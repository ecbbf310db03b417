"""Score-distillation inner loop -- host-side mirror of the loop body of sparsefusion/distillation.py:174-352 (reference).

The reference's ``distillation_loop`` interleaves the hot loop with dataset / pytorch3d / EFT / matplotlib plumbing.
This module keeps the LOOP BODY -- photometric sub-step A (:185-256) and fusion sub-step B (:259-352) -- as
``Distiller.step(itr)`` over a ``SceneCache`` of device tensors, with the boundary the survey fixes (SURVEY.md §8c):
rays arrive as ``rays_o / rays_d`` tensors (the reference gets them from pytorch3d's GridRaysampler, :201-204,:274-277)
and the per-view EFT features / images arrive cached (:95-125).  Loss formulas, weights, schedules and the order of
RNG draws follow the reference line by line (citations inline).  ``INTEGRATION.md`` shows how the reference's
``distillation_loop`` calls this.

What runs where: both NGP renders (fused sm_90a kernels, analytic backward), the PLMS sampler's UNet evaluations
(wgmma engine, one CUDA graph replay per evaluation), the SD VAE encode / decode (``ldm_autoencoder.py``, same engine), the
image-space losses with their gradients (``image_glue.py``), the LPIPS-VGG term when a ``percep`` module is given (``lpips_vgg.py``;
:312-314), fused Adam.

Two step semantics:

* ``Distiller.step`` with ``views_per_step=None`` on one rank is EXACTLY the reference's iteration: sub-step A, Adam, sub-step B on ONE
  target view, Adam (distillation.py:244-247, :345-352).
* ``views_per_step=V`` (SURVEY.md §8e, BASELINE configs[3]) is the view-batched extension: the photometric sub-step and V target views are
  evaluated against the SAME parameters, gradient = grad(A) + mean_v grad(B_v), ONE Adam step -- mathematically one optimiser step on a
  V-view minibatch, not V sequential reference steps.  The V views are entries 1..V of the step's permutation (the reference takes entry 1);
  rank r distils views ``views[r::R]`` as ONE batch through the VAE and the PLMS sampler (UNet batch = V/R, one shared ``max_thres`` per
  step, as many renders as views), the photometric sub-step is computed by one rank (``itr % R``), and the flat 7.46 MB gradient is summed
  with ONE all-reduce per step.  Every random draw of a view (render jitter, inverse-CDF samples, PLMS noise) comes from a generator
  keyed by (seed, iteration, view), so the step's result does not depend on R (up to fp32 summation order).
* ``MultiSceneDistiller`` / ``distill_scenes`` distil S scenes at once, each on the reference's iteration exactly; only the SDS sub-step's VAE
  encode, PLMS sampling (``PLMSSampler.sample_rows``: every scene at its own noise level) and decode are batched over the scenes.

``fusion_substep`` / ``photometric_substep`` with world_size > 1 remain as the one-view-per-rank form (rank r takes entry 1 + r of the
permutation, all-reduce, Adam with grad_scale 1/R) that ``tests/test_multirank_gpu.py`` pins against the single-rank minibatch.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

from . import _lib as lib
from . import image_glue as glue
from .plms import PLMSSampler, _log_snr as plms_log_snr, _sigmoid as plms_sigmoid


def normalize(x):  # utils/common_utils.py:9-13
    return torch.clip(x * 2 - 1.0, -1.0, 1.0)


def unnormalize(x):  # utils/common_utils.py:15-19
    return torch.clip((x + 1.0) / 2.0, 0.0, 1.0)


def huber(x, y, scaling=0.1):  # utils/common_utils.py:183-190
    diff_sq = (x - y) ** 2
    return ((1 + diff_sq / (scaling ** 2)).clamp(1e-4).sqrt() - 1) * float(scaling)


def shard_target_view(perm: torch.Tensor, rank: int) -> int:
    """which target view a rank distils this step: entry (1 + rank) of the step's permutation, wrapping (the reference,
    single process, takes entry 1: distillation.py:264).  Ranks < n_targets therefore get distinct views."""
    return int(perm[(1 + rank) % perm.numel()])


def step_views(perm: torch.Tensor, views_per_step: int) -> list:
    """the V target views of a minibatch step: entries 1..V of the step's permutation, wrapping (V = 1 is the reference's choice, :264)"""
    n = perm.numel()
    return [int(perm[(1 + j) % n]) for j in range(views_per_step)]


def shard_views(views: list, rank: int, world_size: int) -> list:
    """rank r's share of a step's views: views[r::R] (SURVEY.md §8e: {v : v mod R = r} over the step's list)"""
    return list(views[rank::world_size])


def view_seed(seed: int, itr: int, view: int, stream: int) -> int:
    """seed of the generator that serves ONE (iteration, view, stream) -- stream 0: photometric render, 1: fusion render, 2: PLMS noise, 3: evaluation
    render (``evaluate.evaluate_scene``, with iteration 0), 4: circle-path render (``evaluate.render_views`` for the fly-around gif, iteration 0).
    Keyed draws make a minibatch step independent of how its views are spread over ranks."""
    x = (seed * 0x9E3779B97F4A7C15 + itr * 0xBF58476D1CE4E5B9 + view * 0x94D049BB133111EB + stream * 0xD6E8FEB86659FD93) & 0xFFFFFFFFFFFFFFFF
    x ^= x >> 31
    return x & 0x7FFFFFFFFFFFFFFF


class KeyedNoise:
    """``noise_fn`` of the PLMS sampler for a batch of views: row i of every draw comes from view i's own generator (one randn of ``chunk`` draws
    per view per sampling run, sliced by the sampler's calls), so a view's noise does not depend on which other views share its batch.

    ``rows`` (``PLMSSampler.sample_rows``): the draw serves only those views, row i of it view ``rows[i]``.  A view left out of a draw has
    finished its run and may not draw again, so every view still drawing is at the same position of its own stream."""

    def __init__(self, seeds, device, chunk: int = 128):
        self.gens = []
        for sd in seeds:
            g = torch.Generator(device=device)
            g.manual_seed(int(sd))
            self.gens.append(g)
        self.device, self.chunk, self.buf, self.pos = device, chunk, None, 0
        self.finished = set()

    def __call__(self, like: torch.Tensor, rows=None) -> torch.Tensor:
        n = len(self.gens)
        if rows is None:
            assert like.shape[0] == n, 'KeyedNoise: batch rows must match the views it was keyed for'
        else:
            rows = [int(r) for r in rows]
            assert like.shape[0] == len(rows) and not self.finished & set(rows), 'KeyedNoise: a view that stopped drawing may not draw again'
            self.finished |= set(range(n)) - set(rows)
        if self.buf is None or self.pos >= self.chunk:
            self.buf = torch.stack([torch.randn(self.chunk, *like.shape[1:], generator=g, device=self.device, dtype=like.dtype) for g in self.gens], dim=1)
            self.pos = 0
        out = self.buf[self.pos]
        self.pos += 1
        if rows is not None and rows != list(range(n)):
            out = torch.stack([out[r] for r in rows])        # one launch, no host-to-device index copy
        return out


@dataclass
class SceneCache:
    """what the reference holds per scene before the loop starts (distillation.py:65-125), as device tensors"""
    input_rgb: torch.Tensor        # [Vi,3,256,256]  scene_rgb[input_idx]
    input_mask: torch.Tensor       # [Vi,1,256,256]  scene_mask[input_idx]
    input_rays_o: torch.Tensor     # [Vi,N,3]  sampler_feat(camera_vox) origins, N = 128*128 (:201-204)
    input_rays_d: torch.Tensor     # [Vi,N,3]
    target_features: torch.Tensor  # [Vt,256,32,32]  eft_feature_cache[ci]['features'] (:116,:124)
    target_eft_image: torch.Tensor  # [Vt,3,256,256] eft_feature_cache[ci]['eft_image'] (:118-119)
    target_rays_o: torch.Tensor    # [Vt,N,3]
    target_rays_d: torch.Tensor    # [Vt,N,3]

    def to(self, device, non_blocking=False):
        return SceneCache(*[getattr(self, f).to(device, non_blocking=non_blocking) for f in self.__dataclass_fields__])

    def pin(self):
        return SceneCache(*[getattr(self, f).pin_memory() for f in self.__dataclass_fields__])


class FlatAdam:
    """torch.optim.Adam(ngp.get_params(lr)) + StepLR(step_size, gamma) (distillation.py:165-166) over ONE flat buffer:
    parameters, gradients and both moments are contiguous so that the gradient all-reduce is a single collective and
    the update a single fused kernel per parameter group (encoder lr*10, MLP lr: network_grid.py:223-234)."""

    def __init__(self, net, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, step_size=3000, gamma=0.2):
        groups = [dict(g, params=list(g['params'])) for g in net.get_params(lr)]   # get_params hands out generators
        params = [p for g in groups for p in g['params']]
        dev = params[0].device
        sizes = [p.numel() for p in params]
        self.flat = torch.empty(sum(sizes), device=dev)
        self.grad = torch.zeros_like(self.flat)
        self.m, self.v = torch.zeros_like(self.flat), torch.zeros_like(self.flat)
        self.groups = []
        off = 0
        for g in groups:
            start = off
            for p in g['params']:
                n = p.numel()
                self.flat[off:off + n].copy_(p.data.reshape(-1))
                p.data = self.flat[off:off + n].view_as(p)          # parameters become views of the flat buffer
                p.grad = self.grad[off:off + n].view_as(p)          # autograd accumulates in place into the flat gradient
                off += n
            self.groups.append((start, off, g['lr']))
        self.params = params
        self.betas, self.eps, self.step_size, self.gamma = betas, eps, step_size, gamma
        self.t = 0          # optimizer.step() count
        self.sched = 0      # scheduler.step() count

    def zero_grad(self):
        self.grad.zero_()  # parameters' .grad are views of this buffer; never set them to None

    def sync_grads(self, world_size: int = 1, process_group=None) -> float:
        """N>1: ONE sum all-reduce of the flat gradient buffer (NCCL over NVLink on the GPU box, gloo in the CPU tests);
        returns the grad_scale (1/world_size) the following step() must use so that the update is the mean over ranks"""
        if world_size > 1:
            torch.distributed.all_reduce(self.grad, op=torch.distributed.ReduceOp.SUM, group=process_group)
        return 1.0 / world_size

    def step(self, grad_scale: float = 1.0):
        if not self.flat.is_cuda:
            raise RuntimeError('FlatAdam.step: the fused Adam kernel needs CUDA parameters (there is no CPU path)')
        self.t += 1
        lr_mult = self.gamma ** (self.sched // self.step_size)
        for start, end, lr in self.groups:
            lib.call('sfb_adam_step', self.flat[start:end].data_ptr(), self.grad[start:end].data_ptr(), self.m[start:end].data_ptr(),
                     self.v[start:end].data_ptr(), end - start, lr * lr_mult, self.betas[0], self.betas[1], self.eps, self.t, grad_scale, lib.stream())

    def scheduler_step(self):
        self.sched += 1


class Distiller:
    def __init__(self, ngp, vae, vldm, opt, cache: SceneCache, *, z_scale_factor=0.18215, plms_steps=50, start_fusion_step=1000,
                 lambda_color=1.0, lambda_sil=1.0, lambda_opacity=1e-3, seed=0, rank=0, world_size=1, process_group=None,
                 use_cuda_graph=True, fused_glue=True, percep=None, lambda_percep=0.1, start_percep_step=1000, views_per_step=None, max_batch=32):
        self.ngp, self.vae, self.vldm, self.opt, self.cache = ngp, vae, vldm, opt, cache
        self.z_scale_factor = z_scale_factor
        self.start_fusion_step = start_fusion_step
        self.lambda_color, self.lambda_sil, self.lambda_opacity = lambda_color, lambda_sil, lambda_opacity
        self.rank, self.world_size, self.pg = rank, world_size, process_group
        # None: the reference's two-update iteration on one view (one rank) / one view per rank (N ranks, legacy form); V: view-batched minibatch step
        self.views_per_step = views_per_step
        self.max_batch = max_batch     # views per VAE / PLMS batch on one rank (activations of the VAE decoder: 0.27 GB per tensor per 8 views at 256^2)
        self.seed = seed
        # perceptual term (distillation.py:161, :176-178, :312-314): a PerceptualLoss module (lpips_vgg.py) or None; lambda switches on at start_percep_step
        self.percep, self.lambda_percep, self.start_percep_step = percep, lambda_percep, start_percep_step
        self.fused_glue = fused_glue   # image-space losses + their gradients as fused kernels (image_glue.py) instead of ~50 eager launches + autograd
        self.sampler = PLMSSampler(vldm, plms_steps, use_cuda_graph=use_cuda_graph)          # distillation.py:160
        self.optimizer = FlatAdam(ngp, lr=5e-4)                                              # :165-166
        # the reference draws from torch's global CPU generator (:185,:263,:303); a private generator with the same draw
        # order keeps every rank's view permutation identical
        self.gen = torch.Generator().manual_seed(seed)
        self.render_kw = dict(staged=False, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', force_all_rays=True, **vars(opt))
        self.render_noise = None   # parity tests: callable('A'|'B') -> (perturb_noise [N,64], pdf_noise [N,64]) replacing torch.rand
        self.render_noise_keyed = None   # parity tests (minibatch step): callable('A'|'B', view) -> the same pair for that view
        self.plms_noise = None     # parity tests (minibatch step): callable(views) -> noise_fn for that batch, replacing KeyedNoise
        self.pred_img_hook = None  # parity tests (minibatch step): callable(views, pred_img) -> pred_img, e.g. to inject a fixed denoised target
        self._keyed = False        # MultiSceneDistiller: the reference step draws from the keyed generators too (``_render_draws``)
        self.last = {}

    # ------------------------------------------------------------------------------------------------
    def _render_draws(self, rays_o, itr, view, stream, keyed):
        """(perturb_noise [N, num_steps], pdf_noise [N, upsample_steps]) of one render -- stream 0: photometric, 1: fusion -- or None, which
        lets the renderer draw from torch's global generator as the reference does.  ``keyed`` (the view-batched step, MultiSceneDistiller's
        scenes): ``render_noise_keyed`` or the (seed, itr, view, stream) generator; otherwise ``render_noise``."""
        which = 'AB'[stream]
        if not keyed:
            return None if self.render_noise is None else self.render_noise(which)
        if self.render_noise_keyed is not None:
            return self.render_noise_keyed(which, view)
        n, dev = rays_o.shape[0], rays_o.device
        g = torch.Generator(device=dev)
        g.manual_seed(view_seed(self.seed, itr, view, stream))
        return (torch.rand(n, self.opt.num_steps, generator=g, device=dev),             # renderer_df.py:363
                torch.rand(n, self.opt.upsample_steps, generator=g, device=dev))        # renderer_df.py:31

    def _render(self, rays_o, rays_d, draws):
        """(image [N,3], weights_sum [N], hw) with the autograd graph of the render attached; ``draws`` from ``_render_draws``"""
        kw = self.render_kw if draws is None else dict(self.render_kw, perturb_noise=draws[0], pdf_noise=draws[1])
        out = self.ngp.render(rays_o[None], rays_d[None], **kw)
        n = rays_o.shape[0]
        return out['image'].reshape(n, 3), out['weights_sum'].reshape(n), int(round(n ** 0.5))

    def _render_nchw(self, rays_o, rays_d, draws):
        """the render as the eager path uses it: image [1,3,hw,hw] and silhouette [1,1,hw,hw] (:210-211)"""
        img, ws, hw = self._render(rays_o, rays_d, draws)
        return img.reshape(1, hw, hw, 3).permute(0, 3, 1, 2).contiguous(), ws.reshape(1, hw, hw, 1).permute(0, 3, 1, 2).contiguous()

    def _photometric_grad(self, idx, draws):
        """photometric term of input view idx with the fused kernels: render, loss value and gradient (:216-234), backward; returns the loss"""
        c = self.cache
        img, ws, hw = self._render(c.input_rays_o[idx], c.input_rays_d[idx], draws)
        loss, g_img, g_ws = glue.photometric_loss(img.detach(), ws.detach(), c.input_rgb[idx], c.input_mask[idx], hw, hw, int(self.opt.hw_scale),
                                                  self.lambda_color, self.lambda_sil, self.lambda_opacity)
        torch.autograd.backward((img, ws), (g_img, g_ws))
        return loss

    def photometric_substep(self, itr: int):
        """distillation.py:185-247"""
        c = self.cache
        n_in = c.input_rgb.shape[0]
        idx = int(torch.randperm(n_in, generator=self.gen)[0])                               # :185-186
        self.ngp.train()
        if self.opt.cuda_ray and itr % 16 == 0:                                               # :181-182
            self.ngp.update_extra_state()
        draws = self._render_draws(c.input_rays_o[idx], itr, 0, 0, self._keyed)              # keyed: view 0, whichever input view is drawn
        if self.fused_glue:
            self.optimizer.zero_grad()                                                        # :244
            loss = self._photometric_grad(idx, draws)
        else:
            image, sil = self._render_nchw(c.input_rays_o[idx], c.input_rays_d[idx], draws)
            scale = 1.0 / self.opt.hw_scale
            batch_rgb = F.interpolate(c.input_rgb[idx:idx + 1], scale_factor=scale)           # :216 (nearest)
            batch_mask = F.interpolate(c.input_mask[idx:idx + 1], scale_factor=scale)         # :217
            color_err = huber(image, batch_rgb).abs().mean()                                  # :218
            sil_err = huber(sil, batch_mask).abs().mean()                                     # :222
            loss = self.lambda_color * color_err + self.lambda_sil * sil_err                  # :227
            opacity = torch.sqrt(sil ** 2 + .01).mean()                                       # :233
            loss = loss + self.lambda_opacity * opacity                                       # :234
            self.optimizer.zero_grad()                                                        # :244
            loss.backward()
            loss = loss.detach()
        # replicated sub-step: for N>1 the reduce only removes atomic-order drift so that ranks stay bit-identical
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))
        self.optimizer.scheduler_step()                                                       # :247
        self.last['photo_loss'] = loss
        return loss

    def fusion_substep(self, itr: int, max_thres: Optional[float] = None):
        """distillation.py:259-352; rank r takes the (1 + r)-th entry of the step's permutation (the reference takes entry 1, :264)"""
        c = self.cache
        self.optimizer.zero_grad()                                                            # :261
        n_t = c.target_features.shape[0]
        perm = torch.randperm(n_t, generator=self.gen)                                        # :263
        vi = shard_target_view(perm, self.rank)                                               # :264
        u = torch.rand(1, generator=self.gen)                                                 # :303 (drawn every step to keep the stream aligned)
        feats = c.target_features[vi:vi + 1]
        if self.fused_glue and int(self.opt.hw_scale) == 2:
            return self._fusion_substep_fused(itr, max_thres, vi, u, feats)
        image, sil = self._render_nchw(c.target_rays_o[vi], c.target_rays_d[vi], self._render_draws(c.target_rays_o[vi], itr, vi, 1, self._keyed))
        image = F.interpolate(image, scale_factor=self.opt.hw_scale, mode='bilinear')         # :287
        sil = F.interpolate(sil, scale_factor=self.opt.hw_scale, mode='bilinear')             # :288
        if itr > self.start_fusion_step:                                                      # :294
            if max_thres is None:
                max_thres = u.clamp(min=0.0, max=0.99).item()                                 # :303
            pred_img, alpha_cumprod = self._fusion_target([image[0]], feats, max_thres, None)
            fusion_weight = (1 - alpha_cumprod).to(pred_img.device)                           # :307 (the sampler's fp32 value)
            fusion_loss = (fusion_weight * (image - pred_img).abs().mean()).sum()             # :310 ([1]-shaped in the reference)
            if self.percep is not None and itr >= self.start_percep_step:                     # :176-178, :312-314
                fusion_loss = fusion_loss + self.percep(image, pred_img, normalize=True).mean() * self.lambda_percep
            self.last['unet_calls'] = self.sampler.last_unet_calls
        else:                                                                                 # EFT bootstrap :316-329
            noisy_rgb = c.target_eft_image[vi:vi + 1]
            noisy_mask = (noisy_rgb.mean(dim=1, keepdim=True) > .1).float()                   # :269-271
            fusion_loss = self.lambda_color * huber(image, noisy_rgb).abs().mean() + self.lambda_sil * huber(sil, noisy_mask).abs().mean()
        opacity = torch.sqrt(sil ** 2 + .01).mean()                                           # :336
        loss = fusion_loss + self.lambda_opacity * opacity                                    # :344
        loss.backward()                                                                       # :345
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))   # :352
        self.last['fusion_loss'] = loss.detach()
        return loss.detach()

    def _fusion_substep_fused(self, itr, max_thres, vi, u, feats):
        """the same sub-step on target view vi (conditioning ``feats``) with the fused image-space kernels, then Adam (:352)"""
        if itr > self.start_fusion_step and max_thres is None:
            max_thres = u.clamp(min=0.0, max=0.99).item()                                     # :303
        loss = self._fusion_views(itr, [vi], feats, max_thres, self._keyed, 1.0)[0]
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))   # :352
        self.last['fusion_loss'] = loss
        return loss

    def _fusion_views(self, itr, views, feats, max_thres, keyed, scale):
        """fusion term of target views ``views`` (conditioning ``feats``, read in the SDS phase only) with the image-space work in three kernels
        (bilinear x2 to NCHW for the VAE, loss value + gradient at full resolution, adjoint of the bilinear back to the render's [N,3] / [N]
        outputs): renders, ONE SDS target batch passed through ``pred_img_hook`` (or the EFT bootstrap), each view's gradient scaled by
        ``scale``.  PLMS draws: keyed per view (``plms_noise`` or ``KeyedNoise``) when ``keyed``, else the sampler's own.  Returns the views'
        losses, unscaled; the caller steps the optimiser."""
        renders = self._fusion_renders(itr, views, keyed)
        pred = [None] * len(views)
        if itr > self.start_fusion_step:                                                      # :294
            noise_fn = None
            if keyed:
                noise_fn = self.plms_noise(views) if self.plms_noise is not None else KeyedNoise([view_seed(self.seed, itr, v, 2) for v in views],
                                                                                                 renders[0][0].device)
            pred = self._fusion_target([r[3] for r in renders], feats, max_thres, noise_fn)[0]
            if self.pred_img_hook is not None:
                pred = self.pred_img_hook(views, pred)
            self.last['unet_calls'] = self.sampler.last_unet_calls
        return [self._fusion_grad(itr, *r, v, p, max_thres, scale) for r, v, p in zip(renders, views, pred)]

    def _fusion_renders(self, itr, views, keyed):
        """renders of target views (:274-277), then their x2 bilinear upsampling (:287-288): [(image [N,3], weights_sum [N], hw, planes
        [4,2hw,2hw] (r, g, b, opacity))]"""
        c = self.cache
        renders = [self._render(c.target_rays_o[v], c.target_rays_d[v], self._render_draws(c.target_rays_o[v], itr, v, 1, keyed)) for v in views]
        return [(img, ws, hw, glue.upsample2x_render(img.detach(), ws.detach(), hw, hw)) for img, ws, hw in renders]

    @torch.no_grad()
    def _fusion_target(self, images, feats, max_thres, noise_fn, sampler=None):
        """the denoised targets of a batch of renders ([C>=3,H,W] each, colour first): VAE encode (:299), PLMS sampling (:304), decode (:309).
        Returns (pred_img [B,3,H,W], alpha_cumprod [B] of the run's first noise level, fp32).  ``max_thres`` is one float shared by the batch
        (``PLMSSampler.sample``) or one per row (``PLMSSampler.sample_rows``); ``noise_fn`` serves the run's draws, None: the sampler's own."""
        sampler = self.sampler if sampler is None else sampler
        batch = images[0][None, :3] if len(images) == 1 else torch.stack([im[:3] for im in images])
        latents = self.vae.encode(normalize(batch)).mode() * self.z_scale_factor                # :299
        if isinstance(max_thres, (list, tuple)):
            out = sampler.sample_rows(latents, max_thres, feats, noise_fn=noise_fn)
        else:
            prev = sampler.noise_fn
            if noise_fn is not None:
                sampler.noise_fn = noise_fn
            try:
                out = sampler.sample(latents, cond_images=feats, use_tqdm=False, return_noise=True, max_thres=max_thres)   # :304
            finally:
                sampler.noise_fn = prev
        return unnormalize(self.vae.decode(1.0 / self.z_scale_factor * out[0])).clip(0.0, 1.0), out[3]     # :309

    def _fusion_grad(self, itr, img, ws, hw, up, vi, pred_img, max_thres, scale=1.0):
        """loss value and gradient of target view vi (:307-344; SDS against ``pred_img`` [3,2hw,2hw], or the EFT bootstrap when it is None),
        backward (:345) of the gradient times ``scale``; returns the loss.  The caller steps the optimiser (:352)."""
        if pred_img is not None:
            weight = 1.0 - plms_sigmoid(plms_log_snr(float(max_thres)))                      # 1 - alpha_cumprod of the run's first noise level (:307)
            g_extra, percep_term = None, None
            if self.percep is not None and itr >= self.start_percep_step:                     # :176-178, :312-314: value and gradient together
                pv, pg = self.percep.value_and_grad(up[:3], pred_img, normalize=True)
                percep_term, g_extra = pv * self.lambda_percep, pg * self.lambda_percep
            loss, g_img, g_ws = glue.fusion_loss(up, pred_img, hw, hw, 'sds', weight, self.lambda_color, self.lambda_sil, self.lambda_opacity,
                                                 g_extra=g_extra)
            if percep_term is not None:
                loss = loss + percep_term
        else:                                                                                 # EFT bootstrap :316-329
            loss, g_img, g_ws = glue.fusion_loss(up, self.cache.target_eft_image[vi], hw, hw, 'eft', 1.0, self.lambda_color, self.lambda_sil,
                                                 self.lambda_opacity)
        if scale != 1.0:
            g_img, g_ws = g_img * scale, g_ws * scale
        torch.autograd.backward((img, ws), (g_img, g_ws))                                     # :345
        return loss

    def step(self, itr: int, max_thres: Optional[float] = None):
        """one iteration of the reference's main loop (distillation.py:174-352); returns the two losses as device scalars"""
        with torch.cuda.device(self.cache.input_rgb.device):
            if self.views_per_step is not None:
                return self.minibatch_step(itr, max_thres)
            a = self.photometric_substep(itr)
            b = self.fusion_substep(itr, max_thres)
        return a, b

    # ------------------------------------------------------------------------------------------------ view-batched step (SURVEY.md §8e)
    def minibatch_step(self, itr: int, max_thres: Optional[float] = None):
        """one optimiser step on (photometric view + V target views); returns (photometric loss, mean fusion loss) as device scalars.  With
        world_size R each rank handles views[r::R]; the losses returned are the GLOBAL ones only on the rank(s) that computed every term --
        use them for logging, not for control flow."""
        if not self.fused_glue or int(self.opt.hw_scale) != 2:
            raise NotImplementedError('the view-batched step uses the fused image-space kernels (fused_glue=True, hw_scale=2)')
        c = self.cache
        V, R, r = int(self.views_per_step), self.world_size, self.rank
        n_in, n_t = c.input_rgb.shape[0], c.target_features.shape[0]
        idx = int(torch.randperm(n_in, generator=self.gen)[0])                                 # :185-186
        perm = torch.randperm(n_t, generator=self.gen)                                         # :263
        u = torch.rand(1, generator=self.gen)                                                  # :303: ONE noise level per step, shared by its views
        views = step_views(perm, V)
        mine = shard_views(views, r, R)
        self.ngp.train()
        self.optimizer.zero_grad()
        loss_a = loss_b = torch.zeros((), device=c.input_rgb.device)
        if self.opt.cuda_ray and itr % 16 == 0:
            self.ngp.update_extra_state()
        # ---- photometric term: one rank (round-robin over iterations), gradient joins the step's single all-reduce
        if itr % R == r:
            loss_a = self._photometric_grad(idx, self._render_draws(c.input_rays_o[idx], itr, idx, 0, True))
        # ---- fusion term over this rank's views, in batches of at most max_batch, gradient = mean over the step's V views
        sds = itr > self.start_fusion_step
        if sds and max_thres is None:
            max_thres = u.clamp(min=0.0, max=0.99).item()
        if sds and not mine:                               # a rank with no views this step (V < R); otherwise _fusion_views sets it
            self.last['unet_calls'] = 0
        inv_v = 1.0 / V
        for lo in range(0, len(mine), self.max_batch):
            chunk = mine[lo:lo + self.max_batch]
            feats = c.target_features[chunk] if sds else None         # cache fields take int, one-row slice or list indices (bench.py's staged cache)
            for lv in self._fusion_views(itr, chunk, feats, max_thres, True, inv_v):
                loss_b = loss_b + lv * inv_v
        self.optimizer.sync_grads(R, self.pg)              # the step's ONE collective: sum of every rank's (photometric + fusion) gradient
        self.optimizer.step(grad_scale=1.0)
        self.optimizer.scheduler_step()                                                        # :247
        self.last['photo_loss'], self.last['fusion_loss'] = loss_a, loss_b
        self.last['views'] = mine
        return loss_a, loss_b


# ----------------------------------------------------------------------------------------------------------------------
# scene-batched distillation: S scenes, each on the reference's iteration, sharing the VAE and UNet batches
# ----------------------------------------------------------------------------------------------------------------------
class MultiSceneDistiller:
    """Distils S scenes at once on one GPU.  Every scene runs the reference's iteration exactly -- photometric sub-step and Adam, then ONE
    target view and Adam (``Distiller.step`` with ``views_per_step=None``) -- with its own network, optimiser and random streams, held by one
    ``Distiller`` per scene.  What is shared is the SDS work: the S upsampled renders go through ONE VAE encode, ONE ``PLMSSampler.sample_rows``
    (each scene at its own noise level, so with its own number of UNet evaluations; the UNet runs at the batch of scenes still sampling) and
    ONE decode, in chunks of at most ``max_batch`` scenes.  The SDS phase's UNet and VAE run at batch S instead of S times at batch 1.

    Draws of scene k: the view permutation and ``u`` from ``torch.Generator().manual_seed(seeds[k])`` in the reference's order (as in
    ``Distiller(seed=seeds[k])``); the render jitter / inverse-CDF samples of the photometric render from ``view_seed(seeds[k], itr, 0, 0)``, those
    of the fusion render of view v from ``view_seed(seeds[k], itr, v, 1)`` and the PLMS noise from ``view_seed(seeds[k], itr, v, 2)``.  A scene's
    trajectory therefore does not depend on which scenes share its batch.  Parity tests replace them through ``render_noise(scene, 'A'|'B')`` and
    ``plms_noise(scene) -> noise_fn``, the per-scene counterparts of ``Distiller.render_noise`` and ``PLMSSampler.noise_fn``.

    Not supported: ``views_per_step`` (NotImplementedError), ``fused_glue=False`` and ``opt.hw_scale != 2`` (NotImplementedError), scenes of
    different image, latent or ray sizes (ValueError), CPU tensors (RuntimeError)."""

    def __init__(self, ngps, vae, vldm, opt, caches, *, seeds, percep=None, max_batch=8, **kw):
        if kw.get('views_per_step') is not None:
            raise NotImplementedError('MultiSceneDistiller runs the reference iteration (one target view per scene); views_per_step is not supported')
        if not kw.get('fused_glue', True) or int(opt.hw_scale) != 2:
            raise NotImplementedError('MultiSceneDistiller uses the fused image-space kernels (fused_glue=True, hw_scale=2)')
        if kw.get('world_size', 1) != 1:
            raise NotImplementedError('MultiSceneDistiller runs on one rank: give each rank its own share of the scenes')
        if not (len(ngps) == len(caches) == len(seeds)) or len(caches) == 0:
            raise ValueError(f'MultiSceneDistiller: {len(ngps)} networks, {len(caches)} caches, {len(seeds)} seeds')
        fields = list(SceneCache.__dataclass_fields__)
        for c in caches:
            for f in fields:
                t = getattr(c, f)
                if not t.is_cuda:
                    raise RuntimeError(f'MultiSceneDistiller: SceneCache.{f} must be a CUDA tensor (there is no CPU path)')
                if tuple(t.shape[1:]) != tuple(getattr(caches[0], f).shape[1:]):
                    raise ValueError(f'MultiSceneDistiller: scenes differ in SceneCache.{f} size ({tuple(t.shape[1:])} vs '
                                     f'{tuple(getattr(caches[0], f).shape[1:])}); batched scenes need equal image, latent and ray sizes')
        self.scenes = [Distiller(ngp, vae, vldm, opt, cache, seed=int(sd), percep=percep, **kw) for ngp, cache, sd in zip(ngps, caches, seeds)]
        for d in self.scenes:
            d._keyed = True
        self.seeds = [int(s) for s in seeds]
        self.max_batch = int(max_batch)
        lead = self.scenes[0]
        self.start_fusion_step = lead.start_fusion_step
        # one sampler for all scenes: its UnetGraph holds one graph per batch size (at most max_batch of them)
        self.sampler = PLMSSampler(vldm, lead.sampler.plms_steps, use_cuda_graph=lead.sampler.use_cuda_graph)
        self.render_noise = None
        self.plms_noise = None     # parity tests: callable(scene) -> noise_fn(like) serving that scene's PLMS draws
        self.last = {}

    def __len__(self):
        return len(self.scenes)

    @property
    def render_noise(self):
        """parity tests: callable(scene, 'A'|'B') -> (perturb_noise, pdf_noise) of that scene's render, in place of its keyed draws"""
        return self._render_noise

    @render_noise.setter
    def render_noise(self, fn):
        self._render_noise = fn
        for k, d in enumerate(self.scenes):
            d.render_noise_keyed = None if fn is None else (lambda which, view, k=k: fn(k, which))

    def _plms_noise_fn(self, ks, views, itr, dev):
        """noise_fn of one sample_rows run over scenes ks: row i is scene ks[i]'s own stream"""
        if self.plms_noise is None:
            return KeyedNoise([view_seed(self.seeds[k], itr, v, 2) for k, v in zip(ks, views)], dev)
        fns = [self.plms_noise(k) for k in ks]

        def route(like, rows=None):
            rows = range(len(ks)) if rows is None else rows
            return torch.cat([fns[r](like[i:i + 1]) for i, r in enumerate(rows)])
        return route

    def photometric_substep(self, itr: int):
        """every scene's photometric sub-step (:185-247) through ``Distiller.photometric_substep``; returns the [S] losses"""
        return torch.stack([d.photometric_substep(itr) for d in self.scenes])

    def fusion_substep(self, itr: int, max_thres: Optional[float] = None):
        """every scene's fusion sub-step (:259-352) with the VAE encode, PLMS sampling and decode batched over chunks of scenes; returns the [S]
        losses.  ``max_thres`` forces one noise level for every scene (tests); by default scene k uses its own ``u`` (:303)."""
        S = len(self.scenes)
        sds = itr > self.start_fusion_step
        losses, calls, replays = [None] * S, [0] * S, 0
        for lo in range(0, S, self.max_batch):
            ks = list(range(lo, min(S, lo + self.max_batch)))
            views, mts, renders = [], [], []
            for k in ks:
                d, c = self.scenes[k], self.scenes[k].cache
                d.optimizer.zero_grad()                                                        # :261
                perm = torch.randperm(c.target_features.shape[0], generator=d.gen)            # :263
                vi = shard_target_view(perm, 0)                                                # :264
                u = torch.rand(1, generator=d.gen)                                             # :303
                views.append(vi)
                mts.append(float(max_thres) if max_thres is not None else u.clamp(min=0.0, max=0.99).item())
                renders += d._fusion_renders(itr, [vi], True)
            pred = [None] * len(ks)
            if sds:
                feats = torch.cat([self.scenes[k].cache.target_features[v:v + 1] for k, v in zip(ks, views)])
                pred = self.scenes[ks[0]]._fusion_target([r[3] for r in renders], feats, mts, self._plms_noise_fn(ks, views, itr, renders[0][0].device),
                                                         sampler=self.sampler)[0]
                replays += self.sampler.last_graph_replays
                for j, k in enumerate(ks):
                    calls[k] = self.sampler.last_row_calls[j]
                    self.scenes[k].last['unet_calls'] = calls[k]
            for j, k in enumerate(ks):
                d = self.scenes[k]
                losses[k] = d.last['fusion_loss'] = d._fusion_grad(itr, *renders[j], views[j], pred[j], mts[j])
                d.optimizer.step()                                                             # :352 (one rank: grad_scale 1)
            del renders
        if sds:
            self.last['unet_calls'] = calls
            self.last['graph_replays'] = replays
        return torch.stack(losses)

    def step(self, itr: int, max_thres: Optional[float] = None):
        """one iteration of the reference's loop (distillation.py:174-352) for every scene; returns ([S] photometric, [S] fusion) losses"""
        with torch.cuda.device(self.scenes[0].cache.input_rgb.device):
            a = self.photometric_substep(itr)
            b = self.fusion_substep(itr, max_thres)
        self.last['photo_loss'], self.last['fusion_loss'] = a, b
        return a, b


# ----------------------------------------------------------------------------------------------------------------------
# distillation_loop: the reference's entry point (sparsefusion/distillation.py:26-497), same signature
# ----------------------------------------------------------------------------------------------------------------------
from .network_grid import NeRFNetwork, get_default_torch_ngp_opt  # noqa: E402,F401  (re-exported: demo.py:9 imports both names from this module)


class ReferenceSceneBuilder:
    """distillation.py:60-127 -- what the reference prepares per scene before its loop: relative / voxel-frame cameras, 50 circle-path
    augmentation cameras, the 128x128 ray sampler, and the EFT feature cache of every (scene + augmentation) view.  These steps are outside the
    hot path (SURVEY.md §2, §8f row 4): they are executed by the REFERENCE's own utilities -- ``utils.camera_utils``, ``utils.render_utils`` (pytorch3d)
    and the EFT model handed in through ``model_tuple`` -- imported at call time from the reference tree the caller runs in.  The result is the
    ``SceneCache`` the hot loop consumes: rays as tensors, cached features / low-res EFT images per target view."""

    def __init__(self, gpu):
        self.gpu = gpu

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True) -> 'SceneCache':
        try:
            from utils.camera_utils import RelativeCameraLoader, get_interpolated_path
            from utils.render_utils import init_light_field_renderer, init_ray_sampler
        except ImportError as e:
            raise RuntimeError('distillation_loop needs the reference tree (utils/camera_utils.py, utils/render_utils.py) and pytorch3d on sys.path to turn '
                               'pytorch3d cameras into rays and to run the EFT; pass scene_builder=... to supply a SceneCache another way') from e
        from einops import rearrange
        gpu = self.gpu
        relative_cam = RelativeCameraLoader(relative=True, center_at_origin=True)                                    # :65-66
        relative_cam_no_origin = RelativeCameraLoader(relative=True, center_at_origin=False)
        scene_cameras_vox = relative_cam_no_origin.get_relative_camera(scene_cameras, query_idx=[0], center_at_origin=False)   # :70
        scene_cameras_aug = get_interpolated_path(scene_cameras, n=50, method='circle', theta_offset_max=0.17)      # :73
        scene_cameras_aug = relative_cam.concat_cameras([scene_cameras, scene_cameras_aug])                          # :74
        scene_cameras_aug_rel = relative_cam.get_relative_camera(scene_cameras_aug, query_idx=[0], center_at_origin=True)      # :75
        scene_cameras_aug_vox = relative_cam_no_origin.get_relative_camera(scene_cameras_aug, query_idx=[0], center_at_origin=False)
        blank_rgb = torch.zeros_like(scene_rgb[:1]).repeat(len(scene_cameras_aug), 1, 1, 1)                          # :77-79
        scene_rgb_aug = torch.cat((scene_rgb, blank_rgb))
        cam_dist_mean = torch.mean(torch.linalg.norm(scene_cameras.get_camera_center(), axis=1))                     # :82-84
        min_depth, volume_extent_world = cam_dist_mean - 5.0, cam_dist_mean + 5.0
        _, _, sampler_feat = init_ray_sampler(gpu, 256, 256, min=min_depth, max=volume_extent_world, scale_factor=2)            # :85
        _, _, renderer_feat = init_light_field_renderer(gpu, 256, 256, min=min_depth, max=volume_extent_world, scale_factor=8.0)   # :86

        def rays_of(cam):
            rb = sampler_feat(cam)                                                                                  # :201-204, :274-277
            return rearrange(rb.origins, 'b h w c -> b (h w) c')[0].contiguous(), rearrange(rb.directions, 'b h w c -> b (h w) c')[0].contiguous()
        in_o, in_d = zip(*[rays_of(relative_cam.get_camera_slice(scene_cameras_vox, [i])) for i in input_idx])
        feats, eft_imgs, t_o, t_d = [], [], [], []
        n_cache = len(scene_cameras_aug_rel) if use_diffusion else 0
        for ci in range(n_cache):                                                                                   # :95-125
            q_cam, _, _, input_cameras, input_rgb, _ = relative_cam(scene_cameras_aug_rel, scene_rgb_aug, query_idx=[ci], context_idx=input_idx)
            eft.encode(input_cameras, input_rgb)
            with torch.no_grad():
                epi, _, _ = renderer_feat(cameras=q_cam, volumetric_function=eft.batched_forward, n_batches=16, input_cameras=input_cameras, input_rgb=input_rgb)
                lr_render, latents = epi.split([3, 256], dim=-1)
            feats.append(rearrange(latents, 'b h w f -> b f h w'))
            eft_imgs.append(F.interpolate(rearrange(lr_render, 'b h w f -> b f h w'), scale_factor=8.0, mode='bilinear'))
            o, d = rays_of(relative_cam.get_camera_slice(scene_cameras_aug_vox, [ci]))
            t_o.append(o)
            t_d.append(d)
        dev = scene_rgb.device
        n_rays = in_o[0].shape[0]
        empty = lambda *s: torch.zeros(0, *s, device=dev)
        return SceneCache(input_rgb=scene_rgb[input_idx].float(), input_mask=scene_mask[input_idx].float(), input_rays_o=torch.stack(in_o), input_rays_d=torch.stack(in_d),
                          target_features=torch.cat(feats) if feats else empty(256, 32, 32), target_eft_image=torch.cat(eft_imgs) if eft_imgs else empty(3, 256, 256),
                          target_rays_o=torch.stack(t_o) if t_o else empty(n_rays, 3), target_rays_d=torch.stack(t_d) if t_d else empty(n_rays, 3))

    def _grid_rays(self, scene_cameras, circle_n=None):
        """rays [V, 256*256, 3] (origins, directions) of the 256x256 ``sampler_grid`` (:85) for every scene camera in the voxel frame (:70,
        :395-402), or for the ``circle_n`` cameras of the circle path through them (:463-469)"""
        try:
            from utils.camera_utils import RelativeCameraLoader, get_interpolated_path
            from utils.render_utils import init_ray_sampler
        except ImportError as e:
            raise RuntimeError('distillation_loop(evaluate=True / visualize=True) needs the reference tree (utils/camera_utils.py, utils/render_utils.py) '
                               'and pytorch3d on sys.path to turn pytorch3d cameras into rays; pass a scene_builder with its own eval_views / '
                               'circle_views') from e
        from einops import rearrange
        relative_cam = RelativeCameraLoader(relative=True, center_at_origin=True)
        relative_cam_no_origin = RelativeCameraLoader(relative=True, center_at_origin=False)
        scene_cameras_vox = relative_cam_no_origin.get_relative_camera(scene_cameras, query_idx=[0], center_at_origin=False)   # :70
        cam_dist_mean = torch.mean(torch.linalg.norm(scene_cameras.get_camera_center(), axis=1))                     # :82-84
        sampler_grid = init_ray_sampler(self.gpu, 256, 256, min=cam_dist_mean - 5.0, max=cam_dist_mean + 5.0, scale_factor=2)[0]   # :85
        cams = scene_cameras_vox if circle_n is None else get_interpolated_path(scene_cameras_vox, n=circle_n, method='circle')   # :463
        o, d = [], []
        for ci in range(len(cams)):
            rb = sampler_grid(relative_cam.get_camera_slice(cams, [ci]))
            o.append(rearrange(rb.origins, 'b h w c -> b (h w) c')[0].contiguous())
            d.append(rearrange(rb.directions, 'b h w c -> b (h w) c')[0].contiguous())
        return torch.stack(o), torch.stack(d)

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        """the views the reference scores the distilled scene on (:393-406): every scene camera in the voxel frame (:70) through the 256x256
        ``sampler_grid`` (:85), with ``scene_rgb`` / ``scene_mask`` as ground truth -> ``evaluate.EvalViews``"""
        from .evaluate import EvalViews
        o, d = self._grid_rays(scene_cameras)
        return EvalViews(rays_o=o, rays_d=d, rgb=scene_rgb.float(), mask=scene_mask.float())

    def circle_views(self, scene_cameras, n=50):
        """the views of the reference's fly-around gif (:461-469): ``get_interpolated_path(scene_cameras_vox, n=50, method='circle')`` through
        the 256x256 ``sampler_grid`` -> (rays_o, rays_d), each [n, 256*256, 3]"""
        return self._grid_rays(scene_cameras, circle_n=n)


def distillation_loop(gpu, args, opt, model_tuple, save_dir, seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx,
                      use_diffusion=True, max_itr=3000, loss_fn_vgg=None, *, scene_builder=None, views_per_step=None, on_iteration=None, seed=None,
                      process_group=None, evaluate=False, visualize=False):
    """sparsefusion/distillation.py:26-497 with the reference's signature (demo.py:87-103 calls it unchanged): builds the per-scene cache
    (``ReferenceSceneBuilder``, or ``scene_builder.build(...)``), optimises a fresh ``NeRFNetwork(opt)`` for ``max_itr`` iterations with
    ``Distiller.step`` and saves ``{'model_state_dict': ngp.state_dict()}`` to ``{save_dir}/{seq_name}.pt`` (:495-496).

    ``evaluate=True`` adds the reference's scene scores (:391-443): before the first iteration the builder's ``eval_views(scene_cameras, scene_rgb,
    scene_mask)`` gives the views (a ``scene_builder`` without it fails then, not after the loop); after the loop ``evaluate.evaluate_scene`` renders
    every view in eval mode (jitter keyed by the scene's seed) and scores it with PSNR, SSIM and LPIPS-VGG on the GPU, and
    ``{save_dir}/metrics/{seq_name}.txt`` is written in the reference's format.  LPIPS uses ``loss_fn_vgg``'s weights (an ``lpips.LPIPS``, as
    demo.py:33 passes it, or a ``PerceptualLoss``); without it the LPIPS entry is nan rather than a distance from random VGG weights.

    ``visualize=True`` adds the reference's pictures (:129-141, :444-493; ``_write_scene_pictures``): before the first iteration the builder's
    ``eval_views`` and ``circle_views(scene_cameras)`` give the scene views and the 50 circle-path views (a builder without them fails then),
    and with ``use_diffusion`` the grid of cached EFT images is written to ``{args.exp_dir}/log/{seq_name}_eft_grid.jpg``.  After the loop
    ``{save_dir}/render_gifs/{seq_name}.gif`` (gt | EFT image | render | gt mask | silhouette per scene view, without the EFT panel when not
    ``use_diffusion``), ``{save_dir}/render_imgs/{seq_name}/{view:03d}.jpg`` (gt | render) and ``{save_dir}/render_gifs/{seq_name}_circle.gif``
    (render | silhouette per circle view) are written; the sequence frames are the renders ``evaluate`` scores.  GIF palettes are quantised on
    the GPU (``video.py``); Pillow writes the files.

    Not reproduced: the matplotlib loss plots and the periodic ``_vis.jpg`` renders (:355-388) -- logging, outside the hot path;
    ``on_iteration(itr, distiller)`` is the hook for them (``distiller.ngp.render_batched`` is the same call the reference makes).
    ``scene_valid_region`` is accepted and unused, as in the reference's loop body (:192-195 overwrites the region with ones), and so is
    ``loss_fn_vgg`` unless ``evaluate``.  Extensions, keyword-only: ``views_per_step`` (view-batched step, see the module docstring; with
    torch.distributed initialised and ``process_group`` given the views are sharded over its ranks), ``seed``, ``evaluate``, ``visualize``.
    Returns the optimised network."""
    eft, vae, vldm = model_tuple
    rank, world = 0, 1
    if process_group is not None:
        rank, world = torch.distributed.get_rank(process_group), torch.distributed.get_world_size(process_group)

    def make(ngps, caches, percep, seed):
        return Distiller(ngps[0], vae, vldm, opt, caches[0], plms_steps=50, start_fusion_step=1000, lambda_color=1.0, lambda_sil=1.0,   # :148-160
                         lambda_opacity=1e-3, seed=seed, rank=rank, world_size=world, process_group=process_group, percep=percep, lambda_percep=0.1,
                         start_percep_step=1000, views_per_step=views_per_step)
    ngp_network, = _run_distillation(gpu, args, opt, eft, save_dir, [(seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx)],
                                     make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate, loss_fn_vgg, visualize)
    print('input idx', input_idx)
    return ngp_network


def distill_scenes(gpu, args, opt, model_tuple, save_dir, scenes, *, use_diffusion=True, max_itr=3000, scene_builder=None, seed=None, on_iteration=None,
                   evaluate=False, loss_fn_vgg=None, visualize=False):
    """``distillation_loop`` for several scenes at once on one GPU (``MultiSceneDistiller``): demo.py's per-scene loop (demo.py:87-103) becomes
    one call.  ``scenes`` is a list of ``(seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx)``, the per-scene
    arguments demo.py passes to ``distillation_loop``.  Each scene's cache is built as ``distillation_loop`` builds it (``ReferenceSceneBuilder``,
    or ``scene_builder.build(...)``), one ``PerceptualLoss`` serves all scenes, scene k is seeded with ``seed + k`` (``seed`` drawn from torch's
    seed when None), and every network is saved as ``{'model_state_dict': ngp.state_dict()}`` to ``{save_dir}/{seq_name}.pt`` (:495-496).
    Scenes of one call must share image, latent and ray sizes.  With several GPUs, each rank passes its own share of the scenes.
    ``on_iteration(itr, multi_scene_distiller)`` runs after every iteration.  ``evaluate`` / ``loss_fn_vgg``: each scene is scored and its
    ``{save_dir}/metrics/{seq_name}.txt`` written as ``distillation_loop(evaluate=True)`` does, scene k's render jitter keyed by ``seed + k``.
    ``visualize``: each scene's EFT grid, gifs and jpegs as ``distillation_loop(visualize=True)`` writes them, jitter keyed by ``seed + k``.
    Returns the optimised networks in the order of ``scenes``."""
    eft, vae, vldm = model_tuple

    def make(ngps, caches, percep, base):
        return MultiSceneDistiller(ngps, vae, vldm, opt, caches, seeds=[base + k for k in range(len(ngps))], percep=percep,
                                   plms_steps=50, start_fusion_step=1000, lambda_color=1.0, lambda_sil=1.0, lambda_opacity=1e-3,   # :148-160
                                   lambda_percep=0.1, start_percep_step=1000)
    return _run_distillation(gpu, args, opt, eft, save_dir, scenes, make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate,
                             loss_fn_vgg, visualize)


EFT_GRID_COLUMNS = 8     # cached EFT images per row of the grid the reference writes before its loop (:129-141)


def _write_eft_grid(path, eft_images, n_views):
    """the reference's ``{exp_dir}/log/{seq_name}_eft_grid.jpg`` (:129-141): the first 8 * ceil(n_views / 8) cached EFT images [N,3,h,w],
    8 per row"""
    from .video import to_uint8, write_jpeg
    rows = -(-n_views // EFT_GRID_COLUMNS)
    t = eft_images[:rows * EFT_GRID_COLUMNS].float().permute(0, 2, 3, 1)
    h, w = t.shape[1:3]
    grid = t.reshape(rows, EFT_GRID_COLUMNS, h, w, 3).permute(0, 2, 1, 3, 4).reshape(1, rows * h, EFT_GRID_COLUMNS * w, 3)
    write_jpeg(path, to_uint8(grid)[0])


def _write_scene_pictures(save_dir, seq_name, ngp, opt, views, circle, eft_images, seed, scores=None):
    """the reference's sequence gif, per-view jpegs and circle gif of one distilled scene (:444-493).  The sequence frames are ``scores``'
    renders (``evaluate_scene``'s, the ones the metrics come from) or, without scores, the same renders by ``render_views`` (stream 3);
    the circle frames are ``render_views`` of the circle rays with stream 4.  ``eft_images``: the scene views' cached EFT images [V,3,h,w]
    (``use_diffusion``) or None."""
    from .evaluate import CIRCLE_STREAM, EVAL_STREAM, render_views
    from .video import to_uint8, write_gif, write_jpegs
    V = views.rgb.shape[0]
    H, W = views.rgb.shape[2:]
    if scores is None:
        image, sil = render_views(ngp, views.rays_o, views.rays_d, (H, W), opt, seed=seed, stream=EVAL_STREAM)
    else:
        image, sil = scores.image, scores.silhouette
    gt, gt_mask = views.rgb.float().permute(0, 2, 3, 1), views.mask.float().permute(0, 2, 3, 1)
    eft = [] if eft_images is None else [eft_images[:V].float().permute(0, 2, 3, 1)]
    gif_path = f'{save_dir}/render_gifs/{seq_name}.gif'
    write_gif(gif_path, to_uint8(gt, *eft, image, gt_mask, sil[..., None]))                                      # :449-453
    write_jpegs([f'{save_dir}/render_imgs/{seq_name}/{si:03d}.jpg' for si in range(V)], to_uint8(gt, image))         # :455-456
    print('saved video', gif_path)
    rays_o, rays_d = circle
    hw = int(round(rays_o.shape[1] ** 0.5))
    if hw * hw != rays_o.shape[1]:
        raise ValueError(f'circle views must be square images (got {rays_o.shape[1]} rays per view)')
    c_image, c_sil = render_views(ngp, rays_o, rays_d, (hw, hw), opt, seed=seed, stream=CIRCLE_STREAM)           # :461-485
    gif_path = f'{save_dir}/render_gifs/{seq_name}_circle.gif'
    write_gif(gif_path, to_uint8(c_image, c_sil[..., None]))                                                         # :487-490
    print('saved video', gif_path)


def _run_distillation(gpu, args, opt, eft, save_dir, scenes, make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate=False,
                      loss_fn_vgg=None, visualize=False):
    """what ``distillation_loop`` and ``distill_scenes`` share: the reference's output directories, one cache per scene of ``scenes`` (as
    ``distill_scenes`` takes them), a fresh ``NeRFNetwork(opt)`` per scene, the distiller ``make(ngps, caches, percep, seed)`` builds, the
    ``max_itr`` iterations and one checkpoint per scene; with ``evaluate``, the scene scores and metrics files, with ``visualize`` the EFT
    grids before the loop and the gifs and jpegs after it (scene k seeded ``seed + k``).  Returns the networks."""
    import os
    from .lpips_vgg import PerceptualLoss
    builder = scene_builder if scene_builder is not None else ReferenceSceneBuilder(gpu)
    if visualize:
        from .video import require_pillow
        require_pillow()
    for flag, name, sig in ((evaluate or visualize, 'eval_views', '(scene_cameras, scene_rgb, scene_mask)'), (visualize, 'circle_views', '(scene_cameras)')):
        if flag and not callable(getattr(builder, name, None)):
            raise TypeError(f'{"evaluate=True" if name == "eval_views" and evaluate else "visualize=True"} needs the scene builder to provide '
                            f'{name}{sig}; {type(builder).__name__} has none')
    exp_dir = getattr(args, 'exp_dir', save_dir)
    for sc in scenes:
        os.makedirs(f'{exp_dir}/render_imgs/{sc[0]}/', exist_ok=True)                                                # :57-58
    os.makedirs(f'{exp_dir}/render_gifs/', exist_ok=True)
    os.makedirs(save_dir, exist_ok=True)
    device = torch.device('cuda', gpu) if isinstance(gpu, int) else torch.device(gpu)
    eval_views = [builder.eval_views(cams, rgb, mask).to(device) for _, cams, rgb, mask, _, _ in scenes] if evaluate or visualize else None
    circles = [tuple(t.to(device) for t in builder.circle_views(cams)) for _, cams, _, _, _, _ in scenes] if visualize else None
    caches = [builder.build(eft, cams, rgb, mask, input_idx, use_diffusion=use_diffusion).to(device)
              for _, cams, rgb, mask, _, input_idx in scenes]
    if visualize and use_diffusion:
        for (seq_name, *_rest), views, cache in zip(scenes, eval_views, caches):
            need = -(-views.rgb.shape[0] // EFT_GRID_COLUMNS) * EFT_GRID_COLUMNS
            if cache.target_eft_image.shape[0] < need:
                raise ValueError(f'visualize=True: scene {seq_name} has {views.rgb.shape[0]} views, so its EFT grid needs {need} cached EFT images; '
                                 f'the cache holds {cache.target_eft_image.shape[0]}')
        with torch.cuda.device(device):
            for (seq_name, *_rest), views, cache in zip(scenes, eval_views, caches):
                _write_eft_grid(f'{exp_dir}/log/{seq_name}_eft_grid.jpg', cache.target_eft_image, views.rgb.shape[0])   # :129-141
    with torch.cuda.device(device):
        perceptual_loss = PerceptualLoss('vgg', device=device) if use_diffusion else None                          # :161
        ngps = [NeRFNetwork(opt).to(device).train() for _ in scenes]                                               # :164
        base_seed = torch.seed() % (2 ** 31) if seed is None else int(seed)
        dist = make(ngps, caches, perceptual_loss, base_seed)
        for itr in range(max_itr):                                                                                  # :174
            if use_diffusion:
                dist.step(itr)
            else:
                dist.photometric_substep(itr)
            if on_iteration is not None:
                on_iteration(itr, dist)
        torch.cuda.synchronize(device)
    for (seq_name, *_rest), ngp in zip(scenes, ngps):
        torch.save({'model_state_dict': ngp.state_dict()}, f'{save_dir}/{seq_name}.pt')                             # :495-496
    if evaluate or visualize:
        from .evaluate import evaluate_scene, write_scene_metrics
        with torch.cuda.device(device):
            eval_percep = None if loss_fn_vgg is None or not evaluate else PerceptualLoss('vgg', device=device).load_state_dict(loss_fn_vgg.state_dict())
            for k, ((seq_name, *_rest), ngp, views) in enumerate(zip(scenes, ngps, eval_views)):
                scores = None
                if evaluate:
                    scores = evaluate_scene(ngp, views, opt, eval_percep, seed=base_seed + k)                       # :391-433
                    print('warning: this metric is used for debugging only and not the final metric')
                    print(f'{getattr(args, "category", "")} scene {seq_name}')
                    write_scene_metrics(f'{save_dir}/metrics/{seq_name}.txt', scores)                              # :434-441
                if visualize:
                    _write_scene_pictures(save_dir, seq_name, ngp, opt, views, circles[k], caches[k].target_eft_image if use_diffusion else None,
                                          base_seed + k, scores)                                                    # :444-493
    return ngps
