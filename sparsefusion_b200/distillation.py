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

Every entry point takes ``sds_method``: 'plms' (default) samples the SDS target with the reference's multi-step PLMS run, 'onestep' with
``DDPM.forward_noloss`` -- one UNet evaluation per target at the same noise level (see ``Distiller``).

``fusion_substep`` / ``photometric_substep`` with world_size > 1 remain as the one-view-per-rank form (rank r takes entry 1 + r of the
permutation, all-reduce, Adam with grad_scale 1/R) that ``tests/test_multirank_gpu.py`` pins against the single-rank minibatch.

Checkpoints: ``Distiller.state_dict`` / ``MultiSceneDistiller.state_dict`` hold everything a run needs to continue -- parameters, Adam
moments and counts, the cuda_ray density grid and counters, the view-permutation generator, the global CPU / CUDA generators of every rank,
the seed -- with a fingerprint of the step's settings and a digest of the scene cache, so that ``load_state_dict`` refuses a state it cannot
continue.  The loops write them with ``checkpoint_every`` and continue from them with ``resume``.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

from . import _lib as lib
from . import image_glue as glue
from .plms import PLMSSampler, _log_snr as plms_log_snr, _sigmoid as plms_sigmoid, check_cond_scale
from .vldm import keep_mask


def _check_cond_scale(vldm, cond_scale, where):
    """ValueError, before any device work, for a guidance scale of the SDS target that is not finite, or not 1 on a VLDM without
    conditional dropout"""
    if not math.isfinite(float(cond_scale)):
        raise ValueError(f'{where}: cond_scale must be finite (got {cond_scale!r})')
    check_cond_scale(vldm, cond_scale, where)


SDS_METHODS = ('plms', 'onestep')


def _check_sds_method(sds_method, where):
    """ValueError, before any device work, for an SDS target method other than 'plms' (the reference's multi-step PLMS run) and 'onestep'
    (``DDPM.forward_noloss``)"""
    if sds_method not in SDS_METHODS:
        raise ValueError(f'{where}: sds_method must be one of {SDS_METHODS} (got {sds_method!r})')


def _check_lambda_entropy(lambda_entropy, where):
    """ValueError, before any device work, for an entropy weight that is negative or not finite"""
    le = float(lambda_entropy)
    if not (math.isfinite(le) and le >= 0.0):
        raise ValueError(f'{where}: lambda_entropy must be a finite value >= 0 (got {lambda_entropy!r})')


# columns of the loss history (``Distiller.history``): the reference's loss_list, opacity_loss_list, entropy_loss_list and fusion_loss_list
HISTORY_COLUMNS = ('volumetric', 'opacity', 'entropy', 'fusion')


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
    render (``evaluate.evaluate_scene``, with iteration 0), 4: circle-path render (``evaluate.render_views`` for the fly-around gif, iteration 0), 5: VLDM
    baseline samples (``baselines.sample_vldm_views``, iteration 0), 6: the periodic snapshot render of the photometric input view (``progress.py``).
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


CHECKPOINT_VERSION = 1     # format of Distiller.state_dict; load_state_dict refuses any other


def cache_digest(cache: SceneCache) -> dict:
    """{field: (shape, digest)} of a scene cache, each digest a 64-bit checksum of the field's bits computed on its device
    (``sfb_digest_u32``).  A resumed run rebuilds its cache and compares this instead of saving the cache."""
    fields = list(SceneCache.__dataclass_fields__)
    for f in fields:
        t = getattr(cache, f)
        if not t.is_cuda:
            raise RuntimeError(f'cache_digest: SceneCache.{f} must be a CUDA tensor (the digest runs on the device)')
        if (t.numel() * t.element_size()) % 4:
            raise ValueError(f'cache_digest: SceneCache.{f} is not a whole number of 32-bit words')
    sums = []
    for f in fields:
        t = getattr(cache, f).contiguous()
        out = torch.empty(1, dtype=torch.int64, device=t.device)
        with torch.cuda.device(t.device):
            lib.call('sfb_digest_u32', t.data_ptr() if t.numel() else None, t.numel() * t.element_size() // 4, out.data_ptr(), lib.stream())
        sums.append(out)
    words = torch.cat([s.cpu() for s in sums]).tolist()
    return {f: (tuple(getattr(cache, f).shape), w & 0xFFFFFFFFFFFFFFFF) for f, w in zip(fields, words)}


def _plain(v):
    """``v`` as plain, comparable Python values (lists for tuples, repr for anything else), for a fingerprint"""
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, dict):
        return {str(k): _plain(x) for k, x in v.items()}
    return repr(v)


def _rng_states(device, world_size=1, process_group=None) -> list:
    """[per rank] the global CPU generator's state and the CUDA generator's state of the rank's device (None on a CPU device); with
    world_size > 1 gathered from every rank of the process group"""
    mine = dict(cpu=torch.get_rng_state(), cuda=torch.cuda.get_rng_state(device) if device.type == 'cuda' else None)
    if world_size == 1:
        return [mine]
    out = [None] * world_size
    torch.distributed.all_gather_object(out, mine, group=process_group)
    return out


def _restore_rng(states, device, rank):
    """restore this rank's entry of ``_rng_states`` (entry rank mod the saved world size)"""
    st = states[rank % len(states)]
    torch.set_rng_state(st['cpu'])
    if st['cuda'] is not None and device.type == 'cuda':
        torch.cuda.set_rng_state(st['cuda'], device)


def _mismatch(what, saved, now):
    return ValueError(f'load_state_dict: {what} differs: the checkpoint has {saved!r}, this run {now!r}; the saved state cannot be continued here')


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

    def state_dict(self) -> dict:
        """Adam moments ``m`` / ``v`` (host copies) and the step and scheduler counts; the parameters are the network's"""
        return dict(m=self.m.detach().to('cpu', copy=True), v=self.v.detach().to('cpu', copy=True), t=self.t, sched=self.sched,
                    groups=[list(g) for g in self.groups])

    def check_state(self, sd):
        """ValueError when ``sd`` is not a state of an optimiser with this one's parameter groups"""
        for k in ('m', 'v'):
            if tuple(sd[k].shape) != tuple(self.m.shape):
                raise _mismatch(f'optimizer.{k} size', tuple(sd[k].shape), tuple(self.m.shape))
        if [list(g) for g in sd['groups']] != [list(g) for g in self.groups]:
            raise _mismatch('optimizer parameter groups', sd['groups'], [list(g) for g in self.groups])

    def load_state_dict(self, sd):
        """copy ``m`` / ``v`` into the existing buffers in place -- the parameters and their .grad are views of ``flat`` / ``grad`` and
        must stay so -- and restore the counts"""
        self.check_state(sd)
        self.m.copy_(sd['m'])
        self.v.copy_(sd['v'])
        self.t, self.sched = int(sd['t']), int(sd['sched'])


class Distiller:
    """One scene's distillation loop body (see the module docstring for the step semantics).

    ``sds_method`` picks the SDS target of each view's VAE latent.  'plms' (the default, the reference's): the multi-step PLMS run from
    ``max_thres`` (``PLMSSampler``, about 38 UNet evaluations on average).  'onestep': ``DDPM.forward_noloss`` at the step's own noise
    level -- times = the ``max_thres`` PLMS would start from, so both methods use the same levels and the same fusion weight
    1 - alpha_cumprod -- ONE UNet evaluation per target (a graph replay of the chunk's B rows, 2B guided), then the same decode, loss,
    LPIPS and Adam.  ``cond_scale`` guides either target.  Draws of the one-step target: torch's global generator in ``step`` (the
    reference's order: noise, then the conditional-dropout keep mask); in ``minibatch_step`` (and in ``MultiSceneDistiller``'s scenes) each
    view's noise, then its keep uniform, from its own ``view_seed(seed, itr, view, 2)`` generator, so a view's target does not depend on its
    batch-mates.  An unknown ``sds_method`` raises ValueError before any device work."""

    def __init__(self, ngp, vae, vldm, opt, cache: SceneCache, *, z_scale_factor=0.18215, plms_steps=50, start_fusion_step=1000,
                 lambda_color=1.0, lambda_sil=1.0, lambda_opacity=1e-3, seed=0, rank=0, world_size=1, process_group=None,
                 use_cuda_graph=True, fused_glue=True, percep=None, lambda_percep=0.1, start_percep_step=1000, views_per_step=None, max_batch=32,
                 cond_scale=1.0, sds_method='plms', lambda_entropy=0.0, max_itr=3000):
        _check_cond_scale(vldm, cond_scale, 'Distiller')
        _check_sds_method(sds_method, 'Distiller')
        _check_lambda_entropy(lambda_entropy, 'Distiller')
        self.ngp, self.vae, self.vldm, self.opt, self.cache = ngp, vae, vldm, opt, cache
        self.z_scale_factor = z_scale_factor
        self.start_fusion_step = start_fusion_step
        self.lambda_color, self.lambda_sil, self.lambda_opacity = lambda_color, lambda_sil, lambda_opacity
        self.lambda_entropy = float(lambda_entropy)    # entropy regulariser of both sub-steps (:236-241, :338-344); the reference's loop sets 0
        self.rank, self.world_size, self.pg = rank, world_size, process_group
        # None: the reference's two-update iteration on one view (one rank) / one view per rank (N ranks, legacy form); V: view-batched minibatch step
        self.views_per_step = views_per_step
        self.max_batch = max_batch     # views per VAE / PLMS batch on one rank (activations of the VAE decoder: 0.27 GB per tensor per 8 views at 256^2)
        # classifier-free guidance scale of the SDS target's PLMS run (1: none); with guidance the UNet evaluates 2 rows per view
        self.cond_scale = float(cond_scale)
        self.sds_method = sds_method   # SDS target: 'plms' (multi-step PLMS run) or 'onestep' (DDPM.forward_noloss, one UNet evaluation)
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
        self.next_itr = 0          # the iteration after the last one run: what state_dict saves as ``itr``
        self.last = {}
        # loss history (see ``history``): rows for max_itr iterations, grown by doubling should a step run past them
        self._history = torch.full((max(int(max_itr), 1), len(HISTORY_COLUMNS)), math.nan, dtype=torch.float32, device=cache.input_rgb.device)

    # ------------------------------------------------------------------------------------------------ loss history
    @property
    def history(self) -> torch.Tensor:
        """[next_itr, 4] device tensor, row itr = the terms the reference logs at iteration itr (distillation.py:249-256, :349), columns
        ``HISTORY_COLUMNS``: 'volumetric' (the photometric sub-step's loss, opacity and entropy included), 'opacity' (lambda_opacity *
        opacity), 'entropy' (lambda_entropy * entropy) of the photometric sub-step, and 'fusion' (the fusion sub-step's SDS L1 plus the
        perceptual term, or its EFT-bootstrap term; without opacity and entropy).  Each step writes its row with device-to-device copies, so
        recording costs no host synchronisation.  nan marks a term not computed: the fusion term of a loop without diffusion, the photometric
        terms of a rank that skipped the photometric sub-step in the view-batched step (the reference has no such case), and rows before the
        iteration a run was resumed at from a checkpoint without history.  The view-batched step logs the mean over its V views (with
        world_size R, over this rank's views' share of that mean)."""
        return self._history[:self.next_itr]

    def _history_rows(self, rows):
        """grow the history buffer (nan rows, by doubling) until it holds ``rows`` rows"""
        if rows > self._history.shape[0]:
            grown = torch.full((max(2 * self._history.shape[0], rows), self._history.shape[1]), math.nan, dtype=self._history.dtype,
                               device=self._history.device)
            grown[:self._history.shape[0]].copy_(self._history)
            self._history = grown

    def _record(self, itr, col, values):
        """row ``itr``, columns col.. of the history <- ``values`` (device tensor), without a host synchronisation"""
        self._history_rows(itr + 1)
        values = values.detach().reshape(-1)
        self._history[itr, col:col + values.numel()].copy_(values)

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
        """photometric term of input view idx with the fused kernels: render, loss value and gradient (:216-241), backward; returns the loss
        and leaves its [4] logged terms (``image_glue.photometric_loss``) in ``last['photo_terms']``"""
        c = self.cache
        img, ws, hw = self._render(c.input_rays_o[idx], c.input_rays_d[idx], draws)
        loss, g_img, g_ws, terms = glue.photometric_loss(img.detach(), ws.detach(), c.input_rgb[idx], c.input_mask[idx], hw, hw,
                                                         int(self.opt.hw_scale), self.lambda_color, self.lambda_sil, self.lambda_opacity,
                                                         lambda_entropy=self.lambda_entropy, return_terms=True)
        torch.autograd.backward((img, ws), (g_img, g_ws))
        self.last['photo_terms'] = terms
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
        self.last['input_view'] = idx
        if self.fused_glue:
            self.optimizer.zero_grad()                                                        # :244
            loss = self._photometric_grad(idx, draws)
            terms = self.last['photo_terms']
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
            entropy = torch.zeros_like(loss)
            if self.lambda_entropy > 0:
                alphas = sil.clamp(1e-5, 1 - 1e-5)                                            # :238-240
                entropy = (- alphas * torch.log2(alphas) - (1 - alphas) * torch.log2(1 - alphas)).mean()
                loss = loss + self.lambda_entropy * entropy                                   # :241
            self.optimizer.zero_grad()                                                        # :244
            loss.backward()
            loss = loss.detach()
            terms = torch.stack((loss, (self.lambda_opacity * opacity).detach(), (self.lambda_entropy * entropy).detach()))   # :254-256
        # replicated sub-step: for N>1 the reduce only removes atomic-order drift so that ranks stay bit-identical
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))
        self.optimizer.scheduler_step()                                                       # :247
        self._record(itr, 0, terms[:3])                                                       # :254-256
        self.last['photo_loss'] = loss
        self.next_itr = itr + 1
        return loss

    def fusion_substep(self, itr: int, max_thres: Optional[float] = None):
        """distillation.py:259-352; rank r takes the (1 + r)-th entry of the step's permutation (the reference takes entry 1, :264)"""
        c = self.cache
        self.next_itr = itr + 1
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
            self._note_target_calls()
        else:                                                                                 # EFT bootstrap :316-329
            noisy_rgb = c.target_eft_image[vi:vi + 1]
            noisy_mask = (noisy_rgb.mean(dim=1, keepdim=True) > .1).float()                   # :269-271
            fusion_loss = self.lambda_color * huber(image, noisy_rgb).abs().mean() + self.lambda_sil * huber(sil, noisy_mask).abs().mean()
        opacity = torch.sqrt(sil ** 2 + .01).mean()                                           # :336
        loss = fusion_loss + self.lambda_opacity * opacity                                    # :344
        if self.lambda_entropy > 0:
            alphas = sil.clamp(1e-5, 1 - 1e-5)                                                # :340-342
            entropy = (- alphas * torch.log2(alphas) - (1 - alphas) * torch.log2(1 - alphas)).mean()
            loss = loss + self.lambda_entropy * entropy                                       # :344
        loss.backward()                                                                       # :345
        self._record(itr, 3, fusion_loss)                                                     # :349
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))   # :352
        self.last['fusion_loss'] = loss.detach()
        return loss.detach()

    def _fusion_substep_fused(self, itr, max_thres, vi, u, feats):
        """the same sub-step on target view vi (conditioning ``feats``) with the fused image-space kernels, then Adam (:352)"""
        if itr > self.start_fusion_step and max_thres is None:
            max_thres = u.clamp(min=0.0, max=0.99).item()                                     # :303
        loss, logged = self._fusion_views(itr, [vi], feats, max_thres, self._keyed, 1.0)[0]
        self._record(itr, 3, logged)                                                          # :349
        self.optimizer.step(grad_scale=self.optimizer.sync_grads(self.world_size, self.pg))   # :352
        self.last['fusion_loss'] = loss
        return loss

    def _fusion_views(self, itr, views, feats, max_thres, keyed, scale, first=True):
        """fusion term of target views ``views`` (conditioning ``feats``, read in the SDS phase only) with the image-space work in three kernels
        (bilinear x2 to NCHW for the VAE, loss value + gradient at full resolution, adjoint of the bilinear back to the render's [N,3] / [N]
        outputs): renders, ONE SDS target batch passed through ``pred_img_hook`` (or the EFT bootstrap), each view's gradient scaled by
        ``scale``.  PLMS draws: keyed per view (``plms_noise`` or ``KeyedNoise``) when ``keyed``, else the sampler's own.  Returns the views'
        (loss, logged fusion term) pairs (``_fusion_grad``), unscaled; the caller steps the optimiser."""
        renders = self._fusion_renders(itr, views, keyed)
        pred = [None] * len(views)
        if itr > self.start_fusion_step:                                                      # :294
            noise_fn = seeds = None
            if keyed and self.sds_method == 'onestep':
                seeds = [view_seed(self.seed, itr, v, 2) for v in views]
            elif keyed:
                noise_fn = self.plms_noise(views) if self.plms_noise is not None else KeyedNoise([view_seed(self.seed, itr, v, 2) for v in views],
                                                                                                 renders[0][0].device)
            pred = self._fusion_target([r[3] for r in renders], feats, max_thres, noise_fn, seeds=seeds)[0]
            if self.pred_img_hook is not None:
                pred = self.pred_img_hook(views, pred)
            self._note_target_calls(first)
        return [self._fusion_grad(itr, *r, v, p, max_thres, scale) for r, v, p in zip(renders, views, pred)]

    def _fusion_renders(self, itr, views, keyed):
        """renders of target views (:274-277), then their x2 bilinear upsampling (:287-288): [(image [N,3], weights_sum [N], hw, planes
        [4,2hw,2hw] (r, g, b, opacity))]"""
        c = self.cache
        renders = [self._render(c.target_rays_o[v], c.target_rays_d[v], self._render_draws(c.target_rays_o[v], itr, v, 1, keyed)) for v in views]
        return [(img, ws, hw, glue.upsample2x_render(img.detach(), ws.detach(), hw, hw)) for img, ws, hw in renders]

    def _note_target_calls(self, first=True):
        """``last['unet_calls']`` of the SDS target batch just made: the PLMS run's evaluations, or 1 for the one-step target, whose graph
        replays of the sub-step (one per batch; ``first``: the sub-step's first batch) ``last['graph_replays']`` counts"""
        if self.sds_method == 'onestep':
            self.last['unet_calls'] = 1
            self.last['graph_replays'] = 1 if first else self.last.get('graph_replays', 0) + 1
        else:
            self.last['unet_calls'] = self.sampler.last_unet_calls

    @torch.no_grad()
    def _onestep_target(self, latents, max_thres, feats, seeds):
        """``DDPM.forward_noloss`` of the B latents at times = ``max_thres`` (one float, or one per row): ONE UNet evaluation of the batch
        (2B rows guided).  ``seeds``: per row, the generator of its noise and then its keep uniform; None: torch's global generator, in the
        reference's order.  Returns what ``PLMSSampler.sample`` returns: (pred_x0, x_noisy, noise, alpha_cumprod)."""
        b, dev = latents.shape[0], latents.device
        mts = [float(m) for m in max_thres] if isinstance(max_thres, (list, tuple)) else [float(max_thres)] * b
        times = torch.tensor(mts, dtype=torch.float32).to(dev)
        noise = keep = None
        if seeds is not None:
            prob = 1 - self.vldm.cond_drop_prob
            draw_u = self.cond_scale == 1 and prob not in (0, 1)
            noise, u = [], []
            for sd in seeds:
                g = torch.Generator(device=dev)
                g.manual_seed(int(sd))
                noise.append(torch.randn(latents.shape[1:], generator=g, device=dev))
                if draw_u:
                    u.append(torch.rand(1, generator=g, device=dev))
            noise = torch.stack(noise)
            if self.cond_scale == 1:
                keep = keep_mask(torch.cat(u) if draw_u else None, prob, b, dev)
        _, x0, x_noisy, noise, acp = self.vldm.forward_noloss(latents, cond_images=feats, return_noise=True, times=times, noise=noise, keep=keep,
                                                              cond_scale=self.cond_scale)
        return self.vldm.unnormalize_img(x0), x_noisy, noise, acp

    @torch.no_grad()
    def _fusion_target(self, images, feats, max_thres, noise_fn, sampler=None, seeds=None):
        """the denoised targets of a batch of renders ([C>=3,H,W] each, colour first): VAE encode (:299), PLMS sampling (:304), decode (:309).
        Returns (pred_img [B,3,H,W], alpha_cumprod [B] of the run's first noise level, fp32).  ``max_thres`` is one float shared by the batch
        (``PLMSSampler.sample``) or one per row (``PLMSSampler.sample_rows``); ``noise_fn`` serves the run's draws, None: the sampler's own.
        The run is guided with ``self.cond_scale``.  With ``sds_method='onestep'`` the sampling is ``_onestep_target`` at the same levels, its
        draws from the per-row generators of ``seeds`` (None: torch's global generator)."""
        sampler = self.sampler if sampler is None else sampler
        batch = images[0][None, :3] if len(images) == 1 else torch.stack([im[:3] for im in images])
        latents = self.vae.encode(normalize(batch)).mode() * self.z_scale_factor                # :299
        if self.sds_method == 'onestep':
            out = self._onestep_target(latents, max_thres, feats, seeds)
        elif isinstance(max_thres, (list, tuple)):
            out = sampler.sample_rows(latents, max_thres, feats, noise_fn=noise_fn, cond_scale=self.cond_scale)
        else:
            prev = sampler.noise_fn
            if noise_fn is not None:
                sampler.noise_fn = noise_fn
            try:
                out = sampler.sample(latents, cond_images=feats, cond_scale=self.cond_scale, use_tqdm=False, return_noise=True,
                                     max_thres=max_thres)                                                             # :304
            finally:
                sampler.noise_fn = prev
        return unnormalize(self.vae.decode(1.0 / self.z_scale_factor * out[0])).clip(0.0, 1.0), out[3]     # :309

    def _fusion_grad(self, itr, img, ws, hw, up, vi, pred_img, max_thres, scale=1.0):
        """loss value and gradient of target view vi (:307-344; SDS against ``pred_img`` [3,2hw,2hw], or the EFT bootstrap when it is None),
        backward (:345) of the gradient times ``scale``; returns the loss and the fusion term the reference logs (:349: the SDS L1 plus the
        perceptual term, or the EFT-bootstrap term; no opacity or entropy).  The caller steps the optimiser (:352)."""
        if pred_img is not None:
            weight = 1.0 - plms_sigmoid(plms_log_snr(float(max_thres)))                      # 1 - alpha_cumprod of the run's first noise level (:307)
            g_extra, percep_term = None, None
            if self.percep is not None and itr >= self.start_percep_step:                     # :176-178, :312-314: value and gradient together
                pv, pg = self.percep.value_and_grad(up[:3], pred_img, normalize=True)
                percep_term, g_extra = pv * self.lambda_percep, pg * self.lambda_percep
            loss, g_img, g_ws, terms = glue.fusion_loss(up, pred_img, hw, hw, 'sds', weight, self.lambda_color, self.lambda_sil,
                                                        self.lambda_opacity, g_extra=g_extra, lambda_entropy=self.lambda_entropy, return_terms=True)
            logged = terms[3]
            if percep_term is not None:
                loss = loss + percep_term
                logged = logged + percep_term
        else:                                                                                 # EFT bootstrap :316-329
            loss, g_img, g_ws, terms = glue.fusion_loss(up, self.cache.target_eft_image[vi], hw, hw, 'eft', 1.0, self.lambda_color,
                                                        self.lambda_sil, self.lambda_opacity, lambda_entropy=self.lambda_entropy, return_terms=True)
            logged = terms[3]
        if scale != 1.0:
            g_img, g_ws = g_img * scale, g_ws * scale
        torch.autograd.backward((img, ws), (g_img, g_ws))                                     # :345
        return loss, logged

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
        loss_a = loss_b = logged_b = torch.zeros((), device=c.input_rgb.device)
        if self.opt.cuda_ray and itr % 16 == 0:
            self.ngp.update_extra_state()
        self.last['input_view'] = idx
        # ---- photometric term: one rank (round-robin over iterations), gradient joins the step's single all-reduce
        if itr % R == r:
            loss_a = self._photometric_grad(idx, self._render_draws(c.input_rays_o[idx], itr, idx, 0, True))
            self._record(itr, 0, self.last['photo_terms'][:3])
        else:
            self._record(itr, 0, torch.full((3,), math.nan, device=c.input_rgb.device))
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
            for lv, gv in self._fusion_views(itr, chunk, feats, max_thres, True, inv_v, first=lo == 0):
                loss_b = loss_b + lv * inv_v
                logged_b = logged_b + gv * inv_v
        self._record(itr, 3, logged_b if mine else torch.full((1,), math.nan, device=c.input_rgb.device))
        self.optimizer.sync_grads(R, self.pg)              # the step's ONE collective: sum of every rank's (photometric + fusion) gradient
        self.optimizer.step(grad_scale=1.0)
        self.optimizer.scheduler_step()                                                        # :247
        self.last['photo_loss'], self.last['fusion_loss'] = loss_a, loss_b
        self.last['views'] = mine
        self.next_itr = itr + 1
        return loss_a, loss_b

    # ------------------------------------------------------------------------------------------------ checkpoint / resume
    def fingerprint(self, use_diffusion=True) -> dict:
        """everything besides the parameters, optimiser state, draws and cache that decides what the next step computes; a checkpoint
        continues only under an equal fingerprint.  ``use_diffusion``: whether the loop runs the fusion sub-step at all"""
        return dict(opt=_plain(vars(self.opt)), views_per_step=self.views_per_step, max_batch=self.max_batch, cond_scale=self.cond_scale,
                    sds_method=self.sds_method, use_diffusion=bool(use_diffusion), lambda_color=self.lambda_color, lambda_sil=self.lambda_sil,
                    lambda_opacity=self.lambda_opacity, lambda_percep=self.lambda_percep, start_fusion_step=self.start_fusion_step,
                    start_percep_step=self.start_percep_step, plms_steps=self.sampler.plms_steps, fused_glue=self.fused_glue,
                    percep=self.percep is not None, z_scale_factor=self.z_scale_factor, keyed=self._keyed,
                    # only when on: checkpoints made before the entropy term existed carry no such key and continue at lambda_entropy 0
                    **({'lambda_entropy': self.lambda_entropy} if self.lambda_entropy != 0 else {}),
                    # likewise for pretrained perceptual weights (``percep_weights``): a run with them and one with the random initialisation
                    # distil different losses
                    **({'percep_pretrained': True} if getattr(self.percep, 'pretrained', False) else {}))

    def _scene_state(self, itr, use_diffusion):
        """this scene's part of a checkpoint: everything but the global generators"""
        extra = {k: getattr(self.ngp, k) for k in ('mean_density', 'iter_density', 'mean_count', 'local_step')} if self.opt.cuda_ray else {}
        return dict(version=CHECKPOINT_VERSION, itr=int(itr), world_size=self.world_size, seed=self.seed,
                    fingerprint=self.fingerprint(use_diffusion), cache=cache_digest(self.cache),
                    ngp={k: v.detach().to('cpu', copy=True) for k, v in self.ngp.state_dict().items()}, ngp_extra=extra,
                    optimizer=self.optimizer.state_dict(), gen=self.gen.get_state(),
                    history=self._history[:int(itr)].to('cpu', copy=True))

    def state_dict(self, itr: Optional[int] = None, use_diffusion=True) -> dict:
        """everything needed to continue this run at iteration ``itr`` (default: the one after the last step run): a format version,
        ``itr``, the world size, the seed, ``fingerprint(use_diffusion)``, the cache digest (``cache_digest``), the network's state dict
        (with cuda_ray its density grid, bitfield and step counter) and plain counters (``ngp_extra``), the optimiser's state, the
        permutation generator's state and ``rng``: every rank's global CPU and CUDA generator states.  Host tensors throughout.  With
        world_size > 1 every rank must call it (the generator states are gathered); parameters and Adam state are the same on every rank."""
        sd = self._scene_state(self.next_itr if itr is None else itr, use_diffusion)
        sd['rng'] = _rng_states(self.cache.input_rgb.device, self.world_size, self.pg)
        return sd

    def check_state(self, sd, use_diffusion=True):
        """ValueError naming the first field that keeps ``sd`` from being continued by this distiller; touches no device state"""
        if sd.get('version') != CHECKPOINT_VERSION:
            raise _mismatch('the checkpoint format version', sd.get('version'), CHECKPOINT_VERSION)
        if sd['world_size'] != self.world_size:
            if self.views_per_step is None:
                raise _mismatch('world_size (the reference step and the one-view-per-rank form continue on the same ranks only)',
                                sd['world_size'], self.world_size)
            if self.opt.cuda_ray:
                raise _mismatch('world_size (with cuda_ray the density grid and the CUDA generator are per rank)', sd['world_size'],
                                self.world_size)
        now = self.fingerprint(use_diffusion)
        for k in sorted(set(now) | set(sd['fingerprint'])):
            a, b = sd['fingerprint'].get(k), now.get(k)
            if k == 'opt' and isinstance(a, dict) and isinstance(b, dict):
                for o in sorted(set(a) | set(b)):
                    if a.get(o) != b.get(o):
                        raise _mismatch(f'opt.{o}', a.get(o), b.get(o))
            elif a != b:
                raise _mismatch(k, a, b)
        if sd['seed'] != self.seed:
            raise _mismatch('seed', sd['seed'], self.seed)
        digest = cache_digest(self.cache)
        for f in SceneCache.__dataclass_fields__:
            if tuple(sd['cache'][f][0]) != digest[f][0]:
                raise _mismatch(f'scene cache field {f} shape', tuple(sd['cache'][f][0]), digest[f][0])
            if sd['cache'][f][1] != digest[f][1]:
                raise _mismatch(f'scene cache field {f} contents (digest)', f'{sd["cache"][f][1]:016x}', f'{digest[f][1]:016x}')
        mine = self.ngp.state_dict()
        if set(sd['ngp']) != set(mine):
            raise _mismatch('network state keys', sorted(sd['ngp']), sorted(mine))
        for k, v in mine.items():
            if tuple(sd['ngp'][k].shape) != tuple(v.shape):
                raise _mismatch(f'ngp.{k} shape', tuple(sd['ngp'][k].shape), tuple(v.shape))
        self.optimizer.check_state(sd['optimizer'])
        hist = sd.get('history')            # optional: checkpoints made before the loss history have none
        if hist is not None and (hist.dim() != 2 or hist.shape[1] != len(HISTORY_COLUMNS) or hist.shape[0] > sd['itr']):
            raise _mismatch('history shape', tuple(hist.shape), f'(<= {sd["itr"]}, {len(HISTORY_COLUMNS)})')

    def _load_scene_state(self, sd):
        self.ngp.load_state_dict(sd['ngp'])          # copies into the existing tensors: the parameters stay views of the flat buffer
        for k, v in sd['ngp_extra'].items():
            setattr(self.ngp, k, v)
        self.optimizer.load_state_dict(sd['optimizer'])
        self.gen.set_state(sd['gen'])
        self.next_itr = int(sd['itr'])
        self._history.fill_(math.nan)
        hist = sd.get('history')
        if hist is not None:
            self._history_rows(hist.shape[0])
            self._history[:hist.shape[0]].copy_(hist)

    def load_state_dict(self, sd, use_diffusion=True):
        """continue from ``state_dict``'s ``sd``: ``check_state`` first (ValueError before any device state is touched), then the network,
        optimiser and generator states in place, and last this rank's global CPU / CUDA generator states -- call it immediately before the
        first resumed step.  The view-batched step (``views_per_step``) may continue at another world size unless cuda_ray is on; rank r
        then takes the generator states of saved rank r mod the saved world size."""
        self.check_state(sd, use_diffusion)
        self._load_scene_state(sd)
        _restore_rng(sd['rng'], self.cache.input_rgb.device, self.rank)


# ----------------------------------------------------------------------------------------------------------------------
# scene-batched distillation: S scenes, each on the reference's iteration, sharing the VAE and UNet batches
# ----------------------------------------------------------------------------------------------------------------------
class MultiSceneDistiller:
    """Distils S scenes at once on one GPU.  Every scene runs the reference's iteration exactly -- photometric sub-step and Adam, then ONE
    target view and Adam (``Distiller.step`` with ``views_per_step=None``) -- with its own network, optimiser and random streams, held by one
    ``Distiller`` per scene.  What is shared is the SDS work: the S upsampled renders go through ONE VAE encode, ONE ``PLMSSampler.sample_rows``
    (each scene at its own noise level, so with its own number of UNet evaluations; the UNet runs at the batch of scenes still sampling) and
    ONE decode, in chunks of at most ``max_batch`` scenes.  The SDS phase's UNet and VAE run at batch S instead of S times at batch 1.

    ``sds_method`` ('plms' or 'onestep', see ``Distiller``) is every scene's SDS target.  With 'onestep' a chunk's targets are ONE
    ``DDPM.forward_noloss`` call -- one graph replay of its b scenes (2b guided), each at its own level, one UNet evaluation per scene --
    whose draws come from each scene's ``view_seed(seeds[k], itr, v, 2)`` generator (noise, then the keep uniform); ``plms_noise`` is not
    used.

    ``cond_scale`` guides every scene's SDS target with the same classifier-free guidance scale (1: none; ValueError at construction when the
    VLDM has no conditional dropout).  ``max_batch`` counts scenes, guided or not: a guided chunk of b scenes still sampling evaluates its
    conditional and null rows as one UNet batch of 2b rows, so the sampler's CUDA graphs cover the batch sizes 1..max_batch unguided and
    2, 4, .., 2 * max_batch guided, each captured when a run first reaches it.

    Draws of scene k: the view permutation and ``u`` from ``torch.Generator().manual_seed(seeds[k])`` in the reference's order (as in
    ``Distiller(seed=seeds[k])``); the render jitter / inverse-CDF samples of the photometric render from ``view_seed(seeds[k], itr, 0, 0)``, those
    of the fusion render of view v from ``view_seed(seeds[k], itr, v, 1)`` and the PLMS noise from ``view_seed(seeds[k], itr, v, 2)``.  A scene's
    trajectory therefore does not depend on which scenes share its batch.  Parity tests replace them through ``render_noise(scene, 'A'|'B')`` and
    ``plms_noise(scene) -> noise_fn``, the per-scene counterparts of ``Distiller.render_noise`` and ``PLMSSampler.noise_fn``.

    Not supported: ``views_per_step`` (NotImplementedError), ``fused_glue=False`` and ``opt.hw_scale != 2`` (NotImplementedError), scenes of
    different image, latent or ray sizes (ValueError), CPU tensors (RuntimeError).  ``lambda_entropy`` and ``max_itr`` (the rows of each
    scene's loss history) pass to every scene's ``Distiller``."""

    def __init__(self, ngps, vae, vldm, opt, caches, *, seeds, percep=None, max_batch=8, cond_scale=1.0, sds_method='plms', **kw):
        _check_cond_scale(vldm, cond_scale, 'MultiSceneDistiller')
        _check_sds_method(sds_method, 'MultiSceneDistiller')
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
        self.scenes = [Distiller(ngp, vae, vldm, opt, cache, seed=int(sd), percep=percep, cond_scale=cond_scale, sds_method=sds_method, **kw)
                       for ngp, cache, sd in zip(ngps, caches, seeds)]
        for d in self.scenes:
            d._keyed = True
        self.seeds = [int(s) for s in seeds]
        self.max_batch = int(max_batch)
        self.cond_scale = float(cond_scale)
        self.sds_method = sds_method
        lead = self.scenes[0]
        self.start_fusion_step = lead.start_fusion_step
        # one sampler for all scenes: its UnetGraph holds one graph per UNet batch size (at most max_batch of them: see the class docstring)
        self.sampler = PLMSSampler(vldm, lead.sampler.plms_steps, use_cuda_graph=lead.sampler.use_cuda_graph)
        self.render_noise = None
        self.plms_noise = None     # parity tests: callable(scene) -> noise_fn(like) serving that scene's PLMS draws
        self.next_itr = 0          # the iteration after the last one run
        self.last = {}

    def __len__(self):
        return len(self.scenes)

    @property
    def history(self) -> list:
        """every scene's loss history (``Distiller.history``), in scene order"""
        return [d.history for d in self.scenes]

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
        self.next_itr = itr + 1
        return torch.stack([d.photometric_substep(itr) for d in self.scenes])

    def fusion_substep(self, itr: int, max_thres: Optional[float] = None):
        """every scene's fusion sub-step (:259-352) with the VAE encode, PLMS sampling and decode batched over chunks of scenes; returns the [S]
        losses.  ``max_thres`` forces one noise level for every scene (tests); by default scene k uses its own ``u`` (:303)."""
        S = len(self.scenes)
        self.next_itr = itr + 1
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
            if sds and self.sds_method == 'onestep':                                           # one forward_noloss of the chunk's scenes
                feats = torch.cat([self.scenes[k].cache.target_features[v:v + 1] for k, v in zip(ks, views)])
                pred = self.scenes[ks[0]]._fusion_target([r[3] for r in renders], feats, mts, None,
                                                         seeds=[view_seed(self.seeds[k], itr, v, 2) for k, v in zip(ks, views)])[0]
                replays += 1
                for k in ks:
                    calls[k] = self.scenes[k].last['unet_calls'] = 1
            elif sds:
                feats = torch.cat([self.scenes[k].cache.target_features[v:v + 1] for k, v in zip(ks, views)])
                pred = self.scenes[ks[0]]._fusion_target([r[3] for r in renders], feats, mts, self._plms_noise_fn(ks, views, itr, renders[0][0].device),
                                                         sampler=self.sampler)[0]
                replays += self.sampler.last_graph_replays
                for j, k in enumerate(ks):
                    calls[k] = self.sampler.last_row_calls[j]
                    self.scenes[k].last['unet_calls'] = calls[k]
            for j, k in enumerate(ks):
                d = self.scenes[k]
                losses[k], logged = d._fusion_grad(itr, *renders[j], views[j], pred[j], mts[j])
                d.last['fusion_loss'] = losses[k]
                d._record(itr, 3, logged)                                                      # :349
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

    def state_dict(self, itr: Optional[int] = None, use_diffusion=True) -> dict:
        """``{'version', 'itr', 'scenes'}``: the shared iteration (default: the one after the last step run) and one ``Distiller.state_dict``
        per scene, each holding the process's global generator states"""
        itr = self.next_itr if itr is None else int(itr)
        rng = _rng_states(self.scenes[0].cache.input_rgb.device)
        return dict(version=CHECKPOINT_VERSION, itr=itr, scenes=[dict(d._scene_state(itr, use_diffusion), rng=rng) for d in self.scenes])

    def load_state_dict(self, sd, use_diffusion=True):
        """continue from ``state_dict``'s ``sd``: every scene checked first (ValueError naming the scene and the field, before any device
        state is touched), then every scene's state loaded, then the global generators restored -- immediately before the first resumed step"""
        if sd.get('version') != CHECKPOINT_VERSION:
            raise _mismatch('the checkpoint format version', sd.get('version'), CHECKPOINT_VERSION)
        if len(sd['scenes']) != len(self.scenes):
            raise _mismatch('the number of scenes', len(sd['scenes']), len(self.scenes))
        for k, (d, s) in enumerate(zip(self.scenes, sd['scenes'])):
            if s['itr'] != sd['itr']:
                raise ValueError(f'load_state_dict: scene {k} is saved at iteration {s["itr"]}, the others at {sd["itr"]}')
            try:
                d.check_state(s, use_diffusion)
            except ValueError as e:
                raise ValueError(f'scene {k}: {e}') from None
        for d, s in zip(self.scenes, sd['scenes']):
            d._load_scene_state(s)
        self.next_itr = int(sd['itr'])
        _restore_rng(sd['scenes'][0]['rng'], self.scenes[0].cache.input_rgb.device, 0)


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


class NativeSceneBuilder:
    """``ReferenceSceneBuilder`` without pytorch3d or the reference tree: the same protocol (``build``, ``eval_views``, ``circle_views``) and
    the same ``SceneCache`` / ``EvalViews`` contents in the same view order, following distillation.py:65-125 step by step.  The camera maths
    runs on the host (``cameras.py``: relative / voxel-frame cameras, the 50 jittered circle-path cameras drawn with ``torch.rand`` from
    torch's global generator as the reference draws them), every ray grid of a call in one ``sfb_grid_rays`` launch, and the EFT feature
    cache of all (scene + circle) views through ``EpipolarFeatureTransformer.feature_cache`` -- the ResNet-18 pyramid once per scene instead
    of twice per view.  ``scene_cameras``: pytorch3d-style cameras (any object with R, T, focal_length, principal_point, image_size)."""

    RAYS_HW = 128           # sampler_feat: 256 // 2 (:85)
    EFT_HW = 32             # renderer_feat: 256 // 8, 20 points per ray (:86; utils/render_utils.py:133-144)
    EFT_DEPTHS = 20
    EVAL_HW = 256           # sampler_grid (:85)
    IMAGE_HW = 256          # every grid's pixel centres are those of the 256 x 256 image (utils/render_utils.py:38-41)

    def __init__(self, gpu):
        self.gpu = gpu
        self.device = torch.device('cuda', gpu) if isinstance(gpu, int) else torch.device(gpu)

    def _rays(self, cams, hw):
        from .cameras import grid_rays
        return grid_rays(cams, hw, hw, self.device, self.IMAGE_HW, self.IMAGE_HW)

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True) -> 'SceneCache':
        from . import cameras as C
        cams = C.as_cameras(scene_cameras).cpu()
        input_idx = [int(i) for i in input_idx]
        vox = C.relative_cameras(cams, [0], center_at_origin=False)                                                  # :70
        in_o, in_d = self._rays(C.camera_slice(vox, input_idx), self.RAYS_HW)                                        # :201-204
        dev = self.device
        n_rays = self.RAYS_HW * self.RAYS_HW
        empty = lambda *s: torch.zeros(0, *s, device=dev)
        feats, eft_imgs, t_o, t_d = empty(256, self.EFT_HW, self.EFT_HW), empty(3, self.IMAGE_HW, self.IMAGE_HW), empty(n_rays, 3), empty(n_rays, 3)
        if use_diffusion:
            aug = C.concat_cameras([cams, C.interpolated_path(cams, n=50, theta_offset_max=0.17)])                   # :73-74
            aug_rel = C.relative_cameras(aug, [0], center_at_origin=True)                                            # :75
            aug_vox = C.relative_cameras(aug, [0], center_at_origin=False)                                           # :76
            cam_dist_mean = torch.mean(torch.linalg.norm(cams.get_camera_center(), axis=1))                          # :82-84
            V = len(aug_rel)
            per_view = [C.relative_cameras(aug_rel, [ci], center_at_origin=True) for ci in range(V)]                 # :98 relative_cam(..., query_idx=[ci])
            q_o, q_d = self._rays(C.concat_cameras([c[ci] for ci, c in enumerate(per_view)]), self.EFT_HW)
            lengths = torch.linspace(float(cam_dist_mean - 5.0), float(cam_dist_mean + 5.0), self.EFT_DEPTHS, device=dev)
            context = [c[input_idx] for c in per_view]                                                               # input_cameras of view ci (:98)
            input_rgb = scene_rgb[input_idx].to(dev)                                                                 # scene_rgb_aug[input_idx] (:77-79, :98)
            feats, lr = eft.feature_cache(q_o, q_d, lengths.expand(V, q_o.shape[1], -1), context, input_rgb, (self.EFT_HW, self.EFT_HW))   # :99-116
            eft_imgs = F.interpolate(lr, scale_factor=float(self.IMAGE_HW // self.EFT_HW), mode='bilinear')          # :118-119
            t_o, t_d = self._rays(aug_vox, self.RAYS_HW)                                                             # :115, :274-277
        return SceneCache(input_rgb=scene_rgb[input_idx].float(), input_mask=scene_mask[input_idx].float(), input_rays_o=in_o, input_rays_d=in_d,
                          target_features=feats, target_eft_image=eft_imgs, target_rays_o=t_o, target_rays_d=t_d)

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        """``ReferenceSceneBuilder.eval_views``: every scene camera in the voxel frame (:70) through the 256 x 256 grid (:85, :393-406)"""
        from . import cameras as C
        from .evaluate import EvalViews
        vox = C.relative_cameras(C.as_cameras(scene_cameras).cpu(), [0], center_at_origin=False)
        o, d = self._rays(vox, self.EVAL_HW)
        return EvalViews(rays_o=o, rays_d=d, rgb=scene_rgb.float(), mask=scene_mask.float())

    def circle_views(self, scene_cameras, n=50):
        """``ReferenceSceneBuilder.circle_views``: ``get_interpolated_path(scene_cameras_vox, n, method='circle')`` (no jitter) through the
        256 x 256 grid (:461-469) -> (rays_o, rays_d), each [n, 256*256, 3]"""
        from . import cameras as C
        vox = C.relative_cameras(C.as_cameras(scene_cameras).cpu(), [0], center_at_origin=False)
        return self._rays(C.interpolated_path(vox, n=n), self.EVAL_HW)


def distillation_loop(gpu, args, opt, model_tuple, save_dir, seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx,
                      use_diffusion=True, max_itr=3000, loss_fn_vgg=None, *, scene_builder=None, views_per_step=None, on_iteration=None, seed=None,
                      process_group=None, evaluate=False, visualize=False, visualize_shadings=(), evaluate_baselines=False, vldm_cond_scale=1.0,
                      cond_scale=1.0, sds_method='plms', checkpoint_every=None, resume=False, lambda_entropy=0.0, progress_every=None,
                      percep_weights=None):
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
    the GPU (``video.py``); Pillow writes the files.  ``visualize_shadings`` (with ``visualize``), e.g. ``('normal', 'textureless')``, adds one
    ``{save_dir}/render_gifs/{seq_name}_circle_{shading}.gif`` per listed shading of ``NeRFNetwork.forward``: the circle views rendered with
    that shading under a headlight (``evaluate.render_views``), at ambient ratio 0.1 for the lit shadings ('lambertian', 'textureless') so the
    geometry shows, 1.0 for 'normal' and 'albedo'.

    ``lambda_entropy`` weights the reference's entropy regulariser of both sub-steps (:236-241, :338-344; its loop sets 0, the default
    here); a negative value is a ValueError.  Every step records the logged terms in ``Distiller.history`` on the device.

    ``progress_every=K`` writes the reference's periodic outputs (:355-388; ``progress.ProgressWriter``) after every iteration ``itr`` with
    ``itr % K == 0`` (the reference: K = 20): ``{args.exp_dir}/log/{seq_name}_loss.jpg`` and ``{seq_name}_fusionloss.jpg``, the loss curves
    of every iteration so far drawn with Pillow, and ``{seq_name}_vis.jpg``, the eval-mode render | silhouette of the iteration's photometric
    input view through the builder's ``eval_views`` rays (a builder without ``eval_views`` fails before the loop).  Writing them draws from
    no global generator and leaves the network in train mode, so the run's steps are those of a run without them.  With a process group
    rank 0 writes.  None (the default) writes nothing; K <= 0 is a ValueError.  The tqdm bar and the ``running_loss`` print stay out.
    With a process group the plots show rank 0's own history (``Distiller.history``): in the view-batched step its photometric terms exist
    every R-th iteration only, so those curves are dots rather than lines, and its fusion curve is its views' share of the step's mean,
    not the mean over all V views.
    ``scene_valid_region`` is accepted and unused, as in the reference's loop body (:192-195 overwrites the region with ones), and so is
    ``loss_fn_vgg`` unless ``evaluate``.  Extensions, keyword-only: ``views_per_step`` (view-batched step, see the module docstring; with
    torch.distributed initialised and ``process_group`` given the views are sharded over its ranks), ``seed``, ``evaluate``, ``visualize``,
    ``visualize_shadings``.

    ``evaluate_baselines=True`` (needs ``use_diffusion`` and the builder's ``eval_views``) also scores the paper's two intermediate stages on
    the scene views after the loop (``baselines.evaluate_baselines``): the cached EFT images and VLDM samples from pure noise conditioned on
    the cached EFT features (guidance scale ``vldm_cond_scale``, draws keyed by the scene's seed), with the same metrics as ``evaluate``, and
    writes ``{save_dir}/metrics/{seq_name}_eft.txt``, ``{seq_name}_vldm.txt`` and ``{save_dir}/render_gifs/{seq_name}_baselines.gif``.

    ``cond_scale`` is the classifier-free guidance scale of the distillation itself: every SDS target is sampled with
    eps = null + (cond - null) * cond_scale, the conditional and null branches as one UNet batch (1, the default, is the reference's unguided
    loop).  It is independent of ``vldm_cond_scale``, which only guides the VLDM baseline's samples.  Guidance needs a VLDM trained with
    conditional dropout (ValueError before any work otherwise); with ``use_diffusion=False`` there is no SDS target and it is ignored.

    ``sds_method`` is the SDS target (``Distiller``): 'plms', the default, is the reference's multi-step PLMS run; 'onestep' is
    ``DDPM.forward_noloss`` at the same noise level, one UNet evaluation per target instead of about 38 -- the paper's one-step ablation
    and a much cheaper distillation.  Any other value raises ValueError before any work.

    ``checkpoint_every=K`` writes ``{save_dir}/checkpoints/{seq_name}.ckpt`` (``Distiller.state_dict``: network, Adam state, counters, every
    generator, seed, fingerprint and cache digest) after every iteration ``itr`` with ``(itr + 1) % K == 0`` and after the last one, before
    ``on_iteration`` sees it.  Each write goes to a temporary file in the same directory, is fsynced and then renamed over the old one, so an
    interruption mid-write keeps the previous checkpoint; with ``process_group`` rank 0 writes and every rank waits at a barrier.
    ``resume=True`` builds the cache as a fresh run does and then, if the checkpoint exists, continues from it: the base seed is the saved one
    (an explicit ``seed`` that differs is a ValueError), the global generators are restored right before the first resumed iteration, and
    ``on_iteration`` sees only the iterations run.  A state the run cannot continue (other settings, cache, or world size where that matters:
    ``Distiller.check_state``) is a ValueError.  With ``max_itr`` at or below the saved iteration no iteration runs and the outputs come from
    the saved state, so a finished run with a checkpoint can be extended by a larger ``max_itr``; without a checkpoint the run starts fresh,
    so an interrupted command can be re-issued unchanged.

    ``percep_weights`` (a state dict in ``lpips.LPIPS(net='vgg')``'s key layout, e.g. ``loss_fn_vgg.state_dict()`` or
    ``lpips_vgg.load_lpips_state_dict(path)``) is loaded into the loop's ``PerceptualLoss`` before the first iteration, so the perceptual
    term of the fusion loss is the reference's pretrained LPIPS-VGG (:161, :312-314).  None (the default) keeps ``PerceptualLoss``'s seeded
    random initialisation.  The checkpoint fingerprint records pretrained weights, so a resume that mixes the two is a ValueError.
    Returns the optimised network."""
    eft, vae, vldm = model_tuple
    _check_sds_method(sds_method, 'distillation_loop')
    _check_lambda_entropy(lambda_entropy, 'distillation_loop')
    if use_diffusion:
        _check_cond_scale(vldm, cond_scale, 'distillation_loop')
    rank, world = 0, 1
    if process_group is not None:
        rank, world = torch.distributed.get_rank(process_group), torch.distributed.get_world_size(process_group)

    def make(ngps, caches, percep, seed):
        return Distiller(ngps[0], vae, vldm, opt, caches[0], plms_steps=50, start_fusion_step=1000, lambda_color=1.0, lambda_sil=1.0,   # :148-160
                         lambda_opacity=1e-3, seed=seed, rank=rank, world_size=world, process_group=process_group, percep=percep, lambda_percep=0.1,
                         start_percep_step=1000, views_per_step=views_per_step, cond_scale=cond_scale if use_diffusion else 1.0, sds_method=sds_method,
                         lambda_entropy=lambda_entropy, max_itr=max_itr)
    ngp_network, = _run_distillation(gpu, args, opt, eft, save_dir, [(seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx)],
                                     make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate, loss_fn_vgg, visualize,
                                     visualize_shadings, _baselines(evaluate_baselines, vae, vldm, vldm_cond_scale), checkpoint_every, resume,
                                     progress_every, percep_weights)
    print('input idx', input_idx)
    return ngp_network


def distill_scenes(gpu, args, opt, model_tuple, save_dir, scenes, *, use_diffusion=True, max_itr=3000, scene_builder=None, seed=None, on_iteration=None,
                   evaluate=False, loss_fn_vgg=None, visualize=False, visualize_shadings=(), evaluate_baselines=False, vldm_cond_scale=1.0,
                   cond_scale=1.0, sds_method='plms', checkpoint_every=None, resume=False, lambda_entropy=0.0, progress_every=None,
                   percep_weights=None, seeds=None):
    """``distillation_loop`` for several scenes at once on one GPU (``MultiSceneDistiller``): demo.py's per-scene loop (demo.py:87-103) becomes
    one call.  ``scenes`` is a list of ``(seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx)``, the per-scene
    arguments demo.py passes to ``distillation_loop``.  Each scene's cache is built as ``distillation_loop`` builds it (``ReferenceSceneBuilder``,
    or ``scene_builder.build(...)``), one ``PerceptualLoss`` serves all scenes, scene k is seeded with ``seed + k`` (``seed`` drawn from torch's
    seed when None), and every network is saved as ``{'model_state_dict': ngp.state_dict()}`` to ``{save_dir}/{seq_name}.pt`` (:495-496).
    Scenes of one call must share image, latent and ray sizes.  With several GPUs, each rank passes its own share of the scenes.
    ``on_iteration(itr, multi_scene_distiller)`` runs after every iteration.  ``evaluate`` / ``loss_fn_vgg``: each scene is scored and its
    ``{save_dir}/metrics/{seq_name}.txt`` written as ``distillation_loop(evaluate=True)`` does, scene k's render jitter keyed by ``seed + k``.
    ``visualize`` / ``visualize_shadings``: each scene's EFT grid, gifs and jpegs as ``distillation_loop(visualize=True)`` writes them, jitter
    keyed by ``seed + k``.  ``evaluate_baselines`` / ``vldm_cond_scale``: each scene's EFT and VLDM baselines scored and written as
    ``distillation_loop(evaluate_baselines=True)`` does, scene k's VLDM draws keyed by ``seed + k``.  ``cond_scale``: the guidance scale of
    every scene's SDS targets, as ``distillation_loop(cond_scale=...)``, independent of ``vldm_cond_scale``.  ``sds_method``: every scene's
    SDS target, 'plms' or 'onestep', as ``distillation_loop(sds_method=...)``; a chunk's one-step targets are one ``forward_noloss`` call.
    ``checkpoint_every`` / ``resume``: as ``distillation_loop``'s, one ``{save_dir}/checkpoints/{seq_name}.ckpt`` per scene (scene k's part
    of ``MultiSceneDistiller.state_dict``).  Resuming needs a checkpoint at the same iteration for every scene of the call, or none (then
    the call starts fresh); anything else is a ValueError naming the scenes.  ``lambda_entropy`` / ``progress_every``: as
    ``distillation_loop``'s, every scene's entropy weight, history and progress files, scene k's snapshot jitter keyed by ``seed + k``.
    ``percep_weights``: as ``distillation_loop``'s, loaded into the one ``PerceptualLoss`` of all scenes.

    ``seeds`` (one non-negative int per scene, instead of ``seed``) seeds scene k with ``seeds[k]`` wherever the above says ``seed + k``, and
    also seeds torch's global CPU generator with ``seeds[k]`` immediately before scene k's cache is built; that stream serves the scene's
    circle-path jitter (``NativeSceneBuilder``) and then its network's initialisation.  A scene's outputs then depend on its own seed and
    inputs only, not on which other scenes share the call or their order.  Its checkpoint stores ``seeds[k]`` (and no base seed); resuming
    it under another seed, or with ``seed`` instead of ``seeds``, or the other way round, is a ValueError.
    Returns the optimised networks in the order of ``scenes``."""
    eft, vae, vldm = model_tuple
    _check_sds_method(sds_method, 'distill_scenes')
    _check_lambda_entropy(lambda_entropy, 'distill_scenes')
    if use_diffusion:
        _check_cond_scale(vldm, cond_scale, 'distill_scenes')
    if seeds is not None:
        if seed is not None:
            raise ValueError('distill_scenes: pass seed (scene k seeded seed + k) or seeds (one per scene), not both')
        seeds = list(seeds)
        if len(seeds) != len(scenes) or not all(isinstance(s, int) and not isinstance(s, bool) and 0 <= s < 2 ** 63 for s in seeds):
            raise ValueError(f'distill_scenes: seeds must hold one int in [0, 2**63) per scene ({len(scenes)} scenes, got {seeds!r})')

    def make(ngps, caches, percep, base):       # base: the base seed, or the list of per-scene seeds
        scene_seeds = list(base) if isinstance(base, list) else [base + k for k in range(len(ngps))]
        return MultiSceneDistiller(ngps, vae, vldm, opt, caches, seeds=scene_seeds, percep=percep,
                                   plms_steps=50, start_fusion_step=1000, lambda_color=1.0, lambda_sil=1.0, lambda_opacity=1e-3,   # :148-160
                                   lambda_percep=0.1, start_percep_step=1000, cond_scale=cond_scale if use_diffusion else 1.0, sds_method=sds_method,
                                   lambda_entropy=lambda_entropy, max_itr=max_itr)
    return _run_distillation(gpu, args, opt, eft, save_dir, scenes, make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate,
                             loss_fn_vgg, visualize, visualize_shadings, _baselines(evaluate_baselines, vae, vldm, vldm_cond_scale),
                             checkpoint_every, resume, progress_every, percep_weights, seeds)


def _baselines(enabled, vae, vldm, cond_scale):
    """what ``_run_distillation`` needs to score the EFT / VLDM baselines, or None when they are off"""
    return dict(vae=vae, vldm=vldm, cond_scale=float(cond_scale)) if enabled else None


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


LIT_SHADING_AMBIENT = 0.1     # ambient ratio of the lit shadings' circle gifs: mostly light, so the geometry shows


def _write_scene_pictures(save_dir, seq_name, ngp, opt, views, circle, eft_images, seed, scores=None, shadings=()):
    """the reference's sequence gif, per-view jpegs and circle gif of one distilled scene (:444-493).  The sequence frames are ``scores``'
    renders (``evaluate_scene``'s, the ones the metrics come from) or, without scores, the same renders by ``render_views`` (stream 3);
    the circle frames are ``render_views`` of the circle rays with stream 4.  ``eft_images``: the scene views' cached EFT images [V,3,h,w]
    (``use_diffusion``) or None.  Each of ``shadings`` adds ``{seq_name}_circle_{shading}.gif``: the circle views rendered with that shading
    (headlit, ``render_views``), one panel per frame."""
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
    for shading in shadings:
        ratio = 1.0 if shading in ('albedo', 'normal') else LIT_SHADING_AMBIENT
        s_image, _ = render_views(ngp, rays_o, rays_d, (hw, hw), opt, seed=seed, stream=CIRCLE_STREAM, shading=shading, ambient_ratio=ratio)
        gif_path = f'{save_dir}/render_gifs/{seq_name}_circle_{shading}.gif'
        write_gif(gif_path, to_uint8(s_image))
        print('saved video', gif_path)


def _atomic_save(obj, path):
    """torch.save to ``path`` through a temporary file in the same directory, fsynced and then renamed over ``path``: an interruption
    leaves either the old file or the new one, never a partial one"""
    tmp = f'{path}.tmp'
    try:
        with open(tmp, 'wb') as f:
            torch.save(obj, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise


def _checkpoint_paths(save_dir, scenes):
    return [f'{save_dir}/checkpoints/{sc[0]}.ckpt' for sc in scenes]


def _read_checkpoints(paths, names, seed, seeds=None):
    """the scenes' saved states for ``resume``, or None when no scene has one; ValueError when only some have one, when they are at
    different iterations or base seeds, or when an explicit ``seed`` differs from the saved base seed.  With per-scene ``seeds``
    (``distill_scenes``): ValueError unless every scene was saved with its own seed (base seed None) equal to ``seeds[k]``."""
    have = [os.path.exists(p) for p in paths]
    if not any(have):
        return None
    if not all(have):
        raise ValueError(f'resume: checkpoints exist for scenes {[n for n, h in zip(names, have) if h]} but not for '
                         f'{[n for n, h in zip(names, have) if not h]}; a call resumes all its scenes or none')
    states = [torch.load(p, map_location='cpu', weights_only=True) for p in paths]
    itrs = {n: s['itr'] for n, s in zip(names, states)}
    if len(set(itrs.values())) > 1:
        raise ValueError(f'resume: the scenes\' checkpoints are at different iterations {itrs}; a call resumes scenes saved together')
    if seeds is not None:
        for n, s, want in zip(names, states, seeds):
            if s['base_seed'] is not None:
                raise ValueError(f'resume: scene {n} was saved by a run with seed={s["base_seed"]} (scene k seeded seed + k); this call passes '
                                 f'seeds')
            if s['seed'] != want:
                raise ValueError(f'resume: scene {n} was saved with seed {s["seed"]}, this call passes {want} in seeds')
        return states
    unseeded = [n for n, s in zip(names, states) if s['base_seed'] is None]
    if unseeded:
        raise ValueError(f'resume: scenes {unseeded} were saved by a run with per-scene seeds; resume them with the same seeds')
    bases = {n: s['base_seed'] for n, s in zip(names, states)}
    if len(set(bases.values())) > 1:
        raise ValueError(f'resume: the scenes\' checkpoints come from different runs (base seeds {bases})')
    base = states[0]['base_seed']
    if seed is not None and int(seed) != base:
        raise ValueError(f'resume: seed={seed} differs from the base seed {base} the checkpoints were made with (pass seed=None or {base})')
    return states


def _write_checkpoints(dist, paths, itr, use_diffusion, base_seed):
    """every scene's checkpoint at iteration ``itr`` (the next one to run), each with the call's ``base_seed`` (None for a call with
    per-scene seeds; every scene's state holds its own seed); with a process group every rank takes part in gathering the generator
    states, rank 0 writes and all ranks wait at a barrier"""
    sd = dist.state_dict(itr, use_diffusion)
    states = sd['scenes'] if isinstance(dist, MultiSceneDistiller) else [sd]
    pg = getattr(dist, 'pg', None)
    if getattr(dist, 'rank', 0) == 0:
        os.makedirs(os.path.dirname(paths[0]), exist_ok=True)
        for st, p in zip(states, paths):
            _atomic_save(dict(st, base_seed=base_seed), p)
    if pg is not None:
        torch.distributed.barrier(group=pg)


def _run_distillation(gpu, args, opt, eft, save_dir, scenes, make, use_diffusion, max_itr, scene_builder, seed, on_iteration, evaluate=False,
                      loss_fn_vgg=None, visualize=False, visualize_shadings=(), baselines=None, checkpoint_every=None, resume=False,
                      progress_every=None, percep_weights=None, seeds=None):
    """what ``distillation_loop`` and ``distill_scenes`` share: the reference's output directories, one cache per scene of ``scenes`` (as
    ``distill_scenes`` takes them), a fresh ``NeRFNetwork(opt)`` per scene, the distiller ``make(ngps, caches, percep, seed)`` builds
    (``seed``: the base seed, or the list ``seeds``), the ``max_itr`` iterations and one saved network per scene; with ``evaluate``, the scene scores and metrics files, with
    ``visualize`` the EFT grids before the loop and the gifs and jpegs after it (scene k seeded ``scene_seeds[k]``: ``seed + k``, or
    ``seeds[k]``, which also seeds the global CPU generator before the scene's cache and network); with ``baselines`` (``_baselines``), the
    EFT and VLDM scores, metrics files and gifs after it; with ``checkpoint_every`` / ``resume`` the checkpoints, with ``progress_every`` the
    progress files and with ``percep_weights`` the pretrained perceptual term of ``distillation_loop``'s docstring.  Returns the networks."""
    from .lpips_vgg import PerceptualLoss
    from .progress import ProgressWriter, check_progress_every
    check_progress_every(progress_every)
    if checkpoint_every is not None and (isinstance(checkpoint_every, bool) or not isinstance(checkpoint_every, int) or checkpoint_every < 1):
        raise ValueError(f'checkpoint_every must be a positive int or None (got {checkpoint_every!r})')
    ckpt_paths = _checkpoint_paths(save_dir, scenes)
    saved = _read_checkpoints(ckpt_paths, [sc[0] for sc in scenes], seed, seeds) if resume else None
    builder = scene_builder if scene_builder is not None else ReferenceSceneBuilder(gpu)
    visualize_shadings = tuple(visualize_shadings)
    if not all(isinstance(sh, str) and sh and '/' not in sh for sh in visualize_shadings):
        raise ValueError(f'visualize_shadings must be shading names, got {visualize_shadings!r}')
    if visualize or progress_every is not None:
        from .video import require_pillow
        require_pillow()
    if baselines is not None:
        from .baselines import check_baseline_options
        check_baseline_options(baselines['vldm'], baselines['cond_scale'], use_diffusion)
        from .video import require_pillow
        require_pillow()
    scored = evaluate or visualize or baselines is not None
    need_views = scored or progress_every is not None
    for flag, name, sig in ((need_views, 'eval_views', '(scene_cameras, scene_rgb, scene_mask)'), (visualize, 'circle_views', '(scene_cameras)')):
        if flag and not callable(getattr(builder, name, None)):
            raise TypeError(f'{_needs(name, evaluate, visualize, baselines is not None)} needs the scene builder to provide '
                            f'{name}{sig}; {type(builder).__name__} has none')
    exp_dir = getattr(args, 'exp_dir', save_dir)
    for sc in scenes:
        os.makedirs(f'{exp_dir}/render_imgs/{sc[0]}/', exist_ok=True)                                                # :57-58
    os.makedirs(f'{exp_dir}/render_gifs/', exist_ok=True)
    os.makedirs(save_dir, exist_ok=True)
    device = torch.device('cuda', gpu) if isinstance(gpu, int) else torch.device(gpu)
    all_views = [builder.eval_views(cams, rgb, mask) for _, cams, rgb, mask, _, _ in scenes] if need_views else None
    eval_views = [v.to(device) for v in all_views] if scored else None
    # the snapshots render input views only: a copy of those rows, so the other views' rays need not stay on the device for the run
    input_views = [_view_rows(v, sc[5]).to(device) for v, sc in zip(all_views, scenes)] if progress_every is not None else None
    del all_views
    circles = [tuple(t.to(device) for t in builder.circle_views(cams)) for _, cams, _, _, _, _ in scenes] if visualize else None
    caches, cpu_streams = [], []
    for k, (_, cams, rgb, mask, _, input_idx) in enumerate(scenes):
        if seeds is not None:
            torch.default_generator.manual_seed(seeds[k])
        caches.append(builder.build(eft, cams, rgb, mask, input_idx, use_diffusion=use_diffusion).to(device))
        cpu_streams.append(torch.get_rng_state())      # where scene k's network initialisation continues its stream (with seeds)
    if baselines is not None:
        from .baselines import check_baseline_cache
        for views, cache in zip(eval_views, caches):
            check_baseline_cache(cache, views)
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
        if perceptual_loss is not None and percep_weights is not None:
            perceptual_loss.load_state_dict(percep_weights)
        ngps = []
        for k in range(len(scenes)):
            if seeds is not None:
                torch.set_rng_state(cpu_streams[k])
            ngps.append(NeRFNetwork(opt).to(device).train())                                                       # :164
        if seeds is not None:
            base_seed, scene_seeds = None, list(seeds)
        else:
            if saved is not None:
                base_seed = saved[0]['base_seed']
            else:
                base_seed = torch.seed() % (2 ** 31) if seed is None else int(seed)
            scene_seeds = [base_seed + k for k in range(len(scenes))]
        dist = make(ngps, caches, perceptual_loss, scene_seeds if seeds is not None else base_seed)
        progress = None
        if progress_every is not None and getattr(dist, 'rank', 0) == 0:
            progress = ProgressWriter(exp_dir, [sc[0] for sc in scenes], input_views, [sc[5] for sc in scenes], opt)
        start = 0
        if saved is not None:                  # restores the global generators too: nothing may draw between here and the first step
            multi = isinstance(dist, MultiSceneDistiller)
            dist.load_state_dict(dict(version=saved[0]['version'], itr=saved[0]['itr'], scenes=saved) if multi else saved[0], use_diffusion)
            start = saved[0]['itr']
        for itr in range(start, max_itr):                                                                           # :174
            if use_diffusion:
                dist.step(itr)
            else:
                dist.photometric_substep(itr)
            if checkpoint_every is not None and ((itr + 1) % checkpoint_every == 0 or itr == max_itr - 1):
                _write_checkpoints(dist, ckpt_paths, itr + 1, use_diffusion, base_seed)
            if progress is not None and itr % progress_every == 0:                                                   # :355
                progress.write(itr, getattr(dist, 'scenes', [dist]))
            if on_iteration is not None:
                on_iteration(itr, dist)
        torch.cuda.synchronize(device)
    for (seq_name, *_rest), ngp in zip(scenes, ngps):
        torch.save({'model_state_dict': ngp.state_dict()}, f'{save_dir}/{seq_name}.pt')                             # :495-496
    if evaluate or visualize or baselines is not None:
        from .evaluate import evaluate_scene, write_scene_metrics
        with torch.cuda.device(device):
            eval_percep = None if loss_fn_vgg is None or not (evaluate or baselines) else PerceptualLoss('vgg', device=device).load_state_dict(loss_fn_vgg.state_dict())
            for k, ((seq_name, *_rest), ngp, views) in enumerate(zip(scenes, ngps, eval_views)):
                scores = None
                if evaluate:
                    scores = evaluate_scene(ngp, views, opt, eval_percep, seed=scene_seeds[k])                    # :391-433
                    print('warning: this metric is used for debugging only and not the final metric')
                    print(f'{getattr(args, "category", "")} scene {seq_name}')
                    write_scene_metrics(f'{save_dir}/metrics/{seq_name}.txt', scores)                              # :434-441
                if visualize:
                    _write_scene_pictures(save_dir, seq_name, ngp, opt, views, circles[k], caches[k].target_eft_image if use_diffusion else None,
                                          scene_seeds[k], scores, visualize_shadings)                                 # :444-493
            if baselines is not None:
                from .baselines import evaluate_baselines
                sampler = PLMSSampler(baselines['vldm'], 50)                                                        # plms_steps of the loop (:160)
                for k, ((seq_name, *_rest), views) in enumerate(zip(scenes, eval_views)):
                    evaluate_baselines(save_dir, seq_name, baselines['vldm'], baselines['vae'], caches[k], views, eval_percep, seed=scene_seeds[k],
                                       cond_scale=baselines['cond_scale'], sampler=sampler)
    return ngps


def _view_rows(views, idx):
    """the rows ``idx`` of ``views`` (``evaluate.EvalViews``) as new tensors"""
    from .evaluate import EvalViews
    idx = [int(i) for i in idx]
    return EvalViews(*[getattr(views, f)[idx] for f in EvalViews.__dataclass_fields__])


def _needs(name, evaluate, visualize, baselines=False):
    """the option that asked the scene builder for ``name``, for the error message"""
    if name == 'eval_views':
        return ('evaluate=True' if evaluate else 'visualize=True' if visualize else 'evaluate_baselines=True' if baselines
                else 'progress_every')
    return 'visualize=True'
