"""oracle/distill_oracle.py -- CPU restatement of one iteration of the reference's distillation loop
(sparsefusion/distillation.py:174-352), assembled from the oracle's parts: ngp_oracle.run (renderer_df.run + the
field), unet_oracle.plms_sample / unet_forward (PLMSSampler + Unet), torch autograd + torch.optim.Adam.

TEST INFRASTRUCTURE ONLY.  Used by tests/test_distillation_gpu.py as the checker of Distiller.step and by bench.py as
the CPU baseline / `--impl reference` arm (the reference itself has no CPU path for the NGP render -- CUDA-only
extensions -- and cannot be imported on the GPU box at all).

The VAE handed in is oracle/vae_oracle.TorchVAE (torch restatement pinned bit-exact to the reference's Encoder / Decoder by
tests/golden/vae.npz); the product's AutoencoderKL has no torch / CPU execution path.
"""
from __future__ import annotations

import time
from typing import Callable, Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import ngp_oracle as no
from . import unet_oracle as uo


def normalize(x):
    return torch.clip(x * 2 - 1.0, -1.0, 1.0)


def unnormalize(x):
    return torch.clip((x + 1.0) / 2.0, 0.0, 1.0)


def huber(x, y, scaling=0.1):
    return ((1 + (x - y) ** 2 / (scaling ** 2)).clamp(1e-4).sqrt() - 1) * float(scaling)


class OracleDistiller:
    """mirrors sparsefusion_b200.distillation.Distiller on CPU tensors; every random draw is injectable"""

    def __init__(self, field_params: Dict[str, torch.Tensor], vae, unet_sd, unet_cfg, cache, *, hw_scale=2, z_scale_factor=0.18215,
                 plms_steps=50, start_fusion_step=1000, seed=0, rank=0, level_scales=None, lr=5e-4, percep=None, lambda_percep=0.1,
                 start_percep_step=1000):
        self.params = {k: v.clone().requires_grad_(True) for k, v in field_params.items()}
        self.field = no.Field(self.params, level_scales=level_scales)
        self.vae, self.unet_sd, self.cfg, self.cache = vae, unet_sd, unet_cfg, cache
        self.hw_scale, self.z, self.plms_steps, self.start_fusion_step = hw_scale, z_scale_factor, plms_steps, start_fusion_step
        self.opt = torch.optim.Adam([{'params': [self.params['encoder.embeddings']], 'lr': lr * 10},
                                     {'params': [self.params[k] for k in no.PARAM_KEYS[1:]], 'lr': lr}])
        self.sched = torch.optim.lr_scheduler.StepLR(self.opt, step_size=3000, gamma=0.2)
        self.gen = torch.Generator().manual_seed(seed)
        self.rank = rank
        self.percep, self.lambda_percep, self.start_percep_step = percep, lambda_percep, start_percep_step   # lpips_oracle.PerceptualLoss or None
        self.timing: Dict[str, float] = {}

    def _render(self, ro, rd, noise):
        pn, un = noise
        r = no.run(self.field, ro, rd, perturb_noise=pn, pdf_noise=un, min_near=0.1, bg_color=0.0, training=True)
        hw = int(round(ro.shape[0] ** 0.5))
        image = r['image'].reshape(1, hw, hw, 3).permute(0, 3, 1, 2).contiguous()
        sil = r['weights_sum'].reshape(1, hw, hw, 1).permute(0, 3, 1, 2).contiguous()
        return image, sil

    def step(self, itr: int, render_noise: Callable[[str], tuple], plms_noise, max_thres: Optional[float] = None):
        c = self.cache
        t0 = time.perf_counter()
        # --- A (distillation.py:185-247)
        idx = int(torch.randperm(c.input_rgb.shape[0], generator=self.gen)[0])
        image, sil = self._render(c.input_rays_o[idx], c.input_rays_d[idx], render_noise('A'))
        rgb = F.interpolate(c.input_rgb[idx:idx + 1], scale_factor=1.0 / self.hw_scale)
        mask = F.interpolate(c.input_mask[idx:idx + 1], scale_factor=1.0 / self.hw_scale)
        loss_a = huber(image, rgb).abs().mean() + huber(sil, mask).abs().mean() + 1e-3 * torch.sqrt(sil ** 2 + .01).mean()
        self.opt.zero_grad()
        loss_a.backward()
        self.opt.step()
        self.sched.step()
        t1 = time.perf_counter()
        # --- B (:259-352)
        self.opt.zero_grad()
        perm = torch.randperm(c.target_features.shape[0], generator=self.gen)
        vi = int(perm[(1 + self.rank) % c.target_features.shape[0]])
        u = torch.rand(1, generator=self.gen)
        image, sil = self._render(c.target_rays_o[vi], c.target_rays_d[vi], render_noise('B'))
        image = F.interpolate(image, scale_factor=self.hw_scale, mode='bilinear')
        sil = F.interpolate(sil, scale_factor=self.hw_scale, mode='bilinear')
        t2 = time.perf_counter()
        calls = 0
        if itr > self.start_fusion_step:
            with torch.no_grad():
                latents = self.vae.encode(normalize(image)).mode() * self.z
                t3 = time.perf_counter()
                if max_thres is None:
                    max_thres = u.clamp(min=0.0, max=0.99).item()
                feats = c.target_features[vi:vi + 1]
                pred_x0, _, _, acp, calls = uo.plms_sample(lambda xx, ls: uo.unet_forward(self.unet_sd, self.cfg, xx, ls, feats), latents,
                                                           max_thres, plms_noise, self.plms_steps)
                t4 = time.perf_counter()
                pred_img = unnormalize(self.vae.decode(1.0 / self.z * pred_x0)).clip(0.0, 1.0)
                t5 = time.perf_counter()
            fusion = ((1 - acp) * (image - pred_img).abs().mean()).sum()
            if self.percep is not None and itr >= self.start_percep_step:           # distillation.py:176-178, :312-314
                fusion = fusion + self.percep(image, pred_img, normalize=True).mean() * self.lambda_percep
            self.timing.update(vae_encode=t3 - t2, plms=t4 - t3, vae_decode=t5 - t4)
        else:
            nrgb = c.target_eft_image[vi:vi + 1]
            nmask = (nrgb.mean(dim=1, keepdim=True) > .1).float()
            fusion = huber(image, nrgb).abs().mean() + huber(sil, nmask).abs().mean()
        loss_b = fusion + 1e-3 * torch.sqrt(sil ** 2 + .01).mean()
        loss_b.backward()
        self.opt.step()
        t6 = time.perf_counter()
        self.timing.update(substep_a=t1 - t0, render_b=t2 - t1, total=t6 - t0, unet_calls=calls)
        return loss_a.detach(), loss_b.detach()


def synthetic_scene(n_input=2, n_target=64, image_size=256, latent=32, feat_ch=256, render_hw=128, seed=0, radius=5.0):
    """BASELINE.json config 3's synthetic hydrant-style scene (SURVEY.md §8d C3): object-centric circle cameras, random
    images with a disc mask, N(0,1) EFT features.  Returns a dict of CPU tensors with the SceneCache field names."""
    rng = np.random.default_rng(seed)
    cams = no.circle_cameras(n_target, radius=radius)
    yy, xx = np.mgrid[0:image_size, 0:image_size]
    disc = (((yy - image_size / 2) ** 2 + (xx - image_size / 2) ** 2) < (0.35 * image_size) ** 2).astype(np.float32)

    def rays(idx):
        o, d = zip(*[no.camera_rays(cams[i], render_hw, render_hw) for i in idx])
        return torch.from_numpy(np.stack(o)), torch.from_numpy(np.stack(d))
    in_idx = [int(i * n_target / n_input) for i in range(n_input)]
    iro, ird = rays(in_idx)
    tro, trd = rays(range(n_target))
    return dict(
        input_rgb=torch.from_numpy(rng.random((n_input, 3, image_size, image_size), dtype=np.float32) * disc),
        input_mask=torch.from_numpy(np.broadcast_to(disc, (n_input, 1, image_size, image_size)).copy()),
        input_rays_o=iro, input_rays_d=ird,
        target_features=torch.from_numpy(rng.standard_normal((n_target, feat_ch, latent, latent), dtype=np.float32)),
        target_eft_image=torch.from_numpy(rng.random((n_target, 3, image_size, image_size), dtype=np.float32) * disc),
        target_rays_o=tro, target_rays_d=trd)
