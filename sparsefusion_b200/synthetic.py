"""Synthetic scenes for benches and smoke runs (no dataset, no pytorch3d): BASELINE.json config 3's "synthetic
hydrant-shaped cameras" -- an object-centric fly-around as utils/camera_utils.py:190-259 (get_interpolated_path) produces,
rays on the 128x128 pixel-centre grid of utils/render_utils.py:40-65 (NDC from 1-1/W to -1+1/W, directions not
normalised, as pytorch3d's GridRaysampler emits them; SURVEY.md §8c/§8d).
"""
from __future__ import annotations

import math

import numpy as np
import torch


def circle_cameras(n_views: int, radius: float = 5.0, elevation_deg: float = 15.0):
    """camera centres on a circle at the given elevation, looking at the origin, +y up -> list of (centre [3], R [3,3] rows right/up/fwd)"""
    el = math.radians(elevation_deg)
    cams = []
    for i in range(n_views):
        az = 2 * math.pi * i / n_views
        c = np.array([radius * math.cos(el) * math.sin(az), radius * math.sin(el), radius * math.cos(el) * math.cos(az)])
        fwd = -c / np.linalg.norm(c)
        right = np.cross(np.array([0.0, 1.0, 0.0]), fwd)
        right /= np.linalg.norm(right)
        up = np.cross(fwd, right)
        cams.append((c.astype(np.float32), np.stack([right, up, fwd]).astype(np.float32)))
    return cams


def camera_rays(cam, H: int, W: int, focal_ndc: float = 4.0):
    c, R = cam
    xs = np.linspace(1 - 1 / W, -1 + 1 / W, W, dtype=np.float32)
    ys = np.linspace(1 - 1 / H, -1 + 1 / H, H, dtype=np.float32)
    yy, xx = np.meshgrid(ys, xs, indexing='ij')
    d = np.stack([xx / focal_ndc, yy / focal_ndc, np.ones_like(xx)], axis=-1).reshape(-1, 3) @ R
    return np.ascontiguousarray(np.broadcast_to(c, d.shape), np.float32), np.ascontiguousarray(d, np.float32)


def synthetic_scene(n_input=2, n_target=64, image_size=256, latent=32, feat_ch=256, render_hw=128, seed=0, radius=5.0):
    """dict of CPU tensors with the field names of distillation.SceneCache"""
    rng = np.random.default_rng(seed)
    cams = circle_cameras(n_target, radius=radius)
    yy, xx = np.mgrid[0:image_size, 0:image_size]
    disc = (((yy - image_size / 2) ** 2 + (xx - image_size / 2) ** 2) < (0.35 * image_size) ** 2).astype(np.float32)

    def rays(idx):
        o, d = zip(*[camera_rays(cams[i], render_hw, render_hw) for i in idx])
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


def toy_scene(k: int, n_views: int = 12) -> dict:
    """scene k of a synthetic toy dataset in the reference's layout (utils/co3d_toy_dataloader.py): ``n_views`` pytorch3d cameras on a
    ``circle_cameras`` ring (radius and elevation vary with k) looking at a lit disc, R [N,3,3], T [N,3], f [N,2], c [N,2], image_size,
    images [N,3,256,256], masks and valid_region [N,1,256,256]"""
    g = torch.Generator().manual_seed(100 + k)
    R, T = [], []
    for c, rows in circle_cameras(n_views, radius=4.0 + 0.5 * k, elevation_deg=10.0 + 5 * k):
        r = torch.from_numpy(rows).T.contiguous()          # x_view = x_world R + T: R's columns are the camera axes
        R.append(r)
        T.append(-torch.from_numpy(c) @ r)
    yy, xx = torch.meshgrid(torch.arange(256.0), torch.arange(256.0), indexing='ij')
    disc = (((yy - 128) ** 2 + (xx - 128) ** 2) < (70 + 5 * k) ** 2).float()
    images = (torch.rand(n_views, 3, 1, 1, generator=g) * 0.8 + 0.2) * disc
    return dict(R=torch.stack(R), T=torch.stack(T), f=torch.full((n_views, 2), 3.0), c=torch.zeros(n_views, 2),
                image_size=torch.full((n_views, 2), 256.0), images=images, masks=disc.expand(n_views, 1, 256, 256).clone(),
                valid_region=torch.ones(n_views, 1, 256, 256))


def write_demo_inputs(d: str, cat: str = 'hydrant', n_scenes: int = 2, n_views: int = 12, seed: int = 0) -> dict:
    """what ``python -m sparsefusion_b200.demo`` reads, with random weights: ``{d}/data/{cat}/{cat}_toy.pt`` (``toy_scene`` 0..n_scenes-1),
    the EFT, VLDM and SD-VAE checkpoints of the released configuration in the released files' layouts, and LPIPS-VGG weights.  Returns
    the paths (root, eft, vldm, vae, lpips) and the LPIPS state dict (lpips_sd)."""
    import os
    from . import demo
    from .eft import EpipolarFeatureTransformer
    from .imagen_pytorch import Unet
    from .ldm_autoencoder import AutoencoderKL
    from .lpips_vgg import PerceptualLoss
    from .vldm import DDPM
    os.makedirs(f'{d}/data/{cat}', exist_ok=True)
    torch.save({cat: [toy_scene(k, n_views) for k in range(n_scenes)]}, f'{d}/data/{cat}/{cat}_toy.pt')
    torch.manual_seed(seed)
    eft = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=False)
    torch.save({'model_state_dict': eft.state_dict()}, f'{d}/eft.pt')
    vldm = DDPM(unets=(Unet(**demo.UNET_KW),), **demo.DDPM_KW)
    torch.save({'model_state_dict': vldm.state_dict()}, f'{d}/vldm.pt')
    del vldm
    vae = AutoencoderKL(**demo.VAE_KW)
    torch.save({'state_dict': {f'first_stage_model.{k}': v for k, v in vae.state_dict().items()}}, f'{d}/vae.ckpt')
    lp = PerceptualLoss('vgg', seed=seed + 11).state_dict()
    torch.save(lp, f'{d}/lpips.pt')
    return dict(root=f'{d}/data', eft=f'{d}/eft.pt', vldm=f'{d}/vldm.pt', vae=f'{d}/vae.ckpt', lpips=f'{d}/lpips.pt', lpips_sd=lp)
