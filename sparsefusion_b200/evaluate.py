"""Scores of a distilled scene on the GPU: what the reference's ``distillation_loop`` does after its iterations (sparsefusion/distillation.py:391-443).
Every scene view is rendered in eval mode at the rays' resolution and scored against the ground truth with PSNR, SSIM (scikit-image's
semantics, utils/common_utils.py:48-64; kernel in csrc/metrics.cu, header section 10) and LPIPS-VGG (``PerceptualLoss``, value only), and the
reference's ``{save_dir}/metrics/{seq_name}.txt`` is written.

The reference copies each render to the host for scikit-image and runs LPIPS on the CPU; here renders, SSIM / PSNR and LPIPS stay on the GPU.
Every function takes CUDA tensors; CPU tensors raise RuntimeError (there is no CPU fallback).
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib as lib
from .distillation import view_seed

EVAL_STREAM = 3      # view_seed stream of the evaluation renders' jitter
CIRCLE_STREAM = 4    # view_seed stream of the circle-path renders' jitter (video.py's fly-around gif)


@dataclass
class EvalViews:
    """the scene views a distilled scene is scored on (distillation.py:393-406), as device tensors"""
    rays_o: torch.Tensor    # [V, H*W, 3]  sampler_grid(scene_cameras_vox[ci]) origins, row-major pixels (:85, :400-402)
    rays_d: torch.Tensor    # [V, H*W, 3]
    rgb: torch.Tensor       # [V, 3, H, W] scene_rgb, the ground truth in [0, 1]
    mask: torch.Tensor      # [V, 1, H, W] scene_mask

    def to(self, device, non_blocking=False):
        return EvalViews(*[getattr(self, f).to(device, non_blocking=non_blocking) for f in self.__dataclass_fields__])


@dataclass
class SceneEval:
    """per-view scores (fp64) and the renders they were computed on"""
    psnr: torch.Tensor        # [V]
    ssim: torch.Tensor        # [V]  fp32 values, as scikit-image returns them for fp32 images
    lpips: torch.Tensor       # [V]  nan without a perceptual network
    image: torch.Tensor       # [V, H, W, 3]
    silhouette: torch.Tensor  # [V, H, W]  weights_sum


def image_metrics(pred: torch.Tensor, gt: torch.Tensor):
    """(ssim [B], psnr [B]) fp64 CUDA tensors of image pairs [B, H, W, 3] (or one pair [H, W, 3]) of float32 CUDA tensors:
    ``skimage.metrics.structural_similarity(pred, gt, channel_axis=-1, data_range=1)`` and ``peak_signal_noise_ratio(pred, gt, data_range=1)``
    as scikit-image computes them for float32 images (header section 10); PSNR is inf for identical images.  Images smaller than the 7x7
    window raise ValueError, as scikit-image does."""
    for name, t in (('pred', pred), ('gt', gt)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f'image_metrics: {name} must be a CUDA tensor (no CPU fallback)')
        if t.dtype != torch.float32:
            raise RuntimeError(f'image_metrics: {name} must be float32 (got {t.dtype})')
    if pred.shape != gt.shape or pred.dim() not in (3, 4) or pred.shape[-1] != 3:
        raise ValueError(f'image_metrics: pred and gt must both be [B, H, W, 3] or [H, W, 3] (got {tuple(pred.shape)} and {tuple(gt.shape)})')
    if pred.device != gt.device:
        raise RuntimeError(f'image_metrics: pred and gt are on different devices ({pred.device}, {gt.device})')
    a, b = (t.reshape(-1, *t.shape[-3:]).contiguous() for t in (pred, gt))
    B, H, W = a.shape[:3]
    n_work = lib.load().sfb_image_ssim_psnr_work(B, H, W)
    if n_work == 0:
        raise ValueError(f'image_metrics: images must be at least 7 x 7 (the SSIM window) in batches of 1..65535 (got {B} x {H} x {W})')
    with torch.cuda.device(a.device):
        out = torch.empty(B, 2, dtype=torch.float64, device=a.device)
        work = torch.empty(n_work, dtype=torch.float64, device=a.device)
        lib.call('sfb_image_ssim_psnr', lib.fptr(a), lib.fptr(b), B, H, W, out.data_ptr(), work.data_ptr(), lib.stream())
        psnr = 10.0 * torch.log10(1.0 / out[:, 1])
    return out[:, 0].clone(), psnr


@torch.no_grad()
def render_views(ngp, rays_o: torch.Tensor, rays_d: torch.Tensor, hw, opt, *, seed: int, stream: int):
    """(images [V, H, W, 3] fp32, silhouettes [V, H, W]) of V views (rays [V, H*W, 3], ``hw`` = (H, W)) with the reference's eval-mode render
    call (distillation.py:404-406, :480-482).  Its ``perturb=True`` jitter, which the reference draws from torch's unseeded global generator,
    comes from the CUDA generator seeded with ``view_seed(seed, 0, view, stream)`` inside ``torch.random.fork_rng``, so the renders are
    reproducible and the callers' generators are left as they were.  ``ngp.training`` is restored on return."""
    dev = rays_o.device
    if dev.type != 'cuda':
        raise RuntimeError('render_views: the rays must be CUDA tensors (no CPU fallback)')
    H, W = hw
    V, N = rays_o.shape[:2]
    if N != H * W or rays_d.shape != rays_o.shape:
        raise ValueError(f'render_views: rays {tuple(rays_o.shape)} / {tuple(rays_d.shape)} do not match {H} x {W} images')
    was_training = ngp.training
    ngp.eval()
    images, sils = [], []
    try:
        with torch.cuda.device(dev):
            for v in range(V):
                with torch.random.fork_rng(devices=[dev]):
                    torch.cuda.manual_seed(view_seed(seed, 0, v, stream))
                    out = ngp.render_batched(rays_o[v][None], rays_d[v][None], batched=True, perturb=True, bg_color=0, ambient_ratio=1.0,
                                             shading='albedo', force_all_rays=True, **vars(opt))
                images.append(out['image'].reshape(H, W, 3))
                sils.append(out['weights_sum'].reshape(H, W))
            return torch.stack(images).float(), torch.stack(sils)
    finally:
        ngp.train(was_training)


@torch.no_grad()
def evaluate_scene(ngp, views: EvalViews, opt, percep, *, seed: int) -> SceneEval:
    """scores of ``ngp`` on every view of ``views`` (distillation.py:393-433).  The renders are ``render_views`` with ``stream=3``: the
    reference's eval-mode render call, jitter from ``view_seed(seed, 0, view, 3)``, the callers' generators left as they were.  SSIM / PSNR:
    ``image_metrics`` over all views at once.  LPIPS: ``percep.value_and_grad(render, gt, normalize=True, want_grad=False)`` per view, which is the reference's ``loss_fn_vgg(gt * 2 - 1, pred * 2 - 1)`` (the distance is symmetric); nan when ``percep`` is None.
    ``ngp.training`` is restored on return."""
    dev = views.rays_o.device
    if dev.type != 'cuda':
        raise RuntimeError('evaluate_scene: the views must be CUDA tensors (no CPU fallback)')
    V, N = views.rays_o.shape[:2]
    H, W = views.rgb.shape[2:]
    if N != H * W or views.rgb.shape[:2] != (V, 3) or views.rays_d.shape != views.rays_o.shape:
        raise ValueError(f'evaluate_scene: rays {tuple(views.rays_o.shape)} / {tuple(views.rays_d.shape)} do not match images {tuple(views.rgb.shape)}')
    image, sil = render_views(ngp, views.rays_o, views.rays_d, (H, W), opt, seed=seed, stream=EVAL_STREAM)
    with torch.cuda.device(dev):
        gt = views.rgb.float().permute(0, 2, 3, 1).contiguous()
        ssim, psnr = image_metrics(image, gt)
        if percep is None:
            lp = torch.full((V,), float('nan'), dtype=torch.float64, device=dev)
        else:
            lp = torch.stack([percep.value_and_grad(image[v].permute(2, 0, 1), views.rgb[v].float(), normalize=True, want_grad=False)[0]
                              for v in range(V)]).double()
    return SceneEval(psnr=psnr, ssim=ssim, lpips=lp, image=image, silhouette=sil)


def _array(values) -> np.ndarray:
    if isinstance(values, torch.Tensor):
        values = values.detach().cpu().numpy()
    return np.array(values)


def write_metrics(path: str, ssim, psnr, lpips) -> None:
    """the reference's metrics file (distillation.py:437-441), byte for byte: each entry is ``str(np.array(values).mean())`` of the per-view
    values, so pass them as the reference holds them -- SSIM as float32 (scikit-image's type for float32 images), PSNR and LPIPS as float64.
    The warning line has no newline and LPIPS is labelled ``pip:``, as in the reference.  Creates the file's directory and prints the
    reference's ``psnr:`` / ``lpips:`` lines (:434-435)."""
    s, p, l = _array(ssim).mean(), _array(psnr).mean(), _array(lpips).mean()
    print('psnr:', p)
    print('lpips:', l)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, 'w') as fp:
        fp.write('warning: this metric is used for debugging only and not the final metric')
        fp.write('psnr:\n' + str(p) + '\n')
        fp.write('ssim:\n' + str(s) + '\n')
        fp.write('pip:\n' + str(l) + '\n')


def write_scene_metrics(path: str, scores: SceneEval) -> None:
    """``write_metrics`` of an ``evaluate_scene`` result, with each score in the type the reference's file is formatted from"""
    write_metrics(path, scores.ssim.cpu().numpy().astype(np.float32), scores.psnr.cpu().numpy(), scores.lpips.cpu().numpy())
