"""Ray generation and the image-space glue of a distillation step as fused kernels (SURVEY.md §8f row 2; C ABI section 6).

The reference does these with ~50 eager launches per sub-step plus their autograd backward (sparsefusion/distillation.py:201-241, :274-288,
:307-344; utils/common_utils.py:183-190; utils/render_utils.py:40-47).  Here a sub-step's loss is one kernel that returns the value together
with d loss / d image and d loss / d weights_sum; `Distiller` feeds those two gradients straight into the render's backward.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import _lib as lib


def rays_from_camera(center: torch.Tensor, rot: torch.Tensor, height: int, width: int, focal_ndc: float = 4.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """(rays_o, rays_d) [H*W, 3] of the pixel-centre NDC grid; rot rows = (right, up, forward); directions un-normalised (plane at depth 1)"""
    cam = torch.cat((center.reshape(3), rot.reshape(9))).float().contiguous()
    assert cam.is_cuda
    o = torch.empty(height * width, 3, dtype=torch.float32, device=cam.device)
    d = torch.empty_like(o)
    lib.call('sfb_rays_from_camera', lib.fptr(cam), height, width, float(focal_ndc), lib.fptr(o), lib.fptr(d), lib.stream())
    return o, d


def _combine(sums: torch.Tensor, n: int, lc: float, ls: float, lo: float, colour_scale: float = 1.0) -> torch.Tensor:
    return colour_scale * lc * sums[0] / (3.0 * n) + ls * sums[1] / n + lo * sums[2] / n


def _check_entropy(lambda_entropy) -> float:
    le = float(lambda_entropy)
    if not le >= 0.0:
        raise ValueError(f'lambda_entropy must be >= 0 (got {lambda_entropy!r})')
    return le


def _terms(loss: torch.Tensor, data: torch.Tensor, sums: torch.Tensor, n: int, lo: float, le: float) -> torch.Tensor:
    """[4] device tensor (loss, lo * opacity, le * entropy, data term): the sub-step's weighted terms in the reference's logging units
    (distillation.py:254-256, :349), from the kernel's sums; the entropy entry is 0 when the sums hold no entropy"""
    ent = le * sums[3] / n if le > 0.0 else torch.zeros_like(loss)
    return torch.stack((loss, lo * sums[2] / n, ent, data))


def photometric_loss(img: torch.Tensor, sil: torch.Tensor, rgb: torch.Tensor, mask: torch.Tensor, h: int, w: int, scale: int,
                     lambda_color: float, lambda_sil: float, lambda_opacity: float, *, lambda_entropy: float = 0.0, return_terms: bool = False):
    """distillation.py:210-241.  img [h*w,3], sil [h*w] (detached render outputs); rgb [3,H,W], mask [1,H,W] of the input view, H = h*scale.
    Returns (loss, d loss/d img, d loss/d sil), and with ``return_terms`` a fourth entry: the [4] device tensor (loss, lambda_opacity *
    opacity, lambda_entropy * entropy, lambda_color * colour + lambda_sil * silhouette) -- the first three are what the reference logs
    (:254-256).  ``lambda_entropy`` > 0 adds the entropy regulariser (:236-241) through ``sfb_photometric_loss_ent``; at 0 the kernel is
    ``sfb_photometric_loss``, the same launch as without it."""
    assert img.shape == (h * w, 3) and sil.numel() == h * w and rgb.shape[-2:] == (h * scale, w * scale)
    le = _check_entropy(lambda_entropy)
    sums = torch.empty(4 if le > 0.0 else 3, dtype=torch.float32, device=img.device)
    g_img, g_sil = torch.empty_like(img), torch.empty(h * w, dtype=torch.float32, device=img.device)
    rgb, mask = rgb.contiguous(), mask.contiguous()     # bound to names: a temporary would be freed (and its block reused) before the launch
    if le > 0.0:
        lib.call('sfb_photometric_loss_ent', lib.fptr(img), lib.fptr(sil), lib.fptr(rgb), lib.fptr(mask), h, w, scale, float(lambda_color),
                 float(lambda_sil), float(lambda_opacity), le, lib.fptr(sums), lib.fptr(g_img), lib.fptr(g_sil), lib.stream())
    else:
        lib.call('sfb_photometric_loss', lib.fptr(img), lib.fptr(sil), lib.fptr(rgb), lib.fptr(mask), h, w, scale,
                 float(lambda_color), float(lambda_sil), float(lambda_opacity), lib.fptr(sums), lib.fptr(g_img), lib.fptr(g_sil), lib.stream())
    n = h * w
    loss = _combine(sums, n, lambda_color, lambda_sil, lambda_opacity)
    if le > 0.0:
        loss = loss + le * sums[3] / n
    if not return_terms:
        return loss, g_img, g_sil
    data = lambda_color * sums[0] / (3.0 * n) + lambda_sil * sums[1] / n
    return loss, g_img, g_sil, _terms(loss, data, sums, n, lambda_opacity, le)


def upsample2x_render(img: torch.Tensor, sil: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """[4, 2h, 2w]: bilinear x2 (align_corners False) of the rendered colours (planes 0..2) and opacity (plane 3), distillation.py:287-288"""
    up = torch.empty(4, 2 * h, 2 * w, dtype=torch.float32, device=img.device)
    lib.call('sfb_upsample2x_render', lib.fptr(img), lib.fptr(sil), h, w, lib.fptr(up), lib.stream())
    return up


def fusion_loss(up: torch.Tensor, target: torch.Tensor, h: int, w: int, mode: str, weight: float, lambda_color: float, lambda_sil: float,
                lambda_opacity: float, g_extra: torch.Tensor = None, *, lambda_entropy: float = 0.0, return_terms: bool = False):
    """distillation.py:310 ('sds': weight * L1 to the decoded image) / :316-329 ('eft': huber to the cached EFT image and its mask), plus the
    opacity term (:336-344) and, with ``lambda_entropy`` > 0, the entropy term over the up-sampled silhouette (:338-344, through
    ``sfb_fusion_loss_ent``).  up = upsample2x_render(...); target [3,2h,2w].  Returns (loss, d loss/d img [h*w,3], d loss/d sil [h*w]), and
    with ``return_terms`` a fourth entry: the [4] device tensor (loss, lambda_opacity * opacity, lambda_entropy * entropy, fusion term) whose
    last entry is the reference's logged ``fusion_loss`` (:349) before the perceptual term, without opacity and entropy."""
    H, W = 2 * h, 2 * w
    assert up.shape == (4, H, W) and target.shape[-3:] == (3, H, W)
    le = _check_entropy(lambda_entropy)
    sums = torch.empty(4 if le > 0.0 else 3, dtype=torch.float32, device=up.device)
    g_up = torch.empty_like(up)
    g_img, g_sil = torch.empty(h * w, 3, dtype=torch.float32, device=up.device), torch.empty(h * w, dtype=torch.float32, device=up.device)
    m = {'sds': 0, 'eft': 1}[mode]
    # g_extra [3,2h,2w]: gradient of further terms w.r.t. the up-sampled colour planes (the perceptual term), joined before the bilinear adjoint
    assert g_extra is None or tuple(g_extra.shape) == (3, H, W)
    target = target.contiguous()                         # named: temporaries would be freed before the launch and may alias each other
    g_extra = None if g_extra is None else g_extra.contiguous()
    if le > 0.0:
        lib.call('sfb_fusion_loss_ent', lib.fptr(up), lib.fptr(target), H, W, m, float(weight), float(lambda_color), float(lambda_sil),
                 float(lambda_opacity), le, None if g_extra is None else lib.fptr(g_extra), lib.fptr(sums), lib.fptr(g_up), h, w, lib.fptr(g_img),
                 lib.fptr(g_sil), lib.stream())
    else:
        lib.call('sfb_fusion_loss_ex', lib.fptr(up), lib.fptr(target), H, W, m, float(weight), float(lambda_color), float(lambda_sil),
                 float(lambda_opacity), None if g_extra is None else lib.fptr(g_extra), lib.fptr(sums), lib.fptr(g_up), h, w, lib.fptr(g_img),
                 lib.fptr(g_sil), lib.stream())
    n = H * W
    if m == 0:
        loss = float(weight) * sums[0] / (3.0 * n) + lambda_opacity * sums[2] / n
    else:
        loss = _combine(sums, n, lambda_color, lambda_sil, lambda_opacity)
    if le > 0.0:
        loss = loss + le * sums[3] / n
    if not return_terms:
        return loss, g_img, g_sil
    if m == 0:
        data = float(weight) * sums[0] / (3.0 * n)
    else:
        data = lambda_color * sums[0] / (3.0 * n) + lambda_sil * sums[1] / n
    return loss, g_img, g_sil, _terms(loss, data, sums, n, lambda_opacity, le)
