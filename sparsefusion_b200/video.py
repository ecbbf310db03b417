"""The distilled scene's pictures, as the reference's ``distillation_loop`` writes them (sparsefusion/distillation.py:129-141, :444-493): uint8
frames from fp32 panels, GIF palettes quantised on the GPU (csrc/palette.cu, header section 11), and GIF / JPEG files written with Pillow.

The reference hands RGB frames to imageio, which quantises every frame on the host (Pillow's adaptive palette: ~0.2 s per 256x1280 frame).
Here the palettes and index planes are computed on the GPU and copied to the host once; Pillow only packs the indexed frames into the GIF
container.  Every function takes CUDA tensors; CPU tensors raise RuntimeError (there is no CPU fallback).
"""
from __future__ import annotations

import os

import torch

from . import _lib as lib

GIF_DURATION_MS = 200     # imageio's duration=0.2 (seconds) of the reference's gif writers (:444, :489)


def require_pillow():
    """the Pillow ``Image`` module, or ImportError naming what needs it (call this before a long run, not after it)"""
    try:
        from PIL import Image
    except ImportError as e:
        raise ImportError('writing gifs and jpegs needs Pillow (the PIL package)') from e
    return Image


def _check_cuda(name, t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor (no CPU fallback)')


def to_uint8(*panels: torch.Tensor) -> torch.Tensor:
    """uint8 frames [B, H, sum W, 3] of fp32 panels [B, H, W, C] (C = 1 is repeated to 3) placed side by side: on [0, 1] exactly the
    reference's ``(np.hstack(panels) * 255).astype(np.uint8)`` (fp32 multiply, truncation); values outside [0, 1] are clamped first.
    Panels of different heights or batch sizes raise ValueError, as ``np.hstack`` fails on them."""
    if not panels:
        raise ValueError('to_uint8: no panels')
    for i, p in enumerate(panels):
        _check_cuda(f'to_uint8: panel {i}', p)
        if p.dim() != 4 or p.shape[-1] not in (1, 3):
            raise ValueError(f'to_uint8: panel {i} must be [B, H, W, 1 or 3] (got {tuple(p.shape)})')
        if p.shape[:2] != panels[0].shape[:2]:
            raise ValueError(f'to_uint8: panel {i} is {tuple(p.shape)}, panel 0 {tuple(panels[0].shape)}: panels need one batch size and height')
    x = torch.cat([p.float().expand(*p.shape[:3], 3) for p in panels], dim=2)
    return (x.clamp(0.0, 1.0) * 255.0).to(torch.uint8)


def _quantize(frames: torch.Tensor, colors: int):
    """(buffer, palette, ncolors, indices): the three outputs as views of ONE uint8 buffer, so that a single copy brings them to the host"""
    _check_cuda('quantize_palette: frames', frames)
    if frames.dtype != torch.uint8:
        raise RuntimeError(f'quantize_palette: frames must be uint8 (got {frames.dtype})')
    if frames.dim() != 4 or frames.shape[-1] != 3:
        raise ValueError(f'quantize_palette: frames must be [B, H, W, 3] (got {tuple(frames.shape)})')
    if not 2 <= int(colors) <= 256:
        raise ValueError(f'quantize_palette: colors must be in 2..256 (got {colors})')
    frames = frames.contiguous()
    B, H, W = frames.shape[:3]
    n_work = lib.load().sfb_palette_work_bytes(B, H, W)
    if n_work == 0:
        raise ValueError(f'quantize_palette: {B} frames of {H} x {W} are out of range (1..65535 frames of 1..16843009 pixels)')
    with torch.cuda.device(frames.device):
        n_pal, n_cnt = B * 256 * 3, B * 4
        buf = torch.empty(n_pal + n_cnt + B * H * W, dtype=torch.uint8, device=frames.device)
        work = torch.empty(n_work, dtype=torch.uint8, device=frames.device)
        palette, ncolors, indices = buf[:n_pal], buf[n_pal:n_pal + n_cnt], buf[n_pal + n_cnt:]
        lib.call('sfb_palette_quantize', frames.data_ptr(), B, H, W, int(colors), palette.data_ptr(), ncolors.data_ptr(), indices.data_ptr(),
                 work.data_ptr(), lib.stream())
    return buf, (B, H, W)


def _split(buf: torch.Tensor, B: int, H: int, W: int):
    n_pal, n_cnt = B * 256 * 3, B * 4
    return buf[:n_pal].view(B, 256, 3), buf[n_pal:n_pal + n_cnt].view(torch.int32), buf[n_pal + n_cnt:].view(B, H, W)


def quantize_palette(frames: torch.Tensor, colors: int = 256):
    """(palette [B, 256, 3] uint8, ncolors [B] int32, indices [B, H, W] uint8) of uint8 CUDA frames [B, H, W, 3]: each frame's median-cut
    palette of at most ``colors`` entries (zero beyond ``ncolors``) and every pixel's nearest entry (header section 11)"""
    buf, shape = _quantize(frames, colors)
    return _split(buf, *shape)


def write_gif(path: str, frames: torch.Tensor, duration_ms: int = GIF_DURATION_MS) -> None:
    """an animated GIF of uint8 CUDA frames [B, H, W, 3], as the reference's ``imageio.get_writer(path, mode='I', duration=0.2)`` writes it:
    ``duration_ms`` per frame, looping forever.  Palettes are quantised on the GPU and copied to the host with the index planes in one copy;
    Pillow stores the indexed frames.  Pillow merges identical consecutive frames into one of the summed duration."""
    Image = require_pillow()
    buf, (B, H, W) = _quantize(frames, 256)
    palette, ncolors, indices = _split(buf.cpu(), B, H, W)
    images = []
    for b in range(B):
        im = Image.frombytes('P', (W, H), indices[b].numpy().tobytes())
        im.putpalette(palette[b, :int(ncolors[b])].numpy().tobytes())
        images.append(im)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    images[0].save(path, save_all=True, append_images=images[1:], duration=int(duration_ms), loop=0)


def write_jpeg(path: str, frame: torch.Tensor) -> None:
    """a JPEG of one uint8 CUDA frame [H, W, 3] with Pillow's defaults (quality 75), which imageio's JPEG writer uses too"""
    write_jpegs([path], frame[None])


def write_jpegs(paths, frames: torch.Tensor) -> None:
    """one JPEG per uint8 CUDA frame of [B, H, W, 3] (one device-to-host copy for all of them)"""
    Image = require_pillow()
    _check_cuda('write_jpeg: frame', frames)
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3 or frames.shape[0] != len(paths):
        raise ValueError(f'write_jpeg: frames must be uint8 [B, H, W, 3] with one path each (got {frames.dtype} {tuple(frames.shape)}, '
                         f'{len(paths)} paths)')
    host = frames.cpu().numpy()
    for p, f in zip(paths, host):
        d = os.path.dirname(p)
        if d:
            os.makedirs(d, exist_ok=True)
        Image.fromarray(f).save(p)
