"""Mesh extraction from a density lattice on the GPU (include/sparsefusion_b200.h section 9): what NeRFRenderer.export_mesh strings together.

    python -m sparsefusion_b200.mesh CKPT OUT_DIR [--resolution R]

loads a checkpoint saved by ``distillation_loop`` (``{'model_state_dict': ...}``) into ``NeRFNetwork(get_default_torch_ngp_opt())`` on
cuda:0 and writes ``OUT_DIR/mcubes_mesh.obj`` (the file the reference's ``export_mesh`` writes, vertices in lattice index units).

Every function takes CUDA tensors; CPU tensors raise RuntimeError (there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

from . import _lib as lib

STATS_WORK = 1024       # SFB_VOLUME_STATS_WORK: doubles of scratch for sfb_volume_mean_std
MAX_AXIS = 1024         # SFB_MC_MAX_AXIS: lattice points per axis accepted by marching cubes


def _volume(volume: torch.Tensor, name: str = 'volume') -> torch.Tensor:
    if not isinstance(volume, torch.Tensor) or not volume.is_cuda:
        raise RuntimeError(f'{name} must be a CUDA tensor (no CPU fallback)')
    if volume.dim() != 3 or volume.dtype != torch.float32:
        raise RuntimeError(f'{name} must be a [X, Y, Z] float32 tensor (got {tuple(volume.shape)} {volume.dtype})')
    return volume.contiguous()


def smooth_gaussian(volume: torch.Tensor, sigma: float = 1.5) -> torch.Tensor:
    """scipy.ndimage.gaussian_filter(volume, sigma) in fp32: radius int(4 sigma + 0.5), mode 'reflect'.  PyMCubes' smooth_gaussian filters
    ``volume - 0.5`` in float64; that constant offset moves the mean and not the std, so the isosurface at mean + 0.25 std is the same
    and it is not reproduced here (the smoothed volume differs from PyMCubes' by it)."""
    v = _volume(volume)
    with torch.cuda.device(v.device):
        out, tmp = torch.empty_like(v), torch.empty_like(v)
        lib.call('sfb_gaussian_filter3d', lib.fptr(v), lib.fptr(out), lib.fptr(tmp), *v.shape, float(sigma), lib.stream())
    return out


def volume_mean_std(volume: torch.Tensor):
    """(mean, std) of every value (population std, ddof = 0, as numpy computes it), accumulated in fp64; one device sync"""
    v = _volume(volume)
    with torch.cuda.device(v.device):
        out = torch.empty(2, dtype=torch.float64, device=v.device)
        work = torch.empty(STATS_WORK, dtype=torch.float64, device=v.device)
        lib.call('sfb_volume_mean_std', lib.fptr(v), v.numel(), out.data_ptr(), work.data_ptr(), lib.stream())
        mean, std = out.tolist()
    return mean, std


def marching_cubes(volume: torch.Tensor, isovalue: float):
    """(verts [V,3] float32, tris [F,3] int32) CUDA tensors in index units (axis order of the volume).  A corner is inside the surface's
    lower side when v <= isovalue; each face's normal points toward decreasing value (outward for a density).  Vertices are shared between
    faces and the order is fixed by the volume (header section 9), so repeated calls give identical tensors.  Syncs once to read V and F."""
    v = _volume(volume)
    X, Y, Z = v.shape
    dev = v.device
    with torch.cuda.device(dev):
        nbytes = lib.load().sfb_marching_cubes_scratch_bytes(X, Y, Z)
        if nbytes == 0:
            raise RuntimeError(f'marching_cubes: lattice {X} x {Y} x {Z} is outside 1..{MAX_AXIS} points per axis')
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        iso = float(np.float32(isovalue))
        lib.call('sfb_marching_cubes_count', lib.fptr(v), X, Y, Z, iso, scratch.data_ptr(), counts.data_ptr(), lib.stream())
        nv, nf = counts.tolist()
        if nv >= 2 ** 31:
            raise RuntimeError(f'marching_cubes: {nv} vertices do not fit int32 triangle indices')
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        tris = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        lib.call('sfb_marching_cubes_emit', lib.fptr(v), X, Y, Z, iso, scratch.data_ptr(), verts.data_ptr() if nv else None,
                 tris.data_ptr() if nf else None, lib.stream())
    return verts, tris


def density_lattice(net, resolution: int = 128, S: int = 128) -> torch.Tensor:
    """sigma of the field ``net`` (a NeRFNetwork) on the lattice torch.linspace(-bound, bound, R) per axis, indexing 'ij' -> [R, R, R] on
    the parameters' device.  The field is queried in slabs of S x-planes, so point memory stays at S R^2 x 12 bytes."""
    R, S = int(resolution), int(S)
    if not 2 <= R <= MAX_AXIS or S < 1:
        raise ValueError(f'the lattice needs 2..{MAX_AXIS} points per axis and S >= 1 (got {R}, {S})')
    emb, w0, b0, w1, b1, w2, b2 = net._field_params()
    dev = emb.device
    if dev.type != 'cuda':
        raise RuntimeError('export_mesh needs the network on a CUDA device (no CPU fallback)')
    enc = net.encoder
    geo = (float(np.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound))
    f = lib.fptr
    with torch.cuda.device(dev):
        lin = torch.linspace(-net.bound, net.bound, R).to(dev)          # on the CPU in fp32 as the reference builds it, then moved
        sigma = torch.empty(R, R, R, device=dev)
        for x0 in range(0, R, S):
            xs = lin[x0:x0 + S]
            xx, yy, zz = torch.meshgrid(xs, lin, lin, indexing='ij')
            pts = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], dim=-1).contiguous()
            lib.call('sfb_ngp_field_forward', f(pts), None, None, None, 0, pts.shape[0], f(emb), lib.iptr(enc.offsets), *geo, f(w0), f(b0),
                     f(w1), f(b1), f(w2), f(b2), f(sigma[x0:x0 + S]), None, lib.stream())
    return sigma


def _digits(a: np.ndarray, pad: int) -> np.ndarray:
    """[n] non-negative int64 -> [n, width] ASCII digits, leading zeros replaced by `pad` (the last digit is always kept)"""
    width = max(1, len(str(int(a.max())))) if a.size else 1
    p = 10 ** np.arange(width - 1, -1, -1, dtype=np.int64)
    d = (a[:, None] // p) % 10
    out = (d + ord('0')).astype(np.uint8)
    lead = np.cumsum(d != 0, axis=1) == 0
    lead[:, -1] = False
    out[lead] = pad
    return out


def _obj_block(tag: bytes, cols) -> bytes:
    """rows of `tag c0 c1 c2\\n`, each column given as a [n, w] uint8 byte block in which 0 marks padding; padding is dropped"""
    n = cols[0].shape[0]
    parts = [np.frombuffer(tag, dtype=np.uint8)[None].repeat(n, 0)]
    for i, c in enumerate(cols):
        parts.append(c)
        parts.append(np.full((n, 1), ord(' ') if i < len(cols) - 1 else ord('\n'), dtype=np.uint8))
    buf = np.concatenate(parts, axis=1).reshape(-1)
    return buf[buf != 0].tobytes()


def _float_col(x: np.ndarray, decimals: int = 6) -> np.ndarray:
    q = np.rint(np.abs(x.astype(np.float64)) * 10 ** decimals).astype(np.int64)
    sign = np.where((x < 0) & (q > 0), ord('-'), 0).astype(np.uint8)[:, None]
    ip = _digits(q // 10 ** decimals, 0)
    fp = _digits(q % 10 ** decimals + 10 ** decimals, 0)[:, 1:]        # zero-padded fraction: 1ffffff without its leading 1
    return np.concatenate([sign, ip, np.full((len(x), 1), ord('.'), dtype=np.uint8), fp], axis=1)


def write_obj(path: str, verts, tris) -> None:
    """OBJ in mcubes.export_obj's layout: `v x y z` lines (6 decimals), then `f a b c` lines with 1-based indices.  Formatted with numpy
    array operations (no per-vertex Python loop): a 512^3 lattice gives meshes of millions of vertices."""
    v = (verts.detach().cpu().numpy() if isinstance(verts, torch.Tensor) else np.asarray(verts)).reshape(-1, 3)
    t = (tris.detach().cpu().numpy() if isinstance(tris, torch.Tensor) else np.asarray(tris)).reshape(-1, 3).astype(np.int64)
    if not np.isfinite(v).all():
        raise ValueError('write_obj: vertices must be finite')
    if t.size and (t.min() < 0 or t.max() >= len(v)):
        raise ValueError('write_obj: triangle index out of range')
    with open(path, 'wb') as fh:
        if len(v):
            fh.write(_obj_block(b'v ', [_float_col(v[:, c]) for c in range(3)]))
        if len(t):
            fh.write(_obj_block(b'f ', [_digits(t[:, c] + 1, 0) for c in range(3)]))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog='python -m sparsefusion_b200.mesh', description='marching-cubes mesh of a distilled NeRF checkpoint')
    ap.add_argument('ckpt', help="checkpoint saved by distillation_loop ({'model_state_dict': ...})")
    ap.add_argument('out_dir', help='directory for mcubes_mesh.obj (created if missing)')
    ap.add_argument('--resolution', type=int, default=128, help='lattice points per axis (default 128, as the reference)')
    a = ap.parse_args(argv)
    if not os.path.isfile(a.ckpt):
        ap.error(f'checkpoint not found: {a.ckpt}')
    if not 2 <= a.resolution <= MAX_AXIS:
        ap.error(f'--resolution must be in 2..{MAX_AXIS} (got {a.resolution})')
    if not torch.cuda.is_available():
        raise RuntimeError('mesh export runs on the GPU: no CUDA device is available')
    from .network_grid import NeRFNetwork, get_default_torch_ngp_opt
    ck = torch.load(a.ckpt, map_location='cpu')
    if not isinstance(ck, dict) or 'model_state_dict' not in ck:
        ap.error(f"{a.ckpt} has no 'model_state_dict' (expected a checkpoint saved by distillation_loop)")
    sd = ck['model_state_dict']
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = 'density_grid' in sd
    net = NeRFNetwork(opt)
    net.load_state_dict(sd)
    net = net.to('cuda:0').eval()
    os.makedirs(a.out_dir, exist_ok=True)
    verts, tris = net.export_mesh(a.out_dir, grid_resolution=a.resolution)
    print(f'{os.path.join(a.out_dir, "mcubes_mesh.obj")}: {verts.shape[0]} vertices, {tris.shape[0]} triangles ({a.resolution}^3 lattice)')
    return 0


if __name__ == '__main__':
    sys.exit(main())
