"""Mesh extraction from a density lattice on the GPU (include/sparsefusion_b200.h section 9) and its albedo texture (section 12): what
NeRFRenderer.export_mesh strings together.

    python -m sparsefusion_b200.mesh CKPT OUT_DIR [--resolution R] [--texture-size T]

loads a checkpoint saved by ``distillation_loop`` (``{'model_state_dict': ...}``) into ``NeRFNetwork(get_default_torch_ngp_opt())`` on
cuda:0 and writes ``OUT_DIR/mcubes_mesh.obj`` (the file the reference's ``export_mesh`` writes, vertices in lattice index units); with
``--texture-size T`` also ``mesh.obj`` (world units, with UVs), ``mesh.mtl`` and the T x T ``albedo.png``.

Every function takes CUDA tensors; CPU tensors raise RuntimeError (there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import math
import os
import sys

import numpy as np
import torch

from . import _lib as lib

STATS_WORK = 1024       # SFB_VOLUME_STATS_WORK: doubles of scratch for sfb_volume_mean_std
MAX_AXIS = 1024         # SFB_MC_MAX_AXIS: lattice points per axis accepted by marching cubes
TEXTURE_MIN, TEXTURE_MAX, TEXTURE_MIN_CELL = 16, 8192, 4      # SFB_TEXTURE_MIN / _MAX / _MIN_CELL: texture sizes and atlas cell size


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


def _atlas_cell(F: int, T: int) -> int:
    if not isinstance(T, (int, np.integer)) or not TEXTURE_MIN <= T <= TEXTURE_MAX:
        raise ValueError(f'texture_size must be an integer in {TEXTURE_MIN}..{TEXTURE_MAX} (got {T!r})')
    c = lib.load().sfb_mesh_atlas_cell(int(F), int(T))
    if c == 0:
        n = max(1, math.isqrt(max(0, (F + 1) // 2 - 1)) + 1) if F > 0 else 1
        raise ValueError(f'a {T} x {T} texture is too small for {F} triangles (cells of {T // n} < {TEXTURE_MIN_CELL} texels): '
                         f'texture_size >= {max(TEXTURE_MIN, TEXTURE_MIN_CELL * n)} is needed')
    return c


def _cuda_device(device) -> torch.device:
    dev = torch.device(device) if device is not None else (torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else None)
    if dev is None or dev.type != 'cuda':
        raise RuntimeError('the texture atlas is built on a CUDA device (no CPU fallback)')
    return dev


def uv_atlas(F: int, T: int, device=None) -> torch.Tensor:
    """[F, 3, 2] float32 UV corners (x = column, y = row from the top) in texel units of a T x T texture, corners in tris[t, 0..2] order
    (header section 12): triangles 2k and 2k+1 share square cell k.  ValueError when T is outside 16..8192 or the cells would be smaller
    than 4 texels."""
    F = int(F)
    _atlas_cell(F, T)
    dev = _cuda_device(device)
    with torch.cuda.device(dev):
        uv = torch.empty(F, 3, 2, device=dev)
        lib.call('sfb_mesh_uv_atlas', F, int(T), uv.data_ptr() if F else None, lib.stream())
    return uv


def bake_albedo(net, verts_world: torch.Tensor, tris: torch.Tensor, texture_size: int, rows: int = None):
    """Albedo texture of the mesh (verts_world [V,3] float32 in world units, tris [F,3] int32, CUDA tensors) for the field ``net`` (a
    NeRFNetwork): (uv [F,3,2] float32 texel units, texture [T,T,3] uint8, owner [T,T] int32, -1 = no triangle) on the parameters' device.
    Each owned texel takes the point of its triangle closest, in the atlas, to the texel centre, and stores trunc(255 albedo) of the field
    there; the rest are black (header section 12).  The field is queried in slabs of ``rows`` texel rows (default: 2^21 texels per slab),
    so point memory stays near 64 MB whatever T is.  Repeated calls give identical bytes."""
    T = texture_size
    for name, t, dt in (('verts_world', verts_world, torch.float32), ('tris', tris, torch.int32)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f'bake_albedo: {name} must be a CUDA tensor (no CPU fallback)')
        if t.dim() != 2 or t.shape[1] != 3 or t.dtype != dt:
            raise RuntimeError(f'bake_albedo: {name} must be a [N, 3] {dt} tensor (got {tuple(t.shape)} {t.dtype})')
    emb, w0, b0, w1, b1, w2, b2 = net._field_params()
    dev = emb.device
    if dev.type != 'cuda' or verts_world.device != dev or tris.device != dev:
        raise RuntimeError('bake_albedo needs the network, verts and tris on one CUDA device (no CPU fallback)')
    F = tris.shape[0]
    c = _atlas_cell(F, T)
    verts, tris = verts_world.contiguous(), tris.contiguous()
    if F and (int(tris.min()) < 0 or int(tris.max()) >= verts.shape[0]):
        raise ValueError(f'bake_albedo: triangle index out of range 0..{verts.shape[0] - 1}')
    rows = max(1, (1 << 21) // T) if rows is None else int(rows)
    if rows < 1:
        raise ValueError(f'bake_albedo: rows must be >= 1 (got {rows})')
    rows = min(rows, T)
    enc = net.encoder
    geo = (float(np.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound))
    f = lib.fptr
    with torch.cuda.device(dev):
        uv = uv_atlas(F, T, dev)
        texture = torch.empty(T, T, 3, dtype=torch.uint8, device=dev)
        owner = torch.empty(T, T, dtype=torch.int32, device=dev)
        xyz = torch.empty(rows * T, 3, device=dev)
        sigma = torch.empty(rows * T, device=dev)
        rgb = torch.empty(rows * T, 3, device=dev)
        st = lib.stream()
        vp, tp = (f(verts), lib.iptr(tris)) if F else (None, None)
        for y0 in range(0, T, rows):
            h = min(rows, T - y0)
            own = owner[y0:y0 + h]
            lib.call('sfb_mesh_texel_points', vp, tp, F, T, y0, h, own.data_ptr(), xyz.data_ptr(), st)
            lib.call('sfb_ngp_field_forward', xyz.data_ptr(), None, None, None, 0, h * T, f(emb), lib.iptr(enc.offsets), *geo, f(w0), f(b0),
                     f(w1), f(b1), f(w2), f(b2), sigma.data_ptr(), rgb.data_ptr(), st)
            lib.call('sfb_mesh_texture_pack', own.data_ptr(), rgb.data_ptr(), h * T, texture[y0:y0 + h].data_ptr(), st)
    return uv, texture, owner


MTL = ('newmtl mat0\nKa 1.000000 1.000000 1.000000\nKd 1.000000 1.000000 1.000000\nKs 0.000000 0.000000 0.000000\nd 1.000000\nillum 1\n'
       'Ns 0.000000\nmap_Kd albedo.png\n')


def write_textured_obj(dir: str, verts, tris, uv, texture) -> None:
    """``dir/mesh.obj``, ``dir/mesh.mtl`` and ``dir/albedo.png`` (the reference's textured export names).  mesh.obj: `mtllib mesh.mtl`,
    `v x y z` lines, then (F > 0) one `vt u v` line per triangle corner, u = x / T, v = 1 - y / T (6 decimals), `usemtl mat0` and
    `f a/at b/bt c/ct` lines with 1-based indices.  mesh.mtl: the reference's material with `d 1.000000` (opaque) in place of its
    `Tr 1.000000`, which several loaders read as full transparency.  albedo.png: texture [T,T,3] uint8, row 0 at the top (y = 0)."""
    from PIL import Image
    v = (verts.detach().cpu().numpy() if isinstance(verts, torch.Tensor) else np.asarray(verts)).reshape(-1, 3)
    t = (tris.detach().cpu().numpy() if isinstance(tris, torch.Tensor) else np.asarray(tris)).reshape(-1, 3).astype(np.int64)
    q = (uv.detach().cpu().numpy() if isinstance(uv, torch.Tensor) else np.asarray(uv)).reshape(-1, 2).astype(np.float64)
    img = texture.detach().cpu().numpy() if isinstance(texture, torch.Tensor) else np.asarray(texture)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or img.shape[0] != img.shape[1]:
        raise ValueError(f'write_textured_obj: texture must be [T, T, 3] uint8 (got {img.shape} {img.dtype})')
    T = img.shape[0]
    if len(q) != 3 * len(t):
        raise ValueError(f'write_textured_obj: uv has {len(q)} corners for {len(t)} triangles')
    if not np.isfinite(v).all() or not np.isfinite(q).all():
        raise ValueError('write_textured_obj: vertices and uv must be finite')
    if t.size and (t.min() < 0 or t.max() >= len(v)):
        raise ValueError('write_textured_obj: triangle index out of range')
    with open(os.path.join(dir, 'mesh.obj'), 'wb') as fh:
        fh.write(b'mtllib mesh.mtl\n')
        if len(v):
            fh.write(_obj_block(b'v ', [_float_col(v[:, c]) for c in range(3)]))
        if len(t):
            fh.write(_obj_block(b'vt ', [_float_col(q[:, 0] / T), _float_col(1.0 - q[:, 1] / T)]))
            fh.write(b'usemtl mat0\n')
            slash = np.full((len(t), 1), ord('/'), dtype=np.uint8)
            vt = np.arange(1, 3 * len(t) + 1, dtype=np.int64).reshape(-1, 3)
            # _digits pads every column to its widest value; the padding (0 bytes) is dropped by _obj_block
            fh.write(_obj_block(b'f ', [np.concatenate([_digits(t[:, c] + 1, 0), slash, _digits(vt[:, c], 0)], axis=1) for c in range(3)]))
    with open(os.path.join(dir, 'mesh.mtl'), 'w') as fh:
        fh.write(MTL)
    Image.fromarray(np.ascontiguousarray(img), 'RGB').save(os.path.join(dir, 'albedo.png'))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog='python -m sparsefusion_b200.mesh', description='marching-cubes mesh of a distilled NeRF checkpoint')
    ap.add_argument('ckpt', help="checkpoint saved by distillation_loop ({'model_state_dict': ...})")
    ap.add_argument('out_dir', help='directory for mcubes_mesh.obj (created if missing)')
    ap.add_argument('--resolution', type=int, default=128, help='lattice points per axis (default 128, as the reference)')
    ap.add_argument('--texture-size', type=int, default=None, metavar='T',
                    help=f'also write mesh.obj, mesh.mtl and a T x T albedo.png ({TEXTURE_MIN}..{TEXTURE_MAX}; default: no texture)')
    a = ap.parse_args(argv)
    if not os.path.isfile(a.ckpt):
        ap.error(f'checkpoint not found: {a.ckpt}')
    if not 2 <= a.resolution <= MAX_AXIS:
        ap.error(f'--resolution must be in 2..{MAX_AXIS} (got {a.resolution})')
    if a.texture_size is not None and not TEXTURE_MIN <= a.texture_size <= TEXTURE_MAX:
        ap.error(f'--texture-size must be in {TEXTURE_MIN}..{TEXTURE_MAX} (got {a.texture_size})')
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
    verts, tris = net.export_mesh(a.out_dir, grid_resolution=a.resolution, texture_size=a.texture_size)
    print(f'{os.path.join(a.out_dir, "mcubes_mesh.obj")}: {verts.shape[0]} vertices, {tris.shape[0]} triangles ({a.resolution}^3 lattice)')
    if a.texture_size is not None:
        print(f'{os.path.join(a.out_dir, "mesh.obj")}: textured by a {a.texture_size}^2 albedo.png')
    return 0


if __name__ == '__main__':
    sys.exit(main())
