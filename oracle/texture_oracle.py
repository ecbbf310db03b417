"""Plain-numpy fp64 restatement of the mesh texture contract (include/sparsefusion_b200.h section 12, sparsefusion_b200/mesh.py), test-only.

* ``atlas_cell``, ``uv_atlas``: the cell layout and each triangle's UV corners in texel units.
* ``ownership``: owner [T, T] (-1 = none) from the integer rule of the header.
* ``texel_points``: barycentrics of the point of the owner's UV triangle closest to each texel centre, computed by the general
  closest-point-on-triangle test (Voronoi regions of the vertices and edges, Ericson, Real-Time Collision Detection 5.1.5), not by the
  leg-frame clamp the kernel uses, and the surface point they give.
* ``bilinear_taps``: texels a bilinear lookup weights nonzero at given texel-unit points.
* ``read_textured_obj``, ``read_mtl``: readers for mesh.obj (v, vt, f a/at b/bt c/ct) and mesh.mtl.
"""
from __future__ import annotations

import math

import numpy as np

M, D = 0.5, 2.0          # margin to the cell border and gap between the two hypotenuses, in texels
T_MIN, T_MAX, C_MIN = 16, 8192, 4


def atlas_cols(F):
    return max(1, math.isqrt(max(0, (F + 1) // 2 - 1)) + 1) if F > 0 else 1


def atlas_cell(F, T):
    """cell size c in texels; ValueError outside the limits"""
    if not T_MIN <= T <= T_MAX:
        raise ValueError(f'texture_size must be in {T_MIN}..{T_MAX} (got {T})')
    n = atlas_cols(F)
    c = T // n
    if c < C_MIN:
        raise ValueError(f'a {T} x {T} texture is too small for {F} triangles: texture_size >= {max(T_MIN, C_MIN * n)} is needed')
    return c


def uv_atlas(F, T):
    """[F, 3, 2] float64 UV corners (x, y) in texel units, corners in tris[t, 0..2] order"""
    c, n = atlas_cell(F, T), atlas_cols(F)
    t = np.arange(F)
    k = t // 2
    origin = np.stack([(k % n) * c, (k // n) * c], axis=1).astype(np.float64)
    lower = np.array([[M, M], [c - M - D, M], [M, c - M - D]])
    upper = np.array([[c - M, c - M], [M + D, c - M], [c - M, M + D]])
    local = np.where((t % 2 == 0)[:, None, None], lower[None], upper[None])
    return origin[:, None, :] + local


def ownership(F, T):
    """owner [T, T] int64 (row y, column x), -1 where no triangle owns the texel"""
    c, n = atlas_cell(F, T), atlas_cols(F)
    y, x = np.meshgrid(np.arange(T), np.arange(T), indexing='ij')
    cx, cy, i, j = x // c, y // c, x % c, y % c
    t = 2 * (cy * n + cx) + ((2 * i + 1) + (2 * j + 1) >= 2 * c)
    return np.where((cx < n) & (cy < n) & (t < F), t, -1)


def closest_barycentrics(p, a, b, c):
    """barycentrics [N, 3] of the point of triangle (a, b, c) closest to p; every argument [N, 2]"""
    p, a, b, c = (np.asarray(q, dtype=np.float64) for q in (p, a, b, c))
    ab, ac, ap = b - a, c - a, p - a
    dot = lambda u, v: (u * v).sum(-1)
    d1, d2 = dot(ab, ap), dot(ac, ap)
    bp = p - b
    d3, d4 = dot(ab, bp), dot(ac, bp)
    cp = p - c
    d5, d6 = dot(ab, cp), dot(ac, cp)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    with np.errstate(divide='ignore', invalid='ignore'):
        denom = va + vb + vc
        lam = np.stack([va / denom, vb / denom, vc / denom], axis=1)                              # interior
        w = d6 / (d6 - d5)
        lam = np.where(((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0))[:, None],                     # edge bc
                       np.stack([0 * w, 1 - (d4 - d3) / ((d4 - d3) + (d5 - d6)), (d4 - d3) / ((d4 - d3) + (d5 - d6))], 1), lam)
        lam = np.where(((vb <= 0) & (d2 >= 0) & (d6 <= 0))[:, None], np.stack([1 - d2 / (d2 - d6), 0 * w, d2 / (d2 - d6)], 1), lam)   # ac
        lam = np.where(((vc <= 0) & (d1 >= 0) & (d3 <= 0))[:, None], np.stack([1 - d1 / (d1 - d3), d1 / (d1 - d3), 0 * w], 1), lam)   # ab
    one = lambda q: np.broadcast_to(np.array(q, dtype=np.float64), lam.shape)
    lam = np.where(((d6 >= 0) & (d5 <= d6))[:, None], one([0, 0, 1]), lam)                        # vertex c
    lam = np.where(((d3 >= 0) & (d4 <= d3))[:, None], one([0, 1, 0]), lam)                        # vertex b
    lam = np.where(((d1 <= 0) & (d2 <= 0))[:, None], one([1, 0, 0]), lam)                         # vertex a
    return lam


def texel_points(verts, tris, T):
    """(owner [T, T] int64, lam [T, T, 3], xyz [T, T, 3]) in fp64; lam and xyz are 0 where there is no owner"""
    verts, tris = np.asarray(verts, dtype=np.float64).reshape(-1, 3), np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    F = len(tris)
    owner = ownership(F, T)
    lam = np.zeros((T, T, 3))
    xyz = np.zeros((T, T, 3))
    ys, xs = np.nonzero(owner >= 0)
    if len(ys):
        t = owner[ys, xs]
        uv = uv_atlas(F, T)[t]
        p = np.stack([xs + 0.5, ys + 0.5], axis=1)
        l = closest_barycentrics(p, uv[:, 0], uv[:, 1], uv[:, 2])
        lam[ys, xs] = l
        xyz[ys, xs] = np.einsum('ni,nic->nc', l, verts[tris[t]])
    return owner, lam, xyz


def bilinear_taps(p):
    """[N, 4, 2] integer texels (x, y) that a bilinear lookup at texel-unit points p [N, 2] reads: floor and ceil of p - 1/2 per axis
    (a tap of weight zero, at an exact texel centre, is not read)"""
    q = np.asarray(p, dtype=np.float64) - 0.5
    lo, hi = np.floor(q).astype(np.int64), np.ceil(q).astype(np.int64)
    return np.stack([np.stack([lo[:, 0], lo[:, 1]], 1), np.stack([hi[:, 0], lo[:, 1]], 1), np.stack([lo[:, 0], hi[:, 1]], 1),
                     np.stack([hi[:, 0], hi[:, 1]], 1)], axis=1)


def read_textured_obj(path):
    """(verts [V,3], vt [Tc,2], tris [F,3], tri_vt [F,3], lines) of a textured OBJ; indices zero-based, lines = its non-empty lines"""
    vs, vts, fs, fts, lines = [], [], [], [], []
    with open(path) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            lines.append(line.rstrip('\n'))
            if tok[0] == 'v':
                vs.append([float(t) for t in tok[1:4]])
            elif tok[0] == 'vt':
                vts.append([float(t) for t in tok[1:3]])
            elif tok[0] == 'f':
                pairs = [t.split('/') for t in tok[1:4]]
                fs.append([int(p[0]) - 1 for p in pairs])
                fts.append([int(p[1]) - 1 for p in pairs])
    return (np.array(vs, dtype=np.float64).reshape(-1, 3), np.array(vts, dtype=np.float64).reshape(-1, 2),
            np.array(fs, dtype=np.int64).reshape(-1, 3), np.array(fts, dtype=np.int64).reshape(-1, 3), lines)


def read_mtl(path):
    with open(path) as f:
        return [l.rstrip('\n') for l in f if l.strip()]
