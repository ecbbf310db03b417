"""oracle/grid_march_fp64.py -- fp64 references, with per-element error bounds, of the grid encoder (csrc/gridencoder.cu) and of the
compositing operators of csrc/raymarching.cu (train forward / backward, inference).

TEST INFRASTRUCTURE ONLY.  Vectorised torch; runs on the CPU (host tests) or on CUDA in float64 (GPU tests).  The helpers
(gamma, fma_f32, violations, assert_within) are field_fp64's.

Grid encoder.  What is an integer or a position in the kernel stays in fp32, exactly as the kernel computes it: the device level
scale (sfb_grid_level_scales), p = fma(x, scale, 0.5 or 0) (the SASS contracts it into one FFMA), cell = floor(p), frac = p - cell
(exact), and the row of each corner, including the tiled-stride quirk (coordinates past the first stride above the level's row count
are dropped) and the hash.  Everything after frac is fp64.  Bounds, as gamma(n) times the same sum on absolute values (Higham, 2nd
ed., sec. 3.1), n counting the fp32 roundings along the longest path:
    weight      D roundings of 1 - frac and D - 1 products                                   n_w  = 2D - 1
    forward     the weight, one product with the value, 2^D adds                             n_w + 1 + 2^D
    dy_dx       scale times D - 1 factors (2(D - 1)), vr - vl (bounded on |vr| + |vl|), one product, 2^(D-1) adds
    embedding   each scatter w * g (n_w + 1), then one add per scatter into the row (the row's hit count)
    grad_inputs L C products and adds of grad * dy_dx, plus the dy_dx bound
Points with any coordinate outside [0, 1] have weight 0: their outputs and dy_dx must be exact zeros and they scatter nothing.

Compositing.  The kernels compute alpha = 1 - __expf(-sigma delta).  CUDA documents __expf's error as 2 + floor(|1.173 x|) ulp
(CUDA C++ Programming Guide, intrinsic functions); ex2.approx returns exactly 1 at 0, so sigma delta = 0 is exact.  Near
sigma delta = 0 that error is all of alpha, so it is carried as an absolute error through alpha = 1 - e and the transmittance:
    e_err = (2 + floor(1.173 x)) ulp(e) + x u e            (the second term: the rounding of x = sigma * delta)
    a_err = e_err + u alpha,  (1 - alpha) carries a_err + u (1 - alpha),
    |dT_{k+1}| <= sum_{j<=k} T_j (a_err_j + u (1 - a_j)) + u T_{j+1},    |dw_k| <= a_k |dT_k| + T_k a_err_k + u w_k,
(the train kernels' T is a product, so |dT_{k+1}| <= T_{k+1} sum_{j<=k} ((a_err_j + u (1 - a_j)) / (1 - a_j) + u) bounds it as well,
which is the tighter of the two once T is small),
and every sum over samples adds gamma(K + 1) of its absolute companion.  These are first-order bounds; the products of two first-order
terms are covered by the factor 1 + 2 max|dT| + gamma(8 T).
The termination step is part of the contract: it is taken from an fp32 restatement, and a ray on which fp64 would stop at another
step must have |T_64 - T_thresh| within the transmittance bound there (``ambiguous``).  The backward is checked against torch
autograd of the fp64 forward truncated at that step, with the loss sum(g_image image) + sum(g_ws ws): depth takes no gradient.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .field_fp64 import ATOL, U32, assert_within, fma_f32, gamma, violations  # noqa: F401  (re-exported for the tests)

PRIMES = (1, 2654435761, 805459861, 3674653429, 2097192037, 1434869437, 2165219737)
MASK32 = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ grid encoder
def level_plan(offsets, scales, D: int, gridtype: int, align_corners: bool, swap_level: Optional[int] = None):
    """per level: (first row, row count, scale, strides of the coordinates that enter the tiled index, whether the hash is used).
    The stride chain is the kernel's uint32 arithmetic (grid_row); ``swap_level`` inverts the tiled / hash choice of one level (a
    negative control)."""
    plan = []
    for l in range(len(offsets) - 1):
        rows = int(offsets[l + 1]) - int(offsets[l])
        scale = float(scales[l])
        res = int(math.ceil(scale)) + 1
        stride, strides = 1, []
        for _ in range(D):
            if stride <= rows:
                strides.append(stride)
                stride = (stride * (res if align_corners else res + 1)) & MASK32
        use_hash = gridtype == 0 and stride > rows
        if swap_level == l:
            use_hash = not use_hash
        plan.append((int(offsets[l]), rows, scale, strides, use_hash))
    return plan


def corner_bits(D: int, device) -> torch.Tensor:
    k = torch.arange(1 << D, device=device)
    return torch.stack([(k >> d) & 1 for d in range(D)], 1)                  # [2^D, D]


def grid_locate(x: torch.Tensor, scale: float, align_corners: bool):
    """fp32 p = fma(x, scale, 0.5 or 0); cell (int64) and frac (fp64, exact) [B, D]"""
    p = fma_f32(x.float(), torch.full_like(x.float(), scale), 0.0 if align_corners else 0.5)
    cell = torch.floor(p)
    return cell.long(), (p.double() - cell.double())


def corner_rows(cell: torch.Tensor, bits: torch.Tensor, level) -> torch.Tensor:
    """row inside the level of every corner: [B, 2^D]"""
    first, rows, _, strides, use_hash = level
    cl = cell[:, None, :] + bits[None]                                         # [B, K, D]
    if use_hash:
        idx = torch.zeros(cl.shape[:2], dtype=torch.int64, device=cl.device)
        for d in range(cl.shape[2]):
            idx = idx ^ ((cl[..., d] * PRIMES[d]) & MASK32)
    else:
        idx = torch.zeros(cl.shape[:2], dtype=torch.int64, device=cl.device)
        for d, s in enumerate(strides):
            idx = idx + cl[..., d] * s
        idx = idx & MASK32
    return idx % rows


def corner_weights(frac: torch.Tensor, bits: torch.Tensor, swap_dim: Optional[int] = None) -> torch.Tensor:
    """fp64 multilinear weights [B, 2^D]; ``swap_dim`` exchanges frac and 1 - frac in one dimension (a negative control)"""
    w = torch.ones(frac.shape[0], bits.shape[0], dtype=torch.float64, device=frac.device)
    for d in range(bits.shape[1]):
        f = frac[:, d:d + 1]
        hi, lo = (1 - f, f) if d == swap_dim else (f, 1 - f)
        w = w * torch.where(bits[None, :, d] == 1, hi, lo)
    return w


def grid_rtols(D: int, C: int, L: int):
    n_w = 2 * D - 1
    n_dy = 2 * (D - 1) + 2 + (1 << (D - 1))
    return dict(n_w=n_w, out=gamma(n_w + 1 + (1 << D)), dy=gamma(n_dy), gi=gamma(L * C + n_dy + 1))


class GridFP64:
    """fp64 forward / backward of the grid encoder for fp32 inputs x [B, D] and embeddings [rows, C], on x's device.

    forward(): out / out_abs [L, B, C], dy / dy_abs [B, L, D, C] (the kernel's layout), rows [L, B, 2^D] (absolute, -1 outside).
    backward(grad [L, B, C]): ge / ge_abs / ge_rtol [rows, C] and, given the kernel's dy_dx, gi / gi_abs [B, D].
    Negative controls: drop_corner=(b, level, corner), swap_dim=d (frac / 1 - frac in dimension d), swap_level=l (tiled <-> hash),
    flip_dy=(b, level, d, c)."""

    def __init__(self, x, emb, offsets, scales, gridtype: int, align_corners: bool, chunk: int = 1 << 16, drop_corner=None,
                 swap_dim=None, swap_level=None, flip_dy=None):
        self.dev = x.device
        self.x = x.float()
        self.emb = emb.to(self.dev).double()
        self.B, self.D = x.shape
        self.C = emb.shape[1]
        self.L = len(offsets) - 1
        self.n_rows = int(offsets[-1])
        self.plan = level_plan(offsets, scales, self.D, gridtype, align_corners, swap_level)
        self.ac, self.chunk = align_corners, chunk
        self.bits = corner_bits(self.D, self.dev)
        self.drop_corner, self.swap_dim, self.flip_dy = drop_corner, swap_dim, flip_dy
        self.rt = grid_rtols(self.D, self.C, self.L)
        self.live = ~((self.x < 0) | (self.x > 1)).any(1)                     # NaN-free inputs only

    def _level(self, l, lo, hi):
        """rows (absolute) and fp64 weights [b, 2^D] of points lo:hi on level l, plus frac; weights 0 outside [0, 1]"""
        lv = self.plan[l]
        cell, frac = grid_locate(self.x[lo:hi], lv[2], self.ac)
        live = self.live[lo:hi]
        cell = torch.where(live[:, None], cell, torch.zeros_like(cell))
        rows = corner_rows(cell, self.bits, lv) + lv[0]
        w = corner_weights(frac, self.bits, self.swap_dim) * live[:, None]
        if self.drop_corner is not None and self.drop_corner[1] == l and lo <= self.drop_corner[0] < hi:
            w[self.drop_corner[0] - lo, self.drop_corner[2]] = 0
        return rows, w, frac, live

    def forward(self) -> Dict[str, torch.Tensor]:
        B, D, C, L = self.B, self.D, self.C, self.L
        f64 = dict(dtype=torch.float64, device=self.dev)
        out, out_abs = torch.zeros(L, B, C, **f64), torch.zeros(L, B, C, **f64)
        dy, dy_abs = torch.zeros(B, L, D, C, **f64), torch.zeros(B, L, D, C, **f64)
        rows_all = torch.full((L, B, 1 << D), -1, dtype=torch.int64, device=self.dev)
        for lo in range(0, B, self.chunk):
            hi = min(B, lo + self.chunk)
            for l in range(L):
                rows, w, frac, live = self._level(l, lo, hi)
                e = self.emb[rows]                                              # [b, K, C]
                out[l, lo:hi] = (w[..., None] * e).sum(1)
                out_abs[l, lo:hi] = (w[..., None] * e.abs()).sum(1)
                rows_all[l, lo:hi] = torch.where(live[:, None], rows, torch.full_like(rows, -1))
                scale = self.plan[l][2]
                for gd in range(D):
                    right = self.bits[:, gd] == 1                               # corners on the +1 side of dimension gd
                    # the weight of a corner pair without dimension gd: the full weight over the factor of gd
                    others = torch.ones_like(w)
                    for d in range(D):
                        if d != gd:
                            f = frac[:, d:d + 1]
                            hi_, lo_ = (1 - f, f) if d == self.swap_dim else (f, 1 - f)
                            others = others * torch.where(self.bits[None, :, d] == 1, hi_, lo_)
                    wr = (others * scale * live[:, None])[:, right]             # pairs ordered alike on both sides
                    vr, vl = e[:, right], e[:, ~right]
                    dy[lo:hi, l, gd] = (wr[..., None] * (vr - vl)).sum(1)
                    dy_abs[lo:hi, l, gd] = (wr[..., None] * (vr.abs() + vl.abs())).sum(1)
        if self.flip_dy is not None:
            b, l, d, c = self.flip_dy
            dy[b, l, d, c] = -dy[b, l, d, c]
        self.rows_all = rows_all
        return dict(out=out, out_abs=out_abs, dy=dy, dy_abs=dy_abs, rows=rows_all)

    def backward(self, grad: torch.Tensor, dy_kernel: Optional[torch.Tensor] = None, dy_abs: Optional[torch.Tensor] = None,
                 drop_scatter=None) -> Dict[str, torch.Tensor]:
        """grad [L, B, C] fp32.  ``drop_scatter=(b, level, corner)`` leaves one scatter out (a negative control)."""
        B, D, C, L = self.B, self.D, self.C, self.L
        g = grad.to(self.dev).double()
        f64 = dict(dtype=torch.float64, device=self.dev)
        ge, ge_abs, hits = torch.zeros(self.n_rows, C, **f64), torch.zeros(self.n_rows, C, **f64), torch.zeros(self.n_rows, **f64)
        for lo in range(0, B, self.chunk):
            hi = min(B, lo + self.chunk)
            for l in range(L):
                rows, w, _, live = self._level(l, lo, hi)
                if drop_scatter is not None and drop_scatter[1] == l and lo <= drop_scatter[0] < hi:
                    w = w.clone()
                    w[drop_scatter[0] - lo, drop_scatter[2]] = 0
                wg = w[..., None] * g[l, lo:hi, None, :]                       # [b, K, C]
                r = rows.reshape(-1)
                ge.index_add_(0, r, wg.reshape(-1, C))
                ge_abs.index_add_(0, r, wg.abs().reshape(-1, C))
                hits.index_add_(0, r, live[:, None].expand_as(rows).reshape(-1).double())
        out = dict(ge=ge, ge_abs=ge_abs, ge_rtol=gamma(self.rt['n_w'] + 1 + hits)[:, None], hits=hits)
        if dy_kernel is not None:
            dk = dy_kernel.to(self.dev).double().view(B, L, D, C)
            gl = g.permute(1, 0, 2)                                             # [B, L, C]
            out['gi'] = (gl[:, :, None, :] * dk).sum((1, 3))
            out['gi_abs'] = (gl.abs()[:, :, None, :] * dy_abs.view(B, L, D, C)).sum((1, 3))
        return out


def grid_points(B: int, D: int, scales, seed: int) -> torch.Tensor:
    """B fp32 points in [0, 1]^D, then the edges: 0, 1, -0.0, just outside [0, 1], and cell boundaries (k - 0.5) / scale of every
    level with their fp32 neighbours"""
    g = torch.Generator().manual_seed(seed)
    pts = [torch.rand(B, D, generator=g)]
    one, zero = torch.ones(D), torch.zeros(D)
    edge = [zero, one, -zero, torch.full((D,), 0.5)]
    for d in range(D):
        for v in (1.0000001, -1e-7, float(torch.nextafter(torch.tensor(1.0), torch.tensor(2.0))), -1e-45):
            p = torch.full((D,), 0.5)
            p[d] = v
            edge.append(p)
    pts.append(torch.stack(edge))
    for s in scales:
        s = float(s)
        k = torch.randint(1, max(2, int(s) + 1), (8, D), generator=g).double()
        base = ((k - 0.5) / s).clamp(0, 1).float()
        pts += [base, torch.nextafter(base, torch.ones_like(base)), torch.nextafter(base, torch.zeros_like(base))]
    return torch.cat(pts).float().contiguous()


# ------------------------------------------------------------------------------------------------ compositing
def _ulp32(v: torch.Tensor) -> torch.Tensor:
    """one fp32 ulp at |v| (fp64 in, fp64 out), 2^-149 at least"""
    _, ex = torch.frexp(v.abs())
    return torch.ldexp(torch.ones_like(v), (ex - 24).clamp(min=-149))


def _alpha(s: torch.Tensor, dt: torch.Tensor):
    """fp64 alpha = 1 - exp(-s dt) and the absolute bound of the kernel's 1 - __expf(-s * dt) and of its 1 - alpha"""
    x = s * dt
    e = torch.exp(-x)
    n = 2 + torch.floor(1.173 * x.abs())
    e_err = torch.where(x == 0, torch.zeros_like(x), n * _ulp32(e) + x.abs() * U32 * e + (e < 2.0 ** -126) * 2.0 ** -126)
    a = 1 - e
    a_err = e_err + U32 * a
    return a, a_err, a_err + U32 * (1 - a) * (a != 0)           # 1 - alpha is exact where alpha is


def _excl_cumprod(v: torch.Tensor) -> torch.Tensor:
    return torch.cat([torch.ones_like(v[:, :1]), torch.cumprod(v, 1)[:, :-1]], 1)


def _excl_cumsum(v: torch.Tensor) -> torch.Tensor:
    return torch.cumsum(v, 1) - v


def _gam_k(K: torch.Tensor) -> torch.Tensor:
    K = K.double()
    return K * U32 / (1 - K * U32)


def train_stop_fp32(s, dt, counts, T_thresh: float, exp_fn=torch.exp) -> torch.Tensor:
    """the fp32 restatement's termination: number of samples each ray composites (composite_train_fwd_kernel)"""
    s, dt = s.float(), dt.float()
    N, T = s.shape
    T32 = torch.ones(N, dtype=torch.float32, device=s.device)
    K = counts.clone().long()
    alive = counts > 0
    thr = torch.tensor(T_thresh, dtype=torch.float32)
    for k in range(T):
        act = alive & (k < counts)
        if not bool(act.any()):
            break
        alpha = 1.0 - exp_fn(-(s[:, k] * dt[:, k]))
        T32 = torch.where(act, T32 * (1.0 - alpha), T32)
        stop = act & (T32 < thr)
        K = torch.where(stop, torch.full_like(K, k + 1), K)
        alive = alive & ~stop
    return K


def composite_train_fp64(sigmas, rgbs, deltas, counts, T_thresh: float, g_ws=None, g_image=None, K=None) -> Dict[str, torch.Tensor]:
    """fp64 composite_rays_train forward (and backward, given g_ws [N] and g_image [N,3]) on padded rays: sigmas [N,T], rgbs [N,T,3],
    deltas [N,T,2] (fp32), counts [N] samples per ray (0 for empty rays and rays past M).  K [N]: the samples composited (default:
    the fp32 restatement's).  Values come with absolute bounds '<name>_err'."""
    dev = sigmas.device
    s, c, dl = sigmas.double(), rgbs.double(), deltas.double()
    N, T = s.shape
    counts = counts.to(dev).long()
    K32 = train_stop_fp32(sigmas, deltas[..., 0], counts, T_thresh)
    K = K32 if K is None else K.to(dev).long()
    idx = torch.arange(T, device=dev)[None]
    m = (idx < K[:, None]).double()

    a, a_err, f_err = _alpha(s, dl[..., 0])
    a, a_err, f_err = a * m, a_err * m, f_err * m
    Tk = _excl_cumprod(1 - a)
    Tn = Tk * (1 - a)
    loc = Tk * f_err + U32 * Tn * m * (a != 0)                  # T (1 - alpha) is exact where alpha is 0
    # T is a product, so its error is also bounded relatively: sum of the relative errors of its factors; the smaller bound holds
    rloc = torch.where(a < 1, f_err / (1 - a), torch.full_like(a, math.inf)) + U32 * (a != 0)
    rTn = torch.cumsum(rloc, 1)
    rel = lambda r, v: torch.where(torch.isfinite(r), r * v, torch.full_like(v, math.inf))
    dTn = torch.minimum(torch.cumsum(loc, 1), rel(rTn, Tn))
    dTk = torch.minimum(torch.cumsum(loc, 1) - loc, rel(rTn - rloc, Tk))
    w = a * Tk
    dw = (a * dTk + Tk * a_err + U32 * w) * m
    close = 1 + 2 * dTn.amax(1, keepdim=True) + gamma(8 * T)
    gK = _gam_k(K + 1)[:, None]

    ws = w.sum(1)
    ws_err = (dw.sum(1) + gK[:, 0] * w.sum(1)) * close[:, 0]
    image = (w[..., None] * c).sum(1)
    image_err = ((dw[..., None] * c.abs()).sum(1) + gK * (w[..., None] * c.abs()).sum(1)) * close
    t = torch.cumsum(dl[..., 1] * m, 1)
    t_err = _gam_k(idx + 1) * torch.cumsum(dl[..., 1].abs() * m, 1)
    depth = (w * t).sum(1)
    depth_err = ((dw * t.abs() + w * t_err).sum(1) + gK[:, 0] * (w * t.abs()).sum(1)) * close[:, 0]

    # ambiguity of the termination test: T_{k+1} < T_thresh decided within the bound of T_{k+1} at some composited step
    near = ((Tn - T_thresh).abs() <= dTn * close) & (dTn > 0) & (m > 0)            # an exact T decides as fp64 does
    ambiguous = near.any(1) if T_thresh > 0 else torch.zeros(N, dtype=torch.bool, device=dev)
    # where fp64 stops elsewhere, the decision must be one of those ambiguous ones
    valid = idx < counts[:, None]
    a_all, _, _ = _alpha(s, dl[..., 0])
    Tn_all = torch.cumprod(1 - a_all * valid, 1)
    stop64 = (Tn_all < T_thresh) & valid
    K64 = torch.where(stop64.any(1), stop64.double().argmax(1) + 1, counts)

    out = dict(ws=ws, ws_err=ws_err, image=image, image_err=image_err, depth=depth, depth_err=depth_err, K=K, K32=K32, K64=K64,
               ambiguous=ambiguous, w=w, w_err=dw * close, T_next=Tn, T_next_err=dTn * close)
    if g_ws is None:
        return out

    gws, gim = g_ws.to(dev).double(), g_image.to(dev).double()
    # exact derivative of the truncated forward: autograd in fp64
    sg = s.clone().requires_grad_(True)
    cg = c.clone().requires_grad_(True)
    ag = (1 - torch.exp(-sg * dl[..., 0])) * m
    wg = ag * _excl_cumprod(1 - ag)
    loss = ((wg[..., None] * cg).sum(1) * gim).sum() + (wg.sum(1) * gws).sum()
    loss.backward()
    # bounds of the kernel's closed form: T_{k+1} c_k - (final - prefix_k), summed over channels, + gws (1 - ws_final), times delta
    pre = torch.cumsum(w[..., None] * c, 1)
    pre_err = torch.cumsum(dw[..., None] * c.abs(), 1) + _gam_k(idx + 1)[..., None] * torch.cumsum(w[..., None] * c.abs(), 1)
    gia = gim.abs()[:, None, :]
    rel = (gia * (Tn[..., None] * c.abs() + image.abs()[:, None, :] + pre.abs())).sum(-1) + gws.abs()[:, None] * (1 + ws.abs()[:, None])
    prop = (gia * (dTn[..., None] * c.abs() + image_err[:, None, :] + pre_err)).sum(-1) + gws.abs()[:, None] * ws_err[:, None]
    d0 = dl[..., 0].abs()
    out.update(g_sigma=sg.grad * m, g_sigma_err=(d0 * (prop * close + gamma(8) * rel)) * m,
               g_rgb=cg.grad * m[..., None], g_rgb_err=(gia * (dw * close + U32 * w)[..., None]) * m[..., None])
    return out


def closed_form_train_backward(ref: Dict[str, torch.Tensor], c, deltas, g_ws, g_image, drop_ws_term=False) -> torch.Tensor:
    """the kernel's closed form of dL/dsigma evaluated in fp64 on the reference forward; ``drop_ws_term`` leaves out
    g_ws (1 - ws_final) (a negative control)"""
    c, d0 = c.double(), deltas[..., 0].double()
    m = (torch.arange(c.shape[1], device=c.device)[None] < ref['K'][:, None]).double()
    pre = torch.cumsum(ref['w'][..., None] * c, 1)
    term = (g_image.double()[:, None, :] * (ref['T_next'][..., None] * c - (ref['image'][:, None, :] - pre))).sum(-1)
    if not drop_ws_term:
        term = term + g_ws.double()[:, None] * (1 - ref['ws'][:, None])
    return d0 * term * m


def inference_stop_fp32(s, dl, ws0, n_step: int, T_thresh: float):
    """composite_rays_kernel's loop in fp32: samples composited (K) and whether the ray stays alive"""
    s, d0 = s.float(), dl[..., 0].float()
    ws = ws0.float().clone()
    n = s.shape[0]
    K = torch.full((n,), n_step, dtype=torch.long, device=s.device)
    alive = torch.ones(n, dtype=torch.bool, device=s.device)
    thr = torch.tensor(T_thresh, dtype=torch.float32)
    for k in range(n_step):
        zero = alive & (d0[:, k] == 0)
        K = torch.where(zero, torch.full_like(K, k), K)
        alive = alive & ~zero
        alpha = 1.0 - torch.exp(-(s[:, k] * d0[:, k]))
        T = 1.0 - ws
        ws = torch.where(alive, ws + alpha * T, ws)
        stop = alive & (T < thr)
        K = torch.where(stop, torch.full_like(K, k + 1), K)
        alive = alive & ~stop
    return K, alive


def composite_inference_fp64(sigmas, rgbs, deltas, ws0, d0, img0, t0, T_thresh: float, K=None) -> Dict[str, torch.Tensor]:
    """fp64 composite_rays (one iteration of the inference loop) for n alive rays with n_step samples each: sigmas [n,S], rgbs [n,S,3],
    deltas [n,S,2] and the running state ws0, d0 [n], img0 [n,3], t0 [n].  The transmittance is 1 - ws, tested before the sample is
    added; a sample with delta 0 ends the ray before it is composited."""
    dev = sigmas.device
    s, c, dl = sigmas.double(), rgbs.double(), deltas.double()
    n, S = s.shape
    K32, alive32 = inference_stop_fp32(sigmas, deltas, ws0, S, T_thresh)
    K = K32 if K is None else K
    idx = torch.arange(S, device=dev)[None]
    m = (idx < K[:, None]).double()
    a, a_err, _ = _alpha(s, dl[..., 0])
    a, a_err = a * m, a_err * m
    w0 = ws0.double()
    Tk = (1 - w0)[:, None] * _excl_cumprod(1 - a)
    w = a * Tk
    wsn = w0[:, None] + torch.cumsum(w, 1)
    loc = (a * U32 * Tk + Tk * a_err + U32 * w + U32 * wsn) * m
    dws = _excl_cumsum(loc)                                                     # |d ws_k| before sample k
    dT = dws + U32 * Tk * (wsn - w != 0)                        # 1 - ws is exact where ws is 0
    dw = (a * dT + Tk * a_err + U32 * w) * m
    close = 1 + 2 * (dws + loc).amax(1, keepdim=True) + gamma(8 * S)
    gK = _gam_k(K + 1)[:, None]
    ws = w0 + w.sum(1)
    ws_err = ((dws + loc)[:, -1] + gK[:, 0] * (w0.abs() + w.sum(1))) * close[:, 0]
    image = img0.double() + (w[..., None] * c).sum(1)
    image_err = ((dw[..., None] * c.abs()).sum(1) + gK * (img0.double().abs() + (w[..., None] * c.abs()).sum(1))) * close
    t = t0.double()[:, None] + torch.cumsum(dl[..., 1] * m, 1)
    t_err = _gam_k(idx + 1) * (t0.double().abs()[:, None] + torch.cumsum(dl[..., 1].abs() * m, 1))
    depth = d0.double() + (w * t).sum(1)
    depth_err = ((dw * t.abs() + w * t_err).sum(1) + gK[:, 0] * (d0.double().abs() + (w * t.abs()).sum(1))) * close[:, 0]
    near = ((Tk - T_thresh).abs() <= dT * close) & (dT > 0) & (m > 0)
    ambiguous = near.any(1) if T_thresh > 0 else torch.zeros(n, dtype=torch.bool, device=dev)
    return dict(ws=ws, ws_err=ws_err, image=image, image_err=image_err, depth=depth, depth_err=depth_err, K=K, alive=alive32,
                ambiguous=ambiguous)


# ------------------------------------------------------------------------------------------------ sph_from_ray
def sph_from_ray_fp64(rays_o, rays_d, radius: float):
    """coords [N,2] in fp64 and a first-order bound of the kernel's fp32 evaluation.  Each fp32 operation of sph_from_ray_kernel
    is written as op * (1 + delta_i); the bound is sum_i |d coords / d delta_i| * eps_i at delta = 0 (autograd, fp64), with eps_i = u
    for the correctly rounded operations (products, sums, sqrtf, the division) and 3 ulp (3 * 2^-23 relative) for each atan2f (CUDA's
    documented maximum error), doubled for the products of two first-order terms that the linearisation drops."""
    o, d = rays_o.double(), rays_d.double()
    N = o.shape[0]
    deltas, eps = [], []

    def r(v, e=U32):
        dlt = torch.zeros(N, dtype=torch.float64, device=o.device, requires_grad=True)
        deltas.append(dlt)
        eps.append(e)
        return v * (1 + dlt)

    dx, dy, dz = d.unbind(1)
    ox, oy, oz = o.unbind(1)
    A = r(r(r(dx * dx) + r(dy * dy)) + r(dz * dz))
    Bh = r(r(r(ox * dx) + r(oy * dy)) + r(oz * dz))
    Cc = r(r(r(r(ox * ox) + r(oy * oy)) + r(oz * oz)) - r(torch.full_like(ox, radius * radius)))
    disc = r(r(Bh * Bh) - r(A * Cc))
    t = r(r(-Bh + r(torch.sqrt(disc))) / A)
    x, y, z = r(ox + r(t * dx)), r(oy + r(t * dy)), r(oz + r(t * dz))
    theta = r(torch.atan2(r(torch.sqrt(r(r(x * x) + r(z * z)))), y), 3 * 2.0 ** -23)
    phi = r(torch.atan2(z, x), 3 * 2.0 ** -23)
    rpi = float(torch.tensor(1 / math.pi, dtype=torch.float32))
    c0 = r(r(r(2 * theta) * rpi) - 1)
    c1 = r(phi * rpi)
    out, err = [], []
    for v in (c0, c1):
        gs = torch.autograd.grad(v.sum(), deltas, retain_graph=True, allow_unused=True)
        e = torch.zeros(N, dtype=torch.float64, device=o.device)
        for g, ep in zip(gs, eps):
            if g is not None:
                e = e + g.abs() * ep
        out.append(v.detach())
        err.append(2 * e)
    return torch.stack(out, 1), torch.stack(err, 1)


# ------------------------------------------------------------------------------------------------ test geometry
GRID_H, GRID_L = 2, 5          # base resolution 2, per-level scale 2: resolutions 2, 4, 8, 16, 32


def grid_case(D: int, align_corners: bool):
    """level offsets of a GridEncoder geometry whose two coarsest levels are dense tiled grids and whose three finest are capped at
    the hashmap size (hash or tiled-with-wraparound rows), so both branches of grid_row run in one call: (offsets, S, H)"""
    from sparsefusion_b200.gridencoder import level_offsets
    log2_hashmap = math.ceil(math.log2(5 ** D))
    return level_offsets(D, GRID_L, 2.0, GRID_H, log2_hashmap, align_corners), 1.0, GRID_H


def grid_embeddings(n_rows: int, C: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n_rows, C, generator=g) * 2 - 1).float()
