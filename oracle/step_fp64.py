"""oracle/step_fp64.py -- launch plans, fp64 references and per-element error bounds of the sampler updates (plms_update*,
ddpm_dynamic_step in csrc/unet_ops.cu), the distillation loss kernels (csrc/image_glue.cu) and the EFT-only kernels (csrc/eft_ops.cu).

TEST INFRASTRUCTURE ONLY.

Conventions as oracle/simt_fp64.py: every ``ref_*`` returns (y, bound) with |got - y| <= rho * A + slack per element, A the absolute
companion, rho = gamma(n) (``field_fp64.gamma``) for the longest chain of fp32 roundings the kernel runs.  The library is built without
--use_fast_math, so sqrtf and '/' are correctly rounded (one rounding each); FMA contraction is on, which never lengthens a chain.
Positions and weights that select or weight source elements (the resize / grid-sample coordinates, the glue's taps, the mode-1 mask) are
computed in fp32 the kernel's way and then promoted, as ``field_fp64`` does for the trilinear weights: they are part of what the kernel
computes, and the discrete ones must match exactly.

NaN: the references follow torch -- clamp, max-pool, relu and quantile keep NaN -- and the tests compare NaN positions exactly.

``emulate_*`` evaluate the kernels' arithmetic in fp32 (torch on the CPU) with switches that inject single defects; the host tests use them
to show what the bounds see.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from .field_fp64 import ATOL, U32 as U, gamma
from .simt_fp64 import ULP, _softmax_pv_bound

HUBER_S = float(np.float32(0.1))                        # kHuberS
HUBER_S2 = float(np.float32(np.float32(0.1) * np.float32(0.1)))   # kHuberS * kHuberS, folded in fp32
INV_SQRT2 = float(np.float32(0.70710678118654752))
NAN = float('nan')


def f32(v) -> float:
    return float(np.float32(v))


def _ceil_div(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ launch plans
DYN_CHUNK, DYN_MAX_CLUSTER = 8192, 8


def kernel_plan(op: str, g: Dict, sm_count: int = 132) -> Dict:
    """the launches the host makes for ``op``; ``kernels`` lists the traced names (the SFB_LAUNCH kernels only)"""
    if op == 'plms_update':                                            # unet_ops.cu sfb_plms_update
        return dict(grid=(min(_ceil_div(g['n'], 256), 1024), 1), kernels=['sfb::plms_update_kernel'])
    if op in ('plms_update_rows', 'plms_update_rows_cfg'):
        bx = min(_ceil_div(g['row_len'], 256), 1024)
        return dict(grid=(bx, g['rows']), kernels=[f'sfb::{op}_kernel'])
    if op == 'ddpm_dynamic_step':                                      # sfb_ddpm_dynamic_step
        k = _ceil_div(g['row_len'], DYN_CHUNK)
        chunk = _ceil_div(g['row_len'], k)
        return dict(k=k, chunk=chunk, smem=chunk * 4, grid=(k, g['B']),
                    kernels=[f"sfb::ddpm_dynamic_step_kernel<{'true' if k > 1 else 'false'}>"])
    if op in ('photometric_loss', 'fusion_loss'):                      # image_glue.cu: min(ceil(n / 256), 2 SMs) blocks
        n = g['h'] * g['w'] if op == 'photometric_loss' else 4 * g['h'] * g['w']
        blocks = min(_ceil_div(n, 256), 2 * sm_count)
        return dict(blocks=blocks, iters=_ceil_div(n, 256 * blocks), kernels=[])
    raise KeyError(op)


# ------------------------------------------------------------------------------------------------ comparison
def compare(got: torch.Tensor, ref: torch.Tensor, bnd: Optional[torch.Tensor]) -> Dict:
    """NaN-aware per-element comparison: NaN positions must match; where the reference is infinite the value must be equal; elsewhere
    |got - ref| <= bnd (bnd None: equal values, +-0 alike).  Returns dict(nan_ok, ratio) with ratio the largest err / bound."""
    got = got.to(ref.device).double()
    ref = ref.double()
    gn, rn = torch.isnan(got), torch.isnan(ref)
    nan_ok = bool(torch.equal(gn, rn))
    fin = ~gn & ~rn
    inf = fin & torch.isinf(ref)
    bad_inf = bool((got[inf] != ref[inf]).any())
    rest = fin & ~torch.isinf(ref)
    if bnd is None:
        ratio = math.inf if bool((got[rest] != ref[rest]).any()) else 0.0
    else:
        b = bnd.to(ref.device).double().expand_as(ref)[rest]
        r = (got[rest] - ref[rest]).abs() / (b + ATOL)
        r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
        ratio = float(r.max()) if r.numel() else 0.0
    if bad_inf:
        ratio = math.inf
    return dict(nan_ok=nan_ok, ratio=ratio)


def passes(got, ref, bnd) -> bool:
    c = compare(got, ref, bnd)
    return c['nan_ok'] and c['ratio'] <= 1


# ------------------------------------------------------------------------------------------------ sampler updates
def ref_plms(x, eps: Sequence[Optional[torch.Tensor]], coefs, scalars, noise, clip, e_abs=None, e_ref=None):
    """x, eps[i], noise [rows, row_len] fp32 (eps[i] None: a NULL history pointer); coefs (c0..c3) fp32 values; scalars [rows, 5] =
    (alpha, sigma, alpha_next, c, noise_scale) fp32.  Returns {'e', 'x0', 'x_prev'}: (y, bound).

    e = sum c_i e_i: c0 e0 and up to three fmas, gamma(4) on sum |c_i||e_i|.  ``e_ref`` / ``e_abs`` replace the combination and its
    companion (the guided DDPM path: s cond + (1 - s) null against the reference's null + (cond - null) s, companion |s||cond| + |1-s||null|).
    x0 = (x - sigma e) / max(alpha, 1e-8): an fma and a division on (|x| + sigma A_e) / alpha -> gamma(7) with e's error folded in.
    The clamp is 1-Lipschitz (the bound passes through; an element clamped with margin is exact).
    x_prev = alpha_next (x (1 - c) / alpha + c x0) + noise_scale noise: (1 - c), the product, the quotient, the fma, alpha_next and the
    last fma -- gamma(6) on the companion, plus |alpha_next c| times x0's bound."""
    rows = x.shape[0]
    sc = torch.as_tensor(scalars, dtype=torch.float64).reshape(rows, 5).to(x.device)
    al, sg, an, c, ns = (sc[:, i:i + 1] for i in range(5))
    xd, nd = x.double(), noise.double()
    if e_ref is None:
        e = torch.zeros_like(xd)
        ea = torch.zeros_like(xd)
        for ci, ei in zip(coefs, eps):
            if ei is None:
                continue
            e = e + f32(ci) * ei.double()
            ea = ea + abs(f32(ci)) * ei.double().abs()
    else:
        e, ea = e_ref.double(), e_abs.double()
    be = gamma(4) * ea + ATOL
    alc = torch.clamp(al, min=f32(1e-8))
    x0 = (xd - sg * e) / alc
    a0 = (xd.abs() + sg.abs() * ea) / alc
    b0 = gamma(7) * a0 + ATOL
    clip = f32(clip)
    x0c = torch.where(torch.isnan(x0), x0, x0.clamp(-clip, clip))
    clipped = (x0.abs() - b0 > clip) | torch.isinf(x0)
    b0c = torch.where(clipped, torch.zeros_like(b0), b0)
    mean = an * (xd * (1 - c) / al + c * x0c)
    y = mean + ns * nd
    A = an.abs() * (xd.abs() * (1 - c).abs() / al.abs() + c.abs() * x0c.abs()) + ns.abs() * nd.abs()
    bx = gamma(6) * A + (an * c).abs() * b0c + ATOL
    return {'e': (e, be), 'x0': (x0c, b0c), 'x_prev': (y, bx)}


def cfg_eps(e_cond: torch.Tensor, e_null: torch.Tensor, cond_scale: float) -> torch.Tensor:
    """e_null + (e_cond - e_null) * cond_scale in fp32, three roundings, no contraction: what the cfg kernel's e_out must equal bit for bit"""
    ec, en = e_cond.float().cpu(), e_null.float().cpu()
    return en + (ec - en) * torch.tensor(cond_scale, dtype=torch.float32)


def emulate_plms(x, eps, coefs, scalars, noise, clip, defect: Optional[str] = None):
    """fp32 rows kernel.  Defects: 'e1_e2_swap' (c1 pairs with e2), 'row_shift' (row r reads row r - 1's scalars), 'no_alpha_clamp'
    (x0 divides by alpha, not max(alpha, 1e-8)), 'clamp_drops_nan' (fminf / fmaxf)"""
    rows = x.shape[0]
    sc = torch.as_tensor(scalars, dtype=torch.float32).reshape(rows, 5)
    if defect == 'row_shift':
        sc = torch.cat((sc[:1], sc[:-1]))
    al, sg, an, c, ns = (sc[:, i:i + 1] for i in range(5))
    cf = [torch.tensor(f32(v), dtype=torch.float32) for v in coefs]
    ep = list(eps)
    if defect == 'e1_e2_swap':
        ep[1], ep[2] = ep[2], ep[1]
    e = cf[0] * ep[0].float()
    for ci, ei in zip(cf[1:], ep[1:]):
        if ei is not None:
            e = e + ci * ei.float()
    xv = x.float()
    den = al if defect == 'no_alpha_clamp' else torch.clamp(al, min=f32(1e-8))
    x0 = (xv - sg * e) / den
    clip_t = torch.tensor(f32(clip), dtype=torch.float32)
    x0 = torch.nan_to_num(x0, nan=-f32(clip)).clamp(-clip_t, clip_t) if defect == 'clamp_drops_nan' else x0.clamp(-clip_t, clip_t)
    mean = an * (xv * (1 - c) / al + c * x0)
    return {'e': e, 'x0': x0, 'x_prev': mean + ns * noise.float()}


# ------------------------------------------------------------------------------------------------ dynamic thresholding
def dyn_x0(x, e_cond, e_null, cond_scale, alpha, sigma):
    """x0 = (x - sigma e) / max(alpha, 1e-8), e = s e_cond + (1 - s) e_null (e_null None: e_cond): the product, (1 - s), the fma, the
    kernel's fma and the division -> gamma(6) on (|x| + sigma (|s||e_cond| + |1 - s||e_null|)) / alpha"""
    s = f32(cond_scale)
    e = s * e_cond.double()
    ea = abs(s) * e_cond.double().abs()
    if e_null is not None:
        cn = 1.0 - s
        e = e + cn * e_null.double()
        ea = ea + abs(cn) * e_null.double().abs()
    alc = max(f32(alpha), f32(1e-8))
    x0 = (x.double() - f32(sigma) * e) / alc
    return x0, gamma(6) * (x.double().abs() + abs(f32(sigma)) * ea) / alc + ATOL


def quantile_s(x0_rows: torch.Tensor, p: float) -> torch.Tensor:
    """torch.quantile(|x0|, p).clamp(min=1) per row, as DDPM.p_sample computes s (NaN rows give NaN)"""
    return torch.quantile(x0_rows.abs(), p, dim=-1).clamp(min=1)


def ref_dyn_x_prev(x, x0, b0, s, alpha, alpha_next, c, noise_scale, noise):
    """x_prev given the kernel's own s per row (the selection is discontinuous, so it is conditioned on): clamp(x0, +-s) / s is
    1/s-Lipschitz (x0's bound / s) plus the division's rounding; the update's chain is gamma(6) as in ref_plms"""
    sd = s.double().reshape(-1, 1).to(x0.device)
    x0c = torch.where(torch.isnan(x0), x0, torch.maximum(torch.minimum(x0, sd), -sd)) / sd
    b = b0 / sd + U * x0c.abs()
    al, an, c, ns = f32(alpha), f32(alpha_next), f32(c), f32(noise_scale)
    xd = x.double()
    y = an * (xd * (1 - c) / al + c * x0c) + ns * noise.double()
    A = abs(an) * (xd.abs() * abs(1 - c) / abs(al) + abs(c) * x0c.abs()) + abs(ns) * noise.double().abs()
    return y, gamma(6) * A + abs(an * c) * b + ATOL


# ------------------------------------------------------------------------------------------------ image glue
def _huber_grad(d):
    return d / (HUBER_S * torch.sqrt(1 + d * d / HUBER_S2))


def _huber_val(d):
    return (torch.sqrt(1 + d * d / HUBER_S2) - 1) * HUBER_S


def _huber_val_abs(d):
    """companion of huber_val: sqrt(1 + d^2 / s^2) - 1 cancels, so its rounding errors are relative to sqrt(.) + 1"""
    return (torch.sqrt(1 + d * d / HUBER_S2) + 1) * HUBER_S


def glue_nearest(full: torch.Tensor, h: int, w: int, scale: int, defect: Optional[str] = None) -> torch.Tensor:
    """[C, h, w] = full[:, y * scale, x * scale] read through the kernel's flat index (y scale) W + x scale.  Defects: 'hw_swap' (the flat
    index built with h and w exchanged), 'nearest_off_by_one' (source x scale + 1, clamped)"""
    C, Hf, Wf = full.shape
    fl = full.reshape(C, -1)
    y = torch.arange(h).view(h, 1)
    x = torch.arange(w).view(1, w)
    if defect == 'hw_swap':
        src = (x * scale) * (h * scale) + y * scale
    elif defect == 'nearest_off_by_one':
        src = (y * scale) * Wf + torch.clamp(x * scale + 1, max=Wf - 1)
    else:
        src = (y * scale) * Wf + x * scale
    return fl[:, src.reshape(-1).clamp(max=fl.shape[1] - 1)].view(C, h, w)


def sum_chain(plan: Dict) -> int:
    """roundings on one term's way into a sum: its own evaluation (5), one add per grid-stride iteration and channel (3 per iteration),
    5 warp-shuffle levels, 3 levels over the block's 8 warps and one atomic per block"""
    return 5 + 3 * plan['iters'] + 5 + 3 + plan['blocks']


def ref_photometric(img, sil, rgb, mask, h, w, scale, lc, ls, lo, plan, defect: Optional[str] = None):
    """{'g_img' [n,3], 'g_sil' [n], 'sums' [3]}: (y, bound).  g_img = lc huber'(d) / (3 n): huber' is d / (s sqrt(1 + d^2/s^2)) -- its
    relative condition number in d is at most 1 -- so the 9 roundings of d, d^2, / s^2, + 1, sqrt, s *, /, lc * and / (3 n) give gamma(10)
    relative.  g_sil adds lo sv / (sqrt(sv^2 + .01) n): gamma(14) on the companion.  Sums: sum_chain on the companion
    (huber_val's cancellation is relative to sqrt(.) + 1).  ``defect`` is applied to the nearest-source look-up."""
    n = h * w
    lc, ls, lo = f32(lc), f32(ls), f32(lo)
    tgt = glue_nearest(rgb.double().cpu(), h, w, scale, defect).reshape(3, n).t()
    tm = glue_nearest(mask.double().cpu().reshape(1, h * scale, w * scale), h, w, scale, defect).reshape(n)
    d = img.double().cpu() - tgt
    gi = lc * _huber_grad(d) / (3 * n)
    sv = sil.double().cpu()
    dm = sv - tm
    op = torch.sqrt(sv * sv + f32(0.01))
    gs = ls * _huber_grad(dm) / n + lo * sv / (op * n)
    gsa = (ls * _huber_grad(dm) / n).abs() + (lo * sv / (op * n)).abs()
    ch = sum_chain(plan)
    sums = torch.stack((_huber_val(d).sum(), _huber_val(dm).sum(), op.sum()))
    sa = torch.stack((_huber_val_abs(d).sum(), _huber_val_abs(dm).sum(), op.sum()))
    return {'g_img': (gi, gamma(10) * gi.abs() + ATOL), 'g_sil': (gs, gamma(14) * gsa + ATOL), 'sums': (sums, gamma(ch) * sa + ATOL)}


def up2_taps(n: int, edge_clamp: bool = True):
    """[2n, n] matrix of F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) along one axis, taps computed in fp32 as
    up2_taps: s = (d + .5) .5 - .5 clamped at 0, i0 = (int) s, i1 = i0 + (i0 < n - 1), l1 = s - i0 (all exact).  edge_clamp False:
    i1 = i0 + 1 always, a tap past the edge is dropped"""
    M = torch.zeros(2 * n, n, dtype=torch.float64)
    for d in range(2 * n):
        s = max(f32((np.float32(d) + np.float32(0.5)) * np.float32(0.5) - np.float32(0.5)), 0.0)
        i0 = int(s)
        i1 = i0 + (1 if (i0 < n - 1 or not edge_clamp) else 0)
        l1 = s - i0
        M[d, i0] += 1 - l1
        if i1 < n:
            M[d, i1] += l1
    return M


def ref_upsample2x(img, sil, h, w):
    """up [4, 2h, 2w]: exact weights (quarters), four fmas: gamma(4) on sum |w||v|"""
    My, Mx = up2_taps(h), up2_taps(w)
    planes = torch.cat((img.double().cpu().t().reshape(3, h, w), sil.double().cpu().reshape(1, h, w)))
    y = My @ planes @ Mx.t()
    A = My @ planes.abs() @ Mx.t()
    return y, gamma(4) * A + ATOL


def fusion_mask(target: torch.Tensor) -> torch.Tensor:
    """(t0 + t1 + t2) / 3 > 0.1f in fp32, as the kernel and target.mean(dim=1) > .1 compute it"""
    t = target.float().cpu()
    return (((t[0] + t[1]) + t[2]) / 3.0 > torch.tensor(f32(0.1))).double()


def ref_fusion(up, target, mode, wgt, lc, ls, lo, g_extra, plan, defect: Optional[str] = None):
    """{'g_up' [4,H,W], 'sums' [3]}: (y, bound).  mode 0: wgt sign(d) / (3 HW) + g_extra -- sign(d) is exact (an fp32 difference is zero
    only for equal operands), the quotient and the add round: gamma(2).  mode 1: lc huber'(d) / (3 HW) + g_extra, gamma(11); the mask is
    computed in fp32 (``fusion_mask``) and compared exactly through g_up[3].  Defects: 'mask_ge' (>= 0.1f), 'g_extra_on_sil'."""
    H, W = up.shape[1], up.shape[2]
    HW = H * W
    wgt, lc, ls, lo = f32(wgt), f32(lc), f32(ls), f32(lo)
    u = up.double().cpu()
    t = target.double().cpu()
    ge = g_extra.double().cpu() if g_extra is not None else torch.zeros(3, H, W, dtype=torch.float64)
    d = u[:3] - t
    if mode == 0:
        g = wgt * torch.sign(d) / (3 * HW)
        gc = g + ge
        bc = gamma(2) * (g.abs() + ge.abs())
        sc, sca = d.abs().sum(), d.abs().sum()
    else:
        g = lc * _huber_grad(d) / (3 * HW)
        gc = g + ge
        bc = gamma(11) * (g.abs() + ge.abs())
        sc, sca = _huber_val(d).sum(), _huber_val_abs(d).sum()
    sv = u[3]
    op = torch.sqrt(sv * sv + f32(0.01))
    gs = lo * sv / (op * HW)
    gsa = gs.abs()
    ss = ssa = torch.zeros((), dtype=torch.float64)
    if mode == 1:
        m = fusion_mask(target).view(H, W)
        if defect == 'mask_ge':
            tf = target.float().cpu()
            m = (((tf[0] + tf[1]) + tf[2]) / 3.0 >= torch.tensor(f32(0.1))).double()
        dm = sv - m
        gs = gs + ls * _huber_grad(dm) / HW
        gsa = gsa + (ls * _huber_grad(dm) / HW).abs()
        ss, ssa = _huber_val(dm).sum(), _huber_val_abs(dm).sum()
    if defect == 'g_extra_on_sil':
        gs = gs + ge[0]
        gsa = gsa + ge[0].abs()
    y = torch.cat((gc, gs[None]))
    b = torch.cat((bc, gamma(14) * gsa[None])) + ATOL
    ch = sum_chain(plan)
    sums = torch.stack((sc, ss, op.sum()))
    sa = torch.stack((sca, ssa, op.sum()))
    return {'g_up': (y, b), 'sums': (sums, gamma(ch) * sa + ATOL)}


def ref_fusion_adjoint(g_up, h, w):
    """(g_img [n,3], g_sil [n]) of the kernel's own g_up (conditioned on it: g_up has its own check): at most 16 taps, each weight
    product exact, 16 fmas -> gamma(16) on sum |w||g|"""
    My, Mx = up2_taps(h), up2_taps(w)
    g = g_up.double().cpu()
    y = My.t() @ g @ Mx
    A = My.t() @ g.abs() @ Mx
    b = gamma(16) * A + ATOL
    return (y[:3].reshape(3, -1).t(), b[:3].reshape(3, -1).t()), (y[3].reshape(-1), b[3].reshape(-1))


def emulate_fusion_adjoint(g_up, h, w, defect: Optional[str] = None):
    """fp32 adjoint; defect 'adjoint_no_edge_clamp' drops the last tap's clamp (its weight falls off the edge)"""
    My, Mx = up2_taps(h, defect != 'adjoint_no_edge_clamp').float(), up2_taps(w, defect != 'adjoint_no_edge_clamp').float()
    y = My.t() @ g_up.float().cpu() @ Mx
    return y[:3].reshape(3, -1).t(), y[3].reshape(-1)


# ------------------------------------------------------------------------------------------------ EFT: max-pool and activations
def maxpool3x3s2(x: torch.Tensor, defect: Optional[str] = None) -> torch.Tensor:
    """x [NB,H,W,C] -> [NB,(H+1)//2,(W+1)//2,C]: max over the 3x3 window at stride 2, padding 1, NaN-sticky (F.max_pool2d).
    defect 'window_shift': the window starts one row / column later (oh * 2 instead of oh * 2 - 1)"""
    NB, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = torch.full((NB, H + 4, W + 4, C), -math.inf, dtype=x.dtype)
    xp[:, 1:H + 1, 1:W + 1] = x.cpu()
    o = 1 if defect == 'window_shift' else 0
    m = None
    for dy in range(3):
        for dx in range(3):
            v = xp[:, o + dy:o + dy + 2 * Ho:2, o + dx:o + dx + 2 * Wo:2][:, :Ho, :Wo]
            m = v if m is None else torch.maximum(m, v)          # torch.maximum propagates NaN
    return m


def relu(x: torch.Tensor) -> torch.Tensor:
    return torch.where(torch.isnan(x), x, x.clamp_min(0))


def ref_gelu(x):
    """0.5 x (1 + erff(x * 0.70710677f)): the argument product (u), erff (2 ulp of erf, plus erf' <= 2 / sqrt(pi) times the argument's
    error), the add, 0.5 x (exact) and the product -- on 0.5 |x| (1 + |erf|)"""
    xd = x.double().cpu()
    a = xd * INV_SQRT2
    er = torch.erf(a)
    y = 0.5 * xd * (1 + er)
    bnd = 0.5 * xd.abs() * (2 * ULP * er.abs() + 1.13 * gamma(2) * a.abs() + gamma(2) * (1 + er.abs())) + ATOL
    return y, bnd


# ------------------------------------------------------------------------------------------------ EFT: resize and grid-sample
def resize_positions(H, W, Ho, Wo, defect: Optional[str] = None):
    """fp32 source rows / columns and weights as resize_bilinear_ac_kernel: s = (H - 1) / (Ho - 1) (host, fp32), f = s * o, i0 = min((int)
    f, H - 1), i1 = min(i0 + 1, H - 1), l = f - i0, h = 1 - l.  defect 'xy_swap': the row scale on the columns and vice versa"""
    sh = np.float32(H - 1) / np.float32(Ho - 1) if Ho > 1 else np.float32(0)
    sw = np.float32(W - 1) / np.float32(Wo - 1) if Wo > 1 else np.float32(0)
    if defect == 'xy_swap':
        sh, sw = sw, sh

    def axis(s, n, no):
        f = np.float32(s) * np.arange(no, dtype=np.float32)
        i0 = np.minimum(f.astype(np.int64), n - 1)
        i1 = np.minimum(i0 + 1, n - 1)
        l = (f - i0.astype(np.float32)).astype(np.float32)
        return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(l.astype(np.float64)), torch.from_numpy((np.float32(1) - l).astype(np.float64))

    return axis(sh, H, Ho), axis(sw, W, Wo)


def ref_resize(x: torch.Tensor, Ho: int, Wo: int, defect: Optional[str] = None):
    """x [NB,H,W,C] -> [NB,Ho,Wo,C]: fp32 positions and weights, the blend hy (hx v00 + lx v01) + ly (hx v10 + lx v11) in fp64 with
    gamma(4) on the same blend of |v|"""
    NB, H, W, C = x.shape
    xd = x.double()
    (y0, y1, ly, hy), (x0, x1, lx, hx) = (tuple(t.to(xd.device) for t in a) for a in resize_positions(H, W, Ho, Wo, defect))

    def blend(v):
        r0, r1 = v[:, y0], v[:, y1]
        hx_, lx_ = hx.view(1, 1, Wo, 1), lx.view(1, 1, Wo, 1)
        a = hx_ * r0[:, :, x0] + lx_ * r0[:, :, x1]
        b = hx_ * r1[:, :, x0] + lx_ * r1[:, :, x1]
        return hy.view(1, Ho, 1, 1) * a + ly.view(1, Ho, 1, 1) * b

    return blend(xd), gamma(4) * blend(xd.abs()) + ATOL


def grid_weights(grid: torch.Tensor, H: int, W: int, defect: Optional[str] = None):
    """fp32 corner indices and corner weights as border_bilinear: i = (g + 1) .5 (W - 1), clipped to [0, W - 1] (border), floor, w1 = i - i0,
    w0 = 1 - w1, weights w0 w0' ... rounded in fp32; a corner past the last row / column has weight 0.  Defects: 'align_false'
    (((g + 1) W - 1) / 2), 'zeros_pad' (no clip: corners outside the image read zero)"""
    g = grid.float().cpu()
    gx, gy = g[..., 0], g[..., 1]
    if defect == 'align_false':
        ix, iy = ((gx + 1) * W - 1) / 2, ((gy + 1) * H - 1) / 2
    else:
        ix, iy = (gx + 1) * 0.5 * float(W - 1), (gy + 1) * 0.5 * float(H - 1)
    if defect != 'zeros_pad':
        ix, iy = ix.clamp(0, W - 1), iy.clamp(0, H - 1)
    fx0, fy0 = torch.floor(ix), torch.floor(iy)
    wx1, wy1 = ix - fx0, iy - fy0
    wx0, wy0 = 1 - wx1, 1 - wy1
    x0, y0 = fx0.long(), fy0.long()
    corners = []
    for dy, wy in ((0, wy0), (1, wy1)):
        for dx, wx in ((0, wx0), (1, wx1)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
            wgt = torch.where(ok, wx * wy, torch.zeros_like(wx)).double()
            corners.append((yi.clamp(0, H - 1), xi.clamp(0, W - 1), wgt))
    return corners


def ref_grid_sample(x: torch.Tensor, grid: torch.Tensor, defect: Optional[str] = None):
    """x [NB,H,W,C], grid [NB,M,2] -> [NB,M,C]: fp32 weights (``grid_weights``), fp64 blend, gamma(4) on sum |w||v|"""
    NB, H, W, C = x.shape
    xd = x.double()
    y = torch.zeros(NB, grid.shape[1], C, dtype=torch.float64, device=xd.device)
    A = torch.zeros_like(y)
    nb = torch.arange(NB, device=xd.device).view(NB, 1)
    for yi, xi, wgt in grid_weights(grid, H, W, defect):
        yi, xi, wgt = yi.to(xd.device), xi.to(xd.device), wgt.to(xd.device)
        v = xd[nb, yi, xi]
        y = y + wgt[..., None] * v
        A = A + wgt[..., None].abs() * v.abs()
    return y, gamma(4) * A + ATOL


# ------------------------------------------------------------------------------------------------ EFT: sequence attention
def seq_scale(E: int) -> float:
    """1.f / sqrtf((float)E) on the host"""
    return f32(np.float32(1) / np.sqrt(np.float32(E)))


def ref_seq_attention(qkv: torch.Tensor, S: int, B: int, E: int, defect: Optional[str] = None):
    """qkv [S,B,3E] -> [S,B,E] = softmax over the S positions of (q k^T) scale, times v.  Score chain: each lane's E / 128 float4 chunks
    (4 fmas each), 5 shuffles and the scale -> 4 ceil(E / 128) + 6 roundings; __expf's error grows with |s - max| (simt_fp64.expf_fast_rel); the
    denominator and the weighted sum run over S (simt_fp64._softmax_pv_bound).  Defects: 'scale_1_over_E', 'softmax_over_batch'."""
    q, k, v = (t.double().permute(1, 0, 2) for t in qkv.view(S, B, 3 * E).split(E, dim=-1))   # [B,S,E]
    sc = seq_scale(E) if defect != 'scale_1_over_E' else f32(1.0 / E)
    s = q @ k.transpose(1, 2) * sc
    sa = q.abs() @ k.abs().transpose(1, 2) * sc
    if defect == 'softmax_over_batch':                       # softmax over b for each (s, t) pair, then the weighted sum over t
        y = torch.softmax(s, dim=0) @ v
        return y.permute(1, 0, 2), torch.zeros_like(y).permute(1, 0, 2)
    y, bnd = _softmax_pv_bound(s, sa, 4 * _ceil_div(E, 128) + 6, v, S)
    return y.permute(1, 0, 2), bnd.permute(1, 0, 2)


# ------------------------------------------------------------------------------------------------ recorded launches
def _floats(a, *names):
    return tuple(float(a[n]) for n in names)


def _nulls(a, *names):
    return tuple(a[n] is None for n in names)


COEFS = ('c0', 'c1', 'c2', 'c3')
STEP_SCALARS = ('alpha', 'sigma', 'alpha_next', 'c', 'noise_scale')
LAMBDAS = ('lambda_color', 'lambda_sil', 'lambda_opacity')
ENTRIES = {
    'sfb_plms_update': ('plms_update', lambda a: dict(
        n=int(a['n']), nulls=_nulls(a, 'e1', 'e2', 'e3'), coefs=_floats(a, *COEFS), scalars=_floats(a, *STEP_SCALARS), clip=float(a['clip']),
        x0_out=a['x0_out'] is not None, e_out=a['e_out'] is not None)),
    'sfb_plms_update_rows': ('plms_update_rows', lambda a: dict(
        rows=int(a['rows']), row_len=int(a['row_len']), nulls=_nulls(a, 'e1', 'e2', 'e3'), coefs=_floats(a, *COEFS), clip=float(a['clip']),
        x0_out=a['x0_out'] is not None, row_scalars=tuple(a['row_scalars'].tolist()))),
    'sfb_plms_update_rows_cfg': ('plms_update_rows_cfg', lambda a: dict(
        rows=int(a['rows']), row_len=int(a['row_len']), nulls=_nulls(a, 'e1', 'e2', 'e3'), coefs=_floats(a, *COEFS),
        cond_scale=float(a['cond_scale']), clip=float(a['clip']), e_out=a['e_out'] is not None, row_scalars=tuple(a['row_scalars'].tolist()))),
    'sfb_photometric_loss': ('photometric_loss', lambda a: dict(h=a['h'], w=a['w'], scale=a['scale'], lam=_floats(a, *LAMBDAS))),
    'sfb_upsample2x_render': ('upsample2x_render', lambda a: dict(h=a['h'], w=a['w'])),
    'sfb_fusion_loss_ex': ('fusion_loss', lambda a: dict(h=a['h'], w=a['w'], mode=a['mode'], g_extra=a['g_extra'] is not None,
                                                         wgt=float(a['weight']), lam=_floats(a, *LAMBDAS))),
    'sfb_ddpm_dynamic_step': ('ddpm_dynamic_step', lambda a: dict(
        B=int(a['B']), row_len=int(a['row_len']), guided=a['e_null'] is not None, cond_scale=float(a['cond_scale']),
        scalars=_floats(a, *STEP_SCALARS), p=float(a['percentile']), s_out=a['s_out'] is not None, x0_out=a['x0_out'] is not None)),
    'sfb_maxpool3x3s2_nhwc': ('maxpool3x3s2', lambda a: dict(NB=a['NB'], H=a['H'], W=a['W'], C=a['C'])),
    'sfb_resize_bilinear_ac_nhwc': ('resize', lambda a: dict(NB=a['NB'], H=a['H'], W=a['W'], C=a['C'], Ho=a['Ho'], Wo=a['Wo'], ldx=int(a['ldx']),
                                                             ldo=int(a['ldo']))),
    'sfb_grid_sample_nhwc': ('grid_sample', lambda a: dict(NB=a['NB'], H=a['H'], W=a['W'], C=a['C'], M=int(a['M']), ldx=int(a['ldx']),
                                                           ldo=int(a['ldo']))),
    'sfb_seq_attention': ('seq_attention', lambda a: dict(S=a['S'], B=a['B'], E=a['E'])),
    'sfb_act_inplace': ('act', lambda a: dict(n=int(a['n']), kind=a['kind'])),
}


def entry(r) -> Optional[Dict]:
    """the replay entry (tests/test_step_fp64_gpu.py) of an oracle/insitu ``Call`` of a sampler update, a distillation loss kernel or an
    EFT-only kernel, its arguments read by parameter name: geometry, strides, the scalars, each row's five step scalars and which optional
    pointers are NULL (None for any other launch)"""
    if r.op not in ENTRIES:
        return None
    op, fields = ENTRIES[r.op]
    return dict(fields(r.args), op=op, family=r.family, label='recorded')
