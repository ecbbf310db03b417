"""oracle/simt_fp64.py -- launch plans, fp64 references and per-element error bounds of the SIMT kernels of the UNet, the VAE and
LPIPS (sparsefusion_b200/csrc/unet_ops.cu, csrc/lpips_ops.cu).

TEST INFRASTRUCTURE ONLY.

``kernel_plan`` restates the host dispatch of sfb_groupnorm_nhwc, sfb_mq_attention, sfb_gca_pool and sfb_linear_small line by line;
the GPU tests hold it to the kernels the tracer names.

Every ``ref_*`` returns (y, bound): y is the operation in fp64, bound the per-element tolerance of the kernel's fp32 result,
    |got - y| <= rho * A + slack,
where A is the absolute companion (the same computation on |operands|), rho is built from gamma(n) (``field_fp64.gamma``: n chained fp32
roundings of u = 2^-24, Higham sec. 3.1) for the longest chain the kernel runs, and slack carries the terms that are not proportional to A
(statistics, exponentials, the argument error of sin / cos).  Each bound is derived next to its reference.

Transcendentals, from the CUDA C++ Programming Guide (intrinsic and single-precision function tables):
    __expf(x)  2 + floor(|1.173 x|) ulp          expf(x)  2 ulp          sinf / cosf  2 ulp          erff  2 ulp          rsqrtf  2 ulp
An ulp of a normal fp32 result is at most 2^-23 of its magnitude.

'tf32' mode: outputs that feed a tensor-core GEMM are rounded to TF32 (cvt.rna) on write, half a TF32 ulp: 2^-11 of the value on top.

``emulate_*`` evaluate the kernels' arithmetic in fp32 (torch on the CPU) in their fold orders, with switches that inject single defects; the
host tests use them to show what the bounds see.

``entry`` turns an oracle/insitu record of a front end, or a call of an LPIPS entry point, into the geometry and memory layout
tests/test_simt_fp64_gpu.py replays.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .conv_fp64 import nhwc_meta, rows_meta, same_ptr
from .field_fp64 import ATOL, U32 as U, gamma

ULP = 2.0 ** -23          # one ulp of a normal fp32 value, relative to it
TF32_HALF = 2.0 ** -11    # cvt.rna.tf32.f32
LPIPS_NAMES = {'sfb_lpips_prep': 'lpips_prep', 'sfb_lpips_prep_backward': 'lpips_prep_backward', 'sfb_relu_nhwc': 'relu',
               'sfb_maxpool2x2_nhwc': 'maxpool', 'sfb_maxpool2x2_relu_backward_nhwc': 'maxpool_bwd', 'sfb_add_relu_mask': 'add_relu_mask',
               'sfb_lpips_head': 'lpips_head'}


def expf_fast_rel(x: torch.Tensor) -> torch.Tensor:
    """relative error of __expf at x"""
    return (2 + torch.floor((1.173 * x).abs())) * ULP


def _tf32(bnd: torch.Tensor, y: torch.Tensor, precision: str, rounded: bool = True) -> torch.Tensor:
    if precision == 'tf32' and rounded:
        return bnd + TF32_HALF * (y.abs() + bnd)
    return bnd


def is_tf32(t: torch.Tensor) -> bool:
    """every finite element has its 13 low mantissa bits clear"""
    i = t.float().contiguous().view(torch.int32)
    return bool(((i & 0x1FFF) == 0).all())


# ------------------------------------------------------------------------------------------------ launch plans
def _ceil_div(a, b):
    return -(-a // b)


def kernel_plan(op: str, geometry: Dict, sm_count: int = 132, fusion_mask: int = 0x7fffffff, precision: str = 'tf32x3') -> Dict:
    """the launches the host makes for ``op`` (unet_ops.cu line numbers in the comments); ``kernels`` lists the traced names in order"""
    g = geometry
    if op == 'groupnorm':
        NB, HW, C, G = g['NB'], g['HW'], g['C'], g['G']
        C4, Cg = C // 4, C // G
        # :1155-1172
        if (fusion_mask & 4) and Cg % 16 == 0 and HW >= 1 and NB <= 4 and NB * HW * C <= (1 << 20):
            k = 8
            while k > 1 and k > HW:
                k >>= 1
            per_cta = _ceil_div(HW, k) * (Cg // 4)
            items = _ceil_div(per_cta, 256)
            if items <= 16:
                it = 4 if items <= 4 else (8 if items <= 8 else 16)
                return dict(path='cluster', k=k, items=items, ITEMS=it, kernels=[f'gn_cluster_kernel<{it}>'])
        # :1174 (rows_ok: no group crosses a 256-column pass)
        rows_ok = Cg % 4 == 0 and ((256 % C4 == 0) if C4 <= 256 else (C4 % 256 == 0 and 256 % (Cg // 4) == 0))
        if g.get('legacy_rows_gate'):          # the gate before the straddling groups were excluded (host tests only)
            rows_ok = Cg % 4 == 0 and ((256 % C4 == 0) if C4 <= 256 else C4 % 256 == 0) and Cg // 4 <= min(C4, 256)
        S = 1
        if rows_ok:                                                           # :1176-1183
            rpi = 256 // min(C4, 256)
            want = (2 * sm_count + NB - 1) // NB
            S = max(1, min(HW // (rpi * 2), want, 256))
            stats = 'gn_stats_rows_kernel'
        else:                                                                 # :1185-1186
            while S < 64 and G * NB * S * 2 <= sm_count * 2 and HW // (S * 2) >= 8:
                S *= 2
            stats = 'gn_stats_kernel'
        apply = 'gn_apply_cols_kernel' if (C4 <= 256 and 256 % C4 == 0) else 'gn_apply_kernel'     # :1194
        return dict(path='two-launch', rows=rows_ok, S=S, stats=stats, apply=apply, kernels=[stats, apply])
    if op == 'mq_attention':
        n, nc, dh, heads, B = g['n'], g['nc'], g['dh'], g['heads'], g['B']
        nk = nc + 1 + n
        smk = (nk * (2 * dh + 4) + 8 * ((nk + 31) & ~31) + 8 * dh) * 4       # :1245
        sm2 = (nk * 2 * dh + 8 * nk) * 4                                      # :1257
        if nk > 64 and dh % 4 == 0 and dh <= 128 and smk <= 200 * 1024:      # :1244-1246
            qpw = max(1, _ceil_div(heads * n * B, 8 * sm_count))              # :1248
            return dict(nk=nk, smk=smk, sm2=sm2, qpw=qpw, kernel='keys', kernels=['mq_attention_keys_kernel'])
        if dh % 4 == 0 and dh <= 128 and sm2 <= 160 * 1024:                  # :1258
            return dict(nk=nk, smk=smk, sm2=sm2, qpw=1, kernel='smem', kernels=['mq_attention_smem_kernel'])
        sm = 4 * nk * 4                                                       # :1265-1267
        return dict(nk=nk, smk=smk, sm2=sm2, qpw=1, kernel='plain', fits=sm <= 48 * 1024, kernels=['mq_attention_kernel'])
    if op == 'gca_pool':
        HW, C = g['HW'], g['C']
        if HW >= 4096:                                                        # :1288-1291
            sms = ((((HW + 7) // 8 + 4) & ~3) + 64 * 16) * 4
            return dict(split=True, Z=8, smem=sms, fits=sms <= 200 * 1024, kernels=['gca_logits_kernel', 'gca_pool_split_kernel'])
        sm = (((HW + 3) & ~3) + 64 * 16) * 4                                  # :1297-1298
        return dict(split=False, Z=1, smem=sm, fits=sm <= 200 * 1024, kernels=['gca_logits_kernel', 'gca_pool_kernel'])
    if op == 'linear_small':
        MT = 2 if g['M'] <= 2 else 8                                          # :1220
        return dict(MT=MT, smem=MT * g['K'] * 4, kernels=[f'linear_small_kernel<{MT}>'])
    raise KeyError(op)


# ------------------------------------------------------------------------------------------------ GroupNorm (+ FiLM, SiLU)
def stat_chain(plan: Dict) -> int:
    """fp32 roundings in one thread's partial sum before it is promoted to fp64: a float4's sum of squares is 4 products and 3 adds in the
    stats kernels (:158-159, :208-209; the scalar path rounds one product); gn_cluster_kernel keeps s / ss in float over ITEMS float4
    (:261-262): 2 + 2 roundings per item, 4 ITEMS in all"""
    return 4 * plan['ITEMS'] if plan['path'] == 'cluster' else 4


def _silu_bound(z, dz):
    """|silu_f(z~) - silu(z)| for |z~ - z| <= dz: silu' is below 1.1 in magnitude; silu_f = z / (1 + __expf(-z)) rounds the sum and the
    quotient (2 u) and carries __expf's error through e / (1 + e) = 1 - sigmoid"""
    sig = torch.sigmoid(z)
    return 1.1 * dz + (z.abs() * sig) * (expf_fast_rel(-z) * (1 - sig) + 2 * U) + ATOL


def ref_groupnorm(x, G, gamma_, beta, film, act, plan, precision='tf32x3', eps=1e-5):
    """x [NB,HW,C]; film [NB,2C] or None.  y = act(((x - mu) r gamma + beta)(s + 1) + h), r = 1 / sqrt(var + eps).

    Statistics: each partial sum is an fp32 chain of ``stat_chain`` roundings, the rest is folded in fp64, so
        |d mu| <= g_s E|x|,   |d var| <= g_s E[x^2] + 2 |mu| |d mu|  (E[x^2] = var + mu^2: the (1 + mu^2 / var) amplification of the
    one-pass variance); d r / r <= |d var| / (2 (var + eps)) + u (the float cast), and the float cast of mu adds u |mu|.
    Element: (x - mu_f) r_f gamma + beta, then (s + 1) and + h -- at most 7 roundings on the magnitudes (gn_apply_cols folds
    a = r gamma (s + 1) and b = beta (s + 1) + h first: also 7 along any path)."""
    xd = x.double()
    NB, HW, C = xd.shape
    Cg = C // G
    xg = xd.view(NB, HW, G, Cg)
    mu = xg.mean(dim=(1, 3))
    var = xg.var(dim=(1, 3), unbiased=False)
    m1 = xg.abs().mean(dim=(1, 3))
    m2 = (xg * xg).mean(dim=(1, 3))
    r = 1.0 / torch.sqrt(var + eps)
    gs = gamma(stat_chain(plan) + 1) + 2.0 ** -40
    dmu = gs * m1 + U * mu.abs()
    dvar = gs * m2 + 2 * mu.abs() * gs * m1
    dr = dvar / (2 * (var + eps)) + 2 * U
    ex = lambda t: t.repeat_interleave(Cg, dim=1)[:, None, :]          # [NB, 1, C]
    mu_c, r_c, dmu_c, dr_c = ex(mu), ex(r), ex(dmu), ex(dr)
    gm, bt = gamma_.double()[None, None], beta.double()[None, None]
    if film is not None:
        sc = film.double()[:, None, :C] + 1
        sh = film.double()[:, None, C:]
    else:
        sc = torch.ones(NB, 1, C, dtype=torch.float64, device=xd.device)
        sh = torch.zeros_like(sc)
    nrm = (xd - mu_c) * r_c
    z = (nrm * gm + bt) * sc + sh
    A = ((xd.abs() + mu_c.abs()) * r_c * gm.abs() + bt.abs()) * sc.abs() + sh.abs()
    dz = gamma(7) * A + r_c * gm.abs() * sc.abs() * (dmu_c + (xd - mu_c).abs() * dr_c)
    if act:
        y = F.silu(z)
        b = _silu_bound(z, dz)
    else:
        y, b = z, dz + ATOL
    return y, _tf32(b, y, precision)


def gn_partials(x: torch.Tensor, G: int, plan: Dict, defect: Optional[str] = None) -> torch.Tensor:
    """[NB, G, S, 2] fp64 partial (sum, sumsq) pairs as the stats kernels write them, NaN where no CTA writes (the tests' workspace is
    NaN-filled).  x [NB,HW,C] fp32.  gn_stats_rows_kernel's bookkeeping is followed literally (:196-223): the CTA of slab sl sums, per
    256-column pass, thread columns tc = 0..cols-1, and thread t < cols / Cg4 writes group pass * gpp + t from columns t Cg4 .. t Cg4 + Cg4 - 1
    of the pass.  defect 'lost_slab': slab S - 1 of group 0 is never written."""
    NB, HW, C = x.shape
    S = plan['S']
    out = torch.full((NB, G, S, 2), float('nan'), dtype=torch.float64)
    xf = x.float()
    C4, Cg = C // 4, C // G
    v4 = xf.view(NB, HW, C4, 4)
    s4 = ((v4[..., 0] + v4[..., 1]) + v4[..., 2]) + v4[..., 3]            # fp32 per float4 (order immaterial within the bound)
    q4 = v4 * v4
    ss4 = ((q4[..., 0] + q4[..., 1]) + q4[..., 2]) + q4[..., 3]
    for sl in range(S):
        p0, p1 = (HW * sl) // S, (HW * (sl + 1)) // S
        cs, css = s4[:, p0:p1].double().sum(1), ss4[:, p0:p1].double().sum(1)      # [NB, C4]: per float4 column, fp64
        if plan['stats'] == 'gn_stats_rows_kernel':
            Cg4 = Cg // 4
            cols = min(C4, 256)
            passes = 1 if C4 < 256 else C4 // 256
            gpp = cols // Cg4
            for ps in range(passes):
                for t in range(gpp):
                    c0 = ps * 256 + t * Cg4
                    gi = ps * gpp + t
                    if gi < G:
                        out[:, gi, sl, 0] = cs[:, c0:c0 + Cg4].sum(1)
                        out[:, gi, sl, 1] = css[:, c0:c0 + Cg4].sum(1)
        else:
            xs = xf[:, p0:p1].view(NB, p1 - p0, G, Cg)
            out[:, :, sl, 0] = xs.double().sum(dim=(1, 3))
            out[:, :, sl, 1] = (xs * xs).double().sum(dim=(1, 3))
    if defect == 'lost_slab':
        out[:, 0, S - 1] = float('nan')
    return out


def emulate_groupnorm(x, G, gamma_, beta, film, act, plan, eps=1e-5, defect: Optional[str] = None):
    """fp32 result of the two-launch path (or the cluster path: the same statistics with a single slab).  defects: 'lost_slab',
    'wrong_group' (gn_apply_kernel's channel c + k takes the group of c, wrong when 4 does not divide Cg), 'film_no_plus1'"""
    NB, HW, C = x.shape
    Cg = C // G
    p = plan if plan['path'] == 'two-launch' else dict(plan, S=1, stats='gn_stats_kernel')
    part = gn_partials(x, G, p, defect if defect == 'lost_slab' else None)
    tot = part.sum(2)                                                      # fp64 fold
    cnt = HW * Cg
    mean = tot[..., 0] / cnt
    var = (tot[..., 1] / cnt - mean * mean).clamp_min(0)
    mu_f, r_f = mean.float(), (1.0 / torch.sqrt(var + eps)).float()
    cidx = torch.arange(C)
    grp = cidx // Cg
    if defect == 'wrong_group':
        grp = ((cidx // 4) * 4) // Cg
    mu_c, r_c = mu_f[:, grp][:, None], r_f[:, grp][:, None]
    o = (x.float() - mu_c) * r_c * gamma_.float() + beta.float()
    if film is not None:
        sc = film.float()[:, None, :C]
        o = o * (sc if defect == 'film_no_plus1' else sc + 1) + film.float()[:, None, C:]
    if act:
        o = o / (1 + torch.exp(-o))
    return o


# ------------------------------------------------------------------------------------------------ attention
def _softmax_pv_bound(s, s_abs, n_s, v, nk_chain):
    """scores s [.., nk] (fp64), |q| |k| companions s_abs, values v [.., nk, dh]: (out, bound) of softmax(s) v with fp32 scores of
    n_s roundings.  e_j = __expf(s_j - m) errs by  g(n_s) (s_abs_j + s_abs_max) + u |s_j - m| (the subtraction)  in the argument and
    expf_fast_rel(s_j - m) in the value; the denominator is a chain of nk_chain adds and 1 / den one rounding, P.V a chain of nk_chain
    products (plus the inv scaling: 2 roundings)."""
    m = s.max(dim=-1, keepdim=True).values
    p = torch.softmax(s, dim=-1)
    gs = gamma(n_s)
    amax = torch.gather(s_abs, -1, s.argmax(dim=-1, keepdim=True))
    delta = gs * (s_abs + amax) + U * (s - m).abs() + expf_fast_rel(s - m)
    delta = delta * torch.exp(delta)                                       # first order -> exact for e^delta - 1
    y = p @ v
    A = p @ v.abs()
    den = (p * delta).sum(-1, keepdim=True) + gamma(nk_chain + 1)
    bnd = (p * delta) @ v.abs() + A * (den + gamma(nk_chain + 3)) * (1 + den)
    return y, bnd + ATOL


def mq_keys(q, kv, null_kv, ckv, heads, dh):
    """(qs [B,heads,n,dh], k [B,nk,dh], v [B,nk,dh]) fp64 in the kernel's key order: context, null, tokens"""
    B, n = q.shape[0], q.shape[1]
    qd = q.double().view(B, n, heads, dh).transpose(1, 2)
    k, v = kv.double().view(B, n, 2, dh).unbind(2)
    nk_ = null_kv.double()
    k = torch.cat((nk_[0].expand(B, 1, dh), k), 1)
    v = torch.cat((nk_[1].expand(B, 1, dh), v), 1)
    if ckv is not None and ckv.shape[1] > 0:
        ck, cv = ckv.double().view(B, -1, 2, dh).unbind(2)
        k, v = torch.cat((ck, k), 1), torch.cat((cv, v), 1)
    return qd, k, v


def ref_mq_attention(q, kv, null_kv, ckv, heads, dh, plan, precision='tf32x3'):
    """out [B,n,heads*dh].  Score chain: q scale (1) and one product per term, then the kernel's adds -- plain: dh / 32 per lane + 5
    shuffles; smem: 4 + 5; keys: two dh / 8 chains of pairs + 1.  dh + 8 bounds all three.  Denominator and P.V: nk adds (plain and
    smem) -- the keys kernel sums nk / 32 per lane + 5."""
    B, n = q.shape[0], q.shape[1]
    scale = float(torch.tensor(dh ** -0.5, dtype=torch.float32))
    qd, k, v = mq_keys(q, kv, null_kv, ckv, heads, dh)
    s = torch.einsum('bhid,bjd->bhij', qd * scale, k)
    sa = torch.einsum('bhid,bjd->bhij', qd.abs() * scale, k.abs())
    y, bnd = _softmax_pv_bound(s, sa, dh + 8, v[:, None], plan['nk'] + 5)
    y = y.transpose(1, 2).reshape(B, n, heads * dh)
    bnd = bnd.transpose(1, 2).reshape(B, n, heads * dh)
    return y, _tf32(bnd, y, precision)


def ref_cross_attention(q, kvc, null_kv, heads, dh, precision='tf32x3'):
    """keys: null, then the context tokens' per-head slices (:805-827); chains as the plain kernel"""
    B, n = q.shape[0], q.shape[1]
    nc = kvc.shape[1]
    inner = heads * dh
    scale = float(torch.tensor(dh ** -0.5, dtype=torch.float32))
    qd = q.double().view(B, n, heads, dh).transpose(1, 2)
    k, v = kvc.double().view(B, nc, 2, heads, dh).unbind(2)
    k, v = k.transpose(1, 2), v.transpose(1, 2)
    nk_ = null_kv.double()
    k = torch.cat((nk_[0].expand(B, heads, 1, dh), k), 2)
    v = torch.cat((nk_[1].expand(B, heads, 1, dh), v), 2)
    s = torch.einsum('bhid,bhjd->bhij', qd * scale, k)
    sa = torch.einsum('bhid,bhjd->bhij', qd.abs() * scale, k.abs())
    y, bnd = _softmax_pv_bound(s, sa, dh + 8, v, nc + 6)
    y = y.transpose(1, 2).reshape(B, n, inner)
    bnd = bnd.transpose(1, 2).reshape(B, n, inner)
    return y, _tf32(bnd, y, precision)


def emulate_mq_attention(q, kv, null_kv, ckv, heads, dh, defect: Optional[str] = None):
    """fp32 plain-kernel arithmetic.  defects: 'drop_null' (the null key is never staged), 'swap_order' (keys staged null, context, tokens
    while the values stay context, null, tokens)"""
    qd, k, v = mq_keys(q, kv, null_kv, ckv, heads, dh)
    nc = 0 if ckv is None else ckv.shape[1]
    if defect == 'drop_null':
        keep = [j for j in range(k.shape[1]) if j != nc]
        k, v = k[:, keep], v[:, keep]
    if defect == 'swap_order' and nc:
        perm = [nc] + list(range(nc)) + list(range(nc + 1, k.shape[1]))
        k = k[:, perm]
    scale = torch.tensor(dh ** -0.5, dtype=torch.float32)
    s = torch.einsum('bhid,bjd->bhij', (qd.float() * scale), k.float())
    e = torch.exp(s - s.max(-1, keepdim=True).values)
    p = e * (1.0 / e.sum(-1, keepdim=True))
    y = torch.einsum('bhij,bjd->bhid', p, v.float())
    B, n = q.shape[0], q.shape[1]
    return y.transpose(1, 2).reshape(B, n, heads * dh)


# ------------------------------------------------------------------------------------------------ GlobalContext pooling
def ref_gca_pool(x, wk, bk, plan):
    """x [NB,HW,C]; pooled [NB,C] = softmax_p(x wk + bk) x.  Logit chain: per lane C / 128 float4 steps of 5 roundings, 5 shuffles, the
    bias: C / 16 + 8 bounds it.  Softmax weights: __expf(l - M) as in attention; the sum is HW / 256 + 13 adds.  Pooled: HW / 64 FMAs per
    thread, a 64-row fold, the 1 / den scaling (HW / 64 + 66).  The split kernel adds the Z-way merge: __expf(m_z - M) errs by
    expf_fast_rel(m_z - M) <= expf_fast_rel(l_p - M) for every pixel p of slab z (m_z >= l_p), and S, A chains of Z = 8 adds."""
    xd = x.double()
    NB, HW, C = xd.shape
    l = xd @ wk.double().reshape(C) + bk.double().reshape(())
    la = xd.abs() @ wk.double().abs().reshape(C) + bk.double().abs().reshape(())
    chain = HW // 64 + 66 + (2 * plan['Z'] + 2 if plan['split'] else 0)
    y, bnd = _softmax_pv_bound(l[:, None], la[:, None], C // 16 + 8, xd, chain)
    y, bnd = y[:, 0], bnd[:, 0]
    if plan['split']:
        pe = torch.softmax(l, -1) * expf_fast_rel(l - l.max(-1, keepdim=True).values)
        A = torch.einsum('bp,bpc->bc', torch.softmax(l, -1), xd.abs())
        bnd = bnd + 2 * (torch.einsum('bp,bpc->bc', pe, xd.abs()) + pe.sum(-1, keepdim=True) * A)
    return y, bnd


def emulate_gca_pool(x, wk, bk, Z: int = 8, defect: Optional[str] = None):
    """fp32 split-kernel arithmetic: per slab (m_z, s_z, a_z), merged with __expf(m_z - M).  defects: 'lost_pixel' (the last pixel of slab
    0 is skipped), 'merge_sign' (the merge scales by e^(M - m_z))"""
    xf = x.float()
    NB, HW, C = xf.shape
    l = xf @ wk.float().reshape(C) + bk.float().reshape(())
    ms, ss, As = [], [], []
    for z in range(Z):
        p0, p1 = (HW * z) // Z, (HW * (z + 1)) // Z
        if defect == 'lost_pixel' and z == 0:
            p1 -= 1
        lz = l[:, p0:p1]
        mz = lz.max(-1).values
        e = torch.exp(lz - mz[:, None])
        ms.append(mz)
        ss.append(e.sum(-1))
        As.append(torch.einsum('bp,bpc->bc', e, xf[:, p0:p1]))
    M = torch.stack(ms, 1).max(1).values
    S = torch.zeros(NB)
    A = torch.zeros(NB, C)
    for mz, sz, az in zip(ms, ss, As):
        f = torch.exp((M - mz) if defect == 'merge_sign' else (mz - M))
        S = S + sz * f
        A = A + az * f[:, None]
    return A / S[:, None]


# ------------------------------------------------------------------------------------------------ rows: softmax, LayerNorm, linear
def ref_softmax_rows(x, scale):
    """softmax(scale x) per row with expf (2 ulp): argument error u (|x s| + |m| + |x s - m|), value 2 ulp; the sum is cols / 256 + 13
    adds; y = e / den: 2 roundings"""
    xd = x.double() * float(scale)
    m = xd.max(-1, keepdim=True).values
    y = torch.softmax(xd, -1)
    delta = U * (xd.abs() + m.abs() + (xd - m).abs()) + 2 * ULP
    delta = delta * torch.exp(delta)
    den = (y * delta).sum(-1, keepdim=True) + gamma(x.shape[-1] // 256 + 14)
    return y, y * (delta + den + gamma(2)) * (1 + den) + ATOL


def ref_layernorm(x, g, b, res, pre_gelu, round_out, precision='tf32x3'):
    """y = LN(pre(x)) g (+ b) (+ res), eps 1e-5, two-pass fp32 statistics over one 128-thread row.
    pre = GELU: 0.5 v (1 + erff(v / sqrt 2)), erff 2 ulp: |d v| <= |v| (2^-23 + 3 u).
    mean: C / 128 + 5 + 3 adds and / C: g_m = gamma(C / 128 + 10); var = sum (v - mean)^2 / C with d = v - mean exact but for 1 rounding and
    |d mean| + |d v|: |d var| <= g_m var + 2 E|d| (|d mean| + max |d v|) + 2 u var; r = rsqrtf(var + eps): 2 ulp + |d var| / (2 (var + eps)).
    Element: (v - mean) r g + b + res: 5 roundings on the magnitudes."""
    xd = x.double()
    C = xd.shape[-1]
    if pre_gelu:
        v = F.gelu(xd)
        dv = xd.abs() * (ULP + 3 * U)
    else:
        v, dv = xd, torch.zeros_like(xd)
    mean = v.mean(-1, keepdim=True)
    d = v - mean
    var = (d * d).mean(-1, keepdim=True)
    gm = gamma(C // 128 + 10)
    dmean = gm * v.abs().mean(-1, keepdim=True) + dv.mean(-1, keepdim=True)
    dvmax = dv.max(-1, keepdim=True).values
    dvar = gm * var + 2 * d.abs().mean(-1, keepdim=True) * (dmean + dvmax) + (dmean + dvmax) ** 2 + 2 * U * var
    r = 1.0 / torch.sqrt(var + 1e-5)
    dr = dvar / (2 * (var + 1e-5)) + 2 * ULP + 2 * U
    gd = g.double().reshape(-1)
    y = d * r * gd
    A = (v.abs() + mean.abs()) * r * gd.abs()
    if b is not None:
        y = y + b.double()
        A = A + b.double().abs()
    if res is not None:
        y = y + res.double()
        A = A + res.double().abs()
    bnd = gamma(5) * A + r * gd.abs() * (d.abs() * dr + dmean + dv) * (1 + dr) + ATOL
    return y, _tf32(bnd, y, precision, round_out)


def _sigmoid_bound(z, dz):
    sig = torch.sigmoid(z)
    return 0.25 * dz + sig * (expf_fast_rel(-z) * (1 - sig) + 2 * U) + ATOL


def ref_linear_small(x, w, bias, res, pre, post, round_out, precision='tf32x3'):
    """y = post(bias + pre(x) W^T) (+ res).  Dot chain: K / 128 float4 steps of 4 roundings per lane (or K / 32 FMAs), 5 shuffles and the
    bias: K / 32 + 8.  pre = SiLU adds its own error times |W|; post = SiLU / sigmoid as in ``_silu_bound``."""
    xd = x.double()
    if pre == 1:
        a = F.silu(xd)
        sig = torch.sigmoid(xd)
        da = xd.abs() * sig * (expf_fast_rel(-xd) * (1 - sig) + 2 * U)
    else:
        a, da = xd, torch.zeros_like(xd)
    wd = w.double()
    z = a @ wd.T
    A = a.abs() @ wd.abs().T
    if bias is not None:
        z = z + bias.double()
        A = A + bias.double().abs()
    K = x.shape[-1]
    dz = gamma(K // 32 + 8) * A + da @ wd.abs().T
    if post == 1:
        y, bnd = F.silu(z), _silu_bound(z, dz)
    elif post == 2:
        y, bnd = torch.sigmoid(z), _sigmoid_bound(z, dz)
    else:
        y, bnd = z, dz + ATOL
    if res is not None:
        y = y + res.double()
        bnd = bnd + U * (y.abs() + bnd)
    return y, _tf32(bnd, y, precision, round_out)


def ref_gate_mlp_residual(h, hid, w2, b2, res):
    """out = h sigmoid(b2 + W2 hid) + res: the gate's dot is Hd / 32 + 8 roundings (as linear_small), then one FMA"""
    z = hid.double() @ w2.double().T + b2.double()
    A = hid.double().abs() @ w2.double().abs().T + b2.double().abs()
    gte = torch.sigmoid(z)
    dg = _sigmoid_bound(z, gamma(w2.shape[1] // 32 + 8) * A)
    hd, rd = h.double(), res.double()
    y = hd * gte[:, None, :] + rd
    return y, hd.abs() * dg[:, None, :] + gamma(2) * (hd.abs() * gte[:, None, :] + rd.abs()) + ATOL


def ref_gate_residual(h, gate, res):
    """out = h gate + res (or h + res): at most 2 roundings"""
    hd, rd = h.double(), res.double()
    g = gate.double()[:, None, :] if gate is not None else torch.ones_like(hd[:, :1])
    y = hd * g + rd
    return y, gamma(2) * (hd.abs() * g.abs() + rd.abs()) + ATOL


def ref_time_fourier(t, w):
    """[t, sin f, cos f], f = 2 pi t w computed as ((t w) 2) pi_f: 2 roundings and pi's fp32 rounding, so f carries an ABSOLUTE error of
    gamma(3) |f|, which passes unchanged through sin and cos; then 2 ulp of a result below 1"""
    td, wd = t.double(), w.double()
    f = td[:, None] * wd[None, :] * (2 * math.pi)
    y = torch.cat((td[:, None], torch.sin(f), torch.cos(f)), 1)
    df = gamma(3) * f.abs() + 2 * ULP
    bnd = torch.cat((torch.zeros_like(td[:, None]), df, df), 1) + ATOL
    return y, bnd


def ref_pixel_shuffle_silu(y):
    """y [NB,H,W,4 Co] -> [NB,2H,2W,Co] silu, channel c*4 + i*2 + j"""
    yd = y.double()
    NB, H, W, C4 = yd.shape
    o = F.pixel_shuffle(yd.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    return F.silu(o), _silu_bound(o, torch.zeros_like(o))


# ------------------------------------------------------------------------------------------------ exact ops (compared bit for bit)
def upsample2x(x, defect: Optional[str] = None):
    """nearest x2, NHWC; defect 'off_by_one': output row oh reads input row (oh + 1) >> 1 (clamped)"""
    NB, H, W, C = x.shape
    r = torch.arange(2 * H) >> 1 if defect != 'off_by_one' else ((torch.arange(2 * H) + 1) >> 1).clamp(max=H - 1)
    c = torch.arange(2 * W) >> 1
    return x[:, r.to(x.device)][:, :, c.to(x.device)]


def im2col4(x, KH, KW, pad, ldo):
    NB, H, W, _ = x.shape
    xp = F.pad(x.permute(0, 3, 1, 2), (pad, KW - 1 - pad, pad, KH - 1 - pad))
    cols = [xp[:, :, ky:ky + H, kx:kx + W] for ky in range(KH) for kx in range(KW)]
    out = torch.stack(cols, 1).permute(0, 3, 4, 1, 2).reshape(NB, H, W, KH * KW * 4)
    return F.pad(out, (0, ldo - KH * KW * 4))


def maxpool2x2(x):
    NB, H, W, C = x.shape
    return x.view(NB, H // 2, 2, W // 2, 2, C).amax(dim=(2, 4))


def maxpool2x2_relu_backward(x, gy, defect: Optional[str] = None):
    """x [H,W,C] post-ReLU, gy [H/2,W/2,C]: the window's gradient goes to its FIRST maximum in row-major order when that maximum is
    positive; defect 'last_max' picks the last one"""
    H, W, C = x.shape
    win = x.view(H // 2, 2, W // 2, 2, C).permute(0, 2, 4, 1, 3).reshape(H // 2, W // 2, C, 4)
    if defect == 'last_max':
        arg = 3 - win.flip(-1).argmax(-1)
    else:
        arg = (win == win.max(-1, keepdim=True).values).float().argmax(-1)      # first occurrence
    best = win.max(-1).values
    g = torch.where(best > 0, gy, torch.zeros_like(gy))
    out = torch.zeros_like(win)
    out.scatter_(-1, arg[..., None], g[..., None])
    return out.view(H // 2, W // 2, C, 2, 2).permute(0, 3, 1, 4, 2).reshape(H, W, C)


def add_relu_mask(g, g_head, act):
    v = g if g_head is None else g + g_head
    return torch.where(act > 0, v, torch.zeros_like(v))


# ------------------------------------------------------------------------------------------------ LPIPS head
def ref_lpips_head(f0, f1, w, eps_mode: str = 'kernel'):
    """f0, f1 [HW,C], w [C] >= 0.  n = f / (r + 1e-10), value = sum_p sum_c w (n0 - n1)^2 / HW,
    g = d value / d f0 = dn / (r0 + e) - f0 (f0 . dn) / (r0 (r0 + e)^2) with dn = 2 w (n0 - n1) / HW; the second term is 0 when r0 = 0.
    Returns (value, value bound, g, g bound).

    r = sqrtf(sum f^2): the sum is C / 128 float4 steps of 8 roundings per lane + 5 shuffles, sqrt and +eps and 1/ three more, so
    i = 1 / (r + e) errs by g_r = gamma(C / 16 + 16) relative.  d = f0 i0 - f1 i1: 3 roundings on |n0| + |n1| plus both i's errors.
    value per pixel: w d^2 chain of C / 32 + 5 and the atomics' order (HW / 8 CTAs and 8 warps: HW / 8 + 16 adds): bound on the
    companion sum w (|n0| + |n1|)^2 with 2 (g_r + gamma(3)) + gamma(C / 32 + HW / 8 + 24).
    gradient: dn i0 and f0 (f0 . dn) i0^2 / r0 -- the dot has the same chain as the value; 8 roundings per element on top."""
    f0d, f1d, wd = f0.double(), f1.double(), w.double()
    HW, C = f0d.shape
    e = 1e-10
    r0, r1 = f0d.norm(dim=1, keepdim=True), f1d.norm(dim=1, keepdim=True)
    i0, i1 = 1 / (r0 + e), 1 / (r1 + e)
    n0, n1 = f0d * i0, f1d * i1
    d = n0 - n1
    val = (wd * d * d).sum() / HW
    gr = gamma(C // 16 + 16)
    dd = (n0.abs() + n1.abs()) * (gr + gamma(3))
    val_abs = (wd * (n0.abs() + n1.abs()) ** 2).sum() / HW
    vb = 2 * (wd * (n0.abs() + n1.abs()) * dd).sum() / HW + gamma(C // 32 + HW // 8 + 24) * val_abs + ATOL
    dn = 2 * wd * d / HW
    dot = (f0d * dn).sum(1, keepdim=True)
    k2 = torch.where(r0 > 0, dot * i0 * i0 / r0.clamp_min(1e-300), torch.zeros_like(r0))
    g = dn * i0 - f0d * k2
    dn_abs = 2 * wd * (n0.abs() + n1.abs()) / HW
    ddn = 2 * wd * dd / HW + gamma(3) * dn_abs
    dot_abs = (f0d.abs() * dn_abs).sum(1, keepdim=True)
    ddot = (f0d.abs() * ddn).sum(1, keepdim=True) + gamma(C // 32 + 8) * dot_abs
    k2_abs = torch.where(r0 > 0, dot_abs * i0 * i0 / r0.clamp_min(1e-300), torch.zeros_like(r0))
    dk2 = torch.where(r0 > 0, (ddot + 4 * gr * dot_abs) * i0 * i0 / r0.clamp_min(1e-300), torch.zeros_like(r0))
    gb = (ddn + dn_abs * gr) * i0 + f0d.abs() * dk2 + gamma(8) * (dn_abs * i0 + f0d.abs() * k2_abs) + ATOL
    return val, vb, g, gb


def emulate_lpips_head(f0, f1, w, defect: Optional[str] = None):
    """fp32 (value, g); defect 'eps_outside': i = 1 / r + 1e-10 (the epsilon added after the reciprocal)"""
    f0, f1, w = f0.float(), f1.float(), w.float()
    HW, C = f0.shape
    r0, r1 = f0.norm(dim=1, keepdim=True), f1.norm(dim=1, keepdim=True)
    if defect == 'eps_outside':
        i0, i1 = 1 / r0 + 1e-10, 1 / r1 + 1e-10
    else:
        i0, i1 = 1 / (r0 + 1e-10), 1 / (r1 + 1e-10)
    d = f0 * i0 - f1 * i1
    val = (w * d * d).sum() / HW
    dn = 2 * w * d / HW
    dot = (f0 * dn).sum(1, keepdim=True)
    k2 = torch.where(r0 > 0, dot * i0 * i0 / r0, torch.zeros_like(r0))
    return val, dn * i0 - f0 * k2


# ------------------------------------------------------------------------------------------------ comparison
def max_ratio(got: torch.Tensor, ref: torch.Tensor, bnd: torch.Tensor) -> float:
    """largest |got - ref| / bound (NaN counts as infinite)"""
    err = (got.to(ref.device).double() - ref).abs()
    r = err / (bnd + ATOL)
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------ LPIPS input scaling
LPIPS_SHIFT = (-.030, -.088, -.188)
LPIPS_SCALE = (.458, .448, .450)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def ref_lpips_prep(pred, target, normalize):
    """[2,H,W,4]: ((2 v - 1 if normalize) - shift_c) / scale_c, channel 3 zero.  2 v is exact, - 1, - shift and / scale round once each"""
    out, bnd = [], []
    for img in (pred, target):
        v = img.double()
        if normalize:
            v = 2 * v - 1
        sh = torch.tensor([_f32(s) for s in LPIPS_SHIFT], dtype=torch.float64, device=v.device)[:, None, None]
        sc = torch.tensor([_f32(s) for s in LPIPS_SCALE], dtype=torch.float64, device=v.device)[:, None, None]
        y = (v - sh) / sc
        out.append(F.pad(y.permute(1, 2, 0), (0, 1)))
        bnd.append(F.pad((gamma(3) * (v.abs() + sh.abs() + 1) / sc).permute(1, 2, 0), (0, 1)))
    return torch.stack(out), torch.stack(bnd) + ATOL


def ref_lpips_prep_backward(gx, normalize, factor):
    """[3,H,W] = gx[..., c] factor (2 if normalize) / scale_c: the factor product and the division round (the doubling is exact)"""
    sc = torch.tensor([_f32(s) for s in LPIPS_SCALE], dtype=torch.float64, device=gx.device)
    y = (gx.double()[..., :3] * _f32(factor) * (2 if normalize else 1) / sc).permute(2, 0, 1)
    return y, gamma(3) * y.abs() + ATOL


# ------------------------------------------------------------------------------------------------ recorded launches
def _lpips_entry(name, a):
    if name == 'sfb_lpips_prep':
        return dict(H=a['H'], W=a['W'], normalize=a['normalize'])
    if name == 'sfb_lpips_prep_backward':
        return dict(H=a['H'], W=a['W'], normalize=a['normalize'], factor=float(a['factor']))
    if name == 'sfb_relu_nhwc':
        return dict(n=int(a['n']))
    if name == 'sfb_maxpool2x2_nhwc':
        return dict(NB=a['NB'], H=a['H'], W=a['W'], C=a['C'])
    if name == 'sfb_maxpool2x2_relu_backward_nhwc':
        return dict(H=a['H'], W=a['W'], C=a['C'])
    if name == 'sfb_add_relu_mask':
        return dict(n=int(a['n']), head=a['g_head'] is not None)
    return dict(HW=a['HW'], C=a['C'])                                          # sfb_lpips_head


def _front_end_entry(op, t, s):
    if op == 'groupnorm':
        x, y, film = t['x'], t['out'], t['film']
        nb, h, w, c, ldx, xoff = nhwc_meta(x)
        _, _, _, _, ldy, yoff = nhwc_meta(y)
        return dict(NB=nb, H=h, W=w, C=c, G=s['groups'], ldx=ldx, xoff=xoff, ldy=ldy, yoff=yoff, film=film is not None,
                    ldf=film.stride(0) if film is not None else 0, act=s['silu'], alias='x=out' if same_ptr(x, y) else '')
    if op == 'layernorm':
        res = t['residual']
        T, C, ldx, xoff = rows_meta(t['x'])
        return dict(T=T, C=C, ldx=ldx, xoff=xoff, ldy=rows_meta(t['out'])[2], b=t['b'] is not None, res=res is not None,
                    ldr=rows_meta(res)[2] if res is not None else 0, pre_gelu=s['pre_gelu'], round=s['round'],
                    alias='res=out' if same_ptr(res, t['out']) else '')
    if op == 'linear_small':
        res = t['residual']
        M, K, ldx, xoff = rows_meta(t['x'])
        return dict(M=M, K=K, O=t['w'].shape[0], ldx=ldx, xoff=xoff, ldy=rows_meta(t['out'])[2], bias=t['bias'] is not None,
                    res=res is not None, ldr=rows_meta(res)[2] if res is not None else 0, pre=s['pre'], post=s['post'], round=s['round'])
    if op == 'mq_attention':
        q, ckv = t['q'], t['ckv']
        return dict(B=q.shape[0], n=q.shape[1], heads=s['heads'], dh=s['dh'], nc=0 if ckv is None else ckv.shape[1])
    if op == 'cross_attention':
        q = t['q']
        return dict(B=q.shape[0], n=q.shape[1], heads=s['heads'], dh=s['dh'], nc=t['kvc'].shape[1])
    if op == 'gca_pool':
        nb, h, w, c, ldx, xoff = nhwc_meta(t['x'])
        return dict(NB=nb, HW=h * w, C=c, ldx=ldx, xoff=xoff)
    if op == 'gate_mlp_residual':
        nb, hh, ww, c, ldh, _ = nhwc_meta(t['h'])
        return dict(NB=nb, HW=hh * ww, C=c, Hd=t['hid'].shape[-1], ldh=ldh, ldr=nhwc_meta(t['res'])[4])
    if op == 'gate_residual':
        nb, hh, ww, c, ldh, _ = nhwc_meta(t['h'])
        return dict(NB=nb, HW=hh * ww, C=c, ldh=ldh, ldr=nhwc_meta(t['res'])[4], ldo=nhwc_meta(t['out'])[4], gate=t['gate'] is not None)
    if op == 'softmax_rows':
        r, c, ldx, _ = rows_meta(t['x'])
        return dict(rows=r, cols=c, ldx=ldx, ldy=rows_meta(t['out'])[2], scale=s['scale'])
    if op == 'upsample2x':
        nb, h, w, c, ldx, _ = nhwc_meta(t['x'])
        return dict(NB=nb, H=h, W=w, C=c, ldx=ldx)
    if op == 'nchw_to_nhwc':
        nb, c, h, w = t['src'].shape
        return dict(NB=nb, C=c, H=h, W=w, ld=nhwc_meta(t['out'])[4], c_off=s['c_off'], round=s['round'])
    if op == 'nhwc_to_nchw':
        nb, h, w, c, ld, _ = nhwc_meta(t['src'])
        return dict(NB=nb, C=c, H=h, W=w, ld=ld)
    if op == 'im2col4':
        nb, h, w, c, ldx, _ = nhwc_meta(t['x'])
        return dict(NB=nb, H=h, W=w, KH=s['kh'], KW=s['kw'], pad=s['pad'], ldx=ldx)
    if op == 'concat2':
        nb, h, w, c1, lda, _ = nhwc_meta(t['a'])
        return dict(NB=nb, H=h, W=w, C1=c1, lda=lda, C2=t['b'].shape[-1], ldb=nhwc_meta(t['b'])[4], ldo=nhwc_meta(t['out'])[4],
                    scale_b=s['scale_b'])
    if op == 'pixel_shuffle_silu':
        nb, h, w, c4, _, _ = nhwc_meta(t['y'])
        return dict(NB=nb, H=h, W=w, Co=c4 // 4, ldo=nhwc_meta(t['out'])[4])
    if op == 'time_fourier':
        return dict(B=t['t'].shape[0], half=t['w'].shape[0])
    return None                                                                 # conv2d_nhwc: tests/test_conv_fp64_gpu.py


def entry(r) -> Optional[Dict]:
    """the replay entry of an oracle/insitu record: a front-end record other than the GEMM's, or a ``Call`` of an LPIPS entry point read by
    parameter name (None for any other launch).  Row strides, slice offsets, the FiLM row stride, residual and aliasing (an output at the
    address of an input); labelled with the family."""
    if r.op in LPIPS_NAMES:
        return dict(_lpips_entry(r.op, r.args), op=LPIPS_NAMES[r.op], family=r.family, label=r.family)
    f = None if r.op.startswith('sfb_') else _front_end_entry(r.op, r.orig, r.s)       # calls carry the C symbol, records the front end
    return None if f is None else dict(f, op=r.op, family=r.family, label=r.family)
