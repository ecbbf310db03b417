"""oracle/conv_fp64.py -- the launch plan, an fp64 reference and per-element error bounds of the tensor-core GEMM kernel
``conv_gemm_kernel`` (sparsefusion_b200/csrc/conv_wgmma.cu), through which every convolution and linear of the UNet, the VAE,
LPIPS-VGG and the EFT runs.

TEST INFRASTRUCTURE ONLY.

``launch_plan`` restates the host-side dispatch of ``sfb_conv2d_nhwc_tf32_ex`` line by line: tile kind and shape, N tile, split-K
factor and the kernel instantiation the tracer records.  The GPU tests hold it to the real dispatch through that tracer.

``conv_ref`` is the convolution in fp64 with its absolute companion; ``bound`` is the per-element tolerance
    |y_gpu - y| <= (rho_prod + 2 gamma(n_chain)) * conv(|x|, |w|) + gamma(n_epi) * A,
    A = conv(|x|, |w|) + |bias| + |residual| + |prefill|,
with gamma, ``violations`` and ``assert_within`` from ``field_fp64`` (Higham's model: n chained roundings of unit roundoff u = 2^-24).

``emulate`` evaluates the kernel's arithmetic in the kernel's k order (fp64 products of the tf32 operand words, fp32 partial sums),
with switches that inject single defects; the host tests use it to show which defects the bound sees.

``entry`` turns an oracle/insitu record of ``ops.conv2d_nhwc`` into the geometry and memory layout tests/test_conv_fp64_gpu.py replays.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .field_fp64 import ATOL, gamma, violations

KBM = 128          # M-side rows of a CTA (conv_wgmma.cu kBM)
KBK = 32           # fp32 elements per k-step (kBK): one 32-channel chunk of one filter tap

# ------------------------------------------------------------------------------------------------ rounding model
# rho_prod: relative error of ONE product x * w as the tensor core forms it, w.r.t. |x| |w|.
#   3xTF32: x = hi + lo with hi = x & 0xFFFFE000 (exact), so |lo| < 2^-10 |x|.  The kernel issues hi*hi + lo*hi + hi*lo.  The dropped lo*lo
#     is < 2^-20 |x w|.  lo is passed as a full fp32 word and the tensor core reads only its tf32 part: lo carries at most 13 significant
#     bits, so that read drops at most its 2 lowest, < 2^-21 |x| for each operand.  In all 2^-20 + 2 * 2^-21 = 2^-19 = 32 u.  With random
#     mantissas the product error is ~2^-21 (8 u, the figure field_fp64.wgrad_rtol uses); the edge operands of the GPU tests (low words
#     0x1FFF) deliberately approach the worst case, so the per-element bound takes it.
#   single pass: the activation word is read as tf32 (truncated: < 2^-10, or rounded: <= 2^-11); the weights were rounded to nearest
#     at packing (<= 2^-11), or are a raw activation themselves in the attention GEMMs (< 2^-10).  Their product adds the cross term.
RHO_TF32X3 = 2.0 ** -19


def rho_prod(precision: str, w_rounded: bool = True) -> float:
    if precision == 'tf32x3':
        return RHO_TF32X3
    ew = 2.0 ** -11 if w_rounded else 2.0 ** -10
    return 2.0 ** -10 + ew + 2.0 ** -10 * ew


# n_chain: products chained into one CTA's accumulator, ceil(k_iters / splits) k-steps of 32.  The tensor core's fp32 accumulation is
#   not exactly rounded (products are aligned to the largest exponent and truncated); 2 u per chained product bounds it.
# n_epi: the epilogue.  Split 0 adds the bias (1 rounding) and the residual (1); each split's partial sum meets the destination in a
#   red.global.add (splits roundings), the first of them onto the pre-filled value when accumulating (1 more).
def n_chain(plan: dict) -> int:
    return -(-plan['k_iters'] // plan['splits']) * KBK


def n_epi(plan: dict) -> int:
    return plan['splits'] + 3


def rtols(plan: dict, precision: str, w_rounded: bool = True):
    """(relative factor on conv(|x|,|w|), relative factor on A)"""
    return rho_prod(precision, w_rounded) + 2 * gamma(n_chain(plan)), gamma(n_epi(plan))


def bound(plan: dict, precision: str, C: torch.Tensor, A: torch.Tensor, w_rounded: bool = True) -> torch.Tensor:
    r_c, r_a = rtols(plan, precision, w_rounded)
    return r_c * C + r_a * A


# ------------------------------------------------------------------------------------------------ launch plan
def _ceil_div(a: int, b: int) -> int:
    return -(-a // b)


def _pow2_floor(v: int) -> int:
    r = 1
    while r * 2 <= v:
        r *= 2
    return r


def out_size(H, W, KH, KW, stride, pad, pad_after):
    return (H + pad + pad_after - KH) // stride + 1, (W + pad + pad_after - KW) // stride + 1


def launch_plan(NB: int, H: int, W: int, Cin: int, Cout: int, KH: int, KW: int, stride: int = 1, pad: int = 0,
                pad_after: Optional[int] = None, splits: int = 0, bn: int = 0, precision: str = 'tf32x3', variant: int = 2,
                presplit: bool = False, sm: int = 132) -> Dict:
    """the launch sfb_conv2d_nhwc_tf32_ex makes.  ``bn`` in the result is the N width of the launched tile: output channels in
    normal mode, pixels (tile_pix) in swap mode; ``bn_host`` is the host's BN variable, which swap mode does not use."""
    if pad_after is None:
        pad_after = pad
    Ho, Wo = out_size(H, W, KH, KW, stride, pad, pad_after)                 # conv_wgmma.cu:551
    assert Ho > 0 and Wo > 0
    P_total = NB * Ho * Wo                                                  # :560
    v2 = precision == 'tf32x3' and variant >= 2                             # :561
    swap = v2 and P_total <= 64 and bn <= 0                                 # :562
    tile_pix = KBM
    if swap:                                                                # :564
        tile_pix = 16
        while tile_pix < P_total:
            tile_pix *= 2
    TW = tile_pix if Wo >= tile_pix else _pow2_floor(Wo)                    # :565-568
    TH = tile_pix // TW
    if TH > Ho:
        TH = _pow2_floor(Ho)
    TN = tile_pix // (TW * TH)
    tiles_w, tiles_h, tiles_n = _ceil_div(Wo, TW), _ceil_div(Ho, TH), _ceil_div(NB, TN)
    tiles_m = tiles_w * tiles_h * tiles_n                                   # :572
    cin_pad = _ceil_div(Cin, 32) * 32
    k_iters = KH * KW * (cin_pad // 32)                                     # :577
    BN = bn
    if BN <= 0:                                                             # :587-592
        BN = 256 if Cout >= 256 else (128 if Cout >= 128 else (64 if Cout >= 64 else 32))
        while BN > 128 and tiles_m * _ceil_div(Cout, BN) < sm:
            BN //= 2
        if v2 and BN > 128:
            BN = 128
    assert BN in (32, 64, 128, 256)
    tiles_c = _ceil_div(Cout, KBM) if swap else _ceil_div(Cout, BN)         # :594
    if splits <= 0:                                                         # :595-604
        ctas = tiles_m * tiles_c
        splits = 1
        if ctas < sm:
            splits = sm // ctas
            max_by_k = k_iters // 4 if k_iters // 4 > 0 else 1
            splits = min(splits, max_by_k)
            splits = max(splits, 1)
    if precision == 'tf32x3':                                               # :605-610
        splits = max(splits, _ceil_div(k_iters, 96))
    splits = min(splits, k_iters)                                           # :611
    kernel = f'conv<{tile_pix},swap>' if swap else f'conv<{BN}>'            # :451-452, :657-677
    return dict(NB=NB, Ho=Ho, Wo=Wo, P_total=P_total, swap=swap, tile_pix=tile_pix, TW=TW, TH=TH, TN=TN, tiles_w=tiles_w, tiles_h=tiles_h,
                tiles_n=tiles_n, tiles_m=tiles_m, tiles_c=tiles_c, bn=tile_pix if swap else BN, bn_host=BN, splits=splits, k_iters=k_iters,
                cin_pad=cin_pad, presplit=bool(presplit and v2 and not swap), kernel=kernel, np=3 if precision == 'tf32x3' else 1,
                pad_after=pad_after)


def split_ranges(k_iters: int, splits: int):
    """[kb, ke) of every split (blockIdx.z), conv_wgmma.cu:109-110"""
    return [((k_iters * z) // splits, (k_iters * (z + 1)) // splits) for z in range(splits)]


# ------------------------------------------------------------------------------------------------ fp64 reference
def conv_ref(x: torch.Tensor, w: torch.Tensor, bias=None, residual=None, prefill=None, stride: int = 1, pad: int = 0,
             pad_after: Optional[int] = None):
    """x NHWC [NB,H,W,Cin], w [Cout,Cin,KH,KW] -> (y, C, A) NHWC fp64 on x's device: y the exact result (bias, residual and the
    pre-filled destination included), C = conv(|x|, |w|), A = C + |bias| + |residual| + |prefill|"""
    if pad_after is None:
        pad_after = pad
    xd, wd = x.double(), w.double()

    def conv(a, b):
        if b.shape[2:] == (1, 1) and stride == 1 and pad == 0 and pad_after == 0:
            return (a.reshape(-1, a.shape[-1]) @ b[:, :, 0, 0].T).reshape(*a.shape[:-1], b.shape[0])
        a = F.pad(a.permute(0, 3, 1, 2), (pad, pad_after, pad, pad_after))
        return F.conv2d(a, b, stride=stride).permute(0, 2, 3, 1)

    y = conv(xd, wd)
    C = conv(xd.abs(), wd.abs())
    A = C.clone()
    for t in (bias, residual, prefill):
        if t is not None:
            y = y + t.double()
            A = A + t.double().abs()
    return y, C, A


def slice_guard_intact(before: torch.Tensor, after: torch.Tensor, c_off: int, width: int) -> bool:
    """every channel of the rows [.., ld] outside [c_off, c_off + width) (and every element outside the rows: pass flat guards as
    [1, n] with width 0) is bit-identical, compared as int32"""
    b, a = before.contiguous().view(torch.int32), after.contiguous().view(torch.int32)
    keep = torch.ones(b.shape[-1], dtype=torch.bool, device=b.device)
    keep[c_off:c_off + width] = False
    return bool(torch.equal(b[..., keep], a[..., keep]))


# ------------------------------------------------------------------------------------------------ operand words
def tf32_hi(t: torch.Tensor) -> torch.Tensor:
    """fp32 word with its 13 low mantissa bits cleared (the kernel's hi, and the tensor core's truncating tf32 read)"""
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


def tf32_rna(t: torch.Tensor) -> torch.Tensor:
    """round to nearest, ties away (cvt.rna.tf32.f32, ops.round_tf32)"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & -8192).view(torch.float32)


def with_low_bits(t: torch.Tensor, low: int) -> torch.Tensor:
    """t with the 13 low mantissa bits replaced by ``low``"""
    i = t.float().contiguous().view(torch.int32)
    return ((i & -8192) | low).view(torch.float32)


# ------------------------------------------------------------------------------------------------ emulation of the kernel
def _taps(x: torch.Tensor, KH: int, KW: int, stride: int, pad: int, Ho: int, Wo: int, parity_swap: bool = False,
          shift_cols=None) -> torch.Tensor:
    """[KH*KW, NB, Ho, Wo, Cin] fp64: the activation each output pixel reads at each tap, zero outside the image (the TMA fill).
    For stride 2 the read goes through parity plane (py, px) of the tap; ``parity_swap`` reads plane (px, py) instead.
    ``shift_cols`` (bool [Wo]): those output columns read one pixel further right at every tap."""
    NB, H, W, Cin = x.shape
    dev = x.device
    oh = torch.arange(Ho, device=dev)
    ow = torch.arange(Wo, device=dev)
    out = torch.zeros(KH * KW, NB, Ho, Wo, Cin, dtype=torch.float64, device=dev)
    for ky in range(KH):
        for kx in range(KW):
            oy, ox = ky - pad, kx - pad
            if stride == 2:
                py, px = oy & 1, ox & 1
                oy2, ox2 = (oy - py) >> 1, (ox - px) >> 1
                if parity_swap:
                    py, px = px, py
                r = 2 * (oh + oy2) + py
                c = 2 * (ow + ox2) + px
                rv = (oh + oy2 >= 0) & (oh + oy2 < H // 2)
                cv = (ow + ox2 >= 0) & (ow + ox2 < W // 2)
            else:
                r, c = oh + oy, ow + ox
                rv, cv = (r >= 0) & (r < H), (c >= 0) & (c < W)
            if shift_cols is not None:
                c = torch.where(shift_cols, c + 1, c)
                cv = cv & (c < W) & (c >= 0)
            g = x[:, r.clamp(0, H - 1)][:, :, c.clamp(0, W - 1)].double()
            out[ky * KW + kx] = g * (rv[:, None, None] & cv[None, :, None]).to(g.dtype)
    return out


def emulate(x: torch.Tensor, w: torch.Tensor, plan: dict, precision: str = 'tf32x3', bias=None, residual=None, prefill=None,
            stride: int = 1, pad: int = 0, defect: Optional[str] = None, defect_split: int = 0) -> torch.Tensor:
    """fp32 result [NB,Ho,Wo,Cout] (as fp64) of the kernel's arithmetic: k-steps tap-major over 32-channel chunks, each split z summing
    its k range [kb, ke) into an fp32 accumulator (one rounding per k-step), products formed from the tf32 words the tensor core reads
    (3xTF32: hi*hi + lo*hi + hi*lo with lo's tf32 part; single pass: truncated activations times nearest-rounded weights), split 0 adding
    bias and residual in fp32, the splits meeting in fp32 on the pre-filled destination in split order.

    defects: 'lost_kstep' (split ``defect_split`` skips its last k-step), 'lost_tile' (the first M tile of the first channel tile is never
    written), 'bias_every_split', 'residual_every_split', 'parity_swap', 'pad_after_ignored' (the output extent of pad_after = pad: the
    last row and column are never written), 'tap_shift' (the last output column, on a partial tile's edge, reads one pixel to the right),
    'single_pass' (every product in single-pass precision), 'one_chunk_single_pass' (only k-step 0 of split 0 in single-pass precision)."""
    NB, H, W, Cin = x.shape
    Cout, _, KH, KW = w.shape
    Ho, Wo = plan['Ho'], plan['Wo']
    cin_pad = plan['cin_pad']
    shift = None
    if defect == 'tap_shift':
        shift = torch.zeros(Wo, dtype=torch.bool, device=x.device)
        shift[Wo - 1] = True
    X = _taps(x, KH, KW, stride, pad, Ho, Wo, parity_swap=defect == 'parity_swap', shift_cols=shift)
    X = F.pad(X, (0, cin_pad - Cin)).reshape(KH * KW, -1, cin_pad)                       # [taps, P, cin_pad]
    Wt = F.pad(w.double().permute(2, 3, 0, 1).reshape(KH * KW, Cout, Cin), (0, cin_pad - Cin))   # [taps, Cout, cin_pad]

    def words(single):
        if single:
            return (tf32_hi(X).double(),), (tf32_rna(Wt).double(),)
        xh, wh = tf32_hi(X).double(), tf32_hi(Wt).double()
        xl, wl = tf32_hi(X - xh).double(), tf32_hi(Wt - wh).double()
        return (xh, xl, xh), (wh, wh, wl)

    sp = words(True)
    tx = words(precision != 'tf32x3' or defect == 'single_pass')
    P = X.shape[1]
    out = torch.zeros(P, Cout, dtype=torch.float64, device=x.device) if prefill is None else prefill.double().reshape(P, Cout).clone()
    for z, (kb, ke) in enumerate(split_ranges(plan['k_iters'], plan['splits'])):
        acc = torch.zeros(P, Cout, dtype=torch.float64, device=x.device)
        for i in range(kb, ke):
            if defect == 'lost_kstep' and z == defect_split and i == ke - 1:
                continue
            xs, ws = sp if (defect == 'one_chunk_single_pass' and z == 0 and i == kb) else tx
            tap, cc = divmod(i, cin_pad // 32)
            ch = slice(cc * 32, cc * 32 + 32)
            s = sum(a[tap][:, ch] @ b[tap][:, ch].T for a, b in zip(xs, ws))
            acc = (acc + s).float().double()
        if z == 0 or defect in ('bias_every_split', 'residual_every_split'):
            if bias is not None and (z == 0 or defect == 'bias_every_split'):
                acc = (acc + bias.double()[None]).float().double()
            if residual is not None and (z == 0 or defect == 'residual_every_split'):
                acc = (acc + residual.double().reshape(P, Cout)).float().double()
        out = (out + acc).float().double()
    out = out.reshape(NB, Ho, Wo, Cout)
    fill = torch.zeros_like(out) if prefill is None else prefill.double()
    if defect == 'lost_tile':
        bn = KBM if plan['swap'] else plan['bn']
        TW, TH, TN = plan['TW'], plan['TH'], plan['TN']
        out[:TN, :TH, :TW, :bn] = fill[:TN, :TH, :TW, :bn]
    if defect == 'pad_after_ignored':
        out[:, -1] = fill[:, -1]
        out[:, :, -1] = fill[:, :, -1]
    return out


def max_ratio(got: torch.Tensor, bnd: torch.Tensor, ref: torch.Tensor) -> float:
    """largest |got - ref| / bound (NaN counts as infinite)"""
    err = (got.double() - ref).abs()
    r = err / (bnd + ATOL)
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------ recorded launches
def nhwc_meta(t: torch.Tensor):
    """(NB, H, W, C, ld, off) of an NHWC tensor or channel slice of one: ld its row stride, off its first channel within a row (0 when
    the slice does not sit inside one row)"""
    nb, h, w, c = t.shape
    ld = t.stride(2)
    off = t.storage_offset() % ld
    return nb, h, w, c, ld, (off if off + c <= ld else 0)


def rows_meta(t: torch.Tensor):
    """(rows, C, ld, off) of a row-major [..., C] tensor with a uniform row stride ld, off as in ``nhwc_meta``"""
    c = t.shape[-1]
    ld = t.stride(-2) if t.dim() >= 2 else c
    off = t.storage_offset() % ld if ld else 0
    return t.numel() // c, c, ld, (off if off + c <= ld else 0)


def same_ptr(a: Optional[torch.Tensor], b: Optional[torch.Tensor]) -> bool:
    return a is not None and b is not None and a.data_ptr() == b.data_ptr()


def entry(r) -> Optional[Dict]:
    """the replay entry of an oracle/insitu record of ``ops.conv2d_nhwc`` (None for any other launch): geometry, row strides and slice
    offsets of x, out and the residual, the switches, and ``alias`` where two of them start at the same address"""
    if r.op != 'conv2d_nhwc':
        return None
    t, s = r.orig, r.s
    x, y, res = t['x'], t['out'], t['residual']
    nb, h, w, cin, ldx, xoff = nhwc_meta(x)
    ldo, ooff = nhwc_meta(y)[4:]
    ldr, roff = nhwc_meta(res)[4:] if res is not None else (0, 0)
    alias = [n for a, b, n in ((x, y, 'x=out'), (res, y, 'res=out'), (x, res, 'x=res')) if same_ptr(a, b)]
    return dict(NB=nb, H=h, W=w, Cin=cin, ldx=ldx, xoff=xoff, Cout=s['cout'], KH=s['kh'], KW=s['kw'], stride=s['stride'], pad=s['pad'],
                pad_after=s['pad_after'], ldo=ldo, ooff=ooff, bias=t['bias'] is not None, residual=res is not None, ldr=ldr, roff=roff,
                accumulate=s['accumulate'], w_split=t['w_split'] is not None, dyn=s['dyn'], splits=s['splits'], bn=s['bn'],
                alias=','.join(alias), family=r.family, label=r.label)
