"""Torch-tensor front ends of the UNet operators of the C ABI (include/sparsefusion_b200.h §3).

Everything here is plumbing: allocate outputs with torch, pass device pointers + the current
stream to libsparsefusion_b200.so.  Activations are NHWC fp32 tensors ``[NB, H, W, C]``; a
"channel slice" view ``t[..., a:b]`` of a wider NHWC tensor is accepted wherever a leading
dimension is passed (its ``stride(2)`` is the channel stride).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib as lib


# --------------------------------------------------------------------------------------------- precision
def set_precision(mode: str) -> None:
    """'tf32x3' (default; error-compensated, fp32-class accuracy) or 'tf32' (single pass, operands rounded on write).
    Packed weights depend on the mode: call ``Unet.prepare()`` again after switching."""
    lib.call('sfb_set_precision', {'tf32': 0, 'tf32x3': 1}[mode])


def get_precision() -> str:
    return ('tf32', 'tf32x3')[lib.load().sfb_get_precision()]


# --------------------------------------------------------------------------------------------- accounting
_GRAPH_LAUNCHES = 0   # kernels executed through CUDA-graph replays (they do not pass through the C ABI again)


def launch_count() -> int:
    """kernels of libsparsefusion_b200.so launched so far in this process: direct launches + graph-replayed ones"""
    return int(lib.load().sfb_launch_count()) + _GRAPH_LAUNCHES


def note_graph_replay(n_kernels: int) -> None:
    global _GRAPH_LAUNCHES
    _GRAPH_LAUNCHES += n_kernels


# --------------------------------------------------------------------------------------------- helpers
def round_tf32(t: torch.Tensor) -> torch.Tensor:
    """round-to-nearest (ties away from zero) fp32 -> tf32 kept in fp32 storage (== cvt.rna.tf32.f32)"""
    i = t.contiguous().view(torch.int32)
    r = ((i + 0x1000) & ~0x1FFF)
    # values whose exponent is all ones (inf / nan) must not be touched
    keep = (i & 0x7F800000) == 0x7F800000
    return torch.where(keep, i, r).view(torch.float32)


def pack_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """nn.Conv2d weight [Cout,Cin,KH,KW] (or nn.Linear weight [O,K]) -> [Cout, KH*KW*ceil32(Cin)]
    tap-major / channel-minor, zero padded: the K-major B operand of the implicit GEMM.  TF32-rounded in 'tf32' mode,
    raw fp32 in 'tf32x3' mode (the kernel splits hi/lo itself)."""
    if w.dim() == 2:
        w = w[:, :, None, None]
    cout, cin, kh, kw = w.shape
    cin_pad = (cin + 31) // 32 * 32
    p = torch.zeros(cout, kh, kw, cin_pad, dtype=torch.float32, device=w.device)
    p[..., :cin] = w.detach().float().permute(0, 2, 3, 1)
    p = p.reshape(cout, kh * kw * cin_pad)
    return (round_tf32(p) if get_precision() == 'tf32' else p).contiguous()


def split_packed_weight(wp: torch.Tensor) -> torch.Tensor:
    """[2, Cout, K]: hi = the TF32 part the tensor core uses (bits & 0xFFFFE000), lo = w - hi (exact in fp32).  The tensor-bound convolutions
    of the 3xTF32 engine TMA-load both tiles instead of splitting the weight tile in shared memory on every k-step."""
    hi = (wp.contiguous().view(torch.int32) & -8192).view(torch.float32)
    return torch.stack((hi, wp - hi), dim=0).contiguous()


def _nhwc_meta(t: torch.Tensor) -> Tuple[int, int, int, int, int]:
    """(NB, H, W, C, ld) of an NHWC tensor or channel-slice view of one"""
    assert t.dim() == 4 and t.is_cuda and t.dtype == torch.float32, 'expected a CUDA fp32 NHWC tensor'
    nb, h, w, c = t.shape
    ld = t.stride(2)
    assert t.stride(3) == 1 and t.stride(1) == w * ld and t.stride(0) == h * w * ld, 'expected NHWC with a uniform channel stride'
    return nb, h, w, c, ld


def _rows_meta(t: torch.Tensor) -> Tuple[int, int, int]:
    """(rows, cols, ld) of a row-major 2D-like tensor [..., C] with uniform row stride"""
    assert t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1
    c = t.shape[-1]
    rows = t.numel() // c
    ld = t.stride(-2) if t.dim() >= 2 else c
    return rows, c, ld


# --------------------------------------------------------------------------------------------- conv / linear on tensor cores
# --------------------------------------------------------------------------------------------- split-K output arena
# The weight-streaming convolutions split K over up to one CTA per SM and meet in fp32 red.global.add, so their destination must start from
# zero.  One cudaMemset node per convolution costs ~2.3 us inside the replayed UNet graph (and breaks the programmatic-dependent-launch
# edge in front of the convolution); with an arena all conv outputs of one UNet evaluation are carved out of ONE buffer that is
# zero-filled once at the start of the evaluation, and the convolutions run in "accumulate" mode.
class ZeroArena:
    def __init__(self, floats: int, device):
        self.buf = torch.zeros(max(int(floats), 1), dtype=torch.float32, device=device)
        self.off = 0

    def take(self, shape):
        n = 1
        for d in shape:
            n *= int(d)
        if self.off + n > self.buf.numel():
            return None
        t = self.buf[self.off:self.off + n].view(*shape)
        self.off += (n + 63) // 64 * 64          # 256-byte granules keep every tensor 16-byte aligned for TMA
        return t


class ArenaMeter:
    """first evaluation of a shape: count the floats an arena would have to hold"""

    def __init__(self):
        self.floats = 0

    def take(self, shape):
        n = 1
        for d in shape:
            n *= int(d)
        self.floats += (n + 63) // 64 * 64
        return None


_arena = None


class use_arena:
    def __init__(self, arena):
        self.arena = arena

    def __enter__(self):
        global _arena
        self.prev, _arena = _arena, self.arena
        return self.arena

    def __exit__(self, *exc):
        global _arena
        _arena = self.prev
        return False


def _conv_out(shape, device):
    """(tensor, pre-zeroed?)"""
    if _arena is not None:
        t = _arena.take(shape)
        if t is not None:
            return t, True
    return torch.empty(*shape, dtype=torch.float32, device=device), False


def conv2d_nhwc(x: torch.Tensor, w_packed: torch.Tensor, cout: int, kh: int, kw: int, stride: int = 1, pad: int = 0,
                bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                accumulate: bool = False, splits: int = 0, bn: int = 0, pad_after: Optional[int] = None,
                w_split: Optional[torch.Tensor] = None, dynamic_weights: bool = False) -> torch.Tensor:
    nb, h, w, cin, ldx = _nhwc_meta(x)
    if pad_after is None:
        pad_after = pad
    ho = (h + pad + pad_after - kh) // stride + 1
    wo = (w + pad + pad_after - kw) // stride + 1
    if out is None:
        out, zeroed = _conv_out((nb, ho, wo, cout), x.device)
        accumulate = accumulate or zeroed           # pre-zeroed destination: reduce straight into it, no memset node
    onb, oh, ow, oc, ldo = _nhwc_meta(out)
    assert (onb, oh, ow, oc) == (nb, ho, wo, cout), f'out shape {tuple(out.shape)} != {(nb, ho, wo, cout)}'
    assert w_packed.shape == (cout, kh * kw * ((cin + 31) // 32 * 32)), 'packed weight shape mismatch'
    ldr = 0
    if residual is not None:
        rnb, rh, rw, rc, ldr = _nhwc_meta(residual)
        assert (rnb, rh, rw, rc) == (nb, ho, wo, cout)
    if w_split is not None:
        assert w_split.shape == (2,) + tuple(w_packed.shape)
    if dynamic_weights:
        # the K-major operand is an activation produced by an earlier launch (attention GEMMs): the kernel must not prefetch it ahead of its
        # programmatic-dependent-launch wait (sfb_conv2d_nhwc_tf32_dyn)
        assert w_split is None
        lib.call('sfb_conv2d_nhwc_tf32_dyn', x.data_ptr(), nb, h, w, cin, ldx, lib.fptr(w_packed, 'w_packed'), cout, kh, kw, stride, pad, pad_after,
                 lib.fptr(bias, 'bias'), None if residual is None else residual.data_ptr(), ldr, out.data_ptr(), ldo, int(accumulate), splits, bn, lib.stream())
        return out
    lib.call('sfb_conv2d_nhwc_tf32_ex', x.data_ptr(), nb, h, w, cin, ldx,
             lib.fptr(w_packed, 'w_packed'), lib.fptr(w_split, 'w_split'), cout, kh, kw, stride, pad, pad_after, lib.fptr(bias, 'bias'),
             None if residual is None else residual.data_ptr(), ldr, out.data_ptr(), ldo, int(accumulate), splits, bn, lib.stream())
    return out


def linear_tc(x: torch.Tensor, w_packed: torch.Tensor, out_features: int, bias=None, residual=None, out=None, w_split=None,
              dynamic_weights: bool = False) -> torch.Tensor:
    """nn.Linear on the tensor cores: rows [T, K] are treated as T 1x1 'images'.  ``dynamic_weights``: w_packed is an activation (see conv2d_nhwc)"""
    t, k, ld = _rows_meta(x)
    x4 = x.as_strided((t, 1, 1, k), (ld, ld, ld, 1))
    zeroed = False
    if out is None:
        out, zeroed = _conv_out((*x.shape[:-1], out_features), x.device)
    to, co, ldo = _rows_meta(out)
    o4 = out.as_strided((t, 1, 1, out_features), (ldo, ldo, ldo, 1))
    r4 = None
    if residual is not None:
        tr, cr, ldr = _rows_meta(residual)
        r4 = residual.as_strided((t, 1, 1, out_features), (ldr, ldr, ldr, 1))
    conv2d_nhwc(x4, w_packed, out_features, 1, 1, 1, 0, bias, r4, o4, accumulate=zeroed, w_split=w_split, dynamic_weights=dynamic_weights)
    return out


def gate_mlp_residual(h: torch.Tensor, hid: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor, res: torch.Tensor) -> torch.Tensor:
    """out = h * sigmoid(hid @ w2.T + b2)[:, None, None, :] + res   (GlobalContext's last layer + the ResnetBlock tail in one launch)"""
    nb, hh, ww, c, ldh = _nhwc_meta(h)
    _, _, _, _, ldr = _nhwc_meta(res)
    out = torch.empty(nb, hh, ww, c, dtype=torch.float32, device=h.device)
    hd = hid.shape[-1]
    assert tuple(w2.shape) == (c, hd) and hid.numel() == nb * hd
    lib.call('sfb_gate_mlp_residual_nhwc', h.data_ptr(), ldh, lib.fptr(hid), lib.fptr(w2), lib.fptr(b2), hd, res.data_ptr(), ldr, out.data_ptr(), c,
             nb, hh * ww, c, lib.stream())
    return out


def softmax_rows(x: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(scale * x) over the last dim of a [rows, cols] matrix (row stride free)"""
    t, c, ld = _rows_meta(x)
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    lib.call('sfb_softmax_rows', x.data_ptr(), ld, out.data_ptr(), _rows_meta(out)[2], t, c, float(scale), lib.stream())
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    nb, h, w, c, ldx = _nhwc_meta(x)
    out = torch.empty(nb, 2 * h, 2 * w, c, dtype=torch.float32, device=x.device)
    lib.call('sfb_upsample2x_nhwc', x.data_ptr(), ldx, out.data_ptr(), c, nb, h, w, c, lib.stream())
    return out


# --------------------------------------------------------------------------------------------- layout
def nchw_to_nhwc(src: torch.Tensor, dst: torch.Tensor, c_off: int = 0, round_to_tf32: bool = False) -> torch.Tensor:
    nb, c, h, w = src.shape
    dnb, dh, dw, dc, ld = _nhwc_meta(dst)
    assert (dnb, dh, dw) == (nb, h, w) and c_off + c <= dc
    src = src.contiguous()
    lib.call('sfb_nchw_to_nhwc', lib.fptr(src, 'src'), dst.data_ptr(), nb, c, h, w, ld, c_off, int(round_to_tf32), lib.stream())
    return dst


def nhwc_to_nchw(src: torch.Tensor) -> torch.Tensor:
    nb, h, w, c, ld = _nhwc_meta(src)
    dst = torch.empty(nb, c, h, w, dtype=torch.float32, device=src.device)
    lib.call('sfb_nhwc_to_nchw', src.data_ptr(), lib.fptr(dst), nb, c, h, w, ld, lib.stream())
    return dst


def im2col4(x: torch.Tensor, kh: int, kw: int, pad: int) -> torch.Tensor:
    """[NB,H,W,4] -> [NB,H,W,ceil32(4*kh*kw)] patches (tap-major, channel-minor), zero outside the image and in the padding columns"""
    nb, h, w, c, ldx = _nhwc_meta(x)
    assert c == 4
    k = (4 * kh * kw + 31) // 32 * 32
    out = torch.empty(nb, h, w, k, dtype=torch.float32, device=x.device)
    lib.call('sfb_im2col4_nhwc', x.data_ptr(), ldx, out.data_ptr(), k, nb, h, w, kh, kw, pad, lib.stream())
    return out


def concat2(a: torch.Tensor, b: torch.Tensor, scale_b: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    nb, h, w, c1, lda = _nhwc_meta(a)
    _, _, _, c2, ldb = _nhwc_meta(b)
    if out is None:
        out = torch.empty(nb, h, w, c1 + c2, dtype=torch.float32, device=a.device)
    ldo = _nhwc_meta(out)[4]
    lib.call('sfb_concat2_nhwc', a.data_ptr(), c1, lda, b.data_ptr(), c2, ldb, float(scale_b), out.data_ptr(), ldo, nb * h * w, lib.stream())
    return out


def pixel_shuffle_silu(y: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    nb, h, w, c4, ld = _nhwc_meta(y)
    assert ld == c4 and c4 % 4 == 0
    co = c4 // 4
    if out is None:
        out = torch.empty(nb, 2 * h, 2 * w, co, dtype=torch.float32, device=y.device)
    ldo = _nhwc_meta(out)[4]
    lib.call('sfb_pixel_shuffle_silu_nhwc', y.data_ptr(), out.data_ptr(), nb, h, w, co, ldo, lib.stream())
    return out


# --------------------------------------------------------------------------------------------- norms
def groupnorm(x: torch.Tensor, groups: int, gamma: torch.Tensor, beta: torch.Tensor, film: Optional[torch.Tensor] = None,
              silu: bool = True, eps: float = 1e-5, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    nb, h, w, c, ldx = _nhwc_meta(x)
    if out is None:
        out = torch.empty(nb, h, w, c, dtype=torch.float32, device=x.device)
    ldy = _nhwc_meta(out)[4]
    ws = torch.empty(lib.load().sfb_groupnorm_ws_floats(nb, groups), dtype=torch.float32, device=x.device)
    film_ld = 0
    if film is not None:
        assert film.shape == (nb, 2 * c) and film.stride(1) == 1
        film_ld = film.stride(0)
    lib.call('sfb_groupnorm_nhwc', x.data_ptr(), ldx, nb, h * w, c, groups, lib.fptr(gamma), lib.fptr(beta), None if film is None else film.data_ptr(),
             film_ld, int(silu), float(eps),
             lib.fptr(ws), None, out.data_ptr(), ldy, lib.stream())
    return out


def layernorm(x: torch.Tensor, g: torch.Tensor, b: Optional[torch.Tensor] = None, pre_gelu: bool = False, round_to_tf32: bool = True,
              residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    t, c, ldx = _rows_meta(x)
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    ldy = _rows_meta(out)[2]
    ldr = _rows_meta(residual)[2] if residual is not None else 0
    lib.call('sfb_layernorm_rows', x.data_ptr(), ldx, lib.fptr(g.reshape(-1)), lib.fptr(b), None if residual is None else residual.data_ptr(), ldr,
             out.data_ptr(), ldy, t, c, int(pre_gelu), int(round_to_tf32), lib.stream())
    return out


# --------------------------------------------------------------------------------------------- small linears / misc
def linear_small(x: torch.Tensor, w: torch.Tensor, bias=None, pre: int = 0, post: int = 0, residual=None, round_to_tf32: bool = False,
                 out=None) -> torch.Tensor:
    m, k, ldx = _rows_meta(x)
    o = w.shape[0]
    assert w.shape[1] == k and w.is_contiguous()
    if out is None:
        out = torch.empty(*x.shape[:-1], o, dtype=torch.float32, device=x.device)
    ldy = _rows_meta(out)[2]
    ldr = _rows_meta(residual)[2] if residual is not None else 0
    lib.call('sfb_linear_small', x.data_ptr(), ldx, lib.fptr(w), lib.fptr(bias), None if residual is None else residual.data_ptr(), ldr,
             out.data_ptr(), ldy, m, k, o, pre, post, int(round_to_tf32), lib.stream())
    return out


def time_fourier(t: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    b, half = t.shape[0], w.shape[0]
    out = torch.empty(b, 2 * half + 1, dtype=torch.float32, device=t.device)
    t = t.contiguous()
    lib.call('sfb_time_fourier', lib.fptr(t), lib.fptr(w), lib.fptr(out), b, half, lib.stream())
    return out


def mq_attention(q, kv, null_kv, ckv, heads: int, dh: int) -> torch.Tensor:
    b, n = q.shape[0], q.shape[1]
    nc = 0 if ckv is None else ckv.shape[1]
    out = torch.empty(b, n, heads * dh, dtype=torch.float32, device=q.device)
    lib.call('sfb_mq_attention', lib.fptr(q), lib.fptr(kv), lib.fptr(null_kv), lib.fptr(ckv), lib.fptr(out), b, n, heads, dh, nc, float(dh ** -0.5),
             lib.stream())
    return out


def cross_attention(q, kvc, null_kv, heads: int, dh: int) -> torch.Tensor:
    b, n = q.shape[0], q.shape[1]
    nc = kvc.shape[1]
    out = torch.empty(b, n, heads * dh, dtype=torch.float32, device=q.device)
    lib.call('sfb_cross_attention', lib.fptr(q), lib.fptr(kvc), lib.fptr(null_kv), lib.fptr(out), b, n, heads, dh, nc, float(dh ** -0.5), lib.stream())
    return out


def gca_pool(x: torch.Tensor, wk: torch.Tensor, bk: torch.Tensor) -> torch.Tensor:
    nb, h, w, c, ldx = _nhwc_meta(x)
    ws = torch.empty(nb * h * w + 2 * nb + 2, dtype=torch.float32, device=x.device)
    pooled = torch.empty(nb, c, dtype=torch.float32, device=x.device)
    lib.call('sfb_gca_pool', x.data_ptr(), ldx, nb, h * w, c, lib.fptr(wk.reshape(-1)), lib.fptr(bk), lib.fptr(ws), lib.fptr(pooled), lib.stream())
    return pooled


def gate_residual(h: torch.Tensor, gate: Optional[torch.Tensor], res: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    nb, hh, ww, c, ldh = _nhwc_meta(h)
    ldr = _nhwc_meta(res)[4]
    if out is None:
        out = torch.empty(nb, hh, ww, c, dtype=torch.float32, device=h.device)
    ldo = _nhwc_meta(out)[4]
    lib.call('sfb_gate_residual_nhwc', h.data_ptr(), ldh, lib.fptr(gate), res.data_ptr(), ldr, out.data_ptr(), ldo, nb, hh * ww, c, lib.stream())
    return out
