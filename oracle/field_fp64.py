"""oracle/field_fp64.py -- fp64 restatement of the fused NGP field (csrc/ngp_field.cu) and of the compositing tail of
NeRFRenderer.run (renderer_df.py:414-456), with per-element error bounds.

TEST INFRASTRUCTURE ONLY.  It runs on the CPU (host tests) or on CUDA in fp64 (large GPU cases).

Field: the corner rows come from the C oracle (``ngp_oracle.grid_encode_forward(..., want_rows=True)``); the trilinear
weights are computed in fp32 exactly as ``grid_locate`` does (p = fma(u, scale, 0.5), frac = p - floor(p)) and then
promoted: the kernel's fp32 position arithmetic is part of what the field computes (at level 15 one ulp of p is 1e-3 of
a cell).  Everything after that -- MLP 32-64-64-4, blob, trunc_exp, sigmoid, all gradients -- is fp64.

Every output and gradient comes with an "absolute" companion: the same computation carried out on |weights| and
|terms|.  A fp32 evaluation that accumulates at most n rounded operations along any path is within gamma(n) * abs of the
exact value (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 3.1), so comparisons are per element:
    |got - ref| <= rtol * abs + slack + atol.
``slack`` covers the one discontinuity of the field's backward: a ReLU whose pre-activation is within the forward error
bound of 0 may take either branch in fp32, and the gradient routed through it is then either there or not.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import ngp_oracle as no

U32 = 2.0 ** -24     # unit roundoff of fp32 (round to nearest)


def gamma(n) -> float:
    """Higham's gamma_n = n u / (1 - n u): the relative bound of n chained fp32 roundings"""
    return n * U32 / (1 - n * U32)


# Per-point operation counts of the field along its longest rounding path:
#   encode: weights 3 products + 1 - frac (4) and 8 corner FMAs (8)                                  12
#   layer 0: K = 32 FMAs + bias (33); layer 1: K = 64 (65); output layer: K = 64 (65)                163
#   blob, exp / sigmoid, the divisions of the activations (<= 2 ulp each for expf, 8 in all)           8
#   backward: d3 (4), W2^T d3 (K = 4), W1^T D2 (K = 64), W0^T D1 (K = 64), w * dE (1)                137
# -> 320 roundings.  Sums over points (weight and bias gradients, embedding rows hit by several points) add their own
# accumulation length on top (wgrad_chain, rows_hit).
RTOL_POINT = gamma(320)
ATOL = 1e-30         # fp32 subnormal products; no compared value is anywhere near it


# ------------------------------------------------------------------------------------------------ fp32 helpers
def fma_f32(a: torch.Tensor, b: torch.Tensor, c: float) -> torch.Tensor:
    """correctly rounded fp32 fma(a, b, c) for fp32 a, b and an fp32-exact c.  a*b is exact in fp64; the sum is rounded
    once to fp64 and its exact error kept (TwoSum), which decides the only case where rounding to fp32 twice could
    differ from rounding once: an fp64 sum exactly on an fp32 midpoint."""
    a64, b64 = a.double(), b.double()
    prod = a64 * b64
    s = prod + c
    bb = s - prod
    err = (prod - (s - bb)) + (c - bb)
    r = s.float()
    r64 = r.double()
    other = torch.nextafter(r, torch.where(s > r64, torch.full_like(r, math.inf), torch.full_like(r, -math.inf)))
    mid = (r64 + other.double()) * 0.5
    fix = (s == mid) & (err != 0) & (torch.sign(err) == torch.sign(other.double() - r64))
    return torch.where(fix, other, r)


def normalized_inputs(x: torch.Tensor, bound: float) -> torch.Tensor:
    """u = (x + bound) / (2 bound) in fp32, as grid.py:142 and encode_point compute it"""
    x = x.float()
    return (x + np.float32(bound)) / np.float32(2 * bound)


def ray_points(rays_o: torch.Tensor, rays_d: torch.Tensor, z: torch.Tensor, bound: float) -> torch.Tensor:
    """x = clamp(o + d z, -bound, bound) in fp32 with a separate multiply and add (renderer_df.py:367-368, fetch_point).
    rays [N,3], z [N,T] -> [N*T,3]"""
    x = rays_o.float()[:, None, :] + rays_d.float()[:, None, :] * z.float()[:, :, None]
    return x.clamp(-bound, bound).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------ encoding geometry
def encode_geometry(x: torch.Tensor, geo: dict, level_scales, bound: float = 4.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """corner rows (absolute, int64 [B,L,8]) and fp64 trilinear weights [B,L,8] of fp32 points x [B,3], on x's device.
    Points outside the grid get weight 0 (and row 0) at every level."""
    dev = x.device
    u = normalized_inputs(x.cpu(), bound)
    _, _, rows = no.grid_encode_forward(u.numpy(), np.zeros((int(geo['offsets'][-1]), 2), np.float32), geo['offsets'], geo['S'], geo['H'],
                                        geo['gridtype'], geo['align_corners'], False, level_scales, want_rows=True)
    rows = torch.from_numpy(rows).permute(1, 0, 2).to(dev)                     # [B,L,8]
    u = u.to(dev)
    scales = torch.as_tensor(np.asarray(level_scales, np.float32), device=dev)
    L = scales.shape[0]
    p = fma_f32(u[:, None, :].expand(-1, L, -1), scales[None, :, None].expand(u.shape[0], -1, 3), 0.5)   # [B,L,3] fp32
    frac = (p - torch.floor(p)).double()
    w = torch.ones(u.shape[0], L, 8, dtype=torch.float64, device=dev)
    for corner in range(8):
        for d in range(3):
            w[:, :, corner] *= frac[:, :, d] if corner & (1 << d) else 1 - frac[:, :, d]
    live = rows >= 0
    return torch.where(live, rows, torch.zeros_like(rows)).long(), torch.where(live, w, torch.zeros_like(w))


def encode(rows: torch.Tensor, w: torch.Tensor, emb: torch.Tensor):
    """fp64 encoding [B, 32] (feature 2 l + c) and its absolute companion"""
    e = emb.to(w.device).double()[rows]                                          # [B,L,8,2]
    enc = (w[..., None] * e).sum(2).reshape(w.shape[0], -1)
    enc_abs = (w[..., None] * e.abs()).sum(2).reshape(w.shape[0], -1)
    return enc, enc_abs


# ------------------------------------------------------------------------------------------------ the field
def _trunc_exp_grad(pre):
    """ngp_activation.py:19-21: the backward of trunc_exp is exp(clamp(x, -15, 15))"""
    return torch.exp(pre.clamp(-15, 15))


class FieldFP64:
    """The field at fp32 points x [B,3] and its backward, in fp64, each value with its absolute companion ('<name>_abs').

    The backward is the chain rule written out (autograd_reference() restates it through torch autograd; the host tests
    hold the two together).  Written out, single defects can be injected for the sensitivity self-checks of the tests:
    ``flip_relu=(layer, point, unit)`` inverts one ReLU mask, ``drop_level=(point, level)`` skips one level of one
    point's embedding scatter, ``point_keep`` [B] bool drops whole points from every gradient."""

    def __init__(self, params: Dict[str, torch.Tensor], x: torch.Tensor, level_scales, bound: float = 4.0, device=None):
        dev = torch.device(device) if device is not None else x.device
        self.dev, self.bound, self.params = dev, bound, params
        self.geo = no.live_geometry(bound)
        self.x = x.float().to(dev)
        self.rows, self.w = encode_geometry(self.x, self.geo, level_scales, bound)
        self.W = [params[k].detach().to(dev).double() for k in no.PARAM_KEYS[1:]]
        self._forward()

    def _forward(self):
        W0, b0, W1, b1, W2, b2 = self.W
        self.enc, self.enc_abs = encode(self.rows, self.w, self.params['encoder.embeddings'])
        a1 = self.enc @ W0.T + b0
        a1_abs = self.enc_abs @ W0.abs().T + b0.abs()
        self.mask1, self.amb1 = a1 > 0, a1.abs() < RTOL_POINT * a1_abs    # exact zeros (abs 0) are not ambiguous
        self.h1, self.h1_abs = torch.relu(a1), a1_abs * (self.mask1 | self.amb1)
        a2 = self.h1 @ W1.T + b1
        a2_abs = self.h1_abs @ W1.abs().T + b1.abs()
        self.mask2, self.amb2 = a2 > 0, a2.abs() < RTOL_POINT * a2_abs
        self.h2, self.h2_abs = torch.relu(a2), a2_abs * (self.mask2 | self.amb2)
        self.o = self.h2 @ W2.T + b2
        self.o_abs = self.h2_abs @ W2.abs().T + b2.abs()
        r2 = (self.x.double() ** 2).sum(-1)
        blob = 5 * torch.exp(-r2 / 0.08)                                  # network_grid.py:69-75
        self.pre = self.o[:, 0] + blob
        self.pre_abs = self.o_abs[:, 0] + blob * (1 + r2 / 0.08)          # exp's argument carries r2 / 0.08 of relative rounding
        self.sigma = torch.exp(self.pre)
        self.rgb = torch.sigmoid(self.o[:, 1:])

    def forward(self) -> Dict[str, torch.Tensor]:
        s = self.rgb
        return dict(sigma=self.sigma, sigma_abs=self.sigma * (1 + self.pre_abs), rgb=s, rgb_abs=s + s * (1 - s) * self.o_abs[:, 1:])

    def backward(self, g_sigma: torch.Tensor, g_rgb: Optional[torch.Tensor], flip_relu=None, drop_level=None,
                 point_keep: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        W0, b0, W1, b1, W2, b2 = self.W
        B = self.x.shape[0]
        gs = g_sigma.to(self.dev).double()
        gc = torch.zeros(B, 3, dtype=torch.float64, device=self.dev) if g_rgb is None else g_rgb.to(self.dev).double()
        if point_keep is not None:
            k = point_keep.to(self.dev)
            gs, gc = gs * k, gc * k[:, None]
        e = _trunc_exp_grad(self.pre)
        s = self.rgb
        d3 = torch.cat([(gs * e)[:, None], gc * s * (1 - s)], 1)
        # the abs companion of sg (1 - sg) is sg (1 + sg): 1 - sg loses all relative accuracy when the sigmoid saturates
        d3_abs = torch.cat([(gs.abs() * e * (1 + self.pre_abs))[:, None], gc.abs() * s * ((1 + s) + (1 - s) * self.o_abs[:, 1:])], 1)
        dh2, dh2_abs = d3 @ W2, d3_abs @ W2.abs()
        m1, m2 = self.mask1.clone(), self.mask2.clone()
        if flip_relu is not None:
            layer, p, j = flip_relu
            m = m1 if layer == 1 else m2
            m[p, j] = ~m[p, j]
        d2, d2_abs = dh2 * m2, dh2_abs * (m2 | self.amb2)
        f2 = (dh2.abs() + RTOL_POINT * dh2_abs) * self.amb2               # either branch of an ambiguous ReLU
        dh1, dh1_abs, fh1 = d2 @ W1, d2_abs @ W1.abs(), f2 @ W1.abs()
        d1, d1_abs = dh1 * m1, dh1_abs * (m1 | self.amb1)
        self.dh = {1: dh1, 2: dh2}                                        # dL/dh before the masks (for choosing defects)
        f1 = fh1 * (m1 | self.amb1) + (dh1.abs() + RTOL_POINT * dh1_abs) * self.amb1
        denc, denc_abs, fenc = d1 @ W0, d1_abs @ W0.abs(), f1 @ W0.abs()
        out = {}
        zero = torch.zeros(4, 64, dtype=torch.float64, device=self.dev)
        for name, d, da, f, h, ha in (('sigma_net.net.2', d3, d3_abs, None, self.h2, self.h2_abs),
                                      ('sigma_net.net.1', d2, d2_abs, f2, self.h1, self.h1_abs),
                                      ('sigma_net.net.0', d1, d1_abs, f1, self.enc, self.enc_abs)):
            out[name + '.weight'], out[name + '.weight_abs'] = d.T @ h, da.T @ ha
            out[name + '.bias'], out[name + '.bias_abs'] = d.sum(0), da.sum(0)
            out[name + '.weight_slack'] = zero if f is None else f.T @ ha
            out[name + '.bias_slack'] = zero[:, 0] if f is None else f.sum(0)
        L = self.rows.shape[1]
        dl = denc.view(B, L, 1, 2)
        if drop_level is not None:
            dl = dl.clone()
            dl[drop_level[0], drop_level[1]] = 0
        rows = self.rows.reshape(-1)
        n = self.n_rows
        for key, g in (('', dl), ('_abs', denc_abs.view(B, L, 1, 2)), ('_slack', fenc.view(B, L, 1, 2))):
            ge = torch.zeros(n, 2, dtype=torch.float64, device=self.dev)
            ge.index_add_(0, rows, (self.w[..., None] * g).reshape(-1, 2))
            out['encoder.embeddings' + key] = ge
        # accumulation length of every embedding row: the points and corners that scatter into it
        hits = torch.zeros(n, dtype=torch.float64, device=self.dev)
        hits.index_add_(0, rows, (self.w > 0).reshape(-1).double())
        out['encoder.embeddings_hits'] = hits[:, None]
        return out

    @property
    def n_rows(self):
        return int(self.geo['offsets'][-1])

    def autograd_reference(self, g_sigma, g_rgb) -> Dict[str, torch.Tensor]:
        """the same values through torch autograd (fp64): encode as a gather of the embedding rows, trunc_exp with its
        clamped backward"""
        class TruncExp(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x):
                ctx.save_for_backward(x)
                return torch.exp(x)

            @staticmethod
            def backward(ctx, g):
                return g * _trunc_exp_grad(ctx.saved_tensors[0])

        p = {k: self.params[k].detach().to(self.dev).double().requires_grad_(True) for k in no.PARAM_KEYS}
        B, L = self.rows.shape[:2]
        enc = (self.w[..., None] * p['encoder.embeddings'][self.rows]).sum(2).reshape(B, -1)
        h = torch.relu(torch.nn.functional.linear(enc, p['sigma_net.net.0.weight'], p['sigma_net.net.0.bias']))
        h = torch.relu(torch.nn.functional.linear(h, p['sigma_net.net.1.weight'], p['sigma_net.net.1.bias']))
        o = torch.nn.functional.linear(h, p['sigma_net.net.2.weight'], p['sigma_net.net.2.bias'])
        sigma = TruncExp.apply(o[:, 0] + 5 * torch.exp(-(self.x.double() ** 2).sum(-1) / 0.08))
        rgb = torch.sigmoid(o[:, 1:])
        loss = (sigma * g_sigma.to(self.dev).double()).sum()
        if g_rgb is not None:
            loss = loss + (rgb * g_rgb.to(self.dev).double()).sum()
        loss.backward()
        out = {k: p[k].grad for k in no.PARAM_KEYS}
        out.update(sigma=sigma.detach(), rgb=rgb.detach())
        return out


def field_params_fp32(params: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {k: v.detach().float().contiguous() for k, v in params.items()}


# ------------------------------------------------------------------------------------------------ accumulation lengths
def wgrad_rtol(path: str, B: int, sm: int) -> float:
    """relative bound (w.r.t. the absolute companion) of a weight or bias gradient: the per-point bound plus the sum over
    the points, with the accumulation length of the path's reduction (ngp_field.cu):
      v2       each CTA chains 64 points per tile over ceil(tiles / CTAs) tiles, then one fp32 atomic per CTA
      v1-simt  mlp_wgrad_kernel: the same with 64-point chunks over min(Bp / 64, 2 SM) blocks
      v1-tc    3xTF32 wgmma (conv_wgmma.cu): the 64 (or 4) rows of D are one CTA's pixels, so the point range of Bp / 32
               k-steps is split over min(SM, k-steps / 4) CTAs (at least k-steps / 96), whose partial sums meet in fp32 reds;
               the tensor core's fp32 accumulation is not exactly rounded (2 u per add), and a 3xTF32 product carries ~2^-21
               (8 u).  The bias rows are summed by tape_rowsum_kernel: <= 64 chunks of 256 threads, 3 roundings per float4,
               then a warp tree (5), the 8 warps and one atomic per chunk."""
    Bp = (B + 63) // 64 * 64
    if path == 'v2':
        tiles = Bp // 64
        ctas = min(tiles, 2 * sm)
        return RTOL_POINT + gamma(-(-tiles // ctas) * 64 + ctas)
    if path == 'v1-simt':
        chunks = Bp // 64
        blocks = min(chunks, 2 * sm)
        return RTOL_POINT + gamma(-(-chunks // blocks) * 64 + blocks)
    if path == 'v1-tc':
        k_iters = Bp // 32
        splits = min(k_iters, max(-(-k_iters // 96), min(sm, max(k_iters // 4, 1))))
        gemm = -(-k_iters // splits) * 32 + splits
        chunks = min(-(-Bp // 4096), 64)
        rowsum = 3 * -(-(Bp // 4) // (chunks * 256)) + 5 + 8 + chunks
        return RTOL_POINT + 2 * gamma(max(gemm, rowsum)) + 8 * U32
    raise ValueError(path)


def violations(got: torch.Tensor, ref: torch.Tensor, ref_abs: torch.Tensor, rtol, slack=0.0, atol: float = ATOL) -> torch.Tensor:
    """boolean mask of the elements with |got - ref| > rtol * ref_abs + slack + atol (NaN anywhere is a violation)"""
    got = got.to(ref.device).double()
    err = (got - ref).abs()
    bound = rtol * ref_abs + slack + atol
    return ~(err <= bound)


def assert_within(name: str, got, ref, ref_abs, rtol, slack=0.0, atol: float = ATOL):
    bad = violations(got, ref, ref_abs, rtol, slack, atol)
    if bad.any():
        got = got.to(ref.device).double()
        err = (got - ref).abs()
        bound = rtol * ref_abs + slack + atol
        i = int(torch.argmax(torch.where(bad, err / bound, torch.zeros_like(err))).item())
        raise AssertionError(f'{name}: {int(bad.sum())} of {bad.numel()} elements outside |got - ref| <= rtol abs + slack + atol; worst flat index {i}: '
                             f'got {got.reshape(-1)[i].item():.9g} ref {ref.reshape(-1)[i].item():.9g} bound {torch.as_tensor(bound).expand_as(err).reshape(-1)[i].item():.3g}')


# ------------------------------------------------------------------------------------------------ compositing
# renderer_df.py:414-456 in fp64.  Every factor 1 - alpha + 1e-15 of the transmittance carries <= 6 u of absolute fp32 error (exp,
# the product delta * sigma, two subtractions, the epsilon) and the scan one more; summed over the 128 samples of a ray, the error of
# any transmittance, weight or weighted sum is within 11 * 128 roundings of the ray's scale (1 for the opacity and the normalised depth,
# max |rgb| + |bg| for the colour).  The backward's suffix sums are formed as the total minus a prefix, so their error scales with the
# largest |dL/dw| of the ray rather than with the suffix itself.
RTOL_COMP = gamma(12 * 128)


def composite(z: torch.Tensor, sigma: torch.Tensor, rgb: torch.Tensor, nears: torch.Tensor, fars: torch.Tensor, bg: float,
              g_image: torch.Tensor, g_ws: Optional[torch.Tensor], g_depth: Optional[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """forward and autograd backward of the compositing of [N,T] samples, fp64 on z's device, with absolute companions"""
    dev = z.device
    z, nears, fars = z.double(), nears.double()[:, None], fars.double()[:, None]
    sig = sigma.double().clone().requires_grad_(True)
    col = rgb.double().clone().requires_grad_(True)
    sample_dist = (fars - nears) / 64
    deltas = torch.cat([z[:, 1:] - z[:, :-1], sample_dist], 1)
    alphas = 1 - torch.exp(-deltas * sig)
    shifted = torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], 1)
    weights = alphas * torch.cumprod(shifted, 1)[:, :-1]
    ws = weights.sum(1)
    ori_z = ((z - nears) / (fars - nears)).clamp(0, 1)
    depth = (weights * ori_z).sum(1)
    image = (weights[..., None] * col).sum(1) + (1 - ws)[:, None] * bg
    gi = g_image.double().to(dev)
    loss = (image * gi).sum()
    gws = torch.zeros_like(ws) if g_ws is None else g_ws.double().to(dev)
    gdp = torch.zeros_like(ws) if g_depth is None else g_depth.double().to(dev)
    loss = loss + (ws * gws).sum() + (torch.nan_to_num(depth) * gdp).sum()
    loss.backward()
    G_abs = (gi.abs()[:, None, :] * (col.detach().abs() + abs(bg))).sum(-1) + gws.abs()[:, None] + gdp.abs()[:, None]
    scale = col.detach().abs().amax(dim=(1, 2)) + abs(bg)
    return dict(image=image.detach(), image_abs=scale[:, None].expand(-1, 3), weights_sum=ws.detach(), weights_sum_abs=torch.ones_like(ws),
                depth=depth.detach(), depth_abs=torch.ones_like(ws), g_sigma=sig.grad, g_rgb=col.grad,
                g_sigma_abs=deltas.detach().abs() * (G_abs + 2 * G_abs.amax(1, keepdim=True)),
                g_rgb_abs=gi.abs()[:, None, :].expand_as(col))


def upstream_grads(B: int, sigma: torch.Tensor, seed: int, scale_sigma: bool = True):
    """dL/dsigma [B] and dL/drgb [B,3] for the field tests: |N(0, 1)|, sigma's divided by sigma + 1.  They are one-signed on
    purpose: a weight or bias gradient is a sum over the points, and with zero-mean upstream gradients that sum cancels to
    1e-3 .. 1e-7 of its absolute companion, which puts one 64-point tile far below any worst-case summation bound.  One-signed,
    the sums stay within a small factor of their companions, and the bounds see a lost tile in every weight and bias gradient."""
    rng = np.random.default_rng(seed)
    gs = torch.from_numpy(np.abs(rng.standard_normal(B)).astype(np.float32))
    if scale_sigma:
        gs = (gs.double() / (sigma.double().cpu() + 1)).float()
    gc = torch.from_numpy(np.abs(rng.standard_normal((B, 3))).astype(np.float32))
    return gs, gc
