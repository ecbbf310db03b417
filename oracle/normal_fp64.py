"""oracle/normal_fp64.py -- fp64 restatement of the finite-difference normal stencils (csrc/ngp_field.cu, network_grid.py:91-164) on
top of field_fp64.FieldFP64, with absolute companions.

TEST INFRASTRUCTURE ONLY.

Rows: slot s of a point shifts component s // 2 by +eps (even s) or -eps (odd s) and clamps to [-bound, bound] (6 slots), or is the
point itself (1 slot, common_forward_smooth); sample j adds the jitter (u radius) 2 - radius, with u from Philox4x32-10 (counter
(point, slot, sample, 0), key split into two 32-bit words, low first; u = (r >> 8) 2^-24 of lanes 0..2).  The shifted and jittered
points are formed in fp32 exactly as the kernel forms them; the field and everything after it is fp64.

Bounds: sigma carries field_fp64's per-point bound; a slot mean adds its k-term sum; fd = 0.5 (m+ - m-) / eps cancels, so its bound is
rtol (abs+ + abs-) / (2 eps) (``fd_abs``).  A normalised normal is compared only where |fd| is well above that bound.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import field_fp64 as f64

FLT_MAX = float(np.finfo(np.float32).max)
RTOL_STENCIL = f64.RTOL_POINT + f64.gamma(4)          # the point's field, then the slot difference, * 0.5 and / eps


# ------------------------------------------------------------------------------------------------ Philox4x32-10
def philox4x32_10(ctr: np.ndarray, key) -> np.ndarray:
    """Random123's philox4x32-10: ctr [n,4] uint32, key (k0, k1) -> [n,4] uint32"""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    mask, sh = np.uint64(0xFFFFFFFF), np.uint64(32)
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> sh) ^ c[1] ^ k0, p1 & mask, (p0 >> sh) ^ c[3] ^ k1, p0 & mask]
        k0, k1 = (k0 + W0) & mask, (k1 + W1) & mask
    return np.stack(c, 1).astype(np.uint32)


def key_words(key: int):
    k = int(key) & 0xFFFFFFFFFFFFFFFF
    return k & 0xFFFFFFFF, k >> 32


def jitter(B: int, slots: int, k: int, key: int, radius: float) -> np.ndarray:
    """[B, slots, k, 3] fp32 jitter (u radius) 2 - radius, in the reference's operation order (network_grid.py:113)"""
    q, s, j = np.meshgrid(np.arange(B), np.arange(slots), np.arange(k), indexing='ij')
    ctr = np.stack([q.ravel(), s.ravel(), j.ravel(), np.zeros(q.size)], 1).astype(np.uint32)
    r = philox4x32_10(ctr, key_words(key))[:, :3]
    u = (r >> 8).astype(np.float32) * np.float32(2.0 ** -24)
    rad = np.float32(radius)
    return ((u * rad) * np.float32(2) - rad).reshape(B, slots, k, 3)


# ------------------------------------------------------------------------------------------------ stencil points
def stencil_points(x: np.ndarray, slots: int, k: int, eps: float, radius: float, key: Optional[int], bound: float = 4.0,
                   clamp_after_jitter: bool = False):
    """(xg [B, slots, k, 3] where the grid is evaluated, xb [B, slots, 3] where the blob is), fp32"""
    x = np.asarray(x, np.float32)
    B = x.shape[0]
    if slots == 6:
        xb = np.repeat(x[:, None, :], 6, 1).copy()
        e = np.float32(eps)
        for s in range(6):
            xb[:, s, s // 2] = xb[:, s, s // 2] + (-e if s & 1 else e)
        xb = np.clip(xb, np.float32(-bound), np.float32(bound))
    else:
        xb = x[:, None, :].copy()
    xg = np.repeat(xb[:, :, None, :], k, 2)
    if key is not None:
        xg = xg + jitter(B, slots, k, key, radius)
        if clamp_after_jitter:
            xg = np.clip(xg, np.float32(-bound), np.float32(bound))
    return xg.astype(np.float32), xb.astype(np.float32)


class StencilFP64:
    """The stencil at fp32 points x [B,3]: fd, normal (slots = 6) or sigma, albedo (slots = 1), with absolute companions, and the
    plain stencil's backward.  Defects for the sensitivity self-checks: drop_slot (that slot's sigma is 0), flip_slot (its sign in fd
    flips), blob_at_jitter (blob at the jittered point), clamp_after_jitter."""

    def __init__(self, params: Dict[str, torch.Tensor], x, level_scales, *, slots=6, k=1, eps=1e-2, radius=0.0, key=None, bound=4.0,
                 device=None, drop_slot=None, flip_slot=None, blob_at_jitter=False, clamp_after_jitter=False):
        x = x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
        self.B, self.slots, self.k, self.eps = x.shape[0], slots, k, eps
        xg, xb = stencil_points(x, slots, k, eps, radius, key, bound, clamp_after_jitter)
        rows = torch.from_numpy(xg.reshape(-1, 3))
        self.field = f64.FieldFP64(params, rows if device is None else rows.to(device), level_scales, bound)
        dev = self.field.dev
        fld = self.field
        blob_at = torch.from_numpy(xg.reshape(-1, 3) if blob_at_jitter else np.repeat(xb[:, :, None, :], k, 2).reshape(-1, 3)).to(dev).double()
        r2 = (blob_at ** 2).sum(-1)
        blob = 5 * torch.exp(-r2 / 0.08)
        pre = fld.o[:, 0] + blob
        pre_abs = fld.o_abs[:, 0] + blob * (1 + r2 / 0.08)
        sigma = torch.exp(pre)
        sigma = torch.where(sigma > FLT_MAX, torch.full_like(sigma, float('inf')), sigma)       # fp32 overflow
        sigma_abs = sigma * (1 + pre_abs)
        shape = (self.B, slots, k)
        sigma, sigma_abs = sigma.view(shape), sigma_abs.view(shape)
        if drop_slot is not None:
            sigma = sigma.clone()
            sigma[:, drop_slot] = 0
        self.m, self.m_abs = sigma.mean(2), sigma_abs.mean(2)
        if slots == 1:
            rgb = fld.rgb.view(self.B, 1, k, 3)
            rgb_abs = (rgb + rgb * (1 - rgb) * fld.o_abs[:, 1:].view(self.B, 1, k, 3))
            self.sigma, self.sigma_abs = self.m[:, 0], self.m_abs[:, 0]
            self.albedo, self.albedo_abs = rgb.mean(2)[:, 0], rgb_abs.mean(2)[:, 0]
            return
        sign = torch.tensor([1.0, -1.0] * 3, dtype=torch.float64, device=dev)
        if flip_slot is not None:
            sign[flip_slot] = -sign[flip_slot]
        ms = self.m * sign
        self.fd = 0.5 * (ms[:, 0::2] + ms[:, 1::2]) / eps
        self.fd_abs = 0.5 * (self.m_abs[:, 0::2] + self.m_abs[:, 1::2]) / eps

    def rtol(self) -> float:
        return RTOL_STENCIL + f64.gamma(self.k + 1)

    def normal(self):
        """(normal [B,3] with NaN -> 0, reliable [B] bool: |fd| at least 10 times its bound)"""
        fd = self.fd
        r = torch.sqrt(torch.clamp((fd * fd).sum(-1, keepdim=True), min=1e-20))
        n = fd / r
        n = torch.where(torch.isnan(n), torch.zeros_like(n), n)
        err = self.rtol() * self.fd_abs.norm(dim=-1)
        reliable = torch.isfinite(fd).all(-1) & (fd.norm(dim=-1) > 10 * err)
        return n, reliable

    def normal_rtol(self):
        """per-point bound of a normalised normal's elements where normal()'s reliable is set: twice the relative error of fd, plus the
        kernel's normalisation (a square sum, a sqrt and a division)"""
        return 2 * self.rtol() * self.fd_abs.norm(dim=-1, keepdim=True) / self.fd.norm(dim=-1, keepdim=True) + f64.gamma(8)

    def backward(self, fd32: torch.Tensor, g_normal: Optional[torch.Tensor] = None, g_fd: Optional[torch.Tensor] = None):
        """parameter gradients of the plain stencil (k = 1) for dL/dnormal at the kernel's fd32 [B,3] (or dL/dfd directly); the
        returned dict is field_fp64.FieldFP64.backward's over the 6 B rows"""
        dev = self.field.dev
        if g_fd is None:
            fd = fd32.to(dev).double()
            g = g_normal.to(dev).double()
            ss = (fd * fd).sum(-1, keepdim=True)
            r = torch.sqrt(torch.clamp(ss, min=1e-20))
            dot = (g * fd).sum(-1, keepdim=True)
            gfd = g / r - torch.where(ss > 1e-20, fd * dot / r ** 3, torch.zeros_like(fd))
            gfd = torch.where(torch.isfinite(ss), gfd, torch.zeros_like(gfd))
        else:
            gfd = g_fd.to(dev).double()
        gd = 0.5 * gfd / self.eps                                                 # [B,3]
        gs = torch.stack([gd, -gd], -1).reshape(self.B * 6)                       # slot 2a: +, 2a + 1: -
        return self.field.backward(gs, None)


def reference_autograd(params: Dict[str, torch.Tensor], x, level_scales, g_normal, eps=1e-2, bound=4.0):
    """normal(x) (network_grid.py:91-106, 155-164) restated directly in torch fp64 autograd -- six field evaluations at the clamped shifted
    points, 0.5 (pos - neg) / eps, safe_normalize, NaN -> 0 -- and the parameter gradients of <normal, g_normal>"""
    xs, _ = stencil_points(np.asarray(x, np.float32), 6, 1, eps, 0.0, None, bound)
    fld = f64.FieldFP64(params, torch.from_numpy(xs.reshape(-1, 3)), level_scales, bound)

    class TruncExp(torch.autograd.Function):          # ngp_activation.py:10-21
        @staticmethod
        def forward(ctx, v):
            ctx.save_for_backward(v)
            return torch.exp(v)

        @staticmethod
        def backward(ctx, g):
            return g * torch.exp(ctx.saved_tensors[0].clamp(-15, 15))

    p = {k: params[k].detach().double().requires_grad_(True) for k in params}
    B = xs.shape[0]
    Bt, L = fld.rows.shape[:2]
    enc = (fld.w[..., None] * p['encoder.embeddings'][fld.rows]).sum(2).reshape(Bt, -1)
    h = torch.relu(torch.nn.functional.linear(enc, p['sigma_net.net.0.weight'], p['sigma_net.net.0.bias']))
    h = torch.relu(torch.nn.functional.linear(h, p['sigma_net.net.1.weight'], p['sigma_net.net.1.bias']))
    o = torch.nn.functional.linear(h, p['sigma_net.net.2.weight'], p['sigma_net.net.2.bias'])
    sigma = TruncExp.apply(o[:, 0] + 5 * torch.exp(-(fld.x.double() ** 2).sum(-1) / 0.08)).view(B, 6)
    fd = torch.stack([0.5 * (sigma[:, 2 * a] - sigma[:, 2 * a + 1]) / eps for a in range(3)], -1)
    n = fd / torch.sqrt(torch.clamp((fd * fd).sum(-1, keepdim=True), min=1e-20))
    n = torch.where(torch.isnan(n), torch.zeros_like(n), n)
    (n * g_normal.double()).sum().backward()
    out = {k: p[k].grad for k in p}
    out.update(fd=fd.detach(), normal=n.detach())
    return out
