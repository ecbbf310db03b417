"""NeRFNetwork -- host-side mirror of external/nerf/network_grid.py (reference): the Instant-NGP scene that
SparseFusion optimises (sparsefusion/distillation.py:164-165).

Same constructor (``NeRFNetwork(opt)``), parameter names (``encoder.embeddings``, ``encoder.offsets``,
``sigma_net.net.{0,1,2}.{weight,bias}``) so checkpoints round-trip (distillation.py:495-496), same methods
(``common_forward``, ``density``, ``forward(x, d, l, ratio, shading)``, ``get_params(lr)``, ``normal``,
``finite_difference_normal``, ``common_forward_smooth``, ``finite_difference_normal_smooth``).  The field query
(grid encode + MLP + activations) is ONE fused kernel with a fused backward (csrc/ngp_field.cu) instead of the
reference's kernel_grid + permute + three cuBLAS GEMMs + elementwise launches.

``forward`` has every shading of the reference (network_grid.py:167-197): 'albedo' (SparseFusion's), 'textureless'
and 'normal' (the smoothed normal, no gradient) and lambertian for any other string (the plain normal, with gradient).
A normal is a finite-difference stencil evaluated and reduced inside one tiled field kernel (6 field rows per point, or
6 x 10 jittered rows for the smoothed normal), with a stencil backward for the plain one.  The jitter of the smoothed
stencils is Philox4x32-10 keyed by one int64 drawn from the current CUDA generator: ``torch.cuda.manual_seed``
reproduces it, though it is not the stream of numbers ``torch.rand_like`` would give.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib as lib
from .gridencoder import GridEncoder
from .renderer_df import NeRFRenderer


def get_default_torch_ngp_opt():
    """sparsefusion/distillation.py:500-526 (the options the render kernels are parameterised by)"""
    return SimpleNamespace(cuda_ray=False, max_steps=256, num_steps=64, upsample_steps=64, update_extra_interval=16, max_ray_batch=4096,
                           albedo_iters=1000, bg_radius=0, density_thresh=10, fp16=True, backbone='grid', w=128, h=128, hw_scale=2, bound=4,
                           min_near=0.1, dt_gamma=0, lambda_entropy=1e-4, lambda_opacity=0, lambda_orient=1e-2, lambda_smooth=0)


def shade(albedo, normal, l, ratio, shading):
    """network_grid.py:187-197: (color, normal) from the albedo and the normal under light direction l [3]"""
    lam = ratio + (1 - ratio) * (normal @ -l).clamp(min=0)
    if shading == 'textureless':
        color = lam.unsqueeze(-1).repeat(1, 3) * 0.8 + .2
    elif shading == 'normal':
        color = (normal + 1) / 2
    else:
        color = albedo * lam.unsqueeze(-1)
    return color, normal


class MLP(nn.Module):
    """parameter container with the reference's layout (network_grid.py:14-33); evaluated inside the fused field kernel"""

    def __init__(self, dim_in, dim_out, dim_hidden, num_layers, bias=True):
        super().__init__()
        self.dim_in, self.dim_out, self.dim_hidden, self.num_layers = dim_in, dim_out, dim_hidden, num_layers
        self.net = nn.ModuleList([nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=bias)
                                  for l in range(num_layers)])


class _FieldFn(torch.autograd.Function):
    """sigma, albedo = common_forward(x)   (network_grid.py:77-88) for explicit points x [B,3]"""

    @staticmethod
    def forward(ctx, net, x, emb, w0, b0, w1, b1, w2, b2):
        enc = net.encoder
        B = x.shape[0]
        sigma = torch.empty(B, device=x.device)
        rgb = torch.empty(B, 3, device=x.device)
        f = lib.fptr
        ctx.geo = (float(math.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound))
        lib.call('sfb_ngp_field_forward', f(x), None, None, None, 0, B, f(emb), lib.iptr(enc.offsets), *ctx.geo, f(w0), f(b0), f(w1), f(b1), f(w2),
                 f(b2), f(sigma), f(rgb), lib.stream())
        ctx.save_for_backward(x, emb, w0, b0, w1, b1, w2, b2)
        ctx.offsets = enc.offsets
        return sigma, rgb

    @staticmethod
    def backward(ctx, g_sigma, g_rgb):
        x, emb, w0, b0, w1, b1, w2, b2 = ctx.saved_tensors
        B = x.shape[0]
        f = lib.fptr
        g_sigma = torch.zeros(B, device=x.device) if g_sigma is None else g_sigma.contiguous()
        g_rgb = None if g_rgb is None else g_rgb.contiguous()
        tape = torch.empty(lib.load().sfb_ngp_field_tape_floats(B), device=x.device)
        g_emb = torch.zeros_like(emb)
        gw0, gb0, gw1, gb1, gw2, gb2 = (torch.zeros_like(t) for t in (w0, b0, w1, b1, w2, b2))
        lib.call('sfb_ngp_field_backward', f(x), None, None, None, 0, B, f(emb), lib.iptr(ctx.offsets), *ctx.geo, f(w0), f(b0), f(w1), f(b1), f(w2),
                 f(b2), f(g_sigma), f(g_rgb), f(g_emb), f(gw0), f(gb0), f(gw1), f(gb1), f(gw2), f(gb2), f(tape), lib.stream())
        return None, None, g_emb, gw0, gb0, gw1, gb1, gw2, gb2


def _src(x=None, rays=None):
    """the point source of a field kernel call: explicit points x [B,3], or ray samples rays = (rays_o [N,3], rays_d [N,3],
    z [N,T]) at clamp(o + d z, -bound, bound)"""
    f = lib.fptr
    if x is not None:
        return (f(x), None, None, None, 0)
    o, d, z = rays
    return (None, f(o), f(d), f(z), z.shape[1])


def stencil_forward(net, B, *, x=None, rays=None, slots=6, k=1, eps=1e-2, radius=0.0, key=None, want_fd=True, want_normal=True):
    """one sfb_ngp_field_normal_forward call (no autograd): slots = 6 -> (fd [B,3] or None, normal [B,3] or None);
    slots = 1 -> (sigma [B], albedo [B,3]).  key: int64 [1] on the device (the jitter), or None with k = 1"""
    emb, w0, b0, w1, b1, w2, b2 = (t.detach() for t in net._field_params())
    enc = net.encoder
    dev = emb.device
    f = lib.fptr
    a = torch.empty(B, 3, device=dev) if (slots == 1 or want_fd) else None
    b = torch.empty(B, 3, device=dev) if (slots == 6 and want_normal) else None
    sig = torch.empty(B, device=dev) if slots == 1 else None
    lib.call('sfb_ngp_field_normal_forward', *_src(x, rays), B, f(emb), lib.iptr(enc.offsets), float(math.log2(enc.per_level_scale)),
             int(enc.base_resolution), float(net.bound), f(w0), f(b0), f(w1), f(b1), f(w2), f(b2), slots, k, float(eps), float(radius),
             None if key is None else lib.ptr(key, torch.int64, 'key'), f(a) if slots == 6 and a is not None else None, f(b) if b is not None else None,
             f(sig) if sig is not None else None, f(a) if slots == 1 else None, lib.stream())
    return (sig, a) if slots == 1 else (a, b)


def jitter_key(device):
    """the Philox key of one jittered stencil: an int64 drawn on the device from the current CUDA generator (no host sync)"""
    return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=device)


class _NormalFn(torch.autograd.Function):
    """finite_difference_normal(x, eps) (network_grid.py:91-106), or with normalize=True normal(x) = safe_normalize of it with NaN -> 0
    (:155-164), at explicit points x or ray samples; gradients into every field parameter through the 6 stencil rows"""

    @staticmethod
    def forward(ctx, net, x, rays, eps, normalize, emb, w0, b0, w1, b1, w2, b2):
        B = x.shape[0] if x is not None else rays[2].numel()
        fd, n = stencil_forward(net, B, x=x, rays=rays, eps=eps)
        ctx.net, ctx.x, ctx.rays, ctx.eps, ctx.normalize = net, x, rays, eps, normalize
        ctx.save_for_backward(fd, emb, w0, b0, w1, b1, w2, b2)
        return n if normalize else fd

    @staticmethod
    def backward(ctx, g):
        fd, emb, w0, b0, w1, b1, w2, b2 = ctx.saved_tensors
        net = ctx.net
        enc = net.encoder
        f = lib.fptr
        g = g.contiguous()
        g_emb = torch.zeros_like(emb)
        gw0, gb0, gw1, gb1, gw2, gb2 = (torch.zeros_like(t) for t in (w0, b0, w1, b1, w2, b2))
        lib.call('sfb_ngp_field_normal_backward', *_src(ctx.x, ctx.rays), fd.shape[0], f(emb), lib.iptr(enc.offsets),
                 float(math.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound), f(w0), f(b0), f(w1), f(b1), f(w2), f(b2),
                 float(ctx.eps), f(fd), f(g) if ctx.normalize else None, None if ctx.normalize else f(g), f(g_emb), f(gw0), f(gb0), f(gw1), f(gb1),
                 f(gw2), f(gb2), lib.stream())
        return None, None, None, None, None, g_emb, gw0, gb0, gw1, gb1, gw2, gb2


class NeRFNetwork(NeRFRenderer):
    def __init__(self, opt, num_layers=3, hidden_dim=64, num_layers_bg=2, hidden_dim_bg=64):
        super().__init__(opt)
        if num_layers != 3 or hidden_dim != 64:
            raise NotImplementedError('the fused field kernel is built for the SparseFusion MLP (3 layers, 64 hidden)')
        if self.bg_radius > 0:
            raise NotImplementedError('bg_radius > 0 (background network) is not used by SparseFusion (distillation.py:512)')
        self.num_layers, self.hidden_dim = num_layers, hidden_dim
        # get_encoder('tiledgrid', input_dim=3, log2_hashmap_size=16, desired_resolution=2048*bound)  (network_grid.py:50, ngp_encoder.py:69-71)
        self.encoder = GridEncoder(input_dim=3, num_levels=16, level_dim=2, base_resolution=16, log2_hashmap_size=16,
                                   desired_resolution=2048 * self.bound, gridtype='tiled', align_corners=False)
        self.in_dim = self.encoder.output_dim
        self.sigma_net = MLP(self.in_dim, 4, hidden_dim, num_layers, bias=True)
        self.bg_net = None

    def _field_params(self):
        n = self.sigma_net.net
        return (self.encoder.embeddings, n[0].weight, n[0].bias, n[1].weight, n[1].bias, n[2].weight, n[2].bias)

    def gaussian(self, x):
        d = (x ** 2).sum(-1)
        return 5 * torch.exp(-d / (2 * 0.2 ** 2))

    def common_forward(self, x):
        """x: [N, 3] in [-bound, bound] -> sigma [N], albedo [N, 3]"""
        if not x.is_cuda:
            raise RuntimeError('NeRFNetwork.common_forward needs CUDA tensors (no CPU fallback)')
        x = x.contiguous().view(-1, 3).float()
        with torch.cuda.device(x.device):
            return _FieldFn.apply(self, x, *self._field_params())

    def _points(self, x):
        if not x.is_cuda:
            raise RuntimeError('NeRFNetwork needs CUDA tensors (no CPU fallback)')
        return x.detach().contiguous().view(-1, 3).float()

    def finite_difference_normal(self, x, epsilon=1e-2):
        """network_grid.py:91-106: fd [N,3] = 0.5 (sigma(clamp(x + eps e_a)) - sigma(clamp(x - eps e_a))) / eps, with gradient"""
        x = self._points(x)
        with torch.cuda.device(x.device):
            return _NormalFn.apply(self, x, None, float(epsilon), False, *self._field_params())

    @torch.no_grad()
    def common_forward_smooth(self, x, radius=1e-2, k=5):
        """network_grid.py:108-130: sigma [N] and albedo [N,3] averaged over k jittered copies of x (the blob at x itself)"""
        x = self._points(x)
        with torch.cuda.device(x.device):
            return stencil_forward(self, x.shape[0], x=x, slots=1, k=int(k), radius=float(radius), key=jitter_key(x.device))

    @torch.no_grad()
    def finite_difference_normal_smooth(self, x, epsilon=3e-1):
        """network_grid.py:132-152: the stencil of finite_difference_normal on common_forward_smooth (radius 0.3, k = 10, as hard-coded there)"""
        x = self._points(x)
        with torch.cuda.device(x.device):
            return stencil_forward(self, x.shape[0], x=x, k=10, eps=float(epsilon), radius=3e-1, key=jitter_key(x.device), want_normal=False)[0]

    def normal(self, x, smooth=False):
        """network_grid.py:155-164: safe_normalize(fd) with NaN -> 0; the smoothed one carries no gradient"""
        x = self._points(x)
        with torch.cuda.device(x.device):
            if smooth:
                with torch.no_grad():
                    return stencil_forward(self, x.shape[0], x=x, k=10, eps=3e-1, radius=3e-1, key=jitter_key(x.device), want_fd=False)[1]
            return _NormalFn.apply(self, x, None, 1e-2, True, *self._field_params())

    def forward(self, x, d, l=None, ratio=1, shading='textureless'):
        """network_grid.py:167-197 -> (sigma, color, normal); normal is None for 'albedo'"""
        if shading == 'albedo':
            sigma, color = self.common_forward(x)
            return sigma, color, None
        sigma, albedo = self.common_forward(x)
        normal = self.normal(x, smooth=shading in ('textureless', 'normal'))
        return (sigma, *shade(albedo, normal, l, ratio, shading))

    def density(self, x):
        sigma, albedo = self.common_forward(x)
        return {'sigma': sigma, 'albedo': albedo}

    def get_params(self, lr):
        return [{'params': self.encoder.parameters(), 'lr': lr * 10}, {'params': self.sigma_net.parameters(), 'lr': lr}]
