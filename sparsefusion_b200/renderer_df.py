"""NeRFRenderer -- host-side mirror of external/nerf/renderer_df.py (reference), the volume renderer the
distillation loop drives (sparsefusion/distillation.py:209,282,380).

Same class / method names and keyword arguments (``render``, ``render_batched``, ``run``, ``run_cuda``,
``update_extra_state``, ``reset_extra_state``), same result dictionaries, same registered buffers
(``aabb_train``, ``aabb_infer``, and ``density_grid`` / ``density_bitfield`` / ``step_counter`` with cuda_ray), so
``ngp_network.render(rays_o, rays_d, staged=False, perturb=True, bg_color=0, ..., **vars(opt))`` works unchanged.
``export_mesh`` runs the reference's mcubes export on the GPU (sparsefusion_b200/mesh.py: lattice query through the fused field kernel,
Gaussian smoothing, marching cubes, OBJ); with ``texture_size`` it also bakes the field's albedo into a per-triangle UV atlas and writes a
textured OBJ (the reference's xatlas/nvdiffrast export is dead code there).

Every shading of the reference runs on both paths: 'albedo' (SparseFusion's) on the fused path below; 'lambertian' (any other
string), 'textureless' and 'normal' shade the field with finite-difference normals computed as stencils inside the tiled field
kernel (network_grid.py), and return the reference's loss_orient / loss_smooth.

``run`` is the default path (opt.cuda_ray = False, distillation.py:505).  The reference spells it as ~150 eager
launches and evaluates the field three times (coarse, fine, colour); here it is seven kernels and every point is
evaluated once (sigma+rgb at the num_steps coarse and the upsample_steps importance depths, gathered into sorted
order), with an analytic backward -- gradients equal the reference's because its fine/colour passes see the same
points and parameters.  'albedo' renders at any num_steps >= 1, upsample_steps >= 0 with num_steps + upsample_steps
<= 256 (num_steps >= 2 when upsample_steps > 0); the normal-based shadings at 64 + 64.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import _lib as lib
from . import raymarching


def _sorted_samples(net, rays_o, rays_d, aabb, min_near, perturb_noise, pdf_u, emb, w0, b0, w1, b1, w2, b2, num_steps=64, upsample_steps=64):
    """renderer_df.run :328-412: near/far, the num_steps stratified and upsample_steps importance depths, and sigma, rgb at the
    T = num_steps + upsample_steps sorted samples -> (zs [N,T], sigma [N,T], rgb [N,T,3], nears [N], fars [N]).  With upsample_steps = 0
    these are the coarse samples themselves (the reference skips importance sampling, :372)."""
    N = rays_o.shape[0]
    dev = rays_o.device
    enc = net.encoder
    S, H, bound = float(math.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound)
    st = lib.stream()
    f = lib.fptr
    Tc, Tf = num_steps, upsample_steps
    nears, fars = torch.empty(N, device=dev), torch.empty(N, device=dev)
    zc = torch.empty(N, Tc, device=dev)
    lin = torch.linspace(0.0, 1.0, Tc, device=dev)
    lib.call('sfb_ray_coarse_z', f(rays_o), f(rays_d), f(aabb), float(min_near), f(lin), f(perturb_noise), N, Tc, f(nears), f(fars), f(zc), st)
    # the field is evaluated ONCE per sample: coarse pass (sigma + rgb at the Tc stratified depths), importance pass (the Tf new depths),
    # then a gather into sorted order -- the values of the coarse samples are the same numbers a second evaluation would produce
    sig_c, rgb_c = torch.empty(N, Tc, device=dev), torch.empty(N, Tc, 3, device=dev)
    args = (f(emb), lib.iptr(enc.offsets), S, H, bound, f(w0), f(b0), f(w1), f(b1), f(w2), f(b2))
    lib.call('sfb_ngp_field_forward', None, f(rays_o), f(rays_d), f(zc), Tc, N * Tc, *args, f(sig_c), f(rgb_c), st)
    if Tf == 0:
        return zc, sig_c, rgb_c, nears, fars
    zs, zn = torch.empty(N, Tc + Tf, device=dev), torch.empty(N, Tf, device=dev)
    src_of = torch.empty(N, Tc + Tf, dtype=torch.uint8, device=dev)
    lib.call('sfb_ray_resample_ex', f(zc), f(sig_c), f(nears), f(fars), f(pdf_u), 0, N, Tc, Tf, f(zs), f(zn), src_of.data_ptr(), st)
    sig_n, rgb_n = torch.empty(N, Tf, device=dev), torch.empty(N, Tf, 3, device=dev)
    lib.call('sfb_ngp_field_forward', None, f(rays_o), f(rays_d), f(zn), Tf, N * Tf, *args, f(sig_n), f(rgb_n), st)
    sigma, rgb = torch.empty(N, Tc + Tf, device=dev), torch.empty(N, Tc + Tf, 3, device=dev)
    lib.call('sfb_ray_gather_sorted_steps', src_of.data_ptr(), f(sig_c), f(rgb_c), f(sig_n), f(rgb_n), N, Tc, Tf, f(sigma), f(rgb), st)
    return zs, sigma, rgb, nears, fars


def _field_backward_at_samples(net, rays_o, rays_d, zs, g_sigma, g_rgb, emb, w0, b0, w1, b1, w2, b2):
    """parameter gradients of <sigma, g_sigma> + <rgb, g_rgb> over the field at the [N,T] ray samples"""
    enc = net.encoder
    dev = rays_o.device
    f = lib.fptr
    B = zs.numel()
    tape = torch.empty(lib.load().sfb_ngp_field_tape_floats(B), device=dev)
    g_emb = torch.zeros_like(emb)
    gw0, gb0, gw1, gb1, gw2, gb2 = (torch.zeros_like(t) for t in (w0, b0, w1, b1, w2, b2))
    lib.call('sfb_ngp_field_backward', None, f(rays_o), f(rays_d), f(zs), zs.shape[1], B, f(emb), lib.iptr(enc.offsets), float(math.log2(enc.per_level_scale)),
             int(enc.base_resolution), float(net.bound), f(w0), f(b0), f(w1), f(b1), f(w2), f(b2), f(g_sigma), None if g_rgb is None else f(g_rgb),
             f(g_emb), f(gw0), f(gb0), f(gw1), f(gb1), f(gw2), f(gb2), f(tape), lib.stream())
    return g_emb, gw0, gb0, gw1, gb1, gw2, gb2


class _RunRender(torch.autograd.Function):
    """renderer_df.run (:310-468) for shading='albedo', bg_radius == 0: returns (image [N,3], depth [N], weights_sum [N], nears, fars)"""

    @staticmethod
    def forward(ctx, net, rays_o, rays_d, aabb, min_near, bg_color, num_steps, upsample_steps, perturb_noise, pdf_u, emb, w0, b0, w1, b1, w2, b2):
        N = rays_o.shape[0]
        dev = rays_o.device
        f = lib.fptr
        zs, sigma, rgb, nears, fars = _sorted_samples(net, rays_o, rays_d, aabb, min_near, perturb_noise, pdf_u, emb, w0, b0, w1, b1, w2, b2,
                                                      num_steps, upsample_steps)
        image, depth, ws = torch.empty(N, 3, device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev)
        lib.call('sfb_ray_composite_forward_steps', f(zs), f(sigma), f(rgb), f(nears), f(fars), float(bg_color), N, num_steps, upsample_steps, f(image),
                 f(depth), f(ws), lib.stream())
        ctx.save_for_backward(rays_o, rays_d, zs, sigma, rgb, nears, fars, emb, w0, b0, w1, b1, w2, b2)
        ctx.net, ctx.bg, ctx.steps = net, float(bg_color), (num_steps, upsample_steps)
        ctx.mark_non_differentiable(nears, fars)
        return image, depth, ws, nears, fars

    @staticmethod
    def backward(ctx, g_image, g_depth, g_ws, _gn, _gf):
        rays_o, rays_d, zs, sigma, rgb, nears, fars, emb, w0, b0, w1, b1, w2, b2 = ctx.saved_tensors
        g_sigma, g_rgb = _composite_backward(zs, sigma, rgb, nears, fars, ctx.bg, g_image, g_depth, g_ws, *ctx.steps)
        grads = _field_backward_at_samples(ctx.net, rays_o, rays_d, zs, g_sigma, g_rgb, emb, w0, b0, w1, b1, w2, b2)
        return (None, None, None, None, None, None, None, None, None, None, *grads)


def _composite_backward(zs, sigma, rgb, nears, fars, bg, g_image, g_depth, g_ws, num_steps, upsample_steps):
    """sfb_ray_composite_backward_steps: (dL/dsigma [N,T], dL/drgb [N,T,3])"""
    N, T = zs.shape
    dev = zs.device
    f = lib.fptr
    g_image = g_image.contiguous() if g_image is not None else torch.zeros(N, 3, device=dev)
    g_sigma, g_rgb = torch.empty(N, T, device=dev), torch.empty(N, T, 3, device=dev)
    g_ws = None if g_ws is None else g_ws.contiguous()
    g_depth = None if g_depth is None else g_depth.contiguous()
    lib.call('sfb_ray_composite_backward_steps', f(zs), f(sigma), f(rgb), f(nears), f(fars), bg, N, num_steps, upsample_steps, f(g_image),
             None if g_ws is None else f(g_ws), None if g_depth is None else f(g_depth), f(g_sigma), f(g_rgb), lib.stream())
    return g_sigma, g_rgb


class _RaySamples(torch.autograd.Function):
    """the field at the 128 sorted samples of run (renderer_df.py:328-412) as an autograd node: (sigma [N,128], albedo [N,128,3], zs, nears,
    fars); the backward runs the field backward at the same samples"""

    @staticmethod
    def forward(ctx, net, rays_o, rays_d, aabb, min_near, perturb_noise, pdf_u, emb, w0, b0, w1, b1, w2, b2):
        zs, sigma, rgb, nears, fars = _sorted_samples(net, rays_o, rays_d, aabb, min_near, perturb_noise, pdf_u, emb, w0, b0, w1, b1, w2, b2)
        ctx.save_for_backward(rays_o, rays_d, zs, emb, w0, b0, w1, b1, w2, b2)
        ctx.net = net
        ctx.mark_non_differentiable(zs, nears, fars)
        return sigma, rgb, zs, nears, fars

    @staticmethod
    def backward(ctx, g_sigma, g_rgb, _gz, _gn, _gf):
        rays_o, rays_d, zs, emb, w0, b0, w1, b1, w2, b2 = ctx.saved_tensors
        g_sigma = torch.zeros_like(zs) if g_sigma is None else g_sigma.contiguous()
        g_rgb = None if g_rgb is None else g_rgb.contiguous()
        grads = _field_backward_at_samples(ctx.net, rays_o, rays_d, zs, g_sigma, g_rgb, emb, w0, b0, w1, b1, w2, b2)
        return (None, None, None, None, None, None, None, *grads)


class _Composite(torch.autograd.Function):
    """renderer_df.py:414-456 (bg_radius == 0): (image [N,3], depth [N], weights_sum [N]) of colours rgb [N,T,3] at depths zs [N,T],
    T = num_steps + upsample_steps"""

    @staticmethod
    def forward(ctx, zs, sigma, rgb, nears, fars, bg_color, num_steps, upsample_steps):
        N = zs.shape[0]
        dev = zs.device
        f = lib.fptr
        sigma, rgb = sigma.contiguous(), rgb.contiguous()
        image, depth, ws = torch.empty(N, 3, device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev)
        lib.call('sfb_ray_composite_forward_steps', f(zs), f(sigma), f(rgb), f(nears), f(fars), float(bg_color), N, num_steps, upsample_steps, f(image),
                 f(depth), f(ws), lib.stream())
        ctx.save_for_backward(zs, sigma, rgb, nears, fars)
        ctx.bg, ctx.steps = float(bg_color), (num_steps, upsample_steps)
        return image, depth, ws

    @staticmethod
    def backward(ctx, g_image, g_depth, g_ws):
        zs, sigma, rgb, nears, fars = ctx.saved_tensors
        g_sigma, g_rgb = _composite_backward(zs, sigma, rgb, nears, fars, ctx.bg, g_image, g_depth, g_ws, *ctx.steps)
        return None, g_sigma, g_rgb, None, None, None, None, None


def _safe_normalize(x, eps=1e-20):
    """external/nerf/utils.py:41-42"""
    return x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps))


class NeRFRenderer(nn.Module):
    MAX_RAYS_PER_LAUNCH = 65536      # rays per fused-render autograd node at 128 samples per ray (x 1.4 KB of backward tape = 12 GB transient)
    MAX_SAMPLES_PER_RAY = 256        # num_steps + upsample_steps: the fused kernels index a ray's sorted samples with a uint8

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.bound = opt.bound
        self.cascade = 1 + math.ceil(math.log2(opt.bound))
        self.grid_size = 128
        self.cuda_ray = opt.cuda_ray
        self.min_near = opt.min_near
        self.density_thresh = opt.density_thresh
        self.bg_radius = opt.bg_radius
        aabb_train = torch.FloatTensor([-opt.bound, -opt.bound, -opt.bound, opt.bound, opt.bound, opt.bound])
        self.register_buffer('aabb_train', aabb_train)
        self.register_buffer('aabb_infer', aabb_train.clone())
        if self.cuda_ray:
            self.register_buffer('density_grid', torch.zeros([self.cascade, self.grid_size ** 3]))
            self.register_buffer('density_bitfield', torch.zeros(self.cascade * self.grid_size ** 3 // 8, dtype=torch.uint8))
            self.mean_density = 0
            self.iter_density = 0
            self.register_buffer('step_counter', torch.zeros(16, 2, dtype=torch.int32))
            self.mean_count = 0
            self.local_step = 0

    def forward(self, x, d):
        raise NotImplementedError()

    def density(self, x):
        raise NotImplementedError()

    def reset_extra_state(self):
        if not self.cuda_ray:
            return
        self.density_grid.zero_()
        self.mean_density = 0
        self.iter_density = 0
        self.step_counter.zero_()
        self.mean_count = 0
        self.local_step = 0

    @torch.no_grad()
    def export_mesh(self, path, resolution=None, S=128, *, grid_resolution=128, texture_size=None):
        """renderer_df.py:121-153 on the GPU: sigma on the lattice linspace(-bound, bound, R)^3 (indexing 'ij', queried in slabs of S
        x-planes), Gaussian smoothing with sigma = 1.5 voxels, marching cubes at mean + 0.25 std of the smoothed volume, and
        ``{path}/mcubes_mesh.obj`` with vertices in lattice index units, as the reference writes it.  ``resolution`` is accepted and
        ignored (the reference overrides it with 128); ``grid_resolution`` sets R (128 = the reference's lattice).
        ``texture_size=T`` (16..8192) also writes ``{path}/mesh.obj`` (world-unit vertices with per-corner UVs), ``mesh.mtl`` and a T x T
        ``albedo.png``: the field's albedo at the surface point under every texel of a per-triangle atlas (mesh.bake_albedo).  A T outside
        16..8192 raises ValueError before anything is written; one too small for the mesh's triangle count raises it after mcubes_mesh.obj.
        Returns (verts [V,3] float32 in world units, v / (R-1) * 2 bound - bound; tris [F,3] int32) on the parameters' device.
        Works with either cuda_ray setting: it reads neither mean_density nor the density bitfield."""
        import os
        from . import mesh
        R = int(grid_resolution)
        if texture_size is not None:
            mesh._atlas_cell(0, texture_size)
        sigma = mesh.density_lattice(self, R, S)
        smooth = mesh.smooth_gaussian(sigma, 1.5)
        mean, std = mesh.volume_mean_std(smooth)
        verts, tris = mesh.marching_cubes(smooth, mean + 0.25 * std)
        mesh.write_obj(os.path.join(path, 'mcubes_mesh.obj'), verts, tris)
        verts_world = verts / (R - 1) * (2 * self.bound) - self.bound
        if texture_size is not None:
            uv, texture, _ = mesh.bake_albedo(self, verts_world, tris, texture_size)
            mesh.write_textured_obj(path, verts_world, tris, uv, texture)
        return verts_world, tris

    # ------------------------------------------------------------------------------------------ default path
    def run(self, rays_o, rays_d, num_steps=128, upsample_steps=128, light_d=None, ambient_ratio=1.0, shading='albedo', bg_color=None,
            perturb=False, fixed_light=False, perturb_noise=None, pdf_noise=None, normal_noise=None, regularisers=True, **kwargs):
        """rays_o, rays_d: [B, N, 3] (B == 1) -> image [B,N,3], depth [B,N], weights_sum [N], mask [B,N], and with a shading other than
        'albedo' loss_orient and loss_smooth (:427-436).  ``perturb_noise`` [N,num_steps] / ``pdf_noise`` [N,upsample_steps] /
        ``normal_noise`` [N,128,3] override the torch.rand / torch.randn draws (parity tests).  ``regularisers=False`` skips loss_orient and
        loss_smooth (and the randn of :434 with them): ``render(staged=True)`` passes it, since the reference discards them there.
        'albedo' takes num_steps >= 1 and upsample_steps >= 0 with num_steps + upsample_steps <= 256 (num_steps >= 2 when upsample_steps > 0:
        at 1 the reference itself fails); upsample_steps = 0 composites the coarse samples alone.  The other shadings take 64 + 64."""
        if self.bg_radius > 0:
            raise NotImplementedError("the fused renderer covers SparseFusion's configuration: bg_radius=0 (sparsefusion/distillation.py:512)")
        if shading != 'albedo' and (num_steps != 64 or upsample_steps != 64):
            raise NotImplementedError(f"shading={shading!r} renders at num_steps = upsample_steps = 64 (get_default_torch_ngp_opt); 'albedo' takes other counts")
        if num_steps < 1 or upsample_steps < 0 or (num_steps == 1 and upsample_steps > 0):
            raise ValueError(f'num_steps = {num_steps}, upsample_steps = {upsample_steps}: needs num_steps >= 1, upsample_steps >= 0, and num_steps >= 2 '
                             'when upsample_steps > 0 (the importance pdf is over the coarse bins)')
        if num_steps + upsample_steps > self.MAX_SAMPLES_PER_RAY:
            raise NotImplementedError(f'num_steps + upsample_steps = {num_steps + upsample_steps}: the fused renderer takes at most '
                                      f'{self.MAX_SAMPLES_PER_RAY} samples per ray')
        prefix = rays_o.shape[:-1]
        rays_o = rays_o.contiguous().view(-1, 3).float()
        rays_d = rays_d.contiguous().view(-1, 3).float()
        if not rays_o.is_cuda:
            raise RuntimeError('NeRFRenderer.run needs CUDA tensors (the reference has no CPU path either)')
        N = rays_o.shape[0]
        dev = rays_o.device
        aabb = self.aabb_train if self.training else self.aabb_infer
        if bg_color is None:
            bg_color = 1
        if not isinstance(bg_color, (int, float)):
            raise NotImplementedError('per-ray bg_color tensors are not used by the distillation loop (bg_color=0)')
        with torch.cuda.device(dev):
            if shading != 'albedo' and light_d is None:                                         # :333-352, drawn first as there
                if fixed_light:
                    rot_m = torch.tensor([[0.63, .65, -0.43], [-.43, .75, -0.5], [-.65, .13, .75]], device=dev, dtype=torch.float)
                    light_d = _safe_normalize(rays_o[0] @ rot_m)
                else:
                    light_d = _safe_normalize(rays_o[0] + torch.randn(3, device=dev, dtype=torch.float))
            if perturb and perturb_noise is None:
                perturb_noise = torch.rand(N, num_steps, device=dev)                          # renderer_df.py:363
            if not perturb:
                perturb_noise = None
            if upsample_steps == 0:                                                            # no sample_pdf, no draw (:372)
                pdf_u = None
            elif self.training:
                pdf_u = pdf_noise if pdf_noise is not None else torch.rand(N, upsample_steps, device=dev)   # renderer_df.py:31
            else:                                                                              # det = not self.training (:392)
                pdf_u = torch.linspace(0. + 0.5 / upsample_steps, 1. - 0.5 / upsample_steps, steps=upsample_steps, device=dev).expand(N, upsample_steps)
            pdf_u = None if pdf_u is None else pdf_u.contiguous()
            p = self._field_params()
            pn = None if perturb_noise is None else perturb_noise.contiguous()
            if shading != 'albedo':
                return self._run_shaded(rays_o, rays_d, prefix, aabb, bg_color, pn, pdf_u, light_d, ambient_ratio, shading, normal_noise,
                                        regularisers)
            # large images (512x512 rays and up at 128 samples): the backward's activation tapes are 1.4 KB per sample point, so rays go through
            # the fused kernels in slices of a fixed sample count -- each slice is its own autograd node, whose tape exists only while that slice
            # back-propagates
            M = self.MAX_RAYS_PER_LAUNCH * 128 // (num_steps + upsample_steps)
            steps = (num_steps, upsample_steps)
            if N <= M:
                image, depth, ws, nears, fars = _RunRender.apply(self, rays_o, rays_d, aabb, self.min_near, bg_color, *steps, pn, pdf_u, *p)
            else:
                parts = [_RunRender.apply(self, rays_o[i:i + M], rays_d[i:i + M], aabb, self.min_near, bg_color, *steps, None if pn is None else pn[i:i + M],
                                          None if pdf_u is None else pdf_u[i:i + M], *p)
                         for i in range(0, N, M)]
                image, depth, ws, nears, fars = (torch.cat([q[j] for q in parts]) for j in range(5))
        return {'image': image.view(*prefix, 3), 'depth': depth.view(*prefix), 'weights_sum': ws, 'mask': (nears < fars).reshape(*prefix)}

    def _run_shaded(self, rays_o, rays_d, prefix, aabb, bg_color, pn, pdf_u, light_d, ratio, shading, normal_noise, regularisers):
        """run with a normal-based shading, in slices of MAX_RAYS_PER_LAUNCH rays as the albedo path (each slice its own autograd nodes, so
        the v1 field kernels' backward tape exists for one slice at a time); the regularisers are means over all slices' samples"""
        N = rays_o.shape[0]
        M = self.MAX_RAYS_PER_LAUNCH
        parts = [self._shade_slice(rays_o[i:i + M], rays_d[i:i + M], aabb, bg_color, None if pn is None else pn[i:i + M], pdf_u[i:i + M], light_d,
                                   ratio, shading, None if normal_noise is None else normal_noise[i:i + M], regularisers) for i in range(0, N, M)]
        image, depth, ws, nears, fars = (torch.cat([q[j] for q in parts]) for j in range(5))
        out = {'image': image.view(*prefix, 3), 'depth': depth.view(*prefix), 'weights_sum': ws, 'mask': (nears < fars).reshape(*prefix)}
        if regularisers:
            out['loss_orient'] = sum(q[5] for q in parts) / (N * 128)
            out['loss_smooth'] = sum(q[6] for q in parts) / (N * 128 * 3)
        return out

    def _shade_slice(self, rays_o, rays_d, aabb, bg_color, pn, pdf_u, light_d, ratio, shading, normal_noise, regularisers):
        """one slice of rays: the field at the 128 sorted samples (one autograd node), the normal there (the smoothed stencil for 'textureless'
        / 'normal', the plain one with gradient otherwise), shading (network_grid.py:187-195), compositing, and the sums of the orientation and
        smoothness terms (renderer_df.py:427-436, with the weights of :416-418, detached) -> (image, depth, ws, nears, fars, orient, smooth)"""
        from .network_grid import _NormalFn, shade, stencil_forward, jitter_key
        N = rays_o.shape[0]
        dev = rays_o.device
        p = self._field_params()
        sigma, albedo, zs, nears, fars = _RaySamples.apply(self, rays_o, rays_d, aabb, self.min_near, pn, pdf_u, *p)
        rays = (rays_o, rays_d, zs)
        if shading in ('textureless', 'normal'):
            with torch.no_grad():
                normal = stencil_forward(self, N * 128, rays=rays, k=10, eps=3e-1, radius=3e-1, key=jitter_key(dev), want_fd=False)[1]
        else:
            normal = _NormalFn.apply(self, None, rays, 1e-2, True, *p)
        color, _ = shade(albedo.view(-1, 3), normal, light_d, ratio, shading)
        image, depth, ws = _Composite.apply(zs, sigma, color.view(N, 128, 3), nears, fars, bg_color, 64, 64)
        if not regularisers:
            return image, depth, ws, nears, fars
        with torch.no_grad():
            sample_dist = ((fars - nears) / 64)[:, None]
            deltas = torch.cat([zs[:, 1:] - zs[:, :-1], sample_dist], -1)
            alphas = 1 - torch.exp(-deltas * sigma)
            weights = alphas * torch.cumprod(torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], -1), -1)[:, :-1]
            xyzs = torch.min(torch.max(rays_o[:, None, :] + rays_d[:, None, :] * zs[..., None], aabb[:3]), aabb[3:])
            if normal_noise is None:
                normal_noise = torch.randn_like(xyzs)
        normals = normal.view(N, 128, 3)
        dirs = rays_d.view(-1, 1, 3).expand_as(normals)
        orient = (weights * (normals * dirs).sum(-1).clamp(min=0) ** 2).sum()
        normals_perturb = self.normal(xyzs + normal_noise.to(dev) * 1e-2).view(N, 128, 3)
        smooth = (normals - normals_perturb).abs().sum()
        return image, depth, ws, nears, fars, orient, smooth

    # ------------------------------------------------------------------------------------------ cuda_ray path
    def run_cuda(self, rays_o, rays_d, dt_gamma=0, light_d=None, ambient_ratio=1.0, shading='albedo', bg_color=None, perturb=False,
                 force_all_rays=False, max_steps=1024, T_thresh=1e-4, **kwargs):
        prefix = rays_o.shape[:-1]
        rays_o = rays_o.contiguous().view(-1, 3)
        rays_d = rays_d.contiguous().view(-1, 3)
        N = rays_o.shape[0]
        device = rays_o.device
        # NB: like the reference (renderer_df.py:483) min_near is NOT forwarded here -> the wrapper default 0.2
        nears, fars = raymarching.near_far_from_aabb(rays_o, rays_d, self.aabb_train if self.training else self.aabb_infer)
        if shading != 'albedo' and light_d is None:       # :486-489
            light_d = _safe_normalize(rays_o[0] + torch.randn(3, device=device, dtype=torch.float))
        results = {}
        if self.training:
            counter = self.step_counter[self.local_step % 16]
            counter.zero_()
            self.local_step += 1
            xyzs, dirs, deltas, rays = raymarching.march_rays_train(rays_o, rays_d, self.bound, self.density_bitfield, self.cascade, self.grid_size,
                                                                    nears, fars, counter, self.mean_count, perturb, 128, force_all_rays, dt_gamma,
                                                                    max_steps)
            sigmas, rgbs, normals = self(xyzs, dirs, light_d, ratio=ambient_ratio, shading=shading)
            weights_sum, depth, image = raymarching.composite_rays_train(sigmas, rgbs, deltas, rays, T_thresh)
            if normals is not None:                       # :509-519, with the weights 1 - exp(-sigma) used there
                weights = 1 - torch.exp(-sigmas)
                results['loss_orient'] = (weights.detach() * (normals * dirs).sum(-1).clamp(min=0) ** 2).mean()
                normals_perturb = self.normal(xyzs + torch.randn_like(xyzs) * 1e-2)
                results['loss_smooth'] = (normals - normals_perturb).abs().mean()
        else:
            weights_sum = torch.zeros(N, dtype=torch.float32, device=device)
            depth = torch.zeros(N, dtype=torch.float32, device=device)
            image = torch.zeros(N, 3, dtype=torch.float32, device=device)
            n_alive = N
            rays_alive = torch.arange(n_alive, dtype=torch.int32, device=device)
            rays_t = nears.clone()
            step = 0
            while step < max_steps:
                n_alive = rays_alive.shape[0]
                if n_alive <= 0:
                    break
                n_step = max(min(N // n_alive, 8), 1)
                xyzs, dirs, deltas = raymarching.march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, self.bound, self.density_bitfield,
                                                            self.cascade, self.grid_size, nears, fars, 128, perturb if step == 0 else False,
                                                            dt_gamma, max_steps)
                sigmas, rgbs, _ = self(xyzs, dirs, light_d, ratio=ambient_ratio, shading=shading)
                raymarching.composite_rays(n_alive, n_step, rays_alive, rays_t, sigmas, rgbs, deltas, weights_sum, depth, image, T_thresh)
                rays_alive = rays_alive[rays_alive >= 0]
                step += n_step
        if self.bg_radius > 0:
            raise NotImplementedError('bg_radius > 0 is not used by SparseFusion (distillation.py:512)')
        if bg_color is None:
            bg_color = 1
        image = image + (1 - weights_sum).unsqueeze(-1) * bg_color
        image = image.view(*prefix, 3)
        depth = torch.clamp(depth - nears, min=0) / (fars - nears)
        results['image'] = image
        results['depth'] = depth.view(*prefix)
        results['weights_sum'] = weights_sum.reshape(*prefix)
        results['mask'] = (nears < fars).reshape(*prefix)
        return results

    @torch.no_grad()
    def update_extra_state(self, decay=0.95, S=128, jitter=None):
        """renderer_df.py:587-640: refresh the cascaded density grid (EMA max) and its bitfield.  ``jitter``
        [cascade, G^3, 3] in U(0,1) overrides torch.rand_like (parity tests)."""
        if not self.cuda_ray:
            return
        G = self.grid_size
        dev = self.density_bitfield.device
        tmp_grid = -torch.ones_like(self.density_grid)
        ar = torch.arange(G, dtype=torch.int32, device=dev)
        xx, yy, zz = torch.meshgrid(ar, ar, ar, indexing='ij')
        coords = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], dim=-1)
        indices = raymarching.morton3D(coords).long()
        xyzs = 2 * coords.float() / (G - 1) - 1
        for cas in range(self.cascade):
            bound = min(2 ** cas, self.bound)
            half_grid_size = bound / G
            cas_xyzs = xyzs * (bound - half_grid_size)
            noise = torch.rand_like(cas_xyzs) if jitter is None else jitter[cas].to(dev)
            cas_xyzs = cas_xyzs + (noise * 2 - 1) * half_grid_size
            sigmas = self.density(cas_xyzs)['sigma'].reshape(-1).detach()
            tmp_grid[cas, indices] = sigmas
        valid_mask = self.density_grid >= 0
        self.density_grid[valid_mask] = torch.maximum(self.density_grid[valid_mask] * decay, tmp_grid[valid_mask])
        self.mean_density = torch.mean(self.density_grid[valid_mask]).item()
        self.iter_density += 1
        density_thresh = min(self.mean_density, self.density_thresh)
        self.density_bitfield = raymarching.packbits(self.density_grid, density_thresh, self.density_bitfield)
        total_step = min(16, self.local_step)
        if total_step > 0:
            self.mean_count = int(self.step_counter[:total_step, 0].sum().item() / total_step)
        self.local_step = 0

    # ------------------------------------------------------------------------------------------ dispatch
    def render(self, rays_o, rays_d, staged=False, max_ray_batch=4096, **kwargs):
        _run = self.run_cuda if self.cuda_ray else self.run
        B, N = rays_o.shape[:2]
        device = rays_o.device
        if staged and not self.cuda_ray:
            depth = torch.empty((B, N), device=device)
            image = torch.empty((B, N, 3), device=device)
            weights_sum = torch.empty((B, N), device=device)
            for b in range(B):
                head = 0
                while head < N:
                    tail = min(head + max_ray_batch, N)
                    # only three keys survive here (as in the reference), so the shaded path's regularisers are not computed
                    r = _run(rays_o[b:b + 1, head:tail], rays_d[b:b + 1, head:tail], regularisers=False, **kwargs)
                    depth[b:b + 1, head:tail] = r['depth']
                    weights_sum[b:b + 1, head:tail] = r['weights_sum']
                    image[b:b + 1, head:tail] = r['image']
                    head += max_ray_batch
            return {'depth': depth, 'image': image, 'weights_sum': weights_sum}
        return _run(rays_o, rays_d, **kwargs)

    def render_batched(self, rays_o, rays_d, batched=False, max_ray_batch=128 * 128, **kwargs):
        with torch.no_grad():
            return self.render(rays_o, rays_d, staged=batched, max_ray_batch=max_ray_batch, **kwargs)
