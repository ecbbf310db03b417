"""The fused NGP field (csrc/ngp_field.cu) and the per-ray stages (csrc/ngp_render.cu) element by element against fp64 references
(oracle/field_fp64.py), on all three field kernel paths.

Tolerances are per element, |got - ref| <= rtol * ref_abs + slack + atol, where ref_abs is the reference computed on |weights| and
|terms|.  rtol is gamma(n) = n u / (1 - n u) (u = 2^-24) for the longest chain of n fp32 roundings the kernel performs to reach that
element (Higham, Accuracy and Stability of Numerical Algorithms, sec. 3.1):
  * per point (sigma, rgb, and the per-point part of every gradient): 320 roundings, field_fp64.RTOL_POINT (the count is itemised there);
  * weight / bias gradients: plus the reduction over the points, whose length depends on the path and on B (field_fp64.wgrad_rtol);
  * embedding rows: plus the number of (point, corner) scatters into that row, counted by the reference;
  * compositing: 12 roundings per sample over 128 samples of the ray scale (field_fp64.RTOL_COMP).
Upstream gradients are one-signed (field_fp64.upstream_grads) so that the sums over points do not cancel.  The host tests
(test_ngp_field_fp64_host.py) show, tensor by tensor and for each path's bounds, what a single defect the comparison sees: a lost
64-point tile in every weight and bias gradient (B = 20 000); a lost point in every weight and bias gradient at B = 1 000, and at
B = 20 000 in the embedding gradient only (one point is 5e-5 of a 20 000-point sum, below the summation bounds there); a lost level of
one point, and a flipped ReLU mask, in the tensors they reach.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import field_fp64 as f64
from oracle import ngp_oracle as no

pytestmark = pytest.mark.gpu

BOUND = 4.0
FLT_MAX = float(np.finfo(np.float32).max)


def _lib():
    from sparsefusion_b200 import _lib as lib
    return lib


def _sm_count():
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib().call('sfb_device_info', ctypes.addressof(sm), ctypes.addressof(major), ctypes.addressof(minor))
    return sm.value


@pytest.fixture(params=[(0x7fffffff, 'v2'), (0x7fffffff & ~16, 'v1-tc'), (0, 'v1-simt')],
                ids=['field-v2-tiled', 'field-v1-wgrad-tcgen05', 'field-v1-wgrad-simt'])
def field_path(request):
    """the three implementations of the field kernels (sfb_set_fusion bit 4: v2 tiles; bit 0: v1 weight gradients as wgmma GEMMs)"""
    mask, name = request.param
    lib = _lib()
    lib.call('sfb_set_fusion', mask)
    try:
        yield name
    finally:
        lib.call('sfb_set_fusion', 0x7fffffff)


_GEO = no.live_geometry(BOUND)
_SCALES = {}


def _scales():
    if 'd' not in _SCALES:
        from _helpers import device_level_scales
        _SCALES['d'] = device_level_scales(_GEO)
    return _SCALES['d']


# ------------------------------------------------------------------------------------------------ kernel calls
def _field(p, B, xyz=None, rays=None, g_sigma=None, g_rgb=None, prefill=None, want_rgb=True, backward=True):
    """forward (sigma, rgb) and, with g_sigma, backward through the C ABI; gradients accumulate into `prefill` (or zeros)"""
    lib = _lib()
    f = lib.fptr
    q = {k: v.detach().float().cuda().contiguous() for k, v in p.items()}
    offsets = torch.from_numpy(_GEO['offsets']).cuda()
    src = (f(xyz), None, None, None, 0) if xyz is not None else (None, f(rays[0]), f(rays[1]), f(rays[2]), rays[2].shape[1])
    W = [f(q[k]) for k in no.PARAM_KEYS[1:]]
    sigma = torch.full((B,), -7.0, device='cuda')
    rgb = torch.full((B, 3), -7.0, device='cuda') if want_rgb else None
    lib.call('sfb_ngp_field_forward', *src, B, f(q['encoder.embeddings']), lib.iptr(offsets), float(_GEO['S']), 16, BOUND, *W,
             f(sigma), f(rgb) if rgb is not None else None, lib.stream())
    out = dict(sigma=sigma, rgb=rgb)
    if g_sigma is None:
        return out
    grads = {k: (prefill[k].clone() if prefill is not None else torch.zeros_like(q[k])) for k in no.PARAM_KEYS}
    tape = torch.empty(max(int(lib.load().sfb_ngp_field_tape_floats(B)), 1), device='cuda')
    # device copies held in locals: a temporary's memory returns to the caching allocator as soon as its pointer is taken
    gs_d = g_sigma.cuda().contiguous()
    gc_d = g_rgb.cuda().contiguous() if g_rgb is not None else None
    lib.call('sfb_ngp_field_backward', *src, B, f(q['encoder.embeddings']), lib.iptr(offsets), float(_GEO['S']), 16, BOUND, *W,
             f(gs_d), f(gc_d) if gc_d is not None else None, *[f(grads[k]) for k in no.PARAM_KEYS], f(tape), lib.stream())
    out.update(grads)
    return out


def _check_field(got, ref, fwd, bwd, path, B, prefill=None, fwd_rows=None):
    """every gradient in full; the forward on `fwd_rows` (all rows by default)"""
    sel = slice(None) if fwd_rows is None else fwd_rows
    f64.assert_within('sigma', got['sigma'][sel], fwd['sigma'][sel], fwd['sigma_abs'][sel], f64.RTOL_POINT)
    if got['rgb'] is not None:
        f64.assert_within('rgb', got['rgb'][sel], fwd['rgb'][sel], fwd['rgb_abs'][sel], f64.RTOL_POINT)
    if bwd is None:
        return
    sm = _sm_count()
    extra = 0.0 if prefill is None else f64.gamma(1)          # one more rounding: the pre-filled value plus the fresh sum
    for k in no.PARAM_KEYS:
        want, want_abs = bwd[k], bwd[k + '_abs']
        if prefill is not None:
            pf = prefill[k].to(want.device).double()
            want, want_abs = want + pf, want_abs + pf.abs()
        if k == 'encoder.embeddings':
            rtol = f64.RTOL_POINT + f64.gamma(bwd[k + '_hits'] + 1) + extra
        else:
            rtol = f64.wgrad_rtol(path, B, sm) + extra
        f64.assert_within(f'{path} B={B} {k}', got[k], want, want_abs, rtol, bwd[k + '_slack'])


# ------------------------------------------------------------------------------------------------ cases
def _points(B, seed):
    """explicit points: uniform in [-1.1, 1.1] * bound (so some lie outside the box), the blob centre, points exactly on +-bound"""
    rng = np.random.default_rng(seed)
    x = ((rng.random((B, 3), dtype=np.float32) * 2 - 1) * 1.1 * BOUND).astype(np.float32)
    special = np.array([[0, 0, 0], [BOUND, BOUND, BOUND], [-BOUND, -BOUND, -BOUND], [BOUND, 0.3, -BOUND], [0.01, -0.02, 0.015],
                        [np.nextafter(np.float32(BOUND), np.float32(5)), 0, 0]], np.float32)
    n = min(B, len(special))
    x[:n] = special[:n]
    return torch.from_numpy(x)


_REFS = {}


def _reference(key, params, x, seed, scale_sigma=True, g_rgb=True):
    """fp64 reference of one case, shared by the three paths"""
    if key not in _REFS:
        ref = f64.FieldFP64(params, x.cuda(), _scales(), BOUND)
        fwd = ref.forward()
        gs, gc = f64.upstream_grads(x.shape[0], fwd['sigma'], seed, scale_sigma)
        if not g_rgb:
            gc = None
        if key == 'full' or 'full' in _REFS:     # the full-size case is ~10 GB of fp64: never resident next to another one
            _REFS.clear()
        _REFS[key] = (ref, fwd, gs, gc, ref.backward(gs, gc))
    return _REFS[key]


def _sizes():
    return [1, 63, 64, 65, 127, 128, 129, 1000, 20000, 'wrap-fwd', 'wrap-bwd']


def _resolve(B):
    sm = _sm_count()
    # v1 forward launches 3 SM CTAs of 128 points, the v2 kernels 2 SM CTAs of 128 (forward) / 64 (backward) points: one more point
    # than either cap makes every path's grid-stride loop wrap
    return {'wrap-fwd': 3 * sm * 128 + 1, 'wrap-bwd': 2 * sm * 64 + 1}.get(B, B)


@pytest.mark.parametrize('size', _sizes())
def test_field_explicit_points(field_path, size):
    B = _resolve(size)
    p = no.make_field_params(seed=0)
    x = _points(B, seed=B)
    ref, fwd, gs, gc, bwd = _reference(('explicit', B), p, x, seed=B + 1)
    got = _field(p, B, xyz=x.cuda(), g_sigma=gs, g_rgb=gc)
    _check_field(got, ref, fwd, bwd, field_path, B)


def _rays(N, T, seed):
    """rays from outside the box towards it, with depths that run past the far side of the box (the clamp applies)"""
    rng = np.random.default_rng(seed)
    cams = no.circle_cameras(16)
    o = np.stack([cams[i % 16][0] for i in range(N)]).astype(np.float32)
    d = (-o / np.linalg.norm(o, axis=1, keepdims=True) + (rng.random((N, 3), dtype=np.float32) - 0.5) * 0.6).astype(np.float32)
    z = np.sort(rng.random((N, T), dtype=np.float32) * 12.0 + 0.2, axis=1).astype(np.float32)
    return torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(z)


@pytest.mark.parametrize('T', [64, 128])
def test_field_ray_points_and_explicit_equivalence(field_path, T):
    N = 20000 // T + 3
    B = N * T
    o, d, z = _rays(N, T, seed=T)
    x = f64.ray_points(o.cuda(), d.cuda(), z.cuda(), BOUND)
    assert (x.abs() == BOUND).any(dim=1).float().mean() > 0.1, 'depths must push some samples past the box'
    p = no.make_field_params(seed=1)
    ref, fwd, gs, gc, bwd = _reference(('rays', T), p, x, seed=T + 1)
    rays = (o.cuda(), d.cuda(), z.cuda().contiguous())
    got = _field(p, B, rays=rays, g_sigma=gs, g_rgb=gc)
    _check_field(got, ref, fwd, bwd, field_path, B)
    # the explicit source fed the fp32-rounded, clamped points gives the same bits
    ex = _field(p, B, xyz=x.contiguous())
    assert torch.equal(ex['sigma'], got['sigma']) and torch.equal(ex['rgb'], got['rgb'])


def test_field_full_size_render(field_path):
    """one 128x128 render: 16 384 rays x 128 samples = 2^21 points; the forward on every 61st point, every gradient in full"""
    N, T = 128 * 128, 128
    ro, rd = no.camera_rays(no.circle_cameras(8)[3], 128, 128)
    rng = np.random.default_rng(21)
    z = np.sort(rng.random((N, T), dtype=np.float32) * 10.0 + 0.5, axis=1).astype(np.float32)
    o, d, z = torch.from_numpy(ro).cuda(), torch.from_numpy(rd).cuda(), torch.from_numpy(z).cuda()
    x = f64.ray_points(o, d, z, BOUND)
    p = no.make_field_params(seed=0)
    ref, fwd, gs, gc, bwd = _reference('full', p, x, seed=22)
    got = _field(p, N * T, rays=(o, d, z), g_sigma=gs, g_rgb=gc)
    _check_field(got, ref, fwd, bwd, field_path, N * T, fwd_rows=torch.arange(0, N * T, 61, device='cuda'))


def _edge_params():
    """pre-activations of sigma beyond +-15 (trunc_exp's backward clamp), saturated sigmoids, a hidden unit of each layer whose
    pre-activation is exactly 0 for every point (dead; a ReLU' of 1 at 0 would show), one that is always active"""
    p = {k: v.clone() for k, v in no.make_field_params(seed=2).items()}
    p['sigma_net.net.2.weight'][0] *= 40
    p['sigma_net.net.2.weight'][1:] *= 60
    p['sigma_net.net.0.weight'][5] = 0
    p['sigma_net.net.0.bias'][5] = 0
    p['sigma_net.net.1.weight'][9] = 0
    p['sigma_net.net.1.bias'][9] = 0
    p['sigma_net.net.0.weight'][7] *= 0.25
    p['sigma_net.net.0.bias'][7] = 4
    p['sigma_net.net.2.weight'][0] *= 20
    p['sigma_net.net.2.bias'][0] = -121          # centres sigma's pre-activation: about -35 .. 40 over the points
    p['sigma_net.net.2.bias'][3] = 40            # blue saturates at 1, the other channels reach below 1e-6
    return p


def test_field_activation_edges(field_path):
    B = 5000
    p = _edge_params()
    x = _points(B, seed=5)
    ref, fwd, gs, gc, bwd = _reference('edges', p, x, seed=6, scale_sigma=False)
    live = ref.w.sum((1, 2)) > 0
    assert (ref.pre > 15).any() and (ref.pre < -15).any()
    assert not ref.mask1[:, 5].any() and not ref.mask2[:, 9].any() and ref.mask1[live, 7].all()
    assert (fwd['rgb'].float() == 1).any() and (fwd['rgb'] < 1e-6).any()
    got = _field(p, B, xyz=x.cuda(), g_sigma=gs, g_rgb=gc)
    _check_field(got, ref, fwd, bwd, field_path, B)
    assert (got['sigma_net.net.0.weight'][5] == 0).all() and got['sigma_net.net.0.bias'][5] == 0


def test_field_contracts(field_path):
    """gradients accumulate into the buffers; grad_rgb may be NULL; rgb may be NULL; B = 0 touches nothing; the forward is deterministic"""
    B = 20000
    p = no.make_field_params(seed=0)
    x = _points(B, seed=B)
    ref, fwd, gs, gc, bwd = _reference(('explicit', B), p, x, seed=B + 1)
    g = torch.Generator().manual_seed(4)
    prefill = {k: torch.randn(v.shape, generator=g).cuda() * 0.01 for k, v in p.items()}
    got = _field(p, B, xyz=x.cuda(), g_sigma=gs, g_rgb=gc, prefill=prefill)
    _check_field(got, ref, fwd, bwd, field_path, B, prefill=prefill)
    again = _field(p, B, xyz=x.cuda())
    assert torch.equal(again['sigma'], got['sigma']) and torch.equal(again['rgb'], got['rgb'])
    no_rgb = _field(p, B, xyz=x.cuda(), want_rgb=False)
    assert torch.equal(no_rgb['sigma'], got['sigma'])
    # grad_rgb = NULL is the backward with a zero colour gradient
    ref0, fwd0, gs0, _, bwd0 = _reference(('no-rgb-grad', B), p, x, seed=B + 1, g_rgb=False)
    got0 = _field(p, B, xyz=x.cuda(), g_sigma=gs0, g_rgb=None)
    _check_field(got0, ref0, fwd0, bwd0, field_path, B)
    # B = 0: a no-op on every output buffer
    lib, f = _lib(), _lib().fptr
    q = {k: v.cuda() for k, v in p.items()}
    offsets = torch.from_numpy(_GEO['offsets']).cuda()
    sentinel = torch.full((4,), 3.0, device='cuda')
    sg = {k: torch.full_like(q[k], 3.0) for k in no.PARAM_KEYS}
    W = [f(q[k]) for k in no.PARAM_KEYS[1:]]
    xs = torch.zeros(4, 3, device='cuda')
    lib.call('sfb_ngp_field_forward', f(xs), None, None, None, 0, 0, f(q['encoder.embeddings']), lib.iptr(offsets), float(_GEO['S']), 16, BOUND,
             *W, f(sentinel), None, lib.stream())
    lib.call('sfb_ngp_field_backward', f(xs), None, None, None, 0, 0, f(q['encoder.embeddings']), lib.iptr(offsets), float(_GEO['S']), 16, BOUND,
             *W, f(sentinel), None, *[f(sg[k]) for k in no.PARAM_KEYS], f(sentinel), lib.stream())
    torch.cuda.synchronize()
    assert (sentinel == 3).all() and all((v == 3).all() for v in sg.values())


# ------------------------------------------------------------------------------------------------ compositing
def _composite_inputs(N, seed):
    """[N,128] sorted depths, densities, colours; ray n is of kind n % 5 (N = 1 gets the saturated kind):
    0 ordinary, 1 saturated samples (alpha == 1 in fp32: the 1e-15 of the transmittance), 2 zero-length deltas, 3 fully transparent,
    4 missed (near = far = z = FLT_MAX)"""
    g = torch.Generator().manual_seed(seed)
    nears = 0.5 + torch.rand(N, generator=g) * 1.5
    fars = nears + 1 + torch.rand(N, generator=g) * 5
    z = nears[:, None] + (fars - nears)[:, None] * torch.sort(torch.rand(N, 128, generator=g), dim=1).values
    sig = torch.rand(N, 128, generator=g) * torch.rand(N, 1, generator=g) * 4
    rgb = torch.rand(N, 128, 3, generator=g)
    kind = torch.arange(N) % 5 if N > 1 else torch.ones(1, dtype=torch.long)
    for n in range(N):
        k = int(kind[n])
        if k == 1:
            sig[n, 40] = 1e4
            sig[n, 90:92] = 1e5
        elif k == 2:
            z[n, 10:20] = z[n, 10]
            z[n, 127] = z[n, 126]
        elif k == 3:
            sig[n] = 0
        elif k == 4:
            nears[n] = fars[n] = FLT_MAX
            z[n] = FLT_MAX
    return z.float(), sig.float(), rgb.float(), nears.float(), fars.float(), kind


@pytest.mark.parametrize('N', [1, 3, 5, 4097])
@pytest.mark.parametrize('bg', [0.0, 1.0, 0.3])
@pytest.mark.parametrize('grads', ['ws+depth', 'ws', 'depth', 'image-only'])
def test_composite_forward_backward(N, bg, grads):
    """sfb_ray_composite_forward / _backward against fp64 autograd of renderer_df.py:414-456 (the tail of ngp_oracle.run).
    Missed rays (near = far = FLT_MAX, `mask` false for them): torch's normalised depth is 0/0 = NaN there, and so is the depth
    gradient it back-propagates; the kernel gives depth 0 and zero gradients -- pinned here, the one deviation from the reference."""
    lib = _lib()
    f = lib.fptr
    z, sig, rgb, nears, fars, kind = _composite_inputs(N, seed=N)
    g = torch.Generator().manual_seed(N + 7)
    gi = torch.randn(N, 3, generator=g)
    gws = torch.randn(N, generator=g) if 'ws' in grads else None
    gdp = torch.randn(N, generator=g) if 'depth' in grads else None
    # device copies held in locals: a temporary's memory returns to the caching allocator as soon as its pointer is taken
    zd, sd, cd, nd, fd, gid = (t.cuda().contiguous() for t in (z, sig, rgb, nears, fars, gi))
    gwsd = gws.cuda() if gws is not None else None
    gdpd = gdp.cuda() if gdp is not None else None
    image, depth, ws = torch.empty(N, 3, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
    lib.call('sfb_ray_composite_forward', f(zd), f(sd), f(cd), f(nd), f(fd), bg, N, 128, f(image), f(depth), f(ws), lib.stream())
    gsig, grgb = torch.empty(N, 128, device='cuda'), torch.empty(N, 128, 3, device='cuda')
    lib.call('sfb_ray_composite_backward', f(zd), f(sd), f(cd), f(nd), f(fd), bg, N, 128, f(gid), f(gwsd) if gwsd is not None else None,
             f(gdpd) if gdpd is not None else None, f(gsig), f(grgb), lib.stream())
    r = f64.composite(z, sig, rgb, nears, fars, bg, gi, gws, gdp)
    hit = kind != 4
    R = f64.RTOL_COMP
    f64.assert_within('weights_sum', ws.cpu(), r['weights_sum'], r['weights_sum_abs'], R)
    f64.assert_within('image', image.cpu(), r['image'], r['image_abs'], R)
    f64.assert_within('depth', depth.cpu()[hit], r['depth'][hit], r['depth_abs'][hit], R)
    f64.assert_within('g_sigma', gsig.cpu()[hit], r['g_sigma'][hit], r['g_sigma_abs'][hit], R)
    f64.assert_within('g_rgb', grgb.cpu()[hit], r['g_rgb'][hit], r['g_rgb_abs'][hit], R)
    miss = ~hit
    if miss.any():
        assert (depth.cpu()[miss] == 0).all() and (ws.cpu()[miss] == 0).all() and (image.cpu()[miss] == bg).all()
        assert (gsig.cpu()[miss] == 0).all() and (grgb.cpu()[miss] == 0).all()
    if (kind == 1).any():
        sat = kind == 1
        assert (ws.cpu()[sat] > 0.999).all()


# ------------------------------------------------------------------------------------------------ resampling
def test_resample_and_gather():
    """sfb_ray_resample_ex: src_of is a permutation of the 128 slots, z_sorted[slot] is the depth it names, sorted with ties coarse
    first (then by index), z_new is fp64 sample_pdf wherever the sample's bin is above the pdf's 1e-5 floor (see below); and
    sfb_ray_gather_sorted is an exact gather"""
    lib = _lib()
    f = lib.fptr
    N = 4097
    g = torch.Generator().manual_seed(9)
    nears = 0.5 + torch.rand(N, generator=g)
    fars = nears + 2 + torch.rand(N, generator=g) * 4
    lin = torch.linspace(0, 1, 64)
    zc = nears[:, None] + (fars - nears)[:, None] * lin + (torch.rand(N, 64, generator=g) - 0.5) * ((fars - nears) / 64)[:, None]
    zc[::7, 20:24] = zc[::7, 20:21]                          # equal coarse depths: ties among coarse samples and with new ones
    zc = torch.sort(zc, dim=1).values.float()
    sig = (torch.rand(N, 64, generator=g) * 30 * (torch.rand(N, 1, generator=g) > 0.1)).float()
    for det in (0, 1):
        u = torch.rand(N, 64, generator=g).float()
        u[::11, :4] = 0.0
        zs, zn = torch.empty(N, 128, device='cuda'), torch.empty(N, 64, device='cuda')
        src = torch.empty(N, 128, dtype=torch.uint8, device='cuda')
        zcd, sigd, nd, fd, ud = (t.cuda().contiguous() for t in (zc, sig, nears, fars, u))
        lib.call('sfb_ray_resample_ex', f(zcd), f(sigd), f(nd), f(fd), f(ud), det, N, 64, 64, f(zs), f(zn), lib.bptr(src), lib.stream())
        zs, zn, src = zs.cpu(), zn.cpu(), src.cpu().long()
        assert torch.equal(torch.sort(src, dim=1).values, torch.arange(128).expand(N, -1))
        both = torch.cat([zc, zn], 1)
        assert torch.equal(torch.gather(both, 1, src), zs)
        assert (zs[:, 1:] >= zs[:, :-1]).all()
        tie = zs[:, 1:] == zs[:, :-1]
        assert tie.any() and (src[:, 1:][tie] > src[:, :-1][tie]).all()
        # fp64 sample_pdf on the same fp32 inputs (renderer_df.py:381-395)
        zc64, s64 = zc.double(), sig.double()
        sd = ((fars - nears) / 64).double()[:, None]
        d = torch.cat([zc64[:, 1:] - zc64[:, :-1], sd], 1)
        a = 1 - torch.exp(-d * s64)
        w = a * torch.cumprod(torch.cat([torch.ones(N, 1, dtype=torch.float64), 1 - a + 1e-15], 1), 1)[:, :-1]
        mid = zc64[:, :-1] + 0.5 * d[:, :-1]
        uu = torch.linspace(0.5 / 64, 1 - 0.5 / 64, 64, dtype=torch.float64).expand(N, 64) if det else u.double()
        ref = no.sample_pdf(mid, w[:, 1:-1], 64, det=False, u=uu)
        wi = w[:, 1:-1] + 1e-5
        cdf = torch.cat([torch.zeros(N, 1, dtype=torch.float64), torch.cumsum(wi / wi.sum(1, keepdim=True), 1)], 1)
        inds = torch.searchsorted(cdf, uu.contiguous(), right=True)
        below, above = (inds - 1).clamp(min=0), inds.clamp(max=62)
        cb, ca = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
        bb, ba = torch.gather(mid, 1, below), torch.gather(mid, 1, above)
        # the kernel's cdf: weights within 10 u per sample of the transmittance scale (see field_fp64.RTOL_COMP) plus the scans and the
        # normalisation, <= 800 roundings of 1; the sample moves by that over the bin's mass, times the bin width
        e_cdf = f64.gamma(800)
        # compared: samples in bins whose weight is above the 1e-5 floor and whose cdf step exceeds the kernel's denom < 1e-5 switch
        # by more than the cdf error (so both sides interpolate in the same branch), away from the bin edges by more than that error
        # (so both pick the same bin); the bound divides by the step, so small steps are compared loosely rather than excluded
        w_bin = torch.gather(w[:, 1:-1], 1, below.clamp(max=61))         # pdf index k spans cdf[k] .. cdf[k + 1]
        ok = (w_bin > 1e-5) & ((ca - cb) > 1e-5 + 2 * e_cdf) & ((uu - cb) > 2 * e_cdf) & ((ca - uu) > 2 * e_cdf)
        bound = (ba - bb).abs() * (2 * e_cdf / (ca - cb) + f64.gamma(4)) + f64.gamma(4) * (bb.abs() + ba.abs())
        assert ok.float().mean() > 0.5
        f64.assert_within(f'z_new det={det}', zn[ok], ref[ok], torch.zeros_like(ref[ok]), 0.0, bound[ok])
    # gather
    sc, sn = torch.rand(N, 64, generator=g).cuda(), torch.rand(N, 64, generator=g).cuda()
    cc, cn = torch.rand(N, 64, 3, generator=g).cuda(), torch.rand(N, 64, 3, generator=g).cuda()
    so, co = torch.empty(N, 128, device='cuda'), torch.empty(N, 128, 3, device='cuda')
    srcd = src.to(torch.uint8).cuda()
    lib.call('sfb_ray_gather_sorted', lib.bptr(srcd), f(sc), f(cc), f(sn), f(cn), N, 128, f(so), f(co), lib.stream())
    idx = src.cuda()
    assert torch.equal(so, torch.gather(torch.cat([sc, sn], 1), 1, idx))
    assert torch.equal(co, torch.gather(torch.cat([cc, cn], 1), 1, idx[..., None].expand(-1, -1, 3)))


# ------------------------------------------------------------------------------------------------ Adam
@pytest.mark.parametrize('n', [1, 3, 4097])
def test_adam_step_vs_fp64_torch_adam(n):
    """sfb_adam_step with grad_scale 0.5 (a 2-rank sum all-reduce) for three steps against fp64 torch.optim.Adam on the fp32-rounded
    hyper-parameters.  Per step the update rounds <= 30 times; bias corrections 1 - beta^k are formed in fp32 from powf, which costs
    u / (1 - beta^k) relatively; the parameter itself is rounded once per step."""
    lib = _lib()
    lr, b1, b2, eps = (float(np.float32(v)) for v in (5e-3, 0.9, 0.999, 1e-8))
    g = torch.Generator().manual_seed(n)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * (10.0 ** (k - 1)) for k in range(3)]
    ref = p0.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps)
    p, m, v = p0.cuda(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    p_abs = p0.double().abs()
    m_abs, v_abs = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    p_rtol_terms = torch.zeros(n, dtype=torch.float64)
    for k, gr in enumerate(grads, start=1):
        gd = gr.cuda()
        lib.call('sfb_adam_step', lib.fptr(p), lib.fptr(gd), lib.fptr(m), lib.fptr(v), n, lr, b1, b2, eps, k, 0.5, lib.stream())
        before = ref.detach().clone()
        ref.grad = gr.double() * 0.5
        opt.step()
        gs = gr.double().abs() * 0.5
        m_abs = b1 * m_abs + (1 - b1) * gs
        v_abs = b2 * v_abs + (1 - b2) * gs * gs
        rel = f64.gamma(30 + 4 * k) + 0.5 * f64.U32 / (1 - b2 ** k) + f64.U32 / (1 - b1 ** k)
        p_rtol_terms += rel * (ref.detach() - before).abs()
        p_abs += (ref.detach() - before).abs()
    st = opt.state[ref]
    torch.cuda.synchronize()
    f64.assert_within('exp_avg', m.cpu(), st['exp_avg'], m_abs, f64.gamma(4 * 3))
    f64.assert_within('exp_avg_sq', v.cpu(), st['exp_avg_sq'], v_abs, f64.gamma(5 * 3))
    f64.assert_within('param', p.cpu(), ref.detach(), p_abs, f64.gamma(3), p_rtol_terms)
