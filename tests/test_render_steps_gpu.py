"""The fused renderer at sample counts other than 64 + 64 (num_steps coarse + upsample_steps importance samples, up to 256 per ray):
the per-ray kernels of csrc/ngp_render.cu element by element against fp64, NeRFNetwork.render against the reference's own render
(ngp_run_steps.npz, tools/gen_run_steps_golden.py) and the oracle, slicing at 256 samples, and the distillation / evaluation entry points
at the new counts.  Tolerances follow test_ngp_field_fp64_gpu.py: compositing within gamma(12 T) of the ray scale, resampling within
the admissible-sample bound of test_resample_and_gather."""
import numpy as np
import pytest
import torch

from oracle import field_fp64 as f64
from oracle import ngp_oracle as no

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
GOLDEN_STEPS = [(128, 128), (32, 32), (48, 16), (100, 28), (64, 0)]


def _lib():
    from sparsefusion_b200 import _lib as lib
    return lib


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _draws(N, num_steps, upsample_steps):
    """the golden's injected torch.rand draws (perturbation, then sample_pdf)"""
    rng = np.random.default_rng(1000 * num_steps + upsample_steps)
    return rng.random((N, num_steps), dtype=np.float32), rng.random((N, upsample_steps), dtype=np.float32)


def _net(seed=0):
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    net = NeRFNetwork(opt)
    p = no.make_field_params(seed=seed)
    sd = net.state_dict()
    sd.update(p)
    net.load_state_dict(sd)
    return net.cuda().train(), p, opt


# ------------------------------------------------------------------------------------------------ compositing
def _composite_inputs(N, T, seed):
    """[N,T] sorted depths, densities, colours; ray n is of kind n % 5 (N = 1 gets the saturated kind): 0 ordinary, 1 saturated samples
    (alpha == 1 in fp32), 2 zero-length deltas, 3 fully transparent, 4 missed (near = far = z = FLT_MAX)"""
    g = torch.Generator().manual_seed(seed)
    nears = 0.5 + torch.rand(N, generator=g) * 1.5
    fars = nears + 1 + torch.rand(N, generator=g) * 5
    z = nears[:, None] + (fars - nears)[:, None] * torch.sort(torch.rand(N, T, generator=g), dim=1).values
    sig = torch.rand(N, T, generator=g) * torch.rand(N, 1, generator=g) * 4
    rgb = torch.rand(N, T, 3, generator=g)
    kind = torch.arange(N) % 5 if N > 1 else torch.ones(1, dtype=torch.long)
    for n in range(N):
        k = int(kind[n])
        if k == 1:
            sig[n, T // 3] = 1e4
            sig[n, (2 * T) // 3:(2 * T) // 3 + 2] = 1e5
        elif k == 2:
            z[n, T // 12:T // 6 + 1] = z[n, T // 12]
            z[n, T - 1] = z[n, max(T - 2, 0)]
        elif k == 3:
            sig[n] = 0
        elif k == 4:
            nears[n] = fars[n] = FLT_MAX
            z[n] = FLT_MAX
    return z.float(), sig.float(), rgb.float(), nears.float(), fars.float(), kind


def _composite_fp64(z, sig, rgb, nears, fars, bg, gi, gws, gdp, num_steps):
    """field_fp64.composite with the last delta (far - near) / num_steps: one more sample, of zero density and colour, at
    z_last + (far - near) / num_steps (in fp64) gives the last real sample that delta and adds nothing to any output or gradient"""
    zz = z.double()
    z_pad = torch.cat([zz, zz[:, -1:] + ((fars.double() - nears.double()) / num_steps)[:, None]], 1)
    r = f64.composite(z_pad, torch.cat([sig, torch.zeros_like(sig[:, :1])], 1), torch.cat([rgb, torch.zeros_like(rgb[:, :1])], 1), nears, fars, bg,
                      gi, gws, gdp)
    for k in ('g_sigma', 'g_sigma_abs', 'g_rgb', 'g_rgb_abs'):
        r[k] = r[k][:, :-1]
    return r


@pytest.mark.parametrize('num_steps, T', [(1, 1), (33, 33), (48, 80), (128, 256), (200, 256)])
@pytest.mark.parametrize('bg', [0.0, 0.3])
def test_composite_steps_forward_backward(num_steps, T, bg):
    lib = _lib()
    f = lib.fptr
    N = 1001
    z, sig, rgb, nears, fars, kind = _composite_inputs(N, T, seed=T + num_steps)
    g = torch.Generator().manual_seed(T + 7)
    gi, gws, gdp = torch.randn(N, 3, generator=g), torch.randn(N, generator=g), torch.randn(N, generator=g)
    zd, sd, cd, nd, fd, gid, gwsd, gdpd = (t.cuda().contiguous() for t in (z, sig, rgb, nears, fars, gi, gws, gdp))
    image, depth, ws = torch.empty(N, 3, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
    lib.call('sfb_ray_composite_forward_steps', f(zd), f(sd), f(cd), f(nd), f(fd), bg, N, num_steps, T - num_steps, f(image), f(depth), f(ws),
             lib.stream())
    gsig, grgb = torch.empty(N, T, device='cuda'), torch.empty(N, T, 3, device='cuda')
    lib.call('sfb_ray_composite_backward_steps', f(zd), f(sd), f(cd), f(nd), f(fd), bg, N, num_steps, T - num_steps, f(gid), f(gwsd), f(gdpd),
             f(gsig), f(grgb), lib.stream())
    r = _composite_fp64(z, sig, rgb, nears, fars, bg, gi, gws, gdp, num_steps)
    hit = kind != 4
    R = f64.gamma(12 * T)
    f64.assert_within('weights_sum', ws.cpu(), r['weights_sum'], r['weights_sum_abs'], R)
    f64.assert_within('image', image.cpu(), r['image'], r['image_abs'], R)
    f64.assert_within('depth', depth.cpu()[hit], r['depth'][hit], r['depth_abs'][hit], R)
    f64.assert_within('g_sigma', gsig.cpu()[hit], r['g_sigma'][hit], r['g_sigma_abs'][hit], R)
    f64.assert_within('g_rgb', grgb.cpu()[hit], r['g_rgb'][hit], r['g_rgb_abs'][hit], R)
    miss = ~hit
    assert (depth.cpu()[miss] == 0).all() and (ws.cpu()[miss] == 0).all() and (image.cpu()[miss] == bg).all()
    assert (gsig.cpu()[miss] == 0).all() and (grgb.cpu()[miss] == 0).all()
    assert (ws.cpu()[kind == 1] > 0.999).all()


# ------------------------------------------------------------------------------------------------ resampling
def _sample_pdf_fp64(zc, sig, nears, fars, u):
    """renderer_df.py:381-395 + sample_pdf in fp64 on the fp32 inputs, with an explicit leading zero in the cdf (so num_steps = 2, no bins,
    puts every sample at z_mid[0]) -> (samples, admissible mask, bound) as in test_resample_and_gather"""
    N, Tc = zc.shape
    zc64, s64 = zc.double(), sig.double()
    sd = ((fars - nears) / Tc).double()[:, None]
    d = torch.cat([zc64[:, 1:] - zc64[:, :-1], sd], 1)
    a = 1 - torch.exp(-d * s64)
    w = a * torch.cumprod(torch.cat([torch.ones(N, 1, dtype=torch.float64), 1 - a + 1e-15], 1), 1)[:, :-1]
    mid = zc64[:, :-1] + 0.5 * d[:, :-1]
    wi = w[:, 1:-1] + 1e-5
    cdf = torch.cat([torch.zeros(N, 1, dtype=torch.float64), torch.cumsum(wi / wi.sum(1, keepdim=True), 1)], 1)
    inds = torch.searchsorted(cdf, u.contiguous(), right=True)
    below, above = (inds - 1).clamp(min=0), inds.clamp(max=Tc - 2)
    cb, ca = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bb, ba = torch.gather(mid, 1, below), torch.gather(mid, 1, above)
    denom = torch.where(ca - cb < 1e-5, torch.ones_like(ca), ca - cb)
    ref = bb + (u - cb) / denom * (ba - bb)
    e_cdf = f64.gamma(800)
    if Tc > 2:
        # a single bin has the exact cdf [0, 1] whatever its weight, so its weight need not be above the floor
        w_bin = torch.gather(w[:, 1:-1], 1, below.clamp(max=Tc - 3)) if Tc > 3 else torch.ones_like(u)
        ok = (w_bin > 1e-5) & ((ca - cb) > 1e-5 + 2 * e_cdf) & ((u - cb) > 2 * e_cdf) & ((ca - u) > 2 * e_cdf)
    else:
        ok = torch.zeros_like(u, dtype=torch.bool)
    bound = (ba - bb).abs() * (2 * e_cdf / (ca - cb).clamp(min=1e-300) + f64.gamma(4)) + f64.gamma(4) * (bb.abs() + ba.abs())
    return ref, ok, bound


@pytest.mark.parametrize('Tc, Tf', [(2, 8), (3, 1), (32, 32), (48, 16), (100, 28), (128, 128), (200, 56)])
def test_resample_and_gather_steps(Tc, Tf):
    lib = _lib()
    f = lib.fptr
    N, T = 4097, Tc + Tf
    g = torch.Generator().manual_seed(Tc * 1000 + Tf)
    nears = 0.5 + torch.rand(N, generator=g)
    fars = nears + 2 + torch.rand(N, generator=g) * 4
    lin = torch.linspace(0, 1, Tc)
    zc = nears[:, None] + (fars - nears)[:, None] * lin + (torch.rand(N, Tc, generator=g) - 0.5) * ((fars - nears) / Tc)[:, None]
    a = Tc // 3
    zc[::7, a:a + 4] = zc[::7, a:a + 1]                      # equal coarse depths: ties among coarse samples and with new ones
    zc = torch.sort(zc, dim=1).values.float()
    sig = (torch.rand(N, Tc, generator=g) * 30 * (torch.rand(N, 1, generator=g) > 0.1)).float()
    for det in (0, 1):
        u = torch.rand(N, Tf, generator=g).float()
        u[::11, :4] = 0.0
        zs, zn = torch.empty(N, T, device='cuda'), torch.empty(N, Tf, device='cuda')
        src = torch.empty(N, T, dtype=torch.uint8, device='cuda')
        zcd, sigd, nd, fd, ud = (t.cuda().contiguous() for t in (zc, sig, nears, fars, u))
        lib.call('sfb_ray_resample_ex', f(zcd), f(sigd), f(nd), f(fd), f(ud), det, N, Tc, Tf, f(zs), f(zn), lib.bptr(src), lib.stream())
        zs, zn, src = zs.cpu(), zn.cpu(), src.cpu().long()
        assert torch.equal(torch.sort(src, dim=1).values, torch.arange(T).expand(N, -1))
        assert torch.equal(torch.gather(torch.cat([zc, zn], 1), 1, src), zs)
        assert (zs[:, 1:] >= zs[:, :-1]).all()
        tie = zs[:, 1:] == zs[:, :-1]
        assert tie.any() and (src[:, 1:][tie] > src[:, :-1][tie]).all()
        uu = torch.linspace(0.5 / Tf, 1 - 0.5 / Tf, Tf, dtype=torch.float64).expand(N, Tf) if det else u.double()
        ref, ok, bound = _sample_pdf_fp64(zc, sig, nears, fars, uu)
        if Tc == 2:                                          # no bins: every sample is z_mid[0], exactly as fp32 forms it
            mid0 = zc[:, :1] + 0.5 * (zc[:, 1:2] - zc[:, :1])
            assert torch.equal(zn, mid0.expand(N, Tf))
        else:
            assert ok.float().mean() > 0.5
            f64.assert_within(f'z_new {Tc}+{Tf} det={det}', zn[ok], ref[ok], torch.zeros_like(ref[ok]), 0.0, bound[ok])
    sc, sn = torch.rand(N, Tc, generator=g).cuda(), torch.rand(N, Tf, generator=g).cuda()
    cc, cn = torch.rand(N, Tc, 3, generator=g).cuda(), torch.rand(N, Tf, 3, generator=g).cuda()
    so, co = torch.empty(N, T, device='cuda'), torch.empty(N, T, 3, device='cuda')
    srcd = src.to(torch.uint8).cuda()
    lib.call('sfb_ray_gather_sorted_steps', lib.bptr(srcd), f(sc), f(cc), f(sn), f(cn), N, Tc, Tf, f(so), f(co), lib.stream())
    idx = src.cuda()
    assert torch.equal(so, torch.gather(torch.cat([sc, sn], 1), 1, idx))
    assert torch.equal(co, torch.gather(torch.cat([cc, cn], 1), 1, idx[..., None].expand(-1, -1, 3)))


@pytest.mark.parametrize('num_steps', [1, 2, 33, 64, 128, 256])
def test_coarse_depths_equal_the_torch_expression(num_steps):
    lib = _lib()
    f = lib.fptr
    net, _, _ = _net()
    ro, rd = (torch.from_numpy(a).cuda() for a in no.camera_rays(no.circle_cameras(8)[3], 40, 40))
    N = ro.shape[0]
    nears, fars, zc = torch.empty(N, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, num_steps, device='cuda')
    lin, noise = torch.linspace(0, 1, num_steps, device='cuda'), torch.rand(N, num_steps, device='cuda')
    lib.call('sfb_ray_coarse_z', f(ro), f(rd), f(net.aabb_train), 0.1, f(lin), f(noise), N, num_steps, f(nears), f(fars), f(zc), lib.stream())
    zref = nears[:, None] + (fars - nears)[:, None] * lin[None] + (noise - 0.5) * ((fars - nears) / num_steps)[:, None]   # renderer_df.py:356-364
    assert torch.equal(zc, zref)


def test_64_plus_64_through_the_steps_entry_points_is_unchanged():
    """the count-taking entry points at 64 + 64 give exactly what the fixed 64 + 64 ones give"""
    lib = _lib()
    f = lib.fptr
    N = 3001
    z, sig, rgb, nears, fars, _ = _composite_inputs(N, 128, seed=5)
    g = torch.Generator().manual_seed(6)
    gi, gws, gdp = torch.randn(N, 3, generator=g).cuda(), torch.randn(N, generator=g).cuda(), torch.randn(N, generator=g).cuda()
    zd, sd, cd, nd, fd = (t.cuda().contiguous() for t in (z, sig, rgb, nears, fars))
    # device copies held in locals: a temporary's memory returns to the caching allocator as soon as its pointer is taken
    zc = torch.sort(z[:, :64], dim=1).values.cuda()
    sc, sn, cc, cn = (t.cuda().contiguous() for t in (sig[:, :64], sig[:, 64:], rgb[:, :64], rgb[:, 64:]))
    u = torch.rand(N, 64, generator=g).cuda()
    outs = []
    for steps in (None, (64, 64)):
        cnt = (128,) if steps is None else steps
        sfx = '' if steps is None else '_steps'
        image, depth, ws = torch.empty(N, 3, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
        lib.call('sfb_ray_composite_forward' + sfx, f(zd), f(sd), f(cd), f(nd), f(fd), 0.3, N, *cnt, f(image), f(depth), f(ws), lib.stream())
        gsig, grgb = torch.empty(N, 128, device='cuda'), torch.empty(N, 128, 3, device='cuda')
        lib.call('sfb_ray_composite_backward' + sfx, f(zd), f(sd), f(cd), f(nd), f(fd), 0.3, N, *cnt, f(gi), f(gws), f(gdp), f(gsig), f(grgb),
                 lib.stream())
        zs, zn, src = torch.empty(N, 128, device='cuda'), torch.empty(N, 64, device='cuda'), torch.empty(N, 128, dtype=torch.uint8, device='cuda')
        lib.call('sfb_ray_resample' + ('_ex' if steps is None else ''), f(zc), f(sc), f(nd), f(fd), f(u), 0, N, 64, 64, f(zs),
                 *((f(zn), lib.bptr(src)) if steps is None else ()), lib.stream())
        if steps is not None:                            # the merged depths of sfb_ray_resample equal those of sfb_ray_resample_ex
            src = outs[0][6]
        so, co = torch.empty(N, 128, device='cuda'), torch.empty(N, 128, 3, device='cuda')
        lib.call('sfb_ray_gather_sorted' + sfx, lib.bptr(src), f(sc), f(cc), f(sn), f(cn), N, *cnt, f(so), f(co), lib.stream())
        outs.append((image, depth, ws, gsig, grgb, zs, src, so, co))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    # the fixed entry points still refuse other counts
    with pytest.raises(RuntimeError):
        lib.call('sfb_ray_composite_forward', f(zd), f(sd), f(cd), f(nd), f(fd), 0.3, N, 96, f(outs[0][0]), f(outs[0][1]), f(outs[0][2]), lib.stream())


# ------------------------------------------------------------------------------------------------ NeRFNetwork.render
def _device_merged_depths(net, ro, rd, pn, un, Tc, Tf):
    lib = _lib()
    f = lib.fptr
    N = ro.shape[0]
    nears, fars, zc = torch.empty(N, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, Tc, device='cuda')
    lib.call('sfb_ray_coarse_z', f(ro), f(rd), f(net.aabb_train), 0.1, f(torch.linspace(0, 1, Tc, device='cuda')), f(pn), N, Tc, f(nears), f(fars),
             f(zc), lib.stream())
    emb, w0, b0, w1, b1, w2, b2 = [t.detach() for t in net._field_params()]
    sig_c = torch.empty(N, Tc, device='cuda')
    lib.call('sfb_ngp_field_forward', None, f(ro), f(rd), f(zc), Tc, N * Tc, f(emb), lib.iptr(net.encoder.offsets), float(np.log2(net.encoder.per_level_scale)),
             16, 4.0, f(w0), f(b0), f(w1), f(b1), f(w2), f(b2), f(sig_c), None, lib.stream())
    zs = torch.empty(N, Tc + Tf, device='cuda')
    lib.call('sfb_ray_resample', f(zc), f(sig_c), f(nears), f(fars), f(un), 0, N, Tc, Tf, f(zs), lib.stream())
    return zs


@pytest.mark.parametrize('Tc, Tf', GOLDEN_STEPS)
def test_render_at_count_vs_reference_and_oracle(golden_dir, Tc, Tf):
    from _helpers import device_level_scales as _device_scales
    net, p, opt = _net()
    opt.num_steps, opt.upsample_steps = Tc, Tf
    g, ref = np.load(f'{golden_dir}/ngp_run.npz'), np.load(f'{golden_dir}/ngp_run_steps.npz')
    tag = f'{Tc}_{Tf}'
    ro, rd = g['rays_o'], g['rays_d']
    N = ro.shape[0]
    pn, un = _draws(N, Tc, Tf)
    dev = lambda a: torch.from_numpy(a).cuda()
    out = net.render(dev(ro)[None], dev(rd)[None], staged=False, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', force_all_rays=True,
                     perturb_noise=dev(pn), pdf_noise=dev(un), **vars(opt))
    image = out['image'][0]
    r_img, r_ws, r_dp = _rel(image, ref[f'image_{tag}']), _rel(out['weights_sum'], ref[f'weights_sum_{tag}']), _rel(out['depth'][0], ref[f'depth_{tag}'])
    print(f'  {Tc} + {Tf}: vs the reference: image rel {r_img:.2e}, opacity {r_ws:.2e}, depth {r_dp:.2e}')
    assert r_img < 1e-3 and r_ws < 1e-3 and r_dp < 1e-3
    tgt = dev(np.random.default_rng(int(g['target_seed'])).random((N, 3), dtype=np.float32))
    loss = ((image - tgt) ** 2).mean() + 0.1 * out['weights_sum'].mean()
    assert abs(loss.item() - float(ref[f'loss_{tag}'])) < 1e-4 * float(ref[f'loss_{tag}'])
    loss.backward()
    got = dict(net.named_parameters())
    ge = got['encoder.embeddings'].grad.cpu().numpy()
    # loose against the golden (a few ill-conditioned importance samples land in other cells, see test_run_render_vs_oracle_and_golden) ...
    assert _rel(ge[ref['gemb_rows']], ref[f'gemb_vals_{tag}']) < 5e-2
    assert abs(np.abs(ge).sum() - float(ref[f'gemb_abs_sum_{tag}'])) < 3e-3 * float(ref[f'gemb_abs_sum_{tag}'])
    for k in no.PARAM_KEYS[1:]:
        assert _rel(got[k].grad, ref[f'g_{k}_{tag}']) < 2e-2, (k, _rel(got[k].grad, ref[f'g_{k}_{tag}']))
    # ... and tight against the oracle fed the device's merged depths
    rot, rdt = dev(ro), dev(rd)
    zs = _device_merged_depths(net, rot, rdt, dev(pn), dev(un), Tc, Tf) if Tf > 0 else None
    params = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    r = no.run(no.Field(params, level_scales=_device_scales(no.live_geometry())), torch.from_numpy(ro), torch.from_numpy(rd), num_steps=Tc,
               upsample_steps=Tf, perturb_noise=torch.from_numpy(pn), pdf_noise=torch.from_numpy(un), z_sorted_override=None if zs is None else zs.cpu())
    (((r['image'] - tgt.cpu()) ** 2).mean() + 0.1 * r['weights_sum'].mean()).backward()
    assert _rel(image, r['image']) < 1e-5
    for k in no.PARAM_KEYS:
        rr = _rel(got[k].grad, params[k].grad)
        print(f'  {Tc} + {Tf} same depths: grad {k:26s} rel {rr:.3e}')
        assert rr < 2e-3, (k, rr)
    # eval mode: deterministic importance sampling, render_batched chunks
    net.eval()
    with torch.no_grad():
        e = net.render_batched(dev(ro)[None], dev(rd)[None], batched=True, bg_color=0, perturb=False, shading='albedo', **dict(vars(opt), max_ray_batch=500))
    eo = no.run(no.Field(p, level_scales=_device_scales(no.live_geometry())), torch.from_numpy(ro), torch.from_numpy(rd), num_steps=Tc, upsample_steps=Tf,
                training=False)
    assert _rel(e['image'][0], eo['image']) < 1e-3 and _rel(e['image'][0], ref[f'eval_image_{tag}']) < 1e-3
    assert _rel(e['weights_sum'].reshape(-1), ref[f'eval_weights_sum_{tag}']) < 1e-3


def test_render_without_counts_uses_the_references_defaults():
    """render / run default to num_steps = upsample_steps = 128 as the reference's do (renderer_df.py:310)"""
    net, _, _ = _net()
    ro, rd = (torch.from_numpy(a).cuda() for a in no.camera_rays(no.circle_cameras(8)[2], 32, 32))
    outs = []
    for kw in ({}, {'num_steps': 128, 'upsample_steps': 128}):
        torch.cuda.manual_seed(17)
        outs.append(net.render(ro[None], rd[None], perturb=True, bg_color=0, **kw))
    for k in ('image', 'depth', 'weights_sum'):
        assert torch.equal(outs[0][k], outs[1][k]), k
    assert (outs[0]['weights_sum'] > 0).any()


def test_sliced_render_equals_single_launch_at_256_samples():
    net, _, opt = _net()
    opt.num_steps, opt.upsample_steps = 128, 128
    ro, rd = (torch.from_numpy(a).cuda() for a in no.camera_rays(no.circle_cameras(8)[1], 48, 48))
    N = ro.shape[0]
    g = torch.Generator(device='cuda').manual_seed(3)
    pn, un = torch.rand(N, 128, device='cuda', generator=g), torch.rand(N, 128, device='cuda', generator=g)
    kw = dict(staged=False, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', force_all_rays=True, perturb_noise=pn, pdf_noise=un, **vars(opt))
    outs = []
    for cap in (65536, 2000):                            # 2000 rays at 128 samples = 1000 rays per slice at 256: three slices
        net.MAX_RAYS_PER_LAUNCH = cap
        net.zero_grad(set_to_none=True)
        r = net.render(ro[None], rd[None], **kw)
        (r['image'].square().mean() + 0.1 * r['weights_sum'].mean() + 0.01 * r['depth'].mean()).backward()
        outs.append((r['image'].detach().clone(), r['weights_sum'].detach().clone(), r['mask'].clone(), [q.grad.clone() for q in net.parameters()]))
    del net.MAX_RAYS_PER_LAUNCH
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    # float atomics: the order differs between one launch and three.  At 256 samples twice as many points scatter into each embedding
    # row as at 128, and the embedding gradient, whose entries cancel, moves by up to ~1.4e-5 of its norm (1e-5 bounds it at 128)
    for a, b in zip(outs[0][3], outs[1][3]):
        assert ((a - b).norm() / a.norm().clamp(min=1e-30)).item() < 5e-5


# ------------------------------------------------------------------------------------------------ distillation and evaluation
def _small_models():
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.vldm import DDPM
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval()
    vae.load_state_dict(vo.make_params(seed=0, ch=32, ch_mult=(1, 2, 4, 4)))
    cfg = uo.SMALL
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0))
    ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()
    return vae.cuda(), ddpm


def _scenes(S):
    from oracle import distill_oracle as do, unet_oracle as uo
    from sparsefusion_b200.distillation import SceneCache
    return [SceneCache(**do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels, render_hw=64,
                                            seed=3 + k)).to('cuda') for k in range(S)]


@pytest.mark.parametrize('Tc, Tf', [(32, 32), (64, 0)])
def test_distillation_steps_at_count(Tc, Tf):
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, view_seed
    vae, ddpm = _small_models()
    caches = _scenes(2)
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    nets = [_net(seed=k)[0] for k in range(2)]
    opt = get_default_torch_ngp_opt()
    opt.num_steps, opt.upsample_steps = Tc, Tf
    # the photometric render of a step is net.render at the step's keyed draws
    d = Distiller(_net(seed=0)[0], vae, ddpm, opt, caches[0], seed=11)
    ro, rd = caches[0].input_rays_o[0], caches[0].input_rays_d[0]
    draws = d._render_draws(ro, 5, 0, 0, keyed=True)
    assert draws[0].shape == (ro.shape[0], Tc) and draws[1].shape == (ro.shape[0], Tf)
    with torch.no_grad():
        img, ws, _ = d._render(ro, rd, draws)
        gg = torch.Generator(device='cuda')
        gg.manual_seed(view_seed(11, 5, 0, 0))
        pn, un = torch.rand(ro.shape[0], Tc, generator=gg, device='cuda'), torch.rand(ro.shape[0], Tf, generator=gg, device='cuda')
        direct = d.ngp.render(ro[None], rd[None], **dict(d.render_kw, perturb_noise=pn, pdf_noise=un))
    assert torch.equal(img, direct['image'].reshape(-1, 3)) and torch.equal(ws, direct['weights_sum'].reshape(-1))
    before = d.optimizer.flat.clone()
    la, lb = d.step(5)
    assert torch.isfinite(la).all() and torch.isfinite(lb).all() and not torch.equal(d.optimizer.flat, before)
    msd = MultiSceneDistiller(nets, vae, ddpm, opt, caches, seeds=[11, 12])
    before = [s.optimizer.flat.clone() for s in msd.scenes]
    la, lb = msd.step(5)
    assert torch.isfinite(la).all() and torch.isfinite(lb).all()
    assert all(not torch.equal(s.optimizer.flat, b) for s, b in zip(msd.scenes, before))


def test_render_views_at_128_plus_128():
    from sparsefusion_b200.distillation import view_seed
    from sparsefusion_b200.evaluate import render_views
    net, _, opt = _net()
    opt.num_steps, opt.upsample_steps = 128, 128
    H = 32
    cams = no.circle_cameras(8)
    o, d = (torch.stack([torch.from_numpy(no.camera_rays(cams[v], H, H)[i]) for v in (0, 3)]).cuda() for i in (0, 1))
    img, sil = render_views(net, o, d, (H, H), opt, seed=1, stream=0)
    net.eval()
    for k, v in enumerate((0, 3)):
        torch.cuda.manual_seed(view_seed(1, 0, k, 0))
        with torch.no_grad():
            out = net.render_batched(o[k][None], d[k][None], batched=True, perturb=True, bg_color=0, shading='albedo', force_all_rays=True, **vars(opt))
        assert torch.equal(img[k], out['image'].reshape(H, H, 3))
