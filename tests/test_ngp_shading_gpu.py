"""The finite-difference normal stencils (sfb_ngp_field_normal_forward / _backward, csrc/ngp_field.cu) element by element against the fp64
oracle (oracle/normal_fp64.py), and the shadings of NeRFNetwork.forward, NeRFRenderer.run and run_cuda that use them.

Bounds follow test_ngp_field_fp64_gpu.py: per element, |got - ref| <= rtol * ref_abs + slack, rtol the longest chain of fp32 roundings.
fd = 0.5 (m+ - m-) / eps cancels, so its companion is (abs+ + abs-) / (2 eps); normalised normals are compared where |fd| is at least 10
times its bound.  Jitter is reproduced bit for bit from the key by the oracle's numpy Philox4x32-10.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import field_fp64 as f64
from oracle import ngp_oracle as no
from oracle import normal_fp64 as nf

pytestmark = pytest.mark.gpu

BOUND = 4.0
GEO = no.live_geometry(BOUND)
KEY = 0x0123_4567_89ab_cdef - (1 << 62)


def _lib():
    from sparsefusion_b200 import _lib as lib
    return lib


def _scales():
    from _helpers import device_level_scales
    return device_level_scales(GEO)


def _sm_count():
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib().call('sfb_device_info', ctypes.addressof(sm), ctypes.addressof(major), ctypes.addressof(minor))
    return sm.value


def _stencil(p, B, xyz=None, rays=None, slots=6, k=1, eps=1e-2, radius=0.0, key=None):
    lib = _lib()
    f = lib.fptr
    q = {n: v.detach().float().cuda().contiguous() for n, v in p.items()}
    offsets = torch.from_numpy(GEO['offsets']).cuda()
    src = (f(xyz), None, None, None, 0) if xyz is not None else (None, f(rays[0]), f(rays[1]), f(rays[2]), rays[2].shape[1])
    a = torch.full((B, 3), -7.0, device='cuda')
    b = torch.full((B, 3), -7.0, device='cuda')
    s = torch.full((B,), -7.0, device='cuda')
    kt = None if key is None else torch.tensor([key], dtype=torch.int64, device='cuda')
    lib.call('sfb_ngp_field_normal_forward', *src, B, f(q['encoder.embeddings']), lib.iptr(offsets), float(GEO['S']), 16, BOUND,
             *[f(q[n]) for n in no.PARAM_KEYS[1:]], slots, k, float(eps), float(radius), None if kt is None else kt.data_ptr(),
             f(a) if slots == 6 else None, f(b) if slots == 6 else None, f(s) if slots == 1 else None, f(a) if slots == 1 else None, lib.stream())
    torch.cuda.synchronize()
    return (a, b) if slots == 6 else (s, a)


def _stencil_backward(p, B, fd, xyz=None, rays=None, g_normal=None, g_fd=None, prefill=None):
    lib = _lib()
    f = lib.fptr
    q = {n: v.detach().float().cuda().contiguous() for n, v in p.items()}
    offsets = torch.from_numpy(GEO['offsets']).cuda()
    src = (f(xyz), None, None, None, 0) if xyz is not None else (None, f(rays[0]), f(rays[1]), f(rays[2]), rays[2].shape[1])
    grads = {n: (prefill[n].clone().cuda() if prefill is not None else torch.zeros_like(q[n])) for n in no.PARAM_KEYS}
    gn = None if g_normal is None else g_normal.float().cuda().contiguous()
    gf = None if g_fd is None else g_fd.float().cuda().contiguous()
    lib.call('sfb_ngp_field_normal_backward', *src, B, f(q['encoder.embeddings']), lib.iptr(offsets), float(GEO['S']), 16, BOUND,
             *[f(q[n]) for n in no.PARAM_KEYS[1:]], 1e-2, f(fd), None if gn is None else f(gn), None if gf is None else f(gf),
             *[f(grads[n]) for n in no.PARAM_KEYS], lib.stream())
    torch.cuda.synchronize()
    return grads


def _points(B, seed):
    """uniform in [-1.02, 1.02] bound (some outside the box), plus points within eps of the faces and near the blob"""
    rng = np.random.default_rng(seed)
    x = ((rng.random((B, 3), dtype=np.float32) * 2 - 1) * 1.02 * BOUND).astype(np.float32)
    x[:64, 0] = np.float32(BOUND - 0.004)
    x[64:128, 1] = np.float32(-BOUND + 0.006)
    x[128:192, 2] = np.float32(BOUND)
    x[192:256] = (rng.random((64, 3), dtype=np.float32) * 2 - 1) * np.float32(0.3)
    return torch.from_numpy(x)


def _rays(N, T, seed):
    rng = np.random.default_rng(seed)
    o = torch.from_numpy((rng.standard_normal((N, 3)) * 1.5).astype(np.float32))
    d = torch.from_numpy(rng.standard_normal((N, 3)).astype(np.float32))
    d = d / d.norm(dim=-1, keepdim=True)
    z = torch.from_numpy(np.sort(rng.random((N, T), dtype=np.float32) * 7, 1).astype(np.float32))
    return o, d, z


def _check_fd_normal(fd, n, st: nf.StencilFP64, what):
    f64.assert_within(f'{what} fd', fd, st.fd, st.fd_abs, st.rtol())
    ref, reliable = st.normal()
    assert int(reliable.sum()) >= 50, 'too few points with a well-determined normal'
    bound = st.normal_rtol().expand_as(ref)
    f64.assert_within(f'{what} normal', n[reliable.to(n.device)], ref[reliable], torch.ones_like(ref[reliable]), bound[reliable])
    live = torch.isfinite(st.fd).all(-1) & (st.fd.abs().sum(-1) > 0)
    assert int(live.sum()) > 0 and ((n.norm(dim=-1)[live] - 1).abs() < 1e-5).all()      # every finite, non-zero fd gives a unit normal
    assert (n[~live] == 0).all()


@pytest.mark.parametrize('B', [5000, 7001])          # 7001 > 2 SM x 21 points per tile on an H100: the grid-stride loop wraps
def test_plain_stencil_explicit_points(B):
    p = no.make_field_params(seed=3)
    x = _points(B, B)
    fd, n = _stencil(p, B, xyz=x.cuda())
    _check_fd_normal(fd, n, nf.StencilFP64(p, x, _scales(), device='cuda'), f'B={B}')


def test_plain_stencil_ray_samples():
    p = no.make_field_params(seed=5)
    o, d, z = _rays(60, 128, 7)
    B = 60 * 128
    fd, n = _stencil(p, B, rays=(o.cuda(), d.cuda(), z.cuda()))
    x = f64.ray_points(o, d, z, BOUND)
    _check_fd_normal(fd, n, nf.StencilFP64(p, x, _scales(), device='cuda'), 'rays')


def test_overflowing_sigma_gives_zero_normals():
    p = no.make_field_params(seed=3)
    p['sigma_net.net.2.bias'] = p['sigma_net.net.2.bias'].clone()
    p['sigma_net.net.2.bias'][0] = 200.0
    x = _points(1000, 1)
    fd, n = _stencil(p, 1000, xyz=x.cuda())
    st = nf.StencilFP64(p, x, _scales(), device='cuda')
    assert torch.isnan(st.fd).all() and torch.isnan(fd).all()
    assert (n == 0).all()


def test_smoothed_stencil_reproduces_jitter():
    p = no.make_field_params(seed=4)
    x = _points(3000, 9)
    fd, n = _stencil(p, 3000, xyz=x.cuda(), k=10, eps=0.3, radius=0.3, key=KEY)
    _check_fd_normal(fd, n, nf.StencilFP64(p, x, _scales(), k=10, eps=0.3, radius=0.3, key=KEY, device='cuda'), 'smooth')


def test_common_forward_smooth_reproduces_jitter():
    p = no.make_field_params(seed=4)
    x = _points(4000, 10)
    sigma, albedo = _stencil(p, 4000, xyz=x.cuda(), slots=1, k=5, radius=1e-2, key=KEY)
    st = nf.StencilFP64(p, x, _scales(), slots=1, k=5, radius=1e-2, key=KEY, device='cuda')
    f64.assert_within('smooth sigma', sigma, st.sigma, st.sigma_abs, st.rtol())
    f64.assert_within('smooth albedo', albedo, st.albedo, st.albedo_abs, st.rtol())


def _net(seed=3, cuda_ray=False):
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = cuda_ray
    net = NeRFNetwork(opt).cuda()
    sd = net.state_dict()
    for k, v in no.make_field_params(seed=seed).items():
        sd[k] = v
    net.load_state_dict(sd)
    return net


def test_seed_reproducibility():
    net = _net()
    x = _points(2000, 11).cuda()
    torch.cuda.manual_seed(5)
    a = net.normal(x, smooth=True)
    s1, _ = net.common_forward_smooth(x)
    torch.cuda.manual_seed(5)
    b = net.normal(x, smooth=True)
    s2, _ = net.common_forward_smooth(x)
    torch.cuda.manual_seed(6)
    c = net.normal(x, smooth=True)
    assert torch.equal(a, b) and torch.equal(s1, s2)
    assert not torch.equal(a, c)


def test_plain_stencil_backward_accumulates():
    p = no.make_field_params(seed=3)
    B = 7001
    x = _points(B, 12)
    fd, _ = _stencil(p, B, xyz=x.cuda())
    rng = np.random.default_rng(13)
    g_fd = torch.from_numpy(np.abs(rng.standard_normal((B, 3))).astype(np.float32) * 1e-3)
    prefill = {k: torch.from_numpy(rng.standard_normal(v.shape).astype(np.float32)) for k, v in p.items()}
    got = _stencil_backward(p, B, fd, xyz=x.cuda(), g_fd=g_fd, prefill=prefill)
    st = nf.StencilFP64(p, x, _scales(), device='cuda')
    bwd = st.backward(fd, g_fd=g_fd)
    sm = _sm_count()
    tiles = -(-B // 10)
    for k in no.PARAM_KEYS:
        pf = prefill[k].cuda().double()
        want, want_abs = bwd[k] + pf, bwd[k + '_abs'] + pf.abs()
        if k == 'encoder.embeddings':
            rtol = f64.RTOL_POINT + f64.gamma(bwd[k + '_hits'] + 2)
        else:
            rtol = f64.wgrad_rtol('v2', tiles * 64, sm) + f64.gamma(3)
        f64.assert_within(k, got[k], want, want_abs, rtol, bwd[k + '_slack'])


def _relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def test_normal_autograd_matches_oracle_backward():
    """NeRFNetwork.normal's gradient (safe_normalize backward in the kernel) against the oracle's at the kernel's fd"""
    net = _net()
    B = 3000
    x = _points(B, 14)
    g = torch.from_numpy(np.random.default_rng(15).standard_normal((B, 3)).astype(np.float32))
    n = net.normal(x.cuda())
    (n * g.cuda()).sum().backward()
    fd = net.finite_difference_normal(x.cuda()).detach()
    bwd = nf.StencilFP64(no.make_field_params(seed=3), x, _scales(), device='cuda').backward(fd, g_normal=g)
    names = dict(net.named_parameters())
    for k in no.PARAM_KEYS:
        # relative to the absolute companion: the output bias's sigma row gets sum_q g_fd . fd = 0 exactly (a common factor on sigma
        # leaves the normal unchanged), so both sides are rounding residue there
        err = (names[k].grad.double() - bwd[k]).norm().item()
        assert err <= 1e-4 * bwd[k + '_abs'].norm().item(), k


@pytest.mark.parametrize('shading', ['albedo', 'lambertian', 'textureless', 'normal', 'anything-else'])
def test_network_forward_shadings(shading):
    net = _net()
    x = _points(2000, 16).cuda()
    l = torch.nn.functional.normalize(torch.tensor([0.3, -0.5, 0.8]), dim=0).cuda()
    torch.cuda.manual_seed(1)
    sigma, color, normal = net(x, None, l, ratio=0.2, shading=shading)
    s0, a0 = net.common_forward(x)
    assert torch.equal(sigma, s0)
    if shading == 'albedo':
        assert normal is None and torch.equal(color, a0)
        return
    torch.cuda.manual_seed(1)
    n0 = net.normal(x, smooth=shading in ('textureless', 'normal'))
    assert torch.equal(normal.detach(), n0.detach())
    # network_grid.py:188-195 in closed form, per element; the light leaves n . (-l) strictly inside (0, 1) for many points, where a swap of
    # ratio and 1 - ratio, a lost clamp or a flipped light would show
    n, a = n0.detach().double(), a0.detach().double()
    c = (n @ -l.double()).clamp(min=0)
    assert ((c > 0.05) & (c < 0.95)).double().mean() > 0.2
    lam = 0.2 + 0.8 * c
    want = {'textureless': (lam * 0.8 + 0.2)[:, None].expand(-1, 3), 'normal': (n + 1) / 2}.get(shading, a * lam[:, None])
    assert (color.detach().double() - want).abs().max() < 1e-6
    if shading in ('lambertian', 'anything-else'):
        assert color.requires_grad and normal.requires_grad
    else:
        assert not normal.requires_grad


def _run_case(net, shading, train, N=512, seed=20):
    rng = np.random.default_rng(seed)
    o = torch.from_numpy((rng.standard_normal((N, 3)) * 0.3 + np.array([0, 0, 2.5])).astype(np.float32)).cuda()
    d = torch.from_numpy((np.array([0, 0, -1]) + rng.standard_normal((N, 3)) * 0.3).astype(np.float32)).cuda()
    d = d / d.norm(dim=-1, keepdim=True)
    pn = torch.from_numpy(rng.random((N, 64), dtype=np.float32)).cuda()
    pdf = torch.from_numpy(rng.random((N, 64), dtype=np.float32)).cuda()
    nn_ = torch.from_numpy(rng.standard_normal((N, 128, 3)).astype(np.float32)).cuda()
    l = torch.nn.functional.normalize(torch.tensor([0.2, 0.4, 0.9]), dim=0).cuda()
    net.train(train)
    return o, d, dict(num_steps=64, upsample_steps=64, light_d=l, ambient_ratio=0.3, shading=shading, bg_color=0, perturb=True,
                      perturb_noise=pn, pdf_noise=pdf, normal_noise=nn_)


def _composed(net, o, d, kw, zs, nears, fars):
    """the same render from independent pieces: explicit-point field and stencil calls at the materialised samples, shading and the
    reference's compositing (renderer_df.py:414-456) and regularisers (:427-436) in torch autograd"""
    from sparsefusion_b200.network_grid import shade
    N = o.shape[0]
    x = torch.min(torch.max(o[:, None, :] + d[:, None, :] * zs[..., None], net.aabb_train[:3]), net.aabb_train[3:])
    sigma, albedo = net.common_forward(x.reshape(-1, 3))
    normal = net.normal(x.reshape(-1, 3), smooth=kw['shading'] in ('textureless', 'normal'))
    color, _ = shade(albedo, normal, kw['light_d'], kw['ambient_ratio'], kw['shading'])
    sigma, color = sigma.view(N, 128), color.view(N, 128, 3)
    deltas = torch.cat([zs[:, 1:] - zs[:, :-1], ((fars - nears) / 64)[:, None]], -1)
    alphas = 1 - torch.exp(-deltas * sigma)
    weights = alphas * torch.cumprod(torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], -1), -1)[:, :-1]
    ws = weights.sum(-1)
    depth = (weights * ((zs - nears[:, None]) / (fars - nears)[:, None]).clamp(0, 1)).sum(-1)
    image = (weights[..., None] * color).sum(-2) + (1 - ws)[:, None] * kw['bg_color']
    normals = normal.view(N, 128, 3)
    loss_orient = (weights.detach() * (normals * d[:, None, :]).sum(-1).clamp(min=0) ** 2).mean()
    npert = net.normal(x + kw['normal_noise'] * 1e-2).view(N, 128, 3)
    loss_smooth = (normals - npert).abs().mean()
    return dict(image=image, depth=depth, weights_sum=ws, loss_orient=loss_orient, loss_smooth=loss_smooth)


@pytest.mark.parametrize('train', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('shading', ['lambertian', 'textureless', 'normal'])
def test_run_with_shading(shading, train):
    from sparsefusion_b200.renderer_df import _sorted_samples
    net = _net(seed=6)
    o, d, kw = _run_case(net, shading, train)
    N = o.shape[0]
    g = torch.from_numpy(np.random.default_rng(21).standard_normal((N, 3)).astype(np.float32)).cuda()
    torch.cuda.manual_seed(3)
    out = net.run(o[None], d[None], **kw)
    loss = (out['image'][0] * g).sum() + out['loss_orient'] + out['loss_smooth']
    net.zero_grad()
    loss.backward()
    got = {k: v.grad.clone() for k, v in net.named_parameters()}
    with torch.no_grad():
        pdf_u = kw['pdf_noise'] if train else torch.linspace(0.5 / 64, 1 - 0.5 / 64, 64, device='cuda').expand(N, 64).contiguous()
        zs, _, _, nears, fars = _sorted_samples(net, o, d, net.aabb_train if train else net.aabb_infer, net.min_near, kw['perturb_noise'],
                                                pdf_u, *net._field_params())
    torch.cuda.manual_seed(3)
    want = _composed(net, o, d, kw, zs, nears, fars)
    wl = (want['image'] * g).sum() + want['loss_orient'] + want['loss_smooth']
    net.zero_grad()
    wl.backward()
    for k in ('image', 'depth', 'weights_sum'):          # per ray: values on [0, 1]
        assert (out[k].detach().reshape(-1) - want[k].detach().reshape(-1)).abs().max() < 2e-5, k
    for k in ('loss_orient', 'loss_smooth'):
        assert abs(out[k].item() - want[k].item()) <= 1e-5 * abs(want[k].item()), k
    for k, v in net.named_parameters():                   # per element, on the scale of the tensor
        assert (got[k] - v.grad).abs().max() <= 1e-3 * v.grad.abs().max(), k


def test_run_cuda_with_shading():
    """run_cuda in training: the default light (renderer_df.py:486-489), the lambertian colour per marched sample, and loss_orient /
    loss_smooth (:509-519) restated from the samples the network was queried at"""
    net = _net(seed=6, cuda_ray=True)
    net.update_extra_state()
    o, d, _ = _run_case(net, 'lambertian', True, N=1024)
    calls, fwd0, normal0 = [], net.forward, net.normal

    def forward(x, dirs, l=None, ratio=1, shading='textureless'):
        out = fwd0(x, dirs, l, ratio, shading)
        calls.append(('forward', x.detach().clone(), dirs.detach().clone(), l.detach().clone(), *[t.detach().clone() for t in out]))
        return out

    def normal(x, smooth=False):
        calls.append(('normal', x.detach().clone(), smooth))
        return normal0(x, smooth)
    net.forward, net.normal = forward, normal
    torch.cuda.manual_seed(9)
    out = net.run_cuda(o[None], d[None], ambient_ratio=0.3, shading='lambertian', bg_color=0, perturb=False, force_all_rays=True)
    torch.cuda.manual_seed(9)
    light = o[0] + torch.randn(3, device='cuda')
    light = light / light.norm().clamp(min=1e-10)
    fw = [c for c in calls if c[0] == 'forward']
    assert len(fw) == 1
    _, x, dirs, l, sigma, color, n = fw[0]
    assert x.shape[0] > 1000, 'too few marched samples'
    assert (l - light).abs().max() < 1e-6
    c = (n.double() @ -l.double()).clamp(min=0)
    _, albedo = net.common_forward(x)
    assert (color.double() - albedo.double() * (0.3 + 0.7 * c)[:, None]).abs().max() < 1e-6
    w = 1 - torch.exp(-sigma.double())
    want_orient = (w * (n.double() * dirs.double()).sum(-1).clamp(min=0) ** 2).mean()
    assert abs(out['loss_orient'].item() - want_orient.item()) <= 1e-5 * want_orient.item()
    kind, xp, smooth = calls[-1]
    assert kind == 'normal' and not smooth and 0 < (xp - x).abs().max() < 0.1
    want_smooth = (n.double() - normal0(xp).detach().double()).abs().mean()
    assert abs(out['loss_smooth'].item() - want_smooth.item()) <= 1e-5 * want_smooth.item()
    (out['image'].sum() + out['loss_orient'] + out['loss_smooth']).backward()
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
    assert net.encoder.embeddings.grad.abs().sum() > 0
    net.forward, net.normal = fwd0, normal0
    net.eval()
    with torch.no_grad():
        out = net.run_cuda(o[None], d[None], shading='normal', bg_color=0)
    assert torch.isfinite(out['image']).all() and 'loss_orient' not in out
    assert (out['image'] >= 0).all() and (out['image'] <= 1 + 1e-5).all()


def test_render_views_with_normal_shading():
    from sparsefusion_b200.evaluate import render_views
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    net = _net(seed=6)
    opt = get_default_torch_ngp_opt()
    V, H = 2, 32
    rng = np.random.default_rng(30)
    o = torch.from_numpy(np.tile(np.array([0, 0, 2.5], np.float32), (V, H * H, 1))).cuda()
    d = torch.from_numpy((np.array([0, 0, -1]) + rng.standard_normal((V, H * H, 3)) * 0.2).astype(np.float32)).cuda()
    d = d / d.norm(dim=-1, keepdim=True)
    a, sa = render_views(net, o, d, (H, H), opt, seed=1, stream=0)
    img, sil = render_views(net, o, d, (H, H), opt, seed=1, stream=0, shading='normal')
    img2, _ = render_views(net, o, d, (H, H), opt, seed=1, stream=0, shading='normal')
    assert img.shape == (V, H, H, 3) and torch.isfinite(img).all() and torch.equal(img, img2)
    assert torch.equal(sil, sa)                        # same samples and densities; only the colours differ
    assert not torch.equal(img, a) and (img >= 0).all() and (img <= 1 + 1e-5).all()


def test_visualize_shadings_writes_circle_gifs(tmp_path, capsys):
    """distillation_loop(visualize=True, visualize_shadings=('normal', 'textureless')): one 50-frame circle gif per shading, the headlit
    render_views frames of the circle path (stream 4; ambient 0.1 for the lit shading), through the GPU palette path"""
    from types import SimpleNamespace
    from test_video_gpu import N_CIRCLE, _VisBuilder, _assert_gif, _decode_gif, _models
    from sparsefusion_b200.distillation import distill_scenes, distillation_loop, get_default_torch_ngp_opt
    from sparsefusion_b200.evaluate import CIRCLE_STREAM, render_views
    from sparsefusion_b200.video import to_uint8
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    rgb, mask = torch.zeros(3, 3, 128, 128), torch.zeros(3, 1, 128, 128)
    builder = _VisBuilder(cfg)
    out = tmp_path / 'out'
    net = distillation_loop(0, SimpleNamespace(exp_dir=str(tmp_path / 'exp')), opt, models, str(out), 'hydrant_000', 3, rgb, mask, None, [0, 1],
                            use_diffusion=False, max_itr=2, scene_builder=builder, seed=5, visualize=True,
                            visualize_shadings=('normal', 'textureless'))
    printed = capsys.readouterr().out
    co, cd = (t.cuda() for t in builder.circle_views(3))
    for shading, ratio in (('normal', 1.0), ('textureless', 0.1)):
        path = out / 'render_gifs' / f'hydrant_000_circle_{shading}.gif'
        assert f'saved video {path}\n' in printed
        img, _ = render_views(net, co, cd, (128, 128), opt, seed=5, stream=CIRCLE_STREAM, shading=shading, ambient_ratio=ratio)
        assert img.shape[0] == N_CIRCLE == 50
        _assert_gif(path, to_uint8(img), (128, 128, 3))
        assert sum(dur for _, dur in _decode_gif(path)) == 50 * 200          # 50 frames of 200 ms (identical neighbours merged)
    assert (out / 'render_gifs' / 'hydrant_000_circle.gif').exists()
    # the default writes no shading gifs; distill_scenes takes the option too; names that are not shading names are refused
    nets = distill_scenes(0, SimpleNamespace(exp_dir=str(tmp_path / 'b')), opt, models, str(tmp_path / 'b'), [('s0', 3, rgb, mask, None, [0, 1])],
                          use_diffusion=False, max_itr=1, scene_builder=builder, seed=5, visualize=True, visualize_shadings=('lambertian',))
    assert len(nets) == 1 and (tmp_path / 'b' / 'render_gifs' / 's0_circle_lambertian.gif').exists()
    assert not list((tmp_path / 'b' / 'render_gifs').glob('s0_circle_normal*'))
    with pytest.raises(ValueError, match='visualize_shadings'):
        distillation_loop(0, SimpleNamespace(exp_dir=str(tmp_path / 'c')), opt, models, str(tmp_path / 'c'), 'h', 3, rgb, mask, None, [0, 1],
                          use_diffusion=False, max_itr=1, scene_builder=builder, seed=5, visualize=True, visualize_shadings=('../x',))
