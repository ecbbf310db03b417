"""oracle/distill_grad_fp64.py on the CPU: the staged fp64 restatement of a distillation sub-step's gradient equals fp64 autograd of the
reference's loss (distillation.py:185-352) end to end, agrees with central differences, accepts an fp32 evaluation of the fused loss path,
and rejects the wiring defects the GPU suite (tests/test_distill_grad_fp64_gpu.py) is there to catch."""
import math

import numpy as np
import pytest
import torch

from oracle import distill_grad_fp64 as dg, lpips_oracle as lo, ngp_oracle as no
from oracle.step_fp64 import f32

HW = 8                      # rays per side; the fusion images are 16 x 16 (LPIPS takes multiples of 16)
LE = 1e-2


def _cfg(le=0.0):
    return dg.StepConfig(lambda_entropy=le)


def _render(seed, hw=HW):
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(hw * hw, 3, generator=g).float()
    ws = (torch.rand(hw * hw, generator=g) * 0.98 + 0.01).float()
    return img, ws


def _targets(seed, hw=HW):
    g = torch.Generator().manual_seed(seed + 100)
    rgb = torch.rand(1, 3, 2 * hw, 2 * hw, generator=g).float()
    mask = (torch.rand(1, 1, 2 * hw, 2 * hw, generator=g) > 0.5).float()
    return rgb, mask


def _autograd_s1(kind, img, ws, cfg, hw=HW, view_scale=1.0, **kw):
    """d (view_scale * loss) / d (image, weights_sum) by fp64 autograd of the reference's expressions"""
    x = img.double().clone().requires_grad_(True)
    s = ws.double().clone().requires_grad_(True)
    im, sil = dg.nchw(x, s, hw)
    (view_scale * dg.reference_loss(kind, im, sil, cfg, **kw)).backward()
    return x.grad, s.grad


def _percep():
    p = {k: v.double() for k, v in lo.make_params(seed=1).items()}
    return lambda a, b: lo.lpips(p, 2 * a - 1, 2 * b - 1).mean()


def _percep_grad(up3, target, percep):
    u = up3.double().clone().requires_grad_(True)
    percep(u[None], target.double()).backward()
    return u.grad


def _rel(a, b):
    return dg.rel_l2(a, b)


@pytest.mark.parametrize('le', [0.0, LE], ids=['no-entropy', 'entropy'])
@pytest.mark.parametrize('kind', ['photo', 'eft', 'sds', 'sds-lpips', 'sds-view-batched'])
def test_s1_equals_autograd_of_the_reference_loss(kind, le):
    cfg = _cfg(le)
    img, ws = _render(1)
    rgb, mask = _targets(1)
    if kind == 'photo':
        got = dg.photometric_grad(img, ws, rgb[0], mask[0], HW, 2, cfg, eager=True)
        want = _autograd_s1('photo', img, ws, cfg, rgb=rgb.double(), mask=mask.double())
    elif kind == 'eft':
        got = dg.fusion_grad(img, ws, HW, rgb[0], 'eft', cfg, eager=True)
        want = _autograd_s1('eft', img, ws, cfg, target=rgb.double())
    else:
        w, _ = dg.sds_weight(0.13)
        percep = _percep() if kind == 'sds-lpips' else None
        vs = 1.0 / 3 if kind == 'sds-view-batched' else 1.0
        gp = None
        if percep is not None:
            gp = _percep_grad(dg.upsample(img, ws, HW)[0][:3], rgb, percep)
        got = dg.fusion_grad(img, ws, HW, rgb[0], 'sds', cfg, weight=w, g_percep=gp, eager=True, view_scale=vs)
        want = _autograd_s1('sds', img, ws, cfg, view_scale=vs, target=rgb.double(), weight=w, percep=percep)
    assert _rel(got['g_img'][0], want[0]) < 1e-12 and _rel(got['g_ws'][0], want[1]) < 1e-12


def test_sds_weight_is_one_minus_the_schedules_alpha_cumprod():
    """sin^2 of the cosine schedule's angle equals 1 - sigmoid(log_snr) of the fp64 schedule, and the bound covers the fp32 log-SNR the
    sampler conditions on"""
    from sparsefusion_b200.plms import _log_snr, _sigmoid
    for t in (0.02, 0.13, 0.37, 0.6, 0.95):
        w, b = dg.sds_weight(t)
        a = (t + 0.008) / 1.008 * math.pi / 2
        ls64 = -math.log(math.cos(a) ** -2 - 1)
        assert abs(w - (1 - 1 / (1 + math.exp(-ls64)))) < 1e-15
        w32 = 1.0 - _sigmoid(_log_snr(t))
        assert abs(w32 - w) <= b, (t, w32, w, b)
        assert b < 1e-3 * w


# ------------------------------------------------------------------------------------------------ S1 o S2 o S3 end to end
def _scene(seed=0):
    geo = no.live_geometry()
    scales = no.level_scales_host(geo['L'], geo['S'], geo['H'])
    ro, rd = no.camera_rays(no.circle_cameras(8)[3], HW, HW)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    aabb = np.array([-4, -4, -4, 4, 4, 4], np.float32)
    nears, fars = (torch.from_numpy(a) for a in no.near_far_from_aabb(ro.numpy(), rd.numpy(), aabb, 0.1))
    rng = np.random.default_rng(seed)
    u = np.sort(rng.random((HW * HW, 128), dtype=np.float32), axis=1)
    zs = (nears[:, None] + (fars - nears)[:, None] * torch.from_numpy(u)).float()
    return no.make_field_params(seed=seed), ro, rd, zs, nears, fars, scales


def _forward32(params, ro, rd, zs, nears, fars, scales):
    """the render the chain starts from: fp64 field and compositing at the samples"""
    from oracle import field_fp64 as f64
    x = f64.ray_points(ro, rd, zs, 4.0)
    fld = f64.FieldFP64(params, x, scales, 4.0)
    fw = fld.forward()
    sigma, rgb = fw['sigma'].view(zs.shape), fw['rgb'].view(*zs.shape, 3)
    r = f64.composite(zs, sigma, rgb, nears, fars, 0.0, torch.zeros(zs.shape[0], 3), None, None)
    return sigma, rgb, r['image'], r['weights_sum']


def _chain(kind, cfg, params, ro, rd, zs, nears, fars, scales, rgb, mask, weight=None, percep=None):
    sigma, col, img, ws = _forward32(params, ro, rd, zs, nears, fars, scales)
    if kind == 'photo':
        s1 = dg.photometric_grad(img, ws, rgb[0], mask[0], HW, 2, cfg, eager=True)
    else:
        gp = None if percep is None else _percep_grad(dg.upsample(img, ws, HW)[0][:3], rgb, percep)
        s1 = dg.fusion_grad(img, ws, HW, rgb[0], kind, cfg, weight=weight, g_percep=gp, eager=True)
    s2 = dg.composite_grad(zs, sigma, col, nears, fars, 0.0, s1['g_img'][0], s1['g_ws'][0])
    return dg.field_grad(params, ro, rd, zs, s2['g_sigma'][0], s2['g_rgb'][0], scales, 'v2', 132)


@pytest.mark.parametrize('kind,le,lpips', [('photo', 0.0, False), ('photo', LE, False), ('eft', 0.0, False), ('eft', LE, False),
                                           ('sds', LE, False), ('sds', 0.0, True), ('sds', LE, True)])
def test_chain_equals_end_to_end_autograd(kind, le, lpips):
    """S3(S2(S1)) -- each stage fed the previous stage's fp64 output -- against one fp64 autograd graph of field, compositing and loss"""
    cfg = _cfg(le)
    params, ro, rd, zs, nears, fars, scales = _scene()
    rgb, mask = _targets(2)
    w = dg.sds_weight(0.13)[0]
    percep = _percep() if lpips else None
    chain = _chain(kind, cfg, params, ro, rd, zs, nears, fars, scales, rgb, mask, weight=w, percep=percep)
    kw = dict(rgb=rgb.double(), mask=mask.double()) if kind == 'photo' else dict(target=rgb.double(), weight=w, percep=percep)
    e2e = dg.end_to_end_grad(params, ro, rd, zs, nears, fars, HW, lambda im, sil: dg.reference_loss(kind, im, sil, cfg, **kw), scales)
    for k in no.PARAM_KEYS:
        r = _rel(chain[k][0], e2e[k])
        assert r < 1e-12, (k, r)


def test_end_to_end_gradient_agrees_with_central_differences():
    """the fp64 end-to-end gradient against central differences of the same fp64 loss on embedding rows the render hits and on MLP
    weights (photometric and EFT terms with entropy: smooth away from ReLU kinks)"""
    cfg = _cfg(LE)
    params, ro, rd, zs, nears, fars, scales = _scene(1)
    rgb, mask = _targets(3)

    def loss(p):
        out = {}

        def fn(im, sil):
            v = dg.reference_loss('photo', im, sil, cfg, rgb=rgb.double(), mask=mask.double()) \
                + dg.reference_loss('eft', im, sil, cfg, target=rgb.double())
            out['v'] = v.item()
            return v
        g = dg.end_to_end_grad(p, ro, rd, zs, nears, fars, HW, fn, scales)
        return out['v'], g

    _, grad = loss(params)
    emb_rows = torch.nonzero(grad['encoder.embeddings'].abs().sum(1) > 0).reshape(-1)
    picks = [('encoder.embeddings', (int(r), c)) for r, c in zip(emb_rows[torch.randperm(emb_rows.numel(), generator=torch.Generator().manual_seed(0))[:6]], range(6))]
    picks = [(k, (i[0], i[1] % 2)) for k, i in picks]
    picks += [('sigma_net.net.0.weight', (3, 7)), ('sigma_net.net.1.weight', (10, 20)), ('sigma_net.net.2.weight', (0, 5)),
              ('sigma_net.net.2.weight', (2, 9)), ('sigma_net.net.2.bias', (1,))]
    for k, idx in picks:
        h = 1e-4 * max(1.0, abs(float(params[k][idx])))
        pp = {kk: v.double().clone() for kk, v in params.items()}
        pp[k][idx] += h
        lp, _ = loss(pp)
        pp[k][idx] -= 2 * h
        lm, _ = loss(pp)
        fd = (lp - lm) / (2 * h)
        an = float(grad[k][idx])
        assert abs(fd - an) <= 1e-5 * abs(an) + 1e-12, (k, idx, fd, an)


# ------------------------------------------------------------------------------------------------ the bounds' teeth
def _fused_bounds(img, ws, target, mode, cfg, weight, g_percep=None, view_scale=1.0):
    return dg.fusion_grad(img, ws, HW, target, mode, cfg, weight=weight, g_percep=g_percep, view_scale=view_scale)


@pytest.mark.parametrize('mode', ['sds', 'eft'])
def test_fp32_emulation_passes_and_defects_are_flagged(mode):
    cfg = _cfg(LE)
    img, ws = _render(5)
    rgb, _ = _targets(5)
    target = rgb[0] * 0.5
    w, _ = dg.sds_weight(0.13)
    gp = None
    if mode == 'sds':
        gp = _percep_grad(dg.upsample(img, ws, HW)[0][:3], target[None], _percep())
    vs = 1.0 / 3
    ref = _fused_bounds(img, ws, target, mode, cfg, w, gp, vs)
    ok = dg.emulate_fusion(img, ws, HW, target, mode, cfg, w, g_percep=gp, view_scale=vs)
    ratios = (dg.within(ok[0], ref['g_img']), dg.within(ok[1], ref['g_ws']))
    print(f'{mode}: fp32 emulation err/bound {ratios}')
    assert max(ratios) <= 1
    w_last = 1.0 - 1.0 / (1.0 + math.exp(-(-math.log(math.cos((0.01 + 0.008) / 1.008 * math.pi / 2) ** -2 - 1))))   # t = 0.01, the run's last level
    defects = ['double', 'no_opacity_grad', 'no_entropy_grad', 'unscaled_view']
    gp_target = None
    if mode == 'sds':
        defects += ['weight', 'percep_wrt_target']
        # LPIPS called as (pred_img, up[:3]): its gradient is the one with respect to the target, at the same pair of images
        up3 = dg.upsample(img, ws, HW)[0][:3]
        t = target.double().clone().requires_grad_(True)
        _percep()(t[None], up3[None]).backward()
        gp_target = t.grad
    for defect in defects:
        bad = dg.emulate_fusion(img, ws, HW, target, mode, cfg, w_last if defect == 'weight' else w,
                                g_percep=gp_target if defect == 'percep_wrt_target' else gp, view_scale=vs,
                                defect=None if defect in ('weight', 'percep_wrt_target') else defect)
        r = max(dg.within(bad[0], ref['g_img']), dg.within(bad[1], ref['g_ws']))
        print(f'  {defect}: err/bound {r:.3g}')
        assert r > 1, defect


def test_step_lr_pins_the_steplr_boundaries():
    """torch's StepLR after 2999 / 3000 / 5999 / 6000 scheduler steps, and a swap of the two groups' rates is not one of them"""
    cfg = dg.StepConfig()
    want = {0: 1.0, 2999: 1.0, 3000: 0.2, 5999: 0.2, 6000: 0.04}
    for s, mult in want.items():
        lrs = dg.step_lr(cfg, s)
        assert [f32(v) for v in lrs] == [f32(5e-3 * mult), f32(5e-4 * mult)], (s, lrs)
        assert [f32(v) for v in lrs[::-1]] != [f32(v) for v in lrs]


def test_adam_reference_bounds_an_fp32_update():
    """adam_reference's bound holds for an fp32 Adam step from a restored state, and not for the step with its group rates swapped"""
    cfg = dg.StepConfig()
    g = torch.Generator().manual_seed(0)
    n0, n1 = 300, 200
    flat = torch.randn(n0 + n1, generator=g)
    grad = torch.randn(n0 + n1, generator=g) * 1e-4
    m = torch.randn(n0 + n1, generator=g) * 1e-5
    v = torch.rand(n0 + n1, generator=g) * 1e-9
    t, lrs = 7, [5e-3, 5e-4]
    b1, b2 = (f32(b) for b in cfg.betas)

    def fp32_step(lr_list):
        out = flat.clone()
        for (s, e), lr in zip(((0, n0), (n0, n0 + n1)), lr_list):
            mm = b1 * m[s:e] + (1 - b1) * grad[s:e]
            vv = b2 * v[s:e] + (1 - b2) * grad[s:e] ** 2
            mh, vh = mm / (1 - b1 ** t), vv / (1 - b2 ** t)
            out[s:e] = flat[s:e] - f32(lr) * mh / (vh.sqrt() + f32(cfg.eps))
        return out
    y, a, sl = dg.adam_reference(flat, grad, m, v, t, lrs, ((0, n0), (n0, n0 + n1)), cfg)
    ok = fp32_step(lrs)
    err = (ok.double() - y).abs()
    assert (err <= dg.gamma(3) * a + sl + 1e-30).all()
    bad = fp32_step(lrs[::-1])
    assert ((bad.double() - y).abs() > dg.gamma(3) * a + sl).any()
