"""oracle/step_fp64.py checked on the CPU: the launch plans against hand-derived ones, the fp64 references against torch autograd of the
distillation.py expressions and against F.grid_sample / F.interpolate / nn.MultiheadAttention in fp64, and sensitivity self-checks: the
defect-free fp32 evaluation passes each per-element bound and every injected defect is rejected.

Seen: h / w swapped in the glue's flat index, the nearest source one column off, the adjoint without its edge clamp, the mode-1 mask with
>= at a mean of exactly 0.1f, g_extra added to the silhouette plane, the e1 / e2 coefficients swapped, a row reading row r - 1's scalars,
the alpha clamp missing, a clamp that drops NaN, align_corners=False or zero padding in grid_sample, x / y swapped in resize, the max-pool
window shifted by one, the attention scale 1 / E and the softmax over the batch instead of the sequence."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import insitu, step_fp64 as sp

SM = 132      # H100 SXM
g = torch.Generator().manual_seed(0)


def rn(*s):
    return torch.randn(*s, generator=g)


def rand(*s):
    return torch.rand(*s, generator=g)


# ------------------------------------------------------------------------------------------------ plans and bounds
def test_plans():
    assert sp.kernel_plan('plms_update', dict(n=1))['grid'] == (1, 1)
    assert sp.kernel_plan('plms_update', dict(n=257))['grid'] == (2, 1)
    assert sp.kernel_plan('plms_update', dict(n=1024 * 256 + 1))['grid'] == (1024, 1)          # the grid-stride loop takes over
    assert sp.kernel_plan('plms_update_rows', dict(rows=3, row_len=4096))['grid'] == (16, 3)
    assert sp.kernel_plan('plms_update_rows_cfg', dict(rows=2, row_len=10 ** 6))['kernels'] == ['sfb::plms_update_rows_cfg_kernel']
    d = lambda L: sp.kernel_plan('ddpm_dynamic_step', dict(B=2, row_len=L))
    assert (d(8192)['k'], d(8192)['kernels']) == (1, ['sfb::ddpm_dynamic_step_kernel<false>'])
    assert (d(8193)['k'], d(8193)['chunk'], d(8193)['smem']) == (2, 4097, 4097 * 4)
    assert (d(57345)['k'], d(57345)['chunk']) == (8, 7169)                                    # uneven: the last CTA holds 7162
    assert (d(65536)['k'], d(65536)['smem'], d(65536)['kernels']) == (8, 32768, ['sfb::ddpm_dynamic_step_kernel<true>'])
    p = sp.kernel_plan('photometric_loss', dict(h=128, w=128), SM)
    assert (p['blocks'], p['iters']) == (64, 1)
    p = sp.kernel_plan('fusion_loss', dict(h=128, w=128), SM)
    assert (p['blocks'], p['iters']) == (256, 1)                                              # 65 536 full-resolution pixels
    p = sp.kernel_plan('fusion_loss', dict(h=256, w=256), SM)
    assert (p['blocks'], p['iters']) == (264, 4)


def test_bound_arithmetic():
    assert sp.sum_chain(dict(blocks=264, iters=4)) == 5 + 12 + 8 + 264
    x = torch.tensor([[1.0]])
    r = sp.ref_plms(x, [torch.tensor([[2.0]]), None, None, None], (1.0, 0, 0, 0), [[0.5, 0.25, 1.0, 0.5, 0.0]], torch.zeros(1, 1), 10.0)
    e, be = r['e']
    assert float(e) == 2.0 and math.isclose(float(be), sp.gamma(4) * 2.0, rel_tol=1e-12)
    x0, b0 = r['x0']
    assert float(x0) == 1.0 and math.isclose(float(b0), sp.gamma(7) * (1 + 0.25 * 2) / 0.5, rel_tol=1e-9)
    r = sp.ref_plms(x, [torch.tensor([[-100.0]]), None, None, None], (1.0, 0, 0, 0), [[0.5, 0.25, 1.0, 0.5, 0.0]], torch.zeros(1, 1), 1.0)
    assert float(r['x0'][0]) == 1.0 and float(r['x0'][1]) == 0.0                              # clamped with margin: exact


# ------------------------------------------------------------------------------------------------ references against torch
def _huber(x, y, s=0.1):
    return ((1 + (x - y) ** 2 / s ** 2).clamp(1e-4).sqrt() - 1) * s


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


@pytest.mark.parametrize('hw', [(16, 16), (37, 53)])
def test_photometric_reference_matches_autograd(hw):
    h, w = hw
    n = h * w
    img, sil, rgb = rand(n, 3), rand(n), rand(3, 2 * h, 2 * w)
    mask = (rand(1, 2 * h, 2 * w) > 0.5).float()
    lc, ls, lo = 1.0, 0.7, 1e-3
    r = sp.ref_photometric(img, sil, rgb, mask, h, w, 2, lc, ls, lo, sp.kernel_plan('photometric_loss', dict(h=h, w=w)))
    a, b = img.double().requires_grad_(True), sil.double().requires_grad_(True)
    image, s = a.reshape(1, h, w, 3).permute(0, 3, 1, 2), b.reshape(1, 1, h, w)
    c_ = _huber(image, F.interpolate(rgb[None].double(), scale_factor=0.5)).mean()
    s_ = _huber(s, F.interpolate(mask[None].double(), scale_factor=0.5)).mean()
    o_ = torch.sqrt(s ** 2 + .01).mean()
    (lc * c_ + ls * s_ + lo * o_).backward()
    assert _rel(r['g_img'][0], a.grad) < 1e-6 and _rel(r['g_sil'][0], b.grad) < 1e-6
    sums = r['sums'][0]
    assert _rel(torch.stack((sums[0] / (3 * n), sums[1] / n, sums[2] / n)), torch.stack((c_, s_, o_)).detach()) < 1e-6


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('hw', [(16, 16), (5, 9)])
def test_fusion_references_match_autograd(mode, hw):
    h, w = hw
    img, sil = rand(h * w, 3), rand(h * w)
    target = rand(3, 2 * h, 2 * w) * 0.3
    ge = rn(3, 2 * h, 2 * w) * 1e-3
    wgt, lc, ls, lo = 0.37, 1.0, 0.7, 1e-3
    up, _ = sp.ref_upsample2x(img, sil, h, w)
    a, b = img.double().requires_grad_(True), sil.double().requires_grad_(True)
    image = F.interpolate(a.reshape(1, h, w, 3).permute(0, 3, 1, 2), scale_factor=2, mode='bilinear')
    s = F.interpolate(b.reshape(1, 1, h, w), scale_factor=2, mode='bilinear')
    assert _rel(up[:3], image[0].detach()) < 1e-12 and _rel(up[3], s[0, 0].detach()) < 1e-12
    t = target[None].double()
    fl = wgt * (image - t).abs().mean() if mode == 0 else \
        lc * _huber(image, t).mean() + ls * _huber(s, (t.mean(dim=1, keepdim=True) > .1).double()).mean()
    (fl + lo * torch.sqrt(s ** 2 + .01).mean() + (image[0] * ge.double()).sum()).backward()     # g_extra: the perceptual term's gradient
    r = sp.ref_fusion(up.float(), target, mode, wgt, lc, ls, lo, ge, sp.kernel_plan('fusion_loss', dict(h=h, w=w)))
    (gi, _), (gs, _) = sp.ref_fusion_adjoint(r['g_up'][0], h, w)
    assert _rel(gi, a.grad) < 1e-6 and _rel(gs, b.grad) < 1e-6


def test_fusion_mask_is_torch_mean():
    t = rand(3, 64, 64) * 0.3
    assert torch.equal(sp.fusion_mask(t).bool(), t.mean(dim=0) > 0.1)


def test_eft_references_match_torch():
    x = rn(2, 5, 7, 8)
    y, _ = sp.ref_resize(x, 16, 11)
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), (16, 11), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    assert (y - ref).abs().max() < 1e-5                      # the fp32 source positions: an ulp of the position times the slope
    x = rn(2, 9, 11, 7)
    grid = rand(2, 300, 2) * 2.6 - 1.3
    y, _ = sp.ref_grid_sample(x, grid)
    ref = F.grid_sample(x.double().permute(0, 3, 1, 2), grid.double()[:, :, None], mode='bilinear', padding_mode='border',
                        align_corners=True)[..., 0].permute(0, 2, 1)
    assert (y - ref).abs().max() < 1e-5
    x = rn(2, 17, 22, 8)
    assert torch.equal(sp.maxpool3x3s2(x), F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1))
    x[0, 3, 4, 1] = math.nan
    assert torch.equal(torch.isnan(sp.maxpool3x3s2(x)), torch.isnan(F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)))
    v = torch.tensor([math.nan, -1.0, 0.0, 2.0, -math.inf])
    assert torch.equal(torch.isnan(sp.relu(v)), torch.isnan(F.relu(v))) and torch.equal(sp.relu(v)[1:], F.relu(v)[1:])
    xg = rn(4000) * 3
    yg, bg = sp.ref_gelu(xg)
    assert ((yg - F.gelu(xg.double())).abs() <= bg).all()
    for S, B, E in ((2, 30, 256), (20, 6, 132), (1, 3, 4)):
        qkv = rn(S, B, 3 * E)
        y, _ = sp.ref_seq_attention(qkv, S, B, E)
        mha = torch.nn.MultiheadAttention(E, 1, bias=False).double()
        with torch.no_grad():
            mha.in_proj_weight.copy_(torch.eye(E).repeat(3, 1))
            mha.out_proj.weight.copy_(torch.eye(E))
        q, k, v = qkv.double().split(E, dim=-1)
        qkv_in = torch.cat((q, k, v), -1)
        # with identity projections MHA computes softmax(q k^T / sqrt(E)) v; feed q, k, v through the three identity blocks
        ref, _ = mha(qkv_in[..., :E], qkv_in[..., E:2 * E], qkv_in[..., 2 * E:], need_weights=False)
        assert (y - ref).abs().max() < 1e-6, (S, B, E)


# ------------------------------------------------------------------------------------------------ defect-free emulations pass, defects are rejected
def _plms_case(rows=3, L=500):
    x, noise = rn(rows, L), rn(rows, L)
    eps = [rn(rows, L) * 0.7 for _ in range(4)]
    r = torch.arange(rows, dtype=torch.float64)
    al = 0.3 + 0.6 * (r + 1) / (rows + 1)
    sc = torch.stack((al, torch.sqrt(1 - al * al), al + 0.05, 0.2 + 0.1 * r / rows, 0.05 + 0.01 * r), 1).float()
    return x, eps, (55 / 24, -59 / 24, 37 / 24, -9 / 24), sc, noise


def _plms_ok(defect, clip=1.0, scalars=None, nan=False):
    x, eps, cf, sc, noise = _plms_case()
    if scalars is not None:
        sc = torch.tensor(scalars, dtype=torch.float32).expand(3, 5).contiguous()
    if nan:
        eps[0][0, ::7] = math.nan
    ref = sp.ref_plms(x, eps, cf, sc, noise, clip)
    got = sp.emulate_plms(x, eps, cf, sc, noise, clip, defect)
    return all(sp.passes(got[k], *ref[k]) for k in ('e', 'x0', 'x_prev'))


def test_plms_emulation_and_defects():
    assert _plms_ok(None) and _plms_ok(None, nan=True) and _plms_ok(None, math.inf, (1e-10, 0.6, 0.9, 0.3, 0.1))
    assert not _plms_ok('e1_e2_swap')
    assert not _plms_ok('row_shift')
    assert not _plms_ok('no_alpha_clamp', math.inf, (1e-10, 0.6, 0.9, 0.3, 0.1))
    assert not _plms_ok('clamp_drops_nan', nan=True)


def test_cfg_eps_rounds_three_times():
    """cfg_eps against numpy's fp32 scalar arithmetic, one correctly rounded operation at a time: (e_cond - e_null), the product with the
    scale and the add each round once, as __fsub_rn / __fmul_rn / __fadd_rn do; contracting the product into the add (an fma) is caught"""
    ec, en = rn(1000), rn(1000)
    f = np.float32
    want = torch.tensor([f(b) + f(f(a) - f(b)) * f(3.0) for a, b in zip(ec.tolist(), en.tolist())])
    e = sp.cfg_eps(ec, en, 3.0)
    assert torch.equal(e, want)
    d = (ec - en).double()
    fma = (en.double() + d * 3.0).float()              # the product kept exact, one rounding for product and add
    assert not torch.equal(fma, want)


def test_dynamic_x_prev_bound_sees_a_wrong_s():
    x, e = rn(2, 4096) * 2, rn(2, 4096)
    x0, b0 = sp.dyn_x0(x, e, None, 1.0, 0.8, 0.6)
    s = sp.quantile_s(x0.float(), 0.95)
    noise = rn(2, 4096)
    y, b = sp.ref_dyn_x_prev(x, x0, b0, s, 0.8, 0.9, 0.3, 0.1, noise)
    x0c = torch.maximum(torch.minimum(x0.float(), s.float()[:, None]), -s.float()[:, None]) / s.float()[:, None]
    got = 0.9 * (x.float() * (1 - 0.3) / 0.8 + 0.3 * x0c) + 0.1 * noise
    assert sp.passes(got, y, b)
    y2, _ = sp.ref_dyn_x_prev(x, x0, b0, s * (1 + 1e-4), 0.8, 0.9, 0.3, 0.1, noise)
    assert not sp.passes(y2, y, b)


@pytest.mark.parametrize('defect', ['hw_swap', 'nearest_off_by_one'])
def test_photometric_defects(defect):
    h, w = 37, 53
    img, sil, rgb = rand(h * w, 3), rand(h * w), rand(3, 2 * h, 2 * w)
    mask = (rand(1, 2 * h, 2 * w) > 0.5).float()
    plan = sp.kernel_plan('photometric_loss', dict(h=h, w=w))
    ref = sp.ref_photometric(img, sil, rgb, mask, h, w, 2, 1.0, 0.7, 1e-3, plan)
    # defect-free fp32 evaluation
    tgt = sp.glue_nearest(rgb, h, w, 2).reshape(3, -1).t()
    d = img - tgt
    gi = 1.0 * (d / (sp.HUBER_S * torch.sqrt(1 + d * d / sp.HUBER_S2))) / (3 * h * w)
    assert sp.passes(gi, *ref['g_img'])
    bad = sp.ref_photometric(img, sil, rgb, mask, h, w, 2, 1.0, 0.7, 1e-3, plan, defect)
    assert not sp.passes(bad['g_img'][0].float(), *ref['g_img'])


def test_fusion_defects():
    h, w = 6, 9
    H, W = 2 * h, 2 * w
    up = rand(4, H, W)
    target = torch.zeros(3, H, W)
    t0 = [np.float32(0.1) * np.float32(3)]
    while np.float32(t0[0] / np.float32(3)) != np.float32(0.1):
        t0[0] = np.nextafter(t0[0], np.float32(1) if np.float32(t0[0] / np.float32(3)) < np.float32(0.1) else np.float32(0))
    target[0] = float(t0[0])                                                   # every channel mean exactly 0.1f
    ge = rn(3, H, W) * 1e-3
    plan = sp.kernel_plan('fusion_loss', dict(h=h, w=w))
    ref = sp.ref_fusion(up, target, 1, 0.37, 1.0, 0.7, 1e-3, ge, plan)
    for defect in ('mask_ge', 'g_extra_on_sil'):
        bad = sp.ref_fusion(up, target, 1, 0.37, 1.0, 0.7, 1e-3, ge, plan, defect)
        assert not sp.passes(bad['g_up'][0].float(), *ref['g_up']), defect
    g_up = ref['g_up'][0].float()
    (gi, gib), (gs, gsb) = sp.ref_fusion_adjoint(g_up, h, w)
    ei, es = sp.emulate_fusion_adjoint(g_up, h, w)
    assert sp.passes(ei, gi, gib) and sp.passes(es, gs, gsb)
    ei, es = sp.emulate_fusion_adjoint(g_up, h, w, 'adjoint_no_edge_clamp')
    assert not (sp.passes(ei, gi, gib) and sp.passes(es, gs, gsb))


def test_eft_defects():
    x = rn(2, 9, 7, 4)
    ref = sp.maxpool3x3s2(x)
    fp32 = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert sp.passes(fp32, ref, None)                                          # the GPU suite's exact, NaN-aware comparison
    assert not sp.passes(sp.maxpool3x3s2(x, 'window_shift'), ref, None)
    x = rn(1, 5, 9, 4)
    y, b = sp.ref_resize(x, 13, 17)
    fp32 = F.interpolate(x.permute(0, 3, 1, 2), (13, 17), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    assert sp.passes(fp32, y, b)
    assert not sp.passes(sp.ref_resize(x, 13, 17, 'xy_swap')[0].float(), y, b)
    x = rn(2, 9, 11, 7)
    grid = rand(2, 300, 2) * 2.6 - 1.3
    y, b = sp.ref_grid_sample(x, grid)
    fp32 = F.grid_sample(x.permute(0, 3, 1, 2), grid[:, :, None], mode='bilinear', padding_mode='border', align_corners=True)[..., 0].permute(0, 2, 1)
    assert sp.passes(fp32, y, b)
    for defect in ('align_false', 'zeros_pad'):
        assert not sp.passes(sp.ref_grid_sample(x, grid, defect)[0].float(), y, b), defect
    S, B, E = 20, 6, 132
    qkv = rn(S, B, 3 * E)
    y, b = sp.ref_seq_attention(qkv, S, B, E)
    q, k, v = (t.permute(1, 0, 2) for t in qkv.split(E, dim=-1))
    fp32 = (torch.softmax(q @ k.transpose(1, 2) * sp.seq_scale(E), dim=-1) @ v).permute(1, 0, 2)
    assert sp.passes(fp32, y, b)
    for defect in ('scale_1_over_E', 'softmax_over_batch'):
        assert not sp.passes(sp.ref_seq_attention(qkv, S, B, E, defect)[0].float(), y, b), defect


# ------------------------------------------------------------------------------------------------ catalogue entries of recorded launches
def _call(name, *args, family='Distill'):
    """an oracle/insitu ``Call``: positional C ABI arguments bound to the header's parameter names, as the recorder binds them"""
    return insitu.Call(name, dict(zip(insitu.c_params()[name], args)), family)


def test_entry_reads_sampler_calls_by_parameter_name():
    # x, e0, e1, e2, e3, c0..c3, noise, alpha, sigma, alpha_next, c, noise_scale, clip, x_prev, x0_out, e_out, n, stream
    e = sp.entry(_call('sfb_plms_update', 1, 2, None, 4, None, 0.5, 1.5, 2.5, 3.5, 10, 0.8, 0.6, 0.9, 0.3, 0.1, 7.0, 20, None, 22, 4096, 0,
                       family='DDPM'))
    assert e == dict(n=4096, nulls=(True, False, True), coefs=(0.5, 1.5, 2.5, 3.5), scalars=(0.8, 0.6, 0.9, 0.3, 0.1), clip=7.0,
                     x0_out=False, e_out=True, op='plms_update', family='DDPM', label='recorded')
    # x, e_cond, e_null, cond_scale, e1, e2, e3, c0..c3, noise, row_scalars (copied at call time), clip, x_prev, e_out, rows, row_len, stream
    table = torch.arange(10, dtype=torch.float32) / 16
    e = sp.entry(_call('sfb_plms_update_rows_cfg', 1, 2, 3, 3.0, 5, None, None, 0.5, 1.5, 2.5, 3.5, 12, table, 1.0, 15, None, 2, 8192, 0,
                       family='PLMS'))
    assert e == dict(rows=2, row_len=8192, nulls=(False, True, True), coefs=(0.5, 1.5, 2.5, 3.5), cond_scale=3.0, clip=1.0, e_out=False,
                     row_scalars=tuple(table.tolist()), op='plms_update_rows_cfg', family='PLMS', label='recorded')
    # x, e_cond, e_null, cond_scale, noise, alpha, sigma, alpha_next, c, noise_scale, percentile, row_len, B, x_prev, s_out, x0_out, stream
    e = sp.entry(_call('sfb_ddpm_dynamic_step', 1, 2, None, 1.0, 5, 0.8, 0.6, 0.9, 0.3, 0.1, 0.95, 65536, 2, 14, 15, None, 0))
    assert (e['B'], e['row_len'], e['guided'], e['p'], e['s_out'], e['x0_out']) == (2, 65536, False, 0.95, True, False)


def test_entry_reads_glue_and_eft_calls_by_parameter_name():
    # up, target, H, W, mode, weight, lambda_color, lambda_sil, lambda_opacity, g_extra, sums, g_up, h, w, g_img, g_sil, stream
    e = sp.entry(_call('sfb_fusion_loss_ex', 1, 2, 128, 96, 1, 0.25, 1.0, 0.5, 0.125, None, 11, 12, 64, 48, 15, 16, 0))
    assert e == dict(h=64, w=48, mode=1, g_extra=False, wgt=0.25, lam=(1.0, 0.5, 0.125), op='fusion_loss', family='Distill', label='recorded')
    # x, ldx, y, ldo, NB, H, W, C, Ho, Wo, stream
    e = sp.entry(_call('sfb_resize_bilinear_ac_nhwc', 1, 12, 3, 20, 2, 5, 7, 8, 16, 9, 0, family='EFT'))
    assert e == dict(NB=2, H=5, W=7, C=8, Ho=16, Wo=9, ldx=12, ldo=20, op='resize', family='EFT', label='recorded')
    # x, ldx, grid, out, ldo, NB, H, W, C, M, stream
    e = sp.entry(_call('sfb_grid_sample_nhwc', 1, 64, 3, 4, 70, 1, 6, 5, 60, 33, 0, family='EFT'))
    assert e == dict(NB=1, H=6, W=5, C=60, M=33, ldx=64, ldo=70, op='grid_sample', family='EFT', label='recorded')
    assert sp.entry(_call('sfb_relu_nhwc', 1, 64, 0)) is None
    assert sp.entry(insitu.Rec('groupnorm', {}, (), {})) is None
