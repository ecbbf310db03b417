"""The fp64 restatement of the fused NGP field (oracle/field_fp64.py) checked on the CPU: its encoding against the C oracle's fp32
grid encoder, its hand-written backward against fp64 autograd, its values and gradients against the fp32 autograd restatement
(ngp_oracle.Field) -- and sensitivity self-checks.  Each self-check injects one defect into the reference and asserts, tensor by
tensor and with each kernel path's own bounds, that the per-element comparison of the GPU tests rejects it.  What is and is not
visible, stated plainly:
  * a lost 64-point tile: every weight, bias and embedding gradient, every path (B = 20 000);
  * the lost 32-point partial last tile of B = 20 000: the embedding gradient, dW1, db1 and db2 on every path (dW0, db0 and dW2 carry
    32 / 20 000 of their sums there, at the edge of the v1 wgmma path's summation bound);
  * a lost point: every weight, bias and embedding gradient at B = 1 000; at B = 20 000 the embedding gradient only -- one point is
    5e-5 of a 20 000-point sum, below the summation bounds;
  * a lost level of one point: the embedding gradient, the only tensor the scatter writes;
  * a flipped ReLU mask: the gradients of that layer's weights and biases and the embedding gradient.
Upstream gradients are one-signed (field_fp64.upstream_grads): zero-mean ones make the sums over points cancel far below any
worst-case summation bound."""
import numpy as np
import pytest
import torch

from oracle import field_fp64 as f64
from oracle import ngp_oracle as no

SM = 132      # H100 SXM: the CTA counts the tolerances are derived for
PATHS = ('v2', 'v1-simt', 'v1-tc')
W_KEYS = no.PARAM_KEYS[1:]
E_KEY = 'encoder.embeddings'


def _make_case(B):
    geo = no.live_geometry()
    scales = no.level_scales_host(geo['L'], geo['S'], geo['H'])
    p = no.make_field_params(seed=0)
    rng = np.random.default_rng(3)
    x = ((rng.random((B, 3), dtype=np.float32) * 2 - 1) * 4).astype(np.float32)
    x[:200] *= 0.05                                     # inside the density blob
    x[200:210] = 4.0                                    # on the box boundary
    x[210:220] = -4.0
    x[220:230] *= 1.1                                   # some outside the box
    ref = f64.FieldFP64(p, torch.from_numpy(x), scales)
    fwd = ref.forward()
    gs, gc = f64.upstream_grads(B, fwd['sigma'], seed=4)
    return dict(B=B, geo=geo, scales=scales, p=p, x=x, gs=gs, gc=gc, ref=ref, fwd=fwd, bwd=ref.backward(gs, gc))


@pytest.fixture(scope='module')
def case():
    return _make_case(20000)


@pytest.fixture(scope='module')
def case_small():
    return _make_case(1000)


def test_fma_f32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a = torch.from_numpy(rng.random(100000, dtype=np.float32))
    b = torch.from_numpy((rng.random(100000, dtype=np.float32) * 4096).astype(np.float32))
    got = f64.fma_f32(a, b, 0.5)
    # the fp32 result is within half an ulp of the exact a*b + 0.5 (exact in fp64 for these operands)
    exact = a.double() * b.double() + 0.5
    assert ((got.double() - exact).abs() <= torch.nextafter(got, torch.full_like(got, np.inf)).double().sub(got.double()) * 0.5).all()
    # double rounding: a = 2^-12 (1 + 2^-23), b = 2^-12 (1 - 2^-23), so a b = 2^-24 - 2^-70; c = 1 + 2^-23 (odd last bit).  The exact
    # sum 1 + 2^-23 + 2^-24 - 2^-70 rounds to the fp64 value 1 + 2^-23 + 2^-24, exactly halfway between two fp32 values, and
    # ties-to-even would then go up to 1 + 2^-22.  The exact value is below the midpoint: the correct fp32 result is 1 + 2^-23.
    a = torch.tensor([2.0 ** -12 * (1 + 2.0 ** -23)], dtype=torch.float32)
    b = torch.tensor([2.0 ** -12 * (1 - 2.0 ** -23)], dtype=torch.float32)
    c = 1 + 2.0 ** -23
    assert (a.double() * b.double() + c).float().item() == 1 + 2.0 ** -22           # what rounding twice gives
    assert f64.fma_f32(a, b, c).item() == 1 + 2.0 ** -23


def test_encoding_matches_the_fp32_grid_encoder(case):
    ref, geo, B = case['ref'], case['geo'], case['B']
    u = f64.normalized_inputs(torch.from_numpy(case['x']), 4.0).numpy()
    out, _, rows = no.grid_encode_forward(u, case['p']['encoder.embeddings'].numpy(), geo['offsets'], geo['S'], geo['H'], 1, False, False,
                                          case['scales'], want_rows=True)
    want = torch.from_numpy(out).permute(1, 0, 2).reshape(B, -1).double()
    # the oracle rounds 8 fp32 FMAs and 3 weight products per level: 12 roundings of the absolute value
    f64.assert_within('encoding', want, ref.enc, ref.enc_abs, f64.gamma(12))
    assert ((ref.enc == 0) == (want == 0)).all()
    dead = (torch.from_numpy(rows) < 0).permute(1, 0, 2).all(-1).all(-1)
    outside = torch.from_numpy((np.abs(case['x']) > 4).any(1))
    assert outside.sum() > 0 and torch.equal(dead, outside) and (ref.enc[dead] == 0).all()


def test_written_out_backward_equals_autograd(case):
    ref = case['ref']
    ag = ref.autograd_reference(case['gs'], case['gc'])
    assert torch.allclose(ag['sigma'], case['fwd']['sigma'], rtol=1e-13, atol=0)
    assert torch.allclose(ag['rgb'], case['fwd']['rgb'], rtol=1e-13, atol=0)
    for k in no.PARAM_KEYS:
        a, b = ag[k], case['bwd'][k]
        assert ((a - b).abs() <= 1e-11 * case['bwd'][k + '_abs'] + 1e-300).all(), k


def test_restatement_vs_fp32_autograd_oracle(case):
    """the fp32 oracle on the CPU sums its GEMM reductions blockwise; bound its accumulation length by B"""
    bwd, fwd, B = case['bwd'], case['fwd'], case['B']
    params = {k: v.clone().requires_grad_(True) for k, v in case['p'].items()}
    field = no.Field(params, level_scales=case['scales'])
    so, co = field.common_forward(torch.from_numpy(case['x']))
    (so * case['gs']).sum().add((co * case['gc']).sum()).backward()
    f64.assert_within('sigma', so.detach(), fwd['sigma'], fwd['sigma_abs'], f64.RTOL_POINT)
    f64.assert_within('rgb', co.detach(), fwd['rgb'], fwd['rgb_abs'], f64.RTOL_POINT)
    for k in W_KEYS:
        f64.assert_within(k, params[k].grad, bwd[k], bwd[k + '_abs'], f64.RTOL_POINT + f64.gamma(B), bwd[k + '_slack'])
    f64.assert_within('embeddings', params[E_KEY].grad, bwd[E_KEY], bwd[E_KEY + '_abs'], f64.RTOL_POINT + f64.gamma(bwd[E_KEY + '_hits']),
                      bwd[E_KEY + '_slack'])


def _seen_by(c, bad_bwd, path):
    """the tensors in which the GPU tests' comparison (with `path`'s bounds) rejects `bad_bwd` as the kernel's result"""
    ref_bwd = c['bwd']
    rtol_w = f64.wgrad_rtol(path, c['B'], SM)
    seen = {k for k in W_KEYS if f64.violations(bad_bwd[k], ref_bwd[k], ref_bwd[k + '_abs'], rtol_w, ref_bwd[k + '_slack']).any()}
    if f64.violations(bad_bwd[E_KEY], ref_bwd[E_KEY], ref_bwd[E_KEY + '_abs'], f64.RTOL_POINT + f64.gamma(ref_bwd[E_KEY + '_hits']),
                      ref_bwd[E_KEY + '_slack']).any():
        seen.add(E_KEY)
    return seen


def _drop(c, points):
    keep = torch.ones(c['B'], dtype=torch.bool)
    keep[points] = False
    return c['ref'].backward(c['gs'], c['gc'], point_keep=keep)


ALL = set(no.PARAM_KEYS)


@pytest.mark.parametrize('path', PATHS)
def test_reference_passes_its_own_comparison(case, case_small, path):
    assert _seen_by(case, case['bwd'], path) == set()
    assert _seen_by(case_small, case_small['bwd'], path) == set()


@pytest.mark.parametrize('path', PATHS)
def test_sensitivity_one_64_point_tile_removed(case, path):
    for t in (0, 7, 123, 200):
        assert _seen_by(case, _drop(case, slice(t * 64, (t + 1) * 64)), path) == ALL, t
    last = (case['B'] - 1) // 64                                 # 20 000 = 312 * 64 + 32: a 32-point partial tile
    assert _seen_by(case, _drop(case, slice(last * 64, None)), path) >= {E_KEY, 'sigma_net.net.1.weight', 'sigma_net.net.1.bias',
                                                                         'sigma_net.net.2.bias'}


@pytest.mark.parametrize('path', PATHS)
def test_sensitivity_one_point_removed(case, case_small, path):
    for pt in (5, 333, 999):
        assert _seen_by(case_small, _drop(case_small, pt), path) == ALL, pt
    for pt in (5, 4321, 19999):
        assert E_KEY in _seen_by(case, _drop(case, pt), path), pt


def test_sensitivity_one_level_of_one_point(case):
    for pt, lvl in ((7, 0), (999, 8), (15000, 15)):
        bad = case['ref'].backward(case['gs'], case['gc'], drop_level=(pt, lvl))
        for path in PATHS:
            assert E_KEY in _seen_by(case, bad, path), (pt, lvl, path)


@pytest.mark.parametrize('path', PATHS)
def test_sensitivity_one_relu_mask_flipped(case_small, path):
    c = case_small
    ref = c['ref']
    clear = torch.nonzero(~(ref.amb1.any(1) | ref.amb2.any(1)))[:, 0]     # points with no ReLU within the error bound of 0
    for layer, pt in ((1, int(clear[11])), (1, int(clear[500])), (2, int(clear[12])), (2, int(clear[700]))):
        amb = ref.amb1 if layer == 1 else ref.amb2
        mask = ref.mask1 if layer == 1 else ref.mask2
        # the unambiguously active unit of this point that routes the most gradient
        j = int(torch.argmax(torch.where(~amb[pt] & mask[pt], ref.dh[layer][pt].abs(), torch.zeros(64, dtype=torch.float64))))
        seen = _seen_by(c, ref.backward(c['gs'], c['gc'], flip_relu=(layer, pt, j)), path)
        lin = 'sigma_net.net.0' if layer == 1 else 'sigma_net.net.1'
        assert seen >= {lin + '.weight', lin + '.bias', E_KEY}, (layer, pt, j, seen)


def test_sensitivity_of_the_forward(case):
    """a one-point change of sigma or rgb: a point's value from its neighbour, one ulp-scale relative error above the bound"""
    fwd = case['fwd']
    s = fwd['sigma'].clone()
    s[17] = s[18]
    assert f64.violations(s, fwd['sigma'], fwd['sigma_abs'], f64.RTOL_POINT).any()
    s = fwd['sigma'] * (1 + 64 * f64.RTOL_POINT)
    assert f64.violations(s, fwd['sigma'], fwd['sigma_abs'], f64.RTOL_POINT).any()


def test_ambiguous_relus_are_rare(case):
    """the slack that ambiguous ReLUs allow is for a small fraction of the (point, unit) pairs, not for the bulk"""
    ref = case['ref']
    assert int(ref.amb1.sum()) + int(ref.amb2.sum()) < 1e-3 * case['B'] * 128


def test_composite_reference_handles_edge_rays():
    """fp64 compositing: opacity + final transmittance = 1; background enters with 1 - opacity"""
    N = 3
    z = torch.linspace(1, 3, 128).repeat(N, 1)
    sig = torch.rand(N, 128) * 3
    sig[1] = 0
    rgb = torch.rand(N, 128, 3)
    nears, fars = torch.full((N,), 1.0), torch.full((N,), 3.0)
    r = f64.composite(z, sig, rgb, nears, fars, 0.3, torch.ones(N, 3), None, None)
    assert abs(r['weights_sum'][1].item()) < 1e-15 and torch.allclose(r['image'][1], torch.full((3,), 0.3, dtype=torch.float64))
    assert (r['weights_sum'] <= 1).all()
