"""The fp64 references of oracle/grid_march_fp64.py checked on the CPU against the C restatement (oracle/ngp_oracle.c) of the grid
encoder, the compositing operators and sph_from_ray, within their derived bounds -- and negative controls: each single defect below,
applied to an otherwise exact result, must be rejected by the same per-element comparison the GPU tests make."""
import itertools

import numpy as np
import pytest
import torch

from oracle import grid_march_fp64 as gm
from oracle import ngp_oracle as no

VARIANTS = list(itertools.product((1, 2, 3, 4, 5), (1, 2, 4, 8), (0, 1), (False, True)))


def _grid(D, C, gridtype, ac, B=64, seed=0):
    offsets, S, H = gm.grid_case(D, ac)
    scales = no.level_scales_host(len(offsets) - 1, S, H)
    x = gm.grid_points(B, D, scales, seed)
    emb = gm.grid_embeddings(int(offsets[-1]), C, seed + 1)
    return offsets, S, H, scales, x, emb


@pytest.mark.parametrize('D,C,gridtype,ac', VARIANTS)
def test_grid_reference_vs_c_restatement(D, C, gridtype, ac):
    offsets, S, H, scales, x, emb = _grid(D, C, gridtype, ac)
    out, dy, rows = no.grid_encode_forward(x.numpy(), emb.numpy(), offsets, S, H, gridtype, ac, True, scales, want_rows=True)
    ref = gm.GridFP64(x, emb, offsets, scales, gridtype, ac)
    f = ref.forward()
    assert np.array_equal(f['rows'].numpy(), rows), 'corner rows differ from the C restatement'
    rt = ref.rt
    gm.assert_within('out', torch.from_numpy(out), f['out'], f['out_abs'], rt['out'])
    gm.assert_within('dy_dx', torch.from_numpy(dy).view(f['dy'].shape), f['dy'], f['dy_abs'], rt['dy'])
    dead = ~ref.live
    assert dead.sum() > 0 and (torch.from_numpy(out)[:, dead] == 0).all() and (torch.from_numpy(dy)[dead] == 0).all()
    grad = torch.from_numpy(np.random.default_rng(2).standard_normal(out.shape).astype(np.float32))
    ge, gi = no.grid_encode_backward(grad.numpy(), x.numpy(), offsets, int(offsets[-1]), S, H, gridtype, ac, dy, scales)
    b = ref.backward(grad, torch.from_numpy(dy), f['dy_abs'])
    gm.assert_within('grad_embeddings', torch.from_numpy(ge), b['ge'], b['ge_abs'], b['ge_rtol'])
    gm.assert_within('grad_inputs', torch.from_numpy(gi), b['gi'], b['gi_abs'], rt['gi'])
    # both levels kinds present: dense tiled levels and levels past the hashmap cap
    dense = [(int(np.ceil(p[2])) + 1 + (0 if ac else 1)) ** D for p in ref.plan]
    capped = [p[1] < n for p, n in zip(ref.plan, dense)]
    assert not all(capped) and any(capped)
    assert any(p[4] for p in ref.plan) == (gridtype == 0)


@pytest.fixture(scope='module')
def grid3():
    offsets, S, H, scales, x, emb = _grid(3, 2, 0, False, B=512)
    ref = gm.GridFP64(x, emb, offsets, scales, 0, False)
    f = ref.forward()
    grad = torch.from_numpy(np.random.default_rng(2).standard_normal(f['out'].shape).astype(np.float32))
    return dict(offsets=offsets, scales=scales, x=x, emb=emb, ref=ref, f=f, grad=grad, b=ref.backward(grad))


def _fwd_rejected(c, **defect):
    bad = gm.GridFP64(c['x'], c['emb'], c['offsets'], c['scales'], 0, False, **defect).forward()
    f, rt = c['f'], c['ref'].rt
    return bool(gm.violations(bad['out'], f['out'], f['out_abs'], rt['out']).any()), \
        bool(gm.violations(bad['dy'], f['dy'], f['dy_abs'], rt['dy']).any())


def _interior(c, level):
    """a live point whose frac is well inside (0.1, 0.9) in every dimension on `level`"""
    _, frac = gm.grid_locate(c['x'], c['ref'].plan[level][2], False)
    ok = ((frac > 0.1) & (frac < 0.9)).all(1) & c['ref'].live
    return int(torch.nonzero(ok)[3])


def test_negative_control_one_corner_dropped(grid3):
    for level in (0, 4):
        assert _fwd_rejected(grid3, drop_corner=(_interior(grid3, level), level, 5))[0]


def test_negative_control_frac_swapped_in_one_dimension(grid3):
    for d in range(3):
        assert all(_fwd_rejected(grid3, swap_dim=d))


def test_negative_control_tiled_and_hash_rows_swapped_on_one_level(grid3):
    for level in (0, 1, 3):
        assert _fwd_rejected(grid3, swap_level=level)[0], level


def test_negative_control_dy_dx_sign_flipped(grid3):
    b = _interior(grid3, 2)
    f = grid3['f']
    assert f['dy'][b, 2, 1, 0].abs() > 1e-3
    assert _fwd_rejected(grid3, flip_dy=(b, 2, 1, 0))[1]


def test_negative_control_one_lost_scatter(grid3):
    """one scatter of weight > 0.05 left out of the row of the finest level that the fewest points hit"""
    c = grid3
    b = c['b']
    rows4, w4 = c['ref']._level(4, 0, c['x'].shape[0])[:2]
    big = (w4 > 0.05) & (c['grad'][4].abs().min(1).values > 0.1)[:, None] & c['ref'].live[:, None]
    hits = torch.where(big, b['hits'][rows4], torch.full_like(w4, 1e9))
    pt, corner = divmod(int(torch.argmin(hits)), w4.shape[1])
    assert hits[pt, corner] <= 32
    bad = c['ref'].backward(c['grad'], drop_scatter=(pt, 4, corner))
    assert gm.violations(bad['ge'], b['ge'], b['ge_abs'], b['ge_rtol']).any()


# ------------------------------------------------------------------------------------------------ compositing
def _rays(N=400, T=300, seed=0):
    """padded rays with the edge samples: sigma 0, sigma delta >= 104 (alpha = 1 in fp32), delta 0, and rays of 0 and 1 samples"""
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, T + 1, (N,), generator=g)
    counts[:8] = torch.tensor([0, 1, 1, 2, 0, 1, T, T])
    s = torch.rand(N, T, generator=g) * 30
    s[torch.rand(N, T, generator=g) < 0.1] = 0
    s[torch.rand(N, T, generator=g) < 0.01] = 5000
    dl = torch.stack([torch.rand(N, T, generator=g) * 0.05, torch.rand(N, T, generator=g) * 0.05], -1)
    dl[torch.rand(N, T, generator=g) < 0.02, 0] = 0
    s[9, :] = 0
    c = torch.rand(N, T, 3, generator=g)
    return s.float(), c.float(), dl.float(), counts


def _pack(s, c, dl, counts):
    """padded -> the operators' flat layout with a rays table in ray order"""
    N, T = s.shape
    valid = torch.arange(T)[None] < counts[:, None]
    off = torch.cumsum(counts, 0) - counts
    rays = torch.stack([torch.arange(N), off, counts], 1).int()
    return s[valid].contiguous(), c[valid].contiguous(), dl[valid].contiguous(), rays


@pytest.mark.parametrize('thr', (0.0, 1e-4, 1e-2, 1.0))
def test_train_composite_reference_vs_c_restatement(thr):
    s, c, dl, counts = _rays()
    sf, cf, df, rays = _pack(s, c, dl, counts)
    ws, dp, im = no.composite_rays_train_forward(sf.numpy(), cf.numpy(), df.numpy(), rays.numpy(), thr)
    g = torch.Generator().manual_seed(7)
    gws, gim = torch.randn(s.shape[0], generator=g), torch.randn(s.shape[0], 3, generator=g)
    gs, gc = no.composite_rays_train_backward(gws.numpy(), gim.numpy(), sf.numpy(), cf.numpy(), df.numpy(), rays.numpy(), ws, im, thr)
    ref = gm.composite_train_fp64(s, c, dl, counts, thr, gws, gim)
    # where fp64 stops at another step than fp32, the transmittance is within its bound of the threshold there
    assert (ref['ambiguous'] | (ref['K64'] == ref['K32'])).all()
    ok = ~ref['ambiguous']
    assert ok.float().mean() > 0.95
    for name, got in (('ws', ws), ('depth', dp), ('image', im)):
        got = torch.from_numpy(got)[ok]
        gm.assert_within(name, got, ref[name][ok], 0, 0, ref[name + '_err'][ok])
    valid = torch.arange(s.shape[1])[None] < counts[:, None]
    gsp, gcp = torch.zeros(s.shape, dtype=torch.float32), torch.zeros(c.shape, dtype=torch.float32)
    gsp[valid], gcp[valid] = torch.from_numpy(gs), torch.from_numpy(gc)
    gm.assert_within('grad_sigmas', gsp[ok], ref['g_sigma'][ok], 0, 0, ref['g_sigma_err'][ok])
    gm.assert_within('grad_rgbs', gcp[ok], ref['g_rgb'][ok], 0, 0, ref['g_rgb_err'][ok])


def test_negative_control_termination_one_step_late():
    s, c, dl, counts = _rays(seed=3)
    ref = gm.composite_train_fp64(s, c, dl, counts, 1e-2)
    late = gm.composite_train_fp64(s, c, dl, counts, 1e-2, K=torch.minimum(ref['K'] + 1, counts))
    moved = (late['K'] != ref['K']) & ~ref['ambiguous']
    assert moved.sum() > 10
    assert gm.violations(late['ws'][moved], ref['ws'][moved], 0, 0, ref['ws_err'][moved]).any()
    assert gm.violations(late['image'][moved], ref['image'][moved], 0, 0, ref['image_err'][moved]).any()


def test_closed_form_equals_autograd_and_the_ws_term_is_needed():
    s, c, dl, counts = _rays(seed=4)
    g = torch.Generator().manual_seed(8)
    gws, gim = torch.rand(s.shape[0], generator=g) + 0.5, torch.randn(s.shape[0], 3, generator=g)
    ref = gm.composite_train_fp64(s, c, dl, counts, 1e-4, gws, gim)
    closed = gm.closed_form_train_backward(ref, c, dl, gws, gim)
    gm.assert_within('closed form', closed, ref['g_sigma'], 0, 0, ref['g_sigma_err'])
    bad = gm.closed_form_train_backward(ref, c, dl, gws, gim, drop_ws_term=True)
    assert gm.violations(bad, ref['g_sigma'], 0, 0, ref['g_sigma_err']).any()


@pytest.mark.parametrize('thr', (0.0, 1e-4, 1e-2, 1.0))
def test_inference_composite_reference_vs_c_restatement(thr):
    g = torch.Generator().manual_seed(5)
    n, S = 300, 8
    s, c, dl, _ = _rays(n, S, seed=6)
    dl[:20, 3:] = 0                                                      # rays whose march ended
    ws0 = (torch.rand(n, generator=g) * 0.9).float()
    ws0[:50] = 0
    d0, img0, t0 = torch.rand(n, generator=g), torch.rand(n, 3, generator=g) * 0.5, torch.rand(n, generator=g) * 3
    alive = np.arange(n, dtype=np.int32)
    rt, wsa, dpa, ima = t0.numpy().copy(), ws0.numpy().copy(), d0.numpy().copy(), img0.numpy().copy()
    no.composite_rays(n, S, alive, rt, s.numpy(), c.numpy(), dl.reshape(-1, 2).numpy(), wsa, dpa, ima, thr)
    ref = gm.composite_inference_fp64(s, c, dl, ws0, d0, img0, t0, thr)
    ok = ~ref['ambiguous']
    assert ok.float().mean() > 0.95
    assert np.array_equal((alive >= 0)[ok.numpy()], ref['alive'][ok].numpy())
    for name, got in (('ws', wsa), ('depth', dpa), ('image', ima)):
        gm.assert_within(name, torch.from_numpy(got)[ok], ref[name][ok], 0, 0, ref[name + '_err'][ok])


def test_sph_from_ray_reference_vs_c_restatement():
    g = torch.Generator().manual_seed(9)
    o = (torch.rand(2000, 3, generator=g) * 2 - 1).float()
    d = (torch.randn(2000, 3, generator=g)).float()
    d[:10, 0] = 0
    d[10:20, :2] = 0
    got = torch.from_numpy(no.sph_from_ray(o.numpy(), d.numpy(), 3.0))
    ref, err = gm.sph_from_ray_fp64(o, d, 3.0)
    gm.assert_within('sph_from_ray', got, ref, 0, 0, err)
