"""Host checks of the shading oracle (oracle/normal_fp64.py) and of NeRFNetwork's shading dispatch: the numpy Philox4x32-10 against the
published Random123 known-answer vectors, the fp64 stencil and its backward against a direct torch-autograd restatement of
network_grid.py:91-164, and the sensitivity of the oracle's bounds to single defects of the stencil."""
import numpy as np
import pytest
import torch

from oracle import field_fp64 as f64
from oracle import ngp_oracle as no
from oracle import normal_fp64 as nf

BOUND = 4.0
GEO = no.live_geometry(BOUND)


def _scales():
    return no.level_scales_host(16, GEO['S'], 16)


def test_philox_known_answers():
    """Random123 kat_vectors, philox4x32 with 10 rounds"""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = nf.philox4x32_10(np.array([ctr], np.uint32), key)[0]
        assert tuple(int(v) for v in got) == want, (ctr, [hex(int(v)) for v in got])


def test_jitter_range_and_key_split():
    j = nf.jitter(50, 6, 10, -1234567890123, 0.3)
    assert j.dtype == np.float32 and j.shape == (50, 6, 10, 3)
    assert (j >= np.float32(-0.3)).all() and (j < np.float32(0.3)).all()
    assert nf.key_words(-1) == (0xFFFFFFFF, 0xFFFFFFFF) and nf.key_words(1 << 32) == (0, 1)


def _points(B, seed, near_face=True):
    rng = np.random.default_rng(seed)
    x = ((rng.random((B, 3), dtype=np.float32) * 2 - 1) * 0.9 * BOUND).astype(np.float32)
    if near_face:        # within eps of a face: the clamp of the shifted point engages
        x[:4, 0] = np.float32(BOUND - 0.004)
        x[4:8, 1] = np.float32(-BOUND + 0.002)
    return x


def test_stencil_and_backward_match_autograd_restatement():
    params = no.make_field_params(seed=3)
    x = _points(24, 0)
    g = torch.from_numpy(np.random.default_rng(1).standard_normal((24, 3)))
    want = nf.reference_autograd(params, x, _scales(), g)
    st = nf.StencilFP64(params, x, _scales())
    torch.testing.assert_close(st.fd, want['fd'], rtol=1e-12, atol=1e-12)
    n, _ = st.normal()
    torch.testing.assert_close(n, want['normal'], rtol=1e-12, atol=1e-12)
    got = st.backward(st.fd, g_normal=g)
    for k in no.PARAM_KEYS:
        torch.testing.assert_close(got[k], want[k], rtol=1e-9, atol=1e-12, msg=k)


def _outside(defect: nf.StencilFP64, clean: nf.StencilFP64):
    """some fd element of the defective stencil lies outside the clean oracle's per-element bound"""
    return bool(f64.violations(defect.fd, clean.fd, clean.fd_abs, clean.rtol()).any())


@pytest.mark.parametrize('defect', [dict(drop_slot=3), dict(flip_slot=4)])
def test_plain_stencil_defects_are_seen(defect):
    params = no.make_field_params(seed=3)
    x = _points(32, 2)
    clean = nf.StencilFP64(params, x, _scales())
    assert not _outside(clean, clean)
    assert _outside(nf.StencilFP64(params, x, _scales(), **defect), clean)


@pytest.mark.parametrize('defect', [dict(blob_at_jitter=True), dict(clamp_after_jitter=True)])
def test_smoothed_stencil_defects_are_seen(defect):
    params = no.make_field_params(seed=4)
    rng = np.random.default_rng(5)
    x = ((rng.random((32, 3), dtype=np.float32) * 2 - 1) * 0.2).astype(np.float32)     # near the blob: its gradient is large there
    x[16:, 0] = np.float32(BOUND - 0.1)                                                 # the +-0.3 jitter leaves the box here
    kw = dict(k=10, eps=0.3, radius=0.3, key=0x1234_5678_9abc_def0)
    clean = nf.StencilFP64(params, x, _scales(), **kw)
    assert _outside(nf.StencilFP64(params, x, _scales(), **kw, **defect), clean)


def _net_cpu():
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    return NeRFNetwork(get_default_torch_ngp_opt())


def test_unknown_shading_is_lambertian():
    net = _net_cpu()
    seen = []
    albedo = torch.full((5, 3), 0.5)
    net.common_forward = lambda x: (torch.ones(5), albedo)

    def fake_normal(x, smooth=False):
        seen.append(smooth)
        return torch.tensor([[0.0, 0.0, -1.0]]).expand(5, 3)
    net.normal = fake_normal
    l = torch.tensor([0.75 ** 0.5, 0.0, 0.5])                     # n . (-l) = 0.5: lam = 0.25 + 0.75 * 0.5 = 0.625
    sigma, color, normal = net(torch.zeros(5, 3), None, l, ratio=0.25, shading='shiny')
    assert seen == [False]
    torch.testing.assert_close(color, albedo * 0.625)
    _, color, _ = net(torch.zeros(5, 3), None, l, ratio=0.25, shading='textureless')
    assert seen[-1] is True
    torch.testing.assert_close(color, torch.full((5, 3), 0.625 * 0.8 + 0.2))
    _, color, _ = net(torch.zeros(5, 3), None, l, ratio=0.25, shading='normal')
    torch.testing.assert_close(color, torch.tensor([[0.5, 0.5, 0.0]]).expand(5, 3))
    _, color, _ = net(torch.zeros(5, 3), None, -l, ratio=0.25, shading='lambertian')
    torch.testing.assert_close(color, albedo * 0.25)                # light from behind: the clamp leaves the ambient term only
    _, _, normal = net(torch.zeros(5, 3), None, l, shading='albedo')
    assert normal is None


def test_run_still_refuses_background_net_and_other_step_counts():
    net = _net_cpu()
    rays = torch.zeros(1, 4, 3)
    with pytest.raises(NotImplementedError):
        net.run(rays, rays, num_steps=32, upsample_steps=64, shading='normal')
    net.bg_radius = 1.0
    with pytest.raises(NotImplementedError):
        net.run(rays, rays, num_steps=64, upsample_steps=64, shading='lambertian')
