"""Epipolar Feature Transformer on the sm_90a engine (SURVEY §8f row 4) against tests/golden/eft.npz -- outputs of the REFERENCE's own
EpipolarFeatureTransformer (sparsefusion/eft.py) on the same deterministic weights and inputs -- and its new operators against torch.
Bar: 1e-3 relative L2 (BASELINE.json north_star tolerance for floating-point outputs)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm()).item()


def _model():
    from oracle import eft_oracle as eo
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    m = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=False)
    m.load_state_dict(eo.make_params({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0), strict=True)
    return m.cuda()


def test_eft_vs_reference_golden(golden_dir):
    from oracle import eft_oracle as eo
    g = np.load(f'{golden_dir}/eft.npz')
    m = _model()
    images, cams, rb = eo.scene_inputs()
    dev = lambda t: t.cuda()
    cams = eo.NdcCameras(dev(cams.R), dev(cams.T), dev(cams.focal_length), dev(cams.principal_point))
    rbd = eo.RayBundle(dev(rb.origins), dev(rb.directions), dev(rb.lengths), None)
    _, latent = m.encode(cams, images.cuda())
    assert tuple(latent.shape) == (2, 64, 64, 512)                                   # NHWC here, [2,512,64,64] in the reference
    r_lat = _rel(latent.reshape(-1)[::997], torch.from_numpy(g['latent_sample']))
    r_norm = abs(latent.norm().item() - float(g['latent_norm'])) / float(g['latent_norm'])
    rgb, f3, _ = m.forward(rbd)
    r_rgb, r_f3 = _rel(rgb, torch.from_numpy(g['rgb'])), _rel(f3, torch.from_numpy(g['f3']))
    print(f'EFT vs reference: ResNet-18 pyramid sample rel {r_lat:.3e} (norm {r_norm:.2e}); rgb rel {r_rgb:.3e}; conditioning feature rel {r_f3:.3e}')
    assert max(r_lat, r_norm, r_rgb, r_f3) < 1e-3
    # the cache-building call of sparsefusion/distillation.py:103-110: a [1,H,W] bundle through batched_forward -> same numbers
    b3 = eo.RayBundle(rbd.origins.view(1, 6, 8, 3), rbd.directions.view(1, 6, 8, 3), rbd.lengths.view(1, 6, 8, -1), None)
    rgb_b, f3_b, reg = m.batched_forward(b3, n_batches=16)
    assert rgb_b.shape == (1, 6, 8, 3) and f3_b.shape == (1, 6, 8, 256) and reg == 0
    assert _rel(f3_b.reshape(-1, 256), f3) < 1e-5


def test_eft_operators_vs_torch():
    from sparsefusion_b200 import _lib as lib
    g = torch.Generator(device='cuda').manual_seed(0)
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
    st = lib.stream
    # 3x3 / 2 max-pool with padding 1
    x = rn(2, 17, 22, 8)
    y = torch.empty(2, 9, 11, 8, device='cuda')
    lib.call('sfb_maxpool3x3s2_nhwc', lib.fptr(x), lib.fptr(y), 2, 17, 22, 8, st())
    assert torch.equal(y, F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1))
    # bilinear resize, align_corners=True, into a channel slice
    x = rn(2, 5, 7, 8)
    out = torch.zeros(2, 16, 16, 20, device='cuda')
    lib.call('sfb_resize_bilinear_ac_nhwc', x.data_ptr(), 8, out[..., 4:12].data_ptr(), 20, 2, 5, 7, 8, 16, 16, st())
    ref = F.interpolate(x.permute(0, 3, 1, 2), (16, 16), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    assert (out[..., 4:12] - ref).abs().max() < 1e-5 and out[..., :4].abs().max() == 0 and out[..., 12:].abs().max() == 0
    # grid_sample, border padding, align_corners=True (coordinates beyond [-1,1] included), odd channel count
    x = rn(2, 9, 11, 7)
    grid = (torch.rand(2, 300, 2, device='cuda', generator=g) * 2.6 - 1.3).contiguous()
    out = torch.empty(2, 300, 12, device='cuda').fill_(7.0)
    lib.call('sfb_grid_sample_nhwc', x.data_ptr(), 7, lib.fptr(grid), out[..., 3:].data_ptr(), 12, 2, 9, 11, 7, 300, st())
    ref = F.grid_sample(x.permute(0, 3, 1, 2), grid[:, :, None, :], mode='bilinear', padding_mode='border', align_corners=True)[..., 0].permute(0, 2, 1)
    assert (out[..., 3:10] - ref).abs().max() < 1e-5 and (out[..., :3] == 7.0).all() and (out[..., 10:] == 7.0).all()
    # single-head attention core vs nn.MultiheadAttention's arithmetic (sequence-first)
    for S, B in ((2, 300), (20, 64), (6, 5)):
        E = 256
        qkv = rn(S, B, 3 * E)
        out = torch.empty(S, B, E, device='cuda')
        lib.call('sfb_seq_attention', lib.fptr(qkv), lib.fptr(out), S, B, E, st())
        q, k, v = (t.double().permute(1, 0, 2) for t in qkv.split(E, dim=-1))
        ref = (torch.softmax(q @ k.transpose(1, 2) / E ** 0.5, dim=-1) @ v).permute(1, 0, 2).float()
        assert (out - ref).abs().max() < 2e-5, (S, B)
    # activations in place
    x = rn(1000 * 4)
    a, b = x.clone(), x.clone()
    lib.call('sfb_act_inplace', lib.fptr(a), a.numel(), 0, st())
    lib.call('sfb_act_inplace', lib.fptr(b), b.numel(), 1, st())
    assert torch.equal(a, F.relu(x)) and (b - F.gelu(x)).abs().max() < 1e-6


def test_transformer_encoder_engine_vs_torch_module():
    """one TransformerEncoder of the EFT (pre Linear + GELU, 4 post-norm layers) on the engine against the torch modules it holds as containers"""
    from oracle import eft_oracle as eo
    m = _model()
    m.prepare()
    S, Bn, din = 20, 96, 425
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(S, Bn, din, device='cuda', generator=g)
    xp = torch.zeros(S * Bn, 428, device='cuda')
    xp[:, :din] = x.view(S * Bn, din)
    with torch.no_grad():
        got = m._transformer('t2', xp, S, Bn).view(S, Bn, 256)
        t2 = m.t2.double()
        ref = t2.encoder(t2.pre(x.double()))
        m.t2.float()
    r = _rel(got, ref)
    print(f'transformer encoder (20 positions x 96) rel vs torch fp64: {r:.3e}')
    assert r < 1e-3
