"""Epipolar Feature Transformer on the sm_90a engine (SURVEY §8f row 4) against tests/golden/eft.npz -- outputs of the REFERENCE's own
EpipolarFeatureTransformer (sparsefusion/eft.py) on the same deterministic weights and inputs -- and its transformer encoder against torch.
Bar: 1e-3 relative L2 (BASELINE.json north_star tolerance for floating-point outputs).  The EFT-only operators are checked per element
against fp64 in tests/test_step_fp64_gpu.py."""
import numpy as np
import pytest
import torch

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
