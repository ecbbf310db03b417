"""Ray generation (SURVEY §8f row 2, C ABI section 6) against the harness' ray function.  The fused image-space losses are checked per
element against fp64 in tests/test_step_fp64_gpu.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('hw', [(128, 128), (37, 53), (256, 256)])
def test_rays_match_the_harness_camera_function(hw):
    from oracle import ngp_oracle as no
    from sparsefusion_b200 import image_glue as glue
    h, w = hw
    for cam in no.circle_cameras(5)[:3]:
        o_ref, d_ref = no.camera_rays(cam, h, w, 4.0)
        o, d = glue.rays_from_camera(torch.from_numpy(cam[0]).cuda(), torch.from_numpy(cam[1]).cuda(), h, w, 4.0)
        assert np.array_equal(o.cpu().numpy(), o_ref)
        assert np.abs(d.cpu().numpy() - d_ref).max() < 2e-7          # same expression; numpy's matmul may order / fuse the 3-term sum differently


@pytest.mark.parametrize('mode', ['photometric', 'sds', 'eft'])
def test_loss_wrappers_combine_the_sums(mode):
    """the loss image_glue.py assembles from the kernels' three sums, against the fp64 loss of distillation.py's expressions: the sums'
    own bounds (oracle/step_fp64.py) weighted by the loss coefficients, plus a few roundings of the combination"""
    from oracle import step_fp64 as sp
    from oracle.field_fp64 import gamma
    from sparsefusion_b200 import image_glue as glue
    g = torch.Generator(device='cuda').manual_seed(7)
    h, w = 37, 53
    n = h * w
    lc, ls, lo, wgt = 1.0, 0.7, 1e-3, 0.37
    img, sil = torch.rand(n, 3, device='cuda', generator=g), torch.rand(n, device='cuda', generator=g)
    if mode == 'photometric':
        rgb = torch.rand(3, 2 * h, 2 * w, device='cuda', generator=g)
        mask = (torch.rand(1, 2 * h, 2 * w, device='cuda', generator=g) > 0.5).float()
        loss = glue.photometric_loss(img, sil, rgb, mask, h, w, 2, lc, ls, lo)[0]
        (S, B) = sp.ref_photometric(img, sil, rgb, mask, h, w, 2, lc, ls, lo, sp.kernel_plan('photometric_loss', dict(h=h, w=w)))['sums']
        k = torch.tensor([lc / (3 * n), ls / n, lo / n], dtype=torch.float64)
    else:
        up = glue.upsample2x_render(img, sil, h, w)
        target = torch.rand(3, 2 * h, 2 * w, device='cuda', generator=g) * 0.3
        ge = torch.randn(3, 2 * h, 2 * w, device='cuda', generator=g) * 1e-4
        m = 0 if mode == 'sds' else 1
        loss = glue.fusion_loss(up, target, h, w, mode, wgt, lc, ls, lo, g_extra=ge)[0]
        (S, B) = sp.ref_fusion(up, target, m, wgt, lc, ls, lo, ge, sp.kernel_plan('fusion_loss', dict(h=h, w=w)))['sums']
        N = 4 * n
        k = torch.tensor([(wgt if m == 0 else lc) / (3 * N), 0.0 if m == 0 else ls / N, lo / N], dtype=torch.float64)
    ref = float((k * S).sum())
    bound = float((k.abs() * B).sum() + gamma(8) * (k * S).abs().sum())
    err = abs(float(loss) - ref)
    print(f'{mode}: loss {float(loss):.9g} vs fp64 {ref:.9g}, err/bound {err / bound:.3f}')
    assert err <= bound
