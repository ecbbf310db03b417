"""wgmma implicit-GEMM convolution (sfb_conv2d_nhwc_tf32) against a plain PyTorch reference (fp64 accumulate).

Tolerances, all written here:
  * operands pre-rounded to TF32 on both sides -> only the fp32 accumulation order differs: rel L2 <= 2e-6 (both modes);
  * raw fp32 operands, 'tf32x3' mode (default: hi/lo split, 3 MMAs) -> fp32-class: rel L2 <= 5e-6;
  * raw fp32 operands, 'tf32' mode (single pass; what the reference GPU build's cuDNN/cuBLAS did) -> rel L2 <= 1e-3.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(params=['tf32x3', 'tf32'])
def mode(request):
    from sparsefusion_b200 import ops
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision('tf32x3')


def _ref_conv(x_nhwc, w, b, stride, pad):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2).double(), w.double(), None if b is None else b.double(), stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).float().contiguous()


CASES = [
    # NB, H, W, Cin, Cout, K, stride, pad
    (2, 8, 8, 32, 32, 1, 1, 0),
    (1, 16, 16, 64, 128, 3, 1, 1),
    (1, 32, 32, 260, 64, 7, 1, 3),      # K tail: 260 channels -> 9 chunks of 32, last zero filled by TMA
    (1, 32, 32, 16, 64, 15, 1, 7),      # CrossEmbed 15x15
    (2, 16, 16, 64, 128, 4, 2, 1),      # Downsample: stride-2 parity planes
    (3, 4, 4, 128, 256, 3, 1, 1),       # pixel tile spans 8 images, NB = 3 -> TMA box beyond the batch
    (5, 1, 1, 96, 64, 1, 1, 0),         # nn.Linear as 1x1 conv on 5 rows
    (1, 32, 32, 256, 4, 3, 1, 1),       # final_conv: Cout = 4
    (2, 8, 8, 512, 1024, 3, 1, 1),      # weight-streaming shape: split-K kicks in
    (1, 24, 24, 32, 32, 3, 1, 1),       # non power-of-two width: partial tiles
]


@pytest.mark.parametrize('case', CASES)
def test_conv_matches_fp32_reference(case, mode):
    from sparsefusion_b200 import ops
    nb, h, w, cin, cout, k, stride, pad = case
    g = torch.Generator(device='cuda').manual_seed(1234 + cin + cout + k)
    x = torch.randn(nb, h, w, cin, device='cuda', generator=g)
    wt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device='cuda', generator=g)
    # (1) exact-operand test
    xr, wr = ops.round_tf32(x), ops.round_tf32(wt)
    y = ops.conv2d_nhwc(xr, ops.pack_conv_weight(wr), cout, k, k, stride, pad, bias=b)
    ref = _ref_conv(xr, wr, b, stride, pad)
    rel = ((y - ref).norm() / ref.norm()).item()
    assert rel < 2e-6, f'{case}: tf32-exact operands rel {rel:.3e}'
    # (2) raw fp32 activations (hardware truncation of A), weights rounded at pack time
    y2 = ops.conv2d_nhwc(x, ops.pack_conv_weight(wt), cout, k, k, stride, pad, bias=b)
    ref2 = _ref_conv(x, wt, b, stride, pad)
    rel2 = ((y2 - ref2).norm() / ref2.norm()).item()
    assert rel2 < (5e-6 if mode == 'tf32x3' else 1e-3), f'{case} [{mode}]: raw operands rel {rel2:.3e}'


@pytest.mark.parametrize('bn', [32, 64, 128, 256])
@pytest.mark.parametrize('splits', [1, 3, 0])
def test_conv_tilings_agree(bn, splits, mode):
    from sparsefusion_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(7)
    x = ops.round_tf32(torch.randn(2, 16, 16, 96, device='cuda', generator=g))
    wt = ops.round_tf32(torch.randn(256, 96, 3, 3, device='cuda', generator=g) / 30)
    b = torch.randn(256, device='cuda', generator=g)
    y = ops.conv2d_nhwc(x, ops.pack_conv_weight(wt), 256, 3, 3, 1, 1, bias=b, splits=splits, bn=bn)
    ref = _ref_conv(x, wt, b, 1, 1)
    rel = ((y - ref).norm() / ref.norm()).item()
    assert rel < 2e-6, f'bn={bn} splits={splits}: rel {rel:.3e}'


def test_conv_epilogue_residual_accumulate_and_channel_slices(mode):
    from sparsefusion_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(9)
    wide_in = ops.round_tf32(torch.randn(2, 8, 8, 160, device='cuda', generator=g))
    x = wide_in[..., 32:96]                                   # read a 64-channel slice of a 160-channel tensor
    wt = ops.round_tf32(torch.randn(64, 64, 3, 3, device='cuda', generator=g) / 24)
    b = torch.randn(64, device='cuda', generator=g)
    res = torch.randn(2, 8, 8, 64, device='cuda', generator=g)
    wide_out = torch.full((2, 8, 8, 192), 7.0, device='cuda')
    out = wide_out[..., 64:128]                               # write a slice of a 192-channel tensor
    ops.conv2d_nhwc(x, ops.pack_conv_weight(wt), 64, 3, 3, 1, 1, bias=b, residual=res, out=out)
    ref = _ref_conv(x.contiguous(), wt, b, 1, 1) + res
    assert ((out - ref).norm() / ref.norm()).item() < 2e-6
    assert (wide_out[..., :64] == 7.0).all() and (wide_out[..., 128:] == 7.0).all()
    # accumulate a second convolution into the same slice (Parallel(conv3x3, conv1x1), imagen_pytorch.py:1322)
    w1 = ops.round_tf32(torch.randn(64, 64, 1, 1, device='cuda', generator=g) / 8)
    ops.conv2d_nhwc(x, ops.pack_conv_weight(w1), 64, 1, 1, 1, 0, out=out, accumulate=True)
    ref2 = ref + _ref_conv(x.contiguous(), w1, None, 1, 0)
    assert ((out - ref2).norm() / ref2.norm()).item() < 2e-6


def test_linear_tc():
    from sparsefusion_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(11)
    x = ops.round_tf32(torch.randn(3, 50, 128, device='cuda', generator=g))
    w = ops.round_tf32(torch.randn(64, 128, device='cuda', generator=g) / 11)
    y = ops.linear_tc(x, ops.pack_conv_weight(w), 64)
    ref = (x.double() @ w.double().t()).float()
    assert ((y - ref).norm() / ref.norm()).item() < 2e-6


def test_round_tf32_matches_definition():
    from sparsefusion_b200 import ops
    x = torch.randn(4096, device='cuda')
    r = ops.round_tf32(x)
    assert ((r.view(torch.int32) & 0x1FFF) == 0).all()
    assert ((r - x).abs() <= x.abs() * 2.0 ** -11 + 1e-45).all()
