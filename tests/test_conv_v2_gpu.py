"""Second-generation 3xTF32 conv kernel (M-side operand split in registers, swap-AB for <= 64 output pixels) against fp64
references and against the first-generation kernel.  Tolerance: fp32-class, rel L2 <= 1e-5 (the accumulation chain per CTA is capped at 96 k-steps; longer chains drift, see conv_wgmma.cu)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

CASES = [
    # NB, H, W, Cin, Cout, K, stride, pad          (P = NB*Ho*Wo output pixels)
    (1, 4, 4, 1024, 1024, 3, 1, 1),     # swap-AB, 16 pixels
    (1, 4, 4, 2048, 1024, 1, 1, 0),     # swap-AB 1x1, many channel chunks
    (2, 4, 4, 256, 512, 3, 1, 1),       # swap-AB, 32 pixels over two images
    (1, 8, 8, 512, 512, 3, 1, 1),       # swap-AB, 64 pixels
    (1, 16, 16, 256, 512, 4, 2, 1),     # swap-AB through the stride-2 parity planes (8x8 outputs)
    (3, 1, 1, 1024, 512, 1, 1, 0),      # linear rows (3 "pixels")
    (1, 4, 4, 64, 12, 3, 1, 1),         # Cout tail inside the 128-row weight box
    (1, 16, 16, 256, 256, 3, 1, 1),     # normal mode, 256 pixels
    (1, 32, 32, 260, 64, 7, 1, 3),      # normal mode, K tail
    (8, 8, 8, 512, 512, 3, 1, 1),       # normal mode, batch 8
    (1, 32, 32, 256, 4, 3, 1, 1),       # normal mode, Cout = 4
]


def _ref(x, w, b, stride, pad):
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), None if b is None else b.double(), stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).float().contiguous()


@pytest.mark.parametrize('case', CASES)
def test_v2_matches_reference_and_v1(case):
    from sparsefusion_b200 import _lib as lib, ops
    nb, h, w, cin, cout, k, stride, pad = case
    ops.set_precision('tf32x3')
    g = torch.Generator(device='cuda').manual_seed(77 + cin + cout + k + nb)
    x = torch.randn(nb, h, w, cin, device='cuda', generator=g)
    wt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device='cuda', generator=g)
    res = torch.randn(nb, (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1, cout, device='cuda', generator=g)
    wp = ops.pack_conv_weight(wt)
    ref = _ref(x, wt, b, stride, pad) + res
    out = {}
    for v in (2, 1):
        lib.call('sfb_conv_set_variant', v)
        try:
            out[v] = ops.conv2d_nhwc(x, wp, cout, k, k, stride, pad, bias=b, residual=res)
            for splits in (2, 0):
                y = ops.conv2d_nhwc(x, wp, cout, k, k, stride, pad, bias=b, residual=res, splits=splits)
                rel = ((y - ref).norm() / ref.norm()).item()
                # 3xTF32 drops the lo*lo term (2^-22 per product) and the tensor core's fp32 accumulator truncates; measured 0.3-1.02e-5
                assert rel < 2e-5, f'{case} variant {v} splits {splits}: rel {rel:.3e}'
        finally:
            lib.call('sfb_conv_set_variant', 2)
    assert ((out[1] - out[2]).norm() / ref.norm()).item() < 1e-5
    # accumulate mode
    y0 = torch.ones_like(ref)
    ops.conv2d_nhwc(x, wp, cout, k, k, stride, pad, out=y0, accumulate=True)
    assert ((y0 - (_ref(x, wt, None, stride, pad) + 1)).norm() / ref.norm()).item() < 1e-5


def test_tensor_core_reads_tf32_by_truncation():
    """Experiment recorded as a test: feeding the un-masked fp32 word as the 'hi' operand (variant 3) must give bit-identical
    results to the explicitly masked operand (variant 2) if -- and only if -- the tensor core's tf32 read ignores the 13 low mantissa bits."""
    from sparsefusion_b200 import _lib as lib, ops
    ops.set_precision('tf32x3')
    g = torch.Generator(device='cuda').manual_seed(5)
    same = []
    for (nb, h, w, cin, cout, k) in [(1, 4, 4, 1024, 1024, 3), (1, 32, 32, 256, 256, 3), (1, 8, 8, 512, 512, 1)]:
        x = torch.randn(nb, h, w, cin, device='cuda', generator=g)
        wt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
        wp = ops.pack_conv_weight(wt)
        out = {}
        for v in (2, 3):
            lib.call('sfb_conv_set_variant', v)
            try:
                out[v] = ops.conv2d_nhwc(x, wp, cout, k, k, 1, k // 2, splits=1)
            finally:
                lib.call('sfb_conv_set_variant', 2)
        same.append(bool(torch.equal(out[2], out[3])))
        rel = ((out[3] - out[2]).norm() / out[2].norm()).item()
        print(f'raw-hi vs masked-hi {(nb, h, w, cin, cout, k)}: bit-identical={same[-1]} rel diff {rel:.3e}')
    print('TENSOR CORE TF32 READ IS A TRUNCATION' if all(same) else 'tensor core tf32 read is NOT a plain truncation')


@pytest.mark.parametrize('case', [(1, 32, 32, 256, 256, 3, 1, 1), (2, 16, 16, 96, 160, 3, 1, 1), (1, 64, 64, 128, 128, 3, 2, 1), (300, 1, 1, 512, 384, 1, 1, 0)])
def test_presplit_weights_match_in_kernel_split(case):
    """(hi, lo) copies of the weights loaded by TMA vs the same split done by the converter warps: the operands of every MMA are
    bit-identical, so the results must be (for equal split-K factors)."""
    from sparsefusion_b200 import ops
    nb, h, w, cin, cout, k, stride, pad = case
    ops.set_precision('tf32x3')
    g = torch.Generator(device='cuda').manual_seed(9 + cin)
    x = torch.randn(nb, h, w, cin, device='cuda', generator=g)
    wt = torch.randn(cout, cin, k, k, device='cuda', generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device='cuda', generator=g)
    wp = ops.pack_conv_weight(wt)
    sp = ops.split_packed_weight(wp)
    assert torch.equal(sp[0] + sp[1], wp) and ((sp[0].view(torch.int32) & 0x1FFF) == 0).all()
    y0 = ops.conv2d_nhwc(x, wp, cout, k, k, stride, pad, bias=b, splits=1)
    y1 = ops.conv2d_nhwc(x, wp, cout, k, k, stride, pad, bias=b, splits=1, w_split=sp)
    assert torch.equal(y0, y1)
    ref = _ref(x, wt, b, stride, pad)
    assert ((y1 - ref).norm() / ref.norm()).item() < 2e-5
