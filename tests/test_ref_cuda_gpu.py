"""Cross-validation against the REFERENCE's own CUDA operators: tests/golden/ref_cuda.npz holds their outputs on seeded inputs
(oracle/ref_cuda_golden.py, run on a GPU against the reference's sources compiled by oracle/build_ref.py).  Checked here against them:
(a) our sm_90a kernels, (b) the C restatement.

This is what pins the NGP half of the oracle to the reference: the reference has no tests or golden vectors
for this path, and its operators are CUDA-only.
"""
import numpy as np
import pytest
import torch

from oracle import ref_cuda_golden as rg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(f'{golden_dir}/ref_cuda.npz')


def test_grid_forward_bit_identical_to_reference_cuda(gold):
    from sparsefusion_b200 import _gridencoder as ours
    geo, x, emb = rg.grid_problem(1 << 18)
    B, L, C, D = x.shape[0], geo['L'], geo['C'], 3
    xt, et, off = torch.from_numpy(x).cuda(), emb.cuda(), torch.from_numpy(geo['offsets']).cuda()
    o_our, d_our = torch.empty(L, B, C, device='cuda'), torch.empty(B, L * D * C, device='cuda')
    ours.grid_encode_forward(xt, et, off, o_our, B, D, C, L, geo['S'], geo['H'], d_our, 1, False)
    torch.cuda.synchronize()
    # identical indices AND identical interpolation arithmetic -> identical bits
    o_s = rg.sample(o_our.cpu().numpy(), 10)
    assert np.array_equal(o_s, gold['fwd_out']), f'{(o_s != gold["fwd_out"]).sum()} of {o_s.size} sampled outputs differ'
    np.testing.assert_allclose(rg.sample(d_our.cpu().numpy(), 11), gold['fwd_dy_dx'], rtol=1e-6, atol=1e-6)
    # hash grid type
    offs, emb_h = rg.hash_problem()
    b = torch.empty(8, B, 2, device='cuda')
    ours.grid_encode_forward(xt, torch.from_numpy(emb_h).cuda(), torch.from_numpy(offs).cuda(), b, B, 3, 2, 8, 1.0, 16, None, 0, False)
    assert np.array_equal(rg.sample(b.cpu().numpy(), 12), gold['hash_out'])


def test_grid_backward_matches_reference_cuda(gold):
    from sparsefusion_b200 import _gridencoder as ours
    geo, x, emb = rg.grid_problem(1 << 16)
    B, L, C, D = x.shape[0], geo['L'], geo['C'], 3
    xt, et, off = torch.from_numpy(x).cuda(), emb.cuda(), torch.from_numpy(geo['offsets']).cuda()
    grad = torch.from_numpy(rg.backward_grad(L, B, C)).cuda()
    g_our = torch.zeros_like(et)
    ours.grid_encode_backward(grad, xt, et, off, g_our, B, D, C, L, geo['S'], geo['H'], None, None, 1, False)
    gn = g_our.cpu().numpy()
    np.testing.assert_allclose(rg.sample(gn, 13), gold['bwd_grad'], rtol=1e-4, atol=1e-5)      # atomic order differs
    assert np.array_equal(np.packbits((gn != 0).reshape(-1)), gold['bwd_touched'])             # same rows touched


def test_c_restatement_matches_reference_cuda_grid(gold):
    from oracle import ngp_oracle as no
    from sparsefusion_b200 import _lib as lib
    geo, x, emb = rg.grid_problem(1 << 14)
    L = geo['L']
    s = torch.empty(L, device='cuda')
    lib.call('sfb_grid_level_scales', L, float(geo['S']), geo['H'], lib.fptr(s), lib.stream())
    out, _, _ = no.grid_encode_forward(x, emb.numpy(), geo['offsets'], geo['S'], geo['H'], 1, False, False, s.cpu().numpy())
    out = rg.sample(out, 14)
    diff = np.abs(out - gold['small_fwd_out'])
    print('oracle-vs-reference-CUDA grid forward: max abs diff', diff.max(), 'exact fraction', (diff == 0).mean())
    np.testing.assert_allclose(out, gold['small_fwd_out'], rtol=1e-5, atol=1e-6)


def test_raymarching_operators_match_reference_cuda(gold, golden_dir):
    from sparsefusion_b200 import _raymarching as ours
    from oracle import ngp_oracle as no
    ro, rd, bitfield, noises = rg.march_problem(golden_dir)
    our = rg.run_march(ours, ro, rd, bitfield, noises)
    ref = {k[len('march_'):]: gold[k] for k in gold.files if k.startswith('march_')}
    assert np.array_equal(ref['nears'], our['nears']) and np.array_equal(ref['fars'], our['fars'])
    assert np.array_equal(ref['counter'], our['counter'])
    assert np.array_equal(ref['counts'], our['counts']), 'per-ray sample counts differ from the reference CUDA kernel'
    # oracle counts too
    _, _, _, rays_o, cnt_o = no.march_rays_train(ro, rd, 4.0, bitfield, 3, 128, ref['nears'], ref['fars'], noises, 0.0, rg.STEPS)
    assert np.array_equal(rays_o[:, 2], ref['counts']) and int(cnt_o[0]) == int(ref['counter'][0])
    # points of a few rays, and composite forward / backward keyed by (ray, sample)
    np.testing.assert_array_equal(our['xyzs'], ref['xyzs'])
    for k in ('ws', 'depth', 'image', 'grad_sigma', 'grad_rgb'):
        np.testing.assert_allclose(our[k], ref[k], rtol=1e-6, atol=1e-7, err_msg=k)
    # morton / packbits
    i2 = torch.empty(50000, dtype=torch.int32, device='cuda')
    ours.morton3D(torch.from_numpy(rg.morton_coords()).cuda(), 50000, i2)
    assert np.array_equal(rg.sample(i2.cpu().numpy(), 15), gold['morton'])
    b2 = torch.empty(3 * 128 ** 3 // 8, dtype=torch.uint8, device='cuda')
    ours.packbits(torch.from_numpy(rg.density_grid()).cuda(), b2.numel(), 0.1, b2)
    assert np.array_equal(rg.sample(b2.cpu().numpy(), 16), gold['packbits'])
