"""oracle/ref_cuda_golden.py -- outputs of the REFERENCE's own CUDA operators (grid encoder, ray marching; compiled into oracle/_ref/ by
oracle/build_ref.py) on seeded inputs, stored as tests/golden/ref_cuda.npz, which tests/test_ref_cuda_gpu.py compares our kernels and the
C restatement against.  The test regenerates the inputs from the seeds below; large outputs are stored as a fixed, seeded sample of their
elements.  Point-wise quantities of the ray marcher are keyed by (ray, sample along the ray), which does not depend on the order in which
rays claim their slots in the point buffer.

    python -m oracle.ref_cuda_golden tests/golden/ref_cuda.npz      (on a GPU, after build() made oracle/_ref/)
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

SAMPLE = 8192
STEPS = 256          # max samples per ray of the march
RAYS_CHECKED = 128   # rays whose points / point gradients are stored whole


def grid_problem(B, seed=0):
    from oracle import ngp_oracle as no
    geo = no.live_geometry()
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.random((B, 3), dtype=np.float32), no.golden_grid_inputs()])
    emb = no.make_field_params(seed=1)['encoder.embeddings']
    return geo, x, emb


def hash_problem():
    from oracle import ngp_oracle as no
    offs, _ = no.grid_geometry(3, 8, 2, 2.0, 16, 14, None, False)
    emb = np.random.default_rng(3).random((int(offs[-1]), 2), dtype=np.float32) - 0.5
    return offs, emb


def backward_grad(L, B, C):
    return np.random.default_rng(4).standard_normal((L, B, C), dtype=np.float32)


def sample(a, seed, k=SAMPLE):
    """fixed, seeded sample of the elements of a (flattened)"""
    a = a.reshape(-1)
    idx = np.sort(np.random.default_rng(seed).choice(a.shape[0], min(a.shape[0], k), replace=False))
    return a[idx]


def march_problem(golden_dir):
    from oracle import ngp_oracle as no
    g = np.load(os.path.join(golden_dir, 'ngp_march.npz'))
    ro, rd = no.camera_rays(no.circle_cameras(8)[2], 128, 128)
    noises = np.random.default_rng(1).random(ro.shape[0], dtype=np.float32)
    return ro, rd, g['bitfield'], noises


def per_ray_inputs(N):
    """density / colour of sample k of ray n: [N, STEPS], [N, STEPS, 3]"""
    rng = np.random.default_rng(5)
    return rng.random((N, STEPS), dtype=np.float32) * 20, rng.random((N, STEPS, 3), dtype=np.float32)


def checked_rays(N):
    return np.random.default_rng(2).choice(N, RAYS_CHECKED, replace=False)


def point_index(rays):
    """for a rays table [N, 3] (ray index, offset, count): (ray index, sample k, point slot) of every point, as int64 tensors"""
    idx, off, cnt = rays[:, 0].long(), rays[:, 1].long(), rays[:, 2].long()
    r = torch.repeat_interleave(idx, cnt)
    first = torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    k = torch.arange(r.shape[0], device=rays.device) - first
    return r, k, torch.repeat_interleave(off, cnt) + k


def ray_segments(values, rays, which):
    """values of the points of rays `which` (in that order, then by sample), concatenated"""
    by_ray = {int(i): (int(o), int(c)) for i, o, c in rays.tolist()}
    return np.concatenate([values[by_ray[int(n)][0]:by_ray[int(n)][0] + by_ray[int(n)][1]] for n in which])


def run_march(m, ro, rd, bitfield, noises):
    """march_rays_train + composite forward / backward of one operator module on the march problem"""
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    N = ro.shape[0]
    rot, rdt, aabb = dev(ro), dev(rd), dev(np.array([-4, -4, -4, 4, 4, 4], np.float32))
    nears, fars = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
    m.near_far_from_aabb(rot, rdt, aabb, N, 0.2, nears, fars)
    M = N * STEPS
    xyzs, dirs, deltas = torch.zeros(M, 3, device='cuda'), torch.zeros(M, 3, device='cuda'), torch.zeros(M, 2, device='cuda')
    rays = torch.empty(N, 3, dtype=torch.int32, device='cuda')
    counter = torch.zeros(2, dtype=torch.int32, device='cuda')
    m.march_rays_train(rot, rdt, dev(bitfield), 4.0, 0.0, STEPS, N, 3, 128, M, nears, fars, xyzs, dirs, deltas, rays, counter, dev(noises))
    torch.cuda.synchronize()
    n_pts = int(counter[0].item())
    sig_t, rgb_t = per_ray_inputs(N)
    r, k, slot = point_index(rays)
    sig, rgb = torch.zeros(n_pts, device='cuda'), torch.zeros(n_pts, 3, device='cuda')
    sig[slot] = dev(sig_t)[r, k]
    rgb[slot] = dev(rgb_t)[r, k]
    ws, dp, im = torch.empty(N, device='cuda'), torch.empty(N, device='cuda'), torch.empty(N, 3, device='cuda')
    dl = deltas[:n_pts].contiguous()
    m.composite_rays_train_forward(sig, rgb, dl, rays, n_pts, N, 1e-4, ws, dp, im)
    gs, gc = torch.zeros(n_pts, device='cuda'), torch.zeros(n_pts, 3, device='cuda')
    gws, gim = torch.ones(N, device='cuda') * 0.3, torch.ones(N, 3, device='cuda') * 0.7
    m.composite_rays_train_backward(gws, gim, sig, rgb, dl, rays, ws, im, n_pts, N, 1e-4, gs, gc)
    torch.cuda.synchronize()
    rt = rays.cpu().numpy()
    which = checked_rays(N)
    return dict(nears=nears.cpu().numpy(), fars=fars.cpu().numpy(), counter=counter.cpu().numpy(), counts=rt[np.argsort(rt[:, 0])][:, 2],
                xyzs=ray_segments(xyzs.cpu().numpy(), rt, which), ws=ws.cpu().numpy(), depth=dp.cpu().numpy(), image=im.cpu().numpy(),
                grad_sigma=ray_segments(gs.cpu().numpy(), rt, which), grad_rgb=ray_segments(gc.cpu().numpy(), rt, which))


def morton_coords():
    return np.random.default_rng(6).integers(0, 128, (50000, 3), dtype=np.int32)


def density_grid():
    return np.random.default_rng(7).standard_normal(3 * 128 ** 3, dtype=np.float32)


def generate(golden_dir):
    from oracle import build_ref
    ge, rm = build_ref.load_module('_ref_gridencoder'), build_ref.load_module('_ref_raymarching')
    out = {}
    # grid encoder forward (tiled live geometry + a hash grid)
    geo, x, emb = grid_problem(1 << 18)
    B, L, C, D = x.shape[0], geo['L'], geo['C'], 3
    xt, et, off = torch.from_numpy(x).cuda(), emb.cuda(), torch.from_numpy(geo['offsets']).cuda()
    o, d = torch.empty(L, B, C, device='cuda'), torch.empty(B, L * D * C, device='cuda')
    ge.grid_encode_forward(xt, et, off, o, B, D, C, L, geo['S'], geo['H'], d, 1, False)
    out['fwd_out'], out['fwd_dy_dx'] = sample(o.cpu().numpy(), 10), sample(d.cpu().numpy(), 11)
    offs, emb_h = hash_problem()
    a = torch.empty(8, B, 2, device='cuda')
    ge.grid_encode_forward(xt, torch.from_numpy(emb_h).cuda(), torch.from_numpy(offs).cuda(), a, B, 3, 2, 8, 1.0, 16, None, 0, False)
    out['hash_out'] = sample(a.cpu().numpy(), 12)
    # grid encoder backward
    geo, x, emb = grid_problem(1 << 16)
    B = x.shape[0]
    g = torch.zeros_like(emb.cuda())
    ge.grid_encode_backward(torch.from_numpy(backward_grad(L, B, C)).cuda(), torch.from_numpy(x).cuda(), emb.cuda(), off, g, B, D, C, L, geo['S'],
                            geo['H'], None, None, 1, False)
    gn = g.cpu().numpy()
    out['bwd_touched'] = np.packbits((gn != 0).reshape(-1))
    out['bwd_grad'] = sample(gn, 13)
    # forward at the size the C restatement is checked at
    geo, x, emb = grid_problem(1 << 14)
    B = x.shape[0]
    o = torch.empty(L, B, C, device='cuda')
    ge.grid_encode_forward(torch.from_numpy(x).cuda(), emb.cuda(), off, o, B, D, C, L, geo['S'], geo['H'], None, 1, False)
    out['small_fwd_out'] = sample(o.cpu().numpy(), 14)
    # ray marching, compositing, morton codes, bitfield packing
    for k, v in run_march(rm, *march_problem(golden_dir)).items():
        out['march_' + k] = v
    i1 = torch.empty(50000, dtype=torch.int32, device='cuda')
    rm.morton3D(torch.from_numpy(morton_coords()).cuda(), 50000, i1)
    out['morton'] = sample(i1.cpu().numpy(), 15)
    b1 = torch.empty(3 * 128 ** 3 // 8, dtype=torch.uint8, device='cuda')
    rm.packbits(torch.from_numpy(density_grid()).cuda(), b1.numel(), 0.1, b1)
    out['packbits'] = sample(b1.cpu().numpy(), 16)
    return out


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    res = generate(os.path.join(root, 'tests', 'golden'))
    np.savez_compressed(sys.argv[1], **res)
    print({k: v.shape for k, v in res.items()}, os.path.getsize(sys.argv[1]))
