"""The grid-encoder and ray-marching operators on the GPU, at every configuration they accept, against three references: the fp64
restatements of oracle/grid_march_fp64.py (per-element derived bounds), the C restatement (oracle/ngp_oracle.c) and the reference's own
`_gridencoder` / `_raymarching` modules built into oracle/_ref/ by build().  Without oracle/_ref/ the reference-build comparisons skip;
the fp64 ones still run.

Grid encoder: all 80 (D, C, gridtype, align_corners) instantiations, on level geometries whose coarse levels are dense tiled grids and
whose fine levels are capped at the hashmap size, so both branches of grid_row run in one call.  Corner rows equal the fp64 restatement's
integer contract; the forward and dy_dx are bit-identical to the reference build (same arithmetic in the same order) and within the fp64
bound; embedding gradients and grad_inputs are within the fp64 bound, with the same set of touched rows as the reference build.

Marching: bit-identical to the reference build and to the C restatement, per ray through the `rays` table (point order follows atomic
arrival).  Compositing: within the fp64 bound; the inference loop's alive sets and rays_t equal the reference build's after every
iteration.  No ray sent here has a zero direction or an unbounded skip target (`do t += dt while t < tt` would never end).

The catalogue test at the end asserts that every variant of the matrix ran: run the file whole."""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import build_ref
from oracle import grid_march_fp64 as gm
from oracle import ngp_oracle as no

pytestmark = pytest.mark.gpu

RAN = {k: set() for k in ('grid', 'grid_B', 'march', 'composite', 'inference', 'packbits')}
NO_REF = 'oracle/_ref/ is absent: build() compiles the reference operators there (only where the reference sources are present)'
VARIANTS = list(itertools.product((1, 2, 3, 4, 5), (1, 2, 4, 8), (0, 1), (False, True)))


@pytest.fixture(scope='module')
def ref():
    if not build_ref.available():
        return None
    return dict(grid=build_ref.load_module('_ref_gridencoder'), march=build_ref.load_module('_ref_raymarching'))


def _need(ref, which):
    if ref is None:
        pytest.skip(NO_REF)
    return ref[which]


def _scales(L, S, H):
    from sparsefusion_b200 import _lib as lib
    s = torch.empty(L, device='cuda')
    lib.call('sfb_grid_level_scales', L, float(S), H, lib.fptr(s), lib.stream())
    return s.cpu()


def _sync():
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ grid encoder
def _grid_run(mod, x, emb, offsets, S, H, D, C, L, gridtype, ac, grad):
    B = x.shape[0]
    off = torch.from_numpy(offsets).cuda()
    out, dy = torch.empty(L, B, C, device='cuda'), torch.empty(B, L * D * C, device='cuda')
    mod.grid_encode_forward(x, emb, off, out, B, D, C, L, S, H, dy, gridtype, ac)
    _sync()
    ge, gi = torch.zeros_like(emb), torch.zeros(B, D, device='cuda')
    mod.grid_encode_backward(grad, x, emb, off, ge, B, D, C, L, S, H, dy, gi, gridtype, ac)
    _sync()
    return out, dy, ge, gi


def _corner_rows(x, offsets, D, L, S, H, gridtype, ac):
    from sparsefusion_b200 import _lib as lib
    rows = torch.empty(L, x.shape[0], 1 << D, dtype=torch.int32, device='cuda')
    lib.call('sfb_grid_corner_rows', lib.fptr(x), lib.iptr(torch.from_numpy(offsets).cuda()), lib.iptr(rows), x.shape[0], D, L, float(S), H,
             gridtype, int(ac), lib.stream())
    _sync()
    return rows


def _check_grid(x, D, C, gridtype, ac, ref, seed, record):
    from sparsefusion_b200 import _gridencoder as ours
    offsets, S, H = gm.grid_case(D, ac)
    L = len(offsets) - 1
    scales = _scales(L, S, H)
    emb = gm.grid_embeddings(int(offsets[-1]), C, seed).cuda()
    B = x.shape[0]
    grad = torch.randn(L, B, C, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    out, dy, ge, gi = _grid_run(ours, x, emb, offsets, S, H, D, C, L, gridtype, ac, grad)
    r = gm.GridFP64(x, emb, offsets, scales, gridtype, ac)
    f = r.forward()
    rt = r.rt
    assert torch.equal(_corner_rows(x, offsets, D, L, S, H, gridtype, ac).long(), f['rows']), 'corner rows'
    gm.assert_within('outputs', out, f['out'], f['out_abs'], rt['out'])
    gm.assert_within('dy_dx', dy.view(B, L, D, C), f['dy'], f['dy_abs'], rt['dy'])
    dead = ~r.live
    assert (out[:, dead] == 0).all() and (dy[dead] == 0).all(), 'out-of-range points must give exact zeros'
    b = r.backward(grad, dy, f['dy_abs'])
    gm.assert_within('grad_embeddings', ge, b['ge'], b['ge_abs'], b['ge_rtol'])
    gm.assert_within('grad_inputs', gi, b['gi'], b['gi_abs'], rt['gi'])
    record.add((D, C, gridtype, ac) if B != 1 << 20 else B)
    m = _need(ref, 'grid')
    o2, dy2, ge2, gi2 = _grid_run(m, x, emb, offsets, S, H, D, C, L, gridtype, ac, grad)
    assert torch.equal(out, o2), f'{int((out != o2).sum())} outputs differ from the reference build'
    assert torch.equal(dy, dy2), f'{int((dy != dy2).sum())} dy_dx differ from the reference build'
    gm.assert_within('grad_embeddings (reference build)', ge2, b['ge'], b['ge_abs'], b['ge_rtol'])
    assert torch.equal(ge != 0, ge2 != 0), 'touched rows differ from the reference build'
    assert torch.equal(gi, gi2), 'grad_inputs differ from the reference build (same dy_dx, same order)'


@pytest.mark.parametrize('D,C,gridtype,ac', VARIANTS)
def test_grid_variant(D, C, gridtype, ac, ref):
    offsets, S, H = gm.grid_case(D, ac)
    x = gm.grid_points(257, D, _scales(len(offsets) - 1, S, H), seed=D * 100 + C).cuda()
    _check_grid(x, D, C, gridtype, ac, ref, seed=7 * D + C, record=RAN['grid'])


@pytest.mark.parametrize('B', (1, 255, 257, 1 << 20))
@pytest.mark.parametrize('gridtype', (0, 1))
def test_grid_batch_sizes(B, gridtype, ref):
    x = torch.rand(B, 3, generator=torch.Generator().manual_seed(B)).cuda()
    _check_grid(x, 3, 2, gridtype, False, ref, seed=B % 1000, record=RAN['grid_B'])
    RAN['grid_B'].add(B)


@pytest.mark.parametrize('gridtype', ('hash', 'tiled'))
def test_grid_encoder_module_autograd(gridtype):
    """GridEncoder with calc_grad_inputs (inputs that require grad): embeddings and input gradients within the fp64 bound"""
    from sparsefusion_b200.gridencoder import GridEncoder
    D, C = 3, 4
    offsets, S, H = gm.grid_case(D, False)
    enc = GridEncoder(input_dim=D, num_levels=gm.GRID_L, level_dim=C, per_level_scale=2, base_resolution=H,
                      log2_hashmap_size=math.ceil(math.log2(5 ** D)), gridtype=gridtype).cuda()
    assert np.array_equal(enc.offsets.cpu().numpy(), offsets)
    with torch.no_grad():
        enc.embeddings.copy_(gm.grid_embeddings(int(offsets[-1]), C, 3))
    g = torch.Generator().manual_seed(4)
    x = (torch.rand(4000, D, generator=g) * 2.2 - 1.1).cuda().requires_grad_(True)
    G = torch.randn(4000, gm.GRID_L * C, generator=g).cuda()
    (enc(x) * G).sum().backward()
    u = (x.detach() + 1) / 2                                               # the module's fp32 normalisation
    r = gm.GridFP64(u, enc.embeddings.detach(), offsets, _scales(gm.GRID_L, S, H), 0 if gridtype == 'hash' else 1, False)
    f = r.forward()
    grad = G.view(-1, gm.GRID_L, C).permute(1, 0, 2).contiguous()
    b = r.backward(grad, None)
    gm.assert_within('embeddings.grad', enc.embeddings.grad, b['ge'], b['ge_abs'], b['ge_rtol'])
    gi = 0.5 * (grad.double().permute(1, 0, 2)[:, :, None, :] * f['dy']).sum((1, 3))
    gi_abs = 0.5 * (grad.double().abs().permute(1, 0, 2)[:, :, None, :] * f['dy_abs']).sum((1, 3))
    gm.assert_within('inputs.grad', x.grad, gi, gi_abs, r.rt['gi'])
    assert (x.grad[~r.live] == 0).all() and (~r.live).sum() > 100


# ------------------------------------------------------------------------------------------------ marching
def _rays(N, bound, seed):
    """from outside the box, from inside it (near clamped to min_near), missing it, axis-parallel with one or two zero direction
    components; directions not normalised (|d| in [0.3, 3]), no component between 0 and 1e-2 in magnitude"""
    g = torch.Generator().manual_seed(seed)
    n = N // 6
    unit = lambda v: v / v.norm(dim=1, keepdim=True)
    o_out = unit(torch.randn(n, 3, generator=g)) * bound * 2.5
    d_out = (torch.rand(n, 3, generator=g) * 1.6 - 0.8) * bound - o_out
    o_in = (torch.rand(n, 3, generator=g) * 1.8 - 0.9) * bound
    d_in = torch.randn(n, 3, generator=g)
    o_miss = unit(torch.randn(n, 3, generator=g)) * bound * 3
    d_miss = torch.linalg.cross(o_miss, torch.randn(n, 3, generator=g))      # the line passes 3 bound from the centre
    o_ax1 = (torch.rand(n, 3, generator=g) * 1.8 - 0.9) * bound
    d_ax1 = torch.randn(n, 3, generator=g)
    d_ax1[torch.arange(n), torch.arange(n) % 3] = 0
    o_ax2 = (torch.rand(n, 3, generator=g) * 1.8 - 0.9) * bound
    k = torch.arange(n) % 3
    d_ax2 = torch.zeros(n, 3)
    d_ax2[torch.arange(n), k] = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    o_ax2[torch.arange(n), k] = o_ax2[torch.arange(n), k] * 2.5           # some from outside along the axis
    o_far = unit(torch.randn(N - 5 * n, 3, generator=g)) * bound * 1.5
    d_far = -o_far + torch.randn(N - 5 * n, 3, generator=g) * 0.3 * bound
    o = torch.cat([o_out, o_in, o_miss, o_ax1, o_ax2, o_far])
    d = torch.cat([d_out, d_in, d_miss, d_ax1, d_ax2, d_far])
    d = torch.where((d.abs() < 1e-2) & (d != 0), torch.full_like(d, 1e-2), d)
    d = unit(d) * (0.3 + 2.7 * torch.rand(N, 1, generator=g))
    return o.float().contiguous(), d.float().contiguous()


def _product_bitfield(golden_dir):
    """the density bitfield that NeRFRenderer.update_extra_state builds for the seeded field of tests/golden/ngp_march.npz (C = 3,
    H = 128): tests/test_ngp_render_gpu.py::test_cuda_ray_mode_vs_oracle holds the product's to this one"""
    return np.load(f'{golden_dir}/ngp_march.npz')['bitfield']


BASE = dict(C=3, bound=4.0, H=128, dtg=0.0, steps=256, noise=True, overflow=False, occ=0.5)
MARCH = [dict(BASE)]
MARCH += [dict(BASE, C=c, bound=float(2 ** (c - 1))) for c in (1, 2, 4, 5)] + [dict(BASE, bound=3.0), dict(BASE, C=5, bound=11.0)]
MARCH += [dict(BASE, H=64), dict(BASE, dtg=1 / 256), dict(BASE, dtg=1 / 64), dict(BASE, C=5, bound=16.0, dtg=1 / 64)]
MARCH += [dict(BASE, steps=s) for s in (1, 16, 1024)] + [dict(BASE, noise=False), dict(BASE, overflow=True)]
MARCH += [dict(BASE, occ=o) for o in (0.0, 0.02, 1.0, 'update_extra_state')]
MARCH += [dict(C=5, bound=16.0, H=64, dtg=1 / 64, steps=1024, noise=True, overflow=True, occ=0.02),
          dict(C=2, bound=2.0, H=64, dtg=1 / 256, steps=16, noise=False, overflow=False, occ=1.0),
          dict(C=1, bound=1.0, H=128, dtg=1 / 64, steps=1024, noise=True, overflow=True, occ=0.5),
          dict(C=4, bound=8.0, H=128, dtg=1 / 256, steps=1024, noise=True, overflow=False, occ='update_extra_state')]
MIN_NEAR = 0.05


def _march_inputs(cfg, golden_dir, N=1536):
    ro, rd = _rays(N, cfg['bound'], seed=hash((cfg['C'], cfg['H'], cfg['steps'])) % 1000)
    if cfg['occ'] == 'update_extra_state':
        assert cfg['H'] == 128
        bf = _product_bitfield(golden_dir)
        bf = np.concatenate([bf, np.packbits(np.random.default_rng(1).random((cfg['C'] - 3) * 128 ** 3) < 0.3, bitorder='little')]) \
            if cfg['C'] > 3 else bf[:cfg['C'] * 128 ** 3 // 8]
    else:
        bf = np.packbits(np.random.default_rng(2).random(cfg['C'] * cfg['H'] ** 3) < cfg['occ'], bitorder='little')
    noises = np.random.default_rng(3).random(N, dtype=np.float32) if cfg['noise'] else np.zeros(N, np.float32)
    return ro, rd, bf, noises


def _march(mod, ro, rd, bf, noises, cfg, M):
    N = ro.shape[0]
    b = cfg['bound']
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()
    rot, rdt = ro.cuda(), rd.cuda()
    nears, fars = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
    mod.near_far_from_aabb(rot, rdt, dev(np.array([-b, -b, -b, b, b, b], np.float32)), N, MIN_NEAR, nears, fars)
    xyzs, dirs, deltas = torch.zeros(M, 3, device='cuda'), torch.zeros(M, 3, device='cuda'), torch.zeros(M, 2, device='cuda')
    rays = torch.full((N, 3), -7, dtype=torch.int32, device='cuda')
    counter = torch.zeros(2, dtype=torch.int32, device='cuda')
    mod.march_rays_train(rot, rdt, dev(bf), b, cfg['dtg'], cfg['steps'], N, cfg['C'], cfg['H'], M, nears, fars, xyzs, dirs, deltas, rays, counter,
                         dev(noises))
    _sync()
    return dict(nears=nears.cpu(), fars=fars.cpu(), xyzs=xyzs.cpu(), dirs=dirs.cpu(), deltas=deltas.cpu(), rays=rays.cpu(), counter=counter.cpu())


def _per_ray(res, M, width):
    """points of every ray written whole within M, by (ray, sample): [N, width, 8] (xyz, dir, deltas), and the written mask [N]"""
    rays = res['rays'].long()
    N = rays.shape[0]
    pts = torch.cat([res['xyzs'], res['dirs'], res['deltas']], 1)
    dense = torch.zeros(N, width, 8)
    written = (rays[:, 2] > 0) & (rays[:, 1] + rays[:, 2] <= M)
    for i, o, c in rays[written].tolist():
        dense[i, :c] = pts[o:o + c]
    wmask = torch.zeros(N, dtype=torch.bool)
    wmask[rays[written, 0]] = True
    return dense, wmask


def _check_rays_table(rays, N, total):
    """a permutation of the rays, whose point ranges tile [0, total) in claim order"""
    r = rays.long()
    assert torch.equal(torch.sort(r[:, 0]).values, torch.arange(N))
    order = torch.argsort(r[:, 1] * 2 + (r[:, 2] > 0))                     # empty rays may share an offset
    off, cnt = r[order, 1], r[order, 2]
    assert torch.equal(off, torch.cumsum(cnt, 0) - cnt) and int(cnt.sum()) == total


@pytest.mark.parametrize('cfg', MARCH, ids=lambda c: '-'.join(f'{k}{v}' for k, v in c.items()))
def test_march_rays_train(cfg, ref, golden_dir):
    from sparsefusion_b200 import _raymarching as ours
    ro, rd, bf, noises = _march_inputs(cfg, golden_dir)
    N = ro.shape[0]
    full = N * cfg['steps']
    o = _march(ours, ro, rd, bf, noises, cfg, full)
    total = int(o['counter'][0])
    M = max(1, total // 2) if cfg['overflow'] else full
    if cfg['overflow']:
        o = _march(ours, ro, rd, bf, noises, cfg, M)
    nears, fars = no.near_far_from_aabb(ro.numpy(), rd.numpy(), np.array([-1, -1, -1, 1, 1, 1], np.float32) * cfg['bound'], MIN_NEAR)
    assert torch.equal(o['nears'], torch.from_numpy(nears)) and torch.equal(o['fars'], torch.from_numpy(fars))
    miss = nears == np.finfo(np.float32).max
    assert miss.sum() > 0 and (fars[miss] == np.finfo(np.float32).max).all() and (nears[~miss] == MIN_NEAR).sum() > 0
    xo, do, lo, rays_o, cnt_o = no.march_rays_train(ro.numpy(), rd.numpy(), cfg['bound'], bf, cfg['C'], cfg['H'], nears, fars, noises,
                                                    cfg['dtg'], cfg['steps'], full)
    counts_o = torch.from_numpy(rays_o[:, 2]).long()
    r = o['rays'].long()
    counts = torch.zeros(N, dtype=torch.long)
    counts[r[:, 0]] = r[:, 2]
    assert torch.equal(counts, counts_o), 'per-ray sample counts differ from the C restatement'
    assert int(o['counter'][0]) == int(cnt_o[0]) and int(o['counter'][1]) == N
    _check_rays_table(o['rays'], N, total)
    width = max(1, int(counts.max()))
    mine, written = _per_ray(o, M, width)
    orc, _ = _per_ray(dict(xyzs=torch.from_numpy(xo), dirs=torch.from_numpy(do), deltas=torch.from_numpy(lo), rays=torch.from_numpy(rays_o)),
                      full, width)
    assert torch.equal(mine[written], orc[written]), 'points differ from the C restatement'
    assert bool(written.any()) == (total > 0) and cfg['overflow'] == bool((~written & (counts > 0)).any())
    if cfg['overflow']:
        # points of rays past M are not written: every slot in [0, M) that no written ray owns stays zero
        own = torch.zeros(M, dtype=torch.bool)
        for i, off, c in r[(r[:, 2] > 0) & (r[:, 1] + r[:, 2] <= M)].tolist():
            own[off:off + c] = True
        assert (o['deltas'][~own] == 0).all() and (o['xyzs'][~own] == 0).all()
    RAN['march'].add(tuple(sorted(cfg.items())))
    m = _need(ref, 'march')
    rf = _march(m, ro, rd, bf, noises, cfg, M)
    for k in ('nears', 'fars', 'counter'):
        assert torch.equal(rf[k], o[k]), k
    theirs, w2 = _per_ray(rf, M, width)
    assert torch.equal(torch.sort(rf['rays'][:, 0]).values, torch.arange(N, dtype=torch.int32))
    c2 = torch.zeros(N, dtype=torch.long)
    c2[rf['rays'][:, 0].long()] = rf['rays'][:, 2].long()
    assert torch.equal(c2, counts)
    both = written & w2
    assert torch.equal(theirs[both], mine[both]), 'points differ from the reference build'


# ------------------------------------------------------------------------------------------------ compositing
def _comp_rays(N, T, seed):
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, T + 1, (N,), generator=g)
    counts[:6] = torch.tensor([0, 1, 1, 0, T, 1])
    s = torch.rand(N, T, generator=g) * 30
    s[torch.rand(N, T, generator=g) < 0.1] = 0                            # sigma 0
    s[torch.rand(N, T, generator=g) < 0.01] = 5000                        # sigma delta >= 104: alpha = 1 in fp32
    dl = torch.stack([torch.rand(N, T, generator=g) * 0.05, torch.rand(N, T, generator=g) * 0.05], -1)
    dl[torch.rand(N, T, generator=g) < 0.02, 0] = 0                       # delta 0
    return s.float(), torch.rand(N, T, 3, generator=g).float(), dl.float(), counts


def _pack(s, c, dl, counts, seed, overflow):
    """the flat layout, point ranges claimed in a random ray order, M cut so that the last rays claimed fall past it"""
    N, T = s.shape
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(seed))
    off = torch.zeros(N, dtype=torch.long)
    off[perm] = torch.cumsum(counts[perm], 0) - counts[perm]
    total = int(counts.sum())
    M = int(total * 0.9) if overflow else total
    rays = torch.stack([torch.arange(N), off, counts], 1)[perm].int()
    sf, cf, df = torch.zeros(total), torch.zeros(total, 3), torch.zeros(total, 2)
    valid = torch.arange(T)[None] < counts[:, None]
    slot = (off[:, None] + torch.arange(T)[None])[valid]
    sf[slot], cf[slot], df[slot] = s[valid], c[valid], dl[valid]
    past = off + counts > M
    return sf[:M].contiguous(), cf[:M].contiguous(), df[:M].contiguous(), rays, M, past, slot, valid


def _composite_train(mod, sf, cf, df, rays, M, N, thr, gws, gim):
    sf, cf, df, rays = sf.cuda(), cf.cuda(), df.cuda(), rays.cuda()
    ws, dp, im = torch.full((N,), 9.0, device='cuda'), torch.full((N,), 9.0, device='cuda'), torch.full((N, 3), 9.0, device='cuda')
    mod.composite_rays_train_forward(sf, cf, df, rays, M, N, thr, ws, dp, im)
    gs, gc = torch.zeros(M, device='cuda'), torch.zeros(M, 3, device='cuda')
    mod.composite_rays_train_backward(gws.cuda(), gim.cuda(), sf, cf, df, rays, ws, im, M, N, thr, gs, gc)
    _sync()
    return ws.cpu(), dp.cpu(), im.cpu(), gs.cpu(), gc.cpu()


def _unpack(gs, gc, slot, valid, M):
    N, T = valid.shape
    keep = slot < M
    gsp, gcp = torch.zeros(N, T), torch.zeros(N, T, 3)
    idx = torch.nonzero(valid)
    gsp[idx[keep, 0], idx[keep, 1]] = gs[slot[keep]]
    gcp[idx[keep, 0], idx[keep, 1]] = gc[slot[keep]]
    return gsp, gcp


@pytest.mark.parametrize('overflow', (False, True))
@pytest.mark.parametrize('thr', (0.0, 1e-4, 1e-2, 1.0))
def test_composite_rays_train(thr, overflow, ref):
    """forward and backward within the fp64 bound of the truncated forward and its autograd derivative; rays of 0 and 1 samples,
    rays past M composite to exact zeros and take no gradient"""
    from sparsefusion_b200 import _raymarching as ours
    N, T = 3000, 320
    s, c, dl, counts = _comp_rays(N, T, seed=int(thr * 1e4) + overflow)
    sf, cf, df, rays, M, past, slot, valid = _pack(s, c, dl, counts, 11, overflow)
    assert past.any() == overflow
    g = torch.Generator().manual_seed(12)
    gws, gim = torch.randn(N, generator=g), torch.randn(N, 3, generator=g)
    eff = torch.where(past, torch.zeros_like(counts), counts)
    r = gm.composite_train_fp64(s.cuda(), c.cuda(), dl.cuda(), eff.cuda(), thr, gws.cuda(), gim.cuda())
    assert (r['ambiguous'] | (r['K64'] == r['K32'])).all()
    ok = (~r['ambiguous']).cpu()
    assert ok.float().mean() > 0.98

    def check(tag, ws, dp, im, gs, gc):
        for name, got in (('ws', ws), ('depth', dp), ('image', im)):
            gm.assert_within(f'{tag} {name}', got[ok], r[name].cpu()[ok], 0, 0, r[name + '_err'].cpu()[ok])
        gsp, gcp = _unpack(gs, gc, slot, valid, M)
        gm.assert_within(f'{tag} grad_sigmas', gsp[ok], r['g_sigma'].cpu()[ok], 0, 0, r['g_sigma_err'].cpu()[ok])
        gm.assert_within(f'{tag} grad_rgbs', gcp[ok], r['g_rgb'].cpu()[ok], 0, 0, r['g_rgb_err'].cpu()[ok])
        assert (ws[past] == 0).all() and (im[past] == 0).all() and (dp[past] == 0).all()
        own = torch.zeros(M, dtype=torch.bool)
        for i, o, n in rays.long().tolist():
            if n > 0 and o + n <= M:
                own[o:o + n] = True
        assert (gs[~own] == 0).all() and (gc[~own] == 0).all(), 'slots of rays past M took gradient'

    check('ours', *_composite_train(ours, sf, cf, df, rays, M, N, thr, gws, gim))
    RAN['composite'].add(('train', thr, overflow))
    # through the product's autograd function: a depth gradient is dropped, as the reference drops it
    import sparsefusion_b200.raymarching as rm
    sg, cg = sf.cuda().requires_grad_(True), cf.cuda().requires_grad_(True)
    ws, dp, im = rm.composite_rays_train(sg, cg, df.cuda(), rays.cuda(), thr)
    ((im * gim.cuda()).sum() + (ws * gws.cuda()).sum() + (dp * 3.0).sum()).backward()
    check('autograd', ws.detach().cpu(), dp.detach().cpu(), im.detach().cpu(), sg.grad.cpu(), cg.grad.cpu())
    m = _need(ref, 'march')
    check('reference build', *_composite_train(m, sf, cf, df, rays, M, N, thr, gws, gim))


def _composite_inf(mod, n, S, thr, alive, rt, s, c, dl, ws, dp, im):
    alive, rt, ws, dp, im = alive.clone().cuda(), rt.clone().cuda(), ws.clone().cuda(), dp.clone().cuda(), im.clone().cuda()
    mod.composite_rays(n, S, thr, alive, rt, s.cuda(), c.cuda(), dl.cuda(), ws, dp, im)
    _sync()
    return alive.cpu(), rt.cpu(), ws.cpu(), dp.cpu(), im.cpu()


@pytest.mark.parametrize('thr', (0.0, 1e-4, 1e-2, 1.0))
def test_composite_rays_inference(thr, ref):
    """one iteration of the inference loop from a running state: samples with delta 0 end the ray before it is composited"""
    from sparsefusion_b200 import _raymarching as ours
    n, S, R = 2000, 8, 2600
    s, c, dl, _ = _comp_rays(n, S, seed=21)
    dl[:40, 2:] = 0
    g = torch.Generator().manual_seed(22)
    ids = torch.randperm(R, generator=g)[:n].int()
    ws = (torch.rand(R, generator=g) * 0.95).float()
    ws[ids[:300].long()] = 0
    dp, im, rt = torch.rand(R, generator=g), torch.rand(R, 3, generator=g) * 0.5, torch.rand(R, generator=g) * 3
    out = _composite_inf(ours, n, S, thr, ids, rt, s, c, dl, ws, dp, im)
    i = ids.long()
    r = gm.composite_inference_fp64(s, c, dl, ws[i], dp[i], im[i], rt[i], thr)
    ok = ~r['ambiguous']
    assert ok.float().mean() > 0.98
    assert torch.equal((out[0] >= 0)[ok], r['alive'][ok])
    for name, got in (('ws', out[2][i]), ('depth', out[3][i]), ('image', out[4][i])):
        gm.assert_within(name, got[ok], r[name][ok], 0, 0, r[name + '_err'][ok])
    RAN['inference'].add(thr)
    m = _need(ref, 'march')
    theirs = _composite_inf(m, n, S, thr, ids, rt, s, c, dl, ws, dp, im)
    assert torch.equal(theirs[0], out[0]) and torch.equal(theirs[1], out[1])


def _field(xyzs):
    """a deterministic density / colour of the marched points (fp32, on their device)"""
    s = 8 * (torch.sin(3 * xyzs[:, 0]) * torch.cos(2 * xyzs[:, 1]) + 1) * (xyzs[:, 2].abs() < 2.5)
    return s.contiguous(), torch.sigmoid(xyzs * 2).contiguous()


@pytest.mark.parametrize('cfg', [dict(BASE, steps=1024), dict(C=5, bound=16.0, H=64, dtg=1 / 64, steps=256, noise=False, overflow=False, occ=0.5)],
                         ids=('base', 'cascade5-dtgamma'))
@pytest.mark.parametrize('thr', (1e-4, 1e-2))
def test_inference_loop_vs_reference_build(cfg, thr, ref, golden_dir):
    """NeRFRenderer.run_cuda's eval loop (renderer_df.py:521-557) run with our operators and the reference build side by side: equal
    alive sets and rays_t after every iteration, each iteration's compositing within the fp64 bound"""
    from sparsefusion_b200 import _raymarching as ours
    m = _need(ref, 'march')
    ro, rd, bf, _ = _march_inputs(cfg, golden_dir, N=1024)
    N, b = ro.shape[0], cfg['bound']
    bft, rot, rdt = torch.from_numpy(bf).cuda(), ro.cuda(), rd.cuda()
    nears, fars = torch.empty(N, device='cuda'), torch.empty(N, device='cuda')
    ours.near_far_from_aabb(rot, rdt, torch.tensor([-b, -b, -b, b, b, b], device='cuda'), N, MIN_NEAR, nears, fars)
    state = {k: (torch.arange(N, dtype=torch.int32, device='cuda'), nears.clone(), torch.zeros(N, device='cuda'), torch.zeros(N, device='cuda'),
                 torch.zeros(N, 3, device='cuda')) for k in ('ours', 'ref')}
    step, iters = 0, 0
    while step < cfg['steps']:
        alive = state['ours'][0].clone()                                  # composite_rays marks finished rays in place
        n_alive = alive.shape[0]
        if n_alive == 0:
            break
        n_step = max(min(N // n_alive, 8), 1)
        outs = {}
        for k, mod in (('ours', ours), ('ref', m)):
            al, rt, ws, dp, im = state[k]
            assert torch.equal(al, alive)
            xyzs, dirs, deltas = (torch.zeros(n_alive * n_step, w, device='cuda') for w in (3, 3, 2))
            mod.march_rays(n_alive, n_step, al, rt, rot, rdt, b, cfg['dtg'], cfg['steps'], cfg['C'], cfg['H'], bft, nears, fars, xyzs, dirs,
                           deltas, torch.zeros(n_alive, device='cuda'))
            sig, rgb = _field(xyzs)
            before = (ws.clone(), dp.clone(), im.clone(), rt.clone())
            mod.composite_rays(n_alive, n_step, thr, al, rt, sig, rgb, deltas, ws, dp, im)
            _sync()
            outs[k] = (xyzs, deltas, sig, rgb, before)
        assert torch.equal(outs['ours'][0], outs['ref'][0]) and torch.equal(outs['ours'][1], outs['ref'][1]), f'march_rays, iteration {iters}'
        assert torch.equal(state['ours'][0], state['ref'][0]), f'alive set, iteration {iters}'
        assert torch.equal(state['ours'][1], state['ref'][1]), f'rays_t, iteration {iters}'
        xyzs, deltas, sig, rgb, (ws0, d0, im0, rt0) = outs['ours']
        i = alive.long()
        r = gm.composite_inference_fp64(sig.view(n_alive, n_step), rgb.view(n_alive, n_step, 3), deltas.view(n_alive, n_step, 2), ws0[i], d0[i],
                                        im0[i], rt0[i], thr)
        ok = ~r['ambiguous']
        al, rt, ws, dp, im = state['ours']
        assert torch.equal((al >= 0)[ok], r['alive'][ok])
        for name, got in (('ws', ws[i]), ('depth', dp[i]), ('image', im[i])):
            gm.assert_within(f'{name}, iteration {iters}', got[ok], r[name][ok], 0, 0, r[name + '_err'][ok])
        for k in state:
            al = state[k][0]
            state[k] = (al[al >= 0].contiguous(),) + state[k][1:]
        step += n_step
        iters += 1
    assert iters > 3
    RAN['inference'].add(('loop', thr, cfg['C']))


# ------------------------------------------------------------------------------------------------ packbits, sph_from_ray
def test_packbits_edges(ref):
    import sparsefusion_b200.raymarching as rm
    from sparsefusion_b200 import _raymarching as ours
    g = torch.Generator().manual_seed(31)
    grid = torch.randn(3, 64 ** 3, generator=g)
    thr = 0.25
    grid[0, :4096] = thr                                                   # equal to the threshold: not occupied (strict >)
    grid[1, 100:4000:7] = float('nan')
    grid[2, :64] = float(np.nextafter(np.float32(thr), np.float32(1)))
    want = np.packbits((grid.numpy() > thr).reshape(-1), bitorder='little')
    assert np.array_equal(no.packbits(grid.numpy(), thr), want)
    got = rm.packbits(grid.cuda(), thr).cpu().numpy()
    assert np.array_equal(got, want)
    assert (got[:512] == 0).all() and (got[2 * 64 ** 3 // 8:2 * 64 ** 3 // 8 + 8] == 255).all()
    base = torch.zeros(3 * 64 ** 3 + 1, device='cuda')
    with pytest.raises(RuntimeError, match='aligned'):
        rm.packbits(base[1:].view(3, 64 ** 3), thr)                        # contiguous but 4 bytes off: must not launch
    RAN['packbits'].add('edges')
    m = _need(ref, 'march')
    b2 = torch.empty(3 * 64 ** 3 // 8, dtype=torch.uint8, device='cuda')
    m.packbits(grid.cuda(), b2.numel(), thr, b2)
    b1 = torch.empty_like(b2)
    ours.packbits(grid.cuda(), b1.numel(), thr, b1)
    assert torch.equal(b1, b2)


def test_sph_from_ray(ref):
    from sparsefusion_b200 import _raymarching as ours
    g = torch.Generator().manual_seed(41)
    N = 20000
    o = (torch.rand(N, 3, generator=g) * 2 - 1).float()
    d = torch.randn(N, 3, generator=g).float()
    d[:100, 0] = 0
    d[100:200, :2] = 0
    d[200:300] *= 7
    want, err = gm.sph_from_ray_fp64(o, d, 3.0)
    got = torch.empty(N, 2, device='cuda')
    ours.sph_from_ray(o.cuda(), d.cuda(), 3.0, N, got)
    _sync()
    gm.assert_within('sph_from_ray', got.cpu(), want, 0, 0, err)
    m = _need(ref, 'march')
    theirs = torch.empty(N, 2, device='cuda')
    m.sph_from_ray(o.cuda(), d.cuda(), 3.0, N, theirs)
    _sync()
    gm.assert_within('sph_from_ray (reference build)', theirs.cpu(), want, 0, 0, err)


# ------------------------------------------------------------------------------------------------ catalogue
def test_catalogue_every_variant_ran():
    """the whole matrix ran in this session (run the file whole)"""
    assert len(VARIANTS) == 80 and RAN['grid'] == set(VARIANTS), sorted(set(VARIANTS) - RAN['grid'])
    assert {1, 255, 257, 1 << 20} <= RAN['grid_B']
    want = {tuple(sorted(c.items())) for c in MARCH}
    assert RAN['march'] == want, len(want - RAN['march'])
    cover = lambda k: {dict(c)[k] for c in RAN['march']}
    assert {(dict(c)['C'], dict(c)['bound']) for c in RAN['march']} >= {(c, float(2 ** (c - 1))) for c in range(1, 6)}
    assert any(not math.log2(dict(c)['bound']).is_integer() for c in RAN['march'])
    assert cover('H') == {64, 128} and cover('dtg') == {0.0, 1 / 256, 1 / 64} and cover('steps') == {1, 16, 256, 1024}
    assert cover('noise') == {True, False} and cover('overflow') == {True, False}
    assert cover('occ') == {0.0, 0.02, 0.5, 1.0, 'update_extra_state'}
    assert RAN['composite'] == {('train', t, o) for t in (0.0, 1e-4, 1e-2, 1.0) for o in (False, True)}
    assert {0.0, 1e-4, 1e-2, 1.0} <= RAN['inference'] and len(RAN['inference']) == 8
    assert RAN['packbits'] == {'edges'}
    print(f"catalogue: {len(RAN['grid'])} grid-encoder variants, {len(RAN['march'])} marching configurations, "
          f"{len(RAN['composite'])} train compositing and {len(RAN['inference'])} inference compositing cases")
