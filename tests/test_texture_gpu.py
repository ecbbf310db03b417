"""Mesh texture on the GPU (csrc/texture.cu, mesh.uv_atlas / bake_albedo / write_textured_obj, export_mesh(texture_size=T)) against the fp64
restatement of header section 12 (oracle/texture_oracle.py) and the fp64 NGP field oracle.

Bars: uv within 1e-6 texel and owner exactly equal to the oracle; the texel surface points within 1e-5 x bound of the fp64 closest-point
barycentrics; texture bytes exactly trunc(255 albedo) of sfb_ngp_field_forward at the kernel's points, whose albedo is within 2e-4 relative
of the oracle field (the lattice test's bar); colours recomputed in fp64 from the written mesh.obj within 1 LSB of albedo.png; repeated
exports byte-identical.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUND = 4.0


def _net(seed=0, emb_range=0.5):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    net = NeRFNetwork(get_default_torch_ngp_opt())
    p = no.make_field_params(seed=seed, emb_range=emb_range)
    sd = net.state_dict()
    sd.update(p)
    net.load_state_dict(sd)
    return net.cuda().eval(), p


def _mc_mesh(net, R):
    from sparsefusion_b200 import mesh
    sm = mesh.smooth_gaussian(mesh.density_lattice(net, R), 1.5)
    mean, std = mesh.volume_mean_std(sm)
    verts, tris = mesh.marching_cubes(sm, mean + 0.25 * std)
    return verts / (R - 1) * (2 * BOUND) - BOUND, tris


def _synthetic(F, seed=0):
    rng = np.random.default_rng(seed)
    V = max(F + 2, 3)
    verts = torch.from_numpy(rng.uniform(-3, 3, (V, 3)).astype(np.float32)).cuda()
    tris = torch.from_numpy(rng.integers(0, V, (F, 3)).astype(np.int32)).cuda()
    return verts, tris


def _field_rgb(net, pts):
    from sparsefusion_b200 import _lib as lib
    emb, w0, b0, w1, b1, w2, b2 = net._field_params()
    enc = net.encoder
    f = lib.fptr
    pts = pts.contiguous()
    sigma, rgb = torch.empty(pts.shape[0], device='cuda'), torch.empty(pts.shape[0], 3, device='cuda')
    lib.call('sfb_ngp_field_forward', f(pts), None, None, None, 0, pts.shape[0], f(emb), lib.iptr(enc.offsets), float(np.log2(enc.per_level_scale)),
             int(enc.base_resolution), float(net.bound), f(w0), f(b0), f(w1), f(b1), f(w2), f(b2), f(sigma), f(rgb), lib.stream())
    return rgb


def _texel_points(verts, tris, T):
    from sparsefusion_b200 import _lib as lib
    F = tris.shape[0]
    owner = torch.empty(T, T, dtype=torch.int32, device='cuda')
    xyz = torch.full((T, T, 3), 7.0, device='cuda')
    lib.call('sfb_mesh_texel_points', verts.data_ptr() if F else None, tris.data_ptr() if F else None, F, T, 0, T, owner.data_ptr(), xyz.data_ptr(),
             lib.stream())
    return owner, xyz


CASES = [('mc48', 512), ('mc128', 1024), ('F0', 16), ('F1', 16), ('F2', 16), ('F7', 16), ('F7', 40)]


@pytest.mark.parametrize('case,T', CASES)
def test_atlas_texel_points_and_texture_match_the_oracle(case, T):
    from _helpers import device_level_scales
    from oracle import ngp_oracle as no, texture_oracle as to
    from sparsefusion_b200 import mesh
    net, p = _net()
    verts, tris = _mc_mesh(net, int(case[2:])) if case.startswith('mc') else _synthetic(int(case[1:]))
    F = tris.shape[0]
    print(f'  {case}: {verts.shape[0]} vertices, {F} triangles, T = {T}')
    vn, tn = verts.cpu().double().numpy(), tris.cpu().numpy()
    # atlas
    uv = mesh.uv_atlas(F, T)
    assert uv.shape == (F, 3, 2) and uv.dtype == torch.float32
    assert np.abs(uv.cpu().double().numpy() - to.uv_atlas(F, T)).max(initial=0) <= 1e-6
    # texel points
    owner, xyz = _texel_points(verts, tris, T)
    wo, _, wx = to.texel_points(vn, tn, T)
    assert (owner.cpu().numpy() == wo).all()
    err = np.abs(xyz.cpu().double().numpy() - wx).max()
    print(f'  texel points: {(wo >= 0).sum()} owned, max |xyz - oracle| {err:.2e}')
    assert err <= 1e-5 * BOUND
    # texture: trunc(255 albedo) of the field kernel at the kernel's points, in slabs that do and do not divide T
    uv2, tex, own2 = mesh.bake_albedo(net, verts, tris, T)
    assert torch.equal(uv2, uv) and torch.equal(own2, owner)
    rgb = _field_rgb(net, xyz.reshape(-1, 3)).reshape(T, T, 3)
    want = torch.where(owner[..., None] >= 0, (rgb * 255).to(torch.uint8), torch.zeros_like(rgb, dtype=torch.uint8))
    assert torch.equal(tex, want)
    for rows in (7, T):
        assert torch.equal(mesh.bake_albedo(net, verts, tris, T, rows=rows)[1], tex)
    if F == 0:
        assert not tex.any() and (owner == -1).all()
        return
    # the field's albedo against the fp64 oracle at (a sample of) the owned texels' points
    sel = torch.nonzero(owner.reshape(-1) >= 0).reshape(-1)
    sel = sel[torch.randperm(sel.numel(), generator=torch.Generator().manual_seed(0))[:200000].to(sel.device)]
    field = no.Field({k: v.clone() for k, v in p.items()}, level_scales=device_level_scales(no.live_geometry()))
    with torch.no_grad():
        _, ro = field.common_forward(xyz.reshape(-1, 3)[sel].cpu())
    got = rgb.reshape(-1, 3)[sel].cpu().double()
    rel = ((got - ro.double()).norm() / ro.double().norm()).item()
    print(f'  albedo vs oracle field: rel {rel:.2e}')
    assert rel < 2e-4


@pytest.mark.parametrize('R,T', [(48, 1000), (128, 2000)])
def test_bilinear_taps_from_the_written_obj_stay_in_the_owning_triangle(R, T, tmp_path):
    """T divides 500000, so every vt = (half-integer texel) / T is exact in the OBJ's 6 decimals"""
    from oracle import texture_oracle as to
    from sparsefusion_b200 import mesh
    net, _ = _net()
    verts, tris = _mc_mesh(net, R)
    uv, tex, owner = mesh.bake_albedo(net, verts, tris, T)
    mesh.write_textured_obj(str(tmp_path), verts, tris, uv, tex)
    v, vt, t, tt, _ = to.read_textured_obj(str(tmp_path / 'mesh.obj'))
    F = len(t)
    assert F == tris.shape[0] and (t == tris.cpu().numpy()).all()
    corners = np.stack([vt[tt][..., 0] * T, (1 - vt[tt][..., 1]) * T], -1)                  # [F, 3, 2] texel units
    lam = np.random.default_rng(R).dirichlet(np.ones(3), size=(F, 16))
    pts = np.einsum('fsi,fic->fsc', lam, corners).reshape(-1, 2)
    taps = to.bilinear_taps(pts)
    own = owner.cpu().numpy()
    got = own[taps[..., 1], taps[..., 0]]
    assert (got == np.repeat(np.arange(F), 16)[:, None]).all()


def test_export_mesh_with_a_texture(tmp_path):
    """T = 1000 keeps every vt exact in the OBJ's 6 decimals, and the +-0.05 embeddings keep the albedo smooth enough that the vertices'
    6-decimal rounding (5e-7 world units) moves no colour by a whole LSB: with +-0.5 embeddings the seeded field's albedo changes by about
    1 LSB per 1e-6 world units"""
    from PIL import Image
    from oracle import texture_oracle as to
    net, _ = _net(emb_range=0.05)
    R, T = 64, 1000
    a, b, c = tmp_path / 'plain', tmp_path / 'tex', tmp_path / 'tex2'
    for d in (a, b, c):
        d.mkdir()
    v0, t0 = net.export_mesh(str(a), grid_resolution=R)
    assert sorted(os.listdir(a)) == ['mcubes_mesh.obj']
    v1, t1 = net.export_mesh(str(b), grid_resolution=R, texture_size=T)
    net.export_mesh(str(c), grid_resolution=R, texture_size=T)
    assert torch.equal(v0, v1) and torch.equal(t0, t1)
    assert sorted(os.listdir(b)) == ['albedo.png', 'mcubes_mesh.obj', 'mesh.mtl', 'mesh.obj']
    assert (a / 'mcubes_mesh.obj').read_bytes() == (b / 'mcubes_mesh.obj').read_bytes()
    for name in ('mesh.obj', 'mesh.mtl', 'albedo.png', 'mcubes_mesh.obj'):
        assert (b / name).read_bytes() == (c / name).read_bytes(), name
    # colours recomputed in fp64 from the written mesh.obj (vertices and vt) and the field
    img = np.asarray(Image.open(b / 'albedo.png'))
    assert img.shape == (T, T, 3)
    v, vt, t, tt, _ = to.read_textured_obj(str(b / 'mesh.obj'))
    F = len(t)
    corners = np.stack([vt[tt][..., 0] * T, (1 - vt[tt][..., 1]) * T], -1)
    own = to.ownership(F, T)
    ys, xs = np.nonzero(own >= 0)
    tri = own[ys, xs]
    lam = to.closest_barycentrics(np.stack([xs + 0.5, ys + 0.5], 1), corners[tri, 0], corners[tri, 1], corners[tri, 2])
    xyz = np.einsum('ni,nic->nc', lam, v[t[tri]])
    rgb = _field_rgb(net, torch.from_numpy(xyz.astype(np.float32)).cuda()).cpu().numpy()
    want = np.floor(255.0 * rgb.astype(np.float64))
    diff = np.abs(img[ys, xs].astype(np.int64) - want.astype(np.int64)).max()
    print(f'  export at R = {R}, T = {T}: {F} triangles, {len(ys)} owned texels, max colour difference {diff} LSB')
    assert diff <= 1
    assert not img[own < 0].any()
    assert np.abs(v - v1.cpu().double().numpy()).max() <= 5e-7 + 1e-9
    with pytest.raises(ValueError, match='16..8192'):
        net.export_mesh(str(tmp_path / 'plain'), grid_resolution=R, texture_size=8)


def test_cli_writes_a_textured_mesh(tmp_path):
    from PIL import Image
    from oracle import texture_oracle as to
    net, _ = _net(seed=1)
    ckpt = tmp_path / 'scene.pt'
    torch.save({'model_state_dict': {k: v.cpu() for k, v in net.state_dict().items()}}, str(ckpt))
    out = tmp_path / 'mesh'
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'sparsefusion_b200.mesh', str(ckpt), str(out), '--texture-size', '1024'], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr[-2000:])
    assert r.returncode == 0
    assert sorted(os.listdir(out)) == ['albedo.png', 'mcubes_mesh.obj', 'mesh.mtl', 'mesh.obj']
    v, vt, t, tt, lines = to.read_textured_obj(str(out / 'mesh.obj'))
    assert lines[0] == 'mtllib mesh.mtl' and len(t) > 0 and len(vt) == 3 * len(t)
    assert Image.open(out / 'albedo.png').size == (1024, 1024)
    here = tmp_path / 'here'
    here.mkdir()
    net.export_mesh(str(here), texture_size=1024)
    for name in ('mesh.obj', 'albedo.png', 'mcubes_mesh.obj'):
        assert (here / name).read_bytes() == (out / name).read_bytes(), name
