"""Mesh texture, host side: the atlas and ownership contract as the oracle states it (oracle/texture_oracle.py), the size limits shared by the
library and the oracle, the textured OBJ / MTL / PNG writer, and the refusals that need no GPU."""
import numpy as np
import pytest
import torch


def _used_cells(F, T):
    from oracle import texture_oracle as to
    c, n = to.atlas_cell(F, T), to.atlas_cols(F)
    return c, n, (F + 1) // 2


@pytest.mark.parametrize('F,T', [(1, 16), (2, 16), (7, 64), (8, 64), (31, 100), (32, 16), (1001, 512), (1000, 333)])
def test_every_texel_of_a_used_cell_has_one_owner(F, T):
    from oracle import texture_oracle as to
    c, n, cells = _used_cells(F, T)
    own = to.ownership(F, T)
    assert own.shape == (T, T) and own.max() < F
    for k in range(cells):
        x0, y0 = (k % n) * c, (k // n) * c
        blk = own[y0:y0 + c, x0:x0 + c]
        i, j = np.meshgrid(np.arange(c), np.arange(c), indexing='xy')
        lower = i + j + 1 < c
        assert (blk[lower] == 2 * k).all()
        assert (blk[~lower] == (2 * k + 1 if 2 * k + 1 < F else -1)).all()
    # everything outside the used cells is unowned, and each triangle owns texels
    mask = np.zeros((T, T), bool)
    for k in range(cells):
        mask[(k // n) * c:(k // n + 1) * c, (k % n) * c:(k % n + 1) * c] = True
    assert (own[~mask] == -1).all()
    assert set(np.unique(own[own >= 0])) == set(range(F))


@pytest.mark.parametrize('F', [31, 32])
def test_bilinear_taps_stay_inside_the_owning_triangle(F):
    """n = 4 cells per row, T = 4c: every cell size 4..32, odd F (last cell half used) and even F.  Random points of every triangle, its
    corners and its edge midpoints: each texel a bilinear lookup weights nonzero is owned by that triangle."""
    from oracle import texture_oracle as to
    rng = np.random.default_rng(F)
    for c in range(4, 33):
        T = 4 * c
        assert to.atlas_cell(F, T) == c
        uv, own = to.uv_atlas(F, T), to.ownership(F, T)
        lam = rng.dirichlet(np.ones(3), size=(F, 400))
        special = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [.5, .5, 0], [0, .5, .5], [.5, 0, .5], [1 / 3, 1 / 3, 1 / 3]])
        lam = np.concatenate([lam, np.broadcast_to(special, (F, len(special), 3))], axis=1)
        p = np.einsum('fsi,fic->fsc', lam, uv).reshape(-1, 2)
        taps = to.bilinear_taps(p)
        tri = np.repeat(np.arange(F), lam.shape[1])
        assert (taps >= 0).all() and (taps < T).all()
        got = own[taps[..., 1], taps[..., 0]]
        bad = got != tri[:, None]
        assert not bad.any(), (c, p[bad.any(1)][:5])


def test_closest_barycentrics_are_the_closest_point():
    """the oracle's closest-point test against a dense sampling of the triangle, for points around it in every Voronoi region"""
    from oracle import texture_oracle as to
    rng = np.random.default_rng(3)
    a, b, c = np.array([0.5, 0.5]), np.array([6.5, 0.5]), np.array([0.5, 6.5])
    p = rng.uniform(-4, 11, (3000, 2))
    lam = to.closest_barycentrics(p, *(np.broadcast_to(q, p.shape) for q in (a, b, c)))
    assert (lam >= -1e-12).all() and np.allclose(lam.sum(1), 1)
    q = lam @ np.stack([a, b, c])
    g = np.linspace(0, 1, 161)
    s, r = np.meshgrid(g, g)
    keep = s + r <= 1
    samples = a + s[keep, None] * (b - a) + r[keep, None] * (c - a)
    dense = np.sqrt(((p[:, None] - samples[None]) ** 2).sum(-1)).min(1)
    got = np.sqrt(((p - q) ** 2).sum(-1))
    assert (got <= dense + 1e-12).all() and (dense - got).max() < 6 / 160
    inside = rng.dirichlet(np.ones(3), 100)
    assert np.allclose(to.closest_barycentrics(inside @ np.stack([a, b, c]), *(np.broadcast_to(q, (100, 2)) for q in (a, b, c))), inside)


def test_size_limits_agree_between_library_and_oracle():
    from oracle import texture_oracle as to
    from sparsefusion_b200 import _lib, mesh
    lib = _lib.load()
    for F in (0, 1, 2, 3, 7, 8, 31, 32, 33, 1000, 12345, 200000, 2 ** 31 - 1):
        for T in (15, 16, 17, 100, 1024, 2048, 8191, 8192, 8193):
            try:
                want = to.atlas_cell(F, T)
            except ValueError:
                want = 0
            assert lib.sfb_mesh_atlas_cell(F, T) == want, (F, T)
            if want:
                assert mesh._atlas_cell(F, T) == want
            else:
                with pytest.raises(ValueError):
                    mesh._atlas_cell(F, T)
    with pytest.raises(ValueError, match='16..8192'):
        mesh._atlas_cell(8, 15)
    with pytest.raises(ValueError, match='16..8192'):
        mesh._atlas_cell(8, 8193)
    with pytest.raises(ValueError, match='texture_size >= 20 is needed'):        # 33 triangles: 17 cells, 5 per row, 3 texels each at 16
        mesh._atlas_cell(33, 16)
    with pytest.raises(ValueError, match='texture_size >= 20 is needed'):
        to.atlas_cell(33, 16)
    assert mesh._atlas_cell(32, 16) == 4 and lib.sfb_mesh_atlas_cell(-1, 64) == 0


def _textured(tmp_path, F, T, V=None, seed=0):
    from sparsefusion_b200.mesh import write_textured_obj
    from oracle import texture_oracle as to
    rng = np.random.default_rng(seed)
    V = V if V is not None else F + 5
    verts = (rng.standard_normal((V, 3)) * 2).astype(np.float32)
    tris = rng.integers(0, max(V, 1), (F, 3)).astype(np.int32)
    uv = to.uv_atlas(F, T).astype(np.float32)
    tex = rng.integers(0, 256, (T, T, 3)).astype(np.uint8)
    write_textured_obj(str(tmp_path), torch.from_numpy(verts), torch.from_numpy(tris), torch.from_numpy(uv), torch.from_numpy(tex))
    return verts, tris, uv, tex


def test_write_textured_obj_round_trips(tmp_path):
    from PIL import Image
    from oracle import texture_oracle as to
    F, T = 101, 256
    verts, tris, uv, tex = _textured(tmp_path, F, T)
    v, vt, t, tt, lines = to.read_textured_obj(str(tmp_path / 'mesh.obj'))
    assert lines[0] == 'mtllib mesh.mtl'
    assert len(lines) == 1 + len(verts) + 3 * F + 1 + F
    assert lines[1 + len(verts) + 3 * F] == 'usemtl mat0'
    kinds = [l.split()[0] for l in lines]
    assert kinds == ['mtllib'] + ['v'] * len(verts) + ['vt'] * (3 * F) + ['usemtl'] + ['f'] * F
    assert np.abs(v - verts).max() <= 5e-7 + 1e-9
    assert (t == tris).all() and (tt == np.arange(3 * F).reshape(F, 3)).all()
    want = np.stack([uv[..., 0] / T, 1 - uv[..., 1].astype(np.float64) / T], -1).reshape(-1, 2)
    assert np.abs(vt - want).max() <= 5e-7 + 1e-12
    first_vt = lines[1 + len(verts)].split()
    assert len(first_vt) == 3 and all(len(x.split('.')[1]) == 6 for x in first_vt[1:])
    f0 = lines[-F].split()
    assert f0[1:] == [f'{tris[0, i] + 1}/{i + 1}' for i in range(3)]
    assert '  ' not in open(tmp_path / 'mesh.obj').read()
    assert to.read_mtl(str(tmp_path / 'mesh.mtl')) == ['newmtl mat0', 'Ka 1.000000 1.000000 1.000000', 'Kd 1.000000 1.000000 1.000000',
                                                      'Ks 0.000000 0.000000 0.000000', 'd 1.000000', 'illum 1', 'Ns 0.000000', 'map_Kd albedo.png']
    img = Image.open(tmp_path / 'albedo.png')
    assert img.mode == 'RGB' and img.size == (T, T)
    assert (np.asarray(img) == tex).all()


def test_empty_mesh_writes_vertices_only(tmp_path):
    from PIL import Image
    from oracle import texture_oracle as to
    from sparsefusion_b200.mesh import write_textured_obj
    write_textured_obj(str(tmp_path), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), np.zeros((0, 3, 2), np.float32),
                       np.zeros((16, 16, 3), np.uint8))
    assert open(tmp_path / 'mesh.obj').read() == 'mtllib mesh.mtl\n'
    verts, *_ = _textured(tmp_path, 0, 16, V=4)
    v, vt, t, tt, lines = to.read_textured_obj(str(tmp_path / 'mesh.obj'))
    assert len(v) == 4 and len(vt) == 0 and len(t) == 0 and [l.split()[0] for l in lines] == ['mtllib'] + ['v'] * 4
    assert Image.open(tmp_path / 'albedo.png').size == (16, 16)


def test_write_textured_obj_rejects_bad_input(tmp_path):
    from sparsefusion_b200.mesh import write_textured_obj
    v, t, uv = np.zeros((3, 3), np.float32), np.array([[0, 1, 2]], np.int32), np.zeros((1, 3, 2), np.float32)
    with pytest.raises(ValueError, match='uint8'):
        write_textured_obj(str(tmp_path), v, t, uv, np.zeros((16, 16, 3), np.float32))
    with pytest.raises(ValueError, match='corners'):
        write_textured_obj(str(tmp_path), v, t, np.zeros((2, 3, 2), np.float32), np.zeros((16, 16, 3), np.uint8))
    with pytest.raises(ValueError, match='out of range'):
        write_textured_obj(str(tmp_path), v, t + 1, uv, np.zeros((16, 16, 3), np.uint8))


def test_cpu_tensors_are_refused():
    from sparsefusion_b200 import mesh
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    net = NeRFNetwork(get_default_torch_ngp_opt())
    verts, tris = torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(RuntimeError):
        mesh.bake_albedo(net, verts, tris, 64)
    with pytest.raises(RuntimeError):
        mesh.uv_atlas(8, 64, device='cpu')
    with pytest.raises(RuntimeError):
        net.export_mesh('/nonexistent-dir', grid_resolution=8, texture_size=64)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from sparsefusion_b200 import _lib
    with pytest.raises(RuntimeError, match='no atlas'):
        _lib.call('sfb_mesh_uv_atlas', 8, 15, 16, None)
    with pytest.raises(RuntimeError, match='no atlas'):
        _lib.call('sfb_mesh_uv_atlas', 33, 16, 16, None)
    with pytest.raises(RuntimeError, match='negative'):
        _lib.call('sfb_mesh_uv_atlas', -1, 64, 16, None)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_mesh_uv_atlas', 8, 64, None, None)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_mesh_texel_points', None, None, 8, 64, 0, 4, 16, 16, None)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_mesh_texel_points', 16, 16, 0, 64, 0, 4, None, 16, None)
    with pytest.raises(RuntimeError, match='outside'):
        _lib.call('sfb_mesh_texel_points', 16, 16, 8, 64, 60, 5, 16, 16, None)
    with pytest.raises(RuntimeError, match='outside'):
        _lib.call('sfb_mesh_texel_points', 16, 16, 8, 64, -1, 5, 16, 16, None)
    with pytest.raises(RuntimeError, match='no atlas'):
        _lib.call('sfb_mesh_texel_points', 16, 16, 8, 8193, 0, 5, 16, 16, None)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_mesh_texture_pack', None, 16, 10, 16, None)
    with pytest.raises(RuntimeError, match='negative'):
        _lib.call('sfb_mesh_texture_pack', 16, 16, -1, 16, None)
    # empty work returns before touching the device
    _lib.call('sfb_mesh_uv_atlas', 0, 64, None, None)
    _lib.call('sfb_mesh_texel_points', None, None, 8, 64, 3, 0, None, None, None)
    _lib.call('sfb_mesh_texture_pack', None, None, 0, None, None)


def test_cli_rejects_a_bad_texture_size(tmp_path, capsys):
    from sparsefusion_b200 import mesh
    ckpt = tmp_path / 'scene.pt'
    ckpt.write_bytes(b'')
    with pytest.raises(SystemExit) as e:
        mesh.main([str(ckpt), str(tmp_path / 'out'), '--texture-size', '8'])
    assert e.value.code == 2
    assert '--texture-size must be in 16..8192 (got 8)' in capsys.readouterr().err
    assert not (tmp_path / 'out').exists()
