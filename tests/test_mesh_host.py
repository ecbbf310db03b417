"""Mesh extraction, host side: the marching-cubes contract as the oracle states it (topology, orientation, volume), the triangle table shared
by the kernels and the oracle, the OBJ writer, and the refusals that need no GPU."""
import importlib.util
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen_tables():
    spec = importlib.util.spec_from_file_location('gen_mc_tables', os.path.join(ROOT, 'tools', 'gen_mc_tables.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _closed_oriented(tris):
    from oracle import mesh_oracle as mo
    ucount, dcount = mo.edge_face_counts(tris)
    return bool((ucount == 2).all() and (dcount == 1).all())


def test_sphere_is_a_closed_outward_2_manifold():
    """-SDF of a sphere of radius 20 voxels in 64^3: every edge in exactly two faces, each directed edge once (consistent orientation),
    chi = V - E + F = 2, and the divergence-theorem volume is positive (faces point outward, toward decreasing value) and within 1% of
    4/3 pi r^3.  The triangles are chords of the sphere (edges up to sqrt(2) voxels, sagitta <= 2 / (8 r) = 0.0125 voxels), which puts the
    expected deficit near 3 x 0.0125 / 20 = 0.2%; 1% leaves room for the linear interpolation of the distance along each edge."""
    from oracle import mesh_oracle as mo
    verts, tris = mo.marching_cubes(mo.sphere(64, 20.0), 0.0)
    assert len(tris) > 1000 and _closed_oriented(tris)
    assert len(np.unique(tris)) == len(verts)                   # every vertex is used
    assert mo.euler_characteristic(verts, tris) == 2
    vol, want = mo.signed_volume(verts, tris), 4.0 / 3.0 * np.pi * 20.0 ** 3
    assert vol > 0 and abs(vol - want) < 0.01 * want, (vol, want)


def test_torus_has_genus_one():
    from oracle import mesh_oracle as mo
    verts, tris = mo.marching_cubes(mo.torus(64, 16.0, 6.0), 0.0)
    assert _closed_oriented(tris)
    assert mo.euler_characteristic(verts, tris) == 0
    assert mo.signed_volume(verts, tris) > 0


@pytest.mark.parametrize('seed', [0, 1])
def test_every_case_closes_on_random_volumes(seed):
    """noise padded by a below-iso shell: all 256 cases and both kinds of ambiguous face occur, and the surface must still be closed and
    consistently oriented (the face rule of the table is what makes neighbouring cells agree)"""
    from oracle import mesh_oracle as mo
    rng = np.random.default_rng(seed)
    vol = np.full((22, 25, 28), -1.0)
    vol[1:-1, 1:-1, 1:-1] = rng.standard_normal((20, 23, 26))
    below = vol <= 0.0
    case = sum(below[dx:21 + dx, dy:24 + dy, dz:27 + dz].astype(int) << (dx | dy << 1 | dz << 2)
               for dx in (0, 1) for dy in (0, 1) for dz in (0, 1))
    assert len(np.unique(case)) == 256
    verts, tris = mo.marching_cubes(vol, 0.0)
    assert _closed_oriented(tris)
    # integer volume with an integer isovalue: many corners equal iso, and v <= iso counts them as below
    ivol = np.pad(rng.integers(0, 4, (10, 11, 12)).astype(np.float64), 1, constant_values=-1.0)
    verts, tris = mo.marching_cubes(ivol, 2.0)
    assert _closed_oriented(tris)
    on_corner = (verts == np.round(verts)).all(axis=1)         # t = 0: the lower end sits exactly at iso
    assert on_corner.any() and not on_corner.all()


def test_vertex_and_triangle_order_follow_the_lattice():
    from oracle import mesh_oracle as mo
    vol = mo.sphere(24, 7.0)
    verts, tris = mo.marching_cubes(vol, 0.0)
    lo = np.floor(verts + 1e-12).astype(int)
    key = np.ravel_multi_index(lo.T, vol.shape)
    assert (np.diff(key) >= 0).all()                            # lattice order of the owning point
    assert np.abs(verts - np.round(verts)).max() < 1.0 and (verts >= 0).all()
    # a single corner above iso: one triangle around it, facing away from it (toward decreasing value)
    one = np.zeros((2, 2, 2))
    one[0, 0, 0] = 1.0
    v1, t1 = mo.marching_cubes(one, 0.5)
    assert v1.shape == (3, 3) and t1.shape == (1, 3)
    a, b, c = v1[t1[0]]
    n = np.cross(b - a, c - a)
    assert np.dot(n, (a + b + c) / 3 - np.zeros(3)) > 0
    # constant and all-below volumes have no surface
    for vol in (np.full((5, 6, 7), 3.0), np.full((5, 6, 7), -3.0)):
        v, t = mo.marching_cubes(vol, float(vol.mean()))
        assert v.shape == (0, 3) and t.shape == (0, 3)


def test_triangle_tables_agree_between_kernels_oracle_and_generator():
    from oracle import mesh_oracle as mo
    gen = _gen_tables()
    tab, cnt = gen.tables()
    assert [tuple(int(e) for e in row if e >= 0) for row in tab] == [tuple(r) for r in mo.TRI_TABLE]
    assert [len(r) // 3 for r in mo.TRI_TABLE] == cnt.tolist()
    with open(os.path.join(ROOT, 'sparsefusion_b200', 'csrc', 'mc_tables.cuh')) as f:
        assert f.read() == gen.header_text()
    # a case uses exactly the edges whose two corners differ, each once
    for c in range(256):
        crossing = [e for e in range(12) if ((c >> gen.edge_corners(e)[0]) & 1) != ((c >> gen.edge_corners(e)[1]) & 1)]
        assert sorted(set(mo.TRI_TABLE[c])) == crossing


def test_write_obj_round_trips(tmp_path):
    from oracle import mesh_oracle as mo
    from sparsefusion_b200.mesh import write_obj
    rng = np.random.default_rng(4)
    verts = np.concatenate([rng.random((500, 3)) * 1023, rng.standard_normal((100, 3)) * 5, [[0, 0, 0], [1e-7, -1e-7, 0.5], [1023, 0.000001, 10]]])
    verts = verts.astype(np.float32)
    tris = rng.integers(0, len(verts), (700, 3)).astype(np.int32)
    path = str(tmp_path / 'm.obj')
    write_obj(path, torch.from_numpy(verts), torch.from_numpy(tris))
    v, t = mo.read_obj(path)
    assert np.abs(v - verts.astype(np.float64)).max() <= 5e-7 + 1e-9
    assert (t == tris).all()
    lines = open(path).read().splitlines()
    assert len(lines) == len(verts) + len(tris)
    assert lines[0].startswith('v ') and lines[-1].startswith('f ') and '  ' not in open(path).read()
    assert lines[len(verts) - 3] == 'v 0.000000 0.000000 0.000000'
    assert lines[len(verts)].split()[1:] == [str(i + 1) for i in tris[0]]
    # empty mesh: empty file
    write_obj(path, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    assert open(path).read() == ''


def test_cpu_tensors_are_refused():
    from sparsefusion_b200 import mesh
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    vol = torch.zeros(8, 8, 8)
    with pytest.raises(RuntimeError):
        mesh.marching_cubes(vol, 0.0)
    with pytest.raises(RuntimeError):
        mesh.smooth_gaussian(vol)
    with pytest.raises(RuntimeError):
        mesh.volume_mean_std(vol)
    for cuda_ray in (False, True):
        opt = get_default_torch_ngp_opt()
        opt.cuda_ray = cuda_ray
        with pytest.raises(RuntimeError):
            NeRFNetwork(opt).export_mesh('/nonexistent-dir', grid_resolution=8)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from sparsefusion_b200 import _lib
    lib = _lib.load()
    assert lib.sfb_marching_cubes_scratch_bytes(1025, 8, 8) == 0 and lib.sfb_marching_cubes_scratch_bytes(0, 8, 8) == 0
    with pytest.raises(RuntimeError, match='outside 1..1024'):
        _lib.call('sfb_marching_cubes_count', 16, 1025, 8, 8, 0.0, 16, 16, None)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_marching_cubes_emit', None, 8, 8, 8, 0.0, 16, 16, 16, None)
    with pytest.raises(RuntimeError, match='sigma'):
        _lib.call('sfb_gaussian_filter3d', 16, 32, 48, 8, 8, 8, 0.0, None)
    with pytest.raises(RuntimeError, match='sigma'):
        _lib.call('sfb_gaussian_filter3d', 16, 32, 48, 8, 8, 8, 9.0, None)
    with pytest.raises(RuntimeError, match='distinct'):
        _lib.call('sfb_gaussian_filter3d', 16, 16, 48, 8, 8, 8, 1.5, None)
    with pytest.raises(RuntimeError, match='empty'):
        _lib.call('sfb_volume_mean_std', 16, 0, 16, 16, None)


def test_cli_rejects_a_missing_checkpoint(tmp_path, capsys):
    from sparsefusion_b200 import mesh
    missing = str(tmp_path / 'no-such-scene.pt')
    with pytest.raises(SystemExit) as e:
        mesh.main([missing, str(tmp_path / 'out')])
    assert e.value.code == 2
    assert f'checkpoint not found: {missing}' in capsys.readouterr().err
    assert not (tmp_path / 'out').exists()
