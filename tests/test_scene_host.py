"""Host camera maths of the per-scene preparation (sparsefusion_b200/cameras.py) against tests/golden/scene_prep.npz -- outputs of the
reference's own utils/camera_utils.py / utils/render_utils.py over a restatement of the pytorch3d primitives they touch -- and the native
scene builder's view order and shapes."""
import numpy as np
import pytest
import torch

from sparsefusion_b200 import cameras as C


@pytest.fixture(scope='module')
def g(golden_dir):
    return np.load(f'{golden_dir}/scene_prep.npz')


def _cams(g):
    t = lambda k: torch.from_numpy(g[k])
    return C.PerspectiveCameras(t('R'), t('T'), t('focal_length'), t('principal_point'), t('image_size'))


def _close(a, b, tol=1e-5):
    a = a.detach().float().numpy() if torch.is_tensor(a) else a
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max()
    assert err <= tol, err


def test_relative_vox_and_concatenated_cameras(g):
    cams = _cams(g)
    rel = C.relative_cameras(cams, [0], center_at_origin=True)
    vox = C.relative_cameras(cams, [0], center_at_origin=False)
    _close(rel.R, g['rel_R']), _close(rel.T, g['rel_T']), _close(vox.R, g['vox_R']), _close(vox.T, g['vox_T'])
    _close(cams.get_camera_center().norm(dim=1).mean(), g['cam_dist_mean'])
    path = C.PerspectiveCameras(torch.from_numpy(g['path_R']), torch.from_numpy(g['path_T']), torch.from_numpy(g['path_focal_length']),
                                torch.from_numpy(g['path_principal_point']), cams.image_size[:1].expand(50, 2))
    aug = C.concat_cameras([cams, path])
    assert len(aug) == 58 and aug.image_size.shape == (58, 2)
    _close(C.relative_cameras(aug, [0], True).R, g['aug_rel_R']), _close(C.relative_cameras(aug, [0], True).T, g['aug_rel_T'])
    _close(C.relative_cameras(aug, [0], False).R, g['aug_vox_R']), _close(C.relative_cameras(aug, [0], False).T, g['aug_vox_T'])
    aug_rel = C.relative_cameras(aug, [0], True)
    for ci in g['views']:                                       # each cached view's own frame (distillation.py:98)
        pv = C.relative_cameras(aug_rel, [int(ci)], True)
        q, ctx = pv[int(ci)], pv[[int(i) for i in g['context_idx']]]
        _close(q.R, g[f'view{ci}_query_R']), _close(q.T, g[f'view{ci}_query_T'])
        _close(ctx.R, g[f'view{ci}_ctx_R']), _close(ctx.T, g[f'view{ci}_ctx_T'])


def test_circle_path_with_seeded_jitter_and_nearest_centroid(g):
    cams = _cams(g)
    _close(C.get_nearest_centroid(cams), g['centroid'])
    torch.manual_seed(int(g['jitter_seed']))
    path = C.interpolated_path(cams, n=50, theta_offset_max=0.17)
    _close(path.R, g['path_R']), _close(path.T, g['path_T'])
    _close(path.focal_length, g['path_focal_length']), _close(path.principal_point, g['path_principal_point'])
    assert path.image_size.shape == (50, 2)
    circle = C.interpolated_path(C.relative_cameras(cams, [0], False), n=50)          # no jitter: no draw from the generator
    _close(circle.R, g['circle_R']), _close(circle.T, g['circle_T'])
    torch.manual_seed(0)
    a = torch.rand(3)
    torch.manual_seed(0)
    C.interpolated_path(cams, n=50)
    assert torch.equal(torch.rand(3), a)


def _rel_close(a, b, tol=1e-6):
    a = a.reshape(b.shape).numpy()
    err = np.abs(a - b).max() / np.abs(b).max()
    assert err <= tol, err


def test_ray_grid_restatement(g):
    """GridRaysampler of render_utils.py:38-65 restated in torch (the host path get_nearest_centroid uses) at the three sizes"""
    cams = _cams(g)
    aug = C.concat_cameras([cams, C.PerspectiveCameras(torch.from_numpy(g['path_R']), torch.from_numpy(g['path_T']),
                                                       torch.from_numpy(g['path_focal_length']), torch.from_numpy(g['path_principal_point']),
                                                       cams.image_size[:1].expand(50, 2))])
    aug_vox, aug_rel = C.relative_cameras(aug, [0], False), C.relative_cameras(aug, [0], True)
    circle = C.PerspectiveCameras(torch.from_numpy(g['circle_R']), torch.from_numpy(g['circle_T']), torch.from_numpy(g['path_focal_length']),
                                  torch.from_numpy(g['path_principal_point']))
    cdm = float(g['cam_dist_mean'])
    for cam, hw, key, n in ((aug_vox[int(g['ray_camera_128'])], 128, 'rays128', 20), (aug_rel[[int(i) for i in g['ray_cameras_32']]], 32, 'rays32', 20),
                            (circle[int(g['ray_camera_256'])], 256, 'rays256', 128)):
        xy = C.pixel_grid(hw, hw, 256, 256)[None].expand(len(cam), hw, hw, 2)
        o, d, l = C.xy_to_ray_bundle(cam, xy, cdm - 5.0, cdm + 5.0, n, False)
        if key == 'rays256':
            o, d = o.reshape(-1, 3)[::int(g['ray_stride_256'])], d.reshape(-1, 3)[::int(g['ray_stride_256'])]
        _rel_close(o, g[f'{key}_o']), _rel_close(d, g[f'{key}_d'])
        if key == 'rays32':
            _rel_close(l, g['rays32_lengths'])


def test_camera_container_accepts_foreign_cameras_and_slices():
    from types import SimpleNamespace
    R = torch.eye(3)[None].repeat(4, 1, 1)
    foreign = SimpleNamespace(R=R, T=torch.arange(12.0).view(4, 3), focal_length=torch.full((4, 2), 2.0), principal_point=torch.zeros(4, 2),
                              image_size=torch.full((4, 2), 256.0))
    c = C.as_cameras(foreign)
    assert len(c) == 4 and len(c[[1, 3]]) == 2 and torch.equal(c[2].T, foreign.T[2:3])
    assert torch.allclose(c.get_camera_center(), -foreign.T)
    m = c.get_world_to_view_matrix()
    assert m.shape == (4, 4, 4) and torch.equal(m[:, 3, :3], foreign.T) and torch.equal(m[:, :3, :3], R)
    d = C.PerspectiveCameras(R=R[:1], T=torch.zeros(1, 3))
    assert torch.equal(d.focal_length, torch.ones(1, 2)) and torch.equal(d.principal_point, torch.zeros(1, 2))


def test_native_builder_view_order_and_shapes(monkeypatch, g):
    """NativeSceneBuilder.build on the host side: the rays and the EFT are replaced by recorders, so the test sees which cameras go where and in
    which order (distillation.py:65-125): input views of the voxel frame at 128x128, then the 8 + 50 cached views, query = view ci of its own
    relative frame at 32x32 with 20 depths, target rays of the augmented voxel frame at 128x128"""
    from sparsefusion_b200 import distillation as D
    calls = []

    def fake_rays(self, cams, hw):
        calls.append((hw, cams))
        n = len(cams)
        return torch.zeros(n, hw * hw, 3), torch.zeros(n, hw * hw, 3)

    class Eft:
        def feature_cache(self, o, d, lengths, input_cameras, input_images, hw):
            self.args = (o, d, lengths, input_cameras, input_images, hw)
            return torch.zeros(o.shape[0], 256, *hw), torch.zeros(o.shape[0], 3, *hw)
    monkeypatch.setattr(D.NativeSceneBuilder, '_rays', fake_rays)
    monkeypatch.setattr(D.NativeSceneBuilder, '__init__', lambda self, gpu: setattr(self, 'device', torch.device('cpu')))
    monkeypatch.setattr(D.F, 'interpolate', lambda x, scale_factor, mode: x.repeat_interleave(int(scale_factor), 2).repeat_interleave(int(scale_factor), 3))
    cams = _cams(g)
    rgb, mask = torch.rand(8, 3, 256, 256), torch.rand(8, 1, 256, 256)
    eft = Eft()
    torch.manual_seed(int(g['jitter_seed']))
    cache = D.NativeSceneBuilder(0).build(eft, cams, rgb, mask, [0, 5])
    assert [c[0] for c in calls] == [128, 32, 128]
    assert len(calls[0][1]) == 2 and len(calls[1][1]) == 58 and len(calls[2][1]) == 58
    vox = C.relative_cameras(cams, [0], False)
    _close(calls[0][1].R, vox.R[[0, 5]].numpy())
    _close(calls[2][1].R, g['aug_vox_R']), _close(calls[2][1].T, g['aug_vox_T'])
    for ci in g['views']:
        _close(calls[1][1][int(ci)].R, g[f'view{ci}_query_R'][0:1]), _close(calls[1][1][int(ci)].T, g[f'view{ci}_query_T'][0:1])
        _close(eft.args[3][int(ci)].R, g[f'view{ci}_ctx_R']), _close(eft.args[3][int(ci)].T, g[f'view{ci}_ctx_T'])
    o, d, lengths, ctx, images, hw = eft.args
    assert lengths.shape == (58, 1024, 20) and hw == (32, 32) and len(ctx) == 58 and torch.equal(images, rgb[[0, 5]])
    _rel_close(lengths[0, 0], g['rays32_lengths'][0, 0, 0])
    assert cache.target_features.shape == (58, 256, 32, 32) and cache.target_eft_image.shape == (58, 3, 256, 256)
    assert cache.input_rays_o.shape == (2, 128 * 128, 3) and cache.target_rays_o.shape == (58, 128 * 128, 3)
    assert torch.equal(cache.input_rgb, rgb[[0, 5]]) and torch.equal(cache.input_mask, mask[[0, 5]])
    calls.clear()
    cache = D.NativeSceneBuilder(0).build(eft, cams, rgb, mask, [0, 5], use_diffusion=False)
    assert [c[0] for c in calls] == [128] and cache.target_features.shape == (0, 256, 32, 32) and cache.target_rays_o.shape == (0, 128 * 128, 3)
