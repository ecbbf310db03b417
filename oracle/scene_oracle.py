"""oracle/scene_oracle.py -- golden vectors of the per-scene preparation (sparsefusion/distillation.py:65-86): relative / voxel-frame cameras,
the jittered circle path, nearest centroid and GridRaysampler rays, minted by the REFERENCE's own utils/camera_utils.py and
utils/render_utils.py.

TEST INFRASTRUCTURE ONLY, run where the reference tree is (it is not on the GPU machines):

    python -m oracle.scene_oracle          # writes tests/golden/scene_prep.npz

Both reference modules import pytorch3d, which is not installed anywhere here.  pytorch3d is stubbed with a restatement, written from its
documented behaviour, of the few primitives they touch: ``PerspectiveCameras`` (NDC, row vectors: x_view = x_world R + T, x_ndc = f x / z + p),
``Transform3d`` (4x4 matrices; compose = product left to right; inverse = the inverses of the pieces in reverse order), ``Rotate`` /
``Translate``, ``look_at_view_transform``, ``_xy_to_ray_bundle`` and ``GridRaysampler``.  Everything above those primitives -- the relative
composition, the plane and circle fits, the Rodrigues rotations with their quirks, the θ jitter and its draw order, the nearest-centroid
solve, the samplers' grid bounds -- is the reference's code, run unmodified.  So parity is pinned to the REFERENCE's code, not to pytorch3d
itself, which no machine here has to check against.
"""
from __future__ import annotations

import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference'


# ---------------------------------------------------------------------------------------------------------- pytorch3d restatement
class Transform3d:
    def __init__(self, matrix=None, device='cpu', dtype=torch.float32):
        self._matrix = torch.eye(4, dtype=dtype)[None] if matrix is None else matrix
        self._transforms = []

    def _get_matrix_inverse(self):
        return torch.inverse(self._matrix)

    def get_matrix(self):
        m = self._matrix
        for t in self._transforms:
            m = torch.matmul(m, t.get_matrix())
        return m

    def compose(self, *others):
        out = Transform3d(self._matrix.clone())
        out._transforms = self._transforms + list(others)
        return out

    def inverse(self):
        t = Transform3d()
        i = self._get_matrix_inverse()
        if self._transforms:
            last = Transform3d(i)
            t._transforms = [x.inverse() for x in reversed(self._transforms)] + [last]
        else:
            t._matrix = i
        return t

    def transform_points(self, pts):
        h = torch.cat((pts, torch.ones_like(pts[..., :1])), dim=-1)
        out = torch.matmul(h, self.get_matrix())
        return out[..., :3] / out[..., 3:]


class Translate(Transform3d):
    def __init__(self, T):
        m = torch.eye(4).repeat(T.shape[0], 1, 1)
        m[:, 3, :3] = T
        super().__init__(m)

    def _get_matrix_inverse(self):
        mask = torch.ones(1, 4, 4)
        mask[0, 3, :3] = -1.0
        return self._matrix * mask

    def inverse(self):
        t = Transform3d(self._get_matrix_inverse())
        return t


class Rotate(Transform3d):
    def __init__(self, R):
        m = torch.zeros(R.shape[0], 4, 4)
        m[:, :3, :3] = R
        m[:, 3, 3] = 1.0
        super().__init__(m)


class PerspectiveCameras:
    def __init__(self, R=None, T=None, focal_length=1.0, principal_point=((0.0, 0.0),), image_size=None, device='cpu', **_):
        tt = lambda x: x.float() if torch.is_tensor(x) else torch.tensor(x, dtype=torch.float32)
        R = torch.eye(3)[None] if R is None else tt(R)
        T = torch.zeros(1, 3) if T is None else tt(T)
        f, p = tt(focal_length), tt(principal_point)
        if f.dim() < 2 or f.shape[-1] == 1:
            f = f.reshape(-1, 1).expand(-1, 2)
        n = max(R.shape[0], T.shape[0], f.shape[0], p.shape[0])
        self.R, self.T, self.focal_length, self.principal_point = R.expand(n, 3, 3), T.expand(n, 3), f.expand(n, 2), p.expand(n, 2)
        self.image_size = None if image_size is None else tt(image_size).expand(n, 2)
        self.device = torch.device('cpu')

    def __len__(self):
        return self.R.shape[0]

    def cpu(self):
        return self

    def to(self, device):
        return self

    def get_world_to_view_transform(self):
        return Rotate(self.R).compose(Translate(self.T))

    def get_projection_transform(self):
        n = len(self)
        K = torch.zeros(n, 4, 4)
        K[:, 0, 0], K[:, 1, 1] = self.focal_length[:, 0], self.focal_length[:, 1]
        K[:, 0, 2], K[:, 1, 2] = self.principal_point[:, 0], self.principal_point[:, 1]
        K[:, 3, 2] = 1.0
        K[:, 2, 3] = 1.0
        return Transform3d(K.transpose(1, 2))

    def get_camera_center(self):
        return self.get_world_to_view_transform().inverse().get_matrix()[:, 3, :3]

    def unproject_points(self, xy_depth, world_coordinates=True, from_ndc=False):
        assert world_coordinates
        t = self.get_world_to_view_transform().compose(self.get_projection_transform())
        if from_ndc:
            t = t.compose(Transform3d())                      # cameras defined in NDC: the NDC transform is the identity
        xy_inv_depth = torch.cat((xy_depth[..., :2], 1.0 / xy_depth[..., 2:3]), dim=-1)
        return t.inverse().transform_points(xy_inv_depth)


def look_at_view_transform(eye=None, at=((0, 0, 0),), up=((0, 1, 0),), device='cpu', **_):
    eye, at, up = torch.broadcast_tensors(eye.float(), torch.as_tensor(at).float(), torch.as_tensor(up).float())
    z = F.normalize(at - eye, eps=1e-5)
    x = F.normalize(torch.cross(up, z, dim=1), eps=1e-5)
    y = F.normalize(torch.cross(z, x, dim=1), eps=1e-5)
    close = torch.isclose(x, torch.tensor(0.0), atol=5e-3).all(dim=1, keepdim=True)
    if close.any():
        x = torch.where(close, F.normalize(torch.cross(y, z, dim=1), eps=1e-5), x)
    R = torch.cat((x[:, None], y[:, None], z[:, None]), dim=1).transpose(1, 2)
    T = -torch.bmm(R.transpose(1, 2), eye[:, :, None])[:, :, 0]
    return R, T


RayBundle = types.SimpleNamespace


def _xy_to_ray_bundle(cameras, xy_grid, min_depth, max_depth, n_pts_per_ray, unit_directions=False):
    b = xy_grid.shape[0]
    spatial = xy_grid.shape[1:-1]
    m = spatial.numel()
    zs = torch.linspace(min_depth, max_depth, n_pts_per_ray, dtype=xy_grid.dtype)[None, None].expand(b, m, n_pts_per_ray)
    to_unproject = torch.cat((xy_grid.view(b, 1, m, 2).expand(b, 2, m, 2).reshape(b, m * 2, 2),
                              torch.cat((xy_grid.new_ones(b, m, 1), 2.0 * xy_grid.new_ones(b, m, 1)), dim=1)), dim=-1)
    un = cameras.unproject_points(to_unproject, from_ndc=True)
    p1, p2 = un[:, :m], un[:, m:]
    d = p2 - p1
    o = p1 - d
    if unit_directions:
        d = F.normalize(d, dim=-1)
    return RayBundle(origins=o.view(b, *spatial, 3), directions=d.view(b, *spatial, 3), lengths=zs.reshape(b, *spatial, n_pts_per_ray), xys=xy_grid)


class GridRaysampler(torch.nn.Module):
    def __init__(self, min_x, max_x, min_y, max_y, image_width, image_height, n_pts_per_ray, min_depth, max_depth):
        super().__init__()
        gy, gx = torch.meshgrid(torch.linspace(min_y, max_y, image_height, dtype=torch.float32),
                                torch.linspace(min_x, max_x, image_width, dtype=torch.float32), indexing='ij')
        self._xy_grid = torch.stack((gx, gy), dim=-1)
        self.n_pts, self.min_depth, self.max_depth = n_pts_per_ray, min_depth, max_depth

    def forward(self, cameras, **_):
        xy = self._xy_grid[None].expand(len(cameras), *self._xy_grid.shape)
        return _xy_to_ray_bundle(cameras, xy, self.min_depth, self.max_depth, self.n_pts, False)


def import_reference():
    """the reference's utils.camera_utils and utils.render_utils with pytorch3d replaced by the restatement above"""
    sys.path.insert(0, REF)
    sys.dont_write_bytecode = True

    class _Any:
        def __init__(self, *a, **k): pass
        def __call__(self, *a, **k): return self
        def __getattr__(self, k): return _Any()

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__getattr__ = lambda k: _Any
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
    for n in ('pytorch3d', 'pytorch3d.ops', 'pytorch3d.ops.utils', 'pytorch3d.structures', 'pytorch3d.transforms', 'pytorch3d.renderer.implicit',
              'pytorch3d.renderer.implicit.utils', 'pytorch3d.renderer.implicit.raymarching'):
        stub(n)
    stub('pytorch3d.renderer', PerspectiveCameras=PerspectiveCameras, GridRaysampler=GridRaysampler)
    stub('pytorch3d.renderer.cameras', look_at_view_transform=look_at_view_transform, PerspectiveCameras=PerspectiveCameras)
    stub('pytorch3d.renderer.implicit.raysampling', _xy_to_ray_bundle=_xy_to_ray_bundle, RayBundle=RayBundle)
    import utils.camera_utils as cu
    import utils.render_utils as ru
    return cu, ru


def ring_cameras(n=8, seed=11):
    """a seeded, non-planar ring: centres at radius 4-6 with heights varying around the ring, looking near the origin, different focal lengths
    per axis and non-zero principal points"""
    rng = np.random.default_rng(seed)
    eyes, ats = [], []
    for i in range(n):
        az = 2 * math.pi * i / n + rng.uniform(-0.2, 0.2)
        r = rng.uniform(4.0, 6.0)
        eyes.append([r * math.sin(az), 1.2 * math.sin(2 * az) + rng.uniform(0.5, 1.5), r * math.cos(az)])
        ats.append(rng.uniform(-0.3, 0.3, 3))
    R, T = look_at_view_transform(eye=torch.tensor(eyes, dtype=torch.float32), at=torch.tensor(np.array(ats), dtype=torch.float32),
                                  up=torch.tensor([[0.0, 1.0, 0.0]]))
    f = torch.from_numpy(rng.uniform(2.5, 3.5, (n, 2)).astype(np.float32))
    p = torch.from_numpy(rng.uniform(-0.08, 0.08, (n, 2)).astype(np.float32))
    return PerspectiveCameras(R=R, T=T, focal_length=f, principal_point=p, image_size=torch.tensor([[256.0, 256.0]]).expand(n, 2))


def main(out=os.path.join(ROOT, 'tests', 'golden', 'scene_prep.npz')):
    cu, ru = import_reference()
    cams = ring_cameras()
    loader = cu.RelativeCameraLoader(relative=True, center_at_origin=True)
    rel = loader.get_relative_camera(cams, query_idx=[0], center_at_origin=True)                       # distillation.py:69-70
    vox = loader.get_relative_camera(cams, query_idx=[0], center_at_origin=False)
    seed = 1234
    torch.manual_seed(seed)
    path = cu.get_interpolated_path(cams, n=50, method='circle', theta_offset_max=0.17)               # :73
    aug = loader.concat_cameras([cams, path])                                                         # :74
    aug_rel = loader.get_relative_camera(aug, query_idx=[0], center_at_origin=True)                   # :75-76
    aug_vox = loader.get_relative_camera(aug, query_idx=[0], center_at_origin=False)
    circle = cu.get_interpolated_path(vox, n=50, method='circle')                                     # :463
    views = [3, 20]
    per_view = {}
    for ci in views:                                                                                   # :98
        q, _, _, ctx, _, _ = loader(aug_rel, None, query_idx=[ci], context_idx=[0, 5])
        per_view.update({f'view{ci}_query_R': q.R, f'view{ci}_query_T': q.T, f'view{ci}_ctx_R': ctx.R, f'view{ci}_ctx_T': ctx.T})
    cdm = torch.mean(torch.linalg.norm(cams.get_camera_center(), axis=1))                            # :82-86
    grid, _, feat = ru.init_ray_sampler(0, 256, 256, min=cdm - 5.0, max=cdm + 5.0, scale_factor=2)
    eft = ru.init_ray_sampler(0, 256, 256, min=cdm - 5.0, max=cdm + 5.0, scale_factor=8.0)[2]
    sl = lambda c, i: loader.get_camera_slice(c, i)
    rb128 = feat(sl(aug_vox, [9]))
    rb32 = eft(sl(aug_rel, [0, 3, 20, 57]))
    rb256 = grid(sl(circle, [7]))
    d = dict(R=cams.R, T=cams.T, focal_length=cams.focal_length, principal_point=cams.principal_point, image_size=cams.image_size,
             rel_R=rel.R, rel_T=rel.T, vox_R=vox.R, vox_T=vox.T, path_R=path.R, path_T=path.T, path_focal_length=path.focal_length,
             path_principal_point=path.principal_point, aug_rel_R=aug_rel.R, aug_rel_T=aug_rel.T, aug_vox_R=aug_vox.R, aug_vox_T=aug_vox.T,
             circle_R=circle.R, circle_T=circle.T, centroid=cu.get_nearest_centroid(cams), cam_dist_mean=cdm,
             rays128_o=rb128.origins, rays128_d=rb128.directions, rays32_o=rb32.origins, rays32_d=rb32.directions, rays32_lengths=rb32.lengths,
             rays256_o=rb256.origins.reshape(-1, 3)[::7], rays256_d=rb256.directions.reshape(-1, 3)[::7], **per_view)
    d = {k: v.detach().numpy().astype(np.float32) for k, v in d.items()}
    np.savez_compressed(out, jitter_seed=seed, views=np.array(views), context_idx=np.array([0, 5]), ray_camera_128=9,
                        ray_cameras_32=np.array([0, 3, 20, 57]), ray_camera_256=7, ray_stride_256=7, **d)
    print(f'wrote {out}: ' + ', '.join(f'{k} {tuple(v.shape)}' for k, v in d.items()))


if __name__ == '__main__':
    main()
