"""Camera maths of the per-scene preparation (sparsefusion/distillation.py:65-86) on the host, without pytorch3d.

A line-by-line restatement of what the reference's ``utils/camera_utils.py`` does with pytorch3d's ``PerspectiveCameras``: relative and
voxel-frame cameras (camera_utils.py:98-135), camera slices and concatenation (:51-95), the circle path through the scene cameras
(:190-259) with its helpers (:261-400), and the pytorch3d primitives they touch, restated from pytorch3d's documented conventions:
cameras defined in NDC, row vectors (x_view = x_world R + T, x_ndc = f x / z + p), transforms as 4x4 matrices composed left to right.
Everything here handles at most about a hundred cameras, so it runs on the CPU by design; the ray grids of these cameras are computed on
the GPU (``grid_rays``).
"""
from __future__ import annotations

import math
from typing import Sequence

import torch
import torch.nn.functional as F

from . import _lib as lib


class PerspectiveCameras:
    """the fields of pytorch3d.renderer.PerspectiveCameras (in NDC) the preparation uses: R [N,3,3], T [N,3], focal_length [N,2],
    principal_point [N,2], image_size [N,2] (or None).  Defaults and broadcasting as pytorch3d's: identity R, zero T, focal 1, principal
    point 0, every field broadcast to the largest batch."""

    def __init__(self, R=None, T=None, focal_length=1.0, principal_point=((0.0, 0.0),), image_size=None, device='cpu'):
        t = lambda x: x.to(device=device, dtype=torch.float32) if torch.is_tensor(x) else torch.tensor(x, dtype=torch.float32, device=device)
        R = torch.eye(3)[None] if R is None else R
        T = torch.zeros(1, 3) if T is None else T
        R, T = t(R), t(T)
        f, p = t(focal_length), t(principal_point)
        f = f.reshape(-1, 1).expand(-1, 2) if f.dim() < 2 or f.shape[-1] == 1 else f
        n = max(R.shape[0], T.shape[0], f.shape[0], p.shape[0])
        self.R, self.T = R.expand(n, 3, 3), T.expand(n, 3)
        self.focal_length, self.principal_point = f.expand(n, 2), p.expand(n, 2)
        self.image_size = None if image_size is None else t(image_size).expand(n, 2)

    @property
    def device(self):
        return self.R.device

    def __len__(self):
        return self.R.shape[0]

    def __getitem__(self, idx):
        return camera_slice(self, idx)

    def to(self, device):
        return PerspectiveCameras(self.R, self.T, self.focal_length, self.principal_point, self.image_size, device=device)

    def cpu(self):
        return self.to('cpu')

    def get_world_to_view_matrix(self) -> torch.Tensor:
        return world_to_view_matrix(self.R, self.T)

    def get_camera_center(self) -> torch.Tensor:
        return camera_center(self)


def as_cameras(cams) -> PerspectiveCameras:
    """any object with R, T, focal_length, principal_point (and image_size), e.g. a pytorch3d camera -> PerspectiveCameras on the same device"""
    if isinstance(cams, PerspectiveCameras):
        return cams
    return PerspectiveCameras(cams.R, cams.T, cams.focal_length, cams.principal_point, getattr(cams, 'image_size', None), device=cams.R.device)


def camera_slice(cams, indices) -> PerspectiveCameras:
    """RelativeCameraLoader.get_camera_slice (camera_utils.py:76-95)"""
    c = as_cameras(cams)
    if isinstance(indices, int):
        indices = [indices]
    return PerspectiveCameras(c.R[indices], c.T[indices], c.focal_length[indices], c.principal_point[indices],
                              None if c.image_size is None else c.image_size[indices], device=c.device)


def concat_cameras(camera_list: Sequence) -> PerspectiveCameras:
    """RelativeCameraLoader.concat_cameras (camera_utils.py:51-74)"""
    cs = [as_cameras(c) for c in camera_list]
    dev = cs[0].device
    cat = lambda k: torch.cat([getattr(c, k).to(dev) for c in cs])
    return PerspectiveCameras(cat('R'), cat('T'), cat('focal_length'), cat('principal_point'), cat('image_size'), device=dev)


# ---------------------------------------------------------------------------------------------------------- pytorch3d's transforms
def _rotate4(R):            # Rotate(R).get_matrix()
    m = torch.zeros(R.shape[0], 4, 4, dtype=R.dtype, device=R.device)
    m[:, :3, :3] = R
    m[:, 3, 3] = 1.0
    return m


def _translate4(T):         # Translate(T).get_matrix()
    m = torch.eye(4, dtype=T.dtype, device=T.device).repeat(T.shape[0], 1, 1)
    m[:, 3, :3] = T
    return m


def world_to_view_matrix(R, T) -> torch.Tensor:
    """get_world_to_view_transform(R, T).get_matrix() = Rotate(R).compose(Translate(T)): [[R, 0], [T, 1]] (row vectors)"""
    return torch.matmul(_rotate4(R), _translate4(T))


def world_to_view_inverse(R, T) -> torch.Tensor:
    """get_world_to_view_transform(R, T).inverse().get_matrix(): Transform3d.inverse inverts a composed transform piece by piece in reverse
    order -- Translate(-T) (exact), then torch.inverse of the rotation's 4x4 matrix (the composition's own matrix is a general Transform3d)"""
    return torch.matmul(_translate4(-T), torch.linalg.inv(_rotate4(R)))


def camera_center(cams) -> torch.Tensor:
    """PerspectiveCameras.get_camera_center: the translation row of the inverse world-to-view transform"""
    c = as_cameras(cams)
    return world_to_view_inverse(c.R, c.T)[:, 3, :3]


def _projection4(f, p):     # PerspectiveCameras.get_projection_transform() in NDC: Transform3d(matrix=K^T)
    K = torch.zeros(f.shape[0], 4, 4, dtype=f.dtype, device=f.device)
    K[:, 0, 0], K[:, 1, 1] = f[:, 0], f[:, 1]
    K[:, 0, 2], K[:, 1, 2] = p[:, 0], p[:, 1]
    K[:, 3, 2] = 1.0
    K[:, 2, 3] = 1.0
    return K.transpose(1, 2)


def unproject_points(cams, xy_depth: torch.Tensor) -> torch.Tensor:
    """PerspectiveCameras.unproject_points(xy_depth, world_coordinates=True, from_ndc=True) for cameras defined in NDC: the inverse of
    world-to-view . projection (. the identity NDC transform), inverted piece by piece in reverse order, applied to (x, y, 1/depth, 1) with
    the homogeneous divide.  xy_depth [N,P,3] -> world points [N,P,3]"""
    c = as_cameras(cams)
    m = torch.matmul(torch.linalg.inv(_projection4(c.focal_length, c.principal_point)), _translate4(-c.T))
    m = torch.matmul(m, torch.linalg.inv(_rotate4(c.R)))
    pts = torch.cat((xy_depth[..., :2], 1.0 / xy_depth[..., 2:3], torch.ones_like(xy_depth[..., :1])), dim=-1)
    out = torch.matmul(pts, m)
    return out[..., :3] / out[..., 3:]


def xy_to_ray_bundle(cams, xy_grid: torch.Tensor, min_depth, max_depth, n_pts_per_ray: int, unit_directions: bool):
    """pytorch3d.renderer.implicit.raysampling._xy_to_ray_bundle: xy_grid [N,...,2] NDC -> (origins, directions, lengths) with the points
    at depths 1 and 2 unprojected, directions = p2 - p1, origins = p1 - directions; lengths a linspace of n_pts_per_ray depths"""
    n = xy_grid.shape[0]
    spatial = xy_grid.shape[1:-1]
    m = spatial.numel()
    lengths = torch.linspace(float(min_depth), float(max_depth), n_pts_per_ray, dtype=xy_grid.dtype, device=xy_grid.device)
    lengths = lengths[None, None].expand(n, m, n_pts_per_ray)
    ones = xy_grid.new_ones(n, m, 1)
    to_unproject = torch.cat((xy_grid.reshape(n, 1, m, 2).expand(n, 2, m, 2).reshape(n, m * 2, 2), torch.cat((ones, 2.0 * ones), dim=1)), dim=-1)
    unprojected = unproject_points(cams, to_unproject)
    p1, p2 = unprojected[:, :m], unprojected[:, m:]
    directions = p2 - p1
    origins = p1 - directions
    if unit_directions:
        directions = F.normalize(directions, dim=-1)
    return origins.view(n, *spatial, 3), directions.view(n, *spatial, 3), lengths.reshape(n, *spatial, n_pts_per_ray)


def pixel_grid(height: int, width: int, full_height: int = None, full_width: int = None) -> torch.Tensor:
    """GridRaysampler's xy grid [H,W,2] (x, y) as utils/render_utils.py:38-65 configures it: pixel centres of the FULL image
    (min_x = 1 - 1/full_width, max_x = -1 + 1/full_width, likewise y), linspace'd over height x width samples"""
    fh, fw = full_height or height, full_width or width
    ys = torch.linspace(1.0 - 1.0 / fh, -1.0 + 1.0 / fh, height, dtype=torch.float32)
    xs = torch.linspace(1.0 - 1.0 / fw, -1.0 + 1.0 / fw, width, dtype=torch.float32)
    gy, gx = torch.meshgrid(ys, xs, indexing='ij')
    return torch.stack((gx, gy), dim=-1)


# ---------------------------------------------------------------------------------------------------------- camera_utils.py
def relative_cameras(cams, query_idx, center_at_origin: bool = False) -> PerspectiveCameras:
    """RelativeCameraLoader.get_relative_camera (camera_utils.py:98-135): every camera re-expressed relative to the query camera,
    g_q^{-1} g_j on the 4x4 world-to-view matrices; with center_at_origin=False only the query's rotation is undone (the voxel frame)"""
    c = as_cameras(cams)
    q = camera_slice(c, query_idx)
    T = q.T if center_at_origin else torch.zeros(1, 3, device=c.device)
    rel = torch.matmul(world_to_view_inverse(q.R, T), world_to_view_matrix(c.R, c.T))
    return PerspectiveCameras(rel[:, :3, :3], rel[:, 3, :3], c.focal_length, c.principal_point, c.image_size, device=c.device)


def _cross(a, b):
    """torch.cross without dim (camera_utils.py:274, :328, :348): the first dimension of size 3 of the broadcast shape"""
    shape = torch.broadcast_shapes(a.shape, b.shape)
    return torch.linalg.cross(a.expand(shape), b.expand(shape), dim=list(shape).index(3))


def generate_circle_by_vectors(t, C, r, n, u):
    """camera_utils.py:271-275: P(t) = r cos(t) u + r sin(t) (n x u) + C"""
    n = n / torch.linalg.norm(n)
    u = u / torch.linalg.norm(u)
    return r * torch.cos(t)[:, None] * u + r * torch.sin(t)[:, None] * _cross(n, u) + C


def fit_circle_2d(x, y):
    """camera_utils.py:292-310: least-squares circle through 2-D points -> (xc, yc, r)"""
    A = torch.stack([x, y, torch.ones(len(x))]).T
    b = x ** 2 + y ** 2
    c = torch.linalg.lstsq(A, b, rcond=None)[0]
    xc, yc = c[0] / 2, c[1] / 2
    return xc, yc, torch.sqrt(c[2] + xc ** 2 + yc ** 2)


def rodrigues_rot(P, n0, n1):
    """camera_utils.py:319-337: rotate points P [N,3] by the rotation taking n0 to n1"""
    if P.ndim == 1:
        P = P[None, ...]
    n0 = n0 / torch.linalg.norm(n0)
    n1 = n1 / torch.linalg.norm(n1)
    k = _cross(n0, n1)
    k = k / torch.linalg.norm(k)
    theta = torch.arccos(torch.dot(n0, n1))
    P_rot = torch.zeros((len(P), 3))
    for i in range(len(P)):
        P_rot[i] = P[i] * torch.cos(theta) + _cross(k, P[i]) * torch.sin(theta) + k * torch.dot(k, P[i]) * (1 - torch.cos(theta))
    return P_rot


def rodrigues_rot2(P, n1, theta):
    """camera_utils.py:339-356: rotate each point P[i] by theta[i] about k_i = P[i] x n1.  As in the reference, k is divided by the norm of
    the whole [N,3] matrix (:348-349), not row by row"""
    if P.ndim == 1:
        P = P[None, ...]
    k = _cross(P, n1.unsqueeze(0))
    k = k / torch.linalg.norm(k)
    P_rot = torch.zeros((len(P), 3))
    for i in range(len(P)):
        P_rot[i] = P[i] * torch.cos(theta[i]) + _cross(k[i], P[i]) * torch.sin(theta[i]) + k[i] * torch.dot(k[i], P[i]) * (1 - torch.cos(theta[i]))
    return P_rot


def get_nearest_centroid(cams) -> torch.Tensor:
    """camera_utils.py:370-400: the least-squares point nearest to every camera's principal ray (the ray through the mean principal point,
    unit directions), by the SVD pseudo-inverse"""
    c = as_cameras(cams)
    n = len(c)
    camera_centers = c.get_camera_center()
    c_mean = c.principal_point.mean(dim=0)
    xy_grid = c_mean.unsqueeze(0).unsqueeze(0)
    _, camera_directions, _ = xy_to_ray_bundle(c, xy_grid.expand(n, -1, -1), 1.0, 15.0, 20, True)
    A = torch.zeros((3 * n), n + 3)
    b = torch.zeros((3 * n, 1))
    A[:, :3] = torch.eye(3).repeat(n, 1)
    for ci in range(n):
        A[3 * ci:3 * ci + 3, ci + 3] = -camera_directions[ci]
        b[3 * ci:3 * ci + 3, 0] = camera_centers[ci]
    U, s, VT = torch.linalg.svd(A)
    Sinv = torch.diag(1 / s)
    if len(s) < 3 * n:
        Sinv = torch.cat((Sinv, torch.zeros((Sinv.shape[0], 3 * n - Sinv.shape[1]), device=Sinv.device)), dim=1)
    x = torch.matmul(VT.T, torch.matmul(Sinv, torch.matmul(U.T, b)))
    return x[:3, 0]


def look_at_rotation(camera_position, at, up) -> torch.Tensor:
    """pytorch3d.renderer.cameras.look_at_rotation: columns x, y, z of the camera in world coordinates (z towards ``at``)"""
    z_axis = F.normalize(at - camera_position, eps=1e-5)
    x_axis = F.normalize(torch.linalg.cross(up, z_axis, dim=1), eps=1e-5)
    y_axis = F.normalize(torch.linalg.cross(z_axis, x_axis, dim=1), eps=1e-5)
    is_close = torch.isclose(x_axis, torch.tensor(0.0), atol=5e-3).all(dim=1, keepdim=True)
    if is_close.any():
        replacement = F.normalize(torch.linalg.cross(y_axis, z_axis, dim=1), eps=1e-5)
        x_axis = torch.where(is_close, replacement, x_axis)
    R = torch.cat((x_axis[:, None, :], y_axis[:, None, :], z_axis[:, None, :]), dim=1)
    return R.transpose(1, 2)


def look_at_view_transform(eye, at, up):
    """pytorch3d.renderer.cameras.look_at_view_transform(eye=..., at=..., up=...): (R [N,3,3], T [N,3]), eye / at / up broadcast"""
    eye, at, up = torch.broadcast_tensors(eye, at, up)
    R = look_at_rotation(eye, at, up)
    T = -torch.bmm(R.transpose(1, 2), eye[:, :, None])[:, :, 0]
    return R, T


def interpolated_path(cams, n: int = 50, theta_offset_max: float = 0.0) -> PerspectiveCameras:
    """get_interpolated_path(cameras, n, method='circle', theta_offset_max) (camera_utils.py:190-259): a circle fitted through the camera
    centres (SVD plane fit, the normal flipped to face away from the centroid, least-squares circle in the plane), n cameras on it from the
    first camera's angle, each jittered by a uniform angle in +-theta_offset_max (``torch.rand(n)`` from torch's global CPU generator, as the
    reference draws it), all looking at the nearest centroid of the principal rays with up = -normal; mean focal length and principal point"""
    c = as_cameras(cams)
    device = c.device
    c = c.cpu()
    P = c.get_camera_center().cpu()
    P_mean = P.mean(axis=0)
    P_centered = P - P_mean
    U, s, V = torch.linalg.svd(P_centered)
    normal = V[2, :]
    if (normal * 2 - P_mean).norm() < (normal - P_mean).norm():
        normal = -normal
    P_xy = rodrigues_rot(P_centered, normal, torch.tensor([0.0, 0.0, 1.0]))
    xc, yc, r = fit_circle_2d(P_xy[:, 0], P_xy[:, 1])
    C = rodrigues_rot(torch.tensor([xc, yc, 0.0]), torch.tensor([0.0, 0.0, 1.0]), normal) + P_mean
    C = C.flatten()
    t = torch.linspace(0, 2 * math.pi, n)
    u = P[0] - C
    new_camera_centers = generate_circle_by_vectors(t, C, r, normal, u)
    if theta_offset_max > 0.0:
        aug_theta = (torch.rand((new_camera_centers.shape[0])) * (2 * theta_offset_max)) - theta_offset_max
        new_camera_centers = rodrigues_rot2(new_camera_centers, normal, aug_theta)
    new_camera_look_at = get_nearest_centroid(c)
    up_vec = -normal
    R, T = look_at_view_transform(new_camera_centers, new_camera_look_at.unsqueeze(0), up_vec.unsqueeze(0))
    pp = c.principal_point.mean(dim=0, keepdim=True).expand(R.shape[0], -1)
    f = c.focal_length.mean(dim=0, keepdim=True).expand(R.shape[0], -1)
    image_size = None if c.image_size is None else c.image_size[:1].expand(R.shape[0], -1)
    return PerspectiveCameras(R, T, f, pp, image_size, device=device)


# ---------------------------------------------------------------------------------------------------------- GPU ray grids
def pack_cameras(cams, device) -> torch.Tensor:
    """[..., 16] float32 rows (R row-major, T, focal_length, principal_point) of cameras whose tensors have any leading shape"""
    R, T, f, p = cams.R, cams.T, cams.focal_length, cams.principal_point
    lead = R.shape[:-2]
    return torch.cat((R.reshape(*lead, 9), T.reshape(*lead, 3), f.reshape(*lead, 2), p.reshape(*lead, 2)), dim=-1).to(
        device=device, dtype=torch.float32).contiguous()


def grid_rays(cams, height: int, width: int, device, full_height: int = None, full_width: int = None):
    """GridRaysampler(cameras) rays (utils/render_utils.py:16-65, pytorch3d's _xy_to_ray_bundle without unit directions) for every camera in
    ONE launch of ``sfb_grid_rays``: the height x width pixel-centre grid of the full_height x full_width image -> origins, directions
    [V, height*width, 3] on ``device``, row-major pixels.  The ray lengths are one linspace shared by every ray; ``torch.linspace`` gives them."""
    c = as_cameras(cams)
    fh, fw = full_height or height, full_width or width
    packed = pack_cameras(c, device)
    V = packed.shape[0]
    o = torch.empty(V, height * width, 3, dtype=torch.float32, device=device)
    d = torch.empty_like(o)
    with torch.cuda.device(o.device):
        lib.call('sfb_grid_rays', lib.fptr(packed), V, height, width, 1.0 - 1.0 / fw, -1.0 + 1.0 / fw, 1.0 - 1.0 / fh, -1.0 + 1.0 / fh,
                 lib.fptr(o), lib.fptr(d), lib.stream())
    return o, d
