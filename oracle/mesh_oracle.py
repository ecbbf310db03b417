"""Plain-numpy restatement of the mesh extraction contract (include/sparsefusion_b200.h section 9, sparsefusion_b200/mesh.py), test-only.

* ``smooth_gaussian``: scipy.ndimage.gaussian_filter in float64 (what PyMCubes' smooth_gaussian builds on).
* ``mean_std``: numpy's population statistics in float64.
* ``marching_cubes``: the same corner / edge numbering, below test (v <= iso), vertex placement, vertex and triangle order as the CUDA
  kernels, in float64, vectorised over the lattice.  TRI_TABLE is the triangle table of sparsefusion_b200/csrc/mc_tables.cuh, written out
  by tools/gen_mc_tables.py (corner c = dx | dy << 1 | dz << 2; edge e = 4 * axis + r from the corner whose other two coordinates are
  (r & 1, r >> 1) in axis order).
* ``read_obj``, ``euler_characteristic``, ``edge_face_counts``, ``signed_volume``: mesh checks for the tests.
"""
from __future__ import annotations

import numpy as np

# triangles of each case as edge-id triples, flattened (tools/gen_mc_tables.py)
TRI_TABLE = (
    (), (0, 8, 4), (0, 5, 9), (4, 5, 9, 4, 9, 8),
    (1, 4, 10), (0, 8, 10, 0, 10, 1), (0, 5, 9, 1, 4, 10), (1, 5, 9, 1, 9, 8, 1, 8, 10),
    (1, 11, 5), (0, 8, 4, 1, 11, 5), (0, 1, 11, 0, 11, 9), (1, 11, 9, 1, 9, 8, 1, 8, 4),
    (4, 10, 11, 4, 11, 5), (0, 8, 10, 0, 10, 11, 0, 11, 5), (0, 4, 10, 0, 10, 11, 0, 11, 9), (8, 10, 11, 8, 11, 9),
    (2, 6, 8), (0, 2, 6, 0, 6, 4), (0, 5, 9, 2, 6, 8), (2, 6, 4, 2, 4, 5, 2, 5, 9),
    (1, 4, 10, 2, 6, 8), (0, 2, 6, 0, 6, 10, 0, 10, 1), (0, 5, 9, 1, 4, 10, 2, 6, 8), (1, 5, 9, 1, 9, 2, 1, 2, 6, 1, 6, 10),
    (1, 11, 5, 2, 6, 8), (0, 2, 6, 0, 6, 4, 1, 11, 5), (0, 1, 11, 0, 11, 9, 2, 6, 8), (1, 11, 9, 1, 9, 2, 1, 2, 6, 1, 6, 4),
    (2, 6, 8, 4, 10, 11, 4, 11, 5), (0, 2, 6, 0, 6, 10, 0, 10, 11, 0, 11, 5), (0, 4, 10, 0, 10, 11, 0, 11, 9, 2, 6, 8), (2, 6, 10, 2, 10, 11, 2, 11, 9),
    (2, 9, 7), (0, 8, 4, 2, 9, 7), (0, 5, 7, 0, 7, 2), (2, 8, 4, 2, 4, 5, 2, 5, 7),
    (1, 4, 10, 2, 9, 7), (0, 8, 10, 0, 10, 1, 2, 9, 7), (0, 5, 7, 0, 7, 2, 1, 4, 10), (1, 5, 7, 1, 7, 2, 1, 2, 8, 1, 8, 10),
    (1, 11, 5, 2, 9, 7), (0, 8, 4, 1, 11, 5, 2, 9, 7), (0, 1, 11, 0, 11, 7, 0, 7, 2), (1, 11, 7, 1, 7, 2, 1, 2, 8, 1, 8, 4),
    (2, 9, 7, 4, 10, 11, 4, 11, 5), (0, 8, 10, 0, 10, 11, 0, 11, 5, 2, 9, 7), (0, 4, 10, 0, 10, 11, 0, 11, 7, 0, 7, 2), (2, 8, 10, 2, 10, 11, 2, 11, 7),
    (6, 8, 9, 6, 9, 7), (0, 9, 7, 0, 7, 6, 0, 6, 4), (0, 5, 7, 0, 7, 6, 0, 6, 8), (4, 5, 7, 4, 7, 6),
    (1, 4, 10, 6, 8, 9, 6, 9, 7), (0, 9, 7, 0, 7, 6, 0, 6, 10, 0, 10, 1), (0, 5, 7, 0, 7, 6, 0, 6, 8, 1, 4, 10), (1, 5, 7, 1, 7, 6, 1, 6, 10),
    (1, 11, 5, 6, 8, 9, 6, 9, 7), (0, 9, 7, 0, 7, 6, 0, 6, 4, 1, 11, 5), (0, 1, 11, 0, 11, 7, 0, 7, 6, 0, 6, 8), (1, 11, 7, 1, 7, 6, 1, 6, 4),
    (4, 10, 11, 4, 11, 5, 6, 8, 9, 6, 9, 7), (0, 9, 7, 0, 7, 6, 0, 6, 10, 0, 10, 11, 0, 11, 5), (0, 4, 10, 0, 10, 11, 0, 11, 7, 0, 7, 6, 0, 6, 8), (6, 10, 11, 6, 11, 7),
    (3, 10, 6), (0, 8, 4, 3, 10, 6), (0, 5, 9, 3, 10, 6), (3, 10, 6, 4, 5, 9, 4, 9, 8),
    (1, 4, 6, 1, 6, 3), (0, 8, 6, 0, 6, 3, 0, 3, 1), (0, 5, 9, 1, 4, 6, 1, 6, 3), (1, 5, 9, 1, 9, 8, 1, 8, 6, 1, 6, 3),
    (1, 11, 5, 3, 10, 6), (0, 8, 4, 1, 11, 5, 3, 10, 6), (0, 1, 11, 0, 11, 9, 3, 10, 6), (1, 11, 9, 1, 9, 8, 1, 8, 4, 3, 10, 6),
    (3, 11, 5, 3, 5, 4, 3, 4, 6), (0, 8, 6, 0, 6, 3, 0, 3, 11, 0, 11, 5), (0, 4, 6, 0, 6, 3, 0, 3, 11, 0, 11, 9), (3, 11, 9, 3, 9, 8, 3, 8, 6),
    (2, 3, 10, 2, 10, 8), (0, 2, 3, 0, 3, 10, 0, 10, 4), (0, 5, 9, 2, 3, 10, 2, 10, 8), (2, 3, 10, 2, 10, 4, 2, 4, 5, 2, 5, 9),
    (1, 4, 8, 1, 8, 2, 1, 2, 3), (0, 2, 3, 0, 3, 1), (0, 5, 9, 1, 4, 8, 1, 8, 2, 1, 2, 3), (1, 5, 9, 1, 9, 2, 1, 2, 3),
    (1, 11, 5, 2, 3, 10, 2, 10, 8), (0, 2, 3, 0, 3, 10, 0, 10, 4, 1, 11, 5), (0, 1, 11, 0, 11, 9, 2, 3, 10, 2, 10, 8), (1, 11, 9, 1, 9, 2, 1, 2, 4, 2, 3, 10, 2, 10, 4),
    (2, 3, 11, 2, 11, 5, 2, 5, 4, 2, 4, 8), (0, 2, 3, 0, 3, 11, 0, 11, 5), (0, 4, 3, 4, 8, 2, 4, 2, 3, 0, 3, 11, 0, 11, 9), (2, 3, 11, 2, 11, 9),
    (2, 9, 7, 3, 10, 6), (0, 8, 4, 2, 9, 7, 3, 10, 6), (0, 5, 7, 0, 7, 2, 3, 10, 6), (2, 8, 4, 2, 4, 5, 2, 5, 7, 3, 10, 6),
    (1, 4, 6, 1, 6, 3, 2, 9, 7), (0, 8, 6, 0, 6, 3, 0, 3, 1, 2, 9, 7), (0, 5, 7, 0, 7, 2, 1, 4, 6, 1, 6, 3), (1, 5, 7, 1, 7, 2, 1, 2, 8, 1, 8, 6, 1, 6, 3),
    (1, 11, 5, 2, 9, 7, 3, 10, 6), (0, 8, 4, 1, 11, 5, 2, 9, 7, 3, 10, 6), (0, 1, 11, 0, 11, 7, 0, 7, 2, 3, 10, 6), (1, 11, 7, 1, 7, 2, 1, 2, 8, 1, 8, 4, 3, 10, 6),
    (2, 9, 7, 3, 11, 5, 3, 5, 4, 3, 4, 6), (0, 8, 6, 0, 6, 3, 0, 3, 11, 0, 11, 5, 2, 9, 7), (0, 4, 6, 0, 6, 3, 0, 3, 11, 0, 11, 7, 0, 7, 2), (2, 8, 11, 8, 6, 3, 8, 3, 11, 2, 11, 7),
    (3, 10, 8, 3, 8, 9, 3, 9, 7), (0, 9, 7, 0, 7, 3, 0, 3, 10, 0, 10, 4), (0, 5, 7, 0, 7, 3, 0, 3, 10, 0, 10, 8), (3, 10, 4, 3, 4, 5, 3, 5, 7),
    (1, 4, 8, 1, 8, 9, 1, 9, 7, 1, 7, 3), (0, 9, 7, 0, 7, 3, 0, 3, 1), (0, 5, 7, 0, 7, 3, 0, 3, 8, 3, 1, 4, 3, 4, 8), (1, 5, 7, 1, 7, 3),
    (1, 11, 5, 3, 10, 8, 3, 8, 9, 3, 9, 7), (0, 9, 7, 0, 7, 3, 0, 3, 10, 0, 10, 4, 1, 11, 5), (0, 1, 11, 0, 11, 7, 0, 7, 3, 0, 3, 10, 0, 10, 8), (1, 11, 7, 1, 7, 4, 7, 3, 10, 7, 10, 4),
    (3, 11, 5, 3, 5, 4, 3, 4, 8, 3, 8, 9, 3, 9, 7), (0, 9, 7, 0, 7, 3, 0, 3, 11, 0, 11, 5), (0, 4, 8, 3, 11, 7), (3, 11, 7),
    (3, 7, 11), (0, 8, 4, 3, 7, 11), (0, 5, 9, 3, 7, 11), (3, 7, 11, 4, 5, 9, 4, 9, 8),
    (1, 4, 10, 3, 7, 11), (0, 8, 10, 0, 10, 1, 3, 7, 11), (0, 5, 9, 1, 4, 10, 3, 7, 11), (1, 5, 9, 1, 9, 8, 1, 8, 10, 3, 7, 11),
    (1, 3, 7, 1, 7, 5), (0, 8, 4, 1, 3, 7, 1, 7, 5), (0, 1, 3, 0, 3, 7, 0, 7, 9), (1, 3, 7, 1, 7, 9, 1, 9, 8, 1, 8, 4),
    (3, 7, 5, 3, 5, 4, 3, 4, 10), (0, 8, 10, 0, 10, 3, 0, 3, 7, 0, 7, 5), (0, 4, 10, 0, 10, 3, 0, 3, 7, 0, 7, 9), (3, 7, 9, 3, 9, 8, 3, 8, 10),
    (2, 6, 8, 3, 7, 11), (0, 2, 6, 0, 6, 4, 3, 7, 11), (0, 5, 9, 2, 6, 8, 3, 7, 11), (2, 6, 4, 2, 4, 5, 2, 5, 9, 3, 7, 11),
    (1, 4, 10, 2, 6, 8, 3, 7, 11), (0, 2, 6, 0, 6, 10, 0, 10, 1, 3, 7, 11), (0, 5, 9, 1, 4, 10, 2, 6, 8, 3, 7, 11), (1, 5, 9, 1, 9, 2, 1, 2, 6, 1, 6, 10, 3, 7, 11),
    (1, 3, 7, 1, 7, 5, 2, 6, 8), (0, 2, 6, 0, 6, 4, 1, 3, 7, 1, 7, 5), (0, 1, 3, 0, 3, 7, 0, 7, 9, 2, 6, 8), (1, 3, 7, 1, 7, 9, 1, 9, 2, 1, 2, 6, 1, 6, 4),
    (2, 6, 8, 3, 7, 5, 3, 5, 4, 3, 4, 10), (0, 2, 6, 0, 6, 10, 0, 10, 3, 0, 3, 7, 0, 7, 5), (0, 4, 10, 0, 10, 3, 0, 3, 7, 0, 7, 9, 2, 6, 8), (2, 6, 10, 2, 10, 9, 10, 3, 7, 10, 7, 9),
    (2, 9, 11, 2, 11, 3), (0, 8, 4, 2, 9, 11, 2, 11, 3), (0, 5, 11, 0, 11, 3, 0, 3, 2), (2, 8, 4, 2, 4, 5, 2, 5, 11, 2, 11, 3),
    (1, 4, 10, 2, 9, 11, 2, 11, 3), (0, 8, 10, 0, 10, 1, 2, 9, 11, 2, 11, 3), (0, 5, 11, 0, 11, 3, 0, 3, 2, 1, 4, 10), (1, 5, 2, 5, 11, 3, 5, 3, 2, 1, 2, 8, 1, 8, 10),
    (1, 3, 2, 1, 2, 9, 1, 9, 5), (0, 8, 4, 1, 3, 2, 1, 2, 9, 1, 9, 5), (0, 1, 3, 0, 3, 2), (1, 3, 2, 1, 2, 8, 1, 8, 4),
    (2, 9, 5, 2, 5, 4, 2, 4, 10, 2, 10, 3), (0, 8, 10, 0, 10, 3, 0, 3, 5, 3, 2, 9, 3, 9, 5), (0, 4, 10, 0, 10, 3, 0, 3, 2), (2, 8, 10, 2, 10, 3),
    (3, 6, 8, 3, 8, 9, 3, 9, 11), (0, 9, 11, 0, 11, 3, 0, 3, 6, 0, 6, 4), (0, 5, 11, 0, 11, 3, 0, 3, 6, 0, 6, 8), (3, 6, 4, 3, 4, 5, 3, 5, 11),
    (1, 4, 10, 3, 6, 8, 3, 8, 9, 3, 9, 11), (0, 9, 11, 0, 11, 3, 0, 3, 6, 0, 6, 10, 0, 10, 1), (0, 5, 11, 0, 11, 3, 0, 3, 6, 0, 6, 8, 1, 4, 10), (1, 5, 6, 5, 11, 3, 5, 3, 6, 1, 6, 10),
    (1, 3, 6, 1, 6, 8, 1, 8, 9, 1, 9, 5), (0, 9, 3, 9, 5, 1, 9, 1, 3, 0, 3, 6, 0, 6, 4), (0, 1, 3, 0, 3, 6, 0, 6, 8), (1, 3, 6, 1, 6, 4),
    (3, 6, 8, 3, 8, 9, 3, 9, 5, 3, 5, 4, 3, 4, 10), (0, 9, 5, 3, 6, 10), (0, 4, 10, 0, 10, 3, 0, 3, 6, 0, 6, 8), (3, 6, 10),
    (6, 7, 11, 6, 11, 10), (0, 8, 4, 6, 7, 11, 6, 11, 10), (0, 5, 9, 6, 7, 11, 6, 11, 10), (4, 5, 9, 4, 9, 8, 6, 7, 11, 6, 11, 10),
    (1, 4, 6, 1, 6, 7, 1, 7, 11), (0, 8, 6, 0, 6, 7, 0, 7, 11, 0, 11, 1), (0, 5, 9, 1, 4, 6, 1, 6, 7, 1, 7, 11), (1, 5, 9, 1, 9, 8, 1, 8, 6, 1, 6, 7, 1, 7, 11),
    (1, 10, 6, 1, 6, 7, 1, 7, 5), (0, 8, 4, 1, 10, 6, 1, 6, 7, 1, 7, 5), (0, 1, 10, 0, 10, 6, 0, 6, 7, 0, 7, 9), (1, 10, 6, 1, 6, 7, 1, 7, 9, 1, 9, 8, 1, 8, 4),
    (4, 6, 7, 4, 7, 5), (0, 8, 6, 0, 6, 7, 0, 7, 5), (0, 4, 6, 0, 6, 7, 0, 7, 9), (6, 7, 9, 6, 9, 8),
    (2, 7, 11, 2, 11, 10, 2, 10, 8), (0, 2, 7, 0, 7, 11, 0, 11, 10, 0, 10, 4), (0, 5, 9, 2, 7, 11, 2, 11, 10, 2, 10, 8), (2, 7, 11, 2, 11, 10, 2, 10, 4, 2, 4, 5, 2, 5, 9),
    (1, 4, 8, 1, 8, 2, 1, 2, 7, 1, 7, 11), (0, 2, 7, 0, 7, 11, 0, 11, 1), (0, 5, 9, 1, 4, 8, 1, 8, 2, 1, 2, 7, 1, 7, 11), (1, 5, 9, 1, 9, 2, 1, 2, 7, 1, 7, 11),
    (1, 10, 8, 1, 8, 2, 1, 2, 7, 1, 7, 5), (0, 2, 7, 0, 7, 10, 7, 5, 1, 7, 1, 10, 0, 10, 4), (0, 1, 10, 0, 10, 7, 10, 8, 2, 10, 2, 7, 0, 7, 9), (1, 10, 4, 2, 7, 9),
    (2, 7, 5, 2, 5, 4, 2, 4, 8), (0, 2, 7, 0, 7, 5), (0, 4, 7, 4, 8, 2, 4, 2, 7, 0, 7, 9), (2, 7, 9),
    (2, 9, 11, 2, 11, 10, 2, 10, 6), (0, 8, 4, 2, 9, 11, 2, 11, 10, 2, 10, 6), (0, 5, 11, 0, 11, 10, 0, 10, 6, 0, 6, 2), (2, 8, 4, 2, 4, 5, 2, 5, 11, 2, 11, 10, 2, 10, 6),
    (1, 4, 6, 1, 6, 2, 1, 2, 9, 1, 9, 11), (0, 8, 6, 0, 6, 11, 6, 2, 9, 6, 9, 11, 0, 11, 1), (0, 5, 11, 0, 11, 6, 11, 1, 4, 11, 4, 6, 0, 6, 2), (1, 5, 11, 2, 8, 6),
    (1, 10, 6, 1, 6, 2, 1, 2, 9, 1, 9, 5), (0, 8, 4, 1, 10, 6, 1, 6, 2, 1, 2, 9, 1, 9, 5), (0, 1, 10, 0, 10, 6, 0, 6, 2), (1, 10, 6, 1, 6, 2, 1, 2, 8, 1, 8, 4),
    (2, 9, 5, 2, 5, 4, 2, 4, 6), (0, 8, 6, 0, 6, 5, 6, 2, 9, 6, 9, 5), (0, 4, 6, 0, 6, 2), (2, 8, 6),
    (8, 9, 11, 8, 11, 10), (0, 9, 11, 0, 11, 10, 0, 10, 4), (0, 5, 11, 0, 11, 10, 0, 10, 8), (4, 5, 11, 4, 11, 10),
    (1, 4, 8, 1, 8, 9, 1, 9, 11), (0, 9, 11, 0, 11, 1), (0, 5, 11, 0, 11, 8, 11, 1, 4, 11, 4, 8), (1, 5, 11),
    (1, 10, 8, 1, 8, 9, 1, 9, 5), (0, 9, 10, 9, 5, 1, 9, 1, 10, 0, 10, 4), (0, 1, 10, 0, 10, 8), (1, 10, 4),
    (4, 8, 9, 4, 9, 5), (0, 9, 5), (0, 4, 8), (),
)


def smooth_gaussian(volume, sigma=1.5):
    from scipy import ndimage
    return ndimage.gaussian_filter(np.asarray(volume, dtype=np.float64), sigma)


def mean_std(volume):
    v = np.asarray(volume, dtype=np.float64)
    return float(v.mean()), float(v.std())


def _owner_offset(e):
    a, r = divmod(e, 4)
    lo, hi = r & 1, r >> 1
    return ((0, lo, hi), (lo, 0, hi), (lo, hi, 0))[a], a


def marching_cubes(volume, iso):
    """(verts [V,3] float64 in index units, tris [F,3] int64), ordered as the kernels order them"""
    v = np.asarray(volume, dtype=np.float64)
    X, Y, Z = v.shape
    iso = float(iso)
    below = v <= iso
    flags = np.zeros((X, Y, Z, 3), dtype=bool)                 # owned edges to +i, +j, +k that cross
    flags[:-1, :, :, 0] = below[:-1] != below[1:]
    flags[:, :-1, :, 1] = below[:, :-1] != below[:, 1:]
    flags[:, :, :-1, 2] = below[:, :, :-1] != below[:, :, 1:]
    flat = flags.reshape(-1, 3)
    first = np.concatenate([[0], np.cumsum(flat.sum(1))[:-1]])           # index of a point's first vertex
    rank = np.cumsum(flat, axis=1) - flat                                 # rank of each owned edge among the point's crossing edges
    pidx, axis = np.nonzero(flat)                                         # lattice order, then axis order
    ijk = np.stack(np.unravel_index(pidx, (X, Y, Z)), axis=1)
    nxt = ijk.copy()
    nxt[np.arange(len(axis)), axis] += 1
    v0 = v[ijk[:, 0], ijk[:, 1], ijk[:, 2]]
    v1 = v[nxt[:, 0], nxt[:, 1], nxt[:, 2]]
    verts = ijk.astype(np.float64)
    verts[np.arange(len(axis)), axis] += (iso - v0) / (v1 - v0)
    if min(X, Y, Z) < 2:
        return verts, np.zeros((0, 3), dtype=np.int64)
    case = np.zeros((X - 1, Y - 1, Z - 1), dtype=np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= below[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz].astype(np.int64) << c
    width = max(len(r) for r in TRI_TABLE)
    table = np.full((256, width), -1, dtype=np.int64)
    for c, r in enumerate(TRI_TABLE):
        table[c, :len(r)] = r
    cells = np.stack(np.nonzero(case), axis=1)                            # lattice order
    if len(cells) == 0:
        return verts, np.zeros((0, 3), dtype=np.int64)
    rows = table[case[cells[:, 0], cells[:, 1], cells[:, 2]]]             # [M, width]
    valid = rows >= 0
    cell_of = np.broadcast_to(np.arange(len(cells))[:, None], rows.shape)[valid]
    edges = rows[valid]
    off = np.array([_owner_offset(e)[0] for e in range(12)], dtype=np.int64)
    ax = np.array([_owner_offset(e)[1] for e in range(12)], dtype=np.int64)
    owner = cells[cell_of] + off[edges]
    op = np.ravel_multi_index((owner[:, 0], owner[:, 1], owner[:, 2]), (X, Y, Z))
    assert flat[op, ax[edges]].all(), 'a triangle uses an edge that does not cross'
    tris = (first[op] + rank[op, ax[edges]]).reshape(-1, 3)
    return verts, tris


def read_obj(path):
    """(verts [V,3] float64, tris [F,3] int64 zero-based) of an OBJ file with `v x y z` and `f a b c` lines"""
    vs, fs = [], []
    with open(path) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == 'v':
                vs.append([float(t) for t in tok[1:4]])
            elif tok[0] == 'f':
                fs.append([int(t.split('/')[0]) - 1 for t in tok[1:4]])
    return np.array(vs, dtype=np.float64).reshape(-1, 3), np.array(fs, dtype=np.int64).reshape(-1, 3)


def edge_face_counts(tris):
    """how many faces use each undirected edge, and how often each directed edge occurs (1 everywhere on a consistently oriented mesh)"""
    t = np.asarray(tris, dtype=np.int64)
    d = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    _, dcount = np.unique(d, axis=0, return_counts=True)
    _, ucount = np.unique(np.sort(d, axis=1), axis=0, return_counts=True)
    return ucount, dcount


def euler_characteristic(verts, tris):
    ucount, _ = edge_face_counts(tris)
    used = np.unique(np.asarray(tris).reshape(-1))
    return int(len(used) - len(ucount) + len(tris))


def signed_volume(verts, tris):
    """divergence theorem: sum over faces of det(a, b, c) / 6 (positive for outward-facing normals)"""
    p = np.asarray(verts, dtype=np.float64)[np.asarray(tris)]
    return float(np.einsum('ij,ij->i', p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0)


def sphere(n=64, radius=20.0):
    """-SDF of a sphere centred in an n^3 lattice (positive inside, like a density)"""
    g = np.arange(n, dtype=np.float64) - (n - 1) / 2
    x, y, z = np.meshgrid(g, g, g, indexing='ij')
    return radius - np.sqrt(x * x + y * y + z * z)


def torus(n=64, major=16.0, minor=6.0):
    """-SDF of a torus around the k axis, centred in an n^3 lattice"""
    g = np.arange(n, dtype=np.float64) - (n - 1) / 2
    x, y, z = np.meshgrid(g, g, g, indexing='ij')
    return minor - np.sqrt((np.sqrt(x * x + y * y) - major) ** 2 + z * z)
