"""Generate the marching-cubes triangle table of sparsefusion_b200/csrc/mc_tables.cuh (and oracle/mesh_oracle.py's copy).

    python tools/gen_mc_tables.py            # rewrites csrc/mc_tables.cuh, prints the Python literal

Numbering (shared by the kernels and the oracle):
  corner c = dx | dy << 1 | dz << 2 of cell (i, j, k) is lattice point (i + dx, j + dy, k + dz); bit c of the case index is set when that
  corner is "below" (v <= iso).
  edge e = 4 * axis + r runs along `axis` (0 = x/i, 1 = y/j, 2 = z/k) from its lower-index corner, whose two other coordinates are
  (r & 1, r >> 1) in axis order (x: (dy, dz), y: (dx, dz), z: (dx, dy)).  That corner is the lattice point that owns the edge.

Construction, per case: on each of the six faces the crossing edges are paired into segments.  Two crossings give one segment; four
(diagonally opposite below corners) give two segments, each cutting off one below corner, so the above corners stay connected.  The rule
depends on the face alone, so the two cells sharing a face draw the same segments there and the surface is closed.  Each segment is
directed so that, seen from outside the cell, the below corners lie on its left; the directed segments chain into loops around the
below part of the cell's surface, and each loop is fanned into triangles (l0, li, li+1) -- unless a chord of that fan joins two
vertices of a four-crossing face, which the neighbouring cell might also join; then the loop takes the first triangulation without such
a chord.  Every face of the cell boundary thus carries only segments, each used once per cell, so each mesh edge has exactly two faces.
The resulting faces have their normals pointing toward the below corners, i.e. toward decreasing value.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'sparsefusion_b200', 'csrc', 'mc_tables.cuh')


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], dtype=np.float64)


def edge_corners(e):
    """(lower corner, upper corner) of edge e"""
    axis, r = divmod(e, 4)
    other = [a for a in range(3) if a != axis]
    lo = [0, 0, 0]
    lo[other[0]], lo[other[1]] = r & 1, r >> 1
    hi = list(lo)
    hi[axis] = 1
    return lo[0] | lo[1] << 1 | lo[2] << 2, hi[0] | hi[1] << 1 | hi[2] << 2


def _faces():
    """(outward normal, the four corners in cyclic order, the edge between consecutive corners)"""
    out = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            cyc = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[axis], p[u], p[v] = side, du, dv
                cyc.append(p[0] | p[1] << 1 | p[2] << 2)
            edges = []
            for t in range(4):
                a, b = cyc[t], cyc[(t + 1) % 4]
                edges.append(next(e for e in range(12) if set(edge_corners(e)) == {a, b}))
            n = np.zeros(3)
            n[axis] = 1.0 if side else -1.0
            out.append((n, cyc, edges))
    return out


FACES = _faces()


def _triangulations(poly):
    """every triangulation of the polygon `poly` (a list of vertex ids), as lists of triangles; fans from poly[0] come first"""
    if len(poly) < 3:
        yield []
        return
    a, b = poly[0], poly[-1]
    for k in range(len(poly) - 2, 0, -1):
        for left in _triangulations(poly[:k + 1]):
            for right in _triangulations(poly[k:]):
                yield left + [(a, poly[k], b)] + right


def _loop_triangles(loop, forbidden):
    """triangles of one loop: the fan (l0, li, li+1) unless one of its chords joins two vertices that lie on the same four-crossing face
    (the neighbouring cell may draw the same chord there, which would give an edge four faces); then the first triangulation without one"""
    for tris in _triangulations(loop):
        chords = {frozenset(p) for t in tris for p in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))}
        if not chords & forbidden:
            # orient as the loop runs: (a, b, c) in loop order
            pos = {e: i for i, e in enumerate(loop)}
            return [tuple(sorted(t, key=lambda e: pos[e])) for t in tris]
    raise AssertionError(f'no admissible triangulation of loop {loop}')


def case_triangles(case):
    below = [(case >> c) & 1 for c in range(8)]
    mid = {e: (corner_pos(edge_corners(e)[0]) + corner_pos(edge_corners(e)[1])) / 2 for e in range(12)}
    nxt = {}
    forbidden = set()
    for n, cyc, edges in FACES:
        cross = [t for t in range(4) if below[cyc[t]] != below[cyc[(t + 1) % 4]]]
        if not cross:
            continue
        if len(cross) == 2:
            segs = [((edges[cross[0]], edges[cross[1]]), [c for c in cyc if below[c]])]
        else:       # four crossings: cut off each below corner (corner t sits between face edges t-1 and t)
            segs = [((edges[(t - 1) % 4], edges[t]), [cyc[t]]) for t in range(4) if below[cyc[t]]]
            forbidden |= {frozenset((edges[s], edges[t])) for s in range(4) for t in range(s + 1, 4)} - {frozenset(s[0]) for s in segs}
        for (a, b), bc in segs:
            p = np.mean([corner_pos(c) for c in bc], axis=0)
            if np.dot(np.cross(mid[b] - mid[a], p - mid[a]), n) < 0:
                a, b = b, a
            assert a not in nxt, (case, a)
            nxt[a] = b
    tris = []
    todo = set(nxt)
    while todo:
        loop = [min(todo)]
        while nxt[loop[-1]] != loop[0]:
            loop.append(nxt[loop[-1]])
        todo -= set(loop)
        tris += _loop_triangles(loop, forbidden)
    return tris


def tables():
    """tri_table [256][3 * max_tris] int (-1 padded), tri_count [256]"""
    rows = [case_triangles(c) for c in range(256)]
    width = 3 * max(len(r) for r in rows)
    tab = np.full((256, width), -1, dtype=np.int64)
    for c, r in enumerate(rows):
        flat = [e for t in r for e in t]
        tab[c, :len(flat)] = flat
    return tab, np.array([len(r) for r in rows], dtype=np.int64)


def header_text():
    tab, cnt = tables()
    lines = ['// mc_tables.cuh -- marching-cubes triangle table, generated by tools/gen_mc_tables.py (numbering and construction documented there)',
             '#pragma once', '#include <stdint.h>', '', 'namespace sfb {', '',
             f'constexpr int kMcMaxTris = {tab.shape[1] // 3};', '',
             '// triangles per case', '__constant__ uint8_t c_mc_tri_count[256] = {']
    for r in range(0, 256, 32):
        lines.append('    ' + ', '.join(str(int(v)) for v in cnt[r:r + 32]) + ',')
    lines += ['};', '', '// edge ids of the triangles of each case, three per triangle, -1 padded',
              f'__constant__ int8_t c_mc_tri_table[256][{tab.shape[1]}] = {{']
    for c in range(256):
        lines.append('    {' + ', '.join(str(int(v)) for v in tab[c]) + '},')
    lines += ['};', '', '}  // namespace sfb', '']
    return '\n'.join(lines)


def python_literal():
    tab, _ = tables()
    rows = [[int(v) for v in tab[c] if v >= 0] for c in range(256)]
    out = ['TRI_TABLE = (']
    for c in range(0, 256, 4):
        out.append('    ' + ' '.join(f'{tuple(r)!r},' if len(r) != 1 else f'({r[0]},),' for r in rows[c:c + 4]))
    out.append(')')
    return '\n'.join(out)


if __name__ == '__main__':
    with open(HEADER, 'w') as f:
        f.write(header_text())
    print(python_literal())
    sys.stderr.write(f'wrote {HEADER}; max {tables()[0].shape[1] // 3} triangles per case\n')
