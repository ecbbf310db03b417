"""numpy restatement of the GIF palette quantiser (include/sparsefusion_b200.h section 11, csrc/palette.cu): 32^3 histogram by bincount, median
cut over boxes shrunk to their non-empty cells, rounded box means as the palette, brute-force nearest entry per pixel.  Integer arithmetic
throughout, so the kernel must match it bit for bit."""
from __future__ import annotations

import numpy as np

SIDE = 32


def histogram(frame: np.ndarray):
    """(n, sums) of one uint8 [H, W, 3] frame: n [32, 32, 32] pixel counts, sums [3, 32, 32, 32] channel sums, int64"""
    px = frame.reshape(-1, 3).astype(np.int64)
    cell = (px[:, 0] >> 3) * SIDE * SIDE + (px[:, 1] >> 3) * SIDE + (px[:, 2] >> 3)
    n = np.bincount(cell, minlength=SIDE ** 3)
    sums = np.stack([np.bincount(cell, weights=px[:, c], minlength=SIDE ** 3).astype(np.int64) for c in range(3)])
    return n.reshape(SIDE, SIDE, SIDE), sums.reshape(3, SIDE, SIDE, SIDE)


def _shrink(n, lo, hi):
    """the bounding box of the non-empty cells inside the inclusive range [lo, hi]"""
    sub = n[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] > 0
    new_lo, new_hi = [], []
    for a in range(3):
        occupied = np.flatnonzero(sub.any(axis=tuple(b for b in range(3) if b != a)))
        new_lo.append(lo[a] + int(occupied[0]))
        new_hi.append(lo[a] + int(occupied[-1]))
    return new_lo, new_hi


def _count(n, lo, hi):
    return int(n[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1].sum())


def median_cut(n, sums, colors):
    """palette [256, 3] uint8 (zero beyond the boxes) and the number of boxes"""
    boxes = [_shrink(n, [0, 0, 0], [SIDE - 1] * 3)]
    counts = [_count(n, *boxes[0])]
    while len(boxes) < colors:
        splittable = [k for k, (lo, hi) in enumerate(boxes) if any(h > l for l, h in zip(lo, hi))]
        if not splittable:
            break
        k = max(splittable, key=lambda i: (counts[i], -i))                 # most pixels, lowest index on ties
        lo, hi = boxes[k]
        axis = max(range(3), key=lambda a: (hi[a] - lo[a], -a))            # longest axis, r before g before b on ties
        sub = n[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1]
        per_slice = sub.sum(axis=tuple(b for b in range(3) if b != axis))
        cum = np.cumsum(per_slice)
        t = hi[axis] - 1
        for s in range(lo[axis], hi[axis]):
            if 2 * int(cum[s - lo[axis]]) >= counts[k]:
                t = s
                break
        lo_hi, up_lo = list(hi), list(lo)
        lo_hi[axis], up_lo[axis] = t, t + 1
        boxes[k] = _shrink(n, lo, lo_hi)
        boxes.append(_shrink(n, up_lo, hi))
        counts[k] = _count(n, *boxes[k])
        counts.append(_count(n, *boxes[-1]))
    palette = np.zeros((256, 3), np.uint8)
    for k, (lo, hi) in enumerate(boxes):
        N = counts[k]
        for c in range(3):
            S = int(sums[c, lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1].sum())
            palette[k, c] = (2 * S + N) // (2 * N)
    return palette, len(boxes)


def nearest(frame: np.ndarray, palette: np.ndarray, ncolors: int, chunk: int = 4096) -> np.ndarray:
    """indices [H, W] uint8: the entry of smallest squared distance, the lowest index on ties (argmin's first minimum)"""
    colours, inverse = np.unique(frame.reshape(-1, 3), axis=0, return_inverse=True)
    pal = palette[:ncolors].astype(np.int32)
    best = np.empty(len(colours), np.uint8)
    for i in range(0, len(colours), chunk):
        d = ((colours[i:i + chunk, None, :].astype(np.int32) - pal[None]) ** 2).sum(-1)
        best[i:i + chunk] = d.argmin(axis=1)
    return best[inverse.reshape(-1)].reshape(frame.shape[:2])


def quantize(frames: np.ndarray, colors: int = 256):
    """(palette [B, 256, 3] uint8, ncolors [B] int32, indices [B, H, W] uint8) of uint8 frames [B, H, W, 3]"""
    if not 2 <= colors <= 256:
        raise ValueError(f'colors must be in 2..256 (got {colors})')
    B = frames.shape[0]
    palette, ncolors = np.zeros((B, 256, 3), np.uint8), np.zeros(B, np.int32)
    indices = np.zeros(frames.shape[:3], np.uint8)
    for b in range(B):
        palette[b], ncolors[b] = median_cut(*histogram(frames[b]), colors)
        indices[b] = nearest(frames[b], palette[b], int(ncolors[b]))
    return palette, ncolors, indices
