"""Progress outputs of a distillation run: the reference's periodic loss plots and snapshot renders (sparsefusion/distillation.py:355-388).

Every ``progress_every`` iterations (the reference: 20) ``ProgressWriter.write`` writes, per scene,
``{exp_dir}/log/{seq_name}_loss.jpg`` (curves 'volumetric', 'opacity' and 'entropy', legend at upper right), ``{seq_name}_fusionloss.jpg``
(the fusion curve) and ``{seq_name}_vis.jpg`` (eval-mode render | silhouette of the iteration's photometric input view).  The losses come
from the distillers' on-device history (``Distiller.history``): one device-to-host copy of the rows added since the previous write.

The reference draws its plots with matplotlib, which these outputs do not need: ``plot_lines`` draws them with Pillow at matplotlib's
default figure size (640 x 480), axes box and colours (C0, C1, C2), so the files look alike but are not the same bytes.
"""
from __future__ import annotations

import math
import os
from typing import Optional, Sequence

import numpy as np
import torch

PROGRESS_STREAM = 6      # view_seed stream of the snapshot renders' jitter (5 serves the VLDM baseline's samples)
FIG_W, FIG_H = 640, 480  # matplotlib's default figure: 6.4 x 4.8 in at 100 dpi
AXES = (0.125, 0.11, 0.9, 0.88)   # matplotlib's default subplot box: left, bottom, right, top as fractions of the figure
COLORS = ((0x1f, 0x77, 0xb4), (0xff, 0x7f, 0x0e), (0x2c, 0xa0, 0x2c))   # matplotlib's default cycle C0, C1, C2
LOSS_LABELS = ('volumetric', 'opacity', 'entropy')


def check_progress_every(progress_every):
    """ValueError for a ``progress_every`` that is not None or a positive int"""
    if progress_every is not None and (isinstance(progress_every, bool) or not isinstance(progress_every, int) or progress_every < 1):
        raise ValueError(f'progress_every must be a positive int or None (got {progress_every!r})')


def _nice_ticks(lo: float, hi: float, n: int = 8):
    """tick values covering [lo, hi] at a step of 1, 2, 2.5 or 5 times a power of ten, at most about ``n`` of them"""
    raw = (hi - lo) / n
    mag = 10.0 ** math.floor(math.log10(raw))
    step = next(m * mag for m in (1, 2, 2.5, 5, 10) if m * mag >= raw)
    first = math.ceil(lo / step - 1e-9) * step
    return [first + i * step for i in range(int(math.floor((hi - first) / step + 1e-9)) + 1)]


def _limits(vals: np.ndarray):
    """matplotlib's autoscaled limits: the data range with 5 % margins, widened when it is a single value"""
    lo, hi = float(vals.min()), float(vals.max())
    if hi - lo <= 1e-12 * max(abs(lo), abs(hi), 1e-30):
        pad = 0.05 * abs(lo) if lo != 0 else 0.055
        return lo - pad, hi + pad
    m = 0.05 * (hi - lo)
    return lo - m, hi + m


def _label(v: float, step: float) -> str:
    digits = max(0, -int(math.floor(math.log10(step) + 1e-9)))
    if abs(v) < step * 1e-6:
        v = 0.0
    return f'{v:.{digits}f}'


def plot_lines(path: str, ys: Sequence[np.ndarray], labels: Optional[Sequence[str]] = None) -> None:
    """a line plot of the series ``ys`` (each against 0, 1, 2, ..) as a 640 x 480 JPEG, in matplotlib's default colours and axes box, with
    a legend at upper right when ``labels`` are given.  A nan ends a line segment (the curve breaks there), as in matplotlib; a finite
    value with nan on both sides, which matplotlib would not show, is drawn as a dot so that a series logged every few iterations shows."""
    from .video import require_pillow
    Image = require_pillow()
    from PIL import ImageDraw, ImageFont
    im = Image.new('RGB', (FIG_W, FIG_H), (255, 255, 255))
    dr = ImageDraw.Draw(im)
    font = ImageFont.load_default()
    x0, x1 = AXES[0] * FIG_W, AXES[2] * FIG_W
    y0, y1 = (1 - AXES[1]) * FIG_H, (1 - AXES[3]) * FIG_H          # pixel rows of the axes' bottom and top
    ys = [np.asarray(y, dtype=np.float64).reshape(-1) for y in ys]
    n = max((y.size for y in ys), default=0)
    finite = np.concatenate([y[np.isfinite(y)] for y in ys]) if ys else np.zeros(0)
    xl = _limits(np.array([0.0, max(n - 1, 0)], dtype=np.float64))
    yl = _limits(finite) if finite.size else (-0.055, 0.055)
    px = lambda x: x0 + (x - xl[0]) / (xl[1] - xl[0]) * (x1 - x0)
    py = lambda y: y0 - (y - yl[0]) / (yl[1] - yl[0]) * (y0 - y1)
    for axis, (lo, hi) in (('x', xl), ('y', yl)):
        ticks = _nice_ticks(lo, hi)
        step = ticks[1] - ticks[0] if len(ticks) > 1 else max(hi - lo, 1e-30)
        for t in ticks:
            s = _label(t, step)
            tw, th = dr.textbbox((0, 0), s, font=font)[2:]
            if axis == 'x':
                p = px(t)
                dr.line([(p, y0), (p, y0 + 3.5)], fill=(0, 0, 0), width=1)
                dr.text((p - tw / 2, y0 + 6), s, fill=(0, 0, 0), font=font)
            else:
                p = py(t)
                dr.line([(x0 - 3.5, p), (x0, p)], fill=(0, 0, 0), width=1)
                dr.text((x0 - 6 - tw, p - th / 2), s, fill=(0, 0, 0), font=font)
    for k, y in enumerate(ys):
        color = COLORS[k % len(COLORS)]
        ok = np.isfinite(y)
        seg = []
        for i in range(y.size + 1):
            if i < y.size and ok[i]:
                seg.append((px(i), py(y[i])))
                continue
            if len(seg) > 1:
                dr.line(seg, fill=color, width=2)          # 1 pt at 100 dpi is 1.4 px
            elif seg:
                (cx, cy), = seg
                dr.ellipse([cx - 1.5, cy - 1.5, cx + 1.5, cy + 1.5], fill=color)
            seg = []
    dr.rectangle([x0, y1, x1, y0], outline=(0, 0, 0), width=1)
    if labels:
        rows = [dr.textbbox((0, 0), s, font=font)[2:] for s in labels]
        line_w, pad, gap = 20, 5, 4
        row_h = max(h for _, h in rows) + gap
        w = pad + line_w + 6 + max(tw for tw, _ in rows) + pad
        h = pad + row_h * len(labels) - gap + pad
        lx, ly = x1 - 8 - w, y1 + 8
        dr.rounded_rectangle([lx, ly, lx + w, ly + h], radius=3, fill=(255, 255, 255), outline=(204, 204, 204), width=1)
        for k, s in enumerate(labels):
            cy = ly + pad + k * row_h + row_h / 2 - gap / 2
            dr.line([(lx + pad, cy), (lx + pad + line_w, cy)], fill=COLORS[k % len(COLORS)], width=2)
            dr.text((lx + pad + line_w + 6, cy - rows[k][1] / 2), s, fill=(0, 0, 0), font=font)
    os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
    im.save(path, format='JPEG', quality=90, subsampling=0)      # full-resolution chroma: thin coloured lines keep their colour


def write_loss_plots(exp_dir: str, seq_name: str, rows: np.ndarray) -> None:
    """the reference's ``{exp_dir}/log/{seq_name}_loss.jpg`` (volumetric, opacity and entropy curves, legend upper right; :356-362) and
    ``{seq_name}_fusionloss.jpg`` (:364-367) of the history rows [n, 4] (``Distiller.history`` columns)"""
    plot_lines(f'{exp_dir}/log/{seq_name}_loss.jpg', [rows[:, 0], rows[:, 1], rows[:, 2]], LOSS_LABELS)
    plot_lines(f'{exp_dir}/log/{seq_name}_fusionloss.jpg', [rows[:, 3]])


class ProgressWriter:
    """the periodic outputs of one run's scenes (module docstring).  ``names``: the scenes' seq_names; ``views``: their ``EvalViews`` (the
    builder's ``eval_views`` rows ``input_idx[k]``), whose row j gives the snapshot of scene k when its photometric sub-step drew input j.
    The snapshot is ``evaluate.render_views``' eval-mode render (``render_batched(..., batched=True, perturb=True, bg_color=0,
    shading='albedo', force_all_rays=True)``, :369-382) with its jitter from ``view_seed(seed, itr, view, PROGRESS_STREAM)`` inside
    ``torch.random.fork_rng``: no draw from the global generators, and the network goes back to train mode, so a run with progress
    outputs takes the same steps as one without."""

    def __init__(self, exp_dir, names, views, input_idx, opt):
        """``views[k]``: scene k's input views, row j that of ``input_idx[k][j]``, the scene view whose number keys the jitter"""
        self.exp_dir, self.names, self.views, self.opt = exp_dir, list(names), list(views), opt
        self.input_idx = [[int(i) for i in idx] for idx in input_idx]
        self.rows = [np.full((0, 4), np.nan, dtype=np.float32) for _ in self.names]
        self.synced = 0            # history rows already on the host

    def write(self, itr: int, distillers) -> None:
        """the three files of every scene after iteration ``itr``; ``distillers``: one ``Distiller`` per scene"""
        from .evaluate import render_views
        from .video import to_uint8, write_jpeg
        lo, hi = self.synced, itr + 1
        if hi > lo:
            fresh = torch.stack([d._history[lo:hi] for d in distillers]).cpu().numpy()     # ONE device-to-host copy per write
            self.rows = [np.concatenate((r[:lo], f)) for r, f in zip(self.rows, fresh)]
            self.synced = hi
        os.makedirs(f'{self.exp_dir}/log', exist_ok=True)
        for k, (name, d) in enumerate(zip(self.names, distillers)):
            write_loss_plots(self.exp_dir, name, self.rows[k][:hi])
            views = self.views[k]
            j = d.last['input_view']
            H, W = views.rgb.shape[2:]
            image, sil = render_views(d.ngp, views.rays_o[j:j + 1], views.rays_d[j:j + 1], (H, W), self.opt, seed=d.seed,
                                      stream=PROGRESS_STREAM, itr=itr, view_ids=[self.input_idx[k][j]])
            write_jpeg(f'{self.exp_dir}/log/{name}_vis.jpg', to_uint8(image, sil[..., None])[0])              # :384-388
