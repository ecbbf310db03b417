"""Device time to build one scene's EFT feature cache (sparsefusion/distillation.py:65-125): 32 scene views + 50 circle-path views, 256^2
images, NC input views, two ways, timed alternately in one process:

* ``per_view``: the reference's drive -- for each of the 82 views its relative cameras, its 32^2 x 20 query bundle, ``eft.encode(cameras,
  images)`` and ``eft.batched_forward(bundle, input_cameras=..., input_rgb=...)`` (which encodes the images a second time, as the reference's
  keyword call does), the x8 up-sampling of the EFT image and the view's 128^2 target rays;
* ``native``: ``NativeSceneBuilder.build`` (view-batched ``feature_cache``, every ray grid in one launch).

Both include the same host camera maths.  Each number is the median of ``--reps`` runs after one warm-up run, from CUDA events around work
that ends in a device synchronise; with the peak device memory of a run and the card's name and power limit.

    python tools/scene_bench.py [--reps 3] [--nc 2 6]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def _scene(n=32):
    """a seeded ring of n cameras around the origin (elevation varying around the ring), 256^2 images"""
    import math
    from sparsefusion_b200 import cameras as C
    g = torch.Generator().manual_seed(0)
    az = torch.arange(n) * (2 * math.pi / n)
    eye = torch.stack((5 * torch.sin(az), 1.0 + 0.5 * torch.sin(2 * az), 5 * torch.cos(az)), dim=-1)
    R, T = C.look_at_view_transform(eye, torch.zeros(1, 3), torch.tensor([[0.0, 1.0, 0.0]]))
    cams = C.PerspectiveCameras(R, T, torch.full((n, 2), 3.0), torch.zeros(n, 2), torch.full((n, 2), 256.0))
    return cams, torch.rand(n, 3, 256, 256, generator=g), torch.ones(n, 1, 256, 256)


def per_view_build(eft, cams, rgb, input_idx, dev):
    """the cache the way the reference builds it, view by view (distillation.py:73-125), with this package's cameras and ray grids"""
    from sparsefusion_b200 import cameras as C
    from sparsefusion_b200.eft import RayBundle
    cams = C.as_cameras(cams).cpu()
    aug = C.concat_cameras([cams, C.interpolated_path(cams, n=50, theta_offset_max=0.17)])
    aug_rel, aug_vox = C.relative_cameras(aug, [0], True), C.relative_cameras(aug, [0], False)
    cdm = torch.mean(torch.linalg.norm(cams.get_camera_center(), axis=1))
    lengths = torch.linspace(float(cdm - 5.0), float(cdm + 5.0), 20, device=dev).expand(1, 32, 32, 20)
    images = rgb[input_idx].to(dev)
    feats, imgs, t_o = [], [], []
    for ci in range(len(aug_rel)):
        rel = C.relative_cameras(aug_rel, [ci], True)
        q, ctx = rel[ci], rel[input_idx].to(dev)
        o, d = C.grid_rays(q, 32, 32, dev, 256, 256)
        eft.encode(ctx, images)
        rgb_lr, f, _ = eft.batched_forward(RayBundle(o.view(1, 32, 32, 3), d.view(1, 32, 32, 3), lengths, None), n_batches=16, input_cameras=ctx,
                                           input_rgb=images)
        feats.append(f.permute(0, 3, 1, 2))
        imgs.append(F.interpolate(rgb_lr.permute(0, 3, 1, 2), scale_factor=8.0, mode='bilinear'))
        t_o.append(C.grid_rays(aug_vox[ci], 128, 128, dev, 256, 256))
    return torch.cat(feats), torch.cat(imgs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--nc', type=int, nargs='+', default=[2, 6])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('scene_bench needs a CUDA device')
    from oracle import eft_oracle as eo
    from sparsefusion_b200.distillation import NativeSceneBuilder
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    dev = torch.device('cuda', 0)
    eft = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=True)
    eft.load_state_dict(eo.make_params({k: tuple(v.shape) for k, v in eft.state_dict().items()}, seed=0))
    eft = eft.to(dev)
    cams, rgb, mask = _scene()
    builder = NativeSceneBuilder(0)
    card = _card()
    for nc in a.nc:
        idx = [int(i) for i in torch.linspace(0, 31, nc).round().long()]
        ways = {'per_view': lambda: per_view_build(eft, cams, rgb, idx, dev),
                'native': lambda: (lambda c: (c.target_features, c.target_eft_image))(builder.build(eft, cams, rgb, mask, idx))}
        times, peaks, outs = {k: [] for k in ways}, {}, {}
        for rep in range(a.reps + 1):
            for name, fn in ways.items():
                torch.manual_seed(rep)                               # the same circle-path jitter for both ways
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                out = fn()
                e.record()
                torch.cuda.synchronize()
                if rep:
                    times[name].append(s.elapsed_time(e))
                peaks[name] = max(peaks.get(name, 0), torch.cuda.max_memory_allocated(dev))
                outs[name] = out
        rel = lambda a, b: ((a - b).double().norm() / b.double().norm()).item()
        res = dict(card=card, views=82, input_views=nc, query='32x32x20', reps=a.reps,
                   per_view_ms=round(statistics.median(times['per_view']), 1), native_ms=round(statistics.median(times['native']), 1),
                   per_view_ms_all=[round(t, 1) for t in times['per_view']], native_ms_all=[round(t, 1) for t in times['native']],
                   per_view_peak_gb=round(peaks['per_view'] / 2 ** 30, 2), native_peak_gb=round(peaks['native'] / 2 ** 30, 2),
                   features_rel=rel(outs['native'][0], outs['per_view'][0]), eft_image_rel=rel(outs['native'][1], outs['per_view'][1]))
        res['speedup'] = round(res['per_view_ms'] / res['native_ms'], 2)
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
