"""Cost of the periodic progress outputs and of the entropy term, on bench.py's flagship scene and models (FULL UNet, SD VAE, LPIPS, 128^2
rays, 256^2 images).

    python tools/progress_bench.py [--steps 20] [--repeats 5] [--out progress_bench.json]

(1) One progress write (``progress.ProgressWriter.write``: the history rows' device-to-host copy, the two Pillow plots, the 256^2 eval-mode
    snapshot render and the JPEG encodes), median over ``--repeats`` writes after one warm-up, against ``--steps`` reference iterations
    (``Distiller.step`` in the SDS phase, at bench.py's noise levels): the reference writes every 20 iterations.
(2) The reference iteration's time with lambda_entropy 0 against 1e-2 after a warm-up: per repeat, ``--steps`` of bench.py's noise levels,
    each run once per arm back to back (the order alternating), so both arms do the same UNet work; the per-repeat differences are printed.
Times are wall clock around work that ends in a device synchronise.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f'unknown ({e})'


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('progress_bench.py measures on the GPU; no CUDA device is visible')
    import bench
    from sparsefusion_b200.evaluate import EvalViews
    from sparsefusion_b200.progress import ProgressWriter
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    Distiller, nets, scene, kw = bench.build_gpu(0, 1, dev)
    thres = bench.max_thres_sequence(2, 2 * a.steps + 2)
    cache = scene.to(dev)
    res = dict(card=_card())
    # (2) step time at lambda_entropy 0 and 1e-2 on the same workload: each noise level runs once per arm, back to back (the order alternating),
    # so both arms make the same PLMS runs (min(int(100 max_thres), 50) UNet evaluations each)
    dist = Distiller(cache=cache, max_itr=3000, **nets, **kw)
    for i in range(2):
        dist.step(1001 + i, max_thres=thres[i])
    arms = (0.0, 1e-2)
    times, calls, diffs = {le: [] for le in arms}, {le: 0 for le in arms}, []
    itr = 1003
    for rep in range(a.repeats):
        t = {le: 0.0 for le in arms}
        for i in range(a.steps):
            mt = thres[(rep * a.steps + i) % len(thres)]
            for le in (arms if i % 2 == 0 else arms[::-1]):
                dist.lambda_entropy = le
                t[le] += _timed(lambda: dist.step(itr, max_thres=mt))
                calls[le] += dist.last['unet_calls']
                itr += 1
        for le in arms:
            times[le].append(t[le] / a.steps)
        diffs.append(100 * (t[1e-2] - t[0.0]) / t[0.0])
    assert calls[0.0] == calls[1e-2], calls
    ms0, ms1 = 1e3 * statistics.median(times[0.0]), 1e3 * statistics.median(times[1e-2])
    res.update(step_ms_lambda_entropy_0=ms0, step_ms_lambda_entropy_1e_2=ms1, entropy_cost_pct=100 * (ms1 - ms0) / ms0,
               entropy_cost_pct_per_repeat=diffs, unet_evals_per_arm=calls[0.0])
    # (1) one progress write against --steps reference iterations
    dist.lambda_entropy = 0.0
    n_in = cache.input_rgb.shape[0]
    views = EvalViews(rays_o=torch.nn.functional.interpolate(cache.input_rays_o.reshape(n_in, 128, 128, 3).permute(0, 3, 1, 2), size=(256, 256),
                                                             mode='bilinear').permute(0, 2, 3, 1).reshape(n_in, -1, 3).contiguous(),
                      rays_d=torch.nn.functional.interpolate(cache.input_rays_d.reshape(n_in, 128, 128, 3).permute(0, 3, 1, 2), size=(256, 256),
                                                             mode='bilinear').permute(0, 2, 3, 1).reshape(n_in, -1, 3).contiguous(),
                      rgb=cache.input_rgb, mask=cache.input_mask)
    with tempfile.TemporaryDirectory() as tmp:
        w = ProgressWriter(tmp, ['scene'], [views], [list(range(n_in))], nets['opt'])
        w.write(itr - 1, [dist])                               # warm-up
        writes = []
        for rep in range(a.repeats):
            t20 = _timed(lambda: [dist.step(itr + i, max_thres=thres[(itr + i) % len(thres)]) for i in range(a.steps)])
            itr += a.steps
            writes.append((_timed(lambda: w.write(itr - 1, [dist])), t20))
    wm = 1e3 * statistics.median(x for x, _ in writes)
    sm = 1e3 * statistics.median(y for _, y in writes)
    res.update(progress_write_ms=wm, steps=a.steps, steps_ms=sm, write_share_pct=100 * wm / sm)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
