"""Device time of the SDS (fusion) sub-step with the multi-step PLMS target against the one-step target: ``sds_method`` 'plms' against
'onestep', the full UNet at 32^2 latents, the full VAE at 256^2, LPIPS on, 128^2 rays, in the SDS phase (itr > 1000), at cond_scale 1 and 3.

* S = 1: ``Distiller.fusion_substep``, the reference's iteration (one target view);
* S = 2, 4, 8: ``MultiSceneDistiller.fusion_substep`` (every scene at its own noise level; one ``sample_rows`` run or one ``forward_noloss``
  call per chunk).

Both arms hold their own networks; scene k is seeded k in both, so they draw the same views and the same noise levels.  The arms are timed
alternately with CUDA events around the same max(steps, 12 / S) sub-steps per repetition, after a warm-up that captures every UNet graph a
run can reach.  Reported per arm: ms per sub-step (total over all repetitions over the sub-steps), UNet rows evaluated and graph replays per
sub-step, the peak allocated memory, and ``onestep_speedup`` (the ratio of the totals); with the card's name and power limit.

    python tools/onestep_sds_bench.py [--scenes 1 2 4 8] [--scales 1 3] [--steps 3] [--reps 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

METHODS = ('plms', 'onestep')


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def _arm(S, cs, method, models, percep, dev):
    """the distiller of one arm; the PLMS arm's graphs of every active-row count are captured here"""
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, SceneCache
    from sparsefusion_b200.network_grid import NeRFNetwork
    from sparsefusion_b200.synthetic import synthetic_scene
    vae, vldm, opt = models['vae'], models['vldm'], models['opt']

    def ngp():
        n = NeRFNetwork(opt)
        n.encoder.embeddings.data.uniform_(-0.5, 0.5)
        return n.to(dev).train()
    caches = [SceneCache(**synthetic_scene(n_target=8, seed=k)).to(dev) for k in range(S)]
    if S == 1:
        d = Distiller(ngp(), vae, vldm, opt, caches[0], seed=0, percep=percep, cond_scale=cs, sds_method=method)
    else:
        d = MultiSceneDistiller([ngp() for _ in range(S)], vae, vldm, opt, caches, seeds=list(range(S)), percep=percep, max_batch=8,
                                cond_scale=cs, sds_method=method)
    if method == 'plms':
        with torch.no_grad():                               # S distinct run lengths: every active-row count 1..S, so every graph of the arm
            lat = torch.randn(S, 4, 32, 32, device=dev)
            feats = torch.cat([c.target_features[:1] for c in caches])
            d.sampler.sample_rows(lat, [0.99 - 0.1 * k for k in range(S)], feats, cond_scale=cs)
    return d


def _counts(d, S, cs, method):
    """(UNet rows evaluated, graph replays) of the sub-step just run"""
    mult = 2 if cs != 1 else 1
    if method == 'onestep':
        return S * mult, d.last['graph_replays']
    if S == 1:
        return d.sampler.last_unet_calls * mult, d.sampler.last_graph_replays
    return sum(d.sampler.last_row_calls) * mult, d.last['graph_replays']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, nargs='+', default=[1, 2, 4, 8])
    ap.add_argument('--scales', type=float, nargs='+', default=[1.0, 3.0])
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('onestep_sds_bench: needs a CUDA device')
    from bench import build_gpu
    card = _card()
    print('card', card, flush=True)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    _, models, _, kw = build_gpu(0, 1, dev)
    res = dict(card=card, latent=32, image=256, rays=128, plms_steps=50, lpips=True, steps=a.steps, reps=a.reps, runs={})
    for S in a.scenes:
        K = max(a.steps, 12 // S)                           # at least ~1 s of device time per timed window of the PLMS arm
        for cs in a.scales:
            arms = {m: _arm(S, cs, m, models, kw['percep'], dev) for m in METHODS}
            itr = 1001
            for _ in range(3):                              # warm-up: the one-step arm captures its graph here
                for m in METHODS:
                    arms[m].fusion_substep(itr)
                itr += 1
            times, rows, replays, peak = ({m: [] for m in METHODS}, {m: 0 for m in METHODS}, {m: 0 for m in METHODS}, {m: 0 for m in METHODS})
            for _ in range(a.reps):
                for m in METHODS:
                    d = arms[m]
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for i in range(K):
                        d.fusion_substep(itr + i)
                        r, g = _counts(d, S, cs, m)
                        rows[m] += r
                        replays[m] += g
                    e1.record()
                    torch.cuda.synchronize()
                    times[m].append(e0.elapsed_time(e1) / K)
                    peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
                itr += K
            rec = dict(substeps_per_rep=K)
            n = K * a.reps
            for m in METHODS:
                rec[m] = dict(ms_per_substep=round(sum(times[m]) / len(times[m]), 1), all_ms=[round(t, 1) for t in times[m]],
                              unet_rows_per_substep=round(rows[m] / n, 1), graph_replays_per_substep=round(replays[m] / n, 1),
                              peak_allocated_gb=round(peak[m] / 1e9, 2))
            rec['onestep_speedup'] = round(sum(times['plms']) / sum(times['onestep']), 2)
            res['runs'][f'S{S}_cs{cs:g}'] = rec
            print(f'S={S} cond_scale={cs:g}:', json.dumps(rec), flush=True)
            del arms
            torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
