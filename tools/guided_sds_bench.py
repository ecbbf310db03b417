"""Device time of the SDS (fusion) sub-step with and without classifier-free guidance: cond_scale 1 against cond_scale 3, the full UNet at
32^2 latents, the full VAE at 256^2, LPIPS on, 128^2 rays, in the SDS phase (itr > 1000).

* S = 1: ``Distiller.fusion_substep``, the reference's iteration (one target view, guided runs through ``PLMSSampler.sample``);
* S = 2, 4, 8: ``MultiSceneDistiller.fusion_substep`` (every scene at its own noise level, guided runs through ``sample_rows``).

Both arms hold their own networks and samplers; scene k is seeded k in both, so they draw the same views and noise levels and run the same
number of UNet evaluations.  The arms are timed alternately: CUDA events around the same max(steps, 12 / S) sub-steps per repetition, after
a warm-up that captures every UNet graph a run can reach (batch sizes 1..S unguided, 2, 4, .., 2S guided).  The repetitions draw different
noise levels, so each arm's time is the total over all repetitions divided by the sub-steps, and ``guidance_ratio`` the ratio of those
totals (the per-repetition ratios are listed too).  Reported per arm: ms per sub-step, UNet rows evaluated per sub-step, the device memory
reserved by the private pools of the arm's graph captures, and the peak allocated memory; with the card's name and power limit.

    python tools/guided_sds_bench.py [--scenes 1 2 4 8] [--steps 3] [--reps 5] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SCALES = (1.0, 3.0)


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def _graph_pools():
    """reserved bytes per private memory pool (every captured CUDA graph allocates from its own pool; (0, 0) is the default pool)"""
    pools = {}
    for seg in torch.cuda.memory._snapshot()['segments']:
        pid = tuple(seg['segment_pool_id'])
        if pid != (0, 0):
            pools[pid] = pools.get(pid, 0) + seg['total_size']
    return pools


def _arm(S, cs, models, percep, dev):
    """(fusion_substep, sampler) of one arm, with every graph shape of its runs captured; returns also the MB its captures reserved"""
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
        d = Distiller(ngp(), vae, vldm, opt, caches[0], seed=0, percep=percep, cond_scale=cs)
        run, sampler = d.fusion_substep, d.sampler
    else:
        d = MultiSceneDistiller([ngp() for _ in range(S)], vae, vldm, opt, caches, seeds=list(range(S)), percep=percep, max_batch=8, cond_scale=cs)
        run, sampler = d.fusion_substep, d.sampler
    torch.cuda.synchronize()
    before = _graph_pools()
    with torch.no_grad():                                   # S distinct run lengths: every active-row count 1..S, so every graph of the arm
        lat = torch.randn(S, 4, 32, 32, device=dev)
        feats = torch.cat([c.target_features[:1] for c in caches])
        sampler.sample_rows(lat, [0.99 - 0.1 * k for k in range(S)], feats, cond_scale=cs)
    torch.cuda.synchronize()
    after = _graph_pools()
    return run, sampler, sum(b for pid, b in after.items() if pid not in before) / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, nargs='+', default=[1, 2, 4, 8])
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('guided_sds_bench: needs a CUDA device')
    from bench import build_gpu
    card = _card()
    print('card', card, flush=True)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    _, models, _, kw = build_gpu(0, 1, dev)
    from sparsefusion_b200.plms import PLMSSampler
    with torch.no_grad():       # one-time allocations (packed weights, workspaces) outside every arm's capture measurement
        for cs in SCALES:
            PLMSSampler(models['vldm'], 50).sample_rows(torch.randn(1, 4, 32, 32, device=dev), [0.5], torch.randn(1, 256, 32, 32, device=dev),
                                                        cond_scale=cs)
    res = dict(card=card, latent=32, image=256, rays=128, plms_steps=50, lpips=True, steps=a.steps, reps=a.reps, scenes={})
    for S in a.scenes:
        K = max(a.steps, 12 // S)                           # at least ~1 s of device time per timed window
        arms, captured = {}, {}
        for cs in SCALES:
            run, sampler, mb = _arm(S, cs, models, kw['percep'], dev)
            arms[cs], captured[cs] = (run, sampler), mb
        itr = 1001
        for _ in range(3):                                  # warm-up
            for cs in SCALES:
                arms[cs][0](itr)
            itr += 1
        times, rows, peak = {cs: [] for cs in SCALES}, {cs: 0 for cs in SCALES}, {cs: 0 for cs in SCALES}
        for _ in range(a.reps):
            for cs in SCALES:
                run, sampler = arms[cs]
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(K):
                    run(itr + i)
                    calls = sampler.last_row_calls if S > 1 else [sampler.last_unet_calls]
                    rows[cs] += sum(calls) * (2 if cs != 1 else 1)
                e1.record()
                torch.cuda.synchronize()
                times[cs].append(e0.elapsed_time(e1) / K)
                peak[cs] = max(peak[cs], torch.cuda.max_memory_allocated())
            itr += K
        rec = dict(substeps_per_rep=K)
        for cs in SCALES:
            rec[f'cs{cs:g}'] = dict(ms_per_substep=round(sum(times[cs]) / len(times[cs]), 1), all_ms=[round(t, 1) for t in times[cs]],
                                    unet_rows_per_substep=round(rows[cs] / (K * a.reps), 1), graph_capture_mb=round(captured[cs], 1),
                                    peak_allocated_gb=round(peak[cs] / 1e9, 2))
        rec['guidance_ratio'] = round(sum(times[3.0]) / sum(times[1.0]), 3)
        rec['guidance_ratio_per_rep'] = [round(g / u, 3) for g, u in zip(times[3.0], times[1.0])]
        res['scenes'][str(S)] = rec
        print(f'S={S}:', json.dumps(rec), flush=True)
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
