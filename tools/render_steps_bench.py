"""Device time of the fused NeRF render at several (num_steps, upsample_steps) counts, on cuda:0:

    python tools/render_steps_bench.py [--reps 7] [--warmup 3]

  train: one train-mode NeRFNetwork.render of 128 x 128 rays (perturbed, the distillation step's render) plus its backward
         through the field parameters -- what a distillation step pays per render;
  eval:  one eval-mode render_batched of 256 x 256 rays (16 384-ray chunks, the scoring render).
Each figure is the median over `reps` repetitions of CUDA-event time, with the counts alternated inside every repetition so that
clock drift and other tenants of the GPU spread over all of them alike.  The GPU name and power limit are read in the same run and
printed with the table; nothing is written.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COUNTS = ((32, 32), (64, 0), (64, 64), (128, 128))


def gpu_identity():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    name, power = (s.strip() for s in q.stdout.strip().split(',')) if q.returncode == 0 else (torch.cuda.get_device_name(0), 'unknown')
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('render_steps_bench needs a CUDA device')
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200 import image_glue as glue
    torch.cuda.set_device(0)
    opt = get_default_torch_ngp_opt()
    net = NeRFNetwork(opt)
    sd = net.state_dict()
    sd.update(no.make_field_params(seed=0))
    net.load_state_dict(sd)
    net = net.cuda()
    cam = no.circle_cameras(64)[17]
    rays = {hw: glue.rays_from_camera(torch.from_numpy(cam[0]).cuda(), torch.from_numpy(cam[1]).cuda(), hw, hw, 4.0) for hw in (128, 256)}

    def train(Tc, Tf):
        net.train()
        ro, rd = rays[128]
        out = net.render(ro[None], rd[None], staged=False, perturb=True, bg_color=0, shading='albedo', force_all_rays=True,
                         **dict(vars(opt), num_steps=Tc, upsample_steps=Tf))
        (out['image'].square().mean() + 0.1 * out['weights_sum'].mean()).backward()
        net.zero_grad(set_to_none=True)

    def evaluate(Tc, Tf):
        net.eval()
        ro, rd = rays[256]
        with torch.no_grad():
            net.render_batched(ro[None], rd[None], batched=True, bg_color=0, perturb=False, shading='albedo',
                               **dict(vars(opt), num_steps=Tc, upsample_steps=Tf, max_ray_batch=16384))

    work = {'train': train, 'eval': evaluate}
    for _ in range(a.warmup):
        for fn in work.values():
            for c in COUNTS:
                fn(*c)
    torch.cuda.synchronize()
    times = {(k, c): [] for k in work for c in COUNTS}
    for _ in range(a.reps):
        for k, fn in work.items():
            for c in COUNTS:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn(*c)
                e.record()
                e.synchronize()
                times[(k, c)].append(s.elapsed_time(e))
    name, power = gpu_identity()
    med = {key: sorted(v)[len(v) // 2] for key, v in times.items()}
    print(f'{name}, power limit {power}; median of {a.reps} alternating repetitions (CUDA events), ms')
    print(f'{"num_steps + upsample_steps":>28s} {"train 128^2 fwd+bwd":>20s} {"eval 256^2":>12s}')
    for c in COUNTS:
        print(f'{f"{c[0]} + {c[1]}":>28s} {med[("train", c)]:20.2f} {med[("eval", c)]:12.2f}')
    print(json.dumps({'gpu': name, 'power_limit': power, 'reps': a.reps,
                      'ms': {f'{k} {c[0]}+{c[1]}': {'median': med[(k, c)], 'min': min(times[(k, c)]), 'max': max(times[(k, c)])} for k, c in times}}))


if __name__ == '__main__':
    main()
