"""Device time of the finite-difference normal stencils (sfb_ngp_field_normal_forward / _backward) against the composed form the
reference uses (network_grid.py:91-152): 6 or 60 field evaluations on materialised shifted / jittered points, one sfb_ngp_field_forward
(or _backward) call each, and a torch reduction.  Both run alternately in one process, on the points of 128^2 and 256^2 rays x 128 samples.
Also one 256^2 frame of evaluate.render_views(shading='normal').

    python tools/shading_bench.py [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('shading_bench needs a CUDA device')
    from sparsefusion_b200 import _lib as lib
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt, jitter_key, stencil_forward
    torch.manual_seed(0)
    net = NeRFNetwork(get_default_torch_ngp_opt()).cuda()
    with torch.no_grad():
        net.encoder.embeddings.uniform_(-0.5, 0.5)
    f = lib.fptr
    enc = net.encoder
    P = [t.detach() for t in net._field_params()]
    geo = (f(P[0]), lib.iptr(enc.offsets), float(math.log2(enc.per_level_scale)), int(enc.base_resolution), float(net.bound))
    W = [f(t) for t in P[1:]]
    res = {'card': _card(), 'reps': args.reps}

    def field_fwd(x):
        s = torch.empty(x.shape[0], device='cuda')
        lib.call('sfb_ngp_field_forward', f(x), None, None, None, 0, x.shape[0], *geo, *W, f(s), None, lib.stream())
        return s

    def composed_plain(x, eps=1e-2):
        sig = []
        for a in range(3):
            for sgn in (1, -1):
                e = torch.zeros(3, device='cuda')
                e[a] = sgn * eps
                sig.append(field_fwd((x + e).clamp(-net.bound, net.bound).contiguous()))
        return torch.stack([0.5 * (sig[2 * a] - sig[2 * a + 1]) / eps for a in range(3)], -1)

    def composed_smooth(x, eps=0.3, k=10):
        m = []
        for a in range(3):
            for sgn in (1, -1):
                e = torch.zeros(3, device='cuda')
                e[a] = sgn * eps
                xs = (x + e).clamp(-net.bound, net.bound)
                m.append(torch.stack([field_fwd((xs + torch.rand_like(xs) * 0.6 - 0.3).contiguous()) for _ in range(k)]).mean(0))
        return torch.stack([0.5 * (m[2 * a] - m[2 * a + 1]) / eps for a in range(3)], -1)

    for R in (128, 256):
        B = R * R * 128
        x = ((torch.rand(B, 3, device='cuda') * 2 - 1) * 1.5).contiguous()
        g = torch.randn(B, 3, device='cuda')
        grads = [torch.zeros_like(t) for t in P]

        def stencil_bwd():
            fd = torch.empty(B, 3, device='cuda')
            lib.call('sfb_ngp_field_normal_forward', f(x), None, None, None, 0, B, *geo, *W, 6, 1, 1e-2, 0.0, None, f(fd), None, None, None,
                     lib.stream())
            lib.call('sfb_ngp_field_normal_backward', f(x), None, None, None, 0, B, *geo, *W, 1e-2, None, None, f(g), *[f(t) for t in grads],
                     lib.stream())

        def composed_bwd():
            gs = torch.empty(B, device='cuda')
            for a in range(3):
                for sgn in (1, -1):
                    e = torch.zeros(3, device='cuda')
                    e[a] = sgn * 1e-2
                    xs = (x + e).clamp(-net.bound, net.bound).contiguous()
                    torch.mul(g[:, a], sgn * 0.5 / 1e-2, out=gs)
                    lib.call('sfb_ngp_field_backward', f(xs), None, None, None, 0, B, *geo, *W, f(gs), None, *[f(t) for t in grads], None,
                             lib.stream())

        key = jitter_key('cuda')
        cases = {'plain_fwd': (lambda: stencil_forward(net, B, x=x, want_normal=False), lambda: composed_plain(x)),
                 'plain_fwd_bwd': (stencil_bwd, lambda: (composed_plain(x), composed_bwd())),
                 'smooth_fwd': (lambda: stencil_forward(net, B, x=x, k=10, eps=0.3, radius=0.3, key=key, want_normal=False),
                                lambda: composed_smooth(x))}
        for name, (ours, base) in cases.items():
            t_ours, t_base = [], []
            for _ in range(3):                       # alternate the two forms
                t_ours.append(_time(ours, args.reps))
                t_base.append(_time(base, args.reps))
            res[f'{R}x{R}x128/{name}'] = {'stencil_ms': round(min(t_ours), 3), 'composed_ms': round(min(t_base), 3),
                                          'speedup': round(min(t_base) / min(t_ours), 2)}
        del x, g, grads
        torch.cuda.empty_cache()

    # one 256^2 eval frame with the smoothed-normal shading, as evaluate.render_views renders it (headlight, per-view seeded jitter)
    from sparsefusion_b200.evaluate import CIRCLE_STREAM, render_views
    o = torch.zeros(1, 256 * 256, 3, device='cuda')
    o[..., 2] = 2.5
    d = torch.randn(1, 256 * 256, 3, device='cuda') * 0.2
    d[..., 2] = -1
    d = d / d.norm(dim=-1, keepdim=True)
    opt = get_default_torch_ngp_opt()
    frame = lambda: render_views(net, o, d, (256, 256), opt, seed=0, stream=CIRCLE_STREAM, shading='normal')      # noqa: E731
    res['render_views_256x256_normal_ms'] = round(min(_time(frame, 2) for _ in range(3)), 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
