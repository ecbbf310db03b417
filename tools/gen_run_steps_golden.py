"""Mint tests/golden/ngp_run_steps.npz: the REFERENCE's own NeRFNetwork.render (external/nerf/network_grid.py over renderer_df.py,
imported unmodified through oracle.gen_golden._import_reference_ngp) at sample counts other than 64 + 64, on the CPU.  Needs the
reference source tree at oracle/gen_golden.py's REF:

    python tools/gen_run_steps_golden.py

Rays, field parameters and the loss target are those of ngp_run.npz.  For each (num_steps, upsample_steps) of STEPS the two torch.rand
draws of run() (perturbation :363, sample_pdf :31; none at upsample_steps = 0) are injected from np.random.default_rng(seed) with
seed = 1000 * num_steps + upsample_steps, perturbation first.  Recorded per count: the train-mode image, weights_sum and depth, the
parameter gradients of ((image - target)^2).mean() + 0.1 weights_sum.mean() (embeddings at every 4th row of ngp_run.npz's rows plus the absolute
sum), and the eval-mode (deterministic) image and weights_sum.

num_steps = 2 with importance samples is not among them: the reference's sample_pdf fails there (weights[1:-1] is empty, and so is the
leading zero it slices from the empty cdf), so the renderer's z_mid[0] convention at that count is pinned by the per-stage tests only.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ngp_oracle as no  # noqa: E402
from oracle.gen_golden import GOLD, _import_reference_ngp  # noqa: E402

STEPS = ((128, 128), (32, 32), (48, 16), (100, 28), (64, 0))


def draws_for(N, num_steps, upsample_steps):
    """the injected torch.rand draws of run() at one count, in call order"""
    rng = np.random.default_rng(1000 * num_steps + upsample_steps)
    pn = rng.random((N, num_steps), dtype=np.float32)
    un = rng.random((N, upsample_steps), dtype=np.float32)
    return pn, un


def main():
    ng, _ = _import_reference_ngp()
    g = np.load(os.path.join(GOLD, 'ngp_run.npz'))
    ro, rd = torch.from_numpy(g['rays_o']), torch.from_numpy(g['rays_d'])
    N = ro.shape[0]
    tgt = torch.from_numpy(np.random.default_rng(int(g['target_seed'])).random((N, 3), dtype=np.float32))
    rows = g['gemb_rows'][::4]
    out = {'steps': np.array(STEPS, dtype=np.int64)}
    orig_rand = torch.rand
    for Tc, Tf in STEPS:
        opt = SimpleNamespace(cuda_ray=False, max_steps=256, num_steps=Tc, upsample_steps=Tf, update_extra_interval=16, max_ray_batch=4096,
                              albedo_iters=1000, bg_radius=0, density_thresh=10, fp16=True, backbone='grid', w=128, h=128, hw_scale=2, bound=4,
                              min_near=0.1, dt_gamma=0, lambda_entropy=1e-4, lambda_opacity=0, lambda_orient=1e-2, lambda_smooth=0)
        net = ng.NeRFNetwork(opt).train()
        sd = net.state_dict()
        sd.update(no.make_field_params(seed=0))
        net.load_state_dict(sd)
        pn, un = draws_for(N, Tc, Tf)
        draws = [torch.from_numpy(pn)] + ([torch.from_numpy(un)] if Tf > 0 else [])

        def fake_rand(*shape, **kw):
            t = draws.pop(0)
            want = tuple(shape[0]) if len(shape) == 1 and not isinstance(shape[0], int) else tuple(shape)
            assert tuple(t.shape) == want, (t.shape, want)
            return t
        torch.rand = fake_rand
        try:
            r = net.render(ro[None], rd[None], staged=False, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', force_all_rays=True, **vars(opt))
        finally:
            torch.rand = orig_rand
        assert not draws
        image, ws, depth = r['image'].reshape(N, 3), r['weights_sum'].reshape(N), r['depth'].reshape(N)
        loss = ((image - tgt) ** 2).mean() + 0.1 * ws.mean()
        loss.backward()
        grads = {k: v.grad.numpy() for k, v in net.named_parameters()}
        net.eval()
        with torch.no_grad():
            e = net.render(ro[None], rd[None], staged=False, perturb=False, bg_color=0, ambient_ratio=1.0, shading='albedo', **vars(opt))
        tag = f'{Tc}_{Tf}'
        gemb = grads['encoder.embeddings']
        out.update({f'image_{tag}': image.detach().numpy(), f'weights_sum_{tag}': ws.detach().numpy(), f'depth_{tag}': depth.detach().numpy(),
                    f'loss_{tag}': float(loss.detach()), f'gemb_vals_{tag}': gemb[rows], f'gemb_abs_sum_{tag}': float(np.abs(gemb).sum()),
                    f'eval_image_{tag}': e['image'].reshape(N, 3).numpy(), f'eval_weights_sum_{tag}': e['weights_sum'].reshape(N).numpy(),
                    **{f'g_{k}_{tag}': grads[k] for k in no.PARAM_KEYS[1:]}})
        print(f'[run steps {Tc} + {Tf}] loss {float(loss):.8f}  opacity mean {float(ws.mean()):.5f}  eval opacity mean {float(e["weights_sum"].mean()):.5f}')
    np.savez_compressed(os.path.join(GOLD, 'ngp_run_steps.npz'), gemb_rows=rows, **out)


if __name__ == '__main__':
    torch.set_num_threads(os.cpu_count())
    main()
