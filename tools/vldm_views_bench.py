"""Device time of the VLDM baseline of one scene: V novel views (default 32) sampled from pure noise by PLMS (50 steps, max_thres .999) with
the full UNet at 32^2 latents, conditioned on EFT features [V, 256, 32, 32], and decoded by the full VAE to 256^2, at cond_scale 1 and 3.
Two ways, timed alternately in one process:

* ``batched``: ``baselines.sample_vldm_views`` -- the views in one batch (``--max-batch``), one CUDA-graph replay per evaluation (batch 2V
  with guidance: conditional and null rows together), the guided eps formed inside the fused update kernel, one VAE decode;
* ``per_view``: the reference's order -- one view at a time through the reference-shaped ``PLMSSampler.p_sample`` with eager evaluations,
  two ``Unet.forward`` calls per guided step (``forward_with_cond_scale``), then a decode of that view.

Both arms draw every view's noise from the same keyed generators, so their images agree up to fp32 summation order (printed as
``rel``).  Each time is the median of ``--reps`` runs after one warm-up run of each arm (the warm-up of ``per_view`` is one view), from CUDA
events around work that ends in a device synchronise; with the peak device memory and the card's name and power limit.  Random weights:
the timing does not depend on them.

    python tools/vldm_views_bench.py [--views 32] [--reps 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PLMS_STEPS = 50


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        return 'unknown'


def _models():
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.vldm import DDPM
    torch.manual_seed(0)
    unet = Unet(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
                layer_cross_attns=(False,) * 4, cond_images_channels=256, attn_pool_text=False, cond_on_z=False, conditional_embed_dim=None)
    ddpm = DDPM(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(32,), timesteps=500, cond_drop_prob=0.1,
                pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False, clip_value=10).cuda()
    torch.nn.init.normal_(ddpm.unets[0].get_parameter('final_conv.weight'), std=0.02)   # the reference zero-initialises it: eps would be 0
    return ddpm, AutoencoderKL().cuda().eval()


@torch.no_grad()
def per_view(ddpm, vae, feats, seed, cond_scale, views):
    """the reference's order: one view at a time, eager evaluations, the reference-shaped p_sample, then that view's decode"""
    from sparsefusion_b200.baselines import VLDM_MAX_THRES, VLDM_STREAM
    from sparsefusion_b200.distillation import KeyedNoise, unnormalize, view_seed
    from sparsefusion_b200.imagen_pytorch import GaussianDiffusionContinuousTimes
    from sparsefusion_b200.plms import PLMSSampler
    unet, sched = ddpm.unets[0], ddpm.noise_schedulers[0]
    short = GaussianDiffusionContinuousTimes(noise_schedule='cosine', timesteps=PLMS_STEPS)
    out = []
    for v in views:
        sampler = PLMSSampler(ddpm, PLMS_STEPS, use_cuda_graph=False, noise_fn=KeyedNoise([view_seed(seed, 0, v, VLDM_STREAM)], 'cuda'))
        img = sampler.noise_fn(torch.empty(1, 4, 32, 32, device='cuda'))                     # plms.py:73
        sampler.noise_fn(img)                                                               # q_sample's draw (:81)
        old_eps = []
        assert VLDM_MAX_THRES >= .99                                                        # the 50-step schedule from t = 1 (:80-85)
        for t, t_next in short.get_sampling_timesteps(1, device='cuda'):
            img, _, e_t = sampler.p_sample(unet, img, t, t_next, feats[v:v + 1], cond_scale, sched, 'noise', False, old_eps)
            old_eps = (old_eps + [e_t])[-3:]
        x0 = img.clamp(-ddpm.clip_value, ddpm.clip_value)
        out.append(unnormalize(vae.decode(x0 / 0.18215)).clip(0.0, 1.0))
    return torch.cat(out)


def _timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=32)
    ap.add_argument('--max-batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('vldm_views_bench: needs a CUDA device')
    from sparsefusion_b200.baselines import sample_vldm_views
    from sparsefusion_b200.plms import PLMSSampler
    card = _card()
    print('card', card, flush=True)
    ddpm, vae = _models()
    feats = torch.randn(a.views, 256, 32, 32, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
    sampler = PLMSSampler(ddpm, PLMS_STEPS)
    res = dict(card=card, views=a.views, max_batch=a.max_batch, plms_steps=PLMS_STEPS, latent=32, image=256, reps=a.reps)
    all_views = list(range(a.views))
    arms = {'batched': lambda cs: sample_vldm_views(ddpm, vae, feats, seed=0, cond_scale=cs, plms_steps=PLMS_STEPS, max_batch=a.max_batch,
                                                    sampler=sampler),
            'per_view': lambda cs: per_view(ddpm, vae, feats, 0, cs, all_views)}
    for cs in (1.0, 3.0):                                                                   # warm-up: graph capture, time features, allocator
        arms['batched'](cs)
        per_view(ddpm, vae, feats, 0, cs, [0])
    torch.cuda.reset_peak_memory_stats()
    times = {(arm, cs): [] for arm in arms for cs in (1.0, 3.0)}
    images = {}
    peak = {}
    for _ in range(a.reps):
        for cs in (1.0, 3.0):
            for arm, fn in arms.items():
                torch.cuda.reset_peak_memory_stats()
                ms, img = _timed(lambda: fn(cs))
                peak[arm, cs] = max(peak.get((arm, cs), 0), torch.cuda.max_memory_allocated())
                times[arm, cs].append(ms)
                images[arm, cs] = img
                print(f'{arm} cond_scale={cs:g}: {ms:.1f} ms', flush=True)
    for cs in (1.0, 3.0):
        b, p = statistics.median(times['batched', cs]), statistics.median(times['per_view', cs])
        x, y = images['batched', cs].double(), images['per_view', cs].double()
        rel = ((x - y).norm() / y.norm()).item()
        rec = dict(batched_ms=round(b, 1), per_view_ms=round(p, 1), speedup=round(p / b, 2), batched_ms_per_view=round(b / a.views, 2),
                   per_view_ms_per_view=round(p / a.views, 2), batched_all_ms=[round(t, 1) for t in times['batched', cs]],
                   per_view_all_ms=[round(t, 1) for t in times['per_view', cs]], rel_batched_vs_per_view=rel,
                   peak_gb_batched=round(peak['batched', cs] / 1e9, 2), peak_gb_per_view=round(peak['per_view', cs] / 1e9, 2))
        res[f'cs{cs:g}'] = rec
        print(f'cond_scale={cs:g}:', json.dumps(rec), flush=True)
    res['guidance_ratio_batched'] = round(res['cs3']['batched_ms'] / res['cs1']['batched_ms'], 3)
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
