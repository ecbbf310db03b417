"""Mint tests/golden/plms_cfg_small.npz: classifier-free-guided PLMS sampling from pure noise by the REFERENCE's own
external.plms.PLMSSampler (with sparsefusion.vldm.DDPM and external.imagen_pytorch.Unet, imported unmodified) on the SMALL UNet
of oracle.unet_oracle, on the CPU.  Needs the reference source tree at oracle/gen_golden.py's REF:

    python tools/gen_plms_cfg_golden.py

Every Gaussian draw of the sampler is injected from oracle.unet_oracle.NoiseSource(seed=7) in the reference's call order, as
oracle/gen_golden.py's PLMS vectors are, so the GPU test can replay the same draws.  Batch 2, cond_scale 3 and 1.5.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import unet_oracle as uo  # noqa: E402
from oracle.gen_golden import GOLD, REF, _inputs, _reference_unet  # noqa: E402

BATCH = 2
SCALES = (3.0, 1.5)


def main():
    sys.path.insert(0, REF)
    from sparsefusion.vldm import DDPM
    from external.plms import PLMSSampler
    cfg = uo.SMALL
    sd = uo.make_params(cfg, seed=0)
    unet = _reference_unet(cfg, sd)
    ddpm = DDPM(channels=cfg.channels, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None,
                image_sizes=(cfg.image_size,), timesteps=500, cond_drop_prob=0.1, pred_objectives='noise',
                conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False,
                dynamic_thresholding_percentile=.68, clip_value=10)
    ddpm.unets[0].load_state_dict(sd)
    ddpm.eval()
    sampler = PLMSSampler(ddpm, 50)
    _, cond, _ = _inputs(cfg, BATCH, seed=5)
    ref_unet = ddpm.unets[0]
    forward_with_cond_scale = ref_unet.forward_with_cond_scale
    out = {'cond': cond.numpy(), 'batch': BATCH, 'noise_seed': 7}
    for s in SCALES:
        calls = [0]

        def counted(*a, **k):
            calls[0] += 1
            return forward_with_cond_scale(*a, **k)
        src = uo.NoiseSource(seed=7)
        orig, orig_randn = torch.randn_like, torch.randn
        torch.randn_like = lambda t, **kw: src(t)                          # every draw in plms.py goes through randn_like ...
        torch.randn = lambda shape, **kw: src(torch.empty(tuple(shape)))   # ... except the start image of sample() from noise (plms.py:73)
        ref_unet.forward_with_cond_scale = counted
        try:
            img = sampler.sample(cond_images=cond, cond_scale=s, use_tqdm=False)
        finally:
            torch.randn_like, torch.randn = orig, orig_randn
            del ref_unet.forward_with_cond_scale
        key = f'{s:.1f}'
        print(f'[plms_cfg cond_scale={s}] unet evaluations {calls[0]} draws {src.count} |img| {img.norm():.4f}')
        out[f'img_{key}'] = img.numpy()
        out[f'calls_{key}'] = calls[0]
        out[f'draws_{key}'] = src.count
    np.savez_compressed(os.path.join(GOLD, 'plms_cfg_small.npz'), **out)


if __name__ == '__main__':
    main()
