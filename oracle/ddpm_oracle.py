"""oracle/ddpm_oracle.py -- CPU restatement of the reference's ancestral sampler ``DDPM.sample`` and the recipe that mints its golden vectors.

TEST INFRASTRUCTURE ONLY, like oracle/unet_oracle.py (whose UNet restatement, schedule functions and ``NoiseSource`` it uses).

    python oracle/ddpm_oracle.py      # tests/golden/ddpm_small.npz, tests/golden/ddpm_full.npz

Run in the BUILD container only: minting imports the reference's own ``sparsefusion.vldm.DDPM`` from /root/reference (unmodified), routes its
``torch.randn`` / ``torch.randn_like`` draws to a ``NoiseSource`` exactly as ``oracle/gen_golden.py gen_plms`` does, and asserts that
``ddpm_sample`` reproduces the reference with the same draw count.  ``ddpm_sample`` itself runs anywhere.
"""
from __future__ import annotations

import os
import sys
from typing import Callable, Tuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.unet_oracle import _pad, alpha_cosine_log_snr, predict_start_from_noise, q_posterior  # noqa: E402


def ddpm_sample(eps_fn: Callable[[torch.Tensor, torch.Tensor, float], torch.Tensor], shape: Tuple[int, ...], T: int,
                noise: Callable[[torch.Tensor], torch.Tensor], cond_scale: float = 1.0, dynamic: bool = False,
                percentile: float = 0.95, clip_value: float = 1.0, dtype=torch.float32) -> torch.Tensor:
    """Restates ``DDPM.sample(cond_images=..., batch_size=B, cond_scale=...)`` (sparsefusion/vldm.py:289-443) for one
    cosine-schedule unet, ``pred_objective='noise'``, ``clip_output=True``, no inpainting: ``p_sample_loop`` (:363-443),
    ``p_sample`` (:337-361) and ``p_mean_variance`` (:289-335).

    ``eps_fn(x, log_snr, cond_drop_prob)`` is the UNet with its conditioning bound; ``cond_drop_prob=1`` is the null
    branch of ``forward_with_cond_scale`` (cond_images zeroed).  ``noise`` replaces every Gaussian draw: the start image
    (``torch.randn(shape)``, :385) then one per step (:356), T + 1 in all.  Returns the final latents, clamped to
    +-clip_value (:434-435); ``unnormalize_img`` is the identity for ``auto_normalize_img=False``.
    """
    b = shape[0]
    img = noise(torch.empty(shape, dtype=dtype))
    lin = torch.linspace(1., 0., T + 1, dtype=torch.float32)                 # get_sampling_timesteps (imagen_pytorch.py:226-231)
    for i in range(T):
        t, t_next = lin[i].to(dtype).expand(b), lin[i + 1].to(dtype).expand(b)
        log_snr = alpha_cosine_log_snr(t)
        e = eps_fn(img, log_snr, 0.)
        if cond_scale != 1:                                                      # imagen_pytorch.py:1464-1468
            null = eps_fn(img, log_snr, 1.)
            e = null + (e - null) * cond_scale
        x0 = predict_start_from_noise(img, t, e)
        if dynamic:                                                              # vldm.py:318-330
            s = torch.quantile(x0.reshape(b, -1).abs(), percentile, dim=-1).clamp(min=1.)
            s = _pad(x0, s)
            x0 = x0.clamp(-s, s) / s
        else:
            x0 = x0.clamp(-clip_value, clip_value)
        mean, _, logvar = q_posterior(x0, img, t, t_next)
        z = noise(img)
        mask = (1 - (t_next == 0).to(dtype)).view(b, *((1,) * (len(shape) - 1)))
        img = mean + mask * (0.5 * logvar).exp() * z
    return img.clamp(-clip_value, clip_value)


CASES = {   # tag: (config, timesteps, batch, cond_scale, dynamic_thresholding, clip_value, file)
    'a': ('SMALL', 500, 1, 1.0, False, 10.0, 'ddpm_small'),    # SparseFusion's VLDM (utils/load_model.py:76-91)
    'b': ('SMALL', 500, 2, 3.0, False, 10.0, 'ddpm_small'),    # classifier-free guidance, two views with distinct conditioning
    'c': ('SMALL', 100, 1, 1.0, True, 1.0, 'ddpm_small'),      # DDPM's constructor defaults: dynamic thresholding at percentile 0.95
    'd': ('FULL', 500, 1, 1.0, False, 10.0, 'ddpm_full'),
}
NOISE_SEED, COND_SEED = 13, 5


def cond_images(cfg, batch, seed=COND_SEED) -> torch.Tensor:
    """the conditioning of a case: oracle/gen_golden.py's ``_inputs`` stream (x drawn first, then cond_images)"""
    rng = np.random.default_rng(seed)
    h = cfg.image_size
    rng.standard_normal((batch, cfg.channels, h, h), dtype=np.float32)
    return torch.from_numpy(rng.standard_normal((batch, cfg.cond_images_channels, h, h), dtype=np.float32))


def mint(gold_dir: str = os.path.join(ROOT, 'tests', 'golden')) -> None:
    """final latents of the REFERENCE's own DDPM.sample (sparsefusion/vldm.py:446-555) with every Gaussian draw routed to a NoiseSource, and the
    check that ``ddpm_sample`` reproduces them"""
    from oracle import unet_oracle as uo
    from oracle.gen_golden import REF, _reference_unet
    sys.path.insert(0, REF)
    from sparsefusion.vldm import DDPM
    out = {'small': {}, 'full': {}}
    for tag, (cfg_name, T, batch, cond_scale, dynamic, clip, fname) in CASES.items():
        cfg = getattr(uo, cfg_name)
        sd = uo.make_params(cfg, seed=0)
        ddpm = DDPM(channels=cfg.channels, unets=(_reference_unet(cfg, sd),), conditional_encoder=None, conditional_embed_dim=None,
                    image_sizes=(cfg.image_size,), timesteps=T, cond_drop_prob=0.1, pred_objectives='noise', conditional=False,
                    auto_normalize_img=False, clip_output=True, dynamic_thresholding=dynamic, dynamic_thresholding_percentile=0.95, clip_value=clip)
        ddpm.unets[0].load_state_dict(sd)
        ddpm.eval()
        cond = cond_images(cfg, batch)
        src = uo.NoiseSource(seed=NOISE_SEED)
        orig, orig_randn = torch.randn_like, torch.randn
        torch.randn_like = lambda t, **kw: src(t)                                  # p_sample's draw (vldm.py:356) ...
        torch.randn = lambda shape, **kw: src(torch.empty(tuple(shape)))          # ... and the start image (:385)
        try:
            img = ddpm.sample(cond_images=cond, batch_size=batch, cond_scale=cond_scale, use_tqdm=False)
        finally:
            torch.randn_like, torch.randn = orig, orig_randn
        src2 = uo.NoiseSource(seed=NOISE_SEED)
        eps_fn = lambda x, ls, drop: uo.unet_forward(sd, cfg, x, ls, cond * (1. - drop))
        with torch.no_grad():
            mine = ddpm_sample(eps_fn, tuple(img.shape), T, src2, cond_scale=cond_scale, dynamic=dynamic, percentile=0.95, clip_value=clip)
        rel = ((mine - img).norm() / img.norm()).item()
        print(f'[ddpm {tag}] {cfg_name} T={T} B={batch} cond_scale={cond_scale} dynamic={dynamic}: draws {src.count}/{src2.count} rel {rel:.3e}')
        assert src.count == src2.count == T + 1 and rel < 1e-4
        o = out['small' if fname == 'ddpm_small' else 'full']
        o[f'img_{tag}'] = img.numpy()
        o[f'case_{tag}'] = np.array([T, batch, cond_scale, float(dynamic), clip, 0.95], dtype=np.float64)
    for k, o in out.items():
        np.savez_compressed(os.path.join(gold_dir, f'ddpm_{k}.npz'), noise_seed=NOISE_SEED, cond_seed=COND_SEED, param_seed=0, **o)


if __name__ == '__main__':
    torch.set_num_threads(os.cpu_count())
    mint(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden'))
