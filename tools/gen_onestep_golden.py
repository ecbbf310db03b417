"""Mint tests/golden/forward_noloss_small.npz: the one-step denoising target by the REFERENCE's own sparsefusion.vldm.DDPM.forward_noloss
(with external.imagen_pytorch.Unet, imported unmodified) on the SMALL UNet of oracle.unet_oracle, on the CPU.  Needs the reference source
tree at oracle/gen_golden.py's REF:

    python tools/gen_onestep_golden.py

The time and noise draws are routed to recorded values at run time (the scheduler's ``sample_random_times_bounded`` and ``torch.randn_like``),
so one row can sit at t >= 0.99, where the fp32 cosine log-SNR is the value the reference conditions on.  The conditional-dropout keep mask
is the reference's own draw from torch's global generator under ``torch.manual_seed(KEEP_SEED)``; the seed is picked so that one row is
dropped, and the recorded mask is checked by re-evaluating the reference UNet with the conditioning multiplied by it.  The latents are
scaled so that the +-clip_value clamp of x0 binds on some elements.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import unet_oracle as uo  # noqa: E402
from oracle.gen_golden import GOLD, REF, _reference_unet  # noqa: E402

TIMES = (0.02, 0.3, 0.6, 0.85, 0.995)
KEEP_SEED = 6          # under this seed the keep draw drops row 2 and keeps the other rows (asserted below)
SCALE = 4.0            # latent magnitude: with clip_value 10 the clamp binds on the rows at high noise levels


def main():
    sys.path.insert(0, REF)
    from sparsefusion.vldm import DDPM
    cfg = uo.SMALL
    sd = uo.make_params(cfg, seed=0)
    unet = _reference_unet(cfg, sd)
    ddpm = DDPM(channels=cfg.channels, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None,
                image_sizes=(cfg.image_size,), timesteps=500, cond_drop_prob=0.1, pred_objectives='noise',
                conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False,
                dynamic_thresholding_percentile=.68, clip_value=10)
    ddpm.unets[0].load_state_dict(sd)
    ddpm.eval()
    b, h = len(TIMES), cfg.image_size
    rng = np.random.default_rng(11)
    images = torch.from_numpy(SCALE * rng.standard_normal((b, cfg.channels, h, h), dtype=np.float32))
    cond = torch.from_numpy(rng.standard_normal((b, cfg.cond_images_channels, h, h), dtype=np.float32))
    times = torch.tensor(TIMES, dtype=torch.float32)
    noise = torch.from_numpy(rng.standard_normal((b, cfg.channels, h, h), dtype=np.float32))

    sched = ddpm.noise_schedulers[0]
    calls = []

    def times_draw(batch_size, min_thres=0.0, max_thres=0.999, *, device):
        calls.append('times')
        assert batch_size == b
        return times.clone()

    def noise_draw(like, **kw):
        calls.append('noise')
        assert tuple(like.shape) == tuple(noise.shape)
        return noise.clone()
    orig = torch.randn_like
    sched.sample_random_times_bounded = times_draw
    torch.randn_like = noise_draw
    try:
        torch.manual_seed(KEEP_SEED)
        pred, pred_x0, x_noisy, noise_out, acp = ddpm.forward_noloss(images, cond_images=cond, return_noise=True)
    finally:
        torch.randn_like = orig
        del sched.sample_random_times_bounded
    assert calls == ['times', 'noise'], calls

    torch.manual_seed(KEEP_SEED)        # the keep mask: the only draw left on the global generator (prob_mask_like, imagen_pytorch.py:185)
    keep = torch.zeros((b,)).float().uniform_(0, 1) < (1 - ddpm.cond_drop_prob)
    assert not keep.all() and keep.any(), keep
    with torch.no_grad():
        again = ddpm.unets[0].forward(x_noisy, sched.get_condition(times), cond_images=cond * keep.view(b, 1, 1, 1).float(), cond_drop_prob=0.)
    assert torch.equal(again, pred), 'the recorded keep mask does not reproduce the reference evaluation'
    clipped = int((pred_x0.abs() == ddpm.clip_value).sum())
    assert clipped > 0
    print(f'[forward_noloss] rows {b} keep {keep.tolist()} alpha_cumprod {acp.tolist()} clamped elements {clipped} |pred| {pred.norm():.4f}')
    np.savez_compressed(os.path.join(GOLD, 'forward_noloss_small.npz'), images=images.numpy(), cond=cond.numpy(), times=times.numpy(),
                        noise=noise_out.numpy(), keep=keep.numpy(), pred=pred.numpy(), pred_x0=pred_x0.numpy(), x_noisy=x_noisy.numpy(),
                        alpha_cumprod=acp.numpy(), clip_value=np.float32(ddpm.clip_value))


if __name__ == '__main__':
    main()
