"""DDPM.sample host side: the oracle's restatement of the reference's ancestral sampler reproduces the reference's own vectors, the
per-step scalars equal the reference's fp32 schedule terms, and every unsupported argument is refused before any GPU work."""
import math

import numpy as np
import pytest
import torch


def _ddpm(cfg, **kw):
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults),
                cond_images_channels=cfg.cond_images_channels, attn_pool_text=False, attn_dim_head=cfg.attn_dim_head,
                attn_heads=cfg.attn_heads)
    args = dict(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,),
                timesteps=500, cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False,
                clip_output=True, dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10)
    args.update(kw)
    return DDPM(**args)


@pytest.mark.parametrize('tag', ['a', 'b', 'c'])
def test_oracle_ddpm_sample_reproduces_reference(golden_dir, tag):
    from oracle import ddpm_oracle as do, unet_oracle as uo
    g = np.load(f'{golden_dir}/ddpm_small.npz')
    T, batch, cond_scale, dynamic, clip, pct = g[f'case_{tag}']
    cfg = uo.SMALL
    sd = uo.make_params(cfg, seed=int(g['param_seed']))
    cond = do.cond_images(cfg, int(batch), int(g['cond_seed']))
    src = uo.NoiseSource(seed=int(g['noise_seed']))
    with torch.no_grad():
        img = do.ddpm_sample(lambda x, ls, drop: uo.unet_forward(sd, cfg, x, ls, cond * (1. - drop)), tuple(g[f'img_{tag}'].shape), int(T),
                             src, cond_scale=float(cond_scale), dynamic=bool(dynamic), percentile=float(pct), clip_value=float(clip))
    ref = torch.from_numpy(g[f'img_{tag}'])
    assert src.count == int(T) + 1
    assert ((img - ref).norm() / ref.norm()).item() < 1e-4


def test_step_scalars_match_reference_fp32_schedule():
    """plms._step_scalars at the 500 steps of DDPM.sample against the fp32 q_posterior / predict_start_from_noise terms
    (imagen_pytorch.py:240-258), including t = 1.0 (fp32 log-SNR -33.9) and the last step, whose noise is multiplied by 0"""
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import _step_scalars
    T = 500
    lin = torch.linspace(1., 0., T + 1)
    t, tn = lin[:-1], lin[1:]
    ls, lsn = uo.alpha_cosine_log_snr(t), uo.alpha_cosine_log_snr(tn)
    assert abs(ls[0].item() - (-33.9)) < 0.05
    alpha, sigma = uo.log_snr_to_alpha_sigma(ls)
    alpha_n, sigma_n = uo.log_snr_to_alpha_sigma(lsn)
    c = -torch.expm1(ls - lsn)
    ns = (1 - (tn == 0).float()) * (0.5 * torch.log((sigma_n ** 2 * c).clamp(min=1e-20))).exp()
    got = torch.tensor([_step_scalars(a, b) for a, b in zip(lin[:-1].tolist(), lin[1:].tolist())], dtype=torch.float32)
    want = torch.stack((alpha, sigma, alpha_n, c, ns), 1)
    assert torch.allclose(got, want, rtol=4e-6, atol=0)
    assert got[-1, 4].item() == 0.0 and got[:-1, 4].min().item() > 0


def test_sample_refuses_unsupported_arguments_and_cpu():
    from oracle import unet_oracle as uo
    cfg = uo.SMALL
    d = _ddpm(cfg)
    cond = torch.zeros(1, cfg.cond_images_channels, cfg.image_size, cfg.image_size)
    for kw in (dict(conditional_input=torch.zeros(1, 3)), dict(conditional_embeds=torch.zeros(1, 4, 8)), dict(video_frames=4),
               dict(inpaint_images=torch.zeros(1, 4, 16, 16), inpaint_masks=torch.ones(1, 16, 16, dtype=torch.bool)),
               dict(return_pil_images=True)):
        with pytest.raises(NotImplementedError):
            d.sample(cond_images=cond, batch_size=1, **kw)
    with pytest.raises(NotImplementedError, match='pred_objective'):
        _ddpm(cfg, pred_objectives='x_start').sample(cond_images=cond, batch_size=1)
    with pytest.raises(NotImplementedError, match='cosine'):
        _ddpm(cfg, noise_schedules='linear').sample(cond_images=cond, batch_size=1)
    with pytest.raises(ValueError, match='batch_size'):
        d.sample(cond_images=cond, batch_size=2)
    with pytest.raises(RuntimeError, match='GPU'):
        d.sample(cond_images=cond, batch_size=1)
    with pytest.raises(RuntimeError, match='GPU'):
        d.sample(cond_images=cond, batch_size=1, cond_scale=3.)


def test_guidance_needs_conditional_dropout():
    from oracle import unet_oracle as uo
    cfg = uo.SMALL
    cond = torch.zeros(1, cfg.cond_images_channels, cfg.image_size, cfg.image_size)
    with pytest.raises(AssertionError, match='classifier free guidance'):
        _ddpm(cfg, cond_drop_prob=0.).sample(cond_images=cond, batch_size=1, cond_scale=3.)


def test_dynamic_step_validates_arguments():
    from sparsefusion_b200 import _lib
    args = dict(alpha=0.5, sigma=0.5, alpha_next=0.6, c=0.1, noise_scale=0.1)
    with pytest.raises(RuntimeError, match='null pointer'):
        _lib.call('sfb_ddpm_dynamic_step', None, None, None, 1.0, None, *args.values(), 0.95, 4096, 1, None, None, None, None)
    with pytest.raises(RuntimeError, match='row_len'):
        _lib.call('sfb_ddpm_dynamic_step', 8, 8, None, 1.0, 8, *args.values(), 0.95, 65537, 1, 8, None, None, None)
    with pytest.raises(RuntimeError, match='percentile'):
        _lib.call('sfb_ddpm_dynamic_step', 8, 8, None, 1.0, 8, *args.values(), 1.5, 4096, 1, 8, None, None, None)
