"""Host side of guided PLMS sampling and the EFT / VLDM baselines: guidance without conditional dropout is refused, every argument is checked
before any device work, and the baselines' metrics files have the scene metrics' format."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _ddpm(**kw):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    cfg = uo.SMALL
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults),
                cond_images_channels=cfg.cond_images_channels, attn_pool_text=False, attn_dim_head=cfg.attn_dim_head,
                attn_heads=cfg.attn_heads)
    args = dict(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,),
                timesteps=500, cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False,
                clip_output=True, dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10)
    args.update(kw)
    return DDPM(**args), cfg


def _feats(cfg, n=2):
    return torch.zeros(n, cfg.cond_images_channels, cfg.image_size, cfg.image_size)


class _Builder:
    """a scene builder that records every call: the refusals below must come before it is asked for anything"""

    def __init__(self):
        self.calls = []

    def build(self, *a, **k):
        self.calls.append('build')
        raise AssertionError('build reached')

    def eval_views(self, *a, **k):
        self.calls.append('eval_views')
        raise AssertionError('eval_views reached')


class _BuilderWithoutEval:
    def build(self, *a, **k):
        raise AssertionError('build reached')


def test_guidance_without_conditional_dropout_is_refused(tmp_path):
    from sparsefusion_b200.baselines import sample_vldm_views, score_baselines
    from sparsefusion_b200.distillation import distill_scenes, distillation_loop
    from sparsefusion_b200.plms import PLMSSampler
    ddpm, cfg = _ddpm(cond_drop_prob=0.)
    with pytest.raises(ValueError, match='conditional dropout'):
        PLMSSampler(ddpm, 50).sample(cond_images=_feats(cfg), cond_scale=3.0, use_tqdm=False)
    with pytest.raises(ValueError, match='conditional dropout'):
        sample_vldm_views(ddpm, None, _feats(cfg), seed=0, cond_scale=3.0)
    models = ('eft', None, ddpm)
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    scenes = [('s0', 0, None, None, None, [0])]
    b = _Builder()
    with pytest.raises(ValueError, match='conditional dropout'):
        distill_scenes(0, args, None, models, str(tmp_path / 'o'), scenes, scene_builder=b, evaluate_baselines=True, vldm_cond_scale=3.0)
    with pytest.raises(ValueError, match='conditional dropout'):
        distillation_loop(0, args, None, models, str(tmp_path / 'o'), 's0', 0, None, None, None, [0], scene_builder=b, evaluate_baselines=True,
                          vldm_cond_scale=3.0)
    with pytest.raises(ValueError, match='conditional dropout'):
        score_baselines(0, args, models, str(tmp_path / 'o'), scenes, scene_builder=b, cond_scale=3.0)
    assert b.calls == [] and not (tmp_path / 'o').exists() and not (tmp_path / 'exp').exists()
    # cond_scale 1 needs no dropout, and with dropout guidance is allowed: both get as far as the device (none here, or not yet touched)
    PLMSSampler(ddpm, 50)        # constructing a sampler does no device work


def test_arguments_are_checked_before_device_work(tmp_path):
    from sparsefusion_b200.baselines import check_baseline_cache, sample_vldm_views
    from sparsefusion_b200.distillation import SceneCache, distill_scenes
    from sparsefusion_b200.evaluate import EvalViews
    ddpm, cfg = _ddpm()
    f = _feats(cfg)
    for kw, msg in ((dict(max_batch=0), 'max_batch'), (dict(max_batch=2.5), 'max_batch'), (dict(plms_steps=0), 'plms_steps'),
                    (dict(cond_scale=float('nan')), 'finite')):
        with pytest.raises(ValueError, match=msg):
            sample_vldm_views(ddpm, None, f, seed=0, **kw)
    with pytest.raises(ValueError, match='features'):
        sample_vldm_views(ddpm, None, f[0], seed=0)
    with pytest.raises(RuntimeError, match='CUDA'):            # valid arguments, CPU features: no CPU path
        sample_vldm_views(ddpm, None, f, seed=0, cond_scale=3.0)
    assert not torch.cuda.is_initialized()
    # the cache's first V entries stand for the V scene views: enough of them, at the ground truth's size
    views = EvalViews(rays_o=torch.zeros(3, 4, 3), rays_d=torch.zeros(3, 4, 3), rgb=torch.zeros(3, 3, 64, 64), mask=torch.zeros(3, 1, 64, 64))

    def cache(n, hw):
        return SceneCache(input_rgb=None, input_mask=None, input_rays_o=None, input_rays_d=None, target_features=torch.zeros(n, 12, 8, 8),
                          target_eft_image=torch.zeros(n, 3, hw, hw), target_rays_o=None, target_rays_d=None)
    check_baseline_cache(cache(5, 64), views)
    with pytest.raises(ValueError, match='3 views'):
        check_baseline_cache(cache(2, 64), views)
    with pytest.raises(ValueError, match='EFT images'):
        check_baseline_cache(cache(5, 32), views)
    # the distillation entries: the baselines need the feature cache (use_diffusion) and the builder's eval_views, checked before any work
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    scenes = [('s0', 0, None, None, None, [0])]
    with pytest.raises(ValueError, match='use_diffusion'):
        distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), scenes, use_diffusion=False, scene_builder=_Builder(),
                       evaluate_baselines=True)
    with pytest.raises(TypeError, match='evaluate_baselines=True needs the scene builder to provide eval_views'):
        distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), scenes, scene_builder=_BuilderWithoutEval(), evaluate_baselines=True)
    assert not (tmp_path / 'o').exists() and not torch.cuda.is_initialized()


def test_baseline_metrics_files_have_the_scene_metrics_format(tmp_path):
    from sparsefusion_b200.evaluate import SceneEval, write_scene_metrics
    se = SceneEval(psnr=torch.tensor([20.0, 22.5], dtype=torch.float64), ssim=torch.tensor([0.5, 0.75], dtype=torch.float64),
                   lpips=torch.tensor([0.25, 0.5], dtype=torch.float64), image=torch.zeros(2, 8, 8, 3), silhouette=None)
    path = tmp_path / 'metrics' / 'hydrant_000_vldm.txt'
    write_scene_metrics(str(path), se)
    want = ('warning: this metric is used for debugging only and not the final metric'
            f'psnr:\n{np.float64(21.25)}\nssim:\n{np.float32(0.625)}\npip:\n{np.float64(0.375)}\n')
    assert path.read_text() == want
