"""Host side of distillation with classifier-free guidance: ``cond_scale`` is refused before any device work when the VLDM has no conditional
dropout or the scale is not finite, ``use_diffusion=False`` ignores it, and the entry points keep the reference's positional signature."""
import inspect
from types import SimpleNamespace

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


class _Builder:
    """a scene builder that records every call: a refusal must come before it is asked for anything"""

    def __init__(self):
        self.calls = []

    def build(self, *a, **k):
        self.calls.append('build')
        raise AssertionError('build reached')


def test_guidance_without_conditional_dropout_is_refused_before_device_work(tmp_path):
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, distill_scenes, distillation_loop
    from sparsefusion_b200.plms import PLMSSampler
    ddpm, cfg = _ddpm(cond_drop_prob=0.)
    h = cfg.image_size
    cuda0 = torch.cuda.is_initialized()
    with pytest.raises(ValueError, match='conditional dropout'):
        PLMSSampler(ddpm, 50).sample_rows(torch.zeros(2, 4, h, h), [0.3, 0.6], torch.zeros(2, cfg.cond_images_channels, h, h), cond_scale=3.0)
    with pytest.raises(ValueError, match='conditional dropout'):
        Distiller(None, None, ddpm, None, None, cond_scale=3.0)
    with pytest.raises(ValueError, match='conditional dropout'):
        MultiSceneDistiller([None], None, ddpm, None, [None], seeds=[0], cond_scale=3.0)
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    b = _Builder()
    with pytest.raises(ValueError, match='conditional dropout'):
        distillation_loop(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), 's0', 0, None, None, None, [0], scene_builder=b, cond_scale=3.0)
    with pytest.raises(ValueError, match='conditional dropout'):
        distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), [('s0', 0, None, None, None, [0])], scene_builder=b, cond_scale=3.0)
    assert b.calls == [] and not (tmp_path / 'o').exists() and not (tmp_path / 'exp').exists()
    assert torch.cuda.is_initialized() == cuda0
    # without the diffusion model there is no SDS target to guide: the scale is ignored and the loop gets as far as building the scene
    for call in (lambda: distillation_loop(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), 's0', 0, None, None, None, [0],
                                           use_diffusion=False, scene_builder=b, cond_scale=3.0),
                 lambda: distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), [('s0', 0, None, None, None, [0])],
                                        use_diffusion=False, scene_builder=b, cond_scale=3.0)):
        with pytest.raises(AssertionError, match='build reached'):
            call()
    assert b.calls == ['build', 'build'] and torch.cuda.is_initialized() == cuda0


def test_non_finite_scale_is_refused():
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller
    ddpm, _ = _ddpm()
    cuda0 = torch.cuda.is_initialized()
    for s in (float('nan'), float('inf')):
        with pytest.raises(ValueError, match='finite'):
            Distiller(None, None, ddpm, None, None, cond_scale=s)
        with pytest.raises(ValueError, match='finite'):
            MultiSceneDistiller([None], None, ddpm, None, [None], seeds=[0], cond_scale=s)
    assert torch.cuda.is_initialized() == cuda0


def test_entry_points_keep_the_reference_signature():
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, distill_scenes, distillation_loop
    from sparsefusion_b200.plms import PLMSSampler
    reference = ['gpu', 'args', 'opt', 'model_tuple', 'save_dir', 'seq_name', 'scene_cameras', 'scene_rgb', 'scene_mask', 'scene_valid_region',
                 'input_idx', 'use_diffusion', 'max_itr', 'loss_fn_vgg']          # sparsefusion/distillation.py:26-41, demo.py:87-103
    sig = inspect.signature(distillation_loop)
    positional = [n for n, p in sig.parameters.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == reference
    assert [sig.parameters[n].default for n in reference[-3:]] == [True, 3000, None]
    for fn in (distillation_loop, distill_scenes, Distiller, MultiSceneDistiller):
        p = inspect.signature(fn).parameters['cond_scale']
        assert p.kind == p.KEYWORD_ONLY and p.default == 1.0, fn
    # the baselines' scale stays its own keyword
    assert inspect.signature(distillation_loop).parameters['vldm_cond_scale'].default == 1.0
    assert inspect.signature(PLMSSampler.sample_rows).parameters['cond_scale'].default == 1.0
