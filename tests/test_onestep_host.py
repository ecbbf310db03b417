"""Host side of the one-step SDS target: ``DDPM.forward_noloss`` and ``sds_method`` refuse what they do not provide before any device work,
keep the reference's signature, and ``sds_method`` reaches the steps from ``distillation_loop`` / ``distill_scenes``."""
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


def test_forward_noloss_refusals_come_before_device_work():
    ddpm, cfg = _ddpm()
    h, cc = cfg.image_size, cfg.cond_images_channels
    x, cond = torch.zeros(2, 4, h, h), torch.zeros(2, cc, h, h)
    cuda0 = torch.cuda.is_initialized()
    with pytest.raises(NotImplementedError, match='onestep'):
        ddpm.forward_noloss(x, cond_images=cond, method='multistep')
    with pytest.raises(NotImplementedError, match='conditioning'):
        ddpm.forward_noloss(x, cond_images=cond, conditional_embeds=torch.zeros(2, 4, 8))
    with pytest.raises(NotImplementedError, match='conditioning'):
        ddpm.forward_noloss(x, cond_images=cond, conditional_input=torch.zeros(2, 3, 8, 8))
    with pytest.raises(NotImplementedError, match='resizing'):
        ddpm.forward_noloss(torch.zeros(2, 4, 2 * h, 2 * h), cond_images=cond)
    with pytest.raises(ValueError, match='min_thres'):
        ddpm.forward_noloss(x, cond_images=cond, min_thres=0.6, max_thres=0.5)
    with pytest.raises(ValueError, match='finite'):
        ddpm.forward_noloss(x, cond_images=cond, cond_scale=float('nan'))
    with pytest.raises(ValueError, match='keep'):
        ddpm.forward_noloss(x, cond_images=cond, keep=torch.ones(2, dtype=torch.bool), cond_scale=3.0)
    with pytest.raises(ValueError, match='times'):
        ddpm.forward_noloss(x, cond_images=cond, times=torch.zeros(3))
    with pytest.raises(ValueError, match='noise'):
        ddpm.forward_noloss(x, cond_images=cond, noise=torch.zeros(2, 4, h, h + 1))
    with pytest.raises(RuntimeError, match='GPU only'):          # a DDPM and tensors on the CPU: no CPU fallback
        ddpm.forward_noloss(x, cond_images=cond)
    plain, _ = _ddpm(cond_drop_prob=0.)
    with pytest.raises(ValueError, match='conditional dropout'):
        plain.forward_noloss(x, cond_images=cond, cond_scale=3.0)
    assert torch.cuda.is_initialized() == cuda0


class _Builder:
    def __init__(self):
        self.calls = []

    def build(self, *a, **k):
        self.calls.append('build')
        raise AssertionError('build reached')


def test_unknown_sds_method_is_refused_before_device_work(tmp_path):
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, distill_scenes, distillation_loop
    ddpm, _ = _ddpm()
    cuda0 = torch.cuda.is_initialized()
    with pytest.raises(ValueError, match='sds_method'):
        Distiller(None, None, ddpm, None, None, sds_method='ddim')
    with pytest.raises(ValueError, match='sds_method'):
        MultiSceneDistiller([None], None, ddpm, None, [None], seeds=[0], sds_method='one-step')
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    b = _Builder()
    for use_diffusion in (True, False):
        with pytest.raises(ValueError, match='sds_method'):
            distillation_loop(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), 's0', 0, None, None, None, [0], use_diffusion=use_diffusion,
                              scene_builder=b, sds_method='PLMS')
        with pytest.raises(ValueError, match='sds_method'):
            distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), [('s0', 0, None, None, None, [0])], use_diffusion=use_diffusion,
                           scene_builder=b, sds_method=None)
    assert b.calls == [] and not (tmp_path / 'o').exists() and not (tmp_path / 'exp').exists()
    assert torch.cuda.is_initialized() == cuda0


def test_signatures_keep_the_reference_and_add_keywords_only():
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, distill_scenes, distillation_loop
    from sparsefusion_b200.vldm import DDPM
    # sparsefusion/vldm.py:632-647
    reference = [('images', inspect.Parameter.empty), ('unet', None), ('conditional_input', None), ('conditional_embeds', None),
                 ('conditional_masks', None), ('unet_number', None), ('cond_images', None), ('loss_mask', None), ('return_noise', False),
                 ('min_thres', 0.0), ('max_thres', 0.999), ('method', 'onestep')]
    sig = inspect.signature(DDPM.forward_noloss)
    positional = [(n, p.default) for n, p in sig.parameters.items() if p.kind == p.POSITIONAL_OR_KEYWORD and n != 'self']
    assert positional == reference
    extra = {n: p.default for n, p in sig.parameters.items() if p.kind == p.KEYWORD_ONLY}
    assert extra == dict(times=None, noise=None, keep=None, cond_scale=1.0)
    # sparsefusion/distillation.py:26-41, demo.py:87-103: the loop's positional signature is unchanged
    loop = ['gpu', 'args', 'opt', 'model_tuple', 'save_dir', 'seq_name', 'scene_cameras', 'scene_rgb', 'scene_mask', 'scene_valid_region',
            'input_idx', 'use_diffusion', 'max_itr', 'loss_fn_vgg']
    sig = inspect.signature(distillation_loop)
    assert [n for n, p in sig.parameters.items() if p.kind == p.POSITIONAL_OR_KEYWORD] == loop
    for fn in (distillation_loop, distill_scenes, Distiller, MultiSceneDistiller):
        p = inspect.signature(fn).parameters['sds_method']
        assert p.kind == p.KEYWORD_ONLY and p.default == 'plms', fn


def test_sds_method_is_threaded_to_the_steps(monkeypatch, tmp_path):
    import sparsefusion_b200.distillation as D
    ddpm, _ = _ddpm()
    seen = []

    class Recorder:
        def __init__(self, *a, **k):
            seen.append((type(self).__name__, k.get('sds_method'), k.get('cond_scale')))
    monkeypatch.setattr(D, 'Distiller', type('Distiller', (Recorder,), {}))
    monkeypatch.setattr(D, 'MultiSceneDistiller', type('MultiSceneDistiller', (Recorder,), {}))
    monkeypatch.setattr(D, '_run_distillation', lambda gpu, args, opt, eft, save_dir, scenes, make, *a, **k:
                        [make([None] * len(scenes), [None] * len(scenes), None, 0)])
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    for method in ('plms', 'onestep'):
        D.distillation_loop(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), 's0', 0, None, None, None, [0], sds_method=method, cond_scale=2.0)
        D.distill_scenes(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), [('s0', 0, None, None, None, [0])], sds_method=method)
    D.distillation_loop(0, args, None, ('eft', None, ddpm), str(tmp_path / 'o'), 's0', 0, None, None, None, [0])
    assert seen == [('Distiller', 'plms', 2.0), ('MultiSceneDistiller', 'plms', 1.0), ('Distiller', 'onestep', 2.0),
                    ('MultiSceneDistiller', 'onestep', 1.0), ('Distiller', 'plms', 1.0)]
