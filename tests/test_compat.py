"""Drop-in boundary (SURVEY §8b row 4): after sparsefusion_b200.compat.install() the reference's own import statements and constructor calls
(demo.py:9, utils/load_model.py:9-10,:58-91, sparsefusion/distillation.py:17-19,:160-165, external/ldm/configs/sd-vae.yaml) resolve to the mirrors,
with the reference's class names, keyword arguments and state_dict layouts.  CPU only: construction and key layouts, no kernels."""
import inspect
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_aliases_resolve_and_construct_with_load_model_kwargs():
    import sparsefusion_b200.compat as compat
    table = compat.install()
    try:
        assert 'sparsefusion.distillation' in table and 'external.imagen_pytorch' in table
        # utils/load_model.py:9-10
        from external.imagen_pytorch import Unet
        from sparsefusion.vldm import DDPM
        # sparsefusion/distillation.py:17-19
        from external.nerf.network_grid import NeRFNetwork
        from external.plms import PLMSSampler
        from external.external_utils import PerceptualLoss
        # demo.py:9
        from sparsefusion.distillation import distillation_loop, get_default_torch_ngp_opt
        from utils.eft_renderer import CustomImplicitRenderer
        import raymarching
        import _raymarching
        import _gridencoder
        assert Unet.__module__ == 'sparsefusion_b200.imagen_pytorch' and DDPM.__module__ == 'sparsefusion_b200.vldm'
        assert all(hasattr(_raymarching, n) for n in ('near_far_from_aabb', 'march_rays_train', 'composite_rays_train_forward', 'packbits', 'morton3D'))
        assert hasattr(_gridencoder, 'grid_encode_forward') and hasattr(_gridencoder, 'grid_encode_backward') and hasattr(raymarching, 'near_far_from_aabb')
        # utils/load_model.py:58-91, a narrow width so that the test stays light (the full width is exercised on the GPU box)
        unet1 = Unet(channels=4, dim=32, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
                     layer_cross_attns=(False, False, False, False), cond_images_channels=256, attn_pool_text=False)
        vldm = DDPM(channels=4, unets=(unet1,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(32,), timesteps=500, cond_drop_prob=0.1,
                    pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False,
                    dynamic_thresholding_percentile=.68, clip_value=10)
        keys = list(vldm.state_dict().keys())
        assert len(keys) == 477 and all(k.startswith('unets.0.') for k in keys)                    # SURVEY §5: 477 tensors under unets.0.*
        vldm.load_state_dict({k: v.clone() for k, v in vldm.state_dict().items()})                # load_model.py:94
        sampler = PLMSSampler(vldm, 50)                                                             # distillation.py:160
        assert list(inspect.signature(sampler.sample).parameters)[:6] == ['image', 'max_thres', 'cond_images', 'cond_scale', 'use_tqdm', 'return_noise']
        opt = get_default_torch_ngp_opt()
        ngp = NeRFNetwork(opt)                                                                      # distillation.py:164
        assert set(ngp.state_dict()) >= {'encoder.embeddings', 'encoder.offsets', 'sigma_net.net.0.weight', 'sigma_net.net.2.bias', 'aabb_train', 'aabb_infer'}
        assert [g['lr'] for g in ngp.get_params(5e-4)] == [5e-3, 5e-4]                              # network_grid.py:223-234
        assert isinstance(PerceptualLoss('vgg', device='cpu'), torch.nn.Module)                     # distillation.py:161
        # the reference's signature, argument for argument (sparsefusion/distillation.py:26-41)
        want = ['gpu', 'args', 'opt', 'model_tuple', 'save_dir', 'seq_name', 'scene_cameras', 'scene_rgb', 'scene_mask', 'scene_valid_region', 'input_idx',
                'use_diffusion', 'max_itr', 'loss_fn_vgg']
        sig = inspect.signature(distillation_loop)
        assert list(sig.parameters)[:len(want)] == want
        assert sig.parameters['use_diffusion'].default is True and sig.parameters['max_itr'].default == 3000 and sig.parameters['loss_fn_vgg'].default is None
        assert all(p.kind is inspect.Parameter.KEYWORD_ONLY for n, p in list(sig.parameters.items())[len(want):])
        # external/ldm/configs/sd-vae.yaml through utils/load_model.py:113-126 (instantiate_from_config -> target(**params))
        from external.ldm.models.autoencoder import AutoencoderKL
        vae = AutoencoderKL(embed_dim=4, monitor='val/rec_loss', lossconfig={'target': 'torch.nn.Identity'},
                            ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                                          attn_resolutions=[], dropout=0.0))
        sd = vae.state_dict()
        assert len(sd) == 248 and 'encoder.down.3.block.1.conv2.weight' in sd and 'post_quant_conv.bias' in sd
        # utils/eft_renderer.py:107-167: (images, ray_bundle, reg) with the reference's call conventions
        calls = []
        r = CustomImplicitRenderer(raysampler=lambda cameras, **kw: calls.append('sample') or 'bundle',
                                   raymarcher=lambda rays_densities, rays_features, ray_bundle, **kw: calls.append('march') or (rays_densities + rays_features))
        images, bundle, reg = r(cameras='cams', volumetric_function=lambda ray_bundle, cameras, **kw: (1.0, 2.0, 7.0), n_batches=16)
        assert (images, bundle, reg) == (3.0, 'bundle', 0) and calls == ['sample', 'march']
        r2 = CustomImplicitRenderer(lambda cameras, **kw: 'b', lambda rays_densities, rays_features, ray_bundle, **kw: 0, reg=True)
        assert r2(cameras=None, volumetric_function=lambda ray_bundle, cameras, **kw: (1, 2, 7.0))[2] == 7.0
        with pytest.raises(ValueError):
            CustomImplicitRenderer(raysampler=None, raymarcher=lambda **k: 0)
    finally:
        compat.uninstall()
    assert 'external.imagen_pytorch' not in sys.modules and 'sparsefusion.vldm' not in sys.modules


def test_aliases_shadow_the_reference_tree_when_it_is_on_the_path(tmp_path):
    """with the reference's tree first on sys.path (how demo.py runs), install() must win over the reference's own modules of the same names.
    The tree here is a stand-in with the reference's package layout whose modules define the same names."""
    ref = tmp_path / 'reference'
    for pkg, mods in {'external': {'imagen_pytorch': 'Unet', 'plms': 'PLMSSampler'}, 'sparsefusion': {'vldm': 'DDPM', 'distillation': 'distillation_loop'}}.items():
        (ref / pkg).mkdir(parents=True)
        (ref / pkg / '__init__.py').write_text('')
        for mod, name in mods.items():
            (ref / pkg / f'{mod}.py').write_text(f'{name} = None\n')
    code = ("import sys; sys.dont_write_bytecode = True; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import sparsefusion_b200.compat as c; c.install()\n"
            "from external.imagen_pytorch import Unet\nfrom external.plms import PLMSSampler\nfrom sparsefusion.vldm import DDPM\n"
            "from sparsefusion.distillation import distillation_loop\nimport external\n"
            "assert Unet.__module__ == 'sparsefusion_b200.imagen_pytorch' and PLMSSampler.__module__ == 'sparsefusion_b200.plms'\n"
            "assert DDPM.__module__ == 'sparsefusion_b200.vldm' and distillation_loop.__module__ == 'sparsefusion_b200.distillation'\n"
            "assert external.__path__ and 'reference' in list(external.__path__)[0]\nprint('ok')\n") % (str(ref), ROOT)
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith('ok'), out.stderr[-2000:]
