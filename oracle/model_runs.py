"""oracle/model_runs.py -- the model evaluations whose kernel launches the per-element GPU tests record and replay.

TEST INFRASTRUCTURE ONLY.  ``record_models(rec)`` runs, on seeded weights: the FULL UNet at 32^2 latents with batch 1, 2 and 8, precompute_time
with 51 rows, precompute_cond + forward(cond_features=...); the SMALL UNet at 128^2; the full VAE encode + decode at 256^2;
PerceptualLoss.value_and_grad at 256^2; the EFT (encode at 256^2, a feature_cache of three views).  ``rec(family)`` is entered around each
family ('UNet', 'VAE', 'LPIPS', 'EFT'), so the GEMM catalogue (tests/test_conv_fp64_gpu.py) and the SIMT catalogue
(tests/test_simt_fp64_gpu.py) record the same evaluations.
"""
import dataclasses

import numpy as np
import torch


def _unet(cfg):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults), cond_images_channels=cfg.cond_images_channels,
                attn_pool_text=False, attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0), strict=True)
    return unet.cuda()


def record_models(rec):
    from oracle import eft_oracle as eo, unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200 import cameras as C
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    g = torch.Generator(device='cuda').manual_seed(0)
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
    with torch.no_grad():
        unet = _unet(uo.FULL)
        for nb in (1, 2, 8):
            with rec('UNet'):
                unet.forward(rn(nb, 4, 32, 32), uo.alpha_cosine_log_snr(torch.full((nb,), 0.37)).cuda(), cond_images=rn(nb, 256, 32, 32))
        with rec('UNet'):
            unet.precompute_time(uo.alpha_cosine_log_snr(torch.linspace(0.02, 0.98, 51)).cuda())
            feat = unet.precompute_cond(rn(1, 256, 32, 32))
            unet.forward(rn(1, 4, 32, 32), uo.alpha_cosine_log_snr(torch.tensor([0.5])).cuda(), cond_features=feat)
        del unet
        unet = _unet(dataclasses.replace(uo.SMALL, image_size=128))
        with rec('UNet'):
            unet.forward(rn(1, 4, 128, 128), uo.alpha_cosine_log_snr(torch.tensor([0.37])).cuda(), cond_images=rn(1, 12, 128, 128))
        del unet
        vae = AutoencoderKL().eval()
        vae.load_state_dict(vo.make_params(seed=0))
        vae = vae.cuda()
        with rec('VAE'):
            vae.encode(torch.rand(1, 3, 256, 256, device='cuda', generator=g) * 2 - 1)
            vae.decode(rn(1, 4, 32, 32))
        del vae
        with rec('LPIPS'):
            PerceptualLoss('vgg', device='cuda', seed=2).value_and_grad(torch.rand(3, 256, 256, device='cuda', generator=g),
                                                                         torch.rand(3, 256, 256, device='cuda', generator=g))
        m = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=True)
        m.load_state_dict(eo.make_params({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0), strict=True)
        m = m.cuda()
        images = torch.rand(2, 3, 256, 256, device='cuda', generator=g)
        # three query views of a ring of 8 cameras, each with its own two input cameras (NativeSceneBuilder's layout)
        c = eo.look_at_cameras(8, radius=4.0)
        rng = np.random.default_rng(0)
        cams = C.PerspectiveCameras(c.R, c.T, torch.from_numpy(rng.uniform(2.6, 3.4, (8, 2)).astype(np.float32)),
                                    torch.from_numpy(rng.uniform(-0.05, 0.05, (8, 2)).astype(np.float32)), torch.full((8, 2), 256.0))
        rel = C.relative_cameras(cams, [0], True)
        views = [1, 4, 6]
        per_view = [C.relative_cameras(rel, [v], True) for v in views]
        q_o, q_d = C.grid_rays(C.concat_cameras([pv[v] for v, pv in zip(views, per_view)]), 32, 32, 'cuda', 256, 256)
        cdm = float(cams.get_camera_center().norm(dim=1).mean())
        lengths = torch.linspace(cdm - 5.0, cdm + 5.0, 20, device='cuda').expand(len(views), 1024, 20)
        with rec('EFT'):
            m.encode(None, images)
            m.feature_cache(q_o, q_d, lengths, [pv[[0, 3]] for pv in per_view], images, (32, 32))
        del m
    torch.cuda.empty_cache()
