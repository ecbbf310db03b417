"""oracle/model_runs.py -- the model evaluations whose kernel launches the per-element GPU tests record and replay.

TEST INFRASTRUCTURE ONLY.  ``record_models(rec)`` runs, on seeded weights: the FULL UNet at 32^2 latents with batch 1, 2 and 8, precompute_time
with 51 rows, precompute_cond + forward(cond_features=...); the SMALL UNet at 128^2; the full VAE encode + decode at 256^2;
PerceptualLoss.value_and_grad at 256^2; the EFT (``record_eft``: encode at 256^2, a feature_cache of three views).  ``rec(family)`` is
entered around each family ('UNet', 'VAE', 'LPIPS', 'EFT'), so the GEMM catalogue (tests/test_conv_fp64_gpu.py) and the SIMT catalogue
(tests/test_simt_fp64_gpu.py) record the same evaluations.

``record_steps(rec)`` runs what tests/test_step_fp64_gpu.py replays, on the SMALL UNet: DDPM.sample for three steps at 32^2 latents
(row_len 4096), static and dynamic thresholding, guided and unguided, and one dynamic run at 128^2 latents (row_len 65 536: an 8-CTA
cluster per row) under rec('DDPM'); PLMSSampler scene-batched over two schedules (sample_rows) and guided (sample, cond_scale 3) under
rec('PLMS'); and Distiller steps in the configuration of tests/test_distillation_gpu.py -- iteration 5 (photometric + EFT bootstrap) and
iteration 1500 (SDS with the perceptual term, whose gradient joins the fusion loss) -- under rec('Distill').
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
    from oracle import unet_oracle as uo, vae_oracle as vo
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
    record_eft(rec, g)


def record_eft(rec, g=None, warmup=None):
    """``warmup(m)``, when given, is called after one evaluation of the same model on the same inputs outside ``rec`` (prepared plans,
    allocator), right before the recorded one"""
    from oracle import eft_oracle as eo
    from sparsefusion_b200 import cameras as C
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    if g is None:
        g = torch.Generator(device='cuda').manual_seed(0)
    with torch.no_grad():
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
        inputs = [pv[[0, 3]] for pv in per_view]
        if warmup is not None:
            m.encode(None, images)
            m.feature_cache(q_o, q_d, lengths, inputs, images, (32, 32))
            warmup(m)
        with rec('EFT'):
            m.encode(None, images)
            m.feature_cache(q_o, q_d, lengths, inputs, images, (32, 32))
        del m
    torch.cuda.empty_cache()


def record_steps(rec):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.vldm import DDPM
    g = torch.Generator(device='cuda').manual_seed(3)
    for size, runs in ((32, ((False, 1.0), (False, 3.0), (True, 1.0), (True, 3.0))), (128, ((True, 1.0),))):
        cfg = dataclasses.replace(uo.SMALL, image_size=size)
        for dynamic, cond_scale in runs:
            d = DDPM(channels=4, unets=(_unet(cfg),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(size,), timesteps=3,
                     cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                     dynamic_thresholding=dynamic, dynamic_thresholding_percentile=0.95, clip_value=1.).cuda()
            with rec('DDPM'), torch.no_grad():
                d.sample(cond_images=torch.randn(2, cfg.cond_images_channels, size, size, device='cuda', generator=g), batch_size=2,
                         cond_scale=cond_scale, use_tqdm=False)
            del d
    torch.cuda.empty_cache()
    _record_plms(rec, g)
    _record_distill(rec)


def _ddpm500(cfg):
    from sparsefusion_b200.vldm import DDPM
    return DDPM(channels=4, unets=(_unet(cfg),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()


def _record_plms(rec, g):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import PLMSSampler
    cfg = uo.SMALL
    ddpm = _ddpm500(cfg)
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
    h = cfg.image_size
    with rec('PLMS'), torch.no_grad():
        PLMSSampler(ddpm, 50).sample_rows(rn(2, 4, h, h), [0.13, 0.37], rn(2, cfg.cond_images_channels, h, h))
        PLMSSampler(ddpm, 50).sample(rn(2, 4, h, h), max_thres=0.13, cond_images=rn(2, cfg.cond_images_channels, h, h), cond_scale=3.0,
                                     use_tqdm=False)
    del ddpm
    torch.cuda.empty_cache()


def _record_distill(rec):
    from oracle import distill_oracle as do, ngp_oracle as no, unet_oracle as uo
    from sparsefusion_b200.distillation import Distiller, SceneCache
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    cfg = uo.SMALL                                              # 16x16 latents <-> 128x128 images <-> 64x64 rays
    scene = do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=cfg.cond_images_channels, render_hw=64, seed=3)
    torch.manual_seed(0)
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval().cuda()
    opt = get_default_torch_ngp_opt()
    ngp = NeRFNetwork(opt)
    st = ngp.state_dict()
    st.update(no.make_field_params(seed=0))
    ngp.load_state_dict(st)
    dist = Distiller(ngp.cuda().train(), vae, _ddpm500(cfg), opt, SceneCache(**scene).to('cuda'), seed=11, fused_glue=True,
                     percep=PerceptualLoss('vgg', device='cuda', seed=2))
    with rec('Distill'):
        dist.step(5)
        dist.step(1500, max_thres=0.13)
    del dist
    torch.cuda.empty_cache()
