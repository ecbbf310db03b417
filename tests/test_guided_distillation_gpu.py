"""Distillation with classifier-free guidance (``cond_scale``) on the GPU: one SDS iteration (itr > start_fusion_step, LPIPS on) of the three
steps, reduced scenes (64x64 rays, 128^2 images, 16^2 latents, small UNet / VAE of the same architecture), every draw injected or keyed.

(1) ``Distiller.step`` with cond_scale 3 against the same iteration restated from its parts: the photometric sub-step, the fusion render,
    VAE encode, guided ``PLMSSampler.sample``, decode, the fusion-loss and LPIPS kernels, Adam;
(2) ``Distiller.minibatch_step`` (3 views in one batch) against the restatement that samples each view alone with its keyed draws;
(3) ``MultiSceneDistiller.step`` (3 scenes at their own noise levels, so guided ``sample_rows`` on per-row schedules) against each scene's own
    guided ``Distiller.step``.
Bar, as tests/test_distillation_gpu.py: losses within 1e-3 relative; every NGP parameter after the step within 1e-3 relative of the
restatement's and within a fifth of how far the step moved it.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SCALE = 3.0
ITR = 1500
MAX_THRES = 0.37


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _models():
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    from sparsefusion_b200.vldm import DDPM
    cfg = uo.SMALL
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval()
    vae.load_state_dict(vo.make_params(seed=0, ch=32, ch_mult=(1, 2, 4, 4)))
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0))
    ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()
    return vae.cuda(), ddpm, PerceptualLoss('vgg', device='cuda', seed=2)


def _cache(k):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.distillation import SceneCache
    from sparsefusion_b200.synthetic import synthetic_scene
    return SceneCache(**synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels, render_hw=64,
                                        seed=3 + k)).to('cuda')


def _ngp(k):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    ngp = NeRFNetwork(get_default_torch_ngp_opt())
    st = ngp.state_dict()
    st.update(no.make_field_params(seed=k))
    ngp.load_state_dict(st)
    return ngp.cuda().train()


def _draws(n_rays, seed):
    rng = np.random.default_rng(seed)
    return {w: (torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda(), torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda())
            for w in 'AB'}


def _distiller(models, k, seed, **kw):
    from sparsefusion_b200.distillation import Distiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    vae, ddpm, pl = models
    return Distiller(_ngp(k), vae, ddpm, get_default_torch_ngp_opt(), _cache(k), seed=seed, percep=pl, **kw)


def _sds_grad(d, itr, img, ws, hw, vi, max_thres, noise_fn, scale=1.0):
    """the SDS term of one view restated: x2 upsampling of the render, VAE encode, guided PLMS on this view alone, decode, then the fusion
    loss kernels with the LPIPS value and gradient, backward of the gradient times ``scale``; returns the loss"""
    from sparsefusion_b200 import image_glue as glue
    from sparsefusion_b200.distillation import normalize, unnormalize
    from sparsefusion_b200.plms import PLMSSampler, _log_snr, _sigmoid
    up = glue.upsample2x_render(img.detach(), ws.detach(), hw, hw)
    with torch.no_grad():
        lat = d.vae.encode(normalize(up[None, :3])).mode() * 0.18215
        sp = PLMSSampler(d.vldm, 50, noise_fn=noise_fn)
        x0 = sp.sample(lat, max_thres=max_thres, cond_images=d.cache.target_features[vi:vi + 1], cond_scale=SCALE, use_tqdm=False)
        pred = unnormalize(d.vae.decode(x0 / 0.18215)).clip(0.0, 1.0)[0]
    pv, pg = d.percep.value_and_grad(up[:3], pred, normalize=True)
    weight = 1.0 - _sigmoid(_log_snr(max_thres))
    loss, g_img, g_ws = glue.fusion_loss(up, pred, hw, hw, 'sds', weight, 1.0, 1.0, 1e-3, g_extra=pg * 0.1)
    torch.autograd.backward((img, ws), (g_img * scale, g_ws * scale))
    return loss + pv * 0.1, sp.last_unet_calls


def _check(label, got_losses, want_losses, got_flat, want_flat, start_flat):
    for a, b in zip(got_losses, want_losses):
        assert abs(a - b) < 1e-3 * abs(b), (label, a, b)
    r, moved = _rel(got_flat, want_flat), _rel(want_flat, start_flat)
    print(f'{label}: losses {got_losses} vs {want_losses}; parameters rel {r:.2e} (the step moved them by {moved:.2e})')
    assert r < 1e-3 and r < 0.2 * moved + 1e-6, (label, r, moved)


def _src_fn(seed):
    from oracle import unet_oracle as uo
    src = uo.NoiseSource(seed=seed)
    return lambda t: src(t.cpu()).to(t.device)


def test_guided_reference_step_matches_restatement():
    from sparsefusion_b200.distillation import shard_target_view
    models = _models()
    draws = _draws(64 * 64, 21)

    d = _distiller(models, 0, 11, cond_scale=SCALE)
    start = d.optimizer.flat.clone()
    d.sampler.noise_fn = _src_fn(5)
    d.render_noise = lambda w: draws[w]
    la, lb = d.step(ITR, max_thres=MAX_THRES)
    calls = d.last['unet_calls']

    r = _distiller(models, 0, 11)                       # unguided: only its photometric sub-step, render and Adam are used
    r.render_noise = lambda w: draws[w]
    ra = r.photometric_substep(ITR)
    c = r.cache
    r.optimizer.zero_grad()
    vi = shard_target_view(torch.randperm(c.target_features.shape[0], generator=r.gen), 0)
    torch.rand(1, generator=r.gen)
    img, ws, hw = r._render(c.target_rays_o[vi], c.target_rays_d[vi], draws['B'])
    rb, r_calls = _sds_grad(r, ITR, img, ws, hw, vi, MAX_THRES, _src_fn(5))
    r.optimizer.step()
    assert calls == r_calls == 38
    _check('Distiller.step', [la.item(), lb.item()], [ra.item(), rb.item()], d.optimizer.flat, r.optimizer.flat, start)

    u = _distiller(models, 0, 11)                       # the same step unguided: the scale must reach the sampler
    u.sampler.noise_fn = _src_fn(5)
    u.render_noise = lambda w: draws[w]
    _, ub = u.step(ITR, max_thres=MAX_THRES)
    print(f'unguided fusion loss {ub.item():.6f} vs guided {lb.item():.6f}')
    assert abs(ub.item() - lb.item()) > 1e-3 * abs(lb.item())


def test_guided_minibatch_step_matches_per_view_restatement():
    from sparsefusion_b200.distillation import KeyedNoise, step_views, view_seed
    models = _models()
    V = 3
    d = _distiller(models, 1, 12, cond_scale=SCALE, views_per_step=V)
    start = d.optimizer.flat.clone()
    la, lb = d.step(ITR, max_thres=MAX_THRES)
    assert d.last['unet_calls'] == 38                  # one batch of V views: 38 evaluations of 2V UNet rows

    r = _distiller(models, 1, 12, views_per_step=V)
    c = r.cache
    idx = int(torch.randperm(c.input_rgb.shape[0], generator=r.gen)[0])
    views = step_views(torch.randperm(c.target_features.shape[0], generator=r.gen), V)
    torch.rand(1, generator=r.gen)
    r.optimizer.zero_grad()
    ra = r._photometric_grad(idx, r._render_draws(c.input_rays_o[idx], ITR, idx, 0, True))
    rb = 0.0
    for v in views:                                     # each view alone, its PLMS draws from its own keyed generator
        img, ws, hw = r._render(c.target_rays_o[v], c.target_rays_d[v], r._render_draws(c.target_rays_o[v], ITR, v, 1, True))
        lv, _ = _sds_grad(r, ITR, img, ws, hw, v, MAX_THRES, KeyedNoise([view_seed(12, ITR, v, 2)], 'cuda'), scale=1.0 / V)
        rb = rb + lv / V
    r.optimizer.step()
    _check('Distiller.minibatch_step', [la.item(), lb.item()], [ra.item(), rb.item()], d.optimizer.flat, r.optimizer.flat, start)


def test_guided_multiscene_step_matches_per_scene_guided_steps():
    from sparsefusion_b200.distillation import MultiSceneDistiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    models = _models()
    vae, ddpm, pl = models
    S = 3
    seeds = [13, 14, 12]                                # noise levels 0.23, 0.06, 0.64: 24, 7 and 51 evaluations, longest last
    draws = [_draws(64 * 64, 30 + k) for k in range(S)]
    ref = []
    for k in range(S):
        d = _distiller(models, k, seeds[k], cond_scale=SCALE)
        d.sampler.noise_fn = _src_fn(50 + k)
        d.render_noise = lambda w, k=k: draws[k][w]
        la, lb = d.step(ITR)                            # scene k's own u: the scenes sample at different noise levels
        ref.append(((la.item(), lb.item()), d.optimizer.flat.clone(), d.last['unet_calls']))
    msd = MultiSceneDistiller([_ngp(k) for k in range(S)], vae, ddpm, get_default_torch_ngp_opt(), [_cache(k) for k in range(S)], seeds=seeds,
                              percep=pl, cond_scale=SCALE)
    start = [s.optimizer.flat.clone() for s in msd.scenes]
    srcs = [_src_fn(50 + k) for k in range(S)]
    msd.render_noise = lambda k, w: draws[k][w]
    msd.plms_noise = lambda k: srcs[k]
    la, lb = msd.step(ITR)
    batches = sorted(key[0][0] for key in msd.sampler._graph._graphs)
    print(f'UNet evaluations per scene {msd.last["unet_calls"]}, graph replays {msd.last["graph_replays"]}, graph batch sizes {batches}')
    assert msd.last['unet_calls'] == [24, 7, 51] and batches == [2, 4, 6]
    assert msd.last['graph_replays'] == max(msd.last['unet_calls'])
    for k in range(S):
        (sa, sb), flat, calls = ref[k]
        assert msd.last['unet_calls'][k] == calls
        _check(f'MultiSceneDistiller scene {k}', [la[k].item(), lb[k].item()], [sa, sb], msd.scenes[k].optimizer.flat, flat, start[k])
