"""Scene-batched distillation on the GPU: the per-row PLMS update kernel, PLMSSampler.sample_rows, MultiSceneDistiller and distill_scenes.

(1) sfb_plms_update_rows is bit-identical to one sfb_plms_update launch per row;
(2) sample_rows with six different noise levels in one call equals six single-scene sample() runs fed the same per-scene noise;
(3) MultiSceneDistiller.step equals one Distiller.step per scene with the same injected draws (reduced scenes, both phases, LPIPS in the SDS one),
    and without injected draws equals Distiller.step fed each scene's (seed, iteration, view)-keyed draws;
(4) the same at full size (FULL UNet, full VAE, LPIPS, 128^2 rays), 4 scenes, one SDS step;
(5) distill_scenes writes every scene's checkpoint in the reference layout.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_THRES = [0.004, 0.013, 0.13, 0.37, 0.62, 0.99]


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _ddpm(cfg, seed=0):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=seed))
    return DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()


def _scalars(g):
    a = 0.2 + 0.8 * torch.rand(1, generator=g).item()
    return (a, (1 - a * a) ** 0.5, min(1.0, a + 0.05), 0.3 * torch.rand(1, generator=g).item(), 0.2 * torch.rand(1, generator=g).item())


@pytest.mark.parametrize('rows', [1, 3, 8])
@pytest.mark.parametrize('row_len', [1024, 4096, 65536])
def test_plms_update_rows_is_bit_identical_to_per_row_launches(rows, row_len):
    from sparsefusion_b200 import _lib as lib
    g = torch.Generator().manual_seed(rows * 100003 + row_len)
    x, z = (torch.randn(rows, row_len, generator=g).cuda() * 3 for _ in range(2))
    eps = [torch.randn(rows, row_len, generator=g).cuda() for _ in range(4)]
    tab = [_scalars(g) for _ in range(rows)]
    tab = [t[:4] + (0.0,) if r % 2 else t for r, t in enumerate(tab)]            # odd rows end their run: noise_scale = 0
    tab_d = torch.tensor(tab, dtype=torch.float32).cuda()
    coefs = {1: [1.0], 2: [1.5, -0.5], 3: [23 / 12, -16 / 12, 5 / 12], 4: [55 / 24, -59 / 24, 37 / 24, -9 / 24]}
    for k in (1, 2, 3, 4):
        ptrs = [lib.fptr(e) for e in eps[:k]] + [None] * (4 - k)
        cf = coefs[k] + [0.0] * (4 - k)
        got, got_x0 = torch.empty_like(x), torch.empty_like(x)
        lib.call('sfb_plms_update_rows', lib.fptr(x), *ptrs, *cf, lib.fptr(z), lib.fptr(tab_d), 10.0, lib.fptr(got), lib.fptr(got_x0), rows, row_len,
                 lib.stream())
        want, want_x0 = torch.empty_like(x), torch.empty_like(x)
        for r in range(rows):
            rp = [lib.fptr(e[r]) for e in eps[:k]] + [None] * (4 - k)
            lib.call('sfb_plms_update', lib.fptr(x[r]), *rp, *cf, lib.fptr(z[r]), *tab[r], 10.0, lib.fptr(want[r]), lib.fptr(want_x0[r]), None,
                     row_len, lib.stream())
        assert torch.equal(got, want) and torch.equal(got_x0, want_x0), (rows, row_len, k)


def test_sample_rows_matches_single_scene_runs():
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import PLMSSampler
    cfg = uo.SMALL
    ddpm = _ddpm(cfg)
    S = len(MAX_THRES)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(S, 4, cfg.image_size, cfg.image_size, generator=g).cuda()
    cond = torch.randn(S, cfg.cond_images_channels, cfg.image_size, cfg.image_size, generator=g).cuda()
    single = []
    for k, m in enumerate(MAX_THRES):
        src = uo.NoiseSource(seed=70 + k)
        sp = PLMSSampler(ddpm, 50, noise_fn=lambda t, src=src: src(t.cpu()).to(t.device))
        out = sp.sample(lat[k:k + 1], max_thres=m, cond_images=cond[k:k + 1], use_tqdm=False, return_noise=True)
        single.append((out, sp.last_unet_calls, src.count))
    srcs = [uo.NoiseSource(seed=70 + k) for k in range(S)]

    def noise_fn(like, rows=None):
        rows = range(S) if rows is None else rows
        return torch.cat([srcs[r](like[i:i + 1].cpu()).to(like.device) for i, r in enumerate(rows)])
    sampler = PLMSSampler(ddpm, 50)
    outs = sampler.sample_rows(lat, MAX_THRES, cond, noise_fn=noise_fn)
    print(f'sample_rows: rows {sampler.last_row_calls}, batched evaluations {sampler.last_unet_calls}, graph replays {sampler.last_graph_replays}')
    assert sampler.last_row_calls == [s[1] for s in single] == [0, 2, 14, 38, 51, 51]
    assert sampler.last_graph_replays == sampler.last_unet_calls == 51
    assert [s.count for s in srcs] == [s[2] for s in single]                      # every row drew what its single run drew
    for k in range(S):
        for name, a, b in zip(('pred_x0', 'x_noisy', 'noise', 'alpha_cumprod'), outs, single[k][0]):
            r = _rel(a[k:k + 1], b)
            print(f'  row {k} (max_thres {MAX_THRES[k]}): {name} rel {r:.2e}')
            assert r < 1e-5, (k, name, r)


# ------------------------------------------------------------------------------------------------ MultiSceneDistiller vs Distiller
def _small_models(percep):
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval()
    vae.load_state_dict(vo.make_params(seed=0, ch=32, ch_mult=(1, 2, 4, 4)))
    pl = None
    if percep:
        from sparsefusion_b200.lpips_vgg import PerceptualLoss
        pl = PerceptualLoss('vgg', device='cuda', seed=2)
    return vae.cuda(), _ddpm(uo.SMALL), pl


def _full_models():
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    vae = AutoencoderKL().eval()
    vae.load_state_dict(vo.make_params(seed=0))
    return vae.cuda(), _ddpm(uo.FULL), PerceptualLoss('vgg', device='cuda', seed=2)


def _ngp(k):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    ngp = NeRFNetwork(get_default_torch_ngp_opt())
    st = ngp.state_dict()
    st.update(no.make_field_params(seed=k))
    ngp.load_state_dict(st)
    return ngp.cuda().train()


def _scenes(S, full):
    from oracle import distill_oracle as do, unet_oracle as uo
    from sparsefusion_b200.distillation import SceneCache
    if full:
        return [SceneCache(**do.synthetic_scene(n_input=2, n_target=6, seed=3 + k)).to('cuda') for k in range(S)]
    return [SceneCache(**do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels, render_hw=64,
                                            seed=3 + k)).to('cuda') for k in range(S)]


def _draws(S, n_rays):
    rng = np.random.default_rng(21)
    return [{w: (torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda(), torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda())
             for w in 'AB'} for _ in range(S)]


def _keyed_replay(d, itr):
    """route the draws MultiSceneDistiller keys by view_seed -- photometric (view 0, stream 0), fusion (vi, 1), PLMS (vi, 2) -- through the
    reference step's hooks of Distiller d"""
    from sparsefusion_b200.distillation import KeyedNoise, shard_target_view, view_seed
    g = torch.Generator().manual_seed(d.seed)                   # d.gen's draws of this step, replayed: randperm(n_in), randperm(n_t)
    torch.randperm(d.cache.input_rgb.shape[0], generator=g)
    vi = shard_target_view(torch.randperm(d.cache.target_features.shape[0], generator=g), 0)
    n = d.cache.input_rays_o.shape[1]

    def pair(view, stream):
        gg = torch.Generator(device='cuda')
        gg.manual_seed(view_seed(d.seed, itr, view, stream))
        return (torch.rand(n, d.opt.num_steps, generator=gg, device='cuda'), torch.rand(n, d.opt.upsample_steps, generator=gg, device='cuda'))
    d.render_noise = lambda w: pair(0, 0) if w == 'A' else pair(vi, 1)
    d.sampler.noise_fn = KeyedNoise([view_seed(d.seed, itr, vi, 2)], 'cuda')


def _single_step(models, cache, k, itr, draws, seed):
    """Distiller.step of scene k with the injected draws (None: MultiSceneDistiller's keyed ones); returns (losses, flat parameters)"""
    from oracle import unet_oracle as uo
    from sparsefusion_b200.distillation import Distiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    vae, ddpm, pl = models
    d = Distiller(_ngp(k), vae, ddpm, get_default_torch_ngp_opt(), cache, seed=seed, percep=pl)
    if draws is None:
        _keyed_replay(d, itr)
    else:
        src = uo.NoiseSource(seed=50 + k)
        d.sampler.noise_fn = lambda t: src(t.cpu()).to(t.device)
        d.render_noise = lambda w: draws[w]
    la, lb = d.step(itr)
    return (la.item(), lb.item()), d.optimizer.flat.clone(), d.last.get('unet_calls')


def _compare(S, itr, full, injected=True):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.distillation import MultiSceneDistiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    models = _full_models() if full else _small_models(percep=itr > 1000)
    caches = _scenes(S, full)
    draws = _draws(S, caches[0].input_rays_o.shape[1]) if injected else [None] * S
    seeds = [11 + k for k in range(S)]
    # run-to-run spread of Distiller.step itself: the field backward accumulates with atomics
    ref = [_single_step(models, caches[k], k, itr, draws[k], seeds[k]) for k in range(S)]
    again = _single_step(models, caches[0], 0, itr, draws[0], seeds[0])
    spread_p = _rel(again[1], ref[0][1])
    spread_l = max(abs(a - b) / abs(b) for a, b in zip(again[0], ref[0][0]))
    vae, ddpm, pl = models
    msd = MultiSceneDistiller([_ngp(k) for k in range(S)], vae, ddpm, get_default_torch_ngp_opt(), caches, seeds=seeds, percep=pl)
    if injected:
        srcs = [uo.NoiseSource(seed=50 + k) for k in range(S)]
        msd.render_noise = lambda k, w: draws[k][w]
        msd.plms_noise = lambda k: (lambda t: srcs[k](t.cpu()).to(t.device))
    la, lb = msd.step(itr)
    print(f'itr {itr}, {S} scenes: Distiller.step run-to-run spread: parameters {spread_p:.2e}, losses {spread_l:.2e}; '
          f'UNet evaluations per scene {msd.last.get("unet_calls")}, graph replays {msd.last.get("graph_replays")}')
    for k in range(S):
        (sa, sb), flat, calls = ref[k]
        rp = _rel(msd.scenes[k].optimizer.flat, flat)
        ra, rb = abs(la[k].item() - sa) / abs(sa), abs(lb[k].item() - sb) / abs(sb)
        print(f'  scene {k}: losses {la[k].item():.6f}/{sa:.6f} {lb[k].item():.6f}/{sb:.6f} (rel {ra:.1e}, {rb:.1e}); parameters rel {rp:.2e}')
        assert ra < 1e-5 and rb < 1e-5, (k, ra, rb)
        assert rp < 1e-4, (k, rp)
        if itr > 1000:
            assert msd.last['unet_calls'][k] == calls


@pytest.mark.parametrize('itr', [5, 1500])
def test_multiscene_step_matches_per_scene_distillers(itr):
    _compare(3, itr, full=False)


def test_multiscene_default_draws_are_keyed_by_scene_seed_iteration_and_view():
    """no hooks: each scene draws from view_seed(seed, itr, 0, 0) (photometric), (vi, 1) (fusion render) and (vi, 2) (PLMS), replayed here
    through a Distiller's hooks"""
    _compare(3, 1500, full=False, injected=False)


@pytest.mark.timeout(1200)
def test_multiscene_step_matches_per_scene_distillers_full_size():
    _compare(4, 1500, full=True)


def test_multiscene_refuses_what_it_does_not_support():
    from sparsefusion_b200.distillation import MultiSceneDistiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    vae, ddpm, _ = _small_models(percep=False)
    opt = get_default_torch_ngp_opt()
    caches = _scenes(2, full=False)
    ngps = [_ngp(0), _ngp(1)]
    with pytest.raises(NotImplementedError):
        MultiSceneDistiller(ngps, vae, ddpm, opt, caches, seeds=[0, 1], views_per_step=2)
    with pytest.raises(NotImplementedError):
        MultiSceneDistiller(ngps, vae, ddpm, opt, caches, seeds=[0, 1], fused_glue=False)
    from sparsefusion_b200.distillation import SceneCache
    small = SceneCache(**{f: getattr(caches[1], f)[..., :8, :8] if getattr(caches[1], f).dim() == 4 else getattr(caches[1], f)
                          for f in SceneCache.__dataclass_fields__})
    with pytest.raises(ValueError):
        MultiSceneDistiller(ngps, vae, ddpm, opt, [caches[0], small], seeds=[0, 1])
    with pytest.raises(RuntimeError):
        MultiSceneDistiller(ngps, vae, ddpm, opt, [caches[0], caches[1].to('cpu')], seeds=[0, 1])


def test_distill_scenes_writes_every_checkpoint(tmp_path):
    from types import SimpleNamespace
    from oracle import distill_oracle as do, unet_oracle as uo
    from sparsefusion_b200.distillation import SceneCache, distill_scenes, get_default_torch_ngp_opt
    vae, ddpm, _ = _small_models(percep=False)
    scenes_raw = {f'hydrant_{k:03d}': do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels,
                                                           render_hw=64, seed=3 + k) for k in range(2)}

    class Builder:
        def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
            assert eft == 'eft-model' and input_idx == [0, 1]
            return SceneCache(**scenes_raw[scene_cameras])
    seen = []
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    scenes = [(name, name, s['input_rgb'], s['input_mask'], None, [0, 1]) for name, s in scenes_raw.items()]
    nets = distill_scenes(0, args, get_default_torch_ngp_opt(), ('eft-model', vae, ddpm), str(tmp_path / 'out'), scenes, max_itr=3,
                          scene_builder=Builder(), seed=5,
                          on_iteration=lambda itr, m: seen.append((itr, m.last['photo_loss'].tolist(), m.last['fusion_loss'].tolist())))
    assert [s[0] for s in seen] == [0, 1, 2] and all(np.isfinite(s[1]).all() and np.isfinite(s[2]).all() and len(s[1]) == 2 for s in seen)
    for name, net in zip(scenes_raw, nets):
        sd = torch.load(str(tmp_path / 'out' / f'{name}.pt'), map_location='cpu')['model_state_dict']
        assert set(sd) == set(net.state_dict()) and sd['encoder.embeddings'].shape == (929336, 2)
        assert sd['encoder.embeddings'].abs().max() > 1e-4
