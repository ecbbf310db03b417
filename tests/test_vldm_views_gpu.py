"""Guided PLMS sampling in the fused loop and the EFT / VLDM baselines of a scene (sparsefusion_b200/plms.py, baselines.py).

(1) guided ``PLMSSampler.sample`` from pure noise against the reference's own guided sampler (tests/golden/plms_cfg_small.npz), per row, at
    the bar of the unguided golden test (relative L2 5e-3), with every evaluation a graph replay;
(2) the graph-replayed batch-2B guided path against ``Unet.forward_with_cond_scale`` driven eagerly through the reference-shaped p_sample;
(3) ``sample_vldm_views``: the same images for max_batch 1, 2 and 6 and on a re-run with the same seed, up to fp32 summation order (split-K
    convolutions sum their partial products with red.global.add, in no fixed order, so re-runs are not bit-identical; the keyed draws are);
(4) ``evaluate_baselines``' metrics files equal the scores recomputed on the images it returns; ``distill_scenes(evaluate_baselines=True)``
    writes each scene's files.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _models():
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
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
    return ('eft-model', vae.cuda(), ddpm), cfg


def _noise(src):
    return lambda t: src(t.cpu()).to(t.device)


def test_guided_sample_vs_reference_golden(golden_dir):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import PLMSSampler
    (_, _, ddpm), cfg = _models()
    g = np.load(f'{golden_dir}/plms_cfg_small.npz')
    cond = torch.from_numpy(g['cond']).cuda()
    for s in (3.0, 1.5):
        key = f'{s:.1f}'
        src = uo.NoiseSource(seed=int(g['noise_seed']))
        sampler = PLMSSampler(ddpm, 50, noise_fn=_noise(src))
        img = sampler.sample(cond_images=cond, cond_scale=s, use_tqdm=False)
        want = torch.from_numpy(g[f'img_{key}'])
        rels = [_rel(img[r].cpu(), want[r]) for r in range(int(g['batch']))]
        print(f'guided PLMS cond_scale={s}: {sampler.last_unet_calls} evaluations, {sampler.last_graph_replays} replays, rel per row {rels}')
        assert sampler.last_unet_calls == int(g[f'calls_{key}']) and src.count == int(g[f'draws_{key}'])
        assert sampler.last_graph_replays == sampler.last_unet_calls
        assert max(rels) < 5e-3


def test_graph_guided_path_matches_eager_forward_with_cond_scale():
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import GaussianDiffusionContinuousTimes
    from sparsefusion_b200.plms import PLMSSampler
    (_, _, ddpm), cfg = _models()
    unet, sched = ddpm.unets[0], ddpm.noise_schedulers[0]
    rng = np.random.default_rng(21)
    B, h = 3, cfg.image_size
    cond = torch.from_numpy(rng.standard_normal((B, cfg.cond_images_channels, h, h), dtype=np.float32)).cuda()
    s = 2.5
    # one evaluation: the batch-2B replay's halves combined as the reference combines them, against the two eager forwards
    x = torch.from_numpy(rng.standard_normal((B, 4, h, h), dtype=np.float32)).cuda()
    ls = sched.get_condition(torch.full((B,), 0.6, device='cuda'))
    sampler = PLMSSampler(ddpm, 50)
    pair = sampler._eps_pair(unet, torch.cat((x, x)), torch.cat((ls, ls)), torch.cat((cond, cond * 0)), None).clone()
    eager = unet.forward_with_cond_scale(x, ls, cond_images=cond, cond_scale=s)
    rel_eps = _rel(pair[B:] + (pair[:B] - pair[B:]) * s, eager)
    assert sampler.last_graph_replays == 1 and rel_eps < 1e-5, rel_eps

    # a whole run: the fused loop against the reference-shaped p_sample, whose _eps drives forward_with_cond_scale eagerly
    src = uo.NoiseSource(seed=4)
    fused = PLMSSampler(ddpm, 50, noise_fn=_noise(src))
    got = fused.sample(cond_images=cond, cond_scale=s, use_tqdm=False)
    assert fused.last_graph_replays == fused.last_unet_calls == 51
    src = uo.NoiseSource(seed=4)
    ref = PLMSSampler(ddpm, 50, noise_fn=_noise(src))
    img = ref.noise_fn(torch.empty(B, 4, h, h, device='cuda'))             # plms.py:73
    ref.noise_fn(img)                                                       # q_sample's draw (:81)
    short = GaussianDiffusionContinuousTimes(noise_schedule='cosine', timesteps=50)
    old_eps = []
    for t, t_next in short.get_sampling_timesteps(B, device='cuda'):
        img, _, e_t = ref.p_sample(unet, img, t, t_next, cond, s, sched, 'noise', False, old_eps)
        old_eps = (old_eps + [e_t])[-3:]
    want = img.clamp(-10, 10)
    assert ref.last_graph_replays == 0 and ref.last_unet_calls == 51
    rels = [_rel(got[r], want[r]) for r in range(B)]
    print(f'guided fused (graph, batch 2B) vs eager forward_with_cond_scale: eps rel {rel_eps:.2e}, final latents rel per row {rels}')
    assert max(rels) < 1e-3


def test_sample_vldm_views_batching_and_seed():
    from sparsefusion_b200.baselines import VLDM_STREAM, sample_vldm_views
    from sparsefusion_b200.distillation import KeyedNoise, view_seed
    (_, vae, ddpm), cfg = _models()
    rng = np.random.default_rng(5)
    V, h = 6, cfg.image_size
    feats = torch.from_numpy(rng.standard_normal((V, cfg.cond_images_channels, h, h), dtype=np.float32)).cuda()
    for s in (3.0, 1.0):
        runs = {mb: sample_vldm_views(ddpm, vae, feats, seed=11, cond_scale=s, plms_steps=20, max_batch=mb) for mb in (6, 2, 1)}
        ref = runs[6]
        assert ref.shape == (V, 3, 8 * h, 8 * h) and ref.min().item() >= 0.0 and ref.max().item() <= 1.0
        for mb in (2, 1):
            rels = [_rel(runs[mb][v], ref[v]) for v in range(V)]
            print(f'cond_scale={s} max_batch {mb} vs 6: rel per view max {max(rels):.2e}')
            assert max(rels) < 1e-3
        again = sample_vldm_views(ddpm, vae, feats, seed=11, cond_scale=s, plms_steps=20, max_batch=6)
        other = sample_vldm_views(ddpm, vae, feats, seed=12, cond_scale=s, plms_steps=20, max_batch=6)
        print(f'cond_scale={s}: re-run rel {_rel(again, ref):.2e}, other seed rel {_rel(other, ref):.2e}')
        assert _rel(again, ref) < 1e-5 and _rel(other, ref) > 1e-2
    guided = sample_vldm_views(ddpm, vae, feats[:2], seed=11, cond_scale=3.0, plms_steps=20)
    assert _rel(guided, runs[6][:2]) > 1e-3                                  # guidance changes the samples
    # the draws themselves are keyed per view: bit-identical whichever views share the batch
    a = KeyedNoise([view_seed(11, 0, v, VLDM_STREAM) for v in range(4)], 'cuda')(torch.empty(4, 4, h, h, device='cuda'))
    b = KeyedNoise([view_seed(11, 0, v, VLDM_STREAM) for v in (2, 3)], 'cuda')(torch.empty(2, 4, h, h, device='cuda'))
    assert torch.equal(a[2:], b)


def _scene(cfg, seed, n_target=6):
    from oracle import distill_oracle as do
    from sparsefusion_b200.distillation import SceneCache
    return SceneCache(**do.synthetic_scene(n_input=2, n_target=n_target, image_size=128, latent=16, feat_ch=cfg.cond_images_channels,
                                           render_hw=64, seed=seed))


def _views(n, hw, seed=0):
    from sparsefusion_b200.evaluate import EvalViews
    rng = np.random.default_rng(seed)
    rgb = torch.from_numpy(rng.random((n, 3, hw, hw), dtype=np.float32))
    rays = torch.zeros(n, hw * hw, 3)
    return EvalViews(rays_o=rays, rays_d=rays.clone(), rgb=rgb, mask=torch.ones(n, 1, hw, hw))


def _read(path):
    return open(path).read()


def test_evaluate_baselines_files_match_recomputed_scores(tmp_path):
    from PIL import Image
    from sparsefusion_b200.baselines import evaluate_baselines
    from sparsefusion_b200.evaluate import score_images, write_scene_metrics
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    (_, vae, ddpm), cfg = _models()
    cache = _scene(cfg, 3).to('cuda')
    views = _views(4, 128, seed=3).to('cuda')
    percep = PerceptualLoss('vgg', device='cuda', seed=1)
    out = evaluate_baselines(str(tmp_path), 'hydrant_000', ddpm, vae, cache, views, percep, seed=9, cond_scale=2.0, plms_steps=10, max_batch=3)
    assert set(out) == {'eft', 'vldm'}
    assert torch.equal(out['eft'].image, cache.target_eft_image[:4].permute(0, 2, 3, 1).float())
    for name in ('eft', 'vldm'):
        se = out[name]
        assert se.image.shape == (4, 128, 128, 3) and se.silhouette is None
        # SSIM / PSNR are bit-reproducible; LPIPS-VGG's convolutions sum split-K partials in no fixed order
        again = score_images(se.image, views.rgb, percep)
        assert torch.equal(again.psnr, se.psnr) and torch.equal(again.ssim, se.ssim), name
        assert torch.allclose(again.lpips, se.lpips, rtol=1e-5, atol=0), (name, again.lpips, se.lpips)
        for scores, tag in ((se, 'returned'), (again, 'recomputed')):
            write_scene_metrics(str(tmp_path / f'{tag}_{name}.txt'), scores)
        got = _read(tmp_path / 'metrics' / f'hydrant_000_{name}.txt')
        print(f'{name}: {got!r}')
        assert got == _read(tmp_path / f'returned_{name}.txt')
        g, w = got.split('\n'), _read(tmp_path / f'recomputed_{name}.txt').split('\n')
        assert g[:4] == w[:4] and abs(float(g[5]) - float(w[5])) <= 1e-5 * abs(float(w[5]))   # psnr, ssim exactly; lpips
    gif = Image.open(tmp_path / 'render_gifs' / 'hydrant_000_baselines.gif')
    assert gif.size == (3 * 128, 128) and gif.n_frames == 4


class _Builder:
    def __init__(self, cfg):
        self.cfg = cfg

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        return _scene(self.cfg, scene_cameras)

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        return _views(3, 128, seed=scene_cameras)


def test_distill_scenes_and_standalone_entry_write_baselines(tmp_path):
    from sparsefusion_b200.baselines import score_baselines
    from sparsefusion_b200.distillation import distill_scenes, get_default_torch_ngp_opt
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    rgb, mask = torch.zeros(3, 3, 128, 128), torch.zeros(3, 1, 128, 128)
    scenes = [(f'hydrant_{k:03d}', 3 + k, rgb, mask, None, [0, 1]) for k in range(2)]
    out = tmp_path / 'out'
    distill_scenes(0, args, opt, models, str(out), scenes, max_itr=3, scene_builder=_Builder(cfg), seed=7, evaluate_baselines=True,
                   vldm_cond_scale=3.0)
    texts = {}
    for seq, *_ in scenes:
        for name in ('eft', 'vldm'):
            texts[seq, name] = _read(out / 'metrics' / f'{seq}_{name}.txt')
            assert texts[seq, name].startswith('warning: this metric is used for debugging only and not the final metricpsnr:\n')
        assert (out / 'render_gifs' / f'{seq}_baselines.gif').exists() and (out / f'{seq}.pt').exists()
        assert not (out / 'metrics' / f'{seq}.txt').exists()                 # evaluate stays off
    assert texts['hydrant_000', 'vldm'] != texts['hydrant_001', 'vldm']
    # no distillation: the same scenes, seeds and guidance give the same baselines (the EFT scores exactly; the VLDM ones to fp32 order)
    solo = tmp_path / 'solo'
    res = score_baselines(0, args, models, str(solo), scenes, scene_builder=_Builder(cfg), seed=7, cond_scale=3.0)
    assert len(res) == 2 and not (solo / 'hydrant_000.pt').exists()
    for seq, *_ in scenes:
        assert _read(solo / 'metrics' / f'{seq}_eft.txt') == texts[seq, 'eft']
        assert (solo / 'render_gifs' / f'{seq}_baselines.gif').exists()
    psnr = float(texts['hydrant_001', 'vldm'].split('\n')[1])
    assert abs(res[1]['vldm'].psnr.mean().item() - psnr) <= 1e-3 * abs(psnr)
