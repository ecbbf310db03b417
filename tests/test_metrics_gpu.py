"""Scene scores on the GPU (csrc/metrics.cu, sparsefusion_b200/evaluate.py, distillation_loop / distill_scenes with evaluate=True) against the
numpy / scipy restatement of scikit-image's SSIM and PSNR (oracle/metrics_oracle.py).

Bars: SSIM within 1e-6 absolute and MSE within 1e-6 relative of the oracle on the same fp32 images (the oracle's own fp32 and fp64 forms
differ by up to 3.4e-8 in SSIM on 256^2 images); identical images give SSIM 1.0 and PSNR inf exactly; repeated calls are bit-identical.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _render_like(rng, H, W):
    """a render of an object on a black background: mostly zeros, a smooth blob with texture"""
    yy, xx = np.mgrid[0:H, 0:W]
    cy, cx, r = rng.uniform(0.3, 0.7) * H, rng.uniform(0.3, 0.7) * W, rng.uniform(0.15, 0.35) * min(H, W)
    blob = np.clip(1.0 - ((yy - cy) ** 2 + (xx - cx) ** 2) / r ** 2, 0.0, 1.0)
    img = blob[..., None] * (0.5 + 0.5 * rng.random((H, W, 3)))
    return img.astype(np.float32)


def _pairs(B, H, W, seed):
    """B pairs cycling through three kinds: independent noise, render-like pairs (mostly black), identical pairs"""
    rng = np.random.default_rng(seed)
    a, b, kind = np.empty((B, H, W, 3), np.float32), np.empty((B, H, W, 3), np.float32), []
    for i in range(B):
        k = ('noise', 'render', 'identical')[i % 3]
        if k == 'noise':
            a[i] = rng.random((H, W, 3), dtype=np.float32)
            b[i] = np.clip(a[i] + 0.1 * rng.standard_normal((H, W, 3)).astype(np.float32), 0, 1) if i % 2 else rng.random((H, W, 3), dtype=np.float32)
        elif k == 'render':
            a[i] = _render_like(rng, H, W)
            b[i] = np.clip(a[i] + 0.05 * rng.standard_normal((H, W, 3)).astype(np.float32) * (a[i] > 0), 0, 1)
        else:
            a[i] = _render_like(rng, H, W) if i % 2 else rng.random((H, W, 3), dtype=np.float32)
            b[i] = a[i]
        kind.append(k)
    return a, b, kind


def _check_against_oracle(pred, gt, ssim, psnr, kinds=None):
    from oracle import metrics_oracle as mo
    ssim, psnr = ssim.cpu().numpy(), psnr.cpu().numpy()
    worst = 0.0
    for i in range(pred.shape[0]):
        ws = mo.structural_similarity(pred[i], gt[i])
        wm = mo.mean_squared_error(pred[i], gt[i])
        worst = max(worst, abs(ssim[i] - float(ws)))
        assert abs(ssim[i] - float(ws)) <= 1e-6, (i, ssim[i], ws)
        if wm == 0:
            assert psnr[i] == np.inf and ssim[i] == 1.0, (i, psnr[i], ssim[i])
        else:
            gm = 10.0 ** (-psnr[i] / 10.0)
            assert abs(gm - wm) <= 1e-6 * wm, (i, gm, wm)
            assert abs(psnr[i] - mo.peak_signal_noise_ratio(pred[i], gt[i])) <= 1e-5
        if kinds is not None and kinds[i] == 'identical':
            assert ssim[i] == 1.0 and psnr[i] == np.inf
    return worst


@pytest.mark.parametrize('B', [1, 5, 64])
@pytest.mark.parametrize('hw', [(256, 256), (128, 128), (7, 7), (37, 53)], ids=lambda s: f'{s[0]}x{s[1]}')
def test_kernel_matches_oracle(hw, B):
    from sparsefusion_b200.evaluate import image_metrics
    H, W = hw
    a, b, kinds = _pairs(B, H, W, seed=H * 1000 + W + B)
    ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    ssim, psnr = image_metrics(ad, bd)
    assert ssim.dtype == psnr.dtype == torch.float64 and ssim.shape == psnr.shape == (B,)
    worst = _check_against_oracle(a, b, ssim, psnr, kinds)
    print(f'  {H}x{W} B={B}: max |SSIM - oracle| {worst:.2e}')
    s2, p2 = image_metrics(ad, bd)
    assert torch.equal(ssim, s2) and torch.equal(psnr, p2)
    s1, p1 = image_metrics(ad[0], bd[0])                                      # one [H, W, 3] pair
    assert s1.shape == (1,) and s1[0] == ssim[0] and p1[0] == psnr[0]


def test_kernel_rejects_small_images():
    from sparsefusion_b200.evaluate import image_metrics
    for shape in ((1, 6, 6, 3), (2, 6, 40, 3), (2, 40, 6, 3)):
        x = torch.zeros(shape, device='cuda')
        with pytest.raises(ValueError):
            image_metrics(x, x.clone())
    with pytest.raises(ValueError):
        image_metrics(torch.zeros(2, 8, 8, 3, device='cuda'), torch.zeros(2, 8, 9, 3, device='cuda'))
    with pytest.raises(RuntimeError):
        image_metrics(torch.zeros(8, 8, 3, device='cuda', dtype=torch.float64), torch.zeros(8, 8, 3, device='cuda', dtype=torch.float64))


# ------------------------------------------------------------------------------------------------ evaluate_scene
def _net(cuda_ray, seed=0):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = cuda_ray
    net = NeRFNetwork(opt)
    sd = net.state_dict()
    sd.update(no.make_field_params(seed=seed))
    net.load_state_dict(sd)
    net = net.cuda()
    if cuda_ray:
        net.update_extra_state()
    return net, opt


def _views(n, hw, seed=0, radius=4.5):
    from sparsefusion_b200.evaluate import EvalViews
    from sparsefusion_b200.synthetic import camera_rays, circle_cameras
    o, d = zip(*[camera_rays(c, hw, hw) for c in circle_cameras(n, radius=radius)])
    rng = np.random.default_rng(seed)
    rgb = np.stack([_render_like(rng, hw, hw) for _ in range(n)]).transpose(0, 3, 1, 2)
    return EvalViews(rays_o=torch.from_numpy(np.stack(o)), rays_d=torch.from_numpy(np.stack(d)), rgb=torch.from_numpy(np.ascontiguousarray(rgb)),
                     mask=torch.from_numpy((rgb.max(1, keepdims=True) > 0).astype(np.float32)))


def _render_as_reference(net, views, opt, seed):
    from sparsefusion_b200.distillation import view_seed
    H, W = views.rgb.shape[2:]
    imgs = []
    net.eval()
    for v in range(views.rays_o.shape[0]):
        with torch.random.fork_rng(devices=[views.rays_o.device]):
            torch.cuda.manual_seed(view_seed(seed, 0, v, 3))
            out = net.render_batched(views.rays_o[v][None], views.rays_d[v][None], batched=True, perturb=True, bg_color=0, ambient_ratio=1.0,
                                     shading='albedo', force_all_rays=True, **vars(opt))
        imgs.append(out['image'].reshape(H, W, 3))
    return torch.stack(imgs)


@pytest.mark.parametrize('cuda_ray', [False, True], ids=['default', 'cuda_ray'])
def test_evaluate_scene(cuda_ray):
    from sparsefusion_b200.evaluate import evaluate_scene
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    net, opt = _net(cuda_ray)
    views = _views(4, 256).to('cuda')
    percep = PerceptualLoss('vgg', device='cuda', seed=3)
    net.train()
    torch.manual_seed(123)
    torch.cuda.manual_seed(123)
    before = torch.cuda.get_rng_state().clone(), torch.get_rng_state().clone()
    se = evaluate_scene(net, views, opt, percep, seed=11)
    assert net.training                                                        # restored
    assert torch.equal(torch.cuda.get_rng_state(), before[0]) and torch.equal(torch.get_rng_state(), before[1])
    assert se.image.shape == (4, 256, 256, 3) and se.silhouette.shape == (4, 256, 256)
    assert se.psnr.dtype == se.ssim.dtype == se.lpips.dtype == torch.float64
    ref = _render_as_reference(net, views, opt, 11)
    assert torch.equal(se.image, ref)
    print(f'  render max {se.image.max().item():.3f}, ssim {se.ssim.tolist()}, psnr {se.psnr.tolist()}, lpips {se.lpips.tolist()}')
    gt = views.rgb.permute(0, 2, 3, 1).contiguous().cpu().numpy()
    _check_against_oracle(se.image.cpu().numpy(), gt, se.ssim, se.psnr)
    for v in range(4):
        want = percep.value_and_grad(se.image[v].permute(2, 0, 1), views.rgb[v], normalize=True, want_grad=False)[0]
        assert abs(se.lpips[v].item() - want.item()) <= 1e-6 * abs(want.item()), (v, se.lpips[v].item(), want.item())
    se2 = evaluate_scene(net.eval(), views, opt, None, seed=11)
    assert not net.training
    assert torch.equal(se2.image, se.image) and torch.equal(se2.ssim, se.ssim) and torch.isnan(se2.lpips).all()
    se3 = evaluate_scene(net, views, opt, None, seed=12)                      # another seed, another jitter
    assert not torch.equal(se3.image, se.image)


# ------------------------------------------------------------------------------------------------ distillation_loop / distill_scenes
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


class _Builder:
    """synthetic scenes keyed by the scene_rgb argument's first value; eval_views at 128^2"""
    def __init__(self, cfg):
        self.cfg, self.built = cfg, []

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        from oracle import distill_oracle as do
        from sparsefusion_b200.distillation import SceneCache
        self.built.append(scene_cameras)
        return SceneCache(**do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=self.cfg.cond_images_channels,
                                               render_hw=64, seed=scene_cameras))

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        return _views(3, 128, seed=scene_cameras)


class _BuilderWithoutEval(_Builder):
    eval_views = None


def _read_metrics(path):
    text = open(path).read()
    assert text.startswith('warning: this metric is used for debugging only and not the final metricpsnr:\n')
    lines = text.split('\n')
    return dict(psnr=lines[1], ssim=lines[3], lpips=lines[5]), text


def _assert_same_scores(got, want):
    for k in ('psnr', 'ssim', 'lpips'):
        g, w = float(got[k]), float(want[k])
        assert (np.isnan(g) and np.isnan(w)) or abs(g - w) <= 1e-6 * max(1.0, abs(w)), (k, got[k], want[k])


def _expected_file(tmp_path, se):
    from sparsefusion_b200.evaluate import write_scene_metrics
    p = str(tmp_path / 'expected.txt')
    write_scene_metrics(p, se)
    return _read_metrics(p)


def test_distillation_loop_evaluate(tmp_path):
    from sparsefusion_b200.distillation import distillation_loop, get_default_torch_ngp_opt
    from sparsefusion_b200.evaluate import evaluate_scene
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    rgb, mask = torch.zeros(6, 3, 128, 128), torch.zeros(6, 1, 128, 128)
    builder = _Builder(cfg)
    lpips_w = PerceptualLoss('vgg', seed=1)                                    # stands in for the pretrained lpips.LPIPS demo.py passes
    out = tmp_path / 'out'
    net = distillation_loop(0, args, opt, models, str(out), 'hydrant_000', 3, rgb, mask, None, [0, 1], use_diffusion=True, max_itr=3,
                            loss_fn_vgg=lpips_w, scene_builder=builder, seed=5, evaluate=True)
    assert (out / 'hydrant_000.pt').exists()
    got, text = _read_metrics(out / 'metrics' / 'hydrant_000.txt')
    se = evaluate_scene(net, _views(3, 128, seed=3).to('cuda'), opt, PerceptualLoss('vgg', device='cuda', seed=1), seed=5)
    want, want_text = _expected_file(tmp_path, se)
    print('  metrics file:', got, 'expected:', want, 'same bytes:', text == want_text)
    _assert_same_scores(got, want)
    # without loss_fn_vgg: LPIPS is nan, SSIM and PSNR of the returned network (a second run trains another network: the renders' jitter
    # comes from torch's global generator, as in the reference)
    out2 = tmp_path / 'out2'
    net2 = distillation_loop(0, args, opt, models, str(out2), 'hydrant_000', 3, rgb, mask, None, [0, 1], use_diffusion=True, max_itr=3,
                             scene_builder=builder, seed=5, evaluate=True)
    got2, _ = _read_metrics(out2 / 'metrics' / 'hydrant_000.txt')
    se2 = evaluate_scene(net2, _views(3, 128, seed=3).to('cuda'), opt, None, seed=5)
    want2, _ = _expected_file(tmp_path, se2)
    assert got2['lpips'] == 'nan' == want2['lpips']
    _assert_same_scores(got2, want2)
    # evaluate=False: no metrics directory
    out3 = tmp_path / 'out3'
    distillation_loop(0, args, opt, models, str(out3), 'hydrant_000', 3, rgb, mask, None, [0, 1], use_diffusion=True, max_itr=1,
                      scene_builder=builder, seed=5)
    assert (out3 / 'hydrant_000.pt').exists() and not (out3 / 'metrics').exists()
    # a builder without eval_views fails before any iteration and writes nothing
    seen = []
    out4 = tmp_path / 'out4'
    with pytest.raises(TypeError, match='eval_views'):
        distillation_loop(0, args, opt, models, str(out4), 'hydrant_000', 3, rgb, mask, None, [0, 1], use_diffusion=True, max_itr=3,
                          scene_builder=_BuilderWithoutEval(cfg), seed=5, evaluate=True, on_iteration=lambda itr, d: seen.append(itr))
    assert seen == [] and not (out4 / 'hydrant_000.pt').exists()


def test_distill_scenes_evaluate(tmp_path):
    from sparsefusion_b200.distillation import distill_scenes, get_default_torch_ngp_opt
    from sparsefusion_b200.evaluate import evaluate_scene
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    rgb, mask = torch.zeros(6, 3, 128, 128), torch.zeros(6, 1, 128, 128)
    scenes = [(f'hydrant_{k:03d}', 3 + k, rgb, mask, None, [0, 1]) for k in range(2)]
    out = tmp_path / 'out'
    nets = distill_scenes(0, args, opt, models, str(out), scenes, max_itr=3, scene_builder=_Builder(cfg), seed=7, evaluate=True,
                          loss_fn_vgg=PerceptualLoss('vgg', seed=1))
    percep = PerceptualLoss('vgg', device='cuda', seed=1)
    texts = []
    for k, net in enumerate(nets):
        got, text = _read_metrics(out / 'metrics' / f'hydrant_{k:03d}.txt')
        se = evaluate_scene(net, _views(3, 128, seed=3 + k).to('cuda'), opt, percep, seed=7 + k)
        want, want_text = _expected_file(tmp_path, se)
        print(f'  scene {k}:', got, 'same bytes:', text == want_text)
        _assert_same_scores(got, want)
        texts.append(text)
        assert (out / f'hydrant_{k:03d}.pt').exists()
    assert texts[0] != texts[1]
