"""GIF palettes and the distilled scene's pictures on the GPU (csrc/palette.cu, sparsefusion_b200/video.py, distillation_loop / distill_scenes
with visualize=True) against the numpy restatement of the quantiser (oracle/palette_oracle.py): palettes, colour counts and index planes
equal bit for bit, and every written gif decodes to the quantiser's output for the expected panels."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

from test_metrics_gpu import _Builder, _models, _read_metrics, _render_like, _views

pytestmark = pytest.mark.gpu

KINDS = ('render', 'noise', 'black', 'few')


def _frames(B, H, W, seed):
    """uint8 frames cycling through render-like (black background), uniform noise, all black and few-colour frames"""
    rng = np.random.default_rng(seed)
    out = np.zeros((B, H, W, 3), np.uint8)
    for b in range(B):
        kind = KINDS[b % 4]
        if kind == 'render':
            out[b] = (_render_like(rng, H, W) * 255).astype(np.uint8)
        elif kind == 'noise':
            out[b] = rng.integers(0, 256, (H, W, 3))
        elif kind == 'few':
            out[b] = rng.integers(0, 256, (5, 3))[rng.integers(0, 5, (H, W))]
    return out


@pytest.mark.parametrize('colors', [256, 16, 2])
@pytest.mark.parametrize('shape', [(4, 256, 1280), (50, 256, 512), (3, 37, 53), (1, 1, 1)], ids=lambda s: f'{s[0]}x{s[1]}x{s[2]}')
def test_quantizer_matches_oracle(shape, colors):
    from oracle import palette_oracle as po
    from sparsefusion_b200.video import quantize_palette
    B, H, W = shape
    frames = _frames(B, H, W, seed=B * 7 + H + W + colors)
    fd = torch.from_numpy(frames).cuda()
    pal, nc, idx = quantize_palette(fd, colors)
    assert pal.shape == (B, 256, 3) and nc.shape == (B,) and idx.shape == (B, H, W)
    assert pal.dtype == idx.dtype == torch.uint8 and nc.dtype == torch.int32
    want = po.quantize(frames, colors)
    got = pal.cpu().numpy(), nc.cpu().numpy(), idx.cpu().numpy()
    print(f'  {shape} colors={colors}: ncolors {got[1][:4].tolist()}')
    for b in range(B):
        assert got[1][b] == want[1][b], (b, KINDS[b % 4], got[1][b], want[1][b])
        assert np.array_equal(got[0][b], want[0][b]), (b, KINDS[b % 4])
        assert np.array_equal(got[2][b], want[2][b]), (b, KINDS[b % 4], int((got[2][b] != want[2][b]).sum()))
    for again in (quantize_palette(fd, colors), quantize_palette(fd, colors)):
        assert all(torch.equal(x, y) for x, y in zip(again, (pal, nc, idx)))


def test_quantizer_rejects_bad_arguments():
    from sparsefusion_b200.video import quantize_palette
    x = torch.zeros(2, 4, 4, 3, dtype=torch.uint8, device='cuda')
    for colors in (1, 257):
        with pytest.raises(ValueError):
            quantize_palette(x, colors)
    with pytest.raises(ValueError):
        quantize_palette(torch.zeros(2, 4, 4, 4, dtype=torch.uint8, device='cuda'))
    with pytest.raises(ValueError):
        quantize_palette(torch.zeros(1, 4105, 4104, 3, dtype=torch.uint8, device='cuda'))     # 16 846 920 pixels: a channel sum could overflow
    with pytest.raises(RuntimeError):
        quantize_palette(x.float())


def test_to_uint8_matches_numpy():
    from sparsefusion_b200.video import to_uint8
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    vals = np.concatenate([k, np.nextafter(k, np.float32(0)), np.nextafter(k, np.float32(1)), [1.0, np.nextafter(np.float32(1), np.float32(0))]])
    vals = np.clip(vals, 0, 1).astype(np.float32)
    rng = np.random.default_rng(0)
    a = rng.choice(vals, (2, 9, 13, 3)).astype(np.float32)
    s = rng.choice(vals, (2, 9, 5, 1)).astype(np.float32)
    c = rng.random((2, 9, 7, 3), dtype=np.float32)
    got = to_uint8(*(torch.from_numpy(t).cuda() for t in (a, s, c))).cpu().numpy()
    for b in range(2):
        want = (np.hstack((a[b], np.repeat(s[b], 3, axis=-1), c[b])) * 255).astype(np.uint8)
        assert np.array_equal(got[b], want)
    out = to_uint8(torch.tensor([[[[-0.5, 1.5, 2.0]]]], device='cuda')).cpu().numpy()
    assert out.tolist() == [[[[0, 255, 255]]]]
    with pytest.raises(ValueError):
        to_uint8(torch.zeros(1, 8, 8, 3, device='cuda'), torch.zeros(1, 9, 8, 3, device='cuda'))


# ------------------------------------------------------------------------------------------------ render_views / distillation_loop
def test_render_views_restores_state():
    from sparsefusion_b200.evaluate import render_views
    from test_metrics_gpu import _net
    net, opt = _net(False)
    views = _views(2, 64).to('cuda')
    net.train()
    before = torch.cuda.get_rng_state().clone(), torch.get_rng_state().clone()
    img, sil = render_views(net, views.rays_o, views.rays_d, (64, 64), opt, seed=3, stream=4)
    assert net.training and img.shape == (2, 64, 64, 3) and sil.shape == (2, 64, 64)
    assert torch.equal(torch.cuda.get_rng_state(), before[0]) and torch.equal(torch.get_rng_state(), before[1])
    img2, _ = render_views(net, views.rays_o, views.rays_d, (64, 64), opt, seed=3, stream=4)
    img3, _ = render_views(net, views.rays_o, views.rays_d, (64, 64), opt, seed=3, stream=3)
    assert torch.equal(img, img2) and not torch.equal(img, img3)


N_CIRCLE = 50


class _VisBuilder(_Builder):
    """8 cached target views (one full row of the EFT grid for the 3 scene views) and 50 circle views, all at 128^2"""

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        from oracle import distill_oracle as do
        from sparsefusion_b200.distillation import SceneCache
        return SceneCache(**do.synthetic_scene(n_input=2, n_target=8, image_size=128, latent=16, feat_ch=self.cfg.cond_images_channels,
                                               render_hw=64, seed=scene_cameras))

    def circle_views(self, scene_cameras, n=N_CIRCLE):
        from sparsefusion_b200.synthetic import camera_rays, circle_cameras
        o, d = zip(*[camera_rays(c, 128, 128) for c in circle_cameras(n, radius=4.0 + 0.1 * scene_cameras)])
        return torch.from_numpy(np.stack(o)), torch.from_numpy(np.stack(d))


class _BuilderWithoutCircle(_Builder):
    pass


def _decode_gif(path):
    with Image.open(path) as im:
        assert im.info['loop'] == 0
        frames = []
        for i in range(im.n_frames):
            im.seek(i)
            frames.append((np.asarray(im.convert('RGB')).copy(), im.info['duration']))
    return frames


def _expected_gif(frames_u8):
    """what the gif of these uint8 CUDA frames must decode to: palette[indices] per frame, identical consecutive frames merged as Pillow
    stores them, with their summed duration"""
    from sparsefusion_b200.video import quantize_palette
    pal, nc, idx = (t.cpu().numpy() for t in quantize_palette(frames_u8))
    out = []
    for b in range(len(idx)):
        f = pal[b][idx[b]]
        if out and np.array_equal(out[-1][0], f):
            out[-1] = (f, out[-1][1] + 200)
        else:
            out.append((f, 200))
    return out


def _assert_gif(path, frames_u8, size):
    got, want = _decode_gif(path), _expected_gif(frames_u8)
    assert len(got) == len(want), (path, len(got), len(want))
    for i, ((g, gd), (w, wd)) in enumerate(zip(got, want)):
        assert g.shape == size and np.array_equal(g, w) and gd == wd, (path, i)


def _assert_jpeg(path, frame_u8, size):
    """the file is Pillow's default JPEG encoding of this uint8 CUDA frame [H, W, 3]"""
    import io
    buf = io.BytesIO()
    Image.fromarray(frame_u8.cpu().numpy()).save(buf, format='JPEG')
    with Image.open(path) as im:
        assert im.size == size and im.mode == 'RGB'
    assert open(path, 'rb').read() == buf.getvalue(), path


def _pictures(tmp_path):
    return sorted(str(p.relative_to(tmp_path)) for p in tmp_path.rglob('*') if p.suffix in ('.gif', '.jpg'))


def test_distillation_loop_visualize(tmp_path, capsys):
    from sparsefusion_b200.distillation import distillation_loop, get_default_torch_ngp_opt
    from sparsefusion_b200.evaluate import CIRCLE_STREAM, evaluate_scene, render_views
    from sparsefusion_b200.video import to_uint8
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    rgb, mask = torch.zeros(3, 3, 128, 128), torch.zeros(3, 1, 128, 128)
    builder = _VisBuilder(cfg)
    out = tmp_path / 'out'
    net = distillation_loop(0, args, opt, models, str(out), 'hydrant_000', 3, rgb, mask, None, [0, 1], use_diffusion=True, max_itr=3,
                            scene_builder=builder, seed=5, evaluate=True, visualize=True)
    printed = capsys.readouterr().out
    assert f'saved video {out}/render_gifs/hydrant_000.gif\n' in printed and f'saved video {out}/render_gifs/hydrant_000_circle.gif\n' in printed
    assert _pictures(tmp_path) == ['exp/log/hydrant_000_eft_grid.jpg', 'out/render_gifs/hydrant_000.gif', 'out/render_gifs/hydrant_000_circle.gif',
                                   'out/render_imgs/hydrant_000/000.jpg', 'out/render_imgs/hydrant_000/001.jpg', 'out/render_imgs/hydrant_000/002.jpg']
    views = _views(3, 128, seed=3).to('cuda')
    cache = builder.build(None, 3, None, None, None)
    se = evaluate_scene(net, views, opt, None, seed=5)
    got, _ = _read_metrics(out / 'metrics' / 'hydrant_000.txt')                # the scores come from the same renders as the gif
    assert float(got['psnr']) == pytest.approx(se.psnr.mean().item(), rel=1e-6, abs=1e-6)
    gt, gt_mask = views.rgb.permute(0, 2, 3, 1), views.mask.permute(0, 2, 3, 1)
    eft = cache.target_eft_image[:3].cuda().permute(0, 2, 3, 1)
    _assert_gif(out / 'render_gifs' / 'hydrant_000.gif', to_uint8(gt, eft, se.image, gt_mask, se.silhouette[..., None]), (128, 5 * 128, 3))
    for v in range(3):
        _assert_jpeg(out / 'render_imgs' / 'hydrant_000' / f'{v:03d}.jpg', to_uint8(gt[v:v + 1], se.image[v:v + 1])[0], (256, 128))
    co, cd = (t.cuda() for t in builder.circle_views(3))
    c_img, c_sil = render_views(net, co, cd, (128, 128), opt, seed=5, stream=CIRCLE_STREAM)
    _assert_gif(out / 'render_gifs' / 'hydrant_000_circle.gif', to_uint8(c_img, c_sil[..., None]), (128, 256, 3))
    tiles = to_uint8(cache.target_eft_image.cuda().permute(0, 2, 3, 1))       # one row of 8 tiles side by side
    _assert_jpeg(tmp_path / 'exp' / 'log' / 'hydrant_000_eft_grid.jpg', torch.cat(list(tiles), dim=1), (8 * 128, 128))

    # visualize without evaluate: the same sequence renders (stream 3), four panels without the EFT image, no EFT grid
    out2, exp2 = tmp_path / 'b' / 'out', tmp_path / 'b' / 'exp'
    net2 = distillation_loop(0, SimpleNamespace(exp_dir=str(exp2)), opt, models, str(out2), 'hydrant_000', 3, rgb, mask, None, [0, 1],
                             use_diffusion=False, max_itr=2, scene_builder=builder, seed=6, visualize=True)
    assert not (exp2 / 'log').exists() and not (out2 / 'metrics').exists()
    se2 = evaluate_scene(net2, views, opt, None, seed=6)
    _assert_gif(out2 / 'render_gifs' / 'hydrant_000.gif', to_uint8(gt, se2.image, gt_mask, se2.silhouette[..., None]), (128, 4 * 128, 3))

    # visualize=False: no pictures at all
    out3 = tmp_path / 'c'
    distillation_loop(0, SimpleNamespace(exp_dir=str(out3)), opt, models, str(out3), 'hydrant_000', 3, rgb, mask, None, [0, 1],
                      use_diffusion=True, max_itr=1, scene_builder=builder, seed=5)
    assert (out3 / 'hydrant_000.pt').exists() and _pictures(out3) == []

    # a builder without circle_views fails before any iteration and writes nothing
    seen, out4 = [], tmp_path / 'd'
    with pytest.raises(TypeError, match='circle_views'):
        distillation_loop(0, SimpleNamespace(exp_dir=str(out4)), opt, models, str(out4), 'hydrant_000', 3, rgb, mask, None, [0, 1],
                          max_itr=3, scene_builder=_BuilderWithoutCircle(cfg), seed=5, visualize=True, on_iteration=lambda itr, d: seen.append(itr))
    assert seen == [] and not out4.exists()

    # a cache too short for the EFT grid fails before any iteration
    class _Short(_VisBuilder):
        def eval_views(self, scene_cameras, scene_rgb, scene_mask):
            return _views(9, 128, seed=scene_cameras)                          # 9 views: two grid rows, 16 cached images needed
    with pytest.raises(ValueError, match='EFT grid'):
        distillation_loop(0, SimpleNamespace(exp_dir=str(out4)), opt, models, str(out4), 'hydrant_000', 3, rgb, mask, None, [0, 1],
                          max_itr=3, scene_builder=_Short(cfg), seed=5, visualize=True, on_iteration=lambda itr, d: seen.append(itr))
    assert seen == [] and not (out4 / 'hydrant_000.pt').exists()


def test_distill_scenes_visualize(tmp_path):
    from sparsefusion_b200.distillation import distill_scenes, get_default_torch_ngp_opt
    from sparsefusion_b200.evaluate import evaluate_scene
    from sparsefusion_b200.video import to_uint8
    models, cfg = _models()
    opt = get_default_torch_ngp_opt()
    rgb, mask = torch.zeros(3, 3, 128, 128), torch.zeros(3, 1, 128, 128)
    scenes = [(f'hydrant_{k:03d}', 3 + k, rgb, mask, None, [0, 1]) for k in range(2)]
    out = tmp_path / 'out'
    builder = _VisBuilder(cfg)
    nets = distill_scenes(0, SimpleNamespace(exp_dir=str(out)), opt, models, str(out), scenes, max_itr=2, scene_builder=builder, seed=7,
                          visualize=True)
    circles = []
    for k, net in enumerate(nets):
        name = f'hydrant_{k:03d}'
        assert (out / 'log' / f'{name}_eft_grid.jpg').exists()
        assert sorted(p.name for p in (out / 'render_imgs' / name).iterdir()) == ['000.jpg', '001.jpg', '002.jpg']
        views = _views(3, 128, seed=3 + k).to('cuda')
        se = evaluate_scene(net, views, opt, None, seed=7 + k)
        eft = builder.build(None, 3 + k, None, None, None).target_eft_image[:3].cuda().permute(0, 2, 3, 1)
        _assert_gif(out / 'render_gifs' / f'{name}.gif', to_uint8(views.rgb.permute(0, 2, 3, 1), eft, se.image, views.mask.permute(0, 2, 3, 1),
                                                                  se.silhouette[..., None]), (128, 5 * 128, 3))
        circles.append((out / 'render_gifs' / f'{name}_circle.gif').read_bytes())
        assert len(_decode_gif(out / 'render_gifs' / f'{name}_circle.gif')) >= 1
    assert circles[0] != circles[1]
