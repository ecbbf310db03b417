"""Host side of the entropy term, the loss history and the progress outputs: the Pillow loss plots (size, line colours, legend, nan
breaks), the refusals of lambda_entropy < 0 and progress_every <= 0, the fingerprint at lambda_entropy 0, and old checkpoints (no history,
no lambda_entropy) passing check_state."""
import hashlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _colour_pixels(path, rgb, tol=60):
    from PIL import Image
    a = np.asarray(Image.open(path).convert('RGB')).astype(int)
    return np.abs(a - np.array(rgb)).sum(-1) < tol


def test_loss_plots_are_640x480_with_three_colours_and_a_legend(tmp_path):
    from PIL import Image
    from sparsefusion_b200.progress import COLORS, write_loss_plots
    n = 60
    x = np.arange(n, dtype=np.float32)
    rows = np.stack((2.0 - x / n, 0.5 + 0.2 * np.sin(x / 5), 0.1 + 0.0 * x, 1.0 + x / n), 1).astype(np.float32)
    write_loss_plots(str(tmp_path), 'scene', rows)
    for f in ('scene_loss.jpg', 'scene_fusionloss.jpg'):
        with Image.open(tmp_path / 'log' / f) as im:
            assert im.size == (640, 480) and im.format == 'JPEG'
    loss = str(tmp_path / 'log' / 'scene_loss.jpg')
    for c in COLORS:
        hit = _colour_pixels(loss, c)
        assert hit.sum() > 40, c
        # the legend's line sample sits in the upper right corner of the axes
        assert hit[58:140, 400:576].any(), c
    fus = str(tmp_path / 'log' / 'scene_fusionloss.jpg')
    assert _colour_pixels(fus, COLORS[0]).sum() > 40 and _colour_pixels(fus, COLORS[1]).sum() < 5


def test_a_nan_row_breaks_the_curve(tmp_path):
    from sparsefusion_b200.progress import COLORS, plot_lines
    y = np.full(100, 1.0)
    y[::2] = 0.0
    y[40:60] = np.nan
    plot_lines(str(tmp_path / 'a.jpg'), [y])
    hit = _colour_pixels(str(tmp_path / 'a.jpg'), COLORS[0])
    cols = hit.any(0)
    x0, x1 = 80, 576
    px = lambda i: int(round(x0 + (i + 4.95) / 108.9 * (x1 - x0)))     # x limits: -4.95 .. 103.95 (5 % margins)
    assert cols[px(20)] and cols[px(80)] and not cols[px(45):px(55)].any()
    # all-nan, single-row and constant series draw axes without failing
    plot_lines(str(tmp_path / 'b.jpg'), [np.full(3, np.nan)], ['x'])
    plot_lines(str(tmp_path / 'c.jpg'), [np.zeros(1)], ['x'])
    plot_lines(str(tmp_path / 'd.jpg'), [np.zeros(0)])


@pytest.mark.parametrize('bad', [0, -20, 2.5, True])
def test_progress_every_must_be_a_positive_int(bad):
    from sparsefusion_b200.distillation import distill_scenes, distillation_loop
    from sparsefusion_b200.progress import check_progress_every
    with pytest.raises(ValueError, match='progress_every'):
        check_progress_every(bad)
    args = SimpleNamespace(exp_dir='/nonexistent')
    with pytest.raises(ValueError, match='progress_every'):
        distillation_loop(0, args, None, (None, None, None), '/nonexistent', 's', None, None, None, None, [0], use_diffusion=False,
                          progress_every=bad)
    with pytest.raises(ValueError, match='progress_every'):
        distill_scenes(0, args, None, (None, None, None), '/nonexistent', [('s', None, None, None, None, [0])], use_diffusion=False,
                       progress_every=bad)


@pytest.mark.parametrize('bad', [-1e-4, float('nan'), float('inf')])
def test_lambda_entropy_must_be_finite_and_not_negative(bad):
    from sparsefusion_b200 import image_glue as glue
    from sparsefusion_b200.distillation import Distiller, distill_scenes, distillation_loop
    args = SimpleNamespace(exp_dir='/nonexistent')
    with pytest.raises(ValueError, match='lambda_entropy'):
        distillation_loop(0, args, None, (None, None, None), '/nonexistent', 's', None, None, None, None, [0], use_diffusion=False,
                          lambda_entropy=bad)
    with pytest.raises(ValueError, match='lambda_entropy'):
        distill_scenes(0, args, None, (None, None, None), '/nonexistent', [('s', None, None, None, None, [0])], use_diffusion=False,
                       lambda_entropy=bad)
    with pytest.raises(ValueError, match='lambda_entropy'):
        Distiller(None, None, None, None, None, lambda_entropy=bad)
    if bad < 0:
        with pytest.raises(ValueError, match='lambda_entropy'):
            glue.photometric_loss(torch.zeros(4, 3), torch.zeros(4), torch.zeros(3, 4, 4), torch.zeros(1, 4, 4), 2, 2, 2, 1.0, 1.0, 1e-3,
                                  lambda_entropy=bad)


# ---------------------------------------------------------------------------------------------------- checkpoints
def _host_digest(cache):
    from sparsefusion_b200.distillation import SceneCache
    return {f: (tuple(getattr(cache, f).shape), int.from_bytes(hashlib.sha256(getattr(cache, f).contiguous().numpy().tobytes()).digest()[:8], 'little'))
            for f in SceneCache.__dataclass_fields__}


@pytest.fixture
def distiller(monkeypatch):
    from oracle import distill_oracle as do, unet_oracle as uo
    from sparsefusion_b200 import distillation
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.vldm import DDPM
    monkeypatch.setattr(distillation, 'cache_digest', _host_digest)
    cfg = uo.SMALL
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults),
                cond_images_channels=cfg.cond_images_channels, attn_pool_text=False, attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads)
    ddpm = DDPM(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10)
    cache = distillation.SceneCache(**do.synthetic_scene(n_input=2, n_target=6, image_size=32, latent=16, feat_ch=cfg.cond_images_channels,
                                                         render_hw=16, seed=3))

    def make(**kw):
        opt = get_default_torch_ngp_opt()
        return distillation.Distiller(NeRFNetwork(opt), None, ddpm, opt, cache, **kw)
    return make


def _old_checkpoint(sd):
    """``sd`` as a checkpoint written before the entropy term and the loss history existed"""
    old = {k: v for k, v in sd.items() if k != 'history'}
    old['fingerprint'] = {k: v for k, v in sd['fingerprint'].items() if k != 'lambda_entropy'}
    return old


def test_fingerprint_has_no_entropy_field_at_zero(distiller):
    d0, d1 = distiller(), distiller(lambda_entropy=1e-4)
    fp0 = d0.fingerprint()
    assert 'lambda_entropy' not in fp0
    assert set(d1.fingerprint()) == set(fp0) | {'lambda_entropy'} and d1.fingerprint()['lambda_entropy'] == 1e-4
    assert {k: v for k, v in d1.fingerprint().items() if k != 'lambda_entropy'} == fp0


def test_old_checkpoint_passes_check_state_and_resumes_with_nan_history(distiller):
    d = distiller(max_itr=10)
    sd = d.state_dict(itr=4)
    assert tuple(sd['history'].shape) == (4, 4)
    old = _old_checkpoint(sd)
    fresh = distiller(max_itr=10)
    fresh.check_state(old)
    fresh.load_state_dict(old)
    assert fresh.next_itr == 4 and tuple(fresh.history.shape) == (4, 4) and torch.isnan(fresh.history).all()
    # a nonzero entropy weight cannot continue a run made without it, nor another weight
    with pytest.raises(ValueError, match='lambda_entropy'):
        distiller(lambda_entropy=1e-3).check_state(old)
    with pytest.raises(ValueError, match='lambda_entropy'):
        distiller(lambda_entropy=1e-3).check_state(distiller(lambda_entropy=1e-2).state_dict(itr=0))


def test_history_rows_round_trip_through_a_checkpoint(distiller):
    d = distiller(max_itr=6)
    rows = torch.arange(24, dtype=torch.float32).view(6, 4)
    for i in range(5):
        d._record(i, 0, rows[i])
    d.next_itr = 5
    sd = d.state_dict()
    assert torch.equal(sd['history'], rows[:5])
    e = distiller(max_itr=3)                         # fewer preallocated rows than the checkpoint holds: the buffer grows
    e.load_state_dict(sd)
    assert torch.equal(e.history, rows[:5])
    bad = dict(sd, history=torch.zeros(5, 3))
    with pytest.raises(ValueError, match='history'):
        distiller().check_state(bad)


def test_isolated_values_are_drawn_as_dots(tmp_path):
    """a series logged every other iteration (a rank that computes the photometric term every R-th step) still shows"""
    from sparsefusion_b200.progress import COLORS, plot_lines
    y = np.full(60, np.nan)
    y[::2] = np.linspace(1.0, 2.0, 30)
    plot_lines(str(tmp_path / 'a.jpg'), [y])
    assert _colour_pixels(str(tmp_path / 'a.jpg'), COLORS[0]).sum() > 30


def test_view_rows_copies_only_the_input_views():
    from sparsefusion_b200.distillation import _view_rows
    from sparsefusion_b200.evaluate import EvalViews
    v = EvalViews(rays_o=torch.arange(5.0).view(5, 1, 1).expand(5, 4, 3).contiguous(), rays_d=torch.zeros(5, 4, 3), rgb=torch.zeros(5, 3, 2, 2),
                  mask=torch.zeros(5, 1, 2, 2))
    r = _view_rows(v, [3, 1])
    assert r.rays_o[:, 0, 0].tolist() == [3.0, 1.0] and r.rgb.shape == (2, 3, 2, 2)
    assert r.rays_o.untyped_storage().nbytes() == 2 * 4 * 3 * 4
