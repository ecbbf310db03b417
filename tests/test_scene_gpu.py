"""The per-scene preparation on the GPU: ``sfb_grid_rays`` against tests/golden/scene_prep.npz (the reference's GridRaysampler configurations),
``sfb_eft_t1_tokens`` per element against the eager T1 assembly of ``EpipolarFeatureTransformer.forward``, ``feature_cache`` against per-view
``batched_forward`` in each view's own relative frame, and ``distillation_loop`` end to end with ``NativeSceneBuilder``."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm()).item()


def _model():
    from oracle import eft_oracle as eo
    from sparsefusion_b200.eft import EpipolarFeatureTransformer
    m = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=True)
    m.load_state_dict(eo.make_params({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0), strict=True)
    return m.cuda()


def _ring(n=8, radius=4.0, seed=0):
    """n cameras on a ring looking at the origin with per-camera focal lengths and principal points, image_size 256"""
    from oracle import eft_oracle as eo
    from sparsefusion_b200.cameras import PerspectiveCameras
    c = eo.look_at_cameras(n, radius=radius)
    rng = np.random.default_rng(seed)
    f = torch.from_numpy(rng.uniform(2.6, 3.4, (n, 2)).astype(np.float32))
    p = torch.from_numpy(rng.uniform(-0.05, 0.05, (n, 2)).astype(np.float32))
    return PerspectiveCameras(c.R, c.T, f, p, torch.full((n, 2), 256.0))


def test_grid_rays_against_reference_samplers(golden_dir):
    from sparsefusion_b200 import cameras as C
    g = np.load(f'{golden_dir}/scene_prep.npz')
    t = lambda k: torch.from_numpy(g[k])
    cams = C.PerspectiveCameras(t('R'), t('T'), t('focal_length'), t('principal_point'), t('image_size'))
    path = C.PerspectiveCameras(t('path_R'), t('path_T'), t('path_focal_length'), t('path_principal_point'), cams.image_size[:1].expand(50, 2))
    aug = C.concat_cameras([cams, path])
    circle = C.PerspectiveCameras(t('circle_R'), t('circle_T'), t('path_focal_length'), t('path_principal_point'))
    for cam, hw, key in ((C.relative_cameras(aug, [0], False)[int(g['ray_camera_128'])], 128, 'rays128'),
                         (C.relative_cameras(aug, [0], True)[[int(i) for i in g['ray_cameras_32']]], 32, 'rays32'),
                         (circle[int(g['ray_camera_256'])], 256, 'rays256')):
        o, d = C.grid_rays(cam, hw, hw, 'cuda', 256, 256)
        assert o.shape == (len(cam), hw * hw, 3)
        if key == 'rays256':
            o, d = o.reshape(-1, 3)[::int(g['ray_stride_256'])], d.reshape(-1, 3)[::int(g['ray_stride_256'])]
        for got, ref in ((o, g[f'{key}_o']), (d, g[f'{key}_d'])):
            ref = torch.from_numpy(ref).reshape(got.shape)
            err = ((got.cpu() - ref).abs().max() / ref.abs().max()).item()
            print(f'grid rays {key}: max rel err {err:.2e}')
            assert err < 1e-5, key


def _eager_t1(m, cams, origins, directions, lengths):
    """the T1 token rows exactly as EpipolarFeatureTransformer.forward assembles them (eft.py:215-327), for one view's cameras"""
    from sparsefusion_b200 import _lib as lib
    from sparsefusion_b200.eft import camera_center, transform_points_ndc
    N, D = lengths.shape
    NC = m.encoder_latent.shape[0]
    xyz = origins[:, None, :] + lengths[:, :, None] * directions[:, None, :]
    ndc = transform_points_ndc(cams, xyz.reshape(1, N * D, 3))
    grid = (-ndc[..., :2]).contiguous()
    M, d1p = N * D, 608
    tok1 = torch.zeros(NC, M, d1p, device='cuda')
    lat, img = m.encoder_latent, m._images_nhwc
    lib.call('sfb_grid_sample_nhwc', lat.data_ptr(), lat.stride(2), lib.fptr(grid), tok1[..., 91:].data_ptr(), d1p, NC, lat.shape[1], lat.shape[2], 512, M,
             lib.stream())
    lib.call('sfb_grid_sample_nhwc', img.data_ptr(), img.stride(2), lib.fptr(grid), tok1[..., 603:].data_ptr(), d1p, NC, img.shape[1], img.shape[2], 3, M,
             lib.stream())
    oc = camera_center(cams)[:, None, None, :].expand(NC, N, D, 3)
    ref_plucker = m.encode_plucker(oc, torch.nn.functional.normalize(xyz[None] - oc, dim=-1))
    tok1[..., :78] = ref_plucker.reshape(NC, M, 78)
    tok1[..., 78:91] = m.harmonic_embedding(lengths[..., None]).reshape(1, M, 13)
    return tok1, ndc[..., 2]


@pytest.mark.parametrize('NC', [2, 6])
def test_t1_tokens_per_element_against_forward_assembly(NC):
    from types import SimpleNamespace
    from sparsefusion_b200 import _lib as lib
    m = _model()
    g = torch.Generator().manual_seed(NC)
    images = torch.rand(NC, 3, 96, 80, generator=g).cuda()
    m.encode(None, images)
    V, N, D = 2, 40, 20
    Rs = torch.linalg.qr(torch.randn(V, NC, 3, 3, generator=g))[0]
    cams = SimpleNamespace(R=Rs, T=torch.randn(V, NC, 3, generator=g) + torch.tensor([0.0, 0.0, 3.0]), focal_length=torch.rand(V, NC, 2, generator=g) + 1.5,
                           principal_point=(torch.rand(V, NC, 2, generator=g) - 0.5) * 0.2)
    origins = torch.randn(V, N, 3, generator=g)
    directions = torch.randn(V, N, 3, generator=g)
    lengths = torch.linspace(-4.0, 8.0, D)[None, None].expand(V, N, D) + torch.rand(V, N, 1, generator=g)    # samples behind the origins too
    cu = lambda x: x.cuda().contiguous()
    packed = cu(torch.cat((cams.R.reshape(V, NC, 9), cams.T, cams.focal_length, cams.principal_point), dim=-1))
    o_d, d_d, l_d = cu(origins), cu(directions), cu(lengths)                            # held: the kernel reads them after fptr returns
    out = torch.full((NC, V * N * D, 608), float('nan'), device='cuda')
    lat, img = m.encoder_latent, m._images_nhwc
    lib.call('sfb_eft_t1_tokens', lib.fptr(packed), lib.fptr(o_d), lib.fptr(d_d), lib.fptr(l_d), lat.data_ptr(), lat.stride(2),
             lat.shape[1], lat.shape[2], 512, img.data_ptr(), img.stride(2), img.shape[1], img.shape[2], 3, 1.0, lib.fptr(out), 608, V, NC, N, D, lib.stream())
    behind = outside = 0
    for v in range(V):
        cv = SimpleNamespace(R=cu(cams.R[v]), T=cu(cams.T[v]), focal_length=cu(cams.focal_length[v]), principal_point=cu(cams.principal_point[v]))
        ref, inv_z = _eager_t1(m, cv, cu(origins[v]), cu(directions[v]), cu(lengths[v]))
        got = out[:, v * N * D:(v + 1) * N * D]
        behind += int((inv_z < 0).sum())
        well_posed = inv_z.abs() < 100                  # projections of points within 1e-2 of a camera plane swing by more than float rounding
        assert well_posed.float().mean() > 0.95
        err_emb = (got[..., :91] - ref[..., :91]).abs().max().item()
        err_look = (got[..., 91:606] - ref[..., 91:606])[well_posed].abs().max().item()
        print(f'NC={NC} view {v}: embedding max abs err {err_emb:.2e}, look-ups max abs err {err_look:.2e}')
        assert err_emb < 2e-4 and err_look < 2e-4
        assert torch.equal(got[..., 606:], torch.zeros_like(got[..., 606:]))
        from sparsefusion_b200.eft import transform_points_ndc
        xyz = (cu(origins[v])[:, None, :] + cu(lengths[v])[:, :, None] * cu(directions[v])[:, None, :]).reshape(1, -1, 3)
        outside += int((transform_points_ndc(cv, xyz)[..., :2].abs() > 1).any(-1).sum())
    assert behind > 0 and outside > 0                                                   # both cases are exercised


def _rays_ring(n_views=5, NC=2):
    """query bundles and per-view input cameras as NativeSceneBuilder makes them for a ring of 8 scene cameras"""
    from sparsefusion_b200 import cameras as C
    cams = _ring(8)
    rel = C.relative_cameras(cams, [0], True)
    ctx_idx = [0, 3] if NC == 2 else [0, 1, 2, 4, 5, 7]
    views = [1, 3, 4, 6, 7][:n_views]
    per_view = [C.relative_cameras(rel, [ci], True) for ci in views]
    q_o, q_d = C.grid_rays(C.concat_cameras([pv[ci] for ci, pv in zip(views, per_view)]), 32, 32, 'cuda', 256, 256)
    cdm = float(cams.get_camera_center().norm(dim=1).mean())
    lengths = torch.linspace(cdm - 5.0, cdm + 5.0, 20, device='cuda').expand(len(views), 1024, 20)
    return q_o, q_d, lengths, [pv[ctx_idx] for pv in per_view], ctx_idx


@pytest.mark.parametrize('NC', [2, 6])
def test_feature_cache_against_per_view_forward(NC):
    from oracle import eft_oracle as eo
    m = _model()
    q_o, q_d, lengths, ctx, idx = _rays_ring(5, NC)
    images = torch.rand(NC, 3, 256, 256, generator=torch.Generator().manual_seed(7)).cuda()
    feats, rgb = m.feature_cache(q_o, q_d, lengths, ctx, images, (32, 32))
    assert feats.shape == (5, 256, 32, 32) and rgb.shape == (5, 3, 32, 32)
    for v in range(5):
        c = ctx[v]
        cams = eo.NdcCameras(c.R.cuda(), c.T.cuda(), c.focal_length.cuda(), c.principal_point.cuda())
        m.encode(cams, images)
        rb = eo.RayBundle(q_o[v].view(1, 32, 32, 3), q_d[v].view(1, 32, 32, 3), lengths[v].reshape(1, 32, 32, 20), None)
        r_rgb, r_f = m.batched_forward(rb, n_batches=16)[:2]
        e_f, e_rgb = _rel(feats[v], r_f[0].permute(2, 0, 1)), _rel(rgb[v], r_rgb[0].permute(2, 0, 1))
        print(f'NC={NC} view {v}: features rel {e_f:.2e}, rgb rel {e_rgb:.2e}')
        assert e_f < 1e-4 and e_rgb < 1e-4


def test_distillation_loop_with_native_scene_builder(tmp_path):
    """distillation_loop on a synthetic camera ring with no scene_builder stand-in: the native builder prepares the cache (58 EFT views),
    the evaluation views and the circle views; three iterations, then the checkpoint, the metrics file and the gifs"""
    import dataclasses
    from types import SimpleNamespace
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.distillation import NativeSceneBuilder, distillation_loop, get_default_torch_ngp_opt
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.vldm import DDPM
    cfg = dataclasses.replace(uo.SMALL, cond_images_channels=256, image_size=32)
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval()
    vae.load_state_dict(vo.make_params(seed=0, ch=32, ch_mult=(1, 2, 4, 4)))
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0))
    ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()
    cams = _ring(8)
    g = torch.Generator().manual_seed(3)
    rgb, mask = torch.rand(8, 3, 256, 256, generator=g), (torch.rand(8, 1, 256, 256, generator=g) > 0.5).float()
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    os.makedirs(f'{args.exp_dir}/log', exist_ok=True)
    out = tmp_path / 'out'
    seen = []
    torch.manual_seed(0)
    distillation_loop(0, args, get_default_torch_ngp_opt(), (_model(), vae.cuda(), ddpm), str(out), 'ring_000', cams, rgb, mask, None, [0, 4],
                      use_diffusion=True, max_itr=3, scene_builder=NativeSceneBuilder(0), seed=5, evaluate=True, visualize=True,
                      on_iteration=lambda itr, d: seen.append((itr, float(d.last['photo_loss']), float(d.last['fusion_loss']))))
    assert [s[0] for s in seen] == [0, 1, 2] and all(math.isfinite(s[1]) and math.isfinite(s[2]) for s in seen)
    assert 'model_state_dict' in torch.load(str(out / 'ring_000.pt'), map_location='cpu')
    assert (out / 'metrics' / 'ring_000.txt').stat().st_size > 0
    for f in ('ring_000.gif', 'ring_000_circle.gif'):
        assert (out / 'render_gifs' / f).stat().st_size > 0
    assert os.path.getsize(f'{args.exp_dir}/log/ring_000_eft_grid.jpg') > 0
