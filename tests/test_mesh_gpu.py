"""Mesh extraction on the GPU (csrc/mesh.cu, sparsefusion_b200/mesh.py, NeRFRenderer.export_mesh) against scipy / numpy and the oracle's
restatement of the marching-cubes contract (oracle/mesh_oracle.py).

Bars: smoothing within 1e-6 x max |v| of scipy.ndimage.gaussian_filter in float64 (fp32 taps and accumulation); mean / std within 1e-9
relative of numpy (fp64 accumulation); marching cubes on the same fp32 volume and isovalue: equal counts, equal triangles (the order is part
of the contract), vertices within 1e-5 index units, bit-identical repeats.  The fp32 pipeline is checked stage by stage, never against an
fp64 pipeline in one step: a corner within rounding of the isovalue may legitimately land on the other side.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


@pytest.mark.parametrize('sigma', [0.7, 1.5, 3.0])
@pytest.mark.parametrize('shape', [(37, 41, 53), (3, 5, 64), (64, 2, 7), (1, 9, 4), (16, 16, 300)])
def test_smoothing_and_statistics_match_scipy_numpy(shape, sigma):
    from scipy import ndimage
    from sparsefusion_b200 import mesh
    rng = np.random.default_rng(sum(shape))
    v = (rng.standard_normal(shape) * 3 + 1).astype(np.float32)
    got = mesh.smooth_gaussian(torch.from_numpy(v).cuda(), sigma).cpu().numpy()
    want = ndimage.gaussian_filter(v.astype(np.float64), sigma)
    err = np.abs(got - want).max()
    print(f'  {shape} sigma {sigma}: max abs err {err:.2e} (max |v| {np.abs(v).max():.2f})')
    assert err <= 1e-6 * np.abs(v).max(), err
    mean, std = mesh.volume_mean_std(torch.from_numpy(got).cuda())
    g64 = got.astype(np.float64)
    assert abs(mean - g64.mean()) <= 1e-9 * abs(g64.mean()) and abs(std - g64.std()) <= 1e-9 * g64.std(), (mean, std, g64.mean(), g64.std())


def _check_mc(vol, iso):
    from oracle import mesh_oracle as mo
    from sparsefusion_b200 import mesh
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    iso = float(np.float32(iso))
    vd = torch.from_numpy(vol).cuda()
    verts, tris = mesh.marching_cubes(vd, iso)
    wv, wt = mo.marching_cubes(vol, iso)
    assert verts.shape == (len(wv), 3) and tris.shape == (len(wt), 3) and tris.dtype == torch.int32
    assert (tris.cpu().numpy() == wt).all()
    if len(wv):
        assert np.abs(verts.cpu().numpy() - wv).max() < 1e-5
    v2, t2 = mesh.marching_cubes(vd, iso)
    assert torch.equal(verts, v2) and torch.equal(tris, t2)
    return verts, tris


def test_marching_cubes_matches_oracle():
    from oracle import mesh_oracle as mo
    rng = np.random.default_rng(7)
    v, t = _check_mc(rng.standard_normal((37, 41, 53)), 0.1)                      # every case, open at the lattice boundary
    assert len(t) > 10000
    v, t = _check_mc(mo.sphere(64, 20.0), 0.0)
    assert mo.euler_characteristic(v.cpu().numpy(), t.cpu().numpy()) == 2
    assert mo.signed_volume(v.cpu().numpy(), t.cpu().numpy()) > 0
    v, t = _check_mc(mo.torus(64, 16.0, 6.0), 0.0)
    assert mo.euler_characteristic(v.cpu().numpy(), t.cpu().numpy()) == 0
    ivol = rng.integers(0, 5, (19, 23, 29)).astype(np.float32)                   # many corners equal iso: pins `below` = v <= iso
    v, t = _check_mc(ivol, 2.0)
    assert (v.cpu().numpy() == np.round(v.cpu().numpy())).all(axis=1).any()
    for vol in (np.full((9, 10, 11), -1.0), np.full((9, 10, 11), 0.5), np.full((1, 1, 1), 0.0), rng.standard_normal((1, 6, 7))):
        v, t = _check_mc(vol, 0.5 if vol.size > 1 else 0.0)
        if vol.shape[0] > 1:
            assert v.shape == (0, 3) and t.shape == (0, 3)
        else:
            assert t.shape == (0, 3)                                                # no cells: vertices but no faces
    with pytest.raises(RuntimeError, match='outside'):
        from sparsefusion_b200 import mesh
        mesh.marching_cubes(torch.zeros(1025, 2, 2, device='cuda'), 0.0)


def _net(cuda_ray, seed=0):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = cuda_ray
    net = NeRFNetwork(opt)
    p = no.make_field_params(seed=seed)
    sd = net.state_dict()
    for k, v in p.items():
        sd[k] = v
    net.load_state_dict(sd)
    return net.cuda().eval(), p


@pytest.mark.parametrize('cuda_ray', [False, True], ids=['default', 'cuda_ray'])
@pytest.mark.parametrize('R', [48, 128])
def test_export_mesh_stage_by_stage(R, cuda_ray, tmp_path):
    from _helpers import device_level_scales
    from oracle import mesh_oracle as mo, ngp_oracle as no
    from sparsefusion_b200 import mesh
    from scipy import ndimage
    net, p = _net(cuda_ray)
    verts_w, tris = net.export_mesh(str(tmp_path), grid_resolution=R, S=20)      # slabs that do not divide R
    # density lattice: linspace(-bound, bound, R), indexing 'ij'
    sigma = mesh.density_lattice(net, R, S=128)
    if R == 48:
        lin = torch.linspace(-4, 4, R)
        xx, yy, zz = torch.meshgrid(lin, lin, lin, indexing='ij')
        pts = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1)
        field = no.Field({k: v.clone() for k, v in p.items()}, level_scales=device_level_scales(no.live_geometry()))
        with torch.no_grad():
            so, _ = field.common_forward(pts)
        r = _rel(sigma.reshape(-1), so)
        print(f'  density lattice {R}^3 vs oracle: rel {r:.2e}')
        assert r < 2e-4
    # smoothing, statistics, marching cubes, each on the previous stage's GPU output
    smooth = mesh.smooth_gaussian(sigma, 1.5)
    s64 = sigma.cpu().double().numpy()
    want = ndimage.gaussian_filter(s64, 1.5)
    assert np.abs(smooth.cpu().numpy() - want).max() <= 1e-6 * np.abs(s64).max()
    mean, std = mesh.volume_mean_std(smooth)
    g64 = smooth.cpu().double().numpy()
    assert abs(mean - g64.mean()) <= 1e-9 * abs(g64.mean()) and abs(std - g64.std()) <= 1e-9 * g64.std()
    iso = mean + 0.25 * std
    verts, t2 = _check_mc(smooth.cpu().numpy(), iso)
    assert len(t2) > 0
    # export_mesh ran the same stages: identical mesh, world mapping v / (R-1) * 2 bound - bound
    assert torch.equal(tris, t2)
    assert torch.allclose(verts_w, verts / (R - 1) * 8.0 - 4.0, rtol=0, atol=1e-6)
    ov, ot = mo.read_obj(str(tmp_path / 'mcubes_mesh.obj'))
    assert (ot == tris.cpu().numpy()).all()
    undone = (verts_w.cpu().double().numpy() + 4.0) / 8.0 * (R - 1)
    assert np.abs(ov - undone).max() < 2e-5 * R
    assert np.abs(ov - verts.cpu().double().numpy()).max() <= 5e-7 + 1e-9


def test_cli_on_a_distilled_checkpoint(tmp_path):
    """checkpoint of 3 distillation iterations on the reduced scene (as tests/test_distillation_gpu.py makes it), then
    `python -m sparsefusion_b200.mesh CKPT OUT_DIR`; the initial density blob (network_grid.gaussian) gives a closed surface around the origin"""
    from types import SimpleNamespace
    from oracle import distill_oracle as do, mesh_oracle as mo, unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.distillation import SceneCache, distillation_loop, get_default_torch_ngp_opt
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.vldm import DDPM
    cfg = uo.SMALL
    scene = do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=cfg.cond_images_channels, render_hw=64, seed=3)
    vae = AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval()
    vae.load_state_dict(vo.make_params(seed=0, ch=32, ch_mult=(1, 2, 4, 4)))
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    unet.load_state_dict(uo.make_params(cfg, seed=0))
    ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()

    class Builder:
        def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
            return SceneCache(**scene)
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'), category='hydrant')
    distillation_loop(0, args, get_default_torch_ngp_opt(), ('eft-model', vae.cuda(), ddpm), str(tmp_path / 'out'), 'hydrant_000_c2', None,
                      scene['input_rgb'], scene['input_mask'], None, [0, 1], use_diffusion=True, max_itr=3, loss_fn_vgg=None, scene_builder=Builder(),
                      seed=5)
    ckpt = tmp_path / 'out' / 'hydrant_000_c2.pt'
    assert ckpt.exists()
    out = tmp_path / 'mesh'
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'sparsefusion_b200.mesh', str(ckpt), str(out)], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=600)
    print(r.stdout, r.stderr[-2000:])
    assert r.returncode == 0
    verts, tris = mo.read_obj(str(out / 'mcubes_mesh.obj'))
    print(f'  CLI mesh: {len(verts)} vertices, {len(tris)} triangles, index-unit bbox {verts.min(0)} .. {verts.max(0)}')
    assert len(tris) > 0 and tris.max() < len(verts)
    assert mo.euler_characteristic(verts, tris) == 2 and mo.signed_volume(verts, tris) > 0
    centre = verts.mean(0) / 127 * 8 - 4                                        # world units: the blob sits at the origin
    assert np.abs(centre).max() < 0.5, centre
