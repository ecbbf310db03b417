"""The entropy regulariser, the on-device loss history and the periodic progress outputs on the GPU.

(1) sfb_photometric_loss_ent / sfb_fusion_loss_ent per element against fp64 autograd of the reference's expressions (distillation.py:210-241,
    :287-344), with oracle/step_fp64.py's bounds for the existing terms and the entropy term's own; silhouettes hold exactly 0, 1e-5,
    1 - 1e-5 and 1, and the gradient is exactly 0 where the clamp moves the silhouette;
(2) at lambda_entropy 0 the new kernels give the old ones' gradients bit for bit (and sums, where one block makes them deterministic), and
    the Python path launches only the old kernels;
(3) Distiller.step with lambda_entropy 1e-2: fused glue against the reference's torch expressions (fused_glue=False) with the same injected
    draws, both phases; MultiSceneDistiller against per-scene Distillers; the view-batched step against its per-view terms;
(4) the history against the reference's .item() values, recorded without a host synchronisation;
(5) a progress write changes nothing the next step reads (bit for bit), a loop with progress outputs draws what one without them draws
    (bit for bit, every iteration), and the history's rows survive a checkpoint bit for bit.
"""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LE = 1e-2
SPECIAL = (0.0, float(np.float32(1e-5)), float(np.float32(1 - 1e-5)), 1.0)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


# ---------------------------------------------------------------------------------------------------- (1), (2) kernels
def _with_specials(s, g):
    """silhouette values in (0, 1), a sixteenth of them replaced by exactly 0, 1e-5, 1 - 1e-5 and 1 (fp32)"""
    s = s.clone()
    k = torch.arange(s.numel(), device=s.device)
    for j, v in enumerate(SPECIAL):
        s.view(-1)[k % 64 == j] = v
    return s


def _entropy_ref(sil, le, n):
    """fp64 autograd of the reference's entropy term (:238-241) summed: (sum H, d(le * mean H)/d sil) with per-element bounds"""
    from oracle.field_fp64 import ATOL, gamma
    s = sil.double().cpu().reshape(-1).clone().requires_grad_(True)
    a = s.clamp(SPECIAL[1], SPECIAL[2])
    h = -a * torch.log2(a) - (1 - a) * torch.log2(1 - a)
    (le * h.sum() / n).backward()
    ad = a.detach()
    l0, l1 = torch.log2(ad).abs(), torch.log2(1 - ad).abs()
    # log2f is within an ulp; 1 - a rounds once (u / ln 2 absolute in its log); the product, difference and scaling round a few times more
    hb = ad * l0 + (1 - ad) * l1 + 1
    gb = gamma(12) * le * (l0 + l1 + 1) / n + ATOL
    return h.detach().sum(), hb.sum(), s.grad, gb


def _rand(g, *shape):
    return torch.rand(*shape, generator=g, device='cuda')


@pytest.mark.parametrize('hw', [64, 128])
def test_photometric_loss_ent_against_fp64(hw):
    from oracle import step_fp64 as sp
    from oracle.field_fp64 import ATOL, gamma
    from sparsefusion_b200 import _lib as lib
    g = torch.Generator(device='cuda').manual_seed(hw)
    n, scale, lam = hw * hw, 2, (1.0, 0.7, 1e-3)
    img, sil = _rand(g, n, 3), _with_specials(_rand(g, n), g)
    rgb, mask = _rand(g, 3, hw * scale, hw * scale), (_rand(g, 1, hw * scale, hw * scale) > 0.5).float()
    sums, gi, gs = torch.full((4,), np.nan, device='cuda'), torch.empty(n, 3, device='cuda'), torch.empty(n, device='cuda')
    lib.call('sfb_photometric_loss_ent', lib.fptr(img), lib.fptr(sil), lib.fptr(rgb), lib.fptr(mask), hw, hw, scale, *lam, LE, lib.fptr(sums),
             lib.fptr(gi), lib.fptr(gs), lib.stream())
    torch.cuda.synchronize()
    plan = sp.kernel_plan('photometric_loss', dict(h=hw, w=hw), torch.cuda.get_device_properties(0).multi_processor_count)
    r = sp.ref_photometric(img, sil, rgb, mask, hw, hw, scale, *lam, plan)
    hs, hsa, hg, hgb = _entropy_ref(sil, LE, n)
    ref_sums = torch.cat((r['sums'][0], hs[None]))
    bnd_sums = torch.cat((r['sums'][1], (gamma(sp.sum_chain(plan) + 12) * hsa + ATOL)[None]))
    want_gs = r['g_sil'][0] + hg
    assert sp.passes(sums, ref_sums, bnd_sums), (sums, ref_sums)
    assert sp.passes(gi, *r['g_img'])
    assert sp.passes(gs, want_gs, r['g_sil'][1] + hgb), sp.compare(gs, want_gs, r['g_sil'][1] + hgb)
    # at the clamped elements (0 and 1) the entropy adds nothing: the gradient is the old kernel's, bit for bit
    old = torch.empty_like(gs)
    lib.call('sfb_photometric_loss', lib.fptr(img), lib.fptr(sil), lib.fptr(rgb), lib.fptr(mask), hw, hw, scale, *lam, lib.fptr(sums),
             lib.fptr(torch.empty_like(gi)), lib.fptr(old), lib.stream())
    torch.cuda.synchronize()
    clamped = (sil < SPECIAL[1]) | (sil > SPECIAL[2])
    assert int(clamped.sum()) >= 2 * n // 64 and torch.equal(gs[clamped], old[clamped])     # torch.rand may add a few of its own
    assert (hg[clamped.cpu()] == 0).all()
    loss, _, _, terms = _glue_photometric(img, sil, rgb, mask, hw, scale, lam)
    want = lam[0] * ref_sums[0] / (3 * n) + lam[1] * ref_sums[1] / n + lam[2] * ref_sums[2] / n + LE * hs / n
    assert abs(loss.item() - want.item()) < 1e-5 * abs(want.item())
    assert abs(terms[2].item() - LE * hs.item() / n) < 1e-5 * LE * hs.item() / n and abs(terms[0].item() - loss.item()) == 0


def _glue_photometric(img, sil, rgb, mask, hw, scale, lam, le=LE):
    from sparsefusion_b200 import image_glue as glue
    return glue.photometric_loss(img, sil, rgb, mask, hw, hw, scale, *lam, lambda_entropy=le, return_terms=True)


@pytest.mark.parametrize('g_extra', [False, True], ids=['plain', 'g_extra'])
@pytest.mark.parametrize('mode', [0, 1], ids=['sds', 'eft'])
@pytest.mark.parametrize('hw', [64, 128])
def test_fusion_loss_ent_against_fp64(hw, mode, g_extra):
    from oracle import step_fp64 as sp
    from oracle.field_fp64 import ATOL, gamma
    from sparsefusion_b200 import _lib as lib
    g = torch.Generator(device='cuda').manual_seed(7 * hw + mode)
    H = W = 2 * hw
    HW = H * W
    lam, wgt = (1.0, 0.7, 1e-3), 0.37
    up = _rand(g, 4, H, W)
    up[3] = _with_specials(up[3], g)
    target = _rand(g, 3, H, W) * 0.3
    ge = (_rand(g, 3, H, W) - 0.5) * 1e-4 if g_extra else None
    sums, gu = torch.full((4,), np.nan, device='cuda'), torch.empty(4, H, W, device='cuda')
    gi, gs = torch.empty(hw * hw, 3, device='cuda'), torch.empty(hw * hw, device='cuda')
    lib.call('sfb_fusion_loss_ent', lib.fptr(up), lib.fptr(target), H, W, mode, wgt, *lam, LE, None if ge is None else lib.fptr(ge), lib.fptr(sums),
             lib.fptr(gu), hw, hw, lib.fptr(gi), lib.fptr(gs), lib.stream())
    torch.cuda.synchronize()
    plan = sp.kernel_plan('fusion_loss', dict(h=hw, w=hw), torch.cuda.get_device_properties(0).multi_processor_count)
    r = sp.ref_fusion(up, target, mode, wgt, *lam, ge, plan)
    hs, hsa, hg, hgb = _entropy_ref(up[3], LE, HW)
    ref_sums = torch.cat((r['sums'][0], hs[None]))
    bnd_sums = torch.cat((r['sums'][1], (gamma(sp.sum_chain(plan) + 12) * hsa + ATOL)[None]))
    want_gu, bnd_gu = r['g_up'][0].clone(), r['g_up'][1].clone()
    want_gu[3] += hg.view(H, W)
    bnd_gu[3] += hgb.view(H, W)
    assert sp.passes(sums, ref_sums, bnd_sums), (sums, ref_sums)
    assert sp.passes(gu, want_gu, bnd_gu), sp.compare(gu, want_gu, bnd_gu)
    (gi_r, gs_r) = sp.ref_fusion_adjoint(gu, hw, hw)
    assert sp.passes(gi, *gi_r) and sp.passes(gs, *gs_r)
    clamped = (up[3] < SPECIAL[1]) | (up[3] > SPECIAL[2])
    old = torch.empty_like(gu)
    lib.call('sfb_fusion_loss_ex', lib.fptr(up), lib.fptr(target), H, W, mode, wgt, *lam, None if ge is None else lib.fptr(ge), lib.fptr(sums),
             lib.fptr(old), hw, hw, lib.fptr(torch.empty_like(gi)), lib.fptr(torch.empty_like(gs)), lib.stream())
    torch.cuda.synchronize()
    assert int(clamped.sum()) >= 2 * HW // 64 and torch.equal(gu[3][clamped], old[3][clamped])


@pytest.mark.parametrize('hw', [8, 16, 64])
def test_entropy_kernels_at_zero_weight_equal_the_old_kernels(hw, monkeypatch):
    """lambda_entropy 0 through the new entry points: the old kernels' gradients bit for bit, and their sums bit for bit where one block
    computes them (hw 8 fusion / 16 photometric); more blocks add their partial sums with atomics, in no fixed order"""
    from sparsefusion_b200 import _lib as lib, image_glue as glue
    g = torch.Generator(device='cuda').manual_seed(hw)
    n, lam = hw * hw, (1.0, 0.7, 1e-3)
    img, sil = _rand(g, n, 3), _with_specials(_rand(g, n), g)
    rgb, mask = _rand(g, 3, 2 * hw, 2 * hw), (_rand(g, 1, 2 * hw, 2 * hw) > 0.5).float()
    outs = []
    for name, extra in (('sfb_photometric_loss', ()), ('sfb_photometric_loss_ent', (0.0,))):
        s, gi, gs = torch.zeros(4, device='cuda'), torch.empty(n, 3, device='cuda'), torch.empty(n, device='cuda')
        lib.call(name, lib.fptr(img), lib.fptr(sil), lib.fptr(rgb), lib.fptr(mask), hw, hw, 2, *lam, *extra, lib.fptr(s), lib.fptr(gi), lib.fptr(gs),
                 lib.stream())
        outs.append((s[:3].clone(), gi, gs))
    (s0, gi0, gs0), (s1, gi1, gs1) = outs
    assert torch.equal(gi0, gi1) and torch.equal(gs0, gs1)
    assert torch.equal(s0, s1) if n <= 256 else _rel(s1, s0) < 1e-6
    up, target = glue.upsample2x_render(img, sil, hw, hw), _rand(g, 3, 2 * hw, 2 * hw) * 0.3
    for mode in (0, 1):
        outs = []
        for name, extra in (('sfb_fusion_loss_ex', ()), ('sfb_fusion_loss_ent', (0.0,))):
            s, gu = torch.zeros(4, device='cuda'), torch.empty_like(up)
            gi, gs = torch.empty(n, 3, device='cuda'), torch.empty(n, device='cuda')
            lib.call(name, lib.fptr(up), lib.fptr(target), 2 * hw, 2 * hw, mode, 0.37, *lam, *extra, None, lib.fptr(s), lib.fptr(gu), hw, hw,
                     lib.fptr(gi), lib.fptr(gs), lib.stream())
            outs.append((s[:3].clone(), gu, gi, gs))
        for a, b in zip(outs[0][1:], outs[1][1:]):
            assert torch.equal(a, b), mode
        assert torch.equal(outs[0][0], outs[1][0]) if 4 * n <= 256 else _rel(outs[1][0], outs[0][0]) < 1e-6
    # the Python path at lambda_entropy 0 launches only the old kernels, with or without the logged terms
    called = []
    real = lib.call
    monkeypatch.setattr(lib, 'call', lambda name, *a: called.append(name) or real(name, *a))
    for rt in (False, True):
        glue.photometric_loss(img, sil, rgb, mask, hw, hw, 2, *lam, lambda_entropy=0.0, return_terms=rt)
        glue.fusion_loss(up, target, hw, hw, 'eft', 1.0, *lam, lambda_entropy=0.0, return_terms=rt)
    assert not [c for c in called if c.endswith('_ent')] and called.count('sfb_photometric_loss') == 2


# ---------------------------------------------------------------------------------------------------- (3), (4) steps and history
def _small_models():
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
    return vae.cuda(), ddpm


_MODELS, _CACHES = [None], {}


def _models():
    if _MODELS[0] is None:
        _MODELS[0] = _small_models()
    return _MODELS[0]


def _scene(k):
    from oracle import distill_oracle as do, unet_oracle as uo
    return do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels, render_hw=64, seed=3 + k)


def _cache(k):
    from sparsefusion_b200.distillation import SceneCache
    if k not in _CACHES:
        _CACHES[k] = SceneCache(**_scene(k)).to('cuda')
    return _CACHES[k]


def _ngp(k):
    from oracle import ngp_oracle as no
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    ngp = NeRFNetwork(get_default_torch_ngp_opt())
    st = ngp.state_dict()
    st.update(no.make_field_params(seed=k))
    ngp.load_state_dict(st)
    return ngp.cuda().train()


def _draws(k, n_rays=64 * 64):
    rng = np.random.default_rng(21 + k)
    return {w: (torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda(), torch.from_numpy(rng.random((n_rays, 64), dtype=np.float32)).cuda())
            for w in 'AB'}


def _distiller(k, itr, fused_glue=True, **kw):
    from oracle import unet_oracle as uo
    from sparsefusion_b200.distillation import Distiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    vae, ddpm = _models()
    d = Distiller(_ngp(k), vae, ddpm, get_default_torch_ngp_opt(), _cache(k), seed=11 + k, fused_glue=fused_glue, lambda_entropy=LE, **kw)
    draws = _draws(k)
    src = uo.NoiseSource(seed=50 + k)
    d.sampler.noise_fn = lambda t: src(t.cpu()).to(t.device)
    d.render_noise = lambda w: draws[w]
    return d


@pytest.mark.parametrize('itr', [5, 1500])
def test_fused_entropy_step_matches_the_reference_expressions(itr):
    mt = 0.13 if itr > 1000 else None
    eager = _distiller(0, itr, fused_glue=False)
    ea, eb = eager.step(itr, max_thres=mt)
    fused = _distiller(0, itr)
    fa, fb = fused.step(itr, max_thres=mt)
    ra, rb = abs(fa.item() - ea.item()) / abs(ea.item()), abs(fb.item() - eb.item()) / abs(eb.item())
    rp = _rel(fused.optimizer.flat, eager.optimizer.flat)
    rh = (fused.history[itr] - eager.history[itr]).abs() / eager.history[itr].abs()
    print(f'itr {itr}: losses {fa.item():.6f}/{ea.item():.6f} {fb.item():.6f}/{eb.item():.6f} (rel {ra:.1e}, {rb:.1e}); parameters rel {rp:.2e}; '
          f'history rel {rh.tolist()}')
    assert ra < 1e-5 and rb < 1e-5 and rp < 1e-4
    assert (rh < 1e-5).all() and fused.history[itr, 2] > 0
    # the entropy term moves the step: the same step without it ends elsewhere
    plain = _distiller(0, itr)
    plain.lambda_entropy = 0.0
    plain.step(itr, max_thres=mt)
    assert _rel(plain.optimizer.flat, fused.optimizer.flat) > 10 * rp


def test_multiscene_entropy_step_matches_per_scene_distillers():
    from oracle import unet_oracle as uo
    from sparsefusion_b200.distillation import MultiSceneDistiller
    from sparsefusion_b200.network_grid import get_default_torch_ngp_opt
    itr, S = 1500, 2
    ref = []
    for k in range(S):
        d = _distiller(k, itr)
        la, lb = d.step(itr)
        ref.append((la.item(), lb.item(), d.optimizer.flat.clone(), d.history[itr].clone()))
    vae, ddpm = _models()
    msd = MultiSceneDistiller([_ngp(k) for k in range(S)], vae, ddpm, get_default_torch_ngp_opt(), [_cache(k) for k in range(S)],
                              seeds=[11 + k for k in range(S)], lambda_entropy=LE)
    draws = [_draws(k) for k in range(S)]
    srcs = [uo.NoiseSource(seed=50 + k) for k in range(S)]
    msd.render_noise = lambda k, w: draws[k][w]
    msd.plms_noise = lambda k: (lambda t: srcs[k](t.cpu()).to(t.device))
    la, lb = msd.step(itr)
    for k in range(S):
        sa, sb, flat, hist = ref[k]
        rp = _rel(msd.scenes[k].optimizer.flat, flat)
        ra, rb = abs(la[k].item() - sa) / abs(sa), abs(lb[k].item() - sb) / abs(sb)
        print(f'scene {k}: loss rel {ra:.1e} {rb:.1e}; parameters rel {rp:.2e}')
        assert ra < 1e-5 and rb < 1e-5 and rp < 1e-4
        assert _rel(msd.history[k][itr], hist) < 1e-5


def test_view_batched_entropy_step_matches_its_per_view_terms():
    """minibatch_step's loss and history against the photometric term plus the mean of the per-view fusion terms, each evaluated alone
    through the eager reference expressions (bootstrap phase: no sampled target)"""
    import torch.nn.functional as F
    from sparsefusion_b200.distillation import huber, step_views
    itr, V = 5, 3
    d = _distiller(0, itr, views_per_step=V)
    d.render_noise_keyed = lambda w, view: _draws(0)[w]
    la, lb = d.minibatch_step(itr)
    c = d.cache
    g = torch.Generator().manual_seed(d.seed)
    idx = int(torch.randperm(c.input_rgb.shape[0], generator=g)[0])
    views = step_views(torch.randperm(c.target_features.shape[0], generator=g), V)
    e = _distiller(0, itr, fused_glue=False)
    with torch.no_grad():
        dr = _draws(0)
        img, sil = e._render_nchw(c.input_rays_o[idx], c.input_rays_d[idx], dr['A'])
        rgb, mask = F.interpolate(c.input_rgb[idx:idx + 1], scale_factor=0.5), F.interpolate(c.input_mask[idx:idx + 1], scale_factor=0.5)
        a = sil.clamp(1e-5, 1 - 1e-5)
        ent = (-a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean()
        opac = torch.sqrt(sil ** 2 + .01).mean()
        pa = huber(img, rgb).abs().mean() + huber(sil, mask).abs().mean() + 1e-3 * opac + LE * ent
        fb, lv = 0.0, 0.0
        for v in views:
            img, sil = e._render_nchw(c.target_rays_o[v], c.target_rays_d[v], dr['B'])
            img, sil = F.interpolate(img, scale_factor=2, mode='bilinear'), F.interpolate(sil, scale_factor=2, mode='bilinear')
            t = c.target_eft_image[v:v + 1]
            f = huber(img, t).abs().mean() + huber(sil, (t.mean(dim=1, keepdim=True) > .1).float()).abs().mean()
            a = sil.clamp(1e-5, 1 - 1e-5)
            lv = lv + (f + 1e-3 * torch.sqrt(sil ** 2 + .01).mean() + LE * (-a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean()) / V
            fb = fb + f / V
    want = torch.stack((pa, 1e-3 * opac, LE * ent, fb))
    print(f'minibatch: losses {la.item():.6f}/{pa.item():.6f} {lb.item():.6f}/{lv.item():.6f}; history {d.history[itr].tolist()} vs {want.tolist()}')
    assert abs(la.item() - pa.item()) < 1e-5 * abs(pa.item()) and abs(lb.item() - lv.item()) < 1e-5 * abs(lv.item())
    assert _rel(d.history[itr], want) < 1e-5


def test_history_equals_the_reference_item_values_without_a_sync():
    """N reference steps record, per row, what the reference's .item() calls log (:249-256, :349) -- recomputed here through the eager
    path on the same parameters and draws -- and recording raises nothing under sync debug mode 'error'"""
    N = 4
    fused, eager = _distiller(0, 0), _distiller(0, 0, fused_glue=False)
    for itr in range(N):
        eager.step(itr)
        fused.step(itr)
    assert fused.history.shape == (N, 4) and eager.history.shape == (N, 4)
    rel = ((fused.history - eager.history).abs() / eager.history.abs()).max().item()
    print(f'history after {N} steps: {fused.history.tolist()}; fused vs eager max rel {rel:.2e}')
    assert torch.isfinite(fused.history).all() and rel < 1e-4
    # recording alone: the step's term copies, with sync debug mode raising on any synchronising call
    terms = torch.arange(4.0, device='cuda')
    torch.cuda.set_sync_debug_mode('error')
    try:
        fused._record(N, 0, terms[:3])
        fused._record(N, 3, terms[3])
        fused._record(fused._history.shape[0] + 5, 0, terms)       # past the preallocated rows: the buffer grows on the device
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert fused._history[N].tolist() == [0.0, 1.0, 2.0, 3.0]


# ---------------------------------------------------------------------------------------------------- (5) progress outputs
class _Builder:
    """scene k of ``_scene`` with 256 x 256 eval views: the input views' 64 x 64 ray grids up-sampled"""

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        from sparsefusion_b200.distillation import SceneCache
        return SceneCache(**_scene(scene_cameras))

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        import torch.nn.functional as F
        from sparsefusion_b200.evaluate import EvalViews
        s = _scene(scene_cameras)
        up = lambda r: F.interpolate(r.reshape(-1, 64, 64, 3).permute(0, 3, 1, 2), size=(256, 256), mode='bilinear').permute(0, 2, 3, 1).reshape(-1, 256 * 256, 3)
        return EvalViews(rays_o=up(s['input_rays_o']).contiguous(), rays_d=up(s['input_rays_d']).contiguous(),
                         rgb=F.interpolate(s['input_rgb'], size=(256, 256), mode='bilinear'), mask=F.interpolate(s['input_mask'], size=(256, 256)))


class _Stop(Exception):
    pass


def _loop(out, scenes, n, *, progress_every=None, checkpoint_every=None, resume=False, stop=None, seen=None):
    """distillation_loop (scenes None) or distill_scenes over ``scenes`` scenes for n iterations; returns (in ``seen``, also filled when the
    run is stopped after iteration ``stop``) the networks' flat parameters and Adam moments, each iteration's generator states and the
    history after every iteration"""
    from sparsefusion_b200.distillation import distill_scenes, distillation_loop, get_default_torch_ngp_opt
    vae, ddpm = _models()
    seen = {} if seen is None else seen
    seen.update(states=[], hist={}, moments=None)

    def on_iteration(itr, dist):
        ds = list(getattr(dist, 'scenes', [dist]))
        seen['states'].append((itr, torch.get_rng_state(), torch.cuda.get_rng_state(), [d.gen.get_state() for d in ds]))
        seen['hist'][itr] = [d.history.clone() for d in ds]
        if itr == n - 1:
            seen['moments'] = torch.cat([torch.cat((d.optimizer.flat, d.optimizer.m, d.optimizer.v)) for d in ds]).cpu()
        if itr == stop:
            raise _Stop()
    args = SimpleNamespace(exp_dir=os.path.join(out, 'exp'))
    kw = dict(max_itr=n, on_iteration=on_iteration, scene_builder=_Builder(), seed=5, lambda_entropy=LE, progress_every=progress_every,
              checkpoint_every=checkpoint_every, resume=resume)
    torch.manual_seed(0)
    if scenes is None:
        distillation_loop(0, args, get_default_torch_ngp_opt(), ('eft', vae, ddpm), out, 'scene_000', 0, None, None, None, [0, 1], **kw)
    else:
        distill_scenes(0, args, get_default_torch_ngp_opt(), ('eft', vae, ddpm), out, [(f'scene_{k:03d}', k, None, None, None, [0, 1])
                                                                                      for k in range(scenes)], **kw)
    return seen


@pytest.mark.timeout(1500)
@pytest.mark.parametrize('scenes', [None, 2], ids=['distillation_loop', 'distill_scenes'])
def test_progress_outputs_leave_the_run_unchanged(scenes, tmp_path):
    from PIL import Image
    n = 41
    off = _loop(str(tmp_path / 'off'), scenes, n)
    on = _loop(str(tmp_path / 'on'), scenes, n, progress_every=20)
    # the draws: every iteration's global CPU / CUDA generator states and permutation generators, bit for bit
    assert len(on['states']) == len(off['states']) == n
    for a, b in zip(on['states'], off['states']):
        assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and all(torch.equal(x, y) for x, y in zip(a[3], b[3]))
    # parameters and Adam moments differ only by the field backward's atomics, which no fixed bound separates from a perturbation over 41
    # iterations: printed here, and the state the next step reads is checked bit for bit around one write below
    print(f'{scenes or 1} scene(s), {n} iterations: parameters and moments, progress on vs off: rel {_rel(on["moments"], off["moments"]):.3e}')
    names = ['scene_000'] if scenes is None else [f'scene_{k:03d}' for k in range(scenes)]
    for name in names:
        log = tmp_path / 'on' / 'exp' / 'log'
        for f, size in ((f'{name}_loss.jpg', (640, 480)), (f'{name}_fusionloss.jpg', (640, 480)), (f'{name}_vis.jpg', (512, 256))):
            with Image.open(log / f) as im:
                assert im.size == size, (f, im.size)
        assert not (tmp_path / 'off' / 'exp' / 'log' / f'{name}_vis.jpg').exists()


def _step_state(d):
    """everything of Distiller d the next step reads, plus the process's global generators, as host copies"""
    n, o = d.ngp, d.optimizer
    out = dict(flat=o.flat, grad=o.grad, m=o.m, v=o.v, t=o.t, sched=o.sched, gen=d.gen.get_state(), history=d._history, next_itr=d.next_itr,
               training=n.training, cpu_rng=torch.get_rng_state(), cuda_rng=torch.cuda.get_rng_state())
    out.update({f'ngp.{k}': t for k, t in n.state_dict(keep_vars=True).items()})
    out.update({f'ngp.{k}': getattr(n, k) for k in ('mean_density', 'iter_density', 'mean_count', 'local_step') if hasattr(n, k)})
    return {k: v.detach().cpu().clone() if isinstance(v, torch.Tensor) else v for k, v in out.items()}


def _bits(t):
    return t.contiguous().reshape(-1).view(torch.uint8)          # bitwise: nan rows of the history compare equal to themselves


def _same_state(a, b):
    assert set(a) == set(b)
    bad = [k for k in a if not (a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and torch.equal(_bits(a[k]), _bits(b[k]))
                                if isinstance(a[k], torch.Tensor) else a[k] == b[k])]
    assert not bad, bad


@pytest.mark.parametrize('mode', ['reference-cuda_ray', 'multi2'])
def test_a_progress_write_changes_no_state_a_step_reads(mode, tmp_path):
    """``ProgressWriter.write`` between two steps: the networks (parameters, buffers, the cuda_ray density grid and counters, train mode),
    Adam's flat buffers and counts, the permutation generators, the histories and the global CPU and CUDA generators are bitwise the
    same after it as before -- for the reference step, whose renders draw from the global generators, and for scene-batched scenes"""
    from PIL import Image
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, _view_rows
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.progress import ProgressWriter
    vae, ddpm = _models()
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = mode == 'reference-cuda_ray'
    torch.manual_seed(0)
    if mode == 'multi2':
        dist = MultiSceneDistiller([NeRFNetwork(opt).cuda().train() for _ in range(2)], vae, ddpm, opt, [_cache(k) for k in range(2)],
                                   seeds=[11, 12], lambda_entropy=LE, max_itr=8)
    else:
        dist = Distiller(NeRFNetwork(opt).cuda().train(), vae, ddpm, opt, _cache(0), seed=11, lambda_entropy=LE, max_itr=8)
    scenes = list(getattr(dist, 'scenes', [dist]))
    views = [_view_rows(_Builder().eval_views(k, None, None), [0, 1]).to('cuda') for k in range(len(scenes))]
    w = ProgressWriter(str(tmp_path), [f's{k}' for k in range(len(scenes))], views, [[0, 1]] * len(scenes), opt)
    for itr in range(3):
        dist.step(itr)
    torch.cuda.synchronize()
    before = [_step_state(d) for d in scenes]
    w.write(2, scenes)
    torch.cuda.synchronize()
    for b, d in zip(before, scenes):
        _same_state(b, _step_state(d))
    with Image.open(tmp_path / 'log' / 's0_vis.jpg') as im:
        assert im.size == (512, 256)


@pytest.mark.timeout(1200)
def test_history_continues_across_a_resume(tmp_path):
    n = 41
    full = _loop(str(tmp_path / 'full'), None, n)
    out = str(tmp_path / 'r')
    stopped = {}
    with pytest.raises(_Stop):
        _loop(out, None, n, checkpoint_every=20, stop=21, seen=stopped)
    resumed = _loop(out, None, n, checkpoint_every=20, resume=True)
    assert resumed['states'][0][0] == 20
    a, b = resumed['hist'][n - 1][0], full['hist'][n - 1][0]
    assert a.shape == b.shape == (n, 4)
    assert torch.isfinite(a).all()
    # rows 0..19 are the ones the stopped run recorded before its checkpoint at iteration 20, restored bit for bit
    assert torch.equal(a[:20], stopped['hist'][19][0])
    # later rows are recomputed: they follow the uninterrupted run up to the field backward's atomics
    rel = ((a - b).abs() / b.abs().clamp(min=1e-12)).max().item()
    print(f'resumed history vs uninterrupted: max rel {rel:.2e}')
    assert rel < 1e-3
