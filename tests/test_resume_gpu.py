"""Checkpoint and resume of the distillation on the GPU, on reduced scenes (64x64 rays, 128^2 images, 16^2 latents, small UNet / VAE).

For each step mode -- the reference step with cuda_ray, the view-batched step at V = 4 guided at cond_scale 3, three scenes at once with
the one-step SDS target -- k iterations are run, saved, and loaded into freshly built objects:
(1) round trip: every tensor, counter and generator state of the loaded objects equals the saved run's, bit for bit;
(2) draws: over the next m iterations the resumed run's draws (permutation / u generator, global CPU and CUDA generators at every step, render
    jitter, PLMS noise, one-step noise and keep mask) are bit-identical to those of an uninterrupted run of k + m iterations;
(3) trajectory: the resumed parameters after k + m iterations agree with the uninterrupted run's within a small multiple of the spread
    between two uninterrupted runs measured in the same test (the field backward accumulates with atomics, so runs differ in the last bits).
    For (3) the SDS target, once the sampler has run and drawn, is replaced by a fixed image per target view (``fixed_target``): an L1
    against a sampled target flips sign on near-tie pixels, so two uninterrupted runs drift apart by amounts that vary 1000-fold from run
    to run; against a fixed target they differ by the atomics only, and the spread is a stable yardstick.
Then the loops: ``distillation_loop`` and ``distill_scenes`` interrupted from ``on_iteration`` and resumed, extended past a finished run,
resumed with ``seed=None``; and a checkpoint of two ranks (gloo) resumed on one.
"""
import io
import os
import re
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

K, M = 3, 3            # iterations before the checkpoint, iterations after it
SPREAD_FACTOR = 4      # the resumed run's distance to the uninterrupted one, in units of the run-to-run spread
FLOOR = 1e-6           # relative distance accepted whatever the spread (two runs may happen to agree bit for bit)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


_MODELS = None


def _models():
    global _MODELS
    if _MODELS is None:
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
        ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,),
                    timesteps=500, cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                    dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()
        _MODELS = (vae.cuda(), ddpm)
    return _MODELS


def _scene(k):
    from oracle import distill_oracle as do, unet_oracle as uo
    return do.synthetic_scene(n_input=2, n_target=6, image_size=128, latent=16, feat_ch=uo.SMALL.cond_images_channels, render_hw=64, seed=3 + k)


_CACHES = {}


def _cache(k):
    from sparsefusion_b200.distillation import SceneCache
    if k not in _CACHES:
        _CACHES[k] = SceneCache(**_scene(k)).to('cuda')
    return _CACHES[k]


MODES = ['reference-cuda_ray', 'views4-guided', 'multi3-onestep']


def _build(mode, init_seed, rank=0, world=1):
    """fresh network(s) initialised from ``init_seed`` and a fresh distiller of ``mode``"""
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    vae, ddpm = _models()
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = mode == 'reference-cuda_ray'
    torch.manual_seed(init_seed)
    if mode == 'multi3-onestep':
        return MultiSceneDistiller([NeRFNetwork(opt).cuda().train() for _ in range(3)], vae, ddpm, opt, [_cache(k) for k in range(3)],
                                   seeds=[11, 12, 13], start_fusion_step=1, sds_method='onestep')
    kw = dict(views_per_step=4, cond_scale=3.0) if mode == 'views4-guided' else {}
    if mode == 'views4':
        kw = dict(views_per_step=4)
    return Distiller(NeRFNetwork(opt).cuda().train(), vae, ddpm, opt, _cache(0), seed=11, start_fusion_step=1, rank=rank, world_size=world, **kw)


def _scenes(dist):
    return list(getattr(dist, 'scenes', [dist]))


class _Draws:
    """every draw of a run, in order: the generator states at the start of each iteration, each render's draws (keyed) or the CUDA generator
    state it draws from (reference step), every PLMS noise tensor and every one-step noise / keep mask"""

    def __init__(self):
        self.log, self.starts = [], {}

    def add(self, tag, *ts):
        self.log.append((tag, [t.detach().clone() if isinstance(t, torch.Tensor) else t for t in ts]))

    def since(self, itr):
        return self.log[self.starts[itr]:]


_ACTIVE = [None]


@pytest.fixture(autouse=True)
def _record_shared_draws(monkeypatch):
    """KeyedNoise (view-batched / multi-scene PLMS noise) and DDPM.forward_noloss (one-step noise and keep) record into the active log"""
    from sparsefusion_b200 import distillation, vldm
    call, fwd = distillation.KeyedNoise.__call__, vldm.DDPM.forward_noloss

    def keyed(self, like, rows=None):
        out = call(self, like, rows)
        if _ACTIVE[0] is not None:
            _ACTIVE[0].add('plms', out)
        return out

    def forward_noloss(self, *a, **kw):
        if _ACTIVE[0] is not None:
            _ACTIVE[0].add('onestep', torch.cuda.get_rng_state(), kw.get('noise'), kw.get('keep'), kw.get('times'))
        return fwd(self, *a, **kw)
    monkeypatch.setattr(distillation.KeyedNoise, '__call__', keyed)
    monkeypatch.setattr(vldm.DDPM, 'forward_noloss', forward_noloss)
    yield
    _ACTIVE[0] = None


def _fixed_target(real):
    """``Distiller._fusion_target`` that runs (and draws) as ``real`` does, then returns a fixed image per target view: a function of the
    view's conditioning features"""
    import torch.nn.functional as F

    def fusion_target(self, images, feats, *a, **kw):
        pred, acp = real(self, images, feats, *a, **kw)
        return F.interpolate(torch.sigmoid(feats[:, :3].float()), size=pred.shape[-2:], mode='bilinear'), acp
    return fusion_target


@pytest.fixture
def fixed_target(monkeypatch):
    from sparsefusion_b200.distillation import Distiller
    monkeypatch.setattr(Distiller, '_fusion_target', _fixed_target(Distiller._fusion_target))


def _instrument(dist, rec):
    for d in _scenes(dist):
        orig = d._render_draws

        def render_draws(rays_o, itr, view, stream, keyed, orig=orig):
            out = orig(rays_o, itr, view, stream, keyed)
            rec.add(('render', itr, view, stream), torch.cuda.get_rng_state(), *(out or ()))
            return out
        d._render_draws = render_draws
        d.sampler.noise_fn = lambda like: rec.add('plms', torch.randn_like(like)) or rec.log[-1][1][0]   # the global generator, recorded
    _ACTIVE[0] = rec


def _run(dist, itrs, rec):
    _instrument(dist, rec)
    for itr in itrs:
        rec.starts[itr] = len(rec.log)
        rec.add(('itr', itr), *[d.gen.get_state() for d in _scenes(dist)], torch.get_rng_state(), torch.cuda.get_rng_state())
        dist.step(itr)
    torch.cuda.synchronize()
    _ACTIVE[0] = None


def _flat(dist):
    return torch.cat([d.optimizer.flat for d in _scenes(dist)]).cpu()


def _live_state(dist):
    """every tensor and counter a resumed run depends on, as host values"""
    out = []
    for d in _scenes(dist):
        o, n = d.optimizer, d.ngp
        out += [o.flat, o.m, o.v, o.t, o.sched, d.gen.get_state(), d.seed]
        if n.cuda_ray:
            out += [n.density_grid, n.density_bitfield, n.step_counter, n.mean_density, n.iter_density, n.mean_count, n.local_step]
    return [x.detach().cpu() if isinstance(x, torch.Tensor) else x for x in out] + [torch.get_rng_state(), torch.cuda.get_rng_state()]


def _same(a, b):
    return type(a) is type(b) and (torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b)


def _same_log(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for (ta, xa), (tb, xb) in zip(a, b):
        assert ta == tb, (ta, tb)
        assert len(xa) == len(xb) and all((x is None and y is None) or _same(x, y) for x, y in zip(xa, xb)), ta


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('mode', MODES)
def test_resume_round_trip_draws_and_trajectory(mode, fixed_target):
    # two uninterrupted runs of K + M iterations: the reference trajectory and its run-to-run spread
    full, again = _Draws(), _Draws()
    a = _build(mode, 0)
    _run(a, range(K + M), full)
    b = _build(mode, 0)
    _run(b, range(K + M), again)
    spread = _rel(_flat(b), _flat(a))
    # K iterations, a checkpoint through the file format, fresh objects (another initialisation) loaded from it
    first = _build(mode, 0)
    _run(first, range(K), _Draws())
    sd = first.state_dict()
    want = _live_state(first)
    buf = io.BytesIO()
    torch.save(sd, buf)
    size = buf.tell()
    buf.seek(0)
    sd = torch.load(buf, map_location='cpu', weights_only=True)
    assert sd['itr'] == K
    resumed = _build(mode, 1234)
    assert not torch.equal(_flat(resumed), _flat(first))
    resumed.load_state_dict(sd)
    got = _live_state(resumed)
    assert len(want) == len(got) and all(_same(x, y) for x, y in zip(want, got)), [i for i, (x, y) in enumerate(zip(want, got)) if not _same(x, y)]
    # M more iterations: the same draws as the uninterrupted run's, and the same trajectory within the spread
    rec = _Draws()
    _run(resumed, range(K, K + M), rec)
    _same_log(rec.log, full.since(K))
    dist = _rel(_flat(resumed), _flat(a))
    kinds = sorted({t if isinstance(t, str) else t[0] for t, _ in rec.log})
    print(f'{mode}: checkpoint {size / 1e6:.2f} MB; {len(rec.log)} draws compared ({", ".join(kinds)}); parameters after {K + M} iterations: '
          f'run-to-run spread {spread:.3e}, resumed vs uninterrupted {dist:.3e} (ratio {dist / max(spread, 1e-30):.2f})')
    assert dist <= SPREAD_FACTOR * spread + FLOOR


def _digest_host(words):
    """numpy restatement of sfb_digest_u32 (header section 13)"""
    def mix(x):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))
    with np.errstate(over='ignore'):
        i = np.arange(words.size, dtype=np.uint64)
        return int(mix(words.astype(np.uint64) ^ mix(i + np.uint64(0x9E3779B97F4A7C15))).sum(dtype=np.uint64))


def test_cache_digest_matches_its_definition():
    from sparsefusion_b200.distillation import SceneCache, cache_digest
    cache = _cache(0)
    got = cache_digest(cache)
    for f in SceneCache.__dataclass_fields__:
        t = getattr(cache, f)
        assert got[f] == (tuple(t.shape), _digest_host(t.contiguous().cpu().numpy().view(np.uint32).reshape(-1))), f
    moved = SceneCache(**{f: getattr(cache, f).clone() for f in SceneCache.__dataclass_fields__})
    moved.input_rgb.view(-1)[[7, 8]] = moved.input_rgb.view(-1)[[8, 7]]        # two words swapped: same sum of values, another digest
    assert cache_digest(moved)['input_rgb'] != got['input_rgb'] or torch.equal(moved.input_rgb, cache.input_rgb)


# ---------------------------------------------------------------------------------------------------- the loops
class _Builder:
    def __init__(self, k=0):
        self.k = k

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        from sparsefusion_b200.distillation import SceneCache
        return SceneCache(**_scene(self.k if scene_cameras is None else scene_cameras))

    def eval_views(self, scene_cameras, scene_rgb, scene_mask):
        """two target views at the render size, scored against their EFT images"""
        import torch.nn.functional as F
        from sparsefusion_b200.evaluate import EvalViews
        s = _scene(self.k if scene_cameras is None else scene_cameras)
        rgb = F.interpolate(s['target_eft_image'][:2], size=(64, 64), mode='bilinear')
        return EvalViews(rays_o=s['target_rays_o'][:2], rays_d=s['target_rays_d'][:2], rgb=rgb, mask=(rgb.mean(1, keepdim=True) > .1).float())


class _Stop(Exception):
    pass


def _loop(out, max_itr, *, scenes=None, stop_after=None, seen=None, **kw):
    from sparsefusion_b200.distillation import distill_scenes, distillation_loop, get_default_torch_ngp_opt
    vae, ddpm = _models()
    seen = [] if seen is None else seen

    def on_iteration(itr, d):
        seen.append((itr, [s.seed for s in _scenes(d)]))
        if itr == stop_after:
            raise _Stop()
    args = SimpleNamespace(exp_dir=os.path.join(out, 'exp'), category='hydrant')
    common = dict(max_itr=max_itr, on_iteration=on_iteration, evaluate=True, **kw)
    torch.manual_seed(0)
    if scenes is None:
        distillation_loop(0, args, get_default_torch_ngp_opt(), ('eft', vae, ddpm), out, 'hydrant_000', None, None, None, None, [0, 1],
                          scene_builder=_Builder(), **common)
        names = ['hydrant_000']
    else:
        names = [f'hydrant_{k:03d}' for k in range(scenes)]
        distill_scenes(0, args, get_default_torch_ngp_opt(), ('eft', vae, ddpm), out, [(n, k, None, None, None, [0, 1]) for k, n in enumerate(names)],
                       scene_builder=_Builder(), **common)
    params = torch.cat([torch.cat([v.reshape(-1).float() for v in torch.load(os.path.join(out, f'{n}.pt'), map_location='cpu')['model_state_dict'].values()])
                        for n in names])
    metrics = np.array([float(x) for n in names for x in re.findall(r'[-+]?(?:\d+\.\d*|nan)', open(os.path.join(out, 'metrics', f'{n}.txt')).read())])
    return params, metrics, seen


def _metric_gap(a, b):
    both = np.isfinite(a) & np.isfinite(b)
    assert (np.isfinite(a) == np.isfinite(b)).all()
    return float(np.max(np.abs(a[both] - b[both]) / np.maximum(np.abs(b[both]), 1e-12), initial=0.0))


@pytest.mark.timeout(1500)
@pytest.mark.parametrize('scenes', [None, 2], ids=['distillation_loop', 'distill_scenes'])
def test_loop_interrupted_resumed_and_extended(scenes, tmp_path):
    n = 8
    p1, m1, _ = _loop(str(tmp_path / 'u1'), n, scenes=scenes, seed=5)
    p2, m2, _ = _loop(str(tmp_path / 'u2'), n, scenes=scenes, seed=5)
    spread, mspread = _rel(p2, p1), _metric_gap(m2, m1)
    # interrupted after iteration 3 (checkpoint_every 2 has just saved iteration 4), then the same command with resume=True
    out = str(tmp_path / 'r')
    with pytest.raises(_Stop):
        _loop(out, n, scenes=scenes, seed=5, checkpoint_every=2, stop_after=3)
    assert torch.load(os.path.join(out, 'checkpoints', 'hydrant_000.ckpt'), weights_only=True)['itr'] == 4
    pr, mr, seen = _loop(out, n, scenes=scenes, seed=5, checkpoint_every=2, resume=True)
    assert [s[0] for s in seen] == list(range(4, n))
    # a finished run of 4 iterations extended to 8
    ext = str(tmp_path / 'e')
    _loop(ext, 4, scenes=scenes, seed=5, checkpoint_every=2)
    pe, me, seen_e = _loop(ext, n, scenes=scenes, seed=5, checkpoint_every=2, resume=True)
    assert [s[0] for s in seen_e] == list(range(4, n))
    dr, de = _rel(pr, p1), _rel(pe, p1)
    gr, ge = _metric_gap(mr, m1), _metric_gap(me, m1)
    print(f'{scenes or 1} scene(s), {n} iterations: parameter spread {spread:.3e}, resumed {dr:.3e}, extended {de:.3e}; '
          f'metric spread {mspread:.3e}, resumed {gr:.3e}, extended {ge:.3e}')
    assert dr <= SPREAD_FACTOR * spread + FLOOR and de <= SPREAD_FACTOR * spread + FLOOR
    assert gr <= SPREAD_FACTOR * mspread + 1e-5 and ge <= SPREAD_FACTOR * mspread + 1e-5


def test_resume_uses_the_saved_seed(tmp_path):
    out = str(tmp_path / 'r')
    with pytest.raises(_Stop):
        _loop(out, 3, seed=None, checkpoint_every=1, stop_after=0)
    base = torch.load(os.path.join(out, 'checkpoints', 'hydrant_000.ckpt'), weights_only=True)['base_seed']
    _, _, seen = _loop(out, 3, seed=None, checkpoint_every=1, resume=True)
    assert [s[0] for s in seen] == [1, 2] and all(s[1] == [base] for s in seen)
    # at or past max_itr: no iteration runs, the outputs come from the saved state
    _, _, seen = _loop(out, 3, seed=None, resume=True)
    assert seen == []


# ---------------------------------------------------------------------------------------------------- two ranks
def _worker(rank, world, store, out_dir):
    import torch.distributed as td
    td.init_process_group('gloo', init_method=f'file://{store}', rank=rank, world_size=world)
    try:
        torch.cuda.set_device(rank % torch.cuda.device_count())
        from sparsefusion_b200.distillation import Distiller
        Distiller._fusion_target = _fixed_target(Distiller._fusion_target)      # as the parent's fixed_target fixture
        d = _build('views4', 0, rank=rank, world=world)
        for itr in range(K):
            d.step(itr)
        sd = d.state_dict()                                      # every rank: the generator states are gathered
        one_view = _build('reference', 0, rank=rank, world=world)
        sd1 = one_view.state_dict(itr=0)
        torch.cuda.synchronize()
        if rank == 0:
            torch.save(dict(views=sd, one_view=sd1), os.path.join(out_dir, 'ckpt.pt'))
    finally:
        td.destroy_process_group()


@pytest.mark.timeout(1200)
def test_two_rank_checkpoint_resumes_on_one_rank(fixed_target):
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        try:
            mp.spawn(_worker, args=(2, os.path.join(d, 'store'), d), nprocs=2, join=True)
        except Exception as e:   # noqa: BLE001
            if 'gloo' in str(e).lower() and 'cuda' in str(e).lower():
                pytest.skip(f'gloo without CUDA tensor support in this torch build: {e}')
            raise
        ck = torch.load(os.path.join(d, 'ckpt.pt'), map_location='cpu', weights_only=True)
    assert ck['views']['world_size'] == 2 and len(ck['views']['rng']) == 2
    a, b = _build('views4', 0), _build('views4', 0)
    _run(a, range(K + M), _Draws())
    _run(b, range(K + M), _Draws())
    spread = _rel(_flat(b), _flat(a))
    resumed = _build('views4', 1234)
    resumed.load_state_dict(ck['views'])
    _run(resumed, range(K, K + M), _Draws())
    dist = _rel(_flat(resumed), _flat(a))
    print(f'2-rank checkpoint resumed on 1 rank: spread {spread:.3e}, resumed vs uninterrupted 1-rank run {dist:.3e} '
          f'(ratio {dist / max(spread, 1e-30):.2f})')
    assert dist <= SPREAD_FACTOR * spread + FLOOR
    with pytest.raises(ValueError, match='world_size'):
        _build('reference', 0).load_state_dict(ck['one_view'])
