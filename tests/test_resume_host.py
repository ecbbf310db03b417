"""Host side of checkpoint / resume: what ``Distiller.load_state_dict`` refuses (one case per fingerprint field, per scene-cache field, the
world-size rules, the seed), the checkpoint files of the loop (the mixed-checkpoint and seed refusals of ``distill_scenes`` /
``distillation_loop``, the atomic write, no file without ``checkpoint_every``, where a resumed loop starts), and ``FlatAdam``'s state round
trip on its flat buffers.  The cache digest runs on the device; here it is replaced by a host hash of the same bits."""
import hashlib
import os
from types import SimpleNamespace

import pytest
import torch


def _host_digest(cache):
    from sparsefusion_b200.distillation import SceneCache
    out = {}
    for f in SceneCache.__dataclass_fields__:
        t = getattr(cache, f).contiguous()
        out[f] = (tuple(t.shape), int.from_bytes(hashlib.sha256(t.numpy().tobytes()).digest()[:8], 'little'))
    return out


@pytest.fixture(autouse=True)
def host_digest(monkeypatch):
    from sparsefusion_b200 import distillation
    monkeypatch.setattr(distillation, 'cache_digest', _host_digest)


def _ddpm():
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    cfg = uo.SMALL
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks,
                layer_attns=cfg.layer_attns, layer_cross_attns=tuple(False for _ in cfg.dim_mults),
                cond_images_channels=cfg.cond_images_channels, attn_pool_text=False, attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads)
    return DDPM(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10)


_DDPM = None


def _cache():
    from oracle import distill_oracle as do, unet_oracle as uo
    from sparsefusion_b200.distillation import SceneCache
    return SceneCache(**do.synthetic_scene(n_input=2, n_target=6, image_size=32, latent=16, feat_ch=uo.SMALL.cond_images_channels,
                                           render_hw=16, seed=3))


def _distiller(cache=None, opt_kw=None, **kw):
    global _DDPM
    from sparsefusion_b200.distillation import Distiller
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    if _DDPM is None:
        _DDPM = _ddpm()
    opt = get_default_torch_ngp_opt()
    for k, v in (opt_kw or {}).items():
        setattr(opt, k, v)
    return Distiller(NeRFNetwork(opt), None, _DDPM, opt, _cache() if cache is None else cache, **kw)


def _snapshot(d):
    return (d.optimizer.flat.clone(), d.optimizer.m.clone(), d.optimizer.t, d.gen.get_state().clone(), torch.get_rng_state().clone())


def _unchanged(d, snap):
    flat, m, t, gen, rng = snap
    return (torch.equal(d.optimizer.flat, flat) and torch.equal(d.optimizer.m, m) and d.optimizer.t == t and torch.equal(d.gen.get_state(), gen)
            and torch.equal(torch.get_rng_state(), rng))


FINGERPRINT_CASES = [
    ('opt.num_steps', dict(opt_kw=dict(num_steps=32))),
    ('opt.cuda_ray', dict(opt_kw=dict(cuda_ray=True))),
    ('views_per_step', dict(views_per_step=4)),
    ('max_batch', dict(max_batch=8)),
    ('cond_scale', dict(cond_scale=3.0)),
    ('sds_method', dict(sds_method='onestep')),
    ('lambda_color', dict(lambda_color=0.5)),
    ('lambda_sil', dict(lambda_sil=0.5)),
    ('lambda_opacity', dict(lambda_opacity=0.0)),
    ('lambda_percep', dict(lambda_percep=0.2)),
    ('start_fusion_step', dict(start_fusion_step=10)),
    ('start_percep_step', dict(start_percep_step=10)),
    ('plms_steps', dict(plms_steps=25)),
    ('fused_glue', dict(fused_glue=False)),
    ('percep', dict(percep=object())),
]


@pytest.mark.parametrize('field,kw', FINGERPRINT_CASES, ids=[c[0] for c in FINGERPRINT_CASES])
def test_fingerprint_mismatch_is_refused_before_any_state_changes(field, kw):
    saved = _distiller(seed=4).state_dict(itr=7)
    other = _distiller(seed=4, **kw)
    snap = _snapshot(other)
    with pytest.raises(ValueError, match=rf'\b{field}\b'):
        other.load_state_dict(saved)
    assert _unchanged(other, snap)


def test_use_diffusion_mismatch_is_refused():
    saved = _distiller(seed=4).state_dict(itr=7, use_diffusion=True)
    with pytest.raises(ValueError, match='use_diffusion'):
        _distiller(seed=4).load_state_dict(saved, use_diffusion=False)


@pytest.mark.parametrize('field', ['input_rgb', 'input_mask', 'input_rays_o', 'input_rays_d', 'target_features', 'target_eft_image',
                                   'target_rays_o', 'target_rays_d'])
def test_cache_digest_mismatch_is_refused_per_field(field):
    saved = _distiller(seed=4).state_dict(itr=3)
    cache = _cache()
    getattr(cache, field).view(-1)[5] += 1e-3                    # one word of one field
    other = _distiller(cache=cache, seed=4)
    snap = _snapshot(other)
    with pytest.raises(ValueError, match=rf'scene cache field {field} contents'):
        other.load_state_dict(saved)
    assert _unchanged(other, snap)
    cache = _cache()
    setattr(cache, field, getattr(cache, field)[:1].clone())     # another view count
    with pytest.raises(ValueError, match=rf'scene cache field {field} shape'):
        _distiller(cache=cache, seed=4).load_state_dict(saved)


def test_seed_mismatch_is_refused():
    saved = _distiller(seed=4).state_dict(itr=3)
    with pytest.raises(ValueError, match='seed'):
        _distiller(seed=5).load_state_dict(saved)


def _two_rank_state(**kw):
    sd = _distiller(seed=4, **kw).state_dict(itr=9)
    sd['world_size'] = 2
    sd['rng'] = [sd['rng'][0], dict(sd['rng'][0])]
    return sd


def test_world_size_rules():
    # the reference step / one-view-per-rank form: the same world size only
    with pytest.raises(ValueError, match='world_size'):
        _distiller(seed=4).load_state_dict(_two_rank_state())
    # cuda_ray: the density grid and the CUDA generator are per rank, in every mode
    with pytest.raises(ValueError, match='world_size'):
        _distiller(seed=4, views_per_step=4, opt_kw=dict(cuda_ray=True)).load_state_dict(_two_rank_state(views_per_step=4, opt_kw=dict(cuda_ray=True)))
    # the keyed view-batched step continues at another world size
    d = _distiller(seed=4, views_per_step=4)
    sd = _two_rank_state(views_per_step=4)
    d.load_state_dict(sd)
    assert d.next_itr == 9 and torch.equal(d.optimizer.flat, torch.cat([sd['ngp'][k].reshape(-1) for k, _ in d.ngp.named_parameters()]))


def test_state_round_trip_on_the_host():
    a = _distiller(seed=4, opt_kw=dict(cuda_ray=True))
    g = torch.Generator().manual_seed(1)
    a.optimizer.flat.copy_(torch.randn(a.optimizer.flat.shape, generator=g))
    a.optimizer.m.copy_(torch.randn(a.optimizer.m.shape, generator=g))
    a.optimizer.v.copy_(torch.rand(a.optimizer.v.shape, generator=g))
    a.optimizer.t, a.optimizer.sched = 12, 11
    a.ngp.density_grid.copy_(torch.rand(a.ngp.density_grid.shape, generator=g))
    a.ngp.step_counter.fill_(3)
    a.ngp.mean_density, a.ngp.iter_density, a.ngp.mean_count, a.ngp.local_step = 0.25, 2, 1234, 5
    torch.randperm(6, generator=a.gen)
    sd = a.state_dict(itr=12)
    b = _distiller(seed=4, opt_kw=dict(cuda_ray=True))
    ptrs = [p.data_ptr() for p in b.ngp.parameters()] + [b.optimizer.flat.data_ptr(), b.optimizer.m.data_ptr(), b.optimizer.v.data_ptr()]
    torch.manual_seed(99)                                          # the global generator moves on; load_state_dict restores the saved state
    b.load_state_dict(sd)
    assert ptrs == [p.data_ptr() for p in b.ngp.parameters()] + [b.optimizer.flat.data_ptr(), b.optimizer.m.data_ptr(), b.optimizer.v.data_ptr()]
    for x, y in ((a.optimizer.flat, b.optimizer.flat), (a.optimizer.m, b.optimizer.m), (a.optimizer.v, b.optimizer.v),
                 (a.ngp.density_grid, b.ngp.density_grid), (a.ngp.density_bitfield, b.ngp.density_bitfield), (a.ngp.step_counter, b.ngp.step_counter),
                 (a.gen.get_state(), b.gen.get_state()), (sd['rng'][0]['cpu'], torch.get_rng_state())):
        assert torch.equal(x, y)
    assert (b.optimizer.t, b.optimizer.sched, b.next_itr) == (12, 11, 12)
    assert (b.ngp.mean_density, b.ngp.iter_density, b.ngp.mean_count, b.ngp.local_step) == (0.25, 2, 1234, 5)


def test_flat_adam_state_round_trip_in_place():
    from sparsefusion_b200.distillation import FlatAdam
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    a, b = FlatAdam(NeRFNetwork(opt)), FlatAdam(NeRFNetwork(opt))
    g = torch.Generator().manual_seed(2)
    a.m.copy_(torch.randn(a.m.shape, generator=g))
    a.v.copy_(torch.rand(a.v.shape, generator=g))
    a.t, a.sched = 7, 9
    sd = a.state_dict()
    a.m.zero_()                                                    # the state is a copy, not a view
    bufs = [b.flat.data_ptr(), b.grad.data_ptr(), b.m.data_ptr(), b.v.data_ptr()]
    views = [(p.data_ptr(), p.grad.data_ptr()) for p in b.params]
    b.load_state_dict(sd)
    assert bufs == [b.flat.data_ptr(), b.grad.data_ptr(), b.m.data_ptr(), b.v.data_ptr()]
    assert views == [(p.data_ptr(), p.grad.data_ptr()) for p in b.params]
    assert torch.equal(b.m, sd['m']) and torch.equal(b.v, sd['v']) and (b.t, b.sched) == (7, 9) and not torch.equal(b.m, a.m)
    sd['m'] = sd['m'][:-1]
    with pytest.raises(ValueError, match='optimizer.m'):
        b.load_state_dict(sd)


def test_atomic_write_keeps_the_old_checkpoint(tmp_path, monkeypatch):
    from sparsefusion_b200.distillation import _atomic_save
    path = str(tmp_path / 'scene.ckpt')
    _atomic_save({'itr': 4, 'x': torch.arange(10)}, path)
    before = open(path, 'rb').read()

    def interrupted(src, dst):
        raise KeyboardInterrupt('interrupted between the temporary write and the rename')
    monkeypatch.setattr(os, 'replace', interrupted)
    with pytest.raises(KeyboardInterrupt):
        _atomic_save({'itr': 8, 'x': torch.arange(20)}, path)
    monkeypatch.undo()
    assert open(path, 'rb').read() == before
    assert torch.load(path, weights_only=True)['itr'] == 4
    assert os.listdir(tmp_path) == ['scene.ckpt']


class _FakeDistiller:
    """stands in for the distiller of ``_run_distillation``: records steps, saves / loads a plain state"""

    def __init__(self, seed):
        self.seed, self.steps, self.loaded, self.next_itr = seed, [], None, 0

    def step(self, itr):
        self.steps.append(itr)
        self.next_itr = itr + 1

    photometric_substep = step

    def state_dict(self, itr, use_diffusion=True):
        return dict(version=1, itr=itr, seed=self.seed)

    def load_state_dict(self, sd, use_diffusion=True):
        self.loaded = sd
        self.next_itr = sd['itr']


class _Builder:
    def __init__(self):
        self.calls = 0

    def build(self, eft, scene_cameras, scene_rgb, scene_mask, input_idx, use_diffusion=True):
        self.calls += 1
        return _cache()


def _run(tmp_path, monkeypatch, names=('a',), **kw):
    from contextlib import nullcontext
    from sparsefusion_b200 import distillation
    monkeypatch.setattr(torch.cuda, 'device', lambda d: nullcontext())
    monkeypatch.setattr(torch.cuda, 'synchronize', lambda d=None: None)
    made, seen = [], []

    def make(ngps, caches, percep, seed):
        made.append(_FakeDistiller(seed))
        return made[-1]
    scenes = [(n, None, None, None, None, [0, 1]) for n in names]
    args = dict(use_diffusion=False, max_itr=5, scene_builder=kw.pop('builder', _Builder()), seed=5, on_iteration=lambda i, d: seen.append(i))
    args.update(kw)
    distillation._run_distillation('cpu', SimpleNamespace(exp_dir=str(tmp_path / 'exp')), distillation.get_default_torch_ngp_opt(), None,
                                   str(tmp_path / 'out'), scenes, make, args.pop('use_diffusion'), args.pop('max_itr'), args.pop('scene_builder'),
                                   args.pop('seed'), args.pop('on_iteration'), **args)
    return made[0], seen


def test_no_checkpoint_without_checkpoint_every(tmp_path, monkeypatch):
    d, seen = _run(tmp_path, monkeypatch)
    assert seen == [0, 1, 2, 3, 4] and d.steps == seen
    assert not os.path.exists(tmp_path / 'out' / 'checkpoints')
    assert os.path.exists(tmp_path / 'out' / 'a.pt')


def test_checkpoint_schedule_and_resume_start(tmp_path, monkeypatch):
    written = []
    from sparsefusion_b200 import distillation
    real = distillation._atomic_save
    monkeypatch.setattr(distillation, '_atomic_save', lambda obj, path: (written.append((obj['itr'], os.path.basename(path))), real(obj, path)))
    _run(tmp_path, monkeypatch, checkpoint_every=2)
    assert written == [(2, 'a.ckpt'), (4, 'a.ckpt'), (5, 'a.ckpt')]          # (itr + 1) % 2 == 0, and after the last iteration
    ck = torch.load(str(tmp_path / 'out' / 'checkpoints' / 'a.ckpt'), weights_only=True)
    assert ck['itr'] == 5 and ck['base_seed'] == 5
    # extend the finished run: it continues at iteration 5, with the saved base seed when seed is None
    d, seen = _run(tmp_path, monkeypatch, resume=True, seed=None, max_itr=8, checkpoint_every=2)
    assert d.seed == 5 and d.loaded['itr'] == 5 and seen == [5, 6, 7]
    assert written[3:] == [(6, 'a.ckpt'), (8, 'a.ckpt')]
    # max_itr at or below the saved iteration: no iteration runs
    d, seen = _run(tmp_path, monkeypatch, resume=True, max_itr=8)
    assert d.loaded['itr'] == 8 and seen == [] and d.steps == []
    # resume without a checkpoint starts fresh
    d, seen = _run(tmp_path, monkeypatch, names=('b',), resume=True)
    assert d.loaded is None and seen == [0, 1, 2, 3, 4]


def test_resume_refuses_a_different_seed_before_building(tmp_path, monkeypatch):
    from sparsefusion_b200.distillation import _atomic_save
    os.makedirs(tmp_path / 'out' / 'checkpoints')
    _atomic_save(dict(version=1, itr=4, base_seed=5), str(tmp_path / 'out' / 'checkpoints' / 'a.ckpt'))
    b = _Builder()
    with pytest.raises(ValueError, match='seed=6 differs from the base seed 5'):
        _run(tmp_path, monkeypatch, resume=True, seed=6, builder=b)
    assert b.calls == 0


def test_distill_scenes_refuses_mixed_checkpoints(tmp_path, monkeypatch):
    from sparsefusion_b200.distillation import _atomic_save, distill_scenes, get_default_torch_ngp_opt
    ck = tmp_path / 'out' / 'checkpoints'
    os.makedirs(ck)
    _atomic_save(dict(version=1, itr=4, base_seed=5), str(ck / 'hydrant_000.ckpt'))
    b = _Builder()
    scenes = [(n, None, None, None, None, [0, 1]) for n in ('hydrant_000', 'hydrant_001')]
    args = SimpleNamespace(exp_dir=str(tmp_path / 'exp'))
    model = (None, None, None)
    with pytest.raises(ValueError, match=r"\['hydrant_000'\] but not for \['hydrant_001'\]"):
        distill_scenes('cpu', args, get_default_torch_ngp_opt(), model, str(tmp_path / 'out'), scenes, use_diffusion=False, scene_builder=b,
                       resume=True)
    _atomic_save(dict(version=1, itr=6, base_seed=5), str(ck / 'hydrant_001.ckpt'))
    with pytest.raises(ValueError, match="different iterations.*'hydrant_000': 4, 'hydrant_001': 6"):
        distill_scenes('cpu', args, get_default_torch_ngp_opt(), model, str(tmp_path / 'out'), scenes, use_diffusion=False, scene_builder=b,
                       resume=True)
    assert b.calls == 0


def test_checkpoint_every_must_be_a_positive_int(tmp_path, monkeypatch):
    for bad in (0, -2, 1.5, True):
        with pytest.raises(ValueError, match='checkpoint_every'):
            _run(tmp_path, monkeypatch, checkpoint_every=bad)
