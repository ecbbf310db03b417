"""Every library launch of real model evaluations checked in place, per element against fp64 of the operands it actually read.

The per-launch tests (tests/test_conv_fp64_gpu.py, tests/test_simt_fp64_gpu.py) replay each launch on its own, so they cannot see one launch
reading an operand before the launch that produces it finished.  Here oracle/insitu.py records the launches of the models themselves, with
the production defaults (3xTF32, programmatic dependent launch, ``parallel_res_conv`` and the split-K arena on), keeps every tensor they
read and wrote, and recomputes each launch in fp64 from the final contents of its operands.  A launch that read an operand too early
disagrees with that operand's final contents; outputs are NaN-filled before the checked run, so an early read of an intermediate gives NaN
however close the two replays' values are.  Each configuration runs once.

- UNet graphs (``UnetGraph`` on seeded weights): FULL at 32^2 latents, batch 1 and 8; batch 2 in the guided-pair layout (cond rows [c, 0]);
  SMALL at 128^2; FULL at 128^2, batch 1, in a test of its own.  Capture with the recorder on and replay A; NaN into every recorded output;
  replay B with inputs drawn independently of A's (another log-SNR level, conditioning of the opposite sign); check every record of both
  graphs, none of which may still hold NaN.  Then NaN into the main graph's outputs (not ``feat``, the conditioning graph's output), replay C
  with ``new_cond=False`` and check the main graph's records again.
- Eager models, each after one warm-up evaluation of the same model and with NaN left in the caching allocator's free blocks: the full VAE
  (encode at 256^2, decode from 32^2) and the narrow VAE at 128^2, batch 1 and 2; the eager UNet, SMALL and FULL, batch 1 and 2;
  PerceptualLoss.value_and_grad at 128^2 and 256^2; the EFT encode and feature_cache.
- The sampler loop on the SMALL UNet with its graphs: PLMSSampler.sample unguided and guided (cond_scale 3), and sample_rows over two
  schedules, so that a row drops out.  Every round: the graph's static inputs equal, bit for bit, the active rows' latents, their
  time-feature rows at each row's level and exactly their conditioning; each sfb_plms_update_rows / _cfg launch is within the fp64 bound of
  its operands cloned right after the launch (the guided eps it writes bit for bit); and its eps operands equal what p_sample assigns,
  built from a per-row log of every replay's output.
- Every GEMM record of every configuration passes ``insitu.provenance``: what conv_gemm_kernel reads ahead of griddepcontrol.wait comes from
  the prepared plans, and ``dynamic_weights`` is set exactly where the weight operand was written in the same evaluation.

Every kernel a configuration launches is accounted for: by a checked record, whose traced names are as many as its kernels, or by name
as a C ABI launch without a front end (the LPIPS prep / relu / max-pool / head kernels, the EFT's own kernels), which is not checked here;
their per-element tests replay them (tests/test_simt_fp64_gpu.py, tests/test_step_fp64_gpu.py).  Out of scope: write-after-read hazards
(every tensor is kept alive, so the allocator reuses no buffer inside a recorded evaluation).

Measured on an H100 80GB HBM3 at 700 W: the whole file passes in 75 s (FULL at 128^2 alone 10 s, against its 900 s timeout) and its
largest configuration peaks at 18.2 GiB (the EFT; 8.0 GiB for FULL at 128^2, 0.2 GiB for a sampler run), against the 40 GiB bar that
keeps the file well inside one shared 80 GB card."""
import dataclasses
from collections import defaultdict

import pytest
import torch

from oracle import insitu, model_runs

pytestmark = pytest.mark.gpu

STATS = {}          # configuration -> summary line (printed by the catalogue test)
PEAK = [0]          # largest peak memory of a configuration, bytes


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _mark_side(recs, unet):
    side = {s.cuda_stream for s in unet._side.values()} if unet is not None else set()
    for r in recs:
        r.s['side'] = r.stream in side


def _check(name, recs, fails):
    """check every record; returns {family: worst ratio}; failures appended as lines"""
    sm = _sm()
    worst = defaultdict(float)
    for i, r in enumerate(recs):
        rep = insitu.check(r, sm)
        r.s['checked'] = True
        worst[r.family] = max(worst[r.family], rep.ratio)
        if not rep.ok:
            fails.append(f'{name}: ' + insitu.describe(i, r, rep))
        if r.op == 'conv2d_nhwc' and r.names != [r.s['plan_kernel']]:
            fails.append(f'{name}: #{i} {r.label} traced {r.names}, planned {r.s["plan_kernel"]}')
        if len(r.names) != r.kernels:
            fails.append(f'{name}: #{i} {r.label} launched {r.kernels} kernels, traced {r.names}')
    return worst


def _summary(name, recs, unchecked, worst, extra=''):
    PEAK[0] = max(PEAK[0], torch.cuda.max_memory_allocated())
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    excl = defaultdict(int)
    for n, k, _ in unchecked:
        excl[n] += k
    s = (f'{name}: {len(recs)} records checked ({sum(r.kernels for r in recs)} kernels, {sum(r.snapshots for r in recs)} snapshot clones, '
         f'{sum(bool(r.s.get("side")) for r in recs)} on the side stream); worst err/bound '
         + ', '.join(f'{f} {v:.3f}' for f, v in sorted(worst.items()))
         + (f'; not checked (C ABI launches without a front end): ' + ', '.join(f'{n} x{k}' for n, k in sorted(excl.items())) if excl else '')
         + f'{extra}; peak memory {peak:.2f} GiB')
    print('\n' + s)
    STATS[name] = s
    return s


# ------------------------------------------------------------------------------------------------ UNet graphs
def _graph_run(name, cfg, nb, guided=False):
    from oracle import unet_oracle as uo
    from sparsefusion_b200 import ops
    from sparsefusion_b200.imagen_pytorch import UnetGraph
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    unet = model_runs._unet(cfg)
    assert unet.use_arena and unet.parallel_res_conv and ops.get_precision() == 'tf32x3'
    g = torch.Generator(device='cuda').manual_seed(nb * 7 + cfg.image_size)
    h, cc = cfg.image_size, cfg.cond_images_channels
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)

    def cond(sign):
        c = sign * rn(nb // 2 if guided else nb, cc, h, h)
        return torch.cat((c, torch.zeros_like(c))) if guided else c
    ls = lambda t: uo.alpha_cosine_log_snr(torch.full((nb,), t)).cuda()
    G = UnetGraph(unet)
    fails = []
    with torch.no_grad():
        c_a = cond(1.0)
        with insitu.Recorder('UNet', captured_only=True) as rec:
            G(rn(nb, 4, h, h), ls(0.31), c_a)                          # capture, replay A
        torch.cuda.synchronize()
        (key, entry), = G._graphs.items()
        n_kernels, n_cond = entry[6], entry[7]
        recs = rec.recs
        assert all(r.captured for r in recs) and not rec.unchecked
        _mark_side(recs, unet)
        # the conditioning graph is captured first: its records are the prefix holding its kernels
        acc, split = 0, None
        for i, r in enumerate(recs):
            if acc == n_cond:
                split = i
                break
            acc += r.kernels
        assert split is not None and sum(r.kernels for r in recs) == n_kernels + n_cond, (n_kernels, n_cond)
        cond_recs, main_recs = recs[:split], recs[split:]
        plans = insitu.plan_storages(unet)
        fails += insitu.provenance(recs, plans)
        insitu.poison(recs)
        G(rn(nb, 4, h, h), ls(0.83), -c_a if not guided else cond(-1.0))         # replay B: independent inputs
        torch.cuda.synchronize()
        worst = _check(f'{name} replay B', recs, fails)
        insitu.poison(main_recs)                                                # not feat: the cond graph is not replayed
        G(rn(nb, 4, h, h), ls(0.57), c_a, new_cond=False)                       # replay C
        torch.cuda.synchronize()
        w2 = _check(f'{name} replay C', main_recs, fails)
        for f, v in w2.items():
            worst[f] = max(worst[f], v)
    s = _summary(name, recs, [], worst, f'; graphs: {n_cond} + {n_kernels} kernels')
    _drop(recs)
    del G, unet
    return dict(recs=recs, fails=fails, summary=s)


def _drop(recs):
    """release the recorded tensors once checked (the catalogue keeps the records' metadata only)"""
    for r in recs:
        r.t, r.orig = {}, {}
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ eager models
def _eager_run(name, family, fn, objs, unet=None, warm_nan=True):
    from sparsefusion_b200 import ops
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    fails = []
    with torch.no_grad():
        fn()                                    # warm-up: prepared plans, the arena size, the pre-split weights
        torch.cuda.synchronize()
        plans = insitu.plan_storages(*objs)
        if warm_nan:
            insitu.poison_allocator()
        n0 = ops.launch_count()
        with insitu.Recorder(family) as rec:
            fn()
        torch.cuda.synchronize()
        n1 = ops.launch_count()
    recs = rec.recs
    _mark_side(recs, unet)
    counted = sum(r.kernels for r in recs) + sum(k for _, k, _ in rec.unchecked)
    if counted != n1 - n0:
        fails.append(f'{name}: records account for {counted} of {n1 - n0} kernels')
    if rec.unattributed:
        fails.append(f'{name}: traced kernels no record accounts for: {rec.unattributed}')
    fails += [f'{name}: {m}' for m in insitu.provenance(recs, plans)]
    worst = _check(name, recs, fails)
    s = _summary(name, recs, rec.unchecked, worst)
    _drop(recs)
    return dict(recs=recs, fails=fails, summary=s, unchecked=rec.unchecked)


def _eager_configs():
    from oracle import unet_oracle as uo, vae_oracle as vo
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    g = torch.Generator(device='cuda').manual_seed(5)
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
    for vname, kw, size in (('full', {}, 256), ('narrow', dict(ch=32, ch_mult=(1, 2, 4, 4)), 128)):
        vae = AutoencoderKL(**kw).eval()
        vae.load_state_dict(vo.make_params(seed=0, **kw))
        vae = vae.cuda()
        for nb in (1, 2):
            img = torch.rand(nb, 3, size, size, device='cuda', generator=g) * 2 - 1
            z = rn(nb, 4, size // 8, size // 8)
            yield f'VAE {vname} {size}^2 batch {nb}', 'VAE', (lambda v=vae, i=img, zz=z: (v.encode(i), v.decode(zz))), (vae,), None
        del vae
    for uname, cfg in (('SMALL', uo.SMALL), ('FULL', uo.FULL)):
        unet = model_runs._unet(cfg)
        h = cfg.image_size
        for nb in (1, 2):
            x, c = rn(nb, 4, h, h), rn(nb, cfg.cond_images_channels, h, h)
            ls = uo.alpha_cosine_log_snr(torch.full((nb,), 0.05)).cuda()
            yield f'eager UNet {uname} {h}^2 batch {nb}', 'UNet', (lambda u=unet, x=x, ls=ls, c=c: u.forward(x, ls, cond_images=c)), (unet,), unet
        del unet
    for size in (128, 256):
        pl = PerceptualLoss('vgg', device='cuda', seed=2)
        a, b = torch.rand(3, size, size, device='cuda', generator=g), torch.rand(3, size, size, device='cuda', generator=g)
        yield f'LPIPS {size}^2', 'LPIPS', (lambda pl=pl, a=a, b=b: pl.value_and_grad(a, b)), (pl,), None


@pytest.fixture(scope='module')
def graph_runs():
    from oracle import unet_oracle as uo
    runs = {}
    for name, cfg, nb, guided in (('graph FULL 32^2 batch 1', uo.FULL, 1, False), ('graph FULL 32^2 batch 8', uo.FULL, 8, False),
                                  ('graph FULL 32^2 guided pair', uo.FULL, 2, True),
                                  ('graph SMALL 128^2 batch 1', dataclasses.replace(uo.SMALL, image_size=128), 1, False)):
        runs[name] = _graph_run(name, cfg, nb, guided)
    return runs


@pytest.fixture(scope='module')
def eager_runs():
    runs = {}
    for name, family, fn, objs, unet in _eager_configs():
        runs[name] = _eager_run(name, family, fn, objs, unet)
        torch.cuda.empty_cache()
    runs['EFT encode + feature_cache'] = _eft_run()
    return runs


def _eft_run():
    """oracle/model_runs.record_eft's evaluation (encode at 256^2, a feature_cache of three views), recorded on the model's second run.
    border_bilinear (eft_ops.cu) clamps a NaN coordinate to 0 (fmaxf returns the other operand) before it forms an address, so the NaN
    allocator warm-up is safe here too."""
    from sparsefusion_b200 import ops
    state = {}

    class Rec:
        def __call__(self, family):
            return self

        def __enter__(self):
            state['n0'] = ops.launch_count()
            state['recorder'] = insitu.Recorder('EFT').__enter__()
            return self

        def __exit__(self, *exc):
            state['recorder'].__exit__(*exc)
            state['n1'] = ops.launch_count()
            return False

    def warmup(m):
        torch.cuda.synchronize()
        state['plans'] = insitu.plan_storages(m)
        insitu.poison_allocator()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model_runs.record_eft(Rec(), warmup=warmup)
    torch.cuda.synchronize()
    rec = state['recorder']
    fails = []
    counted = sum(r.kernels for r in rec.recs) + sum(k for _, k, _ in rec.unchecked)
    if counted != state['n1'] - state['n0']:
        fails.append(f"EFT: records account for {counted} of {state['n1'] - state['n0']} kernels")
    if rec.unattributed:
        fails.append(f'EFT: traced kernels no record accounts for: {rec.unattributed}')
    fails += [f'EFT: {m}' for m in insitu.provenance(rec.recs, state['plans'])]
    worst = _check('EFT', rec.recs, fails)
    s = _summary('EFT encode + feature_cache', rec.recs, rec.unchecked, worst)
    _drop(rec.recs)
    return dict(recs=rec.recs, fails=fails, summary=s, unchecked=rec.unchecked)


# ------------------------------------------------------------------------------------------------ sampler loop
def _sampler_run(name, mts, guided):
    """one PLMSSampler run on the SMALL UNet (graphs on), with every replay logged and every update launch recorded; per round: the graph's
    static inputs against what the round's active rows need, the update against fp64 of its operands cloned right after the launch, and
    its eps operands against p_sample's assignment built from the replay log"""
    from oracle import unet_oracle as uo
    from sparsefusion_b200.plms import PLMSSampler, row_schedule
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    ddpm = model_runs._ddpm500(uo.SMALL)
    unet = ddpm.unets[0]
    sampler = PLMSSampler(ddpm, 50)
    S, h = len(mts), uo.SMALL.image_size
    g = torch.Generator(device='cuda').manual_seed(11 + S + int(guided))
    image = torch.randn(S, 4, h, h, device='cuda', generator=g)
    cond = torch.randn(S, uo.SMALL.cond_images_channels, h, h, device='cuda', generator=g)
    cs = 3.0 if guided else 1.0
    log, tf = [], {}
    replay, precompute_time = sampler._replay, unet.precompute_time

    def logged_replay(u, x, log_snr, cond_images, time_features):
        out = replay(u, x, log_snr, cond_images, time_features)
        _, _, sx, sf, sc, _, _, _, _ = sampler._graph._graphs[(tuple(x.shape), tuple(cond_images.shape), x.device.index)]
        log.append(dict(sx=sx.clone(), sf={k: v.clone() for k, v in sf.items()}, sc=sc.clone(), out=out.clone()))
        return out

    def logged_time(t):
        tf.update(precompute_time(t))
        return tf
    sampler._replay, unet.precompute_time = logged_replay, logged_time
    fails = []
    try:
        with torch.no_grad(), insitu.Recorder('PLMS', sampler=True) as rec:
            if len(set(mts)) > 1:
                sampler.sample_rows(image, mts, cond, cond_scale=cs)
            else:
                sampler.sample(image, max_thres=mts[0], cond_images=cond, cond_scale=cs, use_tqdm=False)
        torch.cuda.synchronize()
    finally:
        del unet.precompute_time
    sch = row_schedule(mts, 50)
    recs = rec.recs
    R = sch.rounds
    if not (len(recs) == len(log) == R):
        fails.append(f'{name}: {len(recs)} updates and {len(log)} replays for {R} rounds')
        return dict(recs=recs, fails=fails, summary='')
    # static inputs of every replay: latents of the active rows (the round's x, round 1 evaluates round 0's x_prev), their time-feature
    # rows at each row's level, and exactly their conditioning (guided: then as many zero rows)
    order = torch.tensor(sch.order, device='cuda')
    bits = lambda t: t.float().contiguous().view(torch.int32)
    for j, (r, rp) in enumerate(zip(recs, log)):
        b = sch.batch[j]
        two = (lambda t: torch.cat((t, t))) if guided else (lambda t: t)
        x_need = recs[0].t['out'][:b] if j == 1 else r.t['x']
        c_need = cond.index_select(0, order[:b])
        c_need = torch.cat((c_need, torch.zeros_like(c_need))) if guided else c_need
        lv = torch.tensor(sch.level_idx[j] * (2 if guided else 1), device='cuda')
        checks = [('x', rp['sx'].reshape(len(rp['sx']), -1), two(x_need))] + [('cond', rp['sc'], c_need)] + \
                 [(f'time feature {k}', rp['sf'][k], tf[k].index_select(0, lv)) for k in tf]
        for what, got, want in checks:
            if got.shape != want.shape or not torch.equal(bits(got), bits(want)):
                fails.append(f'{name}: round {j}: the graph\'s static {what} rows are not the active rows\' {what}')
        if j >= 2 and not torch.equal(bits(r.t['x']), bits(recs[j - 1].t['out'][:b])):
            fails.append(f"{name}: round {j}: the update's x is not round {j - 1}'s x_prev")
        if r.s['rows'] != b:
            fails.append(f"{name}: round {j}: the update ran {r.s['rows']} rows, the schedule {b}")
    fails += [f'{name}: {m}' for m in insitu.plms_history_mismatches(recs, insitu.plms_expected_eps([rp['out'] for rp in log], sch.batch,
                                                                                                      guided, cs))]
    worst = _check(name, recs, fails)
    s = _summary(name, recs, [], worst, f'; {R} rounds, rows per round {sch.batch}')
    _drop(recs)
    del sampler, ddpm, log, tf
    return dict(recs=recs, fails=fails, summary=s)


@pytest.fixture(scope='module')
def sampler_runs():
    return {name: _sampler_run(name, mts, guided) for name, mts, guided in (
        ('PLMS sample, unguided', [0.07, 0.07], False), ('PLMS sample, guided (cond_scale 3)', [0.07, 0.07], True),
        ('PLMS sample_rows, two schedules', [0.05, 0.09], False))}


# ------------------------------------------------------------------------------------------------ tests
def test_unet_graph_replays_are_within_the_fp64_bound(graph_runs):
    fails = [f for r in graph_runs.values() for f in r['fails']]
    assert not fails, f'{len(fails)} failures:\n' + '\n'.join(fails[:40])


def test_eager_model_launches_are_within_the_fp64_bound(eager_runs):
    fails = [f for r in eager_runs.values() for f in r['fails']]
    assert not fails, f'{len(fails)} failures:\n' + '\n'.join(fails[:40])


def test_sampler_loop_updates_read_the_rounds_p_sample_assigns(sampler_runs):
    fails = [f for r in sampler_runs.values() for f in r['fails']]
    assert not fails, f'{len(fails)} failures:\n' + '\n'.join(fails[:40])


@pytest.mark.timeout(900)
def test_full_width_unet_graph_at_128x128_latents():
    from oracle import unet_oracle as uo
    r = _graph_run('graph FULL 128^2 batch 1', dataclasses.replace(uo.FULL, image_size=128), 1)
    assert not r['fails'], f"{len(r['fails'])} failures:\n" + '\n'.join(r['fails'][:40])


def test_catalogue_reaches_every_launch_kind(graph_runs, eager_runs, sampler_runs):
    runs = dict(graph_runs, **eager_runs, **sampler_runs)
    recs = [r for run in runs.values() for r in run['recs']]
    assert all(r.s.get('checked') for r in recs)
    ops_by_family = defaultdict(set)
    for r in recs:
        ops_by_family[r.family].add(r.op)
    print('\nin-situ catalogue:')
    for line in STATS.values():
        print('  ' + line)
    for fam, ops_ in sorted(ops_by_family.items()):
        print(f'  {fam}: ' + ', '.join(sorted(ops_)))
    unet_ops = {'conv2d_nhwc', 'groupnorm', 'layernorm', 'linear_small', 'mq_attention', 'gca_pool', 'gate_mlp_residual'}
    assert unet_ops | {'nchw_to_nhwc', 'nhwc_to_nchw', 'im2col4', 'concat2', 'pixel_shuffle_silu', 'time_fourier'} <= ops_by_family['UNet']
    assert {'conv2d_nhwc', 'groupnorm', 'softmax_rows', 'upsample2x', 'nchw_to_nhwc', 'nhwc_to_nchw'} <= ops_by_family['VAE']
    assert {'conv2d_nhwc'} <= ops_by_family['LPIPS'] and {'conv2d_nhwc', 'layernorm'} <= ops_by_family['EFT']
    graph_recs = [r for run in graph_runs.values() for r in run['recs']]
    # side-stream res_conv, split-K arena accumulates, in-place records, all inside the captured graphs
    assert any(r.s.get('side') and r.op == 'conv2d_nhwc' and 'res_conv' in r.label for r in graph_recs)
    assert any(r.s.get('arena') and r.s['plan_splits'] > 1 for r in graph_recs if r.op == 'conv2d_nhwc')   # split-K onto the arena
    assert any('accumulate' in r.alias for r in graph_recs)             # init_conv's x share onto cond_features: an in-place record
    # the VAE's three dynamic-weight GEMMs: q k^T, W_v h^T, P v
    for name, run in eager_runs.items():
        if name.startswith('VAE'):
            assert sum(r.s.get('dyn', False) for r in run['recs']) >= 3, name
    # every kernel name the tracer reported is a checked record's (each record's traced names are as many as its kernels, and no traced
    # name is left unattributed: asserted per configuration) or a listed C ABI launch's; these are the ones the models reach
    names = {n for r in recs for n in r.names}
    want = {'conv<16,swap>', 'conv<32,swap>', 'conv<64,swap>', 'conv<32>', 'conv<64>', 'conv<128>', 'gn_cluster_kernel<4>',
            'gn_cluster_kernel<8>', 'gn_stats_kernel', 'gn_stats_rows_kernel', 'gn_apply_cols_kernel', 'gn_apply_kernel', 'layernorm_rows_kernel',
            'linear_small_kernel<2>', 'linear_small_kernel<8>', 'mq_attention_keys_kernel', 'mq_attention_smem_kernel', 'cross_attention_kernel',
            'gca_logits_kernel', 'gca_pool_kernel', 'gca_pool_split_kernel', 'gate_mlp_residual_kernel', 'softmax_rows_kernel',
            'upsample2x_kernel', 'concat2_kernel', 'pixel_shuffle_silu_kernel', 'im2col_small_kernel', 'time_fourier_kernel',
            'nchw_to_nhwc_kernel', 'nhwc_to_nchw_kernel', 'sfb::plms_update_rows_kernel', 'sfb::plms_update_rows_cfg_kernel'}
    print('  traced kernels of checked records: ' + ', '.join(sorted(names)))
    assert want <= names, sorted(want - names)
    excluded = defaultdict(int)
    for run in eager_runs.values():
        for n, k, _ in run.get('unchecked', []):
            excluded[n] += k
    print('  not checked here (C ABI launches without a front end): ' + ', '.join(f'{n} x{k}' for n, k in sorted(excluded.items())))
    assert set(excluded) <= {'sfb_lpips_prep', 'sfb_lpips_prep_backward', 'sfb_relu_nhwc', 'sfb_maxpool2x2_nhwc', 'sfb_lpips_head',
                             'sfb_add_relu_mask', 'sfb_maxpool2x2_relu_backward_nhwc', 'sfb_act_inplace', 'sfb_seq_attention',
                             'sfb_maxpool3x3s2_nhwc', 'sfb_resize_bilinear_ac_nhwc', 'sfb_grid_sample_nhwc', 'sfb_eft_t1_tokens'}, sorted(excluded)
    print(f'  largest peak memory of a configuration: {PEAK[0] / 2 ** 30:.2f} GiB')
    assert PEAK[0] < 40 * 2 ** 30
