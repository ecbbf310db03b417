#!/usr/bin/env python
"""bench.py -- SparseFusion score-distillation steps/sec on H100 (BASELINE.json metric) + roofline + CPU baseline.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

A "step" is one iteration of the reference's distillation loop in SDS mode (sparsefusion/distillation.py:174-352, itr > 1000):
photometric sub-step on an input view + fusion sub-step on a cached target view (render 128x128 rays x (64+64) samples, bilinear x2,
VAE encode, PLMS sampler with n+1 UNet evaluations, n = min(int(100*max_thres), 50), VAE decode, L1*(1-alpha_bar) + 0.1*LPIPS-VGG loss,
backward, Adam).
Workload = BASELINE.json configs[2] (the configuration the metric is quoted on): 2 input views, 64 cached target views, 256^2 images,
32x32x4 latents, synthetic hydrant-style cameras, random-init networks of the reference's architecture, synthetic data.
With N GPUs every rank runs the step on its own target view (weak scaling over views) and the NGP gradients are all-reduced; `value`
counts view-steps of all ranks per second.  The max_thres sequence is seeded, identical for every arm and rank.

Printed JSON (rank 0): see the driver contract; `roofline` describes the dominant kernel (the wgmma conv/linear GEMM: it streams the
UNet's 1.6 GB of fp32 weights once per evaluation), `cpu_baseline` the oracle port of the same step on the host cores.
--dump-outputs DIR writes what the last timed step returned and left behind (its two losses and the NGP scene parameters) as DIR/<name>.npy,
float32; the workload is seeded, so runs with the same arguments see the same inputs and two builds can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

UNET_KW = dict(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
               layer_cross_attns=(False, False, False, False), cond_images_channels=256, attn_pool_text=False)
DDPM_KW = dict(channels=4, conditional_encoder=None, conditional_embed_dim=None, image_sizes=(32,), timesteps=500, cond_drop_prob=0.1,
               pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False,
               dynamic_thresholding_percentile=.68, clip_value=10)
UNET_WEIGHT_BYTES = 400_675_357 * 4          # SURVEY.md §8d: algorithmic HBM bytes per UNet evaluation (fp32 weights, read once)
UNET_FLOPS = 62.83e9                          # per sample at 32x32 latents
WORKLOAD = ('sds_distillation_step: BASELINE configs[2] -- 2 input views, 64 cached target views, 256x256 images, 32x32x4 latents, '
            '128x128 rays x (64+64) samples, PLMS(50), max_thres~U(0,0.99) seeded')


def workload_config(world, mean_calls):
    """`config` of the JSON line: the WORKLOAD only, built by one function so that both arms (ours and `--impl reference`) print the same object;
    what describes an arm's engine (precision mode, VAE engine, host threads) goes into the sibling `engine` object."""
    return {'workload': WORKLOAD,
            'parallelism': f'dp{world} over target views, ' + ('no collective' if world == 1 else 'ONE 7.46 MB NGP-gradient all-reduce per step'),
            'unet_evals_per_step_mean': None if mean_calls is None else round(float(mean_calls), 2),
            'l2': 'inputs larger than L2: each UNet evaluation streams 1.6 GB of fp32 weights (L2 = 50 MB)',
            'lpips': 'LPIPS-VGG perceptual term included in every arm (lambda 0.1, distillation.py:312-314) with seeded random weights -- the lpips '
                     'package and its pretrained weights are un-vendored'}


def max_thres_sequence(warmup, steps, seed=1234):
    """max_thres of every step (the reference draws U(0,1).clamp(0, .99) per step, distillation.py:303).  Warm-up steps get
    seeded uniform draws; the K timed steps get a seeded permutation of K equal strata of [0, .99], so that the mean PLMS
    length of ANY K-step run equals the expectation of the reference's draw instead of depending on K's luck.  The same
    list is used by the device-resident leg, the end-to-end leg, the reference arm and every rank."""
    g = torch.Generator().manual_seed(seed)
    warm = [float(torch.rand(1, generator=g).clamp(0.0, 0.99)) for _ in range(warmup)]
    order = torch.randperm(steps, generator=g).tolist()
    return warm + [0.99 * (o + 0.5) / steps for o in order]


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))), 'measured'
    except Exception:
        return {'hbm_gbs': 3350.0, 'bf16_tflops': 989.0}, 'fallback'     # H100 SXM data sheet (700 W): HBM3, dense BF16


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region"""
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap')

    def __init__(self, device_index):
        self.idx, self.proc, self.lines = device_index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', f'--query-gpu={self.Q}', '--format=csv,noheader,nounits', '-lms', '100', '-i', str(self.idx)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=lambda: self.lines.extend(self.proc.stdout), daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(',')]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(('hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap'), f[5:9]):
                if v.lower().startswith('active'):
                    reasons.add(name)
        return {'sm_mhz': float(np.median(sm)) if sm else None, 'sm_max_mhz': mx, 'reasons': sorted(reasons), 'samples': len(sm)}


# ------------------------------------------------------------------------------------------------------------------ GPU arm
def build_gpu(rank, world, device, views_per_step=None):
    from sparsefusion_b200.distillation import Distiller, SceneCache
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.synthetic import synthetic_scene
    from sparsefusion_b200.vldm import DDPM
    torch.manual_seed(0)          # identical random-init weights on every rank
    torch.cuda.manual_seed(0)
    unet = Unet(**UNET_KW)
    torch.nn.init.normal_(unet.get_parameter('final_conv.weight'), std=0.02)   # zero-init final conv would make eps == 0 (SURVEY §0.8)
    ddpm = DDPM(unets=(unet,), **DDPM_KW)
    torch.nn.init.normal_(ddpm.unets[0].get_parameter('final_conv.weight'), std=0.02)
    ddpm = ddpm.to(device)
    vae = AutoencoderKL().to(device).eval()
    opt = get_default_torch_ngp_opt()
    ngp = NeRFNetwork(opt)
    ngp.encoder.embeddings.data.uniform_(-0.5, 0.5)                             # SURVEY §8d C2: the default +-1e-4 is a featureless blob
    ngp = ngp.to(device).train()
    scene = SceneCache(**synthetic_scene(seed=0))
    pg = torch.distributed.group.WORLD if world > 1 else None
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    percep = PerceptualLoss('vgg', device=device, seed=0)                       # distillation.py:161 (random weights: see config.lpips)
    return Distiller, dict(ngp=ngp, vae=vae, vldm=ddpm, opt=opt), scene, dict(seed=0, rank=rank, world_size=world, process_group=pg, percep=percep,
                                                                            views_per_step=views_per_step)


def run_gpu(args):
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device (there is no CPU fallback for the product path)'
    torch.cuda.set_device(local)
    device = torch.device('cuda', local)
    if world > 1:
        torch.distributed.init_process_group('nccl', device_id=device)
    torch.backends.cudnn.allow_tf32 = True       # only matters for torch ops outside the product path (none in the timed region)
    torch.backends.cuda.matmul.allow_tf32 = True
    from sparsefusion_b200 import _lib, ops
    _lib.load()
    # step semantics: 1 GPU, no --views: the reference's iteration (one target view, two Adam updates) = BASELINE configs[2].  N GPUs: the view-
    # batched step of SURVEY §8e with V = N views (one per rank, ONE all-reduce, one Adam update) -- weak scaling over views; --views V fixes V.
    V = args.views if args.views else (world if world > 1 else None)
    Distiller, nets, scene, kw = build_gpu(rank, world, device, V)
    views_per_step = V if V else 1
    K, W = args.steps, args.warmup
    thres = max_thres_sequence(W, K)

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    def timed(dist, step_fn, n, offset):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step_fn(dist, 1001 + offset + i, thres[offset + i])
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=device)
        if world > 1:
            torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
        return float(ms)

    # ---- (1) device-resident: the scene cache lives in HBM before the timed region
    dist = Distiller(cache=scene.to(device), **nets, **kw)
    step_dev = lambda d, itr, mt: d.step(itr, max_thres=mt)
    for i in range(W):
        step_dev(dist, 1001 + i, thres[i])
    clocks = ClockSampler(local)
    l0 = ops.launch_count()
    if rank == 0:
        clocks.start()
    if dist.sampler._graph is not None:
        dist.sampler._graph.timing = []
    n_calls = []
    orig_step = step_dev
    last_losses = []

    def step_counting(d, itr, mt):
        last_losses[:] = orig_step(d, itr, mt)
        n_calls.append(d.last.get('unet_calls', 0))
    ms = timed(dist, step_counting, K, W)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last_losses, dist.ngp)
    clk = clocks.stop() if rank == 0 else None
    launches = ops.launch_count() - l0
    unet_events = dist.sampler._graph.timing if dist.sampler._graph is not None else []
    unet_ms = sum(a.elapsed_time(b) for a, b in unet_events)
    n_unet = len(unet_events)
    if dist.sampler._graph is not None:
        dist.sampler._graph.timing = None
    value = views_per_step * K / (ms / 1e3)       # view-steps of the whole job per second (one view per step on one GPU: == steps/s)

    # ---- (2) end to end through the public API with HOST buffers: pinned scene cache, per-step H2D of the step's views, D2H of the losses
    e2e_val, h2d, d2h = None, 0, 0
    if not args.no_e2e:
        from sparsefusion_b200.distillation import shard_views, step_views
        host = scene.pin()
        dist.cache = None
        bytes_per_step = [0]

        def step_e2e(d, itr, mt):
            g = d.gen.get_state()
            n_in, n_t = host.input_rgb.shape[0], host.target_features.shape[0]
            idx = int(torch.randperm(n_in, generator=d.gen)[0])
            perm = torch.randperm(n_t, generator=d.gen)
            d.gen.set_state(g)    # the step itself redraws the same indices
            if d.views_per_step is None:
                mine, need_in = [int(perm[(1 + d.rank) % n_t])], True
            else:
                mine = shard_views(step_views(perm, d.views_per_step), d.rank, d.world_size)
                need_in = (itr % d.world_size) == d.rank
            d.cache = _StagedCache(host, device, idx if need_in else None, mine)   # this step's views: pinned host -> HBM, inside the timed region
            bytes_per_step[0] = d.cache.bytes
            a, b = d.step(itr, max_thres=mt)
            return float(a.item()) + float(b.item())   # D2H read of the step's losses (the reference logs loss.item(), :249,:349)
        for i in range(2):
            step_e2e(dist, 1001 + i, thres[i % max(1, W)])
        ms_e2e = timed(dist, step_e2e, K, W)        # same itr numbers and max_thres list as the device-resident leg
        e2e_val, h2d, d2h = views_per_step * K / (ms_e2e / 1e3), bytes_per_step[0], 8

    # ---- (2b) BASELINE configs[3] as SURVEY §8d/§8e specify it: a FIXED 64-view minibatch step sharded over the ranks (strong scaling: every rank
    # distils 64/N views per step as UNet / VAE batches, one all-reduce, one Adam update) -- all ranks take part
    c4 = None
    if not args.no_c4:
        try:
            c4 = c4_leg(Distiller, nets, scene, kw, device, rank, world, barrier)
        except Exception as e:   # noqa: BLE001  (the headline line must survive a failure of an auxiliary leg)
            c4 = {'error': f'{type(e).__name__}: {e}'[:300]}

    # ---- (3) roofline of the dominant kernel: instrumented eager UNet evaluations (CUDA events around every conv launch)
    roof = None
    if rank == 0:
        pk, pk_kind = peaks()
        unet = nets['vldm'].unets[0]
        x = torch.randn(1, 4, 32, 32, device=device)
        c = torch.randn(1, 256, 32, 32, device=device)
        t = torch.full((1,), 0.3, device=device)
        feat = unet.precompute_cond(c)       # the sampler evaluates the conditioning map's share of init_conv once per run, not per evaluation
        tfeat = unet.precompute_time(t)      # ... and the noise-level branch (time MLPs) once per run for all levels
        for _ in range(2):
            unet.forward(x, None, cond_features=feat, time_features=tfeat)
        torch.cuda.synchronize()
        import ctypes
        tbuf = torch.zeros(4097, dtype=torch.int64, device=device)
        _lib.call('sfb_trace_begin', tbuf.data_ptr(), 4096)     # kernel names in launch order (+ stamps) for the in-graph measurement below
        par0 = unet.parallel_res_conv
        unet.parallel_res_conv = False           # kernel names in single-chain order
        unet.forward(x, None, cond_features=feat, time_features=tfeat)
        unet.parallel_res_conv = par0
        torch.cuda.synchronize()
        nbuf = ctypes.create_string_buffer(1 << 20)
        _lib.load().sfb_trace_names(nbuf, len(nbuf))
        names = nbuf.value.decode().split('\n')[:-1]
        _lib.call('sfb_conv_prof_enable', 1)
        reps = 5
        for _ in range(reps):
            torch.cuda._sleep(int(2e7))   # ~10 ms of GPU idle-spin: the CPU enqueues the whole eager evaluation behind it, so the
            unet.forward(x, None, cond_features=feat, time_features=tfeat)   # events around each conv launch measure kernel time, not CPU launch gaps
            torch.cuda.synchronize()
        tot, nl, wb, fl = ctypes.c_double(), ctypes.c_int(), ctypes.c_double(), ctypes.c_double()
        _lib.load().sfb_conv_prof_collect(ctypes.byref(tot), ctypes.byref(nl), ctypes.byref(wb), ctypes.byref(fl))
        _lib.call('sfb_conv_prof_enable', 0)
        conv_ms_per_eval = tot.value / reps
        per_launch_us = 1e3 * tot.value / max(1, nl.value)
        achieved = (wb.value / reps) / (conv_ms_per_eval * 1e-3) / 1e9
        # the same kernels inside the replayed CUDA graph of the timed region: %globaltimer stamp of every kernel right after its dependency
        # wait (sfb_trace_begin); consecutive stamps = chain cost of a kernel, launch / dependency latency included
        in_graph = None
        if dist.sampler._graph is not None:
            from sparsefusion_b200.imagen_pytorch import UnetGraph
            flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
            # (a) the graph the timed region replays (res_conv on a parallel branch): first-to-last kernel of one evaluation
            runner = dist.sampler._graph
            all_us = []
            for _ in range(5):
                flush.zero_()
                tbuf.zero_()
                runner(x, t, c, new_cond=False, time_features=tfeat)
                torch.cuda.synchronize()
                k = int(tbuf[0])
                stamps = np.sort(tbuf[1:1 + k].cpu().numpy().astype('int64'))
                all_us.append(float(stamps[-1] - stamps[0]) / 1e3)
            # (b) per-kernel attribution needs a single chain: the same evaluation captured without the parallel branch
            par = unet.parallel_res_conv
            unet.parallel_res_conv = False
            try:
                chain = UnetGraph(unet)
                chain(x, t, c, new_cond=True, time_features=tfeat)
                conv_us, chain_us = [], []
                for _ in range(5):
                    flush.zero_()
                    tbuf.zero_()
                    chain(x, t, c, new_cond=False, time_features=tfeat)
                    torch.cuda.synchronize()
                    k = int(tbuf[0])
                    stamps = tbuf[1:1 + k].cpu().numpy().astype('int64')
                    if k != len(names):
                        break
                    iv = np.diff(stamps) / 1e3
                    conv_us.append(float(sum(d for nm, d in zip(names[:-1], iv) if nm.startswith('conv<'))))
                    chain_us.append(float(iv.sum()))
            finally:
                unet.parallel_res_conv = par
            if conv_us:
                cu = float(np.median(conv_us))
                n_conv = sum(1 for nm in names if nm.startswith('conv<'))
                in_graph = {'kernels_per_eval': len(names), 'conv_launches_per_eval': n_conv, 'conv_us_per_eval': round(cu, 1),
                            'eval_us_single_chain': round(float(np.median(chain_us)), 1),
                            'eval_us_first_to_last_kernel': round(float(np.median(all_us)), 1), 'achieved_GBps': round((wb.value / reps) / (cu * 1e-6) / 1e9, 1),
                            'frac': round((wb.value / reps) / (cu * 1e-6) / 1e9 / pk['hbm_gbs'], 4),
                            'note': 'conv_us_per_eval / achieved from a single-chain capture of the same evaluation (per-kernel attribution); '
                                    'eval_us_first_to_last_kernel from the graph the timed region replays (res_conv on a parallel branch)'}
        _lib.call('sfb_trace_end')
        traffic, traffic_src = None, 'not measured (no DRAM counter capture of this kernel)'
        roof = {'kernel': 'conv_gemm_kernel (wgmma 3xTF32 implicit-GEMM conv/linear, weights streamed from HBM)', 'bound': 'hbm',
                'achieved': round(achieved, 1),
                'peak': pk['hbm_gbs'], 'peak_source': f'{pk_kind} MEASURED_PEAKS.json hbm_gbs (copy bandwidth)', 'unit': 'GB/s',
                'frac': round(achieved / pk['hbm_gbs'], 4), 'traffic': traffic, 'traffic_source': traffic_src,
                'algorithmic_bytes_per_launch': int(wb.value / max(1, nl.value)),
                'algorithmic_bytes_per_eval': int(wb.value / reps), 'launches_per_eval': nl.value // reps,
                'avg_launch_us': round(per_launch_us, 2), 'conv_ms_per_unet_eval': round(conv_ms_per_eval, 4),
                'tensor_tflops_equiv': round((fl.value / reps) / (conv_ms_per_eval * 1e-3) / 1e12, 2),
                'in_graph': in_graph,
                'unet_eval_ms_in_timed_region': round(unet_ms / max(1, n_unet), 4), 'unet_evals_in_timed_region': n_unet,
                'unet_share_of_step': round(unet_ms / ms, 4),
                'note': 'B=1 UNet evaluation is weight-streaming bound (SURVEY §7): achieved = fp32 weight bytes of the conv/linear layers '
                        'per evaluation / summed conv-kernel time per evaluation (CUDA events around each launch, eager pass after the timed region)'}

    # ---- (4) CPU baseline (oracle port) on the host cores, rank 0, N == 1 only
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu:
        cpu = cpu_baseline(float(np.mean(n_calls)) if n_calls else 38.0)

    c5 = None
    if args.c5 or (world == 8 and not args.no_c5):
        c5 = c5_leg(device, rank, world, barrier)
    c2 = gref = None
    if rank == 0 and world == 1 and not args.no_c2:
        try:
            c2 = c2_leg(nets['ngp'], device)
        except Exception as e:   # noqa: BLE001
            c2 = {'error': f'{type(e).__name__}: {e}'[:300]}
    if rank == 0 and world == 1 and not args.no_gpuref:
        try:
            gref = gpu_reference_leg(device, float(np.mean(n_calls)) if n_calls else 38.25, ms / K)
        except Exception as e:   # noqa: BLE001
            gref = {'error': f'{type(e).__name__}: {e}'[:300]}

    if rank == 0:
        out = {'metric': 'distillation-steps/sec (2-view, 256^2, 64 rendered views)', 'value': round(value, 4), 'unit': 'steps/s', 'n_gpus': world,
               'steps': K, 'warmup': W, 'ms_per_step': round(ms / K, 3), 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
               'dtype': 'f32 (UNet GEMMs: 3xTF32 error-compensated tensor-core passes, fp32 accumulate; NGP: fp32)', 'data': 'synthetic',
               'config': workload_config(world, float(np.mean(n_calls)) if n_calls else None),
               'engine': {'vae': 'sm_90a engine (wgmma 3xTF32 convolutions / attention GEMMs, NHWC) -- SURVEY §8f row 1', 'precision_mode': ops.get_precision()},
               'clocks': clk, 'gpu_launches': int(launches),
               'e2e': None if e2e_val is None else {'value': round(e2e_val, 4), 'unit': 'steps/s', 'h2d_bytes_per_step': int(h2d), 'd2h_bytes_per_step': int(d2h)},
               'roofline': roof, 'cpu_baseline': cpu,
               # `value` counts view-steps (target views distilled per second over all ranks); a loop iteration (one scene, one parameter update
               # sequence) takes ms_per_step regardless of N in this weak-scaling default -- both rates are stated (SURVEY §8d)
               'views_per_step': views_per_step, 'views_per_s': round(value, 4), 'optimizer_steps_per_s': round(K / (ms / 1e3), 4),
               'step_semantics': ('reference iteration: photometric update, then fusion update on ONE target view (distillation.py:244-247,:345-352)' if V is None else
                                  f'view-batched step (SURVEY 8e): grad(photometric) + mean over {V} target views, {V // world if V >= world else 1} per rank as one UNet/VAE batch, '
                                  'ONE all-reduce and ONE Adam update per step'),
               'c4_fixed_views': c4, 'c2_render': c2, 'c5_large_latents': c5, 'gpu_reference': gref}
        print(json.dumps(out), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


def dump_outputs(out_dir, losses, ngp):
    """the last timed step's results as its caller receives them: the two losses Distiller.step returns and the NGP parameters it updated"""
    os.makedirs(out_dir, exist_ok=True)
    arrays = {'loss_photometric': losses[0], 'loss_fusion': losses[1]}
    arrays.update({'ngp.' + k: v for k, v in ngp.state_dict().items() if v.is_floating_point()})
    total = 0
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy()
        total += a.nbytes
        np.save(os.path.join(out_dir, name + '.npy'), a)
    assert total <= 64 << 20, f'{total} bytes of outputs'


class _StagedCache:
    """SceneCache view for the end-to-end leg: the step's views are copied host(pinned) -> device when the step starts"""

    def __init__(self, host, device, in_idx, tgt_views):
        self.bytes = 0

        def stage(t, idxs):
            out = {}
            for i in idxs:
                d = t[i:i + 1].to(device, non_blocking=True)
                self.bytes += d.numel() * d.element_size()
                out[i] = d
            return _Views(out, t.shape, device)
        ins = [] if in_idx is None else [in_idx]
        self.input_rgb, self.input_mask = stage(host.input_rgb, ins), stage(host.input_mask, ins)
        self.input_rays_o, self.input_rays_d = stage(host.input_rays_o, ins), stage(host.input_rays_d, ins)
        self.target_features = stage(host.target_features, tgt_views)
        self.target_rays_o, self.target_rays_d = stage(host.target_rays_o, tgt_views), stage(host.target_rays_d, tgt_views)
        self.target_eft_image = _Views({}, host.target_eft_image.shape, device)   # not read in SDS mode


class _Views:
    """the staged rows of one SceneCache field, addressed like the full tensor (t[i], t[i:i+1], t[[i, j, ...]])"""

    def __init__(self, rows, shape, device):
        self.rows, self.shape, self.device = rows, tuple(shape), device

    def __getitem__(self, key):
        if isinstance(key, slice):
            assert key.stop == key.start + 1, 'staged view: one-row slices only'
            return self.rows[key.start]
        if isinstance(key, (list, tuple)):
            return torch.cat([self.rows[int(k)] for k in key])
        return self.rows[int(key)][0]


# ------------------------------------------------------------------------------------------------------------------ auxiliary legs
def c4_leg(Distiller, nets, scene, kw, device, rank, world, barrier, views=64, warmup=2, steps=4):
    """fixed `views`-view minibatch step over `world` ranks: ms per step, views/s, optimiser steps/s (max over ranks, CUDA events)"""
    dist = Distiller(cache=scene.to(device), **nets, **dict(kw, views_per_step=views))
    thres = max_thres_sequence(warmup, steps, seed=4321)
    for i in range(warmup):
        dist.step(1001 + i, max_thres=thres[i])
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    calls = []
    for i in range(steps):
        dist.step(1001 + warmup + i, max_thres=thres[warmup + i])
        calls.append(dist.last.get('unet_calls', 0))
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device=device)
    if world > 1:
        torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
    ms = float(ms) / steps
    per_rank = views // world
    return {'workload': f'BASELINE configs[3] (SURVEY 8d C4): one optimiser step on a FIXED {views}-view minibatch, views sharded {per_rank} per rank, UNet / VAE batch '
                        f'{min(per_rank, dist.max_batch)}, per-view RNG keyed by (step, view), one all-reduce per step', 'views': views, 'n_gpus': world,
            'steps': steps, 'warmup': warmup, 'ms_per_step': round(ms, 2), 'views_per_s': round(views / (ms / 1e3), 3),
            'optimizer_steps_per_s': round(1e3 / ms, 4), 'unet_evals_per_view_mean': round(float(np.mean(calls)), 2), 'scaling': 'strong'}


def c2_leg(ngp, device, n_views=64, hw=256):
    """BASELINE configs[1] (SURVEY §8d C2): forward render of the NGP field, 64 views at 256x256, train-mode sampling (perturb + inverse-CDF noise),
    16 384-ray chunks like render_batched (renderer_df.py:681-718).  FLOPs per sample point: 13.3 k (SURVEY §8d: MLP 12.8 k + interpolation 0.5 k)."""
    from sparsefusion_b200.synthetic import camera_rays, circle_cameras
    cams = circle_cameras(n_views)
    rays = [tuple(torch.from_numpy(a).to(device) for a in camera_rays(c, hw, hw)) for c in cams]
    ngp.train()
    out = {}
    for tag, chunk in (('chunk_16384', 128 * 128), ('whole_view', hw * hw)):
        kw = dict(batched=True, max_ray_batch=chunk, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', num_steps=64, upsample_steps=64)
        for ro, rd in rays[:2]:
            ngp.render_batched(ro[None], rd[None], **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for ro, rd in rays:
            ngp.render_batched(ro[None], rd[None], **kw)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        n_rays = n_views * hw * hw
        out[tag] = {'ms': round(ms, 2), 'rays_per_s': round(n_rays / (ms / 1e3), 1), 'fp32_tflops': round(n_rays * 128 * 13.3e3 / (ms / 1e3) / 1e12, 2)}
    out['workload'] = f'{n_views} views x {hw}x{hw} rays x (64+64) samples, forward only (no_grad), fused run() renderer'
    out['note'] = ('fully fused render is FP32-SIMT / L2-gather bound, not HBM bound (SURVEY 8d): the meaningful fractions are fp32_tflops against the '
                   '~80 TFLOP/s FP32 SIMT peak; each point is evaluated once (the reference evaluates the field twice per point)')
    return out


def c5_leg(device, rank, world, barrier, steps=2, warmup=1):
    """BASELINE configs[4] (SURVEY §8d C5): the iteration at 128x128x4 latents -- 1024x1024 images through the VAE and LPIPS, 512x512 rays x (64+64) samples,
    UNet 1004 GFLOP per evaluation with 256 x 259 attention at the lowest stage, 6 input views -- one target view per GPU per step (reference semantics on
    every rank, replicas: no collective inside the leg, so a failing rank cannot stall the others); reports the max over ranks"""
    from sparsefusion_b200.distillation import Distiller, SceneCache
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.synthetic import synthetic_scene
    from sparsefusion_b200.vldm import DDPM
    ms, err, calls = float('nan'), None, []
    try:
        torch.manual_seed(0)
        unet = Unet(**UNET_KW)
        torch.nn.init.normal_(unet.get_parameter('final_conv.weight'), std=0.02)
        ddpm = DDPM(unets=(unet,), **dict(DDPM_KW, image_sizes=(128,)))
        torch.nn.init.normal_(ddpm.unets[0].get_parameter('final_conv.weight'), std=0.02)
        ddpm = ddpm.to(device)
        vae = AutoencoderKL().to(device).eval()
        opt = get_default_torch_ngp_opt()
        opt.w = opt.h = 512
        ngp = NeRFNetwork(opt)
        ngp.encoder.embeddings.data.uniform_(-0.5, 0.5)
        ngp = ngp.to(device).train()
        scene = SceneCache(**synthetic_scene(n_input=6, n_target=4, image_size=1024, latent=128, render_hw=512, seed=rank)).to(device)
        dist = Distiller(ngp, vae, ddpm, opt, scene, seed=rank, percep=PerceptualLoss('vgg', device=device, seed=0))
        thres = [0.13] * warmup + [0.25, 0.49][:steps]          # 26 + 50 UNet evaluations over the two timed steps: mean 38 = the expectation of the reference's draw
        for i in range(warmup):
            dist.step(1001 + i, max_thres=thres[i])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            a, b = dist.step(1001 + warmup + i, max_thres=thres[warmup + i])
            calls.append(dist.last.get('unet_calls', 0))
        e1.record()
        torch.cuda.synchronize()
        if not (torch.isfinite(a) and torch.isfinite(b)):
            raise RuntimeError('non-finite loss')
        ms = e0.elapsed_time(e1) / steps
        del dist, scene, ngp, vae, ddpm, unet
        torch.cuda.empty_cache()
    except Exception as e:   # noqa: BLE001
        err = f'{type(e).__name__}: {e}'[:300]
    t = torch.tensor([ms if err is None else -1.0], device=device)
    if world > 1:
        gathered = [torch.zeros_like(t) for _ in range(world)]
        torch.distributed.all_gather(gathered, t)
        allms = [float(g) for g in gathered]
    else:
        allms = [float(t)]
    ok = [m for m in allms if m > 0]
    out = {'workload': 'BASELINE configs[4] (SURVEY 8d C5): 6 input views, 128x128x4 latents (1024x1024 images, 512x512 rays x 128 samples), one target view per GPU per '
                       'step, reference iteration on every rank (replicas)', 'n_gpus': world, 'steps': steps, 'warmup': warmup, 'ranks_ok': len(ok),
           'unet_evals_per_step_mean': round(float(np.mean(calls)), 2) if calls else None, 'unet_gflop_per_eval': 1004.3}
    if len(ok) == world:
        worst = max(ok)
        out.update({'ms_per_step': round(worst, 1), 'views_per_s': round(world / (worst / 1e3), 4), 'steps_per_s_per_gpu': round(1e3 / worst, 4)})
    if err is not None:
        out['error_rank%d' % rank] = err
    return out


def gpu_reference_leg(device, mean_calls, our_ms_per_step):
    """the "reference GPU build" comparator (BASELINE.md §3.4): the eager-PyTorch restatement of the reference's step on the SAME GPU -- cuDNN / cuBLAS
    with TF32 on (what torch 1.11 defaulted to), the reference's own CUDA operators from oracle/_ref where they exist -- timed component by
    component and assembled into a step (2 renders fwd+bwd + n+1 UNet evaluations + VAE + LPIPS).  A baseline, not the product."""
    from oracle import gpu_reference
    r = gpu_reference.time_step_components(device, mean_calls)
    r['ours_ms_per_step'] = round(our_ms_per_step, 3)
    r['speedup_vs_gpu_reference'] = round(r['ms_per_step'] / our_ms_per_step, 3)
    return r


# ------------------------------------------------------------------------------------------------------------------ CPU arm
def cpu_baseline(mean_calls):
    """rank 0, N == 1: ONE whole step of the oracle port on the host cores at the run's mean PLMS length (plus a 2-evaluation warm-up step)"""
    port = CpuWholeStep()
    port.step(1001, 0.013)
    n = int(round(mean_calls)) - 1
    dt, tm = port.step(1002, min(0.99, (n + 0.5) / 100.0))
    return {'value': round(1.0 / dt, 6), 'unit': 'steps/s', 'cores': port.threads, 'kind': 'port',
            'sample': f'ONE whole step of the oracle port on {port.threads} host threads (fixed count; {os.cpu_count()}-thread host): {dt:.2f} s with {tm["unet_calls"]} FULL-UNet '
                      f'evaluations ({tm["plms"]:.2f} s), photometric sub-step {tm["substep_a"]:.2f} s, fusion render {tm["render_b"]:.2f} s, VAE {tm.get("vae_encode", 0) + tm.get("vae_decode", 0):.2f} s; '
                      'nothing sampled or scaled. The reference has no CPU path for the NGP render (CUDA-only extensions).'}


REF_THREADS = 16     # intra-op threads of the CPU arm: fixed (a start-up probe picked 16 or 32 from run to run); more threads than this slow the 32x32
                     # feature maps down (tools/cpu_threads_probe.py)


class CpuWholeStep:
    """the reference's iteration restated on the host cores (oracle/distill_oracle.OracleDistiller: FULL UNet, 128x128 rays, 256x256 VAE, LPIPS),
    run as WHOLE steps -- nothing sampled or scaled"""

    def __init__(self):
        from oracle import distill_oracle as do, lpips_oracle as lo, ngp_oracle as no, unet_oracle as uo, vae_oracle as vo
        from sparsefusion_b200.distillation import SceneCache
        self.threads = max(1, min(REF_THREADS, os.cpu_count() or 1))
        torch.set_num_threads(self.threads)
        self.uo = uo
        cache = SceneCache(**do.synthetic_scene(seed=0))
        self.n_rays = cache.input_rays_o.shape[1]
        self.dist = do.OracleDistiller(no.make_field_params(seed=0), vo.TorchVAE(vo.make_params(seed=0)), uo.make_params(uo.FULL, seed=0), uo.FULL, cache,
                                       seed=0, percep=lo.PerceptualLoss(lo.make_params(0)))
        self.rng = np.random.default_rng(0)

    def step(self, itr, max_thres):
        n = self.n_rays
        noise = lambda k: (torch.from_numpy(self.rng.random((n, 64), dtype=np.float32)), torch.from_numpy(self.rng.random((n, 64), dtype=np.float32)))
        t0 = time.perf_counter()
        self.dist.step(itr, noise, self.uo.NoiseSource(seed=itr), max_thres=max_thres)
        return time.perf_counter() - t0, dict(self.dist.timing)


def run_reference(args):
    """`--impl reference`: the reference's CPU implementation of the step = the oracle port (the reference cannot be imported on the GPU box and has
    no CPU render path of its own), whole steps on REF_THREADS host threads.  A whole step takes 10-25 s; the K timed steps are all run when they
    fit the time budget (SFB_REF_BUDGET_S, default 420 s: K = 20 takes ~330 s, so the line's steps x ms_per_step is time really spent); on a slower
    host only as many as fit are run (at least one) and the remaining ones are filled in from the measured components of those runs with their own
    PLMS length (n+1 UNet evaluations) -- the line says how many of each (`whole_steps_measured`, `extrapolated_steps`, `wall_s`)."""
    rank = int(os.environ.get('RANK', 0))
    if rank != 0:
        return
    K, W = args.steps, args.warmup
    thres = max_thres_sequence(W, K)
    calls = [min(int(t * 100), 50) + 1 if t >= 0.01 else 0 for t in thres[W:W + K]]
    # 20 whole steps take ~330 s on the pool's 128-thread hosts: nothing extrapolated by default at N = 1.  Under torchrun (the driver's scaling run
    # repeats this arm at every N although only rank 0 works) the budget is 150 s: the same single-host number, 8 whole steps + declared fill-in
    budget = float(os.environ.get('SFB_REF_BUDGET_S', 420 if int(os.environ.get('WORLD_SIZE', 1)) == 1 else 150))
    port = CpuWholeStep()
    t_begin = time.perf_counter()
    if W > 0:       # one short warm-up step (first-touch allocations, thread pool): 2 UNet evaluations
        port.step(1000 + 1, 0.013)
    whole, comps = {}, []
    for i in range(K):
        if i > 0 and time.perf_counter() - t_begin > budget:
            break
        dt, tm = port.step(1001 + W + i, thres[W + i])
        whole[i] = dt
        comps.append((tm['total'] - tm['plms'], tm['plms'] / max(1, tm['unet_calls']), tm))
    fixed = float(np.mean([c[0] for c in comps]))             # everything but the sampler: 2 renders fwd+bwd, VAE, LPIPS, Adam
    per_call = float(np.mean([c[1] for c in comps if c[2]['unet_calls'] > 0] or [0.0]))
    per_step = [whole.get(i, fixed + calls[i] * per_call) for i in range(K)]
    step_s = float(np.mean(per_step))
    val = 1.0 / step_s
    norm = [whole[i] / max(1e-9, fixed + calls[i] * per_call) for i in whole]      # measured / modelled, per whole step: the spread of the measurement
    out = {'impl': 'reference', 'metric': 'distillation-steps/sec (2-view, 256^2, 64 rendered views)', 'value': round(val, 6), 'unit': 'steps/s',
           'n_gpus': int(os.environ.get('WORLD_SIZE', 1)), 'steps': K, 'warmup': W, 'ms_per_step': round(step_s * 1e3, 1), 'higher_is_better': True,
           'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
           'config': workload_config(int(os.environ.get('WORLD_SIZE', 1)), float(np.mean(calls)) if calls else None),
           'engine': {'host': f'CPU, {port.threads} intra-op threads (fixed; the fastest count measured on the {os.cpu_count()}-thread host class); rank 0 only'},
           'whole_steps_measured': len(whole), 'extrapolated_steps': K - len(whole), 'extrapolated': len(whole) < K,
           'whole_step_s': {'min': round(min(whole.values()), 3), 'max': round(max(whole.values()), 3), 'measured_over_model_min': round(min(norm), 3),
                            'measured_over_model_max': round(max(norm), 3)},
           'components_s': {'all_but_sampler': round(fixed, 3), 'per_unet_eval': round(per_call, 4)}, 'wall_s': round(time.perf_counter() - t_begin, 1),
           'cpu_baseline': {'value': round(val, 6), 'unit': 'steps/s', 'cores': port.threads, 'kind': 'port',
                            'sample': f'{len(whole)} WHOLE steps run on the host cores (oracle port: 2 full-size renders fwd+bwd, n+1 FULL-UNet evaluations, VAE '
                                      f'enc/dec, LPIPS fwd/bwd, Adam), the other {K - len(whole)} of the {K} timed steps filled in from those runs\' measured components '
                                      'with their own PLMS length; the reference cannot be imported on this box and has no CPU render path'},
           'e2e': {'value': round(val, 6), 'unit': 'steps/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--no-e2e', dest='no_e2e', action='store_true')
    ap.add_argument('--no-cpu', dest='no_cpu', action='store_true')
    ap.add_argument('--no-c4', dest='no_c4', action='store_true', help='skip the fixed 64-view minibatch leg')
    ap.add_argument('--no-c2', dest='no_c2', action='store_true', help='skip the 64-view 256x256 render leg')
    ap.add_argument('--no-gpuref', dest='no_gpuref', action='store_true', help='skip the eager-PyTorch-on-GPU reference leg')
    ap.add_argument('--c5', action='store_true', help='run the 128x128-latent leg (BASELINE configs[4]); on by default with 8 GPUs')
    ap.add_argument('--no-c5', dest='no_c5', action='store_true', help='skip it with 8 GPUs')
    ap.add_argument('--views', type=int, default=0, help='target views per optimiser step (view-batched step); default: 1 on one GPU, N on N GPUs')
    ap.add_argument('--dump-outputs', dest='dump_outputs', default=None, metavar='DIR',
                    help='write the last timed step\'s losses and NGP parameters to DIR/<name>.npy (float32)')
    a = ap.parse_args()
    a.warmup = max(a.warmup, 3) if a.impl == 'ours' else a.warmup
    if a.impl == 'reference':
        run_reference(a)
    else:
        run_gpu(a)
