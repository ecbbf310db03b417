"""Per-kernel timings on the GPU box (CUDA events, L2 flushed between iterations) -> gpurun_out/microbench.json.
Used to pick tile/split heuristics; not the headline bench."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sparsefusion_b200 import ops  # noqa: E402

FLUSH = None


def timeit(fn, iters=10, warmup=3, flush=True):
    global FLUSH
    if FLUSH is None:
        FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush:
            FLUSH.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def conv_cases():
    # (name, NB scale, H, Cin, Cout, K, stride)
    base = [('init3', 32, 260, 128, 3, 1), ('init7', 32, 260, 64, 7, 1), ('init15', 32, 260, 64, 15, 1), ('d0.conv3', 32, 256, 256, 3, 1),
            ('d0.down4s2', 32, 256, 256, 4, 2), ('d1.conv3', 16, 256, 256, 3, 1), ('d2.conv3', 8, 512, 512, 3, 1),
            ('d3.conv3', 4, 1024, 1024, 3, 1), ('u0.conv3', 4, 2048, 1024, 3, 1), ('u0.res1x1', 4, 2048, 1024, 1, 1),
            ('u1.conv3', 8, 1536, 1024, 3, 1), ('u2.conv3', 16, 768, 512, 3, 1), ('u3.conv3', 32, 512, 256, 3, 1),
            ('ff1x1', 4, 1024, 2048, 1, 1), ('ps1x1', 4, 1024, 4096, 1, 1), ('final', 32, 256, 4, 3, 1)]
    return base


def unet_bench(out):
    import numpy as np
    from sparsefusion_b200 import _lib
    if 'nopdl' in sys.argv:
        _lib.call('sfb_set_pdl', 0)
    if 'nofuse' in sys.argv:
        _lib.call('sfb_set_fusion', 0)
    for a in sys.argv:
        if a.startswith('fuse='):
            _lib.call('sfb_set_fusion', int(a[5:], 0))
    from sparsefusion_b200.imagen_pytorch import Unet, UnetGraph
    unet = Unet(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
                layer_cross_attns=(False,) * 4, cond_images_channels=256, attn_pool_text=False, cond_on_z=False, conditional_embed_dim=None).cuda()
    torch.nn.init.normal_(unet.get_parameter('final_conv.weight'), std=0.02)
    out['unet'] = {}
    for mode in (('tf32x3',) if 'x3only' in sys.argv else ('tf32x3', 'tf32')):
        ops.set_precision(mode)
        unet.prepare()
        for nb in ((16, 32) if 'nb32' in sys.argv else (1, 8, 16) if 'nb16' in sys.argv else (1, 8)):
            x, cond, t = torch.randn(nb, 4, 32, 32, device='cuda'), torch.randn(nb, 256, 32, 32, device='cuda'), torch.full((nb,), 0.3, device='cuda')
            eager = timeit(lambda: unet.forward(x, t, cond_images=cond), iters=5, warmup=2, flush=False)
            runner = UnetGraph(unet)
            tfeat = unet.precompute_time(t)
            graph = timeit(lambda: runner(x, t, cond, new_cond=False, time_features=tfeat), iters=20, warmup=3, flush=True)
            rec = dict(eager_ms=round(eager, 3), graph_ms=round(graph, 3), tflops=round(62.83e-3 * nb / graph, 1), weight_gbs=round(1602.7 / graph, 1))
            out['unet'][f'{mode}_nb{nb}'] = rec
            print('unet', mode, nb, rec, flush=True)
    ops.set_precision('tf32x3')


def unet_trace(out):
    """in-situ chain cost of every UNet kernel inside the replayed graph (sfb_trace_begin): stamp[i+1] - stamp[i]"""
    global FLUSH
    import ctypes
    import collections
    from sparsefusion_b200 import _lib
    if 'nopdl' in sys.argv:
        _lib.call('sfb_set_pdl', 0)
    if 'nocarve' in sys.argv:
        _lib.call('sfb_set_pdl', 3)
    if 'padsmem' in sys.argv:
        _lib.call('sfb_set_pdl', 5)
    for a in sys.argv:
        if a.startswith('fuse='):
            _lib.call('sfb_set_fusion', int(a[5:], 0))
    from sparsefusion_b200.imagen_pytorch import Unet, UnetGraph
    unet = Unet(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
                layer_cross_attns=(False,) * 4, cond_images_channels=256, attn_pool_text=False, cond_on_z=False, conditional_embed_dim=None).cuda()
    torch.nn.init.normal_(unet.get_parameter('final_conv.weight'), std=0.02)
    ops.set_precision('tf32x3')
    unet.parallel_res_conv = 'parallel' in sys.argv      # per-kernel attribution needs a single dependency chain
    unet.prepare()
    hw = 32
    for a in sys.argv:
        if a.startswith('hw='):
            hw = int(a[3:])
    x, cond, t = torch.randn(1, 4, hw, hw, device='cuda'), torch.randn(1, 256, hw, hw, device='cuda'), torch.full((1,), 0.3, device='cuda')
    runner = UnetGraph(unet)
    for _ in range(3):
        runner(x, t, cond)
    torch.cuda.synchronize()
    cap = 4096
    buf = torch.zeros(cap + 1, dtype=torch.int64, device='cuda')
    pbuf = torch.zeros(1 + 8 * 128, dtype=torch.int64, device='cuda')
    _lib.call('sfb_trace_begin', buf.data_ptr(), cap)
    tfeat = unet.precompute_time(t)
    feat = unet.precompute_cond(cond)
    _lib.call('sfb_trace_begin', buf.data_ptr(), cap)     # restart: names of the main evaluation only
    buf.zero_()
    unet.forward(x, None, cond_features=feat, time_features=tfeat)            # names in launch order (same sequence as the captured main graph)
    torch.cuda.synchronize()
    n_eager = int(buf[0])
    nbuf = ctypes.create_string_buffer(1 << 20)
    _lib.load().sfb_trace_names(nbuf, len(nbuf))
    names = nbuf.value.decode().split('\n')[:-1]
    _lib.call('sfb_conv_phase_trace', pbuf.data_ptr(), 128)
    runs = []
    for _ in range(5):
        if FLUSH is None:
            FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
        FLUSH.zero_()
        buf.zero_()
        pbuf.zero_()
        torch.cuda.synchronize()
        runner(x, t, cond, new_cond=False, time_features=tfeat)
        torch.cuda.synchronize()
        k = int(buf[0])
        runs.append(buf[1:1 + k].cpu().numpy().astype('int64'))
    _lib.call('sfb_trace_end')
    _lib.call('sfb_conv_phase_trace', None, 0)
    import numpy as np
    names = names[-int(buf[0]):]                     # the eager pass also recorded precompute_cond's kernels first
    st = runs[-1]
    assert len(st) == len(names) <= n_eager, (len(st), len(names), n_eager)
    iv = np.median(np.stack([np.diff(r) for r in runs[1:]]), axis=0) / 1e3      # us, median over replays
    agg = collections.defaultdict(lambda: [0, 0.0])
    for nm, d in zip(names[:-1], iv):
        agg[nm][0] += 1
        agg[nm][1] += float(d)
    total = float(iv.sum())
    print(f'trace: {len(names)} kernels, first-to-last stamp {total:.1f} us', flush=True)
    for nm, (c, tt) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f'  {tt:9.1f} us  {c:4d} x {tt / c:7.2f}  {nm}')
    tag = '_'.join(['trace'] + [a for a in sys.argv[1:] if a in ('nopdl', 'nocarve', 'padsmem')])
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    npc = int(pbuf[0])
    json.dump(dict(names=names, interval_us=[round(float(v), 3) for v in iv], total_us=total, stamps=[int(v) for v in runs[-1]],
                   conv_phase_stamps=pbuf[1:1 + 8 * npc].cpu().numpy().reshape(npc, 8).tolist()), open(os.path.join(ROOT, 'gpurun_out', tag + '.json'), 'w'))


def vae_trace(out):
    """chain cost of every kernel of one VAE decode / encode (eager launches queued behind a GPU spin so the stamps show GPU time, not CPU gaps)"""
    import ctypes
    import collections
    import numpy as np
    from sparsefusion_b200 import _lib
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    vae = AutoencoderKL().cuda().eval()
    img = torch.rand(1, 3, 256, 256, device='cuda')
    z = torch.randn(1, 4, 32, 32, device='cuda')
    cap = 4096
    buf = torch.zeros(cap + 1, dtype=torch.int64, device='cuda')
    for what, fn in (('decode', lambda: vae.decode(z)), ('encode', lambda: vae.encode(img).mode())):
        with torch.no_grad():
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            _lib.call('sfb_trace_begin', buf.data_ptr(), cap)
            buf.zero_()
            torch.cuda._sleep(int(6e7))
            fn()
            torch.cuda.synchronize()
        nbuf = ctypes.create_string_buffer(1 << 20)
        _lib.load().sfb_trace_names(nbuf, len(nbuf))
        names = nbuf.value.decode().split('\n')[:-1]
        _lib.call('sfb_trace_end')
        k = int(buf[0])
        st = buf[1:1 + k].cpu().numpy().astype('int64')
        iv = np.diff(st) / 1e3
        agg = collections.defaultdict(lambda: [0, 0.0])
        for nm, d in zip(names[:-1], iv):
            agg[nm][0] += 1
            agg[nm][1] += float(d)
        print(f'vae {what}: {len(names)} kernels, first-to-last {iv.sum():.1f} us')
        for nm, (c, tt) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            print(f'  {tt:9.1f} us  {c:4d} x {tt / c:8.2f}  {nm}')
        top = sorted(zip(iv, range(len(iv))), reverse=True)[:12]
        print('  longest:', [(round(float(d), 1), names[i]) for d, i in top])
        json.dump(dict(names=names, interval_us=[round(float(v), 2) for v in iv]), open(os.path.join(ROOT, 'gpurun_out', f'trace_vae_{what}.json'), 'w'))


def conv_phases(out):
    """where a wgmma conv launch spends its time (sfb_conv_phase_trace): medians over 20 launches, cold L2, arena-style accumulate mode"""
    global FLUSH
    import numpy as np
    from sparsefusion_b200 import _lib
    ops.set_precision('tf32x3')
    if FLUSH is None:
        FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    cap = 64
    buf = torch.zeros(1 + 8 * cap, dtype=torch.int64, device='cuda')
    print('phases (us): prologue | dep-wait | first-stage | mainloop | drain | epilogue | total   [grid]')
    rows = []
    for name, h, cin, cout, k, stride in conv_cases():
        x = torch.randn(1, h, h, cin, device='cuda')
        w = ops.pack_conv_weight(torch.randn(cout, cin, k, k, device='cuda') / (cin * k * k) ** 0.5)
        b = torch.zeros(cout, device='cuda')
        pad = (k - 1) // 2 if stride == 1 else 1
        y = ops.conv2d_nhwc(x, w, cout, k, k, stride, pad, bias=b)
        y.zero_()
        _lib.call('sfb_conv_phase_trace', buf.data_ptr(), cap)
        buf.zero_()
        n = 20
        for _ in range(n):
            FLUSH.zero_()
            ops.conv2d_nhwc(x, w, cout, k, k, stride, pad, bias=b, out=y, accumulate=True)
        torch.cuda.synchronize()
        _lib.call('sfb_conv_phase_trace', None, 0)
        st = buf[1:1 + 8 * n].cpu().numpy().reshape(n, 8)[:, :7].astype('float64')
        d = np.median(np.diff(st, axis=1), axis=0) / 1e3
        tot = float(np.median(st[:, 6] - st[:, 0]) / 1e3)
        rec = dict(name=name, hw=h, cin=cin, cout=cout, k=k, prologue=round(float(d[0]), 2), dep_wait=round(float(d[1]), 2), first_stage=round(float(d[2]), 2),
                   mainloop=round(float(d[3]), 2), drain=round(float(d[4]), 2), epilogue=round(float(d[5]), 2), total=round(tot, 2), weight_mb=round(w.numel() * 4 / 1e6, 2))
        rows.append(rec)
        print(f"{name:12s} {d[0]:6.2f} | {d[1]:6.2f} | {d[2]:6.2f} | {d[3]:6.2f} | {d[4]:6.2f} | {d[5]:6.2f} | {tot:6.2f}   W {rec['weight_mb']:6.2f} MB", flush=True)
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, 'gpurun_out', 'conv_phases.json'), 'w'), indent=1)


def vae_bench(out):
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    vae = AutoencoderKL().cuda().eval()
    img = torch.rand(1, 3, 256, 256, device='cuda')
    z = torch.randn(1, 4, 32, 32, device='cuda')
    with torch.no_grad():
        out['vae_sm100'] = dict(encode_ms=round(timeit(lambda: vae.encode(img).mode(), iters=10, flush=False), 3),
                                decode_ms=round(timeit(lambda: vae.decode(z), iters=10, flush=False), 3))
        print('vae sm100', out['vae_sm100'], flush=True)
    from oracle import vae_oracle as vo                     # eager torch / cuDNN (TF32) restatement as the comparison
    tv = vo.TorchVAE(vae.state_dict()).to('cuda')
    with torch.no_grad():
        enc = timeit(lambda: tv.encode(img).mode(), iters=10, flush=False)
        dec = timeit(lambda: tv.decode(z), iters=10, flush=False)
        enc_cl = dec_cl = float('nan')
    out['vae'] = dict(encode_ms=round(enc, 3), decode_ms=round(dec, 3), encode_cl_ms=round(enc_cl, 3), decode_cl_ms=round(dec_cl, 3))
    print('vae', out['vae'], flush=True)


def render_bench(out):
    import numpy as np
    from sparsefusion_b200 import _lib
    for a in sys.argv:
        if a.startswith('fuse='):
            _lib.call('sfb_set_fusion', int(a[5:], 0))
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    net = NeRFNetwork(opt).cuda().train()
    net.encoder.embeddings.data.uniform_(-0.5, 0.5)
    N = 128 * 128
    o = torch.tensor([0.0, 1.3, 4.8], device='cuda').expand(N, 3).contiguous()
    ys, xs = torch.meshgrid(torch.linspace(1, -1, 128, device='cuda'), torch.linspace(1, -1, 128, device='cuda'), indexing='ij')
    d = torch.stack([xs / 4, ys / 4 - 0.27, -torch.ones_like(xs)], dim=-1).reshape(N, 3).contiguous()
    kw = dict(staged=False, perturb=True, bg_color=0, ambient_ratio=1.0, shading='albedo', force_all_rays=True, **vars(opt))
    def fwd():
        with torch.no_grad():
            net.render(o[None], d[None], **kw)
    def fwd_bwd():
        net.zero_grad(set_to_none=True)
        r = net.render(o[None], d[None], **kw)
        (r['image'].mean() + r['weights_sum'].mean()).backward()
    out['render'] = dict(rays=N, fwd_ms=round(timeit(fwd, iters=10), 3), fwd_bwd_ms=round(timeit(fwd_bwd, iters=10), 3))
    print('render', out['render'], flush=True)


def sample_bench(out):
    """one DDPM.sample (T = 500, FULL UNet, 32x32 latents) per batch size and guidance scale, and the dynamic-threshold step kernel alone"""
    import subprocess
    from sparsefusion_b200 import _lib
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.vldm import DDPM
    out['card'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                                 text=True).stdout.strip()
    print('card', out['card'], flush=True)
    unet = Unet(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
                layer_cross_attns=(False,) * 4, cond_images_channels=256, attn_pool_text=False, cond_on_z=False, conditional_embed_dim=None)
    ddpm = DDPM(channels=4, unets=(unet,), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(32,), timesteps=500, cond_drop_prob=0.1,
                pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False, clip_value=10).cuda()
    torch.nn.init.normal_(ddpm.unets[0].get_parameter('final_conv.weight'), std=0.02)
    out['sample'] = {}
    for nb in (1, 4, 8):
        cond = torch.randn(nb, 256, 32, 32, device='cuda')
        for cs in (1.0, 3.0):
            run = lambda: ddpm.sample(cond_images=cond, batch_size=nb, cond_scale=cs, use_tqdm=False)
            run()                                                   # graph capture, time features of the 501 noise levels
            ts = []
            for _ in range(2):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run()
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            rec = dict(sample_ms=round(min(ts), 1), per_step_ms=round(min(ts) / 500, 3), all_ms=[round(t, 1) for t in ts])
            out['sample'][f'b{nb}_cs{cs:g}'] = rec
            print('sample', nb, cs, rec, flush=True)
        if nb == 1:
            mb = sum(v.numel() * v.element_size() for v in next(iter(ddpm._sampling['time'].values())).values()) / 1e6
            out['sample']['time_features_mb'] = round(mb, 1)
            print('sample: time features of the 501 noise levels', round(mb, 1), 'MB', flush=True)
        r = out['sample'][f'b{nb}_cs3']['sample_ms'] / out['sample'][f'b{nb}_cs1']['sample_ms']
        out['sample'][f'b{nb}_guidance_ratio'] = round(r, 3)
        print('sample', nb, 'guided / unguided', round(r, 3), flush=True)
    out['dynamic_step'] = {}
    for n in (4096, 65536):
        for B in (1, 8):
            x, e, z = (torch.randn(B, n, device='cuda') * 3 for _ in range(3))
            y = torch.empty_like(x)
            step = lambda: _lib.call('sfb_ddpm_dynamic_step', _lib.fptr(x), _lib.fptr(e), None, 1.0, _lib.fptr(z), 0.7, 0.7, 0.75, 0.05, 0.1, 0.95,
                                     n, B, _lib.fptr(y), None, None, _lib.stream())
            us = timeit(lambda: [step() for _ in range(100)], iters=10, warmup=2, flush=False) * 10.   # ms per 100 launches -> us per launch
            out['dynamic_step'][f'n{n}_b{B}'] = round(us, 2)
            print('dynamic_step', n, B, f'{us:.2f} us', flush=True)


def mesh_bench(out):
    """NeRFRenderer.export_mesh stage by stage at R = 128, 256, 512 (seeded field, +-0.5 embeddings): device-event times of the lattice
    query, smoothing, statistics (includes the host read of the two doubles), marching-cubes count (includes the host read of V and F) and
    emit, medians of 5 after one warm-up; the host OBJ write is timed separately (wall clock, to a temporary directory)."""
    import subprocess
    import tempfile
    import time
    from oracle import ngp_oracle as no
    from sparsefusion_b200 import _lib, mesh
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    out['card'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                                 text=True).stdout.strip()
    print('card', out['card'], flush=True)
    net = NeRFNetwork(get_default_torch_ngp_opt())
    sd = net.state_dict()
    sd.update(no.make_field_params(seed=0))
    net.load_state_dict(sd)
    net = net.cuda().eval()
    out['mesh'] = {}

    def ev(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        return r, a.elapsed_time(b)

    with torch.no_grad():
        for R in (128, 256, 512):
            rows = []
            for it in range(6):
                sig, t_q = ev(lambda: mesh.density_lattice(net, R, 128))
                sm, t_s = ev(lambda: mesh.smooth_gaussian(sig, 1.5))
                (mean, std), t_st = ev(lambda: mesh.volume_mean_std(sm))
                iso = mean + 0.25 * std
                # the two marching-cubes phases, as mesh.marching_cubes runs them, timed apart
                nbytes = _lib.load().sfb_marching_cubes_scratch_bytes(R, R, R)
                scratch = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
                counts = torch.empty(2, dtype=torch.int64, device='cuda')
                isof = float(np.float32(iso))
                (nv, nf), t_c = ev(lambda: (_lib.call('sfb_marching_cubes_count', _lib.fptr(sm), R, R, R, isof, scratch.data_ptr(), counts.data_ptr(),
                                                      _lib.stream()), counts.tolist())[1])
                verts = torch.empty(nv, 3, device='cuda')
                tris = torch.empty(nf, 3, dtype=torch.int32, device='cuda')
                _, t_e = ev(lambda: _lib.call('sfb_marching_cubes_emit', _lib.fptr(sm), R, R, R, isof, scratch.data_ptr(), verts.data_ptr(),
                                              tris.data_ptr(), _lib.stream()))
                with tempfile.TemporaryDirectory() as d:
                    t0 = time.perf_counter()
                    mesh.write_obj(os.path.join(d, 'mcubes_mesh.obj'), verts, tris)
                    t_w = (time.perf_counter() - t0) * 1e3
                    obj_mb = os.path.getsize(os.path.join(d, 'mcubes_mesh.obj')) / 1e6
                if it:
                    rows.append((t_q, t_s, t_st, t_c, t_e, t_w))
                del sig, sm, scratch
            med = [float(m) for m in np.median(np.array(rows), axis=0)]
            gpu = sum(med[:5])
            rec = dict(field_query_ms=round(med[0], 2), smooth_ms=round(med[1], 2), stats_ms=round(med[2], 2), mc_count_ms=round(med[3], 2),
                       mc_emit_ms=round(med[4], 2), gpu_total_ms=round(gpu, 2), obj_write_ms=round(med[5], 1), vertices=nv, triangles=nf,
                       obj_mb=round(obj_mb, 1), gpu_share=round(gpu / (gpu + med[5]), 3))
            out['mesh'][str(R)] = rec
            print('mesh', R, rec, flush=True)


def scenes_bench(out):
    """scene-batched distillation (MultiSceneDistiller) against the same scenes as S sequential Distiller.step calls, SDS phase: FULL UNet, full
    VAE, LPIPS on, 32^2 latents, 128^2 rays, S in {1, 2, 4, 8}.  Scene k is seeded k in both arms, so both draw the same u sequence and run the
    same iterations; the two arms are timed alternately (device events around K iterations, after a warm-up that captures every graph shape)."""
    import subprocess
    from bench import build_gpu
    from sparsefusion_b200.distillation import MultiSceneDistiller, SceneCache
    from sparsefusion_b200.network_grid import NeRFNetwork
    from sparsefusion_b200.synthetic import synthetic_scene
    out['card'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                                 text=True).stdout.strip()
    print('card', out['card'], flush=True)
    dev = torch.device('cuda', 0)
    Distiller, models, _, kw = build_gpu(0, 1, dev)
    vae, vldm, opt, percep = models['vae'], models['vldm'], models['opt'], kw['percep']

    def ngp():
        n = NeRFNetwork(opt)
        n.encoder.embeddings.data.uniform_(-0.5, 0.5)
        return n.to(dev).train()
    out['scenes'] = {}
    K, reps, itr0 = 3, 3, 1001
    for S in (1, 2, 4, 8):
        caches = [SceneCache(**synthetic_scene(n_target=8, seed=k)).to(dev) for k in range(S)]
        torch.cuda.synchronize()
        mem0 = torch.cuda.memory_reserved()
        msd = MultiSceneDistiller([ngp() for _ in range(S)], vae, vldm, opt, caches, seeds=list(range(S)), percep=percep, max_batch=8)
        seq = [Distiller(ngp(), vae, vldm, opt, caches[k], seed=k, percep=percep) for k in range(S)]
        for d in seq[1:]:
            d.sampler = seq[0].sampler                                     # one graph per shape for the sequential arm too
        # capture every batch size 1..S of the batched arm: S distinct run lengths
        with torch.no_grad():
            lat = torch.randn(S, 4, 32, 32, device=dev)
            feats = torch.cat([c.target_features[:1] for c in caches])
            msd.sampler.sample_rows(lat, [0.99 - 0.1 * k for k in range(S)], feats)
        torch.cuda.synchronize()
        graph_mb = (torch.cuda.memory_reserved() - mem0) / 1e6
        itr = itr0
        for _ in range(2):                                                 # warm-up
            msd.step(itr)
            for d in seq:
                d.step(itr)
            itr += 1
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        tb, ts, rows, replays = [], [], 0, 0
        for _ in range(reps):
            for arm, times in (('batched', tb), ('sequential', ts)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(K):
                    if arm == 'batched':
                        msd.step(itr + i)
                        rows += sum(msd.last['unet_calls'])
                        replays += msd.last['graph_replays']
                    else:
                        for d in seq:
                            d.step(itr + i)
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) / K)
            itr += K
        mb, ms = float(np.median(tb)), float(np.median(ts))
        rec = dict(batched_ms_per_iteration=round(mb, 1), sequential_ms_per_iteration=round(ms, 1), batched_scene_its_per_s=round(S * 1e3 / mb, 2),
                   sequential_scene_its_per_s=round(S * 1e3 / ms, 2), speedup=round(ms / mb, 3), batched_all_ms=[round(t, 1) for t in tb],
                   sequential_all_ms=[round(t, 1) for t in ts], unet_rows_per_iteration=round(rows / (K * reps), 1),
                   graph_replays_per_iteration=round(replays / (K * reps), 1), graph_capture_mb=round(graph_mb, 1),
                   peak_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
        out['scenes'][str(S)] = rec
        print('scenes', S, rec, flush=True)
        del msd, seq, caches
        torch.cuda.empty_cache()


def eval_bench(out):
    """scene scoring (sparsefusion_b200.evaluate): sfb_image_ssim_psnr alone at B = 1 and 32 on 256^2 pairs (CUDA events around 50 calls,
    after a warm-up), and evaluate_scene over 32 views at 256^2 of a seeded field split into its render, LPIPS and SSIM / PSNR parts (device
    events around each part of one view loop, medians of 5 after a warm-up)."""
    import subprocess
    from oracle import ngp_oracle as no
    from sparsefusion_b200 import evaluate as ev
    from sparsefusion_b200.distillation import view_seed
    from sparsefusion_b200.lpips_vgg import PerceptualLoss
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.synthetic import camera_rays, circle_cameras
    out['card'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                                 text=True).stdout.strip()
    print('card', out['card'], flush=True)
    out['eval'] = {}
    g = torch.Generator(device='cuda').manual_seed(0)
    for B in (1, 32):
        a = torch.rand(B, 256, 256, 3, device='cuda', generator=g)
        b = (a + 0.1 * torch.rand(B, 256, 256, 3, device='cuda', generator=g)).clamp(0, 1)
        for _ in range(5):
            ev.image_metrics(a, b)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(50):
            ev.image_metrics(a, b)
        t1.record()
        torch.cuda.synchronize()
        us = t0.elapsed_time(t1) / 50 * 1e3
        rec = dict(us_per_call=round(us, 1), us_per_image=round(us / B, 2), input_gbs=round(2 * a.numel() * 4 / (us * 1e3), 1))
        out['eval'][f'ssim_psnr_b{B}'] = rec
        print('ssim_psnr', B, rec, flush=True)
    opt = get_default_torch_ngp_opt()
    net = NeRFNetwork(opt)
    sd = net.state_dict()
    sd.update(no.make_field_params(seed=0))
    net.load_state_dict(sd)
    net = net.cuda().eval()
    V, hw = 32, 256
    o, d = zip(*[camera_rays(c, hw, hw) for c in circle_cameras(V, radius=4.5)])
    rays_o, rays_d = torch.from_numpy(np.stack(o)).cuda(), torch.from_numpy(np.stack(d)).cuda()
    rgb = torch.rand(V, 3, hw, hw, device='cuda', generator=g)
    views = ev.EvalViews(rays_o, rays_d, rgb, (rgb > 0.5).float()[:, :1])
    percep = PerceptualLoss('vgg', device='cuda', seed=1)

    def stamp():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e
    rows = []
    with torch.no_grad():
        for it in range(6):
            e0 = stamp()
            imgs = []
            for v in range(V):
                with torch.random.fork_rng(devices=[rays_o.device]):
                    torch.cuda.manual_seed(view_seed(0, 0, v, ev.EVAL_STREAM))
                    imgs.append(net.render_batched(rays_o[v][None], rays_d[v][None], batched=True, perturb=True, bg_color=0, ambient_ratio=1.0,
                                                   shading='albedo', force_all_rays=True, **vars(opt))['image'].reshape(hw, hw, 3))
            image = torch.stack(imgs)
            e1 = stamp()
            lp = [percep.value_and_grad(image[v].permute(2, 0, 1), rgb[v], normalize=True, want_grad=False)[0] for v in range(V)]
            e2 = stamp()
            ev.image_metrics(image, rgb.permute(0, 2, 3, 1).contiguous())
            e3 = stamp()
            ev.evaluate_scene(net, views, opt, percep, seed=0)
            e4 = stamp()
            torch.cuda.synchronize()
            if it:
                rows.append((e0.elapsed_time(e1), e1.elapsed_time(e2), e2.elapsed_time(e3), e3.elapsed_time(e4)))
            del lp
    med = [float(m) for m in np.median(np.array(rows), axis=0)]
    rec = dict(views=V, hw=hw, render_ms=round(med[0], 2), lpips_ms=round(med[1], 2), ssim_psnr_ms=round(med[2], 3),
               evaluate_scene_ms=round(med[3], 2))
    out['eval']['evaluate_scene_32x256'] = rec
    print('evaluate_scene', rec, flush=True)


def video_bench(out):
    """gif palettes (sparsefusion_b200.video): sfb_palette_quantize on render-like frames (black background, a textured blob per panel) --
    50 frames of 256x512 (the circle gif) and V = 32 / 200 frames of 256x1280 (the sequence gif) -- by CUDA events around 10 calls after a
    warm-up; Pillow's convert('P', palette=ADAPTIVE) on the same frames by a host clock; and the end-to-end visualize step of one scene
    (_write_scene_pictures: 32 views and 50 circle views at 256^2 rendered, quantised and written) by a host clock around a synchronise."""
    import subprocess
    import tempfile
    import time
    from PIL import Image
    from oracle import ngp_oracle as no
    from sparsefusion_b200 import evaluate as ev, video
    from sparsefusion_b200.distillation import _write_scene_pictures
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    from sparsefusion_b200.synthetic import camera_rays, circle_cameras
    out['card'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                                 text=True).stdout.strip()
    print('card', out['card'], flush=True)
    out['video'] = {}
    g = torch.Generator(device='cuda').manual_seed(0)

    def render_like(B, H, W):
        yy, xx = torch.meshgrid(torch.arange(H, device='cuda'), torch.arange(W // 256 * 256, device='cuda') % 256, indexing='ij')
        c = torch.rand(B, 1, 1, 2, device='cuda', generator=g) * 80 + 88
        blob = (1 - ((yy - c[..., 0]) ** 2 + (xx - c[..., 1]) ** 2) / 70.0 ** 2).clamp(0, 1)
        return video.to_uint8(blob[..., None] * (0.5 + 0.5 * torch.rand(B, H, W, 3, device='cuda', generator=g)))

    for name, (B, H, W) in (('circle_50x256x512', (50, 256, 512)), ('sequence_32x256x1280', (32, 256, 1280)), ('sequence_200x256x1280', (200, 256, 1280))):
        frames = render_like(B, H, W)
        for _ in range(3):
            video.quantize_palette(frames)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(10):
            video.quantize_palette(frames)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 10
        host = frames.cpu().numpy()
        h0 = time.perf_counter()
        for f in host:
            Image.fromarray(f).convert('P', palette=Image.ADAPTIVE)
        pil_ms = (time.perf_counter() - h0) * 1e3
        rec = dict(gpu_ms=round(ms, 3), gpu_us_per_frame=round(ms * 1e3 / B, 1), pillow_ms=round(pil_ms, 1), pillow_ms_per_frame=round(pil_ms / B, 1),
                   ncolors_mean=round(video.quantize_palette(frames)[1].float().mean().item(), 1))
        out['video'][name] = rec
        print('quantize', name, rec, flush=True)
    opt = get_default_torch_ngp_opt()
    net = NeRFNetwork(opt)
    sd = net.state_dict()
    sd.update(no.make_field_params(seed=0))
    net.load_state_dict(sd)
    net = net.cuda().eval()
    V, hw = 32, 256
    o, d = zip(*[camera_rays(c, hw, hw) for c in circle_cameras(V, radius=4.5)])
    rgb = torch.rand(V, 3, hw, hw, device='cuda', generator=g)
    views = ev.EvalViews(torch.from_numpy(np.stack(o)).cuda(), torch.from_numpy(np.stack(d)).cuda(), rgb, (rgb > 0.5).float()[:, :1])
    co, cd = zip(*[camera_rays(c, hw, hw) for c in circle_cameras(50, radius=4.0)])
    circle = torch.from_numpy(np.stack(co)).cuda(), torch.from_numpy(np.stack(cd)).cuda()
    eft = torch.rand(V, 3, hw, hw, device='cuda', generator=g)
    times, renders = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for it in range(4):
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            _write_scene_pictures(tmp, 'scene', net, opt, views, circle, eft, seed=0)
            torch.cuda.synchronize()
            h1 = time.perf_counter()
            ev.render_views(net, views.rays_o, views.rays_d, (hw, hw), opt, seed=0, stream=ev.EVAL_STREAM)     # the same renders alone
            ev.render_views(net, *circle, (hw, hw), opt, seed=0, stream=ev.CIRCLE_STREAM)
            torch.cuda.synchronize()
            if it:
                times.append((h1 - h0) * 1e3)
                renders.append((time.perf_counter() - h1) * 1e3)
    rec = dict(views=V, circle_views=50, hw=hw, visualize_ms=round(float(np.median(times)), 1), renders_ms=round(float(np.median(renders)), 1),
               all_ms=[round(t, 1) for t in times])
    out['video']['visualize_one_scene'] = rec
    print('visualize', rec, flush=True)


def main():
    out = {'device': torch.cuda.get_device_name(0), 'conv': [], 'grid': {}}
    if 'video' in sys.argv:
        video_bench(out)
        print(json.dumps(out), flush=True)
        return
    if 'eval' in sys.argv:
        eval_bench(out)
        print(json.dumps(out), flush=True)
        return
    if 'scenes' in sys.argv:
        scenes_bench(out)
        print(json.dumps(out), flush=True)
        return
    if 'sample' in sys.argv:
        sample_bench(out)
        print(json.dumps(out), flush=True)
        return
    if 'mesh' in sys.argv:
        mesh_bench(out)
        print(json.dumps(out), flush=True)
        return
    if 'unet' in sys.argv or len(sys.argv) == 1:
        unet_bench(out)
    if 'render' in sys.argv or len(sys.argv) == 1:
        render_bench(out)
    if 'trace' in sys.argv:
        unet_trace(out)
    if 'phases' in sys.argv:
        conv_phases(out)
    if 'vaetrace' in sys.argv:
        vae_trace(out)
    if 'vae' in sys.argv or len(sys.argv) == 1:
        vae_bench(out)
    if len(sys.argv) > 1 and 'conv' not in sys.argv:
        json.dump(out, open(os.path.join(ROOT, 'gpurun_out', 'microbench.json'), 'w'), indent=1)
        return
    for nb in (1, 8):
        for name, h, cin, cout, k, stride in conv_cases():
            x = ops.round_tf32(torch.randn(nb, h, h, cin, device='cuda'))
            w = ops.pack_conv_weight(torch.randn(cout, cin, k, k, device='cuda') / (cin * k * k) ** 0.5)
            b = torch.zeros(cout, device='cuda')
            pad = (k - 1) // 2 if stride == 1 else 1
            y = ops.conv2d_nhwc(x, w, cout, k, k, stride, pad, bias=b)
            ms = timeit(lambda: ops.conv2d_nhwc(x, w, cout, k, k, stride, pad, bias=b, out=y))
            ho = y.shape[1]
            flops = 2.0 * nb * ho * ho * cout * cin * k * k
            wbytes = w.numel() * 4
            rec = dict(name=name, nb=nb, hw=h, cin=cin, cout=cout, k=k, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1),
                       weight_gbs=round(wbytes / ms / 1e6, 1))
            print(rec, flush=True)
            out['conv'].append(rec)
    # grid encoder operators at the render's sizes
    from sparsefusion_b200.gridencoder import GridEncoder
    enc = GridEncoder(input_dim=3, num_levels=16, level_dim=2, base_resolution=16, log2_hashmap_size=16, desired_resolution=8192, gridtype='tiled').cuda()
    enc.embeddings.data.uniform_(-0.5, 0.5)
    for B in (1 << 20, 1 << 21):
        x = (torch.rand(B, 3, device='cuda') * 2 - 1) * 4
        ms_f = timeit(lambda: enc(x, bound=4).sum() if False else enc(x, bound=4))
        y = enc(x, bound=4)
        g = torch.randn_like(y)
        def fb():
            enc.embeddings.grad = None
            y2 = enc(x, bound=4)
            y2.backward(g)
        ms_fb = timeit(fb)
        out['grid'][str(B)] = dict(fwd_ms=round(ms_f, 4), fwd_bwd_ms=round(ms_fb, 4), fwd_GBps_alg=round(B * 140 / ms_f / 1e6, 1))
        print('grid', B, out['grid'][str(B)], flush=True)
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, 'gpurun_out', 'microbench.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
