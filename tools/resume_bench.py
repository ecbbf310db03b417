"""Cost of distillation checkpoints: write time and file size per scene with cuda_ray off and on at S = 1 and 8 scenes, the time to read and
load them back, and the overhead of writing every K iterations as a share of step time.

    python tools/resume_bench.py [--repeats 5] [--K 100] [--out resume_bench.json]

A checkpoint holds the network (1,865,204 fp32 parameters), both Adam moments, the counters and generators, and with cuda_ray the density
grid and bitfield; it does not depend on the UNet or VAE, so the small models stand in for them here.  Scenes are full size (64 target views,
256^2 images, 32^2 latents, 128^2 rays), whose cache the checkpoint's digest reads.  A write is what the loops do: ``state_dict`` (device to
host copies, the cache digest on the device) and an atomic, fsynced write of one file per scene to a temporary directory.  A load is
``torch.load`` of every scene's file and ``load_state_dict``.  Times are medians over ``--repeats`` after one warm-up.  The step times the
overhead is computed against are arguments (defaults: the README's H100 figures for the reference iteration and the 64-view step); the
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f'unknown ({e})'


def _models():
    from oracle import unet_oracle as uo
    from sparsefusion_b200.imagen_pytorch import Unet
    from sparsefusion_b200.ldm_autoencoder import AutoencoderKL
    from sparsefusion_b200.vldm import DDPM
    cfg = uo.SMALL
    unet = Unet(channels=cfg.channels, dim=cfg.dim, dim_mults=cfg.dim_mults, num_resnet_blocks=cfg.num_resnet_blocks, layer_attns=cfg.layer_attns,
                layer_cross_attns=(False,) * 4, cond_images_channels=cfg.cond_images_channels, attn_pool_text=False,
                attn_dim_head=cfg.attn_dim_head, attn_heads=cfg.attn_heads, cond_on_z=False, conditional_embed_dim=None)
    ddpm = DDPM(channels=4, unets=(unet.cuda(),), conditional_encoder=None, conditional_embed_dim=None, image_sizes=(cfg.image_size,), timesteps=500,
                cond_drop_prob=0.1, pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True,
                dynamic_thresholding=False, dynamic_thresholding_percentile=.68, clip_value=10).cuda()
    return AutoencoderKL(ch=32, ch_mult=(1, 2, 4, 4)).eval().cuda(), ddpm


def _distiller(S, cuda_ray, models):
    from oracle import distill_oracle as do
    from sparsefusion_b200.distillation import Distiller, MultiSceneDistiller, SceneCache
    from sparsefusion_b200.network_grid import NeRFNetwork, get_default_torch_ngp_opt
    opt = get_default_torch_ngp_opt()
    opt.cuda_ray = cuda_ray
    caches = [SceneCache(**do.synthetic_scene(n_input=2, n_target=64, seed=k)).to('cuda') for k in range(S)]
    ngps = [NeRFNetwork(opt).cuda().train() for _ in range(S)]
    if S == 1:
        return Distiller(ngps[0], *models, opt, caches[0], seed=0)
    return MultiSceneDistiller(ngps, *models, opt, caches, seeds=list(range(S)))


def _median_time(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--K', type=int, default=100, help='checkpoint interval the overhead is reported for')
    ap.add_argument('--ref-step-ms', type=float, default=100.4, help='reference iteration time (README: H100, bench.py)')
    ap.add_argument('--view64-step-ms', type=float, default=3060.0, help='64-view minibatch step time (README: H100)')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('resume_bench needs a GPU: nothing is measured without one')
    from sparsefusion_b200.distillation import MultiSceneDistiller, _checkpoint_paths, _read_checkpoints, _write_checkpoints
    torch.cuda.set_device(0)
    models = _models()
    rows = []
    for cuda_ray in (False, True):
        for S in (1, 8):
            dist = _distiller(S, cuda_ray, models)
            with tempfile.TemporaryDirectory() as d:
                names = [(f'scene_{k:03d}',) for k in range(S)]
                paths = _checkpoint_paths(d, names)
                write = _median_time(lambda: _write_checkpoints(dist, paths, 100, True, 0), a.repeats)
                size = statistics.mean(os.path.getsize(p) for p in paths)

                def load():
                    saved = _read_checkpoints(paths, [n[0] for n in names], None)
                    sd = dict(version=saved[0]['version'], itr=saved[0]['itr'], scenes=saved) if isinstance(dist, MultiSceneDistiller) else saved[0]
                    dist.load_state_dict(sd)
                read = _median_time(load, a.repeats)
            rows.append(dict(cuda_ray=cuda_ray, scenes=S, write_s=write, write_s_per_scene=write / S, load_s=read, bytes_per_scene=size))
            print(f'cuda_ray={cuda_ray!s:5} S={S}: write {write * 1e3:8.1f} ms ({write / S * 1e3:6.1f} ms/scene), load {read * 1e3:8.1f} ms, '
                  f'{size / 1e6:6.2f} MB per scene', flush=True)
            del dist
            torch.cuda.empty_cache()
    one = {r['cuda_ray']: r for r in rows if r['scenes'] == 1}
    overhead = {f'{name}_cuda_ray_{cr}': one[cr]['write_s'] / (a.K * step_ms / 1e3)
                for name, step_ms in (('reference_step', a.ref_step_ms), ('view64_step', a.view64_step_ms)) for cr in (False, True)}
    for k, v in overhead.items():
        print(f'overhead of one write every K={a.K} iterations, {k}: {100 * v:.3f}% of step time')
    res = dict(card=_card(), torch=torch.__version__, K=a.K, ref_step_ms=a.ref_step_ms, view64_step_ms=a.view64_step_ms, rows=rows,
               overhead_share=overhead)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
