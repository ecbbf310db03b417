"""``python -m sparsefusion_b200.demo``: the reference README's "Evaluation" run (demo.py) from a dataset and the released checkpoints,
without the reference tree, pytorch3d, omegaconf, the ``lpips`` package or a network connection.

The flags are demo.py's (demo.py:106-131) with the same defaults and checkpoint paths (:150-154); ``-n/--nodes`` and ``-nr`` are not
provided (one node).  Three flags are added: ``--lpips PATH`` (pretrained LPIPS-VGG weights, required: see ``lpips_vgg.load_lpips_state_dict``),
``--max-itr`` (the reference's hard-coded 3000) and ``--seed``.

Per category, each GPU takes its share of the ``-i`` scenes (``split_list``), loads the three models (``load_models``) and the category's
toy scenes (``load_toy_category``), gives each scene the reference's input views (``input_views``) and name (``seq_name``), and distils its
share as ONE ``distill_scenes`` call with ``NativeSceneBuilder``, evaluation, pictures and the progress files every 20 iterations, the
pretrained LPIPS-VGG both in the loop's perceptual term and in the scores.  Scene ``val_idx`` is seeded ``scene_seed(seed, val_idx)``, so
its outputs depend on the seed, the category, ``val_idx``, ``-v`` and the checkpoints only: not on ``-g``, nor on which other scenes ``-i``
lists or in which order.  Everything goes to ``output/demo/`` as demo.py writes it.
"""
from __future__ import annotations

import argparse
import os
import sys
from types import SimpleNamespace

import torch

EXP_DIR = 'output/demo'                  # demo.py:160
SEED_STRIDE = 1_000_003                  # scene_seed: a prime above any scene index, so the map (seed, val_idx) -> seed is injective
DATASETS = ('co3d_toy',)


# ---------------------------------------------------------------------------------------------------------------- scene bookkeeping
def split_list(a, n: int) -> list:
    """``a`` in ``n`` contiguous chunks whose lengths differ by at most one, the longer ones first (utils/common_utils.py:21-33): chunk r is
    what GPU r distils"""
    k, m = divmod(len(a), n)
    out, lo = [], 0
    for r in range(n):
        hi = lo + k + (1 if r < m else 0)
        out.append(list(a[lo:hi]))
        lo = hi
    return out


def input_views(n_views: int, val_idx: int, v: int) -> list:
    """the reference's input views of scene ``val_idx`` (demo.py:63, :78-81): the first ``v`` entries of a permutation drawn from a CPU
    generator seeded with ``0 + val_idx``"""
    return torch.randperm(n_views, generator=torch.Generator().manual_seed(0 + val_idx))[:v].long().tolist()


def seq_name(cat: str, val_idx: int, v: int) -> str:
    """the reference's scene name (demo.py:86)"""
    return f'{cat}_{val_idx:03d}_c{v}'


def scene_seed(seed: int, val_idx: int) -> int:
    """the seed scene ``val_idx`` is distilled with (``distill_scenes(seeds=...)``): ``seed * 1_000_003 + val_idx``"""
    return seed * SEED_STRIDE + val_idx


def toy_path(root: str, cat: str) -> str:
    return f'{root}/{cat}/{cat}_toy.pt'                    # utils/co3d_toy_dataloader.py


def load_toy_category(root: str, cat: str) -> list:
    """the scenes of ``{root}/{cat}/{cat}_toy.pt`` as the reference reads them (utils/co3d_toy_dataloader.py): ``torch.load(path)[cat]``, a
    list of dicts with R [N,3,3], T [N,3], f [N,2], c [N,2], image_size [N,2], images [N,3,256,256], masks and valid_region [N,1,256,256].
    This is a full unpickle (``weights_only=False``), as in the reference: only load dataset files you trust."""
    data = torch.load(toy_path(root, cat), map_location='cpu', weights_only=False)
    if not isinstance(data, dict) or cat not in data:
        raise ValueError(f'{toy_path(root, cat)} holds no entry {cat!r}')
    return list(data[cat])


def scene_cameras(scene: dict):
    """``cameras.PerspectiveCameras`` of a toy scene (demo.py:72)"""
    from .cameras import PerspectiveCameras
    return PerspectiveCameras(R=scene['R'], T=scene['T'], focal_length=scene['f'], principal_point=scene['c'], image_size=scene['image_size'])


# ---------------------------------------------------------------------------------------------------------------- models
# utils/load_model.py:56-91: the released VLDM's UNet and DDPM keywords
UNET_KW = dict(channels=4, dim=256, dim_mults=(1, 2, 4, 4), num_resnet_blocks=(2, 2, 2, 2), layer_attns=(False, False, False, True),
               layer_cross_attns=(False, False, False, False), cond_images_channels=256, attn_pool_text=False)
DDPM_KW = dict(channels=4, conditional_encoder=None, conditional_embed_dim=None, image_sizes=(32,), timesteps=500, cond_drop_prob=0.1,
               pred_objectives='noise', conditional=False, auto_normalize_img=False, clip_output=True, dynamic_thresholding=False,
               dynamic_thresholding_percentile=.68, clip_value=10)
# the SD-v1 KL-f8 autoencoder (external/ldm/configs/sd-vae.yaml)
VAE_KW = dict(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, out_ch=3, z_channels=4, embed_dim=4)


def _load(path):
    # a full unpickle, as the reference reads its checkpoints (utils/load_model.py:36, :88, :119)
    return torch.load(path, map_location='cpu', weights_only=False)


def load_eft(path):
    """the released EFT on the CPU: of the checkpoint's ``model_state_dict`` only the keys the model has, then a strict load
    (utils/load_model.py:34-45)"""
    from .eft import EpipolarFeatureTransformer
    eft = EpipolarFeatureTransformer(use_r=True, encoder='resnet18', return_features=True, remove_unused_layers=False)
    own = eft.state_dict()
    own.update({k: v for k, v in _load(path)['model_state_dict'].items() if k in own})
    eft.load_state_dict(own)
    return eft


def load_vldm(path):
    """the released VLDM on the CPU (utils/load_model.py:57-91): ``DDPM(unets=(Unet(**UNET_KW),), **DDPM_KW)``, ``model_state_dict``
    loaded strictly"""
    from .imagen_pytorch import Unet
    from .vldm import DDPM
    vldm = DDPM(unets=(Unet(**UNET_KW),), **DDPM_KW)
    vldm.load_state_dict(_load(path)['model_state_dict'])
    return vldm


def load_vae(path):
    """the SD VAE on the CPU, in eval mode (utils/load_model.py:98-151): the checkpoint's ``state_dict`` with each key renamed by the
    reference's ``k.replace('first_stage_model.', '').replace('model.', '')`` and loaded with ``strict=False``, so the UNet and text-encoder
    keys of a full SD checkpoint are ignored.  Where the reference only prints, a VAE weight the checkpoint does not provide is a
    RuntimeError: a VAE with random weights is never what a run wants."""
    from .ldm_autoencoder import AutoencoderKL
    vae = AutoencoderKL(**VAE_KW)
    sd = {k.replace('first_stage_model.', '').replace('model.', ''): v for k, v in _load(path)['state_dict'].items()}
    missing, _ = vae.load_state_dict(sd, strict=False)
    if missing:
        raise RuntimeError(f'{path}: the checkpoint lacks {len(missing)} VAE weights, e.g. {sorted(missing)[:4]}')
    return vae.eval()


def load_models(gpu, eft_ckpt, vldm_ckpt, vae_ckpt):
    """(eft, vae, vldm) of the released configuration on GPU ``gpu`` (utils/load_model.py:13-93), from the mirrored classes"""
    eft = load_eft(eft_ckpt).cuda(gpu)
    print('LOADING 1/3 loaded eft checkpoint from', eft_ckpt)
    vae = load_vae(vae_ckpt).cuda(gpu)
    print('LOADING 2/3 loaded sd vae from', vae_ckpt)
    vldm = load_vldm(vldm_ckpt).cuda(gpu)
    print('LOADING 3/3 loaded diffusion from', vldm_ckpt)
    return eft, vae, vldm


# ---------------------------------------------------------------------------------------------------------------- command line
LPIPS_HELP = ('pretrained LPIPS-VGG weights (required): a state dict saved on any machine with the lpips package by '
              '`torch.save(lpips.LPIPS(net="vgg").state_dict(), PATH)`, or a directory holding that package\'s weights/v0.1/vgg.pth and '
              'torchvision\'s vgg16-397923af.pth')


def build_parser() -> argparse.ArgumentParser:
    """demo.py:106-131's flags and defaults (without -n/-nr), plus --lpips, --max-itr and --seed"""
    p = argparse.ArgumentParser(prog='python -m sparsefusion_b200.demo', description=__doc__.split('\n\n')[0])
    p.add_argument('-g', '--gpus', default=1, type=int, help='number of gpus (one process each)')
    p.add_argument('-p', '--port', default=1, type=int, metavar='N',
                   help='accepted for demo.py compatibility and ignored: distillation runs no collectives, so no process group is created')
    p.add_argument('-c', '--category', type=str, metavar='S', required=True,
                   help='category, comma-separated categories, or "all" (every directory under --root with a {cat}/{cat}_toy.pt)')
    p.add_argument('-r', '--root', type=str, default='data/co3d_toy', metavar='S', help='location of the toy dataset')
    p.add_argument('-d', '--dataset_name', type=str, default='co3d_toy', metavar='S', help='dataset name (co3d_toy)')
    p.add_argument('-e', '--eft', type=str, default='-DNE', metavar='S', help='eft ckpt (default checkpoints/sf/{cat}/ckpt_latest_eft.pt)')
    p.add_argument('-l', '--vldm', type=str, default='-DNE', metavar='S', help='vldm ckpt (default checkpoints/sf/{cat}/ckpt_latest.pt)')
    p.add_argument('-a', '--vae', type=str, default='-DNE', metavar='S', help='vae ckpt (default checkpoints/sd/sd-v1-3-vae.ckpt)')
    p.add_argument('-i', '--idx', type=str, default='-DNE', metavar='N', help='evaluation indices, e.g. 0,5,7 (default 0)')
    p.add_argument('-v', '--input_views', type=int, default=2, metavar='N', help='input views')
    p.add_argument('--lpips', type=str, default=None, metavar='PATH', help=LPIPS_HELP)
    p.add_argument('--max-itr', type=int, default=3000, metavar='N', help='distillation iterations per scene (default 3000)')
    p.add_argument('--seed', type=int, default=0, metavar='S', help='scene val_idx is seeded seed * 1000003 + val_idx (default 0)')
    return p


class ArgumentError(Exception):
    """an invalid command line or a missing input, found before any GPU work"""


def checkpoint_paths(args, cat: str):
    """(eft, vldm, vae) checkpoint paths of category ``cat``: the flags, or demo.py's defaults (:150-154)"""
    eft = args.eft if args.eft != '-DNE' else f'checkpoints/sf/{cat}/ckpt_latest_eft.pt'
    vldm = args.vldm if args.vldm != '-DNE' else f'checkpoints/sf/{cat}/ckpt_latest.pt'
    vae = args.vae if args.vae != '-DNE' else 'checkpoints/sd/sd-v1-3-vae.ckpt'
    return eft, vldm, vae


def parse_idx(idx: str) -> list:
    if idx == '-DNE':
        return [0]                                                                  # demo.py:158
    try:
        return [int(s) for s in idx.split(',')]
    except ValueError:
        raise ArgumentError(f'-i --idx {idx!r} is invalid, please use the form 1,2,3') from None


def categories(root: str, category: str) -> list:
    if category == 'all_ten':
        raise ArgumentError('-c all_ten is not supported here (its ten-category list belongs to the CO3D dataloader); pass the categories '
                            'as a comma-separated list')
    if category == 'all':
        cats = sorted(c for c in os.listdir(root) if os.path.isfile(toy_path(root, c)))
        if not cats:
            raise ArgumentError(f'-c all: no directory under {root} holds a {{cat}}/{{cat}}_toy.pt')
        return cats
    cats = [c for c in category.split(',') if c]
    if not cats:
        raise ArgumentError(f'-c {category!r} names no category')
    return cats


def check_args(args):
    """utils/check_args.py's checks and the ranges of -i and -v, before any GPU work: returns (categories, val_list, the LPIPS state dict);
    ArgumentError with the message otherwise"""
    from .lpips_vgg import load_lpips_state_dict
    if args.dataset_name == 'co3d':
        raise ArgumentError('-d co3d (the full CO3Dv2 set, read through pytorch3d\'s implicitron) is not supported here; use -d co3d_toy')
    if args.dataset_name not in DATASETS:
        raise ArgumentError(f'provided {args.dataset_name} as dataset, but only {", ".join(DATASETS)} is supported')
    if args.lpips is None:
        raise ArgumentError('--lpips PATH is required: the distillation loss and the LPIPS score use the pretrained LPIPS-VGG, and random '
                            f'weights would distil a different loss than the reference.  {LPIPS_HELP}')
    if not os.path.exists(args.lpips):
        raise ArgumentError(f'provided LPIPS weights {args.lpips} do not exist')
    if args.gpus < 1:
        raise ArgumentError(f'-g --gpus must be at least 1 (got {args.gpus})')
    if args.max_itr < 1:
        raise ArgumentError(f'--max-itr must be at least 1 (got {args.max_itr})')
    if not 0 <= args.seed < 2 ** 32:
        raise ArgumentError(f'--seed must be in [0, 2**32) (got {args.seed})')
    if not os.path.exists(args.root):
        raise ArgumentError(f'provided dataset root {args.root} does not exist')
    val_list = parse_idx(args.idx)
    if len(set(val_list)) != len(val_list):
        raise ArgumentError(f'-i --idx lists a scene twice: {val_list}')
    cats = categories(args.root, args.category)
    for cat in cats:
        for what, path in zip(('EFT', 'VLDM', 'VAE'), checkpoint_paths(args, cat)):
            if not os.path.exists(path):
                raise ArgumentError(f'provided {what} weight {path} does not exist')
        if not os.path.isfile(toy_path(args.root, cat)):
            raise ArgumentError(f'toy dataset not found at {toy_path(args.root, cat)}')
        scenes = load_toy_category(args.root, cat)
        for i in val_list:
            if not 0 <= i < len(scenes):
                raise ArgumentError(f'-i index {i} is out of range: category {cat} has {len(scenes)} scenes')
            n = len(scenes[i]['R'])
            if not 1 <= args.input_views < n:
                raise ArgumentError(f'-v --input_views {args.input_views} must be at least 1 and below the {n} views of {seq_name(cat, i, args.input_views)}')
        del scenes
    try:
        lpips_sd = load_lpips_state_dict(args.lpips)
    except (RuntimeError, OSError, KeyError) as e:
        raise ArgumentError(str(e)) from None
    return cats, val_list, lpips_sd


def fit(gpu: int, args, cats: list, val_list: list, lpips_sd: dict):
    """demo.py:18-103 on GPU ``gpu``: per category, this GPU's share of the scenes as one ``distill_scenes`` call"""
    from .distillation import NativeSceneBuilder, distill_scenes, get_default_torch_ngp_opt
    from .lpips_vgg import PerceptualLoss
    torch.cuda.set_device(gpu)
    for d in ('', '/log', '/metrics', '/render_imgs', '/render_gifs'):                   # demo.py:24-28
        os.makedirs(EXP_DIR + d, exist_ok=True)
    mine = split_list(val_list, args.gpus)[gpu]
    print(f'gpu {gpu}: assigned idx {mine}')
    if not mine:
        return
    loss_fn_vgg = PerceptualLoss('vgg', device=torch.device('cuda', gpu)).load_state_dict(lpips_sd)
    for ci, cat in enumerate(cats):
        print(f'gpu {gpu}: setting category to {cat} {ci}/{len(cats)}')
        models = load_models(gpu, *checkpoint_paths(args, cat))
        data = load_toy_category(args.root, cat)
        scenes, seeds = [], []
        for val_idx in mine:
            sc = data[val_idx]
            idx = input_views(len(sc['R']), val_idx, args.input_views)
            print('val_idx', val_idx, idx)
            scenes.append((seq_name(cat, val_idx, len(idx)), scene_cameras(sc), sc['images'].cuda(gpu), sc['masks'].cuda(gpu),
                           sc['valid_region'].cuda(gpu), idx))
            seeds.append(scene_seed(args.seed, val_idx))
        distill_scenes(gpu, SimpleNamespace(exp_dir=EXP_DIR, category=cat), get_default_torch_ngp_opt(), models, EXP_DIR, scenes,
                       max_itr=args.max_itr, scene_builder=NativeSceneBuilder(gpu), evaluate=True, visualize=True, progress_every=20,
                       loss_fn_vgg=loss_fn_vgg, percep_weights=lpips_sd, seeds=seeds)
        del models, data, scenes
        torch.cuda.empty_cache()


def main(argv=None) -> int:
    """the command line; returns 0, or exits with status 1 and a message on an invalid argument (before any GPU work)"""
    args = build_parser().parse_args(argv)
    try:
        cats, val_list, lpips_sd = check_args(args)
        if torch.cuda.device_count() < args.gpus:
            raise ArgumentError(f'-g {args.gpus} needs {args.gpus} GPUs, {torch.cuda.device_count()} visible')
    except ArgumentError as e:
        print(f'ERROR: {e}', file=sys.stderr)
        print('Exiting...', file=sys.stderr)
        sys.exit(1)
    if args.gpus == 1:
        fit(0, args, cats, val_list, lpips_sd)
    else:
        torch.multiprocessing.spawn(fit, nprocs=args.gpus, args=(args, cats, val_list, lpips_sd))      # demo.py:180
    return 0


if __name__ == '__main__':
    sys.exit(main())
