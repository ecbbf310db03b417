"""The two intermediate stages SparseFusion compares the distilled scene against, scored on the GPU like the scene itself:

* EFT: the Epipolar Feature Transformer's own image of each scene view (``SceneCache.target_eft_image``, the low-resolution render of the
  feature cache upsampled to the image size, distillation.py:118-119);
* VLDM: a novel view sampled from pure noise by the view-conditioned diffusion model, conditioned on the EFT features of that view
  (``SceneCache.target_features``): PLMS from ``max_thres = .999`` (``PLMSSampler.sample``'s default), optionally with classifier-free
  guidance, then ``unnormalize(vae.decode(x0 / z_scale_factor)).clip(0, 1)`` as the reference decodes its samples (distillation.py:309).

``sample_vldm_views`` batches a scene's views through the sampler (UNet CUDA graph, fused update kernel; with guidance the conditional and
null rows of a step are one batch-2B evaluation) and the VAE decoder.  ``evaluate_baselines`` scores both stages with ``evaluate_scene``'s
metrics and writes ``{save_dir}/metrics/{seq_name}_eft.txt``, ``{seq_name}_vldm.txt`` and ``{save_dir}/render_gifs/{seq_name}_baselines.gif``.
The cache's first V target entries are the V scene views (the cache lists the scene views first, then the circle-path views).
"""
from __future__ import annotations

import math

import torch

from .distillation import KeyedNoise, SceneCache, unnormalize, view_seed
from .evaluate import EvalViews, score_images, write_scene_metrics
from .plms import PLMSSampler

VLDM_STREAM = 5      # view_seed stream of the VLDM samples' Gaussian draws (iteration 0)
VLDM_MAX_THRES = .999


def _check_sampling_args(vldm, features, cond_scale, plms_steps, max_batch):
    """every argument check of ``sample_vldm_views`` that needs no device work"""
    if not isinstance(features, torch.Tensor) or features.dim() != 4:
        raise ValueError(f'sample_vldm_views: features must be a [V, C, h, w] tensor (got {getattr(features, "shape", type(features))})')
    if isinstance(plms_steps, bool) or not isinstance(plms_steps, int) or plms_steps < 1:
        raise ValueError(f'sample_vldm_views: plms_steps must be a positive int (got {plms_steps!r})')
    if isinstance(max_batch, bool) or not isinstance(max_batch, int) or max_batch < 1:
        raise ValueError(f'sample_vldm_views: max_batch must be a positive int (got {max_batch!r})')
    check_baseline_options(vldm, cond_scale)
    if not features.is_cuda:
        raise RuntimeError('sample_vldm_views: features must be a CUDA tensor (there is no CPU path)')


@torch.no_grad()
def sample_vldm_views(vldm, vae, features: torch.Tensor, *, seed: int, cond_scale: float = 1.0, plms_steps: int = 50, max_batch: int = 32,
                      z_scale_factor: float = 0.18215, sampler: PLMSSampler = None) -> torch.Tensor:
    """novel views [V, 3, H, W] in [0, 1] from the VLDM ``vldm`` (a ``DDPM``), one per row of the EFT features ``features`` [V, C, h, w]:
    ``PLMSSampler.sample`` from pure noise (``max_thres = .999``, ``plms_steps`` steps, ``cond_scale``), then
    ``unnormalize(vae.decode(x0 / z_scale_factor)).clip(0, 1)``.  Views run in batches of at most ``max_batch``.

    Every Gaussian draw of view v comes from the generator seeded ``view_seed(seed, 0, v, VLDM_STREAM)`` (``KeyedNoise``), so a view's
    draws, and up to fp32 summation order its image, do not depend on ``max_batch`` or on the views that share its batch.  ``sampler``
    (optional) is a ``PLMSSampler`` of ``vldm`` with ``plms_steps`` steps to reuse, e.g. to keep its CUDA graphs across scenes.
    Arguments are checked before any device work: ValueError for bad values and for guidance on a VLDM without conditional dropout,
    RuntimeError for CPU features."""
    _check_sampling_args(vldm, features, cond_scale, plms_steps, max_batch)
    if sampler is None:
        sampler = PLMSSampler(vldm, plms_steps)
    elif sampler.diffusion is not vldm or sampler.plms_steps != plms_steps:
        raise ValueError('sample_vldm_views: the sampler given belongs to another VLDM or runs another number of steps')
    dev = features.device
    V = features.shape[0]
    out = []
    prev = sampler.noise_fn
    try:
        with torch.cuda.device(dev):
            for lo in range(0, V, max_batch):
                views = list(range(lo, min(V, lo + max_batch)))
                sampler.noise_fn = KeyedNoise([view_seed(seed, 0, v, VLDM_STREAM) for v in views], dev)
                x0 = sampler.sample(cond_images=features[lo:lo + len(views)].float(), max_thres=VLDM_MAX_THRES, cond_scale=cond_scale, use_tqdm=False)
                out.append(unnormalize(vae.decode(x0 / z_scale_factor)).clip(0.0, 1.0))          # distillation.py:309
    finally:
        sampler.noise_fn = prev
    return torch.cat(out) if out else torch.zeros(0, 3, 0, 0, device=dev)


def check_baseline_options(vldm, cond_scale, use_diffusion=True):
    """the checks of the baseline options a caller can make before any scene is built: ValueError without the diffusion model's features
    (``use_diffusion=False``) or for guidance on a VLDM without conditional dropout"""
    if not use_diffusion:
        raise ValueError('the EFT / VLDM baselines need the EFT feature cache, which only use_diffusion=True builds')
    if not math.isfinite(float(cond_scale)):
        raise ValueError(f'vldm_cond_scale must be finite (got {cond_scale!r})')
    if cond_scale != 1 and not vldm.can_classifier_guidance:
        raise ValueError('the VLDM was not trained with conditional dropout (cond_drop_prob == 0), so classifier-free guidance '
                         f'(cond_scale {cond_scale} != 1) is not available')


def check_baseline_cache(cache, views):
    """ValueError unless the cache's first V target entries can stand for the V scene views of ``views``"""
    V = views.rgb.shape[0]
    hw = tuple(views.rgb.shape[2:])
    n = cache.target_features.shape[0]
    if cache.target_eft_image.shape[0] != n or n < V:
        raise ValueError(f'evaluate_baselines: the cache holds {n} feature maps and {cache.target_eft_image.shape[0]} EFT images; the scene has '
                         f'{V} views, which must be its first entries')
    if tuple(cache.target_eft_image.shape[2:]) != hw:
        raise ValueError(f'evaluate_baselines: EFT images are {tuple(cache.target_eft_image.shape[2:])}, the ground truth {hw}')


@torch.no_grad()
def evaluate_baselines(save_dir: str, seq_name: str, vldm, vae, cache: SceneCache, views: EvalViews, percep, *, seed: int,
                       cond_scale: float = 1.0, plms_steps: int = 50, max_batch: int = 32, z_scale_factor: float = 0.18215,
                       sampler: PLMSSampler = None) -> dict:
    """scores of the EFT and VLDM baselines on the V scene views of ``views``: ``{'eft': SceneEval, 'vldm': SceneEval}``.

    EFT: ``cache.target_eft_image[:V]``.  VLDM: ``sample_vldm_views(vldm, vae, cache.target_features[:V], seed=seed, ...)``.  Both are scored
    against ``views.rgb`` as ``evaluate_scene`` scores a render (``score_images``: PSNR, SSIM, LPIPS by ``percep``, nan without it), and
    written as ``{save_dir}/metrics/{seq_name}_eft.txt`` / ``{seq_name}_vldm.txt`` in ``write_scene_metrics``' format, with
    ``{save_dir}/render_gifs/{seq_name}_baselines.gif``: one GT | EFT | VLDM frame per view.  The VLDM images must come out at the ground
    truth's size (latent size times the VAE's factor)."""
    from .video import require_pillow, to_uint8, write_gif
    require_pillow()
    check_baseline_cache(cache, views)
    V = views.rgb.shape[0]
    _check_sampling_args(vldm, cache.target_features, cond_scale, plms_steps, max_batch)
    dev = cache.target_features.device
    with torch.cuda.device(dev):
        gt = views.rgb.to(dev).float()
        vldm_img = sample_vldm_views(vldm, vae, cache.target_features[:V], seed=seed, cond_scale=cond_scale, plms_steps=plms_steps,
                                     max_batch=max_batch, z_scale_factor=z_scale_factor, sampler=sampler)
        if vldm_img.shape != gt.shape:
            raise ValueError(f'evaluate_baselines: VLDM images are {tuple(vldm_img.shape)}, the ground truth {tuple(gt.shape)}')
        scores = {}
        for name, img in (('eft', cache.target_eft_image[:V]), ('vldm', vldm_img)):
            scores[name] = score_images(img.float().permute(0, 2, 3, 1).contiguous(), gt, percep)
            print(f'{name} baseline, scene {seq_name}')
            write_scene_metrics(f'{save_dir}/metrics/{seq_name}_{name}.txt', scores[name])
        gif_path = f'{save_dir}/render_gifs/{seq_name}_baselines.gif'
        write_gif(gif_path, to_uint8(gt.permute(0, 2, 3, 1), scores['eft'].image, scores['vldm'].image))
        print('saved video', gif_path)
    return scores


def score_baselines(gpu, args, model_tuple, save_dir, scenes, *, scene_builder=None, seed=None, loss_fn_vgg=None, cond_scale=1.0,
                    max_batch=32):
    """the EFT and VLDM baselines of every scene without any distillation: no NeRF network, no loop.  Takes ``distill_scenes``' arguments
    (``model_tuple`` = (eft, vae, vldm); ``scenes`` = [(seq_name, scene_cameras, scene_rgb, scene_mask, scene_valid_region, input_idx)]),
    builds each scene's cache and views with the scene builder (``ReferenceSceneBuilder``, or ``scene_builder``, which must provide
    ``eval_views``), and runs ``evaluate_baselines`` per scene: scene k's VLDM draws keyed by ``seed + k`` (``seed`` drawn from torch's seed
    when None), LPIPS with ``loss_fn_vgg``'s weights (nan without it), guidance scale ``cond_scale``.  Writes
    ``{save_dir}/metrics/{seq_name}_eft.txt``, ``{seq_name}_vldm.txt`` and ``{save_dir}/render_gifs/{seq_name}_baselines.gif``.
    Returns one ``evaluate_baselines`` result per scene, in the order of ``scenes``."""
    from .distillation import ReferenceSceneBuilder
    from .lpips_vgg import PerceptualLoss
    from .video import require_pillow
    eft, vae, vldm = model_tuple
    check_baseline_options(vldm, cond_scale)
    require_pillow()
    builder = scene_builder if scene_builder is not None else ReferenceSceneBuilder(gpu)
    if not callable(getattr(builder, 'eval_views', None)):
        raise TypeError(f'score_baselines needs the scene builder to provide eval_views(scene_cameras, scene_rgb, scene_mask); '
                        f'{type(builder).__name__} has none')
    device = torch.device('cuda', gpu) if isinstance(gpu, int) else torch.device(gpu)
    views = [builder.eval_views(cams, rgb, mask).to(device) for _, cams, rgb, mask, _, _ in scenes]
    caches = [builder.build(eft, cams, rgb, mask, input_idx, use_diffusion=True).to(device) for _, cams, rgb, mask, _, input_idx in scenes]
    for v, c in zip(views, caches):
        check_baseline_cache(c, v)
    base_seed = torch.seed() % (2 ** 31) if seed is None else int(seed)
    with torch.cuda.device(device):
        percep = None if loss_fn_vgg is None else PerceptualLoss('vgg', device=device).load_state_dict(loss_fn_vgg.state_dict())
        sampler = PLMSSampler(vldm, 50)
        return [evaluate_baselines(save_dir, sc[0], vldm, vae, c, v, percep, seed=base_seed + k, cond_scale=cond_scale, max_batch=max_batch,
                                   sampler=sampler)
                for k, (sc, c, v) in enumerate(zip(scenes, caches, views))]
