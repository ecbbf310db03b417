"""DDPM -- host-side mirror of sparsefusion/vldm.py:53-555 (reference): the container the SparseFusion pipeline
builds around the VLDM UNet (utils/load_model.py:76-91) and hands to PLMSSampler (sparsefusion/distillation.py:160).

Kept: constructor keywords, ``unets`` (re-instantiated through ``Unet.cast_model_parameters`` exactly like
vldm.py:165-171, so checkpoints with keys ``unets.0.*`` load), ``noise_schedulers``, ``pred_objectives``,
``dynamic_thresholding``, ``sample_channels``, ``image_sizes``, ``clip_output``, ``clip_value``,
``unnormalize_img`` / ``normalize_img``, ``device``, ``state_dict`` / ``load_state_dict``, and the ancestral sampler
``sample`` / ``p_sample_loop`` (:363-555): a novel view straight from the VLDM, as train.py's validation asks for.
Not kept: the training loss (``forward``, vldm.py:711-776) -- training the diffusion model needs a UNet backward
(SURVEY.md §2.1 row 21); it raises NotImplementedError.

Sampling on the GPU: the T + 1 noise levels of a run are known up front, so every time-only part of the UNet is
evaluated for all of them in one ``Unet.precompute_time`` batch (cached on the DDPM: the schedule is fixed); each of
the T evaluations replays one CUDA graph (``UnetGraph``), whose cond_images share of init_conv is evaluated once per
run; and a step's latent update is one fused kernel -- ``sfb_plms_update`` with the static clip, or
``sfb_ddpm_dynamic_step``, which also finds each sample's exact |x0| quantile, with dynamic thresholding.
Classifier-free guidance evaluates the conditional and the null branch as ONE batch-2B graph (cond_images
followed by zeros, the reference's ``cond_drop_prob=1`` branch) and combines them inside the step kernel.  Every
Gaussian draw goes through ``noise_fn`` (default ``torch.randn_like``) in the reference's order and count: the start
image, then one per step (the last one multiplied by 0), T + 1 in all.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import _lib as lib
from .imagen_pytorch import GaussianDiffusionContinuousTimes, Unet, UnetGraph, alpha_cosine_log_snr, cast_tuple
from .plms import _log_snr, _step_scalars


def _identity(t, *a, **k):
    return t


class DDPM(nn.Module):
    def __init__(self, unets, *, image_sizes, conditional_encoder, conditional_embed_dim=1024, channels=3, timesteps=1000,
                 cond_drop_prob=0.1, loss_type='l2', noise_schedules='cosine', pred_objectives='noise', random_crop_sizes=None,
                 lowres_noise_schedule='linear', lowres_sample_noise_level=0.2, per_sample_random_aug_noise_level=False, conditional=True,
                 auto_normalize_img=False, p2_loss_weight_gamma=0.5, p2_loss_weight_k=1, dynamic_thresholding=True,
                 dynamic_thresholding_percentile=0.95, only_train_unet_number=None, clip_output=True, clip_value=1.0):
        super().__init__()
        self.timesteps = timesteps
        self.loss_type = loss_type
        self.conditional, self.unconditional = conditional, not conditional
        self.channels = channels
        unets = cast_tuple(unets)
        num_unets = len(unets)
        if num_unets != 1:
            raise NotImplementedError('cascaded DDPMs are not part of the SparseFusion path (one base unet: utils/load_model.py:76)')
        timesteps = cast_tuple(timesteps, num_unets)
        noise_schedules = cast_tuple(noise_schedules)
        noise_schedules = (*noise_schedules, *(('cosine',) * max(0, 2 - len(noise_schedules))))[:max(2, num_unets)]
        self.noise_schedulers = nn.ModuleList([GaussianDiffusionContinuousTimes(noise_schedule=ns, timesteps=ts)
                                               for ts, ns in zip(timesteps, noise_schedules)])
        self.lowres_noise_schedule = GaussianDiffusionContinuousTimes(noise_schedule=lowres_noise_schedule)
        self.pred_objectives = cast_tuple(pred_objectives, num_unets)
        self.conditional_embed_dim = conditional_embed_dim
        self.encode_conditional = conditional_encoder
        self.unets = nn.ModuleList([])
        self.unet_being_trained_index = -1
        self.only_train_unet_number = only_train_unet_number
        for ind, one_unet in enumerate(unets):
            assert isinstance(one_unet, Unet)
            one_unet = one_unet.cast_model_parameters(lowres_cond=not (ind == 0), cond_on_z=self.conditional,
                                                      conditional_embed_dim=self.conditional_embed_dim if self.conditional else None,
                                                      channels=self.channels, channels_out=self.channels)
            self.unets.append(one_unet)
        self.image_sizes = cast_tuple(image_sizes)
        assert num_unets == len(self.image_sizes)
        self.sample_channels = cast_tuple(self.channels, num_unets)
        self.is_video = False
        self.lowres_sample_noise_level = lowres_sample_noise_level
        self.per_sample_random_aug_noise_level = per_sample_random_aug_noise_level
        self.cond_drop_prob = cond_drop_prob
        self.can_classifier_guidance = cond_drop_prob > 0.
        self.normalize_img = (lambda img: img * 2 - 1) if auto_normalize_img else _identity
        self.unnormalize_img = (lambda img: (img + 1) * 0.5) if auto_normalize_img else _identity
        self.input_image_range = (0. if auto_normalize_img else -1., 1.)
        self.dynamic_thresholding = cast_tuple(dynamic_thresholding, num_unets)
        self.dynamic_thresholding_percentile = dynamic_thresholding_percentile
        self.clip_output, self.clip_value = clip_output, clip_value
        self.p2_loss_weight_k = p2_loss_weight_k
        self.p2_loss_weight_gamma = cast_tuple(p2_loss_weight_gamma, num_unets)
        self.register_buffer('_temp', torch.tensor([0.]), persistent=False)
        self.to(next(self.unets.parameters()).device)

    @property
    def device(self):
        return self._temp.device

    def get_unet(self, unet_number):
        assert 0 < unet_number <= len(self.unets)
        return self.unets[unet_number - 1]

    def reset_unets_all_one_device(self, device=None):
        self.unets.to(device if device is not None else self.device)

    def forward(self, *a, **k):
        raise NotImplementedError('DDPM.forward is the VLDM training loss (sparsefusion/vldm.py:711-776): outside the distillation hot path')

    @torch.no_grad()
    def sample(self, conditional_input=None, conditional_masks=None, conditional_embeds=None, video_frames=None, cond_images=None,
               inpaint_images=None, inpaint_masks=None, inpaint_resample_times=5, batch_size=1, cond_scale=1., lowres_sample_noise_level=None,
               stop_at_unet_number=None, return_all_unet_outputs=False, return_pil_images=False, device=None, use_tqdm=True, *, noise_fn=None):
        """vldm.py:446-555: ``batch_size`` views from noise, conditioned on ``cond_images`` [batch_size, C, h, w]; returns the latents
        [batch_size, channels, h, h] clamped to +-clip_value (when clip_output) and passed through unnormalize_img.  ``noise_fn(like)``
        replaces every Gaussian draw (default ``torch.randn_like``)."""
        if conditional_input is not None or conditional_embeds is not None or self.conditional:
            raise NotImplementedError('DDPM.sample: text / embedding conditioning (conditional_input, conditional_embeds) is not part of the '
                                      'SparseFusion VLDM path (conditional=False, utils/load_model.py:76-91)')
        if video_frames is not None:
            raise NotImplementedError('DDPM.sample: video_frames -- video diffusion is not part of the SparseFusion VLDM path')
        if inpaint_images is not None or inpaint_masks is not None:
            raise NotImplementedError('DDPM.sample: inpainting (inpaint_images / inpaint_masks) is not provided')
        if return_pil_images:
            raise NotImplementedError('DDPM.sample: return_pil_images=True -- decode the latents with the VAE instead')
        device = torch.device(device if device is not None else self.device)
        cur = next(self.unets.parameters()).device
        if cur.type != device.type or (device.index is not None and cur.index != device.index):
            self.reset_unets_all_one_device(device=device)       # moving drops the unet's packed weights: only when it is elsewhere
        if cond_images is None:
            raise ValueError('DDPM.sample: cond_images is required (the VLDM UNet is conditioned on epipolar features)')
        if cond_images.shape[0] != batch_size:
            raise ValueError(f'DDPM.sample: batch_size ({batch_size}) must equal cond_images.shape[0] ({cond_images.shape[0]})')
        shape = (batch_size, self.sample_channels[0], self.image_sizes[0], self.image_sizes[0])
        img = self.p_sample_loop(self.unets[0], shape, noise_scheduler=self.noise_schedulers[0], cond_images=cond_images,
                                 cond_scale=cast_tuple(cond_scale, 1)[0], pred_objective=self.pred_objectives[0],
                                 dynamic_threshold=self.dynamic_thresholding[0], use_tqdm=use_tqdm, noise_fn=noise_fn)
        return [img] if return_all_unet_outputs else img

    @torch.no_grad()
    def p_sample_loop(self, unet, shape, *, noise_scheduler, lowres_cond_img=None, lowres_noise_times=None, conditional_embeds=None,
                      conditional_mask=None, cond_images=None, inpaint_images=None, inpaint_masks=None, inpaint_resample_times=5, cond_scale=1,
                      pred_objective='noise', dynamic_threshold=True, use_tqdm=True, noise_fn=None):
        """vldm.py:363-443 with p_sample / p_mean_variance (:289-361) fused into one kernel per step"""
        if lowres_cond_img is not None or conditional_embeds is not None or inpaint_images is not None or inpaint_masks is not None:
            raise NotImplementedError('DDPM.p_sample_loop: low-res / text conditioning and inpainting are not provided')
        if pred_objective != 'noise':
            raise NotImplementedError(f"DDPM.p_sample_loop: pred_objective {pred_objective!r} -- only 'noise' (the VLDM's objective) is provided")
        if noise_scheduler.log_snr is not alpha_cosine_log_snr:
            raise NotImplementedError('DDPM.p_sample_loop: only the cosine noise schedule (the VLDM\'s) is provided')
        assert not (cond_scale != 1. and not self.can_classifier_guidance), 'imagen was not trained with conditional dropout, and thus one cannot use classifier free guidance (cond_scale anything other than 1)'
        device = next(unet.parameters()).device
        if device.type != 'cuda' or not cond_images.is_cuda:
            raise RuntimeError('DDPM.sample runs on the GPU only: move the DDPM and cond_images to a CUDA device (there is no CPU fallback)')
        noise_fn = noise_fn if noise_fn is not None else torch.randn_like
        b, T = shape[0], noise_scheduler.num_timesteps
        guided = cond_scale != 1
        row_len = math.prod(shape[1:])
        clip = float(self.clip_value) if self.clip_output else math.inf
        dynamic = bool(dynamic_threshold) and self.clip_output
        percentile = float(self.dynamic_thresholding_percentile)
        st = lib.stream()

        graph, tf_all = self._sampling_state(unet, T, device)
        cond = cond_images.float()
        if cond.shape[-1] != shape[-1]:
            cond = torch.nn.functional.interpolate(cond, shape[-1], mode='nearest')
        # guidance: the conditional rows, then the null rows -- cond_images * 0, the reference's cond_drop_prob = 1 branch (imagen_pytorch.py:1467)
        cond = torch.cat((cond, torch.zeros_like(cond))).contiguous() if guided else cond.contiguous()
        nb = cond.shape[0]
        lin = torch.linspace(1., 0., T + 1).tolist()                               # get_sampling_timesteps, fp32 (imagen_pytorch.py:226-231)

        img = noise_fn(torch.empty(shape, device=device)).to(device=device, dtype=torch.float32).contiguous()   # :385 torch.randn(shape)
        for i in range(T):
            tf = {k: v[i:i + 1].expand(nb, *v.shape[1:]) for k, v in tf_all.items()}
            x_in = torch.cat((img, img)) if guided else img
            eps = graph(x_in, None, cond, new_cond=(i == 0), time_features=tf)   # static output of the graph: consumed by the launch below
            z = noise_fn(img).to(device=device, dtype=torch.float32).contiguous()                               # :356
            alpha, sigma, alpha_next, c, noise_scale = _step_scalars(lin[i], lin[i + 1])
            out = torch.empty_like(img)
            # the guided eps is s * cond + (1 - s) * null; the reference's null + (cond - null) * s (:1468) differs from it by rounding only
            e_cond, e_null = (eps[:b], eps[b:]) if guided else (eps, None)
            if dynamic:
                lib.call('sfb_ddpm_dynamic_step', lib.fptr(img), lib.fptr(e_cond), lib.fptr(e_null), float(cond_scale), lib.fptr(z), alpha, sigma,
                         alpha_next, c, noise_scale, percentile, row_len, b, lib.fptr(out), None, None, st)
            else:
                coefs = (float(cond_scale), 1.0 - float(cond_scale)) if guided else (1.0, 0.0)
                lib.call('sfb_plms_update', lib.fptr(img), lib.fptr(e_cond), lib.fptr(e_null), None, None, *coefs, 0.0, 0.0, lib.fptr(z), alpha,
                         sigma, alpha_next, c, noise_scale, clip, lib.fptr(out), None, None, b * row_len, st)
            img = out
        if self.clip_output:
            img = img.clamp(-self.clip_value, self.clip_value)                     # :434-435
        return self.unnormalize_img(img)

    def _sampling_state(self, unet, T, device):
        """the CUDA-graph runner and the time features of the T + 1 noise levels, kept while the unet's packed weights are"""
        if unet._plan is None:
            unet.prepare()
        st = getattr(self, '_sampling', None)
        if st is None or st['unet'] is not unet or st['plan'] is not unet._plan:
            st = self._sampling = dict(unet=unet, plan=unet._plan, graph=UnetGraph(unet), time={})
        key = (T, device)
        if key not in st['time']:
            lin = torch.linspace(1., 0., T + 1).tolist()
            st['time'][key] = unet.precompute_time(torch.tensor([_log_snr(t) for t in lin], dtype=torch.float32, device=device))
        return st['graph'], st['time'][key]
