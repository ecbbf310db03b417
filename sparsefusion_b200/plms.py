"""PLMSSampler -- host-side mirror of external/plms.py (reference): the pseudo-linear-multistep sampler the
distillation loop calls once per SDS step (sparsefusion/distillation.py:160,304).

Same constructor and ``sample(image, max_thres, cond_images, cond_scale, use_tqdm, return_noise)`` signature and
return values ``(pred_x0, x_noisy, noise, alpha_cumprod)``.  ``n_steps = min(int(max_thres*plms_steps*2), plms_steps)``
steps, ``n_steps + 1`` UNet evaluations (plms.py:87,136-142), Adams-Bashforth 2/3/4 on the eps history (:144-152),
clamp of x0 to +-clip_value (:205), stochastic posterior step (:208-212).

H100 notes: each eps evaluation replays one CUDA graph of the UNet (``UnetGraph``); the schedule scalars (alpha, sigma, c,
posterior variance) are computed on the host from t / t_next and the whole latent update of a step -- Adams-Bashforth
combination, x0 prediction + clamp, posterior mean, noise injection: ~30 eager launches in the reference -- is ONE fused
kernel (``sfb_plms_update``).  Every ``torch.randn_like`` of the reference is routed through ``self.noise_fn`` (default
``torch.randn_like``) in the reference's draw order and count (including the draws whose result the reference discards), so
parity tests can inject the oracle's noise (SURVEY.md Appendix C).  ``p_sample`` / ``get_model_output`` remain as the
reference-shaped (unfused) methods; ``plms_sample_loop`` uses the fused path on CUDA.
"""
from __future__ import annotations

import math

import torch

from . import _lib as lib
from .imagen_pytorch import GaussianDiffusionContinuousTimes, UnetGraph, alpha_cosine_log_snr


def _log_snr(t: float, s: float = 0.008) -> float:
    """alpha_cosine_log_snr (external/imagen_pytorch.py:194-196) for a host scalar, evaluated with the SAME fp32 torch expression the reference's
    ``GaussianDiffusionContinuousTimes.log_snr`` runs on its fp32 time tensor.  This matters at t -> 1: cos(pi/2) is 6e-17 in fp64 but -4.4e-8 in
    fp32, so the fp64 value is -74.7 where the reference conditions the UNet on -33.9 (the ``max_thres >= .99`` branch and ``sample()`` from
    noise start there).  Everything derived from the log-SNR (alpha, sigma, posterior coefficients) is then computed from this fp32 value."""
    v = _LOG_SNR_CACHE.get(t)
    if v is None:
        if len(_LOG_SNR_CACHE) > 4096:
            _LOG_SNR_CACHE.clear()
        v = _LOG_SNR_CACHE[t] = float(alpha_cosine_log_snr(torch.tensor(t, dtype=torch.float32), s))
    return v


_LOG_SNR_CACHE = {}


def _sigmoid(x: float) -> float:
    return 1.0 / (1.0 + math.exp(-x))


def _step_scalars(t: float, t_next: float):
    """alpha, sigma of t and the q_posterior coefficients towards t_next (imagen_pytorch.py:240-258, :293-297)"""
    ls, lsn = _log_snr(t), _log_snr(t_next)
    alpha, sigma = math.sqrt(_sigmoid(ls)), math.sqrt(_sigmoid(-ls))
    alpha_next, sigma_next = math.sqrt(_sigmoid(lsn)), math.sqrt(_sigmoid(-lsn))
    c = -math.expm1(ls - lsn)
    var = sigma_next ** 2 * c
    noise_scale = 0.0 if t_next == 0 else math.exp(0.5 * math.log(max(var, 1e-20)))
    return alpha, sigma, alpha_next, c, noise_scale


class PLMSSampler:
    def __init__(self, diffusion, plms_steps=100, use_cuda_graph: bool = True, noise_fn=None):
        self.diffusion = diffusion
        self.plms_steps = plms_steps
        self.noise_fn = noise_fn if noise_fn is not None else torch.randn_like
        self.use_cuda_graph = use_cuda_graph
        self._graph = None
        self.last_unet_calls = 0

    def _eps(self, unet, x, log_snr, cond_images, cond_scale, time_features=None):
        self.last_unet_calls += 1
        if self.use_cuda_graph and cond_scale == 1:
            if self._graph is None or self._graph.unet is not unet:
                self._graph = UnetGraph(unet)
            # cond_images is fixed for the whole sampling run: its share of init_conv is evaluated by the first call only
            return self._graph(x, log_snr, cond_images, new_cond=(self.last_unet_calls == 1), time_features=time_features).clone()
        return unet.forward_with_cond_scale(x, log_snr, cond_images=cond_images, cond_scale=cond_scale)

    @torch.no_grad()
    def sample(self, image=None, max_thres=.999, cond_images=None, cond_scale=1.0, use_tqdm=True, return_noise=False, **kwargs):
        batch_size = cond_images.shape[0]
        d = self.diffusion
        shape = (batch_size, d.sample_channels[0], d.image_sizes[0], d.image_sizes[0])
        img, x_noisy, noise, alpha_cumprod = self.plms_sample_loop(d.unets[0], image=image, shape=shape, cond_images=cond_images,
                                                                   cond_scale=cond_scale, noise_scheduler=d.noise_schedulers[0],
                                                                   pred_objective=d.pred_objectives[0],
                                                                   dynamic_threshold=d.dynamic_thresholding[0], use_tqdm=use_tqdm,
                                                                   max_thres=max_thres)
        if not return_noise:
            return img
        return img, x_noisy, noise, alpha_cumprod

    @torch.no_grad()
    def plms_sample_loop(self, unet, image, shape, cond_images, cond_scale, noise_scheduler, pred_objective, dynamic_threshold,
                         use_tqdm, max_thres=None):
        batch, device = shape[0], self.diffusion.device
        self.last_unet_calls = 0
        if image is None:
            image = self.noise_fn(torch.empty(shape, device=device))        # plms.py:73 (torch.randn(shape)); routed through noise_fn for parity tests
        else:
            assert max_thres is not None
        if image.is_cuda and pred_objective == 'noise' and not dynamic_threshold and self.diffusion.clip_output:
            return self._fused_loop(unet, image.float().contiguous(), cond_images, cond_scale, float(max_thres))
        short = GaussianDiffusionContinuousTimes(noise_schedule='cosine', timesteps=self.plms_steps)
        if max_thres >= .99:
            timesteps = short.get_sampling_timesteps(batch, device=device)
            noise = self.noise_fn(image)
            x_noisy, log_snr = short.q_sample(image, t=max_thres, noise=noise)
            img = image
        else:
            n_steps = min(int(max_thres * self.plms_steps * 2), self.plms_steps)
            timesteps = short.get_sampling_timesteps_custom(batch, device=device, max_thres=max_thres, n_steps=n_steps)
            noise = self.noise_fn(image)
            img, log_snr = short.q_sample(image, t=max_thres, noise=noise)
            x_noisy = img
        old_eps = []
        for times, times_next in timesteps:
            img, pred_x0, e_t = self.p_sample(unet, img, times, t_next=times_next, cond_images=cond_images, cond_scale=cond_scale,
                                              noise_scheduler=noise_scheduler, pred_objective=pred_objective,
                                              dynamic_threshold=dynamic_threshold, old_eps=old_eps)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
        if self.diffusion.clip_output:
            img = img.clamp(-self.diffusion.clip_value, self.diffusion.clip_value)
        return self.diffusion.unnormalize_img(img), x_noisy, noise, torch.sigmoid(log_snr)

    @torch.no_grad()
    def _fused_loop(self, unet, image, cond_images, cond_scale, max_thres):
        """plms_sample_loop (:54-119) + p_sample (:122-156) with the per-step latent math in one kernel"""
        b = image.shape[0]
        clip = float(self.diffusion.clip_value)
        if max_thres >= .99:                                                      # :80-85
            lin = torch.linspace(1., 0., self.plms_steps + 1).tolist()
            noise = self.noise_fn(image)
            a0, s0 = math.sqrt(_sigmoid(_log_snr(max_thres))), math.sqrt(_sigmoid(-_log_snr(max_thres)))
            x_noisy = a0 * image + s0 * noise
            img = image
        else:                                                                     # :86-93
            n_steps = min(int(max_thres * self.plms_steps * 2), self.plms_steps)
            lin = torch.linspace(max_thres, 0.0, n_steps + 1).tolist()
            noise = self.noise_fn(image)
            a0, s0 = math.sqrt(_sigmoid(_log_snr(max_thres))), math.sqrt(_sigmoid(-_log_snr(max_thres)))
            img = a0 * image + s0 * noise
            x_noisy = img
        n = img.numel()
        st = lib.stream

        # the run's noise levels are known now: everything of the UNet that depends on them only (time embedding, conditioning tokens, all
        # time MLPs) is evaluated for the whole run in one batch (Unet.precompute_time) instead of once per evaluation
        tf_all = None
        if self.use_cuda_graph and cond_scale == 1 and len(lin) > 1 and hasattr(unet, 'precompute_time'):
            tf_all = unet.precompute_time(torch.tensor([_log_snr(t) for t in lin], dtype=torch.float32, device=img.device))
        level = {t: i for i, t in enumerate(lin)}

        def eps_at(x, t):
            ls = torch.full((b,), _log_snr(t), dtype=torch.float32, device=x.device)
            tf = None
            if tf_all is not None:
                i = level[t]
                tf = {k: v[i:i + 1].expand(b, *v.shape[1:]) for k, v in tf_all.items()}
            return self._eps(unet, x, ls, cond_images, cond_scale, time_features=tf)

        def update(x, eps_list, coefs, z, t, t_next):
            alpha, sigma, alpha_next, c, noise_scale = _step_scalars(t, t_next)
            out = torch.empty_like(x)
            eps_list = [e.contiguous() for e in eps_list]      # held until after the launch
            z = z.contiguous()
            ptrs = [lib.fptr(e) for e in eps_list] + [None] * (4 - len(eps_list))
            cf = list(coefs) + [0.0] * (4 - len(coefs))
            lib.call('sfb_plms_update', lib.fptr(x), *ptrs, *cf, lib.fptr(z), alpha, sigma, alpha_next, c, noise_scale, clip, lib.fptr(out),
                     None, None, n, st())
            return out

        old_eps = []
        for i in range(len(lin) - 1):
            t, t_next = lin[i], lin[i + 1]
            e_t = eps_at(img, t)
            self.noise_fn(img)                                                    # draw of the first get_model_output call (:136; result unused)
            if len(old_eps) == 0:                                                 # pseudo improved Euler (:137-143)
                x_prev = update(img, [e_t], [1.0], self.noise_fn(img), t, t_next)
                e_next = eps_at(x_prev, t_next)
                self.noise_fn(x_prev)                                             # draw of the third call (:142; result unused)
                eps_list, coefs = [e_t, e_next], [0.5, 0.5]
            elif len(old_eps) == 1:
                eps_list, coefs = [e_t, old_eps[-1]], [1.5, -0.5]
            elif len(old_eps) == 2:
                eps_list, coefs = [e_t, old_eps[-1], old_eps[-2]], [23 / 12, -16 / 12, 5 / 12]
            else:
                eps_list, coefs = [e_t, old_eps[-1], old_eps[-2], old_eps[-3]], [55 / 24, -59 / 24, 37 / 24, -9 / 24]
            img = update(img, eps_list, coefs, self.noise_fn(img), t, t_next)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
        img = img.clamp(-clip, clip)
        acp = torch.full((b,), _sigmoid(_log_snr(max_thres)), dtype=torch.float32, device=img.device)
        return self.diffusion.unnormalize_img(img), x_noisy, noise, acp

    @torch.no_grad()
    def p_sample(self, unet, x, t, t_next, cond_images, cond_scale, noise_scheduler, pred_objective, dynamic_threshold, old_eps):
        args = (cond_images, cond_scale, noise_scheduler, pred_objective, dynamic_threshold)
        _, _, e_t = self.get_model_output(unet, x, t, t_next, *args)
        if len(old_eps) == 0:
            x_prev, _, _ = self.get_model_output(unet, x, t, t_next, *args, pred_e=e_t)
            _, _, e_t_next = self.get_model_output(unet, x_prev, t_next, t_next, *args)
            e_t_prime = (e_t + e_t_next) / 2
        elif len(old_eps) == 1:
            e_t_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            e_t_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            e_t_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        x_prev, pred_x0, _ = self.get_model_output(unet, x, t, t_next, *args, pred_e=e_t_prime)
        return x_prev, pred_x0, e_t

    def get_model_output(self, unet, x, t, t_next, cond_images, cond_scale, noise_scheduler, pred_objective, dynamic_threshold, pred_e=None):
        assert pred_objective == 'noise'
        b = x.shape[0]
        if pred_e is None:
            pred_e = self._eps(unet, x, noise_scheduler.get_condition(t), cond_images, cond_scale)
        x_start = noise_scheduler.predict_start_from_noise(x, t=t, noise=pred_e)
        if self.diffusion.clip_output:
            if dynamic_threshold:
                raise NotImplementedError('dynamic thresholding is unreachable in the reference too (plms.py:198 reads a missing attribute)')
            x_start = x_start.clamp(-self.diffusion.clip_value, self.diffusion.clip_value)
        model_mean, _, model_log_variance = noise_scheduler.q_posterior(x_start=x_start, x_t=x, t=t, t_next=t_next)
        noise = self.noise_fn(x)
        nonzero_mask = (1 - (t_next == 0).float()).reshape(b, *((1,) * (len(x.shape) - 1)))
        x_prev = model_mean + nonzero_mask * (0.5 * model_log_variance).exp() * noise
        return x_prev, x_start, pred_e
