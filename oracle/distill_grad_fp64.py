"""oracle/distill_grad_fp64.py -- the gradient one distillation sub-step hands to Adam, restated in fp64 from the reference's loss
expressions (sparsefusion/distillation.py:185-352) stage by stage, each stage with a per-element bound.

TEST INFRASTRUCTURE ONLY.

The kernels of every stage have their own fp64 suites (oracle/step_fp64.py, oracle/field_fp64.py), which check a kernel given the
arguments it was called with.  What is new here is the ARGUMENTS: they come from the configuration (``StepConfig``) and the reference's
expressions, never from what the step passed, so a wrong lambda, weight, view scale, argument order or learning rate shows as a stage
whose output is outside its bound.  Stages (inputs are what the GPU run produced at the previous stage's output):

  S1  loss -> render:   ``photometric_grad`` / ``fusion_grad``: d loss / d image [N,3] and d loss / d weights_sum [N]
  S2  composite:        ``composite_grad``: d loss / d sigma [N,T], d loss / d rgb [N,T,3] (field_fp64.composite)
  S3  field:            ``field_grad``: the parameter gradients of one render (field_fp64.FieldFP64.backward)
  S4  Adam:             ``step_lr`` / ``adam_reference``: the learning rates, the step count and the update of fp64 torch.optim.Adam + StepLR

``end_to_end_grad`` is the same gradient through fp64 autograd alone (field, compositing and the reference's loss in one graph); the host
tests hold the staged chain to it.  ``emulate_fusion`` evaluates the fused fusion path's S1 in fp32 with switches that inject the wiring defects the bounds must see.
"""
from __future__ import annotations

import math
import warnings
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import field_fp64 as f64
from .field_fp64 import ATOL, U32, gamma
from .step_fp64 import HUBER_S, f32, fusion_mask, glue_nearest, up2_taps

ENT_LO, ENT_HI = f32(1e-5), f32(1 - 1e-5)        # the entropy clamp (distillation.py:238-240, :340-342)
LOG2_ENT_EDGE = math.log2(1.0 / ENT_LO)          # |log2((1 - a) / a)| at the clamp's edges


@dataclass
class StepConfig:
    """what the reference's loop sets (distillation.py:153-178): the loss weights, Adam's learning rate (encoder x10,
    network_grid.py:230-231) and the StepLR schedule; the tests build the Distiller from the same values and read nothing back"""
    lambda_color: float = 1.0
    lambda_sil: float = 1.0
    lambda_opacity: float = 1e-3
    lambda_entropy: float = 0.0
    lambda_percep: float = 0.1
    lr: float = 5e-4
    step_size: int = 3000
    gamma: float = 0.2
    betas: tuple = (0.9, 0.999)
    eps: float = 1e-8


# ------------------------------------------------------------------------------------------------ SDS weight
def sds_weight(max_thres: float, s: float = 0.008):
    """(1 - alpha_cumprod, bound) at time ``max_thres`` of the cosine schedule (alpha_cosine_log_snr, imagen_pytorch.py:194-196), in fp64:
    alpha_cumprod = sigmoid(log_snr) = cos^2((t + s) / (1 + s) pi / 2), so the weight is sin^2 of the same angle.

    The run forms log_snr = -log(cos^-2 - 1) in fp32 (its sampler conditions the UNet on that value) and the weight from it.  The
    argument, the cosine (amplified by a tan a), the power and the subtraction (amplified by cos^-2 / (cos^-2 - 1)) and the log round; a
    log-SNR error d moves the weight by alpha (1 - alpha) d."""
    a = (max_thres + s) / (1 + s) * math.pi * 0.5
    c2 = math.cos(a) ** 2
    w = math.sin(a) ** 2
    x = 1.0 / c2 - 1.0
    ls = -math.log(x)
    d_ls = gamma(8) * (1.0 / c2) / x * (1 + 2 * a * math.tan(a)) + gamma(2) * abs(ls)
    return w, c2 * w * d_ls + 1e-300


# ------------------------------------------------------------------------------------------------ S1: loss -> render
def _huber_grad(d):
    return d / (HUBER_S * torch.sqrt(1 + d * d / (HUBER_S * HUBER_S)))


def _eager_vanish(d, g):
    """the reference's huber(x, y).abs() in fp32: where sqrt(1 + d^2 / s^2) rounds to 1 (d^2 / s^2 within a few ulps of 0) the value is
    exactly 0 and abs()'s backward (sign(0) = 0) drops the term's gradient; the fused kernels use the analytic derivative there.  Either is
    the reference's arithmetic: slack |g|."""
    return torch.where(d * d / (HUBER_S * HUBER_S) <= 8 * U32, g.abs(), torch.zeros_like(g))


def entropy_grad(sil: torch.Tensor, le: float, n: int):
    """d (le * mean H(clamp(sil, 1e-5, 1 - 1e-5))) / d sil in log2 (distillation.py:238-241) by fp64 autograd, with the per-element bound of
    tests/test_entropy_progress_gpu.py's derivation: log2f within an ulp, 1 - a rounding once, the product, difference and scaling a few
    times more -> gamma(12) le (|log2 a| + |log2 (1 - a)| + 1) / n.  Zero where the clamp moves the silhouette (clamp's backward)."""
    s = sil.double().reshape(-1).clone().requires_grad_(True)
    a = s.clamp(ENT_LO, ENT_HI)
    h = -a * torch.log2(a) - (1 - a) * torch.log2(1 - a)
    (le * h.sum() / n).backward()
    ad = a.detach()
    return s.grad, gamma(12) * le * (torch.log2(ad).abs() + torch.log2(1 - ad).abs() + 1) / n


def _entropy_slack(sv, delta, le, n):
    """how far the entropy gradient can move when the silhouette itself is only known within delta (the eager path's bilinear
    up-sampling): its derivative le / (n ln 2 a (1 - a)) over the interval, and the whole jump where the interval meets a clamp edge"""
    lo = torch.clamp(torch.minimum(sv, 1 - sv) - delta, min=ENT_LO)
    inner = le * delta / (n * math.log(2) * lo * (1 - lo))
    edge = ((sv - ENT_LO).abs() <= delta) | ((sv - ENT_HI).abs() <= delta)
    return torch.where(edge, torch.full_like(sv, le * LOG2_ENT_EDGE / n), inner)


def _scaled(y, b, scale):
    """the view-batched step multiplies a view's gradient by 1/V in fp32: one more rounding"""
    if scale == 1.0:
        return y, b
    return y * scale, b * scale + U32 * (y * scale).abs()


def photometric_grad(img, ws, rgb, mask, hw: int, scale: int, cfg: StepConfig, *, eager=False, view_scale=1.0) -> Dict:
    """S1 of the photometric sub-step (distillation.py:210-241): render img [n,3], ws [n] against input view rgb [3,H,W], mask [1,H,W]
    down-sampled by nearest (:216-217).  Returns {'g_img': (y, bound), 'g_ws': (y, bound)}.  Bounds: the fused kernel's chains
    (step_fp64.ref_photometric: gamma(10), gamma(14)) or, for the reference's torch expressions (``eager``), 24 roundings per term."""
    n = hw * hw
    lc, ls, lo, le = (f32(v) for v in (cfg.lambda_color, cfg.lambda_sil, cfg.lambda_opacity, cfg.lambda_entropy))
    tgt = glue_nearest(rgb.double().cpu(), hw, hw, scale).reshape(3, n).t()
    tm = glue_nearest(mask.double().cpu().reshape(1, hw * scale, hw * scale), hw, hw, scale).reshape(n)
    x, sv = img.double().cpu(), ws.double().cpu().reshape(n)
    gi = lc * _huber_grad(x - tgt) / (3 * n)
    sil = ls * _huber_grad(sv - tm) / n
    op = lo * sv / (torch.sqrt(sv * sv + f32(0.01)) * n)
    ri, rs = (gamma(24), gamma(24)) if eager else (gamma(10), gamma(14))
    gs, bs = sil + op, rs * (sil.abs() + op.abs())
    bi = ri * gi.abs()
    if eager:
        bi, bs = bi + _eager_vanish(x - tgt, gi), bs + _eager_vanish(sv - tm, sil)
    if le > 0:
        ge, be = entropy_grad(sv, le, n)
        gs, bs = gs + ge, bs + be + gamma(2) * ge.abs()
    return {'g_img': _scaled(gi, bi + ATOL, view_scale), 'g_ws': _scaled(gs, bs + ATOL, view_scale)}


def upsample(img, ws, hw):
    """F.interpolate(scale_factor=2, mode='bilinear') of the render's colour and opacity planes [4,2hw,2hw] in fp64 (distillation.py:287-288),
    with the bound of an fp32 evaluation (four products and adds of exact quarter weights: gamma(4) on the sum of |w||v|)"""
    My, Mx = up2_taps(hw), up2_taps(hw)
    planes = torch.cat((img.double().cpu().t().reshape(3, hw, hw), ws.double().cpu().reshape(1, hw, hw)))
    return My @ planes @ Mx.t(), gamma(4) * (My @ planes.abs() @ Mx.t()) + ATOL


def adjoint(g_up, b_up, hw):
    """the bilinear x2's adjoint of a gradient [4,2hw,2hw] and of its bound, plus the adjoint's own rounding (<= 16 taps per render
    pixel, each weight product exact: gamma(16) on sum |w||g|, whatever the order of accumulation -- torch's backward adds with atomics)"""
    My, Mx = up2_taps(hw), up2_taps(hw)
    y = My.t() @ g_up @ Mx
    b = My.t() @ b_up @ Mx + gamma(16) * (My.t() @ g_up.abs() @ Mx) + ATOL
    return (y[:3].reshape(3, -1).t(), b[:3].reshape(3, -1).t()), (y[3].reshape(-1), b[3].reshape(-1))


def fusion_grad_up(u, delta, target, mode: str, cfg: StepConfig, *, weight=None, weight_err=0.0, g_percep=None, eager=False):
    """S1 of the fusion sub-step at the up-sampled planes u [4,H,W] (known within ``delta``, elementwise): (g_up, bound) [4,H,W].
    mode 'sds': weight |u - pred| mean (:307-310) plus lambda_percep times ``g_percep`` (the perceptual gradient w.r.t. the render,
    :312-314); mode 'eft': huber to the EFT image and its mask (:316-329).  Plus opacity (:336) and entropy (:338-344) of u[3]."""
    H, W = u.shape[1], u.shape[2]
    HW = H * W
    lc, ls, lo, le = (f32(v) for v in (cfg.lambda_color, cfg.lambda_sil, cfg.lambda_opacity, cfg.lambda_entropy))
    t = target.double().cpu()
    d = u[:3] - t
    if mode == 'sds':
        g = weight * torch.sign(d) / (3 * HW)
        bc = (gamma(4) if eager else gamma(2)) * g.abs() + weight_err / (3 * HW)
        bc = bc + torch.where(d.abs() <= delta[:3], torch.full_like(d, 2 * (weight + weight_err) / (3 * HW)), torch.zeros_like(d))
        if g_percep is not None:
            ge = f32(cfg.lambda_percep) * g_percep.double().cpu()
            g, bc = g + ge, bc + gamma(2) * ge.abs()
    else:
        g = lc * _huber_grad(d) / (3 * HW)
        bc = (gamma(24) if eager else gamma(11)) * g.abs() + lc * delta[:3] / (HUBER_S * 3 * HW)
        if eager:
            bc = bc + _eager_vanish((d.abs() - delta[:3]).clamp(min=0), g)
    sv, ds = u[3], delta[3]
    op = lo * sv / (torch.sqrt(sv * sv + f32(0.01)) * HW)
    gs, bs = op, op.abs()
    slack = lo * 10 * ds / HW                                  # |d/ds s / sqrt(s^2 + .01)| <= 10
    if mode == 'eft':
        m = fusion_mask(target).view(H, W)
        sg = ls * _huber_grad(sv - m) / HW
        gs, bs = gs + sg, bs + sg.abs()
        slack = slack + ls * ds / (HUBER_S * HW)
        if eager:
            slack = slack + _eager_vanish(((sv - m).abs() - ds).clamp(min=0), sg)
    bs = (gamma(24) if eager else gamma(14)) * bs + slack
    if le > 0:
        ge, be = entropy_grad(sv, le, HW)
        ge, be = ge.view(H, W), be.view(H, W)
        gs, bs = gs + ge, bs + be + gamma(2) * ge.abs() + _entropy_slack(sv, ds, le, HW)
    return torch.cat((g, gs[None])), torch.cat((bc, bs[None])) + ATOL


def fusion_grad(img, ws, hw: int, target, mode: str, cfg: StepConfig, *, up=None, weight=None, weight_err=0.0, g_percep=None, eager=False,
                view_scale=1.0) -> Dict:
    """S1 of the fusion sub-step from the render img [n,3], ws [n]: the up-sampled planes are the kernel's own ``up`` when given (the fused
    path, where they are an output of their own checked kernel), else the fp64 up-sampling of the render, known within its rounding bound
    (where |u - pred| is within it the L1 term's sign is a tie and either sign passes).  Then ``fusion_grad_up`` and the adjoint."""
    if up is None:
        u, delta = upsample(img, ws, hw)
    else:
        u, delta = up.double().cpu(), torch.zeros(up.shape, dtype=torch.float64)
    g_up, b_up = fusion_grad_up(u, delta, target, mode, cfg, weight=weight, weight_err=weight_err, g_percep=g_percep, eager=eager)
    (gi, bi), (gs, bs) = adjoint(g_up, b_up, hw)
    return {'g_img': _scaled(gi, bi, view_scale), 'g_ws': _scaled(gs, bs, view_scale), 'g_up': (g_up, b_up)}


# ------------------------------------------------------------------------------------------------ S1 as the reference writes it
def huber(x, y, scaling=0.1):  # utils/common_utils.py:183-190
    diff_sq = (x - y) ** 2
    return ((1 + diff_sq / (scaling ** 2)).clamp(1e-4).sqrt() - 1) * float(scaling)


def _entropy(sil):
    a = sil.clamp(ENT_LO, ENT_HI)
    return (- a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean()


def reference_loss(kind: str, image, sil, cfg: StepConfig, *, rgb=None, mask=None, target=None, weight=None, percep=None):
    """the reference's loss of one sub-step as torch expressions (image [1,3,h,w], sil [1,1,h,w], any dtype): 'photo' (:210-241, rgb /
    mask the full-size input view), 'eft' (:287-288, :316-344) and 'sds' (:287-288, :307-344, ``percep`` a callable (a, b) -> distance).
    The constants (huber's 0.1, the opacity's .01, the lambdas) are the fp32 values an fp32 run computes with."""
    lc, ls, lo, le, lp = (f32(v) for v in (cfg.lambda_color, cfg.lambda_sil, cfg.lambda_opacity, cfg.lambda_entropy, cfg.lambda_percep))
    if kind == 'photo':
        s = image.shape[-1] / rgb.shape[-1]
        brgb, bmask = F.interpolate(rgb, scale_factor=s), F.interpolate(mask, scale_factor=s)
        loss = lc * huber(image, brgb, HUBER_S).abs().mean() + ls * huber(sil, bmask, HUBER_S).abs().mean()
    else:
        image = F.interpolate(image, scale_factor=2, mode='bilinear')
        sil = F.interpolate(sil, scale_factor=2, mode='bilinear')
        if kind == 'eft':
            noisy_mask = fusion_mask(target[0]).to(target.device, target.dtype).view(1, 1, *target.shape[-2:])   # mean(dim=1) > .1, in fp32
            loss = lc * huber(image, target, HUBER_S).abs().mean() + ls * huber(sil, noisy_mask, HUBER_S).abs().mean()
        else:
            loss = weight * (image - target).abs().mean()
            if percep is not None:
                loss = loss + percep(image, target) * lp
    loss = loss + lo * torch.sqrt(sil ** 2 + f32(.01)).mean()
    if le > 0:
        loss = loss + le * _entropy(sil)
    return loss


def nchw(img, ws, hw):
    return img.reshape(1, hw, hw, 3).permute(0, 3, 1, 2), ws.reshape(1, hw, hw, 1).permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ S2, S3
def composite_grad(zs, sigma, rgb, nears, fars, bg, g_image, g_ws, device=None) -> Dict:
    """S2: field_fp64.composite's backward of the render's upstream gradients; bound RTOL_COMP on its companions.  ``hit``: the rays
    that meet the box (a missed ray's gradients are exactly zero).  Also the forward ('image', 'weights_sum'), which the render the
    loss saw must equal within the same bound."""
    dev = device or zs.device
    r = f64.composite(zs.to(dev), sigma.to(dev), rgb.to(dev), nears.to(dev), fars.to(dev), bg, g_image.to(dev), g_ws.to(dev), None)
    hit = (nears < fars).to(dev)
    return {'g_sigma': (r['g_sigma'], f64.RTOL_COMP * r['g_sigma_abs']), 'g_rgb': (r['g_rgb'], f64.RTOL_COMP * r['g_rgb_abs']), 'hit': hit,
            'image': (r['image'], f64.RTOL_COMP * r['image_abs']), 'weights_sum': (r['weights_sum'], f64.RTOL_COMP * r['weights_sum_abs'])}


def field_grad(params: Dict[str, torch.Tensor], rays_o, rays_d, zs, g_sigma, g_rgb, level_scales, path: str, sm: int, bound=4.0, device=None):
    """S3: the parameter gradients of <sigma, g_sigma> + <rgb, g_rgb> at the render's samples (FieldFP64.backward), each as (y, rtol
    companion, slack): rtol is wgrad_rtol of the field path for the weights and biases, and the per-point bound plus the row's hit count
    for the embeddings.  'sigma' and 'rgb': the field's forward at the samples (RTOL_POINT on the companions), which the values the
    compositing used must equal."""
    dev = device or zs.device
    x = f64.ray_points(rays_o.to(dev), rays_d.to(dev), zs.to(dev), bound)
    ref = f64.FieldFP64(params, x, level_scales, bound, device=dev)
    out = ref.backward(g_sigma.reshape(-1).to(dev), g_rgb.reshape(-1, 3).to(dev))
    B = x.shape[0]
    fw = ref.forward()
    res = {'sigma': (fw['sigma'], f64.RTOL_POINT * fw['sigma_abs']), 'rgb': (fw['rgb'], f64.RTOL_POINT * fw['rgb_abs'])}
    for k in ('encoder.embeddings', 'sigma_net.net.0.weight', 'sigma_net.net.0.bias', 'sigma_net.net.1.weight', 'sigma_net.net.1.bias',
              'sigma_net.net.2.weight', 'sigma_net.net.2.bias'):
        if k == 'encoder.embeddings':
            rtol = f64.RTOL_POINT + gamma(out[k + '_hits'] + 1)
        else:
            rtol = f64.wgrad_rtol(path, B, sm)
        res[k] = (out[k], rtol * out[k + '_abs'], out[k + '_slack'])
    return res


# ------------------------------------------------------------------------------------------------ end to end
def end_to_end_grad(params: Dict[str, torch.Tensor], rays_o, rays_d, zs, nears, fars, hw: int, loss_fn, level_scales, bound=4.0,
                    device=None) -> Dict[str, torch.Tensor]:
    """fp64 autograd of loss_fn(image [1,3,hw,hw], sil [1,1,hw,hw]) through the compositing (renderer_df.py:414-456) and the field
    (network_grid.py:36-88) at the merged depths zs [N,T]: every intermediate in fp64, none from the GPU run"""
    dev = device or zs.device
    zs, nears, fars = zs.to(dev).double(), nears.to(dev).double()[:, None], fars.to(dev).double()[:, None]
    x = f64.ray_points(rays_o.to(dev), rays_d.to(dev), zs.float(), bound)
    rows, w = f64.encode_geometry(x, f64.no.live_geometry(bound), level_scales, bound)
    p = {k: v.detach().to(dev).double().requires_grad_(True) for k, v in params.items()}
    B = x.shape[0]
    enc = (w[..., None] * p['encoder.embeddings'][rows]).sum(2).reshape(B, -1)
    h = torch.relu(F.linear(enc, p['sigma_net.net.0.weight'], p['sigma_net.net.0.bias']))
    h = torch.relu(F.linear(h, p['sigma_net.net.1.weight'], p['sigma_net.net.1.bias']))
    o = F.linear(h, p['sigma_net.net.2.weight'], p['sigma_net.net.2.bias'])
    pre = o[:, 0] + 5 * torch.exp(-(x.double() ** 2).sum(-1) / 0.08)
    sigma = (torch.exp(pre.detach().clamp(-15, 15)) * (pre - pre.detach()) + torch.exp(pre).detach()).view(zs.shape)   # trunc_exp
    rgb = torch.sigmoid(o[:, 1:]).view(*zs.shape, 3)
    deltas = torch.cat([zs[:, 1:] - zs[:, :-1], (fars - nears) / 64], 1)
    alphas = 1 - torch.exp(-deltas * sigma)
    weights = alphas * torch.cumprod(torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], 1), 1)[:, :-1]
    ws = weights.sum(1)
    image = (weights[..., None] * rgb).sum(1)                       # bg_color 0 (distillation.py's render_kw)
    img, sil = nchw(image, ws, hw)
    loss_fn(img, sil).backward()
    return {k: v.grad for k, v in p.items()}


# ------------------------------------------------------------------------------------------------ S4: Adam
def step_lr(cfg: StepConfig, sched: int):
    """[encoder lr, MLP lr] of torch.optim.Adam(net.get_params(lr)) + StepLR(step_size, gamma) after ``sched`` scheduler steps, read from a
    real fp64 torch optimiser and scheduler (the reference's objects, distillation.py:165-166)"""
    opt = torch.optim.Adam([{'params': [torch.zeros(1, dtype=torch.float64)], 'lr': cfg.lr * 10},
                            {'params': [torch.zeros(1, dtype=torch.float64)], 'lr': cfg.lr}], betas=cfg.betas, eps=cfg.eps)
    sch = torch.optim.lr_scheduler.StepLR(opt, cfg.step_size, cfg.gamma)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')              # scheduler steps without optimiser steps: only the lr is wanted here
        for _ in range(sched):
            sch.step()
    return [g['lr'] for g in opt.param_groups]


def adam_reference(flat0, grad, m0, v0, t: int, lrs, bounds_groups, cfg: StepConfig):
    """one fp64 torch.optim.Adam step from the GPU's pre-step state (parameters, moments, step t - 1) with the gradient ``grad`` (times
    grad_scale already), each group at its lr.  Returns (parameters after, abs companion, slack) in the bound form of
    tests/test_ngp_field_fp64_gpu.py::test_adam_step_vs_fp64_torch_adam: the parameter rounds once (gamma(3) on |p| + |update|), the
    update <= 34 times plus the fp32 bias corrections."""
    b1, b2 = (f32(b) for b in cfg.betas)
    out = torch.empty_like(flat0, dtype=torch.float64)
    for (s, e), lr in zip(bounds_groups, lrs):
        p = flat0[s:e].double().clone().requires_grad_(True)
        opt = torch.optim.Adam([p], lr=f32(lr), betas=(b1, b2), eps=f32(cfg.eps))
        if t > 1:
            opt.state[p] = {'step': torch.tensor(float(t - 1), dtype=torch.float64), 'exp_avg': m0[s:e].double().clone(),
                            'exp_avg_sq': v0[s:e].double().clone()}
        p.grad = grad[s:e].double()
        opt.step()
        out[s:e] = p.detach()
    d = (out - flat0.double()).abs()
    rel = gamma(34) + 0.5 * U32 / (1 - b2 ** t) + U32 / (1 - b1 ** t)
    return out, flat0.double().abs() + d, rel * d


# ------------------------------------------------------------------------------------------------ fp32 emulation (host self-checks)
def emulate_fusion(img, ws, hw, target, mode, cfg: StepConfig, weight, *, g_percep=None, view_scale=1.0, defect: Optional[str] = None):
    """S1 of the fused fusion path in fp32 (torch on the CPU): upsample, loss gradient, adjoint.  Defects: 'double' (the upstream
    gradient doubled), 'no_opacity_grad', 'no_entropy_grad', 'unscaled_view' (scale 1 in place of 1/V); the weight of another noise
    level and the perceptual gradient with respect to the target are injected by passing them as ``weight`` / ``g_percep``"""
    H = 2 * hw
    HW = H * H
    My, Mx = up2_taps(hw).float(), up2_taps(hw).float()
    planes = torch.cat((img.float().t().reshape(3, hw, hw), ws.float().reshape(1, hw, hw)))
    u = My @ planes @ Mx.t()
    t = target.float()
    lo = 0.0 if defect == 'no_opacity_grad' else f32(cfg.lambda_opacity)
    le = 0.0 if defect == 'no_entropy_grad' else f32(cfg.lambda_entropy)
    if mode == 'sds':
        g = torch.tensor(f32(weight)) * torch.sign(u[:3] - t) / (3 * HW)
        if g_percep is not None:
            g = g + f32(cfg.lambda_percep) * g_percep.float()
    else:
        d = u[:3] - t
        g = f32(cfg.lambda_color) * d / (HUBER_S * torch.sqrt(1 + d * d / (HUBER_S * HUBER_S))) / (3 * HW)
    sv = u[3]
    gs = lo * sv / (torch.sqrt(sv * sv + f32(0.01)) * HW)
    if mode == 'eft':
        dm = sv - fusion_mask(target).float().view(H, H)
        gs = gs + f32(cfg.lambda_sil) * dm / (HUBER_S * torch.sqrt(1 + dm * dm / (HUBER_S * HUBER_S))) / HW
    if le > 0:
        a = sv.clamp(ENT_LO, ENT_HI)
        inside = (sv >= ENT_LO) & (sv <= ENT_HI)
        gs = gs + torch.where(inside, le * torch.log2((1 - a) / a) / HW, torch.zeros_like(sv))
    g_up = torch.cat((g, gs[None]))
    y = My.t() @ g_up @ Mx
    gi, gw = y[:3].reshape(3, -1).t(), y[3].reshape(-1)
    if defect == 'double':
        gi, gw = 2 * gi, 2 * gw
    sc = 1.0 if defect == 'unscaled_view' else view_scale
    if sc != 1.0:
        gi, gw = gi * sc, gw * sc
    return gi, gw


def within(got, ref_bound) -> float:
    """the largest |got - y| / bound (inf where NaN)"""
    y, b = ref_bound
    r = (got.double().cpu() - y.cpu()).abs() / (b.cpu() + ATOL)
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def rel_l2(a, b) -> float:
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-300))


__all__ = ['StepConfig', 'sds_weight', 'entropy_grad', 'photometric_grad', 'upsample', 'adjoint', 'fusion_grad_up', 'fusion_grad',
           'reference_loss', 'nchw', 'composite_grad', 'field_grad', 'end_to_end_grad', 'step_lr', 'adam_reference', 'emulate_fusion',
           'within', 'rel_l2']
