"""Unet + GaussianDiffusionContinuousTimes -- host-side mirror of external/imagen_pytorch.py (reference).

``Unet`` keeps the reference's constructor keywords, parameter names / shapes (``state_dict()`` keys are
identical: 477 tensors for the SparseFusion config, utils/load_model.py:58-69), ``forward`` /
``forward_with_cond_scale`` / ``cast_model_parameters`` signatures and NCHW tensors at the boundary, so
``sparsefusion/vldm.py`` (DDPM), ``external/plms.py`` and ``utils/load_model.py`` use it unchanged.  The forward
itself never touches torch.nn: it is a sequence of sm_90a kernels from libsparsefusion_b200.so (wgmma
implicit-GEMM convolutions + fused norm/attention kernels, NHWC) launched on the current stream, and can be
captured into a CUDA graph (``UnetGraph``).  It is inference-only: SparseFusion's distillation loop runs the UNet
under no_grad (sparsefusion/distillation.py:302-304).

Supported configuration == what the SparseFusion pipeline instantiates (SURVEY.md Appendix A): cross-embed
init conv, pixel-shuffle upsampling, scaled skip connections, gca resnet blocks, final resnet block,
layer_cross_attns all False, memory_efficient False, no low-res / text conditioning in forward.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import ops

CROSS_DIM_HEAD, CROSS_HEADS = 64, 8  # mid blocks build CrossAttention with its own defaults (imagen_pytorch.py:737-738, :1336)


def exists(v):
    return v is not None


def default(v, d):
    return v if exists(v) else (d() if callable(d) else d)


def cast_tuple(val, length=None):
    if isinstance(val, list):
        val = tuple(val)
    out = val if isinstance(val, tuple) else ((val,) * default(length, 1))
    if exists(length):
        assert len(out) == length
    return out


# ---------------------------------------------------------------------------------------------------------
# continuous-time gaussian diffusion (imagen_pytorch.py:194-297): elementwise schedule math, stays in torch
# ---------------------------------------------------------------------------------------------------------
def alpha_cosine_log_snr(t, s: float = 0.008):
    return -torch.log(((torch.cos((t + s) / (1 + s) * math.pi * 0.5) ** -2) - 1).clamp(min=1e-5))


def beta_linear_log_snr(t):
    return -torch.log(torch.special.expm1(1e-4 + 10 * (t ** 2)))


def log_snr_to_alpha_sigma(log_snr):
    return torch.sqrt(torch.sigmoid(log_snr)), torch.sqrt(torch.sigmoid(-log_snr))


def right_pad_dims_to(x, t):
    pad = x.ndim - t.ndim
    return t if pad <= 0 else t.view(*t.shape, *((1,) * pad))


class GaussianDiffusionContinuousTimes(nn.Module):
    def __init__(self, *, noise_schedule, timesteps=1000):
        super().__init__()
        if noise_schedule == 'linear':
            self.log_snr = beta_linear_log_snr
        elif noise_schedule == 'cosine':
            self.log_snr = alpha_cosine_log_snr
        else:
            raise ValueError(f'invalid noise schedule {noise_schedule}')
        self.num_timesteps = timesteps

    def get_times(self, batch_size, noise_level, *, device):
        return torch.full((batch_size,), noise_level, device=device, dtype=torch.float32)

    def sample_random_times(self, batch_size, max_thres=0.999, *, device):
        return torch.zeros((batch_size,), device=device).float().uniform_(0, max_thres)

    def get_condition(self, times):
        return None if times is None else self.log_snr(times)

    def get_sampling_timesteps(self, batch, *, device):
        times = torch.linspace(1., 0., self.num_timesteps + 1, device=device)
        times = times[None, :].expand(batch, -1)
        return list(zip(times[:, :-1].unbind(dim=-1), times[:, 1:].unbind(dim=-1)))

    def get_sampling_timesteps_custom(self, batch, min_thres=0.0, max_thres=0.999, *, device, n_steps=5):
        times = torch.linspace(max_thres, min_thres, n_steps + 1, device=device)
        times = times[None, :].expand(batch, -1)
        return list(zip(times[:, :-1].unbind(dim=-1), times[:, 1:].unbind(dim=-1)))

    def q_posterior(self, x_start, x_t, t, *, t_next=None):
        t_next = default(t_next, lambda: (t - 1. / self.num_timesteps).clamp(min=0.))
        log_snr, log_snr_next = right_pad_dims_to(x_t, self.log_snr(t)), right_pad_dims_to(x_t, self.log_snr(t_next))
        alpha, sigma = log_snr_to_alpha_sigma(log_snr)
        alpha_next, sigma_next = log_snr_to_alpha_sigma(log_snr_next)
        c = -torch.special.expm1(log_snr - log_snr_next)
        posterior_mean = alpha_next * (x_t * (1 - c) / alpha + c * x_start)
        posterior_variance = (sigma_next ** 2) * c
        return posterior_mean, posterior_variance, torch.log(posterior_variance.clamp(min=1e-20))

    def q_sample(self, x_start, t, noise=None):
        if isinstance(t, float):
            t = torch.full((x_start.shape[0],), t, device=x_start.device, dtype=x_start.dtype)
        noise = default(noise, lambda: torch.randn_like(x_start))
        log_snr = self.log_snr(t)
        alpha, sigma = log_snr_to_alpha_sigma(right_pad_dims_to(x_start, log_snr))
        return alpha * x_start + sigma * noise, log_snr

    def predict_start_from_noise(self, x_t, t, noise):
        alpha, sigma = log_snr_to_alpha_sigma(right_pad_dims_to(x_t, self.log_snr(t)))
        return (x_t - sigma * noise) / alpha.clamp(min=1e-8)


# ---------------------------------------------------------------------------------------------------------
# parameter inventory: {reference state_dict key: shape}
# ---------------------------------------------------------------------------------------------------------
def unet_param_shapes(*, dim, dim_mults, num_resnet_blocks, layer_attns, channels, channels_out, cond_images_channels, cond_dim,
                      attn_dim_head, attn_heads, ff_mult, num_time_tokens, learned_sinu_pos_emb_dim, init_cross_embed_kernel_sizes,
                      max_conditional_len, cond_on_z, conditional_embed_dim) -> Dict[str, Tuple[int, ...]]:
    s: Dict[str, Tuple[int, ...]] = {}
    td = dim * 4
    inner, dh = attn_dim_head * attn_heads, attn_dim_head
    cin = channels + cond_images_channels
    ks = sorted(init_cross_embed_kernel_sizes)
    scales = [int(dim / (2 ** i)) for i in range(1, len(ks))]
    scales = [*scales, dim - sum(scales)]
    s['null_conditional_embed'] = (1, max_conditional_len, cond_dim)
    s['null_conditional_hidden'] = (1, td)
    for i, (k, d) in enumerate(zip(ks, scales)):
        s[f'init_conv.convs.{i}.weight'], s[f'init_conv.convs.{i}.bias'] = (d, cin, k, k), (d,)
    s['to_time_hiddens.0.weights'] = (learned_sinu_pos_emb_dim // 2,)
    s['to_time_hiddens.1.weight'], s['to_time_hiddens.1.bias'] = (td, learned_sinu_pos_emb_dim + 1), (td,)
    s['to_time_cond.0.weight'], s['to_time_cond.0.bias'] = (td, td), (td,)
    s['to_time_tokens.0.weight'], s['to_time_tokens.0.bias'] = (cond_dim * num_time_tokens, td), (cond_dim * num_time_tokens,)
    s['norm_cond.weight'], s['norm_cond.bias'] = (cond_dim,), (cond_dim,)
    if cond_on_z:  # present in the state_dict of a text-conditioned Unet; never used by this forward
        s['conditional_to_cond.weight'], s['conditional_to_cond.bias'] = (cond_dim, conditional_embed_dim), (cond_dim,)
        s['to_conditional_non_attn_cond.0.weight'], s['to_conditional_non_attn_cond.0.bias'] = (cond_dim,), (cond_dim,)
        s['to_conditional_non_attn_cond.1.weight'], s['to_conditional_non_attn_cond.1.bias'] = (td, cond_dim), (td,)
        s['to_conditional_non_attn_cond.3.weight'], s['to_conditional_non_attn_cond.3.bias'] = (td, td), (td,)

    def resnet(p, din, dout, gca, cross):
        s[f'{p}.time_mlp.1.weight'], s[f'{p}.time_mlp.1.bias'] = (dout * 2, td), (dout * 2,)
        if cross:
            ci = CROSS_DIM_HEAD * CROSS_HEADS
            s[f'{p}.cross_attn.fn.null_kv'] = (2, CROSS_DIM_HEAD)
            s[f'{p}.cross_attn.fn.norm.g'] = (dout,)
            s[f'{p}.cross_attn.fn.to_q.weight'] = (ci, dout)
            s[f'{p}.cross_attn.fn.to_kv.weight'] = (ci * 2, cond_dim)
            s[f'{p}.cross_attn.fn.to_out.0.weight'] = (dout, ci)
            s[f'{p}.cross_attn.fn.to_out.1.g'] = (dout,)
        for b, (i, o) in (('block1', (din, dout)), ('block2', (dout, dout))):
            s[f'{p}.{b}.groupnorm.weight'], s[f'{p}.{b}.groupnorm.bias'] = (i,), (i,)
            s[f'{p}.{b}.project.weight'], s[f'{p}.{b}.project.bias'] = (o, i, 3, 3), (o,)
        if gca:
            hid = max(3, dout // 2)
            s[f'{p}.gca.to_k.weight'], s[f'{p}.gca.to_k.bias'] = (1, dout, 1, 1), (1,)
            s[f'{p}.gca.net.0.weight'], s[f'{p}.gca.net.0.bias'] = (hid, dout, 1, 1), (hid,)
            s[f'{p}.gca.net.2.weight'], s[f'{p}.gca.net.2.bias'] = (dout, hid, 1, 1), (dout,)
        if din != dout:
            s[f'{p}.res_conv.weight'], s[f'{p}.res_conv.bias'] = (dout, din, 1, 1), (dout,)

    def attention(p, d, context):
        s[f'{p}.null_kv'], s[f'{p}.norm.g'] = (2, dh), (d,)
        s[f'{p}.to_q.weight'], s[f'{p}.to_kv.weight'] = (inner, d), (dh * 2, d)
        if context:
            s[f'{p}.to_context.0.weight'], s[f'{p}.to_context.0.bias'] = (cond_dim,), (cond_dim,)
            s[f'{p}.to_context.1.weight'], s[f'{p}.to_context.1.bias'] = (dh * 2, cond_dim), (dh * 2,)
        s[f'{p}.to_out.0.weight'], s[f'{p}.to_out.1.g'] = (d, inner), (d,)

    def transformer(p, d):
        attention(f'{p}.layers.0.0.fn', d, True)
        hid = int(d * ff_mult)
        s[f'{p}.layers.0.1.0.g'], s[f'{p}.layers.0.1.1.weight'] = (1, d, 1, 1), (hid, d, 1, 1)
        s[f'{p}.layers.0.1.3.g'], s[f'{p}.layers.0.1.4.weight'] = (1, hid, 1, 1), (d, hid, 1, 1)

    dims = [dim, *[dim * m for m in dim_mults]]
    in_out = list(zip(dims[:-1], dims[1:]))
    n = len(in_out)
    for i, (din, dout) in enumerate(in_out):
        resnet(f'downs.{i}.1', din, din, False, False)
        for j in range(num_resnet_blocks[i]):
            resnet(f'downs.{i}.2.{j}', din, din, True, False)
        if layer_attns[i]:
            transformer(f'downs.{i}.3', din)
        if i < n - 1:
            s[f'downs.{i}.4.weight'], s[f'downs.{i}.4.bias'] = (dout, din, 4, 4), (dout,)
        else:
            s[f'downs.{i}.4.fns.0.weight'], s[f'downs.{i}.4.fns.0.bias'] = (dout, din, 3, 3), (dout,)
            s[f'downs.{i}.4.fns.1.weight'], s[f'downs.{i}.4.fns.1.bias'] = (dout, din, 1, 1), (dout,)
    mid = dims[-1]
    resnet('mid_block1', mid, mid, False, True)
    attention('mid_attn.fn.fn', mid, False)
    resnet('mid_block2', mid, mid, False, True)
    for i, (din, dout) in enumerate(reversed(in_out)):
        ri = n - 1 - i
        resnet(f'ups.{i}.0', dout + din, dout, False, False)
        for j in range(num_resnet_blocks[ri]):
            resnet(f'ups.{i}.1.{j}', dout + din, dout, True, False)
        if layer_attns[ri]:
            transformer(f'ups.{i}.2', dout)
        if i < n - 1:
            s[f'ups.{i}.3.net.0.weight'], s[f'ups.{i}.3.net.0.bias'] = (din * 4, dout, 1, 1), (din * 4,)
    resnet('final_res_block', dim, dim, True, False)
    s['final_conv.weight'], s['final_conv.bias'] = (channels_out, dim, 3, 3), (channels_out,)
    return s


class _Node(nn.Module):
    """bare container: gives parameters the reference's dotted state_dict names"""


def _register(root: nn.Module, dotted: str, p: nn.Parameter) -> None:
    parts = dotted.split('.')
    m = root
    for part in parts[:-1]:
        if part not in m._modules:
            m.add_module(part, _Node())
        m = m._modules[part]
    m.register_parameter(parts[-1], p)


class Unet(nn.Module):
    def __init__(self, *, dim, image_embed_dim=1024, conditional_embed_dim=1024, num_resnet_blocks=1, cond_dim=None, num_image_tokens=4,
                 num_time_tokens=2, learned_sinu_pos_emb_dim=16, out_dim=None, dim_mults=(1, 2, 4, 8), cond_images_channels=0, channels=3,
                 channels_out=None, attn_dim_head=64, attn_heads=8, ff_mult=2., lowres_cond=False, layer_attns=True, layer_attns_depth=1,
                 layer_attns_add_conditional_cond=True, attend_at_middle=True, layer_cross_attns=True, use_linear_attn=False,
                 use_linear_cross_attn=False, cond_on_z=True, max_conditional_len=256, init_dim=None, resnet_groups=8,
                 init_conv_kernel_size=7, init_cross_embed=True, init_cross_embed_kernel_sizes=(3, 7, 15), cross_embed_downsample=False,
                 cross_embed_downsample_kernel_sizes=(2, 4), attn_pool_text=True, attn_pool_num_latents=32, dropout=0.,
                 memory_efficient=False, init_conv_to_final_conv_residual=False, use_global_conconditional_attn=True,
                 scale_skip_connection=True, final_resnet_block=True, final_conv_kernel_size=3, cosine_sim_attn=False,
                 combine_upsample_fmaps=False, pixel_shuffle_upsample=True):
        super().__init__()
        self._locals = {k: v for k, v in locals().items() if k not in ('self', '__class__')}
        n = len(dim_mults)
        num_resnet_blocks, layer_attns = cast_tuple(num_resnet_blocks, n), cast_tuple(layer_attns, n)
        layer_cross_attns = cast_tuple(layer_cross_attns, n)
        unsupported = []
        if any(layer_cross_attns): unsupported.append('layer_cross_attns')
        if memory_efficient: unsupported.append('memory_efficient')
        if not init_cross_embed: unsupported.append('init_cross_embed=False')
        if cross_embed_downsample: unsupported.append('cross_embed_downsample')
        if not pixel_shuffle_upsample: unsupported.append('pixel_shuffle_upsample=False')
        if use_linear_attn or use_linear_cross_attn: unsupported.append('linear attention')
        if init_conv_to_final_conv_residual or combine_upsample_fmaps: unsupported.append('final residual / fmap combiner')
        if not (use_global_conconditional_attn and scale_skip_connection and final_resnet_block and attend_at_middle): unsupported.append('block switches')
        if cosine_sim_attn or lowres_cond or attn_pool_text or cast_tuple(layer_attns_depth, n) != (1,) * n or final_conv_kernel_size != 3:
            unsupported.append('cosine_sim_attn / lowres_cond / attn_pool_text / attention depth / final kernel size')
        if init_dim is not None and init_dim != dim: unsupported.append('init_dim')
        if cast_tuple(resnet_groups, n) != (cast_tuple(resnet_groups, n)[0],) * n: unsupported.append('per-stage resnet_groups')
        if unsupported:
            raise NotImplementedError('sparsefusion_b200.Unet implements the SparseFusion VLDM configuration only '
                                      f'(utils/load_model.py:58-69); unsupported: {unsupported}')
        self.channels, self.channels_out = channels, default(channels_out, channels)
        self.lowres_cond, self.cond_on_z = lowres_cond, cond_on_z
        self.has_cond_image, self.cond_images_channels = cond_images_channels > 0, cond_images_channels
        self.dim, self.dim_mults, self.num_resnet_blocks, self.layer_attns = dim, tuple(dim_mults), num_resnet_blocks, layer_attns
        self.cond_dim = default(cond_dim, dim)
        self.time_cond_dim = dim * 4
        self.groups = cast_tuple(resnet_groups, n)[0]
        self.attn_heads, self.attn_dim_head, self.num_time_tokens = attn_heads, attn_dim_head, num_time_tokens
        self.kernel_sizes = tuple(sorted(init_cross_embed_kernel_sizes))
        self.skip_connect_scale = 2 ** -0.5
        self.max_conditional_len = max_conditional_len

        shapes = unet_param_shapes(dim=dim, dim_mults=self.dim_mults, num_resnet_blocks=num_resnet_blocks, layer_attns=layer_attns,
                                   channels=channels, channels_out=self.channels_out, cond_images_channels=cond_images_channels,
                                   cond_dim=self.cond_dim, attn_dim_head=attn_dim_head, attn_heads=attn_heads, ff_mult=ff_mult,
                                   num_time_tokens=num_time_tokens, learned_sinu_pos_emb_dim=learned_sinu_pos_emb_dim,
                                   init_cross_embed_kernel_sizes=self.kernel_sizes, max_conditional_len=max_conditional_len,
                                   cond_on_z=cond_on_z, conditional_embed_dim=conditional_embed_dim)
        self._shapes = shapes
        for name, shape in shapes.items():
            _register(self, name, nn.Parameter(torch.empty(shape)))
        self.reset_parameters()
        self._plan = None  # packed weights etc., rebuilt lazily
        self.use_arena = True      # split-K conv outputs from one zero-filled buffer per evaluation (ops.ZeroArena)
        self._arena_floats = {}    # (nb, h, w) -> floats, measured on the first evaluation of that shape
        self.parallel_res_conv = True   # res_conv on a side stream = a parallel branch of the captured graph (see _resnet)
        self._side = {}

    # ------------------------------------------------------------------------------------------ parameters
    @torch.no_grad()
    def reset_parameters(self):
        """PyTorch-default-like init; final_conv zero as in the reference (imagen_pytorch.py:1388)"""
        for name, p in self.named_parameters():
            leaf = name.rsplit('.', 1)[-1]
            if leaf == 'g' or (leaf == 'weight' and p.dim() == 1):
                p.fill_(1.0)
            elif leaf in ('null_kv', 'weights') or name.startswith('null_conditional'):
                p.normal_()
            elif leaf == 'bias':
                if p.dim() == 1 and (name.endswith('groupnorm.bias') or name in ('norm_cond.bias',) or name.endswith('to_context.0.bias')
                                     or name.endswith('to_conditional_non_attn_cond.0.bias')):
                    p.zero_()
                else:
                    w = self._shapes[name[:-4] + 'weight']
                    bound = 1.0 / math.sqrt(max(1, int(torch.tensor(w[1:]).prod())))
                    p.uniform_(-bound, bound)
            else:
                bound = 1.0 / math.sqrt(max(1, int(torch.tensor(p.shape[1:]).prod())))
                p.uniform_(-bound, bound)
        self.get_parameter('final_conv.weight').zero_()
        self.get_parameter('final_conv.bias').zero_()
        for name, p in self.named_parameters():  # PixelShuffleUpsample.init_conv_ (:596-603): 4 identical sub-filters, zero bias
            if name.endswith('.3.net.0.weight'):
                o = p.shape[0] // 4
                p.copy_(p[:o].repeat_interleave(4, dim=0))
            if name.endswith('.3.net.0.bias'):
                p.zero_()
        self._plan = None

    def _apply(self, fn, *a, **k):
        self._plan = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._plan = None
        return super().load_state_dict(*a, **k)

    def cast_model_parameters(self, *, lowres_cond, conditional_embed_dim, channels, channels_out, cond_on_z):
        """imagen_pytorch.py:1392-1416: re-instantiate when DDPM asks for a different conditioning set-up"""
        if (lowres_cond == self.lowres_cond and channels == self.channels and cond_on_z == self.cond_on_z
                and conditional_embed_dim == self._locals['conditional_embed_dim'] and channels_out == self.channels_out):
            return self
        upd = dict(lowres_cond=lowres_cond, conditional_embed_dim=conditional_embed_dim, channels=channels, channels_out=channels_out,
                   cond_on_z=cond_on_z)
        return self.__class__(**{**self._locals, **upd})

    def to_config_and_state_dict(self):
        return self._locals, self.state_dict()

    @classmethod
    def from_config_and_state_dict(klass, config, state_dict):
        unet = klass(**config)
        unet.load_state_dict(state_dict)
        return unet

    # ------------------------------------------------------------------------------------------ plan
    @torch.no_grad()
    def prepare(self):
        """pack every tensor-core weight ([Cout][tap][Cin_pad], TF32-rounded) and fuse the 27 time MLPs into one GEMV"""
        P = {n: p.detach() for n, p in self.named_parameters()}
        dev = next(iter(P.values())).device
        if dev.type != 'cuda':
            raise RuntimeError('sparsefusion_b200.Unet runs on CUDA only (there is no CPU fallback); call .cuda() first')
        packed = {}
        for n, p in P.items():
            if n.endswith('.weight') and p.dim() == 4 and 'gca.' not in n:
                packed[n] = ops.pack_conv_weight(p)
            elif n.endswith(('to_q.weight', 'to_kv.weight', 'to_out.0.weight')):
                packed[n] = ops.pack_conv_weight(p)
        if self.has_cond_image:
            # CrossEmbedLayer input = cat(cond_images, x): conv(W, cat) = conv(W[:, :Cc], cond) + conv(W[:, Cc:], x).  The first term does not change
            # during a PLMS sampling run (33 evaluations per distillation step share one cond_images): precompute_cond() evaluates it once.
            cc = self.cond_images_channels
            for i in range(len(self.kernel_sizes)):
                w = P[f'init_conv.convs.{i}.weight']
                packed[f'init_conv.convs.{i}.weight@cond'] = ops.pack_conv_weight(w[:, :cc].contiguous())
                packed[f'init_conv.convs.{i}.weight@x'] = ops.pack_conv_weight(w[:, cc:].contiguous())
            # the x share: few channels (4 latents).  As implicit GEMMs the three kernel sizes would each pad those channels to 32 per tap (8x the
            # work: 16 % of a batch-16 evaluation's convolution time); unfolded by ops.im2col4 they are ONE 1x1 convolution over 4 kmax^2 columns whose
            # weight rows are the three filters, centred in the largest window
            if self.channels == 4:
                km = max(self.kernel_sizes)
                wm = torch.zeros(self.dim, km, km, 4, dtype=torch.float32, device=dev)
                o = 0
                for i, k in enumerate(self.kernel_sizes):
                    w = P[f'init_conv.convs.{i}.weight'][:, cc:]                      # [co, 4, k, k]
                    off = (km - k) // 2
                    wm[o:o + w.shape[0], off:off + k, off:off + k, :] = w.permute(0, 2, 3, 1)
                    o += w.shape[0]
                packed['init_conv.merged@x'] = ops.pack_conv_weight(wm.reshape(self.dim, km * km * 4))
        # last down stage: Parallel(conv3x3, conv1x1) summed (:1322) == ONE 3x3 convolution whose centre tap carries the 1x1 weights too
        for n in list(P):
            if n.endswith('.4.fns.0.weight') and n.replace('fns.0', 'fns.1') in P:
                w3, w1 = P[n], P[n.replace('fns.0', 'fns.1')]
                if w3.shape[2:] == (3, 3) and w1.shape[2:] == (1, 1):
                    wm = w3.clone()
                    wm[:, :, 1, 1] += w1[:, :, 0, 0]
                    base = n[:-len('.fns.0.weight')]
                    packed[base + '.merged.weight'] = ops.pack_conv_weight(wm)
                    P[base + '.merged.bias'] = (P[n[:-len('weight')] + 'bias'] + P[n.replace('fns.0', 'fns.1')[:-len('weight')] + 'bias']).contiguous()
        film_names = [n[:-len('.time_mlp.1.weight')] for n in P if n.endswith('.time_mlp.1.weight')]
        film_w = torch.cat([P[f'{b}.time_mlp.1.weight'] for b in film_names], dim=0).contiguous()
        film_b = torch.cat([P[f'{b}.time_mlp.1.bias'] for b in film_names], dim=0).contiguous()
        film_off, o = {}, 0
        for b in film_names:
            film_off[b] = (o, P[f'{b}.time_mlp.1.weight'].shape[0])
            o += P[f'{b}.time_mlp.1.weight'].shape[0]
        self._plan = dict(P=P, packed=packed, split={}, film_w=film_w, film_b=film_b, film_off=film_off)
        return self

    # ------------------------------------------------------------------------------------------ forward pieces (NHWC)
    def _split(self, key, x_pixels):
        """pre-split (hi, lo) copy of a packed weight for launches that run the tensor-bound (non swap-AB) kernel: more than 64 output pixels in
        3xTF32 mode.  Made on first use; the weight-streaming layers of a batch-1 evaluation never get one."""
        pl = self._plan
        if x_pixels <= 64 or ops.get_precision() != 'tf32x3':
            return None
        sp = pl['split'].get(key)
        if sp is None:
            sp = pl['split'][key] = ops.split_packed_weight(pl['packed'][key])
        return sp

    def _conv(self, name, x, k, stride=1, pad=0, residual=None, out=None, accumulate=False):
        pl = self._plan
        w = pl['packed'][name + '.weight']
        npix = x.shape[0] * (x.shape[1] // stride) * (x.shape[2] // stride)
        return ops.conv2d_nhwc(x, w, w.shape[0], k, k, stride, pad, bias=pl['P'].get(name + '.bias'), residual=residual, out=out,
                               accumulate=accumulate, w_split=self._split(name + '.weight', npix))

    def _linear_rows(self, name, x, bias=True, round_out=False):
        """token projection [.., K] -> [.., O]: fp32 GEMV for a handful of rows, tensor cores (swap-AB tile: the rows are the N side) from 16 rows up --
        in the replayed graph the 8-row GEMV tile costs 13.8 us per projection of the 4x4 stage's 16 tokens, the wgmma path ~5 us"""
        pl = self._plan
        w = pl['P'][name + '.weight']
        b = pl['P'].get(name + '.bias') if bias else None
        rows = x.numel() // x.shape[-1]
        if rows < 16 or (name + '.weight') not in pl['packed']:
            return ops.linear_small(x, w.reshape(w.shape[0], -1), b, round_to_tf32=round_out)
        return ops.linear_tc(x, pl['packed'][name + '.weight'], w.shape[0], bias=b, w_split=self._split(name + '.weight', rows))

    def _side_stream(self, device):
        key = torch.device(device).index
        if key not in self._side:
            self._side[key] = torch.cuda.Stream(device=device)
        return self._side[key]

    def _resnet(self, pfx, x, film_all, c_tokens, taps=None):
        pl = self._plan
        P = pl['P']
        off, width = pl['film_off'][pfx]
        film = film_all[:, off:off + width]
        g = self.groups
        # res_conv(x) only depends on the block input and is consumed at the very end of the block: issue it on a side stream, so that in the
        # captured graph it is a parallel branch running in the shadow of the GroupNorm launches instead of one more link of the dependent chain
        join = None
        if f'{pfx}.res_conv.weight' in P:
            if self.parallel_res_conv:
                main = torch.cuda.current_stream()
                side = self._side_stream(x.device)
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    res = self._conv(f'{pfx}.res_conv', x, 1)
                res.record_stream(main)
                join = side
            else:
                res = self._conv(f'{pfx}.res_conv', x, 1)
        else:
            res = x
        a1 = ops.groupnorm(x, g, P[f'{pfx}.block1.groupnorm.weight'], P[f'{pfx}.block1.groupnorm.bias'], None, True)
        h = self._conv(f'{pfx}.block1.project', a1, 3, 1, 1)
        if f'{pfx}.cross_attn.fn.null_kv' in P:
            h = self._cross_attn(f'{pfx}.cross_attn.fn', h, c_tokens)
        a2 = ops.groupnorm(h, g, P[f'{pfx}.block2.groupnorm.weight'], P[f'{pfx}.block2.groupnorm.bias'], film, True)
        if f'{pfx}.gca.to_k.weight' in P:
            h2 = self._conv(f'{pfx}.block2.project', a2, 3, 1, 1)
            pooled = ops.gca_pool(h2, P[f'{pfx}.gca.to_k.weight'], P[f'{pfx}.gca.to_k.bias'])
            w0, w2 = P[f'{pfx}.gca.net.0.weight'], P[f'{pfx}.gca.net.2.weight']
            hid = ops.linear_small(pooled, w0.reshape(w0.shape[0], -1), P[f'{pfx}.gca.net.0.bias'], post=1)
            if join is not None:
                torch.cuda.current_stream().wait_stream(join)
            # (GlobalContext + gate + residual as ONE thread-block-cluster kernel was built and measured: 21 us per block against 16.9 us for these four
            #  launches -- five dependent global / DSMEM round trips do not shrink by sharing a launch -- and taken out again)
            out = ops.gate_mlp_residual(h2, hid, w2.reshape(w2.shape[0], -1), P[f'{pfx}.gca.net.2.bias'], res)   # gate GEMV + sigmoid + h*gate + res
        else:
            if join is not None:
                torch.cuda.current_stream().wait_stream(join)
            out = self._conv(f'{pfx}.block2.project', a2, 3, 1, 1, residual=res)
        if taps is not None:
            taps[pfx] = out
        return out

    def _cross_attn(self, pfx, h, c_tokens):
        """CrossAttention(h tokens, context c) + h   (imagen_pytorch.py:721-723, :764-805)"""
        P = self._plan['P']
        nb, hh, ww, c = h.shape
        rows = h.view(nb, hh * ww, c)
        xn = ops.layernorm(rows, P[f'{pfx}.norm.g'], None, round_to_tf32=True)
        q = self._linear_rows(f'{pfx}.to_q', xn, bias=False)
        kvc = self._linear_rows(f'{pfx}.to_kv', c_tokens, bias=False)
        o = ops.cross_attention(q, kvc, P[f'{pfx}.null_kv'], CROSS_HEADS, CROSS_DIM_HEAD)
        y = self._linear_rows(f'{pfx}.to_out.0', o, bias=False)
        out = ops.layernorm(y, P[f'{pfx}.to_out.1.g'], None, round_to_tf32=False, residual=rows)
        return out.view(nb, hh, ww, c)

    def _self_attn(self, pfx, x, c_tokens):
        """Attention(x tokens, optional context) + x   (imagen_pytorch.py:511-566 inside Residual / TransformerBlock)"""
        P = self._plan['P']
        nb, hh, ww, c = x.shape
        rows = x.view(nb, hh * ww, c)
        xn = ops.layernorm(rows, P[f'{pfx}.norm.g'], None, round_to_tf32=True)
        q = self._linear_rows(f'{pfx}.to_q', xn, bias=False)
        kv = self._linear_rows(f'{pfx}.to_kv', xn, bias=False)
        ckv = None
        if c_tokens is not None and f'{pfx}.to_context.1.weight' in P:
            cn = ops.layernorm(c_tokens, P[f'{pfx}.to_context.0.weight'], P[f'{pfx}.to_context.0.bias'], round_to_tf32=False)
            ckv = ops.linear_small(cn, P[f'{pfx}.to_context.1.weight'], P[f'{pfx}.to_context.1.bias'])
        o = ops.mq_attention(q, kv, P[f'{pfx}.null_kv'], ckv, self.attn_heads, self.attn_dim_head)
        y = self._linear_rows(f'{pfx}.to_out.0', o, bias=False)
        out = ops.layernorm(y, P[f'{pfx}.to_out.1.g'], None, round_to_tf32=False, residual=rows)
        return out.view(nb, hh, ww, c)

    def _transformer(self, pfx, x, c_tokens):
        P = self._plan['P']
        x = self._self_attn(f'{pfx}.layers.0.0.fn', x, c_tokens)
        nb, hh, ww, c = x.shape
        f = ops.layernorm(x.view(nb * hh * ww, c), P[f'{pfx}.layers.0.1.0.g'], None, round_to_tf32=True).view(nb, hh, ww, c)
        f = self._conv(f'{pfx}.layers.0.1.1', f, 1)
        hid = f.shape[-1]
        f = ops.layernorm(f.view(nb * hh * ww, hid), P[f'{pfx}.layers.0.1.3.g'], None, pre_gelu=True, round_to_tf32=True).view(nb, hh, ww, hid)
        return self._conv(f'{pfx}.layers.0.1.4', f, 1, residual=x)

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def precompute_cond(self, cond_images: torch.Tensor) -> torch.Tensor:
        """the cond_images share of init_conv (NHWC [nb, h, w, dim], biases included): pass it to forward(cond_features=...) for every evaluation
        that uses the same cond_images -- a PLMS run evaluates the UNet ~33 times on one conditioning map (external/plms.py:96-119), and the
        15x15 / 7x7 / 3x3 CrossEmbed convolutions over its 256 channels are 5% of an evaluation."""
        assert self.has_cond_image and cond_images.shape[1] == self.cond_images_channels
        if self._plan is None:
            self.prepare()
        pl = self._plan
        nb, _, hh, ww = cond_images.shape
        dev = cond_images.device
        with torch.cuda.device(dev):
            cn = torch.empty(nb, hh, ww, self.cond_images_channels, dtype=torch.float32, device=dev)
            ops.nchw_to_nhwc(cond_images.float(), cn, 0, True)
            h0 = torch.empty(nb, hh, ww, self.dim, dtype=torch.float32, device=dev)
            o = 0
            for i, k in enumerate(self.kernel_sizes):
                w = pl['packed'][f'init_conv.convs.{i}.weight@cond']
                ops.conv2d_nhwc(cn, w, w.shape[0], k, k, 1, (k - 1) // 2, bias=pl['P'].get(f'init_conv.convs.{i}.bias'), out=h0[..., o:o + w.shape[0]],
                                w_split=self._split(f'init_conv.convs.{i}.weight@cond', nb * hh * ww))
                o += w.shape[0]
        return h0

    @torch.no_grad()
    def precompute_time(self, time: torch.Tensor) -> dict:
        """everything of an evaluation that depends on the noise level only (imagen_pytorch.py:1517-1522, :1600-1604 and every block's time MLP,
        :698-704): rows of ``t`` [T, time_cond_dim], ``c`` [T, tokens, cond_dim] and ``film`` [T, sum 2*dim_out] for T log-SNR values.  A PLMS run knows
        its n+1 noise levels up front: evaluating them in one batch reads the 143 MB of time-MLP weights once per run instead of once per UNet
        evaluation, and takes six launches (66 us) off the critical path of every evaluation.  Pass row i as ``forward(time_features=...)``."""
        if self._plan is None:
            self.prepare()
        pl = self._plan
        P = pl['P']
        time = time.float().contiguous()
        rows = time.shape[0]
        with torch.cuda.device(time.device):
            four = ops.time_fourier(time, P['to_time_hiddens.0.weights'])
            th = ops.linear_small(four, P['to_time_hiddens.1.weight'], P['to_time_hiddens.1.bias'], post=1)
            tokens = ops.linear_small(th, P['to_time_tokens.0.weight'], P['to_time_tokens.0.bias']).view(rows, self.num_time_tokens, self.cond_dim)
            t = ops.linear_small(th, P['to_time_cond.0.weight'], P['to_time_cond.0.bias'])
            c = ops.layernorm(tokens, P['norm_cond.weight'], P['norm_cond.bias'], round_to_tf32=False)
            if rows >= 16:      # many noise levels at once: one pass over the fused time-MLP weights on the tensor cores (swap-AB tile)
                if 'film_w' not in pl['packed']:
                    pl['packed']['film_w'] = ops.pack_conv_weight(pl['film_w'])
                film_all = ops.linear_tc(torch.nn.functional.silu(t), pl['packed']['film_w'], pl['film_w'].shape[0], bias=pl['film_b'],
                                         w_split=self._split('film_w', rows))
            else:
                film_all = ops.linear_small(t, pl['film_w'], pl['film_b'], pre=1)  # every block's SiLU->Linear time MLP at once
        return dict(t=t, c=c, film=film_all)

    def forward_with_cond_scale(self, *args, cond_scale=1., **kwargs):
        logits = self.forward(*args, **kwargs)
        if cond_scale == 1:
            return logits
        null_logits = self.forward(*args, cond_drop_prob=1., **kwargs)
        return null_logits + (logits - null_logits) * cond_scale

    @torch.no_grad()
    def forward(self, x, time, *, lowres_cond_img=None, lowres_noise_times=None, conditional_embeds=None, conditional_mask=None,
                cond_images=None, cond_drop_prob=0., taps: Optional[dict] = None, cond_features: Optional[torch.Tensor] = None,
                time_features: Optional[dict] = None):
        if exists(lowres_cond_img) or exists(conditional_embeds):
            raise NotImplementedError('sparsefusion_b200.Unet: low-res / text conditioning are not part of the SparseFusion VLDM path')
        assert not (self.has_cond_image ^ (exists(cond_images) or exists(cond_features))), 'cond_images must be given iff the unet was built with cond_images_channels'
        if self._plan is None:
            self.prepare()
        P = self._plan['P']
        nb, _, hh, ww = x.shape
        dev = x.device
        # split-K destinations: one zero-filled arena per evaluation (ops.ZeroArena); the first evaluation of a shape only measures it
        need = self._arena_floats.get((nb, hh, ww)) if self.use_arena else None
        arena = ops.ArenaMeter() if (need is None and self.use_arena) else (ops.ZeroArena(need, dev) if need is not None else None)
        with torch.cuda.device(dev), ops.use_arena(arena):
            y = self._forward_nhwc(x, time, cond_images, cond_drop_prob, taps, P, nb, hh, ww, dev, cond_features, time_features)
        if isinstance(arena, ops.ArenaMeter):
            self._arena_floats[(nb, hh, ww)] = arena.floats
        return y

    def _forward_nhwc(self, x, time, cond_images, cond_drop_prob, taps, P, nb, hh, ww, dev, cond_features=None, time_features=None):
        pl = self._plan
        if cond_features is not None:
            # init_conv = cached conv(W[:, :Cc], cond_images) (+ bias) + conv(W[:, Cc:], x): only the 4-channel term is evaluated here
            assert cond_drop_prob == 0. and tuple(cond_features.shape) == (nb, hh, ww, self.dim)
            x4 = torch.empty(nb, hh, ww, self.channels, dtype=torch.float32, device=dev)
            ops.nchw_to_nhwc(x.float(), x4, 0, True)
            h0 = cond_features.clone()
            if 'init_conv.merged@x' in pl['packed']:
                km = max(self.kernel_sizes)
                w = pl['packed']['init_conv.merged@x']
                ops.conv2d_nhwc(ops.im2col4(x4, km, km, (km - 1) // 2), w, w.shape[0], 1, 1, 1, 0, out=h0, accumulate=True,
                                w_split=self._split('init_conv.merged@x', nb * hh * ww))
            else:
                o = 0
                for i, k in enumerate(self.kernel_sizes):
                    w = pl['packed'][f'init_conv.convs.{i}.weight@x']
                    ops.conv2d_nhwc(x4, w, w.shape[0], k, k, 1, (k - 1) // 2, out=h0[..., o:o + w.shape[0]], accumulate=True,
                                    w_split=self._split(f'init_conv.convs.{i}.weight@x', nb * hh * ww))
                    o += w.shape[0]
        else:
            # cat(cond_images * keep_mask, x) -> NHWC (imagen_pytorch.py:1496-1504); prob 0 keeps, prob 1 drops everything
            cin = self.channels + self.cond_images_channels
            xin = torch.zeros(nb, hh, ww, cin, dtype=torch.float32, device=dev)
            if exists(cond_images):
                assert cond_images.shape[1] == self.cond_images_channels
                if cond_images.shape[-1] != ww:
                    cond_images = torch.nn.functional.interpolate(cond_images, ww, mode='nearest')
                if cond_drop_prob == 0.:
                    ops.nchw_to_nhwc(cond_images.float(), xin, 0, True)
                elif cond_drop_prob != 1.:
                    keep = (torch.zeros((nb,), device=dev).float().uniform_(0, 1) < (1 - cond_drop_prob)).view(nb, 1, 1, 1)
                    ops.nchw_to_nhwc(cond_images.float() * keep, xin, 0, True)
            ops.nchw_to_nhwc(x.float(), xin, self.cond_images_channels, True)
            # CrossEmbedLayer: three convolutions write adjacent channel slices (:1040-1042)
            h0 = torch.empty(nb, hh, ww, self.dim, dtype=torch.float32, device=dev)
            o = 0
            for i, k in enumerate(self.kernel_sizes):
                co = P[f'init_conv.convs.{i}.weight'].shape[0]
                self._conv(f'init_conv.convs.{i}', xin, k, 1, (k - 1) // 2, out=h0[..., o:o + co])
                o += co
        xcur = h0
        if taps is not None:
            taps['init_conv'] = xcur
        # time conditioning (:1517-1522, :1600-1604): depends on `time` only -- evaluated here, or ahead of time for a whole sampling run
        if time_features is None:
            time_features = self.precompute_time(time)
        t, c, film_all = time_features['t'], time_features['c'], time_features['film']
        assert film_all.shape[0] == nb and c.shape[0] == nb, 'time_features rows must match the batch'
        if taps is not None:
            taps['t'], taps['c'] = t, c

        n = len(self.dim_mults)
        hiddens: List[torch.Tensor] = []
        for i in range(n):
            xcur = self._resnet(f'downs.{i}.1', xcur, film_all, c, taps)
            for j in range(self.num_resnet_blocks[i]):
                xcur = self._resnet(f'downs.{i}.2.{j}', xcur, film_all, None, taps)
                hiddens.append(xcur)
            if self.layer_attns[i]:
                xcur = self._transformer(f'downs.{i}.3', xcur, c)
                if taps is not None:
                    taps[f'downs.{i}.3'] = xcur
            hiddens.append(xcur)
            if i < n - 1:
                xcur = self._conv(f'downs.{i}.4', xcur, 4, 2, 1)
            else:  # Parallel(conv3x3, conv1x1) summed (:1322)
                if f'downs.{i}.4.merged.weight' in self._plan['packed']:
                    xcur = self._conv(f'downs.{i}.4.merged', xcur, 3, 1, 1)
                else:
                    y = self._conv(f'downs.{i}.4.fns.0', xcur, 3, 1, 1)
                    xcur = self._conv(f'downs.{i}.4.fns.1', xcur, 1, 1, 0, out=y, accumulate=True)
            if taps is not None:
                taps[f'downs.{i}.4'] = xcur

        xcur = self._resnet('mid_block1', xcur, film_all, c, taps)
        xcur = self._self_attn('mid_attn.fn.fn', xcur, None)
        if taps is not None:
            taps['mid_attn'] = xcur
        xcur = self._resnet('mid_block2', xcur, film_all, c, taps)

        for i in range(n):
            ri = n - 1 - i
            xcur = self._resnet(f'ups.{i}.0', ops.concat2(xcur, hiddens.pop(), self.skip_connect_scale), film_all, c, taps)
            for j in range(self.num_resnet_blocks[ri]):
                xcur = self._resnet(f'ups.{i}.1.{j}', ops.concat2(xcur, hiddens.pop(), self.skip_connect_scale), film_all, None, taps)
            if self.layer_attns[ri]:
                xcur = self._transformer(f'ups.{i}.2', xcur, c)
                if taps is not None:
                    taps[f'ups.{i}.2'] = xcur
            if i < n - 1:
                xcur = ops.pixel_shuffle_silu(self._conv(f'ups.{i}.3.net.0', xcur, 1))
                if taps is not None:
                    taps[f'ups.{i}.3'] = xcur
        xcur = self._resnet('final_res_block', xcur, film_all, None, taps)
        y = self._conv('final_conv', xcur, 3, 1, 1)
        return ops.nhwc_to_nchw(y)


class UnetGraph:
    """CUDA graphs around ``Unet.forward`` per batch size: ~340 kernel launches replayed with one driver call.  Inputs are copied into static
    buffers; the returned tensor is the graph's static output (clone to keep it).

    Two graphs per shape: ``cond`` evaluates ``Unet.precompute_cond`` (the cond_images share of init_conv) into a static buffer, ``main`` is the
    evaluation proper reading that buffer.  ``new_cond=False`` tells the call that cond_images is unchanged since the previous call, so only
    ``main`` is replayed -- the PLMS sampler does that for evaluations 2..n+1 of a run."""

    def __init__(self, unet: Unet):
        self.unet = unet
        self._graphs = {}
        self.timing = None   # set to [] to collect (start, stop) CUDA event pairs around every replay (bench.py)

    @torch.no_grad()
    def __call__(self, x, time, cond_images, new_cond: bool = True, time_features: Optional[dict] = None):
        """``time_features`` = the rows of ``Unet.precompute_time`` for this batch (the PLMS sampler computes them for all its noise levels in one
        batch); when absent they are evaluated here from ``time``, outside the graph."""
        key = (tuple(x.shape), tuple(cond_images.shape), x.device.index)
        g = self._graphs.get(key)
        launches = lambda: int(ops.lib.load().sfb_launch_count())
        if time_features is None:
            time_features = self.unet.precompute_time(time)
        if g is None:
            sx, sc = x.clone(), cond_images.clone()
            sf = {k: v.clone() for k, v in time_features.items()}
            if self.unet._plan is None:
                self.unet.prepare()
            side = torch.cuda.Stream(device=x.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):  # warm-up outside capture: lazy attribute setting, tensor-map cache, allocator, arena size
                    feat = self.unet.precompute_cond(sc)
                    self.unet.forward(sx, None, cond_features=feat, time_features=sf)
            torch.cuda.current_stream().wait_stream(side)
            cond_graph, graph = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            n0 = launches()
            with torch.cuda.graph(cond_graph):
                feat = self.unet.precompute_cond(sc)
            n1 = launches()
            with torch.cuda.graph(graph):
                out = self.unet.forward(sx, None, cond_features=feat, time_features=sf)
            g = self._graphs[key] = (graph, cond_graph, sx, sf, sc, out, launches() - n1, n1 - n0, feat)
            new_cond = True
        graph, cond_graph, sx, sf, sc, out, n_kernels, n_cond_kernels, _ = g
        sx.copy_(x)
        for k, v in sf.items():
            if v.data_ptr() != time_features[k].data_ptr():
                v.copy_(time_features[k])
        if new_cond:
            if sc.data_ptr() != cond_images.data_ptr():
                sc.copy_(cond_images)
            cond_graph.replay()
            ops.note_graph_replay(n_cond_kernels)
        if self.timing is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            self.timing.append((e0, e1))
        else:
            graph.replay()
        ops.note_graph_replay(n_kernels)
        return out
