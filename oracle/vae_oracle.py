"""oracle/vae_oracle.py -- plain-torch restatement of the SD-v1 KL-f8 autoencoder the distillation loop calls
(external/ldm/models/autoencoder.py:285-333 encode / decode, external/ldm/modules/diffusionmodules/model.py:82-142 ResnetBlock,
:150-203 AttnBlock, :368-460 Encoder, :462-568 Decoder, external/ldm/modules/distributions/distributions.py:24-62).

TEST INFRASTRUCTURE ONLY (checker for sparsefusion_b200/ldm_autoencoder.py's sm_90a engine, and the VAE of bench.py's CPU /
eager-GPU baseline arms).  The product never imports this module and has no torch / CPU execution path of its own.

Pinning: oracle/gen_golden.py `vae` loads make_params() into the REFERENCE's own Encoder / Decoder modules (imported from
/root/reference in the build container), checks that this restatement reproduces them bit for bit, and stores their outputs as
tests/golden/vae.npz; tests/test_oracle_vae.py replays that on CPU.

Functional over a state dict with the reference's keys (``encoder.*``, ``decoder.*``, ``quant_conv.*``, ``post_quant_conv.*``), any
dtype / device -- fp64 on the GPU box is the tolerance reference of tests/test_vae_gpu.py.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

GROUPS, EPS = 32, 1e-6          # Normalize(): GroupNorm(32, eps=1e-6) (model.py:37-38)


def param_shapes(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, out_ch=3, z_channels=4, embed_dim=4) -> Dict[str, tuple]:
    s: Dict[str, tuple] = {}

    def conv(name, o, i, k):
        s[name + '.weight'], s[name + '.bias'] = (o, i, k, k), (o,)

    def norm(name, c):
        s[name + '.weight'], s[name + '.bias'] = (c,), (c,)

    def resnet(p, i, o):
        norm(p + '.norm1', i); conv(p + '.conv1', o, i, 3); norm(p + '.norm2', o); conv(p + '.conv2', o, o, 3)
        if i != o:
            conv(p + '.nin_shortcut', o, i, 1)

    def attn(p, c):
        norm(p + '.norm', c)
        for n in ('q', 'k', 'v', 'proj_out'):
            conv(f'{p}.{n}', c, c, 1)

    n = len(ch_mult)
    conv('encoder.conv_in', ch, in_channels, 3)
    in_mult = (1,) + tuple(ch_mult)
    block_in = ch
    for i in range(n):
        block_in, block_out = ch * in_mult[i], ch * ch_mult[i]
        for j in range(num_res_blocks):
            resnet(f'encoder.down.{i}.block.{j}', block_in, block_out)
            block_in = block_out
        if i != n - 1:
            conv(f'encoder.down.{i}.downsample.conv', block_in, block_in, 3)
    resnet('encoder.mid.block_1', block_in, block_in); attn('encoder.mid.attn_1', block_in); resnet('encoder.mid.block_2', block_in, block_in)
    norm('encoder.norm_out', block_in)
    conv('encoder.conv_out', 2 * z_channels, block_in, 3)
    block_in = ch * ch_mult[-1]
    conv('decoder.conv_in', block_in, z_channels, 3)
    resnet('decoder.mid.block_1', block_in, block_in); attn('decoder.mid.attn_1', block_in); resnet('decoder.mid.block_2', block_in, block_in)
    for i in reversed(range(n)):
        block_out = ch * ch_mult[i]
        for j in range(num_res_blocks + 1):
            resnet(f'decoder.up.{i}.block.{j}', block_in, block_out)
            block_in = block_out
        if i != 0:
            conv(f'decoder.up.{i}.upsample.conv', block_in, block_in, 3)
    norm('decoder.norm_out', block_in)
    conv('decoder.conv_out', out_ch, block_in, 3)
    conv('quant_conv', 2 * embed_dim, 2 * z_channels, 1)
    conv('post_quant_conv', z_channels, embed_dim, 1)
    return s


def make_params(seed: int = 0, **cfg) -> Dict[str, torch.Tensor]:
    """deterministic weights (numpy generator keyed by parameter order): kaiming-uniform-like convolutions, norm gains in [0.5, 1.5], small biases
    -- every term of every block is exercised"""
    rng = np.random.default_rng(seed)
    sd = {}
    for name, shape in param_shapes(**cfg).items():
        if len(shape) == 4:
            bound = 1.0 / np.sqrt(shape[1] * shape[2] * shape[3])
            v = (rng.random(shape, dtype=np.float32) * 2 - 1) * bound
        elif name.endswith('.weight'):
            v = rng.random(shape, dtype=np.float32) + 0.5
        else:
            v = rng.standard_normal(shape, dtype=np.float32) * 0.05
        sd[name] = torch.from_numpy(v.astype(np.float32))
    return sd


def _swish(x):
    return x * torch.sigmoid(x)                                   # nonlinearity(), model.py:32-34


def _gn(sd, p, x):
    return F.group_norm(x, GROUPS, sd[p + '.weight'], sd[p + '.bias'], EPS)


def _conv(sd, p, x, stride=1, padding=0):
    return F.conv2d(x, sd[p + '.weight'], sd[p + '.bias'], stride=stride, padding=padding)


def _resnet(sd, p, x):                                             # model.py:82-142 (temb is None, dropout 0)
    h = _conv(sd, p + '.conv1', _swish(_gn(sd, p + '.norm1', x)), padding=1)
    h = _conv(sd, p + '.conv2', _swish(_gn(sd, p + '.norm2', h)), padding=1)
    if (p + '.nin_shortcut.weight') in sd:
        x = _conv(sd, p + '.nin_shortcut', x)
    return x + h


def _attn(sd, p, x):                                               # model.py:150-203
    h = _gn(sd, p + '.norm', x)
    q, k, v = _conv(sd, p + '.q', h), _conv(sd, p + '.k', h), _conv(sd, p + '.v', h)
    b, c, hh, ww = q.shape
    w_ = torch.bmm(q.reshape(b, c, hh * ww).permute(0, 2, 1), k.reshape(b, c, hh * ww)) * (int(c) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    h = torch.bmm(v.reshape(b, c, hh * ww), w_.permute(0, 2, 1)).reshape(b, c, hh, ww)
    return x + _conv(sd, p + '.proj_out', h)


def _levels(sd, prefix):
    i = 0
    while f'{prefix}.{i}.block.0.norm1.weight' in sd:
        i += 1
    return i


def _blocks(sd, prefix):
    j = 0
    while f'{prefix}.{j}.norm1.weight' in sd:
        j += 1
    return j


def encoder(sd, x):                                                # Encoder.forward, model.py:427-460
    h = _conv(sd, 'encoder.conv_in', x, padding=1)
    n = _levels(sd, 'encoder.down')
    for i in range(n):
        for j in range(_blocks(sd, f'encoder.down.{i}.block')):
            h = _resnet(sd, f'encoder.down.{i}.block.{j}', h)
        if i != n - 1:
            h = _conv(sd, f'encoder.down.{i}.downsample.conv', F.pad(h, (0, 1, 0, 1), mode='constant', value=0), stride=2)   # model.py:73-75
    h = _resnet(sd, 'encoder.mid.block_2', _attn(sd, 'encoder.mid.attn_1', _resnet(sd, 'encoder.mid.block_1', h)))
    return _conv(sd, 'encoder.conv_out', _swish(_gn(sd, 'encoder.norm_out', h)), padding=1)


def decoder(sd, z):                                                # Decoder.forward, model.py:530-568
    h = _conv(sd, 'decoder.conv_in', z, padding=1)
    h = _resnet(sd, 'decoder.mid.block_2', _attn(sd, 'decoder.mid.attn_1', _resnet(sd, 'decoder.mid.block_1', h)))
    n = _levels(sd, 'decoder.up')
    for i in reversed(range(n)):
        for j in range(_blocks(sd, f'decoder.up.{i}.block')):
            h = _resnet(sd, f'decoder.up.{i}.block.{j}', h)
        if i != 0:
            h = _conv(sd, f'decoder.up.{i}.upsample.conv', F.interpolate(h, scale_factor=2.0, mode='nearest'), padding=1)   # model.py:47-52
    return _conv(sd, 'decoder.conv_out', _swish(_gn(sd, 'decoder.norm_out', h)), padding=1)


class DiagonalGaussianDistribution:
    """distributions.py:24-62 (mode / sample)"""

    def __init__(self, parameters):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def mode(self):
        return self.mean

    def sample(self):
        return self.mean + self.std * torch.randn_like(self.mean)


class TorchVAE:
    """AutoencoderKL.encode / decode (autoencoder.py:311-323) over a state dict; ``.to(device, dtype)`` returns a converted copy"""

    def __init__(self, sd: Dict[str, torch.Tensor]):
        self.sd = {k: v.detach() for k, v in sd.items()}

    def to(self, device=None, dtype=None):
        return TorchVAE({k: v.to(device=device, dtype=dtype) for k, v in self.sd.items()})

    def double(self):
        return self.to(dtype=torch.float64)

    def eval(self):
        return self

    @torch.no_grad()
    def encode(self, x):
        return DiagonalGaussianDistribution(_conv(self.sd, 'quant_conv', encoder(self.sd, x)))

    @torch.no_grad()
    def decode(self, z):
        return decoder(self.sd, _conv(self.sd, 'post_quant_conv', z))
