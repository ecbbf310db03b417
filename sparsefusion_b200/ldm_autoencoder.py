"""AutoencoderKL -- host-side mirror of the SD-v1 KL-f8 VAE the distillation loop calls every SDS step
(external/ldm/models/autoencoder.py:285-333, external/ldm/modules/diffusionmodules/model.py:82-142,150-203,368-568,
external/ldm/modules/distributions/distributions.py:24-62, config external/ldm/configs/sd-vae.yaml).

SURVEY.md §8f "next" row #1.  Same module tree and state_dict keys as the reference (``encoder.*``, ``decoder.*``,
``quant_conv``, ``post_quant_conv``), without the pytorch_lightning / taming base classes the reference drags in.

ONE execution path behind ``encode`` / ``decode`` (both inference-only in the loop: ``vae.encode(...).mode()`` at
sparsefusion/distillation.py:299 and ``vae.decode(...)`` at :309 run under no_grad): the sm_90a engine (``_Sm90Engine`` below) -- NHWC
activations, every convolution / 1x1 projection / attention matmul on the wgmma 3xTF32 implicit-GEMM kernel (``ops.conv2d_nhwc``),
GroupNorm(32)+swish fused in one pass over the data, nearest upsampling and the row softmax as small kernels.  No cuDNN, no torch matmul,
no CPU fallback: the module classes below are PARAMETER CONTAINERS with the reference's names and shapes (checkpoints load unchanged);
calling them, or calling encode / decode with non-CUDA tensors, raises.  The plain-torch restatement that checks this engine lives in
the test oracle's ``vae_oracle`` module (test infrastructure, pinned to the reference's own Encoder / Decoder by tests/golden/vae.npz).
"""
from __future__ import annotations

import torch
import torch.nn as nn


def _norm(c):
    return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6, affine=True)


class _Container(nn.Module):
    """parameter container: the arithmetic of these blocks runs in _Sm90Engine, never through torch.nn"""

    def forward(self, *a, **k):
        raise RuntimeError(f'{type(self).__name__} is a parameter container of sparsefusion_b200.AutoencoderKL: the VAE runs on the sm_90a engine '
                           '(AutoencoderKL.encode / decode with CUDA tensors); there is no torch / CPU execution path')


class ResnetBlock(_Container):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = _norm(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.norm2 = _norm(out_channels)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        if in_channels != out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, 1, 1, 0)



class AttnBlock(_Container):
    def __init__(self, c):
        super().__init__()
        self.norm = _norm(c)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(c, c, 1) for _ in range(4))



class Downsample(_Container):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 2, 0)



class Upsample(_Container):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 1, 1)



class _Level(_Container):
    pass


class Encoder(_Container):
    def __init__(self, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, z_channels=4, double_z=True):
        super().__init__()
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.conv_in = nn.Conv2d(in_channels, ch, 3, 1, 1)
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        block_in = ch
        for i in range(self.num_resolutions):
            lvl = _Level()
            block_in, block_out = ch * in_ch_mult[i], ch * ch_mult[i]
            blocks = []
            for _ in range(num_res_blocks):
                blocks.append(ResnetBlock(block_in, block_out))
                block_in = block_out
            lvl.block = nn.ModuleList(blocks)
            lvl.attn = nn.ModuleList()
            if i != self.num_resolutions - 1:
                lvl.downsample = Downsample(block_in)
            self.down.append(lvl)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        self.norm_out = _norm(block_in)
        self.conv_out = nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, 3, 1, 1)



class Decoder(_Container):
    def __init__(self, ch=128, out_ch=3, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4):
        super().__init__()
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        block_in = ch * ch_mult[-1]
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        ups = []
        for i in reversed(range(self.num_resolutions)):
            lvl = _Level()
            block_out = ch * ch_mult[i]
            blocks = []
            for _ in range(num_res_blocks + 1):
                blocks.append(ResnetBlock(block_in, block_out))
                block_in = block_out
            lvl.block = nn.ModuleList(blocks)
            lvl.attn = nn.ModuleList()
            if i != 0:
                lvl.upsample = Upsample(block_in)
            ups.insert(0, lvl)
        self.up = nn.ModuleList(ups)
        self.norm_out = _norm(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)



class DiagonalGaussianDistribution:
    """distributions.py:24-62 (only what the loop uses: mode / sample)"""

    def __init__(self, parameters):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def mode(self):
        return self.mean

    def sample(self):
        return self.mean + self.std * torch.randn_like(self.mean)


class _Sm90Engine:
    """Encoder / Decoder forward on the sm_90a operators (NHWC, 3xTF32 tensor cores).  Weights are packed once (``prepare``)."""

    GROUPS, EPS = 32, 1e-6

    def __init__(self, vae: 'AutoencoderKL'):
        from . import ops
        self.ops = ops
        self.vae = vae
        P = {n: p.detach() for n, p in vae.named_parameters()}
        if next(iter(P.values())).device.type != 'cuda':
            raise RuntimeError('the sm_90a VAE engine needs CUDA parameters')
        self.P, self.W, self.B, self.S = P, {}, {}, {}
        for n, p in P.items():
            if n.endswith('.weight') and p.dim() == 4:
                base = n[:-len('.weight')]
                w, b = p, P.get(base + '.bias')
                if w.shape[0] % 4:                                   # decoder.conv_out: 3 output channels -> pad to 4 (TMA / vector stores)
                    padc = 4 - w.shape[0] % 4
                    w = torch.cat((w, w.new_zeros(padc, *w.shape[1:])), dim=0)
                    b = torch.cat((b, b.new_zeros(padc))) if b is not None else None
                self.W[base] = ops.pack_conv_weight(w)
                self.S[base] = ops.split_packed_weight(self.W[base]) if ops.get_precision() == 'tf32x3' else None   # these convolutions are tensor-bound
                self.B[base] = None if b is None else b.float().contiguous()

    # ---- building blocks
    def conv(self, name, x, k, stride=1, pad=None, pad_after=None, residual=None):
        w = self.W[name]
        pad = (k - 1) // 2 if pad is None else pad
        return self.ops.conv2d_nhwc(x, w, w.shape[0], k, k, stride, pad, bias=self.B[name], residual=residual, pad_after=pad_after, w_split=self.S[name])

    def gn(self, name, x, swish):
        return self.ops.groupnorm(x, self.GROUPS, self.P[name + '.weight'], self.P[name + '.bias'], None, swish, eps=self.EPS)

    def resnet(self, pfx, x):                                         # model.py:82-142
        h = self.conv(pfx + '.conv1', self.gn(pfx + '.norm1', x, True), 3)
        h = self.gn(pfx + '.norm2', h, True)
        sc = self.conv(pfx + '.nin_shortcut', x, 1) if (pfx + '.nin_shortcut') in self.W else x
        return self.conv(pfx + '.conv2', h, 3, residual=sc)

    def attn(self, pfx, x):                                           # model.py:150-203, single head over h*w tokens
        ops = self.ops
        nb, hh, ww, c = x.shape
        n = hh * ww
        if n % 32 or c % 32:
            raise NotImplementedError('sm_90a VAE attention needs h*w and channels to be multiples of 32')
        hn = self.gn(pfx + '.norm', x, False)
        out = torch.empty_like(x)
        wv = self.P[pfx + '.v.weight'].reshape(c, c)
        for b in range(nb):
            rows = hn[b].reshape(n, c)
            q = ops.linear_tc(rows, self.W[pfx + '.q'], c, bias=self.B[pfx + '.q'], w_split=self.S[pfx + '.q'])
            k = ops.linear_tc(rows, self.W[pfx + '.k'], c, bias=self.B[pfx + '.k'], w_split=self.S[pfx + '.k'])
            # in these three GEMMs the K-major "weight" operand is an ACTIVATION made by an earlier launch: dynamic_weights keeps the kernel from
            # prefetching it ahead of its programmatic-dependent-launch wait (the prologues of a PDL chain run far ahead of the bodies)
            scores = ops.linear_tc(q, k, n, dynamic_weights=True)     # q k^T: the keys are the GEMM's [Cout = n][K = c] operand
            probs = ops.softmax_rows(scores, scale=float(c) ** -0.5)
            vt = ops.linear_tc(wv, rows, n, dynamic_weights=True)     # (W_v h^T) = v^T without bias: [c][n], the K-major operand of P.V
            o = ops.linear_tc(probs, vt, c, bias=self.B[pfx + '.v'], dynamic_weights=True)   # rows of P sum to 1, so v's bias is added once per output row
            ops.linear_tc(o, self.W[pfx + '.proj_out'], c, bias=self.B[pfx + '.proj_out'], residual=x[b].reshape(n, c), out=out[b].reshape(n, c),
                          w_split=self.S[pfx + '.proj_out'])
        return out

    # ---- Encoder.forward (model.py:368-460) + quant_conv (autoencoder.py:311-315)
    def encode_moments(self, x):
        ops, enc = self.ops, self.vae.encoder
        nb, cin, hh, ww = x.shape
        xin = torch.zeros(nb, hh, ww, (cin + 3) // 4 * 4, dtype=torch.float32, device=x.device)
        ops.nchw_to_nhwc(x.float(), xin, 0)
        h = self.conv('encoder.conv_in', xin, 3)
        for i in range(enc.num_resolutions):
            for j in range(enc.num_res_blocks):
                h = self.resnet(f'encoder.down.{i}.block.{j}', h)
            if i != enc.num_resolutions - 1:
                h = self.conv(f'encoder.down.{i}.downsample.conv', h, 3, stride=2, pad=0, pad_after=1)      # F.pad (0,1,0,1), model.py:73-75
        h = self.resnet('encoder.mid.block_1', h)
        h = self.attn('encoder.mid.attn_1', h)
        h = self.resnet('encoder.mid.block_2', h)
        h = self.conv('encoder.conv_out', self.gn('encoder.norm_out', h, True), 3)
        return ops.nhwc_to_nchw(self.conv('quant_conv', h, 1))

    # ---- post_quant_conv + Decoder.forward (model.py:462-568)
    def decode(self, z):
        ops, dec = self.ops, self.vae.decoder
        nb, cz, hh, ww = z.shape
        zin = torch.zeros(nb, hh, ww, (cz + 3) // 4 * 4, dtype=torch.float32, device=z.device)
        ops.nchw_to_nhwc(z.float(), zin, 0)
        h = self.conv('decoder.conv_in', self.conv('post_quant_conv', zin, 1), 3)
        h = self.resnet('decoder.mid.block_1', h)
        h = self.attn('decoder.mid.attn_1', h)
        h = self.resnet('decoder.mid.block_2', h)
        for i in reversed(range(dec.num_resolutions)):
            for j in range(dec.num_res_blocks + 1):
                h = self.resnet(f'decoder.up.{i}.block.{j}', h)
            if i != 0:
                h = self.conv(f'decoder.up.{i}.upsample.conv', ops.upsample2x(h), 3)
        y = self.conv('decoder.conv_out', self.gn('decoder.norm_out', h, True), 3)
        out_ch = self.P['decoder.conv_out.weight'].shape[0]
        return ops.nhwc_to_nchw(y[..., :out_ch])


class AutoencoderKL(nn.Module):
    def __init__(self, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, out_ch=3, z_channels=4, embed_dim=4):
        super().__init__()
        self.encoder = Encoder(ch, ch_mult, num_res_blocks, in_channels, z_channels, True)
        self.decoder = Decoder(ch, out_ch, ch_mult, num_res_blocks, z_channels)
        self.quant_conv = nn.Conv2d(2 * z_channels, 2 * embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, z_channels, 1)
        self.embed_dim = embed_dim
        self._sm100 = None

    def prepare(self):
        """(re)pack the weights for the sm_90a engine; call again after loading a checkpoint or switching ops.set_precision"""
        self._sm100 = _Sm90Engine(self)
        return self

    def _engine_for(self, t):
        if not t.is_cuda:
            raise RuntimeError('sparsefusion_b200.AutoencoderKL runs on CUDA tensors only (sm_90a engine; there is no CPU fallback)')
        if torch.is_grad_enabled() and (t.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError('the sm_90a VAE engine is inference-only (the distillation loop calls the VAE under no_grad): wrap the call in '
                               'torch.no_grad()')
        if self._sm100 is None:
            self.prepare()
        return self._sm100

    def load_state_dict(self, *args, **kwargs):
        self._sm100 = None
        return super().load_state_dict(*args, **kwargs)

    def _apply(self, fn, *a, **k):
        # .to(device) / .float() / .half() move or recast the parameters: the packed copies the engine holds would be stale
        self._sm100 = None
        return super()._apply(fn, *a, **k)

    def encode(self, x):
        eng = self._engine_for(x)
        with torch.no_grad(), torch.cuda.device(x.device):
            return DiagonalGaussianDistribution(eng.encode_moments(x))

    def decode(self, z):
        eng = self._engine_for(z)
        with torch.no_grad(), torch.cuda.device(z.device):
            return eng.decode(z)

    def forward(self, x, sample_posterior=True):
        post = self.encode(x)
        z = post.sample() if sample_posterior else post.mode()
        return self.decode(z), post
