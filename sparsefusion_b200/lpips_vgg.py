"""PerceptualLoss -- host-side mirror of external/external_utils.py:11-49 (``lpips.LPIPS(net='vgg')`` behind a thin wrapper), the perceptual
term the distillation loop adds to the fusion loss from iteration 1000 on (sparsefusion/distillation.py:161, :176-178, :312-314).
SURVEY.md §8f row 3.

Same call: ``PerceptualLoss('vgg', device)(pred, target, normalize=True) -> [B,1,1,1]`` with images in [0,1]; differentiable w.r.t. ``pred``
(the loop back-propagates it into the render); ``target`` is treated as a constant, which is how the loop uses it (``pred_img`` is produced under
no_grad, distillation.py:302-309).

``state_dict`` keys follow the ``lpips`` package (``net.slice{1..5}.{torchvision index}.weight/bias``, ``lin{k}.model.1.weight``), so the package's
weights load unchanged; this repository cannot ship them, so a fresh module is randomly initialised and says so (``pretrained``).
``load_lpips_state_dict`` reads the pretrained weights from a local file or from the two files the ``lpips`` package is built from.

Engine (CUDA only, C ABI section 7): both images go through the VGG16 trunk as ONE batch of two NHWC tensors; the 13 convolutions and, for the
gradient, their 13 data-gradient convolutions (same kernel, weights transposed and flipped) run on the wgmma 3xTF32 implicit-GEMM engine with
pre-split weights; ReLU / 2x2 max-pool (forward, and backward fused with the ReLU mask) / the per-tap LPIPS head (value and gradient in one
launch) / input scaling are small NHWC kernels.  Value and gradient are produced together; autograd only sees one custom Function.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib as lib
from . import ops

CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512]
TV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)          # torchvision vgg16.features index of the 13 convolutions
SLICE_OF = (1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5)                   # lpips slice each of them lives in
TAPS = (1, 3, 6, 9, 12)                                              # convolution after whose ReLU a tap is taken (relu1_2 ... relu5_3)
CHNS = (64, 128, 256, 512, 512)


def conv_names() -> List[str]:
    return [f'net.slice{s}.{i}' for s, i in zip(SLICE_OF, TV_INDEX)]


LPIPS_LIN_FILE = 'vgg.pth'                    # the lpips package's weights/v0.1/vgg.pth: the lin{k}.model.1.weight heads
TORCHVISION_VGG16_FILE = 'vgg16-397923af.pth'  # torchvision's ImageNet VGG-16: features.{N}.weight / .bias


def _lpips_keys() -> List[str]:
    return [n + s for n in conv_names() for s in ('.weight', '.bias')] + [f'lin{k}.model.1.weight' for k in range(len(CHNS))]


def load_lpips_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """the pretrained LPIPS-VGG weights as a state dict in ``PerceptualLoss``'s (= ``lpips.LPIPS(net='vgg')``'s) key layout, from either

    * a file holding such a state dict, e.g. ``torch.save(lpips.LPIPS(net='vgg').state_dict(), path)`` on a machine with the ``lpips``
      package (extra keys such as ``scaling_layer.*`` are dropped), or
    * a directory holding the two files that package builds the network from: its ``weights/v0.1/vgg.pth`` (``LPIPS_LIN_FILE``, the
      ``lin*`` heads) and torchvision's ``vgg16-397923af.pth`` (``TORCHVISION_VGG16_FILE``, whose ``features.N`` convolutions become
      ``net.sliceK.N``).

    Files are read with ``torch.load(weights_only=True)``.  RuntimeError naming the keys when any LPIPS key is missing."""
    import os
    if os.path.isdir(path):
        lin = torch.load(os.path.join(path, LPIPS_LIN_FILE), map_location='cpu', weights_only=True)
        vgg = torch.load(os.path.join(path, TORCHVISION_VGG16_FILE), map_location='cpu', weights_only=True)
        src = {f'lin{k}.model.1.weight': lin[f'lin{k}.model.1.weight'] for k in range(len(CHNS)) if f'lin{k}.model.1.weight' in lin}
        for name, i in zip(conv_names(), TV_INDEX):
            for s in ('weight', 'bias'):
                if f'features.{i}.{s}' in vgg:
                    src[f'{name}.{s}'] = vgg[f'features.{i}.{s}']
    else:
        src = torch.load(path, map_location='cpu', weights_only=True)
    keys = _lpips_keys()
    missing = [k for k in keys if k not in src]
    if missing:
        raise RuntimeError(f'load_lpips_state_dict({path!r}): {len(missing)} LPIPS-VGG weights missing, e.g. {missing[:4]}')
    return {k: src[k] for k in keys}


class PerceptualLoss(nn.Module):
    def __init__(self, net: str = 'vgg', device=None, seed: int = 0):
        super().__init__()
        if net != 'vgg':
            raise NotImplementedError("sparsefusion_b200.PerceptualLoss: the distillation loop uses net='vgg' (distillation.py:161)")
        g = torch.Generator().manual_seed(seed)
        cin = 3
        for name, v in zip(conv_names(), [c for c in CFG if c != 'M']):
            w = torch.randn(v, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
            self._reg(name + '.weight', w)
            self._reg(name + '.bias', torch.randn(v, generator=g) * 0.05)
            cin = v
        for k, c in enumerate(CHNS):
            self._reg(f'lin{k}.model.1.weight', torch.rand(1, c, 1, 1, generator=g) * 4 / c)
        self.pretrained = False          # random weights until load_state_dict() is given the lpips package's
        self._plan = None
        self.device = device
        if device is not None:
            self.to(device)
        for p in self.parameters():
            p.requires_grad_(False)      # the metric network is frozen (lpips: requires_grad False)

    # parameters live in a flat dict under their dotted lpips names
    def _reg(self, name: str, value: torch.Tensor):
        self.register_parameter(name.replace('.', '/'), nn.Parameter(value))

    def state_dict(self, *a, **k):
        return {n.replace('/', '.'): v for n, v in super().state_dict(*a, **k).items()}

    def load_state_dict(self, sd, strict: bool = True):
        own = {n.replace('/', '.'): n for n, _ in self.named_parameters()}
        missing = [n for n in own if n not in sd]
        if strict and missing:
            raise RuntimeError(f'PerceptualLoss.load_state_dict: missing keys {missing[:4]}...')
        with torch.no_grad():
            for n, raw in own.items():
                if n in sd:
                    self.get_parameter(raw).copy_(sd[n])
        self.pretrained = True
        self._plan = None
        return self

    def _apply(self, fn, *a, **k):
        self._plan = None           # packed weights follow the parameters (device / dtype moves)
        return super()._apply(fn, *a, **k)

    def _p(self, name: str) -> torch.Tensor:
        return self.get_parameter(name.replace('.', '/'))

    # ------------------------------------------------------------------------------------------------ plan
    @torch.no_grad()
    def prepare(self):
        """pack the forward weights and the data-gradient weights (transposed over channels, flipped over taps), both pre-split for 3xTF32"""
        dev = self._p('lin0.model.1.weight').device
        if dev.type != 'cuda':
            raise RuntimeError('sparsefusion_b200.PerceptualLoss runs on CUDA only (there is no CPU fallback); call .cuda() first')
        fw, bw, bias = [], [], []
        for i, name in enumerate(conv_names()):
            w = self._p(name + '.weight').float()
            wp = ops.pack_conv_weight(w)
            fw.append((wp, ops.split_packed_weight(wp) if ops.get_precision() == 'tf32x3' else None))
            wt = w.permute(1, 0, 2, 3).flip(2, 3).contiguous()                  # [Cin, Cout, 3, 3]: d x = conv(d y, wt)
            if wt.shape[0] % 4:                                                  # first layer: 3 input channels -> 4 gradient channels
                wt = torch.cat((wt, wt.new_zeros(4 - wt.shape[0] % 4, *wt.shape[1:])), dim=0)
            wtp = ops.pack_conv_weight(wt)
            bw.append((wtp, ops.split_packed_weight(wtp) if ops.get_precision() == 'tf32x3' else None))
            bias.append(self._p(name + '.bias').float().contiguous())
        lin = [self._p(f'lin{k}.model.1.weight').float().reshape(-1).contiguous() for k in range(5)]
        self._plan = dict(fw=fw, bw=bw, bias=bias, lin=lin)
        return self

    # ------------------------------------------------------------------------------------------------ engine
    @torch.no_grad()
    def value_and_grad(self, pred: torch.Tensor, target: torch.Tensor, normalize: bool = True, want_grad: bool = True
                       ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """pred, target [3,H,W] planes in [0,1] -> (LPIPS distance as a 0-d tensor, d distance / d pred [3,H,W] or None)"""
        if self._plan is None:
            self.prepare()
        pl = self._plan
        assert pred.is_cuda and pred.shape == target.shape and pred.dim() == 3 and pred.shape[0] == 3
        _, H, W = pred.shape
        assert H % 16 == 0 and W % 16 == 0, 'four 2x2 max-pools: H and W must be multiples of 16'
        dev = pred.device
        st = lib.stream
        with torch.cuda.device(dev):
            x = torch.empty(2, H, W, 4, dtype=torch.float32, device=dev)
            p32, t32 = pred.float().contiguous(), target.float().contiguous()   # named: two temporaries could share one recycled block
            lib.call('sfb_lpips_prep', lib.fptr(p32), lib.fptr(t32), H, W, int(normalize), lib.fptr(x), st())
            acts: List[torch.Tensor] = []          # post-ReLU output of every convolution (both images)
            pooled_from: Dict[int, torch.Tensor] = {}
            h, i = x, 0
            for v in CFG:
                if v == 'M':
                    nb, hh, ww, c = h.shape
                    y = torch.empty(nb, hh // 2, ww // 2, c, dtype=torch.float32, device=dev)
                    lib.call('sfb_maxpool2x2_nhwc', lib.fptr(h), lib.fptr(y), nb, hh, ww, c, st())
                    pooled_from[i] = h            # conv i reads the pooled version of this activation
                    h = y
                    continue
                wp, sp = pl['fw'][i]
                h = ops.conv2d_nhwc(h, wp, v, 3, 3, 1, 1, bias=pl['bias'][i], w_split=sp)
                lib.call('sfb_relu_nhwc', lib.fptr(h), h.numel(), st())
                acts.append(h)
                i += 1
            value = torch.zeros(1, dtype=torch.float32, device=dev)
            g_head: Dict[int, torch.Tensor] = {}
            for k, ci in enumerate(TAPS):
                f = acts[ci]
                _, hh, ww, c = f.shape
                gh = torch.empty(1, hh, ww, c, dtype=torch.float32, device=dev)
                lib.call('sfb_lpips_head', lib.fptr(f[0]), lib.fptr(f[1]), lib.fptr(pl['lin'][k]), hh * ww, c, lib.fptr(value), lib.fptr(gh), st())
                g_head[ci] = gh
            if not want_grad:
                return value[0], None
            # ---- backward through the trunk for image 0.  G = d value / d (post-ReLU activation of conv i) arriving from the deeper layers
            G = None
            for i in range(12, -1, -1):
                a = acts[i][0:1]
                head = g_head.get(i)
                if G is None:                                                     # deepest layer (a tap): only its head feeds it
                    g, head = head.clone(), None
                else:
                    g = G
                lib.call('sfb_add_relu_mask', lib.fptr(g), None if head is None else lib.fptr(head), lib.fptr(a), g.numel(), st())
                # g = d value / d (pre-ReLU output of conv i); its data gradient is a convolution with the transposed, flipped weights
                wtp, sp = pl['bw'][i]
                d_in = ops.conv2d_nhwc(g, wtp, wtp.shape[0], 3, 3, 1, 1, w_split=sp)  # [1, h, w, Cin(i)] (4 channels for the first layer)
                if i == 0:
                    g = d_in
                    break
                if i in pooled_from:                                              # conv i read max_pool(act[i-1]): route to the window maxima
                    src = pooled_from[i][0:1]
                    _, hh, ww, c = src.shape
                    G = torch.empty(1, hh, ww, c, dtype=torch.float32, device=dev)
                    lib.call('sfb_maxpool2x2_relu_backward_nhwc', lib.fptr(src), lib.fptr(d_in), lib.fptr(G), hh, ww, c, st())
                else:
                    G = d_in
            g_pred = torch.empty(3, H, W, dtype=torch.float32, device=dev)
            lib.call('sfb_lpips_prep_backward', lib.fptr(g), H, W, int(normalize), 1.0, lib.fptr(g_pred), st())
        return value[0], g_pred

    # ------------------------------------------------------------------------------------------------ reference-shaped call
    def __call__(self, pred, target, normalize=True):
        if pred.shape[1] != 3:                                           # external_utils.py:33-35
            pred = pred.permute(0, 3, 1, 2)
            target = target.permute(0, 3, 1, 2)
        outs = [_LpipsFn.apply(self, pred[b], target[b].detach(), bool(normalize)) for b in range(pred.shape[0])]
        return torch.stack(outs).view(-1, 1, 1, 1)


class _LpipsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, pred, target, normalize):
        value, grad = module.value_and_grad(pred.detach(), target, normalize, want_grad=pred.requires_grad)
        ctx.save_for_backward(grad if grad is not None else pred.new_zeros(()))
        ctx.has_grad = grad is not None
        return value.clone()

    @staticmethod
    def backward(ctx, g_out):
        (grad,) = ctx.saved_tensors
        return None, (grad * g_out if ctx.has_grad else None), None, None
