"""EpipolarFeatureTransformer -- host-side mirror of sparsefusion/eft.py (reference): the frozen network that turns the 2-6 posed input views
into the per-target-view conditioning the VLDM consumes (a 256-channel 32x32 feature map + a low-res RGB estimate), evaluated once per scene
for every cached view (sparsefusion/distillation.py:92-127; SURVEY.md §8f row 4).

Same constructor keywords, ``encode(input_cameras, input_images)``, ``forward(ray_bundle, **kwargs)``, ``batched_forward(ray_bundle, n_batches,
**kwargs)`` and the same state_dict keys (``encoder_model.*`` = torchvision's resnet18, ``t1|t2|t3.pre.0``, ``t*.encoder.layers.N.{self_attn.in_proj_*,
self_attn.out_proj, linear1, linear2, norm1, norm2}``, ``t2_attn``, ``t3_attn``, ``color_layer.0``), so utils/load_model.py:34-41 loads its
checkpoint unchanged.  The torch modules registered here are PARAMETER CONTAINERS; the arithmetic runs on the sm_90a engine:

* ResNet-18 pyramid (eft.py:172-204): every convolution on the wgmma implicit-GEMM kernel with the (eval-mode) BatchNorm folded into the
  packed weights, ReLU / residual adds in its epilogue or one elementwise pass, 3x3/2 max-pool, bilinear (align_corners) resize of the four
  levels into ONE 512-channel NHWC tensor;
* epipolar look-up (eft.py:230-275): ``grid_sample`` of that tensor and of the input images at the NDC projections of all ray samples, one
  warp per point, written straight into the (padded) token rows of transformer T1;
* T1 / T2 / T3 (eft.py:18-50, :396-440): nn.TransformerEncoder(4 layers, d 256, 1 head, ff 256, post-norm, ReLU) as wgmma linears (3xTF32) +
  a one-warp-per-query attention core over the short sequences (2-6 views or 20 depth samples) + the fused residual LayerNorm kernel.

Camera maths (pytorch3d's PerspectiveCameras in NDC: x_view = x_world R + T, x_ndc = f x/z + p; centre = -T R^T) is used through the camera
object's own ``transform_points_ndc`` / ``get_camera_center`` when it has them (the reference environment), else through the restatement below
(any object with R, T, focal_length, principal_point).  Supported configuration = what utils/load_model.py:34 builds: encoder='resnet18',
return_features=True, out_sigmoid=True.
"""
from __future__ import annotations

import math
from collections import namedtuple
from typing import Optional

import torch
import torch.nn as nn

from . import _lib as lib
from . import ops

RayBundle = namedtuple('RayBundle', 'origins directions lengths xys')     # pytorch3d.renderer.RayBundle's fields


def transform_points_ndc(cameras, pts: torch.Tensor) -> torch.Tensor:
    """PerspectiveCameras.transform_points_ndc for cameras defined in NDC: pts [1 or NC, M, 3] world -> [NC, M, 3] (x_ndc, y_ndc, 1/z)"""
    if hasattr(cameras, 'transform_points_ndc'):
        return cameras.transform_points_ndc(pts)
    R, T = cameras.R, cameras.T                                              # [NC,3,3], [NC,3]
    f, p = cameras.focal_length, cameras.principal_point                    # [NC,2], [NC,2]
    v = torch.matmul(pts.expand(R.shape[0], -1, -1), R) + T[:, None, :]      # row-vector convention
    z = v[..., 2:3]
    xy = f[:, None, :] * v[..., :2] / z + p[:, None, :]
    return torch.cat((xy, 1.0 / z), dim=-1)


def camera_center(cameras) -> torch.Tensor:
    if hasattr(cameras, 'get_camera_center'):
        return cameras.get_camera_center()
    return -torch.matmul(cameras.T[:, None, :], cameras.R.transpose(1, 2))[:, 0, :]


def ray_bundle_to_ray_points(rb) -> torch.Tensor:
    return rb.origins[..., None, :] + rb.lengths[..., :, None] * rb.directions[..., None, :]


class HarmonicEmbedding(nn.Module):
    """utils/common_utils.py:68-140: [sin(f_k x), cos(f_k x), x] with f_k = omega0 * 2^k"""

    def __init__(self, n_harmonic_functions: int = 6, omega_0: float = 1.0, logspace: bool = True, append_input: bool = True):
        super().__init__()
        freq = 2.0 ** torch.arange(n_harmonic_functions, dtype=torch.float32) if logspace else \
            torch.linspace(1.0, 2.0 ** (n_harmonic_functions - 1), n_harmonic_functions, dtype=torch.float32)
        self.register_buffer('_frequencies', freq * omega_0, persistent=False)
        self.append_input = append_input
        self.n = n_harmonic_functions

    def get_output_dim(self, input_dims: int = 3) -> int:
        return input_dims * (2 * self.n + int(self.append_input))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        embed = (x[..., None] * self._frequencies).reshape(*x.shape[:-1], -1)
        return torch.cat((embed.sin(), embed.cos(), x), dim=-1) if self.append_input else torch.cat((embed.sin(), embed.cos()), dim=-1)


class TransformerEncoder(nn.Module):
    """parameter container with the reference's layout (eft.py:18-35); evaluated by _Engine.transformer"""

    def __init__(self, d_in, d_out, n_hidden=256, n_layer=4, post_linear=False):
        super().__init__()
        if post_linear:
            raise NotImplementedError('post_linear=True is not used by the EFT (eft.py:121,130,138)')
        self.post_linear = post_linear
        self.pre = nn.Sequential(nn.Linear(d_in, n_hidden), nn.GELU())
        self.encoder = nn.TransformerEncoder(nn.TransformerEncoderLayer(n_hidden, 1, n_hidden, 0.1), n_layer, enable_nested_tensor=False)

    def forward(self, *a, **k):
        raise RuntimeError('TransformerEncoder is a parameter container of sparsefusion_b200.EpipolarFeatureTransformer (sm_90a engine; no torch path)')


class EpipolarFeatureTransformer(nn.Module):
    def __init__(self, use_r=True, n_harmonic_functions=6, conv_dims=[32, ], return_features=False, encoder='lite', remove_unused_layers=True,
                 in_dim=3, out_dim=3, out_sigmoid=True, omega0=1.0, verbose=False):
        super().__init__()
        if encoder != 'resnet18' or in_dim != 3:
            raise NotImplementedError("sparsefusion_b200.EpipolarFeatureTransformer implements the released configuration: encoder='resnet18', in_dim=3 "
                                      '(utils/load_model.py:34)')
        import torchvision
        self.use_r, self.return_features, self.encoder, self.in_dim = use_r, return_features, encoder, in_dim
        self.omega0 = omega0
        self.harmonic_embedding = HarmonicEmbedding(n_harmonic_functions, omega0)
        self.conv_dims = 'default'
        self.encoder_num_layers = 4
        self.encoder_model = torchvision.models.resnet18(weights=None)         # container; the reference loads ImageNet weights, then the EFT checkpoint overwrites them
        if remove_unused_layers:
            self.encoder_model.layer4 = nn.Identity()
            self.encoder_model.fc = nn.Identity()
        self.feat_size = 64 + 64 + 128 + 256
        patch_dim = self.feat_size + in_dim
        ray_dim, depth_dim = self.harmonic_embedding.get_output_dim(6), self.harmonic_embedding.get_output_dim(1)
        d = 256
        self.t1 = TransformerEncoder(ray_dim + depth_dim + patch_dim, d)
        self.t2 = TransformerEncoder((2 if use_r else 1) * ray_dim + depth_dim + d, d)
        self.t2_attn = nn.Linear(d, 1)
        self.t3 = TransformerEncoder((2 if use_r else 1) * ray_dim + d, d)
        self.t3_attn = nn.Linear(d, 1)
        self.color_layer = nn.Sequential(nn.Linear(d, out_dim), nn.Sigmoid()) if out_sigmoid else nn.Sequential(nn.Linear(d, out_dim))
        self.out_sigmoid = out_sigmoid
        self.input_bbox = None
        self._plan = None
        self.eval()

    def get_config(self):
        return {'model': 'patch_nerf', 'conv_dims': self.conv_dims, 'encoder': self.encoder}

    def _apply(self, fn, *a, **k):
        self._plan = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._plan = None
        return super().load_state_dict(*a, **k)

    # ------------------------------------------------------------------------------------------------ plan
    @torch.no_grad()
    def prepare(self):
        dev = self.t2_attn.weight.device
        if dev.type != 'cuda':
            raise RuntimeError('sparsefusion_b200.EpipolarFeatureTransformer runs on CUDA only (there is no CPU fallback); call .cuda() first')
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        W, B = {}, {}

        def fold(conv, bn):             # eval-mode BatchNorm folded into the convolution: w' = w g / sqrt(var + eps), b' = beta - mean g / sqrt(var + eps)
            w = sd[f'encoder_model.{conv}.weight']
            scale = sd[f'encoder_model.{bn}.weight'] / torch.sqrt(sd[f'encoder_model.{bn}.running_var'] + 1e-5)
            w = w * scale[:, None, None, None]
            if w.shape[1] % 4:          # conv1: 3 input channels -> 4 (TMA strides)
                w = torch.cat((w, w.new_zeros(w.shape[0], 4 - w.shape[1] % 4, *w.shape[2:])), dim=1)
            W[conv] = ops.pack_conv_weight(w)
            B[conv] = (sd[f'encoder_model.{bn}.bias'] - sd[f'encoder_model.{bn}.running_mean'] * scale).contiguous()
        fold('conv1', 'bn1')
        for li, blocks in ((1, 2), (2, 2), (3, 2)):
            for bi in range(blocks):
                fold(f'layer{li}.{bi}.conv1', f'layer{li}.{bi}.bn1')
                fold(f'layer{li}.{bi}.conv2', f'layer{li}.{bi}.bn2')
                if f'encoder_model.layer{li}.{bi}.downsample.0.weight' in sd:
                    fold(f'layer{li}.{bi}.downsample.0', f'layer{li}.{bi}.downsample.1')
        for t in ('t1', 't2', 't3'):
            W[f'{t}.pre'] = ops.pack_conv_weight(sd[f'{t}.pre.0.weight'])
            B[f'{t}.pre'] = sd[f'{t}.pre.0.bias'].contiguous()
            for l in range(4):
                p = f'{t}.encoder.layers.{l}'
                for name, key in (('in', 'self_attn.in_proj_weight'), ('out', 'self_attn.out_proj.weight'), ('l1', 'linear1.weight'), ('l2', 'linear2.weight')):
                    W[f'{p}.{name}'] = ops.pack_conv_weight(sd[f'{p}.{key}'])
                for name, key in (('in', 'self_attn.in_proj_bias'), ('out', 'self_attn.out_proj.bias'), ('l1', 'linear1.bias'), ('l2', 'linear2.bias'),
                                  ('n1w', 'norm1.weight'), ('n1b', 'norm1.bias'), ('n2w', 'norm2.weight'), ('n2b', 'norm2.bias')):
                    B[f'{p}.{name}'] = sd[f'{p}.{key}'].contiguous()
        self._plan = dict(W=W, B=B, sd=sd)
        return self

    # ------------------------------------------------------------------------------------------------ engine pieces
    def _conv(self, name, x, k, stride, pad, relu=False, residual=None):
        pl = self._plan
        w = pl['W'][name]
        y = ops.conv2d_nhwc(x, w, w.shape[0], k, k, stride, pad, bias=pl['B'][name], residual=residual)
        if relu:
            lib.call('sfb_act_inplace', y.data_ptr(), y.numel(), 0, lib.stream())
        return y

    def _block(self, pfx, x, stride):
        """torchvision BasicBlock: relu(bn2(conv2(relu(bn1(conv1(x))))) + shortcut)"""
        h = self._conv(f'{pfx}.conv1', x, 3, stride, 1, relu=True)
        sc = self._conv(f'{pfx}.downsample.0', x, 1, stride, 0) if f'{pfx}.downsample.0' in self._plan['W'] else x
        return self._conv(f'{pfx}.conv2', h, 3, 1, 1, relu=True, residual=sc)

    def _linear(self, name, x, residual=None, act=None):
        pl = self._plan
        w = pl['W'][name]
        y = ops.linear_tc(x, w, w.shape[0], bias=pl['B'][name], residual=residual)
        if act is not None:
            lib.call('sfb_act_inplace', y.data_ptr(), y.numel(), act, lib.stream())
        return y

    def _transformer(self, t: str, x: torch.Tensor, S: int, Bn: int) -> torch.Tensor:
        """TransformerEncoder.forward (eft.py:37-50) on tokens x [S*Bn, d_in rounded up to a multiple of 4, pad columns zero] in sequence-major order
        -> [S*Bn, 256] (the packed weights are zero-padded to the next multiple of 32 columns, so the pad columns contribute nothing)"""
        h = self._linear(f'{t}.pre', x, act=1)                                                       # Linear + GELU
        B = self._plan['B']
        for l in range(4):                                                                           # post-norm encoder layers, ReLU feed-forward
            p = f'{t}.encoder.layers.{l}'
            qkv = self._linear(f'{p}.in', h)
            a = torch.empty(S * Bn, 256, dtype=torch.float32, device=x.device)
            lib.call('sfb_seq_attention', lib.fptr(qkv), lib.fptr(a), S, Bn, 256, lib.stream())
            h = ops.layernorm(self._linear(f'{p}.out', a, residual=h), B[f'{p}.n1w'], B[f'{p}.n1b'], round_to_tf32=False)
            f = self._linear(f'{p}.l1', h, act=0)
            h = ops.layernorm(self._linear(f'{p}.l2', f, residual=h), B[f'{p}.n2w'], B[f'{p}.n2b'], round_to_tf32=False)
        return h

    # ------------------------------------------------------------------------------------------------ reference API
    @torch.no_grad()
    def encode(self, input_cameras, input_images, input_bbox=None):
        """eft.py:155-204.  Returns (input_images NCHW, encoder_latent); the latent is kept NHWC [NC, H/2, W/2, 512] for the look-ups."""
        if input_bbox is not None:
            raise NotImplementedError('input_bbox masking is dead code in the reference (eft.py:267 resets the mask to ones)')
        if input_images.shape[1] != self.in_dim:
            input_images = input_images.permute(0, 3, 1, 2)
        if not input_images.is_cuda:
            raise RuntimeError('EpipolarFeatureTransformer.encode needs CUDA tensors (no CPU fallback)')
        if self._plan is None:
            self.prepare()
        self.input_images, self.input_cameras, self.input_bbox = input_images, input_cameras, input_bbox
        nc, _, H, W = input_images.shape
        dev = input_images.device
        with torch.cuda.device(dev):
            x = torch.zeros(nc, H, W, 4, dtype=torch.float32, device=dev)
            ops.nchw_to_nhwc(input_images.float(), x, 0)
            self._images_nhwc = x
            h = self._conv('conv1', x, 7, 2, 3, relu=True)                                           # conv1 + bn1 + relu
            lat = [h]
            hh, ww = h.shape[1], h.shape[2]
            p = torch.empty(nc, (hh + 1) // 2, (ww + 1) // 2, 64, dtype=torch.float32, device=dev)
            lib.call('sfb_maxpool3x3s2_nhwc', lib.fptr(h), lib.fptr(p), nc, hh, ww, 64, lib.stream())
            h = self._block('layer1.1', self._block('layer1.0', p, 1), 1)
            lat.append(h)
            h = self._block('layer2.1', self._block('layer2.0', h, 2), 1)
            lat.append(h)
            h = self._block('layer3.1', self._block('layer3.0', h, 2), 1)
            lat.append(h)
            out = torch.empty(nc, hh, ww, self.feat_size, dtype=torch.float32, device=dev)
            o = 0
            for t in lat:                                                                            # eft.py:194-204: all levels to the first level's size, concatenated
                c = t.shape[-1]
                lib.call('sfb_resize_bilinear_ac_nhwc', t.data_ptr(), t.stride(2), out[..., o:o + c].data_ptr(), self.feat_size, nc, t.shape[1], t.shape[2], c, hh, ww,
                         lib.stream())
                o += c
        self.encoder_latent = out
        return self.input_images, self.encoder_latent

    def encode_plucker(self, ray_origins, ray_dirs):
        plucker = torch.cat((ray_dirs, torch.cross(ray_origins, ray_dirs, dim=-1)), dim=-1)
        return self.harmonic_embedding(plucker)

    @torch.no_grad()
    def forward(self, ray_bundle, return_intermediates=False, **kwargs):
        """eft.py:330-470 for a flat bundle: origins / directions [N,3], lengths [N,D] (what batched_forward hands down).  Returns (rgb [N,3], f3 [N,256], 0)
        with return_features=True, else (rgb, coarse_rgb, 0)."""
        if kwargs.get('input_cameras') is not None:
            self.encode(kwargs['input_cameras'], kwargs['input_rgb'])
        origins, directions, lengths = ray_bundle.origins, ray_bundle.directions, ray_bundle.lengths
        lead = origins.shape[:-1]
        origins, directions = origins.reshape(-1, 3).float(), directions.reshape(-1, 3).float()
        lengths = lengths.reshape(-1, lengths.shape[-1]).float()
        N, D = lengths.shape
        cams = self.input_cameras
        dev = origins.device
        NC = self.encoder_latent.shape[0]
        he = self.harmonic_embedding
        with torch.cuda.device(dev):
            xyz = origins[:, None, :] + lengths[:, :, None] * directions[:, None, :]                 # [N,D,3]
            ray_dirs = torch.nn.functional.normalize(directions, dim=-1)
            query_plucker = self.encode_plucker(origins, ray_dirs)                                   # [N,78]
            # ---- index (eft.py:215-327): projections, look-ups, reference Pluecker coordinates, depth embedding
            ndc = transform_points_ndc(cams, xyz.reshape(1, N * D, 3))                               # [NC, N*D, 3]
            grid = (-ndc[..., :2]).contiguous()                                                      # grid_sample(-xy) (eft.py:250,272)
            M = N * D
            d1 = 78 + 13 + self.feat_size + self.in_dim                                              # T1 token width: 606
            d1p = (d1 + 3) // 4 * 4
            tok1 = torch.zeros(NC, M, d1p, dtype=torch.float32, device=dev)                          # rows: (camera, ray, depth); padded row stride for TMA
            fo = 78 + 13
            lat = self.encoder_latent
            lib.call('sfb_grid_sample_nhwc', lat.data_ptr(), lat.stride(2), lib.fptr(grid), tok1[..., fo:].data_ptr(), d1p, NC, lat.shape[1], lat.shape[2],
                     self.feat_size, M, lib.stream())
            img = self._images_nhwc
            lib.call('sfb_grid_sample_nhwc', img.data_ptr(), img.stride(2), lib.fptr(grid), tok1[..., fo + self.feat_size:].data_ptr(), d1p, NC, img.shape[1],
                     img.shape[2], self.in_dim, M, lib.stream())
            centers = camera_center(cams)                                                            # [NC,3]
            oc = centers[:, None, None, :].expand(NC, N, D, 3)
            input_dirs = torch.nn.functional.normalize(xyz[None] - oc, dim=-1)
            ref_plucker = self.encode_plucker(oc, input_dirs)                                        # [NC,N,D,78]
            depths = he(lengths[..., None])                                                          # [N,D,13]
            tok1[..., :78] = ref_plucker.reshape(NC, M, 78)
            tok1[..., 78:91] = depths.reshape(1, M, 13)
            # ---- T1: sequence = input views, batch = ray samples
            f1 = self._transformer('t1', tok1.view(NC * M, d1p), NC, M)                                  # zero pad columns meet zero pad weights                      # [NC*M,256]
            rgb, f3, t2_w, t3_w = self._heads(tok1, f1, query_plucker, NC, N, D)
            if self.return_features:
                return rgb.view(*lead, -1), f3.view(*lead, -1), 0
            ref_rgb = tok1[..., fo + self.feat_size:fo + self.feat_size + 3].view(NC, N, D, 3)       # get_coarse_rgb (eft.py:316-328)
            coarse = ((ref_rgb * t2_w.permute(1, 2, 0)[..., None]).sum(-2) * t3_w[..., None]).sum(0).clip(0, 1)
            if return_intermediates:
                return rgb, coarse, t2_w.permute(1, 2, 0)[..., None], t3_w[..., None]
            return rgb.view(*lead, -1), coarse.view(*lead, -1), 0

    def _heads(self, tok1, f1, query_plucker, NC: int, N: int, D: int):
        """everything after T1 (eft.py:396-470): T2 over the depth samples, its softmax pool, T3 over the input views, its softmax pool and the
        colour head.  tok1 [NC, N*D, >= 91] are T1's token rows, whose first 91 columns hold the reference Pluecker embedding (78) and the depth
        embedding (13) T2 / T3 reuse; f1 [NC*N*D, 256] is T1's output; query_plucker [N, 78].  Returns (rgb [N,3], f3 [N,256], t2_w [D,NC,N],
        t3_w [NC,N])."""
        dev = f1.device
        ref_plucker = tok1[..., :78].view(NC, N, D, 78)
        depths = tok1[0, :, 78:91].view(N, D, 13)
        # ---- T2: sequence = depth samples, batch = (view, ray)
        d2 = (2 if self.use_r else 1) * 78 + 13 + 256
        d2p = (d2 + 3) // 4 * 4
        tok2 = torch.zeros(D, NC * N, d2p, dtype=torch.float32, device=dev)
        t2v = tok2.view(D, NC, N, d2p)
        t2v[..., :78] = query_plucker[None, None]
        o = 78
        if self.use_r:
            t2v[..., o:o + 78] = ref_plucker.permute(2, 0, 1, 3)
            o += 78
        t2v[..., o:o + 13] = depths.permute(1, 0, 2)[:, None]
        t2v[..., o + 13:o + 13 + 256] = f1.view(NC, N, D, 256).permute(2, 0, 1, 3)
        f2 = self._transformer('t2', tok2.view(D * NC * N, d2p), D, NC * N).view(D, NC, N, 256)
        sd = self._plan['sd']
        t2 = torch.einsum('dcnf,f->dcn', f2, sd['t2_attn.weight'][0]) + sd['t2_attn.bias']      # Linear(256, 1)
        t2_w = torch.softmax(t2, dim=0)                                                          # over the depth samples (eft.py:415)
        f2 = (f2 * t2_w[..., None]).sum(dim=0)                                                   # [NC,N,256]
        # ---- T3: sequence = input views, batch = rays
        d3 = (2 if self.use_r else 1) * 78 + 256
        d3p = (d3 + 3) // 4 * 4
        tok3 = torch.zeros(NC, N, d3p, dtype=torch.float32, device=dev)
        tok3[..., :78] = query_plucker[None]
        o = 78
        if self.use_r:
            tok3[..., o:o + 78] = ref_plucker[:, :, D // 2, :]
            o += 78
        tok3[..., o:o + 256] = f2
        f3 = self._transformer('t3', tok3.view(NC * N, d3p), NC, N).view(NC, N, 256)
        t3_w = torch.softmax(torch.einsum('cnf,f->cn', f3, sd['t3_attn.weight'][0]) + sd['t3_attn.bias'], dim=0)   # over the views (eft.py:436)
        f3 = (f3 * t3_w[..., None]).sum(dim=0)                                                   # [N,256]
        rgb = f3 @ sd['color_layer.0.weight'].t() + sd['color_layer.0.bias']
        if self.out_sigmoid:
            rgb = torch.sigmoid(rgb)
        return rgb, f3, t2_w, t3_w

    @torch.no_grad()
    def batched_forward(self, ray_bundle, n_batches: int = 32, return_intermediates=False, **kwargs):
        """eft.py:472-525.  The reference splits the rays into n_batches chunks to bound its activation memory; every ray is independent of the others,
        so the chunking does not change any value -- here chunks of <= 4096 rays are used whatever n_batches says."""
        if return_intermediates:
            raise NotImplementedError('batched_forward(return_intermediates=True) is only used by visualisation scripts')
        if kwargs.get('input_cameras') is not None:
            self.encode(kwargs['input_cameras'], kwargs['input_rgb'])
        n_pts = ray_bundle.lengths.shape[-1]
        spatial = list(ray_bundle.origins.shape[:-1])
        o, d, l = ray_bundle.origins.reshape(-1, 3), ray_bundle.directions.reshape(-1, 3), ray_bundle.lengths.reshape(-1, n_pts)
        outs = [self.forward(RayBundle(o[i:i + 4096], d[i:i + 4096], l[i:i + 4096], None)) for i in range(0, o.shape[0], 4096)]
        a, b = (torch.cat([t[j] for t in outs], dim=0).view(*spatial, -1) for j in (0, 1))
        return a, b, 0

    # ------------------------------------------------------------------------------------------------ view-batched feature cache
    CACHE_RAYS = 4096       # rays (all depth samples, all input views) per transformer pass of feature_cache: the bound batched_forward keeps

    @torch.no_grad()
    def feature_cache(self, origins, directions, lengths, input_cameras, input_images, hw=None):
        """the EFT feature cache of V query views at once (sparsefusion/distillation.py:95-125 without the per-view loop): what
        ``batched_forward`` returns for each view v after ``encode(input_cameras[v], input_images)``, for all views in one pass.

        origins / directions [V,N,3], lengths [V,N,D]: the query bundles; ``input_cameras``: the NC input cameras of every view in that view's
        own frame -- one object whose R is [V,NC,3,3] (T [V,NC,3], focal_length / principal_point [V,NC,2]) or a sequence of V camera objects
        with NC cameras each; ``input_images`` [NC,3,H,W] in [0,1], shared by every view.  ``hw`` = (h, w) with h * w = N (a square grid when
        None).  Returns (features [V,256,h,w], rgb [V,3,h,w]): the conditioning features and the colour head's low-resolution image,
        ``batched_forward``'s two outputs with return_features=True (utils/load_model.py:34) rearranged 'b h w f -> b f h w' (:110-118).

        The ResNet-18 pyramid runs once (it depends on the images only; ``encode(None, input_images)``, which leaves ``input_cameras`` None).
        Each T1 token row -- point, projection by its view's camera, look-ups, embeddings -- is written by one kernel (``sfb_eft_t1_tokens``);
        the transformers run on whole views, at most ``CACHE_RAYS`` rays per pass (batched_forward's chunk), so the activations are bounded
        whatever V is: building a scene's 82-view cache peaked at 2.7 GB (NC = 2) and 7.3 GB (NC = 6) of device memory on an H100
        (tools/scene_bench.py)."""
        if isinstance(input_cameras, (list, tuple)):
            R = torch.stack([c.R for c in input_cameras])
            T = torch.stack([c.T for c in input_cameras])
            f = torch.stack([c.focal_length for c in input_cameras])
            p = torch.stack([c.principal_point for c in input_cameras])
        else:
            R, T, f, p = input_cameras.R, input_cameras.T, input_cameras.focal_length, input_cameras.principal_point
        V, N, D = lengths.shape
        NC = R.shape[1]
        if R.shape[0] != V or origins.shape[:2] != (V, N) or directions.shape[:2] != (V, N):
            raise ValueError(f'feature_cache: {R.shape[0]} camera sets for bundles of {tuple(origins.shape[:2])} / {tuple(lengths.shape)}')
        if hw is None:
            s = math.isqrt(N)
            if s * s != N:
                raise ValueError(f'feature_cache: {N} rays per view is not a square grid; pass hw')
            hw = (s, s)
        self.encode(None, input_images)
        if NC != self.encoder_latent.shape[0]:
            raise ValueError(f'feature_cache: {NC} cameras per view for {self.encoder_latent.shape[0]} input images')
        dev = self.encoder_latent.device
        cams = torch.cat((R.reshape(V, NC, 9), T.reshape(V, NC, 3), f.reshape(V, NC, 2), p.reshape(V, NC, 2)), dim=-1).to(dev, torch.float32).contiguous()
        origins, directions = origins.to(dev, torch.float32).contiguous(), directions.to(dev, torch.float32).contiguous()
        lengths = lengths.to(dev, torch.float32).contiguous()
        lat, img = self.encoder_latent, self._images_nhwc
        d1p = (78 + 13 + self.feat_size + self.in_dim + 3) // 4 * 4
        feats = torch.empty(V, 256, N, dtype=torch.float32, device=dev)
        rgbs = torch.empty(V, 3, N, dtype=torch.float32, device=dev)
        step = max(1, self.CACHE_RAYS // N)
        with torch.cuda.device(dev):
            for v0 in range(0, V, step):
                v1 = min(V, v0 + step)
                Vc = v1 - v0
                M = Vc * N * D
                tok1 = torch.empty(NC, M, d1p, dtype=torch.float32, device=dev)
                lib.call('sfb_eft_t1_tokens', lib.fptr(cams[v0:v1]), lib.fptr(origins[v0:v1]), lib.fptr(directions[v0:v1]), lib.fptr(lengths[v0:v1]),
                         lat.data_ptr(), lat.stride(2), lat.shape[1], lat.shape[2], self.feat_size, img.data_ptr(), img.stride(2), img.shape[1],
                         img.shape[2], self.in_dim, float(self.omega0), lib.fptr(tok1), d1p, Vc, NC, N, D, lib.stream())
                o, d = origins[v0:v1].reshape(Vc * N, 3), directions[v0:v1].reshape(Vc * N, 3)
                query_plucker = self.encode_plucker(o, torch.nn.functional.normalize(d, dim=-1))             # [Vc*N, 78]
                f1 = self._transformer('t1', tok1.view(NC * M, d1p), NC, M)
                rgb, f3, _, _ = self._heads(tok1, f1, query_plucker, NC, Vc * N, D)
                feats[v0:v1] = f3.view(Vc, N, 256).transpose(1, 2)
                rgbs[v0:v1] = rgb.view(Vc, N, 3).transpose(1, 2)
        return feats.view(V, 256, *hw), rgbs.view(V, 3, *hw)
