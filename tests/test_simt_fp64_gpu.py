"""Every SIMT launch of the UNet, the VAE and LPIPS (csrc/unet_ops.cu, csrc/lpips_ops.cu) replayed per element against fp64.

A module fixture runs the models of tests/test_conv_fp64_gpu.py (oracle/model_runs.py) with the ``ops.*`` front ends -- and ``_lib.call`` for
the LPIPS entry points -- wrapped, so that every launch's geometry and memory layout is recorded: row strides, slice offsets, the FiLM row
stride, residual and aliasing.  Entries are deduplicated per family; synthetic entries add the dispatch boundaries the models do not reach.

Each entry is replayed through the C ABI with fresh operands in its recorded layout, in 'tf32x3' and 'tf32' precision (GroupNorm also with
fusion bit 2 cleared), with three operand sets -- 'randn', 'one-signed' and 'edges' (zeros, powers of two, GroupNorm / LayerNorm inputs whose
mean is 10^2 standard deviations, softmax logits large enough to be near one-hot, exact ties for max-pool, all-zero LPIPS feature rows) --
and compared per element with the bounds of oracle/simt_fp64.py.  Operands sit inside NaN-filled buffers (floats before and after every
tensor and the channels between a slice and its row stride), the GroupNorm workspace is NaN-filled, and output channels outside a slice must
stay bit-identical.  The tracer names the kernels that ran; they must equal ``kernel_plan``.  Kernels with a fixed fold order run twice and
must agree bit for bit.

Out of scope: GEMMs (tests/test_conv_fp64_gpu.py), the sampler updates, image_glue.cu and the EFT-only kernels of eft_ops.cu
(tests/test_step_fp64_gpu.py) and ordering hazards between launches (tests/test_insitu_fp64_gpu.py checks every launch in place)."""
import ctypes
import math
from collections import defaultdict

import pytest
import torch

from oracle import model_runs, simt_fp64 as sf
from oracle.conv_fp64 import slice_guard_intact

pytestmark = pytest.mark.gpu

GUARD = 256
PRECISIONS = ('tf32x3', 'tf32')
SETS = ('randn', 'one-signed', 'edges')
FULL_MASK = 0x7fffffff
NAN = float('nan')

# the kernel each single-launch op runs (the LPIPS launches bypass the tracer)
FIXED = {'layernorm': 'layernorm_rows_kernel', 'cross_attention': 'cross_attention_kernel', 'gate_mlp_residual': 'gate_mlp_residual_kernel',
         'gate_residual': 'gate_residual_kernel', 'softmax_rows': 'softmax_rows_kernel', 'upsample2x': 'upsample2x_kernel',
         'nchw_to_nhwc': 'nchw_to_nhwc_kernel', 'nhwc_to_nchw': 'nhwc_to_nchw_kernel', 'im2col4': 'im2col_small_kernel', 'concat2': 'concat2_kernel',
         'pixel_shuffle_silu': 'pixel_shuffle_silu_kernel', 'time_fourier': 'time_fourier_kernel'}
LPIPS_NAMES = {'sfb_lpips_prep': 'lpips_prep', 'sfb_lpips_prep_backward': 'lpips_prep_backward', 'sfb_relu_nhwc': 'relu',
               'sfb_maxpool2x2_nhwc': 'maxpool', 'sfb_maxpool2x2_relu_backward_nhwc': 'maxpool_bwd', 'sfb_add_relu_mask': 'add_relu_mask',
               'sfb_lpips_head': 'lpips_head'}
DETERMINISTIC = {'groupnorm', 'mq_attention', 'cross_attention', 'gca_pool', 'layernorm'}


# ------------------------------------------------------------------------------------------------ catalogue
def _nhwc(t):
    from sparsefusion_b200 import ops
    nb, h, w, c, ld = ops._nhwc_meta(t)
    off = t.storage_offset() % ld
    return nb, h, w, c, ld, (off if off + c <= ld else 0)


def _rows(t):
    from sparsefusion_b200 import ops
    r, c, ld = ops._rows_meta(t)
    off = t.storage_offset() % ld if ld else 0
    return r, c, ld, (off if off + c <= ld else 0)


def _same(a, b):
    return a is not None and b is not None and a.data_ptr() == b.data_ptr()


class _Recorder:
    """wraps the ops front ends and _lib.call; entries deduplicated on their geometry within a family"""

    def __init__(self):
        self.entries = {}
        self.family = None

    def __call__(self, family):
        self.family = family
        return self

    def add(self, op, **f):
        key = (self.family, op) + tuple(sorted(f.items()))
        if key not in self.entries:
            self.entries[key] = dict(f, op=op, family=self.family, label=self.family, calls=0)
        self.entries[key]['calls'] += 1

    def __enter__(self):
        from sparsefusion_b200 import _lib as lib, ops
        self.saved = {n: getattr(ops, n) for n in ('groupnorm', 'layernorm', 'linear_small', 'mq_attention', 'cross_attention', 'gca_pool',
                                                   'gate_mlp_residual', 'gate_residual', 'softmax_rows', 'upsample2x', 'nchw_to_nhwc',
                                                   'nhwc_to_nchw', 'im2col4', 'concat2', 'pixel_shuffle_silu', 'time_fourier')}
        self.lib_call = lib.call
        o = self.saved
        rec = self

        def groupnorm(x, groups, gamma, beta, film=None, silu=True, eps=1e-5, out=None):
            y = o['groupnorm'](x, groups, gamma, beta, film, silu, eps, out)
            nb, h, w, c, ldx, xoff = _nhwc(x)
            _, _, _, _, ldy, yoff = _nhwc(y)
            rec.add('groupnorm', NB=nb, H=h, W=w, C=c, G=groups, ldx=ldx, xoff=xoff, ldy=ldy, yoff=yoff, film=film is not None,
                    ldf=film.stride(0) if film is not None else 0, act=bool(silu), alias='x=out' if _same(x, y) else '')
            return y

        def layernorm(x, g, b=None, pre_gelu=False, round_to_tf32=True, residual=None, out=None):
            y = o['layernorm'](x, g, b, pre_gelu, round_to_tf32, residual, out)
            T, C, ldx, xoff = _rows(x)
            rec.add('layernorm', T=T, C=C, ldx=ldx, xoff=xoff, ldy=_rows(y)[2], b=b is not None, res=residual is not None,
                    ldr=_rows(residual)[2] if residual is not None else 0, pre_gelu=bool(pre_gelu), round=bool(round_to_tf32),
                    alias='res=out' if _same(residual, y) else '')
            return y

        def linear_small(x, w, bias=None, pre=0, post=0, residual=None, round_to_tf32=False, out=None):
            y = o['linear_small'](x, w, bias, pre, post, residual, round_to_tf32, out)
            M, K, ldx, xoff = _rows(x)
            rec.add('linear_small', M=M, K=K, O=w.shape[0], ldx=ldx, xoff=xoff, ldy=_rows(y)[2], bias=bias is not None, res=residual is not None,
                    ldr=_rows(residual)[2] if residual is not None else 0, pre=pre, post=post, round=bool(round_to_tf32))
            return y

        def mq_attention(q, kv, null_kv, ckv, heads, dh):
            rec.add('mq_attention', B=q.shape[0], n=q.shape[1], heads=heads, dh=dh, nc=0 if ckv is None else ckv.shape[1])
            return o['mq_attention'](q, kv, null_kv, ckv, heads, dh)

        def cross_attention(q, kvc, null_kv, heads, dh):
            rec.add('cross_attention', B=q.shape[0], n=q.shape[1], heads=heads, dh=dh, nc=kvc.shape[1])
            return o['cross_attention'](q, kvc, null_kv, heads, dh)

        def gca_pool(x, wk, bk):
            nb, h, w, c, ldx, xoff = _nhwc(x)
            rec.add('gca_pool', NB=nb, HW=h * w, C=c, ldx=ldx, xoff=xoff)
            return o['gca_pool'](x, wk, bk)

        def gate_mlp_residual(h, hid, w2, b2, res):
            nb, hh, ww, c, ldh, hoff = _nhwc(h)
            rec.add('gate_mlp_residual', NB=nb, HW=hh * ww, C=c, Hd=hid.shape[-1], ldh=ldh, ldr=_nhwc(res)[4])
            return o['gate_mlp_residual'](h, hid, w2, b2, res)

        def gate_residual(h, gate, res, out=None):
            y = o['gate_residual'](h, gate, res, out)
            nb, hh, ww, c, ldh, _ = _nhwc(h)
            rec.add('gate_residual', NB=nb, HW=hh * ww, C=c, ldh=ldh, ldr=_nhwc(res)[4], ldo=_nhwc(y)[4], gate=gate is not None)
            return y

        def softmax_rows(x, scale=1.0, out=None):
            y = o['softmax_rows'](x, scale, out)
            r, c, ldx, _ = _rows(x)
            rec.add('softmax_rows', rows=r, cols=c, ldx=ldx, ldy=_rows(y)[2], scale=float(scale))
            return y

        def upsample2x(x):
            nb, h, w, c, ldx, _ = _nhwc(x)
            rec.add('upsample2x', NB=nb, H=h, W=w, C=c, ldx=ldx)
            return o['upsample2x'](x)

        def nchw_to_nhwc(src, dst, c_off=0, round_to_tf32=False):
            nb, c, h, w = src.shape
            rec.add('nchw_to_nhwc', NB=nb, C=c, H=h, W=w, ld=_nhwc(dst)[4], c_off=c_off, round=bool(round_to_tf32))
            return o['nchw_to_nhwc'](src, dst, c_off, round_to_tf32)

        def nhwc_to_nchw(src):
            nb, h, w, c, ld, _ = _nhwc(src)
            rec.add('nhwc_to_nchw', NB=nb, C=c, H=h, W=w, ld=ld)
            return o['nhwc_to_nchw'](src)

        def im2col4(x, kh, kw, pad):
            nb, h, w, c, ldx, _ = _nhwc(x)
            rec.add('im2col4', NB=nb, H=h, W=w, KH=kh, KW=kw, pad=pad, ldx=ldx)
            return o['im2col4'](x, kh, kw, pad)

        def concat2(a, b, scale_b, out=None):
            y = o['concat2'](a, b, scale_b, out)
            nb, h, w, c1, lda, _ = _nhwc(a)
            rec.add('concat2', NB=nb, H=h, W=w, C1=c1, lda=lda, C2=b.shape[-1], ldb=_nhwc(b)[4], ldo=_nhwc(y)[4], scale_b=float(scale_b))
            return y

        def pixel_shuffle_silu(y, out=None):
            r = o['pixel_shuffle_silu'](y, out)
            nb, h, w, c4, _, _ = _nhwc(y)
            rec.add('pixel_shuffle_silu', NB=nb, H=h, W=w, Co=c4 // 4, ldo=_nhwc(r)[4])
            return r

        def time_fourier(t, w):
            rec.add('time_fourier', B=t.shape[0], half=w.shape[0])
            return o['time_fourier'](t, w)

        def call(name, *args):
            if name in LPIPS_NAMES:
                op = LPIPS_NAMES[name]
                a = args
                if op == 'lpips_prep':
                    rec.add(op, H=a[2], W=a[3], normalize=a[4])
                elif op == 'lpips_prep_backward':
                    rec.add(op, H=a[1], W=a[2], normalize=a[3], factor=float(a[4]))
                elif op == 'relu':
                    rec.add(op, n=int(a[1]))
                elif op == 'maxpool':
                    rec.add(op, NB=a[2], H=a[3], W=a[4], C=a[5])
                elif op == 'maxpool_bwd':
                    rec.add(op, H=a[3], W=a[4], C=a[5])
                elif op == 'add_relu_mask':
                    rec.add(op, n=int(a[3]), head=a[1] is not None)
                elif op == 'lpips_head':
                    rec.add(op, HW=a[3], C=a[4])
            return rec.lib_call(name, *args)

        for n, f in dict(groupnorm=groupnorm, layernorm=layernorm, linear_small=linear_small, mq_attention=mq_attention,
                         cross_attention=cross_attention, gca_pool=gca_pool, gate_mlp_residual=gate_mlp_residual, gate_residual=gate_residual,
                         softmax_rows=softmax_rows, upsample2x=upsample2x, nchw_to_nhwc=nchw_to_nhwc, nhwc_to_nchw=nhwc_to_nchw, im2col4=im2col4,
                         concat2=concat2, pixel_shuffle_silu=pixel_shuffle_silu, time_fourier=time_fourier).items():
            setattr(ops, n, f)
        lib.call = call
        return self

    def __exit__(self, *exc):
        from sparsefusion_b200 import _lib as lib, ops
        for n, f in self.saved.items():
            setattr(ops, n, f)
        lib.call = self.lib_call
        torch.cuda.synchronize()
        return False


def _gn(label, NB, H, W, C, G, ldx=None, xoff=0, ldy=None, yoff=0, film=True, ldf=None):
    return dict(op='groupnorm', NB=NB, H=H, W=W, C=C, G=G, ldx=ldx or C, xoff=xoff, ldy=ldy or C, yoff=yoff, film=film,
                ldf=(ldf or 2 * C) if film else 0, act=True, alias='', label=label)


def _att(label, B, n, heads, dh, nc=0):
    return dict(op='mq_attention', B=B, n=n, heads=heads, dh=dh, nc=nc, label=label)


def _boundary_n(dh, limit, key):
    """the largest n (nc = 0, B = 1, one head) whose ``key`` shared-memory size is within ``limit``"""
    n = 1
    while sf.kernel_plan('mq_attention', dict(B=1, n=n + 1, heads=1, dh=dh, nc=0))[key] <= limit:
        n += 1
    return n


def _synthetic():
    E = [
        # GroupNorm: straddling groups on the row path (C / 4 a multiple of 256, 256 not a multiple of C / G / 4), past the cluster's 1 Mi
        _gn('C=3072 G=8 row path', 1, 32, 32, 3072, 8),
        _gn('C=3072 G=32 row path', 1, 24, 24, 3072, 32, ldx=3080, xoff=4),
        _gn('C=5120 G=16 row path', 1, 16, 16, 5120, 16),
        _gn('C=2048 G=8: whole groups per pass', 1, 32, 32, 2048, 8),
        # narrow groups (scalar statistics) and C / 4 > 256 with the generic apply kernel
        _gn('Cg = 3', 2, 8, 8, 24, 8, ldx=32, xoff=4),
        _gn('Cg = 5', 1, 9, 7, 40, 8, ldy=48, yoff=8),
        _gn('C / 4 = 384, generic apply', 2, 8, 8, 1536, 8),
        # cluster ITEMS at its thresholds: C = 256, 8 groups -> items = ceil(HW / 8) / 32; 17 falls back to the two launches
        _gn('ITEMS 4', 1, 32, 32, 256, 8),
        _gn('ITEMS 5', 1, 32, 40, 256, 8),
        _gn('ITEMS 8', 1, 32, 64, 256, 8),
        _gn('ITEMS 9', 1, 48, 48, 256, 8),
        _gn('ITEMS 16, exactly 2^20 elements', 1, 64, 64, 256, 8),
        _gn('one pixel more than 2^20 / 256', 1, 1, 4097, 256, 8),
        _gn('ITEMS 17 (C = 128, 2 groups)', 1, 34, 64, 128, 2),
        # batch at the cluster threshold, tiny images (the cluster width shrinks), FiLM rows with a stride
        _gn('NB 4', 4, 8, 8, 256, 8, ldf=768),
        _gn('NB 5', 5, 8, 8, 256, 8),
        _gn('HW 3: cluster of 2', 2, 1, 3, 256, 8),
        _gn('HW 1: cluster of 1', 1, 1, 1, 512, 8, film=False),
        _gn('HW 5: cluster of 4, slices', 1, 1, 5, 128, 8, ldx=160, xoff=16, ldy=192, yoff=32),
        # attention: the 64-key switch, the shared-memory limits, head widths
        _att('nk = 64', 1, 63, 2, 64), _att('nk = 65', 1, 64, 2, 64),
        _att('dh 16', 2, 16, 4, 16, nc=2), _att('dh 96', 1, 40, 2, 96, nc=1), _att('dh 128 keys', 1, 80, 2, 128),
        _att('dh 30 (plain)', 1, 20, 2, 30), _att('dh 160 (plain)', 1, 12, 2, 160), _att('dh 30, > 64 keys (plain)', 1, 90, 1, 30, nc=3),
        _att('qpw 4', 2, 256, 8, 64, nc=2),
        dict(op='cross_attention', B=2, n=16, heads=4, dh=64, nc=0, label='cross nc 0'),
        dict(op='cross_attention', B=2, n=16, heads=4, dh=64, nc=8, label='cross nc 8'),
        dict(op='cross_attention', B=1, n=8, heads=2, dh=36, nc=3, label='cross dh 36'),
        # GlobalContext around the split threshold and a channel count off the 16-channel tile
        dict(op='gca_pool', NB=2, HW=4095, C=64, ldx=64, xoff=0, label='HW 4095'),
        dict(op='gca_pool', NB=1, HW=4096, C=64, ldx=96, xoff=16, label='HW 4096 (split)'),
        dict(op='gca_pool', NB=2, HW=100, C=36, ldx=40, xoff=4, label='C 36'),
        dict(op='gca_pool', NB=1, HW=20000, C=20, ldx=20, xoff=0, label='HW 20000, C 20 (split)'),
        # small kernels
        dict(op='gate_mlp_residual', NB=2, HW=700, C=36, Hd=37, ldh=40, ldr=44, label='Hd 37, C % 8 = 4'),
        dict(op='gate_residual', NB=2, HW=50, C=36, ldh=40, ldr=36, ldo=48, gate=True, label='gate, slices'),
        dict(op='gate_residual', NB=1, HW=50, C=16, ldh=16, ldr=16, ldo=16, gate=False, label='no gate'),
        dict(op='softmax_rows', rows=3, cols=1, ldx=4, ldy=4, scale=0.5, label='cols 1'),
        dict(op='softmax_rows', rows=5, cols=257, ldx=260, ldy=257, scale=0.125, label='cols 257'),
        dict(op='softmax_rows', rows=4, cols=4096, ldx=4096, ldy=4100, scale=0.0625, label='cols 4096'),
        dict(op='layernorm', T=7, C=40, ldx=48, xoff=0, ldy=40, b=True, res=True, ldr=44, pre_gelu=False, round=True, alias='', label='C 40'),
        dict(op='layernorm', T=5, C=200, ldx=200, xoff=0, ldy=208, b=False, res=False, ldr=0, pre_gelu=True, round=True, alias='', label='C 200'),
        dict(op='upsample2x', NB=2, H=5, W=7, C=12, ldx=16, label='odd H, W'),
        dict(op='concat2', NB=1, H=3, W=5, C1=8, lda=12, C2=12, ldb=16, ldo=24, scale_b=0.25, label='slices, scale 1/4'),
        dict(op='nchw_to_nhwc', NB=2, C=36, H=5, W=9, ld=48, c_off=8, round=True, label='slice, rounded'),
        dict(op='nhwc_to_nchw', NB=2, C=36, H=5, W=9, ld=40, label='row stride 40'),
        dict(op='im2col4', NB=1, H=5, W=6, KH=3, KW=3, pad=1, ldx=8, label='3x3 in an 8-float row'),
        dict(op='pixel_shuffle_silu', NB=1, H=3, W=5, Co=8, ldo=12, label='slice'),
        dict(op='time_fourier', B=5, half=8, label='5 x 8'),
        dict(op='lpips_head', HW=100, C=68, label='C 68'),
        dict(op='maxpool_bwd', H=6, W=10, C=5, label='C 5'),
    ]
    for m, k, o in ((2, 8192, 24), (3, 17, 100), (8, 256, 300), (9, 1000, 64), (1, 33, 7)):
        E.append(dict(op='linear_small', M=m, K=k, O=o, ldx=k, xoff=0, ldy=o, bias=True, res=m % 2 == 1, ldr=o, pre=m % 2, post=m % 3,
                      round=m == 8, label=f'M {m} K {k} O {o}'))
    # the keys kernel's 200 KB limit at dh = 128 and the smem kernel's 160 KB limit (reachable only at dh = 4, beyond the keys kernel's limit)
    n200 = _boundary_n(128, 200 * 1024, 'smk')
    E += [_att('keys at 200 KB', 1, n200, 1, 128), _att('past 200 KB: plain', 1, n200 + 1, 1, 128)]
    n160 = _boundary_n(4, 160 * 1024, 'sm2')
    E += [_att('smem at 160 KB', 1, n160, 1, 4), _att('past 160 KB: plain', 1, n160 + 1, 1, 4)]
    for e in E:
        e.setdefault('family', 'synthetic')
        e.setdefault('calls', 0)
    return E


@pytest.fixture(scope='module')
def catalogue():
    rec = _Recorder()
    model_runs.record_models(rec)
    entries = list(rec.entries.values()) + _synthetic()
    fam = defaultdict(int)
    for e in entries:
        fam[e['family']] += 1
    print('\nSIMT catalogue: ' + ', '.join(f'{k} {v}' for k, v in fam.items()))
    return entries


# ------------------------------------------------------------------------------------------------ operands and guarded buffers
def _edge(t, g):
    """one in four of each: exact zero, a power of two, the value itself (twice)"""
    cat = torch.randint(0, 4, t.shape, device=t.device, generator=g)
    p2 = torch.exp2(torch.floor(torch.log2(t.abs().clamp_min(1e-30)))) * torch.sign(t)
    return torch.where(cat == 0, torch.zeros_like(t), torch.where(cat == 1, p2, t))


class _Gen:
    def __init__(self, kind, seed):
        self.kind = kind
        self.g = torch.Generator(device='cuda').manual_seed(seed)

    def __call__(self, *shape, signed=True, scale=1.0):
        t = torch.randn(*shape, device='cuda', generator=self.g) * scale
        if self.kind == 'one-signed' or not signed:
            t = t.abs()
        elif self.kind == 'edges':
            t = _edge(t, self.g)
        return t

    def rand(self, *shape):
        return torch.rand(*shape, device='cuda', generator=self.g)


_ALIVE = []     # the current replay's operand buffers: callers keep only raw pointers, so the buffers must outlive the launch


def _guarded(rows, ld, off, values):
    """NaN buffer [GUARD | rows x ld | GUARD] holding ``values`` [rows, width] at channel ``off``; returns (buffer, pointer, [rows, width] view)"""
    w = values.shape[-1]
    buf = torch.full((rows * ld + 2 * GUARD,), NAN, device='cuda')
    _ALIVE.append(buf)
    body = buf[GUARD:GUARD + rows * ld].view(rows, ld)
    body[:, off:off + w] = values.reshape(rows, w)
    return buf, body[:, off:].data_ptr(), body[:, off:off + w]


class _Out:
    """an output slot: [rows, ld] rows with the result at channel ``off``; everything else random with NaN in every other float, and the
    slot itself NaN before the launch"""

    def __init__(self, rows, ld, off, width):
        g = torch.Generator(device='cuda').manual_seed(rows * 7 + ld)
        self.rows, self.ld, self.off, self.width = rows, ld, off, width
        self.buf = torch.randn(rows * ld + 2 * GUARD, device='cuda', generator=g)
        self.buf[::2] = NAN
        self.body = self.buf[GUARD:GUARD + rows * ld].view(rows, ld)
        self.body[:, off:off + width] = NAN
        self.before = self.buf.clone()
        self.ptr = self.body[:, off:].data_ptr()

    def value(self):
        return self.body[:, self.off:self.off + self.width].clone()

    def guard_ok(self):
        b, a = self.before.view(torch.int32), self.buf.view(torch.int32)
        return (torch.equal(b[:GUARD], a[:GUARD]) and torch.equal(b[-GUARD:], a[-GUARD:])
                and slice_guard_intact(self.before[GUARD:-GUARD].view(self.rows, -1), self.buf[GUARD:-GUARD].view(self.rows, -1), self.off, self.width))


def _flat(t):
    return _guarded(1, t.numel(), 0, t.reshape(1, -1))


# ------------------------------------------------------------------------------------------------ replays
class _Tracer:
    def __init__(self):
        from sparsefusion_b200 import _lib as lib
        self.lib = lib
        self.buf = torch.zeros(65, dtype=torch.int64, device='cuda')
        self.names = ctypes.create_string_buffer(1 << 12)

    def run(self, fn):
        self.lib.call('sfb_trace_begin', self.buf.data_ptr(), 64)
        try:
            fn()
            torch.cuda.synchronize()
        finally:
            self.lib.load().sfb_trace_names(self.names, len(self.names))
            self.lib.call('sfb_trace_end')
        return self.names.value.decode().split('\n')[:-1]


def _replay(e, kind, seed, precision, mask, tracer, sm):
    """one replay: returns dict(outputs=[(name, got, ref, bound, exact, rounded)], guard_ok, names, planned, again (bit-identical rerun))"""
    from sparsefusion_b200 import _lib as lib, ops
    G = _Gen(kind, seed)
    op = e['op']
    _ALIVE.clear()
    call = lib.call
    S = lib.stream()
    res = dict(outputs=[], guard=True, names=None, planned=None, again=True)
    outs = []

    def run(fn):
        names = tracer.run(fn)
        first = [o.value() for o in outs]
        if op in DETERMINISTIC:                       # fixed fold orders: a second launch must reproduce every bit
            fn()
            torch.cuda.synchronize()
            res['again'] = all(torch.equal(a.view(torch.int32), o.value().view(torch.int32)) for a, o in zip(first, outs))
        res['names'] = names
        res['guard'] = all(o.guard_ok() for o in outs)
        return first

    if op == 'groupnorm':
        NB, HW, C, Gr = e['NB'], e['H'] * e['W'], e['C'], e['G']
        x = G(NB, HW, C) + (100.0 if kind == 'edges' else 0.0)
        gam, bet = G(C), G(C)
        film = G(NB, 2 * C, scale=0.5) if e['film'] else None
        _, xp, _ = _guarded(NB * HW, e['ldx'], e['xoff'], x.reshape(-1, C))
        fb = _guarded(NB, e['ldf'], 0, film) if film is not None else None
        gb, bb = _flat(gam), _flat(bet)
        ws = torch.full((lib.load().sfb_groupnorm_ws_floats(NB, Gr) + 64,), NAN, device='cuda')
        out = _Out(NB * HW, e['ldy'], e['yoff'], C)
        outs.append(out)
        got = run(lambda: call('sfb_groupnorm_nhwc', xp, e['ldx'], NB, HW, C, Gr, gb[1], bb[1], fb[1] if fb else None, e['ldf'], int(e['act']),
                               1e-5, ws.data_ptr(), None, out.ptr, e['ldy'], S))
        plan = sf.kernel_plan('groupnorm', dict(NB=NB, HW=HW, C=C, G=Gr), sm, mask, precision)
        y, b = sf.ref_groupnorm(x, Gr, gam, bet, film, e['act'], plan, precision)
        res['outputs'].append(('y', got[0].view(NB, HW, C), y, b, False, True))
        res['planned'] = plan['kernels']
        res['plan'] = plan
    elif op in ('mq_attention', 'cross_attention'):
        B, n, heads, dh, nc = e['B'], e['n'], e['heads'], e['dh'], e['nc']
        big = 32.0 if kind == 'edges' else 1.0
        q = G(B, n, heads * dh, scale=big)
        nkv = G(2, dh)
        qb = _flat(q)
        nb_ = _flat(nkv)
        out = _Out(1, B * n * heads * dh, 0, B * n * heads * dh)
        outs.append(out)
        scale = float(dh ** -0.5)
        if op == 'mq_attention':
            kv, ckv = G(B, n, 2 * dh), (G(B, nc, 2 * dh) if nc else None)
            kb, cb = _flat(kv), (_flat(ckv) if nc else None)
            got = run(lambda: call('sfb_mq_attention', qb[1], kb[1], nb_[1], cb[1] if cb else None, out.ptr, B, n, heads, dh, nc, scale, S))
            plan = sf.kernel_plan('mq_attention', dict(B=B, n=n, heads=heads, dh=dh, nc=nc), sm)
            y, b = sf.ref_mq_attention(q, kv, nkv, ckv, heads, dh, plan, precision)
            res['planned'] = plan['kernels']
            res['plan'] = plan
        else:
            kvc = G(B, nc, 2 * heads * dh) if nc else torch.zeros(B, 1, 2 * heads * dh, device='cuda')
            kb = _flat(kvc)
            got = run(lambda: call('sfb_cross_attention', qb[1], kb[1], nb_[1], out.ptr, B, n, heads, dh, nc, scale, S))
            y, b = sf.ref_cross_attention(q, kvc[:, :nc], nkv, heads, dh, precision)
            res['planned'] = [FIXED[op]]
        res['outputs'].append(('out', got[0].view(B, n, heads * dh), y, b, False, True))
    elif op == 'gca_pool':
        NB, HW, C = e['NB'], e['HW'], e['C']
        x = G(NB, HW, C)
        wk, bk = G(C, scale=(4.0 if kind == 'edges' else 1.0) / math.sqrt(C)), G(1)
        _, xp, _ = _guarded(NB * HW, e['ldx'], e['xoff'], x.reshape(-1, C))
        wb, bb = _flat(wk), _flat(bk)
        lg = torch.full((NB * HW + 2 * NB + 2,), NAN, device='cuda')
        out = _Out(NB, C, 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_gca_pool', xp, e['ldx'], NB, HW, C, wb[1], bb[1], lg.data_ptr(), out.ptr, S))
        plan = sf.kernel_plan('gca_pool', dict(HW=HW, C=C), sm)
        y, b = sf.ref_gca_pool(x, wk, bk, plan)
        res['outputs'].append(('pooled', got[0], y, b, False, False))
        res['planned'] = plan['kernels']
        res['plan'] = plan
    elif op == 'linear_small':
        M, K, O = e['M'], e['K'], e['O']
        x, w = G(M, K), G(O, K, scale=1 / math.sqrt(K))
        bias = G(O) if e['bias'] else None
        r = G(M, O) if e['res'] else None
        _, xp, _ = _guarded(M, e['ldx'], e['xoff'], x)
        wb = _flat(w)
        bb = _flat(bias) if bias is not None else None
        rb = _guarded(M, e['ldr'], 0, r) if r is not None else None
        out = _Out(M, e['ldy'], 0, O)
        outs.append(out)
        got = run(lambda: call('sfb_linear_small', xp, e['ldx'], wb[1], bb[1] if bb else None, rb[1] if rb else None, e['ldr'], out.ptr, e['ldy'],
                               M, K, O, e['pre'], e['post'], int(e['round']), S))
        y, b = sf.ref_linear_small(x, w, bias, r, e['pre'], e['post'], e['round'], precision)
        res['outputs'].append(('y', got[0], y, b, False, e['round']))
        res['planned'] = sf.kernel_plan('linear_small', dict(M=M, K=K), sm)['kernels']
    elif op == 'layernorm':
        T, C = e['T'], e['C']
        x = G(T, C) + (100.0 if kind == 'edges' else 0.0)
        g, b_ = G(C), (G(C) if e['b'] else None)
        r = G(T, C) if e['res'] else None
        _, xp, _ = _guarded(T, e['ldx'], e['xoff'], x)
        gb = _flat(g)
        bb = _flat(b_) if b_ is not None else None
        rb = _guarded(T, e['ldr'], 0, r) if r is not None else None
        out = _Out(T, e['ldy'], 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_layernorm_rows', xp, e['ldx'], gb[1], bb[1] if bb else None, rb[1] if rb else None, e['ldr'], out.ptr, e['ldy'],
                               T, C, int(e['pre_gelu']), int(e['round']), S))
        y, b = sf.ref_layernorm(x, g, b_, r, e['pre_gelu'], e['round'], precision)
        res['outputs'].append(('y', got[0], y, b, False, e['round']))
        res['planned'] = [FIXED[op]]
    elif op == 'gate_mlp_residual':
        NB, HW, C, Hd = e['NB'], e['HW'], e['C'], e['Hd']
        h, r, hid = G(NB, HW, C), G(NB, HW, C), G(NB, Hd)
        w2, b2 = G(C, Hd, scale=1 / math.sqrt(Hd)), G(C)
        _, hp, _ = _guarded(NB * HW, e['ldh'], 0, h.reshape(-1, C))
        _, rp, _ = _guarded(NB * HW, e['ldr'], 0, r.reshape(-1, C))
        hb, wb, bb = _flat(hid), _flat(w2), _flat(b2)
        out = _Out(NB * HW, C, 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_gate_mlp_residual_nhwc', hp, e['ldh'], hb[1], wb[1], bb[1], Hd, rp, e['ldr'], out.ptr, C, NB, HW, C, S))
        y, b = sf.ref_gate_mlp_residual(h, hid, w2, b2, r)
        res['outputs'].append(('out', got[0].view(NB, HW, C), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'gate_residual':
        NB, HW, C = e['NB'], e['HW'], e['C']
        h, r = G(NB, HW, C), G(NB, HW, C)
        gate = G(NB, C) if e['gate'] else None
        _, hp, _ = _guarded(NB * HW, e['ldh'], 0, h.reshape(-1, C))
        _, rp, _ = _guarded(NB * HW, e['ldr'], 0, r.reshape(-1, C))
        gb = _flat(gate) if gate is not None else None
        out = _Out(NB * HW, e['ldo'], 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_gate_residual_nhwc', hp, e['ldh'], gb[1] if gb else None, rp, e['ldr'], out.ptr, e['ldo'], NB, HW, C, S))
        y, b = sf.ref_gate_residual(h, gate, r)
        res['outputs'].append(('out', got[0].view(NB, HW, C), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'softmax_rows':
        R, Cc = e['rows'], e['cols']
        x = G(R, Cc, scale=30.0 if kind == 'edges' else 1.0)
        _, xp, _ = _guarded(R, e['ldx'], 0, x)
        out = _Out(R, e['ldy'], 0, Cc)
        outs.append(out)
        got = run(lambda: call('sfb_softmax_rows', xp, e['ldx'], out.ptr, e['ldy'], R, Cc, e['scale'], S))
        y, b = sf.ref_softmax_rows(x, e['scale'])
        res['outputs'].append(('y', got[0], y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'time_fourier':
        B, half = e['B'], e['half']
        t, w = G(B, scale=20.0), G(half)
        tb, wb = _flat(t), _flat(w)
        out = _Out(1, B * (2 * half + 1), 0, B * (2 * half + 1))
        outs.append(out)
        got = run(lambda: call('sfb_time_fourier', tb[1], wb[1], out.ptr, B, half, S))
        y, b = sf.ref_time_fourier(t, w)
        res['outputs'].append(('four', got[0].view(B, -1), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'pixel_shuffle_silu':
        NB, H, W, Co = e['NB'], e['H'], e['W'], e['Co']
        yv = G(NB, H, W, 4 * Co)
        yb = _flat(yv)
        out = _Out(NB * 4 * H * W, e['ldo'], 0, Co)
        outs.append(out)
        got = run(lambda: call('sfb_pixel_shuffle_silu_nhwc', yb[1], out.ptr, NB, H, W, Co, e['ldo'], S))
        y, b = sf.ref_pixel_shuffle_silu(yv)
        res['outputs'].append(('out', got[0].view(NB, 2 * H, 2 * W, Co), y, b, False, False))
        res['planned'] = [FIXED[op]]
    else:
        _exact_replay(e, G, res, outs, run, precision)
    return res


def _exact_replay(e, G, res, outs, run, precision):
    """ops whose result is a copy, a select or a single correctly rounded operation, and the LPIPS kernels"""
    from sparsefusion_b200 import _lib as lib
    call, S, op = lib.call, lib.stream(), e['op']
    res['planned'] = [FIXED[op]] if op in FIXED else None
    exact = lambda name, got, ref, rounded=False: res['outputs'].append((name, got, ref, None, True, rounded))
    if op == 'upsample2x':
        NB, H, W, C = e['NB'], e['H'], e['W'], e['C']
        x = G(NB, H, W, C)
        _, xp, _ = _guarded(NB * H * W, e['ldx'], 0, x.reshape(-1, C))
        out = _Out(NB * 4 * H * W, C, 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_upsample2x_nhwc', xp, e['ldx'], out.ptr, C, NB, H, W, C, S))
        exact('out', got[0].view(NB, 2 * H, 2 * W, C), sf.upsample2x(x))
    elif op == 'nchw_to_nhwc':
        NB, C, H, W = e['NB'], e['C'], e['H'], e['W']
        x = G(NB, C, H, W)
        xb = _flat(x)
        out = _Out(NB * H * W, e['ld'], e['c_off'], C)
        outs.append(out)
        rnd = e['round'] and precision == 'tf32'
        got = run(lambda: call('sfb_nchw_to_nhwc', xb[1], out.ptr - 4 * e['c_off'], NB, C, H, W, e['ld'], e['c_off'], int(e['round']), S))
        from sparsefusion_b200 import ops
        ref = x.permute(0, 2, 3, 1).reshape(-1, C)
        exact('out', got[0], ops.round_tf32(ref) if rnd else ref, rnd)
    elif op == 'nhwc_to_nchw':
        NB, C, H, W = e['NB'], e['C'], e['H'], e['W']
        x = G(NB, H, W, C)
        _, xp, _ = _guarded(NB * H * W, e['ld'], 0, x.reshape(-1, C))
        out = _Out(1, NB * C * H * W, 0, NB * C * H * W)
        outs.append(out)
        got = run(lambda: call('sfb_nhwc_to_nchw', xp, out.ptr, NB, C, H, W, e['ld'], S))
        exact('out', got[0].view(NB, C, H, W), x.permute(0, 3, 1, 2))
    elif op == 'im2col4':
        NB, H, W, KH, KW, pad = e['NB'], e['H'], e['W'], e['KH'], e['KW'], e['pad']
        k = (4 * KH * KW + 31) // 32 * 32
        x = G(NB, H, W, 4)
        _, xp, _ = _guarded(NB * H * W, e['ldx'], 0, x.reshape(-1, 4))
        out = _Out(NB * H * W, k, 0, k)
        outs.append(out)
        got = run(lambda: call('sfb_im2col4_nhwc', xp, e['ldx'], out.ptr, k, NB, H, W, KH, KW, pad, S))
        exact('out', got[0].view(NB, H, W, k), sf.im2col4(x, KH, KW, pad, k))
    elif op == 'concat2':
        npix = e['NB'] * e['H'] * e['W']
        a, b = G(npix, e['C1']), G(npix, e['C2'])
        _, ap, _ = _guarded(npix, e['lda'], 0, a)
        _, bp, _ = _guarded(npix, e['ldb'], 0, b)
        out = _Out(npix, e['ldo'], 0, e['C1'] + e['C2'])
        outs.append(out)
        got = run(lambda: call('sfb_concat2_nhwc', ap, e['C1'], e['lda'], bp, e['C2'], e['ldb'], e['scale_b'], out.ptr, e['ldo'], npix, S))
        sb = e['scale_b']
        ref = torch.cat((a, b * sb), -1)
        if sb != 0 and math.frexp(abs(sb))[0] == 0.5:       # a power of two: bit-exact
            exact('out', got[0], ref)
        else:
            res['outputs'].append(('out', got[0], ref.double(), sf.U * ref.double().abs() + sf.ATOL, False, False))
    elif op == 'relu':
        n = min(e['n'], 1 << 22)
        x = G(1, n)
        buf, xp, view = _guarded(1, n, 0, x)
        run(lambda: call('sfb_relu_nhwc', xp, n, S))
        exact('x', view.clone(), x.clamp_min(0))
        res['guard'] = bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())
    elif op == 'maxpool':
        NB, H, W, C = e['NB'], e['H'], e['W'], e['C']
        x = G(NB, H, W, C)
        if G.kind == 'edges':
            x = torch.round(x).clamp(-1, 2) + 0.0      # ties (+ 0.0 turns -0 into +0: fmaxf may return either zero of a tie)
        xb = _flat(x)
        out = _Out(1, NB * H * W * C // 4, 0, NB * H * W * C // 4)
        outs.append(out)
        got = run(lambda: call('sfb_maxpool2x2_nhwc', xb[1], out.ptr, NB, H, W, C, S))
        exact('y', got[0].view(NB, H // 2, W // 2, C), sf.maxpool2x2(x))
    elif op == 'maxpool_bwd':
        H, W, C = e['H'], e['W'], e['C']
        x = G(H, W, C).clamp_min(0)
        if G.kind != 'randn':
            x = torch.round(x).clamp(0, 2)             # ties, zero windows
        gy = G(H // 2, W // 2, C)
        xb, gb = _flat(x), _flat(gy)
        out = _Out(1, H * W * C, 0, H * W * C)
        outs.append(out)
        got = run(lambda: call('sfb_maxpool2x2_relu_backward_nhwc', xb[1], gb[1], out.ptr, H, W, C, S))
        exact('gx', got[0].view(H, W, C), sf.maxpool2x2_relu_backward(x, gy))
    elif op == 'add_relu_mask':
        n = min(e['n'], 1 << 22)
        g, act = G(1, n), G(1, n)
        gh = G(1, n) if e['head'] else None
        buf, gp, view = _guarded(1, n, 0, g)
        hb = _flat(gh) if gh is not None else None
        ab = _flat(act)
        run(lambda: call('sfb_add_relu_mask', gp, hb[1] if hb else None, ab[1], n, S))
        exact('g', view.clone(), sf.add_relu_mask(g, gh, act))
        res['guard'] = bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())
    elif op == 'lpips_head':
        HW, C = e['HW'], e['C']
        f0, f1 = G(HW, C), G(HW, C)
        w = G(C, signed=False)
        if G.kind == 'edges':
            f0[::7] = 0                                # r0 = 0
            f1[::5] = 0
        fb0, fb1, wb = _flat(f0), _flat(f1), _flat(w)
        val = torch.zeros(1, device='cuda')
        out = _Out(HW, C, 0, C)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_head', fb0[1], fb1[1], wb[1], HW, C, val.data_ptr(), out.ptr, S))
        v, vb, g, gbnd = sf.ref_lpips_head(f0, f1, w)
        res['outputs'].append(('value', val.view(()), v, vb, False, False))
        res['outputs'].append(('g_f0', got[0], g, gbnd, False, False))
    elif op == 'lpips_prep':
        H, W = e['H'], e['W']
        p, t = G.rand(3, H, W), G.rand(3, H, W)
        pb, tb = _flat(p), _flat(t)
        out = _Out(1, 2 * H * W * 4, 0, 2 * H * W * 4)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_prep', pb[1], tb[1], H, W, e['normalize'], out.ptr, S))
        y, b = sf.ref_lpips_prep(p, t, e['normalize'])
        res['outputs'].append(('x', got[0].view(2, H, W, 4), y, b, False, False))
    elif op == 'lpips_prep_backward':
        H, W = e['H'], e['W']
        gx = G(H, W, 4)
        gb = _flat(gx)
        out = _Out(1, 3 * H * W, 0, 3 * H * W)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_prep_backward', gb[1], H, W, e['normalize'], e['factor'], out.ptr, S))
        y, b = sf.ref_lpips_prep_backward(gx, e['normalize'], e['factor'])
        res['outputs'].append(('g', got[0].view(3, H, W), y, b, False, False))
    else:
        raise KeyError(op)


def _runs(e):
    """(precision, fusion mask) pairs an entry is replayed on"""
    masks = (FULL_MASK, FULL_MASK & ~4) if e['op'] == 'groupnorm' else (FULL_MASK,)
    return [(p, m) for p in PRECISIONS for m in masks]


def _key(e):
    skip = ('op', 'family', 'label', 'calls')
    return f"{e['family']} {e['op']} [{e['label']}] " + ' '.join(f'{k}={v}' for k, v in e.items() if k not in skip and v not in (0, False, ''))


@pytest.fixture(scope='module')
def replays(catalogue):
    from sparsefusion_b200 import _lib as lib, ops
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    tracer = _Tracer()
    out = dict(fail=[], names=set(), table={}, fixture_runs=0)
    table = {}
    try:
        for n, e in enumerate(catalogue):
            for precision, mask in _runs(e):
                ops.set_precision(precision)
                lib.call('sfb_set_fusion', mask)
                for si, kind in enumerate(SETS):
                    r = _replay(e, kind, 1000 * n + si, precision, mask, tracer, sm)
                    out['fixture_runs'] += 1
                    msg = []
                    kern = '/'.join(r['names'] or []) if e['op'] not in LPIPS_NAMES.values() else e['op']
                    if r['planned'] is not None:
                        if r['names'] != r['planned']:
                            msg.append(f"traced {r['names']}, planned {r['planned']}")
                        out['names'] |= set(r['names'])
                    for name, got, ref, bnd, is_exact, rounded in r['outputs']:
                        if is_exact:
                            if not torch.equal(got.float().contiguous().view(torch.int32), ref.float().contiguous().view(torch.int32)):
                                msg.append(f'{name} not bit-identical')
                            ratio = 0.0
                        else:
                            ratio = sf.max_ratio(got, ref, bnd)
                            if ratio > 1:
                                msg.append(f'{name} err/bound {ratio:.3g}')
                            tk = (e['family'], precision, kern)
                            cur = table.get(tk, (0.0, ''))
                            if ratio > cur[0]:
                                table[tk] = (ratio, kind)
                            elif tk not in table:
                                table[tk] = cur
                        if precision == 'tf32' and rounded and not sf.is_tf32(got):
                            msg.append(f'{name} not TF32-rounded')
                    if not r['guard']:
                        msg.append('memory outside the output changed')
                    if not r['again']:
                        msg.append('second run not bit-identical')
                    if msg:
                        out['fail'].append(f"{_key(e)} [{precision} mask={mask:#x} {kind}]: " + '; '.join(msg))
    finally:
        ops.set_precision('tf32x3')
        lib.call('sfb_set_fusion', FULL_MASK)
    out['table'] = table
    print('\nfamily      precision kernel                                          max err/bound  operand set')
    for (fam, prec, kern), (ratio, kind) in sorted(table.items()):
        print(f'{fam:11s} {prec:9s} {kern:48s} {ratio:13.3f}  {kind}')
    if out['fail']:
        print('\n'.join(out['fail'][:60]))
    return out


# ------------------------------------------------------------------------------------------------ tests
def test_catalogue_holds_the_launches_of_every_family(catalogue):
    by = defaultdict(list)
    for e in catalogue:
        by[(e['family'], e['op'])].append(e)
    fams = {f for f, _ in by}
    assert {'UNet', 'VAE', 'LPIPS', 'EFT', 'synthetic'} <= fams, fams
    assert by[('UNet', 'groupnorm')] and by[('VAE', 'groupnorm')] and by[('UNet', 'mq_attention')] and by[('UNet', 'gca_pool')]
    assert by[('VAE', 'softmax_rows')] and by[('LPIPS', 'lpips_head')] and by[('EFT', 'layernorm')]
    assert any(e['film'] and e['ldf'] > 2 * e['C'] for e in by[('UNet', 'groupnorm')])     # FiLM rows of the batched time MLP
    assert any(e['HW'] >= 4096 for e in by[('UNet', 'gca_pool')])                          # 128^2 latents: split pooling
    assert any(e['cols'] == 1024 for e in by[('VAE', 'softmax_rows')])
    assert not any(e.get('alias') for e in catalogue), [_key(e) for e in catalogue if e.get('alias')]


def test_no_model_groupnorm_has_straddling_groups(catalogue):
    """the recorded channel widths never reached the straddling row-path bookkeeping"""
    bad = [e for e in catalogue if e['op'] == 'groupnorm' and e['family'] != 'synthetic' and e['C'] // 4 > 256 and (e['C'] // 4) % 256 == 0
           and 256 % (e['C'] // e['G'] // 4) != 0]
    assert not bad, [_key(e) for e in bad]


def test_every_replay_is_within_its_fp64_bound(replays):
    assert not replays['fail'], f"{len(replays['fail'])} failures:\n" + '\n'.join(replays['fail'][:60])


def test_replays_reach_every_kernel(replays):
    want = {'gn_cluster_kernel<4>', 'gn_cluster_kernel<8>', 'gn_cluster_kernel<16>', 'gn_stats_kernel', 'gn_stats_rows_kernel', 'gn_apply_kernel',
            'gn_apply_cols_kernel', 'mq_attention_kernel', 'mq_attention_smem_kernel', 'mq_attention_keys_kernel', 'gca_logits_kernel',
            'gca_pool_kernel', 'gca_pool_split_kernel', 'linear_small_kernel<2>', 'linear_small_kernel<8>'} | set(FIXED.values())
    assert want <= replays['names'], sorted(want - replays['names'])
