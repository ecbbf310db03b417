"""Every SIMT launch of the UNet, the VAE and LPIPS (csrc/unet_ops.cu, csrc/lpips_ops.cu) replayed per element against fp64.

A module fixture runs the models of tests/test_conv_fp64_gpu.py (oracle/model_runs.py) under oracle/insitu.Catalogue, which records every
front-end launch and every call of an LPIPS entry point with its geometry and memory layout (``simt_fp64.entry``): row strides, slice
offsets, the FiLM row stride, residual and aliasing.  Entries are deduplicated per family; synthetic entries add the dispatch boundaries the
models do not reach.

Each entry is replayed through the C ABI with fresh operands in its recorded layout, in 'tf32x3' and 'tf32' precision (GroupNorm also with
fusion bit 2 cleared), with three operand sets -- 'randn', 'one-signed' and 'edges' (zeros, powers of two, GroupNorm / LayerNorm inputs whose
mean is 10^2 standard deviations, softmax logits large enough to be near one-hot, exact ties for max-pool, all-zero LPIPS feature rows) --
and compared per element with the bounds of oracle/simt_fp64.py.  Operands sit inside NaN-filled buffers (floats before and after every
tensor and the channels between a slice and its row stride), the GroupNorm workspace is NaN-filled, and every float of an output buffer
outside the output (random, NaN in every other one) must stay bit-identical.  The tracer names the kernels that ran; they must equal
``kernel_plan``.  Kernels with a fixed fold order run twice and must agree bit for bit.

Out of scope: GEMMs (tests/test_conv_fp64_gpu.py), the sampler updates, image_glue.cu and the EFT-only kernels of eft_ops.cu
(tests/test_step_fp64_gpu.py) and ordering hazards between launches (tests/test_insitu_fp64_gpu.py checks every launch in place)."""
import math
from collections import defaultdict

import pytest
import torch

from _helpers import NAN, Out, Tracer, guarded, ptr, release
from oracle import insitu, model_runs, simt_fp64 as sf

pytestmark = pytest.mark.gpu

PRECISIONS = ('tf32x3', 'tf32')
SETS = ('randn', 'one-signed', 'edges')
FULL_MASK = 0x7fffffff

# the kernel each single-launch op runs (the LPIPS launches bypass the tracer)
FIXED = {'layernorm': 'layernorm_rows_kernel', 'cross_attention': 'cross_attention_kernel', 'gate_mlp_residual': 'gate_mlp_residual_kernel',
         'gate_residual': 'gate_residual_kernel', 'softmax_rows': 'softmax_rows_kernel', 'upsample2x': 'upsample2x_kernel',
         'nchw_to_nhwc': 'nchw_to_nhwc_kernel', 'nhwc_to_nchw': 'nhwc_to_nchw_kernel', 'im2col4': 'im2col_small_kernel', 'concat2': 'concat2_kernel',
         'pixel_shuffle_silu': 'pixel_shuffle_silu_kernel', 'time_fourier': 'time_fourier_kernel'}
DETERMINISTIC = {'groupnorm', 'mq_attention', 'cross_attention', 'gca_pool', 'layernorm'}


# ------------------------------------------------------------------------------------------------ catalogue
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
    cat = insitu.Catalogue(sf.entry)
    model_runs.record_models(cat)
    entries = list(cat.entries.values()) + _synthetic()
    fam = defaultdict(int)
    for e in entries:
        fam[e['family']] += 1
    print('\nSIMT catalogue: ' + ', '.join(f'{k} {v}' for k, v in fam.items()))
    return entries


# ------------------------------------------------------------------------------------------------ operands
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


# ------------------------------------------------------------------------------------------------ replays
def _replay(e, kind, seed, precision, mask, tracer, sm):
    """one replay: returns dict(outputs=[(name, got, ref, bound, exact, rounded)], guard_ok, names, planned, again (bit-identical rerun))"""
    from sparsefusion_b200 import _lib as lib, ops
    G = _Gen(kind, seed)
    op = e['op']
    release()
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
        xp = ptr(guarded(x.reshape(-1, C), e['ldx'], e['xoff']))
        fb = ptr(guarded(film, e['ldf']))
        gb, bb = ptr(guarded(gam)), ptr(guarded(bet))
        ws = torch.full((lib.load().sfb_groupnorm_ws_floats(NB, Gr) + 64,), NAN, device='cuda')
        out = Out(NB * HW, C, e['ldy'], e['yoff'])
        outs.append(out)
        got = run(lambda: call('sfb_groupnorm_nhwc', xp, e['ldx'], NB, HW, C, Gr, gb, bb, fb, e['ldf'], int(e['act']),
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
        qb = ptr(guarded(q))
        nb_ = ptr(guarded(nkv))
        out = Out(1, B * n * heads * dh)
        outs.append(out)
        scale = float(dh ** -0.5)
        if op == 'mq_attention':
            kv, ckv = G(B, n, 2 * dh), (G(B, nc, 2 * dh) if nc else None)
            kb, cb = ptr(guarded(kv)), ptr(guarded(ckv))
            got = run(lambda: call('sfb_mq_attention', qb, kb, nb_, cb, out.ptr, B, n, heads, dh, nc, scale, S))
            plan = sf.kernel_plan('mq_attention', dict(B=B, n=n, heads=heads, dh=dh, nc=nc), sm)
            y, b = sf.ref_mq_attention(q, kv, nkv, ckv, heads, dh, plan, precision)
            res['planned'] = plan['kernels']
            res['plan'] = plan
        else:
            kvc = G(B, nc, 2 * heads * dh) if nc else torch.zeros(B, 1, 2 * heads * dh, device='cuda')
            kb = ptr(guarded(kvc))
            got = run(lambda: call('sfb_cross_attention', qb, kb, nb_, out.ptr, B, n, heads, dh, nc, scale, S))
            y, b = sf.ref_cross_attention(q, kvc[:, :nc], nkv, heads, dh, precision)
            res['planned'] = [FIXED[op]]
        res['outputs'].append(('out', got[0].view(B, n, heads * dh), y, b, False, True))
    elif op == 'gca_pool':
        NB, HW, C = e['NB'], e['HW'], e['C']
        x = G(NB, HW, C)
        wk, bk = G(C, scale=(4.0 if kind == 'edges' else 1.0) / math.sqrt(C)), G(1)
        xp = ptr(guarded(x.reshape(-1, C), e['ldx'], e['xoff']))
        wb, bb = ptr(guarded(wk)), ptr(guarded(bk))
        lg = torch.full((NB * HW + 2 * NB + 2,), NAN, device='cuda')
        out = Out(NB, C)
        outs.append(out)
        got = run(lambda: call('sfb_gca_pool', xp, e['ldx'], NB, HW, C, wb, bb, lg.data_ptr(), out.ptr, S))
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
        xp = ptr(guarded(x, e['ldx'], e['xoff']))
        wb, bb, rb = ptr(guarded(w)), ptr(guarded(bias)), ptr(guarded(r, e['ldr']))
        out = Out(M, O, e['ldy'])
        outs.append(out)
        got = run(lambda: call('sfb_linear_small', xp, e['ldx'], wb, bb, rb, e['ldr'], out.ptr, e['ldy'], M, K, O, e['pre'], e['post'],
                               int(e['round']), S))
        y, b = sf.ref_linear_small(x, w, bias, r, e['pre'], e['post'], e['round'], precision)
        res['outputs'].append(('y', got[0], y, b, False, e['round']))
        res['planned'] = sf.kernel_plan('linear_small', dict(M=M, K=K), sm)['kernels']
    elif op == 'layernorm':
        T, C = e['T'], e['C']
        x = G(T, C) + (100.0 if kind == 'edges' else 0.0)
        g, b_ = G(C), (G(C) if e['b'] else None)
        r = G(T, C) if e['res'] else None
        xp = ptr(guarded(x, e['ldx'], e['xoff']))
        gb, bb, rb = ptr(guarded(g)), ptr(guarded(b_)), ptr(guarded(r, e['ldr']))
        out = Out(T, C, e['ldy'])
        outs.append(out)
        got = run(lambda: call('sfb_layernorm_rows', xp, e['ldx'], gb, bb, rb, e['ldr'], out.ptr, e['ldy'], T, C, int(e['pre_gelu']),
                               int(e['round']), S))
        y, b = sf.ref_layernorm(x, g, b_, r, e['pre_gelu'], e['round'], precision)
        res['outputs'].append(('y', got[0], y, b, False, e['round']))
        res['planned'] = [FIXED[op]]
    elif op == 'gate_mlp_residual':
        NB, HW, C, Hd = e['NB'], e['HW'], e['C'], e['Hd']
        h, r, hid = G(NB, HW, C), G(NB, HW, C), G(NB, Hd)
        w2, b2 = G(C, Hd, scale=1 / math.sqrt(Hd)), G(C)
        hp, rp = ptr(guarded(h.reshape(-1, C), e['ldh'])), ptr(guarded(r.reshape(-1, C), e['ldr']))
        hb, wb, bb = ptr(guarded(hid)), ptr(guarded(w2)), ptr(guarded(b2))
        out = Out(NB * HW, C)
        outs.append(out)
        got = run(lambda: call('sfb_gate_mlp_residual_nhwc', hp, e['ldh'], hb, wb, bb, Hd, rp, e['ldr'], out.ptr, C, NB, HW, C, S))
        y, b = sf.ref_gate_mlp_residual(h, hid, w2, b2, r)
        res['outputs'].append(('out', got[0].view(NB, HW, C), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'gate_residual':
        NB, HW, C = e['NB'], e['HW'], e['C']
        h, r = G(NB, HW, C), G(NB, HW, C)
        gate = G(NB, C) if e['gate'] else None
        hp, rp = ptr(guarded(h.reshape(-1, C), e['ldh'])), ptr(guarded(r.reshape(-1, C), e['ldr']))
        gb = ptr(guarded(gate))
        out = Out(NB * HW, C, e['ldo'])
        outs.append(out)
        got = run(lambda: call('sfb_gate_residual_nhwc', hp, e['ldh'], gb, rp, e['ldr'], out.ptr, e['ldo'], NB, HW, C, S))
        y, b = sf.ref_gate_residual(h, gate, r)
        res['outputs'].append(('out', got[0].view(NB, HW, C), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'softmax_rows':
        R, Cc = e['rows'], e['cols']
        x = G(R, Cc, scale=30.0 if kind == 'edges' else 1.0)
        xp = ptr(guarded(x, e['ldx']))
        out = Out(R, Cc, e['ldy'])
        outs.append(out)
        got = run(lambda: call('sfb_softmax_rows', xp, e['ldx'], out.ptr, e['ldy'], R, Cc, e['scale'], S))
        y, b = sf.ref_softmax_rows(x, e['scale'])
        res['outputs'].append(('y', got[0], y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'time_fourier':
        B, half = e['B'], e['half']
        t, w = G(B, scale=20.0), G(half)
        tb, wb = ptr(guarded(t)), ptr(guarded(w))
        out = Out(1, B * (2 * half + 1))
        outs.append(out)
        got = run(lambda: call('sfb_time_fourier', tb, wb, out.ptr, B, half, S))
        y, b = sf.ref_time_fourier(t, w)
        res['outputs'].append(('four', got[0].view(B, -1), y, b, False, False))
        res['planned'] = [FIXED[op]]
    elif op == 'pixel_shuffle_silu':
        NB, H, W, Co = e['NB'], e['H'], e['W'], e['Co']
        yv = G(NB, H, W, 4 * Co)
        yb = ptr(guarded(yv))
        out = Out(NB * 4 * H * W, Co, e['ldo'])
        outs.append(out)
        got = run(lambda: call('sfb_pixel_shuffle_silu_nhwc', yb, out.ptr, NB, H, W, Co, e['ldo'], S))
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
        xp = ptr(guarded(x.reshape(-1, C), e['ldx']))
        out = Out(NB * 4 * H * W, C)
        outs.append(out)
        got = run(lambda: call('sfb_upsample2x_nhwc', xp, e['ldx'], out.ptr, C, NB, H, W, C, S))
        exact('out', got[0].view(NB, 2 * H, 2 * W, C), sf.upsample2x(x))
    elif op == 'nchw_to_nhwc':
        NB, C, H, W = e['NB'], e['C'], e['H'], e['W']
        x = G(NB, C, H, W)
        xb = ptr(guarded(x))
        out = Out(NB * H * W, C, e['ld'], e['c_off'])
        outs.append(out)
        rnd = e['round'] and precision == 'tf32'
        got = run(lambda: call('sfb_nchw_to_nhwc', xb, out.ptr - 4 * e['c_off'], NB, C, H, W, e['ld'], e['c_off'], int(e['round']), S))
        from sparsefusion_b200 import ops
        ref = x.permute(0, 2, 3, 1).reshape(-1, C)
        exact('out', got[0], ops.round_tf32(ref) if rnd else ref, rnd)
    elif op == 'nhwc_to_nchw':
        NB, C, H, W = e['NB'], e['C'], e['H'], e['W']
        x = G(NB, H, W, C)
        xp = ptr(guarded(x.reshape(-1, C), e['ld']))
        out = Out(1, NB * C * H * W)
        outs.append(out)
        got = run(lambda: call('sfb_nhwc_to_nchw', xp, out.ptr, NB, C, H, W, e['ld'], S))
        exact('out', got[0].view(NB, C, H, W), x.permute(0, 3, 1, 2))
    elif op == 'im2col4':
        NB, H, W, KH, KW, pad = e['NB'], e['H'], e['W'], e['KH'], e['KW'], e['pad']
        k = (4 * KH * KW + 31) // 32 * 32
        x = G(NB, H, W, 4)
        xp = ptr(guarded(x.reshape(-1, 4), e['ldx']))
        out = Out(NB * H * W, k)
        outs.append(out)
        got = run(lambda: call('sfb_im2col4_nhwc', xp, e['ldx'], out.ptr, k, NB, H, W, KH, KW, pad, S))
        exact('out', got[0].view(NB, H, W, k), sf.im2col4(x, KH, KW, pad, k))
    elif op == 'concat2':
        npix = e['NB'] * e['H'] * e['W']
        a, b = G(npix, e['C1']), G(npix, e['C2'])
        ap, bp = ptr(guarded(a, e['lda'])), ptr(guarded(b, e['ldb']))
        out = Out(npix, e['C1'] + e['C2'], e['ldo'])
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
        out = Out(1, n, prefill=x)                     # in place
        outs.append(out)
        got = run(lambda: call('sfb_relu_nhwc', out.ptr, n, S))
        exact('x', got[0], x.clamp_min(0))
    elif op == 'maxpool':
        NB, H, W, C = e['NB'], e['H'], e['W'], e['C']
        x = G(NB, H, W, C)
        if G.kind == 'edges':
            x = torch.round(x).clamp(-1, 2) + 0.0      # ties (+ 0.0 turns -0 into +0: fmaxf may return either zero of a tie)
        xb = ptr(guarded(x))
        out = Out(1, NB * H * W * C // 4)
        outs.append(out)
        got = run(lambda: call('sfb_maxpool2x2_nhwc', xb, out.ptr, NB, H, W, C, S))
        exact('y', got[0].view(NB, H // 2, W // 2, C), sf.maxpool2x2(x))
    elif op == 'maxpool_bwd':
        H, W, C = e['H'], e['W'], e['C']
        x = G(H, W, C).clamp_min(0)
        if G.kind != 'randn':
            x = torch.round(x).clamp(0, 2)             # ties, zero windows
        gy = G(H // 2, W // 2, C)
        xb, gb = ptr(guarded(x)), ptr(guarded(gy))
        out = Out(1, H * W * C)
        outs.append(out)
        got = run(lambda: call('sfb_maxpool2x2_relu_backward_nhwc', xb, gb, out.ptr, H, W, C, S))
        exact('gx', got[0].view(H, W, C), sf.maxpool2x2_relu_backward(x, gy))
    elif op == 'add_relu_mask':
        n = min(e['n'], 1 << 22)
        g, act = G(1, n), G(1, n)
        gh = G(1, n) if e['head'] else None
        out = Out(1, n, prefill=g)                     # in place
        outs.append(out)
        hb, ab = ptr(guarded(gh)), ptr(guarded(act))
        got = run(lambda: call('sfb_add_relu_mask', out.ptr, hb, ab, n, S))
        exact('g', got[0], sf.add_relu_mask(g, gh, act))
    elif op == 'lpips_head':
        HW, C = e['HW'], e['C']
        f0, f1 = G(HW, C), G(HW, C)
        w = G(C, signed=False)
        if G.kind == 'edges':
            f0[::7] = 0                                # r0 = 0
            f1[::5] = 0
        fb0, fb1, wb = ptr(guarded(f0)), ptr(guarded(f1)), ptr(guarded(w))
        val = torch.zeros(1, device='cuda')
        out = Out(HW, C)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_head', fb0, fb1, wb, HW, C, val.data_ptr(), out.ptr, S))
        v, vb, g, gbnd = sf.ref_lpips_head(f0, f1, w)
        res['outputs'].append(('value', val.view(()), v, vb, False, False))
        res['outputs'].append(('g_f0', got[0], g, gbnd, False, False))
    elif op == 'lpips_prep':
        H, W = e['H'], e['W']
        p, t = G.rand(3, H, W), G.rand(3, H, W)
        pb, tb = ptr(guarded(p)), ptr(guarded(t))
        out = Out(1, 2 * H * W * 4)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_prep', pb, tb, H, W, e['normalize'], out.ptr, S))
        y, b = sf.ref_lpips_prep(p, t, e['normalize'])
        res['outputs'].append(('x', got[0].view(2, H, W, 4), y, b, False, False))
    elif op == 'lpips_prep_backward':
        H, W = e['H'], e['W']
        gx = G(H, W, 4)
        gb = ptr(guarded(gx))
        out = Out(1, 3 * H * W)
        outs.append(out)
        got = run(lambda: call('sfb_lpips_prep_backward', gb, H, W, e['normalize'], e['factor'], out.ptr, S))
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
    tracer = Tracer()
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
                    kern = '/'.join(r['names'] or []) if e['op'] not in sf.LPIPS_NAMES.values() else e['op']
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
