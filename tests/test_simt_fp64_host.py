"""oracle/simt_fp64.py checked on the CPU: ``kernel_plan`` against plans derived by hand from the host dispatch in csrc/unet_ops.cu, the bound
arithmetic, and sensitivity self-checks.

The self-checks run the ``emulate_*`` functions -- the kernels' fp32 arithmetic, with the GroupNorm statistics following the stats kernels'
bookkeeping literally -- and assert that the per-element comparison of tests/test_simt_fp64_gpu.py accepts the defect-free emulation and
rejects each injected defect.  What is seen: a lost slab partial, the straddling-group bookkeeping of gn_stats_rows_kernel at C = 3072 and
5120 (the shapes the old row-path gate let through), the wrong group for a channel when 4 does not divide C / G, FiLM without its + 1, a
dropped null key, keys staged in the wrong order, a pixel missing from a split-pool slab, the merge exponent's sign, an off-by-one in
upsample2x, the last instead of the first maximum in the max-pool backward and the LPIPS epsilon added after the reciprocal.
None of these stays below its bound; ``test_missing_pixel_is_seen_even_under_flat_logits`` checks the weakest case: with all logits equal the
pooled value is a plain mean over 16 384 pixels, and one missing pixel still moves it past the bound."""
import math

import pytest
import torch

from oracle import insitu, simt_fp64 as sf

SM = 132      # H100 SXM


def _gn_plan(**g):
    return sf.kernel_plan('groupnorm', g, SM, g.pop('mask', 0x7fffffff))


# ------------------------------------------------------------------------------------------------ launch plans
def test_plan_groupnorm_cluster_items():
    # C 256, 8 groups: Cg / 4 = 8 float4 per pixel; k = 8 CTAs (:1159-1160), ceil(HW / 8) * 8 / 256 float4 per thread (:1161-1162)
    p = _gn_plan(NB=1, HW=1024, C=256, G=8)
    assert (p['path'], p['k'], p['items'], p['kernels']) == ('cluster', 8, 4, ['gn_cluster_kernel<4>'])
    assert _gn_plan(NB=1, HW=1280, C=256, G=8)['kernels'] == ['gn_cluster_kernel<8>']                # items 5
    assert _gn_plan(NB=1, HW=2304, C=256, G=8)['kernels'] == ['gn_cluster_kernel<16>']               # items 9
    assert _gn_plan(NB=1, HW=4096, C=256, G=8)['items'] == 16                                      # exactly 2^20 elements
    # items 17 (C 128, 2 groups, 2176 pixels): the two-launch row path (:1163), C / 4 = 32 divides 256 -> column apply
    p = _gn_plan(NB=1, HW=2176, C=128, G=2)
    assert (p['path'], p['stats'], p['apply']) == ('two-launch', 'gn_stats_rows_kernel', 'gn_apply_cols_kernel')
    # one pixel past 2^20 elements, batch 5, groups narrower than 16 channels, bit 2 cleared: no cluster (:1155)
    assert _gn_plan(NB=1, HW=4097, C=256, G=8)['path'] == 'two-launch'
    assert _gn_plan(NB=5, HW=64, C=256, G=8)['path'] == 'two-launch'
    assert _gn_plan(NB=4, HW=64, C=256, G=8)['path'] == 'cluster'
    assert _gn_plan(NB=1, HW=64, C=128, G=32)['path'] == 'two-launch'
    assert _gn_plan(NB=1, HW=64, C=256, G=8, mask=0x7fffffff & ~4)['path'] == 'two-launch'
    # tiny images: the cluster narrows to a power of two not above HW (:1160)
    assert _gn_plan(NB=2, HW=3, C=256, G=8)['k'] == 2 and _gn_plan(NB=1, HW=1, C=512, G=8)['k'] == 1 and _gn_plan(NB=1, HW=5, C=128, G=8)['k'] == 4


def test_plan_groupnorm_row_gate_and_slabs():
    # VAE 256^2 x 128, 32 groups: rows, rpi = 256 / 32 = 8, S = min(65536 / 16, 264, 256) = 256 (:1177-1182)
    p = _gn_plan(NB=1, HW=65536, C=128, G=32)
    assert (p['rows'], p['S'], p['kernels']) == (True, 256, ['gn_stats_rows_kernel', 'gn_apply_cols_kernel'])
    # C 3072 / 5120: C / 4 a multiple of 256 but the groups (96 / 24 / 80 float4) straddle the 256-column passes -> group-major statistics
    for C, G in ((3072, 4), (3072, 8), (3072, 16), (3072, 32), (5120, 8), (5120, 16), (5120, 32)):
        p = _gn_plan(NB=1, HW=1024, C=C, G=G)
        assert (p['rows'], p['kernels']) == (False, ['gn_stats_kernel', 'gn_apply_kernel']), (C, G)
        assert _gn_plan(NB=1, HW=1024, C=C, G=G, legacy_rows_gate=True)['rows']            # the old gate took them
    assert not _gn_plan(NB=1, HW=1024, C=5120, G=4)['rows']                                # 320-float4 groups are wider than a pass
    # C 2048, 8 groups: 64 float4 per group, 4 whole groups per pass -> rows
    assert _gn_plan(NB=1, HW=1024, C=2048, G=8)['rows']
    # group-major S doubles while G NB S 2 <= 2 SM and HW / (2 S) >= 8 (:1185): 8 groups, 2 images, 64 pixels -> S = 8 (64 / 16 < 8 stops it)
    p = _gn_plan(NB=2, HW=64, C=1536, G=8, mask=0x7fffffff & ~4)
    assert (p['stats'], p['apply'], p['S']) == ('gn_stats_kernel', 'gn_apply_kernel', 8)
    p = _gn_plan(NB=2, HW=64, C=24, G=8)                                                    # Cg = 3
    assert p['stats'] == 'gn_stats_kernel' and p['apply'] == 'gn_apply_kernel'


def test_plan_attention_and_pool_and_linear():
    a = lambda **g: sf.kernel_plan('mq_attention', g, SM)
    assert a(B=1, n=63, heads=2, dh=64, nc=0)['kernel'] == 'smem'                      # nk 64
    p = a(B=1, n=64, heads=2, dh=64, nc=0)                                             # nk 65
    assert p['kernel'] == 'keys' and p['smk'] == (65 * 132 + 8 * 96 + 8 * 64) * 4 and p['qpw'] == 1
    assert a(B=2, n=256, heads=8, dh=64, nc=2)['qpw'] == 4                             # ceil(4096 / 1056)
    assert a(B=1, n=20, heads=2, dh=30, nc=0)['kernel'] == 'plain' and a(B=1, n=12, heads=2, dh=160, nc=0)['kernel'] == 'plain'
    # the keys kernel's 200 KB: at dh 128 the largest nk is 187 (smk 204 720); beyond it the smem kernel's 160 KB is exceeded too
    assert a(B=1, n=186, heads=1, dh=128, nc=0)['smk'] == 204720 and a(B=1, n=187, heads=1, dh=128, nc=0)['smk'] == 205760
    assert a(B=1, n=186, heads=1, dh=128, nc=0)['kernel'] == 'keys' and a(B=1, n=187, heads=1, dh=128, nc=0)['kernel'] == 'plain'
    # the smem kernel's 160 KB is only reachable past the keys kernel's limit, at dh 4: nk 2560 fits (163 840 bytes), 2561 does not
    assert a(B=1, n=2559, heads=1, dh=4, nc=0)['kernel'] == 'smem' and a(B=1, n=2560, heads=1, dh=4, nc=0)['kernel'] == 'plain'
    g = lambda **k: sf.kernel_plan('gca_pool', k, SM)
    assert not g(HW=4095, C=64)['split'] and g(HW=4096, C=64)['split'] and g(HW=4096, C=64)['smem'] == ((516 & ~3) + 1024) * 4
    assert [sf.kernel_plan('linear_small', dict(M=m, K=64))['MT'] for m in (1, 2, 3, 8, 9)] == [2, 2, 8, 8, 8]


# ------------------------------------------------------------------------------------------------ bound arithmetic
def test_bound_arithmetic():
    assert sf.stat_chain(dict(path='cluster', ITEMS=16)) == 64 and sf.stat_chain(dict(path='two-launch')) == 4
    x = torch.tensor([0.0, 1.0, -10.0, 50.0], dtype=torch.float64)
    assert torch.equal(sf.expf_fast_rel(x), torch.tensor([2.0, 3.0, 13.0, 60.0], dtype=torch.float64) * 2.0 ** -23)
    # the GroupNorm bound grows with the (1 + mean^2 / var) cancellation term
    g = torch.Generator().manual_seed(0)
    x0 = torch.randn(1, 256, 64, generator=g)
    plan = dict(path='two-launch')
    ones, zeros = torch.ones(64), torch.zeros(64)
    _, b0 = sf.ref_groupnorm(x0, 8, ones, zeros, None, False, plan)
    _, b1 = sf.ref_groupnorm(x0 + 100, 8, ones, zeros, None, False, plan)
    assert b1.max() > 1e3 * b0.max() * 0.5
    # time_fourier: the argument error is absolute and proportional to |f|
    _, bt = sf.ref_time_fourier(torch.tensor([1.0, 100.0]), torch.tensor([1.0]))
    assert bt[1, 1] > 50 * bt[0, 1]
    # tf32 rounding adds half a TF32 ulp of the value
    y = torch.tensor([1.0], dtype=torch.float64)
    assert sf._tf32(torch.zeros(1, dtype=torch.float64), y, 'tf32') == 2.0 ** -11 and sf._tf32(torch.zeros(1, dtype=torch.float64), y, 'tf32x3') == 0


# ------------------------------------------------------------------------------------------------ sensitivity self-checks
def _rejected(got, ref, bnd):
    return sf.max_ratio(got, ref, bnd) > 1


def _gn_case(NB, HW, C, G, film=True, seed=0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(NB, HW, C, generator=g) + shift
    gam, bet = torch.randn(C, generator=g), torch.randn(C, generator=g)
    fm = torch.randn(NB, 2 * C, generator=g) * 0.5 if film else None
    return x, gam, bet, fm


@pytest.mark.parametrize('shape', [(1, 256, 128, 32), (2, 64, 1536, 8), (1, 1024, 2048, 8), (2, 64, 24, 8), (1, 64, 256, 8)])
def test_groupnorm_emulation_passes_and_defects_are_rejected(shape):
    NB, HW, C, G = shape
    x, gam, bet, fm = _gn_case(NB, HW, C, G)
    plan = _gn_plan(NB=NB, HW=HW, C=C, G=G, mask=0x7fffffff & ~4)
    y, b = sf.ref_groupnorm(x, G, gam, bet, fm, True, plan)
    assert sf.max_ratio(sf.emulate_groupnorm(x, G, gam, bet, fm, True, plan), y, b) < 0.5
    assert _rejected(sf.emulate_groupnorm(x, G, gam, bet, fm, True, plan, defect='lost_slab'), y, b)
    assert _rejected(sf.emulate_groupnorm(x, G, gam, bet, fm, True, plan, defect='film_no_plus1'), y, b)
    if (C // G) % 4:
        assert _rejected(sf.emulate_groupnorm(x, G, gam, bet, fm, True, plan, defect='wrong_group'), y, b)
    # the mean-shifted operands of the 'edges' set stay within the bound
    xs, *_ = _gn_case(NB, HW, C, G, shift=100.0)
    ys, bs = sf.ref_groupnorm(xs, G, gam, bet, fm, True, plan)
    assert sf.max_ratio(sf.emulate_groupnorm(xs, G, gam, bet, fm, True, plan), ys, bs) < 1


@pytest.mark.parametrize('C,G', [(3072, 4), (3072, 8), (3072, 16), (3072, 32), (5120, 8), (5120, 16), (5120, 32)])
def test_straddling_row_bookkeeping_is_rejected(C, G):
    """the row kernel's bookkeeping at the shapes the old gate sent to it: partials that mix two groups' columns, or are never written"""
    x, gam, bet, fm = _gn_case(1, 16, C, G)
    old = _gn_plan(NB=1, HW=16, C=C, G=G, mask=0, legacy_rows_gate=True)
    new = _gn_plan(NB=1, HW=16, C=C, G=G, mask=0)
    assert old['stats'] == 'gn_stats_rows_kernel' and new['stats'] == 'gn_stats_kernel'
    y, b = sf.ref_groupnorm(x, G, gam, bet, fm, True, new)
    assert _rejected(sf.emulate_groupnorm(x, G, gam, bet, fm, True, old), y, b)
    assert sf.max_ratio(sf.emulate_groupnorm(x, G, gam, bet, fm, True, new), y, b) < 0.5


@pytest.mark.parametrize('nc', [0, 2])
def test_attention_emulation_and_key_defects(nc):
    g = torch.Generator().manual_seed(nc)
    B, n, heads, dh = 2, 20, 2, 32
    q, kv, nkv = torch.randn(B, n, heads * dh, generator=g) * 3, torch.randn(B, n, 2 * dh, generator=g), torch.randn(2, dh, generator=g) * 3
    ckv = torch.randn(B, nc, 2 * dh, generator=g) * 3 if nc else None
    plan = sf.kernel_plan('mq_attention', dict(B=B, n=n, heads=heads, dh=dh, nc=nc))
    y, b = sf.ref_mq_attention(q, kv, nkv, ckv, heads, dh, plan)
    assert sf.max_ratio(sf.emulate_mq_attention(q, kv, nkv, ckv, heads, dh), y, b) < 0.5
    assert _rejected(sf.emulate_mq_attention(q, kv, nkv, ckv, heads, dh, 'drop_null'), y, b)
    if nc:
        assert _rejected(sf.emulate_mq_attention(q, kv, nkv, ckv, heads, dh, 'swap_order'), y, b)


def _gca_case(HW, C, seed, flat=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, HW, C, generator=g)
    wk = torch.zeros(C) if flat else torch.randn(C, generator=g) * 2 / math.sqrt(C)
    return x, wk, torch.randn(1, generator=g)


def test_split_pool_emulation_and_defects():
    x, wk, bk = _gca_case(4096, 32, 0)
    plan = sf.kernel_plan('gca_pool', dict(HW=4096, C=32))
    y, b = sf.ref_gca_pool(x, wk, bk, plan)
    assert sf.max_ratio(sf.emulate_gca_pool(x, wk, bk), y, b) < 0.5
    assert _rejected(sf.emulate_gca_pool(x, wk, bk, defect='merge_sign'), y, b)
    # a missing pixel shows when it carries weight: raise the logit of slab 0's last pixel by 10
    x2 = x.clone()
    x2[0, 511] += 10 * wk / (wk @ wk)
    y2, b2 = sf.ref_gca_pool(x2, wk, bk, plan)
    assert sf.max_ratio(sf.emulate_gca_pool(x2, wk, bk), y2, b2) < 1
    assert _rejected(sf.emulate_gca_pool(x2, wk, bk, defect='lost_pixel'), y2, b2)


def test_missing_pixel_is_seen_even_under_flat_logits():
    x, wk, bk = _gca_case(16384, 16, 1, flat=True)
    plan = sf.kernel_plan('gca_pool', dict(HW=16384, C=16))
    y, b = sf.ref_gca_pool(x, wk, bk, plan)
    assert sf.max_ratio(sf.emulate_gca_pool(x, wk, bk), y, b) < 1
    assert _rejected(sf.emulate_gca_pool(x, wk, bk, defect='lost_pixel'), y, b)


def test_exact_op_defects():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 5, 7, 8, generator=g)
    up = sf.upsample2x(x)
    assert torch.equal(up[:, ::2, ::2], x) and torch.equal(up[:, 1::2, 1::2], x)
    assert not torch.equal(sf.upsample2x(x, 'off_by_one'), up)
    a = torch.round(torch.rand(6, 8, 4, generator=g) * 2)                      # ties: values 0, 1, 2
    gy = torch.randn(3, 4, 4, generator=g)
    first, last = sf.maxpool2x2_relu_backward(a, gy), sf.maxpool2x2_relu_backward(a, gy, 'last_max')
    assert not torch.equal(first, last)
    # torch's own max_pool2d backward routes to the first maximum as well
    t = a.permute(2, 0, 1)[None].clone().requires_grad_(True)
    torch.nn.functional.max_pool2d(t, 2).backward(gy.permute(2, 0, 1)[None])
    want = t.grad[0].permute(1, 2, 0) * (a.view(3, 2, 4, 2, 4).amax(dim=(1, 3)).repeat_interleave(2, 0).repeat_interleave(2, 1) > 0)
    assert torch.equal(first, want)
    col = sf.im2col4(torch.randn(1, 3, 4, 4, generator=g), 3, 3, 1, 64)
    assert (col[..., 36:] == 0).all() and (col[0, 0, 0, :4] == 0).all()


def test_lpips_head_bound_and_epsilon():
    g = torch.Generator().manual_seed(4)
    f0, f1, w = torch.randn(64, 32, generator=g), torch.randn(64, 32, generator=g), torch.rand(32, generator=g)
    f0[::7] = 0                                                                 # r0 = 0 rows take the other branch
    v, vb, gr, gb = sf.ref_lpips_head(f0, f1, w)
    ev, eg = sf.emulate_lpips_head(f0, f1, w)
    assert abs(float(ev) - float(v)) <= float(vb) and sf.max_ratio(eg, gr, gb) < 1
    dv, dg = sf.emulate_lpips_head(f0, f1, w, 'eps_outside')
    assert not (abs(float(dv) - float(v)) <= float(vb)) or _rejected(dg, gr, gb)


# ------------------------------------------------------------------------------------------------ catalogue entries of recorded launches
def _call(name, *args):
    """an oracle/insitu ``Call``: positional C ABI arguments bound to the header's parameter names, as the recorder binds them"""
    return insitu.Call(name, dict(zip(insitu.c_params()[name], args)), 'LPIPS')


def test_entry_reads_front_end_slices_strides_and_aliases():
    rows = torch.zeros(1, 4, 4, 96)
    x = rows[..., 16:80]
    film = torch.zeros(1, 192)[:, :128]
    gn = insitu.Rec('groupnorm', dict(x=x, gamma=torch.zeros(64), beta=torch.zeros(64), film=film, out=x), ('out',),
                    dict(groups=8, silu=True, eps=1e-5), family='VAE')
    assert sf.entry(gn) == dict(NB=1, H=4, W=4, C=64, G=8, ldx=96, xoff=16, ldy=96, yoff=16, film=True, ldf=192, act=True, alias='x=out',
                                op='groupnorm', family='VAE', label='VAE')
    xs = torch.zeros(5, 48)[:, 8:48]
    out = torch.zeros(5, 44)[:, :40]
    ln = insitu.Rec('layernorm', dict(x=xs, g=torch.zeros(40), b=None, residual=out, out=out), ('out',),
                    dict(pre_gelu=True, round=False), family='EFT')
    assert sf.entry(ln) == dict(T=5, C=40, ldx=48, xoff=8, ldy=44, b=False, res=True, ldr=44, pre_gelu=True, round=False, alias='res=out',
                                op='layernorm', family='EFT', label='EFT')
    dst = torch.zeros(2, 3, 3, 48)
    nc = insitu.Rec('nchw_to_nhwc', dict(src=torch.zeros(2, 36, 3, 3), out=dst[..., 8:44]), ('out',), dict(round=True, c_off=8), family='UNet')
    assert sf.entry(nc) == dict(NB=2, C=36, H=3, W=3, ld=48, c_off=8, round=True, op='nchw_to_nhwc', family='UNet', label='UNet')
    assert sf.entry(insitu.Rec('conv2d_nhwc', {}, (), {})) is None


def test_entry_reads_lpips_calls_by_parameter_name():
    bwd = sf.entry(_call('sfb_maxpool2x2_relu_backward_nhwc', 11, 12, 13, 6, 10, 5, 0))      # x, gy, gx, H, W, C, stream
    assert bwd == dict(H=6, W=10, C=5, op='maxpool_bwd', family='LPIPS', label='LPIPS')
    assert sf.entry(_call('sfb_add_relu_mask', 11, None, 13, 4096, 0))['n'] == 4096
    assert sf.entry(_call('sfb_add_relu_mask', 11, 12, 13, 4096, 0))['head'] is True
    assert sf.entry(_call('sfb_add_relu_mask', 11, None, 13, 4096, 0))['head'] is False
    prep = sf.entry(_call('sfb_lpips_prep_backward', 11, 64, 32, 1, 0.25, 12, 0))               # gx, H, W, normalize, factor, g_pred
    assert (prep['H'], prep['W'], prep['normalize'], prep['factor']) == (64, 32, 1, 0.25)
    assert sf.entry(_call('sfb_lpips_head', 11, 12, 13, 100, 68, 14, 15, 0))['HW'] == 100
    assert sf.entry(_call('sfb_seq_attention', 11, 12, 3, 4, 5, 0)) is None
