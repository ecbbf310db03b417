"""oracle/conv_fp64.py checked on the CPU: ``launch_plan`` against plans derived by hand from the host dispatch of
``sfb_conv2d_nhwc_tf32_ex`` (csrc/conv_wgmma.cu), the bound arithmetic, and sensitivity self-checks.

The self-checks run ``conv_fp64.emulate`` -- the kernel's arithmetic in its k order: tap-major k-steps over 32-channel chunks, the k range
of every split, hi / lo words by bit masking, fp32 partial sums -- and assert that the per-element comparison of tests/test_conv_fp64_gpu.py
accepts the defect-free emulation and rejects each injected defect.  What is seen, stated plainly:
  * a lost k-step of one split, a lost output tile, the bias or the residual added by every split, the whole output in single-pass precision:
    at the UNet's 8x8 3x3 512 -> 512 swap-AB launch, the VAE's 64^2 3x3 128, LPIPS's 64-channel 3x3 and a 51-row linear;
  * swapped stride-2 parity planes (the VAE's 3x3 stride-2 downsample and the UNet's 4x4 stride-2 swap-AB launch), an ignored pad_after
    (the VAE downsample), a one-pixel tap shift in the last column of a partial tile (24^2);
  * a write that spills into the neighbouring channel slice (the bit-identical guard comparison).
What is NOT seen: one k-step computed in single-pass precision inside a 96-k-step chain.  Its error, ~2^-12 of 1/96 of the sum, is below
the 2 gamma(3072) accumulation term of that chain."""
import numpy as np
import pytest
import torch

from oracle import conv_fp64 as cf, insitu

SM = 132      # H100 SXM


# ------------------------------------------------------------------------------------------------ launch plans
def _plan(**kw):
    kw.setdefault('sm', SM)
    return cf.launch_plan(**kw)


def _check(p, **want):
    got = {k: p[k] for k in want}
    assert got == want, (got, want)


def test_plan_swap_64_pixels_unet_8x8():
    # 64 output pixels: swap-AB (:562), tile of 64 pixels (:564), TW = TH = 8 (:565-568); 4 channel tiles of 128 (:594);
    # 132 // 4 = 33 splits, under k_iters / 4 = 36 (:599-601) and over ceil(144 / 96) = 2 (:608)
    p = _plan(NB=1, H=8, W=8, Cin=512, Cout=512, KH=3, KW=3, stride=1, pad=1)
    _check(p, swap=True, tile_pix=64, TW=8, TH=8, TN=1, tiles_m=1, tiles_c=4, k_iters=144, splits=33, bn=64, bn_host=128,
           kernel='conv<64,swap>')
    assert cf.n_chain(p) == 5 * 32 and cf.n_epi(p) == 36


def test_plan_swap_16_pixels_and_the_96_step_floor():
    # 4x4 stage, 3x3 1024 -> 1024: 16 pixels (:564); 8 channel tiles; splits 132 // 8 = 16 (:599), above ceil(288 / 96) = 3 (:608)
    p = _plan(NB=1, H=4, W=4, Cin=1024, Cout=1024, KH=3, KW=3, pad=1)
    _check(p, swap=True, tile_pix=16, TW=4, TH=4, TN=1, tiles_c=8, k_iters=288, splits=16, kernel='conv<16,swap>')
    # an explicit split factor below the floor is raised to ceil(k_iters / 96) (:608-609)
    _check(_plan(NB=1, H=4, W=4, Cin=1024, Cout=1024, KH=3, KW=3, pad=1, splits=1), splits=3)
    # ... but not in single-pass mode (no swap there either: :561-562)
    _check(_plan(NB=1, H=4, W=4, Cin=1024, Cout=1024, KH=3, KW=3, pad=1, splits=1, precision='tf32'), splits=1, swap=False, kernel='conv<128>')


def test_plan_17_rows_swap_32_with_a_batch_tile():
    # 17 linear rows: a 32-pixel tile (:564); Wo = Ho = 1, so TW = TH = 1 and the tile spans TN = 32 images (:565-568);
    # 2 channel tiles: 66 CTAs per tile wanted, but k_iters / 4 = 1 caps it (:600-601)
    p = _plan(NB=17, H=1, W=1, Cin=128, Cout=256, KH=1, KW=1)
    _check(p, swap=True, tile_pix=32, TW=1, TH=1, TN=32, tiles_n=1, k_iters=4, splits=1, kernel='conv<32,swap>')


def test_plan_variant_1_has_no_swap_and_no_presplit():
    # variant 1: v2 is false (:561), so 64 pixels take a normal 128-pixel tile: TW = 8, TH = 16 -> 8 (:567), TN = 2;
    # BN 256 halves to 128 for the small grid (:590) and v2's cap does not apply; pre-split weights are not used (:636)
    p = _plan(NB=1, H=8, W=8, Cin=512, Cout=512, KH=3, KW=3, pad=1, variant=1, presplit=True)
    _check(p, swap=False, tile_pix=128, TW=8, TH=8, TN=2, tiles_m=1, bn=128, tiles_c=4, splits=33, presplit=False, kernel='conv<128>')


def test_plan_single_pass_vae_64():
    # 4096 pixels: TW = 64, TH = 2 (:565-566), 32 M tiles; BN 128 (:588); 32 CTAs -> 4 splits (:599), k_iters / 4 = 9 (:600)
    p = _plan(NB=1, H=64, W=64, Cin=128, Cout=128, KH=3, KW=3, pad=1, precision='tf32')
    _check(p, swap=False, TW=64, TH=2, TN=1, tiles_m=32, bn=128, splits=4, k_iters=36, np=1, kernel='conv<128>')


def test_plan_large_grid_presplit_single_split():
    # VAE 256^2: TW = 128, TH = 1, 512 M tiles >= 132 SMs: one split (:598); pre-split weights are used in normal mode (:636)
    p = _plan(NB=1, H=256, W=256, Cin=128, Cout=128, KH=3, KW=3, pad=1, presplit=True)
    _check(p, TW=128, TH=1, tiles_m=512, splits=1, presplit=True, kernel='conv<128>')


def test_plan_bn_256_only_in_single_pass_or_explicit():
    # v2 caps BN at 128 (:591) ...
    _check(_plan(NB=2, H=128, W=128, Cin=256, Cout=256, KH=3, KW=3, pad=1), bn=128, kernel='conv<128>')
    # ... single pass keeps 256 when the grid has >= 132 CTAs (:590): 256 M tiles
    _check(_plan(NB=2, H=128, W=128, Cin=256, Cout=256, KH=3, KW=3, pad=1, precision='tf32'), tiles_m=256, bn=256, splits=1, kernel='conv<256>')
    # an explicit bn is taken as is and turns swap off (:562, :586); 4 CTAs -> 33, capped by k_iters / 4 = 6 (:600)
    _check(_plan(NB=2, H=16, W=16, Cin=96, Cout=256, KH=3, KW=3, pad=1, bn=256), swap=False, bn=256, tiles_m=4, k_iters=27, splits=6,
           kernel='conv<256>')
    # explicit splits above k_iters are capped (:611)
    _check(_plan(NB=2, H=16, W=16, Cin=96, Cout=256, KH=3, KW=3, pad=1, bn=64, splits=100), splits=27, kernel='conv<64>')


def test_plan_stride_2_pad_after():
    # VAE downsample: F.pad (0, 1, 0, 1) + 3x3 stride 2: Ho = (32 + 0 + 1 - 3) / 2 + 1 = 16 (:551); TW = 16, TH = 8; 2 CTAs -> 66 splits,
    # capped by k_iters / 4 = 9 (:600)
    p = _plan(NB=1, H=32, W=32, Cin=128, Cout=128, KH=3, KW=3, stride=2, pad=0, pad_after=1)
    _check(p, Ho=16, Wo=16, TW=16, TH=8, tiles_m=2, splits=9, kernel='conv<128>')


def test_plan_51_row_film_linear_and_the_k_tail():
    # precompute_time with 51 rows: 64-pixel swap tile spanning 64 "images" of 1x1 (:565-568); 16 channel tiles -> 8 splits = k_iters / 4
    p = _plan(NB=51, H=1, W=1, Cin=1024, Cout=2048, KH=1, KW=1)
    _check(p, swap=True, tile_pix=64, TW=1, TH=1, TN=64, tiles_c=16, k_iters=32, splits=8, kernel='conv<64,swap>')
    # im2col of the 15x15 init conv: K = 900 -> 928 = 29 chunks, the last one a 4-channel tail (:574-577)
    p = _plan(NB=1, H=32, W=32, Cin=900, Cout=256, KH=1, KW=1)
    _check(p, cin_pad=928, k_iters=29, tiles_m=8, bn=128, tiles_c=2, splits=7, kernel='conv<128>')


def test_split_ranges_cover_k_once():
    for k, s in ((144, 33), (29, 7), (27, 27), (5, 1)):
        r = cf.split_ranges(k, s)
        assert r[0][0] == 0 and r[-1][1] == k and all(a[1] == b[0] for a, b in zip(r, r[1:])) and all(e > b for b, e in r)
        assert max(e - b for b, e in r) == -(-k // s)


# ------------------------------------------------------------------------------------------------ bound arithmetic
def test_bound_arithmetic():
    u = 2.0 ** -24
    assert cf.rho_prod('tf32x3') == 32 * u
    assert cf.rho_prod('tf32') == 2.0 ** -10 + 2.0 ** -11 + 2.0 ** -21
    assert cf.rho_prod('tf32', w_rounded=False) == 2.0 ** -9 + 2.0 ** -20
    p = _plan(NB=1, H=8, W=8, Cin=512, Cout=512, KH=3, KW=3, pad=1)
    r_c, r_a = cf.rtols(p, 'tf32x3')
    assert r_c == 32 * u + 2 * cf.gamma(160) and r_a == cf.gamma(36)
    C = torch.tensor([1.0, 2.0, 0.0])
    A = torch.tensor([3.0, 2.0, 5.0])
    assert torch.allclose(cf.bound(p, 'tf32x3', C, A), r_c * C + r_a * A, rtol=0, atol=0)
    # the longest chain the dispatch allows, 96 k-steps, stays below single-pass precision
    p96 = _plan(NB=51, H=1, W=1, Cin=3072, Cout=128, KH=1, KW=1, splits=1)
    assert cf.n_chain(p96) == 3072 and sum(cf.rtols(p96, 'tf32x3')) < 2.0 ** -11


def test_operand_words():
    x = torch.tensor([1.0 + 2.0 ** -10 + 2.0 ** -23 * 0x1FFF, 3.0, -0.7], dtype=torch.float32)
    h = cf.tf32_hi(x)
    assert ((h.view(torch.int32) & 0x1FFF) == 0).all() and ((x - h).abs() < 2.0 ** -10 * x.abs()).all()
    assert (cf.with_low_bits(x, 0x1800).view(torch.int32) & 0x1FFF == 0x1800).all()
    r = cf.tf32_rna(x)
    assert ((r - x).abs() <= 2.0 ** -11 * x.abs()).all()


# ------------------------------------------------------------------------------------------------ sensitivity self-checks
def _operands(NB, H, W, Cin, Cout, KH, one_signed, seed, bias=True, residual=True, stride=1, pad=0, pad_after=None):
    rng = np.random.default_rng(seed)
    f = (lambda a: np.abs(a)) if one_signed else (lambda a: a)
    Ho, Wo = cf.out_size(H, W, KH, KH, stride, pad, pad if pad_after is None else pad_after)
    t = lambda *s: torch.from_numpy(f(rng.standard_normal(s)).astype(np.float32))
    x = t(NB, H, W, Cin)
    w = t(Cout, Cin, KH, KH) / float(np.sqrt(Cin * KH * KH))
    return x, w, (t(Cout) if bias else None), (t(NB, Ho, Wo, Cout) if residual else None)


SHAPES = {
    # name: (NB, H, W, Cin, Cout, K, stride, pad, pad_after, residual)
    'unet_8x8_swap': (1, 8, 8, 512, 512, 3, 1, 1, 1, True),
    'vae_64': (1, 64, 64, 128, 128, 3, 1, 1, 1, True),
    'lpips_64ch': (1, 64, 64, 64, 64, 3, 1, 1, 1, False),
    'film_51_rows': (51, 1, 1, 1024, 512, 1, 1, 0, 0, False),
    'vae_downsample': (1, 32, 32, 128, 128, 3, 2, 0, 1, False),
    'unet_downsample_swap': (1, 16, 16, 64, 128, 4, 2, 1, 1, False),
    'partial_tile_24': (1, 24, 24, 64, 64, 3, 1, 1, 1, False),
}
REPRESENTATIVE = ('unet_8x8_swap', 'vae_64', 'lpips_64ch', 'film_51_rows')


def _case(name, one_signed=True, seed=0):
    NB, H, W, Cin, Cout, K, s, pad, pa, res = SHAPES[name]
    x, w, b, r = _operands(NB, H, W, Cin, Cout, K, one_signed, seed, residual=res, stride=s, pad=pad, pad_after=pa)
    plan = _plan(NB=NB, H=H, W=W, Cin=Cin, Cout=Cout, KH=K, KW=K, stride=s, pad=pad, pad_after=pa)
    y, C, A = cf.conv_ref(x, w, b, r, None, s, pad, pa)
    return dict(x=x, w=w, b=b, r=r, plan=plan, y=y, bnd=cf.bound(plan, 'tf32x3', C, A), stride=s, pad=pad)


@pytest.fixture(scope='module')
def cases():
    return {n: _case(n) for n in SHAPES}


def _emulate(c, defect=None, **kw):
    return cf.emulate(c['x'], c['w'], c['plan'], 'tf32x3', c['b'], c['r'], None, c['stride'], c['pad'], defect=defect, **kw)


def _rejected(c, got):
    return bool(cf.violations(got, c['y'], c['bnd'], 1.0).any())


@pytest.mark.parametrize('name', list(SHAPES))
def test_defect_free_emulation_passes(cases, name):
    c = cases[name]
    got = _emulate(c)
    assert not _rejected(c, got), cf.max_ratio(got, c['bnd'], c['y'])
    assert cf.max_ratio(got, c['bnd'], c['y']) < 0.5
    cr = _case(name, one_signed=False, seed=1)                   # zero-mean operands as well
    assert not _rejected(cr, _emulate(cr))


@pytest.mark.parametrize('name', REPRESENTATIVE)
def test_defects_are_rejected(cases, name):
    c = cases[name]
    p = c['plan']
    assert p['splits'] > 1                                       # every representative launch splits K
    for defect, kw in (('lost_kstep', dict(defect_split=p['splits'] - 1)), ('lost_kstep', dict(defect_split=0)), ('lost_tile', {}),
                       ('bias_every_split', {}), ('single_pass', {})):
        assert _rejected(c, _emulate(c, defect, **kw)), (name, defect, kw)
    if c['r'] is not None:
        assert _rejected(c, _emulate(c, 'residual_every_split')), name


@pytest.mark.parametrize('name', ['vae_downsample', 'unet_downsample_swap'])
def test_swapped_parity_planes_are_rejected(cases, name):
    c = cases[name]
    assert _rejected(c, _emulate(c, 'parity_swap'))


def test_ignored_pad_after_and_tap_shift_are_rejected(cases):
    assert _rejected(cases['vae_downsample'], _emulate(cases['vae_downsample'], 'pad_after_ignored'))
    c = cases['partial_tile_24']
    assert c['plan']['Wo'] % c['plan']['TW'] != 0                # the last column is the edge of a partial tile
    assert _rejected(c, _emulate(c, 'tap_shift'))


def test_slice_spill_is_rejected(cases):
    c = cases['lpips_64ch']
    y = _emulate(c).float()
    before = torch.randn(int(y[..., 0].numel()), 160)
    before[:, ::2] = float('nan')
    good = before.clone()
    good[:, 32:96] = y.reshape(-1, 64)
    assert cf.slice_guard_intact(before, good, 32, 64)
    spill = good.clone()
    spill[-1, 96:100] = y.reshape(-1, 64)[-1, :4]                # one more 4-channel store past the slice
    assert not cf.slice_guard_intact(before, spill, 32, 64)
    red = good.clone()
    red[5, 31] += 1.0                                            # a stray add just before the slice
    assert not cf.slice_guard_intact(before, red, 32, 64)


def test_one_single_pass_chunk_in_a_96_step_chain_is_not_visible():
    """the limit of the comparison, pinned: one k-step of 96 in single-pass precision hides under 2 gamma(3072)"""
    x, w, b, _ = _operands(51, 1, 1, 3072, 128, 1, True, 5, residual=False)
    plan = _plan(NB=51, H=1, W=1, Cin=3072, Cout=128, KH=1, KW=1, splits=1)
    assert plan['splits'] == 1 and plan['k_iters'] == 96
    y, C, A = cf.conv_ref(x, w, b)
    bnd = cf.bound(plan, 'tf32x3', C, A)
    got = cf.emulate(x, w, plan, 'tf32x3', b, defect='one_chunk_single_pass')
    assert not cf.violations(got, y, bnd, 1.0).any()
    assert not cf.violations(cf.emulate(x, w, plan, 'tf32x3', b), y, bnd, 1.0).any()


# ------------------------------------------------------------------------------------------------ catalogue entries of recorded launches
def _conv_rec(x, out, residual=None, bias=True, **scalars):
    """an oracle/insitu record of ops.conv2d_nhwc as the recorder builds it, on CPU tensors"""
    s = dict(cout=out.shape[-1], kh=3, kw=3, stride=1, pad=1, pad_after=1, splits=0, bn=0, dyn=False, accumulate=False, arena=False)
    s.update(scalars)
    t = dict(x=x, w_packed=torch.zeros(s['cout'], 9 * 64), bias=torch.zeros(s['cout']) if bias else None, residual=residual, w_split=None,
             out=out)
    return insitu.Rec('conv2d_nhwc', t, ('out',), s, family='UNet', label='unet.py:forward')


def test_entry_reads_the_channel_slices_of_x_out_and_the_residual():
    x, out, res = torch.zeros(2, 6, 6, 40)[..., 8:24], torch.zeros(2, 6, 6, 64)[..., 16:40], torch.zeros(2, 6, 6, 48)[..., 4:28]
    e = cf.entry(_conv_rec(x, out, res, kh=5, kw=1, stride=2, pad=2, pad_after=0, splits=3, bn=64, dyn=True))
    assert (e['NB'], e['H'], e['W'], e['Cin'], e['ldx'], e['xoff']) == (2, 6, 6, 16, 40, 8)
    assert (e['Cout'], e['ldo'], e['ooff'], e['residual'], e['ldr'], e['roff']) == (24, 64, 16, True, 48, 4)
    assert (e['KH'], e['KW'], e['stride'], e['pad'], e['pad_after'], e['splits'], e['bn'], e['dyn']) == (5, 1, 2, 2, 0, 3, 64, True)
    assert (e['bias'], e['w_split'], e['accumulate'], e['alias']) == (True, False, False, '')
    assert (e['family'], e['label']) == ('UNet', 'unet.py:forward')
    assert cf.entry(_conv_rec(x, out, bias=False))['bias'] is False
    assert cf.entry(insitu.Rec('groupnorm', {}, (), {})) is None


def test_entry_alias_is_the_same_address_not_an_overlap():
    buf = torch.zeros(1, 4, 4, 48)
    out = buf[..., 8:32]
    assert cf.entry(_conv_rec(torch.zeros(1, 4, 4, 16), out, out))['alias'] == 'res=out'
    assert cf.entry(_conv_rec(torch.zeros(1, 4, 4, 16), out, buf[..., 0:24]))['alias'] == ''          # overlapping, other address
    x = torch.zeros(1, 4, 4, 24)
    assert cf.entry(_conv_rec(x, x, x))['alias'] == 'x=out,res=out,x=res'


def test_entry_of_a_reduction_into_an_arena_slice():
    """conv2d_nhwc took its output from the split-K arena: the kernel accumulated into the pre-zeroed slice (``accumulate`` is the flag it
    ran with), and the slice's offset in the arena is not a channel offset"""
    arena = torch.zeros(4096)
    out = arena[64:64 + 4 * 4 * 24].view(1, 4, 4, 24)
    e = cf.entry(_conv_rec(torch.zeros(1, 4, 4, 16), out, accumulate=True, arena=True))
    assert (e['accumulate'], e['ldo'], e['ooff']) == (True, 24, 0)
