"""Every tensor-core GEMM launch the models make (``conv_gemm_kernel``, csrc/conv_wgmma.cu), replayed per element against fp64.

A module fixture runs the UNet (FULL at 32^2 latents, batch 1 / 2 / 8, precompute_time with 51 rows, precompute_cond +
forward(cond_features=...); SMALL at 128^2), the full VAE encode + decode at 256^2, PerceptualLoss.value_and_grad at 256^2 and the EFT
(encode at 256^2, a feature_cache of three views), all on seeded weights, under oracle/insitu.Catalogue, which records every launch's
geometry and memory layout (``conv_fp64.entry``).  Synthetic entries add what the models do not reach.

Each entry is replayed with fresh operands in its recorded layout, on the default path (3xTF32, variant 2), variant 1 and single-pass TF32,
with three operand sets -- zero-mean ('randn'), one-signed (the bound is then tight relative to |y|) and 'edges' (exact zeros, powers of
two, low mantissa words 0x1FFF and 0x1800, per-channel magnitudes 2^-8 .. 2^8) -- and compared per element with
    |y_gpu - y| <= (rho_prod + 2 gamma(n_chain)) conv(|x|, |w|) + gamma(n_epi) A            (oracle/conv_fp64.py)
Operands sit inside NaN-filled buffers: the channels between a slice and its row stride, and the floats before and after every tensor,
so a tensor map that reads past Cin, Cout, the last image or a slice shows up as NaN; every float of the output buffer outside the slice
(random, NaN in every other one) must stay bit-identical.  The tracer names every replayed launch, and ``launch_plan`` must name the same
kernel.

Out of scope: ordering hazards between launches, which isolated replays cannot see (tests/test_insitu_fp64_gpu.py checks every launch in
place), the LPIPS head and prep kernels, and the NGP weight-gradient GEMMs issued from C (tests/test_ngp_field_fp64_gpu.py)."""
import math
from collections import defaultdict

import pytest
import torch

from _helpers import Out, Tracer, guarded, release
from oracle import conv_fp64 as cf, insitu, model_runs

pytestmark = pytest.mark.gpu

PATHS = {'tf32x3': ('tf32x3', 2), 'tf32x3-v1': ('tf32x3', 1), 'tf32': ('tf32', 2)}
SETS = ('randn', 'one-signed', 'edges')
FIELDS = ('NB', 'H', 'W', 'Cin', 'ldx', 'xoff', 'Cout', 'KH', 'KW', 'stride', 'pad', 'pad_after', 'ldo', 'ooff', 'bias', 'residual', 'ldr',
          'roff', 'accumulate', 'w_split', 'dyn', 'splits', 'bn', 'alias')


# ------------------------------------------------------------------------------------------------ catalogue
def _entry(label, NB, H, W, Cin, Cout, K, stride=1, pad=0, pad_after=None, ldx=None, xoff=0, ldo=None, ooff=0, bias=True, residual=False,
           ldr=None, roff=0, accumulate=False, w_split=False, dyn=False, splits=0, bn=0):
    return dict(NB=NB, H=H, W=W, Cin=Cin, ldx=ldx or Cin, xoff=xoff, Cout=Cout, KH=K, KW=K, stride=stride, pad=pad,
                pad_after=pad if pad_after is None else pad_after, ldo=ldo or Cout, ooff=ooff, bias=bias, residual=residual, ldr=ldr or Cout,
                roff=roff, accumulate=accumulate, w_split=w_split, dyn=dyn, splits=splits, bn=bn, alias='', family='synthetic', label=label, calls=0)


def _synthetic():
    E = [
        # P_total = NB * Ho * Wo across the swap-AB tile sizes and the first normal tile
        _entry('P=1: 3x3 at H = W = 1', 1, 1, 1, 64, 128, 3, pad=1),
        _entry('P=5 linear rows', 5, 1, 1, 96, 64, 1),
        _entry('P=16 with residual', 1, 4, 4, 64, 128, 3, pad=1, residual=True),
        _entry('P=17 linear rows', 17, 1, 1, 128, 256, 1),
        _entry('P=33 rows, pre-split weights ignored by swap-AB', 33, 1, 1, 256, 128, 1, w_split=True),
        _entry('P=48: NB = 3 not a multiple of TN = 4', 3, 4, 4, 128, 256, 3, pad=1),
        _entry('P=64 accumulating into a pre-filled slice', 1, 8, 8, 256, 256, 3, pad=1, ldo=384, ooff=64, accumulate=True),
        _entry('P=65 rows with residual', 65, 1, 1, 512, 384, 1, residual=True),
        # stride 2 on both tile kinds, the VAE's asymmetric padding
        _entry('stride 2 swap-AB, 4x4 pad 1', 1, 16, 16, 64, 128, 4, stride=2, pad=1),
        _entry('stride 2 swap-AB, pad_after 1', 1, 8, 8, 128, 128, 3, stride=2, pad=0, pad_after=1),
        _entry('stride 2 normal, pad_after 1', 2, 16, 16, 64, 128, 3, stride=2, pad=0, pad_after=1, w_split=True),
        # a 15x15 kernel larger than the image
        _entry('15x15 over 8x8 (swap-AB)', 1, 8, 8, 16, 64, 15, pad=7),
        _entry('15x15 over 12x12, input slice', 1, 12, 12, 16, 64, 15, pad=7, ldx=32, xoff=8),
        # partial batch tile in normal mode, K tails with a wider row stride
        _entry('NB = 3, TN = 2', 3, 8, 8, 64, 128, 3, pad=1),
        _entry('Cin 36 in a 48-float row', 1, 16, 16, 36, 64, 3, pad=1, ldx=48, xoff=8),
        _entry('Cin 4 in an 8-float row, 7x7', 2, 8, 8, 4, 128, 7, pad=3, ldx=8, xoff=4),
        # Cout tails
        _entry('Cout 4', 1, 32, 32, 64, 4, 3, pad=1),
        _entry('Cout 12 (swap-AB)', 1, 4, 4, 64, 12, 3, pad=1),
        _entry('Cout 12 accumulating into a slice', 2, 8, 8, 64, 12, 3, pad=1, ldo=16, ooff=4, accumulate=True),
        # channel slices on every operand
        _entry('slices: x, residual and out', 2, 8, 8, 64, 64, 3, pad=1, ldx=160, xoff=32, residual=True, ldr=96, roff=32, ldo=192, ooff=64),
        # an activation as the K-major operand
        _entry('dynamic K-major operand', 96, 1, 1, 64, 128, 1, dyn=True, bias=False),
    ]
    for bn in (32, 64, 128, 256):
        for splits in (1, 3, 27):            # 27 = k_iters: one k-step per split
            E.append(_entry(f'bn {bn} splits {splits}', 2, 16, 16, 96, 256, 3, pad=1, bn=bn, splits=splits, w_split=bn in (64, 256)))
    return E


@pytest.fixture(scope='module')
def catalogue():
    cat = insitu.Catalogue(cf.entry)
    model_runs.record_models(cat)
    entries = list(cat.entries.values()) + _synthetic()
    fam = defaultdict(int)
    for e in entries:
        fam[e['family']] += 1
    print('\nconv catalogue: ' + ', '.join(f'{k} {v}' for k, v in fam.items()))
    return entries


# ------------------------------------------------------------------------------------------------ operands
def _edge_words(t, g):
    """exact zeros, powers of two (lo = 0), low words 0x1FFF (the largest lo) and 0x1800 (lo = 3/4 of a tf32 ulp), one in four each"""
    cat = torch.randint(0, 4, t.shape, device=t.device, generator=g)
    i = t.contiguous().view(torch.int32)
    pow2 = i & -8388608
    hi = i & -8192
    out = torch.where(cat == 0, torch.zeros_like(i), torch.where(cat == 1, pow2, torch.where(cat == 2, hi | 0x1FFF, hi | 0x1800)))
    return out.view(torch.float32)


def _operands(e, kind, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    Ho, Wo = cf.out_size(e['H'], e['W'], e['KH'], e['KW'], e['stride'], e['pad'], e['pad_after'])
    rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
    x = rn(e['NB'], e['H'], e['W'], e['Cin'])
    w = rn(e['Cout'], e['Cin'], e['KH'], e['KW']) / math.sqrt(e['Cin'] * e['KH'] * e['KW'])
    b = rn(e['Cout']) if e['bias'] else None
    r = rn(e['NB'], Ho, Wo, e['Cout']) if e['residual'] else None
    pre = rn(e['NB'], Ho, Wo, e['Cout']) if e['accumulate'] else None
    if kind == 'one-signed':
        x, w = x.abs(), w.abs()
        b, r, pre = [None if t is None else t.abs() for t in (b, r, pre)]
    elif kind == 'edges':
        x = _edge_words(x, g) * torch.exp2(torch.randint(-8, 9, (e['Cin'],), device='cuda', generator=g).float())
        w = _edge_words(w, g) * torch.exp2(torch.randint(-8, 9, (e['Cout'], 1, 1, 1), device='cuda', generator=g).float())
        b, r, pre = [None if t is None else _edge_words(t, g) for t in (b, r, pre)]
    elif kind == 'control':
        # single-pass negative control: x = 2^k (1 + 0x1800 2^-23), so its tf32 read loses 3/4 of an ulp (truncation) or gains 1/4 (rounding),
        # >= 2^-12 relative either way and one-signed; the weights are exact tf32 words, the epilogue terms zero
        x = torch.exp2(torch.randint(-2, 3, x.shape, device='cuda', generator=g).float())
        x = cf.with_low_bits(x, 0x1800)
        w = cf.tf32_hi(w.abs())
        b, r, pre = [None if t is None else torch.zeros_like(t) for t in (b, r, pre)]
    return x, w, b, r, pre


# ------------------------------------------------------------------------------------------------ replay
def _launch(e, path, ops_in, tracer, sm):
    """one replay of entry e on path with operands (x, w, b, r, pre); returns (got NHWC fp32, guard ok, traced names, plan)"""
    from sparsefusion_b200 import _lib as lib, ops
    precision, variant = PATHS[path]
    x, w, b, r, pre = ops_in
    NB, H, W, Cin, Cout = e['NB'], e['H'], e['W'], e['Cin'], e['Cout']
    Ho, Wo = cf.out_size(H, W, e['KH'], e['KW'], e['stride'], e['pad'], e['pad_after'])
    ops.set_precision(precision)
    lib.call('sfb_conv_set_variant', variant)
    release()
    try:
        if e['dyn']:
            wp = w.reshape(Cout, -1).contiguous()          # an activation: used as it is, in every mode
        else:
            wp = ops.pack_conv_weight(w)                   # rounded to tf32 in single-pass mode
        wpv = guarded(wp)
        spv = guarded(ops.split_packed_weight(wp)) if e['w_split'] and precision == 'tf32x3' else None
        xv = guarded(x, e['ldx'], e['xoff'])
        out = Out(NB * Ho * Wo, Cout, e['ldo'], e['ooff'], prefill=pre)
        ov = out.slot.view(NB, Ho, Wo, Cout)
        rv = None
        if r is not None:
            rv = ov if 'res=out' in e['alias'] else guarded(r, e['ldr'], e['roff'])
        bv = guarded(b)
        plan = cf.launch_plan(NB, H, W, Cin, Cout, e['KH'], e['KW'], e['stride'], e['pad'], e['pad_after'], e['splits'], e['bn'], precision,
                              variant, spv is not None, sm)
        names = tracer.run(lambda: ops.conv2d_nhwc(xv, wpv, Cout, e['KH'], e['KW'], e['stride'], e['pad'], bias=bv, residual=rv, out=ov,
                                                   accumulate=e['accumulate'], splits=e['splits'], bn=e['bn'], pad_after=e['pad_after'],
                                                   w_split=spv, dynamic_weights=e['dyn']))
        return out.value().view(NB, Ho, Wo, Cout), out.guard_ok(), names, plan
    finally:
        ops.set_precision('tf32x3')
        lib.call('sfb_conv_set_variant', 2)


def _features(e, plan):
    f = {'splits>1' if plan['splits'] > 1 else 'splits=1'}
    if e['stride'] == 2:
        f.add('stride2-swap' if plan['swap'] else 'stride2-normal')
    if e['pad_after'] != e['pad']:
        f.add('pad_after')
    if plan['np'] == 3:
        f.add('presplit' if plan['presplit'] else 'in-kernel split')
    if e['dyn']:
        f.add('dyn')
    if e['accumulate']:
        f.add('accumulate into a pre-filled slice')
    return f


def _key(e):
    return f"{e['family']} {e['label']} " + ' '.join(f'{k}={e[k]}' for k in FIELDS if e[k] not in (0, False, ''))


@pytest.fixture(scope='module')
def replays(catalogue):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    tracer = Tracer()
    res = dict(fail=[], names=defaultdict(set), features=defaultdict(set), table={}, control=[])
    table = defaultdict(lambda: [0, 0.0, 0.0])
    for n, e in enumerate(catalogue):
        for si, kind in enumerate(SETS):
            opsn = _operands(e, kind, 1000 * n + si)
            y, C, A = cf.conv_ref(opsn[0], opsn[1], opsn[2], opsn[3], opsn[4], e['stride'], e['pad'], e['pad_after'])
            for path, (precision, _) in PATHS.items():
                got, guard_ok, names, plan = _launch(e, path, opsn, tracer, sm)
                bnd = cf.bound(plan, precision, C, A, w_rounded=not e['dyn'])
                ratio = cf.max_ratio(got, bnd, y)
                t = table[(e['family'], path)]
                if si == 0:
                    t[0] += 1
                t[1] = max(t[1], ratio)
                msg = []
                if ratio > 1:
                    msg.append(f'err/bound {ratio:.3g}')
                if kind == 'randn':
                    rel = ((got.double() - y).norm() / y.norm()).item()
                    t[2] = max(t[2], rel)
                    if precision == 'tf32x3' and rel > 2e-5:
                        msg.append(f'rel L2 {rel:.3g}')
                if not guard_ok:
                    msg.append('output channels outside the slice changed')
                if names != [plan['kernel']]:
                    msg.append(f"traced {names}, planned {plan['kernel']}")
                if msg:
                    res['fail'].append(f"{_key(e)} [{path} {kind}]: " + '; '.join(msg))
                res['names'][path].add(plan['kernel'] if names == [plan['kernel']] else '?')
                res['features'][path] |= _features(e, plan)
            del y, C, A, opsn
        # single-pass negative control: entries whose 3xTF32 bound on the single-pass launch is below 2^-13 relative
        plan_sp = cf.launch_plan(e['NB'], e['H'], e['W'], e['Cin'], e['Cout'], e['KH'], e['KW'], e['stride'], e['pad'], e['pad_after'], e['splits'],
                                 e['bn'], 'tf32', 2, False, sm)
        if sum(cf.rtols(plan_sp, 'tf32x3')) < 2.0 ** -13:
            opsn = _operands(e, 'control', 7 + n)
            y, C, A = cf.conv_ref(opsn[0], opsn[1], opsn[2], opsn[3], opsn[4], e['stride'], e['pad'], e['pad_after'])
            got, guard_ok, names, plan = _launch(e, 'tf32', opsn, tracer, sm)
            assert plan == plan_sp
            bnd3 = cf.bound(plan, 'tf32x3', C, A)
            bad = cf.violations(got, y, bnd3, 1.0)
            live = C > 0
            res['control'].append((_key(e), int(bad.sum()), int(live.sum()), cf.max_ratio(got, bnd3, y)))
            # the single-pass result is still within its own bound
            if cf.max_ratio(got, cf.bound(plan, 'tf32', C, A, w_rounded=not e['dyn']), y) > 1:
                res['fail'].append(f'{_key(e)} [tf32 control]: outside the single-pass bound')
    res['table'] = dict(table)
    print('\nfamily      path        entries  max err/bound  max rel L2 (randn)')
    for (fam, path), (cnt, ratio, rel) in sorted(res['table'].items()):
        print(f'{fam:11s} {path:11s} {cnt:7d}  {ratio:13.3f}  {rel:18.2e}')
    if res['fail']:
        print('\n'.join(res['fail'][:40]))
    return res


# ------------------------------------------------------------------------------------------------ tests
def test_catalogue_holds_the_launches_the_issue_names(catalogue):
    by = defaultdict(list)
    for e in catalogue:
        by[e['family']].append(e)
    assert all(len(by[f]) > 0 for f in ('UNet', 'VAE', 'LPIPS', 'EFT'))
    assert not any(e['alias'] and e['alias'] != 'res=out' for e in catalogue), [_key(e) for e in catalogue if e['alias']]
    assert sum(e['dyn'] for e in by['VAE']) >= 3                                            # q k^T, W_v h^T, P v
    assert any(e['Cin'] == 928 and e['KH'] == 1 and e['accumulate'] for e in by['UNet'])   # im2col of the 15x15 init conv, K 900 -> 928
    assert any(e['ldo'] == 256 and e['Cout'] < 256 and e['ooff'] > 0 for e in by['UNet'])  # init-conv shares into channel slices
    assert any(e['NB'] == 51 and e['H'] == 1 for e in by['UNet'])                          # precompute_time's FiLM linear
    assert any(e['Cout'] == 4 and e['H'] == 256 for e in by['LPIPS'])                      # the first layer's data gradient
    assert any(e['KH'] == 7 and e['stride'] == 2 for e in by['EFT'])                       # ResNet-18 conv1
    assert any(e['H'] == 1 and e['Cin'] % 32 for e in by['EFT'])                           # transformer linears with a K tail
    assert any(e['pad_after'] != e['pad'] for e in by['VAE'])


def test_every_replay_is_within_the_fp64_bound(replays):
    assert not replays['fail'], f"{len(replays['fail'])} failures:\n" + '\n'.join(replays['fail'][:40])


def test_replays_reach_every_kernel_path(replays):
    swap = {'conv<16,swap>', 'conv<32,swap>', 'conv<64,swap>'}
    normal = {'conv<32>', 'conv<64>', 'conv<128>', 'conv<256>'}
    assert replays['names']['tf32x3'] == swap | normal
    assert replays['names']['tf32x3-v1'] == normal and replays['names']['tf32'] == normal
    assert replays['features']['tf32x3'] >= {'stride2-swap', 'stride2-normal', 'pad_after', 'presplit', 'in-kernel split', 'dyn',
                                             'accumulate into a pre-filled slice', 'splits>1', 'splits=1'}


def test_single_pass_negative_control_violates_the_tf32x3_bound(replays):
    ctl = replays['control']
    print(f'\nsingle-pass negative control: {len(ctl)} entries; fewest violating elements '
          f'{min((c[1] / max(c[2], 1) for c in ctl), default=0):.3f} of the live ones; smallest max err/bound {min((c[3] for c in ctl), default=0):.2f}')
    assert len(ctl) >= 20
    missed = [c for c in ctl if c[1] == 0]
    assert not missed, missed[:10]
