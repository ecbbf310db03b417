"""The in-situ checker of oracle/insitu.py on the CPU: it accepts correct records and rejects each single defect an ordering hazard leaves
behind; and the programmatic-dependent-launch contract of the kernel sources.

PDL contract: every kernel launched through SFB_LAUNCH / SFB_LAUNCH_CLUSTER / launch_pdl starts with ``pdl_sync()``.  A kernel that could exit
before its griddepcontrol.wait would let its own dependent's wait return before the kernel ahead of it finished, and the chain would
lose its transitivity.  ``conv_gemm_kernel`` is the one exception: ahead of its wait it reads only the bias, the tensor maps and the first
weight stages, and with ``w_dynamic`` it waits before the weights too."""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import insitu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'sparsefusion_b200', 'csrc')


# ------------------------------------------------------------------------------------------------ synthetic records
def _pack(w):
    cout, cin, kh, kw = w.shape
    cp = (cin + 31) // 32 * 32
    p = torch.zeros(cout, kh, kw, cp)
    p[..., :cin] = w.permute(0, 2, 3, 1)
    return p.reshape(cout, -1)


def _conv_fp32(x, w, bias=None, prefill=None):
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None if bias is None else bias.double(), padding=1).permute(0, 2, 3, 1)
    if prefill is not None:
        y = y + prefill.double()
    return y.float().contiguous()


def _gemm(seed=0, nb=2, bias=True, arena=False, prefill=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(nb, 6, 6, 40, generator=g)
    w = torch.randn(24, 40, 3, 3, generator=g) / 19
    b = torch.randn(24, generator=g) if bias else None
    pre = torch.randn(nb, 6, 6, 24, generator=g) if prefill else None
    out = _conv_fp32(x, w, b, pre)
    t = dict(x=x, w_packed=_pack(w), bias=b, residual=None, w_split=None, out=out)
    if pre is not None:
        t['prefill'] = pre
    s = dict(cout=24, kh=3, kw=3, stride=1, pad=1, pad_after=1, splits=0, bn=0, dyn=False, accumulate=arena or prefill, precision='tf32x3',
             arena=arena)
    return insitu.Rec('conv2d_nhwc', t, ('out',), s, label='synthetic')


def _groupnorm(seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 4, 64, generator=g)
    gam, bet = torch.randn(64, generator=g), torch.randn(64, generator=g)
    film = torch.randn(2, 128, generator=g) * 0.5
    xd = x.double().reshape(2, 16, 8, 8)
    mu, var = xd.mean(dim=(1, 3), keepdim=True), xd.var(dim=(1, 3), unbiased=False, keepdim=True)
    z = ((xd - mu) / torch.sqrt(var + 1e-5)).reshape(2, 4, 4, 64) * gam.double() + bet.double()
    z = z * (film.double()[:, None, None, :64] + 1) + film.double()[:, None, None, 64:]
    out = F.silu(z).float()
    return insitu.Rec('groupnorm', dict(x=x, gamma=gam, beta=bet, film=film, out=out), ('out',),
                      dict(groups=8, silu=True, eps=1e-5, precision='tf32x3'), label='synthetic')


def _softmax(seed=2):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(5, 33, generator=g)
    out = torch.softmax(x.double() * 0.25, -1).float()
    return insitu.Rec('softmax_rows', dict(x=x, out=out), ('out',), dict(scale=0.25, precision='tf32x3'), label='synthetic')


def _stale(rec, name, seed=9):
    """one element of operand ``name`` holds another replay's value: the record read it, the final contents differ"""
    t = rec.t[name].clone()
    g = torch.Generator().manual_seed(seed)
    other = torch.randn(t.shape, generator=g)
    i = tuple(d // 2 for d in t.shape)
    t[i] = other[i] + (1.0 if abs(other[i] - t[i]) < 0.5 else 0.0)
    rec.t[name] = t
    return rec


@pytest.mark.parametrize('make', [_gemm, lambda: _gemm(prefill=True), lambda: _gemm(arena=True, bias=False), _groupnorm, _softmax])
def test_checker_accepts_correct_records(make):
    rep = insitu.check(make())
    assert rep.ok and rep.ratio <= 1, rep


@pytest.mark.parametrize('make,name', [(_gemm, 'x'), (_gemm, 'w_packed'), (_gemm, 'bias'), (lambda: _gemm(prefill=True), 'prefill'),
                                       (_groupnorm, 'x'), (_groupnorm, 'film'), (_softmax, 'x')])
def test_checker_rejects_an_operand_element_from_another_replay(make, name):
    rep = insitu.check(_stale(make(), name))
    assert not rep.ok and rep.n_bad >= 1 and rep.first is not None, rep


@pytest.mark.parametrize('make', [_gemm, _groupnorm, _softmax])
def test_checker_rejects_a_nan_left_in_an_output(make):
    r = make()
    r.t['out'].view(-1)[7] = float('nan')
    rep = insitu.check(r)
    assert rep.n_nonfinite == 1 and rep.n_bad == 1 and math.isinf(rep.ratio), rep


def test_checker_rejects_a_split_k_output_on_an_arena_that_was_not_zeroed():
    r = _gemm(arena=True, bias=False)
    r.t['out'] = r.t['out'] * 2                 # accumulated onto the previous replay's identical result
    rep = insitu.check(r)
    assert not rep.ok and rep.n_bad > rep.numel // 2, rep


def test_checker_rejects_a_guided_pair_with_its_halves_swapped():
    r = _gemm(nb=2)
    r.t['out'] = r.t['out'].flip(0).contiguous()     # [cond, null] rows written as [null, cond]
    rep = insitu.check(r)
    assert not rep.ok and rep.n_bad > rep.numel // 2, rep


def test_provenance_accepts_prepared_operands_and_rejects_operands_written_in_the_evaluation():
    prod = _groupnorm()
    plan_gemm = _gemm()
    plans = insitu.plan_storages(plan_gemm.t['w_packed'], plan_gemm.t['bias'])
    assert insitu.provenance([prod, plan_gemm], plans) == []
    # the bias is an activation written by an earlier record: read before griddepcontrol.wait
    bad_bias = _gemm()
    bad_bias.t['bias'] = bad_bias.orig['bias'] = prod.orig['out'].view(-1)[:24]
    bad_bias.t['w_packed'] = bad_bias.orig['w_packed'] = plan_gemm.orig['w_packed']
    msg = insitu.provenance([prod, bad_bias], plans)
    assert len(msg) == 1 and 'bias' in msg[0], msg
    # a weight an earlier record wrote, without dynamic_weights
    act_w = _gemm()
    act_w.t['bias'] = act_w.orig['bias'] = plan_gemm.orig['bias']
    w_act = torch.zeros(24 * 9 * 32)
    act_w.t['w_packed'] = act_w.orig['w_packed'] = w_act.view(24, -1)
    prod2 = insitu.Rec('softmax_rows', dict(x=torch.zeros(1, 4), out=w_act.view(-1, 8)), ('out',), dict(scale=1.0))
    msg = insitu.provenance([prod2, act_w], plans)
    assert len(msg) == 1 and 'w_packed' in msg[0], msg
    act_w.s['dyn'] = True                        # ... is accepted with the switch set
    assert insitu.provenance([prod2, act_w], plans) == []
    # the switch set on a prepared weight: it is not needed there, and the catalogue would list the launch wrongly
    plan_dyn = _gemm()
    plan_dyn.t = dict(plan_gemm.t)
    plan_dyn.orig = dict(plan_gemm.orig)
    plan_dyn.s['dyn'] = True
    msg = insitu.provenance([prod, plan_dyn], plans)
    assert len(msg) == 1 and 'dynamic_weights' in msg[0], msg


def _plms(seed=3, rows=2, L=48, nulls=(False, False, True), cfg=False):
    from oracle import step_fp64 as st
    g = torch.Generator().manual_seed(seed)
    rn = lambda: torch.randn(rows, L, generator=g)
    x, z = rn(), rn()
    e = [rn()] + [None if n else rn() for n in nulls]
    en = rn() if cfg else None
    coefs = (23 / 12, -16 / 12, 5 / 12, 0.0)
    sc = torch.tensor([[0.9, 0.43, 0.95, 0.3, 0.1]] * rows)
    e0 = st.cfg_eps(e[0], en, 3.0) if cfg else e[0]
    out = st.emulate_plms(x, [e0] + e[1:], coefs, sc, z, 1.0)['x_prev']
    t = dict(x=x, e0=e[0], e1=e[1], e2=e[2], e3=e[3], noise=z, scalars=sc, out=out)
    if cfg:
        t.update(e_null=en, e_out=e0)
    return insitu.Rec('plms_update_rows_cfg' if cfg else 'plms_update_rows', t, ('out', 'e_out') if cfg else ('out',),
                      dict(coefs=coefs, clip=1.0, cond_scale=3.0, rows=rows, row_len=L))


@pytest.mark.parametrize('cfg', [False, True])
def test_checker_accepts_and_rejects_sampler_updates(cfg):
    assert insitu.check(_plms(cfg=cfg)).ok
    assert not insitu.check(_stale(_plms(cfg=cfg), 'e1')).ok
    assert not insitu.check(_stale(_plms(cfg=cfg), 'e_null' if cfg else 'e0')).ok
    if cfg:
        r = _plms(cfg=True)
        r.t['e_out'] = r.t['e_out'].clone()
        r.t['e_out'][1, 3] = float(torch.nextafter(r.t['e_out'][1, 3], torch.tensor(9.0)))     # one ulp off the fp32 guided eps
        assert not insitu.check(r).ok


def _history_run(guided, batch=(3, 3, 3, 3, 2, 2, 1), L=10, seed=4):
    """a replay log and the update records p_sample's assignment gives them"""
    g = torch.Generator().manual_seed(seed)
    outs = [torch.randn((2 if guided else 1) * b, L, generator=g) for b in batch]
    exp = insitu.plms_expected_eps(outs, list(batch), guided, 3.0)
    recs = [insitu.Rec('plms_update_rows_cfg' if guided else 'plms_update_rows', {k: None if v is None else v.clone() for k, v in e.items()},
                       ('out',), {}) for e in exp]
    return outs, exp, recs


@pytest.mark.parametrize('guided', [False, True])
def test_history_check_rejects_eps_from_the_wrong_round_or_row(guided):
    outs, exp, recs = _history_run(guided)
    assert insitu.plms_history_mismatches(recs, exp) == []
    # the assignment itself: round 1 pairs round 0's eps with its own, round 4 reads rounds 3, 2 and 0, newest first
    E = [insitu.st.cfg_eps(o[:len(o) // 2], o[len(o) // 2:], 3.0) if guided else o for o in outs]
    if guided:
        assert torch.equal(exp[1]['e1'], E[0]) and torch.equal(exp[1]['e0'], outs[1][:3])
    else:
        assert torch.equal(exp[1]['e0'], E[0]) and torch.equal(exp[1]['e1'], E[1])
    assert all(torch.equal(exp[4][k], E[i][:2]) for k, i in (('e1', 3), ('e2', 2), ('e3', 0)))
    # the wrong round: round 4's oldest history slot holds round 1's eps instead of round 0's
    _, _, bad = _history_run(guided)
    bad[4].t['e3'] = E[1][:2].clone()
    assert any('round 4: e3' in m for m in insitu.plms_history_mismatches(bad, exp))
    # the wrong row: round 3's newest history rows swapped
    _, _, bad = _history_run(guided)
    bad[3].t['e1'] = bad[3].t['e1'].flip(0).contiguous()
    assert any('round 3: e1' in m for m in insitu.plms_history_mismatches(bad, exp))
    # a history pointer left NULL
    _, _, bad = _history_run(guided)
    bad[5].t['e2'] = None
    assert any('round 5: e2' in m for m in insitu.plms_history_mismatches(bad, exp))


def test_overlap_of_channel_slices_and_views():
    buf = torch.zeros(2, 3, 3, 16)
    a, b, c = buf[..., 0:4], buf[..., 4:12], buf[..., 8:16]
    assert not insitu.overlaps(a, b) and insitu.overlaps(b, c) and insitu.overlaps(a, buf) and insitu.overlaps(buf, buf[1])
    assert not insitu.overlaps(buf[0], buf[1]) and not insitu.overlaps(buf, torch.zeros(2))


def test_poison_touches_exactly_the_output_view():
    buf = torch.arange(2 * 3 * 3 * 16, dtype=torch.float32).view(2, 3, 3, 16)
    before = buf.clone()
    r = insitu.Rec('nchw_to_nhwc', dict(src=torch.zeros(2, 5, 3, 3), out=buf[..., 4:9]), ('out',), dict(round=False))
    insitu.poison([r])
    inside = torch.zeros_like(buf, dtype=torch.bool)
    inside[..., 4:9] = True
    assert torch.isnan(buf[inside]).all() and torch.equal(buf[~inside], before[~inside])


# ------------------------------------------------------------------------------------------------ PDL source contract
def _strip_comments(src):
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return re.sub(r'//[^\n]*', '', src)


def _pdl_launched():
    """{kernel name: file} of every kernel launched through SFB_LAUNCH, SFB_LAUNCH_CLUSTER or launch_pdl / launch_pdl_cluster"""
    out = {}
    for fn in sorted(os.listdir(CSRC)):
        if not fn.endswith('.cu'):
            continue
        src = _strip_comments(open(os.path.join(CSRC, fn)).read())
        for m in re.finditer(r'\b(?:SFB_LAUNCH_CLUSTER|SFB_LAUNCH|launch_pdl_cluster|launch_pdl)\s*\(\s*(?:sfb::)?([A-Za-z_]\w*)', src):
            if m.group(1) not in ('kernel',):             # the helpers' own parameter
                out[m.group(1)] = fn
    return out


def _body(src, name):
    """source of the first __global__ definition of ``name``, from its opening brace"""
    m = re.search(r'__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?' + re.escape(name) + r'\s*\(', src)
    assert m, name
    i = m.end()
    depth = 1
    while depth:                                  # the parameter list
        depth += {'(': 1, ')': -1}.get(src[i], 0)
        i += 1
    j = src.index('{', i)
    depth, k = 1, j + 1
    while depth:
        depth += {'{': 1, '}': -1}.get(src[k], 0)
        k += 1
    return src[j + 1:k - 1]


def test_every_pdl_launched_kernel_waits_at_entry():
    launched = _pdl_launched()
    assert len(launched) >= 25 and 'conv_gemm_kernel' in launched and 'gn_apply_kernel' in launched, sorted(launched)
    bad = []
    for name, fn in sorted(launched.items()):
        if name == 'conv_gemm_kernel':
            continue
        body = _body(_strip_comments(open(os.path.join(CSRC, fn)).read()), name)
        if not body.lstrip().startswith('pdl_sync();'):
            bad.append(f'{fn}:{name} starts with {body.strip()[:60]!r}')
    assert not bad, bad


def test_conv_gemm_kernel_reads_only_bias_tensor_maps_and_weight_stages_before_its_wait():
    src = _strip_comments(open(os.path.join(CSRC, 'conv_wgmma.cu')).read())
    body = _body(src, 'conv_gemm_kernel')
    waits = [m.start() for m in re.finditer(r'pdl_wait\(\);', body)]
    first = next(w for w in waits if not body[:w].rstrip().endswith('if (p.w_dynamic)'))
    dyn = body.index('if (p.w_dynamic) pdl_wait();')
    pre = body[:first]
    # arrays indexed through the parameter block before the wait: the bias (global memory) and tmA (tensor maps in the parameter block)
    assert set(re.findall(r'\bp\.(\w+)\s*\[', pre)) == {'bias', 'tmA'}, set(re.findall(r'\bp\.(\w+)\s*\[', pre))
    assert set(re.findall(r'prefetch_tensormap\(&p\.(\w+)', pre)) <= {'tmA', 'tmB'}
    # TMA loads issued before the wait: load_weights(it) only, and only after the w_dynamic wait
    calls = [(m.start(), m.group(1)) for m in re.finditer(r'\b(load_weights|load_acts)\(it\);', pre)]
    assert calls and all(c == 'load_weights' for _, c in calls), calls
    assert all(pos > dyn for pos, _ in calls)
    assert 'tma_load' not in re.sub(r'auto load_(?:weights|acts) = \[&\]\(int it\) \{.*?\n\s*\};', '', pre, flags=re.S)
    # every thread of the epilogue waits before its residual reads and output writes
    assert re.search(r'pdl_wait\(\);\s*(?:\n[^\n]*)*?\bp\.residual', body[first + 1:]) or 'residual' not in body[first + 1:]


# ------------------------------------------------------------------------------------------------ replay catalogues
def test_catalogue_orders_records_and_calls_as_issued_and_counts_repeats():
    """the replay tests seed each entry's operands by its position, so calls interleave with the front-end records in issue order"""
    from oracle import simt_fp64 as sf
    sm = lambda cols: insitu.Rec('softmax_rows', dict(x=torch.zeros(3, cols), out=torch.zeros(3, cols)), ('out',), dict(scale=1.0),
                                 family='LPIPS')
    relu = lambda n, at: insitu.Call('sfb_relu_nhwc', dict(x=1, n=n, stream=0), 'LPIPS', at)
    gemm = insitu.Rec('conv2d_nhwc', {}, (), {}, family='LPIPS')               # not a SIMT entry
    cat = insitu.Catalogue(sf.entry)
    # issued: relu 8, softmax 4, gemm, relu 16, softmax 4, relu 8
    cat.add([sm(4), gemm, sm(4)], [relu(8, 0), relu(16, 2), relu(8, 3)])
    got = [(e['op'], e.get('n', e.get('cols')), e['calls']) for e in cat.entries.values()]
    assert got == [('relu', 8, 2), ('softmax_rows', 4, 2), ('relu', 16, 1)], got
    cat.add([sm(5)], [relu(8, 1)])                                              # a later family run adds to the same catalogue
    assert [(e['op'], e['calls']) for e in cat.entries.values()][1:] == [('softmax_rows', 2), ('relu', 1), ('softmax_rows', 1)]
    assert next(iter(cat.entries.values()))['calls'] == 3
