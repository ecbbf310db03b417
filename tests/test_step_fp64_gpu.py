"""The sampler updates (plms_update*, ddpm_dynamic_step), the distillation loss kernels (csrc/image_glue.cu) and the EFT-only kernels of
csrc/eft_ops.cu replayed per element against fp64 (oracle/step_fp64.py).

A module fixture records the launches of DDPM.sample, of PLMSSampler (scene-batched and guided) and of two Distiller steps
(oracle/model_runs.record_steps), and of the EFT (record_eft), under oracle/insitu.Catalogue, which reads each C ABI call's arguments by
parameter name (``step_fp64.entry``): geometry, strides, the scalars (alpha, sigma, clip, percentile, cond_scale, the coefficients, each
row's five step scalars, the loss weights) and which history pointers are NULL.  Synthetic
entries add what the models do not reach: h != w and h or w = 1 in the glue, scale 1 / 2 / 4, mode-1 mask means exactly at 0.1f and one ulp
either side, d = 0 exactly; row lengths 1, 255, 256, 257, 8192, 8193, 57 345 and 65 536 and one row past 1024 x 256 floats; every pattern of
NULL history pointers and NULL optional outputs; all |x0| < 1, rank ties that span the cluster's CTAs, +-0 and subnormals, p = 0 and 1;
odd and unit max-pool sizes, Ho / Wo = 1, grid points on +-1, on pixel centres and past the border, C = 3 and 7, S = 1, 2, 20, 31, 32 and
E = 4, 132.

Each entry is replayed through the C ABI with the operand sets 'randn', 'one-signed', 'edges' and -- for the kernels whose clamps and maxima
must keep NaN (the sampler updates, the 3x3 max-pool, ReLU) -- 'non-finite' (NaN and +-inf in eps, x and the activations): NaN positions
must equal the reference's, other elements are held to the usual bound.  Operands sit in NaN-filled guard buffers; every float of an
output buffer outside the output (random, NaN in every other one: channels outside a slice in resize and grid_sample, the floats around
every output) stays bit-identical.  The sampler kernels' traced names must equal the
plan.  Every output except the glue's atomic loss sums must repeat bit for bit.

Out of scope: sfb_eft_t1_tokens (tests/test_scene_gpu.py), sfb_rays_from_camera (bitwise, tests/test_image_glue_gpu.py), NaN grid
coordinates and ordering hazards between launches."""
import math
from collections import defaultdict

import numpy as np
import pytest
import torch

from _helpers import NAN, Out, Tracer, guarded, ptr, release
from oracle import insitu, model_runs, step_fp64 as sp

pytestmark = pytest.mark.gpu

SETS = ('randn', 'one-signed', 'edges', 'non-finite')
NONFINITE = {'plms_update', 'plms_update_rows', 'plms_update_rows_cfg', 'ddpm_dynamic_step', 'maxpool3x3s2', 'act'}
PLMS4 = (55 / 24, -59 / 24, 37 / 24, -9 / 24)
SCAL = (0.8, 0.6, 0.9, 0.3, 0.1)           # alpha, sigma, alpha_next, c, noise_scale


# ------------------------------------------------------------------------------------------------ catalogue
def _plms(label, n, nulls=(False, False, False), x0_out=True, e_out=True, clip=1.0, scalars=SCAL, coefs=PLMS4):
    return dict(op='plms_update', n=n, nulls=nulls, coefs=coefs, scalars=scalars, clip=clip, x0_out=x0_out, e_out=e_out, label=label)


def _rows(label, rows, row_len, nulls=(False, False, False), x0_out=True, clip=1.0):
    return dict(op='plms_update_rows', rows=rows, row_len=row_len, nulls=nulls, coefs=PLMS4, clip=clip, x0_out=x0_out, label=label)


def _cfg(label, rows, row_len, nulls=(False, False, False), e_out=True, cond_scale=3.0):
    return dict(op='plms_update_rows_cfg', rows=rows, row_len=row_len, nulls=nulls, coefs=PLMS4, cond_scale=cond_scale, clip=1.0, e_out=e_out,
                label=label)


def _dyn(label, B, row_len, p=0.95, guided=True, pattern='', s_out=True, x0_out=True, cond_scale=3.0):
    return dict(op='ddpm_dynamic_step', B=B, row_len=row_len, guided=guided, cond_scale=cond_scale if guided else 1.0, scalars=SCAL, p=p,
                s_out=s_out, x0_out=x0_out, pattern=pattern, label=label)


def _synthetic():
    E = []
    # sampler: row lengths around the 256-thread block, the 8192-float chunk and the 8-CTA cluster; every NULL-history pattern
    for n in (1, 255, 256, 257, 8193):
        E.append(_plms(f'n {n}', n))
    E.append(_plms('grid-stride: 1024 x 256 + 1000 floats', 1024 * 256 + 1000))
    for m in range(8):
        nulls = tuple(bool(m >> i & 1) for i in range(3))
        E.append(_plms(f'NULL history {nulls}', 1000, nulls=nulls, x0_out=m % 2 == 0, e_out=m % 3 == 0))
    E.append(_plms('DDPM static guided form', 3000, nulls=(False, True, True), coefs=(3.0, -2.0, 0.0, 0.0), clip=10.0))
    E.append(_plms('alpha below 1e-8, no clip', 600, scalars=(1e-10, 0.6, 0.9, 0.3, 0.1), clip=math.inf))
    for rl in (1, 255, 257):
        E.append(_rows(f'rows row_len {rl}', 3, rl))
        E.append(_cfg(f'cfg row_len {rl}', 3, rl))
    E.append(_rows('rows: one row past 1024 x 256', 1, 1024 * 256 + 300, x0_out=False))
    E.append(_cfg('cfg: one row past 1024 x 256', 1, 1024 * 256 + 300, e_out=False))
    for m in range(8):
        nulls = tuple(bool(m >> i & 1) for i in range(3))
        E.append(_rows(f'rows NULL {nulls}', 5, 700, nulls=nulls, x0_out=m % 2 == 1))
        E.append(_cfg(f'cfg NULL {nulls}', 5, 700, nulls=nulls, e_out=m % 2 == 1, cond_scale=1.0 + m / 2))
    for rl in (1, 255, 256, 257, 8192, 8193, 57345, 65536):
        E.append(_dyn(f'row_len {rl}', 3, rl))
    E += [_dyn('unguided', 2, 4096, guided=False), _dyn('p = 0', 2, 8193, p=0.0), _dyn('p = 1', 2, 8193, p=1.0),
          _dyn('p = 0.5', 2, 5, p=0.5), _dyn('all |x0| < 1: s = 1', 2, 9000, pattern='small'),
          _dyn('rank ties across CTAs', 2, 65536, pattern='ties'), _dyn('ties, one CTA', 2, 4096, pattern='ties'),
          _dyn('+-0 and subnormals', 2, 20000, pattern='tiny'), _dyn('NULL s_out and x0_out', 2, 30000, s_out=False, x0_out=False),
          _dyn('NULL x0_out', 3, 4096, x0_out=False)]
    # image glue
    for h, w, sc in ((37, 53, 2), (1, 40, 2), (40, 1, 2), (16, 16, 1), (9, 12, 4), (64, 64, 2), (128, 128, 2)):
        E.append(dict(op='photometric_loss', h=h, w=w, scale=sc, lam=(1.0, 0.7, 1e-3), label=f'{h}x{w} scale {sc}'))
    for h, w in ((37, 53), (1, 7), (7, 1), (16, 16), (128, 128)):
        E.append(dict(op='upsample2x_render', h=h, w=w, label=f'{h}x{w}'))
        for mode in (0, 1):
            for ge in (False, True):
                E.append(dict(op='fusion_loss', h=h, w=w, mode=mode, g_extra=ge, wgt=0.37, lam=(1.0, 0.7, 1e-3), label=f'{h}x{w}'))
    # EFT
    for NB, H, W, C in ((2, 17, 22, 8), (1, 1, 9, 4), (1, 9, 1, 4), (2, 7, 5, 12), (1, 2, 2, 4), (1, 128, 128, 64)):
        E.append(dict(op='maxpool3x3s2', NB=NB, H=H, W=W, C=C, label=f'{H}x{W}'))
    for NB, H, W, C, Ho, Wo, ldx, ldo, off in ((2, 5, 7, 8, 16, 16, 8, 20, 4), (1, 5, 7, 4, 1, 9, 8, 4, 0), (1, 5, 7, 4, 9, 1, 4, 12, 8),
                                               (1, 1, 1, 4, 3, 5, 4, 4, 0), (2, 8, 8, 12, 32, 32, 16, 24, 12), (1, 64, 64, 8, 64, 64, 8, 8, 0)):
        E.append(dict(op='resize', NB=NB, H=H, W=W, C=C, Ho=Ho, Wo=Wo, ldx=ldx, ldo=ldo, off=off, label=f'{H}x{W}->{Ho}x{Wo}'))
    for NB, H, W, C, M, ldx, ldo, off in ((2, 9, 11, 7, 300, 7, 12, 3), (1, 16, 16, 3, 257, 4, 3, 0), (2, 1, 5, 5, 40, 8, 9, 2),
                                          (1, 6, 1, 64, 33, 64, 70, 4), (1, 32, 32, 512, 100, 512, 512, 0)):
        E.append(dict(op='grid_sample', NB=NB, H=H, W=W, C=C, M=M, ldx=ldx, ldo=ldo, off=off, label=f'C {C}'))
    for S, B, E_ in ((1, 5, 256), (2, 300, 256), (20, 64, 256), (6, 5, 256), (31, 3, 132), (32, 9, 4), (6, 13, 132), (32, 1, 256)):
        E.append(dict(op='seq_attention', S=S, B=B, E=E_, label=f'S {S} B {B} E {E_}'))
    for n, kind in ((4, 0), (4000, 0), (1 << 20, 0), (4, 1), (4000, 1), (1 << 20, 1)):
        E.append(dict(op='act', n=n, kind=kind, label=f'n {n}'))
    for e in E:
        e.setdefault('family', 'synthetic')
    return E


@pytest.fixture(scope='module')
def catalogue():
    cat = insitu.Catalogue(sp.entry)
    model_runs.record_steps(cat)
    model_runs.record_eft(cat)
    entries = list(cat.entries.values()) + _synthetic()
    fam = defaultdict(int)
    for e in entries:
        fam[(e['family'], e['op'])] += 1
    print('\nstep catalogue: ' + ', '.join(f'{f}/{o} {v}' for (f, o), v in sorted(fam.items())))
    return entries


# ------------------------------------------------------------------------------------------------ operands
class _Gen:
    def __init__(self, kind, seed):
        self.kind = kind
        self.g = torch.Generator(device='cuda').manual_seed(seed)

    def __call__(self, *shape, scale=1.0, nonfinite=True):
        t = torch.randn(*shape, device='cuda', generator=self.g) * scale
        if self.kind == 'one-signed':
            t = t.abs()
        elif self.kind == 'edges':
            cat = torch.randint(0, 4, t.shape, device='cuda', generator=self.g)
            p2 = torch.exp2(torch.floor(torch.log2(t.abs().clamp_min(1e-30)))) * torch.sign(t)
            t = torch.where(cat == 0, torch.zeros_like(t), torch.where(cat == 1, p2, t))
        elif self.kind == 'non-finite' and nonfinite:
            cat = torch.randint(0, 48, t.shape, device='cuda', generator=self.g)
            t = torch.where(cat == 0, torch.full_like(t, NAN), torch.where(cat == 1, torch.full_like(t, math.inf),
                                                                             torch.where(cat == 2, torch.full_like(t, -math.inf), t)))
        return t

    def rand(self, *shape):
        return torch.rand(*shape, device='cuda', generator=self.g)


def _opt(flag, rows, width, seed):
    return Out(rows, width, seed=seed) if flag else None


def _row_scalars(rows):
    """a distinct (alpha, sigma, alpha_next, c, noise_scale) per row"""
    r = torch.arange(rows, dtype=torch.float64)
    al = 0.3 + 0.6 * (r + 1) / (rows + 1)
    return torch.stack((al, torch.sqrt(1 - al * al), al + 0.05, 0.2 + 0.1 * r / rows, 0.05 + 0.01 * r), 1).float()


# ------------------------------------------------------------------------------------------------ replays
def _replay(e, kind, seed, tracer, sm):
    """returns dict(checks=[(name, got, ref, bound-or-None)], exact_checks=[(name, ok)], guard, names, planned, again)"""
    from sparsefusion_b200 import _lib as lib
    G = _Gen(kind, seed)
    op = e['op']
    release()
    call, S = lib.call, lib.stream()
    res = dict(checks=[], flags=[], guard=True, names=None, planned=None, again=True)
    outs = []

    def run(fn, repeat=True):
        names = tracer.run(fn)
        first = [o.value() for o in outs]
        if repeat:
            fn()
            torch.cuda.synchronize()
            res['again'] = all(torch.equal(a.view(torch.int32), o.value().view(torch.int32)) for a, o in zip(first, outs))
        res['names'] = names
        res['guard'] = all(o.guard_ok() for o in outs)
        return first

    def chk(name, got, ref_bnd):
        res['checks'].append((name, got, ref_bnd[0], ref_bnd[1]))

    if op in ('plms_update', 'plms_update_rows', 'plms_update_rows_cfg'):
        rows = e.get('rows', 1)
        L = e['n'] if op == 'plms_update' else e['row_len']
        x, noise = G(rows, L), G(rows, L, nonfinite=False)
        eps = [G(rows, L, scale=0.7) if (i == 0 or not e['nulls'][i - 1]) else None for i in range(4)]
        coefs = e['coefs']
        if op == 'plms_update':
            sc = torch.tensor(e['scalars'], dtype=torch.float32).view(1, 5)
        else:
            sc = torch.tensor(e['row_scalars']).view(rows, 5) if 'row_scalars' in e else _row_scalars(rows)
        ptrs = [ptr(guarded(t)) for t in eps]
        xp, zp = ptr(guarded(x)), ptr(guarded(noise))
        xo = Out(rows, L, seed=1)
        outs.append(xo)
        if op == 'plms_update':
            x0o, eo = _opt(e['x0_out'], 1, L, 2), _opt(e['e_out'], 1, L, 3)
            outs += [o for o in (x0o, eo) if o]
            sv = [float(v) for v in sc[0]]
            got = run(lambda: call('sfb_plms_update', xp, *ptrs, *coefs, zp, *sv, e['clip'], xo.ptr, x0o.ptr if x0o else None,
                                   eo.ptr if eo else None, L, S))
            plan = sp.kernel_plan(op, dict(n=L), sm)
            e_ref = e_abs = None
            if (kind != 'non-finite' and eps[1] is not None and all(t is None for t in eps[2:]) and coefs[2] == coefs[3] == 0
                    and abs(coefs[0] + coefs[1] - 1) < 1e-6):
                # DDPM.sample's guided static step: s cond + (1 - s) null against the reference's null + (cond - null) s (the two forms
                # differ by rounding only for finite eps: with -inf cond and +inf null one is -inf, the other NaN)
                s = coefs[0]
                c_, n_ = eps[0].double(), eps[1].double()
                e_ref, e_abs = n_ + (c_ - n_) * s, abs(s) * c_.abs() + abs(1 - s) * n_.abs()
            r = sp.ref_plms(x, eps, coefs, sc, noise, e['clip'], e_abs=e_abs, e_ref=e_ref)
            chk('x_prev', got[0], r['x_prev'])
            k = 1
            if x0o:
                chk('x0', got[k], r['x0'])
                k += 1
            if eo:
                chk('e', got[k], r['e'])
        elif op == 'plms_update_rows':
            scp = ptr(guarded(sc))
            x0o = _opt(e['x0_out'], rows, L, 2)
            if x0o:
                outs.append(x0o)
            got = run(lambda: call('sfb_plms_update_rows', xp, *ptrs, *coefs, zp, scp, e['clip'], xo.ptr, x0o.ptr if x0o else None, rows, L, S))
            plan = sp.kernel_plan(op, dict(rows=rows, row_len=L), sm)
            r = sp.ref_plms(x, eps, coefs, sc, noise, e['clip'])
            chk('x_prev', got[0], r['x_prev'])
            if x0o:
                chk('x0', got[1], r['x0'])
            # each row as its own sfb_plms_update launch with its scalars: bit-identical
            for rr in range(0, rows, max(1, rows - 1)):
                o1 = torch.full((L,), NAN, device='cuda')
                rp = [None if t is None else t[rr].contiguous() for t in eps]
                xr, zr = x[rr].contiguous(), noise[rr].contiguous()
                call('sfb_plms_update', xr.data_ptr(), *[None if t is None else t.data_ptr() for t in rp], *coefs, zr.data_ptr(),
                     *[float(v) for v in sc[rr]], e['clip'], o1.data_ptr(), None, None, L, S)
                torch.cuda.synchronize()
                res['flags'].append((f'row {rr} = its own launch', torch.equal(o1.view(torch.int32), got[0][rr].view(torch.int32))))
        else:
            en = G(rows, L, scale=0.7)
            ec = eps[0]
            enp, scp = ptr(guarded(en)), ptr(guarded(sc))
            eo = _opt(e['e_out'], rows, L, 3)
            if eo:
                outs.append(eo)
            cs = e['cond_scale']
            got = run(lambda: call('sfb_plms_update_rows_cfg', xp, ptrs[0], enp, cs, *ptrs[1:], *coefs, zp, scp, e['clip'], xo.ptr,
                                   eo.ptr if eo else None, rows, L, S))
            plan = sp.kernel_plan(op, dict(rows=rows, row_len=L), sm)
            et = sp.cfg_eps(ec, en, cs).cuda()
            r = sp.ref_plms(x, [et] + eps[1:], coefs, sc, noise, e['clip'])
            chk('x_prev', got[0], r['x_prev'])
            if eo:
                res['flags'].append(('e_out bit-identical to the fp32 emulation', bool(torch.equal(torch.isnan(got[1]), torch.isnan(et)))
                                     and torch.equal(torch.nan_to_num(got[1]).view(torch.int32), torch.nan_to_num(et).view(torch.int32))))
        res['planned'] = plan['kernels']
    elif op == 'ddpm_dynamic_step':
        B, L, pat = e['B'], e['row_len'], e.get('pattern', '')
        al, sg, an, c, ns = e['scalars']
        x, noise = G(B, L, scale=2.0, nonfinite=False), G(B, L, nonfinite=False)
        ec, en = G(B, L, nonfinite=False), (G(B, L, nonfinite=False) if e['guided'] else None)
        if pat in ('small', 'ties', 'tiny'):                          # x0 = x exactly: alpha 1, no eps
            al, sg = 1.0, 0.0
            ec.zero_()
            if en is not None:
                en.zero_()
            if pat == 'small':
                x = (G.rand(B, L) * 1.98 - 0.99)
            elif pat == 'ties':
                x = (torch.randint(0, 4, (B, L), device='cuda', generator=G.g).float() + 0.5) * torch.sign(G.rand(B, L) - 0.5)
            else:
                x = torch.where(G.rand(B, L) < 0.5, torch.full_like(x, 1e-40), torch.zeros_like(x)) * torch.sign(G.rand(B, L) - 0.5)
                x[:, ::97] = 3.0
        if kind == 'non-finite':
            # a NaN x0 from eps: opposite infinities in s e_cond + (1 - s) e_null (a NaN e_cond unguided) -- row 0 when B = 2, the last row
            # when B > 2, where row 0 gets a NaN x.  Row 1: +-inf in x, -inf in e_cond (and +inf in e_null): infinite x0, finite s
            def eps_nan(r, i):
                if en is not None:
                    ec[r, i], en[r, i] = math.inf, math.inf
                else:
                    ec[r, i] = NAN
            if B > 2:
                x[0, L // 3] = NAN
                eps_nan(B - 1, L // 2)
            else:
                eps_nan(0, L // 3)
            if B > 1:
                x[1, L // 2] = math.inf
                ec[1, L // 4] = -math.inf
                if en is not None:
                    en[1, L // 5] = math.inf
                if L > 1:
                    x[1, 0] = -math.inf
        xp, cp, np_, zp = ptr(guarded(x)), ptr(guarded(ec)), ptr(guarded(en)), ptr(guarded(noise))
        xo, so, x0o = Out(B, L, seed=1), Out(1, B, seed=2), Out(B, L, seed=3)
        outs += [xo, so, x0o]
        cs = e['cond_scale']
        args = lambda xo_, so_, x0_: (xp, cp, np_, cs, zp, al, sg, an, c, ns, e['p'], L, B, xo_, so_, x0_, S)
        got = run(lambda: call('sfb_ddpm_dynamic_step', *args(xo.ptr, so.ptr, x0o.ptr)))
        plan = sp.kernel_plan(op, dict(B=B, row_len=L), sm)
        res['planned'] = plan['kernels']
        x0r, b0 = sp.dyn_x0(x, ec, en, cs, al, sg)
        chk('x0', got[2], (x0r, b0))
        s_ref = sp.quantile_s(got[2], e['p'])                          # torch.quantile of the kernel's own x0
        s_got = got[1].view(B)
        res['flags'].append(('s = torch.quantile(|x0|, p).clamp(min=1)', bool(torch.equal(torch.isnan(s_got), torch.isnan(s_ref)))
                             and torch.equal(torch.nan_to_num(s_got).view(torch.int32), torch.nan_to_num(s_ref).view(torch.int32))))
        chk('x_prev', got[0], sp.ref_dyn_x_prev(x, x0r, b0, s_got, al, an, c, ns, noise))
        if pat == 'small' and kind != 'non-finite':                   # the non-finite set puts a NaN in row 0
            res['flags'].append(('s = 1', bool((s_got == 1).all())))
        if not (e['s_out'] and e['x0_out']):                           # the entry's own NULL outputs: the same x_prev
            o2 = Out(B, L, seed=4)
            call('sfb_ddpm_dynamic_step', *args(o2.ptr, so.ptr if e['s_out'] else None, x0o.ptr if e['x0_out'] else None))
            torch.cuda.synchronize()
            res['flags'].append(('NULL outputs leave x_prev unchanged', torch.equal(o2.value().view(torch.int32), got[0].view(torch.int32))))
    elif op == 'photometric_loss':
        h, w, scl = e['h'], e['w'], e['scale']
        n = h * w
        img, sil = G.rand(n, 3), G.rand(n)
        rgb = G.rand(3, h * scl, w * scl)
        mask = (G.rand(h * scl, w * scl) > 0.5).float()
        if kind == 'edges':                                            # d = 0 exactly at a third of the pixels
            src = sp.glue_nearest(rgb.cpu(), h, w, scl).reshape(3, n).t().cuda()
            sel = (torch.arange(n, device='cuda') % 3 == 0)[:, None]
            img = torch.where(sel, src, img)
        elif kind == 'one-signed':
            img = img + 1.0
        lam = e['lam']
        ip, sp_, rp, mp = ptr(guarded(img)), ptr(guarded(sil)), ptr(guarded(rgb)), ptr(guarded(mask))
        so, gi, gs = Out(1, 3, seed=1), Out(n, 3, seed=2), Out(1, n, seed=3)
        outs += [so, gi, gs]
        got = run(lambda: call('sfb_photometric_loss', ip, sp_, rp, mp, h, w, scl, *lam, so.ptr, gi.ptr, gs.ptr, S), repeat=False)
        # the repeat: gradients only (the sums are atomics)
        call('sfb_photometric_loss', ip, sp_, rp, mp, h, w, scl, *lam, so.ptr, gi.ptr, gs.ptr, S)
        torch.cuda.synchronize()
        res['again'] = torch.equal(got[1].view(torch.int32), gi.value().view(torch.int32)) and torch.equal(got[2].view(torch.int32), gs.value().view(torch.int32))
        plan = sp.kernel_plan(op, dict(h=h, w=w), sm)
        r = sp.ref_photometric(img, sil, rgb, mask, h, w, scl, *lam, plan)
        chk('sums', got[0].view(3), r['sums'])
        chk('g_img', got[1], r['g_img'])
        chk('g_sil', got[2].view(n), r['g_sil'])
    elif op == 'upsample2x_render':
        h, w = e['h'], e['w']
        img, sil = G(h * w, 3), G(h * w)
        up = Out(1, 16 * h * w)
        outs.append(up)
        got = run(lambda: call('sfb_upsample2x_render', ptr(guarded(img)), ptr(guarded(sil)), h, w, up.ptr, S))
        chk('up', got[0].view(4, 2 * h, 2 * w), sp.ref_upsample2x(img, sil, h, w))
    elif op == 'fusion_loss':
        h, w, mode = e['h'], e['w'], e['mode']
        H, W = 2 * h, 2 * w
        HW = H * W
        up = G.rand(4, H, W)
        target = G.rand(3, H, W) * 0.3
        if kind == 'edges':
            if mode == 0:                                              # d = 0 exactly
                up[:3, ::2] = target[:, ::2]
            else:                                                      # channel means exactly at 0.1f and one ulp either side
                t01 = torch.tensor(_T0, device='cuda')
                flat = target.view(3, -1)
                k = torch.arange(HW, device='cuda') % 4
                sel = k < 3
                flat[0] = torch.where(sel, t01[k.clamp(max=2), 0], flat[0])
                flat[1] = torch.where(sel, t01[k.clamp(max=2), 1], flat[1])
                flat[2] = torch.where(sel, torch.zeros_like(flat[2]), flat[2])
        elif kind == 'one-signed':
            up[:3] += 1.0
        ge = G(3, H, W, scale=1e-4) if e['g_extra'] else None
        lam = e['lam']
        upp, tp, gep = ptr(guarded(up)), ptr(guarded(target)), ptr(guarded(ge))
        so, gu, gi, gs = Out(1, 3, seed=1), Out(1, 4 * HW, seed=2), Out(h * w, 3, seed=3), Out(1, h * w, seed=4)
        outs += [so, gu, gi, gs]
        fn = lambda: call('sfb_fusion_loss_ex', upp, tp, H, W, mode, e['wgt'], *lam, gep, so.ptr, gu.ptr, h, w, gi.ptr, gs.ptr, S)
        got = run(fn, repeat=False)
        fn()
        torch.cuda.synchronize()
        res['again'] = all(torch.equal(a.view(torch.int32), o.value().view(torch.int32)) for a, o in zip(got[1:], (gu, gi, gs)))
        plan = sp.kernel_plan(op, dict(h=h, w=w), sm)
        r = sp.ref_fusion(up, target, mode, e['wgt'], *lam, ge, plan)
        chk('sums', got[0].view(3), r['sums'])
        chk('g_up', got[1].view(4, H, W), r['g_up'])
        (gi_r, gs_r) = sp.ref_fusion_adjoint(got[1].view(4, H, W), h, w)
        chk('g_img', got[2], gi_r)
        chk('g_sil', got[3].view(-1), gs_r)
    elif op == 'maxpool3x3s2':
        NB, H, W, C = e['NB'], e['H'], e['W'], e['C']
        x = G(NB, H, W, C)
        if kind == 'edges':
            x = torch.round(x).clamp(-1, 2) + 0.0                      # ties
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = Out(1, NB * Ho * Wo * C)
        outs.append(y)
        got = run(lambda: call('sfb_maxpool3x3s2_nhwc', ptr(guarded(x)), y.ptr, NB, H, W, C, S))
        chk('y', got[0].view(NB, Ho, Wo, C), (sp.maxpool3x3s2(x.cpu()), None))
    elif op == 'act':
        n, k = e['n'], e['kind']
        x = G(n, scale=3.0)
        o = Out(1, n, prefill=x)                                       # in place
        tracer.run(lambda: call('sfb_act_inplace', o.ptr, n, k, S))
        got = o.value().view(n)
        res['guard'] = o.guard_ok()
        o.slot[:] = x.view(1, n)
        call('sfb_act_inplace', o.ptr, n, k, S)
        torch.cuda.synchronize()
        res['again'] = torch.equal(got.view(torch.int32), o.value().view(n).view(torch.int32))
        chk('relu' if k == 0 else 'gelu', got, (sp.relu(x.cpu()), None) if k == 0 else sp.ref_gelu(x))
    elif op == 'resize':
        NB, H, W, C, Ho, Wo, ldx, ldo = e['NB'], e['H'], e['W'], e['C'], e['Ho'], e['Wo'], e['ldx'], e['ldo']
        off = e.get('off', (ldo - C) // 4 * 4 if ldo > C else 0)
        x = G(NB, H, W, C)
        xb = torch.full((NB * H * W, ldx), NAN, device='cuda')
        xb[:, :C] = x.view(-1, C)
        y = Out(NB * Ho * Wo, C, ld=ldo, off=off)
        outs.append(y)
        got = run(lambda: call('sfb_resize_bilinear_ac_nhwc', ptr(guarded(xb)), ldx, y.ptr, ldo, NB, H, W, C, Ho, Wo, S))
        chk('y', got[0].view(NB, Ho, Wo, C), sp.ref_resize(x, Ho, Wo))
    elif op == 'grid_sample':
        NB, H, W, C, M, ldx, ldo = e['NB'], e['H'], e['W'], e['C'], e['M'], e['ldx'], e['ldo']
        off = e.get('off', (ldo - C) if ldo > C else 0)
        x = G(NB, H, W, C)
        xb = torch.full((NB * H * W, ldx), NAN, device='cuda')
        xb[:, :C] = x.view(-1, C)
        grid = G.rand(NB, M, 2) * 2.6 - 1.3
        if kind == 'edges':                                            # exactly +-1, pixel centres, beyond the border
            k = torch.arange(M, device='cuda')
            cx = -1 + 2 * (k % max(W, 1)).float() / max(W - 1, 1)
            cy = -1 + 2 * (k % max(H, 1)).float() / max(H - 1, 1)
            g0 = grid[0]
            special = torch.stack((torch.stack((cx, cy), -1), torch.sign(g0), g0 * 3), 0)
            grid = special[k % 3, k].expand(NB, M, 2).contiguous()
        y = Out(NB * M, C, ld=ldo, off=off)
        outs.append(y)
        got = run(lambda: call('sfb_grid_sample_nhwc', ptr(guarded(xb)), ldx, ptr(guarded(grid)), y.ptr, ldo, NB, H, W, C, M, S))
        chk('out', got[0].view(NB, M, C), sp.ref_grid_sample(x, grid))
    elif op == 'seq_attention':
        S_, B, E_ = e['S'], e['B'], e['E']
        qkv = G(S_, B, 3 * E_, scale=(4.0 / math.sqrt(math.sqrt(E_))) if kind == 'edges' else 1.0)
        y = Out(1, S_ * B * E_)
        outs.append(y)
        got = run(lambda: call('sfb_seq_attention', ptr(guarded(qkv)), y.ptr, S_, B, E_, S))
        chk('out', got[0].view(S_, B, E_), sp.ref_seq_attention(qkv, S_, B, E_))
    else:
        raise KeyError(op)
    return res


def _mask_t0():
    """channel pairs (t0, 0) whose fp32 mean (t0 + 0 + 0) / 3 is the largest value below 0.1f that such a mean reaches, 0.1f itself and
    the least value above (a sum near 0.3 has a 2^-25 ulp, so not every fp32 value near 0.1 is a third of one)"""
    f = np.float32
    t = f(f(0.1) * f(3))
    for _ in range(16):
        t = np.nextafter(t, f(0))
    means = {}
    for _ in range(33):
        means.setdefault(float(f(t / f(3))), float(t))
        t = np.nextafter(t, f(1))
    m = float(f(0.1))
    assert m in means
    below, above = max(v for v in means if v < m), min(v for v in means if v > m)
    return [(means[below], 0.0), (means[m], 0.0), (means[above], 0.0)]


_T0 = _mask_t0()


def _key(e):
    skip = ('op', 'family', 'label')
    return f"{e['family']} {e['op']} [{e['label']}] " + ' '.join(f'{k}={v}' for k, v in e.items() if k not in skip)


@pytest.fixture(scope='module')
def replays(catalogue):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    tracer = Tracer()
    out = dict(fail=[], names=set(), table={}, runs=0)
    table = {}
    for n, e in enumerate(catalogue):
        for si, kind in enumerate(SETS):
            if kind == 'non-finite' and e['op'] not in NONFINITE:
                continue
            if kind == 'non-finite' and e['op'] == 'act' and e['kind'] != 0:
                continue
            r = _replay(e, kind, 1000 * n + si, tracer, sm)
            out['runs'] += 1
            msg = []
            if r['planned'] is not None:
                if r['names'] != r['planned']:
                    msg.append(f"traced {r['names']}, planned {r['planned']}")
                out['names'] |= set(r['names'])
            for name, got, ref, bnd in r['checks']:
                c = sp.compare(got, ref, bnd)
                if not c['nan_ok']:
                    msg.append(f'{name}: NaN positions differ from the reference')
                if c['ratio'] > 1:
                    msg.append(f"{name} err/bound {c['ratio']:.3g}" if bnd is not None else f'{name} not equal')
                if bnd is not None:
                    tk = (e['op'], name, kind)
                    table[tk] = max(table.get(tk, 0.0), c['ratio'])
            for name, ok in r['flags']:
                if not ok:
                    msg.append(f'{name}: failed')
            if not r['guard']:
                msg.append('memory outside the output changed')
            if not r['again']:
                msg.append('second run not bit-identical')
            if msg:
                out['fail'].append(f'{_key(e)} [{kind}]: ' + '; '.join(msg))
    out['table'] = table
    print('\nop                    output   operand set   max err/bound')
    for (op, name, kind), ratio in sorted(table.items()):
        print(f'{op:21s} {name:8s} {kind:13s} {ratio:13.3f}')
    if out['fail']:
        print('\n'.join(out['fail'][:80]))
    return out


# ------------------------------------------------------------------------------------------------ tests
def test_catalogue_holds_the_recorded_launches(catalogue):
    by = defaultdict(list)
    for e in catalogue:
        by[(e['family'], e['op'])].append(e)
    for op in ('plms_update', 'ddpm_dynamic_step'):
        assert by[('DDPM', op)], op
    assert by[('PLMS', 'plms_update_rows')] and by[('PLMS', 'plms_update_rows_cfg')]      # scene-batched and guided sampling
    assert by[('Distill', 'plms_update_rows')]                                            # the SDS target
    assert any(e['rows'] == 2 and len(set(e['row_scalars'][0::5])) == 2 for e in by[('PLMS', 'plms_update_rows')])    # two schedules
    assert by[('Distill', 'photometric_loss')] and by[('Distill', 'upsample2x_render')]
    fl = by[('Distill', 'fusion_loss')]
    assert any(e['mode'] == 0 and e['g_extra'] for e in fl) and any(e['mode'] == 1 and not e['g_extra'] for e in fl), fl   # SDS + percep, EFT
    for op in ('maxpool3x3s2', 'resize', 'seq_attention', 'act'):          # the view-batched cache samples in eft_t1_tokens, not grid_sample
        assert by[('EFT', op)], op
    assert any(e['row_len'] == 65536 for e in by[('DDPM', 'ddpm_dynamic_step')])          # 128^2 latents: an 8-CTA cluster per row
    assert any(e['guided'] for e in by[('DDPM', 'ddpm_dynamic_step')]) and any(not e['nulls'][0] for e in by[('DDPM', 'plms_update')])


def test_every_replay_is_within_its_fp64_bound(replays):
    assert not replays['fail'], f"{len(replays['fail'])} failures:\n" + '\n'.join(replays['fail'][:80])


def test_replays_reach_every_sampler_kernel(replays):
    want = {'sfb::plms_update_kernel', 'sfb::plms_update_rows_kernel', 'sfb::plms_update_rows_cfg_kernel',
            'sfb::ddpm_dynamic_step_kernel<false>', 'sfb::ddpm_dynamic_step_kernel<true>'}
    assert want <= replays['names'], sorted(want - replays['names'])
