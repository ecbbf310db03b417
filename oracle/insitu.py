"""oracle/insitu.py -- record the library launches of real model evaluations with the tensors they actually read and wrote, and check every
launch against fp64 of those operands.

TEST INFRASTRUCTURE ONLY.

The per-launch tests (tests/test_conv_fp64_gpu.py, tests/test_simt_fp64_gpu.py) replay each launch's geometry on its own with fresh operands,
so they cannot see an operand read before its producer finished: programmatic dependent launch (PDL), CUDA-graph replays whose
intermediates sit at the same address every time, the UNet's side stream, the split-K arena.  Here the operands are the model's own.

``Recorder`` is the one wrapper of the ``ops.*`` front ends and ``_lib.call``.  Each front-end launch becomes a ``Rec``: the op, its
scalars, references to its input and output tensors (views, slices and strides as passed), the stream it was issued on, whether it was
captured into a graph, the library kernels it launched (``sfb_launch_count``) and their traced names.  Every tensor stays alive as long as
the recorder, so the caching allocator reuses no buffer inside a recorded evaluation: write-after-read hazards between launches are out of
scope.  Each C ABI call made outside a front end becomes a ``Call``: its arguments bound to the header's parameter names.

``Catalogue`` turns the records of oracle/model_runs' evaluations into the entries the per-launch replay tests replay, through the
``entry`` function of oracle/conv_fp64.py, oracle/simt_fp64.py or oracle/step_fp64.py.

A launch that writes memory an earlier record (or the launch itself: x=out, res=out, accumulate into a pre-filled ``out``) read or wrote
would leave that record without the values it saw.  Right before such a launch the recorder clones the overlapping tensor and the record
keeps the clone (``Rec.snapshots``; inside a capture the clone is one more graph node in front of that launch).  C ABI launches that bypass
the front ends (LPIPS, the EFT) are not checked; before each of them every recorded tensor whose storage holds one of its pointer
arguments is cloned the same way, since such a launch may write it in place (``sfb_relu_nhwc``, ``sfb_act_inplace``).

``check(rec)`` recomputes a record in fp64 with the references and bounds of oracle/conv_fp64.py and oracle/simt_fp64.py.  ``poison``
fills the exact element set of recorded outputs with NaN; ``poison_allocator`` leaves NaN in the caching allocator's free blocks before an
eager evaluation.  ``provenance`` checks what every GEMM reads ahead of its griddepcontrol.wait (conv_wgmma.cu: the bias, and the first
weight stages unless ``dynamic_weights``) against the storages of the prepared plans.
"""
from __future__ import annotations

import ctypes
import gc
import inspect
import math
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from . import conv_fp64 as cf, simt_fp64 as sf, step_fp64 as st
from .field_fp64 import ATOL

FRONT_ENDS = ('conv2d_nhwc', 'groupnorm', 'layernorm', 'linear_small', 'mq_attention', 'cross_attention', 'gca_pool', 'gate_mlp_residual',
              'gate_residual', 'softmax_rows', 'upsample2x', 'nchw_to_nhwc', 'nhwc_to_nchw', 'im2col4', 'concat2', 'pixel_shuffle_silu',
              'time_fourier')
NAN = float('nan')


@dataclass
class Rec:
    op: str
    t: Dict[str, Optional[torch.Tensor]]      # operands and outputs as the checker reads them (snapshots substituted)
    outs: tuple                               # names of the outputs in ``t``
    s: Dict                                   # scalars
    stream: int = 0
    captured: bool = False
    family: str = ''
    label: str = ''
    kernels: int = 0
    names: List[str] = field(default_factory=list)
    alias: str = ''
    snapshots: int = 0
    orig: Dict[str, Optional[torch.Tensor]] = field(default_factory=dict)   # the tensors as passed (never substituted)

    def __post_init__(self):
        if not self.orig:
            self.orig = dict(self.t)


@dataclass
class Call:
    op: str                 # the C ABI symbol
    args: Dict              # parameter name (the last identifier of its declaration in the header) -> argument
    family: str = ''
    at: int = 0             # front-end records made before the call


# pointer arguments the recorder copies at call time, with their float counts: the per-row scalar tables of the sampler updates
BY_VALUE = {'row_scalars': lambda a: 5 * a['rows']}


@dataclass
class Report:
    ratio: float            # worst |got - ref| / bound (inf: NaN or a differing bit of an exact op)
    n_bad: int              # elements out of bound
    n_nonfinite: int        # NaN / inf elements of the outputs
    first: Optional[tuple]  # (output, index) of the first offending element
    numel: int

    @property
    def ok(self):
        return self.n_bad == 0 and self.n_nonfinite == 0


# ------------------------------------------------------------------------------------------------ memory helpers
def _extent(t: torch.Tensor):
    """[lo, hi) bytes of t's elements"""
    if t.numel() == 0:
        return t.data_ptr(), t.data_ptr()
    span = sum((s - 1) * abs(st) for s, st in zip(t.shape, t.stride())) + 1
    return t.data_ptr(), t.data_ptr() + span * t.element_size()


def overlaps(a: Optional[torch.Tensor], b: Optional[torch.Tensor]) -> bool:
    """a and b share elements.  Byte ranges that intersect count as overlapping, except for channel slices of the same rows (same shape
    but the last dimension, same strides, one row stride ``ld``): those overlap only where their channel intervals do."""
    if a is None or b is None or a.device != b.device:
        return False
    (a0, a1), (b0, b1) = _extent(a), _extent(b)
    if not (a0 < b1 and b0 < a1):
        return False
    if (a.dim() >= 2 and a.dim() == b.dim() and a.stride() == b.stride() and a.shape[:-1] == b.shape[:-1] and a.stride(-1) == 1
            and a.element_size() == b.element_size()):
        ld, es = a.stride(-2), a.element_size()
        oa, ob = a.data_ptr() // es, b.data_ptr() // es
        ca, cb = oa % ld, ob % ld
        if ca + a.shape[-1] <= ld and cb + b.shape[-1] <= ld and oa - ca == ob - cb:
            return ca < cb + b.shape[-1] and cb < ca + a.shape[-1]
    return True


def _holds(t: torch.Tensor, p: int) -> bool:
    st = t.untyped_storage()
    return st.data_ptr() <= p < st.data_ptr() + st.nbytes()


def storage_of(t: torch.Tensor) -> int:
    return t.untyped_storage().data_ptr()


def device_floats(ptr: int, n: int) -> torch.Tensor:
    """a copy of n floats at a device address, in stream order"""
    class _View:
        __cuda_array_interface__ = dict(shape=(n,), typestr='<f4', data=(ptr, False), version=3)
    return torch.as_tensor(_View(), device='cuda').clone()


# ------------------------------------------------------------------------------------------------ recorder
def c_params() -> Dict[str, List[str]]:
    """symbol -> parameter names of the C ABI header: the last identifier of each declaration"""
    from sparsefusion_b200 import _lib as lib
    return {n: [re.search(r'(\w+)\s*$', d).group(1) for d in decls] for n, (_, decls) in lib.parse_header().items()}


def _specs():
    """op -> (inputs, outputs given before the launch, outputs after the launch, scalars) as functions of the bound arguments"""
    def conv(a, y):
        return dict(x=a['x'], w_packed=a['w_packed'], bias=a['bias'], residual=a['residual'], w_split=a['w_split']), dict(out=y), \
            dict(cout=a['cout'], kh=a['kh'], kw=a['kw'], stride=a['stride'], pad=a['pad'],
                 pad_after=a['pad'] if a['pad_after'] is None else a['pad_after'], splits=a['splits'], bn=a['bn'],
                 dyn=bool(a['dynamic_weights']), accumulate=bool(a['accumulate']))
    return dict(
        conv2d_nhwc=(conv, lambda a: a['out']),
        groupnorm=(lambda a, y: (dict(x=a['x'], gamma=a['gamma'], beta=a['beta'], film=a['film']), dict(out=y),
                                 dict(groups=a['groups'], silu=bool(a['silu']), eps=float(a['eps']))), lambda a: a['out']),
        layernorm=(lambda a, y: (dict(x=a['x'], g=a['g'], b=a['b'], residual=a['residual']), dict(out=y),
                                 dict(pre_gelu=bool(a['pre_gelu']), round=bool(a['round_to_tf32']))), lambda a: a['out']),
        linear_small=(lambda a, y: (dict(x=a['x'], w=a['w'], bias=a['bias'], residual=a['residual']), dict(out=y),
                                    dict(pre=a['pre'], post=a['post'], round=bool(a['round_to_tf32']))), lambda a: a['out']),
        mq_attention=(lambda a, y: (dict(q=a['q'], kv=a['kv'], null_kv=a['null_kv'], ckv=a['ckv']), dict(out=y),
                                    dict(heads=a['heads'], dh=a['dh'])), lambda a: None),
        cross_attention=(lambda a, y: (dict(q=a['q'], kvc=a['kvc'], null_kv=a['null_kv']), dict(out=y), dict(heads=a['heads'], dh=a['dh'])),
                         lambda a: None),
        gca_pool=(lambda a, y: (dict(x=a['x'], wk=a['wk'], bk=a['bk']), dict(out=y), {}), lambda a: None),
        gate_mlp_residual=(lambda a, y: (dict(h=a['h'], hid=a['hid'], w2=a['w2'], b2=a['b2'], res=a['res']), dict(out=y), {}), lambda a: None),
        gate_residual=(lambda a, y: (dict(h=a['h'], gate=a['gate'], res=a['res']), dict(out=y), {}), lambda a: a['out']),
        softmax_rows=(lambda a, y: (dict(x=a['x']), dict(out=y), dict(scale=float(a['scale']))), lambda a: a['out']),
        upsample2x=(lambda a, y: (dict(x=a['x']), dict(out=y), {}), lambda a: None),
        nchw_to_nhwc=(lambda a, y: (dict(src=a['src']), dict(out=a['dst'][..., a['c_off']:a['c_off'] + a['src'].shape[1]]),
                                    dict(round=bool(a['round_to_tf32']), c_off=a['c_off'])),
                      lambda a: a['dst'][..., a['c_off']:a['c_off'] + a['src'].shape[1]]),
        nhwc_to_nchw=(lambda a, y: (dict(src=a['src']), dict(out=y), {}), lambda a: None),
        im2col4=(lambda a, y: (dict(x=a['x']), dict(out=y), dict(kh=a['kh'], kw=a['kw'], pad=a['pad'])), lambda a: None),
        concat2=(lambda a, y: (dict(a=a['a'], b=a['b']), dict(out=y), dict(scale_b=float(a['scale_b']))), lambda a: a['out']),
        pixel_shuffle_silu=(lambda a, y: (dict(y=a['y']), dict(out=y), {}), lambda a: a['out']),
        time_fourier=(lambda a, y: (dict(t=a['t'], w=a['w']), dict(out=y), {}), lambda a: None),
    )


PLMS_CALLS = ('sfb_plms_update_rows', 'sfb_plms_update_rows_cfg')


class Recorder:
    """``with Recorder() as r: <model evaluation>`` -> ``r.recs`` (front-end launches in issue order), ``r.unchecked`` (C ABI launches
    that bypass the front ends: (name, kernels, traced names)) and ``r.calls`` (every C ABI call made outside a front end, as a ``Call``;
    the pointers named in ``BY_VALUE`` replaced by a copy of what they point to).  ``family`` labels the records; ``captured_only`` passes
    launches outside a graph capture straight through (UnetGraph's eager warm-up).  ``unattributed`` collects traced kernel names that no
    record or listed launch accounts for.

    ``sampler=True`` records the sampler's update launches (``PLMS_CALLS``) only and passes everything else through.  Their operands are
    raw pointers; ``_lib.fptr`` is wrapped to map each pointer back to the tensor it came from, and every operand is cloned right after
    the launch, in stream order: the eps operands may be the UNet graph's static output, which the next replay overwrites."""

    def __init__(self, family: str = '', captured_only: bool = False, trace: bool = True, sampler: bool = False):
        self.family = family
        self.captured_only = captured_only
        self.trace = trace
        self.sampler = sampler
        self.recs: List[Rec] = []
        self.unchecked = []
        self.calls: List[Call] = []
        self.unattributed = []
        self.depth = 0
        self._names_len = 0
        self._ptrs = {}

    # -- tracer: kernel names in launch order (host side, so it also names captured launches)
    def _new_names(self):
        from sparsefusion_b200 import _lib as lib
        if not self.trace:
            return []
        n = lib.load().sfb_trace_names(None, 0)
        buf = ctypes.create_string_buffer(n + 1)
        lib.load().sfb_trace_names(buf, n + 1)
        s = buf.value.decode()[self._names_len:]
        self._names_len = n
        return s.split('\n')[:-1]

    def _snapshot_overlapping(self, written: List[torch.Tensor], own: Optional[Rec] = None):
        """clone, before a launch that writes ``written``, every recorded tensor sharing bytes with it"""
        for r in self.recs + ([own] if own is not None else []):
            for k, t in r.t.items():
                if t is None or t is not r.orig.get(k):
                    continue
                if any(overlaps(t, w) for w in written):
                    r.t[k] = t.clone()
                    r.snapshots += 1

    def _snapshot_pointers(self, ptrs: List[int]):
        for r in self.recs:
            for k, t in r.t.items():
                if t is None or t is not r.orig.get(k) or not t.is_cuda:
                    continue
                if any(_holds(t, p) for p in ptrs):
                    r.t[k] = t.clone()
                    r.snapshots += 1

    def __enter__(self):
        from sparsefusion_b200 import _lib as lib, ops
        # torch.cuda.graph does not collect garbage before a capture, so the cyclic collector may free an earlier evaluation's CUDA
        # graphs inside one, which invalidates the capture; the recorder's own allocations make a collection inside a capture likely.
        # Collect here, outside any capture, and hold the collector off until __exit__, which frees what accumulated meanwhile.
        gc.collect()
        self._gc_was_enabled = gc.isenabled()
        gc.disable()
        self.saved = {} if self.sampler else {n: getattr(ops, n) for n in FRONT_ENDS}
        self.lib_call, self.lib_fptr = lib.call, lib.fptr
        specs = _specs()
        params = c_params()
        rec = self
        if self.trace:
            self._tbuf = torch.zeros(65, dtype=torch.int64, device='cuda')
            lib.call('sfb_trace_begin', self._tbuf.data_ptr(), 64)
            self._names_len = 0

        def wrap(name, orig):
            sig = inspect.signature(orig)
            spec, given_out = specs[name]

            def f(*args, **kw):
                if rec.depth or (rec.captured_only and not torch.cuda.is_current_stream_capturing()):
                    return orig(*args, **kw)
                a = sig.bind(*args, **kw)
                a.apply_defaults()
                a = a.arguments
                pre = given_out(a)
                inputs_pre = spec(a, pre)[0]
                own = Rec(name, dict(inputs_pre), (), {})
                prefill = None
                arena = ops._arena
                in_arena = (name == 'conv2d_nhwc' and pre is not None and isinstance(arena, ops.ZeroArena)
                            and storage_of(pre) == storage_of(arena.buf))
                if pre is not None:
                    # in place: the launch's own operands and earlier records' tensors that it overwrites are cloned first
                    rec._snapshot_overlapping([pre], own)
                    if name == 'conv2d_nhwc' and a['accumulate'] and not in_arena:
                        prefill = pre.clone()
                rec._pending()
                n0 = ops.launch_count()
                rec.depth += 1
                try:
                    y = orig(*args, **kw)
                finally:
                    rec.depth -= 1
                inputs, outputs, scal = spec(a, y)
                t = dict(own.t)
                t.update(outputs)
                r = Rec(name, t, tuple(outputs), scal, stream=torch.cuda.current_stream().cuda_stream,
                        captured=torch.cuda.is_current_stream_capturing(), family=rec.family, label=_label(), snapshots=own.snapshots,
                        orig=dict(inputs, **outputs))
                r.kernels = ops.launch_count() - n0
                r.names = rec._new_names()
                r.s['precision'] = ops.get_precision()
                if name == 'conv2d_nhwc':
                    out = outputs['out']
                    # an arena slice: pre-zeroed once per evaluation, reduced into in accumulate mode (linear_tc passes it as ``out``)
                    took_arena = pre is None and isinstance(arena, ops.ZeroArena) and storage_of(out) == storage_of(arena.buf)
                    r.s['arena'] = in_arena or took_arena
                    r.s['accumulate'] = scal['accumulate'] or took_arena      # the flag the kernel ran with
                    if prefill is not None:
                        t['prefill'] = prefill
                        r.orig['prefill'] = prefill
                    al = [n for x_, y_, n in ((a['x'], out, 'x=out'), (a['residual'], out, 'res=out'), (a['x'], a['residual'], 'x=res'))
                          if x_ is not None and y_ is not None and overlaps(x_, y_)]
                    if prefill is not None:
                        al.append('accumulate')
                    r.alias = ','.join(al)
                elif pre is not None and any(overlaps(v, pre) for v in inputs.values() if v is not None):
                    r.alias = 'x=out'
                rec.recs.append(r)
                return y
            return f

        for n, f in self.saved.items():
            setattr(ops, n, wrap(n, f))

        def call(name, *args):
            if rec.sampler:
                if name not in PLMS_CALLS:
                    return rec.lib_call(name, *args)
                rec._new_names()                  # the UNet's own launches (capture, eager time features) pass through
                n0 = ops.launch_count()
                rec.lib_call(name, *args)
                rec.recs.append(rec._plms_rec(name, args, ops.launch_count() - n0))
                return
            if rec.depth or (rec.captured_only and not torch.cuda.is_current_stream_capturing()):
                return rec.lib_call(name, *args)
            a = dict(zip(params[name], args))
            for k, n in BY_VALUE.items():
                if a.get(k) is not None:
                    a[k] = device_floats(a[k], n(a))
            rec.calls.append(Call(name, a, rec.family, len(rec.recs)))
            rec._snapshot_pointers([p for p in args if isinstance(p, int) and p > (1 << 32)])
            rec._pending()
            n0 = ops.launch_count()
            rec.lib_call(name, *args)
            k = ops.launch_count() - n0
            if k:
                rec.unchecked.append((name, k, rec._new_names()))
        def fptr(t, name='tensor'):
            p = rec.lib_fptr(t, name)
            if p is not None:
                rec._ptrs[p] = t
            return p
        lib.call = call
        if self.sampler:
            lib.fptr = fptr
        return self

    def _pending(self):
        """traced names of launches made since the last record: pass-through ones outside a capture, else unaccounted for"""
        names = self._new_names()
        if not self.captured_only:
            self.unattributed += names

    def _plms_rec(self, name, a, kernels):
        """``sfb_plms_update_rows`` / ``_cfg`` as a record whose operands are cloned right after the launch"""
        cfg = name == 'sfb_plms_update_rows_cfg'
        if cfg:
            (x, e0, en, cs, e1, e2, e3, c0, c1, c2, c3, z, sc, clip, out, eo, b, row_len, _) = a
            ptrs = dict(x=x, e0=e0, e_null=en, e1=e1, e2=e2, e3=e3, noise=z, scalars=sc, out=out, e_out=eo)
        else:
            (x, e0, e1, e2, e3, c0, c1, c2, c3, z, sc, clip, out, x0, b, row_len, _) = a
            ptrs = dict(x=x, e0=e0, e1=e1, e2=e2, e3=e3, noise=z, scalars=sc, out=out)
            cs = 1.0
        t = {}
        for k, p in ptrs.items():
            if p is None:
                t[k] = None
                continue
            w = 5 if k == 'scalars' else row_len
            t[k] = self._ptrs[p].reshape(-1)[:b * w].view(b, w).clone()
        outs = ('out', 'e_out') if cfg and eo is not None else ('out',)
        return Rec('plms_update_rows_cfg' if cfg else 'plms_update_rows', t, outs,
                   dict(coefs=(c0, c1, c2, c3), clip=float(clip), cond_scale=float(cs), rows=b, row_len=row_len),
                   stream=torch.cuda.current_stream().cuda_stream, family=self.family, label=name, kernels=kernels,
                   names=self._new_names())

    def __exit__(self, *exc):
        from sparsefusion_b200 import _lib as lib, ops
        for n, f in self.saved.items():
            setattr(ops, n, f)
        lib.call, lib.fptr = self.lib_call, self.lib_fptr
        if self._gc_was_enabled:
            gc.enable()
        gc.collect()
        if self.trace:
            if not self.sampler:
                self._pending()
            lib.call('sfb_trace_end')
        return False


def _label():
    import os
    import sys
    f = sys._getframe(2)
    while f is not None and os.path.basename(f.f_code.co_filename) in ('ops.py', 'insitu.py'):
        f = f.f_back
    if f is None:
        return '?'
    name = f.f_locals.get('name', f.f_locals.get('pfx', ''))
    return f'{os.path.basename(f.f_code.co_filename)}:{f.f_code.co_name}' + (f'({name})' if isinstance(name, str) and name else '')


# ------------------------------------------------------------------------------------------------ replay catalogues
class Catalogue:
    """the ``rec(family)`` that oracle/model_runs enters around each family, building a replay test's catalogue: per family a
    ``Recorder(family, trace=False)``; on exit its records and calls, in issue order, go through ``entry`` (a dict of the launch's
    geometry and scalars with its family and label, or None for a launch the test does not replay), equal entries are counted in
    ``calls``, and the records are dropped, so no family's tensors stay alive while the next one runs.  ``entries``: key -> entry, in
    order of first appearance."""

    def __init__(self, entry):
        self.entry = entry
        self.entries = {}
        self.family = None

    def __call__(self, family):
        self.family = family
        return self

    def __enter__(self):
        self.rec = Recorder(self.family, trace=False).__enter__()
        return self

    def __exit__(self, *exc):
        rec, self.rec = self.rec, None
        rec.__exit__(*exc)
        torch.cuda.synchronize()
        self.add(rec.recs, rec.calls)
        return False

    def add(self, recs: List[Rec], calls: List[Call]) -> None:
        # a call made after the first ``at`` records sorts between record at - 1 and record at
        issued = sorted([(i + 0.5, r) for i, r in enumerate(recs)] + [(c.at, c) for c in calls], key=lambda p: p[0])
        for _, r in issued:
            e = self.entry(r)
            if e is None:
                continue
            key = tuple(sorted((k, v) for k, v in e.items() if k != 'label'))
            self.entries.setdefault(key, dict(e, calls=0))['calls'] += 1


# ------------------------------------------------------------------------------------------------ poison
def poison(recs: List[Rec]) -> None:
    """NaN into exactly the elements of every recorded output view (and of the clones that stand for them); nothing between C and a
    row stride, nothing outside the views"""
    with torch.no_grad():
        for r in recs:
            for k in r.outs:
                r.orig[k].fill_(NAN)
                if r.t[k] is not r.orig[k]:
                    r.t[k].fill_(NAN)


def poison_allocator(device='cuda') -> None:
    """leave NaN in every size class the caching allocator is likely to hand out next (blocks allocated, filled and freed)"""
    blocks = []
    for mb in (0.001, 0.004, 0.016, 0.06, 0.25, 1, 2, 4, 8, 16, 32, 64, 128, 256):
        for _ in range(6):
            blocks.append(torch.full((max(1, int(mb * (1 << 20) // 4)),), NAN, device=device))
    torch.cuda.synchronize()
    del blocks


# ------------------------------------------------------------------------------------------------ provenance
def plan_storages(*objs) -> set:
    """storages of every tensor reachable from the objects (modules: parameters, buffers and attributes such as the prepared plans)"""
    seen, out = set(), set()

    def walk(o, depth):
        if id(o) in seen or depth > 6:
            return
        seen.add(id(o))
        if isinstance(o, torch.Tensor):
            out.add(storage_of(o))
        elif isinstance(o, dict):
            for v in o.values():
                walk(v, depth + 1)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v, depth + 1)
        elif isinstance(o, torch.nn.Module) or type(o).__module__.startswith(('sparsefusion_b200', 'oracle')):
            if isinstance(o, torch.nn.Module):
                for t in list(o.parameters()) + list(o.buffers()):
                    out.add(storage_of(t))
            for v in vars(o).values():
                walk(v, depth + 1)
    for o in objs:
        walk(o, 0)
    return out


def provenance(recs: List[Rec], plans: set) -> List[str]:
    """every GEMM record: its bias from a prepared plan; its packed / split weights from a prepared plan unless ``dynamic_weights``; with
    ``dynamic_weights`` a weight that an earlier record of ``recs`` wrote.  Returns one line per violation."""
    bad = []
    for i, r in enumerate(recs):
        if r.op != 'conv2d_nhwc':
            continue
        earlier = [(j, q, q.orig[k]) for j, q in enumerate(recs[:i]) for k in q.outs]
        b = r.orig.get('bias')
        if b is not None and (storage_of(b) not in plans or any(overlaps(b, o) for _, _, o in earlier)):
            bad.append(f'#{i} {r.label}: bias is not a prepared parameter (read before griddepcontrol.wait)')
        for k in ('w_packed', 'w_split'):
            w = r.orig.get(k)
            if w is None or r.s['dyn']:
                continue
            if storage_of(w) not in plans or any(overlaps(w, o) for _, _, o in earlier):
                bad.append(f'#{i} {r.label}: {k} is not a prepared weight but dynamic_weights is off (read before griddepcontrol.wait)')
        if r.s['dyn'] and not any(overlaps(r.orig['w_packed'], o) for _, _, o in earlier):
            bad.append(f'#{i} {r.label}: dynamic_weights set on a weight no earlier launch of the evaluation wrote')
    return bad


# ------------------------------------------------------------------------------------------------ checker
def _compare(got: torch.Tensor, ref: torch.Tensor, bnd: Optional[torch.Tensor]):
    """(ratio tensor, bad mask); bnd None: bit-exact"""
    got = got.reshape(ref.shape)
    if bnd is None:
        same = got.float().contiguous().view(torch.int32) == ref.float().contiguous().view(torch.int32)
        r = torch.where(same, torch.zeros_like(got, dtype=torch.float64), torch.full_like(got, math.inf, dtype=torch.float64))
    else:
        r = (got.double() - ref).abs() / (bnd + ATOL)
        r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return r, r > 1


def _rows(t):
    return t.reshape(-1, t.shape[-1])


def _nhw_c(t):
    return t.reshape(t.shape[0], -1, t.shape[-1])


def reference(r: Rec, sm: int = 132):
    """[(output name, got, ref, bound or None for bit-exact)] of one record"""
    T, s, op = r.t, r.s, r.op
    prec = s.get('precision', 'tf32x3')
    if op == 'conv2d_nhwc':
        x, wp = T['x'], T['w_packed']
        NB, H, W, Cin = x.shape
        Cout, KH, KW = s['cout'], s['kh'], s['kw']
        cin_pad = (Cin + 31) // 32 * 32
        w = wp.reshape(Cout, KH, KW, cin_pad)[..., :Cin].permute(0, 3, 1, 2)
        prefill = T.get('prefill')
        if s.get('arena'):
            prefill = torch.zeros_like(T['out'])
        y, C, A = cf.conv_ref(x, w, T['bias'], T['residual'], prefill, s['stride'], s['pad'], s['pad_after'])
        plan = cf.launch_plan(NB, H, W, Cin, Cout, KH, KW, s['stride'], s['pad'], s['pad_after'], s['splits'], s['bn'], prec, 2,
                              T['w_split'] is not None, sm)
        r.s['plan_kernel'], r.s['plan_splits'] = plan['kernel'], plan['splits']
        return [('out', T['out'], y, cf.bound(plan, prec, C, A, w_rounded=not s['dyn']))]
    if op == 'groupnorm':
        x = T['x']
        NB, HW, C = x.shape[0], x.shape[1] * x.shape[2], x.shape[3]
        plan = sf.kernel_plan('groupnorm', dict(NB=NB, HW=HW, C=C, G=s['groups']), sm, precision=prec)
        film = T['film']
        y, b = sf.ref_groupnorm(_nhw_c(x), s['groups'], T['gamma'].reshape(-1), T['beta'].reshape(-1), film, s['silu'], plan, prec, s['eps'])
        return [('out', _nhw_c(T['out']), y, b)]
    if op == 'layernorm':
        res = T['residual']
        y, b = sf.ref_layernorm(_rows(T['x']), T['g'].reshape(-1), None if T['b'] is None else T['b'].reshape(-1),
                                None if res is None else _rows(res), s['pre_gelu'], s['round'], prec)
        return [('out', _rows(T['out']), y, b)]
    if op == 'linear_small':
        res = T['residual']
        y, b = sf.ref_linear_small(_rows(T['x']), T['w'], T['bias'], None if res is None else _rows(res), s['pre'], s['post'], s['round'], prec)
        return [('out', _rows(T['out']), y, b)]
    if op == 'mq_attention':
        q = T['q']
        plan = sf.kernel_plan('mq_attention', dict(B=q.shape[0], n=q.shape[1], heads=s['heads'], dh=s['dh'],
                                                   nc=0 if T['ckv'] is None else T['ckv'].shape[1]), sm)
        y, b = sf.ref_mq_attention(q, T['kv'], T['null_kv'], T['ckv'], s['heads'], s['dh'], plan, prec)
        return [('out', T['out'], y, b)]
    if op == 'cross_attention':
        y, b = sf.ref_cross_attention(T['q'], T['kvc'], T['null_kv'], s['heads'], s['dh'], prec)
        return [('out', T['out'], y, b)]
    if op == 'gca_pool':
        x = T['x']
        plan = sf.kernel_plan('gca_pool', dict(HW=x.shape[1] * x.shape[2], C=x.shape[3]), sm)
        y, b = sf.ref_gca_pool(_nhw_c(x), T['wk'].reshape(-1), T['bk'].reshape(-1), plan)
        return [('out', T['out'], y, b)]
    if op == 'gate_mlp_residual':
        hid = T['hid']
        y, b = sf.ref_gate_mlp_residual(_nhw_c(T['h']), hid.reshape(T['h'].shape[0], -1), T['w2'], T['b2'], _nhw_c(T['res']))
        return [('out', _nhw_c(T['out']), y, b)]
    if op == 'gate_residual':
        y, b = sf.ref_gate_residual(_nhw_c(T['h']), T['gate'], _nhw_c(T['res']))
        return [('out', _nhw_c(T['out']), y, b)]
    if op == 'softmax_rows':
        y, b = sf.ref_softmax_rows(_rows(T['x']), s['scale'])
        return [('out', _rows(T['out']), y, b)]
    if op == 'time_fourier':
        y, b = sf.ref_time_fourier(T['t'], T['w'])
        return [('out', T['out'], y, b)]
    if op == 'pixel_shuffle_silu':
        y, b = sf.ref_pixel_shuffle_silu(T['y'])
        return [('out', T['out'], y, b)]
    if op == 'upsample2x':
        return [('out', T['out'], sf.upsample2x(T['x']), None)]
    if op == 'nchw_to_nhwc':
        from sparsefusion_b200 import ops
        ref = T['src'].permute(0, 2, 3, 1)
        if s['round'] and prec == 'tf32':
            ref = ops.round_tf32(ref.contiguous())
        return [('out', T['out'], ref, None)]
    if op == 'nhwc_to_nchw':
        return [('out', T['out'], T['src'].permute(0, 3, 1, 2), None)]
    if op == 'im2col4':
        x = T['x']
        k = (4 * s['kh'] * s['kw'] + 31) // 32 * 32
        return [('out', T['out'], sf.im2col4(x.contiguous(), s['kh'], s['kw'], s['pad'], k), None)]
    if op == 'concat2':
        ref = torch.cat((T['a'], T['b'] * s['scale_b']), -1)
        sb = s['scale_b']
        if sb != 0 and math.frexp(abs(sb))[0] == 0.5:
            return [('out', T['out'], ref, None)]
        rd = ref.double()
        return [('out', T['out'], rd, sf.U * rd.abs() + sf.ATOL)]
    if op in ('plms_update_rows', 'plms_update_rows_cfg'):
        e = [T['e0'], T['e1'], T['e2'], T['e3']]
        res = []
        if op == 'plms_update_rows_cfg':
            e[0] = st.cfg_eps(T['e0'], T['e_null'], s['cond_scale']).to(T['x'].device)
            if T.get('e_out') is not None:
                res.append(('e_out', T['e_out'], e[0], None))          # the guided eps in fp32, bit for bit
        r = st.ref_plms(T['x'], e, s['coefs'], T['scalars'], T['noise'], s['clip'])
        return [('out', T['out']) + r['x_prev']] + res
    raise KeyError(op)


def check(r: Rec, sm: int = 132) -> Report:
    worst, n_bad, n_nf, first, numel = 0.0, 0, 0, None, 0
    with torch.no_grad():
        for name, got, ref, bnd in reference(r, sm):
            ratio, bad = _compare(got, ref, bnd)
            numel += got.numel()
            n_nf += int((~torch.isfinite(got)).sum())
            nb = int(bad.sum())
            if nb and first is None:
                idx = int(bad.reshape(-1).nonzero()[0, 0])
                first = (name, tuple(int(i) for i in torch.unravel_index(torch.tensor(idx), tuple(bad.shape))))
            n_bad += nb
            if ratio.numel():
                worst = max(worst, float(ratio.max()))
    return Report(worst, n_bad, n_nf, first, numel)


def describe(i: int, r: Rec, rep: Report) -> str:
    where = 'side stream' if r.s.get('side') else 'main stream'
    return (f'#{i} {r.family} {r.op} {r.label} [{where}{", captured" if r.captured else ""}{", " + r.alias if r.alias else ""}'
            f'{", arena" if r.s.get("arena") else ""}{", dyn" if r.s.get("dyn") else ""}]: err/bound {rep.ratio:.3g}, {rep.n_bad} of {rep.numel} '
            f'out of bound, {rep.n_nonfinite} non-finite, first at {rep.first}')


# ------------------------------------------------------------------------------------------------ sampler history
def plms_expected_eps(outs: List[torch.Tensor], batch: List[int], guided: bool, cond_scale: float) -> List[Dict]:
    """the eps operands each round's update reads, built from the log of every replay's output ``outs[j]`` ([b_j] rows in the sampler's
    row order; guided [2 b_j]: the conditional rows, then the null rows), as p_sample assigns them (plms.py:_fused_loop): round 0 its own
    eps; round 1 the pseudo improved Euler pair, round 0's eps and its own; round j >= 2 its own eps and p_sample's history, newest first.
    The history holds round 0's eps after round 1 and round j's after round j >= 2.  A guided row's eps is the guided combination of its
    two halves in fp32.  Returns per round {operand name: [b_j, row_len] rows or None}."""
    flat = [o.reshape(o.shape[0], -1) for o in outs]
    E = [st.cfg_eps(o[:b], o[b:2 * b], cond_scale).to(o.device) if guided else o for o, b in zip(flat, batch)]
    exp, old = [], []
    for j, (o, b) in enumerate(zip(flat, batch)):
        if guided:
            d = dict(e0=o[:b], e_null=o[b:2 * b])
            hist = [] if j == 0 else ([E[0]] if j == 1 else old[::-1])
        else:
            lst = [E[0]] if j == 0 else ([E[0], E[1]] if j == 1 else [E[j]] + old[::-1])
            d, hist = dict(e0=lst[0]), lst[1:]
        for i in range(3):
            d[f'e{i + 1}'] = hist[i] if i < len(hist) else None
        exp.append({k: None if v is None else v[:b] for k, v in d.items()})
        if j >= 1:
            old = (old + [E[0] if j == 1 else E[j]])[-3:]
    return exp


def plms_history_mismatches(recs: List[Rec], expected: List[Dict]) -> List[str]:
    """every eps operand of each round's update record equal, bit for bit, to ``plms_expected_eps``"""
    bad = []
    if len(recs) != len(expected):
        return [f'{len(recs)} update records for {len(expected)} rounds']
    for j, (r, e) in enumerate(zip(recs, expected)):
        for k, want in e.items():
            got = r.t.get(k)
            if (got is None) != (want is None):
                bad.append(f'round {j}: {k} is {"NULL" if got is None else "set"}, p_sample assigns {"none" if want is None else "one"}')
            elif got is not None and not torch.equal(got.float().contiguous().view(torch.int32),
                                                     want.to(got.device).float().contiguous().view(torch.int32)):
                bad.append(f'round {j}: {k} differs from the replay log in {int((got != want.to(got.device)).sum())} elements')
    return bad
