"""helpers shared by the GPU tests"""
import ctypes

import torch

from oracle.conv_fp64 import slice_guard_intact

GUARD = 256             # floats before and after every replay buffer (1 KB keeps every tensor 16-byte aligned)
NAN = float('nan')


def device_level_scales(geo):
    """per-level grid scales exactly as the device computes them (exp2f on the GPU; gridencoder.cu:125)"""
    from sparsefusion_b200 import _lib as lib
    s = torch.empty(geo['L'], device='cuda')
    lib.call('sfb_grid_level_scales', geo['L'], float(geo['S']), geo['H'], lib.fptr(s), lib.stream())
    return s.cpu().numpy()


# ------------------------------------------------------------------------------------------------ per-launch replays
class Tracer:
    """the names of the library kernels a replay launches, in launch order"""

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


_ALIVE = []     # the current replay's input buffers: the C ABI takes raw pointers, so the buffers must outlive the launch


def release():
    """free the input buffers of the previous replay"""
    _ALIVE.clear()


def guarded(t, ld=None, off=0):
    """``t`` inside a NaN buffer [GUARD | rows x ld | GUARD]: its rows [rows, t.shape[-1]] at channel ``off`` of rows of ``ld`` floats
    (default: packed), NaN in the channels between.  Returns the view holding ``t``, shaped like it (None passes through); the buffer lives
    until ``release()``."""
    if t is None:
        return None
    w = t.shape[-1]
    rows = t.numel() // w
    ld = ld or w
    buf = torch.full((rows * ld + 2 * GUARD,), NAN, device='cuda')
    _ALIVE.append(buf)
    body = buf[GUARD:GUARD + rows * ld].view(rows, ld)
    body[:, off:off + w] = t.reshape(rows, w)
    return body[:, off:off + w].view(t.shape)


def ptr(t):
    return None if t is None else t.data_ptr()


class Out:
    """an output slot: ``rows`` rows of ``ld`` floats with the result at channel ``off`` (``width`` floats per row), between GUARD floats.
    Every float outside the slot is random with NaN in every other one, so stray stores and stray adds both change its bits; the slot holds
    ``prefill`` (in-place and accumulating launches) or NaN before the launch."""

    def __init__(self, rows, width, ld=None, off=0, seed=0, prefill=None):
        ld = ld or width
        g = torch.Generator(device='cuda').manual_seed(seed + rows * 7 + ld)
        self.rows, self.ld, self.off, self.width = rows, ld, off, width
        self.buf = torch.randn(rows * ld + 2 * GUARD, device='cuda', generator=g)
        self.buf[::2] = NAN
        self.body = self.buf[GUARD:GUARD + rows * ld].view(rows, ld)
        self.slot = self.body[:, off:off + width]
        self.slot[:] = NAN if prefill is None else prefill.reshape(rows, width)
        self.before = self.buf.clone()
        self.ptr = self.slot.data_ptr()

    def value(self):
        return self.slot.clone()

    def guard_ok(self):
        """every float outside the slot bit-identical: the leading and trailing guards, the rows' other channels (``slice_guard_intact``)"""
        b, a = self.before.view(torch.int32), self.buf.view(torch.int32)
        keep = torch.ones_like(self.buf, dtype=torch.bool)
        keep[GUARD:GUARD + self.rows * self.ld].view(self.rows, self.ld)[:, self.off:self.off + self.width] = False
        return (torch.equal(b[:GUARD], a[:GUARD]) and torch.equal(b[-GUARD:], a[-GUARD:]) and torch.equal(b[keep], a[keep])
                and slice_guard_intact(self.before[GUARD:-GUARD].view(self.rows, -1), self.buf[GUARD:-GUARD].view(self.rows, -1), self.off,
                                       self.width))
