"""Helpers of the C-ABI kernel tests (tests/test_head_kernels_gpu.py, tests/test_learn_kernels_gpu.py): the library
handle, bit-for-bit comparison, and device outputs followed by canary elements that must stay untouched."""
import numpy as np
import torch

GUARD = 64                                   # canary elements after every output
CANARY = {torch.float32: 0x7FA5A5A5, torch.float64: 0x7FF4A5A5A5A5A5A5, torch.int64: 0x5A5A5A5A5A5A5A5A,
          torch.int16: 0x5A5A}
INT_VIEW = {torch.float32: torch.int32, torch.float64: torch.int64, torch.int64: torch.int64, torch.int16: torch.int16}


def _lib():
    from coach_b200 import _lib as L
    return L, L.load()


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view({4: np.uint32, 8: np.uint64, 2: np.uint16, 1: np.uint8}[x.dtype.itemsize])


def assert_bits(got, want, name):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = _bits(got) != _bits(want.astype(got.dtype))
    assert not bad.any(), "%s: %d of %d differ, first at %s: got %r want %r" % (
        name, bad.sum(), bad.size, np.argwhere(bad)[0], got[tuple(np.argwhere(bad)[0])],
        want[tuple(np.argwhere(bad)[0])])


class Outs(object):
    """device outputs, each followed by GUARD canary elements that must stay untouched"""

    def __init__(self):
        self.t = {}

    def add(self, name, shape, dtype=torch.float32):
        n = int(np.prod(shape))
        full = torch.empty(n + GUARD, dtype=dtype, device="cuda")
        full.view(INT_VIEW[dtype]).fill_(CANARY[dtype])
        self.t[name] = (full, tuple(shape))
        return full.data_ptr()

    def numpy(self):
        torch.cuda.synchronize()
        out = {}
        for k, (full, shape) in self.t.items():
            n = int(np.prod(shape))
            tail = full[n:].view(INT_VIEW[full.dtype]).cpu().numpy()
            assert (tail == np.array(CANARY[full.dtype]).astype(tail.dtype)).all(), "%s: write past its end" % k
            out[k] = full[:n].cpu().numpy().reshape(shape)
        return out


def _dev(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()
