"""coach_b200.utils.graph_capture: a CUDA-graph capture that Python's cyclic garbage collector cannot interrupt.  Dead
agents are often reference cycles that hold pinned staging buffers; freeing such a buffer records a CUDA event on the
stream of its last asynchronous copy, which must not happen while a capture is in progress."""
import gc
import weakref

import pytest
import torch

pytestmark = pytest.mark.gpu


class _Cycle(object):
    """a dead agent in miniature: a reference cycle holding a pinned buffer that served an asynchronous copy"""

    def __init__(self):
        self.me = self
        self.host = torch.ones(1024, pin_memory=True)
        self.dev = torch.zeros(1024, device="cuda")
        self.dev.copy_(self.host, non_blocking=True)


def test_garbage_is_collected_before_and_held_off_during_the_capture():
    from coach_b200.utils import graph_capture
    x = torch.zeros(16, device="cuda")
    dead = weakref.ref(_Cycle())
    assert dead() is not None                     # only the collector frees it
    seen = {}
    g = torch.cuda.CUDAGraph()
    with graph_capture(g):
        seen["collected"] = dead() is None
        seen["enabled"] = gc.isenabled()
        x.add_(1.0)
    assert seen == {"collected": True, "enabled": False}
    assert gc.isenabled()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert float(x.sum()) == 32.0


def test_collector_state_is_restored_when_the_capture_raises():
    from coach_b200.utils import graph_capture
    x = torch.zeros(1, device="cuda")
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="inside"):
        with graph_capture(g):
            x.add_(1.0)
            raise RuntimeError("inside")
    assert gc.isenabled()
    gc.disable()
    try:
        with graph_capture(torch.cuda.CUDAGraph()):
            x.add_(1.0)
        assert not gc.isenabled()                 # a caller's disabled collector stays disabled
    finally:
        gc.enable()
