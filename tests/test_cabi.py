"""CPU-only checks of the C-ABI boundary: the library builds for sm_90a, loads, and exports every symbol that
include/coach_b200.h declares; the ctypes table in coach_b200/_lib.py covers the same set.  No compute calls."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "coach_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cb200_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    from coach_b200 import build, _lib
    build.build()
    lib = _lib.load()
    names = header_symbols()
    assert len(names) >= 10
    for name in names:
        assert hasattr(lib, name), "libcoach_b200.so does not export %s" % name
    assert lib.cb200_abi_version() == 1


def test_ctypes_table_matches_header():
    from coach_b200 import _lib
    assert sorted(_lib.PROTOTYPES.keys()) == header_symbols()


def test_only_sm90a_code_in_library():
    import subprocess
    from coach_b200 import build
    out = subprocess.run(["cuobjdump", "-lelf", build.build()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_argument_errors_surface_as_valueerror():
    # argument validation happens before any CUDA call, so this is safe without a GPU
    from coach_b200 import _lib
    lib = _lib.load()
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_per_init(None, None, None, None, 8, None))
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_per_sample(1, 1, 12, 1, 4, 4, 0.4, 1, None, None, None))   # size not a power of two
    assert b"power of 2" in lib.cb200_last_error()


def test_tiled_gemm_argument_validation():
    """cb200_gemm_tiled / cb200_split_planes / cb200_scatter_ring_packed reject bad geometry before touching the GPU"""
    import ctypes
    from coach_b200 import _lib
    lib = _lib.load()
    d = _lib.TGemmDesc()
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_gemm_tiled(None, None))
    d.mode, d.batch = 0, 48                                    # not a multiple of 32
    d.a_planes, d.b_planes, d.c = 256, 512, 1024
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_gemm_tiled(ctypes.byref(d), None))
    assert b"batch" in lib.cb200_last_error()
    d.batch, d.a_cols, d.n, d.ldc = 64, 48, 64, 64             # 48 channels: not 32 / 64 / 128 / k*128
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_gemm_tiled(ctypes.byref(d), None))
    assert b"a_cols" in lib.cb200_last_error()
    d.a_cols, d.n = 64, 48                                     # n must be 32 or a multiple of 64
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_gemm_tiled(ctypes.byref(d), None))
    d.n, d.ldc, d.a_num_planes = 64, 64, 1                     # one plane = uint8 operand: needs the divisor
    d.a_rows, d.b_rows = 64, 64
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_gemm_tiled(ctypes.byref(d), None))
    assert b"a_u8_div" in lib.cb200_last_error()
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_split_planes(None, None, 8, None, 0, 0, None))
    cols = (_lib.Column * 1)()
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_scatter_ring_packed(cols, 1, 0, 0, 16, 1, None))     # stride 0
    with pytest.raises(ValueError):
        _lib.check(lib.cb200_u8_s2d_planes(256, 12, 84, 84, 4, 4, 512, None))      # batch not a multiple of 8


def test_plane_format_helpers_roundtrip():
    """host-side mirror of csrc/nn_gemm.cuh tiled_elem: PlaneBuf.to_dense inverts the core-tiled layout"""
    import numpy as np
    import torch
    from coach_b200.architectures import tiled as tl
    rows, cols = 24, 16
    buf = tl.PlaneBuf(rows, cols, "cpu")
    want = torch.arange(rows * cols, dtype=torch.float32).reshape(rows, cols)     # exactly representable in bf16? no:
    want = (want % 128)                                                           # keep 8 significant bits
    flat = torch.zeros(rows * cols)
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    elem = ((r // 8) * (cols // 8) + c // 8) * 64 + (r % 8) * 8 + c % 8
    flat[torch.from_numpy(elem.reshape(-1))] = want.reshape(-1)
    buf.t[0] = flat.to(torch.bfloat16)
    assert torch.equal(buf.to_dense(), want)
    assert tl.channels_ok(64) and tl.channels_ok(256) and not tl.channels_ok(48) and not tl.channels_ok(192 + 8)
    assert tl.width_ok(32) and tl.width_ok(512) and not tl.width_ok(16) and not tl.width_ok(96)
    assert tl.pick_splits_tiled(4, 1296) >= 41          # at most 32 chunks per slice


def test_removed_tune_key_is_rejected():
    # "gemm_persistent" selected a schedule that no longer exists: an error, not a silently ignored switch
    from coach_b200 import _lib
    lib = _lib.load()
    assert lib.cb200_tune(b"gemm_persistent", 1) == -1
    assert b"gemm_persistent" in lib.cb200_last_error()
    assert lib.cb200_tune(b"gemm_tc", 1) == 0
