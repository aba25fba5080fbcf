"""Micro-benchmark of the memory-side kernels at BASELINE config 2 (2^20-leaf PER, 84x84x4 u8, B=512).
Times each kernel with CUDA events on the launching stream, flushing L2 between iterations (a 256 MB memset).
Sweeps the gather tuning knobs.  Prints JSON lines.  Usage: python tools/bench_replay.py [--capacity N]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from coach_b200 import _lib  # noqa: E402


def timed(fn, flush, iters=30, warmup=5):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1)                       # evict L2 (50 MB) with a 256 MB write
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    ts = np.array(ts)
    return float(np.median(ts)), float(ts.min()), float(ts.mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=1 << 18)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--quick", action="store_true", help="a few launches only (for ncu)")
    args = ap.parse_args()
    lib = _lib.load()
    dev = torch.device("cuda")
    size, B, cap = 1 << 20, args.batch, args.capacity
    row = 84 * 84 * 4
    rng = np.random.RandomState(0)
    trees = [torch.empty(2 * size - 1, dtype=torch.float64, device=dev) for _ in range(3)]
    winner = torch.empty(size, dtype=torch.int32, device=dev)
    _lib.check(lib.cb200_per_init(*[t.data_ptr() for t in trees], winner.data_ptr(), size, None))
    pr = torch.from_numpy(np.abs(rng.randn(size)) + 1e-6).to(dev)
    idx_all = torch.arange(size, dtype=torch.int64, device=dev)
    _lib.check(lib.cb200_per_update(*[t.data_ptr() for t in trees], winner.data_ptr(), size, idx_all.data_ptr(),
                                    (pr ** 0.6).data_ptr(), pr.data_ptr(), size, None, None, None))
    state = torch.randint(0, 256, (cap, row), dtype=torch.uint8, device=dev)
    nstate = torch.randint(0, 256, (cap, row), dtype=torch.uint8, device=dev)
    action = torch.randint(0, 6, (cap,), dtype=torch.int64, device=dev)
    reward = torch.randn(cap, dtype=torch.float64, device=dev)
    done = torch.zeros(cap, dtype=torch.uint8, device=dev)
    o_s = torch.empty((B, row), dtype=torch.uint8, device=dev)
    o_n = torch.empty_like(o_s)
    o_a = torch.empty(B, dtype=torch.int64, device=dev)
    o_r = torch.empty(B, dtype=torch.float64, device=dev)
    o_d = torch.empty(B, dtype=torch.uint8, device=dev)
    idx = torch.empty(B, dtype=torch.int64, device=dev)
    w = torch.empty(B, dtype=torch.float64, device=dev)
    w32 = torch.empty(B, dtype=torch.float32, device=dev)
    # priorities only on the first `cap` leaves so that sampled leaves are valid ring rows
    _lib.check(lib.cb200_per_init(*[t.data_ptr() for t in trees], winner.data_ptr(), size, None))
    _lib.check(lib.cb200_per_update(*[t.data_ptr() for t in trees], winner.data_ptr(), size, idx_all.data_ptr(),
                                    (pr ** 0.6).data_ptr(), pr.data_ptr(), cap, None, None, None))
    u = torch.rand(B, dtype=torch.float64, device=dev)
    arr, cnt = _lib.make_columns([(state.data_ptr(), o_s.data_ptr(), row), (nstate.data_ptr(), o_n.data_ptr(), row),
                                  (action.data_ptr(), o_a.data_ptr(), 8), (reward.data_ptr(), o_r.data_ptr(), 8),
                                  (done.data_ptr(), o_d.data_ptr(), 1)])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    alg_bytes = B * (2 * row + 8 + 8 + 1) * 2 + B * 21 * 8 + B * 16      # read + write + tree + idx/weight
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                            "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 6650.0)

    def fused():
        _lib.check(lib.cb200_per_sample_gather(trees[0].data_ptr(), trees[1].data_ptr(), size, u.data_ptr(), B,
                                               2 * cap, 0.4, idx.data_ptr(), w.data_ptr(), w32.data_ptr(), arr, cnt,
                                               None))

    def sample_only():
        _lib.check(lib.cb200_per_sample(trees[0].data_ptr(), trees[1].data_ptr(), size, u.data_ptr(), B, 2 * cap, 0.4,
                                        idx.data_ptr(), w.data_ptr(), w32.data_ptr(), None))

    def gather_only():
        _lib.check(lib.cb200_gather(arr, cnt, idx.data_ptr(), B, None))

    err = torch.rand(B, dtype=torch.float64, device=dev)
    pa = torch.empty(B, dtype=torch.float64, device=dev)
    praw = torch.empty(B, dtype=torch.float64, device=dev)
    maxp = torch.empty(1, dtype=torch.float64, device=dev)

    def update():
        _lib.check(lib.cb200_per_priorities_device(err.data_ptr(), B, 1e-6, 0.6, pa.data_ptr(), praw.data_ptr(), None,
                                                   None))
        _lib.check(lib.cb200_per_update(*[t.data_ptr() for t in trees], winner.data_ptr(), size, idx.data_ptr(),
                                        pa.data_ptr(), praw.data_ptr(), B, maxp.data_ptr(), None, None))

    def torch_copy():
        o_s.copy_(state[:B])
        o_n.copy_(nstate[:B])

    one = torch.zeros(1, dtype=torch.float64, device=dev)

    def tiny():
        _lib.check(lib.cb200_per_priorities_device(one.data_ptr(), 1, 1e-6, 0.6, one.data_ptr(), one.data_ptr(), None,
                                                   None))

    # burst timing: NB back-to-back launches on rotating inputs/outputs (outputs total > L2), one event pair
    NB = 16
    us_ = [torch.rand(B, dtype=torch.float64, device=dev) for _ in range(NB)]
    outs = []
    for _ in range(NB):
        bs, bn = torch.empty_like(o_s), torch.empty_like(o_n)
        outs.append((bs, bn, _lib.make_columns([(state.data_ptr(), bs.data_ptr(), row),
                                                (nstate.data_ptr(), bn.data_ptr(), row),
                                                (action.data_ptr(), o_a.data_ptr(), 8),
                                                (reward.data_ptr(), o_r.data_ptr(), 8),
                                                (done.data_ptr(), o_d.data_ptr(), 1)])))

    def burst(kind):
        def run():
            for k in range(NB):
                if kind == "fused":
                    _lib.check(lib.cb200_per_sample_gather(trees[0].data_ptr(), trees[1].data_ptr(), size,
                                                           us_[k].data_ptr(), B, 2 * cap, 0.4, idx.data_ptr(),
                                                           w.data_ptr(), w32.data_ptr(), outs[k][2][0], outs[k][2][1],
                                                           None))
                elif kind == "sample":
                    _lib.check(lib.cb200_per_sample(trees[0].data_ptr(), trees[1].data_ptr(), size,
                                                    us_[k].data_ptr(), B, 2 * cap, 0.4, idx.data_ptr(), w.data_ptr(),
                                                    w32.data_ptr(), None))
                elif kind == "tiny":
                    tiny()
                elif kind == "update":
                    update()
                else:
                    outs[k][0].copy_(state[k * B:(k + 1) * B])
                    outs[k][1].copy_(nstate[k * B:(k + 1) * B])
        return run

    sample_only()
    if args.quick:
        lib.cb200_tune(b"gather_stages", 0)
        lib.cb200_tune(b"gather_ctas_per_sm", 4)
        for _ in range(8):
            flush.fill_(1)
            fused()
            update()
        torch.cuda.synchronize()
        return
    for kind in ("tiny", "sample", "update", "torch_copy", "fused"):
        med, mn, mean = timed(burst(kind), flush, iters=10, warmup=2)
        print(json.dumps({"burst_of_16": kind, "us_per_call_median": round(med / NB, 2),
                          "us_per_call_min": round(mn / NB, 2)}))
    for name, fn in (("tiny_launch_baseline", tiny), ("per_sample", sample_only), ("gather", gather_only), ("per_update(+prio)", update),
                     ("torch_contiguous_copy_same_bytes", torch_copy)):
        med, mn, mean = timed(fn, flush)
        print(json.dumps({"kernel": name, "us_median": round(med, 2), "us_min": round(mn, 2)}))
    for persist in (0, 1):
        if persist:
            # top 17 levels of the sum tree (2^17 doubles = 1 MiB) + min-tree root stay L2 resident
            rc = lib.cb200_l2_persist(trees[0].data_ptr(), (1 << 17) * 8, None)
            print(json.dumps({"l2_persist_rc": rc}))
        for cps in (1, 2, 3, 4, 6, 8):
            lib.cb200_tune(b"gather_stages", 0)
            lib.cb200_tune(b"gather_ctas_per_sm", cps)
            med, mn, mean = timed(fused, flush)
            bmed, bmn, _ = timed(burst("fused"), flush, iters=8, warmup=2)
            print(json.dumps({"kernel": "per_sample_gather", "l2_persist": persist, "ctas_per_sm": cps,
                              "us_median": round(med, 2), "us_min": round(mn, 2),
                              "burst_us_per_call": round(bmed / NB, 2),
                              "GBps_burst": round(alg_bytes / (bmed / NB) / 1e3, 1),
                              "frac_of_measured_hbm_burst": round(alg_bytes / (bmed / NB) / 1e3 / hbm, 3)}))
        bmed, _, _ = timed(burst("sample"), flush, iters=8, warmup=2)
        print(json.dumps({"burst_of_16": "sample", "l2_persist": persist, "us_per_call_median": round(bmed / NB, 2)}))
        bmed, _, _ = timed(burst("update"), flush, iters=8, warmup=2)
        print(json.dumps({"burst_of_16": "update", "l2_persist": persist, "us_per_call_median": round(bmed / NB, 2)}))
    lib.cb200_l2_persist(None, 0, None)


if __name__ == "__main__":
    main()
