"""GPU benchmark (not a test): a windowed aggregation with and without watermark-driven state cleaning.

Workload per epoch: 2^19 bid rows (auction, price, date_time) with date_time advancing one second per epoch ->
rwgpu_project_device computes tumble_start(date_time, 2 s) -> HashAgg grouped by (window, auction) with count(*) and
max(price) (append-only) -> the barrier, launched and collected one epoch later as in bench.py's agg leg.  The `wm` arm
calls rwgpu_agg_update_watermark(window key, start of the current window) before every barrier; the `none` arm runs the
same stream without it.  The two arms alternate in one process.

Per arm: rows / s over the wall time of the whole stream (inputs already in HBM; the wall time includes the per-barrier
checksum read-back, alike in both arms), p50 of the device time of one barrier (CUDA events
around rwgpu_agg_flush_device_async: the delta and, in the `wm` arm, the cleaning), the final group count and table
capacity (rwgpu_agg_stats), and `verified`: the checksum of every delta row summed over the stream equals that of the
groups of a CPU restatement (numpy group-by over every row).  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from risingwave_b200 import abi, device  # noqa: E402
from risingwave_b200.executor import AggCall, Backend, HashAggExecutor, MockSource, ProjectExecutor  # noqa: E402

M64 = (1 << 64) - 1
SECOND = 1_000_000
WINDOW = 2 * SECOND
WEIGHTS = (3, 5, 7, 11)  # window, auction, count, max


def gen(epochs, rows, auctions, seed):
    rng = np.random.default_rng(seed)
    out = []
    for e in range(epochs):
        auction = rng.integers(0, auctions, rows, dtype=np.int64)
        price = rng.integers(1, 10**7, rows, dtype=np.int64)
        dt = e * SECOND + np.sort(rng.integers(0, SECOND, rows, dtype=np.int64))
        out.append((auction, price, dt))
    return out


def restatement_checksum(data):
    """checksum of the final groups: count(*) and max(price) per (tumble_start(date_time), auction)"""
    win = np.concatenate([d[2] for d in data]) // WINDOW * WINDOW
    auc = np.concatenate([d[0] for d in data])
    price = np.concatenate([d[1] for d in data])
    key = win * (1 << 20) + auc
    order = np.argsort(key, kind="stable")
    k, first, cnt = np.unique(key[order], return_index=True, return_counts=True)
    mx = np.maximum.reduceat(price[order], first)
    w, a = k >> 20, k & ((1 << 20) - 1)
    acc = (w.astype(np.uint64) * np.uint64(WEIGHTS[0]) + a.astype(np.uint64) * np.uint64(WEIGHTS[1])
           + cnt.astype(np.uint64) * np.uint64(WEIGHTS[2]) + mx.astype(np.uint64) * np.uint64(WEIGHTS[3]))
    return len(k), int(acc.sum(dtype=np.uint64)) & M64


def stats(be, ex):
    fn = be.lib.rwgpu_agg_stats
    fn.restype, fn.argtypes = C.c_int32, [C.c_void_p] + [C.POINTER(C.c_uint64)] * 3
    g, cap, n = C.c_uint64(), C.c_uint64(), C.c_uint64()
    be.check(fn(ex._h, C.byref(g), C.byref(cap), C.byref(n)))
    return g.value, cap.value


def run_arm(be, dev_data, with_wm, hint):
    T3 = [abi.T_INT64, abi.T_INT64, abi.T_TIMESTAMP]
    _, s0 = MockSource.channel()
    proj = ProjectExecutor(be, s0.into_executor(T3, []), [f"(tumble_start:timestamp $2:timestamp {WINDOW}:int8)"])
    _, s1 = MockSource.channel()
    agg = HashAggExecutor(be, s1.into_executor([abi.T_TIMESTAMP, abi.T_INT64, abi.T_INT64], []), True,
                          [AggCall.from_pretty("(count:int8)"), AggCall.from_pretty("(max:int8 $2:int8)")], 0, [0, 1],
                          group_capacity_hint=hint)
    st = torch.cuda.Stream()
    ops = torch.ones(dev_data[0][0].numel(), dtype=torch.uint8, device="cuda")
    ev = []
    acc_sum = 0
    keep = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.cuda.stream(st):
        for e, (auction, price, dt) in enumerate(dev_data):
            bid = device.DeviceChunk(ops, [auction, price, dt], T3)
            cols, _, _ = device.project_device(bid, proj._exprs, proj.schema, st)
            ach = device.DeviceChunk(ops, [cols[0], auction, price], [abi.T_TIMESTAMP, abi.T_INT64, abi.T_INT64])
            keep.append((bid, cols, ach))
            device.agg_push_device(agg, ach, st)
            if with_wm:
                agg.update_watermark(0, e * SECOND // WINDOW * WINDOW)
            b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b0.record(st)
            device.agg_flush_device_async(agg, e + 1, st)
            b1.record(st)
            ev.append((b0, b1))
            if e >= 1:
                v = device.agg_flush_collect(agg, st)
                _, s = v.checksum(WEIGHTS)  # (verification: outside the device time of the barriers)
                acc_sum = (acc_sum + s) & M64
                keep = keep[-2:]
        v = device.agg_flush_collect(agg, st)
        _, s = v.checksum(WEIGHTS)
        acc_sum = (acc_sum + s) & M64
    st.synchronize()
    wall = time.perf_counter() - t0
    barrier_ms = sorted(a.elapsed_time(b) for a, b in ev)
    g, cap = stats(be, agg)
    return {"rows_per_s": sum(d[0].numel() for d in dev_data) / wall, "p50_barrier_ms": barrier_ms[len(barrier_ms) // 2],
            "n_groups": g, "capacity": cap, "checksum": acc_sum}


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=40)
    ap.add_argument("--rows", type=int, default=1 << 19)
    ap.add_argument("--auctions", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    be = Backend.cuda()
    data = gen(args.epochs, args.rows, args.auctions, 7)
    want_groups, want_sum = restatement_checksum(data)
    dev_data = [tuple(torch.from_numpy(c).cuda() for c in d) for d in data]
    hint = 2 * args.auctions  # sized for the live windows: the `none` arm grows past it
    res = {"wm": [], "none": []}
    for _ in range(args.reps):
        for arm in ("wm", "none"):
            res[arm].append(run_arm(be, dev_data, arm == "wm", hint))
    line = {"workload": f"Project(tumble_start 2 s) -> HashAgg by (window, auction) count(*), max(price); {args.epochs} epochs x "
                        f"{args.rows} rows, {args.auctions} auctions, 1 s of date_time per epoch",
            "device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "restatement_groups": want_groups}
    for arm, rs in res.items():
        line[arm] = {"rows_per_s": [round(r["rows_per_s"]) for r in rs], "p50_barrier_ms": [round(r["p50_barrier_ms"], 4) for r in rs],
                     "n_groups": rs[-1]["n_groups"], "capacity": rs[-1]["capacity"],
                     "verified": all(r["checksum"] == want_sum for r in rs)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
