"""GPU benchmark (not a test): HashAgg behind the hash shuffle at N GPUs -- the aggregation half of the project's metric
past one GPU.  Run with `torchrun --nproc-per-node N tools/gpu/bench_agg_shuffle.py` (N = 1 is a self-peer exchange).

Per epoch and rank: one flat-exchange batch keyed on the group key (rwgpu_shuffle_exchange_flat_device), the counted
push of the receive buffer into the rank's HashAgg (rwgpu_agg_push_device_counted: the row count is read on the device),
then the barrier, launched and collected one epoch later as in bench.py's agg leg.  Exchange e + 2 reuses the receive
buffer of exchange e, so it waits on an event recorded after push e.

Inputs are bench.py's cfg2 variants A / B / R (SURVEY 8(d)).  At N = 1 the rows are byte-identical to bench.py's agg leg;
at N > 1 the load scales weakly: rank r generates 2^18 rows per epoch at its own row-index offset over 2^20 x N keys.
At N = 1 the plain rwgpu_agg_push_device of the same epochs (no exchange) is timed too, the two arms alternating in one
process: the difference is what going through the exchange costs.

Rank 0 prints one JSON line per variant.  `verified` compares the (delta rows, checksum) of the last epochs, summed over
ranks, with oracle/fastcpu.cc fed every rank's rows."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bench  # noqa: E402
from risingwave_b200 import abi, device, exchange  # noqa: E402
from risingwave_b200.executor import AggCall, Backend, HashAggExecutor, MockSource  # noqa: E402

ROWS = bench.AGG_EPOCH_ROWS
T2 = [abi.T_INT64] * 2
M64 = (1 << 64) - 1


def gen_epoch(variant, e, rank, world, prev):
    """(ops, key, price) of rank `rank`'s epoch e; at world 1 exactly bench.py's agg leg"""
    seed = {"A": bench.AGG_SEED, "B": bench.AGG_SEED + 1, "R": bench.AGG_SEED + 2}[variant]
    k, p = bench.gen_agg_rows(ROWS, (e * world + rank) * ROWS, seed, hot=(variant == "B"))
    ops = np.ones(ROWS, np.uint8)
    if variant == "R" and prev is not None:
        nd = ROWS // 10  # rows 0, 10, 20, ... retract row i of the rank's previous epoch (each at most once)
        sel = np.arange(nd) * 10
        live = prev[0][sel] == 1
        k[sel[live]], p[sel[live]] = prev[1][sel[live]], prev[2][sel[live]]
        ops[sel[live]] = 2
    return ops, k, p


def gen_all(variant, n_epochs, rank, world):
    out, prev = [], None
    for e in range(n_epochs):
        prev = gen_epoch(variant, e, rank, world, prev)
        out.append(prev)
    return out


def gpu_info():
    """read-only query of the card the numbers were measured on"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as ex:  # (the numbers are still reported; the card is then named by torch only)
        return {"name": torch.cuda.get_device_name(), "query_error": str(ex)}


def make_agg(variant, world):
    calls = ("(count:int8)", "(sum:int8 $1:int8)") + (() if variant == "R" else ("(max:int8 $1:int8)",))
    _, src = MockSource.channel()
    agg = HashAggExecutor(Backend.cuda(), src.into_executor(T2, []), variant != "R", [AggCall.from_pretty(c) for c in calls], 0, [0],
                          group_capacity_hint=2 * bench.AGG_KEYS * world)
    return agg, calls


def run_arm(variant, arm, ep_dev, plan, recv, n_ep_w, n_ep, world, stream):
    """one timed pass over the epochs.  arm "exchange": exchange -> counted push; "plain": agg_push_device of the rank's own
    rows (world 1 only).  -> (ms, apply kernel ms, exchange kernel ms, delta rows, agg)"""
    agg, calls = make_agg(variant, world)
    pushed = [torch.cuda.Event() for _ in ep_dev]
    ex_ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in ep_dev]

    def epoch(e, timed):
        if arm == "plain":
            device.agg_push_device(agg, ep_dev[e], stream)
        else:
            if e >= 2:
                stream.wait_event(pushed[e - 2])  # the push of batch e - 2 read this receive buffer
            if timed:
                ex_ev[e][0].record(stream)
            b = plan.start(ep_dev[e], stream)
            if timed:
                ex_ev[e][1].record(stream)
            device.agg_push_device(agg, recv[b], stream, n_rows_dev=plan.count_ptr(b))
        pushed[e].record(stream)

    for e in range(n_ep_w):
        epoch(e, False)
        device.agg_flush_device(agg, e + 1, stream)
    torch.cuda.synchronize()
    dist.barrier()
    device.profile(agg, "agg", True)
    t0 = time.perf_counter()
    delta_rows = 0
    for e in range(n_ep_w, n_ep_w + n_ep):
        epoch(e, True)
        device.agg_flush_device_async(agg, e + 1, stream)
        if e > n_ep_w:
            delta_rows += device.agg_flush_collect(agg, stream).n_rows
    delta_rows += device.agg_flush_collect(agg, stream).n_rows
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    kern_ms, _ = device.profile(agg, "agg", False)
    ex_ms = sum(a.elapsed_time(b) for a, b in ex_ev[n_ep_w:n_ep_w + n_ep]) if arm == "exchange" else 0.0
    return ms, kern_ms, ex_ms, delta_rows, agg, calls


def allreduce(vals, op):
    t = torch.tensor(vals, dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=op)
    return t.tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="A,B,R")
    ap.add_argument("--epochs", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--verify-epochs", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=2, help="passes per arm (the arms alternate)")
    args = ap.parse_args()
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    # weak scaling: 2^20 keys per rank (gen_agg_rows reads the key space from bench.AGG_KEYS; unchanged at N = 1)
    bench.AGG_KEYS = bench.AGG_KEYS * world
    info = gpu_info()
    stream = torch.cuda.Stream()
    plan = exchange.FlatShufflePlan(world, rank, [0], T2, batch_rows=ROWS)
    recv = [device.DeviceChunk(*plan.output(b), T2) for b in range(2)]
    n_ep_w, n_ep, n_v = args.warmup, args.epochs, args.verify_epochs
    for variant in args.variants.split(","):
        host = gen_all(variant, n_ep_w + n_ep + n_v, rank, world)
        ep_dev = [device.DeviceChunk(torch.from_numpy(o).cuda(), [torch.from_numpy(k).cuda(), torch.from_numpy(p).cuda()], T2) for o, k, p in host]
        torch.cuda.synchronize()
        arms = ("exchange", "plain") if world == 1 else ("exchange",)
        runs = {a: [] for a in arms}
        for _ in range(args.repeats):
            for arm in arms:
                ms, kern_ms, ex_ms, delta_rows, agg, calls = run_arm(variant, arm, ep_dev[:n_ep_w + n_ep], plan, recv, n_ep_w, n_ep, world, stream)
                ms_max = allreduce([ms], dist.ReduceOp.MAX)[0]
                runs[arm].append({"ms_per_epoch": ms_max / n_ep, "input_rows_per_s": world * n_ep * ROWS / (ms_max / 1e3),
                                  "apply_kernel_ms_per_epoch": kern_ms / n_ep, "exchange_kernel_ms_per_epoch": ex_ms / n_ep if arm == "exchange" else None,
                                  "delta_rows_per_input_row": delta_rows / (n_ep * ROWS)})
                if arm == "exchange":
                    keep_agg = agg
                else:
                    del agg
        # verification epochs (untimed) through the exchange arm's operator: each delta checksummed
        vr = vc = 0
        for e in range(n_ep_w + n_ep, n_ep_w + n_ep + n_v):
            b = plan.start(ep_dev[e], stream)
            device.agg_push_device(keep_agg, recv[b], stream, n_rows_dev=plan.count_ptr(b))
            r, c = device.agg_flush_device(keep_agg, e + 1, stream).checksum((1,) * (1 + len(calls)))
            vr, vc = vr + r, (vc + c) & M64
            torch.cuda.synchronize()
        tot = torch.tensor([vr, vc - (1 << 64) if vc >= (1 << 63) else vc], dtype=torch.int64, device="cuda")
        dist.all_reduce(tot)
        vr_all, vc_all = int(tot[0]), int(tot[1]) & M64
        # rows received per rank: the vnode owner of every row (all rows are visible)
        sent = np.zeros(world, np.int64)
        for o, k, p in host[n_ep_w:n_ep_w + n_ep]:
            sent += np.bincount(bench.vnode_of_int64(k).astype(np.int64) * world // 256, minlength=world)
        recv_rows = torch.from_numpy(sent).cuda()
        dist.all_reduce(recv_rows)
        recv_per_epoch = recv_rows.cpu().numpy() / n_ep
        if rank == 0:
            fc = bench.FastCpu().f
            fc.rwf_agg_checksum.restype = C.c_uint64
            fc.rwf_agg_checksum.argtypes = [C.c_void_p]
            ha = fc.rwf_agg_new(0 if variant == "R" else 1)
            fc.rwf_agg_reserve(ha, 2 * bench.AGG_KEYS)
            all_host = [host] + [gen_all(variant, n_ep_w + n_ep + n_v, r, world) for r in range(1, world)]
            want_rows, cs0 = 0, 0
            for e in range(n_ep_w + n_ep + n_v):
                for r in range(world):
                    o, k, p = all_host[r][e]
                    fc.rwf_agg_push(ha, len(o), o.ctypes.data, k.ctypes.data, p.ctypes.data)
                rows = fc.rwf_agg_flush(ha)
                if e == n_ep_w + n_ep - 1:
                    cs0 = fc.rwf_agg_checksum(ha)
                if e >= n_ep_w + n_ep:
                    want_rows += rows
            want_cs = (fc.rwf_agg_checksum(ha) - cs0) & M64
            fc.rwf_agg_free(ha)
            best = {a: min(runs[a], key=lambda x: x["ms_per_epoch"]) for a in arms}
            line = {
                "workload": f"nexmark_q4_hashagg_cfg2 variant {variant} behind the flat hash exchange: {', '.join(calls)} GROUP BY auction; "
                            f"{world} GPU(s), 2^18 input rows per rank and epoch, 2^20 x {world} keys",
                "gpus": world, "metric": "input rows/s over all ranks (max time over ranks)",
                "value": best["exchange"]["input_rows_per_s"], "ms_per_epoch": best["exchange"]["ms_per_epoch"],
                "runs": runs,
                "rows_received_per_rank_per_epoch": {"max": float(recv_per_epoch.max()), "mean": float(recv_per_epoch.mean())},
                "verified": bool((vr_all, vc_all) == (want_rows, want_cs)),
                "verification": {"epochs": n_v, "gpu_delta_rows": vr_all, "cpu_delta_rows": want_rows,
                                 "gpu_checksum": f"{vc_all:016x}", "cpu_checksum": f"{want_cs:016x}"},
                "gpu": info,
            }
            if world == 1:
                line["exchange_cost_ms_per_epoch"] = best["exchange"]["ms_per_epoch"] - best["plain"]["ms_per_epoch"]
            print(json.dumps(line), flush=True)
        del keep_agg, ep_dev
        torch.cuda.synchronize()
        dist.barrier()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
