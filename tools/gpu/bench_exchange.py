"""GPU micro-benchmark (not a test): the one-kernel exchange (and the older region exchange) on ONE device with world = 1
(self-peer: every row stays local), 2^20 rows x 4 int64 columns -- the exchange's kernel time without NVLink and without a
neighbour kernel, CUDA events over 20 launches."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bench  # noqa: E402
from risingwave_b200 import abi, device, exchange  # noqa: E402

N = 1 << 20
T4 = [abi.T_INT64] * 4
cols = bench.gen_bids(N, 0, bench.SEED, 10_000_000)
chunk = device.DeviceChunk(torch.ones(N, dtype=torch.uint8, device="cuda"), [torch.from_numpy(c).cuda() for c in cols], T4)
stream = torch.cuda.Stream()
for world in (1, 2, 8):  # world > 1: the destinations are virtual (all buffers on this device); only rank 0's kernel runs -> world 1 for barriers
    pass
total, ops_off, col_off = device.flat_layout(T4, N)
for max_blocks in (0, 2 * 132, 132):  # default (resident grid), two and one blocks per H100 SM
    buf = torch.zeros(total, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(1, dtype=torch.int64, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    tot = torch.zeros(1, dtype=torch.int64, device="cuda")
    call = device.FlatExchangeCall([0], exchange.vnode_to_dest_table(1).cuda(), 1, 0, [buf.data_ptr()], [flags.data_ptr()], N, counts, err, tot.data_ptr(),
                                   None, max_blocks=max_blocks)
    with torch.cuda.stream(stream):
        for e in range(1, 4):
            call(chunk, e, stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for e in range(4, 24):
            call(chunk, e, stream)
        e1.record(stream)
        torch.cuda.synchronize()
    print(f"flat exchange, world 1, max_blocks {max_blocks}: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us per 2^20 rows, total {int(tot.item())} err {int(err.item())}", flush=True)
# the older path: hist, scan, scatter into regions, publish, barrier kernel, unpack
region = device.p2p_region_bytes(T4, N)
recv = torch.zeros(region, dtype=torch.uint8, device="cuda")
flags = torch.zeros(1024, dtype=torch.uint8, device="cuda")
out_ops = torch.empty(N, dtype=torch.uint8, device="cuda")
out_cols = [torch.empty(N, dtype=torch.int64, device="cuda") for _ in T4]
counts = torch.zeros(1, dtype=torch.int64, device="cuda")
overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
total_host = torch.zeros(1, dtype=torch.int64).pin_memory()
call = device.P2PExchangeCall([0], exchange.vnode_to_dest_table(1).cuda(), 1, 0, [recv.data_ptr()], [flags.data_ptr()], N, recv.data_ptr(), out_ops, out_cols,
                              counts, overflow, total_host)
with torch.cuda.stream(stream):
    for e in range(1, 4):
        call(chunk, e, stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for e in range(4, 24):
        call(chunk, e, stream)
    e1.record(stream)
    torch.cuda.synchronize()
print(f"region exchange (6 launches), world 1: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us per 2^20 rows", flush=True)
