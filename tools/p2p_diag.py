"""2-GPU diagnostic for the fused partition+transfer exchange: where does a batch's time go?
torchrun --nproc-per-node 2 tools/p2p_diag.py   (rank 0 prints one report)"""
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from risingwave_b200 import abi, device, exchange  # noqa: E402


def timed(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    import torch.distributed._symmetric_memory as symm_mem
    rep = []
    rep.append(f"can_access_peer(0,1) = {torch.cuda.can_device_access_peer(0, 1) if world > 1 else None}")
    n = 1 << 20
    T4 = [abi.T_INT64] * 4
    g = torch.Generator(device="cuda").manual_seed(1 + rank)
    cols = [torch.randint(0, 1 << 40, (n,), dtype=torch.int64, device="cuda", generator=g) for _ in range(4)]
    chunk = device.DeviceChunk(torch.ones(n, dtype=torch.uint8, device="cuda"), cols, T4)
    stream = torch.cuda.current_stream()

    # raw peer copy bandwidth through a symmetric buffer
    nbytes = 64 << 20
    buf = symm_mem.empty(nbytes, dtype=torch.uint8, device="cuda")
    hdl = symm_mem.rendezvous(buf, dist.group.WORLD)
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    peer = (rank + 1) % world
    pbuf = hdl.get_buffer(peer, (nbytes,), torch.uint8)
    ms = timed(lambda: pbuf.copy_(src))
    rep.append(f"peer copy 64 MiB -> rank {peer}: {ms:.3f} ms = {nbytes / ms / 1e6:.1f} GB/s")
    ms = timed(lambda: hdl.barrier(channel=0))
    rep.append(f"symm_mem barrier: {ms * 1e3:.1f} us")

    plan = exchange.P2PShufflePlan(world, rank, [0], T4, n)
    ms = timed(lambda: plan.exchange(chunk, stream))
    rep.append(f"P2PShufflePlan.exchange (2^20 rows): {ms:.3f} ms")

    nplan = exchange.ShufflePlan(world, rank, [0], T4)
    ms = timed(lambda: nplan.exchange(chunk, stream))
    rep.append(f"ShufflePlan.exchange (NCCL all-to-all-v): {ms:.3f} ms")
    # local partition only
    ms = timed(lambda: device.shuffle_partition(chunk, [0], nplan.v2d, world, 256, stream))
    rep.append(f"  local stable partition only: {ms:.3f} ms")
    if rank == 0:
        print("\n".join(rep))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
