"""Multi-GPU hash shuffle: replaces the Dispatch -> Exchange -> Merge executors for the hash-shuffle
path only (src/stream/src/executor/dispatch.rs:897-1080, exchange/, merge.rs).

One process per GPU.  Per device batch:
  1. `rwgpu_shuffle_partition_device`: vnode = crc32(dist key) % 256 (vnode.rs:45-50), destination =
     vnode_to_dest[vnode] (contiguous equal vnode ranges, the shape of the reference's test mapping
     dispatch.rs:1566-1573), STABLE partition of ops + every column into per-destination regions;
  2. all-to-all of the per-destination row counts, then one all-to-all-v per column buffer over
     NCCL / NVLink (torch.distributed.all_to_all_single with split sizes);
  3. the join / agg kernels consume the received buffers directly (they are ordinary device chunks).
Row order per (source, key) is preserved, and a receiver concatenates sources in rank order, so
per-key order is deterministic.  Barriers are a host-side `dist.barrier()` (they are broadcast in
the reference too, dispatch.rs:940-947).  `U-/U+` pairs whose distribution key changes must be
rewritten to `-/+` before partitioning (`rwgpu_dispatch_rewrite_ops`, dispatch.rs:976-1023).

The split-size logic is backend-agnostic (`plan_splits`) and is covered on CPU with gloo,
world_size 2 (tests/test_exchange_gloo.py).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def vnode_to_dest_table(world: int, vnode_count: int = 256) -> torch.Tensor:
    """contiguous equal vnode ranges -> destination rank."""
    return (torch.arange(vnode_count, dtype=torch.int64) * world // vnode_count).to(torch.int32)


def plan_splits(send_counts: torch.Tensor, group=None) -> Tuple[List[int], List[int]]:
    """Exchange per-destination row counts; returns (input_split_sizes, output_split_sizes)."""
    world = dist.get_world_size(group)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts, group=group)
    ins = [int(x) for x in send_counts.cpu().tolist()]
    outs = [int(x) for x in recv_counts.cpu().tolist()]
    assert len(ins) == world and len(outs) == world
    return ins, outs


def all_to_all_columns(ops: torch.Tensor, cols: Sequence[torch.Tensor], ins: List[int], outs: List[int], group=None):
    """all-to-all-v of the ops bytes and of every column buffer (rows already grouped by destination)."""
    n_out = sum(outs)
    n_in = sum(ins)
    r_ops = torch.empty(n_out, dtype=ops.dtype, device=ops.device)
    dist.all_to_all_single(r_ops, ops[:n_in], outs, ins, group=group)
    r_cols = []
    for c in cols:
        r = torch.empty(n_out, dtype=c.dtype, device=c.device)
        dist.all_to_all_single(r, c[:n_in], outs, ins, group=group)
        r_cols.append(r)
    return r_ops, r_cols


class ShufflePlan:
    def __init__(self, world: int, rank: int, key_indices: Sequence[int], types: Sequence[int], vnode_count: int = 256):
        self.world, self.rank = world, rank
        self.keys = list(key_indices)
        self.types = list(types)
        self.vnode_count = vnode_count
        self.v2d = vnode_to_dest_table(world, vnode_count).cuda()

    def exchange(self, chunk, stream=None):
        """DeviceChunk -> (ops, cols) holding the rows this rank owns, from all ranks."""
        from . import device
        if chunk.visibility is not None or any(v is not None for v in chunk.validity):
            raise ValueError("the exchange does not carry validity / visibility bitmaps (fold visibility into ops; NULLs are unsupported)")
        ops, cols, counts, offsets = device.shuffle_partition(chunk, self.keys, self.v2d, self.world, self.vnode_count, stream)
        ins, outs = plan_splits(counts)
        return all_to_all_columns(ops, cols, ins, outs)

    def start(self, chunk, stream=None):
        """same interface as P2PShufflePlan (the NCCL path needs the split sizes on the host in the
        middle, so the whole exchange happens here)"""
        if stream is None:
            return self.exchange(chunk, stream)
        with torch.cuda.stream(stream):
            return self.exchange(chunk, stream)

    def finish(self, token):
        return token


class P2PShufflePlan:
    """Hash shuffle with the transfer fused into the partition kernel: every rank's scatter kernel
    stores its rows straight into the destination ranks' receive regions over NVLink peer memory
    (torch symmetric memory supplies the peer-mapped buffers; the cross-rank barrier is the library's
    own kernel on peer-mapped flags); no NCCL call is on the data path and one batch is ONE library
    call.  Two receive buffers alternate, so one barrier per batch is enough: a peer
    can only start writing buffer b again after every rank passed the barrier of the batch in between,
    which each rank enqueues AFTER its own unpack of buffer b (stream order).

    Every (source, destination) region is sized for the WORST case -- all `batch_rows` rows of a source going to one
    destination (hot keys) -- so a batch can never overflow its region: W x batch_rows x row bytes per receive buffer
    (8 GPUs, 2^20-row batches of four int64 columns: 277 MB of 180 GB).  The kernels still raise the overflow flag
    for a caller that hands in more rows than it announced; `finish` then raises.

    Columns with validity bitmaps are not carried by either exchange plan (RW_ERR_UNSUPPORTED-style ValueError):
    NULLs would arrive as garbage."""

    def __init__(self, world: int, rank: int, key_indices: Sequence[int], types: Sequence[int], batch_rows: int,
                 group=None, vnode_count: int = 256):
        import torch.distributed._symmetric_memory as symm_mem
        from . import device
        self.world, self.rank = world, rank
        self.keys, self.types, self.vnode_count = list(key_indices), list(types), vnode_count
        self.v2d = vnode_to_dest_table(world, vnode_count).cuda()
        self.cap = int(batch_rows)  # worst case: no skew can overflow a region
        self.region = device.p2p_region_bytes(self.types, self.cap)
        group = group if group is not None else dist.group.WORLD
        self.bufs, self.hdls, self.peers = [], [], []
        for _ in range(2):
            b = symm_mem.empty(world * self.region, dtype=torch.uint8, device="cuda")
            h = symm_mem.rendezvous(b, group)
            self.bufs.append(b)
            self.hdls.append(h)
            self.peers.append([int(h.buffer_ptrs[r]) for r in range(world)])
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.step = 0
        self.fallback = ShufflePlan(world, rank, key_indices, types, vnode_count)
        self.max_rows = world * self.cap
        # double-buffered outputs + row-count read-back (pinned), so that the exchange of batch s+1 can
        # run on its own stream while the consumer still reads the rows of batch s
        self.out, self.totals_host, self.events, self.calls = [], [], [], []
        # flag block of the library's own cross-rank barrier (symmetric, zeroed; epochs only grow)
        self.flags = symm_mem.empty(1024, dtype=torch.uint8, device="cuda")
        self.flags.zero_()
        self.flags_hdl = symm_mem.rendezvous(self.flags, group)
        flag_ptrs = [int(self.flags_hdl.buffer_ptrs[r]) for r in range(world)]
        self._count_base = self.flags.data_ptr() + 512  # device int64 row counts (rwgpu.h): slot = epoch & 1
        self._count_ptr = [0, 0]
        torch.cuda.synchronize()
        self.flags_hdl.barrier(channel=0)  # every rank's flags are zero before anybody signals
        torch.cuda.synchronize()
        for b in range(2):
            ops = torch.empty(self.max_rows, dtype=torch.uint8, device="cuda")
            cols = [torch.empty(self.max_rows, dtype=device.TORCH_DTYPE[t], device="cuda") for t in self.types]
            self.out.append((ops, cols))
            self.totals_host.append(torch.zeros(1, dtype=torch.int64).pin_memory())
            self.events.append(torch.cuda.Event())
            self.calls.append(device.P2PExchangeCall(self.keys, self.v2d, world, rank, self.peers[b], flag_ptrs, self.cap,
                                                     self.bufs[b].data_ptr(), ops, cols, self.counts, self.overflow,
                                                     self.totals_host[b], vnode_count))

    def start(self, chunk, stream=None):
        """enqueue partition + peer stores + barrier + unpack of one batch on `stream` (one library call, five
        launches); returns a token"""
        if chunk.n_rows() > self.cap:
            raise ValueError(f"batch of {chunk.n_rows()} rows exceeds the plan's batch_rows {self.cap}")
        if chunk.visibility is not None or any(v is not None for v in chunk.validity):
            raise ValueError("the exchange does not carry validity / visibility bitmaps (fold visibility into ops; NULLs are unsupported)")
        b = self.step & 1
        self.step += 1
        stream = stream if stream is not None else torch.cuda.current_stream()
        self.calls[b](chunk, self.step, stream)  # epoch = batch number (1, 2, ...)
        self._count_ptr[b] = self._count_base + 8 * (self.step & 1)
        self.events[b].record(stream)
        return b

    def count_ptr(self, b) -> int:
        """device address of the int64 row count of token `b` (valid until the second `start` after it)"""
        return self._count_ptr[b]

    def output(self, b):
        """the FULL output buffers of token `b` (capacity `max_rows`); the row count is on the device at
        `total_dev_ptr` once the batch's work on the stream has run -- for consumers that read it there"""
        return self.out[b]

    def finish(self, b):
        """wait for the batch of token `b`; -> (ops, cols) views of the received rows (valid until the
        second `start` after this one)"""
        self.events[b].synchronize()
        n = int(self.totals_host[b][0])  # the consumer needs the row count on the host
        if n < 0:
            raise RuntimeError("p2p shuffle: a (source, destination) pair exceeded its region capacity "
                               f"({self.cap} rows); use ShufflePlan (NCCL all-to-all-v) for this stream")
        ops, cols = self.out[b]
        return ops[:n], [c[:n] for c in cols]

    def exchange(self, chunk, stream=None):
        return self.finish(self.start(chunk, stream))


class FlatShufflePlan:
    """The N-GPU hash shuffle as ONE kernel per batch (rwgpu_shuffle_exchange_flat_device): histograms,
    scan, count exchange, cross-rank barrier, scatter over NVLink straight into the rows' FINAL place in the
    destination's receive buffer, second barrier, row count -- no NCCL call, no unpack copy; the consumer (the join's
    counted push) reads the receive buffer in place and the row count on the device.

    Two symmetric receive buffers alternate.  Caller contract (rwgpu.h): `start` of batch e is enqueued after the local
    consumer of batch e - 2 has finished (e.g. `stream.wait_event(join_done[e - 2])`).  A buffer holds world x batch_rows
    rows, so no distribution of keys can overflow it.  Columns with validity bitmaps are not carried (ValueError)."""

    def __init__(self, world: int, rank: int, key_indices: Sequence[int], types: Sequence[int], batch_rows: int,
                 group=None, vnode_count: int = 256, max_blocks: int = 0):
        import torch.distributed._symmetric_memory as symm_mem
        from . import abi, device
        self.world, self.rank = world, rank
        self.keys, self.types, self.vnode_count = list(key_indices), list(types), vnode_count
        self.v2d = vnode_to_dest_table(world, vnode_count).cuda()
        self.batch_rows = int(batch_rows)
        self.max_rows = world * self.batch_rows
        total, ops_off, col_off = device.flat_layout(self.types, self.max_rows)
        group = group if group is not None else dist.group.WORLD
        self.bufs, self.hdls, self.out = [], [], []
        self.flags = symm_mem.empty(1024, dtype=torch.uint8, device="cuda")
        self.flags.zero_()
        self.flags_hdl = symm_mem.rendezvous(self.flags, group)
        flag_ptrs = [int(self.flags_hdl.buffer_ptrs[r]) for r in range(world)]
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.err = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.totals_dev = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.totals_host, self.events, self.calls = [], [], []
        for b in range(2):
            buf = symm_mem.empty(total, dtype=torch.uint8, device="cuda")
            buf.zero_()
            h = symm_mem.rendezvous(buf, group)
            self.bufs.append(buf)
            self.hdls.append(h)
            peers = [int(h.buffer_ptrs[r]) for r in range(world)]
            ops = buf[ops_off:ops_off + self.max_rows]
            cols = [buf[o:o + self.max_rows * abi.TYPE_WIDTH[t]].view(device.TORCH_DTYPE[t]) for o, t in zip(col_off, self.types)]
            self.out.append((ops, cols))
            self.totals_host.append(torch.zeros(1, dtype=torch.int64).pin_memory())
            self.events.append(torch.cuda.Event())
            self.calls.append(device.FlatExchangeCall(self.keys, self.v2d, world, rank, peers, flag_ptrs, self.max_rows, self.counts, self.err,
                                                      self.totals_dev.data_ptr() + 8 * b, self.totals_host[b], vnode_count, max_blocks))
        self.step = 0
        torch.cuda.synchronize()
        self.flags_hdl.barrier(channel=0)  # every rank's flags and headers are zero before anybody signals
        torch.cuda.synchronize()

    def start(self, chunk, stream=None):
        """enqueue one batch on `stream` (one launch); -> token"""
        if chunk.n_rows() > self.batch_rows:
            raise ValueError(f"batch of {chunk.n_rows()} rows exceeds the plan's batch_rows {self.batch_rows}")
        if chunk.visibility is not None or any(v is not None for v in chunk.validity):
            raise ValueError("the exchange does not carry validity / visibility bitmaps (fold visibility into ops; NULLs are unsupported)")
        b = self.step & 1
        self.step += 1
        stream = stream if stream is not None else torch.cuda.current_stream()
        self.calls[b](chunk, self.step, stream)
        self.events[b].record(stream)
        return b

    def count_ptr(self, b) -> int:
        """device address of the int64 row count of token `b`"""
        return self.totals_dev.data_ptr() + 8 * b

    def output(self, b):
        """(ops, cols) views of the WHOLE receive buffer of token `b` (capacity world x batch_rows); the first
        `count` rows are the batch"""
        return self.out[b]

    def finish(self, b):
        """wait for token `b`; -> (ops, cols) views of the received rows (valid until the second `start` after it)"""
        self.events[b].synchronize()
        n = int(self.totals_host[b][0])
        if n < 0:
            raise RuntimeError(f"flat shuffle failed on the device (err bits {int(self.err.item())}: 1 = receive buffer too small, "
                               "2 = a peer did not reach the barrier)")
        ops, cols = self.out[b]
        return ops[:n], [c[:n] for c in cols]

    def exchange(self, chunk, stream=None):
        return self.finish(self.start(chunk, stream))
