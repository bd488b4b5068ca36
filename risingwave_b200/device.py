"""Device-resident driver API: torch CUDA tensors in, device views out, through the C ABI's
`*_device` entry points (no torch types cross the ABI: raw device pointers and a cudaStream_t).

Used by bench.py (kernel-only throughput with inputs already in HBM) and by the multi-GPU
hash-shuffle path (exchange.py).  PyTorch is plumbing here: allocation, streams, torch.distributed.
"""
from __future__ import annotations

import collections
import ctypes as C
from typing import List, Optional, Sequence

import torch

from . import abi

TORCH_DTYPE = {abi.T_BOOL: torch.uint8, abi.T_INT16: torch.int16, abi.T_INT32: torch.int32, abi.T_INT64: torch.int64,
               abi.T_FLOAT32: torch.float32, abi.T_FLOAT64: torch.float64, abi.T_DATE: torch.int32,
               abi.T_TIME: torch.int64, abi.T_TIMESTAMP: torch.int64, abi.T_TIMESTAMPTZ: torch.int64,
               abi.T_SERIAL: torch.int64}


class DeviceChunk:
    """A StreamChunk whose buffers are CUDA tensors (ops uint8[n]; columns in native width;
    optional validity / visibility as packed uint64 words held in int64 tensors)."""

    def __init__(self, ops: torch.Tensor, cols: Sequence[torch.Tensor], types: Sequence[int],
                 validity: Optional[Sequence[Optional[torch.Tensor]]] = None, visibility: Optional[torch.Tensor] = None):
        assert ops.dtype == torch.uint8 and ops.is_cuda and ops.is_contiguous()
        self.ops, self.cols, self.types = ops, list(cols), list(types)
        self.validity = list(validity) if validity is not None else [None] * len(cols)
        self.visibility = visibility
        for c, t in zip(self.cols, self.types):
            assert c.is_cuda and c.is_contiguous() and c.dtype == TORCH_DTYPE[t] and c.numel() == ops.numel()

    def n_rows(self) -> int:
        return self.ops.numel()

    def to_abi(self):
        cached = getattr(self, "_abi", None)
        if cached is not None:  # (tensors of a DeviceChunk are never re-bound)
            return cached
        cols = (abi.RwColumn * max(1, len(self.cols)))()
        for k, (c, t) in enumerate(zip(self.cols, self.types)):
            cols[k].type = t
            cols[k].data = c.data_ptr() if c.numel() else None
            cols[k].validity = self.validity[k].data_ptr() if self.validity[k] is not None else None
        ch = abi.RwChunk()
        ch.n_rows = self.ops.numel()
        ch.n_cols = len(self.cols)
        ch.ops = self.ops.data_ptr() if self.ops.numel() else None
        ch.visibility = self.visibility.data_ptr() if self.visibility is not None else None
        ch.columns = cols
        self._abi = (ch, cols)
        return ch, cols


class DeviceView:
    """Device pointers returned by a `*_device` call (valid until the next call on that handle)."""

    def __init__(self, view: abi.RwChunk, stream: Optional[torch.cuda.Stream] = None, chunk: Optional[DeviceChunk] = None):
        # the library may still be packing bitmaps on `stream` when the call returns: readers below wait for it
        self._stream = stream
        self._synced = False
        # a join view's update-side columns may point into the pushed chunk's tensors (rwgpu.h): they live as long as the view
        self._chunk = chunk
        self.n_rows = int(view.n_rows)
        self.n_cols = int(view.n_cols)
        self.ops_ptr = view.ops
        self.vis_ptr = view.visibility
        self.col_ptrs = [view.columns[k].data for k in range(self.n_cols)]
        self.col_types = [int(view.columns[k].type) for k in range(self.n_cols)]
        self.valid_ptrs = [view.columns[k].validity for k in range(self.n_cols)]

    def _wait(self):
        if not self._synced:
            if self._stream is not None:
                self._stream.synchronize()
            else:  # the library's own stream
                torch.cuda.synchronize()
            self._synced = True

    def column(self, k: int) -> torch.Tensor:
        """copy column k out of the library-owned buffer into a fresh tensor (D2D)."""
        self._wait()
        t = self.col_types[k]
        out = torch.empty(self.n_rows, dtype=TORCH_DTYPE[t], device="cuda")
        if self.n_rows:
            _d2d(out.data_ptr(), self.col_ptrs[k], self.n_rows * abi.TYPE_WIDTH[t])
        return out

    def ops(self) -> torch.Tensor:
        self._wait()
        out = torch.empty(self.n_rows, dtype=torch.uint8, device="cuda")
        if self.n_rows:
            _d2d(out.data_ptr(), self.ops_ptr, self.n_rows)
        return out

    def visible(self) -> Optional[torch.Tensor]:
        """bool[n_rows] from the packed visibility words, or None when every row is visible."""
        if not self.vis_ptr or not self.n_rows:
            return None
        self._wait()
        nw = (self.n_rows + 63) // 64
        words = torch.empty(nw, dtype=torch.int64, device="cuda")
        _d2d(words.data_ptr(), self.vis_ptr, nw * 8)
        bits = (words.unsqueeze(1) >> torch.arange(64, device="cuda", dtype=torch.int64).unsqueeze(0)) & 1
        return bits.reshape(-1)[:self.n_rows].to(torch.bool)

    def checksum(self, weights: Sequence[int]) -> tuple:
        """-> (visible rows, order-independent checksum mod 2^64 of the (op, row) multiset): sum over visible rows of
        sign(op) * sum_k weights[k] * col_k, sign = +1 for Insert / UpdateInsert, -1 for Delete / UpdateDelete (the
        same function the CPU baseline of bench.py accumulates; verification only, never inside a timed region)."""
        if not self.n_rows:
            return 0, 0
        acc = torch.zeros(self.n_rows, dtype=torch.int64, device="cuda")
        for k, w in enumerate(weights):
            acc += self.column(k).to(torch.int64) * int(w)
        ops = self.ops()
        sign = torch.where((ops == abi.OP_INSERT) | (ops == abi.OP_UPDATE_INSERT), 1, -1).to(torch.int64)
        acc *= sign
        vis = self.visible()
        if vis is not None:
            acc = acc[vis]
        return int(acc.numel()), int(acc.sum().item()) & ((1 << 64) - 1)


class ViewChunk:
    """Rows [lo, hi) of a DeviceView as a device chunk over the view's own buffers, columns picked and reordered by
    `cols` (a projection by column pointers: nothing is copied).  This is how an operator's delta left in HBM is sent
    through the exchange (q4's outer HashAgg regroups the inner HashAgg's delta by `category`).  Valid as long as the
    view.  A picked column with NULLs keeps its bitmap in `validity`, which the exchange plans refuse (ValueError)."""

    def __init__(self, view: DeviceView, cols: Sequence[int], lo: int = 0, hi: Optional[int] = None):
        self.view, self.lo = view, lo
        self.hi = view.n_rows if hi is None else hi
        assert 0 <= lo <= self.hi <= view.n_rows
        self.types = [view.col_types[k] for k in cols]
        self.ptrs = [view.col_ptrs[k] for k in cols]
        self.validity = [view.valid_ptrs[k] or None for k in cols]
        self.visibility = view.vis_ptr or None

    def n_rows(self) -> int:
        return self.hi - self.lo

    def to_abi(self):
        if self.visibility is not None or any(v is not None for v in self.validity):
            raise ValueError("a slice of a view with validity / visibility bitmaps is not addressable by row offset")
        cols = (abi.RwColumn * max(1, len(self.ptrs)))()
        for k, (p, t) in enumerate(zip(self.ptrs, self.types)):
            cols[k].type = t
            cols[k].data = p + self.lo * abi.TYPE_WIDTH[t]
            cols[k].validity = None
        ch = abi.RwChunk()
        ch.n_rows = self.n_rows()
        ch.n_cols = len(self.ptrs)
        ch.ops = self.view.ops_ptr + self.lo if self.n_rows() else None
        ch.visibility = None
        ch.columns = cols
        return ch, cols


def _d2d(dst: int, src: int, nbytes: int):
    """device-to-device copy ON TORCH'S CURRENT STREAM, so that the tensor operations that follow are ordered behind it.
    (A plain cudaMemcpy runs on the legacy default stream and, device to device, does not wait on the host: kernels torch
    then launches on a non-blocking stream raced with the copy and read the destination's previous contents -- this is
    what made bench.py's retract leg report verified = false in the r2b..r2e runs while the rows were right.)"""
    rc = cudart().cudaMemcpyAsync(C.c_void_p(dst), C.c_void_p(src), C.c_size_t(nbytes), 3, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise RuntimeError(f"cudaMemcpyAsync failed: {rc}")


_cudart = None


def cudart():
    global _cudart
    if _cudart is None:
        import glob
        import os
        cands = glob.glob(os.path.join(os.path.dirname(torch.__file__), "lib", "libcudart*.so*")) + \
            glob.glob("/usr/local/cuda/lib64/libcudart.so*")
        _cudart = C.CDLL(cands[0])
    return _cudart


def _lib():
    lib = abi.load_library()
    if not getattr(lib, "_dev_sigs", False):
        lib.rwgpu_agg_push_device.restype = C.c_int32
        lib.rwgpu_agg_push_device.argtypes = [C.c_void_p, C.POINTER(abi.RwChunk), C.c_void_p]
        lib.rwgpu_agg_push_device_counted.restype = C.c_int32
        lib.rwgpu_agg_push_device_counted.argtypes = [C.c_void_p, C.POINTER(abi.RwChunk), C.c_void_p, C.c_void_p]
        lib.rwgpu_agg_flush_device.restype = C.c_int32
        lib.rwgpu_agg_flush_device.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(abi.RwChunk), C.c_void_p]
        lib.rwgpu_agg_flush_device_async.restype = C.c_int32
        lib.rwgpu_agg_flush_device_async.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        lib.rwgpu_agg_flush_collect.restype = C.c_int32
        lib.rwgpu_agg_flush_collect.argtypes = [C.c_void_p, C.POINTER(abi.RwChunk), C.c_void_p]
        lib.rwgpu_join_push_device.restype = C.c_int32
        lib.rwgpu_join_push_device.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk), C.POINTER(abi.RwChunk), C.c_void_p]
        for name in ("rwgpu_agg_profile", "rwgpu_join_profile"):
            fn = getattr(lib, name)
            fn.restype = C.c_int32
            fn.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        lib.rwgpu_agg_stats.restype = C.c_int32
        lib.rwgpu_agg_stats.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint64)] * 3
        lib.rwgpu_join_stats.restype = C.c_int32
        lib.rwgpu_join_stats.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint64)] * 3
        lib.rwgpu_shuffle_partition_device.restype = C.c_int32
        lib.rwgpu_shuffle_partition_device.argtypes = [C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                                       C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p),
                                                       C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p]
        lib.rwgpu_shuffle_p2p_region_bytes.restype = C.c_int32
        lib.rwgpu_shuffle_p2p_region_bytes.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.c_int64, C.POINTER(C.c_int64)]
        lib.rwgpu_shuffle_partition_p2p_device.restype = C.c_int32
        lib.rwgpu_shuffle_partition_p2p_device.argtypes = [C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p,
                                                           C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.c_int64, C.c_void_p,
                                                           C.c_void_p, C.c_void_p]
        lib.rwgpu_shuffle_unpack_device.restype = C.c_int32
        lib.rwgpu_shuffle_unpack_device.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int64, C.c_void_p,
                                                    C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
        lib.rwgpu_join_push_device_counted.restype = C.c_int32
        lib.rwgpu_join_push_device_counted.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk), C.c_void_p, C.POINTER(abi.RwChunk),
                                                       C.c_void_p]
        lib.rwgpu_join_push_device_async.restype = C.c_int32
        lib.rwgpu_join_push_device_async.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk), C.c_void_p, C.c_void_p]
        lib.rwgpu_join_collect.restype = C.c_int32
        lib.rwgpu_join_collect.argtypes = [C.c_void_p, C.POINTER(abi.RwChunk), C.c_void_p]
        lib.rwgpu_shuffle_exchange_p2p_device.restype = C.c_int32
        lib.rwgpu_shuffle_exchange_p2p_device.argtypes = [C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p,
                                                          C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_uint64,
                                                          C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p,
                                                          C.c_void_p, C.c_void_p, C.c_void_p]
        lib.rwgpu_filter_device.restype = C.c_int32
        lib.rwgpu_filter_device.argtypes = [C.POINTER(abi.RwChunk), C.POINTER(abi.RwFilterTerm), C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        lib.rwgpu_last_error.restype = C.c_char_p
        lib._dev_sigs = True
    return lib


def _check(rc):
    if rc != abi.RW_OK:
        raise abi.RwError(rc, (_lib().rwgpu_last_error() or b"").decode())


def _stream_ptr(stream: Optional[torch.cuda.Stream]):
    return C.c_void_p(stream.cuda_stream) if stream is not None else None


def agg_push_device(executor, chunk: DeviceChunk, stream: Optional[torch.cuda.Stream] = None, n_rows_dev: Optional[int] = None):
    """`n_rows_dev`: device address of an int64 row count produced by earlier work of `stream` (the chunk's
    tensors are then the capacity); no host round trip between the producer and the aggregation.  The chunk's
    tensors and the count must stay unchanged until the push's kernels have run on `stream`."""
    ch, keep = chunk.to_abi()
    if n_rows_dev is None:
        _check(_lib().rwgpu_agg_push_device(executor._h, C.byref(ch), _stream_ptr(stream)))
    else:
        _check(_lib().rwgpu_agg_push_device_counted(executor._h, C.byref(ch), C.c_void_p(n_rows_dev), _stream_ptr(stream)))


def agg_flush_device(executor, epoch: int, stream: Optional[torch.cuda.Stream] = None) -> DeviceView:
    view = abi.RwChunk()
    _check(_lib().rwgpu_agg_flush_device(executor._h, epoch, C.byref(view), _stream_ptr(stream)))
    return DeviceView(view, stream)


def agg_flush_device_async(executor, epoch: int, stream: Optional[torch.cuda.Stream] = None):
    """enqueue the barrier's delta computation (nothing is waited for); collect it with `agg_flush_collect`"""
    _check(_lib().rwgpu_agg_flush_device_async(executor._h, epoch, _stream_ptr(stream)))


def agg_flush_collect(executor, stream: Optional[torch.cuda.Stream] = None) -> DeviceView:
    """wait for the oldest outstanding barrier; -> its delta (device pointers)"""
    view = abi.RwChunk()
    _check(_lib().rwgpu_agg_flush_collect(executor._h, C.byref(view), _stream_ptr(stream)))
    return DeviceView(view, stream)


def join_push_device(executor, side: int, chunk: DeviceChunk, stream: Optional[torch.cuda.Stream] = None,
                     n_rows_dev: Optional[int] = None) -> DeviceView:
    """`n_rows_dev`: device address of an int64 row count produced by earlier work of `stream` (the chunk's
    tensors are then the capacity); no host round trip between the producer and the join."""
    ch, keep = chunk.to_abi()
    view = abi.RwChunk()
    if n_rows_dev is None:
        _check(_lib().rwgpu_join_push_device(executor._h, side, C.byref(ch), C.byref(view), _stream_ptr(stream)))
    else:
        _check(_lib().rwgpu_join_push_device_counted(executor._h, side, C.byref(ch), C.c_void_p(n_rows_dev), C.byref(view),
                                                     _stream_ptr(stream)))
    return DeviceView(view, stream, chunk)


def join_push_device_async(executor, side: int, chunk: DeviceChunk, stream: Optional[torch.cuda.Stream] = None,
                           n_rows_dev: Optional[int] = None):
    """LAUNCH half of a push (nothing is waited for); the chunk is kept alive until `join_collect` hands it to the view"""
    ch, keep = chunk.to_abi()
    _check(_lib().rwgpu_join_push_device_async(executor._h, side, C.byref(ch), C.c_void_p(n_rows_dev) if n_rows_dev else None,
                                               _stream_ptr(stream)))
    if not hasattr(executor, "_pushed_chunks"):
        executor._pushed_chunks = collections.deque()
    executor._pushed_chunks.append(chunk)


def join_collect(executor, stream: Optional[torch.cuda.Stream] = None) -> DeviceView:
    """COLLECT half: wait for the oldest outstanding push; -> its output (device pointers)"""
    view = abi.RwChunk()
    pushed = getattr(executor, "_pushed_chunks", None)
    chunk = pushed.popleft() if pushed else None  # (a collect that fails still takes the oldest push off the handle)
    _check(_lib().rwgpu_join_collect(executor._h, C.byref(view), _stream_ptr(stream)))
    return DeviceView(view, stream, chunk)


def profile(executor, kind: str, enable: bool):
    """-> (dominant-kernel milliseconds, launches) accumulated since the previous call."""
    ms, n = C.c_double(), C.c_uint64()
    fn = _lib().rwgpu_agg_profile if kind == "agg" else _lib().rwgpu_join_profile
    _check(fn(executor._h, int(enable), C.byref(ms), C.byref(n)))
    return ms.value, n.value


def launches(executor, kind: str) -> int:
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fn = _lib().rwgpu_agg_stats if kind == "agg" else _lib().rwgpu_join_stats
    _check(fn(executor._h, C.byref(a), C.byref(b), C.byref(c)))
    return c.value


def shuffle_partition(chunk: DeviceChunk, key_indices: Sequence[int], vnode_to_dest: torch.Tensor, n_dest: int,
                      vnode_count: int = 256, stream: Optional[torch.cuda.Stream] = None):
    """Stable partition of the visible rows by destination = vnode_to_dest[crc32(key) % vnode_count].
    Returns (ops, cols, counts[n_dest], offsets[n_dest]) as CUDA tensors; rows of destination d are
    [offsets[d], offsets[d]+counts[d])."""
    n = chunk.n_rows()
    out_ops = torch.empty(n, dtype=torch.uint8, device="cuda")
    out_cols = [torch.empty_like(c) for c in chunk.cols]
    counts = torch.zeros(n_dest, dtype=torch.int64, device="cuda")
    offsets = torch.zeros(n_dest, dtype=torch.int64, device="cuda")
    ch, keep = chunk.to_abi()
    keys = (C.c_int32 * len(key_indices))(*key_indices)
    colp = (C.c_void_p * len(out_cols))(*[c.data_ptr() for c in out_cols])
    _check(_lib().rwgpu_shuffle_partition_device(C.byref(ch), keys, len(key_indices), vnode_count,
                                                 C.c_void_p(vnode_to_dest.data_ptr()), n_dest, C.c_void_p(out_ops.data_ptr()),
                                                 colp, None, C.c_void_p(counts.data_ptr()), C.c_void_p(offsets.data_ptr()),
                                                 _stream_ptr(stream)))
    return out_ops, out_cols, counts, offsets


def p2p_region_bytes(types: Sequence[int], cap_rows: int) -> int:
    t = (C.c_int32 * len(types))(*types)
    out = C.c_int64()
    _check(_lib().rwgpu_shuffle_p2p_region_bytes(t, len(types), cap_rows, C.byref(out)))
    return out.value


def shuffle_partition_p2p(chunk: DeviceChunk, key_indices: Sequence[int], vnode_to_dest: torch.Tensor, n_dest: int, my_rank: int,
                          peer_ptrs: Sequence[int], cap_rows: int, counts: torch.Tensor, overflow: torch.Tensor,
                          vnode_count: int = 256, stream: Optional[torch.cuda.Stream] = None):
    """fused stable partition + store into the peers' receive regions (NVLink peer memory)."""
    ch, keep = chunk.to_abi()
    keys = (C.c_int32 * len(key_indices))(*key_indices)
    peers = (C.c_void_p * n_dest)(*peer_ptrs)
    _check(_lib().rwgpu_shuffle_partition_p2p_device(C.byref(ch), keys, len(key_indices), vnode_count,
                                                     C.c_void_p(vnode_to_dest.data_ptr()), n_dest, my_rank, peers, cap_rows,
                                                     C.c_void_p(counts.data_ptr()), C.c_void_p(overflow.data_ptr()), _stream_ptr(stream)))


def shuffle_unpack(recv_ptr: int, n_src: int, types: Sequence[int], cap_rows: int, out_ops: torch.Tensor,
                   out_cols: Sequence[torch.Tensor], total: torch.Tensor, stream: Optional[torch.cuda.Stream] = None):
    t = (C.c_int32 * len(types))(*types)
    colp = (C.c_void_p * len(out_cols))(*[c.data_ptr() for c in out_cols])
    _check(_lib().rwgpu_shuffle_unpack_device(C.c_void_p(recv_ptr), n_src, t, len(types), cap_rows, C.c_void_p(out_ops.data_ptr()),
                                              colp, C.c_void_p(total.data_ptr()), _stream_ptr(stream)))


class P2PExchangeCall:
    """Pre-built argument block of rwgpu_shuffle_exchange_p2p_device for one receive-buffer parity: the
    per-batch call is then a single ctypes call (the step is host-latency sensitive)."""

    def __init__(self, key_indices, vnode_to_dest, n_dest, my_rank, peer_ptrs, flag_ptrs, cap_rows, recv_ptr, out_ops, out_cols,
                 counts, overflow, total_host, vnode_count=256):
        self.keys = (C.c_int32 * len(key_indices))(*key_indices)
        self.n_keys = len(key_indices)
        self.peers = (C.c_void_p * n_dest)(*peer_ptrs)
        self.flags = (C.c_void_p * n_dest)(*flag_ptrs)
        self.colp = (C.c_void_p * len(out_cols))(*[c.data_ptr() for c in out_cols])
        self.args = (vnode_count, C.c_void_p(vnode_to_dest.data_ptr()), n_dest, my_rank)
        self.cap_rows, self.recv = cap_rows, C.c_void_p(recv_ptr)
        self.out_ops = C.c_void_p(out_ops.data_ptr())
        self.counts, self.overflow = C.c_void_p(counts.data_ptr()), C.c_void_p(overflow.data_ptr())
        self.total_host = C.c_void_p(total_host.data_ptr())
        self.keep = (vnode_to_dest, out_ops, out_cols, counts, overflow, total_host)

    def __call__(self, chunk: DeviceChunk, epoch: int, stream):
        ch, keep = chunk.to_abi()
        vc, v2d, n_dest, my_rank = self.args
        _check(_lib().rwgpu_shuffle_exchange_p2p_device(C.byref(ch), self.keys, self.n_keys, vc, v2d, n_dest, my_rank, self.peers,
                                                        self.flags, C.c_uint64(epoch), C.c_int64(self.cap_rows), self.recv,
                                                        self.out_ops, self.colp, self.counts, self.overflow, self.total_host,
                                                        _stream_ptr(stream)))


def flat_layout(types: Sequence[int], cap_rows: int):
    """rwgpu_shuffle_flat_layout -> (total bytes, ops offset, [column offsets]) of a flat receive buffer"""
    t = (C.c_int32 * len(types))(*types)
    total, ops_off = C.c_int64(), C.c_int64()
    col_off = (C.c_int64 * max(1, len(types)))()
    _check(_lib().rwgpu_shuffle_flat_layout(t, len(types), C.c_int64(cap_rows), C.byref(total), C.byref(ops_off), col_off))
    return total.value, ops_off.value, [col_off[k] for k in range(len(types))]


class FlatExchangeCall:
    """Pre-built argument block of rwgpu_shuffle_exchange_flat_device for one receive-buffer parity (one ctypes call per
    batch: partition, peer stores, both barriers and the row count are one kernel)."""

    def __init__(self, key_indices, vnode_to_dest, n_dest, my_rank, peer_ptrs, flag_ptrs, cap_rows, counts, err, total_dev_ptr,
                 total_host, vnode_count=256, max_blocks=0):
        self.keys = (C.c_int32 * len(key_indices))(*key_indices)
        self.n_keys = len(key_indices)
        self.peers = (C.c_void_p * n_dest)(*peer_ptrs)
        self.flags = (C.c_void_p * n_dest)(*flag_ptrs)
        self.args = (vnode_count, C.c_void_p(vnode_to_dest.data_ptr()), n_dest, my_rank)
        self.cap_rows = cap_rows
        self.counts, self.err = C.c_void_p(counts.data_ptr()), C.c_void_p(err.data_ptr())
        self.total_dev = C.c_void_p(total_dev_ptr)
        self.total_host = C.c_void_p(total_host.data_ptr()) if total_host is not None else None
        self.max_blocks = max_blocks
        self.keep = (vnode_to_dest, counts, err, total_host)
        lib = _lib()
        if not getattr(lib, "_flat_sig", False):
            lib.rwgpu_shuffle_exchange_flat_device.restype = C.c_int32
            lib.rwgpu_shuffle_exchange_flat_device.argtypes = [
                C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                C.c_int32, C.c_void_p]
            lib._flat_sig = True

    def __call__(self, chunk: DeviceChunk, epoch: int, stream):
        ch, keep = chunk.to_abi()
        vc, v2d, n_dest, my_rank = self.args
        _check(_lib().rwgpu_shuffle_exchange_flat_device(C.byref(ch), self.keys, self.n_keys, vc, v2d, n_dest, my_rank, self.peers, self.flags,
                                                         C.c_uint64(epoch), C.c_int64(self.cap_rows), self.counts, self.err, self.total_dev,
                                                         self.total_host, self.max_blocks, _stream_ptr(stream)))


def project_device(chunk: DeviceChunk, exprs, ret_types: Sequence[int], stream: Optional[torch.cuda.Stream] = None):
    """rwgpu_project_device: `exprs` = (abi.RwProjectExpr * m) postfix programs over the chunk's columns.
    -> (columns, valid bytes, has_null uint32[m]) as CUDA tensors (ops / visibility of the chunk pass through)."""
    lib = _lib()
    if not getattr(lib, "_proj_sig", False):
        lib.rwgpu_project_device.restype = C.c_int32
        lib.rwgpu_project_device.argtypes = [C.POINTER(abi.RwChunk), C.POINTER(abi.RwProjectExpr), C.c_int32, C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
        lib._proj_sig = True
    n, m = chunk.n_rows(), len(ret_types)
    cols = [torch.empty(max(n, 1), dtype=TORCH_DTYPE[t], device="cuda") for t in ret_types]
    valid = [torch.empty(max(n, 1), dtype=torch.uint8, device="cuda") for _ in ret_types]
    has_null = torch.zeros(m, dtype=torch.int32, device="cuda")
    ch, keep = chunk.to_abi()
    dptr = (C.c_void_p * m)(*[c.data_ptr() for c in cols])
    vptr = (C.c_void_p * m)(*[v.data_ptr() for v in valid])
    _check(lib.rwgpu_project_device(C.byref(ch), exprs, m, dptr, vptr, C.c_void_p(has_null.data_ptr()), _stream_ptr(stream)))
    return [c[:n] for c in cols], [v[:n] for v in valid], has_null


def filter_device(chunk_abi, n_rows: int, terms, upsert: bool = False, stream: Optional[torch.cuda.Stream] = None):
    """rwgpu_filter_device on an `abi.RwChunk` with DEVICE pointers (a DeviceChunk.to_abi()[0] or the view of a
    `*_device` call).  -> (ops uint8[n], visibility int64[(n+63)//64] packed bits, n_visible int64[1]) CUDA tensors."""
    ops = torch.empty(max(n_rows, 1), dtype=torch.uint8, device="cuda")
    vis = torch.zeros(max((n_rows + 63) // 64, 1), dtype=torch.int64, device="cuda")
    nvis = torch.zeros(1, dtype=torch.int64, device="cuda")
    _check(_lib().rwgpu_filter_device(C.byref(chunk_abi), terms, len(terms), int(upsert), C.c_void_p(ops.data_ptr()),
                                      C.c_void_p(vis.data_ptr()), C.c_void_p(nvis.data_ptr()), _stream_ptr(stream)))
    return ops[:n_rows], vis, nvis
