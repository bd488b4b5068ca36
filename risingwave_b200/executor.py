"""Host-side mirror of the reference's executor interface for the HashAgg / HashJoin path.

Reference surface being mirrored (Rust, cannot be compiled here):
  * `trait Execute { fn execute(self: Box<Self>) -> BoxedMessageStream }`  src/stream/src/executor/mod.rs:240-253
  * `Message = Chunk | Barrier | Watermark`                                 mod.rs:1283-1299
  * `HashAggExecutor`   src/stream/src/executor/aggregate/hash_agg.rs (execute_inner :561-706)
  * `HashJoinExecutor`  src/stream/src/executor/hash_join.rs (into_stream :582-751)
  * `barrier_align`     src/stream/src/executor/barrier_align.rs:44-165
  * test harness `MockSource` / `MessageSender` / `StreamExecutorTestExt`
    src/stream/src/executor/test_utils/{mock_source.rs:16-137, mod.rs:61-124}

This file is the *driver* used by tests / bench; the production drop-in is the Rust shim shown in
INTEGRATION.md which forwards to the same C ABI (include/rwgpu.h).  All compute happens behind the
`Backend` (a ctypes view of a shared library exporting the rwgpu ABI); the product constructs
`Backend.cuda()`, which loads librwgpu.so and fails loudly if it is absent.
"""
from __future__ import annotations

import ctypes as C
import heapq
import re
from collections import deque
from dataclasses import dataclass, field
from typing import Deque, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .stream_chunk import StreamChunk


# =============================================================================== Backend
class Backend:
    """ctypes binding of one implementation of the rwgpu C ABI (symbol prefix selects it)."""

    def __init__(self, lib: C.CDLL, prefix: str = "rwgpu_"):
        self.lib = lib
        self.prefix = prefix
        f = self._fn
        f("out_num_chunks", C.c_int32, [C.c_void_p])
        f("out_num_rows", C.c_int64, [C.c_void_p])
        f("out_chunk", C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk)])
        f("out_release", None, [C.c_void_p])
        f("agg_create", C.c_int32, [C.POINTER(abi.RwAggDesc), C.POINTER(C.c_void_p)])
        f("agg_destroy", None, [C.c_void_p])
        f("agg_push", C.c_int32, [C.c_void_p, C.POINTER(abi.RwChunk)])
        f("agg_flush", C.c_int32, [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)])
        f("join_create", C.c_int32, [C.POINTER(abi.RwJoinDesc), C.POINTER(C.c_void_p)])
        f("join_destroy", None, [C.c_void_p])
        f("join_push", C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk), C.POINTER(C.c_void_p)])
        f("join_barrier", C.c_int32, [C.c_void_p, C.c_uint64])
        f("vnode_compute", C.c_int32, [C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                       C.POINTER(C.c_uint16)])
        f("dispatch_rewrite_ops", C.c_int32, [C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32,
                                              C.POINTER(C.c_uint8)])
        f("filter", C.c_int32, [C.POINTER(abi.RwChunk), C.POINTER(abi.RwFilterTerm), C.c_int32, C.c_int32, C.POINTER(C.c_uint8),
                                C.POINTER(C.c_uint64), C.POINTER(C.c_int64)])
        f("project", C.c_int32, [C.POINTER(abi.RwChunk), C.POINTER(abi.RwProjectExpr), C.c_int32, C.POINTER(C.c_void_p),
                                 C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)])
        f("last_error", C.c_char_p, [])

    @staticmethod
    def cuda() -> "Backend":
        return Backend(abi.load_library(), "rwgpu_")

    def _fn(self, name, restype, argtypes):
        fn = getattr(self.lib, self.prefix + name)
        fn.restype = restype
        fn.argtypes = argtypes
        setattr(self, "_" + name, fn)

    def check(self, rc: int):
        if rc != abi.RW_OK:
            msg = self._last_error()
            raise abi.RwError(rc, msg.decode() if msg else "")

    def take_out(self, out_ptr) -> List[StreamChunk]:
        chunks = []
        try:
            for i in range(self._out_num_chunks(out_ptr)):
                view = abi.RwChunk()
                self.check(self._out_chunk(out_ptr, i, C.byref(view)))
                chunks.append(StreamChunk.from_abi(view))
        finally:
            self._out_release(out_ptr)
        return chunks

    # ---- shuffle helpers (host)
    def vnode_compute(self, chunk: StreamChunk, keys: Sequence[int], vnode_count: int = 256):
        import numpy as np
        ch, keep = chunk.to_abi()
        k = (C.c_int32 * len(keys))(*keys)
        out = np.zeros(chunk.capacity(), dtype=np.uint16)
        self.check(self._vnode_compute(C.byref(ch), k, len(keys), vnode_count,
                                       out.ctypes.data_as(C.POINTER(C.c_uint16))))
        return out

    def dispatch_rewrite_ops(self, chunk: StreamChunk, keys: Sequence[int]):
        import numpy as np
        ch, keep = chunk.to_abi()
        k = (C.c_int32 * len(keys))(*keys)
        out = np.zeros(chunk.capacity(), dtype=np.uint8)
        self.check(self._dispatch_rewrite_ops(C.byref(ch), k, len(keys), out.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out


# =============================================================================== Message
@dataclass
class Barrier:
    epoch: int
    stop: bool = False


@dataclass
class Watermark:
    col_idx: int
    data_type: int
    val: int


@dataclass
class Message:
    """Message::{Chunk, Barrier, Watermark}  (mod.rs:1283-1299)"""
    chunk: Optional[StreamChunk] = None
    barrier: Optional[Barrier] = None
    watermark: Optional[Watermark] = None


PENDING = object()  # Poll::Pending


class MessageSender:
    """MessageSender (test_utils/mock_source.rs:39-108)."""

    def __init__(self, q: Deque[Message]):
        self._q = q

    def push_chunk(self, chunk: StreamChunk):
        self._q.append(Message(chunk=chunk))

    def push_barrier(self, epoch: int, stop: bool = False):
        self._q.append(Message(barrier=Barrier(epoch, stop)))

    def push_watermark(self, col_idx: int, data_type: int, val: int):
        self._q.append(Message(watermark=Watermark(col_idx, data_type, val)))


class MockSource:
    """MockSource::channel() (test_utils/mock_source.rs:110-137): an input executor fed by hand."""

    def __init__(self, q: Deque[Message], schema: Sequence[int] = (), stream_key: Sequence[int] = ()):
        self._q = q
        self.schema = list(schema)
        self.stream_key = list(stream_key)

    @staticmethod
    def channel() -> Tuple[MessageSender, "MockSource"]:
        q: Deque[Message] = deque()
        return MessageSender(q), MockSource(q)

    def into_executor(self, schema: Sequence[int], stream_key: Sequence[int]) -> "MockSource":
        self.schema = list(schema)
        self.stream_key = list(stream_key)
        return self

    def poll(self):
        return self._q.popleft() if self._q else PENDING


class MessageStream:
    """BoxedMessageStream + StreamExecutorTestExt (test_utils/mod.rs:61-124)."""

    def __init__(self, gen: Iterator):
        self._gen = gen

    def poll_next(self):
        return next(self._gen)

    def next_unwrap_pending(self):
        m = self.poll_next()
        assert m is PENDING, f"expected pending, got {m}"

    def next_unwrap_ready(self) -> Message:
        m = self.poll_next()
        assert m is not PENDING, "expected ready, got pending"
        return m

    def next_unwrap_ready_chunk(self) -> StreamChunk:
        m = self.next_unwrap_ready()
        assert m.chunk is not None, f"expected chunk, got {m}"
        return m.chunk

    def next_unwrap_ready_barrier(self) -> Barrier:
        m = self.next_unwrap_ready()
        assert m.barrier is not None, f"expected barrier, got {m}"
        return m.barrier

    def next_unwrap_ready_watermark(self) -> Watermark:
        m = self.next_unwrap_ready()
        assert m.watermark is not None, f"expected watermark, got {m}"
        return m.watermark

    def drain_until_pending(self) -> List[Message]:
        """check_until_pending (tests/integration_tests/snapshot.rs:180-217)."""
        out = []
        while True:
            m = self.poll_next()
            if m is PENDING:
                return out
            out.append(m)


# =============================================================================== AggCall
_PG_TYPES = {"int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "float4": abi.T_FLOAT32,
             "float8": abi.T_FLOAT64, "decimal": abi.T_DECIMAL, "boolean": abi.T_BOOL, "date": abi.T_DATE,
             "timestamp": abi.T_TIMESTAMP, "timestamptz": abi.T_TIMESTAMPTZ, "serial": abi.T_SERIAL}
_AGG_KINDS = {"count": abi.AGG_COUNT, "sum": abi.AGG_SUM, "min": abi.AGG_MIN, "max": abi.AGG_MAX,
              "sum0": abi.AGG_SUM0}


@dataclass
class AggCall:
    kind: int
    arg_col: int
    ret_type: int
    arg_type: int = 0

    @staticmethod
    def from_pretty(s: str) -> "AggCall":
        """`(sum:int8 $1:int8)` / `(count:int8)`  -- AggCall::from_pretty (src/expr/core/src/aggregate/def.rs)."""
        m = re.fullmatch(r"\(\s*(\w+):(\w+)(?:\s+\$(\d+):(\w+))?\s*\)", s.strip())
        if not m:
            raise ValueError(f"bad agg call {s!r}")
        kind, ret, idx, at = m.groups()
        return AggCall(_AGG_KINDS[kind], -1 if idx is None else int(idx), _PG_TYPES[ret],
                       0 if at is None else _PG_TYPES[at])


# =============================================================================== HashAgg
class HashAggExecutor:
    """Mirror of HashAggExecutor<K,S> (aggregate/hash_agg.rs); arguments follow
    `new_boxed_hash_agg_executor` (test_utils/agg_executor.rs:224-300)."""

    def __init__(self, backend: Backend, input: MockSource, is_append_only: bool, agg_calls: Sequence[AggCall],
                 row_count_index: int, group_key_indices: Sequence[int], chunk_size: int = 1024,
                 strict_consistency: bool = True, group_capacity_hint: int = 0):
        self.backend = backend
        self.input = input
        n_in = len(input.schema)
        self._types = (C.c_int32 * n_in)(*input.schema)
        self._keys = (C.c_int32 * max(1, len(group_key_indices)))(*group_key_indices)
        self._calls = (abi.RwAggCall * max(1, len(agg_calls)))()
        for i, c in enumerate(agg_calls):
            self._calls[i].kind = c.kind
            self._calls[i].arg_col = c.arg_col
            self._calls[i].ret_type = c.ret_type
        d = abi.RwAggDesc()
        d.n_input_cols = n_in
        d.input_types = self._types
        d.n_group_keys = len(group_key_indices)
        d.group_key_indices = self._keys
        d.n_calls = len(agg_calls)
        d.calls = self._calls
        d.row_count_index = row_count_index
        d.is_append_only = int(is_append_only)
        d.chunk_size = chunk_size
        d.strict_consistency = int(strict_consistency)
        d.group_capacity_hint = group_capacity_hint
        self._desc = d
        h = C.c_void_p()
        backend.check(backend._agg_create(C.byref(d), C.byref(h)))
        self._h = h
        self.schema = [input.schema[k] for k in group_key_indices] + [c.ret_type for c in agg_calls]

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self.backend._agg_destroy(h)
            self._h = None

    # direct operator calls (what the Rust shim would issue)
    def apply_chunk(self, chunk: StreamChunk):
        ch, keep = chunk.to_abi()
        self.backend.check(self.backend._agg_push(self._h, C.byref(ch)))

    def flush_data(self, epoch: int) -> List[StreamChunk]:
        out = C.c_void_p()
        self.backend.check(self.backend._agg_flush(self._h, epoch, C.byref(out)))
        return self.backend.take_out(out)

    # state persistence (rwgpu.h rwgpu_agg_snapshot / rwgpu_agg_restore; CUDA backend only)
    def snapshot(self) -> Tuple[List[StreamChunk], List[StreamChunk]]:
        """-> (intermediate-state rows, materialized-input rows of retractable min / max) as chunks"""
        fn = self.backend.lib.rwgpu_agg_snapshot
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        a, b = C.c_void_p(), C.c_void_p()
        self.backend.check(fn(self._h, C.byref(a), C.byref(b)))
        return self.backend.take_out(a), self.backend.take_out(b)

    def restore(self, states: Optional[StreamChunk], minput: Optional[StreamChunk] = None):
        fn = self.backend.lib.rwgpu_agg_restore
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.POINTER(abi.RwChunk), C.POINTER(abi.RwChunk)]
        sa, k1 = states.to_abi()
        if minput is not None:
            ma, k2 = minput.to_abi()
            self.backend.check(fn(self._h, C.byref(sa), C.byref(ma)))
        else:
            self.backend.check(fn(self._h, C.byref(sa), None))

    def execute(self) -> MessageStream:
        return MessageStream(self._run())

    def _run(self):
        # execute_inner (hash_agg.rs:561-706): first barrier initialises; chunks apply; a barrier
        # flushes deltas, then is forwarded.
        first = True
        while True:
            m = self.input.poll()
            if m is PENDING:
                yield PENDING
                continue
            if m.chunk is not None:
                self.apply_chunk(m.chunk)
            elif m.barrier is not None:
                if first:
                    first = False
                    yield m
                    continue
                for ch in self.flush_data(m.barrier.epoch):
                    yield Message(chunk=ch)
                yield m
            else:
                yield m  # watermarks on group keys pass through (hash_agg.rs:628-637, simplified)


# =============================================================================== HashJoin
@dataclass
class JoinParams:
    """JoinParams (hash_join.rs:75-89)."""
    join_key_indices: List[int]
    deduped_pk_indices: List[int]


_CMP = {"less_than": abi.CMP_LT, "less_than_or_equal": abi.CMP_LE, "greater_than": abi.CMP_GT,
        "greater_than_or_equal": abi.CMP_GE, "equal": abi.CMP_EQ, "not_equal": abi.CMP_NE}


def parse_cond(text: Optional[str]) -> Tuple[int, int, int]:
    """`(less_than:boolean $1:int8 $3:int8)` -> (cmp, lhs, rhs) (build_from_pretty subset)."""
    if text is None:
        return (abi.CMP_NONE, 0, 0)
    m = re.fullmatch(r"\(\s*(\w+):boolean\s+\$(\d+):\w+\s+\$(\d+):\w+\s*\)", text.strip())
    if not m:
        raise ValueError(f"unsupported join condition {text!r}")
    return (_CMP[m.group(1)], int(m.group(2)), int(m.group(3)))


class BufferedWatermarks:
    """BufferedWatermarks<Id> (src/stream/src/executor/watermark/mod.rs:38-115): per upstream id the smallest buffered
    watermark sits in a heap, the later ones are staged behind it; a watermark is emitted when EVERY upstream has one in
    the heap (the smallest wins), and equal ones that follow are swallowed.  Watermarks order by value (mod.rs:1219-1222)
    and compare equal on (col_idx, value)."""
    MAX_STAGED = 1024

    def __init__(self, ids: Sequence[int]):
        self.first: List[Tuple[int, int, Watermark]] = []  # heap of (value, id, watermark)
        self.staged = {i: [False, deque()] for i in sorted(ids)}  # id -> [in_heap, staged watermarks]

    def handle_watermark(self, buffer_id: int, wm: Watermark) -> Optional[Watermark]:
        st = self.staged[buffer_id]
        if st[0]:
            if len(st[1]) >= self.MAX_STAGED:
                st[1].popleft()
            st[1].append(wm)
            return None
        st[0] = True
        heapq.heappush(self.first, (wm.val, buffer_id, wm))
        return self.check_watermark_heap()

    def check_watermark_heap(self) -> Optional[Watermark]:
        n, emit = len(self.staged), None
        while self.first and (len(self.first) == n or (emit is not None and (emit.col_idx, emit.val) ==
                                                       (self.first[0][2].col_idx, self.first[0][2].val))):
            _, i, wm = heapq.heappop(self.first)
            emit = wm
            st = self.staged[i]
            if st[1]:
                nxt = st[1].popleft()
                heapq.heappush(self.first, (nxt.val, i, nxt))
            else:
                st[0] = False
        return emit


class HashJoinExecutor:
    """Mirror of HashJoinExecutor<K,S,T,E>::new (hash_join.rs:255-301)."""

    def __init__(self, backend: Backend, join_type: int, input_l: MockSource, input_r: MockSource,
                 params_l: JoinParams, params_r: JoinParams, null_safe: Sequence[bool],
                 output_indices: Optional[Sequence[int]] = None, cond: Optional[str] = None,
                 is_append_only: bool = False, chunk_size: int = 1024, strict_consistency: bool = True,
                 capacity_hint=0, stored_rows_hint=0, watermark_indices_in_jk: Sequence[Tuple[int, bool]] = ()):
        """capacity_hint: expected distinct join keys (one number or (left, right)); stored_rows_hint: expected rows stored
        per side (same shapes; 0 = two per expected key); watermark_indices_in_jk: (join key position, clean state?) pairs
        as in HashJoinExecutor::new (hash_join.rs:255-301)"""
        self.backend = backend
        self.input_l, self.input_r = input_l, input_r
        self._keep = []
        d = abi.RwJoinDesc()
        d.join_type = join_type
        d.n_keys = len(params_l.join_key_indices)
        hints = capacity_hint if isinstance(capacity_hint, (tuple, list)) else (capacity_hint, capacity_hint)
        shints = stored_rows_hint if isinstance(stored_rows_hint, (tuple, list)) else (stored_rows_hint, stored_rows_hint)
        for side, inp, p, hint, shint in ((d.left, input_l, params_l, hints[0], shints[0]), (d.right, input_r, params_r, hints[1], shints[1])):
            types = (C.c_int32 * max(1, len(inp.schema)))(*inp.schema)
            keys = (C.c_int32 * max(1, len(p.join_key_indices)))(*p.join_key_indices)
            pk = (C.c_int32 * max(1, len(p.deduped_pk_indices)))(*p.deduped_pk_indices)
            sk = (C.c_int32 * max(1, len(inp.stream_key)))(*inp.stream_key)
            self._keep += [types, keys, pk, sk]
            side.n_cols = len(inp.schema)
            side.types = types
            side.key_indices = keys
            side.n_pk = len(p.deduped_pk_indices)
            side.pk_indices = pk
            side.n_stream_key = len(inp.stream_key)
            side.stream_key = sk
            side.row_capacity_hint = int(hint)  # expected distinct join keys of the side
            side.stored_rows_hint = int(shint)
        ns = (C.c_uint8 * max(1, len(null_safe)))(*[int(b) for b in null_safe])
        d.null_safe = ns
        if join_type in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
            nat = list(input_l.schema)
        elif join_type in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
            nat = list(input_r.schema)
        else:
            nat = list(input_l.schema) + list(input_r.schema)
        if output_indices is None:
            output_indices = list(range(len(nat)))
        oi = (C.c_int32 * max(1, len(output_indices)))(*output_indices)
        d.n_output = len(output_indices)
        d.output_indices = oi
        cmp_, lhs, rhs = parse_cond(cond)
        d.cond.cmp, d.cond.lhs, d.cond.rhs = cmp_, lhs, rhs
        d.is_append_only = int(is_append_only)
        d.chunk_size = chunk_size
        d.strict_consistency = int(strict_consistency)
        self._keep += [ns, oi]
        self._desc = d
        h = C.c_void_p()
        backend.check(backend._join_create(C.byref(d), C.byref(h)))
        self._h = h
        self.schema = [nat[i] for i in output_indices]
        # watermark handling (hash_join.rs:791-891): i2o_mapping_indexed per side (input column -> output positions)
        n_l = len(input_l.schema)
        semi_l = join_type in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI)
        semi_r = join_type in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI)
        self._i2o = ({}, {})
        for o, i in enumerate(output_indices):
            if semi_l or (not semi_r and i < n_l):
                self._i2o[0].setdefault(i, []).append(o)
            else:
                self._i2o[1].setdefault(i if semi_r else i - n_l, []).append(o)
        self._jk = (list(params_l.join_key_indices), list(params_r.join_key_indices))
        self._wm_in_jk = list(watermark_indices_in_jk)
        self._wm_buffers = {}

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self.backend._join_destroy(h)
            self._h = None

    def handle_watermark(self, side: int, wm: Watermark) -> List[Watermark]:
        """HashJoinExecutor::handle_watermark, the join-key part (hash_join.rs:791-842): a watermark on a join key column
        is buffered per join key position; what BOTH sides have passed is emitted for every output column fed by that
        key on either side (the update side's first), and -- where the plan asks for it -- both sides' state is cleaned
        below it (JoinHashMap::update_watermark = rwgpu_join_update_watermark, applied at the next barrier).  Inequality
        pairs (:844-889) stay with the CPU executor: their `cond` is not offloaded either."""
        out: List[Watermark] = []
        upd, mat = side, 1 - side
        for idx, col in enumerate(self._jk[upd]):
            if col != wm.col_idx:
                continue
            buf = self._wm_buffers.setdefault(idx, BufferedWatermarks([abi.SIDE_LEFT, abi.SIDE_RIGHT]))
            sel = buf.handle_watermark(side, wm)
            if sel is None:
                continue
            if any(p == idx and clean for p, clean in self._wm_in_jk) and hasattr(self.backend.lib, "rwgpu_join_update_watermark") \
                    and self.backend.prefix == "rwgpu_":
                self.update_watermark(mat, idx, sel.val)
                self.update_watermark(upd, idx, sel.val)
            for o in self._i2o[upd].get(self._jk[upd][idx], []) + self._i2o[mat].get(self._jk[mat][idx], []):
                out.append(Watermark(o, sel.data_type, sel.val))
        return out

    # direct operator calls (what the Rust shim would issue)
    def eq_join_oneside(self, side: int, chunk: StreamChunk) -> List[StreamChunk]:
        ch, keep = chunk.to_abi()
        out = C.c_void_p()
        self.backend.check(self.backend._join_push(self._h, side, C.byref(ch), C.byref(out)))
        return self.backend.take_out(out)

    # launch / collect split for host chunks (rwgpu.h rwgpu_join_push_async / rwgpu_join_collect_out; CUDA backend only)
    def eq_join_oneside_launch(self, side: int, chunk: StreamChunk):
        """enqueue the push of `chunk`; its buffers are kept alive here until `eq_join_oneside_collect` returns the output"""
        fn = self.backend.lib.rwgpu_join_push_async
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk)]
        ch, keep = chunk.to_abi()
        self.backend.check(fn(self._h, side, C.byref(ch)))
        if not hasattr(self, "_inflight"):
            self._inflight = []
        self._inflight.append((chunk, ch, keep))

    def eq_join_oneside_collect(self) -> List[StreamChunk]:
        """output of the OLDEST outstanding launch"""
        fn = self.backend.lib.rwgpu_join_collect_out
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p)]
        out = C.c_void_p()
        self.backend.check(fn(self._h, C.byref(out)))
        res = self.backend.take_out(out)  # (copies out of the rwgpu_out, which may alias the input buffers, then releases it)
        self._inflight.pop(0)
        return res

    def flush_data(self, epoch: int):
        self.backend.check(self.backend._join_barrier(self._h, epoch))

    def update_watermark(self, side: int, key_pos: int, value: int):
        """JoinHashMap::update_watermark: rows of `side` with join key column `key_pos` < value leave at the next barrier"""
        fn = self.backend.lib.rwgpu_join_update_watermark
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64]
        self.backend.check(fn(self._h, side, key_pos, value))

    # state persistence (rwgpu.h rwgpu_join_snapshot / rwgpu_join_restore; CUDA backend only)
    def snapshot(self, side: int) -> List[StreamChunk]:
        fn = self.backend.lib.rwgpu_join_snapshot
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        out = C.c_void_p()
        self.backend.check(fn(self._h, side, C.byref(out)))
        return self.backend.take_out(out)

    def restore(self, side: int, rows: StreamChunk):
        fn = self.backend.lib.rwgpu_join_restore
        fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk)]
        ch, keep = rows.to_abi()
        self.backend.check(fn(self._h, side, C.byref(ch)))

    def execute(self) -> MessageStream:
        return MessageStream(self._run())

    def _run(self):
        # into_stream (hash_join.rs:582-751) over barrier_align (barrier_align.rs:44-165).  The
        # reference picks the polled side at random (:67); we prefer left, which is one of its
        # legal interleavings.  A side that delivered its barrier is blocked until the other does.
        blocked = [None, None]
        inputs = (self.input_l, self.input_r)
        while True:
            progressed = False
            for s in (abi.SIDE_LEFT, abi.SIDE_RIGHT):
                if blocked[s] is not None:
                    continue
                m = inputs[s].poll()
                if m is PENDING:
                    continue
                progressed = True
                if m.chunk is not None:
                    for ch in self.eq_join_oneside(s, m.chunk):
                        yield Message(chunk=ch)
                elif m.barrier is not None:
                    blocked[s] = m.barrier
                    if blocked[0] is not None and blocked[1] is not None:
                        assert blocked[0].epoch == blocked[1].epoch, "barrier epoch mismatch"
                        b = blocked[0]
                        blocked = [None, None]
                        self.flush_data(b.epoch)
                        yield Message(barrier=b)
                else:  # AlignedMessage::WatermarkLeft / WatermarkRight (hash_join.rs:711-722)
                    for w in self.handle_watermark(s, m.watermark):
                        yield Message(watermark=w)
                break
            if not progressed:
                yield PENDING


# =============================================================================== Filter
def _filter_terms(text: str) -> List[Tuple[int, int, int, int, str, str]]:
    """parse_filter_expr's terms, each with the type annotations of its two operands"""
    text = text.strip()
    m = re.fullmatch(r"\(\s*and:boolean\s+(\(.*\))\s+(\(.*\))\s*\)", text, re.S)
    if m:
        # split the two operands at the top-level parenthesis boundary
        body = text[text.index("and:boolean") + len("and:boolean"):-1].strip()
        depth, cut = 0, None
        for i, c in enumerate(body):
            depth += c == "("
            depth -= c == ")"
            if depth == 0:
                cut = i + 1
                break
        return _filter_terms(body[:cut]) + _filter_terms(body[cut:])
    m = re.fullmatch(r"\(\s*(\w+):boolean\s+\$(\d+):(\w+)\s+(?:\$(\d+)|(-?\d+)):(\w+)\s*\)", text)
    if not m or m.group(1) not in _CMP:
        raise ValueError(f"unsupported filter expression {text!r}")
    if m.group(4) is not None:
        return [(_CMP[m.group(1)], int(m.group(2)), int(m.group(4)), 0, m.group(3), m.group(6))]
    return [(_CMP[m.group(1)], int(m.group(2)), -1, int(m.group(5)), m.group(3), m.group(6))]


def parse_filter_expr(text: str) -> List[Tuple[int, int, int, int]]:
    """build_from_pretty subset -> conjunction terms (cmp, lhs_col, rhs_col or -1, rhs_const):
    `(greater_than:boolean $0:int8 $1:int8)`, `(greater_than:boolean $1:int8 10:int8)`,
    `(and:boolean (...) (...))`."""
    return [t[:4] for t in _filter_terms(text)]


# the type names build_from_pretty parses (src/expr/core/src/expr/build.rs:325-340), for the column types a chunk carries
_FILTER_TYPES = {"boolean": abi.T_BOOL, "int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "serial": abi.T_SERIAL,
                 "float4": abi.T_FLOAT32, "float8": abi.T_FLOAT64, "decimal": abi.T_DECIMAL, "date": abi.T_DATE,
                 "time": abi.T_TIME, "timestamp": abi.T_TIMESTAMP, "timestamptz": abi.T_TIMESTAMPTZ,
                 "varchar": abi.T_VARCHAR, "bytea": abi.T_BYTEA}
_FILTER_INTS = (abi.T_INT16, abi.T_INT32, abi.T_INT64)


_EX_BIN = {"add": abi.EX_ADD, "subtract": abi.EX_SUB, "multiply": abi.EX_MUL, "divide": abi.EX_DIV, "modulus": abi.EX_MOD,
           "tumble_start": abi.EX_TUMBLE_START, "tumble_end": abi.EX_TUMBLE_END}
_EX_TYPES = {"int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "date": abi.T_DATE, "time": abi.T_TIME,
             "timestamp": abi.T_TIMESTAMP, "timestamptz": abi.T_TIMESTAMPTZ, "serial": abi.T_SERIAL}


def parse_project_expr(text: str) -> Tuple[List[Tuple[int, int, int]], int]:
    """build_from_pretty subset -> (postfix program [(op, arg, value)], return type): `$1:int8`, `42:int8`,
    `(add:int8 $0:int8 $1:int8)`, `(divide:int8 (multiply:int8 $2:int8 908:int8) 1000:int8)`, `(neg:int8 $0:int8)`,
    `(tumble_start:timestamptz $3:timestamptz 10000000:int8)` (the interval in microseconds)."""
    toks = re.findall(r"\(|\)|[^\s()]+", text)
    pos = 0

    def parse():
        nonlocal pos
        t = toks[pos]
        pos += 1
        if t == "(":
            name, ty = toks[pos].split(":")
            pos += 1
            args = []
            while toks[pos] != ")":
                args.append(parse())
            pos += 1
            if ty not in _EX_TYPES:
                raise ValueError(f"unsupported expression type in {text!r}")
            prog = [op for a in args for op in a[0]]
            # an operator's `arg` is its own result type: each checked op overflows at that width (rwgpu.h)
            if name == "neg" and len(args) == 1:
                return prog + [(abi.EX_NEG, _EX_TYPES[ty], 0)], _EX_TYPES[ty]
            if name not in _EX_BIN or len(args) != 2:
                raise ValueError(f"unsupported expression {name!r} in {text!r}")
            return prog + [(_EX_BIN[name], _EX_TYPES[ty], 0)], _EX_TYPES[ty]
        val, ty = t.rsplit(":", 1)
        if ty not in _EX_TYPES:
            raise ValueError(f"unsupported expression type in {text!r}")
        if val.startswith("$"):
            return [(abi.EX_COL, int(val[1:]), 0)], _EX_TYPES[ty]
        return [(abi.EX_CONST, 0, int(val))], _EX_TYPES[ty]

    prog, ty = parse()
    if pos != len(toks):
        raise ValueError(f"trailing tokens in {text!r}")
    return prog, ty


class ProjectExecutor:
    """Mirror of ProjectExecutor::new(ctx, input, exprs, ...) (project/project_scalar.rs:40-76) for the expressions the
    device path evaluates (integer arithmetic, tumble windows); `apply_project_exprs` = :91-108."""

    def __init__(self, backend: Backend, input: MockSource, exprs: Sequence[str]):
        self.backend, self.input = backend, input
        self._keep = []
        self._exprs = (abi.RwProjectExpr * len(exprs))()
        self.schema = []
        for k, text in enumerate(exprs):
            prog, ty = parse_project_expr(text)
            ops = (abi.RwExprOp * len(prog))()
            for i, (op, arg, val) in enumerate(prog):
                ops[i].op, ops[i].arg, ops[i].value = op, arg, val
            self._keep.append(ops)
            self._exprs[k].ops, self._exprs[k].n_ops, self._exprs[k].ret_type = ops, len(prog), ty
            self.schema.append(ty)

    def apply_project_exprs(self, chunk: StreamChunk) -> StreamChunk:
        from .stream_chunk import NP_DTYPE, Column
        ch, keep = chunk.to_abi()
        n, m = chunk.capacity(), len(self.schema)
        data = [np.zeros(max(n, 1), dtype=NP_DTYPE[t]) for t in self.schema]
        valid = [np.zeros(max((n + 63) // 64, 1), dtype=np.uint64) for _ in self.schema]
        dptr = (C.c_void_p * m)(*[d.ctypes.data for d in data])
        vptr = (C.c_void_p * m)(*[v.ctypes.data for v in valid])
        has_null = (C.c_uint32 * m)()
        self.backend.check(self.backend._project(C.byref(ch), self._exprs, m, dptr, vptr, has_null))
        cols = []
        for k, t in enumerate(self.schema):
            v = None
            if has_null[k]:
                v = np.unpackbits(valid[k].view(np.uint8), bitorder="little")[:n].astype(bool)
            cols.append(Column(t, data[k][:n].copy(), v))
        return StreamChunk(chunk.ops.copy(), cols, chunk.vis)

    def execute(self) -> MessageStream:
        return MessageStream(self._run())

    def _run(self):
        while True:
            m = self.input.poll()
            if m is PENDING:
                yield PENDING
            elif m.chunk is not None:
                yield Message(chunk=self.apply_project_exprs(m.chunk))
            else:
                yield m


class FilterExecutor:
    """Mirror of FilterExecutor / UpsertFilterExecutor::new(ctx, input, expr) (filter.rs:33-56) for predicates
    the device path evaluates (conjunctions of integer comparisons)."""

    def __init__(self, backend: Backend, input: MockSource, expr: str, upsert: bool = False):
        self.backend, self.input, self.upsert = backend, input, upsert
        self.schema = list(input.schema)
        terms = _filter_terms(expr)
        self._terms = (abi.RwFilterTerm * len(terms))()
        for k, (cmp, lhs, rhs, const, lty, rty) in enumerate(terms):
            # an operand's annotation is its column's type; a constant's is the left operand's, or another integer type
            # beside an integer one (cmp.rs:44-51 widens them).  The backend sees raw integers and cannot tell.
            for col, ty in ((lhs, lty), (rhs, rty)):
                if col >= 0 and (col >= len(self.schema) or _FILTER_TYPES.get(ty) != self.schema[col]):
                    raise ValueError(f"filter operand ${col}:{ty} does not match the input schema in {expr!r}")
            lt, ct = _FILTER_TYPES.get(lty), _FILTER_TYPES.get(rty)
            if rhs < 0 and ct != lt and not (ct in _FILTER_INTS and lt in _FILTER_INTS):
                raise ValueError(f"filter constant {const}:{rty} does not compare with ${lhs}:{lty} in {expr!r}")
            self._terms[k].cmp, self._terms[k].lhs_col, self._terms[k].rhs_col, self._terms[k].rhs_const = cmp, lhs, rhs, const

    def filter(self, chunk: StreamChunk) -> Optional[StreamChunk]:
        """FilterExecutorInner::filter (filter.rs:58-150): same columns, new ops / visibility; None if no row stays visible"""
        ch, keep = chunk.to_abi()
        n = chunk.capacity()
        ops = np.zeros(max(n, 1), dtype=np.uint8)
        vis = np.zeros(max((n + 63) // 64, 1), dtype=np.uint64)
        nvis = C.c_int64(0)
        self.backend.check(self.backend._filter(C.byref(ch), self._terms, len(self._terms), int(self.upsert),
                                                ops.ctypes.data_as(C.POINTER(C.c_uint8)), vis.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                C.byref(nvis)))
        if nvis.value == 0:
            return None
        bits = np.unpackbits(vis.view(np.uint8), bitorder="little")[:n].astype(bool)
        return StreamChunk(ops[:n].copy(), chunk.columns, bits)

    def execute(self) -> MessageStream:
        return MessageStream(self._run())

    def _run(self):
        # execute_inner (filter.rs:172-194): chunks are filtered, everything else passes through
        while True:
            m = self.input.poll()
            if m is PENDING:
                yield PENDING
            elif m.chunk is not None:
                out = self.filter(m.chunk)
                if out is not None:
                    yield Message(chunk=out)
            else:
                yield m
