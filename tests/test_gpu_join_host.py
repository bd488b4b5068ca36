"""GPU: host-chunk pushes (rwgpu_join_push and the rwgpu_join_push_async / rwgpu_join_collect_out pair).

A positional push (output row r = input row r) onto an 8-byte plan hands back output chunks whose update-side columns
are the caller's input buffers: nothing of them crosses PCIe.  The rwgpu_out views are read through ctypes before
release, so the column pointers can be compared with the input buffers.  Whenever the rows stop lining up -- extra
matches, a visibility bitmap, NULLs in an input column, a plan that is not all 8-byte -- the columns are copied back
instead.  Large chunks are cut into sub-batches (2 from 2^16 rows, 4 from 2^17); a varchar payload column takes the
synchronous call from both entry points.  Every output is compared with the CPU oracle fed the same rows."""
import ctypes as C

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
from risingwave_b200.stream_chunk import Column, StreamChunk, net_multiset

pytestmark = pytest.mark.gpu

I64 = [abi.T_INT64] * 4
N_AUCT = 5000


def make(be, bid_types=I64, auct_types=I64):
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    # left = bids (stream key = column 1), right = auctions (stream key = the join key)
    return HashJoinExecutor(be, abi.JOIN_INNER, sl.into_executor(bid_types, [1]), sr.into_executor(auct_types, [0]),
                            JoinParams([0], [1]), JoinParams([0], []), [False], capacity_hint=1000)


def abi_np(t):
    return {abi.T_INT64: np.int64, abi.T_INT32: np.int32}[t]


def chunk(ops, cols, types=I64):
    return StreamChunk(np.asarray(ops, np.uint8), [Column(t, np.asarray(c, abi_np(t))) for t, c in zip(types, cols)])


def auctions(ids):
    ids = np.asarray(ids)
    return chunk(np.full(len(ids), abi.OP_INSERT), [ids, ids * 3, ids * 5, ids * 7])


def bids(rng, n, pk0, types=I64, key_lo=0, key_hi=N_AUCT):
    """keys in [key_lo, key_hi): below N_AUCT every bid matches exactly one stored auction"""
    return chunk(np.full(n, abi.OP_INSERT), [rng.integers(key_lo, key_hi, n), np.arange(n) + pk0, rng.integers(0, 1 << 30, n),
                                             rng.integers(0, 1 << 30, n)], types)


def read_out(be, out):
    """(output chunks, per chunk: row offset, column data pointers) of an rwgpu_out, which is then released"""
    chunks, views = [], []
    lo = 0
    try:
        for i in range(be._out_num_chunks(out)):
            v = abi.RwChunk()
            be.check(be._out_chunk(out, i, C.byref(v)))
            views.append((lo, [v.columns[k].data or 0 for k in range(v.n_cols)]))
            chunks.append(StreamChunk.from_abi(v))
            lo += int(v.n_rows)
    finally:
        be._out_release(out)
    return chunks, views


def push(g, side, ch):
    """rwgpu_join_push; -> (output chunks, views, the input's abi chunk)"""
    be = g.backend
    c, keep = ch.to_abi()
    out = C.c_void_p()
    be.check(be._join_push(g._h, side, C.byref(c), C.byref(out)))
    return read_out(be, out) + ((c, keep),)


def launch(g, side, ch):
    fn = g.backend.lib.rwgpu_join_push_async
    fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(abi.RwChunk)]
    c, keep = ch.to_abi()
    g.backend.check(fn(g._h, side, C.byref(c)))
    return c, keep


def collect(g, inp):
    """rwgpu_join_collect_out of the oldest launch; `inp` (what launch returned) stays alive until here"""
    fn = g.backend.lib.rwgpu_join_collect_out
    fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p)]
    out = C.c_void_p()
    g.backend.check(fn(g._h, C.byref(out)))
    return read_out(g.backend, out) + (inp,)


def alias_flags(res, first_out, types):
    """per output chunk and update-side column (output columns first_out ..): does it point into the input's buffer"""
    _, views, (c, _) = res
    return [ptrs[first_out + k] == c.columns[k].data + lo * np.dtype(abi_np(t)).itemsize for lo, ptrs in views for k, t in enumerate(types)]


def aliased(res, first_out, types):
    flags = alias_flags(res, first_out, types)
    return bool(flags) and all(flags)


def aliased_any(res, first_out, types):
    return any(alias_flags(res, first_out, types))


def check(res, o, side, ch):
    want = net_multiset(o.eq_join_oneside(side, ch))
    assert net_multiset(res[0]) == want
    return sum(want.values())


def setup(cuda, oracle, bid_types=I64):
    g, o = make(cuda, bid_types), make(oracle, bid_types)
    a = auctions(np.arange(N_AUCT))
    assert g.eq_join_oneside(abi.SIDE_RIGHT, a) == []
    assert o.eq_join_oneside(abi.SIDE_RIGHT, a) == []
    return g, o


def test_positional_host_pushes_alias_the_input(cuda, oracle):
    """one match per bid: synchronous pushes (one sub-batch, then 4 and 8 aligned sub-batches) and async pushes with two
    outstanding hand back the caller's bid columns"""
    rng = np.random.default_rng(11)
    g, o = setup(cuda, oracle)
    for s, n in enumerate((30000, 1 << 17, (1 << 19) + 64 * 8)):
        hc = bids(rng, n, 10 ** 7 * s)
        res = push(g, abi.SIDE_LEFT, hc)
        assert sum(ch.capacity() for ch in res[0]) == n and aliased(res, 0, I64)
        assert check(res, o, abi.SIDE_LEFT, hc) == n
    hcs = [bids(rng, 20000 + 3000 * s, 10 ** 8 + 10 ** 6 * s) for s in range(5)]
    inflight = []
    for s in range(len(hcs) + 1):
        if s < len(hcs):
            inflight.append(launch(g, abi.SIDE_LEFT, hcs[s]))
        if s > 0:
            res = collect(g, inflight.pop(0))
            assert aliased(res, 0, I64)
            assert check(res, o, abi.SIDE_LEFT, hcs[s - 1]) == hcs[s - 1].capacity()


def test_extra_matches_are_copied(cuda, oracle):
    """auctions pushed onto several stored bids each: more output rows than input rows, so nothing is aliased"""
    rng = np.random.default_rng(12)
    g, o = setup(cuda, oracle)
    hb = bids(rng, 6000, 0, key_lo=N_AUCT, key_hi=N_AUCT + 2000)  # bids on auctions that do not exist yet
    res = push(g, abi.SIDE_LEFT, hb)
    assert res[0] == [] and check(res, o, abi.SIDE_LEFT, hb) == 0
    ha = auctions(np.arange(N_AUCT, N_AUCT + 1000))
    res = push(g, abi.SIDE_RIGHT, ha)
    assert sum(ch.capacity() for ch in res[0]) > ha.capacity() and not aliased_any(res, 4, I64)
    check(res, o, abi.SIDE_RIGHT, ha)
    # the same through the async pair, with a second push (auctions without bids: no output) outstanding beside it
    hb2 = bids(rng, 20000, 10 ** 6)
    ha2 = auctions(np.arange(N_AUCT + 1000, N_AUCT + 2000))
    first = launch(g, abi.SIDE_RIGHT, ha2)
    second = launch(g, abi.SIDE_RIGHT, auctions(np.arange(N_AUCT + 2000, N_AUCT + 2500)))
    res = collect(g, first)
    assert sum(ch.capacity() for ch in res[0]) > ha2.capacity() and not aliased_any(res, 4, I64)
    check(res, o, abi.SIDE_RIGHT, ha2)
    res = collect(g, second)
    assert check(res, o, abi.SIDE_RIGHT, auctions(np.arange(N_AUCT + 2000, N_AUCT + 2500))) == 0
    res = push(g, abi.SIDE_LEFT, hb2)
    assert aliased(res, 0, I64)
    check(res, o, abi.SIDE_LEFT, hb2)


def test_bitmaps_are_not_aliased(cuda, oracle):
    """a visibility bitmap on the chunk, or NULLs in an input column: the columns are copied, sync and async"""
    rng = np.random.default_rng(13)
    g, o = setup(cuda, oracle)
    hv = bids(rng, 1 << 17, 0)
    hv.vis = rng.random(hv.capacity()) < 0.8
    hn = bids(rng, 30000, 10 ** 6)
    hn.columns[3].valid = rng.random(hn.capacity()) < 0.9
    for hc in (hv, hn):
        res = push(g, abi.SIDE_LEFT, hc)
        assert not aliased_any(res, 0, I64)
        assert check(res, o, abi.SIDE_LEFT, hc) > 0
    hcs = [bids(rng, 30000, 10 ** 7), bids(rng, 30000, 2 * 10 ** 7)]
    hcs[0].vis = rng.random(30000) < 0.7
    hcs[1].columns[2].valid = rng.random(30000) < 0.9
    inflight = [launch(g, abi.SIDE_LEFT, hc) for hc in hcs]
    for hc in hcs:
        res = collect(g, inflight.pop(0))
        assert not aliased_any(res, 0, I64)
        assert check(res, o, abi.SIDE_LEFT, hc) > 0


def test_plan_with_an_int32_column_is_not_aliased(cuda, oracle):
    types = [abi.T_INT64, abi.T_INT64, abi.T_INT32, abi.T_INT64]
    rng = np.random.default_rng(14)
    g, o = setup(cuda, oracle, types)
    hc = bids(rng, 40000, 0, types)
    res = push(g, abi.SIDE_LEFT, hc)
    assert sum(ch.capacity() for ch in res[0]) == 40000 and not aliased_any(res, 0, types)
    assert check(res, o, abi.SIDE_LEFT, hc) == 40000
    hc = bids(rng, 40000, 10 ** 6, types)
    res = collect(g, launch(g, abi.SIDE_LEFT, hc))
    assert not aliased_any(res, 0, types)
    assert check(res, o, abi.SIDE_LEFT, hc) == 40000


def test_sub_batched_varlen_push(cuda, oracle):
    """a varchar payload column on chunks of more than 2^16 rows (two sub-batches), through rwgpu_join_push and through
    rwgpu_join_push_async, which runs the synchronous call for such plans; then deletes of half the rows"""
    tl = [abi.T_INT64, abi.T_INT64, abi.T_VARCHAR, abi.T_INT64]
    rng = np.random.default_rng(15)
    words = [b"", b"a", b"url-" + bytes(range(65, 91)), b"\xf0\x9f\x9a\x80 unicode", b"x" * 300]
    g_sync, g_async, o = make(cuda, tl), make(cuda, tl), make(oracle, tl)
    a = auctions(np.arange(N_AUCT))
    for ex in (g_sync, g_async, o):
        assert ex.eq_join_oneside(abi.SIDE_RIGHT, a) == []
    n = (1 << 16) + 5000
    key = rng.integers(0, N_AUCT + 300, n)  # some bids match nothing
    url = np.empty(n, dtype=object)
    url[:] = [words[i] for i in rng.integers(0, len(words), n)]
    url_valid = rng.random(n) < 0.95
    cols = [Column(abi.T_INT64, key.astype(np.int64)), Column(abi.T_INT64, np.arange(n, dtype=np.int64)), Column(abi.T_VARCHAR, url, url_valid),
            Column(abi.T_INT64, rng.integers(0, 1000, n).astype(np.int64))]
    ins = StreamChunk(np.full(n, abi.OP_INSERT, np.uint8), cols)
    dels = StreamChunk(np.full(n, abi.OP_DELETE, np.uint8), cols, rng.random(n) < 0.5)
    for hc in (ins, dels):
        want = net_multiset(o.eq_join_oneside(abi.SIDE_LEFT, hc))
        assert sum(abs(v) for v in want.values()) > n // 3
        assert net_multiset(g_sync.eq_join_oneside(abi.SIDE_LEFT, hc)) == want
        g_async.eq_join_oneside_launch(abi.SIDE_LEFT, hc)
        assert net_multiset(g_async.eq_join_oneside_collect()) == want
