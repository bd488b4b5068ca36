"""HashAgg watermark-driven state cleaning at every group-key type, on every barrier entry point, against the typed
restatement of test_agg_types.py / test_state_types.py extended with the state table's range delete, and the host
mirrors' watermark derivation.

The reference (src/stream/src/executor/aggregate/hash_agg.rs):
  * execute_inner (:561-706): a watermark on a column that is not a group key is dropped; one on group key `seq` is
    buffered as `seq`, the later one replacing the earlier; at a barrier the delta chunks go out first, then the
    buffered watermarks in seq order, then the barrier.  The window column is the group key that leads the
    intermediate state table's pk (:569-570; group key 0 in test_utils/agg_executor.rs:157-171);
  * flush_data (:412-514) emits the barrier's delta and then calls update_watermark on every state table (:503-507),
    which drops the range below the watermark when the epoch commits: after that barrier no group whose window key is
    non-NULL and below the watermark is held, nor its materialized-input rows.  NULL is never below a watermark (the
    memcomparable encoding sorts NULL last).
The device rules beyond the reference (rwgpu.h): one pending watermark, a lower value for the same key ignored, another
key position replacing it; a late row of a cleaned group is the first row of a new group.
"""
import copy
import os
import subprocess

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import AggCall, HashAggExecutor, MockSource

import test_agg_types as TA
import test_join_types as TJ
from test_agg_types import Call, Spec, assert_same, chunk_rows, make_chunk
from test_state_types import StateModel, device_state, state_multisets, agg_restore_chunks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INS, DEL, UD, UI = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT
# the key types watermarks clean on (test_agg_types knows the others already)
TA.T_OF.update({"time": abi.T_TIME, "timestamptz": abi.T_TIMESTAMPTZ, "serial": abi.T_SERIAL})
KEY_TYPES = ["int2", "int4", "int8", "date", "time", "timestamp", "timestamptz", "serial"]


class WmModel(StateModel):
    """StateModel plus the state table's range delete below a watermark"""

    def clean(self, key_pos, v):
        for key in list(self.groups):
            if key[key_pos] is not None and key[key_pos] < v:
                del self.groups[key]


# ============================================================================ streams
def key_pool(t):
    lo, hi = TJ.int_edges(t)[0], TJ.int_edges(t)[-1]
    return sorted(set(TJ.int_edges(t) + [lo + 2, hi - 1] + list(range(100, 112))))


def plan(kt, multi, append_only=False):
    """single key: the fast path's shape where the type allows it; multi: (window key, int2 key) with NULLs in both"""
    if multi:
        return Spec([kt, "int2", "int8", "int4"], [0, 1], [Call("count"), Call("sum", 2, "int8", "int8"), Call("min", 3, "int4"),
                                                           Call("max", 2, "int8")], append_only)
    return Spec([kt, "int8", "int4"], [0], [Call("count"), Call("sum", 1, "int8", "int8"), Call("max", 2, "int4"),
                                            Call("min", 1, "int8")], append_only)


class Stream:
    """inserts, deletes and U-/U+ pairs of live rows; window keys drawn at or above a floor (the watermark) or NULL"""

    def __init__(self, spec, kt, seed, key_pos=0):
        self.spec, self.kt, self.key_pos = spec, kt, key_pos
        self.rng = np.random.default_rng(seed)
        self.pool = key_pool(kt)
        self.live = []

    def new_row(self, floor):
        r = self.rng
        row = []
        for k, t in enumerate(self.spec.types):
            if k in self.spec.keys:
                if r.random() < 0.1:
                    row.append(None)
                elif self.spec.keys.index(k) == self.key_pos:
                    pool = [v for v in self.pool if floor is None or v >= floor]
                    row.append(pool[int(r.integers(len(pool)))])
                else:
                    row.append(int(r.integers(0, 5)))
            else:
                row.append(None if r.random() < 0.1 else int(r.integers(-50, 50)))
        return tuple(row)

    def epoch(self, floor=None, pushes=2, rows=40):
        out = []
        for _ in range(pushes):
            p = []
            for _ in range(rows):
                x = self.rng.random()
                if self.live and x < 0.25 and not self.spec.append_only:
                    p.append((DEL, self.live.pop(int(self.rng.integers(len(self.live)))), True))
                elif self.live and x < 0.35 and not self.spec.append_only:
                    old = self.live.pop(int(self.rng.integers(len(self.live))))
                    new = self.new_row(floor)
                    p += [(UD, old, True), (UI, new, True)]
                    self.live.append(new)
                else:
                    new = self.new_row(floor)
                    p.append((INS, new, True))
                    self.live.append(new)
            out.append(p)
        return out

    def clean(self, v):
        kc = self.spec.keys[self.key_pos]
        self.live = [r for r in self.live if r[kc] is None or r[kc] >= v]


def scenario(spec, kt, seed, wm, key_pos=0):
    """-> epochs [(pushes, watermark or None)]: three free epochs, the watermark in the fourth, three that respect it"""
    s = Stream(spec, kt, seed, key_pos)
    eps = [(s.epoch(), None) for _ in range(3)]
    eps.append((s.epoch(), (key_pos, wm)))
    s.clean(wm)
    eps += [(s.epoch(floor=wm), None) for _ in range(3)]
    return eps


def run_model(spec, eps, m=None):
    """-> (model, per-epoch outputs, state after every epoch)"""
    m = m or WmModel(spec.calls, spec.keys, spec.append_only, "barrier")
    res, states = [], []
    for pushes, wm in eps:
        for p in pushes:
            m.push(p)
        res.append(("ok", m.flush()))
        if wm is not None:
            m.clean(*wm)
        states.append(copy.deepcopy(m.snapshot()))
    return m, res, states


# ============================================================================ CPU: the restatement and the mirror
def test_restatement_clean_is_strict_keeps_nulls_and_minput():
    spec = plan("int4", True)
    m = WmModel(spec.calls, spec.keys, False, "barrier")
    m.push([(INS, (k, 1, 5, 7), True) for k in (4, 5, 6, None)])
    m.flush()
    m.clean(0, 5)
    states, minput = m.snapshot()
    assert sorted((r[0] is None, r[0] or 0) for r in states) == [(False, 5), (False, 6), (True, 0)]
    assert all(r[0] != 4 for r in minput) and len(minput) == 6  # (min and max: one row each per group)


def agg_mirror(be, keys, window=0, types=(abi.T_INT64,) * 4):
    tx, src = MockSource.channel()
    ex = HashAggExecutor(be, src.into_executor(list(types), []), False, [AggCall.from_pretty("(count:int8)")], 0, keys,
                         window_col_idx_in_group_key=window)
    return tx, ex, ex.execute()


def kinds(msgs):
    return ["chunk" if m.chunk is not None else ("wm", m.watermark.col_idx, m.watermark.val) if m.watermark else "barrier"
            for m in msgs]


def test_mirror_watermark_derivation(oracle):
    """keys [2, 0]: a watermark on column 1 (not a key) is dropped; column 0 is seq 1, column 2 seq 0; the later one per
    seq wins; at the barrier: chunks, then the watermarks in seq order, then the barrier; nothing is buffered after"""
    from risingwave_b200.stream_chunk import StreamChunk
    tx, ex, st = agg_mirror(oracle, [2, 0])
    tx.push_barrier(1)
    assert kinds(st.drain_until_pending()) == ["barrier"]
    tx.push_chunk(StreamChunk.from_pretty(" I I I I\n + 1 2 3 4\n + 1 5 3 4"))
    tx.push_watermark(1, abi.T_INT64, 100)
    tx.push_watermark(0, abi.T_INT64, 7)
    tx.push_watermark(2, abi.T_INT64, 3)
    tx.push_watermark(0, abi.T_INT64, 9)
    assert st.drain_until_pending() == []
    tx.push_barrier(2)
    assert kinds(st.drain_until_pending()) == ["chunk", ("wm", 0, 3), ("wm", 1, 9), "barrier"]
    tx.push_barrier(3)
    assert kinds(st.drain_until_pending()) == ["barrier"]


@pytest.mark.parametrize("window", [0, 1])
def test_mirror_multi_key_window_column(oracle, window):
    """three group keys [3, 1, 0]: only the window key (seq `window`) would clean -- on the oracle backend nothing is
    called (it has no rwgpu_agg_update_watermark) and every watermark on a group key is still forwarded"""
    from risingwave_b200.stream_chunk import StreamChunk
    tx, ex, st = agg_mirror(oracle, [3, 1, 0], window)
    calls = []
    ex.update_watermark = lambda kp, v: calls.append((kp, v))
    assert ex._window_col == [3, 1, 0][window]
    tx.push_barrier(1)
    tx.push_chunk(StreamChunk.from_pretty(" I I I I\n + 1 2 3 4"))
    tx.push_watermark(1, abi.T_INT64, 11)
    tx.push_watermark(2, abi.T_INT64, 12)
    tx.push_watermark(3, abi.T_INT64, 13)
    tx.push_barrier(2)
    assert kinds(st.drain_until_pending()) == ["barrier", "chunk", ("wm", 0, 13), ("wm", 1, 11), "barrier"]
    assert calls == []


# ============================================================================ GPU
def dev_chunk(spec, p, counted):
    """-> (DeviceChunk, device address of its row count or None); a counted push's chunk has 5 rows of capacity beyond"""
    import torch
    ch = make_chunk(spec.types, p)
    if not counted:
        return TA.device_chunk(ch, False), None, None
    n = torch.tensor([ch.capacity()], dtype=torch.int64, device="cuda")
    return TJ.device_chunk(ch, pad=5), n.data_ptr(), n


def play(spec, cuda, eps, path, hint=0, snapshots=None):
    """through `path`: "host" (rwgpu_agg_push / flush), "device" (push_device / flush_device), "counted" (counted pushes,
    flush_device), "async" (flush_device_async with two barriers outstanding).  `snapshots`: list to receive the
    state after every epoch (sync paths)."""
    import torch
    from risingwave_b200 import device
    ex = spec.executor(cuda, hint)
    res = []
    if path == "host":
        for e, (pushes, wm) in enumerate(eps):
            for p in pushes:
                ex.apply_chunk(make_chunk(spec.types, p))
            if wm is not None:
                ex.update_watermark(*wm)
            res.append(("ok", chunk_rows(ex.flush_data(e + 1), spec.out_types)))
            if snapshots is not None:
                snapshots.append(device_state(spec, ex))
        return ex, res
    st = torch.cuda.Stream()
    keep = []
    with torch.cuda.stream(st):
        for e, (pushes, wm) in enumerate(eps):
            for p in pushes:
                ch, n_dev, n_t = dev_chunk(spec, p, path == "counted")
                keep.append((ch, n_t))
                device.agg_push_device(ex, ch, st, n_rows_dev=n_dev)
            if wm is not None:
                ex.update_watermark(*wm)
            if path == "async":
                device.agg_flush_device_async(ex, e + 1, st)
                if e >= 1:
                    res.append(("ok", TA.view_rows(device.agg_flush_collect(ex, st), spec.out_types)))
            else:
                res.append(("ok", TA.view_rows(device.agg_flush_device(ex, e + 1, st), spec.out_types)))
                if snapshots is not None:
                    snapshots.append(device_state(spec, ex))
        if path == "async":
            res.append(("ok", TA.view_rows(device.agg_flush_collect(ex, st), spec.out_types)))
    st.synchronize()
    return ex, res


def same_state(spec, got, want, what):
    g, w = state_multisets(spec, *got), state_multisets(spec, *want)
    assert g[0] == w[0], f"{what} states: only got {g[0] - w[0]}\n only want {w[0] - g[0]}"
    assert g[1] == w[1], f"{what} minput: only got {g[1] - w[1]}\n only want {w[1] - g[1]}"


def wm_values(kt, seed):
    pool = key_pool(kt)
    k = pool[len(pool) // 2 + seed % 3]
    lo, hi = pool[0], pool[-1]
    return [k - 1, k, k + 1, lo, lo + 1, hi]


@pytest.mark.gpu
@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
@pytest.mark.parametrize("kt", KEY_TYPES)
def test_device_cleaning_at_every_type(cuda, oracle, kt, multi):
    """the cleaning barrier emits the restatement's delta (the one it emits without a watermark), the snapshot after it
    is the restatement's cleaned state (minput included), and the epochs after it equal the restatement and the oracle
    (which never cleans); on every barrier entry point"""
    for key_pos in ((0, 1) if multi else (0,)):
        wt = kt if key_pos == 0 else "int2"  # (the multi-key plan's second key is an int2 column)
        for seed, wm in enumerate(wm_values(wt, key_pos)):
            spec = plan(kt, multi, append_only=(seed == 5 and not multi))
            eps = scenario(spec, wt, 10 * seed + key_pos, wm, key_pos)
            _, want, want_states = run_model(spec, eps)
            plain = [(p, None) for p, _ in eps]
            _, want_plain, _ = run_model(spec, plain)
            assert want[3] == want_plain[3], "the watermark does not change the barrier that applies it"
            loose = spec.loose_cols(True)
            what = f"{kt} {'multi' if multi else 'single'} key {key_pos} wm {wm}"
            assert_same(spec, TA.play_host(spec, oracle, [p for p, _ in eps]), want, loose, what + " oracle")
            for path in ("host", "device", "counted", "async"):
                snaps = [] if path != "async" else None
                ex, got = play(spec, cuda, eps, path, snapshots=snaps)
                assert_same(spec, got, want, loose, f"{what} {path}")
                if snaps is not None:
                    for e in (3, 6):
                        same_state(spec, snaps[e], want_states[e], f"{what} {path} epoch {e}")
                else:
                    same_state(spec, device_state(spec, ex), want_states[-1], f"{what} {path} end")


@pytest.mark.gpu
def test_device_no_watermark_keeps_every_group(cuda):
    """without a watermark the barrier keeps what it kept before: every group with rows stays in the snapshot"""
    spec = plan("int8", False)
    eps = [(p, None) for p, _ in scenario(spec, "int8", 3, 105)]
    _, want, states = run_model(spec, eps)
    ex, got = play(spec, cuda, eps, "host")
    assert_same(spec, got, want, spec.loose_cols(True), "no watermark")
    same_state(spec, device_state(spec, ex), states[-1], "no watermark")


@pytest.mark.gpu
def test_device_growth_in_an_epoch_with_a_pending_watermark(cuda):
    """an operator created for 16 groups receives the watermark, then ~6000 new groups in the same epoch: the table grows
    while the watermark is pending, and the barrier still emits every + before the cleaning drops half of them"""
    spec = plan("int8", True)
    rng = np.random.default_rng(7)
    rows = [(INS, (int(k), int(rng.integers(-3, 3)), int(k), 1), True) for k in rng.permutation(6000)]
    eps = [([[(INS, (1, 1, 1, 1), True)]], None), ([rows[:3000], rows[3000:]], (0, 3000)),
           ([[(INS, (k, 0, 1, 2), True) for k in range(3000, 3100)]], None)]
    _, want, states = run_model(spec, eps)
    for path in ("host", "async"):
        snaps = [] if path == "host" else None
        ex, got = play(spec, cuda, eps, path, hint=16, snapshots=snaps)
        assert_same(spec, got, want, spec.loose_cols(True), path)
        if snaps:
            same_state(spec, snaps[1], states[1], "after the cleaning")
        same_state(spec, device_state(spec, ex), states[-1], path)


def stats(cuda, ex):
    import ctypes as C
    fn = cuda.lib.rwgpu_agg_stats
    fn.restype, fn.argtypes = C.c_int32, [C.c_void_p] + [C.POINTER(C.c_uint64)] * 3
    g, cap, n = C.c_uint64(), C.c_uint64(), C.c_uint64()
    cuda.check(fn(ex._h, C.byref(g), C.byref(cap), C.byref(n)))
    return g.value, cap.value


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "async"])
def test_device_pending_watermark_rules(cuda, path):
    """a lower value for the same key is ignored; another key position replaces the pending watermark; the one applied
    at a barrier is gone after it; NULL keys stay"""
    spec = plan("int4", True)
    base = [(INS, (a, b, 1, 1), True) for a in (1, 5, 9, None) for b in (1, 5, 9, None)]
    cases = [([(0, 6), (0, 2)], (0, 6)), ([(0, 6), (1, 4)], (1, 4)), ([(1, 4), (0, 2), (0, 8)], (0, 8)), ([(0, 2), (0, 9)], (0, 9))]
    for calls, eff in cases:
        m = WmModel(spec.calls, spec.keys, False, "barrier")
        m.push(base)
        m.flush()
        m.flush()
        m.clean(*eff)
        ex, _ = play(spec, cuda, [([base], None), ([], None)], "host")
        for kp, v in calls:
            ex.update_watermark(kp, v)
        if path == "host":
            assert chunk_rows(ex.flush_data(3), spec.out_types) == []
        else:
            from risingwave_b200 import device
            device.agg_flush_device_async(ex, 3, None)
            assert TA.view_rows(device.agg_flush_collect(ex, None), spec.out_types) == []
        same_state(spec, device_state(spec, ex), m.snapshot(), f"{calls}")
        assert stats(cuda, ex)[0] == len(m.snapshot()[0])
        ex.flush_data(4)  # (nothing pending any more)
        same_state(spec, device_state(spec, ex), m.snapshot(), f"{calls} next barrier")


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
def test_device_late_rows(cuda, strict, multi):
    """a row of a cleaned group is the first row of a new group: an insert emits + at the next barrier; a retraction makes
    the row count negative (RW_ERR_INCONSISTENT under strict consistency, else clamped: nothing is emitted); a retracted
    min / max value is missing from the new group's materialized input"""
    spec = plan("int8", multi)

    def mk():
        _, src = MockSource.channel()
        ex = HashAggExecutor(cuda, src.into_executor([TA.T_OF[t] for t in spec.types], []), False,
                             [AggCall.from_pretty(c.pretty()) for c in spec.calls], 0, spec.keys, strict_consistency=strict)
        ex.apply_chunk(make_chunk(spec.types, [(INS, r, True) for r in rows]))
        ex.flush_data(1)
        ex.update_watermark(0, 10)
        ex.flush_data(2)
        return ex

    rows = [(k, 1, 3, 4) if multi else (k, 3, 4) for k in (5, 6, 20)]
    late = rows[0]
    nk = len(spec.keys)
    ex = mk()
    ex.apply_chunk(make_chunk(spec.types, [(INS, late, True)]))
    assert chunk_rows(ex.flush_data(3), spec.out_types) == [(INS, late[:nk] + (1, 3, 4, 3))]  # count, sum, max / min, min / max
    ex = mk()
    ex.apply_chunk(make_chunk(spec.types, [(DEL, late, True)]))
    if strict:
        with pytest.raises(abi.RwError) as e:
            ex.flush_data(3)
        assert e.value.code == abi.RW_ERR_INCONSISTENT
    else:
        assert chunk_rows(ex.flush_data(3), spec.out_types) == []
        ex.apply_chunk(make_chunk(spec.types, [(INS, late, True)]))
        assert len(chunk_rows(ex.flush_data(4), spec.out_types)) == 1
    assert device_state(spec, mk())[0] == [rows[2][:nk] + (1, 3, 4, 3)]


@pytest.mark.gpu
def test_device_refusals(cuda):
    import ctypes as C
    fn = cuda.lib.rwgpu_agg_update_watermark
    fn.restype, fn.argtypes = C.c_int32, [C.c_void_p, C.c_int32, C.c_int64]
    assert fn(None, 0, 0) == abi.RW_ERR_INVALID
    for types, row, keys, code in ((["float8", "int8"], (np.float64(1.0), 2), [0], abi.RW_ERR_UNSUPPORTED),
                                   (["float4", "int8"], (np.float32(1.0), 2), [0], abi.RW_ERR_UNSUPPORTED),
                                   (["boolean", "int8"], (1, 2), [0], abi.RW_ERR_UNSUPPORTED),
                                   (["int8", "float8"], (1, np.float64(2.0)), [0, 1], None)):
        spec = Spec(types, keys, [Call("count")], False)
        ex = spec.executor(cuda)
        ex.apply_chunk(make_chunk(types, [(INS, row, True)]))
        ex.flush_data(1)
        for kp in (-1, len(keys)):
            assert fn(ex._h, kp, 0) == abi.RW_ERR_INVALID
        if code is not None:
            assert fn(ex._h, 0, 10) == code
        else:
            assert fn(ex._h, 1, 10) == abi.RW_ERR_UNSUPPORTED and fn(ex._h, 0, 10) == abi.RW_OK
        ex.flush_data(2)
        assert len(device_state(spec, ex)[0]) == (0 if code is None else 1)


@pytest.mark.gpu
def test_device_restore_keeps_a_pending_watermark(cuda):
    """a watermark set before a restore is applied at the next barrier, to the restored groups (minput included)"""
    spec = plan("date", True)
    eps = scenario(spec, "date", 11, 104)[:3]
    m, _, _ = run_model(spec, eps)
    states, minput = m.snapshot()
    ex = spec.executor(cuda)
    ex.update_watermark(0, 104)
    ex.restore(*agg_restore_chunks(spec, states, minput))
    assert chunk_rows(ex.flush_data(1), spec.out_types) == []
    m.clean(0, 104)
    same_state(spec, device_state(spec, ex), m.snapshot(), "restored then cleaned")
    assert len(m.snapshot()[0]) < len(states)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "async"])
def test_device_value_log_compaction(cuda, path):
    """retractable min / max: windows of many values, most of them retracted, windows cleaned.  After every cleaning
    barrier the value log holds <= 2 x live records + 4096; it is rebuilt along the way; retractions of values that
    survived a rebuild still find them, and the outputs equal the restatement's"""
    spec = Spec(["int8", "int4", "int8"], [0, 1], [Call("count"), Call("min", 2, "int8"), Call("max", 2, "int8")], False)
    rng = np.random.default_rng(3)
    live, eps = [], []
    for e in range(14):
        p = [(INS, (e, int(g), int(rng.integers(-1000, 1000))), True) for g in range(40) for _ in range(60)]
        gone = rng.random(len(live)) < 0.6
        dels = [r for r, x in zip(live, gone) if x]
        live = [r for r, x in zip(live, gone) if not x] + [r for _, r, _ in p]
        eps.append(([p, [(DEL, r, True) for r in dels]], (0, e - 2) if e >= 2 else None))
        live = [r for r in live if r[0] >= e - 2]
    _, want, _ = run_model(spec, eps)
    ex = spec.executor(cuda)
    m = WmModel(spec.calls, spec.keys, False, "barrier")
    from risingwave_b200 import device
    got = []
    for e, (pushes, wm) in enumerate(eps):
        for p in pushes:
            ex.apply_chunk(make_chunk(spec.types, p))
            m.push(p)
        if wm is not None:
            ex.update_watermark(*wm)
        if path == "host":
            got.append(("ok", chunk_rows(ex.flush_data(e + 1), spec.out_types)))
        else:
            device.agg_flush_device_async(ex, e + 1, None)
            got.append(("ok", TA.view_rows(device.agg_flush_collect(ex, None), spec.out_types)))
        m.flush()
        if wm is not None:
            m.clean(*wm)
            n_live = sum(len(g["mi"][c]) for g in m.groups.values() for c in (1, 2))
            used, _ = ex.value_log_stats()
            assert used <= 2 * n_live + 4096, f"epoch {e}: {used} records in use for {n_live} live"
    assert_same(spec, got, want, spec.loose_cols(True), path)
    assert ex.value_log_stats()[1] >= 2
    same_state(spec, device_state(spec, ex), m.snapshot(), "after the rebuilds")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "async"])
def test_device_sliding_window_state_is_bounded(cuda, path):
    """Project(tumble) -> HashAgg by (window, auction) shape: 60 epochs, each in a new window, the watermark two windows
    back.  The group count and the capacity stop growing (the operator's own bound sees the count after cleaning)"""
    from risingwave_b200 import device
    spec = Spec(["timestamp", "int8", "int8"], [0, 1], [Call("count"), Call("max", 2, "int8")], True)
    ex = spec.executor(cuda, 16)
    rng = np.random.default_rng(1)
    seen = []
    for e in range(60):
        w = e * 10_000_000
        rows = [(INS, (w, int(a), int(rng.integers(0, 10**6))), True) for a in rng.integers(0, 3000, 4000)]
        ex.apply_chunk(make_chunk(spec.types, rows))
        ex.update_watermark(0, w - 20_000_000)
        if path == "host":
            ex.flush_data(e + 1)
        else:
            device.agg_flush_device_async(ex, e + 1, None)
            device.agg_flush_collect(ex, None)
        seen.append(stats(cuda, ex))
    assert max(g for g, _ in seen[10:]) <= 3 * 3000
    assert seen[-1][1] == seen[15][1], f"capacity grew: {[c for _, c in seen]}"


@pytest.mark.gpu
def test_device_mirror_cleans_on_the_window_column(cuda):
    """the Python mirror, end to end: keys [2, 0] with the window at seq 1 (column 0); a watermark on column 0 cleans"""
    from risingwave_b200.stream_chunk import StreamChunk
    tx, ex, st = agg_mirror(cuda, [2, 0], window=1)
    tx.push_barrier(1)
    tx.push_chunk(StreamChunk.from_pretty(" I I I I\n + 1 0 7 0\n + 5 0 7 0\n + 9 0 7 0"))
    tx.push_barrier(2)
    tx.push_watermark(0, abi.T_INT64, 5)
    tx.push_watermark(2, abi.T_INT64, 100)  # (seq 0: forwarded, cleans nothing)
    tx.push_barrier(3)
    assert kinds(st.drain_until_pending()) == ["barrier", "chunk", "barrier", ("wm", 0, 100), ("wm", 1, 5), "barrier"]
    g, _ = stats(cuda, ex)
    assert g == 2


@pytest.mark.gpu
def test_cpp_mirror_watermark_kat():
    exe = os.path.join(ROOT, "build", "test_agg_watermarks")
    assert os.path.exists(exe), "run __graft_entry__.build() first"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "agg watermarks: ok" in r.stdout, r.stdout + r.stderr


def test_cpp_mirror_watermark_kat_compiles():
    src = os.path.join(ROOT, "tests", "cpp", "test_agg_watermarks.cc")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
