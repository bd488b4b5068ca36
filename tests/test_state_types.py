"""The operator state lifecycle at every type: HashAgg snapshot / restore (with the materialized input of retractable
min / max), HashJoin snapshot / restore, and join-key watermark cleaning with the unified-table compaction it feeds --
the device against the typed restatements of test_agg_types.py and test_join_types.py, extended here.

HashAgg (src/stream/src/executor/aggregate/agg_group.rs):
  * a snapshot is what the reference persists: one intermediate-state row per group whose row count is > 0, the group
    key and each call's state datum (AggGroup::build_states_change, :473-538; a group whose row count is 0 is deleted
    from the table), and per retractable min / max call one row per live non-NULL input (minput.rs:172-245; the
    MaterializedInputState table).  rwgpu.h fixes the minput row as group key | int4 call index | int8 value, a float
    argument's value being the IEEE bits of the f64;
  * a restored group's state is the loaded row, its previous outputs are the outputs of that row (AggGroup::create,
    :260-316): a barrier right after a restore emits nothing;
  * the device rule for split restores (rwgpu.h): a minput row must name a retractable call of a group whose state row
    was restored in the same call or an earlier one; anything else is RW_ERR_INVALID.
Comparison: bit-exact, except what test_agg_types.py allows (a float sum's NaN bits; a float min / max by OrderedFloat
class on the device) and a float argument's minput value, which compares by class: the device keeps the input in its
sortable encoding, which folds -0 into +0 and every NaN into one.

HashJoin (src/stream/src/executor/join/hash_join.rs, hash_join.rs):
  * the state of a side is its live input rows (JoinHashMap::insert, join/hash_join.rs:591-625); a row whose key has a
    NULL in a column that is not null-safe never matches and the device does not keep it; in an append-only plan with
    pk in the join key a matched row leaves the state (append_only_optimize), so the state is the unmatched rows;
  * a restore replays rows as inserts with the output discarded, in chunk order.  Two live rows of one key with an
    equal pk come only from an inconsistent stream (the reference's state table is keyed by join key | pk and cannot
    hold both); of two such rows in one restore chunk a later delete removes the later one on the unified and fused
    paths and the earlier one on the generic path (DESIGN §9);
  * watermark cleaning (JoinHashMap::update_watermark, join/hash_join.rs:521-527, called from handle_watermark,
    hash_join.rs:791-842): the state table's `update_watermark` takes effect when the epoch commits, so at the first
    barrier after `update_watermark(side, key_pos, v)` every live row of that side whose key column `key_pos` is
    non-NULL and below v in the column type's signed order leaves the state.  NULL is never below a watermark: the
    memcomparable encoding sorts NULL last (src/common/src/util/memcmp_encoding.rs, `encode_value` writes 0 for
    Some and 1 for None with the default ascending nulls-last order).  A lower value while one is pending is ignored;
    another key_pos replaces the pending one (join.cu);
  * late rows (below a watermark after cleaning): the reference leaves their result open (its cache is not cleared,
    `// TODO: remove data in cache`).  The project's rule (rwgpu.h): a late insert is an ordinary insert and matches
    nothing of the cleaned side; a late delete of a cleaned row finds no stored row, which is RW_ERR_INCONSISTENT with
    strict_consistency and is otherwise ignored (the row still probes the other side, as any delete does).
"""
import copy
from collections import Counter

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource, Watermark
from risingwave_b200.stream_chunk import Column, StreamChunk, concat_chunks

import test_agg_types as TA
import test_join_types as TJ
from test_agg_types import Call, Spec, assert_same, chunk_rows, make_chunk
from test_agg_types import Model as AggModel
from test_join_types import PATHS, PLANS, Plan, drive, stream
from test_join_types import Model as JoinModel

INS, DEL, UD, UI = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT
I64MIN, I64MAX = -(1 << 63), (1 << 63) - 1


# ============================================================================ HashAgg: the restatement's state
def f64_bits(v):
    """a float datum as the signed int8 of its f64 bits (rwgpu.h: the minput value of a float argument)"""
    return int(np.array([float(v)], dtype=np.float64).view(np.int64)[0])


def from_f64_bits(at, b):
    return TA.FLOAT_NP[at](np.array([b], dtype=np.int64).view(np.float64)[0])


class StateModel(AggModel):
    """AggModel plus the state rows of agg_group.rs / minput.rs"""

    def snapshot(self):
        states, minput = [], []
        for key, g in self.groups.items():
            if g["states"][0] <= 0:  # (row count 0: no intermediate-state row, and no live input)
                continue
            states.append(key + tuple(g["states"]))
            for c, call in enumerate(self.calls):
                if self.minput(c):
                    for v in g["mi"][c]:
                        minput.append(key + (c, f64_bits(v) if call.is_float() else int(v)))
        return states, minput

    def load(self, states, minput):
        """AggGroup::create over the loaded rows: prev outputs = the loaded states; not dirty"""
        nk = len(self.keys)
        for row in states:
            key = tuple(row[:nk])
            self.groups[key] = {"states": list(row[nk:]), "prev": list(row[nk:]), "mi": [[] for _ in self.calls]}
        for row in minput:
            key, c, v = tuple(row[:nk]), row[nk], row[nk + 1]
            call = self.calls[c]
            self.groups[key]["mi"][c].append(from_f64_bits(call.at, v) if call.is_float() else v)


def minput_types(spec):
    return [spec.types[k] for k in spec.keys] + ["int4", "int8"]


def run_model(spec, epochs, m=None):
    """-> (model, per-epoch outputs); the streams here never fail"""
    m = m or StateModel(spec.calls, spec.keys, spec.append_only, "barrier")
    res = []
    for pushes in epochs:
        for p in pushes:
            m.push(p)
        res.append(("ok", m.flush()))
    return m, res


def state_multisets(spec, states, minput):
    """(state rows, minput rows) -> comparable multisets: see the module docstring"""
    sm = spec.multiset([(INS, r) for r in states], spec.loose_cols(True))
    mm = Counter()
    nk = len(spec.keys)
    for row in minput:
        key = tuple(TA.canon(v, t, "bits") for v, t in zip(row[:nk], spec.types))
        c, v = row[nk], row[nk + 1]
        if spec.calls[c].is_float():
            v = TA.canon(np.float64(from_f64_bits("float8", v)), "float8", "class")
        mm[key + (c, v)] += 1
    return sm, mm


def device_state(spec, ex):
    st, mi = ex.snapshot()
    assert all((ch.ops == INS).all() for ch in st + mi)
    return ([r for _, r in chunk_rows(st, spec.out_types)], [r for _, r in chunk_rows(mi, minput_types(spec))])


def agg_restore_chunks(spec, states, minput):
    return (make_chunk(spec.out_types, [(INS, r, True) for r in states]),
            make_chunk(minput_types(spec), [(INS, r, True) for r in minput]))


# the call signatures check_signatures accepts, each at its own type (test_agg_types.check_signatures)
INT_TYPES = ["int8", "int2", "int4", "int8", "int8", "date", "timestamp"]  # key | int2 | int4 | small int8 | int8 edges | date | ts


def int_state_spec(append_only):
    calls = [Call("count"), Call("count", 1, "int2"), Call("sum", 1, "int2"), Call("sum", 2, "int4"), Call("sum", 3, "int8", "int8"),
             Call("sum0", 3, "int8"), Call("sum", 4, "int8", "decimal"), Call("min", 1, "int2"), Call("max", 1, "int2"),
             Call("min", 2, "int4"), Call("max", 2, "int4"), Call("min", 4, "int8"), Call("max", 4, "int8"), Call("min", 5, "date"),
             Call("max", 6, "timestamp")]
    return Spec(INT_TYPES, [0], calls, append_only)


def int_state_values():
    date_edges = [-(1 << 31), -(1 << 31) + 1, -1, 0, 1, (1 << 31) - 1]
    return [None, [*TA.edges("int2"), None], [*TA.edges("int4"), None], [-3, -1, 0, 2, 5, None], [*TA.edges("int8"), None],
            [*date_edges, None], [*TA.edges("int8"), None]]


FLOAT_TYPES = ["int8", "float4", "float8", "float4", "float8"]  # key | exact f4 | exact f8 | f4 edges | f8 edges


def float_state_spec(append_only):
    calls = [Call("count"), Call("count", 3, "float4"), Call("sum", 1, "float4"), Call("sum", 2, "float8"), Call("min", 3, "float4"),
             Call("max", 3, "float4"), Call("min", 4, "float8"), Call("max", 4, "float8")]
    return Spec(FLOAT_TYPES, [0], calls, append_only)


def float_state_values():
    """sums over quarters: exact in any order (the device's float sums inside one launch are unordered)"""
    q4 = [np.float32(x / 4) for x in (-7, -1, 0, 1, 3, 9)] + [None]
    q8 = [np.float64(x / 4) for x in (-7, -1, 0, 1, 3, 9)] + [None]
    return [None, q4, q8, TA.float_edges("float4") + [None], TA.float_edges("float8") + [None]]


def multikey_state_spec():
    calls = [Call("count"), Call("sum", 2, "int4"), Call("min", 2, "int4"), Call("max", 3, "float8"), Call("count", 3, "float8")]
    return Spec(["int2", "int4", "int4", "float8"], [0, 1], calls, False)


SINGLE_KEYS = (None, I64MIN, I64MIN + 1, -1, 0, 5, I64MAX) + tuple(range(100, 124))
MULTI_KEYS = (-32768, -1, 0, 7, 32767, None) + tuple(range(100, 106))


def agg_case(name):
    """-> (spec, epochs): 8 epochs, every third mostly retracting (groups empty out and come back)"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("int"):
        spec = int_state_spec(name.endswith("ao"))
        vals, keys = int_state_values(), SINGLE_KEYS
    elif name.startswith("float"):
        spec = float_state_spec(name.endswith("ao"))
        vals, keys = float_state_values(), SINGLE_KEYS
    else:
        spec = multikey_state_spec()
        vals, keys = [None, None, [*TA.edges("int4"), None], TA.float_edges("float8") + [None]], MULTI_KEYS
    epochs = TA.random_epochs(rng, spec, vals, n_epochs=8, pushes=2, rows=50, key_values=keys)
    if not spec.append_only:  # two groups of their own that empty out in epoch 5 and stay empty
        extra = [tuple((1000 + g) if k in spec.keys else vals[k][0] for k in range(len(spec.types))) for g in (0, 1)]
        epochs[0].append([(INS, r, True) for r in extra])
        epochs[4].append([(DEL, r, True) for r in extra])
    return spec, epochs


AGG_CASES = ["int_ao", "int_retract", "float_ao", "float_retract", "multikey"]


# ---------------------------------------------------------------------------- CPU: the restatement itself
def test_restatement_agg_snapshot_restore_round_trip():
    """the model restored from its own snapshot emits what the uninterrupted model emits; emptied groups are absent"""
    for name in AGG_CASES:
        spec, epochs = agg_case(name)
        for cut in (3, 5, 6):
            m, _ = run_model(spec, epochs[:cut])
            states, minput = m.snapshot()
            assert all(r[len(spec.keys)] > 0 for r in states)
            assert spec.append_only or cut < 5 or len(states) <= len(m.groups) - 2, f"{name}: emptied groups are in the snapshot"
            _, want = run_model(spec, epochs[cut:], m)
            r = StateModel(spec.calls, spec.keys, spec.append_only, "barrier")
            r.load(states, minput)
            assert r.flush() == []
            _, got = run_model(spec, epochs[cut:], r)
            assert_same(spec, got, want, spec.loose_cols(False), f"model {name} cut {cut}")


def test_restatement_minput_value_encoding():
    assert from_f64_bits("float4", f64_bits(np.float32(-1.5))) == np.float32(-1.5)
    assert f64_bits(np.float64(-0.0)) == I64MIN and f64_bits(np.float32(1.0)) == 0x3FF0000000000000


# ---------------------------------------------------------------------------- GPU: snapshot
def agg_run(spec, cuda, epochs, hint=0):
    ex = spec.executor(cuda, hint)
    for e, pushes in enumerate(epochs):
        for p in pushes:
            ex.apply_chunk(make_chunk(spec.types, p))
        ex.flush_data(e + 1)
    return ex


@pytest.mark.gpu
@pytest.mark.parametrize("name", AGG_CASES)
def test_device_agg_snapshot_is_the_state_rows(cuda, name):
    spec, epochs = agg_case(name)
    for cut in (5, 6):  # (after epoch 6 -- a draining one -- many groups have emptied out)
        m, _ = run_model(spec, epochs[:cut])
        ex = agg_run(spec, cuda, epochs[:cut])
        got, want = state_multisets(spec, *device_state(spec, ex)), state_multisets(spec, *m.snapshot())
        assert got[0] == want[0], f"{name} cut {cut} states: only got {got[0] - want[0]}\n only want {want[0] - got[0]}"
        assert got[1] == want[1], f"{name} cut {cut} minput: only got {got[1] - want[1]}\n only want {want[1] - got[1]}"
        if spec.append_only or not any(m.minput(c) for c in range(len(spec.calls))):
            assert not want[1]


@pytest.mark.gpu
def test_device_agg_snapshot_of_an_empty_operator(cuda):
    for spec in (int_state_spec(False), multikey_state_spec()):
        ex = spec.executor(cuda)
        assert device_state(spec, ex) == ([], [])
        ex.flush_data(1)
        assert device_state(spec, ex) == ([], [])


# ---------------------------------------------------------------------------- GPU: restore
def play_restored(spec, cuda, calls, epochs, path, hint=0):
    """restore through `calls` [(states rows, minput rows)], then a barrier (must emit nothing), then `epochs` through
    the host push, the device push, or the device push with the async flush / collect pair"""
    import torch
    from risingwave_b200 import device
    ex = spec.executor(cuda, hint)
    for states, minput in calls:
        ex.restore(*agg_restore_chunks(spec, states, minput))
    assert chunk_rows(ex.flush_data(1), spec.out_types) == [], "a barrier right after a restore emits nothing"
    res = []
    if path == "host":
        for e, pushes in enumerate(epochs):
            for p in pushes:
                ex.apply_chunk(make_chunk(spec.types, p))
            res.append(("ok", chunk_rows(ex.flush_data(e + 2), spec.out_types)))
        return res
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for e, pushes in enumerate(epochs):
            for p in pushes:
                device.agg_push_device(ex, TA.device_chunk(make_chunk(spec.types, p), False), st)
            if path == "async":
                device.agg_flush_device_async(ex, e + 2, st)
                view = device.agg_flush_collect(ex, st)
            else:
                view = device.agg_flush_device(ex, e + 2, st)
            res.append(("ok", TA.view_rows(view, spec.out_types)))
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("name", AGG_CASES)
def test_device_agg_restore_round_trip(cuda, name):
    """snapshot -> restore into a fresh operator -> the rest of the stream equals the uninterrupted restatement, on
    every path; restored from the device's snapshot and, independently, from the restatement's own state rows"""
    spec, epochs = agg_case(name)
    cut = 4
    m, _ = run_model(spec, epochs[:cut])
    model_rows = m.snapshot()
    _, want = run_model(spec, epochs[cut:], copy.deepcopy(m))
    dev_rows = device_state(spec, agg_run(spec, cuda, epochs[:cut]))
    loose = spec.loose_cols(True)
    for src, rows in (("device snapshot", dev_rows), ("restatement", model_rows)):
        for path in ("host", "device", "async"):
            got = play_restored(spec, cuda, [rows], epochs[cut:], path)
            assert_same(spec, got, want, loose, f"{name} from the {src}, {path}")


@pytest.mark.gpu
def test_device_agg_restore_split_over_calls_and_growth(cuda):
    """the restatement's rows in three restore calls (minput in the call of its states and in later calls), and a
    restore of ~3000 groups into an operator created for 16: the table grows during the restore"""
    for name in ("int_retract", "float_retract", "multikey"):
        spec, epochs = agg_case(name)
        m, _ = run_model(spec, epochs[:4])
        states, minput = m.snapshot()
        _, want = run_model(spec, epochs[4:], copy.deepcopy(m))
        nk = len(spec.keys)
        half = len(states) // 2
        first = {tuple(r[:nk]) for r in states[:half]}
        mi_a = [r for r in minput if tuple(r[:nk]) in first]
        mi_b = [r for r in minput if tuple(r[:nk]) not in first]
        calls = [(states[:half], mi_a[: len(mi_a) // 2]), (states[half:], mi_a[len(mi_a) // 2:] + mi_b[: len(mi_b) // 2]),
                 ([], mi_b[len(mi_b) // 2:])]
        assert_same(spec, play_restored(spec, cuda, calls, epochs[4:], "host"), want, spec.loose_cols(True), f"{name} split")
    spec = int_state_spec(False)
    rng = np.random.default_rng(5)
    keys = tuple(range(-1500, 1500)) + SINGLE_KEYS
    epochs = TA.random_epochs(rng, spec, int_state_values(), n_epochs=5, pushes=3, rows=1500, key_values=keys)
    m, _ = run_model(spec, epochs[:2])
    rows = m.snapshot()
    assert len(rows[0]) > 2000
    _, want = run_model(spec, epochs[2:], copy.deepcopy(m))
    assert_same(spec, play_restored(spec, cuda, [rows], epochs[2:], "host", hint=16), want, spec.loose_cols(True), "growth")


@pytest.mark.gpu
def test_device_agg_restored_extreme_retracted(cuda):
    """retracting a restored max / min makes the barrier recompute it from the restored materialized input
    (minput.rs:184-245), for int2, date, timestamp and float8 arguments"""
    spec = Spec(["int8", "int2", "date", "timestamp", "float8"], [0],
                [Call("count"), Call("max", 1, "int2"), Call("min", 2, "date"), Call("max", 3, "timestamp"), Call("min", 4, "float8")], False)
    f = np.float64
    rows = [(1, -32768, -(1 << 31), I64MIN, f(-np.inf)), (1, 5, 3, 0, f(-0.0)), (1, 32767, 9, I64MAX, f(2.5)), (None, 1, 1, 1, f(1.0))]
    m, _ = run_model(spec, [[[(INS, r, True) for r in rows]]])
    states, minput = m.snapshot()
    epochs = [[[(DEL, rows[2], True)]], [[(DEL, rows[0], True), (DEL, rows[3], True)]], [[(DEL, rows[1], True)]]]
    _, want = run_model(spec, epochs, copy.deepcopy(m))
    assert want[0][1] and want[1][1] and want[2][1]
    for path in ("host", "device"):
        assert_same(spec, play_restored(spec, cuda, [(states, minput)], epochs, path), want, spec.loose_cols(True), path)


@pytest.mark.gpu
def test_device_agg_restore_refusals(cuda):
    from risingwave_b200 import device
    spec = int_state_spec(False)
    m, _ = run_model(spec, agg_case("int_retract")[1][:3])
    states, minput = m.snapshot()
    nk = len(spec.keys)

    def refused(ex, st, mi, code=abi.RW_ERR_INVALID):
        with pytest.raises(abi.RwError) as e:
            ex.restore(st, mi)
        assert e.value.code == code

    good_st, good_mi = agg_restore_chunks(spec, states, minput)
    # after an unflushed push: host (staged, not applied yet) and device
    ex = spec.executor(cuda)
    ex.apply_chunk(make_chunk(spec.types, [(INS, (1,) + (None,) * 6, True)]))
    refused(ex, good_st, good_mi)
    ex = spec.executor(cuda)
    device.agg_push_device(ex, TA.device_chunk(make_chunk(spec.types, [(INS, (1,) + (None,) * 6, True)]), False), None)
    refused(ex, good_st, good_mi)
    # schema / type mismatches
    bad = [Column(c.type, c.data, c.valid) for c in good_st.columns]
    bad[3] = Column(abi.T_INT32, np.zeros(len(states), np.int32))
    refused(spec.executor(cuda), StreamChunk(good_st.ops, bad), None)
    refused(spec.executor(cuda), StreamChunk(good_st.ops, good_st.columns[:-1]), None)
    mt = minput_types(spec)
    for k, t in ((0, "int4"), (nk, "int8"), (nk + 1, "int4")):
        tt = list(mt)
        tt[k] = t
        refused(spec.executor(cuda), good_st, make_chunk(tt, [(INS, (1, 11, 1), True)]))
    # minput for a plan without retractable min / max
    ao = int_state_spec(True)
    m2, _ = run_model(ao, agg_case("int_ao")[1][:2])
    st2, _ = m2.snapshot()
    refused(ao.executor(cuda), make_chunk(ao.out_types, [(INS, r, True) for r in st2]),
            make_chunk(minput_types(ao), [(INS, st2[0][:1] + (7, 1), True)]))
    # call index out of range, or naming a call that is not a retractable min / max
    key = states[0][:nk]
    for c in (-1, len(spec.calls), 0, 2):
        refused(spec.executor(cuda), good_st, make_chunk(mt, [(INS, key + (c, 1), True)]))
    # a minput row whose group has no state row (yet): refused, also when its state row would come in a later call
    ex = spec.executor(cuda)
    ex.restore(*agg_restore_chunks(spec, states[:1], []))
    refused(ex, make_chunk(spec.out_types, []), make_chunk(mt, [(INS, (123456,) + (11, 1), True)]))
    lone = [r for r in minput if tuple(r[:nk]) != tuple(states[0][:nk])][:1]
    assert lone
    ex = spec.executor(cuda)
    refused(ex, *agg_restore_chunks(spec, states[:1], lone))
    # and the good chunks still restore
    ex = spec.executor(cuda)
    ex.restore(good_st, good_mi)
    assert chunk_rows(ex.flush_data(1), spec.out_types) == []


# ============================================================================ HashJoin: the restatement's state
def can_match(plan, row):
    return all(row[k] is not None or ns for k, ns in zip(plan.keys, plan.null_safe))


def stored_rows(m, side):
    """the rows the side's state holds (module docstring): matchable live rows; for an append-only plan, the
    unmatched ones"""
    p = m.p
    out = Counter()
    for g, rows in m.live[side].items():
        for r in rows:
            if not can_match(p, r):
                continue
            if p.append_only:
                other = m.live[1 - side].get(g, [])
                if any(m.match(r, o) if side == 0 else m.match(o, r) for o in other):
                    continue
            out[TJ.exact_row(r)] += 1
    return out


def live_list(m, side):
    """the stored rows as row tuples, oldest first within a key"""
    want = stored_rows(m, side)
    rows = []
    for g in m.live[side].values():
        for r in g:
            e = TJ.exact_row(r)
            if want[e] > 0:
                want[e] -= 1
                rows.append(r)
    return rows


def snapshot_rows(ex, plan, side):
    return TJ.chunk_rows(ex.snapshot(side), plan.types[side])


def drive_on(m, plan, push, pushes, label):
    """test_join_types.drive, continuing an existing restatement"""
    for i, (side, rows) in enumerate(pushes):
        want, _ = m.push(side, rows)
        got = push(side, TJ.make_chunk(plan.types[side], rows))
        net = TJ.signed_net(got)
        assert net == want, (f"{label} {plan} push {i} (side {side}): net change differs\n only in output "
                             f"{dict(Counter(net) - Counter(want))}\n only expected {dict(Counter(want) - Counter(net))}")
        m.check_bits(got)
    return m


def join_restore_chunk(plan, side, rows):
    return TJ.make_chunk(plan.types[side], [(INS, r, True) for r in rows])


def test_restatement_join_state_round_trip():
    """the restatement rebuilt from its own stored rows (either side first) gives the same later net changes"""
    for plan in PLANS:
        lengths = TJ.lengths_for(plan)
        pushes = stream(plan, 31, lengths + lengths[:6], wide=TJ.wide_for(plan))
        k = len(lengths)
        m = JoinModel(plan)
        for side, rows in pushes[:k]:
            m.push(side, rows)
        for order in ((0, 1), (1, 0)):
            a, b = copy.deepcopy(m), JoinModel(plan)
            for s in order:
                b.push(s, [(INS, r, True) for r in live_list(m, s)])
            for s in (0, 1):
                assert stored_rows(b, s) == stored_rows(a, s), (plan, order, s)
                for g, rows in a.live[s].items():  # (never-matching rows are no state, but a later delete names them)
                    b.live[s].setdefault(g, []).extend(r for r in rows if not can_match(plan, r))
            for i, (side, rows) in enumerate(pushes[k:]):
                assert a.push(side, rows)[0] == b.push(side, rows)[0], (plan, order, i)


# ---------------------------------------------------------------------------- GPU: restore
@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS, ids=str)
def test_device_join_restore_round_trip(cuda, plan):
    """drive, snapshot both sides (== the restatement's stored rows), restore into a fresh operator -- left first or
    right first -- and continue with inserts, deletes and U-/U+ on every push path; also restored from the
    restatement's own rows"""
    lengths = TJ.lengths_for(plan)
    pushes = stream(plan, 31, lengths + lengths[:6], wide=TJ.wide_for(plan))
    k = len(lengths)
    ex = plan.executor(cuda)
    try:
        m = drive(plan, TJ.host_push(ex, plan), pushes[:k], label="before snapshot")
        ex.flush_data(1)
        snaps = []
        for s in (0, 1):
            got = snapshot_rows(ex, plan, s)
            assert Counter(TJ.exact_row(r) for _, r in got) == stored_rows(m, s), f"{plan} snapshot side {s}"
            snaps.append([r for _, r in got])
    finally:
        TJ.close(ex)
    runs = [(path, i % 2, "snapshot") for i, path in enumerate(PATHS)] + [("host", 0, "restatement"), ("device", 1, "restatement")]
    for path, flip, src in runs:
        order = (1, 0) if flip else (0, 1)
        rows = snaps if src == "snapshot" else [live_list(m, s) for s in (0, 1)]
        ex2 = plan.executor(cuda)
        try:
            for s in order:
                if rows[s]:
                    ex2.restore(s, join_restore_chunk(plan, s, rows[s]))
            ex2.flush_data(2)
            for s in (0, 1):
                assert Counter(TJ.exact_row(r) for _, r in snapshot_rows(ex2, plan, s)) == stored_rows(m, s), f"{plan} restored side {s}"
            drive_on(copy.deepcopy(m), plan, TJ.gpu_push(path, ex2, plan), pushes[k:], f"restored from the {src} {order}, {path}")
        finally:
            TJ.close(ex2)


# which of two equal-pk rows of one restore chunk a delete removes: the later one on the unified and fused paths; the
# generic path removes the earlier one (DESIGN §9)
EQUAL_PK_PLANS = {"uni_int8": "later", "fused_int4": "later", "generic_left_outer_float8": "earlier"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", EQUAL_PK_PLANS)
def test_device_join_restore_equal_pk_rows_in_chunk_order(cuda, name):
    """two live rows of one key with an equal pk: a restore keeps both, and a delete of that pk removes the one that
    EQUAL_PK_PLANS names for the plan's path"""
    plan = TJ.BY_NAME[name]
    L = plan.types[0]

    def row(pay):
        v = [5 if k in plan.keys else (1 if k in plan.pk else pay) for k in range(len(L))]
        return tuple(TJ.fl(t, x) if t in TJ.FLOAT_NP else x for x, t in zip(v, L))
    a, b = row(10), row(20)
    for first, second in ((a, b), (b, a)):
        ex = plan.executor(cuda)
        try:
            ex.restore(0, join_restore_chunk(plan, 0, [first, second]))
            assert Counter(TJ.exact_row(r) for _, r in snapshot_rows(ex, plan, 0)) == Counter([TJ.exact_row(a), TJ.exact_row(b)])
            ex.eq_join_oneside(0, TJ.make_chunk(L, [(DEL, first, True)]))
            kept = first if EQUAL_PK_PLANS[name] == "later" else second
            assert [TJ.exact_row(r) for _, r in snapshot_rows(ex, plan, 0)] == [TJ.exact_row(kept)], (name, first)
        finally:
            TJ.close(ex)


@pytest.mark.gpu
def test_device_join_restore_past_one_slice(cuda):
    """rwgpu_join_restore replays 2^20 rows per push: a restore of 2^20 + 4099 rows with a validity bitmap and a
    varchar column crosses a slice boundary (bitmap words at lo / 64, varlen offsets at + lo)"""
    n = (1 << 20) + 4099
    tl = [abi.T_INT64, abi.T_INT64, abi.T_VARCHAR, abi.T_INT32]
    tr = [abi.T_INT64, abi.T_INT64]
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    ex = HashJoinExecutor(cuda, abi.JOIN_INNER, sl.into_executor(tl, [1]), sr.into_executor(tr, [1]), JoinParams([0], [1]),
                          JoinParams([0], [1]), [False])
    i = np.arange(n, dtype=np.int64)
    key = i % 70001
    words = np.empty(n, dtype=object)
    for j in range(n):
        words[j] = b"w%d" % (j * 7 % 1000) if j % 5 else b""
    sval = (i % 11) != 3
    ival = (i % 13) != 0
    ch = StreamChunk(np.full(n, INS, np.uint8), [Column(abi.T_INT64, key), Column(abi.T_INT64, i), Column(abi.T_VARCHAR, words, sval),
                                                Column(abi.T_INT32, (i * 3).astype(np.int32), ival)])
    ex.restore(0, ch)
    got = concat_chunks(ex.snapshot(0))
    assert got.capacity() == n
    order = np.argsort(got.columns[1].data, kind="stable")
    assert (got.columns[1].data[order] == i).all() and (got.columns[0].data[order] == key).all()
    gv = got.columns[3].valid
    assert (gv[order] if gv is not None else np.ones(n, bool)).tolist() == ival.tolist()
    assert (got.columns[3].data[order][ival] == (i * 3).astype(np.int32)[ival]).all()
    sv = got.columns[2].valid if got.columns[2].valid is not None else np.ones(n, bool)
    assert sv[order].tolist() == sval.tolist()
    gw = got.columns[2].data[order]
    bad = [j for j in range(n) if sval[j] and bytes(gw[j]) != words[j]]
    assert not bad, bad[:5]
    # a right row meets every left row of its key, wherever in the restore they came
    probe = [0, (1 << 20) - 1, 1 << 20, n - 1]
    rrows = [(INS, (int(key[j]), 10 ** 9 + j)) for j in probe]
    out = ex.eq_join_oneside(1, StreamChunk.from_rows(tr, rrows))
    got_pairs = Counter((r[1], r[5]) for c in out for _, r in c.rows())
    want = Counter((int(l), 10 ** 9 + j) for j in probe for l in i[key == key[j]])
    assert got_pairs == want


# ============================================================================ join-key watermark cleaning
WM_KEY_EDGES = {t: TJ.int_edges(t) for t in ("int2", "int4", "int8", "date", "time", "timestamp", "timestamptz", "serial")}


def wm_plans():
    ps = [TJ.BY_NAME[f"uni_{t}"] for t in ("int8", "timestamp", "timestamptz", "time", "serial")]  # unified, inner
    for jt, kt in (("inner", "int2"), ("left_outer", "int4"), ("right_outer", "date"), ("full_outer", "int8"), ("left_semi", "time"),
                   ("left_anti", "timestamp"), ("right_semi", "timestamptz"), ("right_anti", "serial")):
        ps.append(Plan(f"two_{jt}_{kt}", jt, [kt, "int8", "int4"], [kt, "int8", "int2"], [0], [1]))
    ps.append(Plan("two_multi_inner", "inner", ["int4", "date", "int8", "int8"], ["int4", "date", "int8"], [0, 1], [2], null_safe=[False, True]))
    ps.append(Plan("two_multi_full_outer", "full_outer", ["int8", "int2", "int8"], ["int8", "int2", "int8"], [0, 1], [2],
                   null_safe=[True, False]))
    return ps


WM_PLANS = wm_plans()


def key_pool(t, rng):
    edges = WM_KEY_EDGES[t]
    lo, hi = min(edges), max(edges)
    mid = [int(x) for x in rng.integers(max(lo, -60), min(hi, 60) + 1, 12)]
    return sorted(set(edges + mid))


class WmStream:
    """inserts, deletes of live rows and payload U-/U+ pairs; a floor keeps new keys at or above the watermark"""

    def __init__(self, plan, seed):
        self.p, self.rng = plan, np.random.default_rng(seed)
        self.pools = [key_pool(plan.types[0][k], self.rng) for k in plan.keys]
        self.next_pk = 1 << 20

    def payload(self, t):
        v = int(self.rng.integers(-100, 100))
        return TJ.fl(t, v / 4) if t in TJ.FLOAT_NP else v

    def new_row(self, side, floor):
        p, row = self.p, []
        for k, t in enumerate(p.types[side]):
            if k in p.keys:
                i = p.keys.index(k)
                pool = [v for v in self.pools[i] if floor is None or floor[0] != i or v >= floor[1]]
                nul = p.null_safe[i] or p.jt != abi.JOIN_INNER
                row.append(None if nul and self.rng.random() < 0.08 else pool[int(self.rng.integers(len(pool)))])
            elif k in p.pk:
                self.next_pk += 1
                row.append(self.next_pk)
            else:
                row.append(self.payload(t))
        return tuple(row)

    def chunk(self, m, side, n, floor=None):
        rows = []
        live = [r for g in m.live[side].values() for r in g]
        gone = set()
        while len(rows) < n:
            x = self.rng.random()
            cand = [j for j in range(len(live)) if j not in gone]
            if cand and x < 0.2:
                j = cand[int(self.rng.integers(len(cand)))]
                gone.add(j)
                rows.append((DEL, live[j], True))
            elif cand and x < 0.35:
                j = cand[int(self.rng.integers(len(cand)))]
                gone.add(j)
                old = live[j]
                pay = [k for k in range(len(old)) if k not in self.p.keys and k not in self.p.pk][:1]
                new = tuple(self.payload(self.p.types[side][k]) if k in pay else v for k, v in enumerate(old))
                rows += [(UD, old, True), (UI, new, True)]
            else:
                rows.append((INS, self.new_row(side, floor), True))
        return rows


def wm_clean(m, side, key_pos, v):
    """the restatement's cleaning at the barrier (module docstring)"""
    k = m.p.keys[key_pos]
    for g in list(m.live[side]):
        m.live[side][g] = [r for r in m.live[side][g] if r[k] is None or r[k] >= v]


def wm_values(plan, key_pos, m):
    """watermarks at a stored key - 1, the key and key + 1, and the column type's extremes"""
    t = plan.types[0][plan.keys[key_pos]]
    keys = sorted({r[plan.keys[key_pos]] for s in (0, 1) for g in m.live[s].values() for r in g if r[plan.keys[key_pos]] is not None})
    lo, hi = min(WM_KEY_EDGES[t]), max(WM_KEY_EDGES[t])
    mid = keys[len(keys) // 2]
    return [lo, lo + 1, mid - 1, mid, mid + 1, hi]


def check_state(ex, plan, m, label):
    for s in (0, 1):
        got = Counter(TJ.exact_row(r) for _, r in snapshot_rows(ex, plan, s))
        want = stored_rows(m, s)
        assert got == want, f"{label} side {s}: only got {got - want}\n only want {want - got}"


def test_restatement_wm_clean_is_strict_and_keeps_nulls():
    plan = TJ.BY_NAME["uni_int8"]
    m = JoinModel(plan)
    m.push(0, [(INS, (v, i, TJ.fl("float8", 1.0), 0), True) for i, v in enumerate([I64MIN, -1, 0, 1, I64MAX])])
    wm_clean(m, 0, 0, 0)
    assert sorted(r[0] for g in m.live[0].values() for r in g) == [0, 1, I64MAX]
    p2 = WM_PLANS[-2]
    m = JoinModel(p2)
    m.push(0, [(INS, (1, None, 1, 0), True), (INS, (1, -5, 2, 0), True), (INS, (None, 3, 3, 0), True)])
    wm_clean(m, 0, 1, 0)
    assert sorted(r[2] for g in m.live[0].values() for r in g) == [1, 3]


def test_restatement_reproduces_streaming_hash_join_watermark():
    """hash_join.rs:3648-3715 as test_oracle_golden transcribes it: the watermark that cleans both sides is the smaller
    of the two sides' buffered heads (BufferedWatermarks, watermark/mod.rs:38-115)"""
    events = [(0, 100), (0, 200), (1, 50), (1, 100)]
    heads, emitted = ([], []), []
    for side, v in events:
        heads[side].append(v)
        if heads[0] and heads[1]:
            w = min(heads[0][0], heads[1][0])
            emitted.append(w)
            for s in (0, 1):
                if heads[s][0] == w:
                    heads[s].pop(0)
    assert emitted == [50, 100]


@pytest.mark.gpu
@pytest.mark.parametrize("plan", WM_PLANS, ids=str)
def test_device_watermark_cleaning(cuda, plan):
    """per key position and watermark: drive, update_watermark (nothing changes before the barrier), barrier (the
    state is the restatement's, cleaned), then pushes that respect the watermark on every path"""
    positions = range(len(plan.keys))
    for key_pos in positions:
        for wi in range(6):
            gen = WmStream(plan, 100 * key_pos + wi)
            ex = plan.executor(cuda)
            try:
                m = JoinModel(plan)
                for i in range(6):
                    side = i % 2
                    drive_on(m, plan, TJ.host_push(ex, plan), [(side, gen.chunk(m, side, 40))], "before")
                v = wm_values(plan, key_pos, m)[wi]
                sides = (0, 1) if wi % 3 else ((wi // 3) % 2,)
                for s in sides:
                    ex.update_watermark(s, key_pos, v)
                check_state(ex, plan, m, f"{plan} pending {v}")
                ex.flush_data(1)
                for s in sides:
                    wm_clean(m, s, key_pos, v)
                check_state(ex, plan, m, f"{plan} key_pos {key_pos} wm {v} sides {sides}")
                path = PATHS[wi % len(PATHS)]
                push = TJ.gpu_push(path, ex, plan)
                for i in range(4):
                    side = i % 2
                    drive_on(m, plan, push, [(side, gen.chunk(m, side, 33, floor=(key_pos, v)))], f"after wm {v}, {path}")
            finally:
                TJ.close(ex)


@pytest.mark.gpu
def test_device_watermark_pending_rules(cuda):
    """a lower watermark while one is pending is ignored; another key_pos replaces the pending one"""
    plan = [p for p in WM_PLANS if p.name == "two_multi_inner"][0]
    for calls, clean in (([(0, 30), (0, 10)], (0, 30)), ([(0, 30), (1, 5)], (1, 5)), ([(1, 5), (0, -100), (0, 2)], (0, 2))):
        gen = WmStream(plan, 7)
        ex = plan.executor(cuda)
        try:
            m = JoinModel(plan)
            for i in range(4):
                drive_on(m, plan, TJ.host_push(ex, plan), [(i % 2, gen.chunk(m, i % 2, 60))], "before")
            for kp, v in calls:
                ex.update_watermark(0, kp, v)
            ex.flush_data(1)
            wm_clean(m, 0, *clean)
            check_state(ex, plan, m, f"{calls}")
        finally:
            TJ.close(ex)


@pytest.mark.gpu
def test_device_watermark_through_handle_watermark(cuda):
    """test_oracle_golden.test_streaming_hash_join_watermark (hash_join.rs:3648-3715) on the CUDA backend: the same
    output watermarks, and at the next barrier both sides' state holds only keys >= 100"""
    I = abi.T_INT64
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    ex = HashJoinExecutor(cuda, abi.JOIN_INNER, sl.into_executor([I, I], [1]), sr.into_executor([I, I], [1]),
                          JoinParams([0], [1]), JoinParams([0], [1]), [False], watermark_indices_in_jk=[(0, True)])
    keys = [20, 50, 99, 100, 101, 250, I64MIN]
    for s in (0, 1):
        ex.eq_join_oneside(s, StreamChunk.from_rows([I, I], [(INS, (k, 10 * s + j)) for j, k in enumerate(keys)]))
    ex.flush_data(1)
    assert ex.handle_watermark(0, Watermark(0, I, 100)) == []
    assert ex.handle_watermark(0, Watermark(0, I, 200)) == []
    ex.flush_data(2)
    assert all(len([r for c in ex.snapshot(s) for r in c.rows()]) == len(keys) for s in (0, 1))
    assert ex.handle_watermark(1, Watermark(0, I, 50)) == [Watermark(2, I, 50), Watermark(0, I, 50)]
    assert ex.handle_watermark(1, Watermark(0, I, 100)) == [Watermark(2, I, 100), Watermark(0, I, 100)]
    ex.flush_data(3)
    for s in (0, 1):
        assert sorted(r[0] for c in ex.snapshot(s) for _, r in c.rows()) == [100, 101, 250]


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("name", ["uni_int8", "two_left_outer_int4"])
def test_device_watermark_late_rows(cuda, name, strict):
    """rwgpu.h's rule for rows below the watermark after cleaning: a late insert matches nothing of the cleaned side
    and is stored; a late delete of a cleaned row is RW_ERR_INCONSISTENT with strict_consistency, else a no-op"""
    plan = TJ.BY_NAME.get(name) or [p for p in WM_PLANS if p.name == name][0]
    L, R = plan.types

    def row(side, k, pk):
        return tuple(k if c in plan.keys else (pk if c in plan.pk else (TJ.fl(t, 1.0) if t in TJ.FLOAT_NP else 3))
                     for c, t in enumerate(plan.types[side]))

    def mk():
        srcs = []
        for s in range(2):
            _, src = MockSource.channel()
            srcs.append(src.into_executor([TJ.T_OF[t] for t in plan.types[s]], plan.pk))
        return HashJoinExecutor(cuda, plan.jt, srcs[0], srcs[1], JoinParams(plan.keys, plan.pk), JoinParams(plan.keys, plan.pk),
                                plan.null_safe, plan.out, None, False, strict_consistency=strict)
    for late in ("insert", "delete"):
        ex = mk()
        try:
            ex.eq_join_oneside(0, TJ.make_chunk(L, [(INS, row(0, k, k), True) for k in (1, 2, 3, 10)]))
            ex.eq_join_oneside(1, TJ.make_chunk(R, [(INS, row(1, k, 100 + k), True) for k in (1, 2, 3, 10)]))
            for s in (0, 1):
                ex.update_watermark(s, 0, 5)
            ex.flush_data(1)
            assert [r[0] for _, r in snapshot_rows(ex, plan, 0)] == [10]
            if late == "insert":
                out = TJ.chunk_rows(ex.eq_join_oneside(0, TJ.make_chunk(L, [(INS, row(0, 2, 50), True)])), plan.out_types)
                want_vis = 1 if plan.jt == abi.JOIN_LEFT_OUTER else 0  # (only the NULL-padded row of an outer join)
                assert len(out) == want_vis and all(all(v is None for v in r[len(L):]) for _, r in out), out
                assert sorted(r[0] for _, r in snapshot_rows(ex, plan, 0)) == [2, 10]
            elif strict:
                with pytest.raises(abi.RwError) as e:
                    ex.eq_join_oneside(0, TJ.make_chunk(L, [(DEL, row(0, 2, 2), True)]))
                assert e.value.code == abi.RW_ERR_INCONSISTENT
            else:
                out = TJ.chunk_rows(ex.eq_join_oneside(0, TJ.make_chunk(L, [(DEL, row(0, 2, 2), True)])), plan.out_types)
                assert TJ.signed_net(out) == ({} if plan.jt == abi.JOIN_INNER else TJ.signed_net([(DEL, (2, 2, 3, None, None, None))]))
                assert [r[0] for _, r in snapshot_rows(ex, plan, 0)] == [10]
        finally:
            TJ.close(ex)


@pytest.mark.gpu
def test_device_watermark_refusals(cuda):
    def code(ex, side, kp, v=0):
        with pytest.raises(abi.RwError) as e:
            ex.update_watermark(side, kp, v)
        return e.value.code
    for name in ("fused_float8", "fused_float4", "fused_bool", "generic_left_outer_float8"):
        ex = TJ.BY_NAME[name].executor(cuda)
        assert code(ex, 0, 0) == abi.RW_ERR_UNSUPPORTED, name
        TJ.close(ex)
    ex = TJ.BY_NAME["uni_int8"].executor(cuda)
    assert [code(ex, 2, 0), code(ex, -1, 0), code(ex, 0, 1), code(ex, 0, -1)] == [abi.RW_ERR_INVALID] * 4
    TJ.close(ex)
    ex = TJ.BY_NAME["fused_multi_key"].executor(cuda)
    assert code(ex, 0, 4) == abi.RW_ERR_INVALID
    assert code(ex, 0, 1) == abi.RW_ERR_UNSUPPORTED  # (a bool key column)
    ex.update_watermark(0, 2, 0)  # (a date key column)
    TJ.close(ex)


# ============================================================================ cleaning feeds compaction
def compactions(cuda, ex):
    import ctypes as C
    fn = cuda.lib.rwgpu_join_compactions
    fn.restype, fn.argtypes = C.c_uint64, [C.c_void_p]
    return int(fn(ex._h))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["clean_most", "clean_some_and_delete", "clean_some", "two_table"])
def test_device_cleaning_feeds_compaction(cuda, case):
    """unified plan, left side (the chained side: every row a log record) with 10000 rows: cleaning 6000 compacts
    once; cleaning 4000 and deleting 1500 compacts once; cleaning 4000 alone does not; a second barrier with nothing
    new never compacts again; a two-table plan never compacts.  Snapshot and later pushes follow the restatement."""
    plan = TJ.BY_NAME["uni_int8"] if case != "two_table" else [p for p in WM_PLANS if p.name == "two_full_outer_int8"][0]
    n = 10000
    ex = plan.executor(cuda)
    try:
        m = JoinModel(plan)
        L, R = plan.types

        def row(side, k, pk):
            return tuple(k if c in plan.keys else (pk if c in plan.pk else (TJ.fl(t, 0.5) if t in TJ.FLOAT_NP else k % 7))
                         for c, t in enumerate(plan.types[side]))
        left = [row(0, k - 3000, k) for k in range(n)]
        for lo in range(0, n, 2500):
            drive_on(m, plan, TJ.host_push(ex, plan), [(0, [(INS, r, True) for r in left[lo:lo + 2500]])], "fill")
        drive_on(m, plan, TJ.host_push(ex, plan), [(1, [(INS, row(1, k, n + k), True) for k in range(-3000, 7000, 97)])], "right")
        ex.flush_data(1)
        c0 = compactions(cuda, ex)
        wm = 3000 if case == "clean_most" else 1000
        if case == "clean_some_and_delete":
            dels = [(DEL, r, True) for r in left[5000:6500]]
            drive_on(m, plan, TJ.host_push(ex, plan), [(0, dels)], "deletes")
        ex.update_watermark(0, 0, wm)
        ex.flush_data(2)
        wm_clean(m, 0, 0, wm)
        want = 1 if case in ("clean_most", "clean_some_and_delete") else 0
        assert compactions(cuda, ex) - c0 == want, case
        ex.flush_data(3)
        assert compactions(cuda, ex) - c0 == want, f"{case}: a barrier with nothing new compacted again"
        check_state(ex, plan, m, case)
        gen = WmStream(plan, 3)
        for i, path in enumerate(PATHS):
            drive_on(m, plan, TJ.gpu_push(path, ex, plan), [(i % 2, gen.chunk(m, i % 2, 300, floor=(0, wm)))], f"{case} {path}")
        check_state(ex, plan, m, f"{case} after")
    finally:
        TJ.close(ex)
