"""CPU: pin the oracle (oracle/oracle.cc) to the reference's own golden vectors.

  * every non-watermark #[tokio::test] of src/stream/src/executor/hash_join.rs (exact StreamChunk
    equality incl. visibility, as the reference asserts)
  * src/stream/tests/integration_tests/hash_agg.rs (sorted snapshot comparison)
  * src/expr/impl/src/aggregate/general.rs aggregate-function tests
  * CRC32 vnode against zlib and the routing of test_hash_dispatcher (dispatch.rs:1551-1660)
  * src/stream/src/executor/filter.rs tests (exact StreamChunk equality incl. the hidden halves of U-/U+ pairs)
"""
import ctypes as C
import math
import re
import zlib

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import AggCall, FilterExecutor, MockSource
from risingwave_b200.stream_chunk import StreamChunk

from helpers import load_golden, run_agg_kat, run_join_kat, run_nexmark_q4, run_nexmark_q7, run_nexmark_q8

JOIN_KATS = [k for k in load_golden("hash_join_kats.json") if "skipped" not in k]
AGG_KATS = [k for k in load_golden("hash_agg_kats.json") if "skipped" not in k]
FUNC_KATS = load_golden("agg_func_kats.json")
FILTER_KATS = load_golden("filter_kats.json")


def test_golden_counts():
    assert len(JOIN_KATS) == 24 and len(AGG_KATS) == 3 and len(FUNC_KATS) >= 20


@pytest.mark.parametrize("kat", JOIN_KATS, ids=[k["name"] for k in JOIN_KATS])
def test_hash_join_golden(oracle, kat):
    run_join_kat(oracle, kat, exact=True)


@pytest.mark.parametrize("kat", AGG_KATS, ids=[k["name"] for k in AGG_KATS])
def test_hash_agg_golden(oracle, kat):
    """incl. test_hash_agg_min (hash_agg.rs:97-170): retractable min = MaterializedInput state (minput.rs)"""
    run_agg_kat(oracle, kat)


def _expected_value(expr):
    m = re.search(r"Some\(\(?(-?[\w.:]+)\)?\.into\(\)\)", expr)
    tok = m.group(1) if m else None
    m2 = re.search(r"Decimal::from\((-?\d+)\)", expr)
    if m2:
        return int(m2.group(1))
    if tok is None:
        return None
    if "INFINITY" in tok:
        return math.inf
    if "NAN" in tok:
        return math.nan
    tok = re.sub(r"(i64|f64|f32)$", "", tok)
    return float(tok) if "." in tok else int(tok)


SUPPORTED_FUNCS = [k for k in FUNC_KATS if re.match(r"\((sum|min|max|count):", k["call"])
                   and "varchar" not in k["call"] and "[]" not in k["call"]]


@pytest.mark.parametrize("kat", SUPPORTED_FUNCS, ids=[k["name"] for k in SUPPORTED_FUNCS])
def test_agg_function_golden(oracle, kat):
    call = AggCall.from_pretty(kat["call"])
    chunk = StreamChunk.from_pretty(kat["input"])
    fn = oracle.lib.rwo_agg_eval
    fn.restype = C.c_int32
    c = abi.RwAggCall(call.kind, call.arg_col, call.ret_type, 0)
    ch, keep = chunk.to_abi()
    is_null, lo, hi, f = C.c_int32(), C.c_int64(), C.c_int64(), C.c_double()
    rc = fn(C.byref(c), C.c_int32(call.arg_type), C.byref(ch), C.byref(is_null), C.byref(lo), C.byref(hi), C.byref(f))
    assert rc == 0
    want = _expected_value(kat["expected_expr"])
    if call.ret_type in (abi.T_FLOAT32, abi.T_FLOAT64):
        got = f.value
        assert (math.isnan(got) and math.isnan(want)) or got == want
    else:
        assert not is_null.value
        assert ((hi.value << 64) | (lo.value & (2**64 - 1))) == want


# ------------------------------------------------------------------ vnode / dispatcher
def test_crc32_matches_zlib(oracle):
    fn = oracle.lib.rwo_crc32
    fn.restype = C.c_uint32
    rng = np.random.default_rng(7)
    for n in (0, 1, 3, 4, 8, 9, 64, 1000):
        b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert fn(b, C.c_int64(n)) == zlib.crc32(b)


def test_hash_dispatcher_vnodes(oracle):
    """test_hash_dispatcher (dispatch.rs:1551-1660) recomputes crc32(LE bytes of the i32 key columns)
    % 256 per row; vnode -> output by `vnode % n_outputs`-style mapping.  We check the vnode values."""
    rng = np.random.default_rng(0)
    n = 1000
    a = rng.integers(-2**31, 2**31, n).astype(np.int32)
    b = rng.integers(0, 10, n).astype(np.int32)
    c = rng.integers(0, 10, n).astype(np.int32)
    from risingwave_b200.stream_chunk import Column
    chunk = StreamChunk(np.full(n, 1, np.uint8), [Column(abi.T_INT32, a), Column(abi.T_INT32, b), Column(abi.T_INT32, c)])
    got = oracle.vnode_compute(chunk, [0, 2], 256)
    want = [zlib.crc32(a[i].tobytes() + c[i].tobytes()) % 256 for i in range(n)]
    assert got.tolist() == want
    # NULL datum => u32 0xfffffff0 (array/mod.rs:97); invisible row => crc32("") == 0
    chunk2 = StreamChunk.from_pretty(" I\n + .\n + 5 D\n + 5")
    v = oracle.vnode_compute(chunk2, [0], 256)
    assert v[0] == zlib.crc32((0xfffffff0).to_bytes(4, "little")) % 256
    assert v[1] == 0
    assert v[2] == zlib.crc32((5).to_bytes(8, "little")) % 256


def test_dispatch_update_rewrite(oracle):
    """U-/U+ whose distribution key changes is rewritten to -/+ (dispatch.rs:1001-1019; pinned by the
    reference's test at dispatch.rs:1304-1375)."""
    chunk = StreamChunk.from_pretty(" I I\n U- 1 10\n U+ 1 11\n U- 2 20\n U+ 3 20\n + 4 0")
    ops = oracle.dispatch_rewrite_ops(chunk, [0])
    assert ops.tolist() == [abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT, abi.OP_DELETE, abi.OP_INSERT, abi.OP_INSERT]


def run_filter_kat(backend, kat):
    types = StreamChunk.from_pretty(kat["inputs"][0]).types()
    _, src = MockSource.channel()
    ex = FilterExecutor(backend, src.into_executor(types, []), kat["expr"], upsert=kat["upsert"])
    for inp, exp in zip(kat["inputs"], kat["expected"]):
        got = ex.filter(StreamChunk.from_pretty(inp))
        want = StreamChunk.from_pretty(exp)
        assert got == want, f"{kat['name']}\n got\n{got.to_pretty()}\n want\n{want.to_pretty()}"


@pytest.mark.parametrize("kat", FILTER_KATS, ids=[k["name"] for k in FILTER_KATS])
def test_filter_golden(oracle, kat):
    assert len(FILTER_KATS) == 2
    run_filter_kat(oracle, kat)


def test_filter_oracle_three_valued_all_hidden_and_unpaired_updates(oracle):
    """NULL operands make the row's result false (filter.rs:79); a chunk without visible rows yields nothing (:146-150); a
    U- or U+ without its partner follows the project's pairing rule (rwgpu.h) instead of failing the chunk"""
    _, src = MockSource.channel()
    ex = FilterExecutor(oracle, src.into_executor([abi.T_INT64, abi.T_INT64], []),
                        "(and:boolean (greater_than:boolean $0:int8 $1:int8) (less_than:boolean $0:int8 100:int8))")
    got = ex.filter(StreamChunk.from_pretty(" I I\n + 5 . \n + . 1 \n + 7 3 \n + 700 3 \n - 9 8"))
    assert got == StreamChunk.from_pretty(" I I\n + 5 . D\n + . 1 D\n + 7 3 \n + 700 3 D\n - 9 8")
    assert ex.filter(StreamChunk.from_pretty(" I I\n + 1 2 \n - 1 2")) is None
    # a U- whose U+ is missing (the reference never sees one): filtered like a -, keeping its op, as on the device
    got = ex.filter(StreamChunk.from_pretty(" I I\n U- 5 1 \n U- 50 1 \n + 7 3 \n U- 500 1 \n U+ 5 1"))
    assert got == StreamChunk.from_pretty(" I I\n U- 5 1 \n U- 50 1 \n + 7 3 \n U- 500 1 D\n + 5 1")


def test_nexmark_q4_end_to_end_fixture(oracle):
    """the reference's SQL-level q4 fixture through the oracle's operators (helpers.run_nexmark_q4)"""
    run_nexmark_q4(oracle)


def test_nexmark_q7_end_to_end_fixture(oracle):
    """the reference's SQL-level q7 fixture through the oracle's operators (helpers.run_nexmark_q7): the join's right
    side is an aggregate that retracts and re-emits its maxima"""
    run_nexmark_q7(oracle)


def test_nexmark_q8_end_to_end_fixture(oracle):
    """the reference's SQL-level q8 fixture through the oracle's operators (helpers.run_nexmark_q8): two group-by
    aggregates feeding a join on a three-column key, both sides updating"""
    run_nexmark_q8(oracle)


def test_join_entry_state_iteration_order(oracle):
    """join/hash_join.rs:889-918 `test_managed_join_state`: a key's rows iterate in insertion order while they live in
    the inline `Vec` (<= 4 rows: pk 3, 2, 1) and in pk order once the set spilled to the `BTreeMap` (1, 2, 3, 4, 5).
    Observed through the order of the matches a probe emits (same data; the join key is a constant column).  The
    first probe makes the key's entry resident in the cache (a miss reads the state table in pk order instead:
    hash_join.rs `take_state`), the rows inserted afterwards go into that cached entry."""
    from risingwave_b200.executor import HashJoinExecutor, JoinParams
    I = abi.T_INT64
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    ex = HashJoinExecutor(oracle, abi.JOIN_INNER, sl.into_executor([I, I], [1]), sr.into_executor([I, I, I], [1]),
                          JoinParams([0], [1]), JoinParams([0], [1]), [False])
    matched = lambda out: [(r[1][3], r[1][4]) for c in out for r in c.rows()]
    assert ex.eq_join_oneside(0, StreamChunk.from_pretty(" I I\n + 7 100")) == []          # miss: caches the (empty) entry of key 7
    assert matched(ex.eq_join_oneside(1, StreamChunk.from_pretty(" I I I\n + 7 3 4\n + 7 2 5\n + 7 1 6"))) == [(3, 4), (2, 5), (1, 6)]
    assert matched(ex.eq_join_oneside(0, StreamChunk.from_pretty(" I I\n + 7 101"))) == [(3, 4), (2, 5), (1, 6)]   # `Vec`
    ex.eq_join_oneside(1, StreamChunk.from_pretty(" I I I\n + 7 5 8\n + 7 4 9"))
    assert matched(ex.eq_join_oneside(0, StreamChunk.from_pretty(" I I\n + 7 102"))) == [(1, 6), (2, 5), (3, 4), (4, 9), (5, 8)]  # `BTreeMap`


def test_group_key_null_positions_are_kept_apart(oracle):
    """hash/key.rs:839-866 `test_simple_hash_key_nullable_serde`: the keys <1, NULL> and <NULL, 2> (two Int32 columns)
    are different keys and deserialize back losslessly -- here: they form two groups whose key columns come back
    exactly as they went in."""
    from risingwave_b200.executor import HashAggExecutor
    _, src = MockSource.channel()
    agg = HashAggExecutor(oracle, src.into_executor([abi.T_INT32, abi.T_INT32], []), True, [AggCall.from_pretty("(count:int8)")], 0, [0, 1])
    agg.apply_chunk(StreamChunk.from_pretty(" i i\n + 1 .\n + . 2\n + 1 .\n + . ."))
    rows = sorted((r[1] for c in agg.flush_data(1) for r in c.rows()), key=repr)
    assert rows == sorted([(1, None, 2), (None, 2, 1), (None, None, 1)], key=repr)


# ------------------------------------------------------------------------------------------ Project
def run_project_kat(backend, kat):
    from risingwave_b200.executor import ProjectExecutor
    types = [abi.T_INT64] * 2
    _, src = MockSource.channel()
    pe = ProjectExecutor(backend, src.into_executor(types, [0]), kat["exprs"])
    for inp, exp in zip(kat["inputs"], kat["expected"]):
        got = pe.apply_project_exprs(StreamChunk.from_pretty(inp))
        assert got == StreamChunk.from_pretty(exp), f"{kat['name']}:\n got\n{got}\n want\n{exp}"


@pytest.mark.parametrize("kat", load_golden("project_kats.json"), ids=lambda k: k["name"])
def test_project_golden(oracle, kat):
    """project_scalar.rs test_projection: exact output chunks"""
    run_project_kat(oracle, kat)


def test_project_arithmetic_is_non_strict_with_checked_rem_and_tumble_follows_the_reference_formula(oracle):
    """eval_infallible (project_scalar.rs:98): overflow / division by zero / MIN % -1 (checked_rem, arithmetic_op.rs:98-107)
    / NULL operand -> NULL for that row only; tumble_start = ts - (r < 0 ? r + w : r), r = ts rem w (tumble.rs:96-111),
    checked against a Python restatement"""
    from risingwave_b200.executor import ProjectExecutor
    types = [abi.T_INT64, abi.T_INT64, abi.T_INT32]
    _, src = MockSource.channel()
    exprs = ["(divide:int8 (multiply:int8 $0:int8 908:int8) 1000:int8)", "(tumble_start:int8 $0:int8 10000000:int8)",
             "(tumble_end:int8 $0:int8 $1:int8)", "(modulus:int8 $0:int8 $1:int8)", "(subtract:int4 $2:int4 $0:int8)", "(neg:int8 $0:int8)"]
    pe = ProjectExecutor(oracle, src.into_executor(types, [0]), exprs)
    big = (1 << 63) - 1
    rows = [(abi.OP_INSERT, (v, w, x)) for v, w, x in
            [(1000, 7, 5), (-1000, 7, -5), (big, 2, 1), (-big - 1, -1, 1), (None, 3, 2), (12345678901, 0, 0), (-12345678901, 10_000_000, 2 ** 31 - 1),
             (5, None, None), (0, 1, 0)]]
    out = pe.apply_project_exprs(StreamChunk.from_rows(types, rows))
    got = [r for _, r in out.rows()]

    def trunc_div(a, b):
        q = abs(a) // abs(b)
        return q if (a < 0) == (b < 0) else -q

    def i64(v):
        return v if v is not None and -(1 << 63) <= v <= big else None

    def win(ts, w):
        if w == 0:
            return None
        r = ts - trunc_div(ts, w) * w
        return i64(ts - (r + w if r < 0 else r))

    for (_, (v, w, x)), g in zip(rows, got):
        want = [None] * 6
        if v is not None:
            m = i64(v * 908)
            want[0] = None if m is None else trunc_div(m, 1000)
            want[1] = win(v, 10_000_000)
            want[5] = i64(-v)
            if w is not None:
                s0 = win(v, w)
                want[2] = None if s0 is None else i64(s0 + w)
                want[3] = None if w == 0 or (v == -big - 1 and w == -1) else v - trunc_div(v, w) * w  # checked_rem
            if x is not None:
                d = x - v
                want[4] = d if -(1 << 31) <= d < (1 << 31) else None
        assert list(g) == want, (v, w, x, g, want)


def test_tpch_q3_pipeline_oracle(oracle):
    """SURVEY 8(d) cfg5: the TPC-H q3 streaming plan (two inner joins, two projects, a three-column-key aggregation with a
    128-bit sum) through the oracle's operators, with retractions; the view must equal the SQL evaluated directly."""
    from helpers import run_tpch_q3
    got, deltas = run_tpch_q3(oracle)
    assert len(got) > 50 and any(op == abi.OP_UPDATE_DELETE for d in deltas for (op, _, _) in d)


def test_streaming_hash_join_watermark(oracle):
    """hash_join.rs:3648-3715 `test_streaming_hash_join_watermark`, transcribed: watermarks on the join key are buffered per
    side (BufferedWatermarks, watermark/mod.rs:38-115); what both sides have passed is emitted for the output columns of
    the key, the update side's first.  (create_classical_executor: two int64 columns per side, key = column 0.)"""
    from risingwave_b200.executor import BufferedWatermarks, HashJoinExecutor, JoinParams, MockSource, Watermark
    I = abi.T_INT64
    tx_l, sl = MockSource.channel()
    tx_r, sr = MockSource.channel()
    ex = HashJoinExecutor(oracle, abi.JOIN_INNER, sl.into_executor([I, I], [1]), sr.into_executor([I, I], [1]),
                          JoinParams([0], [1]), JoinParams([0], [1]), [False], watermark_indices_in_jk=[(0, True)])
    st = ex.execute()
    tx_l.push_barrier(1, False)
    tx_r.push_barrier(1, False)
    st.next_unwrap_ready_barrier()
    tx_l.push_watermark(0, I, 100)
    tx_l.push_watermark(0, I, 200)
    tx_l.push_barrier(2, False)
    tx_r.push_barrier(2, False)
    got = st.drain_until_pending()
    assert [m.barrier.epoch for m in got if m.barrier] == [2] and not any(m.watermark for m in got)
    tx_r.push_watermark(0, I, 50)
    w1, w2 = st.next_unwrap_ready_watermark(), st.next_unwrap_ready_watermark()
    tx_r.push_watermark(0, I, 100)
    w3, w4 = st.next_unwrap_ready_watermark(), st.next_unwrap_ready_watermark()
    assert (w1, w2, w3, w4) == (Watermark(2, I, 50), Watermark(0, I, 50), Watermark(2, I, 100), Watermark(0, I, 100))
    st.next_unwrap_pending()
    # BufferedWatermarks on its own: three upstreams, the smallest of the heads wins, equal followers are swallowed
    b = BufferedWatermarks([0, 1, 2])
    assert b.handle_watermark(0, Watermark(0, I, 7)) is None
    assert b.handle_watermark(1, Watermark(0, I, 5)) is None
    assert b.handle_watermark(1, Watermark(0, I, 9)) is None
    assert b.handle_watermark(2, Watermark(0, I, 5)) == Watermark(0, I, 5)   # 5 (id 1), then the equal 5 of id 2
    assert b.handle_watermark(2, Watermark(0, I, 8)) == Watermark(0, I, 7)   # heads now 7, 9, 8
