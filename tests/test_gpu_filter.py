"""GPU: the device Filter (csrc/chain.cu, through the C ABI) vs the reference's golden vectors and the CPU oracle,
and a join -> filter -> project -> agg chain that never leaves the device."""
import ctypes as C

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import AggCall, FilterExecutor, HashAggExecutor, HashJoinExecutor, JoinParams, MockSource, ProjectExecutor, parse_filter_expr
from risingwave_b200.stream_chunk import Column, StreamChunk, net_multiset

from helpers import load_golden, run_nexmark_q4, run_nexmark_q7, run_nexmark_q8
from test_oracle_golden import run_filter_kat

pytestmark = pytest.mark.gpu

FILTER_KATS = load_golden("filter_kats.json")


@pytest.mark.parametrize("kat", FILTER_KATS, ids=[k["name"] for k in FILTER_KATS])
def test_filter_golden(cuda, kat):
    run_filter_kat(cuda, kat)


def random_change_chunk(rng, n, types, null_frac, hidden_frac):
    """well-formed change stream: +, -, and U-/U+ pairs (a pair is hidden or visible as a whole)"""
    ops, vis = [], []
    while len(ops) < n:
        x = rng.random()
        v = rng.random() >= hidden_frac
        if x < 0.35 and len(ops) + 2 <= n:
            ops += [abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT]
            vis += [v, v]
        else:
            ops.append(abi.OP_INSERT if x < 0.75 else abi.OP_DELETE)
            vis.append(v)
    cols = []
    for t in types:
        dt = {abi.T_INT16: np.int16, abi.T_INT32: np.int32}.get(t, np.int64)
        data = rng.integers(-20, 20, n).astype(dt)
        valid = rng.random(n) >= null_frac if null_frac > 0 else None
        cols.append(Column(t, data, valid))
    vis = np.array(vis, bool)
    return StreamChunk(np.array(ops, np.uint8), cols, None if vis.all() else vis)


@pytest.mark.parametrize("upsert", [False, True])
@pytest.mark.parametrize("expr,types", [
    ("(greater_than:boolean $0:int8 $1:int8)", [abi.T_INT64, abi.T_INT64]),
    ("(and:boolean (greater_than_or_equal:boolean $0:int4 $1:int8) (less_than:boolean $2:int2 7:int2))", [abi.T_INT32, abi.T_INT64, abi.T_INT16]),
    ("(not_equal:boolean $1:int8 -3:int8)", [abi.T_INT64, abi.T_INT64]),
])
def test_filter_random_vs_oracle(cuda, oracle, expr, types, upsert):
    rng = np.random.default_rng(len(expr) + int(upsert))
    exs = []
    for be in (cuda, oracle):
        _, src = MockSource.channel()
        exs.append(FilterExecutor(be, src.into_executor(types, []), expr, upsert=upsert))
    for n in (1, 2, 31, 32, 33, 64, 65, 1000, 4097):
        for null_frac, hidden in ((0.0, 0.0), (0.2, 0.0), (0.1, 0.3)):
            ch = random_change_chunk(rng, n, types, null_frac, hidden)
            g, o = exs[0].filter(ch), exs[1].filter(ch)
            assert (g is None) == (o is None)
            if g is not None:
                assert np.array_equal(g.vis, o.vis), f"n={n} visibility differs"
                inv = ch.vis if ch.vis is not None else np.ones(n, bool)
                assert np.array_equal(g.ops[inv], o.ops[inv]) and np.array_equal(g.ops[~inv], ch.ops[~inv])


def test_join_filter_agg_chain_on_device(cuda, oracle):
    """q4-shaped chain: bid JOIN auction ON auction = id -> WHERE bid.date_time BETWEEN auction.date_time AND
    auction.expires -> Project(auction, tumble_start(bid.date_time, 250), price * 908 / 1000) -> max(price * 908 / 1000),
    count(*) GROUP BY auction, window.  On the GPU the join output view feeds the filter kernel, rwgpu_project_device
    (the auction column by pointer, the two computed columns by the project kernel) and the agg push without leaving
    HBM; the oracle runs the same four operators on the host.  A wrong window or price changes the compared deltas:
    the agg deltas of every barrier (net multiset)."""
    import torch
    from risingwave_b200 import device
    rng = np.random.default_rng(8)
    T4 = [abi.T_INT64] * 4
    n_auc, n_bid = 5000, 20000
    auc = [np.arange(n_auc, dtype=np.int64), rng.integers(0, 1000, n_auc).astype(np.int64)]       # id, date_time
    auc.append(auc[1] + rng.integers(1, 500, n_auc)); auc.append(rng.integers(0, 10, n_auc).astype(np.int64))  # expires, category
    bid = [rng.integers(0, n_auc + 50, n_bid).astype(np.int64), np.arange(n_bid, dtype=np.int64),          # auction, bid id (stream key)
           rng.integers(0, 1500, n_bid).astype(np.int64), rng.integers(1, 10 ** 6, n_bid).astype(np.int64)]  # date_time, price
    # join output: bid cols 0..3 then auction cols 4..7
    expr = "(and:boolean (greater_than_or_equal:boolean $2:int8 $5:int8) (less_than_or_equal:boolean $2:int8 $6:int8))"
    calls = [AggCall.from_pretty(c) for c in ("(count:int8)", "(max:int8 $2:int8)")]   # over the projected (auction, window, price')
    proj_exprs = ["(tumble_start:int8 $2:int8 250:int8)", "(divide:int8 (multiply:int8 $3:int8 908:int8) 1000:int8)"]

    def make(be):
        _, sl = MockSource.channel()
        _, sr = MockSource.channel()
        j = HashJoinExecutor(be, abi.JOIN_INNER, sl.into_executor(T4, [1]), sr.into_executor(T4, [0]), JoinParams([0], [1]),
                             JoinParams([0], []), [False], capacity_hint=n_auc)
        _, sa = MockSource.channel()
        a = HashAggExecutor(be, sa.into_executor([abi.T_INT64] * 3, []), True, calls, 0, [0, 1], group_capacity_hint=4 * n_auc)
        return j, a

    jo, ao = make(oracle)
    jg, ag = make(cuda)
    _, fsrc = MockSource.channel()
    fo = FilterExecutor(oracle, fsrc.into_executor(T4 + T4, []), expr)
    po, pg = (ProjectExecutor(be, MockSource.channel()[1].into_executor(T4 + T4, []), proj_exprs) for be in (oracle, cuda))
    terms_py = parse_filter_expr(expr)
    terms = (abi.RwFilterTerm * len(terms_py))()
    for k, (cmp, lhs, rhs, const) in enumerate(terms_py):
        terms[k].cmp, terms[k].lhs_col, terms[k].rhs_col, terms[k].rhs_const = cmp, lhs, rhs, const
    ins = lambda cols: StreamChunk(np.full(len(cols[0]), abi.OP_INSERT, np.uint8), [Column(abi.T_INT64, c) for c in cols])
    assert jo.eq_join_oneside(1, ins(auc)) == []
    dev = lambda cols: device.DeviceChunk(torch.ones(len(cols[0]), dtype=torch.uint8, device="cuda"),
                                          [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in cols], T4)
    assert device.join_push_device(jg, abi.SIDE_RIGHT, dev(auc)).n_rows == 0
    B = 5000
    for e, lo in enumerate(range(0, n_bid, B)):
        part = [c[lo:lo + B] for c in bid]
        # ---- oracle: join -> filter -> project (auction id, window, price') -> agg
        for ch in jo.eq_join_oneside(0, ins(part)):
            f = fo.filter(ch)
            if f is not None:
                p = po.apply_project_exprs(f)
                ao.apply_chunk(StreamChunk(f.ops, [f.columns[0]] + p.columns, f.vis))
        want = net_multiset(ao.flush_data(e + 1))
        # ---- GPU: everything stays in HBM
        view = device.join_push_device(jg, abi.SIDE_LEFT, dev(part))
        raw = abi.RwChunk()
        cols = (abi.RwColumn * view.n_cols)()
        for k in range(view.n_cols):
            cols[k].type, cols[k].data, cols[k].validity = view.col_types[k], view.col_ptrs[k], view.valid_ptrs[k]
        raw.n_rows, raw.n_cols, raw.ops, raw.visibility, raw.columns = view.n_rows, view.n_cols, view.ops_ptr, view.vis_ptr, cols
        f_ops, f_vis, f_n = device.filter_device(raw, view.n_rows, terms)
        raw.ops, raw.visibility = f_ops.data_ptr(), f_vis.data_ptr()
        n = max(view.n_rows, 1)
        pdata = [torch.empty(n, dtype=torch.int64, device="cuda") for _ in proj_exprs]
        pvalid = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in proj_exprs]
        pnull = torch.zeros(len(proj_exprs), dtype=torch.int32, device="cuda")
        device._check(device._lib().rwgpu_project_device(C.byref(raw), pg._exprs, len(proj_exprs), (C.c_void_p * 2)(*[d.data_ptr() for d in pdata]),
                                                         (C.c_void_p * 2)(*[v.data_ptr() for v in pvalid]), C.c_void_p(pnull.data_ptr()), None))
        assert int(pnull.sum().item()) == 0  # non-negative times and prices: neither window nor price' is NULL
        proj = abi.RwChunk()
        pcols = (abi.RwColumn * 3)()
        pcols[0].type, pcols[0].data, pcols[0].validity = view.col_types[0], view.col_ptrs[0], view.valid_ptrs[0]
        for k, d in enumerate(pdata):
            pcols[k + 1].type, pcols[k + 1].data, pcols[k + 1].validity = abi.T_INT64, d.data_ptr(), None
        proj.n_rows, proj.n_cols, proj.ops, proj.visibility, proj.columns = view.n_rows, 3, f_ops.data_ptr(), f_vis.data_ptr(), pcols
        if int(f_n.item()) > 0:
            device._check(device._lib().rwgpu_agg_push_device(ag._h, C.byref(proj), None))
        got = net_multiset(ag.flush_data(e + 1))
        assert got == want, f"epoch {e}: agg deltas differ"
        assert sum(abs(v) for v in want.values()) > 0


def test_nexmark_q4_end_to_end_fixture(cuda):
    """the reference's SQL-level q4 fixture (expected rows of e2e_test/streaming/nexmark/q4.slt.part) through the
    CUDA operators: join -> filter -> agg(max, two group keys) -> agg(count, sum with retractions) -> avg"""
    run_nexmark_q4(cuda)


def test_nexmark_q7_end_to_end_fixture(cuda):
    """the reference's SQL-level q7 fixture (expected rows of e2e_test/streaming/nexmark/q7.slt.part) through the CUDA
    operators: a join whose right side is an aggregate that retracts and re-emits its maxima, then the filter"""
    run_nexmark_q7(cuda)


def test_nexmark_q8_end_to_end_fixture(cuda):
    """the reference's SQL-level q8 fixture (e2e_test/streaming/nexmark/q8.slt.part) through the CUDA operators:
    two group-by aggregates feeding a join on a three-column key"""
    run_nexmark_q8(cuda)


# ------------------------------------------------------------------------------------------ Project (round 2)
def test_project_golden_on_device(cuda):
    """project_scalar.rs test_projection through rwgpu_project: exact output chunks"""
    from test_oracle_golden import run_project_kat
    for kat in load_golden("project_kats.json"):
        run_project_kat(cuda, kat)


def test_project_expressions_match_oracle(cuda, oracle):
    """integer expressions (q1 `price * 908 / 1000`, q7 / q8 tumble windows, narrower result types) over random chunks with
    NULLs, invisible rows and overflowing operands: non-strict evaluation, row by row identical to the oracle"""
    from risingwave_b200.executor import MockSource, ProjectExecutor
    types = [abi.T_INT64, abi.T_INT64, abi.T_INT32, abi.T_TIMESTAMPTZ]
    exprs = ["(divide:int8 (multiply:int8 $0:int8 908:int8) 1000:int8)", "(tumble_start:timestamptz $3:timestamptz 10000000:int8)",
             "(tumble_end:timestamptz $3:timestamptz 10000000:int8)", "(modulus:int8 $0:int8 $1:int8)", "(subtract:int4 $2:int4 $0:int8)",
             "(add:int8 (multiply:int8 $0:int8 $1:int8) (neg:int8 $3:timestamptz))", "(divide:int8 $1:int8 $2:int4)"]
    pes = []
    for be in (cuda, oracle):
        _, src = MockSource.channel()
        pes.append(ProjectExecutor(be, src.into_executor(types, [0]), exprs))
    rng = np.random.default_rng(4)
    for n in (1, 63, 64, 65, 5000):
        a = rng.integers(-(1 << 62), 1 << 62, n) * rng.integers(0, 3, n)  # some overflow 908x, some zero
        b = rng.integers(-5, 6, n).astype(np.int64) * rng.integers(0, 1 << 33, n)
        c = rng.integers(-(1 << 31), 1 << 31, n).astype(np.int32)
        c[rng.random(n) < 0.2] = 0
        d = rng.integers(-(1 << 50), 1 << 50, n)
        cols = [Column(abi.T_INT64, a.astype(np.int64), rng.random(n) > 0.1), Column(abi.T_INT64, b, rng.random(n) > 0.1),
                Column(abi.T_INT32, c, rng.random(n) > 0.1), Column(abi.T_TIMESTAMPTZ, d.astype(np.int64), None)]
        ch = StreamChunk(rng.integers(1, 5, n).astype(np.uint8), cols, rng.random(n) > 0.05)
        g, o = (pe.apply_project_exprs(ch) for pe in pes)
        assert g == o, f"n={n}"


def test_tpch_q3_pipeline(cuda, oracle):
    """SURVEY 8(d) cfg5 (TPC-H q3 streaming plan: customer x orders x lineitem -> sum / count by (orderkey, orderdate,
    shippriority)) through the CUDA operators: the view equals the SQL evaluated directly (checked inside run_tpch_q3) and
    every barrier's delta multiset equals the oracle's.  Mixed-width payload (int64 / date / int32) keeps both joins on
    the general inner-join kernels, the aggregation on the multi-column-key path with a 128-bit sum."""
    from helpers import run_tpch_q3
    got, deltas = run_tpch_q3(cuda)
    want, want_deltas = run_tpch_q3(oracle)
    assert got == want
    assert deltas == want_deltas
    # a second size: larger chunks, more retractions in flight per epoch
    got, deltas = run_tpch_q3(cuda, n_cust=2000, n_orders=20000, n_items=80000, seed=5, epochs=4)
    want, want_deltas = run_tpch_q3(oracle, n_cust=2000, n_orders=20000, n_items=80000, seed=5, epochs=4)
    assert got == want and deltas == want_deltas
