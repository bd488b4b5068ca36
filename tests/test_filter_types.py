"""Filter at the type of every operand, on every entry point: the oracle (CPU) and rwgpu_filter / rwgpu_filter_device
(GPU) against a typed restatement of FilterExecutorInner::filter in Python.

The restatement is independent of oracle/oracle.cc and csrc/: plain Python integers and lists.  A datum is a Python int
or None for NULL: bool is 0 / 1 (false < true), int2 / int4 / date are sign-extended, time / timestamp / timestamptz /
serial are i64.  Rules:
  * signatures (src/expr/impl/src/scalar/cmp.rs): int2 / int4 / int8 compare with each other, widened (`general_lt` etc.,
    cmp.rs:44-51, 191-198); bool, serial, date, time, timestamp and timestamptz compare only with themselves
    (cmp.rs:24-160); a constant right-hand side has the left-hand side's type.  Every other pair is refused with
    RW_ERR_UNSUPPORTED and stays on the CPU FilterExecutor: float4 / float8 / decimal / varchar / bytea, and date against
    timestamp, which the reference evaluates by casting the date to midnight (cmp.rs:35-36, 124-125; DESIGN §9);
  * the predicate: each term is three-valued (a NULL operand makes it NULL), the conjunction is SQL AND, and a row passes
    only if the result is Some(true) (filter.rs:80 `res.unwrap_or(false)`);
  * the op rules: the chunk is compacted first (execute_inner, filter.rs:182), then filter.rs:82-141 apply literally to
    the compacted rows, UPSERT included, and the results are scattered back.  Invisible rows keep their input op and stay
    invisible; n_visible is the popcount and a chunk without a visible row yields no chunk (:146-150);
  * a row whose op is 0 is invisible like a cleared visibility bit (the project's fold of a dropped row, e.g. a join
    view's hole);
  * the reference only sees a U- immediately followed by its U+ (src/common/src/array/stream_chunk.rs:40-42).  For any
    other sequence this file pins the PROJECT's rule, not parity with the reference: a visible U- pairs with the next
    visible row only if that row is a U+ (and that U+ with it); an unpaired U- or U+ is filtered like a - or + and keeps
    its op.
"""
import ctypes as C
import operator

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.stream_chunk import Column, StreamChunk, pack_bits

T_OF = {"bool": abi.T_BOOL, "int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "serial": abi.T_SERIAL,
        "date": abi.T_DATE, "time": abi.T_TIME, "timestamp": abi.T_TIMESTAMP, "timestamptz": abi.T_TIMESTAMPTZ,
        "float4": abi.T_FLOAT32, "float8": abi.T_FLOAT64, "decimal": abi.T_DECIMAL, "varchar": abi.T_VARCHAR,
        "bytea": abi.T_BYTEA}
PRETTY = {"bool": "boolean"}  # build_from_pretty's name where it differs from this file's
NP_OF = {"bool": np.uint8, "int2": np.int16, "int4": np.int32, "int8": np.int64, "serial": np.int64, "date": np.int32,
         "time": np.int64, "timestamp": np.int64, "timestamptz": np.int64, "float4": np.float32, "float8": np.float64}
INTS = ("int2", "int4", "int8")
ORDERED = INTS + ("bool", "serial", "date", "time", "timestamp", "timestamptz")
ALL_TYPES = list(T_OF)
INS, DEL, UI, UD = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_INSERT, abi.OP_UPDATE_DELETE
LT, LE, GT, GE, EQ, NE = 1, 2, 3, 4, 5, 6
CMP = {LT: operator.lt, LE: operator.le, GT: operator.gt, GE: operator.ge, EQ: operator.eq, NE: operator.ne}
CMP_NAME = {LT: "less_than", LE: "less_than_or_equal", GT: "greater_than", GE: "greater_than_or_equal", EQ: "equal",
            NE: "not_equal"}
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
GRID = 132 * 8 * 256  # threads of the filter kernel's capped grid: rows of one grid-stride iteration
GARBAGE = 0xA5


class Refused(Exception):
    def __init__(self, code, what):
        super().__init__(what)
        self.code = code


# ------------------------------------------------------------------------------------------ the restatement
def signature_ok(lt, rt):
    """cmp.rs: is there a comparison function whose operands the raw integers are?"""
    if lt in INTS and rt in INTS:
        return True
    return lt == rt and lt in ORDERED


def check_plan(types, terms):
    """-> None, or raise Refused with the status the C entry points return.  terms: (cmp, lhs, rhs, const)"""
    if not 1 <= len(terms) <= 8:
        raise Refused(abi.RW_ERR_UNSUPPORTED, "1..8 terms")
    for cmp, lhs, rhs, _ in terms:
        if cmp not in CMP:
            raise Refused(abi.RW_ERR_INVALID, "comparison")
        if not 0 <= lhs < len(types) or not -1 <= rhs < len(types):
            raise Refused(abi.RW_ERR_INVALID, "column index")
        if not signature_ok(types[lhs], types[rhs] if rhs >= 0 else types[lhs]):
            raise Refused(abi.RW_ERR_UNSUPPORTED, "operand types")


def term_value(term, vals, r):
    """Option<bool> of one comparison"""
    cmp, lhs, rhs, const = term
    a, b = vals[lhs][r], (vals[rhs][r] if rhs >= 0 else const)
    if a is None or b is None:
        return None
    return CMP[cmp](a, b)


def predicate(terms, vals, r):
    """SQL AND of the terms: FALSE if any term is FALSE, else NULL if any is NULL, else TRUE"""
    out = True
    for t in terms:
        v = term_value(t, vals, r)
        if v is False:
            return False
        if v is None:
            out = None
    return out


def restate(ops, vis, types, vals, terms, upsert):
    """-> (ops, visibility as bool list, n_visible); ops and vis of invisible rows are the input's"""
    check_plan(types, terms)
    n = len(ops)
    pos = [r for r in range(n) if ops[r] != 0 and (vis is None or vis[r])]  # compact_vis (+ op 0 = invisible)
    res = [predicate(terms, vals, r) is True for r in pos]                # unwrap_or(false)
    new_ops, new_vis = [], []
    i = 0
    while i < len(pos):
        op = ops[pos[i]]
        if upsert:  # filter.rs:82-106
            new_ops.append(INS if op in (INS, UI) and res[i] else DEL)
            new_vis.append(True)
        elif op == UD and i + 1 < len(pos) and ops[pos[i + 1]] == UI:  # filter.rs:112-141, one pair
            last_res, r2 = res[i], res[i + 1]
            new_ops += {(True, False): [DEL, UI], (False, True): [UD, INS]}.get((last_res, r2), [UD, UI])
            new_vis += [last_res, r2]
            i += 1
        else:  # + / - (filter.rs:108-111); an unpaired U- / U+ by the project's rule
            new_ops.append(op)
            new_vis.append(res[i])
        i += 1
    out_ops, out_vis = [int(o) for o in ops], [False] * n
    for k, r in enumerate(pos):
        out_ops[r], out_vis[r] = new_ops[k], new_vis[k]
    return out_ops, out_vis, sum(out_vis)


# ------------------------------------------------------------------------------------------ values
def days_from_civil(y, m, d):
    """proleptic Gregorian date -> days since 1970-01-01"""
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + doy - 719468


DAY_US = 86_400_000_000
D_LO, D_HI = days_from_civil(-262000, 1, 1), days_from_civil(262000, 12, 31)  # inside chrono's NaiveDate range
SERIAL_IDS = [I64_MIN, I64_MIN | 1, I64_MIN | (0x2aa << 12), -1 << 40, (0x155 << 12) | 0x7f, 1 << 62, I64_MAX]


def edges(t):
    if t == "bool":
        return [0, 1]
    if t == "time":
        return [0, 1, 2, 43_200_000_000, DAY_US - 2, DAY_US - 1]
    if t == "date":
        return [D_LO, D_LO + 1, -1, 0, 1, D_HI - 1, D_HI]
    if t == "timestamp":
        lo, hi = D_LO * DAY_US, D_HI * DAY_US + DAY_US - 1
        return [lo, lo + 1, -1, 0, 1, hi - 1, hi]
    if t == "serial":
        return SERIAL_IDS + [0, 1]
    b = {"int2": 16, "int4": 32}.get(t, 64)
    lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
    return [lo, lo + 1, -1, 0, 1, hi - 1, hi]


def const_edges(t):
    """constants against a column of type t: its own edges, and i64 extremes against the narrow integers"""
    return edges(t) + ([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1] if t in ("int2", "int4") else [])


class Col:
    """a column: type name, numpy data in the ABI's native width, valid (bool[n]) or None"""

    def __init__(self, t, data, valid=None):
        self.t, self.data, self.valid = t, data, valid

    def values(self):
        raw = [int(x) for x in self.data]
        return raw if self.valid is None else [v if ok else None for v, ok in zip(raw, self.valid)]


def make_col(rng, t, n, null_frac):
    pool = np.array(edges(t), dtype=NP_OF[t])
    data = pool[rng.integers(0, len(pool), n)]
    lo, hi = min(edges(t)), max(edges(t))
    rnd = rng.random(n) < 0.3
    data[rnd] = rng.integers(lo, hi, int(rnd.sum()), endpoint=True, dtype=np.int64).astype(NP_OF[t])
    return Col(t, data, rng.random(n) >= null_frac if null_frac else None)


COMPARED = list(ORDERED)  # one column of every accepted type, then an uncompared float8
SCHEMA = COMPARED + ["float8"]


def random_terms(rng, n_terms, types=SCHEMA):
    terms = []
    for _ in range(n_terms):
        lhs = int(rng.integers(0, len(COMPARED)))
        cmp = int(rng.integers(1, 7))
        x = rng.random()
        if x < 0.45:
            pool = const_edges(types[lhs])
            terms.append((cmp, lhs, -1, pool[int(rng.integers(0, len(pool)))]))
        elif x < 0.55:
            terms.append((cmp, lhs, lhs, 0))  # a column against itself
        else:
            ok = [k for k in range(len(COMPARED)) if signature_ok(types[lhs], types[k])]
            terms.append((cmp, lhs, ok[int(rng.integers(0, len(ok)))], 0))
    return terms


def random_ops(rng, n, op0_frac=0.05):
    """+, -, adjacent U-/U+ pairs, a few unpaired U- / U+ and some op 0 rows"""
    ops = np.zeros(n, np.uint8)
    i = 0
    while i < n:
        x = rng.random()
        if x < 0.3 and i + 1 < n:
            ops[i], ops[i + 1] = UD, UI
            i += 2
            continue
        ops[i] = INS if x < 0.65 else DEL if x < 0.9 else UD if x < 0.94 else UI if x < 0.98 else 0
        i += 1
    ops[rng.random(n) < op0_frac] = 0
    return ops


def place_pairs(rng, ops, vis, boundaries):
    """a visible U- before each boundary and its U+ after it, 0..100 invisible rows between them (cleared bits or op 0)"""
    n = len(ops)
    for b in boundaries:
        gap = int(rng.integers(0, 101))
        before = int(rng.integers(0, gap + 1)) if gap else 0
        lo = b - 1 - before
        hi = lo + gap + 1
        if lo < 0 or hi >= n:
            continue
        ops[lo], ops[hi], vis[lo], vis[hi] = UD, UI, True, True
        for r in range(lo + 1, hi):
            if rng.random() < 0.5:
                vis[r] = False
            else:
                ops[r] = 0


def boundaries_of(n):
    out = [32 * k for k in range(1, 4)] + [64, 128, 256, 512, 768] + [GRID * k for k in range(1, 5)]
    return [b for b in out if b < n]


def make_case(seed, n, n_terms=None, null_frac=0.1, vis_frac=0.9, types=SCHEMA):
    rng = np.random.default_rng(seed)
    cols = [make_col(rng, t, n, null_frac) if t in NP_OF and t not in ("float4", "float8") else
            Col(t, rng.standard_normal(n).astype(NP_OF[t])) for t in types]
    ops = random_ops(rng, n)
    vis = rng.random(n) < vis_frac
    place_pairs(rng, ops, vis, boundaries_of(n))
    terms = random_terms(rng, n_terms if n_terms is not None else [1, 1, 1, 2, 2, 3, 5, 8][int(rng.integers(0, 8))], types)
    return ops, cols, vis, terms


def expected(ops, cols, vis, terms, upsert):
    vals = [c.values() if c.t in ORDERED else None for c in cols]
    return restate(list(ops), None if vis is None else list(vis), [c.t for c in cols], vals, terms, upsert)


# ------------------------------------------------------------------------------------------ calling the entry points
def term_array(terms):
    arr = (abi.RwFilterTerm * max(1, len(terms)))()
    for k, (cmp, lhs, rhs, const) in enumerate(terms):
        arr[k].cmp, arr[k].lhs_col, arr[k].rhs_col, arr[k].rhs_const = cmp, lhs, rhs, const
    return arr


def host_abi(ops, cols, vis):
    """an rw_chunk of HOST pointers -> (chunk, keepalive); varlen columns carry empty values"""
    n, keep = len(ops), []

    def put(a):
        a = np.ascontiguousarray(a)
        keep.append(a)
        return a.ctypes.data
    arr = (abi.RwColumn * max(1, len(cols)))()
    for k, c in enumerate(cols):
        arr[k].type = T_OF[c.t]
        if c.t in ("varchar", "bytea"):
            arr[k].data, arr[k].offsets = put(np.zeros(8, np.uint8)), put(np.zeros(n + 1, np.uint32))
        else:
            arr[k].data = put(c.data) if n else None
        arr[k].validity = put(pack_bits(c.valid)) if c.valid is not None else None
    ch = abi.RwChunk()
    ch.n_rows, ch.n_cols = n, len(cols)
    ch.ops = put(np.asarray(ops, np.uint8)) if n else None
    ch.visibility = put(pack_bits(vis)) if vis is not None else None
    ch.columns = arr
    keep.append(arr)
    return ch, keep


def call_host(fn, ops, cols, vis, terms, upsert):
    """rwo_filter / rwgpu_filter with every output pre-filled with garbage and one guard word / byte past its end
    -> (rc, ops, visibility words, n_visible)"""
    n = len(ops)
    ch, keep = host_abi(ops, cols, vis)
    nw = (n + 63) // 64
    out_ops = np.full(n + 8, GARBAGE, np.uint8)
    out_vis = np.full((nw + 1) * 8, GARBAGE, np.uint8).view(np.uint64)
    nvis = C.c_int64(int(np.full(1, GARBAGE, np.uint8).repeat(8).view(np.int64)[0]))
    rc = fn(C.byref(ch), term_array(terms), len(terms), int(upsert), out_ops.ctypes.data_as(C.POINTER(C.c_uint8)),
            out_vis.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(nvis))
    if rc == abi.RW_OK:
        assert (out_ops[n:] == GARBAGE).all(), "wrote past out_ops[n_rows]"
        assert out_vis[nw] == np.full(8, GARBAGE, np.uint8).view(np.uint64)[0], "wrote past the visibility words"
    return rc, out_ops[:n], out_vis[:nw], nvis.value


def assert_output(what, got, want, n):
    rc, ops, words, nvis = got
    want_ops, want_vis, want_n = want
    assert rc == abi.RW_OK, f"{what}: status {rc}"
    bad = np.nonzero(ops != np.array(want_ops, np.uint8))[0]
    assert not len(bad), f"{what}: op of row {bad[0]} is {ops[bad[0]]}, want {want_ops[bad[0]]} ({len(bad)} rows differ)"
    want_words = pack_bits(np.array(want_vis, bool))[:(n + 63) // 64]
    bad = np.nonzero(words != want_words)[0]
    assert not len(bad), f"{what}: visibility word {bad[0]} is {int(words[bad[0]]):#x}, want {int(want_words[bad[0]]):#x}"
    assert nvis == want_n, f"{what}: n_visible {nvis}, want {want_n}"


def oracle_fn(oracle):
    return oracle.lib.rwo_filter


# ------------------------------------------------------------------------------------------ the restatement's own checks
def test_restatement_reproduces_the_reference_tests():
    """filter.rs:208 test_filter and the upsert test (tests/golden/filter_kats.json), with the I columns as int8"""
    from helpers import load_golden
    for kat in load_golden("filter_kats.json"):
        from risingwave_b200.executor import parse_filter_expr
        terms = parse_filter_expr(kat["expr"])
        for inp, exp in zip(kat["inputs"], kat["expected"]):
            ch, want = StreamChunk.from_pretty(inp), StreamChunk.from_pretty(exp)
            cols = [Col("int8", c.data, c.valid) for c in ch.columns]
            ops, vis, n = expected(ch.ops, cols, ch.vis, terms, kat["upsert"])
            want_vis = want.vis if want.vis is not None else np.ones(len(ops), bool)
            assert ops == [int(o) for o in want.ops] and vis == list(want_vis) and n == int(want_vis.sum()), kat["name"]


def test_restatement_pins_the_projects_rules():
    t = [(LT, 0, -1, 7)]
    # U- + U+ over 5, 9, 5: the U- and the U+ are not adjacent, so each is filtered on its own and keeps its op
    assert expected([UD, INS, UI], [Col("int8", np.array([5, 9, 5]))], None, t, False) == ([UD, INS, UI], [True, False, True], 2)
    # a row with op 0 is invisible: it keeps op 0, and the U- / U+ around it still pair
    assert expected([UD, 0, UI], [Col("int8", np.array([5, 5, 9]))], None, t, False) == ([DEL, 0, UI], [True, False, False], 1)
    assert expected([0, INS], [Col("int8", np.array([5, 5]))], None, t, False) == ([0, INS], [False, True], 1)
    # NULL before / after FALSE is FALSE; NULL with TRUE is NULL: all three filter the row out
    c = [Col("int8", np.array([1]), np.array([False])), Col("int8", np.array([1]))]
    for terms in ([(EQ, 0, 1, 0), (GT, 1, -1, 5)], [(GT, 1, -1, 5), (EQ, 0, 1, 0)], [(EQ, 0, 1, 0), (LT, 1, -1, 5)]):
        assert expected([INS], c, None, terms, False) == ([INS], [False], 0)
    assert expected([INS], c, None, [(LT, 1, -1, 5), (NE, 1, 1, 0)], False) == ([INS], [False], 0)
    assert expected([INS], c, None, [(LT, 1, -1, 5), (EQ, 1, 1, 0)], False) == ([INS], [True], 1)
    # UPSERT: every visible row stays visible, - / U- become -, + / U+ become + or -
    assert expected([UD, UI, DEL, INS], [Col("int8", np.array([9, 5, 5, 9]))], None, t, True) == ([DEL, INS, DEL, DEL], [True] * 4, 4)
    # the signatures: narrow integers against an i64 constant compare widened, mixed non-integer pairs are refused
    assert expected([INS, INS], [Col("int2", np.array([-32768, 32767], np.int16))], None, [(GT, 0, -1, I64_MIN)], False)[2] == 2
    for lt, rt in (("date", "timestamptz"), ("date", "timestamp"), ("bool", "int8"), ("time", "int8"), ("serial", "int8")):
        with pytest.raises(Refused):
            check_plan([lt, rt], [(LT, 0, 1, 0)])
    check_plan(["timestamp", "timestamp"], [(LT, 0, 1, 0)])


# ------------------------------------------------------------------------------------------ checks shared by both backends
SMALL_SIZES = [0, 1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000]
LARGE_SIZES = [GRID - 1, GRID, GRID + 1, GRID + 33, 1_100_003]


def refusal_cases():
    """-> [(name, types, terms, expected status)]"""
    ok = [(LT, 0, -1, 0)]
    out = [("0 terms", ["int8"], [], abi.RW_ERR_UNSUPPORTED), ("9 terms", ["int8"], ok * 9, abi.RW_ERR_UNSUPPORTED),
           ("cmp 0", ["int8"], [(0, 0, -1, 0)], abi.RW_ERR_INVALID), ("cmp 7", ["int8"], [(7, 0, -1, 0)], abi.RW_ERR_INVALID),
           ("lhs -1", ["int8"], [(LT, -1, -1, 0)], abi.RW_ERR_INVALID), ("lhs n_cols", ["int8"], [(LT, 1, -1, 0)], abi.RW_ERR_INVALID),
           ("rhs n_cols", ["int8"], [(LT, 0, 1, 0)], abi.RW_ERR_INVALID), ("rhs -2", ["int8"], [(LT, 0, -2, 0)], abi.RW_ERR_INVALID),
           ("bad cmp after a good term", ["int8"], ok + [(9, 0, -1, 0)], abi.RW_ERR_INVALID)]
    for lt in ALL_TYPES:
        if lt not in ORDERED:
            out.append((f"{lt} vs constant", [lt], ok, abi.RW_ERR_UNSUPPORTED))
        for rt in ALL_TYPES:
            if not signature_ok(lt, rt):
                out.append((f"{lt} vs {rt}", [lt, rt], [(EQ, 1, 1, 0), (GE, 0, 1, 0)], abi.RW_ERR_UNSUPPORTED))
    return out


def refusal_chunk(types):
    cols = [Col(t, np.array(edges(t)[:3], NP_OF[t])) if t in ORDERED else Col(t, np.zeros(3, NP_OF[t])) if t in NP_OF else
            Col(t, None) for t in types]
    return np.full(3, INS, np.uint8), cols, np.ones(3, bool)


def check_refusals(fn):
    for name, types, terms, code in refusal_cases():
        if all(t in ORDERED for t in types):
            with pytest.raises(Refused) as ei:
                check_plan(types, terms)
            assert ei.value.code == code, name
        ops, cols, vis = refusal_chunk(types)
        rc = call_host(fn, ops, cols, vis, terms, False)[0]
        assert rc == code, f"{name}: status {rc}, want {code}"
    # null pointers
    ops, cols, vis = refusal_chunk(["int8"])
    ch, keep = host_abi(ops, cols, vis)
    o, w = np.zeros(8, np.uint8), np.zeros(1, np.uint64)
    po, pw = o.ctypes.data_as(C.POINTER(C.c_uint8)), w.ctypes.data_as(C.POINTER(C.c_uint64))
    t = term_array([(LT, 0, -1, 0)])
    for args in ((None, t, 1, 0, po, pw, None), (C.byref(ch), None, 1, 0, po, pw, None), (C.byref(ch), t, 1, 0, None, pw, None),
                 (C.byref(ch), t, 1, 0, po, None, None)):
        assert fn(*args) == abi.RW_ERR_INVALID
    assert fn(C.byref(ch), t, 1, 0, po, pw, None) == abi.RW_OK  # n_visible may be NULL


def check_signatures(fn):
    """every accepted pair of column types and every accepted column type against constants, at its edges"""
    rng = np.random.default_rng(7)
    for lt in ORDERED:
        for rt in ORDERED:
            if not signature_ok(lt, rt):
                continue
            a, b = edges(lt), edges(rt)
            # every edge of one side against every edge of the other, a NULL on each side and on both
            la = [x for x in a for _ in b] + [a[0], None, None]
            lb = [y for _ in a for y in b] + [None, b[0], None]
            cols = [Col(lt, np.array([0 if v is None else v for v in la], NP_OF[lt]), np.array([v is not None for v in la])),
                    Col(rt, np.array([0 if v is None else v for v in lb], NP_OF[rt]), np.array([v is not None for v in lb]))]
            n = len(la)
            for cmp in CMP:
                ops = random_ops(rng, n, 0.0)
                for upsert in (False, True):
                    terms = [(cmp, 0, 1, 0)]
                    assert_output(f"{lt} {CMP_NAME[cmp]} {rt}", call_host(fn, ops, cols, None, terms, upsert),
                                  expected(ops, cols, None, terms, upsert), n)
        pool = const_edges(lt)
        col = Col(lt, np.array(edges(lt) + [0], NP_OF[lt]), np.array([True] * len(edges(lt)) + [False]))
        for cmp in CMP:
            for k in pool:
                terms = [(cmp, 0, -1, k)]
                ops = np.full(len(col.data), INS, np.uint8)
                assert_output(f"{lt} {CMP_NAME[cmp]} {k}", call_host(fn, ops, [col], None, terms, False),
                              expected(ops, [col], None, terms, False), len(ops))


def check_case(fn, seed, n, upsert, **kw):
    ops, cols, vis, terms = make_case(seed, n, **kw)
    assert_output(f"n={n} seed={seed} upsert={upsert} terms={terms}", call_host(fn, ops, cols, vis, terms, upsert),
                  expected(ops, cols, vis, terms, upsert), n)


def check_shapes(fn, sizes):
    for i, n in enumerate(sizes):
        for upsert in (False, True):
            check_case(fn, 100 + i, n, upsert)
            check_case(fn, 200 + i, n, upsert, vis_frac=0.0)               # fully invisible
            check_case(fn, 300 + i, n, upsert, n_terms=8, null_frac=0.6)   # nothing or almost nothing survives
            check_case(fn, 400 + i, n, upsert, null_frac=0.0, n_terms=1)


def check_invisible_runs(fn):
    """a visible U- and its U+ with 0..100 invisible rows between them, every combination of the pair's two results"""
    for gap in list(range(0, 12)) + [31, 32, 33, 63, 64, 65, 99, 100]:
        for kind in ("bits", "op0", "mixed"):
            n = gap + 4
            ops = np.full(n, INS, np.uint8)
            vis = np.ones(n, bool)
            ops[1], ops[gap + 2] = UD, UI
            for r in range(2, gap + 2):
                if kind == "bits" or (kind == "mixed" and r % 2):
                    vis[r] = False
                    ops[r] = [INS, DEL, UD, UI][r % 4]
                else:
                    ops[r] = 0
            for a in (3, 9):
                for b in (3, 9):
                    x = np.full(n, 5, np.int64)
                    x[1], x[gap + 2] = a, b
                    cols = [Col("int8", x)]
                    for upsert in (False, True):
                        assert_output(f"gap {gap} {kind} ({a}, {b})", call_host(fn, ops, cols, vis, [(LT, 0, -1, 7)], upsert),
                                      expected(ops, cols, vis, [(LT, 0, -1, 7)], upsert), n)


def check_unpaired(fn):
    """sequences the reference never sees: the project's pairing rule"""
    seqs = [[UD, INS, UI], [UD, DEL, UI], [UD, UD, UI, UI], [UI, UD], [UD], [UI], [UD, UI, UI], [UD, UD, UI], [UI, UI, UD, UD],
            [UD, 0, 0, UI], [0, UD, UI, 0]]
    for seq in seqs:
        n = len(seq)
        for bits in range(1 << n):
            x = np.array([3 if (bits >> i) & 1 else 9 for i in range(n)], np.int64)
            for upsert in (False, True):
                ops = np.array(seq, np.uint8)
                assert_output(f"{seq} {bits:b}", call_host(fn, ops, [Col("int8", x)], None, [(LT, 0, -1, 7)], upsert),
                              expected(ops, [Col("int8", x)], None, [(LT, 0, -1, 7)], upsert), n)


# ------------------------------------------------------------------------------------------ CPU: the oracle
def test_oracle_signatures_match_restatement(oracle):
    check_signatures(oracle_fn(oracle))


def test_oracle_refuses_what_the_restatement_refuses(oracle):
    check_refusals(oracle_fn(oracle))


def test_oracle_shapes_match_restatement(oracle):
    check_shapes(oracle_fn(oracle), SMALL_SIZES + [4097])


def test_oracle_invisible_runs_between_a_pair(oracle):
    check_invisible_runs(oracle_fn(oracle))


def test_oracle_unpaired_updates_follow_the_projects_rule(oracle):
    check_unpaired(oracle_fn(oracle))


def test_oracle_op0_rows_are_invisible(oracle):
    """a visible row with op 0 used to be read as a U+ (and [op 0, +] as a U- without its U+)"""
    ops = np.array([0, INS, UD, 0, UI, 0], np.uint8)
    cols = [Col("int8", np.array([5, 5, 5, 5, 9, 5]))]
    assert_output("op 0", call_host(oracle_fn(oracle), ops, cols, None, [(LT, 0, -1, 7)], False),
                  ([0, INS, DEL, 0, UI, 0], [False, True, True, False, False, False], 2), len(ops))


def pretty_expr(terms, types):
    def one(cmp, lhs, rhs, const):
        lt = PRETTY.get(types[lhs], types[lhs])
        r = f"${rhs}:{PRETTY.get(types[rhs], types[rhs])}" if rhs >= 0 else f"{const}:{lt}"
        return f"({CMP_NAME[cmp]}:boolean ${lhs}:{lt} {r})"
    out = one(*terms[-1])
    for t in reversed(terms[:-1]):
        out = f"(and:boolean {one(*t)} {out})"
    return out


@pytest.mark.parametrize("upsert", [False, True])
def test_filter_executor_matches_restatement(oracle, upsert):
    """FilterExecutor over the oracle: the build_from_pretty text of the terms, every accepted type in the schema"""
    from risingwave_b200.executor import FilterExecutor, MockSource
    for seed, n in enumerate([1, 33, 64, 257, 1000]):
        ops, cols, vis, terms = make_case(seed, n)
        ops[ops == 0] = INS  # a host StreamChunk carries ops 1..4
        _, src = MockSource.channel()
        ex = FilterExecutor(oracle, src.into_executor([T_OF[c.t] for c in cols], []), pretty_expr(terms, SCHEMA), upsert=upsert)
        got = ex.filter(StreamChunk(ops, [Column(T_OF[c.t], c.data, c.valid) for c in cols], vis))
        want_ops, want_vis, want_n = expected(ops, cols, vis, terms, upsert)
        if want_n == 0:
            assert got is None
            continue
        assert list(got.ops) == want_ops and list(got.vis) == want_vis, f"seed {seed}"


@pytest.mark.parametrize("expr,why", [
    ("(less_than:boolean $0:varchar 7:date)", "operand"),
    ("(less_than:boolean $0:int4 7:int8)", "operand"),
    ("(less_than:boolean $1:timestamptz $1:timestamptz)", "operand"),
    ("(less_than:boolean $0:int8 $5:int8)", "operand"),
    ("(and:boolean (less_than:boolean $0:int8 1:int8) (greater_than:boolean $2:int8 7:timestamptz))", "operand"),
    ("(less_than:boolean $2:timestamptz 7:int8)", "constant"),
    ("(less_than:boolean $3:date 7:timestamp)", "constant"),
    ("(less_than:boolean $0:int8 7:boolean)", "constant"),
])
def test_filter_executor_checks_annotations(oracle, expr, why):
    from risingwave_b200.executor import FilterExecutor, MockSource
    _, src = MockSource.channel()
    types = [abi.T_INT64, abi.T_TIMESTAMP, abi.T_TIMESTAMPTZ, abi.T_DATE]
    with pytest.raises(ValueError, match=why):
        FilterExecutor(oracle, src.into_executor(types, []), expr)


def test_filter_executor_accepts_matching_annotations(oracle):
    from risingwave_b200.executor import FilterExecutor, MockSource, parse_filter_expr
    types = [abi.T_INT16, abi.T_TIMESTAMP, abi.T_TIMESTAMPTZ, abi.T_DATE]
    expr = ("(and:boolean (less_than:boolean $0:int2 -9223372036854775808:int8) (and:boolean (greater_than:boolean $1:timestamp "
            "$1:timestamp) (equal:boolean $3:date 3:date)))")
    _, src = MockSource.channel()
    FilterExecutor(oracle, src.into_executor(types, []), expr)
    assert parse_filter_expr(expr) == [(LT, 0, -1, I64_MIN), (GT, 1, 1, 0), (EQ, 3, -1, 3)]


# ------------------------------------------------------------------------------------------ GPU: rwgpu_filter (host chunks)
def cuda_fn(cuda):
    lib = cuda.lib
    lib.rwgpu_filter.restype = C.c_int32
    return lib.rwgpu_filter


@pytest.mark.gpu
def test_device_signatures_match_restatement(cuda):
    check_signatures(cuda_fn(cuda))


@pytest.mark.gpu
def test_device_refuses_what_the_oracle_refuses(cuda, oracle):
    check_refusals(cuda_fn(cuda))


@pytest.mark.gpu
def test_device_small_shapes_match_restatement(cuda):
    check_shapes(cuda_fn(cuda), SMALL_SIZES + [4097])


@pytest.mark.gpu
def test_device_invisible_runs_between_a_pair(cuda):
    check_invisible_runs(cuda_fn(cuda))


@pytest.mark.gpu
def test_device_unpaired_updates_follow_the_projects_rule(cuda):
    check_unpaired(cuda_fn(cuda))


@pytest.mark.gpu
@pytest.mark.parametrize("n", LARGE_SIZES)
def test_device_grid_stride_shapes_match_restatement(cuda, n):
    """chunks past one grid-stride iteration of the capped grid, pairs straddling each iteration's end"""
    for upsert in (False, True):
        check_case(cuda_fn(cuda), n, n, upsert, n_terms=2)


# ------------------------------------------------------------------------------------------ GPU: rwgpu_filter_device
def _d_lib():
    from risingwave_b200 import device
    return device._lib()


def call_device(chunk_abi, n, terms, upsert, alias=None):
    """rwgpu_filter_device with garbage-filled DEVICE outputs (a guard byte / word past each) -> like call_host"""
    import torch
    nw = (n + 63) // 64
    out_ops = torch.full((n + 8,), GARBAGE, dtype=torch.uint8, device="cuda")
    out_vis = torch.full(((nw + 1) * 8,), GARBAGE, dtype=torch.uint8, device="cuda")
    nvis = torch.full((8,), GARBAGE, dtype=torch.uint8, device="cuda")
    po, pv = out_ops.data_ptr(), out_vis.data_ptr()
    if alias == "ops":
        po = chunk_abi.ops
    elif alias == "vis":
        pv = chunk_abi.visibility
    rc = _d_lib().rwgpu_filter_device(C.byref(chunk_abi), term_array(terms), len(terms), int(upsert), C.c_void_p(po),
                                      C.c_void_p(pv), C.c_void_p(nvis.data_ptr()), None)
    torch.cuda.synchronize()
    ops, words = out_ops.cpu().numpy(), out_vis.cpu().numpy().view(np.uint64)
    if rc == abi.RW_OK:
        assert (ops[n:] == GARBAGE).all(), "wrote past out_ops[n_rows]"
        assert words[nw] == np.full(8, GARBAGE, np.uint8).view(np.uint64)[0], "wrote past the visibility words"
    return rc, ops[:n], words[:nw], int(nvis.cpu().numpy().view(np.int64)[0])


def dev_abi(ops, cols, vis):
    """an rw_chunk of DEVICE pointers -> (chunk, keepalive)"""
    import torch
    n, keep = len(ops), []

    def put(a):
        t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
        keep.append(t)
        return t.data_ptr()
    arr = (abi.RwColumn * max(1, len(cols)))()
    for k, c in enumerate(cols):
        arr[k].type = T_OF[c.t]
        arr[k].data = put(c.data) if n else None
        arr[k].validity = put(pack_bits(c.valid)) if c.valid is not None else None
    ch = abi.RwChunk()
    ch.n_rows, ch.n_cols = n, len(cols)
    ch.ops = put(np.asarray(ops, np.uint8)) if n else None
    ch.visibility = put(pack_bits(vis)) if vis is not None else None
    ch.columns = arr
    keep.append(arr)
    return ch, keep


@pytest.mark.gpu
@pytest.mark.parametrize("n", SMALL_SIZES + LARGE_SIZES)
def test_filter_device_matches_restatement(cuda, n):
    """rwgpu_filter_device on a device chunk: every op byte, every visibility word (the bits past n_rows zero, the upper
    half of a last odd 32-bit word cleared by the kernel) and the device count"""
    for upsert in (False, True):
        for seed, kw in ((n, {}), (n + 1, {"vis_frac": 0.0}), (n + 2, {"null_frac": 0.0, "n_terms": 1})):
            if n > 100_000 and seed == n + 2:
                continue
            ops, cols, vis, terms = make_case(seed, n, **kw)
            ch, keep = dev_abi(ops, cols, vis)
            assert_output(f"n={n} upsert={upsert} seed={seed}", call_device(ch, n, terms, upsert),
                          expected(ops, cols, vis, terms, upsert), n)


@pytest.mark.gpu
def test_filter_device_refuses_aliased_outputs_and_what_the_oracle_refuses(cuda):
    ops, cols, vis, terms = make_case(3, 100, n_terms=2)
    ch, keep = dev_abi(ops, cols, vis)
    for alias in ("ops", "vis"):
        assert call_device(ch, 100, terms, False, alias)[0] == abi.RW_ERR_INVALID, alias
    for name, types, terms_, code in refusal_cases():
        rops, rcols, rvis = refusal_chunk(types)
        rcols = [c if c.data is not None else Col(c.t, np.zeros(3, np.int64)) for c in rcols]  # varlen: 8-byte handles
        rch, rkeep = dev_abi(rops, rcols, rvis)
        assert call_device(rch, 3, terms_, False)[0] == code, name


def join_view(cuda, plan):
    """an inner join pushed left rows with op 0 and keys without a match (holes in a positional view).  plan "uni" takes the
    unified-table plan (eight-byte columns: the view's left columns alias the pushed chunk), "fused" the fused kernel (an
    int4 payload column)"""
    import torch
    from risingwave_b200 import device
    from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
    lt = ["int8", "int8", "timestamp", "int8"] if plan == "uni" else ["int8", "int8", "timestamp", "int4"]
    rt = ["int8", "int8", "timestamp", "int8"]
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    ex = HashJoinExecutor(cuda, abi.JOIN_INNER, sl.into_executor([T_OF[t] for t in lt], [1]),
                          sr.into_executor([T_OF[t] for t in rt], [0]), JoinParams([0], [1]), JoinParams([0], []), [False],
                          capacity_hint=4096)
    rng = np.random.default_rng(11)
    n_r, n_l = 3000, 20000

    def dev(ops, data, types):
        return device.DeviceChunk(torch.from_numpy(ops).cuda(), [torch.from_numpy(np.ascontiguousarray(d)).cuda() for d in data],
                                  [T_OF[t] for t in types])
    right = [np.arange(n_r, dtype=np.int64), rng.integers(-50, 50, n_r), rng.integers(-10 ** 6, 10 ** 6, n_r),
             rng.integers(-5, 5, n_r)]
    assert device.join_push_device(ex, abi.SIDE_RIGHT, dev(np.full(n_r, INS, np.uint8), right, rt)).n_rows == 0
    ops = np.full(n_l, INS, np.uint8)
    ops[rng.random(n_l) < 0.1] = 0
    left = [rng.integers(0, n_r + 300, n_l), np.arange(n_l, dtype=np.int64), rng.integers(-10 ** 6, 10 ** 6, n_l),
            rng.integers(-50, 50, n_l).astype(np.int64 if plan == "uni" else np.int32)]
    chunk = dev(ops, left, lt)
    view = device.join_push_device(ex, abi.SIDE_LEFT, chunk)
    return ex, chunk, view, lt + rt


@pytest.mark.gpu
@pytest.mark.parametrize("plan", ["uni", "fused"])
def test_filter_device_on_a_join_view(cuda, plan):
    """rwgpu_filter_device on the view a join push returned: holes, columns aliasing the pushed chunk, timestamp
    against timestamp (the Nexmark date_time columns) and the narrow join column against the other side's int8"""
    from risingwave_b200 import device
    ex, chunk, view, types = join_view(cuda, plan)
    n = view.n_rows
    assert n > 0
    vis = view.visible()
    vis = None if vis is None else vis.cpu().numpy()
    ops = view.ops().cpu().numpy()
    cols = []
    for k, t in enumerate(types):
        valid = None
        if view.valid_ptrs[k]:
            import torch
            words = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda")
            device._d2d(words.data_ptr(), view.valid_ptrs[k], words.numel() * 8)
            valid = np.unpackbits(words.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
        cols.append(Col(t, view.column(k).cpu().numpy().astype(NP_OF[t]), valid))
    if plan == "uni":  # positional output: a dropped or unmatched input row leaves a hole (the fused kernel compacts)
        assert (vis is not None and not vis.all()) or (ops == 0).any(), "the view has no holes"
        assert all(view.col_ptrs[k] == chunk.cols[k].data_ptr() for k in range(4)), "the view's left columns are copies"
    raw = abi.RwChunk()
    arr = (abi.RwColumn * view.n_cols)()
    for k in range(view.n_cols):
        arr[k].type, arr[k].data, arr[k].validity = view.col_types[k], view.col_ptrs[k], view.valid_ptrs[k]
    raw.n_rows, raw.n_cols, raw.ops, raw.visibility, raw.columns = n, view.n_cols, view.ops_ptr, view.vis_ptr, arr
    term_sets = [[(LE, 2, 6, 0)], [(GT, 3, 5, 0), (GE, 2, -1, 0)], [(NE, 3, -1, 7), (LT, 6, 2, 0), (EQ, 0, 4, 0)]]
    for terms in term_sets:
        for upsert in (False, True):
            assert_output(f"{plan} {terms} upsert={upsert}", call_device(raw, n, terms, upsert),
                          expected(ops, cols, vis, terms, upsert), n)
    assert call_device(raw, n, term_sets[0], False, "ops")[0] == abi.RW_ERR_INVALID
