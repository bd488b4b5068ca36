"""Project at the type of every operation: the oracle (CPU) and both device entry points (GPU) against a typed
restatement of the reference in Python integers.

The restatement is independent of oracle/oracle.cc and csrc/chain.cu:
  * a leaf is a column value (NULL stays NULL; a narrower column is sign-extended) or a constant;
  * an operation of result type T (int2 / int4 / int8, or a timestamp type for tumble_*) is a `checked_*` op of the
    Rust integer type T, its operands widened `Into<T>` first (src/expr/impl/src/scalar/arithmetic_op.rs:30-114
    `general_add` .. `general_mod`, `general_neg`):
    add / subtract / multiply / divide / neg give NULL when the exact result lies outside T, divide and modulus give
    NULL for a zero divisor, and modulus gives NULL for MIN(T) % -1 (`checked_rem`, :98-107) although its result, 0,
    fits T;
  * tumble_start(ts, w) (src/expr/impl/src/scalar/tumble.rs:34-112): a DATE is the timestamp of its midnight
    (days since 1970-01-01 x 86 400 000 000 us, :34-37), w == 0 is NULL, else ts - (r < 0 ? r + w : r) with
    r = ts rem w, NULL outside i64; tumble_end = that start + w, checked at i64;
  * the row's value is NULL at the first failure or NULL operand (NonStrictExpression::eval_infallible,
    src/stream/src/executor/project/project_scalar.rs:91-108).
Test data keeps to where the reference is defined: `timestamp` values >= 0 (Timestamp::from_timestamp_uncheck is
undefined for a negative start with a sub-second part; `timestamptz` covers the negative range), dates inside chrono's
range, windows >= 0, every constant inside its own type.
"""
import ctypes as C

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import parse_project_expr
from risingwave_b200.stream_chunk import Column, StreamChunk, column_from_values, pack_bits

T_OF = {"int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "serial": abi.T_SERIAL, "date": abi.T_DATE,
        "timestamp": abi.T_TIMESTAMP, "timestamptz": abi.T_TIMESTAMPTZ}
BITS = {"int2": 16, "int4": 32, "date": 32}  # every other integer type here is 64 bits wide
US_PER_DAY = 86_400_000_000
INT_TYPES = ("int2", "int4", "int8")
BIN_OPS = ("add", "subtract", "multiply", "divide", "modulus")
WINDOWS = (0, 1, 7, 10 ** 6, 3_600_000_000, 1 << 62, (1 << 63) - 1)
MAX_EXPRS, MAX_OPS, MAX_STACK = 16, 24, 8  # the device's plan limits (csrc/chain.cu PROJ_*)


def bounds(t):
    b = BITS.get(t, 64)
    return -(1 << (b - 1)), (1 << (b - 1)) - 1


def edges(t):
    lo, hi = bounds(t)
    return [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi]


# ------------------------------------------------------------------------------------------ the restatement
# node: ("col", index, type) | ("const", value, type) | ("op", name, result type, (children...))
def col(k, t):
    return ("col", k, t)


def const(v, t):
    return ("const", v, t)


def op(name, t, *kids):
    return ("op", name, t, tuple(kids))


def node_type(n):
    return n[2]


def render(n):
    """build_from_pretty text, parsed by executor.parse_project_expr"""
    if n[0] == "col":
        return f"${n[1]}:{n[2]}"
    if n[0] == "const":
        return f"{n[1]}:{n[2]}"
    return f"({n[1]}:{n[2]} {' '.join(render(k) for k in n[3])})"


def n_ops(n):
    return 1 if n[0] != "op" else 1 + sum(n_ops(k) for k in n[3])


def nesting(n):
    return 1 if n[0] != "op" else 1 + max(nesting(k) for k in n[3])


def stack_depth(n):
    """values live on the postfix stack while `n` is evaluated"""
    if n[0] != "op":
        return 1
    return max(stack_depth(k) + i for i, k in enumerate(n[3]))


def trunc_div(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def in_i64(v):
    return -(1 << 63) <= v < (1 << 63)


def evaluate(n, row):
    if n[0] == "col":
        return row[n[1]]
    if n[0] == "const":
        return n[1]
    _, name, t, kids = n
    vals = [evaluate(k, row) for k in kids]
    if any(v is None for v in vals):
        return None
    lo, hi = bounds(t)
    if name == "neg":
        r = -vals[0]
    else:
        a, b = vals
        if name == "add":
            r = a + b
        elif name == "subtract":
            r = a - b
        elif name == "multiply":
            r = a * b
        elif name == "divide":
            if b == 0:
                return None
            r = trunc_div(a, b)
        elif name == "modulus":
            if b == 0 or (a == lo and b == -1):  # checked_rem
                return None
            r = a - b * trunc_div(a, b)
        else:  # tumble_start / tumble_end
            if node_type(kids[0]) == "date":
                a *= US_PER_DAY
                if not in_i64(a):
                    return None
            if b == 0:
                return None
            rem = a - b * trunc_div(a, b)
            r = a - (rem + b if rem < 0 else rem)
            if not in_i64(r):
                return None
            if name == "tumble_end":
                r += b
                if not in_i64(r):
                    return None
    return r if lo <= r <= hi else None


# ------------------------------------------------------------------------------------------ calling a backend
def expr_array(progs):
    """[(postfix program [(op, arg, value)], ret type)] -> (RwProjectExpr array, keepalive)"""
    arr = (abi.RwProjectExpr * len(progs))()
    keep = []
    for k, (prog, ty) in enumerate(progs):
        ops = (abi.RwExprOp * max(len(prog), 1))()
        for i, (o, a, v) in enumerate(prog):
            ops[i].op, ops[i].arg, ops[i].value = o, a, v
        keep.append(ops)
        arr[k].ops, arr[k].n_ops, arr[k].ret_type = ops, len(prog), ty
    return arr, keep


def project_host(backend, chunk, progs):
    """rwgpu_project / rwo_project -> per expression ([value or None per row], has_null)"""
    from risingwave_b200.stream_chunk import NP_DTYPE, unpack_bits
    ch, keep = chunk.to_abi()
    n, m = chunk.capacity(), len(progs)
    arr, keep2 = expr_array(progs)
    data = [np.zeros(max(n, 1), dtype=NP_DTYPE[ty]) for _, ty in progs]
    valid = [np.zeros(max((n + 63) // 64, 1), dtype=np.uint64) for _ in progs]
    dptr = (C.c_void_p * m)(*[d.ctypes.data for d in data])
    vptr = (C.c_void_p * m)(*[v.ctypes.data for v in valid])
    has_null = (C.c_uint32 * m)()
    backend.check(backend._project(C.byref(ch), arr, m, dptr, vptr, has_null))
    out = []
    for e in range(m):
        ok = unpack_bits(valid[e], n) if has_null[e] else np.ones(n, bool)
        out.append(([int(data[e][r]) if ok[r] else None for r in range(n)], int(has_null[e])))
    return out


def chunk_of(types, rows, rng=None, vis=False):
    """rows of Python values (None = NULL) -> StreamChunk; with `vis`, random ops and a random visibility"""
    cols = [column_from_values(T_OF[t], [r[k] for r in rows]) for k, t in enumerate(types)]
    n = len(rows)
    if not vis:
        return StreamChunk(np.full(n, abi.OP_INSERT, np.uint8), cols)
    return StreamChunk(rng.integers(1, 5, n).astype(np.uint8), cols, rng.random(n) > 0.3)


def mismatches(exprs, rows, got, limit=6):
    """exprs: trees; got: per expression (values, has_null).  Values are compared where the restatement's row is
    valid, validity everywhere, has_null exactly."""
    bad = []
    for x, (vals, has_null) in zip(exprs, got):
        want = [evaluate(x, r) for r in rows]
        if bool(has_null) != any(w is None for w in want):
            bad.append(f"{render(x)}: has_null={has_null}")
        for r, (g, w) in enumerate(zip(vals, want)):
            if g != w:
                bad.append(f"{render(x)} row {rows[r]}: got {g}, want {w}")
                break
    return bad


def check_grid(backend, types, rows, exprs, label, chunk=None):
    chunk = chunk if chunk is not None else chunk_of(types, rows)
    bad = []
    for lo in range(0, len(exprs), MAX_EXPRS):
        part = exprs[lo:lo + MAX_EXPRS]
        bad += mismatches(part, rows, project_host(backend, chunk, [parse_project_expr(render(x)) for x in part]))
    assert not bad, f"{label}: {len(bad)} expressions differ from the restatement:\n" + "\n".join(bad[:12])


# ------------------------------------------------------------------------------------------ the grid
def with_nulls(rng, rows, frac=0.08):
    return [tuple(None if rng.random() < frac else v for v in r) for r in rows]


def arith_case(t, seed=1):
    """every binary op and neg at type t over columns of type t: the edges crossed, random pairs, NULLs"""
    rng = np.random.default_rng(seed)
    lo, hi = bounds(t)
    e = edges(t)
    rows = [(a, b) for a in e for b in e]
    rows += [(int(rng.integers(lo, hi, endpoint=True)), int(rng.integers(lo, hi, endpoint=True))) for _ in range(48)]
    rows += [(int(rng.integers(-300, 300)), int(rng.integers(-20, 20))) for _ in range(24)]
    rows += with_nulls(rng, rows[:40], 0.5)
    a, b = col(0, t), col(1, t)
    exprs = [op(name, t, a, b) for name in BIN_OPS] + [op("neg", t, a)]
    exprs += [op("modulus", t, a, const(-1, t)), op("divide", t, a, const(-1, t)), op("add", t, op("neg", t, a), const(-1, t)),
              op("multiply", t, a, const(hi, t)), op("subtract", t, const(lo, t), b)]
    return [t, t], rows, exprs


def widening_case(seed=2):
    """narrower columns (sign-extended) and a serial under operations of other widths; narrow under wide and the reverse"""
    rng = np.random.default_rng(seed)
    types = ["int2", "int4", "int8", "serial"]
    cand = [edges(t) + [int(v) for v in rng.integers(-1000, 1000, 4)] for t in types]
    rows = [tuple(int(rng.choice(c)) for c in cand) for _ in range(160)]
    rows += with_nulls(rng, rows[:30], 0.3)
    s, i, l, q = (col(k, t) for k, t in enumerate(types))
    exprs = [op("add", "int8", s, i), op("multiply", "int8", i, i), op("subtract", "int4", s, s), op("multiply", "int2", s, s),
             op("add", "int8", q, l), op("modulus", "int8", q, i), op("divide", "int4", i, s), op("neg", "int2", s),
             op("add", "int8", op("multiply", "int4", i, i), l),                  # narrow inner under a wide outer
             op("multiply", "int4", op("add", "int8", l, l), const(2, "int4")),   # wide inner under a narrow outer
             op("divide", "int4", op("multiply", "int4", i, const(1000, "int4")), const(1000, "int4")),
             op("add", "int2", op("neg", "int4", s), const(-1, "int2")), op("modulus", "int4", op("add", "int8", i, const(0, "int8")), const(-1, "int4")),
             op("subtract", "int8", op("multiply", "int2", s, const(2, "int2")), op("neg", "int8", q))]
    return types, rows, exprs


def random_tree(rng, depth, leaves):
    if depth == 1:
        if rng.random() < 0.7:
            k = int(rng.integers(len(leaves)))
            return col(k, leaves[k])
        t = str(rng.choice(INT_TYPES))
        lo, hi = bounds(t)
        v = int(rng.integers(-9, 10)) if rng.random() < 0.7 else int(rng.choice(edges(t)))
        return const(max(lo, min(hi, v)), t)
    t = str(rng.choice(INT_TYPES))
    name = str(rng.choice(BIN_OPS + ("neg",)))
    deep = random_tree(rng, depth - 1, leaves)
    if name == "neg":
        return op(name, t, deep)
    other = random_tree(rng, int(rng.integers(1, min(depth - 1, 2) + 1)), leaves)
    return op(name, t, *((deep, other) if rng.random() < 0.5 else (other, deep)))


def nested_case(seed):
    """random programs of nesting depth 1..8 and up to 24 operations; every op at a random int width"""
    rng = np.random.default_rng(100 + seed)
    types = ["int2", "int4", "int8", "serial"]
    rows = []
    for _ in range(120):
        row = []
        for t in types:
            x = rng.random()
            lo, hi = bounds(t)
            row.append(int(rng.integers(-12, 13)) if x < 0.6 else int(rng.choice(edges(t))) if x < 0.85
                       else int(rng.integers(lo, hi, endpoint=True)))
        rows.append(tuple(row))
    rows = with_nulls(rng, rows, 0.03)
    exprs = []
    while len(exprs) < 32:
        x = random_tree(rng, int(rng.integers(2, 9)), types)
        if n_ops(x) <= MAX_OPS and stack_depth(x) <= MAX_STACK:
            exprs.append(x)
    return types, rows, exprs


def tumble_case(t, seed=3):
    """tumble_start / tumble_end over a date, timestamp or timestamptz column: constant windows, a window column"""
    rng = np.random.default_rng(seed)
    if t == "date":
        vals = [-94_999_999, -719_528, -1, 0, 1, 2, 19_000, 94_999_999] + [int(v) for v in rng.integers(-94_999_999, 94_999_999, 40)]
    elif t == "timestamp":
        vals = [0, 1, 6, 7, 999_999, 10 ** 6, 3_600_000_000, 1 << 62, (1 << 63) - 2, (1 << 63) - 1] + [int(v) for v in rng.integers(0, 1 << 63, 40)]
    else:
        vals = edges("int8") + [-(1 << 62), -3_600_000_001, -(10 ** 6) - 1] + [int(v) for v in rng.integers(-(1 << 63), (1 << 63) - 1, 40)]
    rows = [(v, WINDOWS[i % len(WINDOWS)]) for i, v in enumerate(vals)]
    rows += [(None, 7), (vals[3], None)]
    out = "timestamptz" if t == "timestamptz" else "timestamp"
    ts, w = col(0, t), col(1, "int8")
    exprs = [op(name, out, ts, const(win, "int8")) for win in WINDOWS for name in ("tumble_start", "tumble_end")]
    exprs += [op("tumble_start", out, ts, w), op("tumble_end", out, ts, w)]
    if t == "date":  # a DATE-typed operation's result is a DATE operand as well
        exprs.append(op("tumble_start", out, op("add", "date", ts, const(0, "int4")), const(3_600_000_000, "int8")))
    return [t, "int8"], rows, exprs


def reference_rows_case():
    """values the reference computes and a 64-bit-intermediate model does not: NULL for the first four, 86 400 000 000 us
    for the last (arithmetic_op.rs:98-107 checked_rem, the int4 checked_mul / checked_neg, tumble.rs:34-37)"""
    types = ["int8", "int4", "int4", "date"]
    rows = [(-(1 << 63), -(1 << 31), 70000, 1), (5, 70000, 70000, -1)]
    exprs = [op("modulus", "int8", col(0, "int8"), const(-1, "int8")), op("modulus", "int4", col(1, "int4"), const(-1, "int4")),
             op("divide", "int4", op("multiply", "int4", col(1, "int4"), col(2, "int4")), const(1000, "int4")),
             op("add", "int4", op("neg", "int4", col(1, "int4")), const(-1, "int4")),
             op("tumble_start", "timestamp", col(3, "date"), const(3_600_000_000, "int8"))]
    return types, rows, exprs


GRID = {f"arith_{t}": (lambda t=t: arith_case(t)) for t in INT_TYPES}
GRID.update({"widening": widening_case, "reference_rows": reference_rows_case})
GRID.update({f"nested_{s}": (lambda s=s: nested_case(s)) for s in range(4)})
GRID.update({f"tumble_{t}": (lambda t=t: tumble_case(t)) for t in ("date", "timestamp", "timestamptz")})


def test_restatement_reproduces_the_reference_rows():
    """the restatement itself, on the values worked out from the reference's source"""
    types, rows, exprs = reference_rows_case()
    assert [evaluate(x, rows[0]) for x in exprs] == [None, None, None, None, US_PER_DAY]
    assert [evaluate(x, rows[1]) for x in exprs] == [0, 0, None, -70001, -US_PER_DAY]


@pytest.mark.parametrize("case", sorted(GRID))
def test_oracle_matches_typed_restatement(oracle, case):
    """CPU: oracle/oracle.cc rwo_project against the restatement, value by value and validity by validity"""
    types, rows, exprs = GRID[case]()
    check_grid(oracle, types, rows, exprs, case)


# ------------------------------------------------------------------------------------------ plan limits
def limit_programs():
    I8 = abi.T_INT64
    c = lambda v: (abi.EX_CONST, 0, v)
    add, sub, neg = (abi.EX_ADD, I8, 0), (abi.EX_SUB, I8, 0), (abi.EX_NEG, I8, 0)
    deep8 = [c(k) for k in range(8)] + [add] * 7                  # stack depth 8, 15 ops
    ops24 = deep8 + [c(1), sub] * 4 + [neg]                        # 24 ops
    return {"ops24_depth8": ops24, "ops25": ops24 + [neg], "depth9": [c(k) for k in range(9)] + [add] * 8}


def limit_value(prog):
    st = []
    for o, _, v in prog:
        if o == abi.EX_CONST:
            st.append(v)
        elif o == abi.EX_NEG:
            st.append(-st.pop())
        else:
            b, a = st.pop(), st.pop()
            st.append(a + b if o == abi.EX_ADD else a - b)
    return st[0]


INVALID_PROGRAMS = {
    "malformed_underflow": [(abi.EX_CONST, 0, 1), (abi.EX_ADD, 0, 0)],
    "malformed_two_left": [(abi.EX_CONST, 0, 1), (abi.EX_CONST, 0, 2)],
    "unknown_op": [(abi.EX_CONST, 0, 1), (11, 0, 0)],
    "unknown_arg_type": [(abi.EX_CONST, 0, 1), (abi.EX_NEG, 99, 0)],
    "negative_arg_type": [(abi.EX_CONST, 0, 1), (abi.EX_CONST, 0, 2), (abi.EX_MUL, -1, 0)],
}


def limit_chunk():
    return StreamChunk(np.full(3, abi.OP_INSERT, np.uint8), [Column(abi.T_INT64, np.arange(3, dtype=np.int64))])


def check_limits_accepted(backend):
    p = limit_programs()["ops24_depth8"]
    got = project_host(backend, limit_chunk(), [(p, abi.T_INT64)] * MAX_EXPRS)
    assert got == [([limit_value(p)] * 3, 0)] * MAX_EXPRS


def check_invalid_refused(backend, name):
    with pytest.raises(abi.RwError) as e:
        project_host(backend, limit_chunk(), [(INVALID_PROGRAMS[name], abi.T_INT64)])
    assert e.value.code == abi.RW_ERR_INVALID


def test_oracle_plan_limits(oracle):
    """16 expressions of 24 operations at stack depth 8 are evaluated; programs with a wrong shape are refused"""
    check_limits_accepted(oracle)
    for name in INVALID_PROGRAMS:
        check_invalid_refused(oracle, name)


# ================================================================================== GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GRID))
def test_project_host_chunk_matches_restatement_and_oracle(cuda, oracle, case):
    """rwgpu_project (host chunk) against the restatement and against the oracle on the same grid: values where valid,
    validity, has_null; with random ops and an invisible share of rows (evaluated all the same)"""
    types, rows, exprs = GRID[case]()
    ch = chunk_of(types, rows, np.random.default_rng(len(case)), vis=True)
    check_grid(cuda, types, rows, exprs, case, chunk=ch)
    for lo in range(0, len(exprs), MAX_EXPRS):
        progs = [parse_project_expr(render(x)) for x in exprs[lo:lo + MAX_EXPRS]]
        assert project_host(cuda, ch, progs) == project_host(oracle, ch, progs), case


DEV_TYPES = ["int2", "int4", "int8", "date", "timestamptz"]
DEV_EXPRS = [op("add", "int2", col(0, "int2"), col(0, "int2")),
             op("divide", "int4", op("multiply", "int4", col(1, "int4"), col(1, "int4")), const(1000, "int4")),
             op("modulus", "int8", col(2, "int8"), const(-1, "int8")), op("modulus", "int4", col(1, "int4"), col(0, "int2")),
             op("neg", "int4", col(1, "int4")), op("add", "int8", op("multiply", "int4", col(1, "int4"), col(0, "int2")), col(2, "int8")),
             op("tumble_start", "timestamp", col(3, "date"), const(3_600_000_000, "int8")),
             op("tumble_end", "timestamptz", col(4, "timestamptz"), const(10 ** 6, "int8"))]


def dev_columns(rng, n):
    """numpy columns of DEV_TYPES: a third at the type edges, the rest small or anywhere in range; dates in chrono's range"""
    out = []
    for t in DEV_TYPES:
        lo, hi = bounds(t)
        if t == "date":
            lo, hi = -94_999_999, 94_999_999
        e = np.array([v for v in edges(t) if lo <= v <= hi] + [lo, hi], dtype=np.int64)
        v = rng.integers(lo, hi, n, endpoint=True, dtype=np.int64)
        pick = rng.random(n)
        v = np.where(pick < 0.33, e[rng.integers(0, len(e), n)], np.where(pick < 0.6, rng.integers(-40, 41, n), v))
        out.append(v.astype({"int2": np.int16, "int4": np.int32, "date": np.int32}.get(t, np.int64)))
    return out


def run_project_device(cols, valid, ops, vis, sliced):
    """DeviceChunk over the numpy columns (validity / visibility as packed words) -> ([values], [valid bytes], has_null)
    on the host, plus whether ops and visibility came back untouched"""
    import torch
    from risingwave_b200 import device

    def to_dev(a, off):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        if not sliced:
            return t
        big = torch.zeros(len(a) + off + 5, dtype=t.dtype, device="cuda")  # the column is a view at an offset
        big[off:off + len(a)] = t
        return big[off:off + len(a)]

    dcols = [to_dev(c, 3 + k) for k, c in enumerate(cols)]
    dvalid = [torch.from_numpy(pack_bits(v).view(np.int64)).cuda() for v in valid]
    dops = to_dev(ops, 1)
    dvis = torch.from_numpy(pack_bits(vis).view(np.int64)).cuda()
    ops0, vis0 = dops.clone(), dvis.clone()
    ch = device.DeviceChunk(dops, dcols, [T_OF[t] for t in DEV_TYPES], dvalid, dvis)
    progs = [parse_project_expr(render(x)) for x in DEV_EXPRS]
    arr, keep = expr_array(progs)
    outs, oks, has_null = device.project_device(ch, arr, [ty for _, ty in progs])
    torch.cuda.synchronize()
    untouched = torch.equal(dops, ops0) and torch.equal(dvis, vis0)
    return [o.cpu().numpy() for o in outs], [v.cpu().numpy() for v in oks], has_null.cpu().numpy(), untouched


def device_rows(cols, valid, idx):
    return [tuple(int(c[r]) if v[r] else None for c, v in zip(cols, valid)) for r in idx]


@pytest.mark.gpu
@pytest.mark.parametrize("sliced", [False, True], ids=["fresh", "sliced"])
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257])
def test_project_device_matches_restatement(cuda, n, sliced):
    """rwgpu_project_device: operand columns with validity bitmaps, a chunk with a visibility bitmap and all four ops
    (passed through untouched; invisible rows are evaluated all the same), columns that are views into larger tensors"""
    rng = np.random.default_rng(n + 7 * sliced)
    cols = dev_columns(rng, n)
    valid = [rng.random(n) > 0.15 for _ in cols]
    ops = rng.integers(1, 5, n).astype(np.uint8)
    vis = rng.random(n) > 0.3
    outs, oks, has_null, untouched = run_project_device(cols, valid, ops, vis, sliced)
    assert untouched
    rows = device_rows(cols, valid, range(n))
    got = [([int(o[r]) if ok[r] else None for r in range(n)], int(h)) for o, ok, h in zip(outs, oks, has_null)]
    bad = mismatches(DEV_EXPRS, rows, got)
    assert not bad, f"n={n}:\n" + "\n".join(bad)


@pytest.mark.gpu
def test_project_device_grid_stride_matches_oracle(cuda, oracle):
    """2^20 + 3 rows: more than the 132 x 8 blocks of 256 threads cover in one round, so every thread strides; all rows
    against the oracle, a sample (both ends and spread over the chunk) against the restatement"""
    n = (1 << 20) + 3
    rng = np.random.default_rng(11)
    cols = dev_columns(rng, n)
    valid = [rng.random(n) > 0.1 for _ in cols]
    ops = rng.integers(1, 5, n).astype(np.uint8)
    vis = rng.random(n) > 0.2
    outs, oks, has_null, untouched = run_project_device(cols, valid, ops, vis, sliced=True)
    assert untouched
    ch = StreamChunk(ops, [Column(T_OF[t], c, v) for t, c, v in zip(DEV_TYPES, cols, valid)], vis)
    from risingwave_b200.stream_chunk import NP_DTYPE, unpack_bits
    progs = [parse_project_expr(render(x)) for x in DEV_EXPRS]
    arr, keep = expr_array(progs)
    c_ch, keep2 = ch.to_abi()
    m = len(progs)
    data = [np.zeros(n, dtype=NP_DTYPE[ty]) for _, ty in progs]
    bits = [np.zeros((n + 63) // 64, dtype=np.uint64) for _ in progs]
    hn = (C.c_uint32 * m)()
    oracle.check(oracle._project(C.byref(c_ch), arr, m, (C.c_void_p * m)(*[d.ctypes.data for d in data]),
                                 (C.c_void_p * m)(*[b.ctypes.data for b in bits]), hn))
    for e in range(m):
        want_ok = unpack_bits(bits[e], n) if hn[e] else np.ones(n, bool)
        assert int(has_null[e]) == hn[e], render(DEV_EXPRS[e])
        assert np.array_equal(oks[e].astype(bool), want_ok), render(DEV_EXPRS[e])
        assert np.array_equal(outs[e][want_ok], data[e][want_ok]), render(DEV_EXPRS[e])
    idx = np.r_[0:300, n - 300:n, rng.choice(n, 3000, replace=False)]
    rows = device_rows(cols, valid, idx)
    for e, x in enumerate(DEV_EXPRS):
        got = [int(outs[e][r]) if oks[e][r] else None for r in idx]
        assert got == [evaluate(x, row) for row in rows], render(x)


@pytest.mark.gpu
def test_device_plan_limits(cuda):
    """accepted: 16 expressions, 24 operations, stack depth 8; refused with RW_ERR_UNSUPPORTED (the shim keeps the
    Project on the CPU): 17 expressions, 25 operations, depth 9; refused with RW_ERR_INVALID: a malformed program, an
    unknown operation, an unknown result type of an operation -- through both device entry points"""
    import torch
    from risingwave_b200 import device
    check_limits_accepted(cuda)
    p = limit_programs()
    refused = {"exprs17": [(p["ops24_depth8"], abi.T_INT64)] * (MAX_EXPRS + 1), "ops25": [(p["ops25"], abi.T_INT64)],
               "depth9": [(p["depth9"], abi.T_INT64)]}
    dch = device.DeviceChunk(torch.ones(3, dtype=torch.uint8, device="cuda"), [torch.arange(3, device="cuda")], [abi.T_INT64])
    for name, progs in refused.items():
        with pytest.raises(abi.RwError) as e:
            project_host(cuda, limit_chunk(), progs)
        assert e.value.code == abi.RW_ERR_UNSUPPORTED, name
        arr, keep = expr_array(progs)
        with pytest.raises(abi.RwError) as e:
            device.project_device(dch, arr, [ty for _, ty in progs])
        assert e.value.code == abi.RW_ERR_UNSUPPORTED, name
    for name, prog in INVALID_PROGRAMS.items():
        check_invalid_refused(cuda, name)
        arr, keep = expr_array([(prog, abi.T_INT64)])
        with pytest.raises(abi.RwError) as e:
            device.project_device(dch, arr, [abi.T_INT64])
        assert e.value.code == abi.RW_ERR_INVALID, name
    arr, keep = expr_array([(p["ops24_depth8"], abi.T_INT64)] * MAX_EXPRS)
    outs, oks, has_null = device.project_device(dch, arr, [abi.T_INT64] * MAX_EXPRS)
    torch.cuda.synchronize()
    want = limit_value(p["ops24_depth8"])
    assert all(o.tolist() == [want] * 3 and v.tolist() == [1] * 3 for o, v in zip(outs, oks)) and not has_null.any()
