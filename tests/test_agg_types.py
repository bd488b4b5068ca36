"""HashAgg at the type of every aggregate: the oracle (CPU) and the device (GPU) against a typed restatement of the
reference in Python integers and numpy floats.

The restatement is independent of oracle/oracle.cc and csrc/agg.cu.  Aggregate functions
(src/expr/impl/src/aggregate/general.rs), one `update` per visible row through the generated wrapper
(src/expr/macro/src/gen.rs:838-912: a NULL argument leaves the state as it is; the first non-NULL argument of a state
that is NULL starts from `S::default()`, or, for `state = "ref"` min / max, becomes the state):
  * count() / count(col) -> int8: +-1 per row (count(col): per non-NULL argument), init_state 0 (:155-162);
  * sum(int2 / int4) -> int8 and the internal sum(int8) -> int8 / sum0(int8) -> int8: an i64 state with
    checked_add / checked_sub (:18-41); sum0 starts at 0 instead of NULL;
  * sum(int8) -> decimal: the same over rust_decimal's 96-bit mantissa, |s| <= 2^96 - 1;
  * sum(float4) -> float4 and sum(float8) -> float8: an F32 / F64 state, rounded after every row;
    OrderedFloat's checked_add never fails (src/common/src/types/ordered_float.rs:431-438), so inf stays inf;
  * append-only min / max: `state.min(input)` / `state.max(input)` (:104,123) under Ord of OrderedFloat (NaN is the
    largest value, +0 == -0, every NaN equals every NaN: ordered_float.rs:182-219).  Rust's Ord::min returns `self` on a
    tie and Ord::max returns `other`: min keeps the state, max takes the input;
  * retractable min / max (AggState::MaterializedInput, minput.rs:172-245): the extreme of the live multiset of
    non-NULL inputs.  A tie between equal values of different bits (+-0, NaN payloads) is broken by the row's pk through
    memcomparable, which the operator's C ABI does not carry: such outputs are compared by OrderedFloat class only.
AggGroup (src/stream/src/executor/aggregate/agg_group.rs): row_count_of (:55-79, strict: a negative count is an
inconsistency), value states reset when the row count is 0 at the barrier (:438-446), OnlyOutputIfHasInput
(:131-166) with Datum equality of the output rows (so a max that moves from +0 to -0 emits nothing and keeps the
previous output, :573-606), and a restored intermediate-state row is the state datum, its outputs the previous
outputs (AggGroup::create, :260-316).

Errors.  The reference raises NumericOutOfRange at the row whose add leaves the state's type (rule "row"); the oracle
does the same, so it fails at that push.  The device keeps every integer sum exact in 128 bits and checks at the
barrier (rule "barrier"): a barrier fails if and only if some dirty group's state, after the reset of a group whose row
count is 0, lies outside its return type.  Overflows that are undone before the barrier therefore pass on the device.

Comparisons are bit-exact except: the NaN bits of a float sum, on every backend (the bits of a NaN that arithmetic
produces are not specified by Rust, a C++ compiler may commute the operands of an add, and the GPU returns its canonical
NaN), and on the device the zero sign / NaN bits of a float min / max (the device orders floats through a sortable
encoding that maps -0 to +0 and every NaN to one value, so it cannot follow row order among equal values): those compare
as NaN, or by OrderedFloat class.  Float sums on the device are order-dependent
inside one launch, and the host pushes of an epoch are applied by one launch: device streams put at most one row per
group into an epoch (or use values whose sums are exact in any order).
"""
from collections import Counter

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import AggCall, HashAggExecutor, MockSource
from risingwave_b200.stream_chunk import DECIMAL_DTYPE, NP_DTYPE, Column, StreamChunk, int_to_decimal, pack_bits, unpack_bits

T_OF = {"int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "float4": abi.T_FLOAT32, "float8": abi.T_FLOAT64,
        "decimal": abi.T_DECIMAL, "boolean": abi.T_BOOL, "date": abi.T_DATE, "timestamp": abi.T_TIMESTAMP}
INT_BITS = {"int2": 16, "int4": 32, "int8": 64}
FLOAT_NP = {"float4": np.float32, "float8": np.float64}
UINT_OF = {"float4": np.uint32, "float8": np.uint64}
DEC_MAX = (1 << 96) - 1
INS, DEL, UD, UI = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT


def bounds(t):
    b = INT_BITS[t]
    return -(1 << (b - 1)), (1 << (b - 1)) - 1


def edges(t):
    lo, hi = bounds(t)
    return [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi]


def fbits(t, bits):
    return np.array([bits], dtype=UINT_OF[t]).view(FLOAT_NP[t])[0]


def tobits(t, v):
    return int(np.array([v], dtype=FLOAT_NP[t]).view(UINT_OF[t])[0])


def float_edges(t):
    """+-0, +-inf, NaN with the sign bit clear and set, the smallest subnormal, f32 max, 2^24, 2^53 and a few plain values"""
    f = FLOAT_NP[t]
    if t == "float4":
        nans, sub = (0x7fc00000, 0xffc00000), 0x00000001
    else:
        nans, sub = (0x7ff8000000000000, 0xfff8000000000000), 0x0000000000000001
    vals = [f(0.0), f(-0.0), f(np.inf), f(-np.inf), fbits(t, nans[0]), fbits(t, nans[1]), fbits(t, sub), -fbits(t, sub),
            f(np.finfo(np.float32).max), -f(np.finfo(np.float32).max), f(2.0 ** 24), f(2.0 ** 53), f(1.0), f(-1.5), f(0.25)]
    return vals


# ------------------------------------------------------------------------------------------ the restatement
class Overflow(Exception):
    pass


class Inconsistent(Exception):
    pass


class Call:
    def __init__(self, kind, arg=None, at=None, ret=None):
        self.kind, self.arg, self.at = kind, arg, at
        if ret is None:  # general.rs: count / sum0 -> int8, sum(int2 / int4) -> int8, otherwise the argument type
            ret = "int8" if kind in ("count", "sum0") or (kind == "sum" and at in ("int2", "int4")) else at
        self.ret = ret

    def pretty(self):
        return f"({self.kind}:{self.ret})" if self.arg is None else f"({self.kind}:{self.ret} ${self.arg}:{self.at})"

    def is_float(self):
        return self.at in FLOAT_NP

    def init(self):
        return 0 if self.kind in ("count", "sum0") else None

    def in_range(self, s):
        if self.ret == "decimal":
            return -DEC_MAX <= s <= DEC_MAX
        lo, hi = bounds(self.ret)
        return lo <= s <= hi


def ord_key(v):
    """Ord of OrderedFloat (NaN largest, -0 == +0) / of the integers"""
    if isinstance(v, np.floating):
        return (1, 0.0) if np.isnan(v) else (0, float(v) + 0.0)
    return (0, v)


def datum_eq(a, b):
    if a is None or b is None:
        return a is None and b is None
    return ord_key(a) == ord_key(b)


def update(call, st, v, retract, rule):
    """one visible row into one value state"""
    if call.kind == "count":
        if call.arg is not None and v is None:
            return st
        return st - 1 if retract else st + 1
    if v is None:
        return st
    if call.kind in ("sum", "sum0"):
        if call.is_float():
            f = FLOAT_NP[call.at]
            s = f(0.0) if st is None else st
            with np.errstate(all="ignore"):
                return f(s - v) if retract else f(s + v)
        s = (0 if st is None else st) + (-v if retract else v)
        if rule == "row" and not call.in_range(s):
            raise Overflow(call.pretty())
        return s
    if retract:
        raise Inconsistent("retract on append-only min / max")
    if st is None:
        return v
    if call.kind == "min":
        return v if ord_key(v) < ord_key(st) else st
    return st if ord_key(v) < ord_key(st) else v


class Model:
    """HashAggExecutor + AggGroup over the restated functions; rule "row" (reference, oracle) or "barrier" (device)"""

    def __init__(self, calls, keys, append_only, rule):
        self.calls, self.keys, self.append_only, self.rule = calls, keys, append_only, rule
        self.groups, self.dirty = {}, []

    def minput(self, c):
        return not self.append_only and self.calls[c].kind in ("min", "max")

    def group(self, key):
        g = self.groups.get(key)
        if g is None:
            g = self.groups[key] = {"states": [c.init() for c in self.calls], "prev": None,
                                    "mi": [[] for _ in self.calls]}
        if key not in self.dirty:
            self.dirty.append(key)
        return g

    def push(self, rows):
        """rows: (op, row tuple, visible)"""
        for op, row, vis in rows:
            if not vis:
                continue
            g = self.group(tuple(row[k] for k in self.keys))
            retract = op in (DEL, UD)
            for c, call in enumerate(self.calls):
                v = None if call.arg is None else row[call.arg]
                if self.minput(c):
                    if v is None:
                        continue
                    mi = g["mi"][c]
                    if retract:
                        hit = [i for i, x in enumerate(mi) if ord_key(x) == ord_key(v)]
                        if not hit:
                            raise Inconsistent("retracting a value that is not in the materialized input")
                        mi.pop(hit[0])
                    else:
                        mi.append(v)
                    pick = min if call.kind == "min" else max
                    g["states"][c] = pick(mi, key=ord_key) if mi else None
                else:
                    g["states"][c] = update(call, g["states"][c], v, retract, self.rule)

    def restore(self, key, states):
        g = self.groups[key] = {"states": list(states), "prev": None, "mi": [[] for _ in self.calls]}
        g["prev"] = list(states)

    def flush(self):
        out = []
        for key in self.dirty:
            g = self.groups[key]
            rc = g["states"][0]
            if rc < 0:
                raise Inconsistent("row count should be non-negative")
            if rc == 0:
                for c, call in enumerate(self.calls):
                    if not self.minput(c):
                        g["states"][c] = call.init()
            if self.rule == "barrier":
                for c, call in enumerate(self.calls):
                    s = g["states"][c]
                    if call.kind in ("sum", "sum0") and not call.is_float() and s is not None and not call.in_range(s):
                        raise Overflow(call.pretty())
        for key in self.dirty:
            g = self.groups[key]
            curr = list(g["states"])
            prev = g["prev"]
            prev_rc = prev[0] if prev is not None else 0
            rc = curr[0]
            if prev_rc == 0 and rc == 0:
                pass
            elif prev_rc == 0:
                out.append((INS, key + tuple(curr)))
                g["prev"] = curr
            elif rc == 0:
                out.append((DEL, key + tuple(prev)))
                g["prev"] = None
            elif not all(datum_eq(a, b) for a, b in zip(prev, curr)):
                out.append((UD, key + tuple(prev)))
                out.append((UI, key + tuple(curr)))
                g["prev"] = curr
        self.dirty = []
        return out


# ------------------------------------------------------------------------------------------ chunks and comparison
def make_chunk(types, rows):
    """rows: (op, row tuple, visible) -> StreamChunk; float values keep their bits"""
    n = len(rows)
    cols = []
    for k, t in enumerate(types):
        data = np.zeros(n, dtype=NP_DTYPE[T_OF[t]])
        valid = np.ones(n, dtype=bool)
        for i, (_, row, _) in enumerate(rows):
            v = row[k]
            if v is None:
                valid[i] = False
            elif t in FLOAT_NP:
                data.view(UINT_OF[t])[i] = tobits(t, v)
            elif t == "decimal":
                data[i] = int_to_decimal(v)
            else:
                data[i] = v
        cols.append(Column(T_OF[t], data, None if valid.all() else valid))
    vis = np.array([r[2] for r in rows], dtype=bool)
    return StreamChunk(np.array([r[0] for r in rows], dtype=np.uint8), cols, None if vis.all() else vis)


def chunk_rows(chunks, out_types):
    """visible (op, row) of output chunks, floats as numpy scalars with their bits"""
    out = []
    for ch in chunks:
        for i in range(ch.capacity()):
            if not ch.is_visible(i):
                continue
            row = []
            for c, t in zip(ch.columns, out_types):
                if c.valid is not None and not c.valid[i]:
                    row.append(None)
                elif t in FLOAT_NP:
                    row.append(FLOAT_NP[t](c.data[i]))
                else:
                    row.append(c.value(i))
            out.append((int(ch.ops[i]), tuple(row)))
    return out


def canon(v, t, how):
    """hashable form of an output value: floats by their bits ("bits"), with every NaN alike ("nan"), or by OrderedFloat
    class ("class": also -0 == +0)"""
    if v is None:
        return None
    if t in FLOAT_NP:
        if np.isnan(v) and how != "bits":
            return "nan"
        if how == "class":
            return float(v) + 0.0
        return (t, tobits(t, v))
    return int(v)


class Spec:
    def __init__(self, types, keys, calls, append_only):
        self.types, self.keys, self.calls, self.append_only = types, keys, calls, append_only
        self.out_types = [types[k] for k in keys] + [c.ret for c in calls]

    def executor(self, backend, hint=0):
        _, src = MockSource.channel()
        return HashAggExecutor(backend, src.into_executor([T_OF[t] for t in self.types], []), self.append_only,
                               [AggCall.from_pretty(c.pretty()) for c in self.calls], 0, self.keys,
                               group_capacity_hint=hint)

    def loose_cols(self, device):
        """how each output column compares (see `canon`): a float sum's NaN bits are those of the hardware's NaN
        arithmetic, which Rust leaves unspecified (even x86 code may commute the operands); a float min / max is
        compared by class on the device and wherever a pk tie-break decides (retractable)"""
        how = ["bits"] * len(self.keys)
        for c in self.calls:
            if not c.is_float():
                how.append("bits")
            elif c.kind in ("min", "max"):
                how.append("class" if device or not self.append_only else "bits")
            else:
                how.append("nan")
        return how

    def multiset(self, rows, loose):
        cnt = Counter()
        for op, row in rows:
            key = tuple(canon(v, t, l) for v, t, l in zip(row, self.out_types, loose))
            cnt[(op, key)] += 1
        return cnt


def play_model(spec, epochs, rule, restored=()):
    """-> per epoch ("ok", rows) until the first error, which is ("err", code, "push" / "flush")"""
    m = Model(spec.calls, spec.keys, spec.append_only, rule)
    for key, states in restored:
        m.restore(key, states)
    res = []
    for pushes in epochs:
        try:
            for p in pushes:
                m.push(p)
        except Overflow:
            return res + [("err", abi.RW_ERR_NUMERIC_OUT_OF_RANGE, "push")]
        except Inconsistent:
            return res + [("err", abi.RW_ERR_INCONSISTENT, "push")]
        try:
            res.append(("ok", m.flush()))
        except Overflow:
            return res + [("err", abi.RW_ERR_NUMERIC_OUT_OF_RANGE, "flush")]
        except Inconsistent:
            return res + [("err", abi.RW_ERR_INCONSISTENT, "flush")]
    return res


def play_host(spec, backend, epochs, restored=None, hint=0):
    """through rwgpu_agg_push / rwgpu_agg_flush (or the oracle's)"""
    ex = spec.executor(backend, hint)
    if restored is not None:
        ex.restore(restored)
    res = []
    for pushes in epochs:
        try:
            for p in pushes:
                ex.apply_chunk(make_chunk(spec.types, p))
        except abi.RwError as e:
            return res + [("err", e.code, "push")]
        try:
            res.append(("ok", chunk_rows(ex.flush_data(len(res) + 1), spec.out_types)))
        except abi.RwError as e:
            return res + [("err", e.code, "flush")]
    return res


def assert_same(spec, got, want, loose, what):
    assert len(got) == len(want), f"{what}: {len(got)} outcomes, want {len(want)}: got {got[-1:]} want {want[-1:]}"
    for e, (g, w) in enumerate(zip(got, want)):
        if w[0] == "err" or g[0] == "err":
            assert g == w, f"{what} epoch {e}: got {g[:3] if g[0] == 'err' else 'rows'}, want {w if w[0] == 'err' else 'rows'}"
            continue
        gm, wm = spec.multiset(g[1], loose), spec.multiset(w[1], loose)
        assert gm == wm, f"{what} epoch {e}:\n only got  {sorted(map(str, (gm - wm).elements()))[:6]}\n only want {sorted(map(str, (wm - gm).elements()))[:6]}"


# ------------------------------------------------------------------------------------------ streams
def random_epochs(rng, spec, values, n_epochs=6, pushes=3, rows=60, key_values=(0, 1, 2, None), p_del=0.3, p_invis=0.1,
                  one_row_per_group=False):
    """inserts, deletes, U-/U+ pairs (not append-only), invisible rows, NULL keys, groups that empty out and come back.
    values[k]: the pool of column k (None = NULL); key columns draw from key_values."""
    live = []
    epochs = []
    for e in range(n_epochs):
        ep = []
        for _ in range(pushes):
            out, used = [], set()

            def new_row():
                return tuple(key_values[int(rng.integers(len(key_values)))] if k in spec.keys
                             else values[k][int(rng.integers(len(values[k])))] for k in range(len(spec.types)))

            for _ in range(rows):
                drain = e % 3 == 2  # every third epoch mostly retracts: groups empty out, and come back later
                if live and not spec.append_only and rng.random() < (0.8 if drain else p_del):
                    i = int(rng.integers(len(live)))
                    old = live[i]
                    gk = tuple(old[k] for k in spec.keys)
                    if one_row_per_group and gk in used:
                        continue
                    if rng.random() < 0.4 and not one_row_per_group:
                        new = new_row()
                        new = tuple(old[k] if k in spec.keys else new[k] for k in range(len(new)))
                        out += [(UD, old, True), (UI, new, True)]
                        live[i] = new
                    else:
                        out.append((DEL, old, True))
                        live.pop(i)
                    used.add(gk)
                else:
                    row = new_row()
                    gk = tuple(row[k] for k in spec.keys)
                    if one_row_per_group and gk in used:
                        continue
                    if rng.random() < p_invis:  # invisible: never applied, never live
                        out.append((INS if spec.append_only else int(rng.integers(1, 5)), row, False))
                        continue
                    out.append((INS, row, True))
                    live.append(row)
                    used.add(gk)
            ep.append(out)
        epochs.append(ep)
    return epochs


def int_spec(t, append_only, wide_sum=False):
    """int8 key | a: t | b: t with NULLs.  Every call at type t."""
    calls = [Call("count"), Call("count", 2, t)]
    if t == "int8":
        calls.append(Call("sum", 1, t, "decimal") if not wide_sum else Call("sum", 1, t, "int8"))
        if wide_sum:
            calls.append(Call("sum0", 2, t))
    else:
        calls.append(Call("sum", 1, t))
        calls.append(Call("sum", 2, t))
    calls += [Call("min", 1, t), Call("max", 2, t)]
    return Spec(["int8", t, t], [0], calls, append_only)


def float_spec(append_only):
    calls = [Call("count"), Call("count", 1, "float4"), Call("sum", 1, "float4"), Call("sum", 2, "float8"),
             Call("min", 1, "float4"), Call("max", 1, "float4"), Call("min", 2, "float8"), Call("max", 2, "float8")]
    return Spec(["int8", "float4", "float8"], [0], calls, append_only)


def multikey_spec():
    calls = [Call("count"), Call("sum", 3, "int4"), Call("max", 3, "int4"), Call("sum", 2, "int2"), Call("min", 2, "int2")]
    return Spec(["int2", "int4", "int2", "int4"], [0, 1], calls, False)


INT_CASES = [(t, ao) for t in INT_BITS for ao in (True, False)]


def int_values(t):
    return [None, [*edges(t), None], [*edges(t), None, None]]


# ------------------------------------------------------------------------------------------ oracle vs restatement (CPU)
@pytest.mark.parametrize("t,append_only", INT_CASES, ids=[f"{t}-{'ao' if a else 'retract'}" for t, a in INT_CASES])
def test_oracle_integer_calls_at_their_types(oracle, t, append_only):
    spec = int_spec(t, append_only)
    rng = np.random.default_rng(INT_BITS[t] + append_only)
    epochs = random_epochs(rng, spec, int_values(t))
    want = play_model(spec, epochs, "row")
    assert all(w[0] == "ok" for w in want)
    assert_same(spec, play_host(spec, oracle, epochs), want, spec.loose_cols(False), f"oracle {t}")


@pytest.mark.parametrize("seed", range(4))
def test_oracle_int8_sums_fail_at_the_overflowing_push(oracle, seed):
    """sum(int8) -> int8 and sum0(int8) over the int8 edges: most streams overflow; the oracle fails at the same push"""
    spec = int_spec("int8", False, wide_sum=True)
    rng = np.random.default_rng(100 + seed)
    vals = [None, [*edges("int8"), None] + [0] * 20, [*edges("int8"), None] + [1, -1] * 10]
    epochs = random_epochs(rng, spec, vals, rows=12)
    assert_same(spec, play_host(spec, oracle, epochs), play_model(spec, epochs, "row"), spec.loose_cols(False), "oracle")


@pytest.mark.parametrize("append_only", [True, False], ids=["ao", "retract"])
def test_oracle_float_calls_at_their_types(oracle, append_only):
    spec = float_spec(append_only)
    rng = np.random.default_rng(7 + append_only)
    epochs = random_epochs(rng, spec, [None, float_edges("float4") + [None], float_edges("float8") + [None]])
    want = play_model(spec, epochs, "row")
    assert_same(spec, play_host(spec, oracle, epochs), want, spec.loose_cols(False), "oracle float")


def test_oracle_multi_column_narrow_keys(oracle):
    spec = multikey_spec()
    rng = np.random.default_rng(11)
    vals = [[*edges("int2")[:3], None], [*edges("int4")[-3:], None], [*edges("int2"), None], [*edges("int4"), None]]
    live, epochs = [], []  # (both key columns draw from their own pools, NULL included)
    for e in range(5):
        ep = []
        for _ in range(3):
            rows = []
            for _ in range(50):
                if live and rng.random() < (0.7 if e % 3 == 2 else 0.3):
                    rows.append((DEL, live.pop(int(rng.integers(len(live)))), True))
                else:
                    row = tuple(vals[k][int(rng.integers(len(vals[k])))] for k in range(4))
                    rows.append((INS, row, True))
                    live.append(row)
            ep.append(rows)
        epochs.append(ep)
    want = play_model(spec, epochs, "row")
    assert all(w[0] == "ok" for w in want)
    assert_same(spec, play_host(spec, oracle, epochs), want, spec.loose_cols(False), "oracle multi-key")


def test_oracle_append_only_max_takes_the_input_on_a_tie(oracle):
    """general.rs:104,123: Ord::min keeps the state on a tie, Ord::max takes the input.  max(+0, -0) = -0,
    min(+0, -0) = +0; among NaNs max ends on the last one, min keeps the first.  A change between equal Datums emits
    nothing (agg_group.rs:160-163)."""
    spec = Spec(["int8", "float8", "float4"], [0],
                [Call("count"), Call("max", 1, "float8"), Call("min", 1, "float8"), Call("max", 2, "float4"),
                 Call("min", 2, "float4")], True)
    n8, n8neg = fbits("float8", 0x7ff8000000000000), fbits("float8", 0xfff8000000000001)
    n4, n4neg = fbits("float4", 0x7fc00000), fbits("float4", 0xffc00001)
    z8, nz8, z4, nz4 = np.float64(0.0), np.float64(-0.0), np.float32(0.0), np.float32(-0.0)
    epochs = [[[(INS, (1, z8, z4), True), (INS, (2, n8, n4), True)]],
              [[(INS, (1, nz8, nz4), True), (INS, (2, n8neg, n4neg), True)]]]
    got = play_host(spec, oracle, epochs)
    assert_same(spec, got, play_model(spec, epochs, "row"), spec.loose_cols(False), "oracle ties")
    new = {r[0]: r for op, r in got[1][1] if op == UI}
    assert tobits("float8", new[1][2]) == tobits("float8", nz8) and tobits("float4", new[1][5]) == 0
    # one push: the states themselves
    got = play_host(spec, oracle, [[[(INS, (1, z8, z4), True), (INS, (1, nz8, nz4), True),
                                     (INS, (2, n8, n4), True), (INS, (2, n8neg, n4neg), True)]]])
    rows = {r[0]: r for _, r in got[0][1]}
    assert tobits("float8", rows[1][2]) == tobits("float8", nz8) and tobits("float8", rows[1][3]) == 0
    assert tobits("float4", rows[1][4]) == tobits("float4", nz4) and tobits("float4", rows[1][5]) == 0
    assert tobits("float8", rows[2][2]) == 0xfff8000000000001 and tobits("float8", rows[2][3]) == 0x7ff8000000000000
    assert tobits("float4", rows[2][4]) == 0xffc00001 and tobits("float4", rows[2][5]) == 0x7fc00000


def test_oracle_output_change_is_datum_equality(oracle):
    """OnlyOutputIfHasInput compares output rows as Datums (agg_group.rs:160-163): a retractable max whose only live value
    moves from +0 to -0 emits no U-/U+, and the previous output (+0) stays the one a later Delete retracts (:573-606)"""
    spec = Spec(["int8", "float8"], [0], [Call("count"), Call("max", 1, "float8")], False)
    z, nz = np.float64(0.0), np.float64(-0.0)
    epochs = [[[(INS, (1, z), True)]], [[(UD, (1, z), True), (UI, (1, nz), True)]], [[(DEL, (1, nz), True)]]]
    got = play_host(spec, oracle, epochs)
    assert [g[0] for g in got] == ["ok"] * 3 and got[1][1] == []
    (op, row), = got[2][1]
    assert op == DEL and tobits("float8", row[2]) == 0
    assert_same(spec, got, play_model(spec, epochs, "row"), ["bits"] * 3, "oracle Datum equality")


def test_oracle_null_arguments_and_all_null_groups(oracle):
    """sum over only NULLs is NULL, sum0 is 0, count(col) is 0, min / max are NULL; a NULL group key is a group"""
    spec = Spec(["int8", "int8", "int4"], [0],
                [Call("count"), Call("count", 1, "int8"), Call("sum", 1, "int8", "decimal"), Call("sum0", 1, "int8"),
                 Call("sum", 2, "int4"), Call("min", 2, "int4"), Call("max", 1, "int8")], False)
    epochs = [[[(INS, (1, None, None), True), (INS, (None, None, None), True), (INS, (2, 5, 7), True)]],
              [[(INS, (2, None, None), True), (DEL, (2, 5, 7), True)]],
              [[(DEL, (1, None, None), True), (DEL, (2, None, None), True), (INS, (2, None, 3), True)]]]
    want = play_model(spec, epochs, "row")
    assert want[0][1][0] == (INS, (1, 1, 0, None, 0, None, None, None))
    # a sum whose every input was retracted is 0, not NULL (its state is Some(0)); min / max of an empty input is NULL
    assert (UI, (2, 1, 0, 0, 0, 0, None, None)) in want[1][1]
    assert (UI, (2, 1, 0, 0, 0, 3, 3, None)) in want[2][1]
    assert_same(spec, play_host(spec, oracle, epochs), want, spec.loose_cols(False), "oracle NULLs")


# ------------------------------------------------------------------------------------------ signatures
BAD_SIGNATURES = ["(sum:decimal $1:int2)", "(sum:decimal $1:int4)", "(sum:int4 $1:int4)", "(sum0:int8 $1:int4)",
                  "(sum0:decimal $2:int8)", "(sum:float8 $3:float4)", "(sum:int8 $4:date)", "(sum:int8 $5:boolean)",
                  "(max:boolean $5:boolean)", "(min:int8 $1:int4)", "(count:int4)", "(sum:int8)"]


def _create(backend, sig):
    """input columns: int8 key | int2 or int4 | int8 | float4 | date | boolean"""
    call = AggCall.from_pretty(sig)
    types = [abi.T_INT64, abi.T_INT16 if "$1:int2" in sig else abi.T_INT32, abi.T_INT64, abi.T_FLOAT32, abi.T_DATE, abi.T_BOOL]
    _, src = MockSource.channel()
    return HashAggExecutor(backend, src.into_executor(types, []), True, [AggCall.from_pretty("(count:int8)"), call], 0, [0])


def check_signatures(backend):
    for sig in BAD_SIGNATURES:
        with pytest.raises(abi.RwError) as e:
            _create(backend, sig)
        assert e.value.code == abi.RW_ERR_INVALID, sig
    for sig in ("(sum:int8 $1:int2)", "(sum:int8 $1:int4)", "(sum:int8 $2:int8)", "(sum:decimal $2:int8)",
                "(sum0:int8 $2:int8)", "(sum:float4 $3:float4)", "(min:date $4:date)", "(count:int8 $5:boolean)"):
        _create(backend, sig)


def test_oracle_refuses_signatures_the_reference_does_not_define(oracle):
    check_signatures(oracle)


# ------------------------------------------------------------------------------------------ the device
def device_chunk(chunk, offset):
    """StreamChunk -> device.DeviceChunk; `offset`: every column starts one element into its allocation (an 8-byte offset
    for int8, never 16-byte aligned) and the ops one byte in (odd address)"""
    import torch
    from risingwave_b200 import device
    pad = 1 if offset else 0
    n = chunk.capacity()

    def up(arr):
        t = torch.from_numpy(np.concatenate([np.zeros(pad, arr.dtype), arr]) if pad else arr.copy()).cuda()
        return t[pad:]

    ops = up(chunk.ops)
    cols = [up(np.ascontiguousarray(c.data)) for c in chunk.columns]
    valid = [None if c.valid is None else torch.from_numpy(pack_bits(c.valid).view(np.int64)).cuda() for c in chunk.columns]
    vis = None if chunk.vis is None else torch.from_numpy(pack_bits(chunk.vis).view(np.int64)).cuda()
    assert all(x.numel() == n for x in cols)
    return device.DeviceChunk(ops, cols, chunk.types(), valid, vis)


def view_rows(view, out_types):
    import torch
    from risingwave_b200 import device
    n = view.n_rows
    ops = view.ops().cpu().numpy()
    cols = []
    for k, t in enumerate(out_types):
        if t == "decimal":  # (no torch dtype: the 16-byte words are copied as int64 pairs)
            view._wait()
            words = torch.empty(2 * n, dtype=torch.int64, device="cuda")
            if n:
                device._d2d(words.data_ptr(), view.col_ptrs[k], n * 16)
            data = words.cpu().numpy().view(DECIMAL_DTYPE)
        else:
            data = view.column(k).cpu().numpy()
        valid = None
        if view.valid_ptrs[k] and n:
            words = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda")
            device._d2d(words.data_ptr(), view.valid_ptrs[k], words.numel() * 8)
            torch.cuda.synchronize()
            valid = unpack_bits(words.cpu().numpy().view(np.uint64), n)
        cols.append(Column(T_OF[t], data, valid))
    return chunk_rows([StreamChunk(ops, cols)], out_types)


def play_device(spec, cuda, epochs, offset, asynchronous):
    """through rwgpu_agg_push_device and rwgpu_agg_flush_device (or the _async / _collect pair)"""
    import torch
    from risingwave_b200 import device
    ex = spec.executor(cuda)
    stream = torch.cuda.Stream()
    res = []
    with torch.cuda.stream(stream):
        for e, pushes in enumerate(epochs):
            try:
                for p in pushes:
                    device.agg_push_device(ex, device_chunk(make_chunk(spec.types, p), offset), stream)
            except abi.RwError as err:
                return res + [("err", err.code, "push")]
            try:
                if asynchronous:
                    device.agg_flush_device_async(ex, e + 1, stream)
                    view = device.agg_flush_collect(ex, stream)
                else:
                    view = device.agg_flush_device(ex, e + 1, stream)
                res.append(("ok", view_rows(view, spec.out_types)))
            except abi.RwError as err:
                return res + [("err", err.code, "flush")]
    return res


def check_device(cuda, oracle, spec, epochs):
    """the host push, the device push at an odd offset, the async pair: all against the restatement (rule "barrier")
    and, when nothing fails, the oracle"""
    want = play_model(spec, epochs, "barrier")
    loose = spec.loose_cols(True)
    assert_same(spec, play_host(spec, cuda, epochs), want, loose, "device host push")
    assert_same(spec, play_device(spec, cuda, epochs, offset=True, asynchronous=False), want, loose, "device push, offset")
    assert_same(spec, play_device(spec, cuda, epochs, offset=False, asynchronous=True), want, loose, "device push, async")
    want_row = play_model(spec, epochs, "row")  # the oracle fails at the push where the reference does
    if all(w[0] == "ok" for w in want_row):
        assert_same(spec, play_host(spec, oracle, epochs), want_row, loose, "oracle")
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("t,append_only", INT_CASES, ids=[f"{t}-{'ao' if a else 'retract'}" for t, a in INT_CASES])
def test_device_integer_calls_at_their_types(cuda, oracle, t, append_only):
    spec = int_spec(t, append_only)
    rng = np.random.default_rng(INT_BITS[t] + append_only)
    epochs = random_epochs(rng, spec, int_values(t))
    want = check_device(cuda, oracle, spec, epochs)
    assert all(w[0] == "ok" for w in want)


@pytest.mark.gpu
@pytest.mark.parametrize("append_only", [True, False], ids=["ao", "retract"])
def test_device_float_calls_at_their_types(cuda, oracle, append_only):
    """one row per group and epoch: the device's float sums are then in row order (the host pushes of an epoch are
    staged and applied by one launch, so only the barrier orders them)"""
    spec = float_spec(append_only)
    rng = np.random.default_rng(7 + append_only)
    epochs = random_epochs(rng, spec, [None, float_edges("float4") + [None], float_edges("float8") + [None]],
                           key_values=tuple(range(12)) + (None,), one_row_per_group=True, n_epochs=16, pushes=1, rows=14)
    check_device(cuda, oracle, spec, epochs)


@pytest.mark.gpu
def test_device_float4_sum_is_an_f32_state(cuda, oracle):
    """general.rs:28-41 over F32: +3e38 +3e38 -3e38 -> 3e38, inf, inf (sticky); 2^24 + 1 in separate pushes stays 2^24;
    the smallest subnormal is kept (not flushed to zero)"""
    spec = Spec(["int8", "float4"], [0], [Call("count"), Call("sum", 1, "float4")], False)
    f = np.float32
    sub = fbits("float4", 1)
    pushes = [[(INS, (1, f(3e38)), True), (INS, (2, f(2.0 ** 24)), True), (INS, (3, sub), True)],
              [(INS, (1, f(3e38)), True), (INS, (2, f(1.0)), True), (INS, (3, sub), True)],
              [(DEL, (1, f(3e38)), True), (INS, (2, f(1.0)), True), (DEL, (3, sub), True)]]
    epochs = [[p] for p in pushes]
    want = check_device(cuda, oracle, spec, epochs)
    last = {r[0]: r for op, r in want[2][1] if op == UI}
    assert np.isinf(last[1][2]) and last[2][2] == f(2.0 ** 24) and tobits("float4", last[3][2]) == 1


@pytest.mark.gpu
def test_device_multi_column_narrow_keys_and_null_keys(cuda, oracle):
    spec = multikey_spec()
    rng = np.random.default_rng(12)
    vals = [[*edges("int2")[:3], None], [*edges("int4")[-3:], None], [*edges("int2"), None], [*edges("int4"), None]]
    live, epochs = [], []
    for e in range(5):
        ep = []
        for _ in range(3):
            rows = []
            for _ in range(60):
                if live and rng.random() < (0.7 if e % 3 == 2 else 0.3):
                    rows.append((DEL, live.pop(int(rng.integers(len(live)))), True))
                else:
                    row = tuple(vals[k][int(rng.integers(len(vals[k])))] for k in range(4))
                    rows.append((INS, row, bool(rng.random() > 0.1)))
                    if rows[-1][2]:
                        live.append(row)
            ep.append(rows)
        epochs.append(ep)
    check_device(cuda, oracle, spec, epochs)


@pytest.mark.gpu
def test_device_barrier_overflow_rule(cuda, oracle):
    """The device's rule: a barrier fails iff some dirty group's integer sum, after the reset of a group whose row count
    is 0, lies outside its return type.  Transient overflows pass on the device and fail the reference / oracle at the
    push; a net overflow fails both; a group that empties out drops its sum before the check."""
    i64max, i64min = (1 << 63) - 1, -(1 << 63)
    i32max = (1 << 31) - 1
    cases = [
        # (calls' argument type, ret, pushes of one epoch, device fails?, oracle fails at push?)
        ("int8", "int8", [[(INS, (1, i64max), True), (INS, (1, 1), True), (DEL, (1, 1), True)]], False, True),
        ("int8", "int8", [[(INS, (1, i64max), True)], [(INS, (1, i64max), True)], [(DEL, (1, i64max), True)]], False, True),
        ("int8", "int8", [[(INS, (1, i64min), True), (INS, (1, -1), True)]], True, True),
        ("int8", "int8", [[(INS, (1, i64max), True), (INS, (1, i64max), True), (DEL, (1, i64max), True),
                           (DEL, (1, i64max), True)]], False, True),  # empties out: reset, nothing emitted
        ("int8", "int8", [[(INS, (1, i64max), True), (INS, (1, 5), True), (DEL, (1, 5), True), (DEL, (1, i64max), True),
                           (INS, (1, i64max), True), (INS, (1, i64max), True)]], True, True),
        ("int8", "decimal", [[(INS, (1, i64max), True)] * 4 + [(DEL, (1, i64max), True)] * 4], False, False),
        ("int4", "int8", [[(INS, (1, i32max), True)] * 8], False, False),
    ]
    for at, ret, pushes, dev_fails, oracle_fails in cases:
        spec = Spec(["int8", at], [0], [Call("count"), Call("sum", 1, at, ret)], False)
        epochs = [pushes]
        want_row, want_bar = play_model(spec, epochs, "row"), play_model(spec, epochs, "barrier")
        assert (want_bar[-1][0] == "err") == dev_fails and (want_row[-1][0] == "err") == oracle_fails, (pushes, want_bar, want_row)
        assert_same(spec, play_host(spec, cuda, epochs), want_bar, spec.loose_cols(True), f"device {pushes}")
        assert_same(spec, play_host(spec, oracle, epochs), want_row, spec.loose_cols(False), f"oracle {pushes}")


@pytest.mark.gpu
def test_device_kernel_paths_same_rows_same_answer(cuda, oracle):
    """The fast kernel (one 16-byte aligned int8 key, no NULLs: host push), the generic kernel (8-byte offset columns
    and an odd ops pointer through rwgpu_agg_push_device), an epoch whose first push is NULL-free and whose second has
    NULLs (the switch to per-row flags), and the async flush/collect pair.  Many i64::MAX / i64::MIN inserts and
    deletes per push exercise the 128-bit carry of concurrent adds."""
    i64max, i64min = (1 << 63) - 1, -(1 << 63)
    # both plans are fast-kernel plans: count(*), sum / sum0(int8) -> int8, and append-only min / max(int8)
    spec = Spec(["int8", "int8", "int8"], [0], [Call("count"), Call("sum", 1, "int8"), Call("sum0", 2, "int8")], False)
    spec_ao = Spec(spec.types, spec.keys, [Call("count"), Call("sum", 2, "int8"), Call("min", 1, "int8"), Call("max", 1, "int8")], True)
    rng = np.random.default_rng(21)
    for sp in (spec, spec_ao):
        epochs = []
        for e in range(4):
            ep = []
            for j in range(2):
                rows = []
                for g in range(40):
                    k = int(rng.integers(-3, 300)) if g else i64min  # (i64::MIN is the table's EMPTY sentinel)
                    m = int(rng.integers(1, 30))
                    if sp.append_only:
                        rows += [(INS, (k, i64max if i % 2 else i64min, int(rng.integers(-5, 5))), True) for i in range(m)]
                    else:  # retracted again inside the push: only the 128-bit carry keeps the net sums right
                        rows += [(INS, (k, i64max, i64min), True)] * m + [(DEL, (k, i64max, i64min), True)] * m
                    rows.append((INS, (k, int(rng.integers(-5, 5)), int(rng.integers(-5, 5))), True))
                if j == 1 and e % 2 == 1:  # NULLs after a NULL-free push of the same epoch
                    rows += [(INS, (None, 1, None), True), (INS, (7, None, 2), True)]
                ep.append([rows[i] for i in rng.permutation(len(rows))])
            epochs.append(ep)
        want = check_device(cuda, oracle, sp, epochs)
        assert all(w[0] == "ok" for w in want)


@pytest.mark.gpu
def test_device_restore_at_the_edges(cuda):
    """rwgpu_agg_restore: a restored state row is the state datum (agg_group.rs:260-316), its outputs the previous
    outputs; pushes continue from it."""
    i64max = (1 << 63) - 1
    f32max = np.float32(np.finfo(np.float32).max)
    cases = []
    # sum(int4) -> int8 at i64::MAX - 5: +5 reaches MAX exactly, +10 fails the barrier
    s4 = Spec(["int8", "int4"], [0], [Call("count"), Call("sum", 1, "int4")], False)
    cases += [(s4, [((1,), [3, i64max - 5])], [[[(INS, (1, 5), True)]]], "ok"),
              (s4, [((1,), [3, i64max - 5])], [[[(INS, (1, 10), True)]]], "err"),
              (s4, [((1,), [3, -i64max + 4])], [[[(INS, (1, -7), True)]]], "err"),
              (s4, [((1,), [3, i64max - 5])], [[[(INS, (1, 10), True), (DEL, (1, 10), True)]]], "ok")]
    s2 = Spec(["int8", "int2"], [0], [Call("count"), Call("sum", 1, "int2")], False)
    cases += [(s2, [((1,), [1, i64max])], [[[(INS, (1, 1), True)]]], "err"),
              (s2, [((1,), [1, i64max])], [[[(INS, (1, -32768), True)]]], "ok")]
    # sum(int8) -> decimal at +-(2^96 - 1) exactly, and one step beyond
    sd = Spec(["int8", "int8"], [0], [Call("count"), Call("sum", 1, "int8", "decimal")], False)
    cases += [(sd, [((1,), [2, DEC_MAX - 7])], [[[(INS, (1, 7), True)]]], "ok"),
              (sd, [((1,), [2, DEC_MAX - 7])], [[[(INS, (1, 8), True)]]], "err"),
              (sd, [((1,), [2, -DEC_MAX + 7])], [[[(INS, (1, -7), True)]]], "ok"),
              (sd, [((1,), [2, -DEC_MAX + 7])], [[[(INS, (1, -8), True)]]], "err")]
    # sum(float4) at f32 max: +max -> inf, -max keeps inf (OrderedFloat checked_add never fails)
    sf = Spec(["int8", "float4"], [0], [Call("count"), Call("sum", 1, "float4")], False)
    cases += [(sf, [((1,), [1, f32max])], [[[(INS, (1, f32max), True)]], [[(INS, (1, -f32max), True)]]], "ok")]
    # narrow min / max states at their type limits
    for t in ("int2", "int4"):
        lo, hi = bounds(t)
        sm = Spec(["int8", t], [0], [Call("count"), Call("min", 1, t), Call("max", 1, t)], True)
        cases += [(sm, [((1,), [2, lo, hi]), ((2,), [1, lo + 1, hi - 1])],
                   [[[(INS, (1, 0), True), (INS, (2, lo), True), (INS, (2, hi), True)]]], "ok")]
    for spec, restored, epochs, outcome in cases:
        want = play_model(spec, epochs, "barrier", restored)
        assert want[-1][0] == outcome, (restored, epochs, want)
        rows = [(INS, key + tuple(st), True) for key, st in restored]
        chunk = make_chunk(spec.out_types, rows)
        assert_same(spec, play_host(spec, cuda, epochs, restored=chunk), want, spec.loose_cols(True),
                    f"restore {[c.pretty() for c in spec.calls]} {restored}")


@pytest.mark.gpu
def test_device_refuses_signatures_the_reference_does_not_define(cuda):
    check_signatures(cuda)
