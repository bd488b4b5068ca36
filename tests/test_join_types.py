"""HashJoin at the type of every key, payload and condition column, on every kernel path: the oracle (CPU) and every
device entry point (GPU) against a typed restatement of the join in Python.

The restatement is independent of oracle/oracle.cc and csrc/.  Values: integers, bool and the temporal types are Python
ints, a decimal is the int of its i128 mantissa, a float is its bit pattern (`OF`, kept as numpy uint32 / uint64 bits)
with OrderedFloat equality: NaN == NaN and -0 == +0 (src/common/src/types/ordered_float.rs:182-219).  Rules:
  * key equality, column by column: both sides non-NULL and equal as Datums (HashKey serialises `normalized()` floats,
    src/common/src/hash/key.rs:400-631), or both NULL where that key is null-safe (hash_join.rs:985-999);
  * the condition `concat_row[lhs] <cmp> concat_row[rhs]` is exact comparison of Python ints; a NULL operand makes it
    false (check_join_condition, hash_join.rs:1362-1384: `unwrap_or(false)`);
  * J(L, R) over the live multisets, as SQL defines the join: inner = the matching pairs; left / right / full outer =
    the pairs plus the NULL-padded unmatched rows of the outer side(s); semi / anti = each row of the kept side that
    has / has no match.  It is projected through `output_indices` (hash_join.rs:337-359);
  * a push's expected net change is J(L', R') - J(L, R), computed per touched key, and is compared with the push's
    net applied output (snapshot.rs `Store::apply_chunk`), both keyed by Datum class;
  * own-side deletes name a live row by pk (join/hash_join.rs:710-713, memcomparable).  The float rule of that
    encoding lives in an external crate the reference tree does not hold, so no reference test pins it; the project
    uses the oracle's rule, Datum class (DESIGN §9), on every backend;
  * every non-NULL output datum is a copy: its bits equal those of an input row of its side.  For inner joins over
    single-match streams (at most one live row per key and side) the emitted rows are predicted exactly: one row per
    matched input row, then eliminate_adjacent_noop_update (src/common/src/array/stream_chunk.rs:331-392), which
    hides a Delete / Insert pair of neighbouring visible rows that are equal as Datums -- also a pair that differs
    only in a column the output does not project.

Comparisons are bit-exact except: the net change and the no-op rule, which are Datum equality by definition; and the
op of a row, compared as its class (Insert / UpdateInsert vs Delete / UpdateDelete): whether a lone U- stays U- depends
on its neighbours in the output, which are the reference's compacted rows but the device's positional ones.
"""
import gc
from collections import Counter

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
from risingwave_b200.stream_chunk import DECIMAL_DTYPE, Column, StreamChunk, decimal_to_int, int_to_decimal, pack_bits, unpack_bits

T_OF = {"bool": abi.T_BOOL, "int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "float4": abi.T_FLOAT32,
        "float8": abi.T_FLOAT64, "date": abi.T_DATE, "time": abi.T_TIME, "timestamp": abi.T_TIMESTAMP,
        "timestamptz": abi.T_TIMESTAMPTZ, "serial": abi.T_SERIAL, "decimal": abi.T_DECIMAL}
NP_OF = {"bool": np.uint8, "int2": np.int16, "int4": np.int32, "int8": np.int64, "date": np.int32, "time": np.int64,
         "timestamp": np.int64, "timestamptz": np.int64, "serial": np.int64}
FLOAT_NP = {"float4": (np.float32, np.uint32), "float8": (np.float64, np.uint64)}
INS, DEL, UD, UI = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT
J = {"inner": abi.JOIN_INNER, "left_outer": abi.JOIN_LEFT_OUTER, "right_outer": abi.JOIN_RIGHT_OUTER,
     "full_outer": abi.JOIN_FULL_OUTER, "left_semi": abi.JOIN_LEFT_SEMI, "left_anti": abi.JOIN_LEFT_ANTI,
     "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI}
CMP_NAME = {abi.CMP_LT: "less_than", abi.CMP_LE: "less_than_or_equal", abi.CMP_GT: "greater_than",
            abi.CMP_GE: "greater_than_or_equal", abi.CMP_EQ: "equal", abi.CMP_NE: "not_equal"}
DEC_MAX = (1 << 127) - 1
CHUNK_LENGTHS = [1, 7, 8, 9, 31, 32, 33, 1023, 1024, 1025, 4097]


# ------------------------------------------------------------------------------------------ values
class OF:
    """a float datum as its bits; equal and hashed as OrderedFloat (NaN == NaN, -0 == +0)"""
    __slots__ = ("t", "bits")

    def __init__(self, t, bits):
        self.t, self.bits = t, int(bits)

    def value(self):
        f, u = FLOAT_NP[self.t]
        return float(np.array([self.bits], dtype=u).view(f)[0])

    def cls(self):
        v = self.value()
        return "nan" if v != v else v + 0.0

    def __eq__(self, other):
        return isinstance(other, OF) and self.cls() == other.cls()

    def __hash__(self):
        return hash(self.cls())

    def __repr__(self):
        return f"{self.t}:{self.bits:#x}"


def fl(t, v):
    f, u = FLOAT_NP[t]
    return OF(t, np.array([v], dtype=f).view(u)[0])


def exact(v):
    return ("f", v.t, v.bits) if isinstance(v, OF) else v


def exact_row(row):
    return tuple(exact(v) for v in row)


def float_classes(t):
    """classes of equal Datums: +-0, NaN (sign bit clear / set, two payloads, a signalling one), +-inf, the smallest
    subnormal of the width, and values whose f32 -> f64 widening is exact"""
    if t == "float4":
        nans = [0x7fc00000, 0xffc00000, 0x7fc00001, 0xffc12345, 0x7f800001]
        zeros, inf, sub = [0x00000000, 0x80000000], 0x7f800000, 0x00000001
    else:
        nans = [0x7ff8000000000000, 0xfff8000000000000, 0x7ff8000000000001, 0xfff8000000abcdef, 0x7ff0000000000001]
        zeros, inf, sub = [0x0000000000000000, 0x8000000000000000], 0x7ff0000000000000, 0x0000000000000001
    sign = 1 << (31 if t == "float4" else 63)
    out = [[OF(t, b) for b in zeros], [OF(t, b) for b in nans], [OF(t, inf)], [OF(t, inf | sign)], [OF(t, sub)],
           [OF(t, sub | sign)]]
    return out + [[fl(t, v)] for v in (1.5, -2.25, 1e-3 if t == "float8" else 16777216.0, 3.0e38)]


def int_edges(t):
    if t == "bool":
        return [0, 1]
    if t == "date":
        return [-(1 << 31), -(1 << 31) + 1, -1, 0, 1, (1 << 31) - 1]
    if t == "time":
        return [0, 1, 43_200_000_000, 86_399_999_999]
    if t == "decimal":
        return [-DEC_MAX, -1, 0, 1, DEC_MAX]
    b = {"int2": 16, "int4": 32}.get(t, 64)
    lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
    return [lo, lo + 1, -1, 0, 1, hi]


def classes(t, wide=0, rng=None):
    """the value classes a column draws from: the edges, plus `wide` random values of the type"""
    if t in FLOAT_NP:
        cl = float_classes(t)
        if wide:
            cl += [[fl(t, float(x) / 4)] for x in rng.choice(1 << 20, wide, replace=False)]
        return cl
    cl = [[v] for v in int_edges(t)]
    if wide and t not in ("bool",):
        lo = min(int_edges(t))
        hi = max(int_edges(t))
        seen = set(int_edges(t))
        for x in rng.integers(max(lo, -(1 << 62)) // 2, min(hi, 1 << 62) // 2, wide * 2, dtype=np.int64):
            if int(x) not in seen and len(cl) < len(int_edges(t)) + wide:
                seen.add(int(x))
                cl.append([int(x)])
    return cl


# ------------------------------------------------------------------------------------------ chunks
def make_chunk(types, rows):
    """rows: (op, row, visible) -> StreamChunk with validity / visibility only where needed"""
    n = len(rows)
    cols = []
    for k, t in enumerate(types):
        vals = [r[1][k] for r in rows]
        valid = np.array([v is not None for v in vals], dtype=bool)
        if t in FLOAT_NP:
            f, u = FLOAT_NP[t]
            data = np.array([0 if v is None else v.bits for v in vals], dtype=u).view(f)
        elif t == "decimal":
            data = np.zeros(n, DECIMAL_DTYPE)
            for i, v in enumerate(vals):
                data[i] = int_to_decimal(0 if v is None else v)
        else:
            data = np.array([0 if v is None else v for v in vals], dtype=NP_OF[t])
        cols.append(Column(T_OF[t], data, None if valid.all() else valid))
    vis = np.array([r[2] for r in rows], dtype=bool)
    return StreamChunk(np.array([r[0] for r in rows], dtype=np.uint8), cols, None if vis.all() else vis)


def column_values(t, data, valid, n):
    data = np.ascontiguousarray(data)
    if t in FLOAT_NP:
        vals = [OF(t, b) for b in data.view(FLOAT_NP[t][1])]
    elif t == "decimal":
        vals = [decimal_to_int(v) for v in data]
    else:
        vals = [int(v) for v in data]
    if valid is not None:
        vals = [v if ok else None for v, ok in zip(vals, valid)]
    return vals[:n]


def chunk_rows(chunks, types):
    """visible (op, row) of host chunks, in order, floats as their bits"""
    out = []
    for ch in chunks:
        n = ch.capacity()
        cols = [column_values(t, c.data, c.valid, n) for t, c in zip(types, ch.columns)]
        for i in range(n):
            if ch.vis is None or ch.vis[i]:
                out.append((int(ch.ops[i]), tuple(c[i] for c in cols)))
    return out


def signed_net(rows):
    c = Counter()
    for op, row in rows:
        c[row] += 1 if op in (INS, UI) else -1
    return {k: v for k, v in c.items() if v}


def emitted_exact(rows):
    return Counter((op in (INS, UI), exact_row(row)) for op, row in rows)


# ------------------------------------------------------------------------------------------ plans
class Plan:
    def __init__(self, name, jt, left, right, keys, pk, null_safe=None, out=None, cond=None, append_only=False,
                 kernel=None, single_match_ok=True):
        """left / right: column type names; keys / pk: column indices, the same on both sides; cond: (cmp, lhs, rhs)"""
        self.name, self.jt, self.types = name, J[jt], (list(left), list(right))
        self.keys, self.pk = list(keys), list(pk)
        self.null_safe = list(null_safe) if null_safe is not None else [False] * len(keys)
        self.cond, self.append_only, self.kernel = cond, append_only, kernel
        self.single_match_ok = single_match_ok
        if self.jt in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
            self.src = [(0, c) for c in range(len(left))]
        elif self.jt in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
            self.src = [(1, c) for c in range(len(right))]
        else:
            self.src = [(0, c) for c in range(len(left))] + [(1, c) for c in range(len(right))]
        self.out = list(range(len(self.src))) if out is None else list(out)
        self.out_types = [self.types[s][c] for s, c in (self.src[i] for i in self.out)]

    def executor(self, be, chunk_size=1024, capacity_hint=16):
        cond = None
        if self.cond is not None:
            cmp_, a, b = self.cond
            cond = f"({CMP_NAME[cmp_]}:boolean ${a}:x ${b}:x)"
        srcs = []
        for s in range(2):
            _, src = MockSource.channel()
            srcs.append(src.into_executor([T_OF[t] for t in self.types[s]], self.pk))
        return HashJoinExecutor(be, self.jt, srcs[0], srcs[1], JoinParams(self.keys, self.pk), JoinParams(self.keys, self.pk),
                                self.null_safe, self.out, cond, self.append_only, chunk_size, capacity_hint=capacity_hint)

    def __repr__(self):
        return self.name


def close(ex):
    """destroy the handle now: a unified-table handle reserves its log segments until then"""
    if getattr(ex, "_h", None):
        ex.backend._join_destroy(ex._h)
        ex._h = None
    gc.collect()


LT, LE, GT, GE, EQ, NE = abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE
UNI, SLOW, W8, FUSED, SERIAL = "uni_hot_kernel", "uni_slow_kernel", "join_inner_w8p_kernel", "join_inner_fused_kernel", "join_serial_kernel"


def plans():
    ps = []
    # unified table: INNER, one 8-byte non-float key, <= 4 eight-byte columns per side, no condition; the left input's
    # last column is not projected
    for kt in ("int8", "timestamp", "timestamptz", "time", "serial"):
        ps.append(Plan(f"uni_{kt}", "inner", [kt, "int8", "float8", "int8"], [kt, "int8", "float8"], [0], [1],
                       out=[0, 1, 2, 4, 5, 6], kernel=UNI))
    ps.append(Plan("uni_float8_pk", "inner", ["int8", "float8", "int8"], ["int8", "float8", "float8"], [0], [1], kernel=UNI))
    ps.append(Plan("uni_bitmaps", "inner", ["int8", "int8", "float8", "int8"], ["int8", "int8", "float8"], [0], [1],
                   out=[0, 1, 2, 4, 5, 6], kernel=SLOW))
    ps.append(Plan("w8", "inner", ["int8", "int8", "float8", "int8", "float8", "int8"], ["int8", "int8", "float8", "int8", "float8"],
                   [0], [1], out=[0, 1, 2, 3, 4, 6, 7, 8, 9, 10], kernel=W8))
    # fused: a narrow or float key, a decimal / bool / int2 payload
    for kt in ("bool", "int2", "int4", "date", "float4", "float8"):
        ps.append(Plan(f"fused_{kt}", "inner", [kt, "int8", "float4", "decimal"], [kt, "int8", "int2", "bool", "float8"], [0], [1],
                       out=[0, 1, 2, 3, 5, 6, 7, 8], kernel=FUSED, single_match_ok=kt != "bool"))
    ps.append(Plan("fused_multi_key", "inner", ["int2", "bool", "date", "float4", "int8", "float8"],
                   ["int2", "bool", "date", "float4", "int8", "float4"], [0, 1, 2, 3], [4], null_safe=[True, False, True, False],
                   kernel=FUSED))
    ps.append(Plan("fused_cond_int2_int8", "inner", ["int8", "int8", "int2"], ["int8", "int8", "int8"], [0], [1], cond=(LE, 2, 5),
                   kernel=FUSED))
    ps.append(Plan("fused_cond_date", "inner", ["int4", "int8", "date"], ["int4", "int8", "date"], [0], [1], cond=(GT, 5, 2),
                   kernel=FUSED))
    ps.append(Plan("fused_float8_pk", "inner", ["int4", "float8", "float4"], ["int4", "float8", "int8"], [0], [1], kernel=FUSED))
    # generic: the seven other join types, and an append-only inner join with pk in the join key on both sides
    for jt, kt, cond in (("left_outer", "float8", None), ("right_outer", "int2", (NE, 3, 7)), ("full_outer", "date", None),
                         ("left_semi", "bool", None), ("left_anti", "float4", (GE, 7, 3)), ("right_semi", "int8", None),
                         ("right_anti", "timestamp", None)):
        ps.append(Plan(f"generic_{jt}_{kt}", jt, [kt, "int8", "float4", "int2"], [kt, "int8", "float8", "int8"], [0], [1],
                       cond=cond, kernel=SERIAL, single_match_ok=kt != "bool"))
    ps.append(Plan("generic_left_outer_float8_pk", "left_outer", ["int4", "float8", "float4"], ["int4", "float8", "int8"], [0], [1],
                   kernel=SERIAL))
    ps.append(Plan("generic_append_only", "inner", ["int8", "float8", "decimal"], ["int8", "int2", "float4"], [0], [0],
                   append_only=True, kernel=SERIAL))
    return ps


PLANS = plans()
BY_NAME = {p.name: p for p in PLANS}
INNER_SINGLE = [p for p in PLANS if p.jt == abi.JOIN_INNER and not p.append_only and p.single_match_ok]


# ------------------------------------------------------------------------------------------ the restatement
class Model:
    """the live multisets of both sides and J(L, R) per key"""

    def __init__(self, plan):
        self.p = plan
        self.live = ({}, {})  # side -> group key -> [rows]
        self.seen = (set(), set())  # exact projections of every row pushed, per side (payload bits)
        self.proj_cols = ([], [])
        for o, i in enumerate(plan.out):
            s, c = plan.src[i]
            self.proj_cols[s].append((o, c))

    def gkey(self, side, row):
        return tuple(row[k] for k in self.p.keys)

    def cond_ok(self, l, r):
        if self.p.cond is None:
            return True
        cmp_, a, b = self.p.cond
        cat = l + r
        x, y = cat[a], cat[b]
        if x is None or y is None:
            return False
        return {LT: x < y, LE: x <= y, GT: x > y, GE: x >= y, EQ: x == y, NE: x != y}[cmp_]

    def match(self, l, r):
        for i, k in enumerate(self.p.keys):
            a, b = l[k], r[k]
            if a is None or b is None:
                if not (a is None and b is None and self.p.null_safe[i]):
                    return False
            elif a != b:
                return False
        return self.cond_ok(l, r)

    def project(self, nat):
        return tuple(nat[i] for i in self.p.out)

    def join(self, L, R):
        T, out = self.p.jt, Counter()
        nl, nr = (None,) * len(self.p.types[0]), (None,) * len(self.p.types[1])
        lm, rm = [False] * len(L), [False] * len(R)
        for i, l in enumerate(L):
            for j, r in enumerate(R):
                if self.match(l, r):
                    lm[i] = rm[j] = True
                    if T in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER):
                        out[self.project(l + r)] += 1
        for i, l in enumerate(L):
            if (T in (abi.JOIN_LEFT_OUTER, abi.JOIN_FULL_OUTER) and not lm[i]):
                out[self.project(l + nr)] += 1
            if (T == abi.JOIN_LEFT_SEMI and lm[i]) or (T == abi.JOIN_LEFT_ANTI and not lm[i]):
                out[self.project(l)] += 1
        for j, r in enumerate(R):
            if T in (abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER) and not rm[j]:
                out[self.project(nl + r)] += 1
            if (T == abi.JOIN_RIGHT_SEMI and rm[j]) or (T == abi.JOIN_RIGHT_ANTI and not rm[j]):
                out[self.project(r)] += 1
        return out

    def j_groups(self, groups):
        tot = Counter()
        for g in groups:
            tot.update(self.join(self.live[0].get(g, []), self.live[1].get(g, [])))
        return tot

    def remove(self, side, row):
        """the newest live row with an equal pk (Datum class) in the row's key group"""
        rows = self.live[side].get(self.gkey(side, row), [])
        pk = tuple(row[k] for k in self.p.pk)
        for i in range(len(rows) - 1, -1, -1):
            if tuple(rows[i][k] for k in self.p.pk) == pk:
                return rows.pop(i)
        raise AssertionError(f"inconsistent stream: delete of a row that is not live: {row}")

    def predict_emitted(self, side, rows):
        """inner join, single match: one output row per matched visible input row, then the no-op elimination"""
        em = []
        for op, row, vis in rows:
            if not vis:
                continue
            for m in self.live[1 - side].get(self.gkey(side, row), []):
                if self.match(row, m) if side == 0 else self.match(m, row):
                    em.append((op in (INS, UI), self.project(row + m if side == 0 else m + row)))
        hidden, prev = set(), None
        for i in range(len(em)):  # stream_chunk.rs:331-392, over the visible rows
            if prev is not None and em[prev][0] != em[i][0] and em[prev][1] == em[i][1]:
                hidden.update((prev, i))
                prev = None
            else:
                prev = i
        return Counter((ins, exact_row(r)) for i, (ins, r) in enumerate(em) if i not in hidden)

    def push(self, side, rows, predict=False):
        """-> (expected signed net change by Datum class, predicted emitted multiset or None)"""
        emitted = self.predict_emitted(side, rows) if predict else None
        touched = {self.gkey(side, r) for _, r, vis in rows if vis}
        before = self.j_groups(touched)
        for op, row, vis in rows:
            self.seen[side].add(tuple(exact(row[c]) for _, c in self.proj_cols[side]))
            if not vis:
                continue
            if op in (INS, UI):
                self.live[side].setdefault(self.gkey(side, row), []).append(row)
            else:
                self.remove(side, row)
        after = self.j_groups(touched)
        net = {k: after.get(k, 0) - before.get(k, 0) for k in set(after) | set(before)}
        return {k: v for k, v in net.items() if v}, emitted

    def live_rows(self, side):
        return Counter(exact_row(r) for g in self.live[side].values() for r in g)

    def check_bits(self, out_rows):
        """every non-NULL output datum carries the bits of an input row of its side"""
        for _, row in out_rows:
            for s in range(2):
                part = tuple(exact(row[o]) for o, _ in self.proj_cols[s])
                if part and any(v is not None for v in part):
                    assert part in self.seen[s], f"output row {row}: side {s} part {part} is no input row's bits"


# ------------------------------------------------------------------------------------------ streams
class Gen:
    """consistent two-sided change stream (StreamGen style): deletes and updates name a live row; updates change the
    key, a payload, a payload only within its Datum class (-0 <-> +0, one NaN encoding -> another), or 0 -> the smallest
    subnormal.  single_match: at most one live row per key class and side."""

    def __init__(self, plan, seed, wide=0, null_frac=0.0, vis_frac=1.0, payload_null=0.1, single_match=False):
        self.p, self.rng = plan, np.random.default_rng(seed)
        self.single, self.null_frac, self.vis_frac, self.payload_null = single_match, null_frac, vis_frac, payload_null
        self.live = ([], [])
        self.next_pk = [0, 0]
        self.cls = [[classes(t, wide if k in plan.keys else 0, self.rng) for k, t in enumerate(plan.types[s])] for s in range(2)]
        for s in range(2):  # key columns of both sides draw from the same classes
            for k in plan.keys:
                self.cls[s][k] = self.cls[0][k]

    def pick(self, side, k):
        cl = self.cls[side][k]
        c = cl[int(self.rng.integers(len(cl)))]
        return c[int(self.rng.integers(len(c)))]

    def key_taken(self, side, key):
        return any(tuple(r[k] for k in self.p.keys) == key for r in self.live[side])

    def new_key(self, side):
        for _ in range(30):
            key = tuple(None if self.rng.random() < self.null_frac else self.pick(side, k) for k in self.p.keys)
            if self.p.append_only or self.single:
                if None in key or self.key_taken(side, key):
                    continue
            return key
        return None

    def pk_value(self, side, k):
        t = self.p.types[side][k]
        v = self.next_pk[side]
        self.next_pk[side] += 1
        return fl(t, v + 0.5) if t in FLOAT_NP else v

    def new_row(self, side, key):
        row = []
        for k, t in enumerate(self.p.types[side]):
            if k in self.p.keys:
                row.append(key[self.p.keys.index(k)])
            elif k in self.p.pk:
                row.append(self.pk_value(side, k))
            else:
                row.append(None if self.rng.random() < self.payload_null else self.pick(side, k))
        return tuple(row)

    def changed(self, side, old):
        """the U+ row of an update of `old`"""
        r = self.rng.random()
        payload = [k for k in range(len(old)) if k not in self.p.keys and k not in self.p.pk]
        if r < 0.3 and not self.p.append_only:
            key = self.new_key(side)
            if key is not None:
                new = list(old)
                for i, k in enumerate(self.p.keys):
                    new[k] = key[i]
                return tuple(new)
        new = list(old)
        if not payload:
            return tuple(new)
        k = payload[int(self.rng.integers(len(payload)))]
        t = self.p.types[side][k]
        if t in FLOAT_NP and r < 0.75 and old[k] is not None:  # same class, other bits (or 0 -> subnormal)
            same = [c for c in self.cls[side][k] if old[k] in c][0]
            if len(same) > 1:
                new[k] = same[int(self.rng.integers(len(same)))]
            elif old[k].cls() == 0.0:
                new[k] = [c for c in float_classes(t)][4][0]
            return tuple(new)
        new[k] = self.pick(side, k)
        return tuple(new)

    def chunk(self, side, n, p_delete=0.2, p_update=0.2):
        rows, live = [], self.live[side]
        while len(rows) < n:
            x = self.rng.random()
            if self.p.append_only:
                x = 1.0
            if live and x < p_delete:
                rows.append((DEL, live.pop(int(self.rng.integers(len(live)))), True))
            elif live and x < p_delete + p_update and len(rows) + 2 <= n:
                old = live.pop(int(self.rng.integers(len(live))))
                new = self.changed(side, old)
                rows += [(UD, old, True), (UI, new, True)]
                live.append(new)
            else:
                key = self.new_key(side)
                if key is None:  # every key class is taken on this side
                    if live and not self.p.append_only:
                        rows.append((DEL, live.pop(int(self.rng.integers(len(live)))), True))
                        continue
                    break
                row = self.new_row(side, key)
                vis = self.rng.random() < self.vis_frac
                rows.append((INS, row, vis))
                if vis:
                    live.append(row)
        return rows


def stream(plan, seed, lengths, wide=0, single_match=False, null_frac=None, vis_frac=None):
    """(side, rows) pushes of the given lengths, sides alternating at random"""
    bitmaps = plan.kernel == SLOW
    g = Gen(plan, seed, wide=wide, single_match=single_match, payload_null=0.0 if plan.kernel in (UNI, W8) else 0.1,
            null_frac=(0.08 if any(plan.null_safe) or plan.jt != abi.JOIN_INNER else 0.0) if null_frac is None else null_frac,
            vis_frac=(0.9 if bitmaps else 1.0) if vis_frac is None else vis_frac)
    out = []
    for n in lengths:
        side = int(g.rng.integers(2))
        rows = g.chunk(side, n)
        if rows:
            out.append((side, rows))
    return out


def lengths_for(plan):
    """chunk lengths: every edge of the kernels' row grouping for plans whose keys spread; narrow keys chain instead"""
    narrow = any(plan.types[0][k] == "bool" for k in plan.keys) or len(plan.keys) > 1
    return [1, 7, 8, 9, 31, 32, 33, 64, 9, 33] if narrow else CHUNK_LENGTHS[:7] + [200, 9, 1023, 1024, 1025, 33]


def wide_for(plan):
    return 0 if any(plan.types[0][k] == "bool" for k in plan.keys) else 400


# ------------------------------------------------------------------------------------------ driving a backend
def host_push(ex, plan):
    def push(side, ch):
        return chunk_rows(ex.eq_join_oneside(side, ch), plan.out_types)
    return push


def drive(plan, push, pushes, exact_emit=False, label=""):
    m = Model(plan)
    for i, (side, rows) in enumerate(pushes):
        want, emit = m.push(side, rows, predict=exact_emit)
        got = push(side, make_chunk(plan.types[side], rows))
        net = signed_net(got)
        assert net == want, (f"{label} {plan} push {i} (side {side}, {len(rows)} rows): net change differs\n"
                             f" only in output {dict(Counter(net) - Counter(want))}\n only expected {dict(Counter(want) - Counter(net))}")
        m.check_bits(got)
        if exact_emit:
            e = emitted_exact(got)
            assert e == emit, f"{label} {plan} push {i}: emitted rows differ\n got-only {e - emit}\n expected-only {emit - e}"
    return m


# ------------------------------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("plan", PLANS, ids=str)
def test_oracle_matches_restatement(oracle, plan):
    ex = plan.executor(oracle, chunk_size=3 if plan.jt != abi.JOIN_INNER else 1024)
    drive(plan, host_push(ex, plan), stream(plan, 7, lengths_for(plan), wide=wide_for(plan)), label="oracle")


@pytest.mark.parametrize("plan", INNER_SINGLE, ids=str)
def test_oracle_single_match_emits_the_predicted_rows(oracle, plan):
    ex = plan.executor(oracle)
    pushes = stream(plan, 11, [1, 8, 9, 33, 200, 400, 31, 1024, 64, 300], wide=wide_for(plan), single_match=True)
    drive(plan, host_push(ex, plan), pushes, exact_emit=True, label="oracle")


def noop_pushes(plan):
    """one key on both sides; then U-/U+ pairs of the left row that change a float payload only within its class
    (-0 -> +0, NaN -> NaN of other bits), a column the output does not project, and 0 -> the smallest subnormal.
    -> [(side, rows, visible output rows expected)]"""
    L, R = plan.types
    fk = [k for k, t in enumerate(L) if t in FLOAT_NP and k not in plan.keys and k not in plan.pk][0]
    ft = L[fk]
    key = {"bool": 1, "float4": fl("float4", 1.5), "float8": fl("float8", 1.5)}

    def row(side, pk, f=None):
        r = []
        for k, t in enumerate(plan.types[side]):
            if k in plan.keys:
                r.append(key.get(t, 5))
            elif k in plan.pk:
                r.append(fl(t, pk) if t in FLOAT_NP else pk)
            elif side == 0 and k == fk:
                r.append(f)
            else:
                r.append(fl(t, 2.0) if t in FLOAT_NP else (1 if t == "bool" else 3))
        return tuple(r)
    sub, zero, nzero = OF(ft, 1), OF(ft, 0), fl(ft, -0.0)
    nan_a, nan_b = float_classes(ft)[1][0], float_classes(ft)[1][3]
    l0, l1, l2, l3 = row(0, 1, nzero), row(0, 1, zero), row(0, 1, nan_a), row(0, 1, nan_b)
    pushes = [(1, [(INS, row(1, 7), True)], None), (0, [(INS, l0, True)], None),
              (0, [(UD, l0, True), (UI, l1, True)], 0),
              (0, [(UD, l1, True), (UI, l2, True)], None),
              (0, [(UD, l2, True), (UI, l3, True)], 0),
              (0, [(UD, l3, True), (UI, l1, True)], None),
              (0, [(UD, l1, True), (UI, row(0, 1, sub), True)], 2)]
    if plan.kernel == SLOW:  # an invisible row behind every left push gives the chunk a visibility bitmap
        pushes = [(s, rows + ([(INS, row(0, 1000 + i, zero), False)] if s == 0 else []), n) for i, (s, rows, n) in enumerate(pushes)]
    hidden_col = [k for k in range(len(L)) if plan.src.index((0, k)) not in plan.out] if (0, 0) in plan.src else []
    if hidden_col:
        k = hidden_col[0]
        old = row(0, 1, sub)
        new = tuple((fl(L[k], 99.0) if L[k] in FLOAT_NP else 99) if i == k else v for i, v in enumerate(old))
        pushes.append((0, [(UD, old, True), (UI, new, True)], 0))
    return pushes


# (not a full outer join: there the pair's two rows are split by the other side's NULL-padded row going and coming back)
NOOP_PLANS = [BY_NAME[n] for n in ("uni_int8", "uni_bitmaps", "w8", "fused_int4", "fused_float8", "generic_left_outer_float8")]


def run_noop(plan, push, label):
    m = Model(plan)
    for i, (side, rows, n_vis) in enumerate(noop_pushes(plan)):
        want, _ = m.push(side, rows)
        got = push(side, make_chunk(plan.types[side], rows))
        assert signed_net(got) == want, f"{label} {plan} push {i}"
        m.check_bits(got)
        if n_vis is not None:
            assert len(got) == n_vis, f"{label} {plan} push {i}: {len(got)} visible rows, want {n_vis}: {got}"


@pytest.mark.parametrize("plan", NOOP_PLANS, ids=str)
def test_oracle_noop_pairs_by_datum_equality(oracle, plan):
    ex = plan.executor(oracle)
    run_noop(plan, host_push(ex, plan), "oracle")


def float4_payload_pushes():
    reps = [v for c in float_classes("float4") for v in c]
    return [(1, [(INS, (5, 0, 1, 1, fl("float8", 1.0)), True)]),
            (0, [(INS, (5, i, v, None), True) for i, v in enumerate(reps)]),
            (0, [(DEL, (5, i, v, None), True) for i, v in enumerate(reps)])]


def test_oracle_carries_float4_payload_bits(oracle):
    """a float4 signalling NaN, and every other float4 edge, leave the join with the bits they came with"""
    plan = BY_NAME["fused_int4"]
    drive(plan, host_push(plan.executor(oracle), plan), float4_payload_pushes(), exact_emit=True, label="oracle")


def float_pk_pushes(plan):
    """left rows with pk -0.0 and NaN, deleted by +0.0 and another NaN: the same rows by Datum class"""
    L, R = plan.types
    pt = L[plan.pk[0]]
    k = 4

    def row(side, pk, pay):
        return tuple(k if c in plan.keys else (pk if c in plan.pk else pay(t)) for c, t in enumerate(plan.types[side]))
    pay = lambda t: fl(t, 2.5) if t in FLOAT_NP else 6
    nan = float_classes(pt)[1]
    right = row(1, fl(R[plan.pk[0]], 100.0), pay)
    a, b = row(0, fl(pt, -0.0), pay), row(0, nan[0], pay)
    a2, b2 = row(0, fl(pt, 0.0), pay), row(0, nan[3], pay)
    right2 = row(1, fl(R[plan.pk[0]], 101.0), pay)
    return [(1, [(INS, right, True)]), (0, [(INS, a, True), (INS, b, True)]), (0, [(DEL, a2, True), (DEL, b2, True)]),
            (1, [(INS, right2, True)]), (0, [(INS, a, True)]), (0, [(DEL, a2, True)])]


FLOAT_PK_PLANS = [BY_NAME[n] for n in ("uni_float8_pk", "fused_float8_pk", "generic_left_outer_float8_pk")]


@pytest.mark.parametrize("plan", FLOAT_PK_PLANS, ids=str)
def test_oracle_float_pk_delete_by_datum_class(oracle, plan):
    ex = plan.executor(oracle)
    m = drive(plan, host_push(ex, plan), float_pk_pushes(plan), label="oracle")
    assert not m.live_rows(0)


def test_oracle_float_keys_match_by_class(oracle):
    """-0 meets +0 and every NaN meets every NaN, at both widths"""
    for name in ("fused_float4", "fused_float8"):
        plan = BY_NAME[name]
        t = plan.types[0][0]
        ex = plan.executor(oracle)
        m = Model(plan)
        for side, reps in ((1, [c[0] for c in float_classes(t)]), (0, [c[-1] for c in float_classes(t)])):
            rows = [(INS, tuple(v if k == 0 else (100 * side + i if k == 1 else None) for k in range(len(plan.types[side]))), True)
                    for i, v in enumerate(reps)]
            want, _ = m.push(side, rows)
            got = chunk_rows(ex.eq_join_oneside(side, make_chunk(plan.types[side], rows)), plan.out_types)
            assert signed_net(got) == want
        assert len(got) == len(float_classes(t)), got  # the second side found one match per class


def refusal_cases():
    """(left types, right types, cond, accepted?)"""
    c = []
    for a, b, ok in (("int2", "int8", True), ("int4", "int2", True), ("date", "date", True), ("timestamp", "timestamp", True),
                     ("bool", "bool", True), ("date", "timestamptz", False), ("date", "timestamp", False), ("bool", "int8", False),
                     ("time", "int8", False), ("serial", "int8", False), ("int8", "timestamp", False), ("float4", "float4", False),
                     ("float8", "int8", False), ("decimal", "decimal", False)):
        c.append(([ "int8", "int8", a], ["int8", "int8", b], (LT, 2, 5), ok))
    return c


def check_refusals(be):
    for left, right, cond, ok in refusal_cases():
        plan = Plan("cond", "inner", left, right, [0], [1], cond=cond)
        if ok:
            close(plan.executor(be))
        else:
            with pytest.raises(abi.RwError) as e:
                plan.executor(be)
            assert e.value.code == abi.RW_ERR_UNSUPPORTED, (left[2], right[2])
    plan = Plan("cond", "inner", ["int8", "int8"], ["int8", "int8"], [0], [1], cond=(LT, 0, 4))
    with pytest.raises(abi.RwError) as e:
        plan.executor(be)
    assert e.value.code == abi.RW_ERR_INVALID


def test_oracle_refuses_what_the_device_refuses(oracle):
    check_refusals(oracle)


def test_restatement_float_classes():
    for t in FLOAT_NP:
        cl = float_classes(t)
        for i, a in enumerate(cl):
            for b in a:
                assert all((b == x) == (j == i) for j, c in enumerate(cl) for x in c)
    assert exact(fl("float4", -0.0)) != exact(fl("float4", 0.0)) and fl("float4", -0.0) == fl("float4", 0.0)


# ------------------------------------------------------------------------------------------ GPU: every device entry point
WIDTH = {"bool": 1, "int2": 2, "int4": 4, "date": 4, "float4": 4, "decimal": 16}
PATHS = ["host", "host_async", "device", "device_async", "device_counted"]


def device_chunk(ch, pad=0):
    """StreamChunk -> device.DeviceChunk; `pad` rows of zeros behind the chunk's rows (a counted push's capacity)"""
    import torch
    from risingwave_b200 import device
    n = ch.capacity()

    def up(a):
        a = np.ascontiguousarray(a)
        if pad:
            a = np.concatenate([a, np.zeros(pad, a.dtype)])
        return torch.from_numpy(a.view(np.int64) if a.dtype == DECIMAL_DTYPE else a).cuda()

    def bits(b):
        return None if b is None else torch.from_numpy(pack_bits(np.concatenate([b, np.zeros(pad, bool)])).view(np.int64)).cuda()
    dc = device.DeviceChunk(up(ch.ops), [], [])
    # (set after the constructor: a decimal column has no torch dtype and travels as int64 pairs)
    dc.cols, dc.types = [up(c.data) for c in ch.columns], ch.types()
    dc.validity = [bits(c.valid) for c in ch.columns]
    dc.visibility = bits(ch.vis)
    assert n >= 1
    return dc


def view_rows(view, types):
    import torch
    from risingwave_b200 import device
    n = view.n_rows
    if n == 0:
        return []
    ops = view.ops().cpu().numpy()
    vis = view.visible()
    cols = []
    for k, t in enumerate(types):
        w = WIDTH.get(t, 8)
        buf = torch.empty(n * w, dtype=torch.uint8, device="cuda")
        device._d2d(buf.data_ptr(), view.col_ptrs[k], n * w)
        dt = DECIMAL_DTYPE if t == "decimal" else (FLOAT_NP[t][0] if t in FLOAT_NP else NP_OF[t])
        data = buf.cpu().numpy().view(dt)
        valid = None
        if view.valid_ptrs[k]:
            words = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda")
            device._d2d(words.data_ptr(), view.valid_ptrs[k], words.numel() * 8)
            valid = unpack_bits(words.cpu().numpy().view(np.uint64), n)
        cols.append(Column(T_OF[t], data, valid))
    return chunk_rows([StreamChunk(ops, cols, None if vis is None else vis.cpu().numpy())], types)


def gpu_push(path, ex, plan):
    import torch
    from risingwave_b200 import device
    if path == "host":
        return host_push(ex, plan)

    def push(side, ch):
        if path == "host_async":
            ex.eq_join_oneside_launch(side, ch)
            return chunk_rows(ex.eq_join_oneside_collect(), plan.out_types)
        if path == "device":
            return view_rows(device.join_push_device(ex, side, device_chunk(ch)), plan.out_types)
        if path == "device_async":
            device.join_push_device_async(ex, side, device_chunk(ch))
            return view_rows(device.join_collect(ex), plan.out_types)
        count = torch.tensor([ch.capacity()], dtype=torch.int64, device="cuda")
        return view_rows(device.join_push_device(ex, side, device_chunk(ch, pad=5), n_rows_dev=count.data_ptr()), plan.out_types)
    return push


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("plan", PLANS, ids=str)
def test_device_matches_restatement(cuda, plan, path):
    """the net change of every push by Datum class, and every output datum's bits; the host push also cuts its output
    into 3-row chunks (non-inner plans) and the stream outgrows the row_capacity_hint of 16 keys"""
    chunk_size = 3 if plan.jt != abi.JOIN_INNER and path == "host" else 1024
    ex = plan.executor(cuda, chunk_size=chunk_size)
    try:
        drive(plan, gpu_push(path, ex, plan), stream(plan, 7, lengths_for(plan), wide=wide_for(plan)), label=path)
    finally:
        close(ex)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("plan", INNER_SINGLE, ids=str)
def test_device_single_match_emits_the_oracles_rows(cuda, oracle, plan, path):
    """single-match inner streams: the emitted rows, keyed by exact bits, are the restatement's prediction and the
    oracle's.  The unified and w8 kernels write row r of the output for input row r, so this holds for chunks of any
    length; the fused kernel reserves its output per 256-row tile in the order the tiles finish, so a U-/U+ pair that
    straddles two tiles can land apart and stay visible (the net change is the same): its pushes stay within a tile."""
    lengths = [1, 8, 9, 33, 200, 400, 31, 1024, 64, 300]
    if plan.kernel == FUSED:  # one 256-row tile: the fused kernel orders its output tile by tile (DESIGN §9)
        lengths = [min(n, 256) for n in lengths]
    pushes = stream(plan, 11, lengths, wide=wide_for(plan), single_match=True)
    ex, ox = plan.executor(cuda), plan.executor(oracle)
    try:
        gp, op = gpu_push(path, ex, plan), host_push(ox, plan)
        m = Model(plan)
        for i, (side, rows) in enumerate(pushes):
            _, emit = m.push(side, rows, predict=True)
            ch = make_chunk(plan.types[side], rows)
            got, want = emitted_exact(gp(side, ch)), emitted_exact(op(side, ch))
            assert want == emit, f"oracle {plan} push {i}"
            assert got == want, f"{path} {plan} push {i}: device-only {got - want}\n oracle-only {want - got}"
    finally:
        close(ex)
        close(ox)


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("plan", NOOP_PLANS, ids=str)
def test_device_noop_pairs_by_datum_equality(cuda, plan, path):
    """a U-/U+ pair that changes a float payload only from -0 to +0, or from one NaN to another, or a column the output
    does not project, is hidden; 0 -> the smallest subnormal stays visible"""
    ex = plan.executor(cuda)
    try:
        run_noop(plan, gpu_push(path, ex, plan), path)
    finally:
        close(ex)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("plan", FLOAT_PK_PLANS, ids=str)
def test_device_float_pk_delete_one_answer(cuda, plan, path):
    """a delete whose float8 pk differs from the stored one only in bits (-0 / +0, NaN encodings) removes that row on
    the unified, fused and generic paths alike"""
    ex = plan.executor(cuda)
    try:
        m = drive(plan, gpu_push(path, ex, plan), float_pk_pushes(plan), label=path)
        assert not m.live_rows(0)
        assert not chunk_rows(ex.snapshot(0), plan.types[0])
    finally:
        close(ex)


@pytest.mark.gpu
def test_device_carries_float4_payload_bits(cuda):
    plan = BY_NAME["fused_int4"]
    for path in PATHS:
        ex = plan.executor(cuda)
        try:
            drive(plan, gpu_push(path, ex, plan), float4_payload_pushes(), exact_emit=True, label=path)
        finally:
            close(ex)


def can_match(plan, row):
    return all(row[k] is not None or ns for k, ns in zip(plan.keys, plan.null_safe))


@pytest.mark.gpu
@pytest.mark.parametrize("plan", [p for p in PLANS if not p.append_only], ids=str)
def test_device_snapshot_is_the_live_rows_bit_for_bit(cuda, plan):
    """rwgpu_join_snapshot returns the restatement's live rows of each side, every datum with its input bits.  Rows
    with a NULL in a key column that is not null-safe can never match; the device does not keep them as state (a delete
    of one is answered from the row itself), so they are not in its snapshot.  The append-only plan is left out: there
    a matched row leaves the state (hash_join.rs append_only_optimize)."""
    ex = plan.executor(cuda)
    try:
        m = drive(plan, host_push(ex, plan), stream(plan, 5, lengths_for(plan)[:9], wide=wide_for(plan)), label="host")
        for side in range(2):
            got = Counter(exact_row(r) for _, r in chunk_rows(ex.snapshot(side), plan.types[side]))
            want = Counter({r: n for r, n in m.live_rows(side).items() if can_match(plan, r)})
            assert got == want, f"{plan} side {side}"
    finally:
        close(ex)


@pytest.mark.gpu
@pytest.mark.parametrize("plan", PLANS, ids=str)
def test_plan_runs_its_kernel_path(cuda, plan):
    """each plan above runs the kernel it is meant to test: a plan cannot drift to another path unnoticed"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    ex = plan.executor(cuda)
    try:
        pushes = stream(plan, 3, [64, 64, 64, 64, 64], wide=wide_for(plan))
        side, rows = pushes[0]  # (the first push loads the module outside the trace)
        ex.eq_join_oneside(side, make_chunk(plan.types[side], rows))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for side, rows in pushes[1:]:
                ex.eq_join_oneside(side, make_chunk(plan.types[side], rows))
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()} | {e.key for e in prof.key_averages()}
        assert any(plan.kernel in n for n in names), (plan.kernel, sorted(n for n in names if "kernel" in n))
    finally:
        close(ex)


@pytest.mark.gpu
def test_device_refuses_what_the_oracle_refuses(cuda):
    check_refusals(cuda)
