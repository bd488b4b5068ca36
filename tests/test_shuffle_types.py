"""Hash shuffle at the type of every key and payload column, on every partition path: the oracle (CPU) and every device
entry point (GPU) against a typed restatement of the dispatcher in Python.

The restatement is independent of oracle/oracle.cc and csrc/: plain Python integers, `zlib.crc32` and `struct`.  A
datum is a Python int (a float is its bit pattern, a decimal the int of its i128 mantissa) or None for NULL.  Rules:
  * the bytes a datum feeds to the hasher, Array::hash_at (src/common/src/array/mod.rs:280-288) -> hash_scalar
    (src/common/src/types/scalar_impl.rs:47-49): int2 / int4 / int8 / serial / timestamptz as native little-endian
    bytes, bool as one byte, float4 / float8 as the 8 bytes of raw_double_bits (ordered_float.rs:852-870), NULL as
    NULL_VAL_FOR_HASH = 0xfffffff0u32 (array/mod.rs:97);
  * date / time / timestamp / decimal hash through chrono / rust_decimal, which the reference tree does not hold.  For
    them this file pins the PROJECT's rule, "the ABI value's little-endian bytes" (DESIGN §2), so that a change to it
    fails here instead of passing silently.  It is not vnode parity with the reference;
  * get_hash_values hashes the visible rows only (data_chunk.rs:338-355): an invisible row's hash is crc32(b"");
    to_vnode is hash % vnode_count (vnode.rs:45-50);
  * compute_chunk (vnode.rs:151-182): a single Serial key takes the row id's vnode bits whatever the visibility
    (util/row_id.rs:135-173); a NULL Serial hashes the whole row, every column in column order;
  * the U-/U+ rewrite of dispatch_data (dispatch.rs:976-1023) pairs a visible U+ with the last visible U- that no
    earlier U+ has taken (`last_update_delete_row_idx.take()`); invisible rows keep their op.  The key compares as a
    projected Row: NULL == NULL, floats by OrderedFloat class (-0 == +0, every NaN equal).  The reference pushes the
    pair's two ops at the U+, so `new_ops` is positional only when the pair is adjacent; the project writes each op at
    its own row;
  * routing: dest = mapping[vnode] for any mapping; within a destination the visible rows keep their input order; a
    receiver concatenates its sources in rank order; ops and column bits travel unchanged.

A device row whose op is 0 is invisible as well (the project's fold of a dropped row); the host entry points get ops
1..4 only.
"""
import ctypes as C
import importlib.util
import os
import re
import struct
import sys
import zlib

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.stream_chunk import DECIMAL_DTYPE, Column, StreamChunk, pack_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_OF = {"bool": abi.T_BOOL, "int2": abi.T_INT16, "int4": abi.T_INT32, "int8": abi.T_INT64, "serial": abi.T_SERIAL,
        "timestamptz": abi.T_TIMESTAMPTZ, "float4": abi.T_FLOAT32, "float8": abi.T_FLOAT64, "date": abi.T_DATE,
        "time": abi.T_TIME, "timestamp": abi.T_TIMESTAMP, "decimal": abi.T_DECIMAL}
NP_OF = {"bool": np.uint8, "int2": np.int16, "int4": np.int32, "int8": np.int64, "serial": np.int64,
         "timestamptz": np.int64, "float4": np.float32, "float8": np.float64, "date": np.int32, "time": np.int64,
         "timestamp": np.int64, "decimal": DECIMAL_DTYPE}
BITS_OF = {"float4": np.uint32, "float8": np.uint64}
PACK_OF = {"bool": "<B", "int2": "<h", "int4": "<i", "date": "<i", "int8": "<q", "serial": "<q", "timestamptz": "<q",
           "time": "<q", "timestamp": "<q"}
WIDE = ["bool", "int2", "int4", "int8", "serial", "timestamptz", "float4", "float8", "date", "time", "timestamp",
        "decimal"]
INS, DEL, UI, UD = abi.OP_INSERT, abi.OP_DELETE, abi.OP_UPDATE_INSERT, abi.OP_UPDATE_DELETE
VNODE_COUNTS = [1, 2, 255, 256, 257, 1023, 1024, 1025, 2048, 4097, 32768]
M64 = (1 << 64) - 1


class Refused(Exception):
    pass


# ------------------------------------------------------------------------------------------ the restatement
# ordered_float.rs:64-70
SIGN_MASK, EXP_MASK, MAN_MASK = 0x8000000000000000, 0x7ff0000000000000, 0x000fffffffffffff
CANONICAL_NAN_BITS, CANONICAL_ZERO_BITS = 0x7ff8000000000000, 0x0
NULL_VAL_FOR_HASH = 0xfffffff0  # array/mod.rs:97


def is_nan(t, bits):
    if t == "float4":
        return (bits >> 23) & 0xff == 0xff and bits & 0x7fffff != 0
    return (bits >> 52) & 0x7ff == 0x7ff and bits & MAN_MASK != 0


def integer_decode(t, bits):
    """num_traits Float::integer_decode from the bits: (mantissa, exponent, sign); subnormals shift the mantissa left"""
    if t == "float4":
        sign = 1 if bits >> 31 == 0 else -1
        exp = (bits >> 23) & 0xff
        man = (bits & 0x7fffff) << 1 if exp == 0 else (bits & 0x7fffff) | 0x800000
        return man, exp - (127 + 23), sign
    sign = 1 if bits >> 63 == 0 else -1
    exp = (bits >> 52) & 0x7ff
    man = (bits & MAN_MASK) << 1 if exp == 0 else (bits & MAN_MASK) | 0x10000000000000
    return man, exp - (1023 + 52), sign


def raw_double_bits(t, bits):
    """ordered_float.rs:857-870"""
    if is_nan(t, bits):
        return CANONICAL_NAN_BITS
    man, exp, sign = integer_decode(t, bits)
    if man == 0:
        return CANONICAL_ZERO_BITS
    exp_u64 = exp & 0xffff  # `exp as u16 as u64`
    return (man & MAN_MASK) | ((exp_u64 << 52) & EXP_MASK) | ((int(sign > 0) << 63) & SIGN_MASK)


def datum_bytes(t, v):
    if v is None:
        return struct.pack("<I", NULL_VAL_FOR_HASH)
    if t in BITS_OF:
        return struct.pack("<Q", raw_double_bits(t, v))
    if t == "decimal":  # project rule: the i128 mantissa's 16 little-endian bytes
        return struct.pack("<QQ", v & M64, (v >> 64) & M64)
    return struct.pack(PACK_OF[t], v)  # date / time / timestamp: project rule, the ABI value's LE bytes


def bit_for_vnode(vnode_count):
    """util/row_id.rs:135-146: COMPAT_VNODE_BITS = 10 up to 1024 vnodes, else next_power_of_two().ilog2()"""
    return 10 if vnode_count <= 1 << 10 else (vnode_count - 1).bit_length()


def vnode_from_row_id(row_id, vnode_count):
    """util/row_id.rs:164-173 (TIMESTAMP_SHIFT_BITS = 22; `>>` of an i64 is arithmetic, as is Python's)"""
    vnode_bit = bit_for_vnode(vnode_count)
    return ((row_id >> (22 - vnode_bit)) & ((1 << vnode_bit) - 1)) % vnode_count


def datum_class(t, v):
    """Datum equality: NULL == NULL, floats by OrderedFloat class"""
    if v is None or t not in BITS_OF:
        return v
    if is_nan(t, v):
        return "nan"
    f = struct.unpack("<f" if t == "float4" else "<d", struct.pack("<I" if t == "float4" else "<Q", v))[0]
    return f + 0.0


class Col:
    """a column: type name, numpy data in the ABI's native width, valid (bool[n]) or None"""

    def __init__(self, t, data, valid=None):
        self.t, self.data, self.valid = t, data, valid

    def values(self):
        """-> list of datums (Python ints / None)"""
        if self.t == "decimal":
            raw = [(int(x["hi"]) << 64) | int(x["lo"]) for x in self.data]
        elif self.t in BITS_OF:
            raw = [int(x) for x in self.data.view(BITS_OF[self.t])]
        else:
            raw = [int(x) for x in self.data]
        if self.valid is not None:
            raw = [v if ok else None for v, ok in zip(raw, self.valid)]
        return raw

    def width(self):
        return self.data.dtype.itemsize

    def row_bytes(self):
        return np.ascontiguousarray(self.data).view(np.uint8).reshape(len(self.data), self.width())


def visible_rows(ops, vis):
    return [bool(op != 0 and (vis is None or vis[i])) for i, op in enumerate(ops)]


def compute_vnodes(ops, cols, vis, keys, vnode_count):
    """VirtualNode::compute_chunk (vnode.rs:151-182) with get_hash_values (data_chunk.rs:338-355)"""
    n = len(ops)
    vals = [c.values() for c in cols]
    if len(keys) == 1 and cols[keys[0]].t == "serial":
        out = []
        for i in range(n):
            rid = vals[keys[0]][i]
            if rid is not None:
                out.append(vnode_from_row_id(rid, vnode_count))
            else:  # the whole row, every column in column order
                out.append(zlib.crc32(b"".join(datum_bytes(c.t, v[i]) for c, v in zip(cols, vals))) % vnode_count)
        return out
    vis_ = visible_rows(ops, vis)
    return [zlib.crc32(b"".join(datum_bytes(cols[k].t, vals[k][i]) for k in keys) if vis_[i] else b"") % vnode_count
            for i in range(n)]


def rewrite_ops(ops, cols, vis, keys):
    """dispatch.rs:976-1023, each op written at its own row"""
    vals = [c.values() for c in cols]
    key = [tuple(datum_class(cols[k].t, vals[k][i]) for k in keys) for i in range(len(ops))]
    out, last = [int(o) for o in ops], None
    for i, vis_i in enumerate(visible_rows(ops, vis)):
        if not vis_i:
            continue
        if ops[i] == UD:
            last = i
        elif ops[i] == UI:
            if last is None:
                raise Refused("missing U- before U+")
            if key[last] != key[i]:
                out[last], out[i] = DEL, INS
            last = None
    if last is not None:
        raise Refused("missing U+ after U-")
    return out


def route(ops, vis, vnodes, mapping, n_dest):
    """-> per destination, the input indices of its rows in input order"""
    per = [[] for _ in range(n_dest)]
    for i, v in enumerate(visible_rows(ops, vis)):
        if v:
            per[mapping[vnodes[i]]].append(i)
    return per


# ------------------------------------------------------------------------------------------ values
FLOAT_EDGES = {
    # +0 -0 +inf -inf qNaN sNaN -NaN NaN-payload min-subnormal -min-subnormal f32-max 2^24 2^53 -1 1
    "float4": [0x00000000, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0x7f800001, 0xffc00000, 0x7fc12345,
               0x00000001, 0x80000001, 0x7f7fffff, 0x4b800000, 0x5a000000, 0xbf800000, 0x3f800000],
    "float8": [0x0, 0x8000000000000000, 0x7ff0000000000000, 0xfff0000000000000, 0x7ff8000000000000,
               0x7ff0000000000001, 0xfff8000000000000, 0x7ff80000000abcde, 0x1, 0x8000000000000001,
               0x47efffffe0000000, 0x4170000000000000, 0x4340000000000000, 0xbff0000000000000, 0x3ff0000000000000],
}
SERIAL_IDS = [1 << b for b in range(7, 22)] + [-(1 << 63) | (0x2aa << 12), -(1 << 63) | (1 << 21) | (1 << 7),
                                              (0x155 << 12) | 0x7f, (0x7fff << 7) | (1 << 40)]


def int_edges(t):
    if t == "bool":
        return [0, 1]
    if t == "decimal":
        return [-((1 << 127) - 1), -(1 << 64), -1, 0, 1, 1 << 64, (1 << 127) - 1]
    b = {"int2": 16, "int4": 32, "date": 32}.get(t, 64)
    lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
    out = [lo, lo + 1, -1, 0, 1, hi] + ([1 << 24] if b >= 32 else []) + ([1 << 53] if b == 64 else [])
    return out + (SERIAL_IDS if t == "serial" else [])


def make_col(rng, t, n, null_frac=0.1, edges_only=False):
    if t in BITS_OF:
        pool = np.array(FLOAT_EDGES[t], dtype=BITS_OF[t])
        bits = pool[rng.integers(0, len(pool), n)]
        if not edges_only:
            rnd = (rng.standard_normal(n) * 1e4).astype(NP_OF[t]).view(BITS_OF[t])
            bits = np.where(rng.random(n) < 0.5, bits, rnd)
        data = bits.view(NP_OF[t]).copy()
    else:
        pool = int_edges(t)
        vals = [pool[j] for j in rng.integers(0, len(pool), n)]
        if not edges_only:
            lo, hi = min(pool), max(pool)
            for i in np.nonzero(rng.random(n) < 0.5)[0]:
                vals[i] = (int(rng.integers(-(1 << 62), 1 << 62)) << 64) | int(rng.integers(0, 1 << 63)) if t == "decimal" \
                    else int(rng.integers(lo, hi, endpoint=True))
        if t == "decimal":
            data = np.zeros(n, DECIMAL_DTYPE)
            data["lo"] = [v & M64 for v in vals]
            data["hi"] = [v >> 64 for v in vals]
        else:
            data = np.array(vals, dtype=NP_OF[t])
    valid = rng.random(n) >= null_frac if null_frac else None
    return Col(t, data, valid)


def host_chunk(ops, cols, vis=None):
    return StreamChunk(np.asarray(ops, np.uint8), [Column(T_OF[c.t], c.data, c.valid) for c in cols], vis)


def wide_chunk(rng, n, null_frac=0.15, vis_frac=0.9):
    cols = [make_col(rng, t, n, null_frac) for t in WIDE]
    ops = rng.integers(1, 5, n).astype(np.uint8)
    vis = rng.random(n) < vis_frac
    return ops, cols, vis


# ------------------------------------------------------------------------------------------ the restatement's own checks
def test_restatement_reproduces_test_hash_dispatcher():
    """dispatch.rs:1593-1606: consecutive i32s from 19260817, crc32 over the LE bytes of the key columns % 256"""
    dimension, n = 4, 64
    start = iter(range(19260817, 19260817 + dimension * n))
    rows = [[next(start) for _ in range(dimension)] for _ in range(n)]
    cols = [Col("int4", np.array([r[k] for r in rows], np.int32)) for k in range(dimension)]
    for key_indices in ([0], [1, 3], [3, 1], [0, 1, 2, 3]):
        want = [zlib.crc32(b"".join(r[k].to_bytes(4, "little", signed=True) for k in key_indices)) % 256 for r in rows]
        assert compute_vnodes([INS] * n, cols, None, key_indices, 256) == want


def test_restatement_float_classes_collapse():
    for t, edges in FLOAT_EDGES.items():
        nans = [b for b in edges if is_nan(t, b)]
        assert len(nans) == 4 and {raw_double_bits(t, b) for b in nans} == {CANONICAL_NAN_BITS}
        zeros = [0, 1 << (31 if t == "float4" else 63)]
        assert {raw_double_bits(t, b) for b in zeros} == {CANONICAL_ZERO_BITS}
        assert len({datum_class(t, b) for b in nans}) == 1 and len({datum_class(t, b) for b in zeros}) == 1
        others = [b for b in edges if not is_nan(t, b) and b not in zeros]
        assert len({raw_double_bits(t, b) for b in others}) == len(others)
    # integer_decode(1.0f64) = (2^52, -52, 1): mantissa bits 0, exponent field 0x7cc, sign bit set for a positive
    assert raw_double_bits("float8", 0x3ff0000000000000) == 0xfcc0000000000000
    # the smallest f32 subnormal: mantissa 2 (shifted left), exponent -150
    assert raw_double_bits("float4", 1) == 2 | (((-150) & 0x7ff) << 52) | (1 << 63)
    assert bit_for_vnode(1024) == 10 and bit_for_vnode(1025) == 11 and bit_for_vnode(32768) == 15


def test_restatement_rewrite_pins_the_take_rule():
    def run(ops, keys, vis=None):
        return rewrite_ops(ops, [Col("int8", np.array(keys, np.int64))], vis, [0])
    assert run([UD, INS, UI], [1, 4, 2]) == [DEL, INS, INS]
    assert run([UD, UD, UI], [1, 1, 1]) == [UD, UD, UI]
    assert run([UD, DEL, UI], [1, 3, 1]) == [UD, DEL, UI]
    for bad, msg in (([UI], "before"), ([UD, UI, UI], "before"), ([UD, UI, UD], "after"), ([INS, UD], "after")):
        with pytest.raises(Refused, match=msg):
            run(bad, [0] * len(bad))


# ------------------------------------------------------------------------------------------ checks shared by both backends
KEY_SETS = [[k] for k in range(len(WIDE))] + [[2, 1], [0, 0], [4, 3], [7, 6], [11, 8, 9, 10], list(range(8))]


def check_vnodes(be, seed):
    rng = np.random.default_rng(seed)
    n = 1025
    ops, cols, vis = wide_chunk(rng, n)
    ch = host_chunk(ops, cols, vis)
    for keys in KEY_SETS:
        for vc in VNODE_COUNTS:
            want = compute_vnodes(ops, cols, vis, keys, vc)
            got = be.vnode_compute(ch, keys, vc).tolist()
            bad = [i for i in range(n) if got[i] != want[i]]
            assert not bad, (keys, vc, bad[:5], [got[i] for i in bad[:5]], [want[i] for i in bad[:5]])


def check_vnodes_small(be):
    """0 / 1 / 31 / 32 / 33 rows, fully invisible chunks and an all-NULL Serial row"""
    rng = np.random.default_rng(5)
    for n in (0, 1, 31, 32, 33):
        ops, cols, vis = wide_chunk(rng, n, null_frac=0.5)
        for v in (vis, np.zeros(n, bool)):
            ch = host_chunk(ops, cols, v)
            for keys in ([4], [3], [6, 7, 11]):
                for vc in (1, 257, 4097):
                    assert be.vnode_compute(ch, keys, vc).tolist() == compute_vnodes(ops, cols, v, keys, vc), (n, keys, vc)


def stream(rng, length, kinds=("+", "pair", "split", "triple", "inv")):
    """a well-formed U-/U+ stream: rows (op, visible, copy_of) where copy_of names the U- whose key a U+ repeats"""
    rows = []
    while len(rows) < length:
        k = kinds[rng.integers(0, len(kinds))]
        if k == "+":
            rows.append((int(rng.choice([INS, DEL])), True, None))
        elif k == "inv":
            rows.append((int(rng.integers(1, 5)), False, None))
        elif k in ("pair", "split"):
            at = len(rows)
            rows.append((UD, True, None))
            for _ in range(int(rng.integers(1, 4)) if k == "split" else 0):
                rows.append((int(rng.integers(1, 5)), False, None) if rng.random() < 0.5 else (int(rng.choice([INS, DEL])), True, None))
            rows.append((UI, True, at if rng.random() < 0.6 else None))
        else:  # U- U- U+: the second U- replaces the first
            at = len(rows)
            rows += [(UD, True, None), (UD, True, None), (UI, True, at + 1 if rng.random() < 0.6 else None)]
    return rows[:length]


def copy_key(cols, src, dst, rng):
    """row dst takes row src's values, floats moved to another encoding of their class (+-0, every NaN)"""
    for c in cols:
        if c.valid is not None:
            c.valid[dst] = c.valid[src]
        c.data[dst] = c.data[src]
        if c.t in BITS_OF:
            b = c.data.view(BITS_OF[c.t])
            sign = 1 << (31 if c.t == "float4" else 63)
            if is_nan(c.t, int(b[src])):
                nans = [x for x in FLOAT_EDGES[c.t] if is_nan(c.t, x)]
                b[dst] = nans[rng.integers(0, len(nans))]
            elif int(b[src]) & ~sign == 0:
                b[dst] = int(rng.integers(0, 2)) * sign


def rewrite_chunk(rng, rows):
    n = len(rows)
    cols = [make_col(rng, t, n, null_frac=0.2, edges_only=True) for t in WIDE]
    for i, (_, _, src) in enumerate(rows):
        if src is not None and i < n:
            copy_key(cols, src, i, rng)
    ops = np.array([r[0] for r in rows], np.uint8)
    vis = np.array([r[1] for r in rows], bool)
    return ops, cols, vis


def close_stream(ops, vis):
    """a stream cut at its length may end inside a pair or a U- U- U+ triple: the U- rows left pending become +"""
    for i in range(len(ops) - 1, -1, -1):
        if vis[i] and ops[i] == UI:
            break
        if vis[i] and ops[i] == UD:
            ops[i] = INS


def check_rewrite(be, ops, cols, vis, keys):
    ch = host_chunk(ops, cols, vis)
    try:
        want = rewrite_ops(ops, cols, vis, keys)
    except Refused as e:
        with pytest.raises(abi.RwError, match=re.escape(str(e))) as ei:
            be.dispatch_rewrite_ops(ch, keys)
        assert ei.value.code == abi.RW_ERR_INCONSISTENT
        return False
    got = be.dispatch_rewrite_ops(ch, keys).tolist()
    bad = [i for i in range(len(ops)) if got[i] != want[i]]
    assert not bad, (keys, len(ops), bad[:5], [got[i] for i in bad[:5]], [want[i] for i in bad[:5]])
    return True


def pinned_rewrites():
    """(name, ops, key values of one int8 column or None for NULL, visibility, keys' type)"""
    f8 = lambda x: struct.unpack("<q", struct.pack("<Q", x))[0]
    return [
        ("changed", [UD, UI], [1, 2], None, "int8"), ("unchanged", [UD, UI], [1, 1], None, "int8"),
        ("U- + U+", [UD, INS, UI], [1, 4, 2], None, "int8"), ("U- - U+", [UD, DEL, UI], [1, 3, 1], None, "int8"),
        ("U- U- U+", [UD, UD, UI], [1, 1, 1], None, "int8"), ("U- U- U+ changed", [UD, UD, UI], [1, 2, 3], None, "int8"),
        ("split by invisible", [UD, UI, INS, UI], [1, 9, 5, 2], [True, False, True, True], "int8"),
        ("invisible U+ / U- pass", [UI, UD, UD, UI], [1, 2, 3, 3], [False, False, True, True], "int8"),
        ("NULL -> value", [UD, UI], [None, 1], None, "int8"), ("NULL -> NULL", [UD, UI], [None, None], None, "int8"),
        ("-0 -> +0", [UD, UI], [f8(0x8000000000000000), 0], None, "float8"),
        ("NaN encodings", [UD, UI], [f8(0x7ff8000000000000), f8(0xfff0000000000001)], None, "float8"),
        ("0 -> subnormal", [UD, UI], [0, 1], None, "float8"),
        ("U+ first", [UI], [1], None, "int8"), ("U- U+ U+", [UD, UI, UI], [1, 1, 1], None, "int8"),
        ("trailing U-", [UD, UI, UD], [1, 1, 1], None, "int8"), ("U- then invisible U+", [UD, UI], [1, 1], [True, False], "int8"),
    ]


PINNED = {case[0]: case for case in pinned_rewrites()}
REFUSED = ("U+ first", "U- U+ U+", "trailing U-", "U- then invisible U+")


def check_pinned_rewrite(be, name):
    _, ops, keys, vis, t = PINNED[name]
    data = np.array([0 if k is None else k for k in keys], np.int64)
    col = Col(t, data.view(NP_OF[t]), np.array([k is not None for k in keys]))
    v = None if vis is None else np.array(vis)
    assert check_rewrite(be, np.array(ops, np.uint8), [col], v, [0]) == (name not in REFUSED), name


def check_rewrites(be):
    rng = np.random.default_rng(11)
    for length in (1, 2, 3, 31, 32, 33, 1023, 1024, 1025, 4097):
        ops, cols, vis = rewrite_chunk(rng, stream(rng, length))
        close_stream(ops, vis)
        for keys in ([3], [6], [7], [0, 1, 2], [11, 8], [7, 6, 4, 5], [2, 1, 0, 9, 10, 11, 3, 5]):
            assert check_rewrite(be, ops, cols, vis, keys), (length, keys)
    # malformed streams: a stray U+ or an unanswered U- somewhere in a long stream
    for length in (33, 1025, 4097):
        for stray in (UI, UD):
            ops, cols, vis = rewrite_chunk(rng, stream(rng, length))
            close_stream(ops, vis)
            at = int(rng.integers(0, length))
            ops[at], vis[at] = stray, True
            check_rewrite(be, ops, cols, vis, [3, 7])


def refusal_cases():
    """(what, ops, cols, keys, vnode_count, code)"""
    rng = np.random.default_rng(3)
    ops, cols, vis = wide_chunk(rng, 40)
    return ops, cols, vis, [
        ("n_keys 0", [], 256, abi.RW_ERR_UNSUPPORTED), ("n_keys 9", [0] * 9, 256, abi.RW_ERR_UNSUPPORTED),
        ("key index -1", [-1], 256, abi.RW_ERR_INVALID), ("key index n_cols", [len(WIDE)], 256, abi.RW_ERR_INVALID),
        ("vnode_count 0", [3], 0, abi.RW_ERR_INVALID), ("vnode_count 32769", [3], 32769, abi.RW_ERR_INVALID),
    ]


def check_refusals(be):
    ops, cols, vis, cases = refusal_cases()
    ch = host_chunk(ops, cols, vis)
    for what, keys, vc, code in cases:
        with pytest.raises(abi.RwError) as ei:
            be.vnode_compute(ch, keys, vc)
        assert ei.value.code == code, what
        if vc == 256:
            with pytest.raises(abi.RwError) as ei:
                be.dispatch_rewrite_ops(ch, keys)
            assert ei.value.code == code, what
    varlen = StreamChunk(ops, [Column(abi.T_INT64, cols[3].data), Column(abi.T_VARCHAR, np.array([b"x"] * len(ops), dtype=object))])
    for call in (lambda: be.vnode_compute(varlen, [0], 256), lambda: be.dispatch_rewrite_ops(varlen, [0])):
        with pytest.raises(abi.RwError) as ei:
            call()
        assert ei.value.code == abi.RW_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_vnodes_match_restatement(oracle, seed):
    check_vnodes(oracle, seed)


def test_oracle_vnodes_small_chunks(oracle):
    check_vnodes_small(oracle)


@pytest.mark.parametrize("name", list(PINNED))
def test_oracle_rewrite_pinned(oracle, name):
    check_pinned_rewrite(oracle, name)


def test_oracle_rewrite_matches_restatement(oracle):
    check_rewrites(oracle)


def test_oracle_refuses_what_the_device_refuses(oracle):
    check_refusals(oracle)


def test_bench_vnode_of_int64_matches_restatement():
    """bench.py pre-partitions the CPU arm's input with its own numpy CRC: it must be the dispatcher's vnode"""
    spec = importlib.util.spec_from_file_location("_bench_for_vnodes", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    dont = sys.dont_write_bytecode
    sys.dont_write_bytecode = True
    try:
        spec.loader.exec_module(mod)
    finally:
        sys.dont_write_bytecode = dont
    rng = np.random.default_rng(9)
    keys = np.concatenate([np.array(int_edges("int8"), np.int64), rng.integers(-2**63, 2**63 - 1, 3000, dtype=np.int64, endpoint=True)])
    want = compute_vnodes([INS] * len(keys), [Col("int8", keys)], None, [0], 256)
    assert mod.vnode_of_int64(keys).tolist() == want


# ------------------------------------------------------------------------------------------ GPU: host entry points
@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_device_vnodes_match_restatement(cuda, seed):
    check_vnodes(cuda, seed)


@pytest.mark.gpu
def test_device_vnodes_small_chunks(cuda):
    check_vnodes_small(cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PINNED))
def test_device_rewrite_pinned(cuda, name):
    check_pinned_rewrite(cuda, name)


@pytest.mark.gpu
def test_device_rewrite_matches_restatement(cuda):
    check_rewrites(cuda)


@pytest.mark.gpu
def test_device_host_entry_points_refuse(cuda):
    check_refusals(cuda)


# ------------------------------------------------------------------------------------------ GPU: the partition paths
def _lib():
    from risingwave_b200 import device
    lib = device._lib()
    if not getattr(lib, "_flat_sig", False):
        lib.rwgpu_shuffle_exchange_flat_device.restype = C.c_int32
        lib.rwgpu_shuffle_exchange_flat_device.argtypes = [
            C.POINTER(abi.RwChunk), C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
            C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
            C.c_int32, C.c_void_p]
        lib._flat_sig = True
    return lib


def _rc(rc, what=""):
    if rc != abi.RW_OK:
        raise abi.RwError(rc, f"{what}: {(_lib().rwgpu_last_error() or b'').decode()}")


def dev_chunk(ops, cols, vis=None, validity=True):
    """an rw_chunk of DEVICE pointers (torch tensors of raw bytes) -> (chunk, keepalive)"""
    import torch
    n = len(ops)
    keep = []

    def put(a):
        t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
        keep.append(t)
        return t.data_ptr()
    arr = (abi.RwColumn * max(1, len(cols)))()
    for k, c in enumerate(cols):
        arr[k].type = T_OF[c.t]
        arr[k].data = put(c.data) if n else None
        arr[k].validity = put(pack_bits(c.valid)) if (validity and c.valid is not None) else None
    ch = abi.RwChunk()
    ch.n_rows, ch.n_cols = n, len(cols)
    ch.ops = put(np.asarray(ops, np.uint8)) if n else None
    ch.visibility = put(pack_bits(vis)) if vis is not None else None
    ch.columns = arr
    keep.append(arr)
    return ch, keep


def i32s(xs):
    return (C.c_int32 * max(1, len(xs)))(*xs)


def ptrs(xs):
    return (C.c_void_p * max(1, len(xs)))(*xs)


def mapping_of(kind, vc, n_dest, rng):
    if kind == "contiguous":
        return [v * n_dest // vc for v in range(vc)]
    if kind == "one":  # everything to the last destination: the others receive nothing
        return [n_dest - 1] * vc
    return [int(x) for x in rng.integers(0, n_dest, vc)]


def partition_device(ops, cols, vis, keys, vc, mapping, n_dest, with_valid=True):
    import torch
    n = len(ops)
    ch, keep = dev_chunk(ops, cols, vis)
    v2d = torch.tensor(mapping, dtype=torch.int32, device="cuda")
    out_ops = torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda")
    out_cols = [torch.zeros(max(n, 1) * c.width(), dtype=torch.uint8, device="cuda") for c in cols]
    out_valid = [torch.full((max(n, 1),), 7, dtype=torch.uint8, device="cuda") for _ in cols]
    counts = torch.full((n_dest,), -1, dtype=torch.int64, device="cuda")
    offsets = torch.full((n_dest,), -1, dtype=torch.int64, device="cuda")
    _rc(_lib().rwgpu_shuffle_partition_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), n_dest,
                                              C.c_void_p(out_ops.data_ptr()), ptrs([t.data_ptr() for t in out_cols]),
                                              ptrs([t.data_ptr() for t in out_valid]) if with_valid else None,
                                              C.c_void_p(counts.data_ptr()), C.c_void_p(offsets.data_ptr()), None), "partition")
    torch.cuda.synchronize()
    return (out_ops.cpu().numpy(), [t.cpu().numpy() for t in out_cols], [t.cpu().numpy() for t in out_valid],
            counts.cpu().numpy().tolist(), offsets.cpu().numpy().tolist())


def assert_rows(what, got_ops, got_cols, srcs):
    """srcs: [(ops, cols, indices)] concatenated in order -> ops and every column's bytes"""
    want_ops = np.concatenate([np.asarray(o, np.uint8)[ix] for o, _, ix in srcs]) if srcs else np.zeros(0, np.uint8)
    m = len(want_ops)
    assert np.array_equal(got_ops[:m], want_ops), (what, "ops")
    for k in range(len(srcs[0][1])):
        w = srcs[0][1][k].width()
        want = np.concatenate([c[k].row_bytes()[ix] for _, c, ix in srcs]).reshape(-1)
        got = got_cols[k][:m * w]
        bad = np.nonzero(got.reshape(-1, w) != want.reshape(-1, w))[0] if m else []
        assert len(bad) == 0, (what, "column", k, srcs[0][1][k].t, "rows", sorted(set(bad.tolist()))[:5])


PART_ROWS = [0, 1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049, 65 * 2048 + 7]
PART_DESTS = [1, 2, 3, 5, 8, 33, 64]
PART_CASES = [(n, PART_DESTS[i % len(PART_DESTS)], ["contiguous", "random", "one"][i % 3], VNODE_COUNTS[i % len(VNODE_COUNTS)])
              for i, n in enumerate(PART_ROWS)] + [(4097, d, "random", 256) for d in PART_DESTS] + [(65 * 2048 + 7, 64, "random", 4097)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,n_dest,kind,vc", PART_CASES)
def test_partition_device_matches_restatement(cuda, n, n_dest, kind, vc):
    """part_hist / part_scan / part_scatter: counts, offsets, ops, every column's bits and the validity bytes, at every
    column width, with ops == 0 and a visibility bitmap, for several key sets"""
    rng = np.random.default_rng(n * 131 + n_dest)
    ops, cols, vis = wide_chunk(rng, n)
    ops[rng.random(n) < 0.1] = 0
    for keys, v in (([3], vis), ([4], None), ([6, 7, 0], vis), ([11, 2, 1, 8, 9, 10, 5], vis)):
        mapping = mapping_of(kind, vc, n_dest, rng)
        per = route(ops, v, compute_vnodes(ops, cols, v, keys, vc), mapping, n_dest)
        got_ops, got_cols, got_valid, counts, offsets = partition_device(ops, cols, v, keys, vc, mapping, n_dest)
        assert counts == [len(p) for p in per], (keys, "counts")
        assert offsets == [sum(len(p) for p in per[:d]) for d in range(n_dest)], (keys, "offsets")
        order = [i for p in per for i in p]
        assert_rows((keys, n_dest), got_ops, got_cols, [(ops, cols, order)])
        for k, c in enumerate(cols):
            want = [1 if (c.valid is None or c.valid[i]) else 0 for i in order]
            assert got_valid[k][:len(order)].tolist() == want, (keys, "valid", k)


@pytest.mark.gpu
def test_partition_device_fully_invisible_and_one_class_per_destination(cuda):
    """a fully invisible chunk sends nothing; rows whose keys are equal as Datums (every NaN encoding, +-0, NULL) land on
    exactly one destination"""
    rng = np.random.default_rng(17)
    n = 3000
    ops, cols, _ = wide_chunk(rng, n)
    _, _, _, counts, _ = partition_device(ops, cols, np.zeros(n, bool), [7], 256, mapping_of("random", 256, 33, rng), 33)
    assert counts == [0] * 33
    for t in ("float4", "float8"):
        edges = FLOAT_EDGES[t]
        bits = np.array([edges[j] for j in rng.integers(0, 8, n)], dtype=BITS_OF[t])  # +-0, +-inf, four NaNs
        col = Col(t, bits.view(NP_OF[t]).copy(), rng.random(n) > 0.2)
        ops = np.full(n, INS, np.uint8)
        mapping = mapping_of("random", 4097, 64, rng)
        got_ops, got_cols, got_valid, counts, offsets = partition_device(ops, [col], None, [0], 4097, mapping, 64)
        dest_of = {}
        out_bits = got_cols[0].view(BITS_OF[t])
        for d in range(64):
            for i in range(offsets[d], offsets[d] + counts[d]):
                dest_of.setdefault(datum_class(t, int(out_bits[i])) if got_valid[0][i] else None, set()).add(d)
        assert len(dest_of) == 5 and all(len(s) == 1 for s in dest_of.values()), dest_of
        per = route(ops, None, compute_vnodes(ops, [col], None, [0], 4097), mapping, 64)
        assert counts == [len(p) for p in per]
        assert_rows(t, got_ops, got_cols, [(ops, [col], [i for p in per for i in p])])


def p2p_types_of(i):
    """payload layouts: every width, and 1-column chunks"""
    layouts = [WIDE, ["int8"], ["bool", "int2"], ["decimal", "float4", "date", "serial"], ["int4", "float8", "timestamp"]]
    return layouts[i % len(layouts)]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8, 33, 64])
def test_p2p_partition_and_unpack_virtual_ranks(cuda, world):
    """part_scatter_p2p_kernel / p2p_publish_counts_kernel / p2p_unpack_kernel with W virtual ranks on one device: each
    receiver holds its sources' routed rows, sources in rank order, every column's bits"""
    import torch
    from risingwave_b200 import device
    lib = _lib()
    rng = np.random.default_rng(world)
    for case in range(2):
        types = p2p_types_of(world + case)
        key_sets = [[0], list(range(min(len(types), 8)))]
        keys = key_sets[case]
        vc = VNODE_COUNTS[(world + case) % len(VNODE_COUNTS)]
        mapping = mapping_of(["random", "contiguous"][case], vc, world, rng)
        v2d = torch.tensor(mapping, dtype=torch.int32, device="cuda")
        sizes = [int(x) for x in rng.choice([0, 1, 33, 1025, 2049], world)] if world > 8 else \
            [int(x) for x in rng.choice([0, 31, 2048, 4097, 65 * 2048 + 7 if world <= 2 else 3000], world)]
        cap = max(1, max(sizes))
        region = device.p2p_region_bytes([T_OF[t] for t in types], cap)
        bufs = [torch.zeros(world * region, dtype=torch.uint8, device="cuda") for _ in range(world)]
        peers = ptrs([b.data_ptr() for b in bufs])
        src = []
        for r in range(world):
            n = sizes[r]
            cols = [make_col(rng, t, n, null_frac=0) for t in types]
            ops = rng.integers(0, 5, n).astype(np.uint8)
            vis = rng.random(n) < 0.9 if r % 2 else None
            per = route(ops, vis, compute_vnodes(ops, cols, vis, keys, vc), mapping, world)
            src.append((ops, cols, per))
            ch, keep = dev_chunk(ops, cols, vis)
            counts = torch.full((world,), -1, dtype=torch.int64, device="cuda")
            overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
            _rc(lib.rwgpu_shuffle_partition_p2p_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), world, r,
                                                       peers, cap, C.c_void_p(counts.data_ptr()), C.c_void_p(overflow.data_ptr()), None))
            torch.cuda.synchronize()
            assert int(overflow.item()) == 0
            assert counts.cpu().numpy().tolist() == [len(p) for p in per], (world, r)
        for d in range(world):
            want = sum(len(s[2][d]) for s in src)
            out_ops = torch.zeros(max(1, want), dtype=torch.uint8, device="cuda")
            out_cols = [torch.zeros(max(1, want) * s.width(), dtype=torch.uint8, device="cuda") for s in src[0][1]]
            total = torch.full((1,), -2, dtype=torch.int64, device="cuda")
            _rc(lib.rwgpu_shuffle_unpack_device(C.c_void_p(bufs[d].data_ptr()), world, i32s([T_OF[t] for t in types]), len(types), cap,
                                                C.c_void_p(out_ops.data_ptr()), ptrs([t.data_ptr() for t in out_cols]),
                                                C.c_void_p(total.data_ptr()), None))
            torch.cuda.synchronize()
            assert int(total.item()) == want, (world, d)
            assert_rows((world, d), out_ops.cpu().numpy(), [t.cpu().numpy() for t in out_cols],
                        [(s[0], s[1], s[2][d]) for s in src])


@pytest.mark.gpu
def test_p2p_exchange_self_peer(cuda):
    """rwgpu_shuffle_exchange_p2p_device at W = 1 over every column width: the unpacked rows, the host and device counts"""
    import torch
    from risingwave_b200 import device
    lib = _lib()
    rng = np.random.default_rng(23)
    types = WIDE
    cap = 4097
    region = device.p2p_region_bytes([T_OF[t] for t in types], cap)
    recv = torch.zeros(region, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    out_ops = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    out_cols = [torch.zeros(cap * (16 if t == "decimal" else abi.TYPE_WIDTH[T_OF[t]]), dtype=torch.uint8, device="cuda") for t in types]
    counts = torch.zeros(1, dtype=torch.int64, device="cuda")
    overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
    total_host = torch.zeros(1, dtype=torch.int64).pin_memory()
    v2d = torch.zeros(1024, dtype=torch.int32, device="cuda")
    for epoch, n in ((1, 4097), (2, 0), (3, 1025)):
        cols = [make_col(rng, t, n, null_frac=0) for t in types]
        ops = rng.integers(0, 5, n).astype(np.uint8)
        vis = rng.random(n) < 0.8
        ch, keep = dev_chunk(ops, cols, vis)
        _rc(lib.rwgpu_shuffle_exchange_p2p_device(C.byref(ch), i32s([7, 6]), 2, 1024, C.c_void_p(v2d.data_ptr()), 1, 0,
                                                  ptrs([recv.data_ptr()]), ptrs([flags.data_ptr()]), epoch, cap, C.c_void_p(recv.data_ptr()),
                                                  C.c_void_p(out_ops.data_ptr()), ptrs([t.data_ptr() for t in out_cols]),
                                                  C.c_void_p(counts.data_ptr()), C.c_void_p(overflow.data_ptr()),
                                                  C.c_void_p(total_host.data_ptr()), None))
        torch.cuda.synchronize()
        idx = [i for i, v in enumerate(visible_rows(ops, vis)) if v]
        dev_count = flags[512 + 8 * (epoch & 1):520 + 8 * (epoch & 1)].view(torch.int64)
        assert int(total_host.item()) == len(idx) == int(dev_count.item()) == int(counts.item()), epoch
        assert int(overflow.item()) == 0
        if n:
            assert_rows(epoch, out_ops.cpu().numpy(), [t.cpu().numpy() for t in out_cols], [(ops, cols, idx)])


# ------------------------------------------------------------------------------------------ GPU: the flat exchange
FLAT_LAYOUTS = {  # name -> column types; staged = every column 8 bytes wide and at most 12 columns (shuffle.cu)
    "staged_1": ["int8"],
    "staged_12": ["int8", "float8", "timestamptz", "serial", "time", "timestamp"] * 2,
    "unstaged_13": ["int8", "float8", "timestamptz", "serial", "time", "timestamp"] * 2 + ["int8"],
    "unstaged_mixed": WIDE,
    "unstaged_int4": ["int4"],
}


def flat_run(world, types, keys, vc, mapping, sizes, rng, epochs=(1, 2), max_blocks=24):
    """-> True if the ranks' kernels met in their barriers; checks every receive buffer against the restatement"""
    import torch
    from risingwave_b200 import device
    lib = _lib()
    tcodes = [T_OF[t] for t in types]
    cap = max(1, world * max(max(s) for s in sizes))
    total, ops_off, col_off = device.flat_layout(tcodes, cap)
    widths = [16 if t == "decimal" else abi.TYPE_WIDTH[T_OF[t]] for t in types]
    flags = [torch.zeros(1024, dtype=torch.uint8, device="cuda") for _ in range(world)]
    bufs = [[torch.zeros(total, dtype=torch.uint8, device="cuda") for _ in range(world)] for _ in range(2)]
    v2d = torch.tensor(mapping, dtype=torch.int32, device="cuda")
    streams = [torch.cuda.Stream() for _ in range(world)]
    for e, epoch in enumerate(epochs):
        buf = bufs[epoch & 1]
        peers = ptrs([b.data_ptr() for b in buf])
        flag_ptrs = ptrs([f.data_ptr() for f in flags])
        src, chunks = [], []
        state = [(torch.full((world,), -1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
                  torch.full((1,), -2, dtype=torch.int64, device="cuda")) for _ in range(world)]
        for r in range(world):
            n = sizes[e][r]
            cols = [make_col(rng, t, n, null_frac=0) for t in types]
            ops = rng.integers(0, 5, n).astype(np.uint8)
            vis = rng.random(n) < 0.85 if (r + e) % 2 else None
            per = route(ops, vis, compute_vnodes(ops, cols, vis, keys, vc), mapping, world)
            src.append((ops, cols, per))
            chunks.append(dev_chunk(ops, cols, vis))
        torch.cuda.synchronize()
        for r in range(world):
            counts, err, tot = state[r]
            _rc(lib.rwgpu_shuffle_exchange_flat_device(C.byref(chunks[r][0]), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), world, r,
                                                       peers, flag_ptrs, epoch, cap, C.c_void_p(counts.data_ptr()), C.c_void_p(err.data_ptr()),
                                                       C.c_void_p(tot.data_ptr()), None, max_blocks, C.c_void_p(streams[r].cuda_stream)), "flat")
        torch.cuda.synchronize()
        errs = [int(s[1].item()) for s in state]
        if any(x & 2 for x in errs):
            return False
        assert errs == [0] * world
        for r in range(world):
            assert state[r][0].cpu().numpy().tolist() == [len(p) for p in src[r][2]], (world, epoch, r)
        for d in range(world):
            want = sum(len(s[2][d]) for s in src)
            assert int(state[d][2].item()) == want, (world, epoch, d)
            b = buf[d].cpu().numpy()
            got_cols = [b[o:o + cap * w] for o, w in zip(col_off, widths)]
            assert_rows((world, epoch, d), b[ops_off:ops_off + cap], got_cols, [(s[0], s[1], s[2][d]) for s in src])
    return True


FLAT_CASES = [(w, name) for w in (1, 2, 3, 4) for name in FLAT_LAYOUTS]


@pytest.mark.gpu
@pytest.mark.parametrize("world,layout", FLAT_CASES)
def test_flat_exchange_virtual_ranks(cuda, world, layout):
    """flat_exchange_kernel, staged and unstaged, with 1-4 virtual ranks side by side on one device (grids capped so that
    they are co-resident): every receive buffer holds its sources' routed rows in rank order, every column's bits"""
    types = FLAT_LAYOUTS[layout]
    rng = np.random.default_rng(world * 17 + len(types))
    vc = [256, 1025, 4097, 32768][world - 1]
    kinds = ["random", "contiguous", "one", "random"]
    mapping = mapping_of(kinds[(world + len(types)) % 4], vc, world, rng)
    keys = [0] if len(types) == 1 else [3, 1] if len(types) > 3 else [0, 1]
    sizes = [[[1023, 1024, 1025, 4097][(r + world) % 4] for r in range(world)],
             [[0, 1, 31, 2 * 1024 + 1][(r + 2) % 4] for r in range(world)]]
    if world == 1:
        sizes = [[65 * 2048 + 7], [1]]
    if not flat_run(world, types, keys, vc, mapping, sizes, rng):
        pytest.skip("this device did not run the ranks' kernels side by side (barrier timed out)")


def flat_kernels_run(layout):
    """-> the flat_exchange_kernel instances a torch.profiler trace sees in one exchange of `layout` at world 1"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    types = FLAT_LAYOUTS[layout]
    rng = np.random.default_rng(2)
    assert flat_run(1, types, [0], 256, [0] * 256, [[1000]], rng, epochs=(1,))  # (loads the module outside the trace)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert flat_run(1, types, [0], 256, [0] * 256, [[1000]], rng, epochs=(1,))
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()} | {e.key for e in prof.key_averages()}
    return sorted({t for t in ("flat_exchange_kernel<true>", "flat_exchange_kernel<false>") for n in names if t in n})


@pytest.mark.gpu
def test_flat_plans_run_their_template(cuda):
    """the staged template runs exactly when every column is 8 bytes wide and there are at most 12 columns.  The traces
    are taken in a fresh interpreter: run late in the whole suite, in the suite's process, the trace came back without
    this kernel's events."""
    import json
    import subprocess
    code = (f"import json, sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_shuffle_types as T; "
            f"print(json.dumps({{l: T.flat_kernels_run(l) for l in T.FLAT_LAYOUTS}}))")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-3000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    for layout, kernels in got.items():
        want = "flat_exchange_kernel<true>" if layout.startswith("staged") else "flat_exchange_kernel<false>"
        assert kernels == [want], (layout, kernels)


# ------------------------------------------------------------------------------------------ GPU: refusals
@pytest.mark.gpu
def test_partition_entry_points_refuse(cuda):
    import torch
    lib = _lib()
    ops, cols, vis, cases = refusal_cases()
    n = len(ops)
    v2d = torch.zeros(32768, dtype=torch.int32, device="cuda")
    out_ops = torch.zeros(n, dtype=torch.uint8, device="cuda")
    outs = [torch.zeros(n * 16, dtype=torch.uint8, device="cuda") for _ in range(len(WIDE) + 1)]
    scratch = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    a = C.c_void_p(scratch.data_ptr())
    bases = ptrs([scratch.data_ptr()] * 65)
    pinned = torch.zeros(1, dtype=torch.int64).pin_memory()

    def part(ch, keys, vc, n_dest, valid=True):
        return lib.rwgpu_shuffle_partition_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), n_dest,
                                                  C.c_void_p(out_ops.data_ptr()), ptrs([t.data_ptr() for t in outs]),
                                                  ptrs([t.data_ptr() for t in outs]) if valid else None, a, a, None)

    def p2p(ch, keys, vc, n_dest, rank=0):
        return lib.rwgpu_shuffle_partition_p2p_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), n_dest, rank,
                                                      bases, 64, a, a, None)

    def xp2p(ch, keys, vc, n_dest, rank=0):
        return lib.rwgpu_shuffle_exchange_p2p_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), n_dest, rank,
                                                     bases, bases, 1, 64, a, C.c_void_p(out_ops.data_ptr()),
                                                     ptrs([t.data_ptr() for t in outs]), a, a, C.c_void_p(pinned.data_ptr()), None)

    def flat(ch, keys, vc, n_dest, rank=0, epoch=1):
        return lib.rwgpu_shuffle_exchange_flat_device(C.byref(ch), i32s(keys), len(keys), vc, C.c_void_p(v2d.data_ptr()), n_dest, rank,
                                                      bases, bases, epoch, 1 << 10, a, a, a, None, 1, None)

    plain, keep1 = dev_chunk(ops, cols, vis, validity=False)
    nulls, keep2 = dev_chunk(ops, cols, vis, validity=True)
    for what, keys, vc, code in cases:
        for fn in (part, p2p, xp2p, flat):
            assert fn(plain, keys, vc, 2) == code, (what, fn.__name__)
    for fn in (p2p, xp2p, flat):  # the peer-memory paths carry no validity
        assert fn(nulls, [3], 256, 2) == abi.RW_ERR_UNSUPPORTED, fn.__name__
        for n_dest in (0, 65):
            assert fn(plain, [3], 256, n_dest) == abi.RW_ERR_INVALID, (fn.__name__, n_dest)
        for rank in (-1, 2):
            assert fn(plain, [3], 256, 2, rank) == abi.RW_ERR_INVALID, (fn.__name__, rank)
    assert part(nulls, [3], 256, 2, valid=False) == abi.RW_ERR_UNSUPPORTED
    for n_dest in (0, 65):
        assert part(plain, [3], 256, n_dest) == abi.RW_ERR_UNSUPPORTED, n_dest
    assert flat(plain, [3], 256, 2, 0, epoch=0) == abi.RW_ERR_INVALID
    # a varlen column anywhere in the chunk
    arr = (abi.RwColumn * 2)()
    arr[0].type, arr[0].data = abi.T_INT64, scratch.data_ptr()
    offs = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    arr[1].type, arr[1].data, arr[1].offsets = abi.T_VARCHAR, scratch.data_ptr(), offs.data_ptr()
    vch = abi.RwChunk()
    vch.n_rows, vch.n_cols, vch.ops, vch.columns = n, 2, out_ops.data_ptr(), arr
    for fn in (part, p2p, xp2p, flat):
        assert fn(vch, [0], 256, 2) == abi.RW_ERR_UNSUPPORTED, fn.__name__
    torch.cuda.synchronize()
