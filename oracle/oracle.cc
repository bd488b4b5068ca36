// oracle.cc -- CPU restatement of RisingWave's streaming HashAgg / HashJoin / hash-dispatch
// algorithms.
//
// *** TEST INFRASTRUCTURE ONLY. ***  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library.  The product path
// (risingwave_b200/, librwgpu.so) never links, imports or calls it.
//
// Parity pinning: this restatement is checked against the reference's own golden vectors --
// the 24 non-watermark tests of src/stream/src/executor/hash_join.rs:1812-3921 (exact chunk
// equality incl. visibility), src/stream/tests/integration_tests/hash_agg.rs:21-242, the agg
// function tests of src/expr/impl/src/aggregate/general.rs:189-416 and test_hash_dispatcher
// (src/stream/src/executor/dispatch.rs:1551-1660) -- extracted by tests/golden/extract_ref_kats.py
// into tests/golden/*.json.  The reference itself is Rust and cannot be compiled here (no
// cargo/rustc), so there is no oracle/_ref.
//
// Third-party arithmetic not in the reference tree: CRC32 = crc32fast 1.5.0 (standard IEEE 802.3,
// reflected 0xEDB88320, init/xorout 0xFFFFFFFF), restated below and cross-checked against zlib.
// XxHash64 values are never observable in operator output and are not restated.
//
// Every function cites the reference file:line it follows (paths relative to the reference checkout).
//
// Exposes the same C structs as include/rwgpu.h under the `rwo_` prefix.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../include/rwgpu.h"

namespace {

thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

typedef __int128 i128;

// ------------------------------------------------------------------ Datum
struct Datum {
  bool null = true;
  i128 i = 0;     // all integer-like types, sign-extended; decimal mantissa
  double f = 0;   // float32 / float64 (float32 kept exactly representable)
  uint32_t f32 = 0;  // float32 read from a column: its bits, so that a copy leaves with them (see write_datum)
  std::string s;  // varchar / bytea (BytesArray, bytes_array.rs:30-34): payload only
};

bool is_float(int t) { return t == RW_T_FLOAT32 || t == RW_T_FLOAT64; }
bool is_varlen(int t) { return t == RW_T_VARCHAR || t == RW_T_BYTEA; }

// which operand types a join condition or filter term compares as raw integers: int2 / int4 / int8 with each other (the
// reference widens them, src/expr/impl/src/scalar/cmp.rs:44-51), any other orderable fixed-width type only with itself
// (cmp.rs:24-160; date against timestamp, which the reference evaluates by casting the date, is not restated)
bool cmp_operands_ok(int a, int b) {
  auto is_int = [](int t) { return t == RW_T_INT16 || t == RW_T_INT32 || t == RW_T_INT64; };
  auto ordered = [&](int t) {
    return is_int(t) || t == RW_T_BOOL || t == RW_T_SERIAL || t == RW_T_DATE || t == RW_T_TIME || t == RW_T_TIMESTAMP ||
           t == RW_T_TIMESTAMPTZ;
  };
  return ordered(a) && ordered(b) && (a == b || (is_int(a) && is_int(b)));
}

int type_width(int t) {
  switch (t) {
    case RW_T_BOOL: return 1;
    case RW_T_INT16: return 2;
    case RW_T_INT32: case RW_T_FLOAT32: case RW_T_DATE: return 4;
    case RW_T_INT64: case RW_T_FLOAT64: case RW_T_TIME: case RW_T_TIMESTAMP:
    case RW_T_TIMESTAMPTZ: case RW_T_SERIAL: return 8;
    case RW_T_DECIMAL: return 16;
    default: return 0;
  }
}

inline bool bit_get(const uint64_t* w, int64_t i) { return w == nullptr || ((w[i >> 6] >> (i & 63)) & 1); }

Datum read_datum(const rw_column& c, int64_t r) {
  Datum d;
  if (!bit_get(c.validity, r)) return d;
  d.null = false;
  const uint8_t* p = (const uint8_t*)c.data;
  if (is_varlen(c.type)) {
    d.s.assign((const char*)p + c.offsets[r], (size_t)(c.offsets[r + 1] - c.offsets[r]));
    return d;
  }
  switch (c.type) {
    case RW_T_BOOL: d.i = p[r] ? 1 : 0; break;
    case RW_T_INT16: { int16_t v; memcpy(&v, p + r * 2, 2); d.i = v; break; }
    case RW_T_INT32: case RW_T_DATE: { int32_t v; memcpy(&v, p + r * 4, 4); d.i = v; break; }
    case RW_T_FLOAT32: { float v; memcpy(&v, p + r * 4, 4); memcpy(&d.f32, &v, 4); d.f = v; break; }
    case RW_T_FLOAT64: { double v; memcpy(&v, p + r * 8, 8); d.f = v; break; }
    case RW_T_DECIMAL: { i128 v; memcpy(&v, p + r * 16, 16); d.i = v; break; }
    default: { int64_t v; memcpy(&v, p + r * 8, 8); d.i = v; break; }
  }
  return d;
}

// the float4 bits of d: those it was read with while d.f is still their widening (a copy), else d.f narrowed.  Widening
// and narrowing back returns every f32 but a signalling NaN unchanged; that one comes back quiet.
uint32_t f32_bits(const Datum& d) {
  float v;
  memcpy(&v, &d.f32, 4);
  const double w = v;
  if (memcmp(&w, &d.f, 8) != 0) v = (float)d.f;
  uint32_t b;
  memcpy(&b, &v, 4);
  return b;
}

// OrderedFloat equality: NaN == NaN, -0 == +0 (src/common/src/types/ordered_float.rs)
bool datum_eq(const Datum& a, const Datum& b, int type) {
  if (a.null || b.null) return a.null && b.null;
  if (is_varlen(type)) return a.s == b.s;
  if (is_float(type)) {
    if (std::isnan(a.f) || std::isnan(b.f)) return std::isnan(a.f) && std::isnan(b.f);
    return a.f == b.f;
  }
  return a.i == b.i;
}
// total order used by min/max (Ord on OrderedFloat: NaN is largest)
int datum_cmp_nonnull(const Datum& a, const Datum& b, int type) {
  if (is_float(type)) {
    bool an = std::isnan(a.f), bn = std::isnan(b.f);
    if (an || bn) return an == bn ? 0 : (an ? 1 : -1);
    return a.f < b.f ? -1 : (a.f > b.f ? 1 : 0);
  }
  return a.i < b.i ? -1 : (a.i > b.i ? 1 : 0);
}

typedef std::vector<Datum> Row;

// order-preserving byte encoding, ascending, NULLs largest (OrderType::ascending(),
// src/common/src/util/sort_util.rs:150-156 + NullsAre::default()==Largest :66-72); stands in for
// memcmp_serialize of the pk (join/hash_join.rs:710-713) and for HashKey equality classes
// (NULL == NULL, floats normalised: hash/key.rs:400-631).
void enc_datum(std::string& out, const Datum& d, int type) {
  if (d.null) { out.push_back((char)1); return; }
  out.push_back((char)0);
  unsigned char b[16];
  if (is_float(type)) {
    double f = d.f;
    if (std::isnan(f)) f = std::nan("");
    if (f == 0.0) f = 0.0;  // -0 -> +0
    uint64_t u; memcpy(&u, &f, 8);
    if (std::isnan(d.f)) u = 0x7ff8000000000000ull;
    u = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
    for (int k = 0; k < 8; k++) b[k] = (unsigned char)(u >> (56 - 8 * k));
    out.append((char*)b, 8);
  } else {
    unsigned __int128 u = (unsigned __int128)d.i ^ ((unsigned __int128)1 << 127);
    for (int k = 0; k < 16; k++) b[k] = (unsigned char)(u >> (120 - 8 * k));
    out.append((char*)b, 16);
  }
}
std::string enc_row(const Row& r, const std::vector<int>& idx, const std::vector<int>& types) {
  std::string s;
  for (int i : idx) enc_datum(s, r[i], types[i]);
  return s;
}

// ------------------------------------------------------------------ output chunks
struct OutCol {
  int type = 0;
  std::vector<uint8_t> data;
  std::vector<uint64_t> valid;
  std::vector<uint32_t> offsets;  // varlen columns: n + 1 entries
  bool has_null = false;
};
struct OutChunk {
  int64_t n = 0;
  std::vector<uint8_t> ops;
  std::vector<uint64_t> vis;
  bool all_vis = true;
  std::vector<OutCol> cols;
  std::vector<rw_column> views;
  std::vector<Row> rows;  // kept for noop elimination / debugging
};

}  // namespace

struct rwgpu_out {
  std::vector<OutChunk> chunks;
};

namespace {

void bit_push(std::vector<uint64_t>& w, int64_t i, bool v) {
  if ((size_t)(i >> 6) >= w.size()) w.push_back(0);
  if (v) w[i >> 6] |= (1ull << (i & 63));
}

void write_datum(OutCol& c, const Datum& d) {
  if (is_varlen(c.type)) {
    if (c.offsets.empty()) c.offsets.push_back(0);
    const int64_t r = (int64_t)c.offsets.size() - 1;
    bit_push(c.valid, r, !d.null);
    if (d.null) c.has_null = true;
    else c.data.insert(c.data.end(), d.s.begin(), d.s.end());
    c.offsets.push_back((uint32_t)c.data.size());
    return;
  }
  int w = type_width(c.type);
  size_t off = c.data.size();
  c.data.resize(off + w, 0);
  int64_t r = (int64_t)(off / w);
  bit_push(c.valid, r, !d.null);
  if (d.null) { c.has_null = true; return; }
  uint8_t* p = c.data.data() + off;
  switch (c.type) {
    case RW_T_BOOL: p[0] = d.i ? 1 : 0; break;
    case RW_T_INT16: { int16_t v = (int16_t)d.i; memcpy(p, &v, 2); break; }
    case RW_T_INT32: case RW_T_DATE: { int32_t v = (int32_t)d.i; memcpy(p, &v, 4); break; }
    case RW_T_FLOAT32: { uint32_t v = f32_bits(d); memcpy(p, &v, 4); break; }
    case RW_T_FLOAT64: { double v = d.f; memcpy(p, &v, 8); break; }
    case RW_T_DECIMAL: { i128 v = d.i; memcpy(p, &v, 16); break; }
    default: { int64_t v = (int64_t)d.i; memcpy(p, &v, 8); break; }
  }
}

// StreamChunk::eliminate_adjacent_noop_update  (src/common/src/array/stream_chunk.rs:331-392)
void eliminate_adjacent_noop_update(OutChunk& c) {
  int64_t len = c.n;
  auto vis = [&](int64_t i) { return (c.vis[i >> 6] >> (i & 63)) & 1; };
  auto set_invis = [&](int64_t i) { c.vis[i >> 6] &= ~(1ull << (i & 63)); c.all_vis = false; };
  auto is_del = [&](int64_t i) { return c.ops[i] == RW_OP_DELETE || c.ops[i] == RW_OP_UPDATE_DELETE; };
  auto is_ins = [&](int64_t i) { return c.ops[i] == RW_OP_INSERT || c.ops[i] == RW_OP_UPDATE_INSERT; };
  auto row_eq = [&](int64_t a, int64_t b) {
    for (size_t k = 0; k < c.cols.size(); k++)
      if (!datum_eq(c.rows[a][k], c.rows[b][k], c.cols[k].type)) return false;
    return true;
  };
  int64_t prev = -1;
  for (int64_t cur = 0; cur < len; cur++) {
    if (!vis(cur)) continue;
    if (prev >= 0 && ((is_del(prev) && is_ins(cur)) || (is_ins(prev) && is_del(cur))) && row_eq(prev, cur)) {
      set_invis(prev);
      set_invis(cur);
      prev = -1;
    } else {
      prev = cur;
    }
  }
  for (int64_t i = 0; i + 1 < len; i++) {
    if (c.ops[i] == RW_OP_UPDATE_DELETE && c.ops[i + 1] == RW_OP_UPDATE_INSERT) {
      bool dv = vis(i), iv = vis(i + 1);
      if (dv && !iv) c.ops[i] = RW_OP_DELETE;
      else if (!dv && iv) c.ops[i + 1] = RW_OP_INSERT;
    }
  }
}

// StreamChunkBuilder (src/common/src/array/stream_chunk_builder.rs:23-219)
struct ChunkBuilder {
  size_t max_chunk_size;
  std::vector<int> types;
  OutChunk cur;
  ChunkBuilder() : max_chunk_size(0) {}
  ChunkBuilder(size_t cap, const std::vector<int>& t) : max_chunk_size(cap), types(t) { reset(); }
  void reset() {
    cur = OutChunk();
    cur.cols.resize(types.size());
    for (size_t i = 0; i < types.size(); i++) cur.cols[i].type = types[i];
  }
  // append_iter_inner :189-219; returns true and moves the finished chunk into `out`
  bool append(uint8_t op, const Row& row, OutChunk* out) {
    cur.ops.push_back(op);
    for (size_t i = 0; i < types.size(); i++) write_datum(cur.cols[i], row[i]);
    bit_push(cur.vis, cur.n, true);
    cur.rows.push_back(row);
    cur.n++;
    if (((size_t)cur.n == max_chunk_size && op != RW_OP_UPDATE_DELETE) || (size_t)cur.n > max_chunk_size)
      return take(out);
    return false;
  }
  bool take(OutChunk* out) {
    if (cur.n == 0) return false;
    *out = std::move(cur);
    reset();
    return true;
  }
};

void finalize_views(rwgpu_out* o) {
  for (auto& c : o->chunks) {
    c.views.resize(c.cols.size());
    for (size_t i = 0; i < c.cols.size(); i++) {
      c.views[i].type = c.cols[i].type;
      c.views[i].reserved = 0;
      c.views[i].data = c.cols[i].data.data();
      c.views[i].validity = c.cols[i].has_null ? c.cols[i].valid.data() : nullptr;
      if (is_varlen(c.cols[i].type)) {
        if (c.cols[i].offsets.empty()) c.cols[i].offsets.push_back(0);
        if (c.cols[i].data.empty()) c.cols[i].data.push_back(0);  // a non-NULL data pointer even for zero bytes
        c.views[i].data = c.cols[i].data.data();
        c.views[i].offsets = c.cols[i].offsets.data();
      } else {
        c.views[i].offsets = nullptr;
      }
    }
  }
}

// ================================================================== HashAgg
struct AggOracle {
  std::vector<int> in_types, key_idx;
  std::vector<rw_agg_call> calls;
  int row_count_index = 0;
  bool append_only = false, strict = true;
  int chunk_size = 1024;
  std::vector<int> out_types;
  struct Group {
    Row key;
    Row states;
    bool has_prev = false;
    Row prev;
    bool dirty = false;
    // AggState::MaterializedInput (agg_state.rs:49-56, minput.rs:45-): the retractable min / max of call c is the
    // first row of the call's materialized input in (value, pk) order -- here the multiset of its non-NULL values
    std::vector<std::vector<Datum>> minput;
  };
  std::unordered_map<std::string, size_t> index;
  std::vector<Group> groups;
  std::vector<size_t> dirty;
  ChunkBuilder builder;

  Datum init_state(const rw_agg_call& c) const {
    Datum d;
    if (c.kind == RW_AGG_COUNT || c.kind == RW_AGG_SUM0) { d.null = false; d.i = 0; }  // init_state = "0i64"
    return d;
  }
};

const i128 DEC_MAX = (((i128)1) << 96) - 1;  // rust_decimal 96-bit mantissa

// the signatures general.rs declares over the types of rwgpu.h: sum :18-27 (sum(int2 / int4) -> int8, sum(int8) ->
// decimal, the internal sum(int8) -> int8 and sum0(int8) -> int8, sum(float4 / float8 / decimal) -> the same type),
// min / max(any type but boolean) -> the argument type :93-128, count() / count(any) -> int8 :155-162
bool agg_signature_ok(int kind, bool has_arg, int at, int ret) {
  switch (kind) {
    case RW_AGG_COUNT: return ret == RW_T_INT64;
    case RW_AGG_SUM0: return has_arg && at == RW_T_INT64 && ret == RW_T_INT64;
    case RW_AGG_SUM:
      if (!has_arg) return false;
      if (at == RW_T_INT16 || at == RW_T_INT32) return ret == RW_T_INT64;
      if (at == RW_T_INT64) return ret == RW_T_INT64 || ret == RW_T_DECIMAL;
      return (at == RW_T_FLOAT32 || at == RW_T_FLOAT64 || at == RW_T_DECIMAL) && ret == at;
    case RW_AGG_MIN:
    case RW_AGG_MAX: return has_arg && at != RW_T_BOOL && ret == at;
    default: return true;
  }
}

// one visible row into one call state: generated `update` wrapper src/expr/macro/src/gen.rs:838-912
// + sum/min/max/count bodies src/expr/impl/src/aggregate/general.rs:28-41,104,123,155-162
int agg_apply(const AggOracle& a, const rw_agg_call& c, Datum& st, const Datum& v, int arg_type, uint8_t op) {
  bool retract = (op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE);
  switch (c.kind) {
    case RW_AGG_COUNT:
      if (c.arg_col >= 0 && v.null) return RW_OK;  // (state, None) => state
      st.i += retract ? -1 : 1;
      return RW_OK;
    case RW_AGG_SUM:
    case RW_AGG_SUM0: {
      if (v.null) return RW_OK;
      if (st.null) { st.null = false; st.i = 0; st.f = 0; }  // S::default()
      if (is_float(arg_type)) {
        if (c.ret_type == RW_T_FLOAT32) {
          float s = (float)st.f, x = (float)v.f;
          st.f = retract ? (float)(s - x) : (float)(s + x);
        } else {
          st.f = retract ? st.f - v.f : st.f + v.f;
        }
        return RW_OK;
      }
      i128 r = retract ? st.i - v.i : st.i + v.i;
      if (c.ret_type == RW_T_DECIMAL) {
        if (r > DEC_MAX || r < -DEC_MAX) return fail(RW_ERR_NUMERIC_OUT_OF_RANGE, "Numeric out of range");
      } else {
        if (r > (i128)INT64_MAX || r < (i128)INT64_MIN) return fail(RW_ERR_NUMERIC_OUT_OF_RANGE, "Numeric out of range");
      }
      st.i = r;
      return RW_OK;
    }
    case RW_AGG_MIN:
    case RW_AGG_MAX: {
      // assert_eq!(op, Op::Insert, "attempt to retract on aggregate function .., but it is append-only")
      if (v.null) return RW_OK;  // also filtered by agg_call_filter_res (aggregate/mod.rs:81-109)
      if (!a.append_only) return fail(RW_ERR_CUDA, "internal: retractable min/max goes through agg_apply_minput");
      if (op != RW_OP_INSERT) return fail(RW_ERR_INCONSISTENT, "attempt to retract on append-only min/max");
      if (st.null) { st = v; return RW_OK; }  // state = "ref": first value
      // state.min(input) / state.max(input) (general.rs:104,123): Ord::min returns `self` and Ord::max `other` when the
      // two compare equal, so on a tie (+0 / -0, two NaNs) min keeps the state and max takes the input
      int cmp = datum_cmp_nonnull(v, st, arg_type);
      if ((c.kind == RW_AGG_MIN && cmp < 0) || (c.kind == RW_AGG_MAX && cmp >= 0)) st = v;
      return RW_OK;
    }
  }
  return fail(RW_ERR_UNSUPPORTED, "agg kind");
}

// retractable min / max: MaterializedInputState::apply_chunk (minput.rs:172-182) inserts / deletes the row in the call's
// materialized input (rows with a NULL argument are filtered out before, aggregate/mod.rs:81-109); get_output
// (minput.rs:184-245) returns the first row in order.  The state datum mirrors that output after every row.
int agg_apply_minput(const AggOracle& a, const rw_agg_call& c, std::vector<Datum>& rows, Datum& st, const Datum& v, int arg_type,
                     uint8_t op) {
  if (v.null) return RW_OK;
  const bool retract = (op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE);
  if (!retract) {
    rows.push_back(v);
  } else {
    size_t i = 0;
    while (i < rows.size() && datum_cmp_nonnull(rows[i], v, arg_type) != 0) i++;
    if (i == rows.size()) {
      if (a.strict) return fail(RW_ERR_INCONSISTENT, "retracting a row that is not in the materialized input");
    } else {
      rows[i] = rows.back();
      rows.pop_back();
    }
  }
  st = Datum();
  for (const Datum& x : rows) {
    if (st.null) { st = x; continue; }
    const int cmp = datum_cmp_nonnull(x, st, arg_type);
    if ((c.kind == RW_AGG_MIN && cmp < 0) || (c.kind == RW_AGG_MAX && cmp > 0)) st = x;
  }
  return RW_OK;
}

}  // namespace

struct rwo_agg {
  AggOracle a;
};
struct rwo_join;

extern "C" {

const char* rwo_last_error(void) { return g_err.c_str(); }
int32_t rwo_type_width(int32_t t) { return type_width(t); }

int32_t rwo_out_num_chunks(const rwgpu_out* o) { return o ? (int32_t)o->chunks.size() : 0; }
int64_t rwo_out_num_rows(const rwgpu_out* o) {
  int64_t n = 0;
  if (o) for (auto& c : o->chunks) n += c.n;
  return n;
}
int32_t rwo_out_chunk(const rwgpu_out* o, int32_t idx, rw_chunk* view) {
  if (!o || idx < 0 || (size_t)idx >= o->chunks.size()) return fail(RW_ERR_INVALID, "chunk index");
  const OutChunk& c = o->chunks[idx];
  view->n_rows = c.n;
  view->n_cols = (int32_t)c.cols.size();
  view->reserved = 0;
  view->ops = c.ops.data();
  view->visibility = c.all_vis ? nullptr : c.vis.data();
  view->columns = c.views.data();
  return RW_OK;
}
void rwo_out_release(rwgpu_out* o) { delete o; }

// ---- HashAggExecutor::new  (hash_agg.rs:185-239; schema: test_utils/agg_executor.rs:38-58)
int32_t rwo_agg_create(const rw_agg_desc* d, rwo_agg** out) {
  if (!d || !out) return fail(RW_ERR_INVALID, "null");
  auto* h = new rwo_agg();
  AggOracle& a = h->a;
  a.in_types.assign(d->input_types, d->input_types + d->n_input_cols);
  a.key_idx.assign(d->group_key_indices, d->group_key_indices + d->n_group_keys);
  a.calls.assign(d->calls, d->calls + d->n_calls);
  for (const rw_agg_call& c : a.calls) {
    const int at = c.arg_col >= 0 && c.arg_col < d->n_input_cols ? a.in_types[c.arg_col] : 0;
    if (c.arg_col >= d->n_input_cols) { delete h; return fail(RW_ERR_INVALID, "agg arg index"); }
    if (!agg_signature_ok(c.kind, c.arg_col >= 0, at, c.ret_type)) {
      delete h;
      return fail(RW_ERR_INVALID, "aggregate signature not defined by the reference (general.rs)");
    }
    if (c.kind < RW_AGG_COUNT || c.kind > RW_AGG_SUM0 || is_varlen(at)) { delete h; return fail(RW_ERR_UNSUPPORTED, "agg kind / argument type"); }
  }
  a.row_count_index = d->row_count_index;
  a.append_only = d->is_append_only != 0;
  a.strict = d->strict_consistency != 0;
  a.chunk_size = d->chunk_size > 0 ? d->chunk_size : 1024;
  for (int k : a.key_idx) a.out_types.push_back(a.in_types[k]);
  for (auto& c : a.calls) a.out_types.push_back(c.ret_type);
  a.builder = ChunkBuilder((size_t)a.chunk_size, a.out_types);
  *out = h;
  return RW_OK;
}
void rwo_agg_destroy(rwo_agg* h) { delete h; }

// ---- apply_chunk  (hash_agg.rs:332-409; per-row order inside a group is chunk order)
int32_t rwo_agg_push(rwo_agg* h, const rw_chunk* ch) {
  AggOracle& a = h->a;
  Row key(a.key_idx.size());
  for (int64_t r = 0; r < ch->n_rows; r++) {
    if (!bit_get(ch->visibility, r)) continue;
    std::string ks;
    for (size_t k = 0; k < a.key_idx.size(); k++) {
      key[k] = read_datum(ch->columns[a.key_idx[k]], r);
      enc_datum(ks, key[k], a.in_types[a.key_idx[k]]);
    }
    auto it = a.index.find(ks);
    size_t gi;
    if (it == a.index.end()) {
      gi = a.groups.size();
      a.index.emplace(ks, gi);
      a.groups.emplace_back();
      AggOracle::Group& g = a.groups.back();
      g.key = key;
      for (auto& c : a.calls) g.states.push_back(a.init_state(c));
      g.minput.resize(a.calls.size());
    } else {
      gi = it->second;
    }
    AggOracle::Group& g = a.groups[gi];
    if (!g.dirty) { g.dirty = true; a.dirty.push_back(gi); }
    uint8_t op = ch->ops[r];
    for (size_t c = 0; c < a.calls.size(); c++) {
      Datum v;
      int at = 0;
      if (a.calls[c].arg_col >= 0) {
        v = read_datum(ch->columns[a.calls[c].arg_col], r);
        at = a.in_types[a.calls[c].arg_col];
      }
      const bool minput = !a.append_only && (a.calls[c].kind == RW_AGG_MIN || a.calls[c].kind == RW_AGG_MAX);
      int rc = minput ? agg_apply_minput(a, a.calls[c], g.minput[c], g.states[c], v, at, op) : agg_apply(a, a.calls[c], g.states[c], v, at, op);
      if (rc != RW_OK) return rc;
    }
  }
  return RW_OK;
}

// ---- flush_data (emit-on-update) hash_agg.rs:412-514; AggGroup::get_outputs agg_group.rs:431-468;
//      build_outputs_change :545-606; OnlyOutputIfHasInput::infer_change_type :131-166
int32_t rwo_agg_flush(rwo_agg* h, uint64_t /*epoch*/, rwgpu_out** out) {
  AggOracle& a = h->a;
  auto* o = new rwgpu_out();
  OutChunk done;
  for (size_t gi : a.dirty) {
    AggOracle::Group& g = a.groups[gi];
    g.dirty = false;
    // row_count_of (agg_group.rs:55-79)
    int64_t rc = (int64_t)g.states[a.row_count_index].i;
    if (rc < 0) {
      if (a.strict) { delete o; return fail(RW_ERR_INCONSISTENT, "row count should be non-negative"); }
      rc = 0;
    }
    if (rc == 0) {  // reset value states (agg_group.rs:438-446); a materialized input is NOT reset ("in fact only
      // value states will be reset"): with zero rows it is empty anyway unless the stream is inconsistent
      for (size_t c = 0; c < a.calls.size(); c++) {
        const bool minput = !a.append_only && (a.calls[c].kind == RW_AGG_MIN || a.calls[c].kind == RW_AGG_MAX);
        if (!minput) g.states[c] = a.init_state(a.calls[c]);
      }
    }
    Row curr = g.states;  // value-state output == state datum
    int64_t prev_rc = 0;
    if (g.has_prev) {
      prev_rc = (int64_t)g.prev[a.row_count_index].i;
      if (prev_rc < 0) prev_rc = 0;
    }
    auto full = [&](const Row& outs) {
      Row r = g.key;
      r.insert(r.end(), outs.begin(), outs.end());
      return r;
    };
    if (prev_rc == 0 && rc == 0) {
      // none
    } else if (prev_rc == 0) {
      if (a.builder.append(RW_OP_INSERT, full(curr), &done)) o->chunks.push_back(std::move(done));
      g.prev = curr; g.has_prev = true;
    } else if (rc == 0) {
      if (a.builder.append(RW_OP_DELETE, full(g.prev), &done)) o->chunks.push_back(std::move(done));
      g.has_prev = false;
    } else {
      bool same = true;
      for (size_t c = 0; c < a.calls.size(); c++)
        if (!datum_eq(g.prev[c], curr[c], a.calls[c].ret_type)) { same = false; break; }
      if (!same) {
        a.builder.append(RW_OP_UPDATE_DELETE, full(g.prev), &done);  // never yields (asserted in reference)
        if (a.builder.append(RW_OP_UPDATE_INSERT, full(curr), &done)) o->chunks.push_back(std::move(done));
        g.prev = curr;
      }
    }
  }
  a.dirty.clear();
  if (a.builder.take(&done)) o->chunks.push_back(std::move(done));
  finalize_views(o);
  *out = o;
  return RW_OK;
}

int32_t rwo_agg_num_groups(rwo_agg* h, uint64_t* n) { *n = h->a.groups.size(); return RW_OK; }

}  // extern "C"

// ================================================================== HashJoin
namespace {

struct JRow {
  Row v;
  uint64_t degree = 0;
};
// JoinEntryState + the rows of one join key in the state table
// (join/hash_join.rs:736-830, join/join_row_set.rs:24-140)
struct Entry {
  std::map<std::string, JRow> table;  // "StateTable" rows under this join key, pk order
  bool cached = false;                // key present in the LRU (complete copy)
  bool btree = false;                 // JoinRowSet::BTree vs ::Vec
  std::vector<std::string> vec;       // Vec-mode order (pks)
};

struct JoinSideO {
  int n_cols = 0;
  std::vector<int> types, key_idx, pk_idx, stream_key;
  bool pk_in_jk = false;
  bool need_degree = false;
  int start_pos = 0;
  std::vector<std::pair<int, int>> i2o;  // (input idx, output idx)
  std::map<std::string, Entry> ht;
  uint64_t n_rows = 0;
};

bool is_subset(const std::vector<int>& a, const std::vector<int>& b) {
  for (int x : a) if (std::find(b.begin(), b.end(), x) == b.end()) return false;
  return true;
}

struct JoinOracle {
  int T = 0;
  JoinSideO side[2];
  std::vector<uint8_t> null_safe;
  std::vector<int> out_types;
  rw_join_cond cond;
  bool append_only_optimize = false;
  bool strict = true;
  size_t chunk_size = 1024;
  size_t entry_state_max_rows = 30000;  // config hash_join_entry_state_max_rows
};

// join/mod.rs:103-169
bool is_outer_side(int T, int S) { return T == RW_JOIN_FULL_OUTER || (T == RW_JOIN_LEFT_OUTER && S == 0) || (T == RW_JOIN_RIGHT_OUTER && S == 1); }
bool outer_side_null(int T, int S) { return T == RW_JOIN_FULL_OUTER || (T == RW_JOIN_LEFT_OUTER && S == 1) || (T == RW_JOIN_RIGHT_OUTER && S == 0); }
bool forward_exactly_once(int T, int S) { return ((T == RW_JOIN_LEFT_SEMI || T == RW_JOIN_LEFT_ANTI) && S == 0) || ((T == RW_JOIN_RIGHT_SEMI || T == RW_JOIN_RIGHT_ANTI) && S == 1); }
bool only_forward_matched_side(int T, int S) { return ((T == RW_JOIN_LEFT_SEMI || T == RW_JOIN_LEFT_ANTI) && S == 1) || ((T == RW_JOIN_RIGHT_SEMI || T == RW_JOIN_RIGHT_ANTI) && S == 0); }
bool is_semi(int T) { return T == RW_JOIN_LEFT_SEMI || T == RW_JOIN_RIGHT_SEMI; }
bool is_anti(int T) { return T == RW_JOIN_LEFT_ANTI || T == RW_JOIN_RIGHT_ANTI; }
bool need_left_degree(int T) { return T == RW_JOIN_FULL_OUTER || T == RW_JOIN_LEFT_OUTER || T == RW_JOIN_LEFT_ANTI || T == RW_JOIN_LEFT_SEMI; }
bool need_right_degree(int T) { return T == RW_JOIN_FULL_OUTER || T == RW_JOIN_RIGHT_OUTER || T == RW_JOIN_RIGHT_ANTI || T == RW_JOIN_RIGHT_SEMI; }

// JoinRowSet::try_insert (join_row_set.rs:60-95) + JoinEntryState::insert (hash_join.rs:760-787)
int entry_cache_insert(JoinOracle& j, Entry& e, const std::string& pk) {
  if (!e.btree && e.vec.size() >= 4) { e.btree = true; e.vec.clear(); }
  if (e.btree) return RW_OK;  // membership == table (checked by caller)
  if (std::find(e.vec.begin(), e.vec.end(), pk) != e.vec.end()) {
    if (j.strict) return fail(RW_ERR_INCONSISTENT, "double inserting a join state entry");
    e.vec.erase(std::find(e.vec.begin(), e.vec.end(), pk));
  }
  e.vec.push_back(pk);
  return RW_OK;
}
// JoinRowSet::remove (join_row_set.rs:97-117); called after the row left `table`
void entry_cache_remove(Entry& e, const std::string& pk) {
  if (e.btree) {
    if (e.table.size() <= 2) {  // MAX_VEC_SIZE / 2
      e.btree = false;
      e.vec.clear();
      for (auto& kv : e.table) e.vec.push_back(kv.first);
    }
  } else {
    auto it = std::find(e.vec.begin(), e.vec.end(), pk);
    if (it != e.vec.end()) {  // swap_remove
      *it = e.vec.back();
      e.vec.pop_back();
    }
  }
}

struct JoinEmit {
  JoinOracle& j;
  int S;  // update side
  ChunkBuilder& b;
  rwgpu_out* o;
  void push(uint8_t op, const Row* upd, const Row* mat) {
    // JoinStreamChunkBuilder::{append_row,append_row_update,append_row_matched} builder.rs:84-148
    Row r(j.out_types.size());
    JoinSideO& su = j.side[S];
    JoinSideO& sm = j.side[1 - S];
    for (auto& m : su.i2o) r[m.second] = upd ? (*upd)[m.first] : Datum();
    for (auto& m : sm.i2o) r[m.second] = mat ? (*mat)[m.first] : Datum();
    OutChunk done;
    if (b.append(op, r, &done)) {
      eliminate_adjacent_noop_update(done);  // JoinChunkBuilder::post_process builder.rs:166-168
      o->chunks.push_back(std::move(done));
    }
  }
};

// check_join_condition (hash_join.rs:1362-1384), restricted to one integer comparison
bool cond_ok(const JoinOracle& j, int S, const Row& upd, const Row& mat) {
  if (j.cond.cmp == RW_CMP_NONE) return true;
  int nl = j.side[0].n_cols;
  auto get = [&](int idx) -> const Datum& {
    bool left = idx < nl;
    int local = left ? idx : idx - nl;
    bool from_upd = (left && S == 0) || (!left && S == 1);
    return from_upd ? upd[local] : mat[local];
  };
  const Datum& a = get(j.cond.lhs);
  const Datum& b = get(j.cond.rhs);
  if (a.null || b.null) return false;  // NULL => unwrap_or(false)
  switch (j.cond.cmp) {
    case RW_CMP_LT: return a.i < b.i;
    case RW_CMP_LE: return a.i <= b.i;
    case RW_CMP_GT: return a.i > b.i;
    case RW_CMP_GE: return a.i >= b.i;
    case RW_CMP_EQ: return a.i == b.i;
    case RW_CMP_NE: return a.i != b.i;
  }
  return false;
}

}  // namespace

struct rwo_join {
  JoinOracle j;
};

extern "C" {

// ---- HashJoinExecutor::new_with_cache_size (hash_join.rs:304-580)
int32_t rwo_join_create(const rw_join_desc* d, rwo_join** out) {
  if (!d || !out) return fail(RW_ERR_INVALID, "null");
  auto* h = new rwo_join();
  JoinOracle& j = h->j;
  j.T = d->join_type;
  const rw_join_side_desc* sd[2] = {&d->left, &d->right};
  for (int s = 0; s < 2; s++) {
    JoinSideO& x = j.side[s];
    x.n_cols = sd[s]->n_cols;
    x.types.assign(sd[s]->types, sd[s]->types + sd[s]->n_cols);
    x.key_idx.assign(sd[s]->key_indices, sd[s]->key_indices + d->n_keys);
    x.pk_idx.assign(sd[s]->pk_indices, sd[s]->pk_indices + sd[s]->n_pk);
    x.stream_key.assign(sd[s]->stream_key, sd[s]->stream_key + sd[s]->n_stream_key);
    x.pk_in_jk = is_subset(x.stream_key, x.key_idx);  // :377-378
    // varlen columns are payload only at this boundary (rwgpu.h): a varlen join key would be `KeySerialized`
    for (int k : x.key_idx) if (is_varlen(x.types[k])) { delete h; return fail(RW_ERR_UNSUPPORTED, "varlen join key"); }
    for (int k : x.pk_idx) if (is_varlen(x.types[k])) { delete h; return fail(RW_ERR_UNSUPPORTED, "varlen pk column"); }
  }
  j.side[0].start_pos = 0;
  j.side[1].start_pos = j.side[0].n_cols;
  j.null_safe.assign(d->null_safe, d->null_safe + d->n_keys);
  j.cond = d->cond;
  if (j.cond.cmp != RW_CMP_NONE) {  // the one integer comparison the C ABI carries (rwgpu.h rw_join_cond)
    const int tot = j.side[0].n_cols + j.side[1].n_cols;
    if (j.cond.cmp < 0 || j.cond.cmp > RW_CMP_NE || j.cond.lhs < 0 || j.cond.lhs >= tot || j.cond.rhs < 0 || j.cond.rhs >= tot) {
      delete h;
      return fail(RW_ERR_INVALID, "join condition");
    }
    auto col_type = [&](int idx) { return idx < j.side[0].n_cols ? j.side[0].types[idx] : j.side[1].types[idx - j.side[0].n_cols]; };
    if (!cmp_operands_ok(col_type(j.cond.lhs), col_type(j.cond.rhs))) { delete h; return fail(RW_ERR_UNSUPPORTED, "join condition operand types"); }
  }
  j.strict = d->strict_consistency != 0;
  j.chunk_size = (size_t)std::max(d->chunk_size > 0 ? d->chunk_size : 1024, 2);  // builder.rs:44-47
  j.append_only_optimize = d->is_append_only && j.side[0].pk_in_jk && j.side[1].pk_in_jk;  // :381
  j.side[0].need_degree = need_left_degree(j.T) && !j.side[1].pk_in_jk;   // :397
  j.side[1].need_degree = need_right_degree(j.T) && !j.side[0].pk_in_jk;  // :398
  // output schema :337-359 and i2o mapping :400-410 / builder.rs:63-80
  int left_len = j.side[0].n_cols;  // columns of the natural output that come from the left input
  std::vector<int> nat;
  if (j.T == RW_JOIN_LEFT_SEMI || j.T == RW_JOIN_LEFT_ANTI) { nat = j.side[0].types; }
  else if (j.T == RW_JOIN_RIGHT_SEMI || j.T == RW_JOIN_RIGHT_ANTI) { nat = j.side[1].types; left_len = 0; }
  else { nat = j.side[0].types; nat.insert(nat.end(), j.side[1].types.begin(), j.side[1].types.end()); }
  for (int oi = 0; oi < d->n_output; oi++) {
    int idx = d->output_indices[oi];
    if (idx < 0 || idx >= (int)nat.size()) { delete h; return fail(RW_ERR_INVALID, "output_indices out of bound"); }
    j.out_types.push_back(nat[idx]);
    if (idx < left_len) j.side[0].i2o.push_back({idx, oi});
    else j.side[1].i2o.push_back({idx - left_len, oi});
  }
  *out = h;
  return RW_OK;
}
void rwo_join_destroy(rwo_join* h) { delete h; }

// ---- eq_join_oneside (hash_join.rs:925-1062) + handle_match_rows (:1072-1244) + handle_match_row (:1247-1357)
int32_t rwo_join_push(rwo_join* h, int32_t S, const rw_chunk* ch, rwgpu_out** out) {
  JoinOracle& j = h->j;
  JoinSideO& su = j.side[S];
  JoinSideO& sm = j.side[1 - S];
  auto* o = new rwgpu_out();
  ChunkBuilder b(j.chunk_size, j.out_types);
  JoinEmit em{j, S, b, o};
  const int T = j.T;
  for (int64_t r = 0; r < ch->n_rows; r++) {
    if (!bit_get(ch->visibility, r)) continue;  // rows_with_holes :977-980
    Row u(su.n_cols);
    for (int c = 0; c < su.n_cols; c++) u[c] = read_datum(ch->columns[c], r);
    uint8_t op = ch->ops[r];
    bool ins = (op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT);  // :1020-1039
    uint8_t jop = ins ? RW_OP_INSERT : RW_OP_DELETE;
    // NULL rule :985-999: key.null_bitmap().is_subset(null_matched)
    bool never = false;
    for (size_t k = 0; k < su.key_idx.size(); k++)
      if (u[su.key_idx[k]].null && !j.null_safe[k]) never = true;
    if (never) {  // CacheResult::NeverMatch :1126-1135
      if ((is_anti(T) && forward_exactly_once(T, S)) || is_outer_side(T, S)) em.push(jop, &u, nullptr);
      continue;
    }
    std::string key = enc_row(u, su.key_idx, su.types);
    Entry& me = sm.ht[key];  // take_state_opt (join/hash_join.rs:537-550)
    bool cache_hit = me.cached;
    std::vector<std::string> order;
    if (cache_hit && !me.btree) order = me.vec;
    else for (auto& kv : me.table) order.push_back(kv.first);
    size_t entry_state_count = 0;
    bool refill_btree = false;
    std::vector<std::string> refill_vec;
    uint64_t degree = 0;
    const std::string* append_only_matched_pk = nullptr;
    for (auto& mpk : order) {
      JRow& m = me.table[mpk];
      if (!cache_hit && entry_state_count <= j.entry_state_max_rows) {  // cache refill :1176-1182
        if (!refill_btree && refill_vec.size() >= 4) { refill_btree = true; refill_vec.clear(); }
        if (!refill_btree) refill_vec.push_back(mpk);
        entry_state_count++;
      }
      // handle_match_row :1247-1357
      if (cond_ok(j, S, u, m.v)) {
        degree++;
        if (ins && !forward_exactly_once(T, S)) {
          // with_match_on_insert builder.rs:184-231 (uses m.degree BEFORE the increment)
          if (is_anti(T)) { if (m.degree == 0 && only_forward_matched_side(T, S)) em.push(RW_OP_DELETE, nullptr, &m.v); }
          else if (is_semi(T)) { if (m.degree == 0 && only_forward_matched_side(T, S)) em.push(RW_OP_INSERT, nullptr, &m.v); }
          else if (m.degree == 0 && outer_side_null(T, S)) { em.push(RW_OP_DELETE, nullptr, &m.v); em.push(RW_OP_INSERT, &u, &m.v); }
          else em.push(RW_OP_INSERT, &u, &m.v);
        }
        if (sm.need_degree) m.degree += ins ? 1 : (uint64_t)-1;  // update_degree join/hash_join.rs:355-380
        if (!ins && !forward_exactly_once(T, S)) {
          // with_match_on_delete builder.rs:233-284 (uses m.degree AFTER the decrement)
          if (is_anti(T)) { if (m.degree == 0 && only_forward_matched_side(T, S)) em.push(RW_OP_INSERT, nullptr, &m.v); }
          else if (is_semi(T)) { if (m.degree == 0 && only_forward_matched_side(T, S)) em.push(RW_OP_DELETE, nullptr, &m.v); }
          else if (m.degree == 0 && outer_side_null(T, S)) { em.push(RW_OP_DELETE, &u, &m.v); em.push(RW_OP_INSERT, nullptr, &m.v); }
          else em.push(RW_OP_DELETE, &u, &m.v);
        }
      }
      if (j.append_only_optimize) append_only_matched_pk = &mpk;  // :1339-1345 (regardless of cond)
    }
    // forward rows depending on join types :1198-1210
    if (degree == 0) {
      if ((is_anti(T) && forward_exactly_once(T, S)) || is_outer_side(T, S)) em.push(jop, &u, nullptr);
    } else if (is_semi(T) && forward_exactly_once(T, S)) {
      em.push(jop, &u, nullptr);
    }
    // cache refill :1212-1215
    if (!cache_hit && entry_state_count <= j.entry_state_max_rows) {
      me.cached = true;
      me.btree = refill_btree;
      me.vec = refill_vec;
    }
    // append-only optimisation :1222-1228
    if (j.append_only_optimize && append_only_matched_pk) {
      std::string pk = *append_only_matched_pk;
      me.table.erase(pk);
      if (me.cached) entry_cache_remove(me, pk);
      sm.n_rows--;
      continue;
    }
    // own-side state update :1230-1242 ; JoinHashMap::insert / delete join/hash_join.rs:591-681
    std::string pk = enc_row(u, su.pk_idx, su.types);
    Entry& ue = su.ht[key];
    if (ins) {
      bool exists = ue.table.count(pk) != 0;
      if (ue.cached) {
        if (exists && ue.btree && j.strict) { delete o; return fail(RW_ERR_INCONSISTENT, "double inserting a join state entry"); }
        int rc = entry_cache_insert(j, ue, pk);
        if (rc != RW_OK) { delete o; return rc; }
      } else if (su.pk_in_jk) {
        ue.cached = true; ue.btree = false; ue.vec.assign(1, pk);
      }
      if (exists && j.strict && !ue.cached) { delete o; return fail(RW_ERR_INCONSISTENT, "double insert into state table"); }
      JRow jr; jr.v = u; jr.degree = su.need_degree ? degree : 0;
      if (!exists) su.n_rows++;
      ue.table[pk] = jr;
    } else {
      bool exists = ue.table.count(pk) != 0;
      if (!exists) {
        if (j.strict) { delete o; return fail(RW_ERR_INCONSISTENT, "removing a join state entry but it is not in the cache"); }
      } else {
        ue.table.erase(pk);
        su.n_rows--;
        if (ue.cached) entry_cache_remove(ue, pk);
      }
    }
  }
  OutChunk done;
  if (b.take(&done)) {  // :1059-1061
    eliminate_adjacent_noop_update(done);
    o->chunks.push_back(std::move(done));
  }
  finalize_views(o);
  *out = o;
  return RW_OK;
}

int32_t rwo_join_barrier(rwo_join*, uint64_t) { return RW_OK; }  // flush_data :754-766 (state stubbed to memory)
int32_t rwo_join_stats(rwo_join* h, uint64_t* l, uint64_t* r) {
  *l = h->j.side[0].n_rows; *r = h->j.side[1].n_rows;
  return RW_OK;
}

// ================================================================== vnode / dispatch
// CRC-32 (IEEE 802.3) as implemented by crc32fast 1.5.0 (Cargo.lock:3247); call sites
// src/common/src/util/hash_util.rs:24-33
static uint32_t crc_table[256];
static bool crc_init_done = false;
static void crc_init() {
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : (c >> 1);
    crc_table[i] = c;
  }
  crc_init_done = true;
}
uint32_t rwo_crc32(const uint8_t* p, int64_t n) {
  if (!crc_init_done) crc_init();
  uint32_t c = 0xFFFFFFFFu;
  for (int64_t i = 0; i < n; i++) c = crc_table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

// raw_double_bits (src/common/src/types/ordered_float.rs:852-870) via Float::integer_decode
static uint64_t raw_double_bits_f64(double f) {
  if (std::isnan(f)) return 0x7ff8000000000000ull;
  uint64_t bits; memcpy(&bits, &f, 8);
  int64_t sign = (bits >> 63) == 0 ? 1 : -1;
  int16_t exp = (int16_t)((bits >> 52) & 0x7ff);
  uint64_t man = exp == 0 ? (bits & 0xfffffffffffffull) << 1 : (bits & 0xfffffffffffffull) | 0x10000000000000ull;
  exp -= 1023 + 52;
  if (man == 0) return 0;
  uint64_t e = (uint64_t)(uint16_t)exp;
  return (man & 0x000fffffffffffffull) | ((e << 52) & 0x7ff0000000000000ull) | (((uint64_t)(sign > 0) << 63));
}
static uint64_t raw_double_bits_f32(float f) {
  if (std::isnan(f)) return 0x7ff8000000000000ull;
  uint32_t bits; memcpy(&bits, &f, 4);
  int64_t sign = (bits >> 31) == 0 ? 1 : -1;
  int16_t exp = (int16_t)((bits >> 23) & 0xff);
  uint32_t man32 = exp == 0 ? (bits & 0x7fffff) << 1 : (bits & 0x7fffff) | 0x800000;
  exp -= 127 + 23;
  uint64_t man = man32;
  if (man == 0) return 0;
  uint64_t e = (uint64_t)(uint16_t)exp;
  return (man & 0x000fffffffffffffull) | ((e << 52) & 0x7ff0000000000000ull) | (((uint64_t)(sign > 0) << 63));
}

// bytes fed to the hasher for one datum: Array::hash_at (src/common/src/array/mod.rs:280-288),
// NULL_VAL_FOR_HASH = 0xfffffff0 (:97); ints = native-endian bytes (types/scalar_impl.rs:47-49).
// Date/Time/Timestamp/Decimal go through chrono / rust_decimal Hash impls that are not in the tree:
// for those we feed the ABI value's LE bytes (self-consistent, "vnode parity unpinned", SURVEY §7.2).
static void hash_bytes(std::string& s, const rw_column& c, int64_t r) {
  if (!bit_get(c.validity, r)) { uint32_t v = 0xfffffff0u; s.append((char*)&v, 4); return; }
  const uint8_t* p = (const uint8_t*)c.data;
  int w = type_width(c.type);
  if (c.type == RW_T_FLOAT64) { double f; memcpy(&f, p + r * 8, 8); uint64_t u = raw_double_bits_f64(f); s.append((char*)&u, 8); }
  else if (c.type == RW_T_FLOAT32) { float f; memcpy(&f, p + r * 4, 4); uint64_t u = raw_double_bits_f32(f); s.append((char*)&u, 8); }
  else s.append((const char*)p + r * w, w);
}

// compute_vnode_from_row_id (src/common/src/util/row_id.rs:135-173)
static uint16_t vnode_from_row_id(int64_t id, int vnode_count) {
  uint32_t vnode_bit = 10;
  if (vnode_count > 1024) { vnode_bit = 0; while ((1u << vnode_bit) < (uint32_t)vnode_count) vnode_bit++; }
  uint32_t seq_bit = 22 - vnode_bit;
  uint64_t part = ((uint64_t)id >> seq_bit) & ((1ull << vnode_bit) - 1);
  return (uint16_t)(part % (uint64_t)vnode_count);
}

// the arguments the device's make_vnode_plan (csrc/shuffle.cu) accepts, refused with the same status codes
static int vnode_args(const rw_chunk* ch, const int32_t* keys, int32_t n_keys, int32_t vnode_count) {
  if (n_keys < 1 || n_keys > 8) return fail(RW_ERR_UNSUPPORTED, "1..8 distribution key columns");
  if (vnode_count < 1 || vnode_count > 32768) return fail(RW_ERR_INVALID, "vnode_count (vnode.rs:79 MAX_COUNT = 2^15)");
  for (int k = 0; k < ch->n_cols; k++)
    if (is_varlen(ch->columns[k].type)) return fail(RW_ERR_UNSUPPORTED, "the hash shuffle does not carry varlen columns");
  for (int k = 0; k < n_keys; k++)
    if (keys[k] < 0 || keys[k] >= ch->n_cols) return fail(RW_ERR_INVALID, "key index");
  return RW_OK;
}

// VirtualNode::compute_chunk (src/common/src/hash/consistent_hash/vnode.rs:151-182);
// get_hash_values hashes only VISIBLE rows (data_chunk.rs:338-355) => invisible rows: crc32("")=0
int32_t rwo_vnode_compute(const rw_chunk* ch, const int32_t* keys, int32_t n_keys, int32_t vnode_count, uint16_t* out) {
  if (!ch || !keys || !out) return fail(RW_ERR_INVALID, "null");
  int rc = vnode_args(ch, keys, n_keys, vnode_count);
  if (rc != RW_OK) return rc;
  if (n_keys == 1 && ch->columns[keys[0]].type == RW_T_SERIAL) {
    const rw_column& c = ch->columns[keys[0]];
    for (int64_t r = 0; r < ch->n_rows; r++) {
      if (bit_get(c.validity, r)) {
        int64_t id; memcpy(&id, (const uint8_t*)c.data + r * 8, 8);
        out[r] = vnode_from_row_id(id, vnode_count);
      } else {  // hash the entire row
        std::string s;
        for (int k = 0; k < ch->n_cols; k++) hash_bytes(s, ch->columns[k], r);
        out[r] = (uint16_t)(rwo_crc32((const uint8_t*)s.data(), (int64_t)s.size()) % (uint32_t)vnode_count);
      }
    }
    return RW_OK;
  }
  for (int64_t r = 0; r < ch->n_rows; r++) {
    std::string s;
    if (bit_get(ch->visibility, r))
      for (int k = 0; k < n_keys; k++) hash_bytes(s, ch->columns[keys[k]], r);
    out[r] = (uint16_t)(rwo_crc32((const uint8_t*)s.data(), (int64_t)s.size()) % (uint32_t)vnode_count);
  }
  return RW_OK;
}

// the op rewrite of HashDataDispatcher::dispatch_data (src/stream/src/executor/dispatch.rs:976-1023): a visible U+
// pairs with the last visible U- that no earlier U+ has taken (`last_update_delete_row_idx.take()`), whatever visible
// +/- rows lie between them; a U- that a later U- replaces keeps its op
int32_t rwo_dispatch_rewrite_ops(const rw_chunk* ch, const int32_t* keys, int32_t n_keys, uint8_t* out_ops) {
  if (!ch || !keys || !out_ops) return fail(RW_ERR_INVALID, "null");
  int rc = vnode_args(ch, keys, n_keys, 256);
  if (rc != RW_OK) return rc;
  int64_t last_ud = -1;
  for (int64_t r = 0; r < ch->n_rows; r++) {
    uint8_t op = ch->ops[r];
    out_ops[r] = op;
    if (!bit_get(ch->visibility, r)) continue;
    if (op == RW_OP_UPDATE_DELETE) last_ud = r;
    else if (op == RW_OP_UPDATE_INSERT) {
      if (last_ud < 0) return fail(RW_ERR_INCONSISTENT, "missing U- before U+");
      bool changed = false;
      for (int k = 0; k < n_keys; k++) {
        const rw_column& c = ch->columns[keys[k]];
        if (!datum_eq(read_datum(c, last_ud), read_datum(c, r), c.type)) changed = true;
      }
      if (changed) { out_ops[last_ud] = RW_OP_DELETE; out_ops[r] = RW_OP_INSERT; }
      last_ud = -1;
    }
  }
  if (last_ud >= 0) return fail(RW_ERR_INCONSISTENT, "missing U+ after U-");
  return RW_OK;
}

// standalone StreamChunk::eliminate_adjacent_noop_update over a host chunk (for tests)
int32_t rwo_eliminate_adjacent_noop_update(const rw_chunk* ch, uint8_t* out_ops, uint64_t* out_vis) {
  OutChunk c;
  c.n = ch->n_rows;
  c.ops.assign(ch->ops, ch->ops + ch->n_rows);
  c.vis.assign((size_t)((ch->n_rows + 63) / 64), 0);
  c.cols.resize(ch->n_cols);
  for (int k = 0; k < ch->n_cols; k++) c.cols[k].type = ch->columns[k].type;
  for (int64_t r = 0; r < ch->n_rows; r++) {
    if (bit_get(ch->visibility, r)) c.vis[r >> 6] |= 1ull << (r & 63);
    Row row(ch->n_cols);
    for (int k = 0; k < ch->n_cols; k++) row[k] = read_datum(ch->columns[k], r);
    c.rows.push_back(row);
  }
  eliminate_adjacent_noop_update(c);
  memcpy(out_ops, c.ops.data(), (size_t)ch->n_rows);
  memcpy(out_vis, c.vis.data(), c.vis.size() * 8);
  return RW_OK;
}

}  // extern "C"

// FilterExecutorInner::filter (src/stream/src/executor/filter.rs:58-150), restated literally: the chunk is
// compacted first (execute_inner, filter.rs:182; a row with op 0 is invisible like a cleared visibility bit), the
// predicate gives Option<bool> per row (`res.unwrap_or(false)`, :79), then the op rules produce new ops / visibility for
// the compacted rows.  The results are scattered back to the positions of the input's visible rows (invisible input rows
// keep their op, op 0 included, and stay invisible) so that the signature equals rwgpu_filter's.
// Predicate = conjunction of integer comparisons with SQL three-valued logic: a NULL operand makes the
// term NULL; AND of terms is NULL/false unless every term is true -> unwrap_or(false) == "all terms true".
// The reference only sees U- immediately followed by U+ (stream_chunk.rs:40-42).  The project's rule for anything else
// (the device's): a U- pairs with the next visible row only if that row is a U+, a U+ with the previous visible row only
// if that row is a U-; an unpaired U- or U+ is filtered like a - or + and keeps its op.
extern "C" int32_t rwo_filter(const rw_chunk* ch, const rw_filter_term* terms, int32_t n_terms, int32_t upsert, uint8_t* out_ops,
                              uint64_t* out_visibility, int64_t* n_visible) {
  if (!ch || !terms || !out_ops || !out_visibility) return fail(RW_ERR_INVALID, "null");
  const int64_t n = ch->n_rows;
  if (n_terms < 1 || n_terms > 8) return fail(RW_ERR_UNSUPPORTED, "filter: 1..8 conjuncts");
  for (int k = 0; k < n_terms; k++) {
    const rw_filter_term& t = terms[k];
    if (t.cmp < RW_CMP_LT || t.cmp > RW_CMP_NE) return fail(RW_ERR_INVALID, "filter: comparison");
    if (t.lhs_col < 0 || t.lhs_col >= ch->n_cols || t.rhs_col < -1 || t.rhs_col >= ch->n_cols) return fail(RW_ERR_INVALID, "filter: column index");
    const int lt = ch->columns[t.lhs_col].type, rt = t.rhs_col >= 0 ? ch->columns[t.rhs_col].type : lt;  // a constant takes the lhs's type
    if (!cmp_operands_ok(lt, rt)) return fail(RW_ERR_UNSUPPORTED, "filter: operand types");
  }
  // compact_vis
  std::vector<int64_t> pos;
  for (int64_t r = 0; r < n; r++)
    if (ch->ops[r] != 0 && bit_get(ch->visibility, r)) pos.push_back(r);
  // pred_output: Option<bool> per compacted row
  auto pred = [&](int64_t r) -> int {  // 1 true, 0 false, -1 NULL
    bool any_null = false, any_false = false;
    for (int k = 0; k < n_terms; k++) {
      const rw_filter_term& t = terms[k];
      Datum a = read_datum(ch->columns[t.lhs_col], r), b;
      if (t.rhs_col >= 0) b = read_datum(ch->columns[t.rhs_col], r);
      else { b.null = false; b.i = t.rhs_const; }
      if (a.null || b.null) { any_null = true; continue; }
      bool v = false;
      switch (t.cmp) {
        case RW_CMP_LT: v = a.i < b.i; break;
        case RW_CMP_LE: v = a.i <= b.i; break;
        case RW_CMP_GT: v = a.i > b.i; break;
        case RW_CMP_GE: v = a.i >= b.i; break;
        case RW_CMP_EQ: v = a.i == b.i; break;
        default: v = a.i != b.i; break;
      }
      if (!v) any_false = true;
    }
    return any_false ? 0 : (any_null ? -1 : 1);
  };
  const size_t m = pos.size();
  std::vector<uint8_t> new_ops(m);
  std::vector<bool> new_vis(m);
  auto op_at = [&](size_t i) { return ch->ops[pos[i]]; };
  for (size_t i = 0; i < m; i++) {
    const uint8_t op = op_at(i);
    const bool res = pred(pos[i]) == 1;  // unwrap_or(false)
    if (upsert) {  // :82-106
      new_ops[i] = (op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT) && res ? RW_OP_INSERT : RW_OP_DELETE;
      new_vis[i] = true;
    } else if (op == RW_OP_UPDATE_DELETE && i + 1 < m && op_at(i + 1) == RW_OP_UPDATE_INSERT) {  // :112-141, one pair
      const bool last_res = res, res2 = pred(pos[i + 1]) == 1;
      if (last_res && !res2) { new_ops[i] = RW_OP_DELETE; new_ops[i + 1] = RW_OP_UPDATE_INSERT; new_vis[i] = true; new_vis[i + 1] = false; }
      else if (!last_res && res2) { new_ops[i] = RW_OP_UPDATE_DELETE; new_ops[i + 1] = RW_OP_INSERT; new_vis[i] = false; new_vis[i + 1] = true; }
      else { new_ops[i] = RW_OP_UPDATE_DELETE; new_ops[i + 1] = RW_OP_UPDATE_INSERT; new_vis[i] = new_vis[i + 1] = last_res; }
      i++;
    } else {  // + / - (:108-111), and an unpaired U- or U+ by the project's rule
      new_ops[i] = op;
      new_vis[i] = res;
    }
  }
  if (n) memcpy(out_ops, ch->ops, (size_t)n);
  memset(out_visibility, 0, (size_t)((n + 63) / 64) * 8);
  int64_t cnt = 0;
  for (size_t i = 0; i < m; i++) {
    out_ops[pos[i]] = new_ops[i];
    if (new_vis[i]) { out_visibility[pos[i] >> 6] |= 1ull << (pos[i] & 63); cnt++; }
  }
  if (n_visible) *n_visible = cnt;
  return RW_OK;
}

// single-state evaluation used to pin agg_apply against the reference's aggregate-function
// tests (src/expr/impl/src/aggregate/general.rs:175-186 `test_agg`): create_state, update over the
// visible rows of `ch`, get_result.
extern "C" int32_t rwo_agg_eval(const rw_agg_call* call, int32_t arg_type, const rw_chunk* ch, int32_t* is_null,
                                int64_t* out_lo, int64_t* out_hi, double* out_f) {
  AggOracle a;
  a.append_only = true;  // the aggregate FUNCTIONS of general.rs are the append-only value states
  Datum st = a.init_state(*call);
  for (int64_t r = 0; r < ch->n_rows; r++) {
    if (!bit_get(ch->visibility, r)) continue;
    Datum v;
    if (call->arg_col >= 0) v = read_datum(ch->columns[call->arg_col], r);
    int rc = agg_apply(a, *call, st, v, arg_type, ch->ops[r]);
    if (rc != RW_OK) return rc;
  }
  *is_null = st.null ? 1 : 0;
  *out_lo = (int64_t)(uint64_t)(unsigned __int128)st.i;
  *out_hi = (int64_t)(st.i >> 64);
  *out_f = st.f;
  return RW_OK;
}


// ================================================================== Project
// apply_project_exprs (src/stream/src/executor/project/project_scalar.rs:91-108) for integer expressions in postfix
// form (include/rwgpu.h RW_EX_*): NonStrictExpression::eval_infallible -- a NULL operand or a failed evaluation
// (checked_add / checked_sub / checked_mul / checked_neg overflow of the operation's own result type `arg`:
// src/expr/impl/src/scalar/arithmetic_op.rs general_*; division by zero; MIN % -1 (checked_rem); a result that does not
// fit the expression's integer type) makes the row's value NULL.  tumble_start: src/expr/impl/src/scalar/tumble.rs:91-112
// (get_window_start_with_offset, zero offset), over a DATE the timestamp of its midnight (:34-37); tumble_end = start +
// window.
extern "C" int32_t rwo_project(const rw_chunk* ch, const rw_project_expr* exprs, int32_t n_exprs, void* const* out_data,
                               uint64_t* const* out_validity, uint32_t* has_null) {
  const int64_t n = ch->n_rows;
  auto int_type = [](int t) {
    switch (t) {
      case RW_T_INT16: case RW_T_INT32: case RW_T_INT64: case RW_T_DATE: case RW_T_TIME: case RW_T_TIMESTAMP: case RW_T_TIMESTAMPTZ:
      case RW_T_SERIAL: return true;
      default: return false;
    }
  };
  auto type_min = [](int t) -> i128 {
    const int w = type_width(t);
    return w == 2 ? (i128)INT16_MIN : w == 4 ? (i128)INT32_MIN : (i128)INT64_MIN;
  };
  if (n_exprs < 1 || n_exprs > 16) { g_err = "project: 1..16 expressions"; return RW_ERR_UNSUPPORTED; }
  // validate every program first (also for an empty chunk); op_type[e][k]: result type of an operation, op_date[e][k]:
  // its first operand is a DATE
  std::vector<std::vector<int>> op_type(n_exprs), op_date(n_exprs);
  for (int e = 0; e < n_exprs; e++) {
    const rw_project_expr& x = exprs[e];
    if (!int_type(x.ret_type)) { g_err = "project: integer-typed expressions only"; return RW_ERR_UNSUPPORTED; }
    if (!x.ops || x.n_ops < 1) { g_err = "project: malformed expression"; return RW_ERR_INVALID; }
    std::vector<int> types;
    for (int k = 0; k < x.n_ops; k++) {
      const rw_expr_op& op = x.ops[k];
      int t = 0, date = 0;
      if (op.op == RW_EX_COL) {
        if (op.arg < 0 || op.arg >= ch->n_cols || !int_type(ch->columns[op.arg].type)) { g_err = "project: operand column"; return RW_ERR_UNSUPPORTED; }
        types.push_back(ch->columns[op.arg].type);
      } else if (op.op == RW_EX_CONST) {
        types.push_back(RW_T_INT64);
      } else if (op.op == RW_EX_NEG || (op.op >= RW_EX_ADD && op.op <= RW_EX_TUMBLE_END)) {
        t = op.arg == 0 ? RW_T_INT64 : op.arg;
        if (t < RW_T_BOOL || t > RW_T_BYTEA) { g_err = "project: unknown result type of an operation"; return RW_ERR_INVALID; }
        if (!int_type(t)) { g_err = "project: integer-typed operations only"; return RW_ERR_UNSUPPORTED; }
        const size_t n_in = op.op == RW_EX_NEG ? 1 : 2;
        if (types.size() < n_in) { g_err = "project: malformed expression"; return RW_ERR_INVALID; }
        date = (op.op == RW_EX_TUMBLE_START || op.op == RW_EX_TUMBLE_END) && types[types.size() - n_in] == RW_T_DATE;
        types.resize(types.size() - n_in);
        types.push_back(t);
      } else {
        g_err = "project: unknown operation";
        return RW_ERR_INVALID;
      }
      op_type[e].push_back(t);
      op_date[e].push_back(date);
    }
    if (types.size() != 1) { g_err = "project: malformed expression"; return RW_ERR_INVALID; }
  }
  for (int e = 0; e < n_exprs; e++) {
    const rw_project_expr& x = exprs[e];
    has_null[e] = 0;
    std::vector<uint64_t> valid((size_t)((n + 63) / 64), 0);
    const int w = type_width(x.ret_type);
    for (int64_t r = 0; r < n; r++) {
      std::vector<i128> st;
      bool ok = true;
      auto window_start = [&](i128 ts, i128 win, i128* out) -> bool {
        if (win == 0) return false;
        i128 rem = ts % win;
        i128 v = ts - (rem < 0 ? rem + win : rem);
        if (v > (i128)INT64_MAX || v < (i128)INT64_MIN) return false;
        *out = v;
        return true;
      };
      for (int k = 0; k < x.n_ops && ok; k++) {
        const rw_expr_op& op = x.ops[k];
        if (op.op == RW_EX_COL) {
          Datum d = read_datum(ch->columns[op.arg], r);
          if (d.null) ok = false; else st.push_back(d.i);
        } else if (op.op == RW_EX_CONST) {
          st.push_back((i128)op.value);
        } else {
          const i128 lo = type_min(op_type[e][k]), hi = -lo - 1;
          i128 v = 0;
          if (op.op == RW_EX_NEG) {
            v = -st.back();
          } else {
            const i128 b = st.back();
            st.pop_back();
            i128 a = st.back();
            switch (op.op) {
              case RW_EX_ADD: v = a + b; break;
              case RW_EX_SUB: v = a - b; break;
              case RW_EX_MUL: v = a * b; break;
              case RW_EX_DIV: if (b == 0) ok = false; else v = a / b; break;
              case RW_EX_MOD: if (b == 0 || (a == lo && b == -1)) ok = false; else v = a % b; break;
              default:  // RW_EX_TUMBLE_START / RW_EX_TUMBLE_END
                if (op_date[e][k]) {  // days -> the microseconds of that midnight, checked at i64
                  a *= (i128)86400000000LL;
                  if (a > (i128)INT64_MAX || a < (i128)INT64_MIN) ok = false;
                }
                ok = ok && window_start(a, b, &v);
                if (op.op == RW_EX_TUMBLE_END) v += b;
                break;
            }
          }
          if (v > hi || v < lo) ok = false;  // checked at the operation's own result type
          st.back() = v;
        }
      }
      int64_t v = ok ? (int64_t)st[0] : 0;
      if (ok && w == 4 && (v < INT32_MIN || v > INT32_MAX)) { ok = false; v = 0; }
      if (ok && w == 2 && (v < INT16_MIN || v > INT16_MAX)) { ok = false; v = 0; }
      switch (w) {
        case 2: ((int16_t*)out_data[e])[r] = (int16_t)v; break;
        case 4: ((int32_t*)out_data[e])[r] = (int32_t)v; break;
        default: ((int64_t*)out_data[e])[r] = v; break;
      }
      if (ok) valid[(size_t)(r >> 6)] |= 1ull << (r & 63); else has_null[e] = 1;
    }
    if (has_null[e] && out_validity[e]) memcpy(out_validity[e], valid.data(), valid.size() * 8);
  }
  return RW_OK;
}
