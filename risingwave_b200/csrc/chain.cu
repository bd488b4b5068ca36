// chain.cu -- stateless operators that sit between the join and the agg of a device-resident plan.
//
// Replaces (reference, Rust):
//   FilterExecutorInner::filter      src/stream/src/executor/filter.rs:58-150
// for conjunctions of integer comparisons.  The chunk's columns are untouched: the kernel writes a new
// ops column and a new packed visibility, one thread per row, 32 rows = one uint32 of the bitmap
// (warp ballot).  Roofline: HBM, W_pred + 1.125 B read and 1.125 B written per row.
#include <algorithm>

#include "common.cuh"

namespace rw {

#define FILTER_MAX_TERMS 8
struct FilterPlanDev {
  int n_terms;
  int upsert;
  rw_filter_term t[FILTER_MAX_TERMS];
};

// three-valued AND of the terms collapsed to "every term is TRUE": a FALSE or NULL term makes the row false
__device__ __forceinline__ bool filter_pred(const FilterPlanDev& p, const DevChunk& ch, int64_t r) {
  bool res = true;
  for (int k = 0; k < p.n_terms && res; k++) {
    const rw_filter_term& t = p.t[k];
    const ColRef& l = ch.cols[t.lhs_col];
    if (col_is_null(l, r)) { res = false; break; }
    const int64_t a = load_i64(l, r);
    int64_t b = t.rhs_const;
    if (t.rhs_col >= 0) {
      const ColRef& rc = ch.cols[t.rhs_col];
      if (col_is_null(rc, r)) { res = false; break; }
      b = load_i64(rc, r);
    }
    switch (t.cmp) {
      case RW_CMP_LT: res = a < b; break;
      case RW_CMP_LE: res = a <= b; break;
      case RW_CMP_GT: res = a > b; break;
      case RW_CMP_GE: res = a >= b; break;
      case RW_CMP_EQ: res = a == b; break;
      default: res = a != b; break;
    }
  }
  return res;
}

__global__ void __launch_bounds__(256) filter_kernel(FilterPlanDev p, DevChunk ch, uint8_t* out_ops, uint32_t* out_vis32,
                                                     unsigned long long* n_visible) {
  const int64_t n32 = (ch.n + 31) >> 5;
  const int lane = lane_id();
  unsigned int cnt = 0;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n32; w += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t r = w * 32 + lane;
    bool vis = false;
    if (r < ch.n) {
      uint8_t op = ch.ops[r];
      if (row_visible(ch, r, op)) {
        const bool res = filter_pred(p, ch, r);
        if (p.upsert) {                                   // filter.rs:82-106
          const bool ins = op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT;
          op = (ins && res) ? RW_OP_INSERT : RW_OP_DELETE;
          vis = true;
        } else if (op == RW_OP_INSERT || op == RW_OP_DELETE) {
          vis = res;                                      // filter.rs:108-111
        } else if (op == RW_OP_UPDATE_DELETE) {           // pairs with the next visible row (filter.rs:112-141)
          int64_t q = r + 1;
          uint8_t oq = 0;
          while (q < ch.n && !row_visible(ch, q, oq = ch.ops[q])) q++;
          if (q < ch.n && oq == RW_OP_UPDATE_INSERT) {
            const bool rq = filter_pred(p, ch, q);
            if (res && !rq) op = RW_OP_DELETE;            // (true, false): Delete | hidden U+
            vis = res;                                    // (false, true): hidden U- | Insert
          } else {
            vis = res;                                    // unpaired U-: not produced by well-formed streams
          }
        } else {                                          // UpdateInsert: pairs with the previous visible row
          int64_t q = r - 1;
          uint8_t oq = 0;
          while (q >= 0 && !row_visible(ch, q, oq = ch.ops[q])) q--;
          if (q >= 0 && oq == RW_OP_UPDATE_DELETE) {
            const bool rq = filter_pred(p, ch, q);
            if (!rq && res) op = RW_OP_INSERT;
            vis = res;
          } else {
            vis = res;
          }
        }
      }
      out_ops[r] = op;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) {
      out_vis32[w] = bal;
      cnt += __popc(bal);
    }
  }
  // the bitmap is handed out as uint64 words: clear the upper half of a last odd word
  if (blockIdx.x == 0 && threadIdx.x == 0 && (n32 & 1)) out_vis32[n32] = 0u;
  if (n_visible && lane == 0 && cnt) atomicAdd(n_visible, (unsigned long long)cnt);
}

static int filter_plan(const rw_chunk* c, const rw_filter_term* terms, int32_t n_terms, int32_t upsert, FilterPlanDev* p) {
  if (n_terms < 1 || n_terms > FILTER_MAX_TERMS) return fail(RW_ERR_UNSUPPORTED, "filter: 1..8 conjuncts");
  p->n_terms = n_terms;
  p->upsert = upsert ? 1 : 0;
  for (int k = 0; k < n_terms; k++) {
    const rw_filter_term& t = terms[k];
    if (t.cmp < RW_CMP_LT || t.cmp > RW_CMP_NE) return fail(RW_ERR_INVALID, "filter: comparison");
    if (t.lhs_col < 0 || t.lhs_col >= c->n_cols || t.rhs_col < -1 || t.rhs_col >= c->n_cols)
      return fail(RW_ERR_INVALID, "filter: column index");
    // a constant right-hand side has the left-hand side's type
    const int lt = c->columns[t.lhs_col].type, rt = t.rhs_col >= 0 ? c->columns[t.rhs_col].type : lt;
    if (!cmp_operands_ok(lt, rt)) return fail(RW_ERR_UNSUPPORTED, "filter: operand types the device does not compare stay on the CPU executor");
    p->t[k] = t;
  }
  return RW_OK;
}

static int filter_launch(const FilterPlanDev& p, const DevChunk& ch, uint8_t* out_ops, uint64_t* out_vis, int64_t* n_visible_dev,
                         cudaStream_t st) {
  if (n_visible_dev) RW_CUDA(cudaMemsetAsync(n_visible_dev, 0, sizeof(int64_t), st));
  if (ch.n == 0) return RW_OK;
  const int64_t blocks = (ch.n + 255) / 256;
  filter_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(blocks, RW_SMS * 8)), 256, 0, st>>>(p, ch, out_ops, (uint32_t*)out_vis,
                                                                                                   (unsigned long long*)n_visible_dev);
  RW_CUDA(cudaGetLastError());
  return RW_OK;
}

// ------------------------------------------------------------------ Project
// apply_project_exprs (src/stream/src/executor/project/project_scalar.rs:91-108): every output column is an expression
// over the input chunk, evaluated NON-STRICTLY (`eval_infallible`): a row whose evaluation fails -- numeric overflow,
// division by zero -- yields NULL, as does a NULL operand.  Ops and visibility pass through.  Offloaded expression
// class: integer arithmetic in postfix form over integer-typed columns and constants (add / subtract / multiply /
// divide / modulus / neg, src/expr/impl/src/scalar/arithmetic_op.rs `general_*` = checked ops) and tumble_start /
// tumble_end over a microsecond interval (src/expr/impl/src/scalar/tumble.rs:91-112).  Every operation is checked at
// its own result type (rw_expr_op.arg), as each checked_* of the reference is an op of that Rust integer type.  One
// thread per row and expression, an 8-deep value stack in registers.  Roofline: HBM, the referenced columns in, one
// column out.
#define PROJ_MAX_EXPRS 16
#define PROJ_MAX_OPS 24
#define PROJ_STACK 8
#define PROJ_US_PER_DAY 86400000000LL
// ops[e][k] as the plan lowers it.  RW_EX_COL / RW_EX_CONST: as passed.  An operator: `value` = MIN of its result type
// (the result must lie in [value, ~value]; a % -1 of value is NULL), `arg` = 1 when its first operand is a DATE (days)
// that tumble_* turns into microseconds first, else 0.
struct ProjectPlanDev {
  int n_exprs;
  int n_ops[PROJ_MAX_EXPRS];
  int ret_width[PROJ_MAX_EXPRS];
  rw_expr_op ops[PROJ_MAX_EXPRS][PROJ_MAX_OPS];
};
struct ProjectOutDev {
  void* data[PROJ_MAX_EXPRS];
  uint8_t* valid[PROJ_MAX_EXPRS];  // 1 byte / row
  unsigned int* has_null;          // per expression
};

// checked_add / checked_sub / checked_mul of i64 (true = overflow)
__device__ __forceinline__ bool add_ovf(long long a, long long b, long long* r) {
  *r = (long long)((unsigned long long)a + (unsigned long long)b);
  return ((a ^ *r) & (b ^ *r)) < 0;
}
__device__ __forceinline__ bool sub_ovf(long long a, long long b, long long* r) {
  *r = (long long)((unsigned long long)a - (unsigned long long)b);
  return ((a ^ b) & (a ^ *r)) < 0;
}
__device__ __forceinline__ bool mul_ovf(long long a, long long b, long long* r) {
  *r = (long long)((unsigned long long)a * (unsigned long long)b);
  const long long hi = __mul64hi(a, b);
  return hi != (*r >> 63);
}

__device__ __forceinline__ bool tumble_window_start(long long ts, long long w, long long* out) {
  if (w == 0) return false;                 // checked_rem: DivisionByZero
  if (ts == INT64_MIN && w == -1) return false;
  const long long r = ts % w;
  long long sub = r < 0 ? r + w : r;        // tumble.rs:101-111
  long long res;
  if (sub_ovf(ts, sub, &res)) return false;
  *out = res;
  return true;
}

__global__ void __launch_bounds__(256) project_kernel(ProjectPlanDev p, DevChunk ch, ProjectOutDev o) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    for (int e = 0; e < p.n_exprs; e++) {
      long long st[PROJ_STACK];
      int sp = 0;
      bool ok = true;  // false: NULL (NULL operand or failed evaluation)
      for (int k = 0; k < p.n_ops[e] && ok; k++) {
        const rw_expr_op op = p.ops[e][k];
        if (op.op == RW_EX_COL) {
          const ColRef& c = ch.cols[op.arg];
          if (col_is_null(c, r)) ok = false;
          else st[sp++] = load_i64(c, r);
        } else if (op.op == RW_EX_CONST) {
          st[sp++] = op.value;
        } else {
          long long v = 0;
          if (op.op == RW_EX_NEG) {
            ok = !sub_ovf(0, st[sp - 1], &v);
          } else {
            const long long b = st[--sp];
            long long a = st[sp - 1];
            switch (op.op) {
              case RW_EX_ADD: ok = !add_ovf(a, b, &v); break;
              case RW_EX_SUB: ok = !sub_ovf(a, b, &v); break;
              case RW_EX_MUL: ok = !mul_ovf(a, b, &v); break;
              case RW_EX_DIV: ok = b != 0 && !(a == INT64_MIN && b == -1); if (ok) v = a / b; break;
              // checked_rem is None for MIN % -1 of the op's type (the quotient overflows), whatever the range check says
              case RW_EX_MOD: ok = b != 0 && !(a == op.value && b == -1); if (ok) v = (b == -1) ? 0 : a % b; break;
              default:  // RW_EX_TUMBLE_START / RW_EX_TUMBLE_END (= window start + window size)
                if (op.arg) ok = !mul_ovf(a, PROJ_US_PER_DAY, &a);  // a DATE is the timestamp of its midnight (tumble.rs:34-37)
                ok = ok && tumble_window_start(a, b, &v) && (op.op == RW_EX_TUMBLE_START || !add_ovf(v, b, &v));
                break;
            }
          }
          if (v < op.value || v > ~op.value) ok = false;  // outside the operation's own result type
          st[sp - 1] = v;
        }
      }
      long long v = ok ? st[0] : 0;
      const int w = p.ret_width[e];
      if (ok && w < 8) {  // the expression's own width: a result outside it is the overflow of the narrower checked op
        const long long lo = w == 4 ? (long long)INT32_MIN : (long long)INT16_MIN, hi = w == 4 ? (long long)INT32_MAX : (long long)INT16_MAX;
        if (v < lo || v > hi) { ok = false; v = 0; }
      }
      switch (w) {
        case 2: ((int16_t*)o.data[e])[r] = (int16_t)v; break;
        case 4: ((int32_t*)o.data[e])[r] = (int32_t)v; break;
        default: ((long long*)o.data[e])[r] = v; break;
      }
      o.valid[e][r] = ok ? 1 : 0;
      if (!ok) o.has_null[e] = 1u;
    }
  }
}

static bool proj_int_type(int t) {
  switch (t) {
    case RW_T_INT16: case RW_T_INT32: case RW_T_INT64: case RW_T_DATE: case RW_T_TIME: case RW_T_TIMESTAMP: case RW_T_TIMESTAMPTZ:
    case RW_T_SERIAL: return true;
    default: return false;
  }
}

static int project_plan(const rw_chunk* c, const rw_project_expr* exprs, int32_t n_exprs, ProjectPlanDev* p) {
  if (n_exprs < 1 || n_exprs > PROJ_MAX_EXPRS) return fail(RW_ERR_UNSUPPORTED, "project: 1..16 expressions");
  p->n_exprs = n_exprs;
  for (int e = 0; e < n_exprs; e++) {
    const rw_project_expr& x = exprs[e];
    if (!x.ops || x.n_ops < 1 || x.n_ops > PROJ_MAX_OPS) return fail(RW_ERR_UNSUPPORTED, "project: 1..24 postfix operations per expression");
    if (!proj_int_type(x.ret_type)) return fail(RW_ERR_UNSUPPORTED, "project: only integer-typed expressions are evaluated on the device");
    p->n_ops[e] = x.n_ops;
    p->ret_width[e] = type_width(x.ret_type);
    int types[PROJ_MAX_OPS];  // RW_T_* of each stack slot: which tumble operand is a DATE is known here, not per row
    int depth = 0;
    for (int k = 0; k < x.n_ops; k++) {
      rw_expr_op op = x.ops[k];
      if (op.op == RW_EX_COL) {
        if (op.arg < 0 || op.arg >= c->n_cols || !proj_int_type(c->columns[op.arg].type))
          return fail(RW_ERR_UNSUPPORTED, "project: operand column must be integer-typed");
        types[depth++] = c->columns[op.arg].type;
      } else if (op.op == RW_EX_CONST) {
        types[depth++] = RW_T_INT64;
      } else if (op.op == RW_EX_NEG || (op.op >= RW_EX_ADD && op.op <= RW_EX_TUMBLE_END)) {
        const int t = op.arg == 0 ? RW_T_INT64 : op.arg;  // 0: INT64, the meaning of programs that predate typed ops
        if (t < RW_T_BOOL || t > RW_T_BYTEA) return fail(RW_ERR_INVALID, "project: unknown result type of an operation");
        if (!proj_int_type(t)) return fail(RW_ERR_UNSUPPORTED, "project: only integer-typed operations are evaluated on the device");
        const int n_in = op.op == RW_EX_NEG ? 1 : 2;
        if (depth < n_in) return fail(RW_ERR_INVALID, "project: malformed postfix expression");
        depth -= n_in;
        const int w = type_width(t);
        op.value = w == 2 ? (int64_t)INT16_MIN : w == 4 ? (int64_t)INT32_MIN : INT64_MIN;
        op.arg = (op.op == RW_EX_TUMBLE_START || op.op == RW_EX_TUMBLE_END) && types[depth] == RW_T_DATE;
        types[depth++] = t;
      } else {
        return fail(RW_ERR_INVALID, "project: unknown operation");
      }
      if (depth > PROJ_STACK) return fail(RW_ERR_UNSUPPORTED, "project: expression too deep");
      p->ops[e][k] = op;
    }
    if (depth != 1) return fail(RW_ERR_INVALID, "project: malformed postfix expression");
  }
  return RW_OK;
}

}  // namespace rw

using namespace rw;

extern "C" {

int32_t rwgpu_project_device(const rw_chunk* c, const rw_project_expr* exprs, int32_t n_exprs, void* const* out_data,
                             uint8_t* const* out_valid_bytes, uint32_t* has_null, void* cuda_stream) {
  if (!c || !exprs || !out_data || !out_valid_bytes || !has_null) return fail(RW_ERR_INVALID, "null");
  ProjectPlanDev p;
  int rc = project_plan(c, exprs, n_exprs, &p);
  if (rc != RW_OK) return rc;
  DevChunk ch;
  rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  RW_CUDA(cudaMemsetAsync(has_null, 0, sizeof(uint32_t) * n_exprs, st));
  if (ch.n == 0) return RW_OK;
  ProjectOutDev o;
  memset(&o, 0, sizeof(o));
  for (int e = 0; e < n_exprs; e++) { o.data[e] = out_data[e]; o.valid[e] = out_valid_bytes[e]; }
  o.has_null = has_null;
  const int64_t blocks = (ch.n + 255) / 256;
  project_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(blocks, RW_SMS * 8)), 256, 0, st>>>(p, ch, o);
  RW_CUDA(cudaGetLastError());
  return RW_OK;
}

int32_t rwgpu_project(const rw_chunk* c, const rw_project_expr* exprs, int32_t n_exprs, void* const* out_data,
                      uint64_t* const* out_validity, uint32_t* has_null) {
  if (!c || !exprs || !out_data || !out_validity || !has_null) return fail(RW_ERR_INVALID, "null");
  int rc = rwgpu_device_check();
  if (rc != RW_OK) return rc;
  ProjectPlanDev p;
  rc = project_plan(c, exprs, n_exprs, &p);
  if (rc != RW_OK) return rc;
  const int64_t n = c->n_rows;
  for (int e = 0; e < n_exprs; e++) has_null[e] = 0;
  if (n == 0) return RW_OK;
  DevBuf in, out;
  DevChunk ch;
  rc = upload_chunk(c, in, &ch, 0);
  if (rc != RW_OK) return rc;
  // device outputs: per expression data | valid bytes | packed validity words; then the has_null flags
  const size_t nw = (size_t)((n + 63) / 64) * 8;
  size_t off = 0;
  auto region = [&](size_t bytes) { size_t o0 = (off + 255) / 256 * 256; off = o0 + bytes; return o0; };
  size_t o_data[PROJ_MAX_EXPRS], o_valid[PROJ_MAX_EXPRS], o_bits[PROJ_MAX_EXPRS];
  for (int e = 0; e < n_exprs; e++) {
    o_data[e] = region((size_t)n * p.ret_width[e]);
    o_valid[e] = region((size_t)n);
    o_bits[e] = region(nw);
  }
  const size_t o_flags = region(sizeof(uint32_t) * PROJ_MAX_EXPRS);
  RW_CUDA(out.reserve(off + 256));
  uint8_t* d = out.as<uint8_t>();
  void* dd[PROJ_MAX_EXPRS];
  uint8_t* dv[PROJ_MAX_EXPRS];
  for (int e = 0; e < n_exprs; e++) { dd[e] = d + o_data[e]; dv[e] = d + o_valid[e]; }
  {
    ProjectOutDev o;
    memset(&o, 0, sizeof(o));
    for (int e = 0; e < n_exprs; e++) { o.data[e] = dd[e]; o.valid[e] = dv[e]; }
    o.has_null = (unsigned int*)(d + o_flags);
    RW_CUDA(cudaMemset(d + o_flags, 0, sizeof(uint32_t) * PROJ_MAX_EXPRS));
    const int64_t blocks = (n + 255) / 256;
    project_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(blocks, RW_SMS * 8)), 256>>>(p, ch, o);
    RW_CUDA(cudaGetLastError());
  }
  RW_CUDA(cudaMemcpy(has_null, d + o_flags, sizeof(uint32_t) * n_exprs, cudaMemcpyDeviceToHost));
  for (int e = 0; e < n_exprs; e++) {
    RW_CUDA(cudaMemcpy(out_data[e], dd[e], (size_t)n * p.ret_width[e], cudaMemcpyDeviceToHost));
    if (has_null[e] && out_validity[e]) {
      pack_bytes_to_bits_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>((n + 63) / 64 / 256 + 1, RW_SMS * 8)), 256>>>(dv[e], (uint64_t*)(d + o_bits[e]), n);
      RW_CUDA(cudaGetLastError());
      RW_CUDA(cudaMemcpy(out_validity[e], d + o_bits[e], nw, cudaMemcpyDeviceToHost));
    }
  }
  return RW_OK;
}

int32_t rwgpu_filter_device(const rw_chunk* c, const rw_filter_term* terms, int32_t n_terms, int32_t upsert, uint8_t* out_ops,
                            uint64_t* out_visibility, int64_t* n_visible_dev, void* cuda_stream) {
  if (!c || !terms || !out_ops || !out_visibility) return fail(RW_ERR_INVALID, "null");
  FilterPlanDev p;
  int rc = filter_plan(c, terms, n_terms, upsert, &p);
  if (rc != RW_OK) return rc;
  // a row reads its neighbours' input ops and visibility while other threads write theirs
  if (out_ops == c->ops || out_visibility == c->visibility) return fail(RW_ERR_INVALID, "filter: outputs alias the input's ops or visibility");
  DevChunk ch;
  rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  return filter_launch(p, ch, out_ops, out_visibility, n_visible_dev, (cudaStream_t)cuda_stream);
}

int32_t rwgpu_filter(const rw_chunk* c, const rw_filter_term* terms, int32_t n_terms, int32_t upsert, uint8_t* out_ops,
                     uint64_t* out_visibility, int64_t* n_visible) {
  if (!c || !terms || !out_ops || !out_visibility) return fail(RW_ERR_INVALID, "null");
  int rc = rwgpu_device_check();
  if (rc != RW_OK) return rc;
  FilterPlanDev p;
  rc = filter_plan(c, terms, n_terms, upsert, &p);
  if (rc != RW_OK) return rc;
  if (n_visible) *n_visible = 0;
  const int64_t n = c->n_rows;
  if (n == 0) return RW_OK;
  DevBuf in, out;
  DevChunk ch;
  rc = upload_chunk(c, in, &ch, 0);
  if (rc != RW_OK) return rc;
  const size_t nw = (size_t)((n + 63) / 64) * 8, o_vis = ((size_t)n + 255) / 256 * 256, o_cnt = o_vis + nw + 8;
  RW_CUDA(out.reserve(o_cnt + 16));
  uint8_t* d = out.as<uint8_t>();
  rc = filter_launch(p, ch, d, (uint64_t*)(d + o_vis), (int64_t*)(d + o_cnt), 0);
  if (rc != RW_OK) return rc;
  RW_CUDA(cudaMemcpy(out_ops, d, (size_t)n, cudaMemcpyDeviceToHost));
  RW_CUDA(cudaMemcpy(out_visibility, d + o_vis, nw, cudaMemcpyDeviceToHost));
  if (n_visible) RW_CUDA(cudaMemcpy(n_visible, d + o_cnt, sizeof(int64_t), cudaMemcpyDeviceToHost));
  return RW_OK;
}

}  // extern "C"
