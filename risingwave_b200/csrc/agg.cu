// agg.cu -- streaming HashAgg on sm_90a: fused group-by hash + atomic partial aggregate, and the
// barrier-time delta (change inference + compaction) kernel.
//
// Replaces (reference, Rust):
//   HashAggExecutor::apply_chunk   src/stream/src/executor/aggregate/hash_agg.rs:332-409
//   AggGroup::apply_chunk          aggregate/agg_group.rs:379-402  (+ generated `update`, expr/macro gen.rs:838-912)
//   HashAggExecutor::flush_data    hash_agg.rs:412-514
//   AggGroup::get_outputs / build_outputs_change / OnlyOutputIfHasInput  agg_group.rs:431-468,545-606,131-166
//
// HBM layout (open-addressed, linear probing, power-of-two capacity `cap`, load <= 1/2):
//   hot  [cap+2][HW] u64 : key word(s) | one state word per agg call     (cfg2: 8+3*8 = 32 B = 1 sector)
//   cold [cap+2][CW] u64 : flags | prev output per call | sum carry (hi) words | prev hi words
//   dirty[(cap+2+31)/32] u32 : one bit per slot touched since the last barrier
// Slots cap / cap+1 are side slots for the NULL key and for the key equal to the EMPTY sentinel
// (single-column-key mode).  Multi-column keys store a tag word (hash bits | null mask | occupied)
// followed by the key words; the tag is claimed with CAS under a lock bit.
#include <algorithm>
#include <atomic>
#include <memory>

#include "common.cuh"

namespace rw {

#define AGG_EMPTY 0x8000000000000000ull
#define AGG_ERR_OVERFLOW 1u
#define AGG_ERR_NEG_COUNT 2u
#define AGG_ERR_RETRACT_APPEND_ONLY 4u
#define AGG_ERR_OUT_CAPACITY 8u
#define AGG_ERR_MM_MISSING 16u   // retracting a value that is not in the call's materialized input
#define AGG_ERR_MM_CAPACITY 32u  // internal: materialized-input log full
#define AGG_ERR_MM_BAD_ROW 64u   // restore: a materialized-input row names no retractable call, or a group without state
#define AGG_ERR_BAD_COUNT 128u   // counted push: the device row count is below 0 or above the chunk's capacity

struct AggStatus {
  unsigned long long out_rows;
  unsigned long long n_groups;
  unsigned int err;
  unsigned int n_dirty;  // entries of the dirty list
  unsigned int blocks_done;  // flush kernel: blocks that have finished (the last one publishes the status)
  unsigned int mm_dead;      // value-log records retracted or left behind by cleaned groups since the last compaction
};

struct AggPlanDev {
  int n_keys;
  int key_col[RW_MAX_KEYS];
  int key_type[RW_MAX_KEYS];
  int n_calls;
  int kind[RW_MAX_CALLS];
  int arg_col[RW_MAX_CALLS];
  int arg_type[RW_MAX_CALLS];
  int ret_type[RW_MAX_CALLS];
  int hi_off[RW_MAX_CALLS];      // cold word of the sum carry (hi) word, -1 if none
  int prevhi_off[RW_MAX_CALLS];  // cold word of prev output hi (decimal ret), -1 if none
  int mm_off[RW_MAX_CALLS];      // retractable min / max: cold word holding the head of the call's value chain, -1 if none
  int KW, HW, CW;
  int single_key;
  int row_count_call;
  int strict;
};

struct AggTable {
  uint64_t* hot;
  uint64_t* cold;
  uint32_t* dirty;       // first-touch filter: one bit per slot
  uint32_t* dirty_list;  // slots touched since the last barrier (each exactly once)
  AggStatus* status;
  uint64_t cap;  // power of two
  // retractable min / max (AggState::MaterializedInput, agg_state.rs:49-56 / minput.rs): every non-NULL input value of
  // such a call is a 16-byte record {u32 link | DEAD, u32 -, i64 value (sortable form)} chained from the group's cold row
  ulonglong2* mm_log;
  unsigned long long* mm_next;  // next free record id (ids start at 1: 0 = end of chain)
  uint64_t mm_cap;
};
#define MM_DEAD 0x80000000u
#define COLD_RECOMPUTE_SHIFT 48  // cold word 0, bit 48 + c: call c's extreme was retracted -> recompute at the barrier

// mark `slot` dirty; the thread that flips the bit appends the slot to the dirty list
// (opportunistic warp aggregation: one atomicAdd per group of converged first-touchers)
__device__ __forceinline__ void mark_dirty(const AggTable& t, uint64_t slot) {
  const uint32_t bit = 1u << (slot & 31);
  uint32_t* dw = t.dirty + (slot >> 5);
  if (__ldcg(dw) & bit) return;
  const uint32_t old = atomicOr(dw, bit);
  if (old & bit) return;
  const unsigned m = __activemask();
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(m) - 1;
  unsigned int base = 0;
  if (lane == leader) base = atomicAdd(&t.status->n_dirty, (unsigned int)__popc(m));
  base = __shfl_sync(m, base, leader);
  t.dirty_list[base + __popc(m & ((1u << lane) - 1))] = (uint32_t)slot;
}

// a chunk whose row count lives on the device (chunk_rows): thread 0 of the apply kernel flags a count out of range,
// which the next barrier reports (chunk_rows makes it no rows: the push applies nothing)
__device__ __forceinline__ void agg_check_count(const AggTable& t, const DevChunk& ch) {
  if (ch.n_dev && blockIdx.x == 0 && threadIdx.x == 0) {
    const int64_t n = *ch.n_dev;
    if (n < 0 || n > ch.n) atomicOr(&t.status->err, AGG_ERR_BAD_COUNT);
  }
}

struct AggOutDev {
  uint8_t* ops;
  void* col[RW_MAX_KEYS + RW_MAX_CALLS];
  uint8_t* valid[RW_MAX_KEYS + RW_MAX_CALLS];  // 1 byte / row
  unsigned int* has_null;                       // per column flag
  int64_t capacity;
};

// cold word 0: bits 0..15 state-non-NULL flag per call, bits 16..31 prev-output NULL mask, bit 32 has_prev
#define COLD_HAS_PREV (1ull << 32)

__device__ __forceinline__ uint64_t state_init(int kind, int arg_type) {
  if (kind == RW_AGG_MIN) return (uint64_t)INT64_MAX;
  if (kind == RW_AGG_MAX) return (uint64_t)INT64_MIN;
  return 0ull;  // count / sum / sum0 (double 0.0 has bit pattern 0 too)
}

// ------------------------------------------------------------------ table init
__global__ void agg_init_kernel(AggTable t, AggPlanDev p, uint64_t from_slot) {
  uint64_t total = t.cap + 2;
  for (uint64_t s = from_slot + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < total;
       s += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t* h = t.hot + s * p.HW;
    h[0] = p.single_key ? AGG_EMPTY : 0ull;
    for (int k = 1; k < p.KW; k++) h[k] = 0;
    for (int c = 0; c < p.n_calls; c++) h[p.KW + c] = state_init(p.kind[c], p.arg_type[c]);
    uint64_t* cw = t.cold + s * p.CW;
    for (int k = 0; k < p.CW; k++) cw[k] = 0;
  }
}

// ------------------------------------------------------------------ slot lookup
__device__ __forceinline__ uint64_t find_or_insert_single(const AggTable& t, int HW, uint64_t key, bool* created) {
  uint64_t mask = t.cap - 1;
  uint64_t idx = mix64(key) & mask;
  while (true) {
    unsigned long long* p = (unsigned long long*)(t.hot + idx * HW);
    unsigned long long cur = *p;
    if (cur == key) return idx;
    if (cur == AGG_EMPTY) {
      unsigned long long old = atomicCAS(p, (unsigned long long)AGG_EMPTY, (unsigned long long)key);
      if (old == AGG_EMPTY) { *created = true; return idx; }
      if (old == key) return idx;
    }
    idx = (idx + 1) & mask;
  }
}

__device__ __forceinline__ uint64_t multi_hash(const AggPlanDev& p, const uint64_t* kw, uint32_t nullmask) {
  uint64_t h = 0x9e3779b97f4a7c15ull ^ nullmask;
  for (int k = 0; k < p.n_keys; k++) h = mix64(h ^ kw[k]) + 0x9e3779b97f4a7c15ull;
  return h;
}

__device__ __forceinline__ uint64_t find_or_insert_multi(const AggTable& t, const AggPlanDev& p, const uint64_t* kw,
                                                          uint32_t nullmask, bool* created) {
  const uint64_t h = multi_hash(p, kw, nullmask);
  uint64_t tag = (h & ~0xFFFFull) | ((uint64_t)nullmask << 8) | 1ull;
  uint64_t mask = t.cap - 1;
  uint64_t idx = (h >> 17) & mask;
  while (true) {
    unsigned long long* ptr = (unsigned long long*)(t.hot + idx * p.HW);
    unsigned long long cur = *(volatile unsigned long long*)ptr;
    if (cur == 0ull) {
      unsigned long long old = atomicCAS(ptr, 0ull, (unsigned long long)(tag | 2ull));
      if (old == 0ull) {
        for (int k = 0; k < p.n_keys; k++) __stcg((unsigned long long*)ptr + 1 + k, (unsigned long long)kw[k]);
        __threadfence();
        atomicExch(ptr, (unsigned long long)tag);
        *created = true;
        return idx;
      }
      cur = old;
    }
    if ((cur & ~2ull) == tag) {
      while (cur & 2ull) cur = *(volatile unsigned long long*)ptr;  // writer publishes within a few cycles
      bool eq = true;
      for (int k = 0; k < p.n_keys; k++) eq = eq && (__ldcg((const unsigned long long*)ptr + 1 + k) == kw[k]);
      if (eq) return idx;
    }
    idx = (idx + 1) & mask;
  }
}

// ------------------------------------------------------------------ apply one row to the group's states
__device__ __forceinline__ void agg_apply_row(const AggTable& t, const AggPlanDev& p, const DevChunk& ch, int64_t r,
                                               uint8_t op, uint64_t slot, int per_row_flags) {
  uint64_t* hot = t.hot + slot * p.HW + p.KW;
  uint64_t* cold = t.cold + slot * p.CW;
  const bool retract = (op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE);
  uint32_t setflags = 0;
#pragma unroll 1
  for (int c = 0; c < p.n_calls; c++) {
    const int kind = p.kind[c];
    const int ac = p.arg_col[c];
    if (ac >= 0 && col_is_null(ch.cols[ac], r)) continue;  // (state, None) => state   gen.rs:894-896
    unsigned long long* sp = (unsigned long long*)(hot + c);
    if (kind == RW_AGG_COUNT) {
      atomicAdd(sp, retract ? ~0ull : 1ull);
      continue;
    }
    setflags |= 1u << c;
    const int at = p.arg_type[c];
    const bool isf = (at == RW_T_FLOAT32 || at == RW_T_FLOAT64);
    if (kind == RW_AGG_SUM || kind == RW_AGG_SUM0) {
      if (at == RW_T_FLOAT32) {
        // sum(float4) -> float4: an f32 state rounded after every add (general.rs:28-41 over F32), in the low half of
        // the state word.  A CAS loop rather than atomicAdd(float*): atom.add.f32 flushes subnormals to zero.
        const float x = ((const float*)ch.cols[ac].data)[r];
        unsigned int* wp = (unsigned int*)sp;
        unsigned int old = __ldcg(wp), seen;
        do {
          seen = old;
          const float s = __uint_as_float(seen);
          old = atomicCAS(wp, seen, __float_as_uint(retract ? __fsub_rn(s, x) : __fadd_rn(s, x)));
        } while (old != seen);
      } else if (isf) {
        double x = load_f64(ch.cols[ac], r);
        atomicAdd((double*)sp, retract ? -x : x);
      } else {
        // exact 128-bit accumulation for every integer width: lo word here, carries into the cold hi word; the state
        // is range-checked against its return type at the barrier (call_output)
        int64_t x = load_i64(ch.cols[ac], r);
        unsigned long long add = retract ? (0ull - (unsigned long long)x) : (unsigned long long)x;
        bool neg = retract ? (x > 0) : (x < 0);
        unsigned long long old = atomicAdd(sp, add);
        unsigned long long nw = old + add;
        long long hd = (neg ? -1ll : 0ll) + ((nw < old) ? 1ll : 0ll);
        if (hd != 0) atomicAdd((unsigned long long*)(cold + p.hi_off[c]), (unsigned long long)hd);
      }
    } else if (p.mm_off[c] >= 0) {  // retractable MIN / MAX: materialized input (minput.rs:172-182)
      if (retract) { setflags &= ~(1u << c); continue; }  // retractions are applied by agg_mm_delete_kernel after this kernel
      long long v = isf ? (long long)f64_sortable(load_f64(ch.cols[ac], r)) : (long long)load_i64(ch.cols[ac], r);
      // one record per value: id from the shared counter (aggregated over the converged lanes), pushed on the chain
      const unsigned m = __activemask();
      const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(t.mm_next, (unsigned long long)__popc(m));
      base = __shfl_sync(m, base, leader);
      const unsigned long long id = base + __popc(m & ((1u << lane) - 1));
      if (id >= t.mm_cap) { atomicOr(&t.status->err, AGG_ERR_MM_CAPACITY); continue; }
      const uint32_t old = atomicExch((uint32_t*)(cold + p.mm_off[c]), (uint32_t)id);
      t.mm_log[id] = make_ulonglong2((unsigned long long)old, (unsigned long long)v);
      if (kind == RW_AGG_MIN) atomicMin((long long*)sp, v); else atomicMax((long long*)sp, v);
    } else {  // MIN / MAX (append-only value state, general.rs:91-125)
      if (op != RW_OP_INSERT) { atomicOr(&t.status->err, AGG_ERR_RETRACT_APPEND_ONLY); continue; }
      long long v = isf ? (long long)f64_sortable(load_f64(ch.cols[ac], r)) : (long long)load_i64(ch.cols[ac], r);
      if (kind == RW_AGG_MIN) atomicMin((long long*)sp, v); else atomicMax((long long*)sp, v);
    }
  }
  if (per_row_flags && setflags) {
    unsigned long long f = __ldcg((const unsigned long long*)cold);
    if ((f & setflags) != setflags) atomicOr((unsigned long long*)cold, (unsigned long long)setflags);
  }
}

// ------------------------------------------------------------------ generic apply kernel (one thread per row)
__global__ void __launch_bounds__(256) agg_apply_kernel(AggTable t, AggPlanDev p, DevChunk ch, int per_row_flags) {
  unsigned int created_local = 0;
  agg_check_count(t, ch);
  // (the count is re-read per row round, an L1 hit: a loop-wide copy costs the kernel register spills)
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < chunk_rows(ch); r += (int64_t)gridDim.x * blockDim.x) {
    uint8_t op = ch.ops[r];
    if (!row_visible(ch, r, op)) continue;
    uint64_t slot;
    bool created = false;
    if (p.single_key) {
      const ColRef& kc = ch.cols[p.key_col[0]];
      if (col_is_null(kc, r)) slot = t.cap;  // NULL is a legal group value (key_v2.rs:216-220)
      else {
        uint64_t key = load_key_word(kc, r);
        if (key == AGG_EMPTY) slot = t.cap + 1;
        else slot = find_or_insert_single(t, p.HW, key, &created);
      }
    } else {
      uint64_t kw[RW_MAX_KEYS];
      uint32_t nm = 0;
      for (int k = 0; k < p.n_keys; k++) {
        const ColRef& kc = ch.cols[p.key_col[k]];
        if (col_is_null(kc, r)) { nm |= 1u << k; kw[k] = 0; }
        else kw[k] = load_key_word(kc, r);
      }
      slot = find_or_insert_multi(t, p, kw, nm, &created);
    }
    if (created) created_local++;
    mark_dirty(t, slot);
    agg_apply_row(t, p, ch, r, op, slot, per_row_flags);
  }
  // warp-aggregated group counter
  for (int o = 16; o > 0; o >>= 1) created_local += __shfl_xor_sync(0xffffffffu, created_local, o);
  if (lane_id() == 0 && created_local) atomicAdd(&t.status->n_groups, (unsigned long long)created_local);
}

// ------------------------------------------------------------------ retractable min / max: the retractions of a chunk
// Runs after the apply kernel (every insert of the chunk is in its chain by then).  A retracted value kills ONE live
// record with that value (the materialized input is a multiset); if it was the group's current extreme the call is
// flagged and the barrier recomputes the extreme from the live records.
__global__ void __launch_bounds__(256) agg_mm_delete_kernel(AggTable t, AggPlanDev p, DevChunk ch) {
  unsigned int kills = 0;  // records this thread retracted: dead for the value-log compaction (agg_mm_compact_kernel)
  // (a count out of range was flagged by the apply kernel; the count is re-read per row round, as there)
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < chunk_rows(ch); r += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t op = ch.ops[r];
    if (!row_visible(ch, r, op) || !(op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE)) continue;
    uint64_t slot;
    bool created = false;
    if (p.single_key) {
      const ColRef& kc = ch.cols[p.key_col[0]];
      if (col_is_null(kc, r)) slot = t.cap;
      else {
        const uint64_t key = load_key_word(kc, r);
        slot = key == AGG_EMPTY ? t.cap + 1 : find_or_insert_single(t, p.HW, key, &created);
      }
    } else {
      uint64_t kw[RW_MAX_KEYS];
      uint32_t nm = 0;
      for (int k = 0; k < p.n_keys; k++) {
        const ColRef& kc = ch.cols[p.key_col[k]];
        if (col_is_null(kc, r)) { nm |= 1u << k; kw[k] = 0; }
        else kw[k] = load_key_word(kc, r);
      }
      slot = find_or_insert_multi(t, p, kw, nm, &created);
    }
    uint64_t* cold = t.cold + slot * p.CW;
    for (int c = 0; c < p.n_calls; c++) {
      if (p.mm_off[c] < 0) continue;
      const int ac = p.arg_col[c];
      if (col_is_null(ch.cols[ac], r)) continue;  // NULL arguments never entered the input (aggregate/mod.rs:81-109)
      const int at = p.arg_type[c];
      const long long v = (at == RW_T_FLOAT32 || at == RW_T_FLOAT64) ? (long long)f64_sortable(load_f64(ch.cols[ac], r))
                                                                     : (long long)load_i64(ch.cols[ac], r);
      bool found = false;
      uint32_t id = __ldcg((const uint32_t*)(cold + p.mm_off[c]));
      while (id != 0u && !found) {
        const ulonglong2 rec = __ldcg(t.mm_log + id);
        const uint32_t lk = (uint32_t)rec.x;
        if (!(lk & MM_DEAD) && (long long)rec.y == v) {
          const uint32_t old = atomicOr((uint32_t*)(t.mm_log + id), MM_DEAD);
          if (!(old & MM_DEAD)) found = true;  // (else another retraction of the same value took this record: go on)
        }
        id = lk & ~MM_DEAD;
      }
      if (!found) {
        if (p.strict) atomicOr(&t.status->err, AGG_ERR_MM_MISSING);
        continue;
      }
      kills++;
      if ((long long)__ldcg(t.hot + slot * p.HW + p.KW + c) == v) atomicOr((unsigned long long*)cold, 1ull << (COLD_RECOMPUTE_SHIFT + c));
    }
  }
  for (int o = 16; o > 0; o >>= 1) kills += __shfl_xor_sync(0xffffffffu, kills, o);
  if (lane_id() == 0 && kills) atomicAdd(&t.status->mm_dead, kills);
}

// ------------------------------------------------------------------ fast path: 1 x 8-byte key, no NULLs anywhere,
// calls = {count(*), sum(int8)->int8, max/min(int8)} in any order (BASELINE cfg2 / Nexmark q4 shape).
// Two rows per thread with 128-bit loads of the key / argument columns.
// One atomic per BLOCK and loop round reserves the dirty-list entries of the block's first-touched groups, one per
// block at the end counts the new groups: an atomicAdd per warp on those two shared counters (the first version)
// serialised in one L2 slice -- thousands of same-address atomics per 2^18-row epoch made up the kernel's
// whole duration.
template <int NCALLS>
__global__ void __launch_bounds__(256) agg_apply_fast_kernel(AggTable t, AggPlanDev p, DevChunk ch) {
  __shared__ unsigned int s_warp[8];
  __shared__ unsigned int s_base;
  unsigned int created_local = 0;
  const int lane = lane_id(), wid = threadIdx.x >> 5;
  agg_check_count(t, ch);
  const int64_t n = chunk_rows(ch);  // grid sized from the capacity: pairs past the count are idle
  const int64_t npair = (n + 1) >> 1;
  const longlong2* keyv = (const longlong2*)ch.cols[p.key_col[0]].data;
  const unsigned short* opv = (const unsigned short*)ch.ops;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x; base < npair; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = base + threadIdx.x;
    uint64_t slot[2] = {0, 0};
    bool first[2] = {false, false};
    if (i < npair) {
      const int64_t r0 = i * 2;
      const bool two = (r0 + 1 < n);
      long long k[2];
      uint8_t op[2];
      long long a[NCALLS][2];
      if (two) {
        longlong2 kv = __ldg(keyv + i);
        k[0] = kv.x; k[1] = kv.y;
        unsigned short o2 = __ldg(opv + i);
        op[0] = (uint8_t)(o2 & 0xff); op[1] = (uint8_t)(o2 >> 8);
#pragma unroll
        for (int c = 0; c < NCALLS; c++) {
          if (p.arg_col[c] >= 0) {
            longlong2 av = __ldg((const longlong2*)ch.cols[p.arg_col[c]].data + i);
            a[c][0] = av.x; a[c][1] = av.y;
          }
        }
      } else {
        k[0] = ((const long long*)ch.cols[p.key_col[0]].data)[r0]; k[1] = 0;
        op[0] = ch.ops[r0]; op[1] = 0;
#pragma unroll
        for (int c = 0; c < NCALLS; c++)
          if (p.arg_col[c] >= 0) { a[c][0] = ((const long long*)ch.cols[p.arg_col[c]].data)[r0]; a[c][1] = 0; }
      }
#pragma unroll
      for (int j = 0; j < 2; j++) {
        if (op[j] == 0) continue;
        bool created = false;
        const uint64_t sl = ((uint64_t)k[j] == AGG_EMPTY) ? t.cap + 1 : find_or_insert_single(t, p.HW, (uint64_t)k[j], &created);
        if (created) created_local++;
        slot[j] = sl;
        {  // first touch of the group in this epoch ?
          const uint32_t bit = 1u << (sl & 31);
          uint32_t* dw = t.dirty + (sl >> 5);
          if (!(__ldcg(dw) & bit)) first[j] = !(atomicOr(dw, bit) & bit);
        }
        unsigned long long* sp = (unsigned long long*)(t.hot + sl * p.HW + 1);
        const bool retract = (op[j] == RW_OP_DELETE || op[j] == RW_OP_UPDATE_DELETE);
#pragma unroll
        for (int c = 0; c < NCALLS; c++) {
          const int kind = p.kind[c];
          if (kind == RW_AGG_COUNT) {
            atomicAdd(sp + c, retract ? ~0ull : 1ull);
          } else if (kind == RW_AGG_SUM || kind == RW_AGG_SUM0) {
            long long x = a[c][j];
            unsigned long long add = retract ? (0ull - (unsigned long long)x) : (unsigned long long)x;
            bool neg = retract ? (x > 0) : (x < 0);
            unsigned long long old = atomicAdd(sp + c, add);
            unsigned long long nw = old + add;
            long long hd = (neg ? -1ll : 0ll) + ((nw < old) ? 1ll : 0ll);
            if (hd != 0) atomicAdd((unsigned long long*)(t.cold + sl * p.CW + p.hi_off[c]), (unsigned long long)hd);
          } else {
            if (op[j] != RW_OP_INSERT) { atomicOr(&t.status->err, AGG_ERR_RETRACT_APPEND_ONLY); continue; }
            if (kind == RW_AGG_MIN) atomicMin((long long*)(sp + c), a[c][j]); else atomicMax((long long*)(sp + c), a[c][j]);
          }
        }
      }
    }
    // dirty-list entries of the block's first touches: warp scan -> block scan -> ONE atomicAdd
    const unsigned int mine = (first[0] ? 1u : 0u) + (first[1] ? 1u : 0u);
    unsigned int incl = mine;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int run = 0;
      for (int w = 0; w < 8; w++) { const unsigned int v = s_warp[w]; s_warp[w] = run; run += v; }
      s_base = run ? atomicAdd(&t.status->n_dirty, run) : 0u;
    }
    __syncthreads();
    unsigned int at = s_base + s_warp[wid] + incl - mine;
    if (first[0]) t.dirty_list[at++] = (uint32_t)slot[0];
    if (first[1]) t.dirty_list[at] = (uint32_t)slot[1];
    __syncthreads();  // s_warp / s_base are rewritten by the next round
  }
  for (int o = 16; o > 0; o >>= 1) created_local += __shfl_xor_sync(0xffffffffu, created_local, o);
  if (lane == 0) s_warp[wid] = created_local;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int tot = 0;
    for (int w = 0; w < 8; w++) tot += s_warp[w];
    if (tot) atomicAdd(&t.status->n_groups, (unsigned long long)tot);
  }
}

// ------------------------------------------------------------------ mark "state non-NULL" for all dirty groups
// (used when every push of the epoch had NULL-free argument columns: then every visible row
// contributed a non-NULL value to every call, so the per-row flag update can be elided)
__global__ void agg_set_flags_kernel(AggTable t, AggPlanDev p, uint32_t mask) {
  const unsigned int n = t.status->n_dirty;
  for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    t.cold[(uint64_t)t.dirty_list[i] * p.CW] |= (uint64_t)mask;
}

// ------------------------------------------------------------------ flush: change inference + compaction
struct OutVal {
  uint64_t lo, hi;
  bool null;
};

// current output of call c from its state (value-state get_output; agg_group.rs:431-468)
__device__ __forceinline__ OutVal call_output(const AggTable& t, const AggPlanDev& p, int c, const uint64_t* hot,
                                               const uint64_t* cold, uint64_t flags) {
  const int kind = p.kind[c];
  const int at = p.arg_type[c];
  const bool isf = (at == RW_T_FLOAT32 || at == RW_T_FLOAT64);
  const uint64_t s = hot[p.KW + c];
  OutVal v;
  v.hi = 0;
  v.lo = 0;
  v.null = false;
  if (kind == RW_AGG_COUNT) {
    v.lo = s;
  } else if (!((flags >> c) & 1)) {
    v.null = (kind != RW_AGG_SUM0);  // sum0: init_state = 0; others NULL until a non-NULL input
  } else if (kind == RW_AGG_SUM || kind == RW_AGG_SUM0) {
    if (at == RW_T_FLOAT32) {  // sum(float4) -> float4: the f32 state, widened exactly (store_word narrows it back)
      v.lo = (uint64_t)__double_as_longlong((double)__uint_as_float((unsigned int)s));
    } else if (isf) {
      v.lo = s;
    } else {
      const long long hi = (long long)cold[p.hi_off[c]];  // every integer sum has a carry word
      v.lo = s;
      v.hi = (uint64_t)hi;
      if (p.ret_type[c] == RW_T_DECIMAL) {  // rust_decimal: 96-bit mantissa
        const bool ok = (hi >= 0) ? (hi < (1ll << 32)) : (hi > -(1ll << 32) || (hi == -(1ll << 32) && s != 0));
        if (!ok) atomicOr(&t.status->err, AGG_ERR_OVERFLOW);
      } else if (hi != (((long long)s) >> 63)) {
        atomicOr(&t.status->err, AGG_ERR_OVERFLOW);
      }
    }
  } else {  // min / max
    v.lo = isf ? (uint64_t)__double_as_longlong(f64_unsortable((int64_t)s)) : s;
  }
  return v;
}

__device__ __forceinline__ void write_out_val(const AggOutDev& o, const AggPlanDev& p, int c, int64_t rr, const OutVal& v) {
  const int oc = p.n_keys + c;
  o.valid[oc][rr] = v.null ? 0 : 1;
  if (v.null) o.has_null[oc] = 1;
  if (p.ret_type[c] == RW_T_DECIMAL) {
    ((uint64_t*)o.col[oc])[rr * 2] = v.lo;
    ((uint64_t*)o.col[oc])[rr * 2 + 1] = v.hi;
  } else {
    store_word(o.col[oc], type_width_dev(p.ret_type[c]), p.ret_type[c], rr, v.lo);
  }
}

// where the last block of the flush kernel publishes the barrier's status (pinned host memory, UVA)
struct AggPublish {
  AggStatus* st_host;
  unsigned int* has_null_host;
  unsigned long long* tag_host;
  unsigned long long tag;
};

__device__ __forceinline__ void agg_publish(AggStatus* st, unsigned int* has_null, const AggPublish& pub, int t) {
  if (t < RW_MAX_KEYS + RW_MAX_CALLS) { pub.has_null_host[t] = __ldcg(has_null + t); has_null[t] = 0; }
  if (t == 0) {
    AggStatus s;
    s.out_rows = __ldcg(&st->out_rows);
    s.n_groups = __ldcg(&st->n_groups);
    s.err = __ldcg(&st->err);
    s.n_dirty = __ldcg(&st->n_dirty);
    s.blocks_done = 0;
    s.mm_dead = 0;
    *pub.st_host = s;
    st->out_rows = 0;
    st->n_dirty = 0;
    st->blocks_done = 0;
  }
  __threadfence_system();
  __syncthreads();
  if (t == 0) {
    *(volatile unsigned long long*)pub.tag_host = pub.tag;  // written last: the host polls it
    __threadfence_system();
  }
}

// one thread per dirty group (the dirty LIST keeps every lane busy however sparse the epoch's touched set is);
// the 0 / 1 / 2 output rows of a BLOCK are compacted with a warp-shuffle scan + one shared-memory pass and ONE
// atomicAdd (an atomic per warp on the shared row counter serialised in one L2 slice), so a U-/U+ pair stays
// adjacent.  The last block to finish publishes the status block to pinned host memory and re-arms the
// per-barrier counters: a barrier is one launch.
//
// The group's hot and cold rows are STAGED IN SHARED MEMORY: every word is fetched once by independent loads issued
// back to back, the generic per-call logic below then runs on the staged copy, and the rows go back with one pass
// of stores.  (Working on the global rows serialised ~20 dependent L2 round trips per thread -- the stores between the
// loads keep the compiler from batching them, leaving both SM and DRAM mostly idle.)
__global__ void __launch_bounds__(256) agg_flush_kernel(AggTable t, AggPlanDev p, AggOutDev o, uint32_t epoch_flag_mask, AggPublish pub) {
  extern __shared__ uint64_t s_rows[];
  const int s_stride = (p.HW + p.CW) | 1;  // odd: conflict-free for 8-byte words
  uint64_t* const hot = s_rows + (size_t)threadIdx.x * s_stride;
  uint64_t* const cold = hot + p.HW;
  __shared__ int s_warp[8];
  __shared__ unsigned long long s_base;
  __shared__ bool s_last;
  const unsigned int n_dirty = __ldcg(&t.status->n_dirty);
  const int lane = lane_id(), wid = threadIdx.x >> 5;
  for (unsigned int base0 = blockIdx.x * blockDim.x; base0 < n_dirty; base0 += gridDim.x * blockDim.x) {
    const unsigned int i = base0 + threadIdx.x;
    const bool active = i < n_dirty;
    int nrows = 0;
    uint8_t op0 = 0, op1 = 0;
    uint64_t slot = 0;
    uint64_t flags = 0;
    bool store_prev = false, hot_changed = false;
    if (active) {
      slot = t.dirty_list[i];
      {
        const uint64_t* gh = t.hot + slot * p.HW;
        const uint64_t* gc = t.cold + slot * p.CW;
#pragma unroll 4
        for (int k = 0; k < p.HW; k++) hot[k] = __ldcg(gh + k);
#pragma unroll 4
        for (int k = 0; k < p.CW; k++) cold[k] = __ldcg(gc + k);
      }
      flags = cold[0] | (uint64_t)epoch_flag_mask;
      // retractable min / max whose extreme was retracted: the first row of the materialized input in order
      // (MaterializedInputState::get_output, minput.rs:184-245) = the extreme of the live records
      if (flags >> COLD_RECOMPUTE_SHIFT) {
        for (int c = 0; c < p.n_calls; c++) {
          if (p.mm_off[c] < 0 || !((flags >> (COLD_RECOMPUTE_SHIFT + c)) & 1ull)) continue;
          const bool is_min = p.kind[c] == RW_AGG_MIN;
          long long best = is_min ? INT64_MAX : INT64_MIN;
          bool any = false;
          for (uint32_t id = (uint32_t)cold[p.mm_off[c]]; id != 0u;) {
            const ulonglong2 rec = t.mm_log[id];
            const uint32_t lk = (uint32_t)rec.x;
            if (!(lk & MM_DEAD)) {
              const long long v = (long long)rec.y;
              best = is_min ? (v < best ? v : best) : (v > best ? v : best);
              any = true;
            }
            id = lk & ~MM_DEAD;
          }
          hot[p.KW + c] = (uint64_t)best;
          hot_changed = true;
          if (!any) flags &= ~(1ull << c);  // empty input: the output is NULL
        }
        flags &= (1ull << COLD_RECOMPUTE_SHIFT) - 1;
      }
      // row_count_of (agg_group.rs:55-79)
      long long rc = (long long)hot[p.KW + p.row_count_call];
      if (rc < 0) {
        if (p.strict) atomicOr(&t.status->err, AGG_ERR_NEG_COUNT);
        rc = 0;
      }
      if (rc == 0) {  // reset value states (agg_group.rs:438-446)
        hot_changed = true;
        for (int c = 0; c < p.n_calls; c++) {
          hot[p.KW + c] = state_init(p.kind[c], p.arg_type[c]);
          if (p.hi_off[c] >= 0) cold[p.hi_off[c]] = 0;
          if (p.mm_off[c] >= 0) cold[p.mm_off[c]] = 0;  // (a group without rows has no live value: drop the dead chain)
        }
        flags &= ~0xFFFFull;
      }
      const bool has_prev = (flags & COLD_HAS_PREV) != 0;
      const uint32_t prev_nm = (uint32_t)((flags >> 16) & 0xFFFF);
      long long prev_rc = 0;
      bool same = true;
      if (has_prev) {
        prev_rc = (long long)cold[1 + p.row_count_call];
        if (prev_rc < 0) prev_rc = 0;
        for (int c = 0; c < p.n_calls; c++) {
          const OutVal v = call_output(t, p, c, hot, cold, flags);
          const bool pnull = (prev_nm >> c) & 1;
          const uint64_t plo = cold[1 + c];
          bool eq = (pnull == v.null) && (v.null || (plo == v.lo && (p.prevhi_off[c] < 0 || cold[p.prevhi_off[c]] == v.hi)));
          if (!eq && !v.null && !pnull && (p.ret_type[c] == RW_T_FLOAT32 || p.ret_type[c] == RW_T_FLOAT64)) {
            // OrderedFloat equality: NaN == NaN, -0 == +0
            const double a = __longlong_as_double((long long)plo), b = __longlong_as_double((long long)v.lo);
            eq = (a != a && b != b) || (a == b);
          }
          same = same && eq;
        }
      } else {
        for (int c = 0; c < p.n_calls; c++) (void)call_output(t, p, c, hot, cold, flags);  // overflow checks
      }
      // OnlyOutputIfHasInput::infer_change_type (agg_group.rs:131-166)
      if (prev_rc == 0 && rc == 0) { nrows = 0; }
      else if (prev_rc == 0) { nrows = 1; op0 = RW_OP_INSERT; store_prev = true; }
      else if (rc == 0) { nrows = 1; op0 = RW_OP_DELETE; }
      else if (!same) { nrows = 2; op0 = RW_OP_UPDATE_DELETE; op1 = RW_OP_UPDATE_INSERT; store_prev = true; }
    }
    // block-wide compaction of the emitted rows
    int incl = nrows;
    for (int d = 1; d < 32; d <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      int run = 0;
      for (int w = 0; w < 8; w++) { const int v = s_warp[w]; s_warp[w] = run; run += v; }
      s_base = run ? atomicAdd(&t.status->out_rows, (unsigned long long)run) : 0ull;
    }
    __syncthreads();
    if (active) {
      const int64_t row = (int64_t)s_base + s_warp[wid] + (incl - nrows);
      if (nrows && row + nrows > o.capacity) {
        atomicOr(&t.status->err, AGG_ERR_OUT_CAPACITY);
      } else if (nrows) {
        // group key
        uint64_t keyw[RW_MAX_KEYS];
        uint32_t key_nm = 0;
        if (p.single_key) {
          if (slot == t.cap) { key_nm = 1; keyw[0] = 0; }
          else keyw[0] = (slot == t.cap + 1) ? AGG_EMPTY : hot[0];
        } else {
          key_nm = (uint32_t)((hot[0] >> 8) & 0xff);
          for (int k = 0; k < p.n_keys; k++) keyw[k] = hot[1 + k];
        }
        const uint32_t prev_nm = (uint32_t)((flags >> 16) & 0xFFFF);
        for (int j = 0; j < nrows; j++) {
          const uint8_t op = j == 0 ? op0 : op1;
          const bool use_prev = (op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE);
          const int64_t rr = row + j;
          o.ops[rr] = op;
          for (int k = 0; k < p.n_keys; k++) {
            const bool nul = (key_nm >> k) & 1;
            o.valid[k][rr] = nul ? 0 : 1;
            if (nul) o.has_null[k] = 1;
            store_word(o.col[k], type_width_dev(p.key_type[k]), p.key_type[k], rr, keyw[k]);
          }
          for (int c = 0; c < p.n_calls; c++) {
            OutVal v;
            if (use_prev) {
              v.lo = cold[1 + c];
              v.hi = (p.prevhi_off[c] >= 0) ? cold[p.prevhi_off[c]] : 0;
              v.null = (prev_nm >> c) & 1;
            } else {
              v = call_output(t, p, c, hot, cold, flags);
            }
            write_out_val(o, p, c, rr, v);
          }
        }
      }
      // remember what was emitted (prev_outputs, agg_group.rs:575-603)
      uint64_t nf = flags;
      if (store_prev) {
        uint32_t curr_nm = 0;
        for (int c = 0; c < p.n_calls; c++) {
          const OutVal v = call_output(t, p, c, hot, cold, flags);
          cold[1 + c] = v.lo;
          if (p.prevhi_off[c] >= 0) cold[p.prevhi_off[c]] = v.hi;
          if (v.null) curr_nm |= 1u << c;
        }
        nf = (nf & ~(0xFFFFull << 16)) | ((uint64_t)curr_nm << 16) | COLD_HAS_PREV;
      } else if (nrows == 1 && op0 == RW_OP_DELETE) {
        nf &= ~(COLD_HAS_PREV | (0xFFFFull << 16));
      }
      cold[0] = nf;
      {  // the staged rows go back
        uint64_t* gc = t.cold + slot * p.CW;
#pragma unroll 4
        for (int k = 0; k < p.CW; k++) gc[k] = cold[k];
        if (hot_changed) {
          uint64_t* gh = t.hot + slot * p.HW;
          for (int k = 0; k < p.HW; k++) gh[k] = hot[k];
        }
      }
      t.dirty[slot >> 5] = 0;  // every dirty slot of this word is in the list; racing zero-stores are benign
    }
    __syncthreads();  // s_warp / s_base are rewritten by the next round
  }
  // the last block to get here publishes the barrier's status
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&t.status->blocks_done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last) {
    __threadfence();
    agg_publish(t.status, o.has_null, pub, threadIdx.x);
  }
}

// a barrier over an epoch without input rows: only the status publication
__global__ void agg_epilogue_kernel(AggStatus* st, unsigned int* has_null, AggPublish pub) { agg_publish(st, has_null, pub, threadIdx.x); }

// ------------------------------------------------------------------ rehash kernel: growth, and watermark cleaning
// live (not retracted) value records on the chains of a group's retractable min / max calls
__device__ __forceinline__ unsigned int mm_live_records(const AggTable& t, const AggPlanDev& p, const uint64_t* cold) {
  unsigned int n = 0;
  for (int c = 0; c < p.n_calls; c++) {
    if (p.mm_off[c] < 0) continue;
    for (uint32_t id = (uint32_t)cold[p.mm_off[c]]; id != 0u;) {
      const uint32_t lk = (uint32_t)t.mm_log[id].x;
      if (!(lk & MM_DEAD)) n++;
      id = lk & ~MM_DEAD;
    }
  }
  return n;
}

// wm_key >= 0: the state-table cleaning below a watermark (rwgpu_agg_update_watermark).  A group whose key column wm_key
// is non-NULL and below `wm` (signed order of the key word: int2 / int4 / date are sign-extended) is not carried over;
// its live value records become unreachable and are counted dead for the value-log compaction.
__global__ void agg_rehash_kernel(AggTable o, AggTable n, AggPlanDev p, int wm_key, long long wm) {
  const uint64_t total = o.cap + 2;
  unsigned int kept = 0, lost = 0;
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < total; s += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t* oh = o.hot + s * p.HW;
    const uint64_t* oc = o.cold + s * p.CW;
    const bool dirty = (o.dirty[s >> 5] >> (s & 31)) & 1;
    uint64_t dst;
    if (s >= o.cap) {
      // single-column keys: slot cap + 1 holds the key INT64_MIN (cap, the NULL key, is never below a watermark)
      if (wm_key >= 0 && p.single_key && s == o.cap + 1 && (long long)AGG_EMPTY < wm) {
        lost += mm_live_records(o, p, oc);
        continue;  // (the new table's side slot stays in its initial state)
      }
      dst = n.cap + (s - o.cap);
    } else {
      uint64_t w0 = oh[0];
      if (p.single_key ? (w0 == AGG_EMPTY) : (w0 == 0)) continue;
      // drop groups that hold no rows, emitted nothing and are not dirty (the reference evicts them
      // from its LRU and deletes their intermediate-state row, agg_group.rs:473-538)
      long long rc = (long long)oh[p.KW + p.row_count_call];
      if (rc == 0 && !(oc[0] & COLD_HAS_PREV) && !dirty) continue;
      if (wm_key >= 0) {
        const bool key_null = !p.single_key && ((w0 >> (8 + wm_key)) & 1ull);
        const long long kv = (long long)(p.single_key ? w0 : oh[1 + wm_key]);
        if (!key_null && kv < wm) {
          lost += mm_live_records(o, p, oc);
          continue;
        }
      }
      kept++;
      uint64_t mask = n.cap - 1;
      if (p.single_key) {
        uint64_t idx = mix64(w0) & mask;
        while (true) {
          unsigned long long* ptr = (unsigned long long*)(n.hot + idx * p.HW);
          if (atomicCAS(ptr, (unsigned long long)AGG_EMPTY, (unsigned long long)w0) == AGG_EMPTY) break;
          idx = (idx + 1) & mask;
        }
        dst = idx;
      } else {
        uint32_t nm = (uint32_t)((w0 >> 8) & 0xff);
        uint64_t h = 0x9e3779b97f4a7c15ull ^ nm;
        for (int k = 0; k < p.n_keys; k++) h = mix64(h ^ oh[1 + k]) + 0x9e3779b97f4a7c15ull;
        uint64_t idx = (h >> 17) & mask;
        while (true) {
          unsigned long long* ptr = (unsigned long long*)(n.hot + idx * p.HW);
          if (atomicCAS(ptr, 0ull, (unsigned long long)w0) == 0ull) break;
          idx = (idx + 1) & mask;
        }
        dst = idx;
      }
    }
    uint64_t* nh = n.hot + dst * p.HW;
    uint64_t* nc = n.cold + dst * p.CW;
    for (int k = (s >= o.cap ? 0 : 1); k < p.HW; k++) nh[k] = oh[k];
    for (int k = 0; k < p.CW; k++) nc[k] = oc[k];
    if (dirty) {
      atomicOr(n.dirty + (dst >> 5), 1u << (dst & 31));
      n.dirty_list[atomicAdd(&n.status->n_dirty, 1u)] = (uint32_t)dst;
    }
  }
  for (int d = 16; d > 0; d >>= 1) {
    kept += __shfl_xor_sync(0xffffffffu, kept, d);
    lost += __shfl_xor_sync(0xffffffffu, lost, d);
  }
  if (lane_id() == 0 && kept) atomicAdd(&n.status->n_groups, (unsigned long long)kept);
  if (lane_id() == 0 && lost) atomicAdd(&n.status->mm_dead, lost);
}

// ------------------------------------------------------------------ value-log compaction (after a cleaning rebuild)
// The records of cleaned groups and retracted records are dead weight in mm_log.  At a cleaning barrier the log is
// rebuilt from the live records of the surviving groups -- like uni_compact for the join's row log -- when more than
// half of it, and more than AGG_MM_COMPACT_FLOOR records, are dead.  A rebuild costs a walk of the table and of the log,
// paid for by the dead records it reclaims; without one the log stays within 2 x live + AGG_MM_COMPACT_FLOOR records.
// The decision is taken on the device (the host never waits for a barrier): every kernel below re-evaluates it from
// counters none of them changes before agg_clean_finish_kernel.
#define AGG_MM_COMPACT_FLOOR 4096ull
struct AggCleanDev {
  unsigned long long new_next;  // next record id of the log being rebuilt (1 between rebuilds)
  unsigned long long compactions;
};

__device__ __forceinline__ bool mm_compact_due(const AggTable& t) {
  const unsigned long long used = __ldcg(t.mm_next) - 1, dead = __ldcg(&t.status->mm_dead);
  return 2 * dead > used + AGG_MM_COMPACT_FLOOR;
}

// one thread per slot: each chain's live records go, contiguous and linked in order, to `dst` (the spare log)
__global__ void __launch_bounds__(256) agg_mm_compact_kernel(AggTable t, AggPlanDev p, ulonglong2* dst, AggCleanDev* cd) {
  if (!mm_compact_due(t)) return;
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < t.cap + 2; s += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t* cold = t.cold + s * p.CW;
    for (int c = 0; c < p.n_calls; c++) {
      if (p.mm_off[c] < 0) continue;
      uint32_t* head = (uint32_t*)(cold + p.mm_off[c]);
      if (*head == 0u) continue;  // (empty slots too: their cold rows are zero)
      unsigned int live = 0;
      for (uint32_t id = *head; id != 0u;) {
        const uint32_t lk = (uint32_t)t.mm_log[id].x;
        if (!(lk & MM_DEAD)) live++;
        id = lk & ~MM_DEAD;
      }
      const unsigned long long base = live ? atomicAdd(&cd->new_next, (unsigned long long)live) : 0ull;
      unsigned long long j = base;
      for (uint32_t id = *head; id != 0u;) {
        const ulonglong2 rec = t.mm_log[id];
        const uint32_t lk = (uint32_t)rec.x;
        if (!(lk & MM_DEAD)) {
          dst[j] = make_ulonglong2(j + 1 < base + live ? j + 1 : 0ull, rec.y);
          j++;
        }
        id = lk & ~MM_DEAD;
      }
      *head = (uint32_t)base;
    }
  }
}

// the rebuilt records go back to the handle's log (whose address the host keeps)
__global__ void __launch_bounds__(256) agg_mm_commit_kernel(AggTable t, const ulonglong2* src, const AggCleanDev* cd) {
  if (!mm_compact_due(t)) return;
  const unsigned long long n = __ldcg(&cd->new_next);
  for (unsigned long long i = 1 + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
    t.mm_log[i] = src[i];
}

// one thread: close the rebuild, and publish the group count and the log's next record id AFTER the cleaning to the
// barrier's pinned status slot (the flush kernel published the count before it), for the host's upper bounds
__global__ void agg_clean_finish_kernel(AggTable t, AggCleanDev* cd, int compact, AggStatus* st_host, unsigned long long* mm_next_host) {
  if (compact && mm_compact_due(t)) {
    *t.mm_next = cd->new_next;
    t.status->mm_dead = 0;
    cd->compactions++;
  }
  cd->new_next = 1;
  st_host->n_groups = t.status->n_groups;
  *mm_next_host = *t.mm_next;
  __threadfence_system();
}

// ------------------------------------------------------------------ state persistence (SURVEY 8(f) rank 3)
// What the reference persists per group is the INTERMEDIATE STATE row  group key | one state datum per call
// (AggGroup::build_states_change agg_group.rs:473-538 -> intermediate_state_table.write_record; a group whose row
// count is 0 is deleted from the table), plus, per retractable min / max call, the rows of its materialized input
// (minput.rs).  On recovery AggGroup::create (agg_group.rs:260-316) loads that row and derives prev_outputs from it.
// The snapshot kernels produce exactly those rows as columnar chunks (the shim hands them to StateTable::write_chunk,
// which does the value / memcomparable encoding and the vnode prefix); restore rebuilds the table from them.
struct AggSnapOut {
  void* col[RW_MAX_KEYS + RW_MAX_CALLS];
  uint8_t* valid[RW_MAX_KEYS + RW_MAX_CALLS];
  unsigned long long* n_rows;
  unsigned int* has_null;  // per column
  // materialized input: key columns | int32 call index | int64 value (sortable form decoded by the host)
  void* mcol[RW_MAX_KEYS + 2];
  uint8_t* mvalid[RW_MAX_KEYS];
  unsigned long long* m_rows;
  int64_t capacity, m_capacity;
};

__device__ __forceinline__ void snap_key(const AggTable& t, const AggPlanDev& p, uint64_t slot, const uint64_t* hot, uint64_t* keyw,
                                         uint32_t* key_nm) {
  *key_nm = 0;
  if (p.single_key) {
    if (slot == t.cap) { *key_nm = 1; keyw[0] = 0; }
    else keyw[0] = (slot == t.cap + 1) ? AGG_EMPTY : hot[0];
  } else {
    *key_nm = (uint32_t)((hot[0] >> 8) & 0xff);
    for (int k = 0; k < p.n_keys; k++) keyw[k] = hot[1 + k];
  }
}

__global__ void __launch_bounds__(256) agg_snapshot_kernel(AggTable t, AggPlanDev p, AggSnapOut o, int count_only) {
  const int lane = lane_id();
  for (uint64_t s0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) & ~31ull; s0 < t.cap + 2; s0 += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t slot = s0 + lane;
    bool live = false;
    const uint64_t* hot = nullptr;
    const uint64_t* cold = nullptr;
    if (slot < t.cap + 2) {
      hot = t.hot + slot * p.HW;
      cold = t.cold + slot * p.CW;
      const bool occupied = slot >= t.cap ? true : (p.single_key ? hot[0] != AGG_EMPTY : hot[0] != 0ull);
      live = occupied && (long long)hot[p.KW + p.row_count_call] > 0;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, live);
    unsigned long long base = 0;
    if (lane == 0 && bal) base = atomicAdd(o.n_rows, (unsigned long long)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (!live) continue;
    const int64_t row = (int64_t)base + __popc(bal & ((1u << lane) - 1u));
    uint64_t keyw[RW_MAX_KEYS];
    uint32_t key_nm;
    snap_key(t, p, slot, hot, keyw, &key_nm);
    if (!count_only && row < o.capacity) {
      for (int k = 0; k < p.n_keys; k++) {
        const bool nul = (key_nm >> k) & 1;
        o.valid[k][row] = nul ? 0 : 1;
        if (nul) o.has_null[k] = 1;
        store_word(o.col[k], type_width_dev(p.key_type[k]), p.key_type[k], row, keyw[k]);
      }
      const uint64_t flags = cold[0];
      for (int c = 0; c < p.n_calls; c++) {
        const OutVal v = call_output(t, p, c, hot, cold, flags);  // a value state's output IS its state datum
        const int oc = p.n_keys + c;
        o.valid[oc][row] = v.null ? 0 : 1;
        if (v.null) o.has_null[oc] = 1;
        if (p.ret_type[c] == RW_T_DECIMAL) {
          ((uint64_t*)o.col[oc])[row * 2] = v.lo;
          ((uint64_t*)o.col[oc])[row * 2 + 1] = v.hi;
        } else {
          store_word(o.col[oc], type_width_dev(p.ret_type[c]), p.ret_type[c], row, v.lo);
        }
      }
    }
    // materialized input of the retractable min / max calls: one row per live value
    for (int c = 0; c < p.n_calls; c++) {
      if (p.mm_off[c] < 0) continue;
      for (uint32_t id = (uint32_t)cold[p.mm_off[c]]; id != 0u;) {
        const ulonglong2 rec = t.mm_log[id];
        const uint32_t lk = (uint32_t)rec.x;
        if (!(lk & MM_DEAD)) {
          const unsigned long long mr = atomicAdd(o.m_rows, 1ull);
          if (!count_only && (int64_t)mr < o.m_capacity) {
            for (int k = 0; k < p.n_keys; k++) {
              o.mvalid[k][mr] = ((key_nm >> k) & 1) ? 0 : 1;
              store_word(o.mcol[k], type_width_dev(p.key_type[k]), p.key_type[k], (int64_t)mr, keyw[k]);
            }
            ((int32_t*)o.mcol[p.n_keys])[mr] = c;
            const bool isf = p.arg_type[c] == RW_T_FLOAT32 || p.arg_type[c] == RW_T_FLOAT64;
            ((long long*)o.mcol[p.n_keys + 1])[mr] = isf ? __double_as_longlong(f64_unsortable((int64_t)rec.y)) : (long long)rec.y;
          }
        }
        id = lk & ~MM_DEAD;
      }
    }
  }
}

// restore: one intermediate-state row -> one group (states, flags, carry words; prev_outputs = the outputs of the
// loaded states, agg_group.rs:305-309)
__global__ void __launch_bounds__(256) agg_restore_kernel(AggTable t, AggPlanDev p, DevChunk ch) {
  unsigned int created_local = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t slot;
    bool created = false;
    if (p.single_key) {
      const ColRef& kc = ch.cols[0];
      if (col_is_null(kc, r)) slot = t.cap;
      else {
        const uint64_t key = load_key_word(kc, r);
        slot = key == AGG_EMPTY ? t.cap + 1 : find_or_insert_single(t, p.HW, key, &created);
      }
    } else {
      uint64_t kw[RW_MAX_KEYS];
      uint32_t nm = 0;
      for (int k = 0; k < p.n_keys; k++) {
        if (col_is_null(ch.cols[k], r)) { nm |= 1u << k; kw[k] = 0; }
        else kw[k] = load_key_word(ch.cols[k], r);
      }
      slot = find_or_insert_multi(t, p, kw, nm, &created);
    }
    if (created) created_local++;
    uint64_t* hot = t.hot + slot * p.HW;
    uint64_t* cold = t.cold + slot * p.CW;
    uint64_t flags = 0;
    for (int c = 0; c < p.n_calls; c++) {
      const ColRef& sc = ch.cols[p.n_keys + c];
      const int kind = p.kind[c], at = p.arg_type[c];
      const bool isf = at == RW_T_FLOAT32 || at == RW_T_FLOAT64;
      if (col_is_null(sc, r)) { hot[p.KW + c] = state_init(kind, at); continue; }
      if (kind != RW_AGG_COUNT) flags |= 1ull << c;
      if (kind == RW_AGG_COUNT) {
        hot[p.KW + c] = (uint64_t)load_i64(sc, r);
      } else if (kind == RW_AGG_SUM || kind == RW_AGG_SUM0) {
        if (at == RW_T_FLOAT32) {
          hot[p.KW + c] = (uint64_t)__float_as_uint(((const float*)sc.data)[r]);  // f32 state (agg_apply_row)
        } else if (isf) {
          hot[p.KW + c] = (uint64_t)__double_as_longlong(load_f64(sc, r));
        } else if (p.ret_type[c] == RW_T_DECIMAL) {
          const uint64_t* d = (const uint64_t*)sc.data + r * 2;
          hot[p.KW + c] = d[0];
          if (p.hi_off[c] >= 0) cold[p.hi_off[c]] = d[1];
        } else {
          const long long v = (long long)load_i64(sc, r);
          hot[p.KW + c] = (uint64_t)v;
          if (p.hi_off[c] >= 0) cold[p.hi_off[c]] = (uint64_t)(v >> 63);
        }
      } else {
        hot[p.KW + c] = isf ? (uint64_t)f64_sortable(load_f64(sc, r)) : (uint64_t)load_i64(sc, r);
      }
    }
    // prev_outputs = get_outputs(loaded states)
    uint32_t prev_nm = 0;
    for (int c = 0; c < p.n_calls; c++) {
      const OutVal v = call_output(t, p, c, hot, cold, flags);
      cold[1 + c] = v.lo;
      if (p.prevhi_off[c] >= 0) cold[p.prevhi_off[c]] = v.hi;
      if (v.null) prev_nm |= 1u << c;
    }
    cold[0] = flags | ((uint64_t)prev_nm << 16) | COLD_HAS_PREV;
  }
  for (int o2 = 16; o2 > 0; o2 >>= 1) created_local += __shfl_xor_sync(0xffffffffu, created_local, o2);
  if (lane_id() == 0 && created_local) atomicAdd(&t.status->n_groups, (unsigned long long)created_local);
}

// restore of a materialized-input row: (group key | call index | value) -> one record on the group's chain.  The group
// must already hold its state row (row count > 0): the row is looked up, never inserted, and refused otherwise.
__global__ void __launch_bounds__(256) agg_restore_minput_kernel(AggTable t, AggPlanDev p, DevChunk ch) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t slot = ~0ull;
    const uint64_t mask = t.cap - 1;
    if (p.single_key) {
      const ColRef& kc = ch.cols[0];
      if (col_is_null(kc, r)) slot = t.cap;
      else {
        const uint64_t key = load_key_word(kc, r);
        if (key == AGG_EMPTY) slot = t.cap + 1;
        else
          for (uint64_t i = mix64(key) & mask; t.hot[i * p.HW] != AGG_EMPTY; i = (i + 1) & mask)
            if (t.hot[i * p.HW] == key) { slot = i; break; }
      }
    } else {
      uint64_t kw[RW_MAX_KEYS];
      uint32_t nm = 0;
      for (int k = 0; k < p.n_keys; k++) {
        if (col_is_null(ch.cols[k], r)) { nm |= 1u << k; kw[k] = 0; }
        else kw[k] = load_key_word(ch.cols[k], r);
      }
      const uint64_t h = multi_hash(p, kw, nm);
      const uint64_t tag = (h & ~0xFFFFull) | ((uint64_t)nm << 8) | 1ull;
      for (uint64_t i = (h >> 17) & mask; t.hot[i * p.HW] != 0ull; i = (i + 1) & mask) {
        bool eq = t.hot[i * p.HW] == tag;
        for (int k = 0; k < p.n_keys && eq; k++) eq = t.hot[i * p.HW + 1 + k] == kw[k];
        if (eq) { slot = i; break; }
      }
    }
    const int c = (int)load_i64(ch.cols[p.n_keys], r);
    if (c < 0 || c >= p.n_calls || p.mm_off[c] < 0 || slot == ~0ull || (long long)t.hot[slot * p.HW + p.KW + p.row_count_call] <= 0) {
      atomicOr(&t.status->err, AGG_ERR_MM_BAD_ROW);
      continue;
    }
    const unsigned long long id = atomicAdd(t.mm_next, 1ull);
    if (id >= t.mm_cap) { atomicOr(&t.status->err, AGG_ERR_MM_CAPACITY); continue; }
    uint64_t* cold = t.cold + slot * p.CW;
    const uint32_t old = atomicExch((uint32_t*)(cold + p.mm_off[c]), (uint32_t)id);
    const bool isf = p.arg_type[c] == RW_T_FLOAT32 || p.arg_type[c] == RW_T_FLOAT64;
    long long v = (long long)load_i64(ch.cols[p.n_keys + 1], r);
    if (isf) v = (long long)f64_sortable(__longlong_as_double(v));
    t.mm_log[id] = make_ulonglong2((unsigned long long)old, (unsigned long long)v);
  }
}

__global__ void pack_bytes_to_bits_kernel(const uint8_t* bytes, uint64_t* words, int64_t n) {
  int64_t nw = (n + 63) >> 6;
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nw; w += (int64_t)gridDim.x * blockDim.x) {
    uint64_t v = 0;
    int64_t base = w << 6;
    int lim = (int)((n - base) < 64 ? (n - base) : 64);
    for (int b = 0; b < lim; b++) v |= (uint64_t)(bytes[base + b] != 0) << b;
    words[w] = v;
  }
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace rw

// =============================================================================== host handle
using namespace rw;

struct AggStage {
  PinnedBuf host;
  DevBuf dev;
  cudaEvent_t done = nullptr;
  bool in_flight = false;
  int64_t rows = 0;
  bool has_valid[RW_MAX_COLS];
};

struct rwgpu_agg {
  AggPlanDev plan;
  std::vector<int> in_types, out_types, used_cols;
  int chunk_size = 1024;
  cudaStream_t stream = nullptr;
  DevBuf hot, cold, dirty, dirty_list, status;
  uint64_t cap = 0;
  uint64_t groups_upper = 0;
  uint64_t epoch_rows = 0;
  bool per_row_mode = false, nullfree_push_seen = false;
  uint32_t all_flag_mask = 0;
  uint64_t launches = 0;
  KernelProf prof;
  bool fast_eligible = false;
  // retractable min / max: log of input values (grows; ids start at 1)
  int n_retract = 0;
  DevBuf mm_log, mm_next;
  uint64_t mm_cap = 0, mm_upper = 1;
  uint64_t mm_charged = 0;  // records ever charged to mm_upper by pushes
  // watermark-driven state cleaning (rwgpu_agg_update_watermark): one pending watermark, applied at the next barrier by
  // a rebuild into the spare table (same capacity; the two swap) and, when due, a rebuild of the value log through the
  // spare log.  Both spares are kept once they have been needed.
  bool wm_pending = false;
  int wm_key_pos = 0;
  int64_t wm_value = 0;
  DevBuf sp_hot, sp_cold, sp_dirty, sp_dlist, mm_spare, clean_dev;
  uint64_t sp_cap = 0;
  // staging (host pushes)
  AggStage stage[2];
  int cur = 0;
  int64_t stage_cap = 1 << 18;
  size_t off_ops = 0, stage_bytes = 0;
  size_t off_data[RW_MAX_COLS], off_valid[RW_MAX_COLS];
  // output buffers (device): two sets, so the delta of barrier e can still be read while barrier e + 1 is computed
  struct OutSet {
    DevBuf ops, col[RW_MAX_KEYS + RW_MAX_CALLS], valid[RW_MAX_KEYS + RW_MAX_CALLS], bits[RW_MAX_KEYS + RW_MAX_CALLS];
    int64_t cap = 0;
  } outs[2];
  int flip = 0;
  DevBuf out_hasnull;
  // barriers enqueued but not collected yet (at most two): status slot = output set
  struct Pending {
    int set;
    unsigned long long tag;
    uint64_t rows_total;
    uint64_t mm_charged;
    bool cleaned;
    cudaStream_t st;
  } pending[2];
  int n_pending = 0;
  unsigned long long tag = 0;
  uint64_t rows_total = 0;  // rows ever pushed
  cudaEvent_t pend_ev[2] = {nullptr, nullptr};
  // one logical stream of work per handle: a call on another stream than the previous one waits for it on the device
  cudaStream_t last_st = nullptr;
  cudaEvent_t order_ev = nullptr;
  PinnedBuf status_host;  // per set: AggStatus @0, has_null flags @64, tag @192, mm_next after cleaning @200 (256 bytes each)
  std::shared_ptr<PinnedPool> pool = std::make_shared<PinnedPool>();
  std::vector<rw_column> dev_view_cols;

  AggTable table() const {
    AggTable t;
    t.hot = hot.as<uint64_t>();
    t.cold = cold.as<uint64_t>();
    t.dirty = dirty.as<uint32_t>();
    t.dirty_list = dirty_list.as<uint32_t>();
    t.status = status.as<AggStatus>();
    t.cap = cap;
    t.mm_log = mm_log.as<ulonglong2>();
    t.mm_next = mm_next.as<unsigned long long>();
    t.mm_cap = mm_cap;
    return t;
  }
  ~rwgpu_agg() {
    for (auto& s : stage) if (s.done) cudaEventDestroy(s.done);
    for (auto e : pend_ev) if (e) cudaEventDestroy(e);
    if (order_ev) cudaEventDestroy(order_ev);
    if (stream) cudaStreamDestroy(stream);
  }
};

static int grid_for(int64_t n_threads, int block) {
  int64_t g = (n_threads + block - 1) / block;
  int64_t maxg = RW_SMS * 8;
  return (int)std::max<int64_t>(1, std::min(g, maxg));
}

static int agg_alloc_table(rwgpu_agg* h, uint64_t cap, DevBuf& hot, DevBuf& cold, DevBuf& dirty, DevBuf& dlist) {
  size_t slots = cap + 2;
  RW_CUDA(hot.reserve(slots * h->plan.HW * 8));
  RW_CUDA(cold.reserve(slots * h->plan.CW * 8));
  RW_CUDA(dirty.reserve(((slots + 31) / 32) * 4));
  RW_CUDA(dlist.reserve(slots * 4));
  return RW_OK;
}

static int agg_init_table(rwgpu_agg* h, AggTable t) {
  RW_CUDA(cudaMemsetAsync(t.dirty, 0, ((t.cap + 2 + 31) / 32) * 4, h->stream));
  agg_init_kernel<<<grid_for((int64_t)t.cap + 2, 256), 256, 0, h->stream>>>(t, h->plan, 0);
  RW_CUDA(cudaGetLastError());
  h->launches++;
  return RW_OK;
}

// make room for `incoming` more rows (each may open a new group); grows + rehashes when needed
static int agg_ensure_capacity(rwgpu_agg* h, uint64_t incoming) {
  if ((h->groups_upper + incoming) * 2 <= h->cap) return RW_OK;
  // the bound is pessimistic: read the real group count.  Work of this handle may be in flight on the handle's own
  // stream AND on a caller's stream (rwgpu_agg_push_device / flush_device): wait for all of it -- reading the
  // count, or re-hashing the table, under a running apply kernel would lose groups or updates.
  RW_CUDA(cudaDeviceSynchronize());
  AggStatus sh_local;
  AggStatus* sh = &sh_local;
  RW_CUDA(cudaMemcpy(sh, h->status.p, sizeof(AggStatus), cudaMemcpyDeviceToHost));
  h->groups_upper = sh->n_groups;
  if ((h->groups_upper + incoming) * 2 <= h->cap) return RW_OK;
  uint64_t need = (h->groups_upper + incoming) * 4;
  uint64_t ncap = h->cap;
  while (ncap < need) ncap <<= 1;
  DevBuf nh, nc, nd, nl;
  int rc = agg_alloc_table(h, ncap, nh, nc, nd, nl);
  if (rc != RW_OK) return rc;
  AggTable ot = h->table();
  AggTable nt = ot;
  nt.hot = nh.as<uint64_t>(); nt.cold = nc.as<uint64_t>(); nt.dirty = nd.as<uint32_t>(); nt.dirty_list = nl.as<uint32_t>(); nt.cap = ncap;
  rc = agg_init_table(h, nt);
  if (rc != RW_OK) return rc;
  RW_CUDA(cudaMemsetAsync(&h->status.as<AggStatus>()->n_groups, 0, sizeof(unsigned long long), h->stream));
  RW_CUDA(cudaMemsetAsync(&h->status.as<AggStatus>()->n_dirty, 0, sizeof(unsigned int), h->stream));
  agg_rehash_kernel<<<grid_for((int64_t)ot.cap + 2, 256), 256, 0, h->stream>>>(ot, nt, h->plan, -1, 0);
  RW_CUDA(cudaGetLastError());
  h->launches++;
  RW_CUDA(cudaStreamSynchronize(h->stream));  // old buffers are freed below
  h->hot = std::move(nh);
  h->cold = std::move(nc);
  h->dirty = std::move(nd);
  h->dirty_list = std::move(nl);
  h->cap = ncap;
  RW_CUDA(cudaMemcpy(sh, h->status.p, sizeof(AggStatus), cudaMemcpyDeviceToHost));
  h->groups_upper = sh->n_groups;
  return RW_OK;
}

// the signatures src/expr/impl/src/aggregate/general.rs declares over the types of rwgpu.h (sum :18-27, min / max
// :93-128, count :155-162); any other (kind, argument, return type) is refused with RW_ERR_INVALID before it is asked
// whether the device runs it.  Unknown kinds pass here and are refused as unsupported.
static bool agg_signature_ok(int kind, bool has_arg, int at, int ret) {
  switch (kind) {
    case RW_AGG_COUNT: return ret == RW_T_INT64;  // count() / count(any) -> int8
    case RW_AGG_SUM0: return has_arg && at == RW_T_INT64 && ret == RW_T_INT64;
    case RW_AGG_SUM:
      if (!has_arg) return false;
      if (at == RW_T_INT16 || at == RW_T_INT32) return ret == RW_T_INT64;
      if (at == RW_T_INT64) return ret == RW_T_INT64 || ret == RW_T_DECIMAL;
      return (at == RW_T_FLOAT32 || at == RW_T_FLOAT64 || at == RW_T_DECIMAL) && ret == at;
    case RW_AGG_MIN:
    case RW_AGG_MAX: return has_arg && at != RW_T_BOOL && ret == at;  // `-> auto`; no min / max(boolean)
    default: return true;
  }
}

static bool chunk_fast_ok(const rwgpu_agg* h, const DevChunk& ch) {
  if (!h->fast_eligible || ch.vis_bits != nullptr) return false;
  if (((uintptr_t)ch.ops & 1) != 0) return false;
  for (int c : h->used_cols) {
    const ColRef& r = ch.cols[c];
    if (r.valid_bits || r.valid_bytes) return false;
    if (((uintptr_t)r.data & 15) != 0) return false;
  }
  return true;
}

// enqueue the apply kernel for a device-resident chunk
static int agg_order(rwgpu_agg* h, cudaStream_t st) {
  if (h->last_st && h->last_st != st) {
    if (!h->order_ev) RW_CUDA(cudaEventCreateWithFlags(&h->order_ev, cudaEventDisableTiming));
    RW_CUDA(cudaEventRecord(h->order_ev, h->last_st));
    RW_CUDA(cudaStreamWaitEvent(st, h->order_ev, 0));
  }
  h->last_st = st;
  return RW_OK;
}

// A chunk with a device row count (ch.n_dev) is charged at its capacity ch.n in every host-side upper bound (groups,
// rows, epoch rows, materialized-input records): the kernels clamp the count themselves, nothing is read back.
static int agg_apply_dev(rwgpu_agg* h, const DevChunk& ch, cudaStream_t st) {
  if (ch.n <= 0) return RW_OK;
  int rc = agg_ensure_capacity(h, (uint64_t)ch.n);
  if (rc != RW_OK) return rc;
  rc = agg_order(h, st);
  if (rc != RW_OK) return rc;
  h->rows_total += (uint64_t)ch.n;
  if (h->n_retract) {
    // every non-NULL input value of a retractable min / max call takes a record
    const uint64_t need = h->mm_upper + (uint64_t)ch.n * (uint64_t)h->n_retract;
    if (need > h->mm_cap) {
      RW_CUDA(cudaDeviceSynchronize());
      unsigned long long used = 1;
      RW_CUDA(cudaMemcpy(&used, h->mm_next.p, 8, cudaMemcpyDeviceToHost));
      h->mm_upper = used;  // (NULL arguments and retractions took none)
      const uint64_t need2 = used + (uint64_t)ch.n * (uint64_t)h->n_retract;
      if (need2 > h->mm_cap) {
        uint64_t ncap = std::max<uint64_t>(h->mm_cap * 2, need2 + need2 / 2);
        if (ncap >= 0x7ffffff0ull) return fail(RW_ERR_OOM, "materialized input of retractable min/max exceeds 2^31 values");
        DevBuf nl;
        RW_CUDA(nl.reserve((size_t)ncap * 16));
        RW_CUDA(cudaMemcpy(nl.p, h->mm_log.p, (size_t)used * 16, cudaMemcpyDeviceToDevice));
        h->mm_log = std::move(nl);
        h->mm_cap = ncap;
      }
    }
    h->mm_upper += (uint64_t)ch.n * (uint64_t)h->n_retract;
    h->mm_charged += (uint64_t)ch.n * (uint64_t)h->n_retract;
  }
  bool has_nulls = h->n_retract > 0;  // retractable min / max keeps its "state is non-NULL" flags per row
  for (int c : h->used_cols) if (ch.cols[c].valid_bits || ch.cols[c].valid_bytes) has_nulls = true;
  if (has_nulls) {
    if (!h->per_row_mode && h->nullfree_push_seen) {
      agg_set_flags_kernel<<<grid_for((int64_t)std::min<uint64_t>(h->epoch_rows + 1, h->cap + 2), 256), 256, 0, st>>>(h->table(), h->plan, h->all_flag_mask);
      RW_CUDA(cudaGetLastError());
      h->launches++;
    }
    h->per_row_mode = true;
  } else if (!h->per_row_mode) {
    h->nullfree_push_seen = true;
  }
  AggTable t = h->table();
  h->prof.begin(st);
  if (!h->per_row_mode && chunk_fast_ok(h, ch)) {
    int g = grid_for((ch.n + 1) / 2, 256);
    switch (h->plan.n_calls) {
      case 1: agg_apply_fast_kernel<1><<<g, 256, 0, st>>>(t, h->plan, ch); break;
      case 2: agg_apply_fast_kernel<2><<<g, 256, 0, st>>>(t, h->plan, ch); break;
      case 3: agg_apply_fast_kernel<3><<<g, 256, 0, st>>>(t, h->plan, ch); break;
      default: agg_apply_fast_kernel<4><<<g, 256, 0, st>>>(t, h->plan, ch); break;
    }
  } else {
    agg_apply_kernel<<<grid_for(ch.n, 256), 256, 0, st>>>(t, h->plan, ch, h->per_row_mode ? 1 : 0);
  }
  h->prof.end(st);
  RW_CUDA(cudaGetLastError());
  h->launches++;
  if (h->n_retract) {
    agg_mm_delete_kernel<<<grid_for(ch.n, 256), 256, 0, st>>>(t, h->plan, ch);
    RW_CUDA(cudaGetLastError());
    h->launches++;
  }
  h->groups_upper += (uint64_t)ch.n;
  h->epoch_rows += (uint64_t)ch.n;
  return RW_OK;
}

static int agg_launch_stage(rwgpu_agg* h) {
  AggStage& s = h->stage[h->cur];
  if (s.rows == 0) return RW_OK;
  uint8_t* hp = s.host.as<uint8_t>();
  uint8_t* dp = s.dev.as<uint8_t>();
  {
    int rc0 = agg_order(h, h->stream);
    if (rc0 != RW_OK) return rc0;
  }
  RW_CUDA(cudaMemcpyAsync(dp + h->off_ops, hp + h->off_ops, (size_t)s.rows, cudaMemcpyHostToDevice, h->stream));
  DevChunk ch;
  memset(&ch, 0, sizeof(ch));
  ch.n = s.rows;
  ch.ops = dp + h->off_ops;
  ch.vis_bits = nullptr;
  ch.n_cols = (int)h->in_types.size();
  for (size_t k = 0; k < h->in_types.size(); k++) {
    ch.cols[k].type = h->in_types[k];
    ch.cols[k].width = type_width(h->in_types[k]);
  }
  for (int c : h->used_cols) {
    int w = type_width(h->in_types[c]);
    RW_CUDA(cudaMemcpyAsync(dp + h->off_data[c], hp + h->off_data[c], (size_t)s.rows * w, cudaMemcpyHostToDevice, h->stream));
    ch.cols[c].data = dp + h->off_data[c];
    if (s.has_valid[c]) {
      RW_CUDA(cudaMemcpyAsync(dp + h->off_valid[c], hp + h->off_valid[c], (size_t)s.rows, cudaMemcpyHostToDevice, h->stream));
      ch.cols[c].valid_bytes = dp + h->off_valid[c];
    }
  }
  int rc = agg_apply_dev(h, ch, h->stream);
  if (rc != RW_OK) return rc;
  RW_CUDA(cudaEventRecord(s.done, h->stream));
  s.in_flight = true;
  s.rows = 0;
  h->cur ^= 1;
  AggStage& nx = h->stage[h->cur];
  if (nx.in_flight) {
    RW_CUDA(cudaEventSynchronize(nx.done));
    nx.in_flight = false;
  }
  nx.rows = 0;
  memset(nx.has_valid, 0, sizeof(nx.has_valid));
  return RW_OK;
}

static int agg_ensure_out(rwgpu_agg* h, int set, int64_t rows) {
  rwgpu_agg::OutSet& os = h->outs[set];
  if (rows <= os.cap) return RW_OK;
  int64_t cap = std::max<int64_t>(rows, 4096);
  RW_CUDA(cudaDeviceSynchronize());  // (growth only) nobody reads the old buffers any more
  RW_CUDA(os.ops.reserve((size_t)cap));
  for (size_t k = 0; k < h->out_types.size(); k++) {
    RW_CUDA(os.col[k].reserve((size_t)cap * type_width(h->out_types[k])));
    RW_CUDA(os.valid[k].reserve((size_t)cap));
    RW_CUDA(os.bits[k].reserve((size_t)((cap + 63) / 64) * 8));
  }
  os.cap = cap;
  return RW_OK;
}

static const char* agg_err_msg(unsigned int e) {
  if (e & AGG_ERR_BAD_COUNT) return "device row count out of range";
  if (e & AGG_ERR_MM_BAD_ROW) return "materialized-input row of no retractable min/max call, or of a group without a state row";
  if (e & AGG_ERR_OVERFLOW) return "Numeric out of range";
  if (e & AGG_ERR_NEG_COUNT) return "row count should be non-negative";
  if (e & AGG_ERR_RETRACT_APPEND_ONLY) return "attempt to retract on append-only min/max";
  if (e & AGG_ERR_MM_MISSING) return "retracting a value that is not in the aggregate's materialized input";
  if (e & AGG_ERR_MM_CAPACITY) return "internal: materialized-input log capacity";
  if (e & AGG_ERR_OUT_CAPACITY) return "internal: output capacity";
  return "unknown";
}
static int agg_err_code(unsigned int e) {
  if (e & (AGG_ERR_MM_BAD_ROW | AGG_ERR_BAD_COUNT)) return RW_ERR_INVALID;
  if (e & AGG_ERR_OVERFLOW) return RW_ERR_NUMERIC_OUT_OF_RANGE;
  if (e & (AGG_ERR_NEG_COUNT | AGG_ERR_RETRACT_APPEND_ONLY | AGG_ERR_MM_MISSING)) return RW_ERR_INCONSISTENT;
  return RW_ERR_CUDA;
}

// watermark cleaning, enqueued on `st` behind the barrier's delta (nothing is waited for; no allocation once the spares
// exist): rebuild into the spare table without the groups below the watermark, swap the tables, compact the value log if
// due, and publish the counts after cleaning to the barrier's status slot `sh`
static int agg_clean_enqueue(rwgpu_agg* h, cudaStream_t st, uint8_t* sh) {
  h->wm_pending = false;
  if (h->sp_cap != h->cap) {
    int rc = agg_alloc_table(h, h->cap, h->sp_hot, h->sp_cold, h->sp_dirty, h->sp_dlist);
    if (rc != RW_OK) return rc;
    h->sp_cap = h->cap;
  }
  if (h->n_retract) RW_CUDA(h->mm_spare.reserve((size_t)h->mm_cap * 16));
  const AggTable ot = h->table();
  AggTable nt = ot;
  nt.hot = h->sp_hot.as<uint64_t>(); nt.cold = h->sp_cold.as<uint64_t>(); nt.dirty = h->sp_dirty.as<uint32_t>(); nt.dirty_list = h->sp_dlist.as<uint32_t>();
  const int g = grid_for((int64_t)h->cap + 2, 256);
  RW_CUDA(cudaMemsetAsync(nt.dirty, 0, ((h->cap + 2 + 31) / 32) * 4, st));
  agg_init_kernel<<<g, 256, 0, st>>>(nt, h->plan, 0);
  RW_CUDA(cudaMemsetAsync(&h->status.as<AggStatus>()->n_groups, 0, sizeof(unsigned long long), st));
  agg_rehash_kernel<<<g, 256, 0, st>>>(ot, nt, h->plan, h->wm_key_pos, (long long)h->wm_value);
  RW_CUDA(cudaGetLastError());
  std::swap(h->hot, h->sp_hot);
  std::swap(h->cold, h->sp_cold);
  std::swap(h->dirty, h->sp_dirty);
  std::swap(h->dirty_list, h->sp_dlist);
  h->launches += 2;
  AggCleanDev* cd = h->clean_dev.as<AggCleanDev>();
  if (h->n_retract) {
    agg_mm_compact_kernel<<<g, 256, 0, st>>>(nt, h->plan, h->mm_spare.as<ulonglong2>(), cd);
    agg_mm_commit_kernel<<<grid_for((int64_t)h->mm_cap, 256), 256, 0, st>>>(nt, h->mm_spare.as<ulonglong2>(), cd);
    RW_CUDA(cudaGetLastError());
    h->launches += 2;
  }
  agg_clean_finish_kernel<<<1, 1, 0, st>>>(nt, cd, h->n_retract ? 1 : 0, (AggStatus*)sh, (unsigned long long*)(sh + 200));
  RW_CUDA(cudaGetLastError());
  h->launches++;
  return RW_OK;
}

// enqueue the barrier's delta computation on `st` (one launch; nothing is waited for): the rows go to output set
// h->flip, the status to that set's pinned slot.  At most two barriers may be outstanding.
static int agg_flush_enqueue(rwgpu_agg* h, cudaStream_t st) {
  if (h->n_pending >= 2) return fail(RW_ERR_INVALID, "two barriers are already outstanding: collect one first");
  int rc = agg_launch_stage(h);
  if (rc != RW_OK) return rc;
  rc = agg_order(h, st);
  if (rc != RW_OK) return rc;
  const int set = h->flip;
  int64_t bound = (int64_t)std::min<uint64_t>(h->epoch_rows, h->groups_upper + 2) * 2 + 2;
  rc = agg_ensure_out(h, set, bound);
  if (rc != RW_OK) return rc;
  rwgpu_agg::OutSet& os = h->outs[set];
  AggStatus* ds = h->status.as<AggStatus>();
  AggOutDev o;
  o.ops = os.ops.as<uint8_t>();
  for (size_t k = 0; k < h->out_types.size(); k++) { o.col[k] = os.col[k].p; o.valid[k] = os.valid[k].as<uint8_t>(); }
  o.has_null = h->out_hasnull.as<unsigned int>();
  o.capacity = os.cap;
  uint8_t* sh = h->status_host.as<uint8_t>() + 256 * set;
  AggPublish pub;
  pub.st_host = (AggStatus*)sh;
  pub.has_null_host = (unsigned int*)(sh + 64);
  pub.tag_host = (unsigned long long*)(sh + 192);
  pub.tag = ++h->tag;
  uint32_t mask = h->per_row_mode ? 0u : h->all_flag_mask;
  if (h->epoch_rows > 0) {
    int64_t max_dirty = (int64_t)std::min<uint64_t>(h->epoch_rows, h->cap + 2);
    const size_t smem = (size_t)((h->plan.HW + h->plan.CW) | 1) * 8 * 256;  // staged hot + cold row per thread
    static std::atomic<size_t> smem_limit{48 * 1024};  // (process-wide: the attribute belongs to the kernel)
    if (smem > smem_limit.load()) {
      RW_CUDA(cudaFuncSetAttribute(agg_flush_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      smem_limit.store(smem);
    }
    agg_flush_kernel<<<grid_for(max_dirty, 256), 256, smem, st>>>(h->table(), h->plan, o, mask, pub);
  } else {
    agg_epilogue_kernel<<<1, 32, 0, st>>>(ds, o.has_null, pub);
  }
  RW_CUDA(cudaGetLastError());
  h->launches++;
  const bool cleaned = h->wm_pending;
  if (cleaned) {
    rc = agg_clean_enqueue(h, st, sh);
    if (rc != RW_OK) return rc;
  }
  if (!h->pend_ev[set]) RW_CUDA(cudaEventCreateWithFlags(&h->pend_ev[set], cudaEventDisableTiming));
  RW_CUDA(cudaEventRecord(h->pend_ev[set], st));
  rwgpu_agg::Pending& pd = h->pending[h->n_pending++];
  pd.set = set;
  pd.tag = pub.tag;
  pd.rows_total = h->rows_total;
  pd.mm_charged = h->mm_charged;
  pd.cleaned = cleaned;
  pd.st = st;
  h->flip ^= 1;
  h->epoch_rows = 0;
  h->per_row_mode = false;
  h->nullfree_push_seen = false;
  return RW_OK;
}

// wait for the OLDEST outstanding barrier; its *n_rows rows sit in output set *set
static int agg_flush_collect(rwgpu_agg* h, int64_t* n_rows, unsigned int* has_null_host, int* set) {
  if (h->n_pending == 0) return fail(RW_ERR_INVALID, "no barrier outstanding");
  const rwgpu_agg::Pending pd = h->pending[0];
  h->pending[0] = h->pending[1];
  h->n_pending--;
  RW_CUDA(cudaEventSynchronize(h->pend_ev[pd.set]));
  uint8_t* sh = h->status_host.as<uint8_t>() + 256 * pd.set;
  if (*(volatile unsigned long long*)(sh + 192) != pd.tag) return fail(RW_ERR_CUDA, "internal: barrier status was not published");
  AggStatus* s = (AggStatus*)sh;
  h->groups_upper = s->n_groups + (h->rows_total - pd.rows_total);  // (after a cleaning: the groups it kept)
  if (pd.cleaned && h->n_retract)
    h->mm_upper = std::min<uint64_t>(h->mm_upper, *(volatile unsigned long long*)(sh + 200) + (h->mm_charged - pd.mm_charged));
  *set = pd.set;
  if (s->err) {
    unsigned int e = s->err;
    cudaMemsetAsync(&h->status.as<AggStatus>()->err, 0, sizeof(unsigned int), pd.st);
    return fail(agg_err_code(e), agg_err_msg(e));
  }
  *n_rows = (int64_t)s->out_rows;
  memcpy(has_null_host, sh + 64, sizeof(unsigned int) * (RW_MAX_KEYS + RW_MAX_CALLS));
  return RW_OK;
}

// synchronous barrier: collect whatever is outstanding first (results discarded would be a caller bug: refuse)
static int agg_flush_dev(rwgpu_agg* h, cudaStream_t st, int64_t* n_rows, unsigned int* has_null_host, int* set) {
  if (h->n_pending) return fail(RW_ERR_INVALID, "collect the outstanding asynchronous barriers first");
  int rc = agg_flush_enqueue(h, st);
  if (rc != RW_OK) return rc;
  return agg_flush_collect(h, n_rows, has_null_host, set);
}

// fill `view` with device pointers into output set `set` (validity bitmaps are packed on `st` when a column has NULLs)
static int agg_fill_view(rwgpu_agg* h, int set, int64_t n, const unsigned int* has_null, rw_chunk* view, cudaStream_t st) {
  rwgpu_agg::OutSet& os = h->outs[set];
  h->dev_view_cols.resize(h->out_types.size());
  for (size_t k = 0; k < h->out_types.size(); k++) {
    rw_column& c = h->dev_view_cols[k];
    c.type = h->out_types[k];
    c.reserved = 0;
    c.data = os.col[k].p;
    c.validity = nullptr;
    if (has_null[k] && n > 0) {
      pack_bytes_to_bits_kernel<<<grid_for((n + 63) / 64, 256), 256, 0, st>>>(os.valid[k].as<uint8_t>(), os.bits[k].as<uint64_t>(), n);
      RW_CUDA(cudaGetLastError());
      h->launches++;
      c.validity = os.bits[k].as<uint64_t>();
    }
  }
  view->n_rows = n;
  view->n_cols = (int32_t)h->out_types.size();
  view->reserved = 0;
  view->ops = os.ops.as<uint8_t>();
  view->visibility = nullptr;
  view->columns = h->dev_view_cols.data();
  return RW_OK;
}

extern "C" {

int32_t rwgpu_agg_create(const rw_agg_desc* d, rwgpu_agg** out) {
  if (!d || !out) return fail(RW_ERR_INVALID, "null descriptor");
  int rc = rwgpu_device_check();
  if (rc != RW_OK) return rc;
  if (d->n_group_keys < 1 || d->n_group_keys > RW_MAX_KEYS) return fail(RW_ERR_UNSUPPORTED, "1..4 group key columns supported");
  if (d->n_calls < 1 || d->n_calls > RW_MAX_CALLS) return fail(RW_ERR_UNSUPPORTED, "1..16 agg calls supported");
  if (d->n_input_cols > RW_MAX_COLS) return fail(RW_ERR_UNSUPPORTED, "too many input columns");
  if (d->row_count_index < 0 || d->row_count_index >= d->n_calls) return fail(RW_ERR_INVALID, "row_count_index");
  auto h = new rwgpu_agg();
  std::unique_ptr<rwgpu_agg> guard(h);
  AggPlanDev& p = h->plan;
  memset(&p, 0, sizeof(p));
  h->in_types.assign(d->input_types, d->input_types + d->n_input_cols);
  for (int t : h->in_types) if (!type_supported(t)) return fail(RW_ERR_UNSUPPORTED, "unsupported input type");
  p.n_keys = d->n_group_keys;
  std::vector<bool> used(d->n_input_cols, false);
  for (int k = 0; k < p.n_keys; k++) {
    int c = d->group_key_indices[k];
    if (c < 0 || c >= d->n_input_cols) return fail(RW_ERR_INVALID, "group key index");
    if (h->in_types[c] == RW_T_DECIMAL) return fail(RW_ERR_UNSUPPORTED, "decimal group key");
    if (type_is_varlen(h->in_types[c])) return fail(RW_ERR_UNSUPPORTED, "varlen group key (KeySerialized) stays on the CPU executor");
    p.key_col[k] = c;
    p.key_type[k] = h->in_types[c];
    used[c] = true;
    h->out_types.push_back(h->in_types[c]);
  }
  p.single_key = (p.n_keys == 1);
  p.KW = p.single_key ? 1 : 1 + p.n_keys;
  p.n_calls = d->n_calls;
  int cw = 1 + p.n_calls;
  bool fast = p.single_key && type_width(p.key_type[0]) == 8 && !type_is_float(p.key_type[0]) && p.n_calls <= 4;
  for (int c = 0; c < p.n_calls; c++) {
    const rw_agg_call& call = d->calls[c];
    p.kind[c] = call.kind;
    p.arg_col[c] = call.arg_col;
    p.ret_type[c] = call.ret_type;
    p.hi_off[c] = -1;
    p.prevhi_off[c] = -1;
    p.mm_off[c] = -1;
    int at = 0;
    if (call.arg_col >= 0) {
      if (call.arg_col >= d->n_input_cols) return fail(RW_ERR_INVALID, "agg arg index");
      at = h->in_types[call.arg_col];
      used[call.arg_col] = true;
    }
    p.arg_type[c] = at;
    if (!agg_signature_ok(call.kind, call.arg_col >= 0, at, call.ret_type))
      return fail(RW_ERR_INVALID, "aggregate signature not defined by the reference (general.rs)");
    if (type_is_varlen(at)) return fail(RW_ERR_UNSUPPORTED, "aggregates over varlen arguments stay on the CPU executor");
    switch (call.kind) {
      case RW_AGG_COUNT:
        if (call.arg_col >= 0) fast = false;
        break;
      case RW_AGG_SUM:
      case RW_AGG_SUM0:
        if (at == RW_T_DECIMAL) return fail(RW_ERR_UNSUPPORTED, "sum(decimal) stays on the CPU executor");
        if (!type_is_float(at)) p.hi_off[c] = cw++;  // every integer sum: exact 128-bit state, range-checked at the barrier
        if (call.ret_type == RW_T_DECIMAL) p.prevhi_off[c] = cw++;
        if (at != RW_T_INT64 || call.ret_type != RW_T_INT64) fast = false;
        h->all_flag_mask |= 1u << c;
        break;
      case RW_AGG_MIN:
      case RW_AGG_MAX:
        if (at == RW_T_DECIMAL) return fail(RW_ERR_UNSUPPORTED, "min/max(decimal) stays on the CPU executor");
        if (type_width(at) != 8 || type_is_float(at)) fast = false;
        if (!d->is_append_only) {
          // retractable min/max is a MaterializedInput state (agg_state.rs:49-56, minput.rs): the call's input values
          // are kept as a chained multiset in HBM, the chain head in a cold word of the group
          p.mm_off[c] = cw++;
          h->n_retract++;
          fast = false;
        }
        h->all_flag_mask |= 1u << c;
        break;
      default:
        return fail(RW_ERR_UNSUPPORTED, "agg kind not offloaded");
    }
    h->out_types.push_back(call.ret_type);
  }
  if (d->calls[d->row_count_index].kind != RW_AGG_COUNT || d->calls[d->row_count_index].arg_col >= 0)
    return fail(RW_ERR_INVALID, "row_count_index must name a count(*) call");
  p.HW = p.KW + p.n_calls;
  p.CW = cw;
  p.row_count_call = d->row_count_index;
  p.strict = d->strict_consistency;
  h->fast_eligible = fast;
  h->chunk_size = d->chunk_size > 0 ? d->chunk_size : 1024;
  for (int c = 0; c < d->n_input_cols; c++) if (used[c]) h->used_cols.push_back(c);

  RW_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  uint64_t want = std::max<uint64_t>(d->group_capacity_hint * 2, 1024);
  uint64_t cap = 1024;
  while (cap < want) cap <<= 1;
  h->cap = cap;
  rc = agg_alloc_table(h, cap, h->hot, h->cold, h->dirty, h->dirty_list);
  if (rc != RW_OK) return rc;
  RW_CUDA(h->status.reserve(sizeof(AggStatus)));
  RW_CUDA(cudaMemsetAsync(h->status.p, 0, sizeof(AggStatus), h->stream));
  RW_CUDA(h->out_hasnull.reserve(sizeof(unsigned int) * (RW_MAX_KEYS + RW_MAX_CALLS)));
  RW_CUDA(cudaMemsetAsync(h->out_hasnull.p, 0, sizeof(unsigned int) * (RW_MAX_KEYS + RW_MAX_CALLS), h->stream));
  RW_CUDA(h->mm_next.reserve(8));
  {
    const unsigned long long one = 1;  // record ids start at 1 (0 terminates a chain)
    RW_CUDA(cudaMemcpyAsync(h->mm_next.p, &one, 8, cudaMemcpyHostToDevice, h->stream));
    RW_CUDA(cudaStreamSynchronize(h->stream));
  }
  {
    const AggCleanDev cd0 = {1ull, 0ull};
    RW_CUDA(h->clean_dev.reserve(sizeof(AggCleanDev)));
    RW_CUDA(cudaMemcpy(h->clean_dev.p, &cd0, sizeof(cd0), cudaMemcpyHostToDevice));
  }
  if (h->n_retract) {
    h->mm_cap = std::max<uint64_t>(1 << 16, d->group_capacity_hint * 4);
    RW_CUDA(h->mm_log.reserve((size_t)h->mm_cap * 16));
  }
  RW_CUDA(h->status_host.reserve(512));
  memset(h->status_host.p, 0, 512);
  rc = agg_init_table(h, h->table());
  if (rc != RW_OK) return rc;
  // staging layout: [ops | per used column: data, valid bytes], 256-byte aligned regions
  size_t off = 0;
  h->off_ops = off; off = align_up(off + (size_t)h->stage_cap, 256);
  for (int c : h->used_cols) {
    h->off_data[c] = off; off = align_up(off + (size_t)h->stage_cap * type_width(h->in_types[c]), 256);
    h->off_valid[c] = off; off = align_up(off + (size_t)h->stage_cap, 256);
  }
  h->stage_bytes = off;
  RW_CUDA(cudaStreamSynchronize(h->stream));
  *out = guard.release();
  return RW_OK;
}

void rwgpu_agg_destroy(rwgpu_agg* h) {
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

static int agg_stage_init(rwgpu_agg* h) {
  for (auto& s : h->stage) {
    if (s.host.p) continue;
    RW_CUDA(s.host.reserve(h->stage_bytes));
    RW_CUDA(s.dev.reserve(h->stage_bytes));
    RW_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    s.rows = 0;
    s.in_flight = false;
    memset(s.has_valid, 0, sizeof(s.has_valid));
  }
  return RW_OK;
}

int32_t rwgpu_agg_push(rwgpu_agg* h, const rw_chunk* c) {
  if (!h || !c) return fail(RW_ERR_INVALID, "null");
  if (c->n_cols != (int)h->in_types.size()) return fail(RW_ERR_INVALID, "chunk schema mismatch");
  for (int k = 0; k < c->n_cols; k++)
    if (c->columns[k].type != h->in_types[k]) return fail(RW_ERR_INVALID, "chunk column type mismatch");
  int rc = agg_stage_init(h);
  if (rc != RW_OK) return rc;
  int64_t done = 0;
  while (done < c->n_rows) {
    AggStage& s = h->stage[h->cur];
    int64_t m = std::min<int64_t>(c->n_rows - done, h->stage_cap - s.rows);
    uint8_t* hp = s.host.as<uint8_t>();
    uint8_t* ops = hp + h->off_ops + s.rows;
    if (c->visibility == nullptr) {
      memcpy(ops, c->ops + done, (size_t)m);
    } else {
      for (int64_t i = 0; i < m; i++) {
        int64_t r = done + i;
        ops[i] = ((c->visibility[r >> 6] >> (r & 63)) & 1) ? c->ops[r] : 0;
      }
    }
    for (int col : h->used_cols) {
      int w = type_width(h->in_types[col]);
      memcpy(hp + h->off_data[col] + (size_t)s.rows * w, (const uint8_t*)c->columns[col].data + (size_t)done * w, (size_t)m * w);
      const uint64_t* vb = c->columns[col].validity;
      uint8_t* vdst = hp + h->off_valid[col];
      if (vb) {
        if (!s.has_valid[col]) { memset(vdst, 1, (size_t)s.rows); s.has_valid[col] = true; }
        for (int64_t i = 0; i < m; i++) {
          int64_t r = done + i;
          vdst[s.rows + i] = (uint8_t)((vb[r >> 6] >> (r & 63)) & 1);
        }
      } else if (s.has_valid[col]) {
        memset(vdst + s.rows, 1, (size_t)m);
      }
    }
    s.rows += m;
    done += m;
    if (s.rows == h->stage_cap) {
      rc = agg_launch_stage(h);
      if (rc != RW_OK) return rc;
    }
  }
  return RW_OK;
}

int32_t rwgpu_agg_push_device(rwgpu_agg* h, const rw_chunk* c, void* cuda_stream) {
  return rwgpu_agg_push_device_counted(h, c, nullptr, cuda_stream);
}

int32_t rwgpu_agg_push_device_counted(rwgpu_agg* h, const rw_chunk* c, const int64_t* n_rows_dev, void* cuda_stream) {
  if (!h || !c) return fail(RW_ERR_INVALID, "null");
  if (c->n_cols != (int)h->in_types.size()) return fail(RW_ERR_INVALID, "chunk schema mismatch");
  DevChunk ch;
  int rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  ch.n_dev = n_rows_dev;
  rc = agg_launch_stage(h);  // keep host-staged rows ordered before this chunk
  if (rc != RW_OK) return rc;
  return agg_apply_dev(h, ch, cuda_stream ? (cudaStream_t)cuda_stream : h->stream);
}

int32_t rwgpu_agg_flush(rwgpu_agg* h, uint64_t /*epoch*/, rwgpu_out** out) {
  if (!h || !out) return fail(RW_ERR_INVALID, "null");
  int64_t n = 0;
  unsigned int has_null[RW_MAX_KEYS + RW_MAX_CALLS];
  int set = 0;
  int rc = agg_flush_dev(h, h->stream, &n, has_null, &set);
  if (rc != RW_OK) return rc;
  rwgpu_agg::OutSet& os = h->outs[set];
  auto o = new rwgpu_out();
  o->chunk_size = h->chunk_size;
  unsigned long long nullm = 0;
  for (size_t k = 0; k < h->out_types.size(); k++) if (has_null[k]) nullm |= 1ull << k;
  if (!o->layout(n, h->out_types, nullm, false, h->pool)) { delete o; return fail(RW_ERR_OOM, "pinned output block"); }
  if (n > 0) {
    cudaMemcpyAsync(o->ops, os.ops.p, (size_t)n, cudaMemcpyDeviceToHost, h->stream);
    for (size_t k = 0; k < h->out_types.size(); k++) {
      size_t w = type_width(h->out_types[k]);
      cudaMemcpyAsync(o->data[k], os.col[k].p, (size_t)n * w, cudaMemcpyDeviceToHost, h->stream);
      if (o->valid_bytes[k]) cudaMemcpyAsync(o->valid_bytes[k], os.valid[k].p, (size_t)n, cudaMemcpyDeviceToHost, h->stream);
    }
    cudaError_t e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) { delete o; return fail(RW_ERR_CUDA, cudaGetErrorString(e)); }
  }
  o->finalize();
  *out = o;
  return RW_OK;
}

int32_t rwgpu_agg_flush_device(rwgpu_agg* h, uint64_t /*epoch*/, rw_chunk* view, void* cuda_stream) {
  if (!h || !view) return fail(RW_ERR_INVALID, "null");
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->stream;
  int64_t n = 0;
  unsigned int has_null[RW_MAX_KEYS + RW_MAX_CALLS];
  int set = 0;
  int rc = agg_flush_dev(h, st, &n, has_null, &set);
  if (rc != RW_OK) return rc;
  return agg_fill_view(h, set, n, has_null, view, st);
}

int32_t rwgpu_agg_flush_device_async(rwgpu_agg* h, uint64_t /*epoch*/, void* cuda_stream) {
  if (!h) return fail(RW_ERR_INVALID, "null");
  return agg_flush_enqueue(h, cuda_stream ? (cudaStream_t)cuda_stream : h->stream);
}

int32_t rwgpu_agg_flush_collect(rwgpu_agg* h, rw_chunk* view, void* cuda_stream) {
  if (!h || !view) return fail(RW_ERR_INVALID, "null");
  int64_t n = 0;
  unsigned int has_null[RW_MAX_KEYS + RW_MAX_CALLS];
  int set = 0;
  int rc = agg_flush_collect(h, &n, has_null, &set);
  if (rc != RW_OK) return rc;
  return agg_fill_view(h, set, n, has_null, view, cuda_stream ? (cudaStream_t)cuda_stream : h->stream);
}

// ---- state persistence: see the comment above agg_snapshot_kernel
int32_t rwgpu_agg_snapshot(rwgpu_agg* h, rwgpu_out** states, rwgpu_out** minput) {
  if (!h || !states || !minput) return fail(RW_ERR_INVALID, "null");
  if (h->n_pending || h->epoch_rows || h->stage[h->cur].rows) return fail(RW_ERR_INVALID, "snapshot between a barrier and the next push only");
  RW_CUDA(cudaDeviceSynchronize());
  const AggPlanDev& p = h->plan;
  const int n_out = (int)h->out_types.size();
  DevBuf counters;
  RW_CUDA(counters.reserve(256));
  RW_CUDA(cudaMemset(counters.p, 0, 256));
  AggSnapOut o;
  memset(&o, 0, sizeof(o));
  o.n_rows = counters.as<unsigned long long>();
  o.m_rows = o.n_rows + 1;
  o.has_null = (unsigned int*)(o.n_rows + 2);
  const int g = grid_for((int64_t)h->cap + 2, 256);
  agg_snapshot_kernel<<<g, 256, 0, h->stream>>>(h->table(), p, o, 1);  // pass 1: sizes
  RW_CUDA(cudaGetLastError());
  unsigned long long cnt[2] = {0, 0};
  RW_CUDA(cudaMemcpyAsync(cnt, counters.p, 16, cudaMemcpyDeviceToHost, h->stream));
  RW_CUDA(cudaStreamSynchronize(h->stream));
  const int64_t n = (int64_t)cnt[0], nm = (int64_t)cnt[1];
  // device staging: columns + valid bytes
  std::vector<DevBuf> col(n_out), val(n_out), mcol(p.n_keys + 2), mval(p.n_keys);
  for (int k = 0; k < n_out; k++) {
    RW_CUDA(col[k].reserve((size_t)std::max<int64_t>(n, 1) * type_width(h->out_types[k])));
    RW_CUDA(val[k].reserve((size_t)std::max<int64_t>(n, 1)));
    o.col[k] = col[k].p;
    o.valid[k] = val[k].as<uint8_t>();
  }
  std::vector<int> mtypes;
  for (int k = 0; k < p.n_keys; k++) mtypes.push_back(p.key_type[k]);
  mtypes.push_back(RW_T_INT32);
  mtypes.push_back(RW_T_INT64);
  for (int k = 0; k < p.n_keys + 2; k++) {
    RW_CUDA(mcol[k].reserve((size_t)std::max<int64_t>(nm, 1) * type_width(mtypes[k])));
    o.mcol[k] = mcol[k].p;
  }
  for (int k = 0; k < p.n_keys; k++) {
    RW_CUDA(mval[k].reserve((size_t)std::max<int64_t>(nm, 1)));
    o.mvalid[k] = mval[k].as<uint8_t>();
  }
  o.capacity = n;
  o.m_capacity = nm;
  RW_CUDA(cudaMemsetAsync(counters.p, 0, 256, h->stream));
  agg_snapshot_kernel<<<g, 256, 0, h->stream>>>(h->table(), p, o, 0);  // pass 2: rows
  RW_CUDA(cudaGetLastError());
  h->launches += 2;
  unsigned int has_null[RW_MAX_KEYS + RW_MAX_CALLS];
  RW_CUDA(cudaMemcpyAsync(has_null, o.has_null, sizeof(has_null), cudaMemcpyDeviceToHost, h->stream));
  RW_CUDA(cudaStreamSynchronize(h->stream));
  auto to_host = [&](int64_t rows, const std::vector<int>& types, std::vector<DevBuf>& cols, std::vector<DevBuf>& vals, const unsigned int* hn,
                     int n_valid, rwgpu_out** out) -> int {
    auto ro = new rwgpu_out();
    ro->chunk_size = h->chunk_size;
    unsigned long long nullm = 0;
    for (int k = 0; k < n_valid; k++) if (hn[k]) nullm |= 1ull << k;
    if (!ro->layout(rows, types, nullm, false, h->pool)) { delete ro; return fail(RW_ERR_OOM, "pinned output block"); }
    if (rows > 0) {
      memset(ro->ops, RW_OP_INSERT, (size_t)rows);
      for (size_t k = 0; k < types.size(); k++) {
        cudaMemcpyAsync(ro->data[k], cols[k].p, (size_t)rows * type_width(types[k]), cudaMemcpyDeviceToHost, h->stream);
        if (ro->valid_bytes[k]) cudaMemcpyAsync(ro->valid_bytes[k], vals[k].p, (size_t)rows, cudaMemcpyDeviceToHost, h->stream);
      }
      cudaError_t e = cudaStreamSynchronize(h->stream);
      if (e != cudaSuccess) { delete ro; return fail(RW_ERR_CUDA, cudaGetErrorString(e)); }
    }
    ro->finalize();
    *out = ro;
    return RW_OK;
  };
  int rc = to_host(n, h->out_types, col, val, has_null, n_out, states);
  if (rc != RW_OK) return rc;
  // (NULL group keys of the materialized input: flagged through the same key-column flags)
  rc = to_host(nm, mtypes, mcol, mval, has_null, p.n_keys, minput);
  if (rc != RW_OK) { rwgpu_out_release(*states); *states = nullptr; return rc; }
  return RW_OK;
}

int32_t rwgpu_agg_restore(rwgpu_agg* h, const rw_chunk* states, const rw_chunk* minput) {
  if (!h || !states) return fail(RW_ERR_INVALID, "null");
  if (h->n_pending || h->epoch_rows || h->stage[h->cur].rows) return fail(RW_ERR_INVALID, "restore into an idle operator only");
  const AggPlanDev& p = h->plan;
  if (states->n_cols != (int)h->out_types.size()) return fail(RW_ERR_INVALID, "state rows: group key columns followed by one state column per call");
  for (int k = 0; k < states->n_cols; k++)
    if (states->columns[k].type != h->out_types[k]) return fail(RW_ERR_INVALID, "state rows: column type mismatch");
  if (minput && minput->n_rows > 0) {
    if (!h->n_retract) return fail(RW_ERR_INVALID, "materialized-input rows for a plan without retractable min/max");
    bool ok = minput->n_cols == p.n_keys + 2 && minput->columns[p.n_keys].type == RW_T_INT32 && minput->columns[p.n_keys + 1].type == RW_T_INT64;
    for (int k = 0; ok && k < p.n_keys; k++) ok = minput->columns[k].type == p.key_type[k];
    if (!ok) return fail(RW_ERR_INVALID, "materialized-input rows: group key columns, int4 call index, int8 value");
  }
  int rc = agg_ensure_capacity(h, (uint64_t)states->n_rows);
  if (rc != RW_OK) return rc;
  if (states->n_rows > 0) {
    DevBuf buf;
    DevChunk ch;
    rc = upload_chunk(states, buf, &ch, h->stream);
    if (rc != RW_OK) return rc;
    agg_restore_kernel<<<grid_for(ch.n, 256), 256, 0, h->stream>>>(h->table(), p, ch);
    RW_CUDA(cudaGetLastError());
    h->launches++;
    RW_CUDA(cudaStreamSynchronize(h->stream));
    h->groups_upper += (uint64_t)states->n_rows;
  }
  if (minput && minput->n_rows > 0) {
    const uint64_t need = h->mm_upper + (uint64_t)minput->n_rows;
    if (need > h->mm_cap) {
      RW_CUDA(cudaDeviceSynchronize());
      unsigned long long used = 1;
      RW_CUDA(cudaMemcpy(&used, h->mm_next.p, 8, cudaMemcpyDeviceToHost));
      uint64_t ncap = std::max<uint64_t>(h->mm_cap * 2, used + (uint64_t)minput->n_rows * 2);
      DevBuf nl;
      RW_CUDA(nl.reserve((size_t)ncap * 16));
      RW_CUDA(cudaMemcpy(nl.p, h->mm_log.p, (size_t)used * 16, cudaMemcpyDeviceToDevice));
      h->mm_log = std::move(nl);
      h->mm_cap = ncap;
    }
    h->mm_upper += (uint64_t)minput->n_rows;
    DevBuf buf;
    DevChunk ch;
    rc = upload_chunk(minput, buf, &ch, h->stream);
    if (rc != RW_OK) return rc;
    agg_restore_minput_kernel<<<grid_for(ch.n, 256), 256, 0, h->stream>>>(h->table(), p, ch);
    RW_CUDA(cudaGetLastError());
    h->launches++;
    RW_CUDA(cudaStreamSynchronize(h->stream));
  }
  AggStatus st;
  RW_CUDA(cudaMemcpy(&st, h->status.p, sizeof(st), cudaMemcpyDeviceToHost));
  if (st.err) {
    cudaMemset(&h->status.as<AggStatus>()->err, 0, sizeof(unsigned int));
    return fail(agg_err_code(st.err), agg_err_msg(st.err));
  }
  return RW_OK;
}

int32_t rwgpu_agg_profile(rwgpu_agg* h, int32_t enable, double* ms, uint64_t* launches) {
  if (!h) return fail(RW_ERR_INVALID, "null");
  RW_CUDA(cudaDeviceSynchronize());
  h->prof.collect();
  if (ms) *ms = h->prof.ms;
  if (launches) *launches = h->prof.n;
  h->prof.ms = 0;
  h->prof.n = 0;
  h->prof.on = enable != 0;
  return RW_OK;
}

int32_t rwgpu_agg_update_watermark(rwgpu_agg* h, int32_t key_pos, int64_t value) {
  if (!h) return fail(RW_ERR_INVALID, "null");
  if (key_pos < 0 || key_pos >= h->plan.n_keys) return fail(RW_ERR_INVALID, "group key position");
  const int t = h->plan.key_type[key_pos];
  if (type_is_float(t) || t == RW_T_BOOL || t == RW_T_DECIMAL)
    return fail(RW_ERR_UNSUPPORTED, "watermarks on this key type keep the state (CPU semantics unchanged)");
  // a later watermark on the same key only moves up
  if (!h->wm_pending || value > h->wm_value || key_pos != h->wm_key_pos) {
    h->wm_pending = true;
    h->wm_key_pos = key_pos;
    h->wm_value = value;
  }
  return RW_OK;
}

int32_t rwgpu_agg_value_log_stats(rwgpu_agg* h, uint64_t* records_in_use, uint64_t* compactions) {
  if (!h) return fail(RW_ERR_INVALID, "null");
  RW_CUDA(cudaDeviceSynchronize());
  unsigned long long next = 1;
  AggCleanDev cd;
  RW_CUDA(cudaMemcpy(&next, h->mm_next.p, 8, cudaMemcpyDeviceToHost));
  RW_CUDA(cudaMemcpy(&cd, h->clean_dev.p, sizeof(cd), cudaMemcpyDeviceToHost));
  if (records_in_use) *records_in_use = next - 1;
  if (compactions) *compactions = cd.compactions;
  return RW_OK;
}

int32_t rwgpu_agg_stats(rwgpu_agg* h, uint64_t* n_groups, uint64_t* capacity, uint64_t* launches) {
  if (!h) return fail(RW_ERR_INVALID, "null");
  AggStatus s;
  RW_CUDA(cudaStreamSynchronize(h->stream));
  RW_CUDA(cudaMemcpy(&s, h->status.p, sizeof(s), cudaMemcpyDeviceToHost));
  if (n_groups) *n_groups = s.n_groups;
  if (capacity) *capacity = h->cap;
  if (launches) *launches = h->launches;
  return RW_OK;
}

}  // extern "C"
