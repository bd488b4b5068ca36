// join_uni.cuh -- ONE hash table for both sides of a Key64 inner join (included by join.cu).
//
// The two-table inner kernels (join.cu) are bound by the NUMBER of random 64-byte DRAM transactions per
// row -- probe line of the other side, own-side line read by the claiming CAS, own-side write-back.  Here a
// join key owns ONE 64-byte bucket that carries the state of BOTH sides, so a row's probe and its own-side
// insert touch the SAME line: one random read + one write-back per row, everything else is sequential.
//
//   bucket (64 B, linear probing bucket by bucket, load <= 1 / U_LOAD_INV = 0.25):
//     +0   key                 J_EMPTY = free
//     +8   WI   inline side:   overflow head (31) | inline state (2) | live rows (31)      (as in join.cu)
//     +16  IH   inline record: null mask (8 bits) | seq << 8
//     +24  WC   chained side:  u32 head of the row chain | u32 live rows
//     +32  the INLINE SIDE's first live row of this key (4 x 8 B columns)
//   inline side IS  = the side whose stream key is inside the join key (at most one live row per key:
//                     the auction side of bid x auction), else the right side.  Its 2nd, 3rd ... row of
//                     a key goes to log[IS], chained from WI.head.
//   chained side CS = the other one.  EVERY row is appended to log[CS] -- a sequential write: the 8 rows a
//                     warp handles per iteration take consecutive ids from the warp's pool -- and pushed
//                     on the key's chain with one 64-bit atomicExch of WC = new head | loaded count + 1 (no CAS
//                     loop: hot keys serialise in L2 only; a RED corrects the count when the key was contended,
//                     uni_chain_push), on the line the probe just loaded.
//   log record (48 B): u32 link | DEAD, u32 null mask, u64 seq, 4 x 8 B columns.
//
// A CS row (bid) therefore costs: one random 64 B read (key, WI, the matched auction row), one L2 atomic on
// that line (one 32/64 B write-back), 48 B appended to the log, 33 B read and 65 B written sequentially.
// An IS row (auction) reads its bucket, walks the CS chain for matches, and claims the inline record.
#pragma once
#include <cooperative_groups.h>

namespace rw {

#define U_NIL 0x7fffffffu
#define U_XCHUNK 64  // extra-match output rows a warp reserves at a time
// blocks of JF_BLOCK threads of uni_hot_kernel, one resident wave (__launch_bounds__(JF_BLOCK, 4)); one id pool per warp
// and side
#define U_MAX_GRID (RW_SMS * 4)
// The bucket array holds at most cap / U_LOAD_INV keys (create-time sizing and uni_grow_table).  At 1/4 (load about 0.15
// at the create-time hint) a key takes ~1.09 bucket probes instead of ~1.21 at 1/2, and about half the warp iterations
// wait on a second probe round instead of 85 %; the bucket array is twice as large (64 B x 2^26 = 4 GiB for 10 M keys).
#define U_LOAD_INV 4

// A side's log is a list of fixed-size SEGMENTS (2^22 records = 192 MiB each) reached through a small device table of
// segment pointers: growing the log allocates one more segment and appends its pointer -- no copy of the existing
// hundreds of megabytes in the middle of the stream (as allocate + copy + free of the whole store would), no
// contiguous virtual range.  Record id -> segment id >> 22, offset (id & 2^22-1) * 48.
#define U_SEG_SHIFT 22
#define U_SEG_RECS (1u << U_SEG_SHIFT)
#define U_MAX_SEGS 512
struct UniDev {
  uint8_t* buckets;   // (cap + 2) x 64 B; slot cap = NULL key (null-safe equality), cap + 1 = the key equal to J_EMPTY
  uint64_t cap;       // power of two
  uint8_t* const* log[2];  // segment tables
  uint64_t log_cap[2];
  uint2* pools[2];                  // per-warp id pools {next, end}, persistent across launches
  unsigned long long* log_next[2];  // ids handed out per side (device counters, absolute)
  unsigned long long* n_dead[2];    // dead log records per side (compaction trigger)
  int is;                           // inline side
};

struct UniRec {
  uint32_t link, nullmask;
  uint64_t seq;
  uint64_t c[4];
};
static_assert(sizeof(UniRec) == 48, "log record");

__device__ __forceinline__ uint8_t* ub(const UniDev& t, int64_t b) { return t.buckets + (uint64_t)b * 64; }
__device__ __forceinline__ unsigned long long* ub_WI(const UniDev& t, int64_t b) { return (unsigned long long*)(ub(t, b) + 8); }
__device__ __forceinline__ unsigned long long* ub_IH(const UniDev& t, int64_t b) { return (unsigned long long*)(ub(t, b) + 16); }
__device__ __forceinline__ uint32_t* ub_chead(const UniDev& t, int64_t b) { return (uint32_t*)(ub(t, b) + 24); }
__device__ __forceinline__ uint32_t* ub_ccount(const UniDev& t, int64_t b) { return (uint32_t*)(ub(t, b) + 28); }
__device__ __forceinline__ uint64_t* ub_cols(const UniDev& t, int64_t b) { return (uint64_t*)(ub(t, b) + 32); }
__device__ __forceinline__ uint8_t* useg_rec(uint8_t* const* segs, uint32_t id) {
  const unsigned long long base = __ldg((const unsigned long long*)segs + (id >> U_SEG_SHIFT));
  return (uint8_t*)(base + (unsigned long long)(id & (U_SEG_RECS - 1u)) * 48ull);
}
__device__ __forceinline__ UniRec* urec(const UniDev& t, int side, uint32_t id) { return (UniRec*)useg_rec(t.log[side], id); }
__device__ __forceinline__ uint64_t uhome(uint64_t key, uint64_t mask) { return mix64(key) & mask; }

__device__ __forceinline__ uint64_t shfl64m(unsigned mask, uint64_t v, int src) {
  return (uint64_t)__shfl_sync(mask, (unsigned long long)v, src);
}

__global__ void uni_init_kernel(uint8_t* buckets, uint64_t from, uint64_t to) {
  for (uint64_t i = from + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < to; i += (uint64_t)gridDim.x * blockDim.x) {
    ulonglong2* s = (ulonglong2*)(buckets + i * 64);
    s[0] = make_ulonglong2(J_EMPTY, W_EMPTY);
    s[1] = make_ulonglong2(0ull, (unsigned long long)U_NIL);  // IH = 0; WC: head NIL, count 0
    s[2] = make_ulonglong2(0ull, 0ull);
    s[3] = make_ulonglong2(0ull, 0ull);
  }
}

// read-only lookup; -1 = absent
__device__ __forceinline__ int64_t uni_find(const UniDev& t, uint64_t key, bool knull) {
  if (knull) return (int64_t)t.cap;
  if (key == J_EMPTY) return (int64_t)t.cap + 1;
  const uint64_t mask = t.cap - 1;
  uint64_t idx = uhome(key, mask);
  while (true) {
    const unsigned long long k = __ldcg((const unsigned long long*)ub(t, (int64_t)idx));
    if (k == key) return (int64_t)idx;
    if (k == J_EMPTY) return -1;
    idx = (idx + 1) & mask;
  }
}
__device__ __forceinline__ int64_t uni_find_or_claim(const UniDev& t, uint64_t key, bool knull, bool* created) {
  if (knull) return (int64_t)t.cap;
  if (key == J_EMPTY) return (int64_t)t.cap + 1;
  const uint64_t mask = t.cap - 1;
  uint64_t idx = uhome(key, mask);
  while (true) {
    unsigned long long* kp = (unsigned long long*)ub(t, (int64_t)idx);
    unsigned long long k = __ldcg(kp);
    if (k == J_EMPTY) {
      k = atomicCAS(kp, (unsigned long long)J_EMPTY, (unsigned long long)key);
      if (k == J_EMPTY) { *created = true; return (int64_t)idx; }
    }
    if (k == key) return (int64_t)idx;
    idx = (idx + 1) & mask;
  }
}

// one output row: update-side columns from the chunk (NULL-aware), matched columns from a stored row
__device__ __forceinline__ void uni_emit(const JoinOutDev& o, const W8Plan& w, JoinStatus* st, int64_t at, uint8_t op, const DevChunk& ch,
                                         int64_t r, const uint64_t* mc, uint32_t mnull) {
  o.ops[at] = op;
  unsigned long long nullbits = 0;
#pragma unroll
  for (int c = 0; c < 4; c++) {
    if (c < w.n_u && w.u_out[c] >= 0) {
      const int oc = w.u_out[c];
      if (col_is_null(ch.cols[c], r)) { o.valid[oc][at] = 0; nullbits |= 1ull << oc; }
      else ((uint64_t*)o.col[oc])[at] = ((const uint64_t*)ch.cols[c].data)[r];
    }
    if (c < w.n_m && w.m_out[c] >= 0) {
      const int oc = w.m_out[c];
      if ((mnull >> c) & 1u) { o.valid[oc][at] = 0; nullbits |= 1ull << oc; }
      else ((uint64_t*)o.col[oc])[at] = mc[c];
    }
  }
  if (nullbits) atomicOr(&st->null_mask, nullbits);
}

// emit the `cnt` matches of chunk row r found in bucket b: one at the positional row `pos`, the others at
// xpos, xpos + 1, ...  (S = side of the chunk row).  The positional row gets the live match that ARRIVED LAST (largest
// arrival number): the positional rows of a U- / U+ pair are adjacent, so that match's pair is the one the no-op pass
// hides, and it must not depend on the order in which concurrent inserts linked the chain.  Rows are pushed at the chain's
// head, so the walk usually meets the last arrival first; when concurrent inserts of one chunk linked out of order, the
// two rows are swapped at the end (matches are kept as references and re-read for the swap: holding their columns
// doubled the kernels' registers).
__device__ __forceinline__ void uni_emit_matches(const UniDev& t, const W8Plan& w, int S, const DevChunk& ch, int64_t r, uint8_t oop, int64_t b,
                                                 uint32_t cnt, const JoinOutDev& o, JoinStatus* st, int64_t pos, int64_t xpos) {
  const uint64_t SEQ56 = (1ull << 56) - 1;
  const uint32_t IL = 0xffffffffu;  // reference to the bucket's inline record (log ids are < 2^31)
  const int mside = S != t.is ? t.is : 1 - t.is;
  // one match: columns + null mask of the inline record or of log record m
  auto load = [&](uint32_t m, uint64_t* mc, uint32_t* nm) {
    const uint8_t* base = m == IL ? ub(t, b) + 32 : (const uint8_t*)urec(t, mside, m) + 16;
    const ulonglong2 c01 = __ldcg((const ulonglong2*)base), c23 = __ldcg((const ulonglong2*)base + 1);
    mc[0] = c01.x; mc[1] = c01.y; mc[2] = c23.x; mc[3] = c23.y;
    *nm = m == IL ? (uint32_t)(__ldcg(ub_IH(t, b)) & 0xffull) : __ldcg(&urec(t, mside, m)->nullmask);
  };
  uint32_t left = cnt, pos_ref = U_NIL, best_ref = U_NIL;
  uint64_t best_seq = 0;
  int64_t best_at = pos;
  auto put = [&](uint32_t m, uint64_t seq) {
    int64_t at = pos;
    if (pos_ref == U_NIL) {
      pos_ref = m;
      best_seq = seq;
    } else {
      at = xpos++;
      o.vis[at] = 1;
      if (seq > best_seq) { best_seq = seq; best_ref = m; best_at = at; }
    }
    uint64_t mc[4];
    uint32_t nm;
    load(m, mc, &nm);
    uni_emit(o, w, st, at, oop, ch, r, mc, nm);
  };
  uint32_t m;
  if (S != t.is) {  // matches are the inline side's rows: the bucket's inline record, then the WI chain
    const unsigned long long WI = __ldcg(ub_WI(t, b));
    if (W_istate(WI) == 1u) {
      put(IL, (__ldcg(ub_IH(t, b)) >> 8) & SEQ56);
      left--;
    }
    m = W_head(WI);
  } else {
    m = __ldcg(ub_chead(t, b));
  }
  while (m != U_NIL && left) {
    const ulonglong2 h0 = __ldcg((const ulonglong2*)urec(t, mside, m));  // link | nullmask, seq
    const uint32_t lk = (uint32_t)h0.x;
    if (!(lk & J_DEAD)) {
      put(m, h0.y & SEQ56);
      left--;
    }
    m = lk & 0x7fffffffu;
  }
  if (best_at != pos) {  // the last arrival goes to the positional row, the row that was there takes its place
    uint64_t mc[4];
    uint32_t pos_nm, best_nm;
    load(pos_ref, mc, &pos_nm);
    load(best_ref, mc, &best_nm);
    for (int c = 0; c < 4; c++) {  // (uni_emit only clears valid bytes: set back the ones the first emission cleared)
      if (c >= w.n_m || w.m_out[c] < 0) continue;
      if ((pos_nm >> c) & 1u) o.valid[w.m_out[c]][pos] = 1;
      if ((best_nm >> c) & 1u) o.valid[w.m_out[c]][best_at] = 1;
    }
    uni_emit(o, w, st, pos, oop, ch, r, mc, best_nm);
    load(pos_ref, mc, &pos_nm);
    uni_emit(o, w, st, best_at, oop, ch, r, mc, pos_nm);
  }
}

// null mask of chunk row r over the side's columns
__device__ __forceinline__ uint32_t uni_row_nullmask(const DevChunk& ch, int n_cols, int64_t r) {
  uint32_t nm = 0;
  for (int c = 0; c < n_cols; c++)
    if (col_is_null(ch.cols[c], r)) nm |= 1u << c;
  return nm;
}

// one id from the side's log without a pool (slow paths only: one atomic on a shared counter)
__device__ __forceinline__ uint32_t uni_alloc_one(const UniDev& t, int S, JoinStatus* st) {
  const unsigned long long id = atomicAdd(t.log_next[S], 1ull);
  if (id >= t.log_cap[S]) { atomicOr(&st->err, JERR_STORE_CAPACITY); return U_NIL; }
  return (uint32_t)id;
}

// Pushes log record `row` on a key's chained-side chain and returns the old head, the record's link.  WC = head | count << 32
// is one aligned 8-byte word, so ONE 64-bit exchange writes both the new head and the count the caller expects, L + 1, where
// L is the count the caller loaded with the bucket.  The exchange returns the count C it replaced; if another push or a
// delete of the key moved the count since that load (C != L), C - L (mod 2^32) is added back.  Every other operation on the
// count during a launch is an addition too (the correction, a delete's atomicSub), and in the order the atomics take effect
// the exchange adds L + 1 - C: whatever the interleaving, the count after the launch is its old value plus the rows pushed
// minus the rows deleted.  The head and the links come out as with an exchange of the head alone.  An uncontended push
// costs one atomic; a push on a contended key costs two, as a separate head exchange and count increment always did.
__device__ __forceinline__ uint32_t uni_chain_push(unsigned long long* wc, uint32_t row, uint32_t L) {
  const unsigned long long old = atomicExch(wc, (unsigned long long)row | ((unsigned long long)(L + 1u) << 32));
  const uint32_t C = (uint32_t)(old >> 32);
  if (C != L) atomicAdd((uint32_t*)wc + 1, C - L);
  return (uint32_t)old;
}

// own-side append of chunk row r to bucket b, by ONE thread (slow paths).  rid = a pre-allocated log id or U_NIL.
__device__ __forceinline__ void uni_insert_row(const UniDev& t, int S, const DevChunk& ch, int n_cols, int64_t r, int64_t b, uint64_t seq,
                                               JoinStatus* st) {
  const uint32_t nm = uni_row_nullmask(ch, n_cols, r);
  uint64_t c[4] = {0, 0, 0, 0};
  for (int k = 0; k < n_cols; k++)
    if (!((nm >> k) & 1u)) c[k] = ((const uint64_t*)ch.cols[k].data)[r];
  if (S == t.is) {
    if (w_claim_inline(ub_WI(t, b))) {
      *ub_IH(t, b) = (unsigned long long)nm | (seq << 8);
      uint64_t* d = ub_cols(t, b);
      d[0] = c[0]; d[1] = c[1]; d[2] = c[2]; d[3] = c[3];
      return;
    }
    const uint32_t rid = uni_alloc_one(t, S, st);
    if (rid == U_NIL) return;
    const uint32_t old = w_push_overflow(ub_WI(t, b), rid);
    UniRec* rec = urec(t, S, rid);
    rec->link = old; rec->nullmask = nm; rec->seq = seq;
    rec->c[0] = c[0]; rec->c[1] = c[1]; rec->c[2] = c[2]; rec->c[3] = c[3];
  } else {
    const uint32_t rid = uni_alloc_one(t, S, st);
    if (rid == U_NIL) return;
    unsigned long long* wc = (unsigned long long*)ub_chead(t, b);
    const uint32_t old = uni_chain_push(wc, rid, (uint32_t)(__ldcg(wc) >> 32));
    UniRec* rec = urec(t, S, rid);
    rec->link = old; rec->nullmask = nm; rec->seq = seq;
    rec->c[0] = c[0]; rec->c[1] = c[1]; rec->c[2] = c[2]; rec->c[3] = c[3];
  }
}

// a whole row by ONE thread: key rules, bucket lookup / claim, probe + emit, own-side append.
// (chunks with bitmaps, the sentinel key, NULL keys; hash_join.rs:985-999 for the never-match rule)
template <bool PROBE_ONLY>
__device__ __forceinline__ void uni_row_generic(const JoinPlanDev* p, const W8Plan& w, int S, const DevChunk& ch, int64_t r, uint8_t op,
                                                const UniDev& t, const JoinOutDev& o, JoinStatus* st, uint64_t seq, int64_t pos, int64_t xarea,
                                                unsigned& new_keys, bool& any_match, bool& any_hole) {
  const bool ins = (op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT);
  const ColRef& kc = ch.cols[w.key_col];
  const bool knull = col_is_null(kc, r);
  if (knull && !p->null_safe[0]) {  // never matches, never stored
    o.vis[pos] = 0;
    any_hole = true;
    return;
  }
  const uint64_t key = knull ? 0ull : ((const uint64_t*)kc.data)[r];
  bool created = false;
  const int64_t b = (PROBE_ONLY || !ins) ? uni_find(t, key, knull) : uni_find_or_claim(t, key, knull, &created);
  if (created) new_keys++;
  uint32_t cnt = 0;
  if (b >= 0) cnt = (S != t.is) ? W_count(__ldcg(ub_WI(t, b))) : __ldcg(ub_ccount(t, b));
  if (cnt == 0) {
    o.vis[pos] = 0;
    any_hole = true;
  } else {
    any_match = true;
    o.vis[pos] = 1;
    int64_t xpos = 0;
    if (cnt > 1) {
      xpos = xarea + (int64_t)atomicAdd(&st->out_rows, (unsigned long long)(cnt - 1));
      if (xpos + (cnt - 1) > o.capacity) { atomicOr(&st->err, JERR_OUT_CAPACITY); cnt = 1; }
    }
    uni_emit_matches(t, w, S, ch, r, ins ? RW_OP_INSERT : RW_OP_DELETE, b, cnt, o, st, pos, xpos);
  }
  if (!PROBE_ONLY && ins) uni_insert_row(t, S, ch, w.n_u, r, b, seq, st);
}

// thread-per-row kernel for chunks that carry validity / visibility bitmaps
template <bool PROBE_ONLY>
__global__ void __launch_bounds__(256) uni_slow_kernel(const JoinPlanDev* __restrict__ p, W8Plan w, int S, DevChunk ch, UniDev t, JoinOutDev o,
                                                       JoinStatus* st, uint64_t seq_base, int64_t out_base) {
  unsigned new_keys = 0, n_del = 0;
  bool any_match = false, any_hole = false;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t op = ch.ops[r];
    if (!row_visible(ch, r, op)) { o.vis[out_base + r] = 0; any_hole = true; continue; }
    if (op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE) n_del++;
    uni_row_generic<PROBE_ONLY>(p, w, S, ch, r, op, t, o, st, seq_base + (uint64_t)r, out_base + r, out_base + ch.n, new_keys, any_match, any_hole);
  }
  if (any_hole) atomicOr(&st->null_mask, 1ull << 63);
  if (any_match) st->pad = 1u;
  if (!PROBE_ONLY && new_keys) atomicAdd(&st->n_keys[0], (unsigned long long)new_keys);
  if (!PROBE_ONLY && n_del) atomicAdd(&st->n_del, (unsigned long long)n_del);
}

__device__ __forceinline__ ulonglong2 ld128_cg(const void* ptr) { return __ldcg((const ulonglong2*)ptr); }

// ------------------------------------------------------------------ quad-cooperative kernel (plain chunks)
// A row is owned by a QUAD of lanes, a warp works on 8 rows per iteration.  Lane q loads 16 bytes of the key's
// bucket in ONE instruction per quad (the cost of a random bucket access is the number of memory instructions
// that reach the line, tools/ubench_bucket.cu):
//     lane 0: key | WI      lane 1: IH | WC      lane 2: inline columns 0,1      lane 3: inline columns 2,3
// lanes 0,1 hold the update row's columns (0,1) / (2,3) and write them to the output; lanes 2,3 write the
// matched columns they loaded themselves -- no shuffle moves payload.  Lane 0 then does the own-side state
// change on the same line, lanes 1..3 write the record (header, columns) with one 16-byte store each.
// Output is positional (output row r = first match of input row r, extra matches behind the n positional rows);
// the extra rows come from a per-warp reservation of U_XCHUNK rows (reserved-but-unused rows are invisible).
//
// The kernel body holds ONLY the common case.  Rows it cannot finish with the quad -- several matches, a match
// that is not the bucket's inline record, NULLs in the matched record, the key equal to the EMPTY sentinel, every
// row of the inline side (its matches live in a chain) -- are DEFERRED: the quad records (bucket, match count,
// reserved extra rows) in the row's worklist entry and sets the row's bit; phase 1 of uni_tail_kernel, launched right
// behind, finishes them one thread per row.  (With those paths inlined the hot loop spilled ~350 bytes.)
struct PlainChunk {      // a chunk without bitmaps, 8-byte columns
  const uint8_t* ops;
  const unsigned long long* c[4];
  const unsigned long long* key;  // the key column (one of c[])
  int64_t n;
  const int64_t* n_dev;  // or nullptr
};
struct UniOwn {          // the pushing side's log, resolved on the host (a side index into UniDev's arrays would make
  uint8_t* const* log;   // the compiler copy the parameter struct to local memory)
  uint64_t log_cap;
  uint2* pools;
  unsigned long long* log_next;
};
struct PlainOut {
  uint8_t* ops;
  uint8_t* vis;
  unsigned long long* ucol[4];  // output column fed by update column c (nullptr = not projected)
  unsigned long long* mcol[4];  // output column fed by matched column c
  int64_t capacity;
};
struct UniDefer {
  int64_t b;       // the key's bucket (-1: look the key up -- sentinel key)
  int64_t xpos;    // first reserved extra-match row
  uint32_t cnt;    // matches to emit (0: whole row through uni_row_generic)
  uint32_t pad;
};
struct UniWork {
  UniDefer* entry;   // [n], written for deferred rows only
  uint8_t* mask;     // [(n + 7) / 8], one bit per input row, every byte written by the hot kernel
};

// 4 blocks of 256 threads per SM (64 registers): the kernel is bound by random DRAM transactions, not by occupancy
template <bool PROBE_ONLY, bool IS_ROW>
__global__ void __launch_bounds__(JF_BLOCK, 4) uni_hot_kernel(PlainChunk ch, uint8_t* buckets, uint64_t cap, UniOwn own, PlainOut o, UniWork wk,
                                                               JoinStatus* st, uint64_t seq_base, int64_t out_base, uint32_t pool_chunk) {
  int64_t n_rows = ch.n;
  if (ch.n_dev) {
    const int64_t nd = *ch.n_dev;
    if (nd < 0 || nd > ch.n) {
      if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&st->err, JERR_BAD_COUNT);
      n_rows = 0;
    } else {
      n_rows = nd;
      if (blockIdx.x == 0 && threadIdx.x == 0) st->n_in = (unsigned long long)nd;
    }
  }
  const int lane = lane_id(), q = lane & 3, qlead = lane & ~3;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  uint32_t pool_next = 0, pool_end = 0;
  if (!PROBE_ONLY) {
    const uint2 pl = own.pools[warp_global];
    pool_next = pl.x;
    pool_end = pl.y;
  }
  int64_t xnext = 0, xend = 0;  // this warp's reservation in the extra-match area (offsets from xarea)
  const int64_t xarea = out_base + n_rows;
  const uint64_t mask = cap - 1;
  unsigned int new_keys = 0, n_del = 0;
  // what this thread has seen, as bits of ONE register (separate booleans, each live across the loop, spilled)
  enum : unsigned { SEEN_MATCH = 1u, SEEN_HOLE = 2u, SEEN_DEFER = 4u, SEEN_SENTINEL = 8u, SEEN_POOL = 16u };
  unsigned seen = 0u;
  // (selected with ?: -- an index computed from the lane would put the parameter arrays in local memory)
  const unsigned long long* pa = (q & 1) ? ch.c[2] : ch.c[0];
  const unsigned long long* pb = (q & 1) ? ch.c[3] : ch.c[1];
  const unsigned long long* pk = ch.key;
  // the two output columns lane q writes, s_po[q] and s_po[4 + q]: read from shared memory where a row is emitted (held in
  // registers across the loop they were spilled to local memory)
  __shared__ unsigned long long* s_po[8];
  if (threadIdx.x < 8) {
    const int c = threadIdx.x;
    s_po[c] = c == 0 ? o.ucol[0] : c == 1 ? o.ucol[2] : c == 2 ? o.mcol[0] : c == 3 ? o.mcol[2]
            : c == 4 ? o.ucol[1] : c == 5 ? o.ucol[3] : c == 6 ? o.mcol[1] : o.mcol[3];
  }
  __syncthreads();
  const uint32_t nwarps = gridDim.x * (blockDim.x >> 5);
  const int64_t groups = (n_rows + 7) >> 3;
  const unsigned long long init_W = IS_ROW ? ((W_EMPTY | W_IL_LIVE) + W_COUNT_ONE) : W_EMPTY;
  // software pipeline: the sequential column loads of the warp's next group are issued right after the random
  // access of the current one
  uint8_t n_op = 0;
  unsigned long long n_key = J_EMPTY, n_va = 0ull, n_vb = 0ull;
#define UNI_FETCH(G2)                                                             \
  do {                                                                            \
    const int64_t g2_ = (G2), r2_ = g2_ * 8 + (lane >> 2);                        \
    n_op = 0;                                                                     \
    if (g2_ < groups && r2_ < n_rows) {                                           \
      n_op = ch.ops[r2_];                                                         \
      n_key = __ldg(pk + r2_);                                                    \
      if (pa) n_va = __ldg(pa + r2_);                                             \
      if (pb) n_vb = __ldg(pb + r2_);                                             \
    }                                                                             \
  } while (0)
  UNI_FETCH(warp_global);
  for (int64_t g = warp_global; g < groups; g += nwarps) {
    const int64_t r = g * 8 + (lane >> 2);
    const bool in = r < n_rows;
    const uint8_t op = n_op;
    const unsigned long long key = n_key, va = n_va, vb = n_vb;
    const int64_t pos = out_base + r;
    const bool act = op != 0;
    const bool ins = act && (op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT);
    if (act && !ins && q == 0) n_del++;
    const bool keyok = act && key != J_EMPTY;
    const bool do_ins = !PROBE_ONLY && ins;
    uint64_t idx = uhome(key, mask);
    // ---- the key's bucket: one 16-byte load per lane; an empty bucket is claimed on the spot by an inserting row
    bool found = false, need = keyok, created = false;
    ulonglong2 pv = make_ulonglong2(0ull, 0ull);
    bool first_iter = true;
    while (__any_sync(0xffffffffu, need)) {
      if (need) pv = ld128_cg(buckets + idx * 64 + 16 * q);
      if (first_iter) {
        UNI_FETCH(g + nwarps);
        first_iter = false;
      }
      const unsigned long long bkey = shfl64m(0xffffffffu, pv.x, qlead);
      const bool empty = need && bkey == J_EMPTY;
      if (need && !empty) {
        if (bkey == key) { found = true; need = false; }
        else idx = (idx + 1) & mask;
      }
      if (__any_sync(0xffffffffu, empty)) {
        ulonglong2 cf = make_ulonglong2(1ull, 0ull);
        if (empty && do_ins && q == 0) {
          ulonglong2 e, d;
          e.x = J_EMPTY; e.y = W_EMPTY;
          d.x = key; d.y = init_W;
          cas128(buckets + idx * 64, e, d, &cf);
        }
        const unsigned long long cfx = shfl64m(0xffffffffu, cf.x, qlead), cfy = shfl64m(0xffffffffu, cf.y, qlead);
        if (empty) {
          if (!do_ins) {
            need = false;  // the key is absent
          } else if ((cfx == J_EMPTY && cfy == W_EMPTY) || cfx == key) {
            // claimed by this row, or a moment ago by another row of this batch with the same key: either way
            // the OTHER side holds nothing for the key (it did not exist before this batch)
            created = cfx == J_EMPTY;
            found = true;
            need = false;
            pv.x = q == 0 ? key : 0ull;
            pv.y = q == 0 ? (created ? init_W : cfy) : (q == 1 ? (unsigned long long)U_NIL : 0ull);
          }
          // else: another key took the bucket -- load it again and move on
        }
      }
    }
    if (first_iter) UNI_FETCH(g + nwarps);
    if (created && q == 0) new_keys++;
    // ---- what does the other side hold for the key ?
    const unsigned long long WI = shfl64m(0xffffffffu, pv.y, qlead);
    uint32_t cnt, own_cnt = 0u;  // own_cnt: the chained side's count as loaded with the bucket (0 after a claim)
    bool fast = false;
    if (!IS_ROW) {
      const uint32_t inull = __shfl_sync(0xffffffffu, (uint32_t)(pv.x & 0xffull), qlead + 1);
      if (!PROBE_ONLY) own_cnt = __shfl_sync(0xffffffffu, (uint32_t)(pv.y >> 32), qlead + 1);
      cnt = found ? W_count(WI) : 0u;
      fast = cnt == 1u && W_istate(WI) == 1u && inull == 0u;
    } else {
      const uint32_t ccount = __shfl_sync(0xffffffffu, (uint32_t)(pv.y >> 32), qlead + 1);
      cnt = found ? ccount : 0u;
    }
    // ---- emit
    if (fast) {  // one match, in the bucket's inline record: the quad writes the row
      seen |= SEEN_MATCH;
      if (q == 0) o.ops[pos] = ins ? RW_OP_INSERT : RW_OP_DELETE;
      if (q == 1) o.vis[pos] = 1;
      unsigned long long* const po0 = *(unsigned long long* volatile*)&s_po[q];  // (volatile: not hoisted out of the loop)
      unsigned long long* const po1 = *(unsigned long long* volatile*)&s_po[4 + q];
      if (po0) po0[pos] = q < 2 ? va : pv.x;
      if (po1) po1[pos] = q < 2 ? vb : pv.y;
    } else if (in && q == 0) {
      // deferred rows get their visibility from uni_tail_kernel's deferred phase; the others are holes
      if (!(act && (!keyok || cnt > 0u))) { o.vis[pos] = 0; seen |= SEEN_HOLE; }
    }
    const bool defer = act && !fast && (!keyok || cnt > 0u);
    // extra-match rows: one reservation per warp and U_XCHUNK rows (an atomic per row on the shared counter
    // serialises in one L2 slice)
    int64_t xoff = 0;
    bool xbad = false;
    {
      const uint32_t xneed = (defer && keyok && q == 0 && cnt > 1u) ? cnt - 1u : 0u;
      if (__any_sync(0xffffffffu, xneed != 0u)) {
        uint32_t incl = xneed;
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        int64_t base = xnext;
        if ((int64_t)total > xend - xnext) {
          // leftover of the old reservation becomes invisible filler
          for (int64_t f = xnext + lane; f < xend; f += 32) { o.ops[xarea + f] = RW_OP_INSERT; o.vis[xarea + f] = 0; }
          if (xend > xnext) seen |= SEEN_HOLE;
          const uint32_t take = total > U_XCHUNK ? total : U_XCHUNK;
          unsigned long long nb = 0;
          if (lane == 0) nb = atomicAdd(&st->out_rows, (unsigned long long)take);
          nb = __shfl_sync(0xffffffffu, nb, 0);
          base = (int64_t)nb;
          xnext = base;
          xend = base + take;
          if (xarea + xend > o.capacity) {  // the host redoes the (state-free) emission with a larger buffer
            if (lane == 0) atomicOr(&st->err, JERR_OUT_CAPACITY);
            xbad = true;
            xend = xnext;
          }
        }
        xoff = base + (int64_t)(incl - xneed);
        if (!xbad) xnext += total;
      }
    }
    // ---- worklist: one mask byte per group of 8 rows (always written), an entry per deferred row
    {
      const unsigned dbal = __ballot_sync(0xffffffffu, defer && q == 0);
      if (dbal) seen |= SEEN_DEFER;
      if (__any_sync(0xffffffffu, defer && !keyok)) seen |= SEEN_SENTINEL;  // whole rows (insert included) go to the tail kernel
      if (lane == 0 && g * 8 < n_rows) {
        unsigned m8 = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) m8 |= ((dbal >> (4 * k)) & 1u) << k;
        wk.mask[g] = (uint8_t)m8;
      }
      if (defer && q == 0) {
        UniDefer e;
        e.b = keyok ? (int64_t)idx : -1;
        e.xpos = xarea + xoff;
        e.cnt = keyok ? (xbad ? 1u : cnt) : 0u;
        e.pad = 0;
        wk.entry[r] = e;
      }
    }
    // ---- append to the own side (same bucket)
    if (!PROBE_ONLY) {
      bool need_id = false, inline_won = false;
      unsigned long long Wcur = WI;
      unsigned long long* Wp = (unsigned long long*)(buckets + idx * 64 + 8);
      const bool mine = do_ins && keyok && q == 0;
      if (IS_ROW) {
        if (mine) {
          inline_won = created;
          if (!inline_won) {
            while (W_istate(Wcur) != 1u) {  // the inline record is free (never used, or its row was deleted)
              const unsigned long long nw = ((Wcur & ~W_IL_MASK) | W_IL_LIVE) + W_COUNT_ONE;
              const unsigned long long old = atomicCAS(Wp, Wcur, nw);
              if (old == Wcur) { inline_won = true; break; }
              Wcur = old;
            }
          }
          need_id = !inline_won;
        }
      } else {
        need_id = mine;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, need_id);
      uint32_t row = U_NIL;
      if (bal) {  // warp-uniform: log ids for the rows that need one, from the warp's pool
        const uint32_t k = __popc(bal), left = pool_end - pool_next;
        uint32_t nb = 0;
        if (left < k) {
          if (lane == 0) {
            const unsigned long long got = atomicAdd(own.log_next, (unsigned long long)pool_chunk);
            if (got + pool_chunk > own.log_cap) { atomicOr(&st->err, JERR_STORE_CAPACITY); nb = 0xffffffffu; }
            else nb = (uint32_t)got;
          }
          nb = __shfl_sync(0xffffffffu, nb, 0);
        }
        const uint32_t i = __popc(bal & ((1u << lane) - 1u));
        const bool bad = left < k && nb == 0xffffffffu;
        if (need_id && !(bad && i >= left)) row = i < left ? pool_next + i : nb + (i - left);
        if (left < k) {
          pool_next = bad ? 0u : nb + (k - left);
          pool_end = bad ? 0u : nb + pool_chunk;
        } else {
          pool_next += k;
        }
        seen |= SEEN_POOL;
      }
      uint32_t link = 0u;
      unsigned long long recp = 0;  // 0 = nothing to write; bit 0 set = the bucket's inline record
      if (IS_ROW) {
        if (inline_won) recp = (unsigned long long)(buckets + idx * 64) | 1ull;
        else if (row != U_NIL) {
          while (true) {  // one CAS pushes the row on the key's overflow chain
            const unsigned long long nw = ((Wcur & ~0x7fffffffull) | (unsigned long long)row) + W_COUNT_ONE;
            const unsigned long long old = atomicCAS(Wp, Wcur, nw);
            if (old == Wcur) break;
            Wcur = old;
          }
          link = W_head(Wcur);
          recp = (unsigned long long)useg_rec(own.log, row);
        }
      } else if (row != U_NIL) {
        link = uni_chain_push((unsigned long long*)(buckets + idx * 64 + 24), row, own_cnt);
        recp = (unsigned long long)useg_rec(own.log, row);
      }
      recp = shfl64m(0xffffffffu, recp, qlead);
      link = __shfl_sync(0xffffffffu, link, qlead);
      if (recp && q != 0) {
        const unsigned long long seq = seq_base + (unsigned long long)r;
        if (recp & 1ull) {  // inline: IH (8 bytes: WC sits next to it) + the columns
          uint8_t* bp = (uint8_t*)(recp & ~1ull);
          if (q == 1) *(unsigned long long*)(bp + 16) = seq << 8;
          else *(ulonglong2*)(bp + 16 + 16 * (q - 1)) = make_ulonglong2(va, vb);
        } else {
          ulonglong2 v;
          if (q == 1) { v.x = (unsigned long long)link; v.y = seq; }  // link | nullmask = 0, seq
          else { v.x = va; v.y = vb; }
          *(ulonglong2*)(recp + 16 * (q - 1)) = v;
        }
      }
    }
  }
#undef UNI_FETCH
  // leftover of the extra-row reservation
  for (int64_t f = xnext + lane; f < xend; f += 32) { o.ops[xarea + f] = RW_OP_INSERT; o.vis[xarea + f] = 0; }
  if (xend > xnext) seen |= SEEN_HOLE;
  if (!PROBE_ONLY && lane == 0 && (seen & SEEN_POOL)) own.pools[warp_global] = make_uint2(pool_next, pool_end);
  unsigned long long flags = ((seen & SEEN_HOLE) ? (1ull << 63) : 0ull);
  const bool warp_match = __any_sync(0xffffffffu, (seen & SEEN_MATCH) != 0u);
  const bool warp_defer = __any_sync(0xffffffffu, (seen & SEEN_DEFER) != 0u);
  const bool warp_sentinel = __any_sync(0xffffffffu, (seen & SEEN_SENTINEL) != 0u);
  for (int d = 16; d > 0; d >>= 1) {
    flags |= __shfl_xor_sync(0xffffffffu, flags, d);
    new_keys += __shfl_xor_sync(0xffffffffu, new_keys, d);
    n_del += __shfl_xor_sync(0xffffffffu, n_del, d);
  }
  if (lane == 0) {
    if (flags && (__ldcg(&st->null_mask) & flags) != flags) atomicOr(&st->null_mask, flags);
    if (warp_match && __ldcg(&st->pad) == 0u) st->pad = 1u;
    {  // bit 0: rows deferred; bit 1: some of them are whole rows whose own-side insert happens in the tail kernel
      const unsigned long long want = (warp_defer ? 1ull : 0ull) | (warp_sentinel ? 2ull : 0ull);
      if (want && (__ldcg(&st->n_defer) & want) != want) atomicOr(&st->n_defer, want);
    }
    if (!PROBE_ONLY && new_keys) atomicAdd(&st->n_keys[0], (unsigned long long)new_keys);
    if (!PROBE_ONLY && n_del) atomicAdd(&st->n_del, (unsigned long long)n_del);
  }
}

// the rows uni_hot_kernel deferred, one thread per input row (phase 1 of uni_tail_kernel)
template <bool PROBE_ONLY>
__device__ __forceinline__ void uni_deferred_body(const JoinPlanDev* __restrict__ p, const W8Plan& w, int S, const DevChunk& ch, const UniDev& t,
                                                  const JoinOutDev& o, const UniWork& wk, JoinStatus* st, uint64_t seq_base, int64_t out_base) {
  const int64_t n_rows = chunk_rows(ch);
  unsigned new_keys = 0;
  bool any_match = false, any_hole = false;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    if (!((wk.mask[r >> 3] >> (r & 7)) & 1u)) continue;
    const UniDefer e = wk.entry[r];
    const uint8_t op = ch.ops[r];
    const int64_t pos = out_base + r;
    if (e.cnt == 0u) {  // whole row (the key equal to the EMPTY sentinel)
      uni_row_generic<PROBE_ONLY>(p, w, S, ch, r, op, t, o, st, seq_base + (uint64_t)r, pos, out_base + n_rows, new_keys, any_match, any_hole);
    } else {
      any_match = true;
      o.vis[pos] = 1;
      const bool ins = (op == RW_OP_INSERT || op == RW_OP_UPDATE_INSERT);
      uni_emit_matches(t, w, S, ch, r, ins ? RW_OP_INSERT : RW_OP_DELETE, e.b, e.cnt, o, st, pos, e.xpos);
    }
  }
  if (any_hole) atomicOr(&st->null_mask, 1ull << 63);
  if (any_match) st->pad = 1u;
  if (!PROBE_ONLY && new_keys) atomicAdd(&st->n_keys[0], (unsigned long long)new_keys);
}

// pk equality of a stored row (columns c[], null mask) with chunk row r; a float8 pk column compares by the class
// load_key_word gives it (-0 == +0, one NaN), as pk_equal of the other paths does
__device__ __forceinline__ bool uni_pk_equal(const JoinPlanDev* p, int S, const uint64_t* c, uint32_t nmask, const DevChunk& ch, int64_t r) {
  for (int i = 0; i < p->n_pk[S]; i++) {
    const int k = p->pk_col[S][i];
    const bool n1 = (nmask >> k) & 1u, n2 = col_is_null(ch.cols[k], r);
    if (n1 != n2) return false;
    if (n1) continue;
    const uint64_t x = c[k], y = ((const uint64_t*)ch.cols[k].data)[r];
    if (x != y) {
      if (p->col_type[S][k] != RW_T_FLOAT64) return false;
      const double fx = __longlong_as_double((long long)x), fy = __longlong_as_double((long long)y);
      if (fx != fy && (fx == fx || fy == fy)) return false;
    }
  }
  return true;
}

// own-side deletes, after the main kernel (exits at once when the batch has none; then it only publishes the
// status block).  Sequential rule: the delete at chunk position r removes the live row with equal pk that
// arrived most recently BEFORE r: rows this very chunk inserted at positions >= r are excluded by their 64-bit
// arrival number (seq_base .. seq_base + n), every other live pk-equal row is older; the newest wins.
// sentinel_mode: 0 = every delete row; 1 = all but the rows whose key is the EMPTY sentinel; 2 = only those, by ONE block
__device__ __forceinline__ void uni_delete_body(const JoinPlanDev* __restrict__ p, int S, const DevChunk& ch, const UniDev& t, JoinStatus* st,
                                                uint64_t seq_base, int sentinel_mode) {
  const int64_t n_rows = chunk_rows(ch);
  const uint64_t SEQ56 = (1ull << 56) - 1;
  unsigned int dead_log = 0;
  const int64_t r_first = sentinel_mode == 2 ? (int64_t)threadIdx.x : blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r_step = sentinel_mode == 2 ? (int64_t)blockDim.x : (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = r_first; r < n_rows; r += r_step) {
    const uint8_t op = ch.ops[r];
    if (!row_visible(ch, r, op) || !(op == RW_OP_DELETE || op == RW_OP_UPDATE_DELETE)) continue;
    const ColRef& kc = ch.cols[p->key_col[S][0]];
    const bool knull = col_is_null(kc, r);
    if (knull && !p->null_safe[0]) continue;  // never-match rows were never stored
    const uint64_t key = knull ? 0ull : ((const uint64_t*)kc.data)[r];
    if (sentinel_mode && ((!knull && key == J_EMPTY) != (sentinel_mode == 2))) continue;
    const int64_t b = uni_find(t, key, knull);
    bool found = false;
    while (b >= 0 && !found) {
      // candidates: the inline record (inline side only) and the side's chain
      int best_kind = 0;  // 0 none, 1 inline, 2 log record
      uint32_t best_id = U_NIL;
      uint64_t best_seq = 0;
      auto consider = [&](int kind, uint32_t id, uint64_t seq, const uint64_t* c, uint32_t nmask) {
        const uint64_t d = (seq - seq_base) & SEQ56;
        if (d < (uint64_t)n_rows && d >= (uint64_t)r) return;  // inserted by this chunk at or after position r
        if (!uni_pk_equal(p, S, c, nmask, ch, r)) return;
        // arrival order: rows of this chunk (d < n) are newer than everything stored before it
        const uint64_t rank = d < (uint64_t)n_rows ? (1ull << 60) + d : (seq & SEQ56);
        if (best_kind == 0 || rank > best_seq) { best_kind = kind; best_id = id; best_seq = rank; }
      };
      uint32_t m;
      if (S == t.is) {
        const unsigned long long WI = __ldcg(ub_WI(t, b));
        if (W_istate(WI) == 1u) {
          const unsigned long long ih = __ldcg(ub_IH(t, b));
          uint64_t c[4];
          const ulonglong2 c01 = __ldcg((const ulonglong2*)(ub(t, b) + 32)), c23 = __ldcg((const ulonglong2*)(ub(t, b) + 48));
          c[0] = c01.x; c[1] = c01.y; c[2] = c23.x; c[3] = c23.y;
          consider(1, 0u, ih >> 8, c, (uint32_t)(ih & 0xffull));
        }
        m = W_head(WI);
      } else {
        m = __ldcg(ub_chead(t, b));
      }
      while (m != U_NIL) {
        const UniRec* rec = urec(t, S, m);
        const ulonglong2 h0 = __ldcg((const ulonglong2*)rec);
        const uint32_t lk = (uint32_t)h0.x;
        if (!(lk & J_DEAD)) {
          uint64_t c[4];
          const ulonglong2 c01 = __ldcg((const ulonglong2*)rec + 1), c23 = __ldcg((const ulonglong2*)rec + 2);
          c[0] = c01.x; c[1] = c01.y; c[2] = c23.x; c[3] = c23.y;
          consider(2, m, h0.y, c, (uint32_t)(h0.x >> 32));
        }
        m = lk & 0x7fffffffu;
      }
      if (best_kind == 0) break;
      if (best_kind == 1) {
        unsigned long long* Wp = ub_WI(t, b);
        unsigned long long cur = __ldcg(Wp);
        while (W_istate(cur) == 1u) {  // live -> dead, count - 1, in one CAS
          const unsigned long long old = atomicCAS(Wp, cur, ((cur & ~W_IL_MASK) | W_IL_DEAD) - W_COUNT_ONE);
          if (old == cur) { found = true; break; }
          cur = old;
        }
      } else {
        const uint32_t old = atomicOr(&urec(t, S, best_id)->link, J_DEAD);
        if (!(old & J_DEAD)) {
          if (S == t.is) atomicAdd(ub_WI(t, b), 0ull - W_COUNT_ONE);
          else atomicSub(ub_ccount(t, b), 1u);
          dead_log++;
          found = true;
        }
      }
      // (lost a race against another delete of the same row: look again)
    }
    if (!found && p->strict) atomicOr(&st->err, JERR_DOUBLE_DELETE);
  }
  if (dead_log) atomicAdd(t.n_dead[S], (unsigned long long)dead_log);
}

// Everything behind the hot kernel in ONE launch: (1) the deferred rows, (2) the own-side deletes, (3) the status block
// published to pinned host memory by the block that finishes last.  Phases 1 and 2 exit at once when the hot kernel
// flagged no such rows (st->n_defer / st->n_del are final when this kernel starts: every block takes the same path).
// The two phases are independent -- deferred emission reads the OTHER side's records, deletes change the OWN side's --
// except for deferred WHOLE rows (the key equal to the EMPTY sentinel: their insert happens in phase 1 and a delete
// later in the chunk may target it).  When a batch has both (n_defer bit 1 and deletes), the deletes of sentinel-key
// rows are left to the LAST block, which runs them after every other block has finished: no block ever waits for
// another one, so the kernel needs no co-residency and no cooperative launch.
// (Separate deferred and delete launches, or one cooperative launch, each cost more per step than this plain one.)
template <bool PROBE_ONLY>
__global__ void __launch_bounds__(256) uni_tail_kernel(const JoinPlanDev* __restrict__ p, W8Plan w, int S, DevChunk ch, UniDev t, JoinOutDev o, UniWork wk,
                                                       JoinStatus* st, uint64_t seq_base, int64_t out_base, JoinStatus* status_host,
                                                       unsigned long long tag, int reset, unsigned int* done) {
  __shared__ bool s_last;
  const unsigned long long defer_flags = *(volatile unsigned long long*)&st->n_defer;
  const bool has_del = !PROBE_ONLY && *(volatile unsigned long long*)&st->n_del != 0ull;
  const bool split = has_del && (defer_flags & 2ull) != 0ull;
  if (defer_flags) uni_deferred_body<PROBE_ONLY>(p, w, S, ch, t, o, wk, st, seq_base, out_base);
  if (has_del) uni_delete_body(p, S, ch, t, st, seq_base, split ? 1 : 0);
  // last block out: the sentinel-key deletes (if any were left), then the status block
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(done, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (split) {
    uni_delete_body(p, S, ch, t, st, seq_base, 2);
    __threadfence();
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    done[0] = 0u;
    st->log_next[0] = *(volatile unsigned long long*)t.log_next[0]; st->log_next[1] = *(volatile unsigned long long*)t.log_next[1];
    st->n_dead[0] = *(volatile unsigned long long*)t.n_dead[0]; st->n_dead[1] = *(volatile unsigned long long*)t.n_dead[1];
    join_status_publish(st, status_host, tag, reset);
  }
}

// watermark-driven state cleaning (JoinHashMap::update_watermark, join/hash_join.rs; applied at the barrier like the
// state table's commit-time range delete): every row of `side` whose join key is below the watermark leaves the state.
// The whole key dies on that side, so the side's part of the bucket is simply reset; its log records become
// unreachable and are counted as dead for the compaction trigger.
__global__ void __launch_bounds__(256) uni_clean_kernel(UniDev t, int side, long long wm) {
  unsigned int dead = 0;
  for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b < t.cap + 2; b += (uint64_t)gridDim.x * blockDim.x) {
    if (b == t.cap) continue;  // NULL keys sort last: never below a watermark
    const unsigned long long key = *(const unsigned long long*)ub(t, (int64_t)b);
    if (b < t.cap && key == J_EMPTY) continue;
    const long long kv = b == t.cap + 1 ? (long long)J_EMPTY : (long long)key;
    if (kv >= wm) continue;
    if (side == t.is) {
      unsigned long long* Wp = ub_WI(t, (int64_t)b);
      const unsigned long long W = *Wp;
      const uint32_t cnt = W_count(W);
      if (cnt) dead += cnt - (W_istate(W) == 1u ? 1u : 0u);
      *Wp = W_EMPTY | (W_istate(W) ? W_IL_DEAD : 0ull);
    } else {
      dead += *ub_ccount(t, (int64_t)b);
      *ub_chead(t, (int64_t)b) = U_NIL;
      *ub_ccount(t, (int64_t)b) = 0u;
    }
  }
  for (int d = 16; d > 0; d >>= 1) dead += __shfl_xor_sync(0xffffffffu, dead, d);
  if (lane_id() == 0 && dead) atomicAdd(t.n_dead[side], (unsigned long long)dead);
}

// status publication after a delete kernel that had real work
__global__ void uni_status_kernel(UniDev t, JoinStatus* st, JoinStatus* status_host, unsigned long long tag, int reset) {
  st->log_next[0] = *t.log_next[0]; st->log_next[1] = *t.log_next[1];
  st->n_dead[0] = *t.n_dead[0]; st->n_dead[1] = *t.n_dead[1];
  join_status_publish(st, status_host, tag, reset);
}

// growth: re-insert every claimed bucket into a larger array
__global__ void uni_rehash_kernel(const uint8_t* ob, uint64_t ocap, uint8_t* nb, uint64_t ncap) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < ocap + 2; i += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2* s = (const ulonglong2*)(ob + i * 64);
    uint64_t dst;
    if (i >= ocap) {
      dst = ncap + (i - ocap);
    } else {
      const uint64_t key = s[0].x;
      if (key == J_EMPTY) continue;
      const uint64_t mask = ncap - 1;
      uint64_t idx = uhome(key, mask);
      while (atomicCAS((unsigned long long*)(nb + idx * 64), (unsigned long long)J_EMPTY, (unsigned long long)key) != J_EMPTY) idx = (idx + 1) & mask;
      dst = idx;
    }
    ulonglong2* d = (ulonglong2*)(nb + dst * 64);
    const ulonglong2 s0 = s[0];
    ((unsigned long long*)d)[1] = s0.y;
    if (i >= ocap) ((unsigned long long*)d)[0] = s0.x;
    d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
  }
}

// compaction of a side's log (barrier time, when dead records dominate): every chain is copied, live records only
// and in chain order, into a fresh log -- ids change, links and heads are rewritten, dead rows disappear.
// One thread per bucket; nothing else runs on the table meanwhile.
__global__ void uni_compact_kernel(UniDev t, int side, uint8_t* const* new_log, unsigned long long* new_next) {
  const int lane = lane_id();
  for (uint64_t i0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) & ~31ull; i0 < t.cap + 2; i0 += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = i0 + lane;
    uint32_t live = 0, head = U_NIL;
    bool has = false;
    if (i < t.cap + 2) {
      const unsigned long long key = __ldcg((const unsigned long long*)ub(t, (int64_t)i));
      has = key != J_EMPTY || i >= t.cap;
      if (has) {
        head = side == t.is ? W_head(__ldcg(ub_WI(t, (int64_t)i))) : __ldcg(ub_chead(t, (int64_t)i));
        for (uint32_t m = head; m != U_NIL;) {
          const uint32_t lk = __ldcg(&urec(t, side, m)->link);
          if (!(lk & J_DEAD)) live++;
          m = lk & 0x7fffffffu;
        }
      }
    }
    // warp-aggregated reservation of new ids
    uint32_t incl = live;
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    unsigned long long base = 0;
    if (lane == 31 && total) base = atomicAdd(new_next, (unsigned long long)total);
    base = __shfl_sync(0xffffffffu, base, 31);
    if (!has) continue;
    uint32_t nid = (uint32_t)base + (incl - live);
    uint32_t new_head = U_NIL;
    UniRec* prev = nullptr;
    for (uint32_t m = head; m != U_NIL;) {
      const UniRec* rec = urec(t, side, m);
      const uint32_t lk = rec->link;
      if (!(lk & J_DEAD)) {
        UniRec* d = (UniRec*)useg_rec(new_log, nid);
        *d = *rec;
        d->link = U_NIL;
        if (prev) prev->link = nid; else new_head = nid;
        prev = d;
        nid++;
      }
      m = lk & 0x7fffffffu;
    }
    if (head != U_NIL) {
      if (side == t.is) {
        unsigned long long* Wp = ub_WI(t, (int64_t)i);
        *Wp = (*Wp & ~0x7fffffffull) | (unsigned long long)new_head;
      } else {
        *ub_chead(t, (int64_t)i) = new_head;
      }
    }
  }
}

}  // namespace rw
