// shuffle.cu -- the hash-shuffle (vnode) path on sm_90a.
//
// Replaces (reference, Rust):
//   VirtualNode::compute_chunk              src/common/src/hash/consistent_hash/vnode.rs:151-182
//   Crc32FastBuilder / to_vnode             src/common/src/util/hash_util.rs:24-33, vnode.rs:45-50
//   HashDataDispatcher::dispatch_data       src/stream/src/executor/dispatch.rs:961-1053
// The reference builds one visibility bitmap per downstream actor over shared column buffers;
// here rows are STABLY partitioned by destination GPU into contiguous regions (the send buffers
// of an NCCL all-to-all-v), preserving per-key row order.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "common.cuh"

namespace rw {

__device__ __forceinline__ uint32_t crc_table_entry(uint32_t i) {
  uint32_t c = i;
#pragma unroll
  for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : (c >> 1);
  return c;
}

__device__ __forceinline__ uint32_t crc_feed(const uint32_t* tab, uint32_t c, uint64_t v, int nbytes) {
  for (int b = 0; b < nbytes; b++) {
    c = tab[(c ^ (uint32_t)(v & 0xff)) & 0xff] ^ (c >> 8);
    v >>= 8;
  }
  return c;
}

// raw_double_bits (src/common/src/types/ordered_float.rs:852-870), via Float::integer_decode
__device__ __forceinline__ uint64_t raw_double_bits_f64(double f) {
  if (f != f) return 0x7ff8000000000000ull;
  uint64_t bits = (uint64_t)__double_as_longlong(f);
  int sign_pos = (bits >> 63) == 0;
  int e = (int)((bits >> 52) & 0x7ff);
  uint64_t man = e == 0 ? (bits & 0xfffffffffffffull) << 1 : (bits & 0xfffffffffffffull) | 0x10000000000000ull;
  short exp = (short)(e - (1023 + 52));
  if (man == 0) return 0;
  uint64_t eu = (uint64_t)(unsigned short)exp;
  return (man & 0x000fffffffffffffull) | ((eu << 52) & 0x7ff0000000000000ull) | ((uint64_t)sign_pos << 63);
}
__device__ __forceinline__ uint64_t raw_double_bits_f32(float f) {
  if (f != f) return 0x7ff8000000000000ull;
  uint32_t bits = __float_as_uint(f);
  int sign_pos = (bits >> 31) == 0;
  int e = (int)((bits >> 23) & 0xff);
  uint32_t man32 = e == 0 ? (bits & 0x7fffff) << 1 : (bits & 0x7fffff) | 0x800000;
  short exp = (short)(e - (127 + 23));
  uint64_t man = man32;
  if (man == 0) return 0;
  uint64_t eu = (uint64_t)(unsigned short)exp;
  return (man & 0x000fffffffffffffull) | ((eu << 52) & 0x7ff0000000000000ull) | ((uint64_t)sign_pos << 63);
}

// bytes of one datum as fed to the hasher (Array::hash_at, src/common/src/array/mod.rs:280-288;
// NULL_VAL_FOR_HASH :97).  Date/Time/Timestamp/Decimal hash through chrono / rust_decimal impls
// that are not in the reference tree: the ABI value's LE bytes are used (self-consistent on both
// join sides; "vnode parity unpinned" for those types, SURVEY §7.2).
__device__ __forceinline__ uint32_t crc_feed_datum(const uint32_t* tab, uint32_t c, const ColRef& col, int64_t r) {
  if (col_is_null(col, r)) return crc_feed(tab, c, 0xfffffff0ull, 4);
  if (col.type == RW_T_FLOAT64) return crc_feed(tab, c, raw_double_bits_f64(((const double*)col.data)[r]), 8);
  if (col.type == RW_T_FLOAT32) return crc_feed(tab, c, raw_double_bits_f32(((const float*)col.data)[r]), 8);
  if (col.width == 16) {
    const uint64_t* p = (const uint64_t*)col.data + r * 2;
    c = crc_feed(tab, c, p[0], 8);
    return crc_feed(tab, c, p[1], 8);
  }
  return crc_feed(tab, c, (uint64_t)load_i64(col, r), col.width);
}

struct VnodePlan {
  int n_keys;
  int key_col[RW_MAX_KEYS * 2];
  int vnode_count;
  int serial_fast;  // single Serial key: vnode taken from the row id (vnode.rs:156-176)
};

// compute_vnode_from_row_id (src/common/src/util/row_id.rs:135-173)
__device__ __forceinline__ uint32_t vnode_from_row_id(int64_t id, int vnode_count) {
  uint32_t vnode_bit = 10;
  if (vnode_count > 1024) { vnode_bit = 0; while ((1u << vnode_bit) < (uint32_t)vnode_count) vnode_bit++; }
  uint32_t seq_bit = 22 - vnode_bit;
  uint64_t part = ((uint64_t)id >> seq_bit) & ((1ull << vnode_bit) - 1);
  return (uint32_t)(part % (uint64_t)vnode_count);
}

__device__ __forceinline__ uint32_t row_vnode(const uint32_t* tab, const VnodePlan& p, const DevChunk& ch, int64_t r,
                                               bool visible) {
  if (p.serial_fast) {
    const ColRef& c = ch.cols[p.key_col[0]];
    if (!col_is_null(c, r)) return vnode_from_row_id(((const int64_t*)c.data)[r], p.vnode_count);
    uint32_t crc = 0xFFFFFFFFu;  // hash the entire row
    for (int k = 0; k < ch.n_cols; k++) crc = crc_feed_datum(tab, crc, ch.cols[k], r);
    return (crc ^ 0xFFFFFFFFu) % (uint32_t)p.vnode_count;
  }
  uint32_t crc = 0xFFFFFFFFu;
  if (visible)  // get_hash_values hashes visible rows only (data_chunk.rs:338-355)
    for (int k = 0; k < p.n_keys; k++) crc = crc_feed_datum(tab, crc, ch.cols[p.key_col[k]], r);
  return (crc ^ 0xFFFFFFFFu) % (uint32_t)p.vnode_count;
}

__global__ void __launch_bounds__(256) vnode_kernel(DevChunk ch, VnodePlan p, uint16_t* out) {
  __shared__ uint32_t tab[256];
  tab[threadIdx.x] = crc_table_entry(threadIdx.x);
  __syncthreads();
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    bool vis = bit_get(ch.vis_bits, r) && (ch.ops == nullptr || ch.ops[r] != 0);
    out[r] = (uint16_t)row_vnode(tab, p, ch, r, vis);
  }
}

// the op rewrite of dispatch.rs:976-1023, one thread per row.  The reference pairs a visible U+ with the last visible U-
// that no earlier U+ has taken (`last_update_delete_row_idx.take()`), whatever visible +/- rows lie between them:
//  * a visible U+ walks back over the visible rows, skipping + / -, to the nearest U- and rewrites both rows; meeting a
//    U+ or the chunk start first is "missing U- before U+" (bit 0 of *err);
//  * a visible U- walks forward the same way: if it meets a U+, that U+ writes its op; if it meets another U-, which
//    replaces it as the pending one, it keeps its op; if it meets the chunk end, it is "missing U+ after U-" (bit 1).
__device__ __forceinline__ bool rewrite_skips(const DevChunk& ch, int64_t r) {
  const uint8_t op = ch.ops[r];
  return !row_visible(ch, r, op) || op == RW_OP_INSERT || op == RW_OP_DELETE;
}
__global__ void dispatch_rewrite_kernel(DevChunk ch, VnodePlan p, uint8_t* out_ops, unsigned int* err) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < ch.n; r += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t op = ch.ops[r];
    if (rewrite_skips(ch, r) || (op != RW_OP_UPDATE_INSERT && op != RW_OP_UPDATE_DELETE)) {
      out_ops[r] = op;
      continue;
    }
    if (op == RW_OP_UPDATE_DELETE) {
      int64_t j = r + 1;
      while (j < ch.n && rewrite_skips(ch, j)) j++;
      if (j >= ch.n) atomicOr(err, 2u);
      if (j >= ch.n || ch.ops[j] != RW_OP_UPDATE_INSERT) out_ops[r] = op;
      continue;
    }
    int64_t j = r - 1;
    while (j >= 0 && rewrite_skips(ch, j)) j--;
    if (j < 0 || ch.ops[j] != RW_OP_UPDATE_DELETE) { atomicOr(err, 1u); out_ops[r] = op; continue; }
    bool changed = false;
    for (int k = 0; k < p.n_keys; k++) {
      const ColRef& c = ch.cols[p.key_col[k]];
      bool n1 = col_is_null(c, j), n2 = col_is_null(c, r);
      if (n1 != n2) changed = true;
      else if (!n1) {
        if (c.width == 16) {
          const uint64_t* a = (const uint64_t*)c.data;
          if (a[j * 2] != a[r * 2] || a[j * 2 + 1] != a[r * 2 + 1]) changed = true;
        } else if (load_key_word(c, j) != load_key_word(c, r)) changed = true;
      }
    }
    out_ops[j] = changed ? RW_OP_DELETE : RW_OP_UPDATE_DELETE;
    out_ops[r] = changed ? RW_OP_INSERT : RW_OP_UPDATE_INSERT;
  }
}

// ------------------------------------------------------------------ stable partition by destination
#define PART_BLOCK 256
#define PART_ROWS_PER_BLOCK 2048
#define PART_MAX_DEST 64

// pass 1: dest per row (255 = dropped: invisible) + per-block histogram
__global__ void __launch_bounds__(PART_BLOCK) part_hist_kernel(DevChunk ch, VnodePlan p, const int32_t* vnode_to_dest,
                                                                int n_dest, uint8_t* dest, uint32_t* block_hist) {
  __shared__ uint32_t tab[256];
  __shared__ uint32_t hist[PART_MAX_DEST];
  tab[threadIdx.x] = crc_table_entry(threadIdx.x);
  if (threadIdx.x < PART_MAX_DEST) hist[threadIdx.x] = 0;
  __syncthreads();
  int64_t base = (int64_t)blockIdx.x * PART_ROWS_PER_BLOCK;
  for (int i = threadIdx.x; i < PART_ROWS_PER_BLOCK; i += PART_BLOCK) {
    int64_t r = base + i;
    if (r >= ch.n) break;
    uint8_t op = ch.ops[r];
    uint8_t d = 255;
    if (row_visible(ch, r, op)) {
      uint32_t v = row_vnode(tab, p, ch, r, true);
      d = (uint8_t)vnode_to_dest[v];
      atomicAdd(&hist[d], 1u);
    }
    dest[r] = d;
  }
  __syncthreads();
  if (threadIdx.x < n_dest) block_hist[(size_t)blockIdx.x * n_dest + threadIdx.x] = hist[threadIdx.x];
}

// pass 2: one block; per destination exclusive scan over blocks -> block offsets; totals + region starts.
// One WARP per destination scans the per-block counts 32 at a time (shuffle scan, the chunk loads do
// not depend on each other); a serial loop over 512 blocks per thread was far slower.
#define PART_SCAN_THREADS 1024
__global__ void __launch_bounds__(PART_SCAN_THREADS) part_scan_kernel(uint32_t* block_hist, int n_blocks, int n_dest, int64_t* counts,
                                                                       int64_t* offsets) {
  __shared__ int64_t totals[PART_MAX_DEST];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (int d = wid; d < n_dest; d += n_warps) {
    uint32_t run = 0;
    for (int b0 = 0; b0 < n_blocks; b0 += 32) {
      const int b = b0 + lane;
      const uint32_t v = b < n_blocks ? block_hist[(size_t)b * n_dest + d] : 0u;
      uint32_t inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (b < n_blocks) block_hist[(size_t)b * n_dest + d] = run + inc - v;
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) {
      totals[d] = run;
      counts[d] = run;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    for (int k = 0; k < n_dest; k++) { offsets[k] = acc; acc += totals[k]; }
  }
}

struct PartOut {
  uint8_t* ops;
  void* col[RW_MAX_COLS];
  uint8_t* valid[RW_MAX_COLS];
};

// pass 3: stable scatter.  Rows of a block are ranked per destination in row order with warp ballots.
__global__ void __launch_bounds__(PART_BLOCK) part_scatter_kernel(DevChunk ch, const uint8_t* dest, const uint32_t* block_off,
                                                                   int n_dest, const int64_t* offsets, PartOut o) {
  __shared__ uint32_t run[PART_MAX_DEST];        // running count per destination within the block
  __shared__ uint32_t warp_cnt[PART_BLOCK / 32][PART_MAX_DEST];
  if (threadIdx.x < PART_MAX_DEST) run[threadIdx.x] = 0;
  __syncthreads();
  const int lane = lane_id(), wid = threadIdx.x >> 5;
  int64_t base = (int64_t)blockIdx.x * PART_ROWS_PER_BLOCK;
  for (int it = 0; it < PART_ROWS_PER_BLOCK / PART_BLOCK; it++) {
    int64_t r = base + it * PART_BLOCK + threadIdx.x;
    uint8_t d = (r < ch.n) ? dest[r] : 255;
    // rank within warp among lanes with the same destination
    unsigned peers = __match_any_sync(0xffffffffu, (unsigned)d);
    unsigned rank_in_warp = __popc(peers & ((1u << lane) - 1));
    bool leader = (rank_in_warp == 0);
    for (int k = lane; k < n_dest; k += 32) warp_cnt[wid][k] = 0;
    __syncwarp();
    if (leader && d != 255) warp_cnt[wid][d] = __popc(peers);
    __syncthreads();
    uint32_t pos = 0;
    if (d != 255) {
      uint32_t before = 0;
      for (int w = 0; w < wid; w++) before += warp_cnt[w][d];
      pos = run[d] + before + rank_in_warp;
    }
    __syncthreads();
    if (threadIdx.x < n_dest) {
      uint32_t tot = 0;
      for (int w = 0; w < PART_BLOCK / 32; w++) tot += warp_cnt[w][threadIdx.x];
      run[threadIdx.x] += tot;
    }
    if (d != 255) {
      int64_t dst = offsets[d] + block_off[(size_t)blockIdx.x * n_dest + d] + pos;
      o.ops[dst] = ch.ops[r];
      for (int k = 0; k < ch.n_cols; k++) {
        const ColRef& c = ch.cols[k];
        if (o.col[k] == nullptr) continue;
        switch (c.width) {
          case 1: ((uint8_t*)o.col[k])[dst] = ((const uint8_t*)c.data)[r]; break;
          case 2: ((uint16_t*)o.col[k])[dst] = ((const uint16_t*)c.data)[r]; break;
          case 4: ((uint32_t*)o.col[k])[dst] = ((const uint32_t*)c.data)[r]; break;
          case 8: ((uint64_t*)o.col[k])[dst] = ((const uint64_t*)c.data)[r]; break;
          default: ((ulonglong2*)o.col[k])[dst] = ((const ulonglong2*)c.data)[r]; break;
        }
        if (o.valid[k]) o.valid[k][dst] = col_is_null(c, r) ? 0 : 1;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ P2P exchange over NVLink peer memory
// Receive buffer of a rank (symmetric on every rank): one REGION per source rank,
//   region = [ header 256 B: int64 row count ][ ops: cap bytes ][ column k: cap * width_k bytes ] (each 256-B aligned).
// The sender's scatter kernel stores its rows for destination d straight into region `my_rank` of d's
// buffer (plain st.global on a peer-mapped pointer: partition and transfer are ONE kernel, no send
// staging, no NCCL call on the data path).  After a device-side barrier the receiver unpacks the W
// regions into contiguous columns.
struct P2PLayout {
  int64_t cap_rows;
  int64_t region_bytes;
  int64_t ops_off;
  int64_t col_off[RW_MAX_COLS];
  int n_cols;
  int col_width[RW_MAX_COLS];
};
struct PeerBases {
  uint8_t* base[PART_MAX_DEST];
};

static int p2p_layout(const int32_t* types, int n_cols, int64_t cap_rows, P2PLayout* L) {
  if (n_cols < 0 || n_cols > RW_MAX_COLS || cap_rows <= 0) return fail(RW_ERR_INVALID, "p2p layout");
  auto up = [](int64_t x) { return (x + 255) / 256 * 256; };
  int64_t off = 256;
  L->cap_rows = cap_rows;
  L->n_cols = n_cols;
  L->ops_off = off;
  off = up(off + cap_rows);
  for (int k = 0; k < n_cols; k++) {
    int w = type_width(types[k]);
    if (!w) return fail(RW_ERR_UNSUPPORTED, "column type");
    L->col_width[k] = w;
    L->col_off[k] = off;
    off = up(off + cap_rows * w);
  }
  L->region_bytes = off;
  return RW_OK;
}

__global__ void __launch_bounds__(PART_BLOCK) part_scatter_p2p_kernel(DevChunk ch, const uint8_t* dest, const uint32_t* block_off,
                                                                       int n_dest, P2PLayout L, PeerBases peers, int my_rank,
                                                                       int* overflow) {
  __shared__ uint32_t run[PART_MAX_DEST];
  __shared__ uint32_t warp_cnt[PART_BLOCK / 32][PART_MAX_DEST];
  if (threadIdx.x < PART_MAX_DEST) run[threadIdx.x] = 0;
  __syncthreads();
  const int lane = lane_id(), wid = threadIdx.x >> 5;
  int64_t base = (int64_t)blockIdx.x * PART_ROWS_PER_BLOCK;
  for (int it = 0; it < PART_ROWS_PER_BLOCK / PART_BLOCK; it++) {
    int64_t r = base + it * PART_BLOCK + threadIdx.x;
    uint8_t d = (r < ch.n) ? dest[r] : 255;
    unsigned peers_m = __match_any_sync(0xffffffffu, (unsigned)d);
    unsigned rank_in_warp = __popc(peers_m & ((1u << lane) - 1));
    for (int k = lane; k < n_dest; k += 32) warp_cnt[wid][k] = 0;
    __syncwarp();
    if (rank_in_warp == 0 && d != 255) warp_cnt[wid][d] = __popc(peers_m);
    __syncthreads();
    uint32_t pos = 0;
    if (d != 255) {
      uint32_t before = 0;
      for (int w = 0; w < wid; w++) before += warp_cnt[w][d];
      pos = run[d] + before + rank_in_warp;
    }
    __syncthreads();
    if (threadIdx.x < n_dest) {
      uint32_t tot = 0;
      for (int w = 0; w < PART_BLOCK / 32; w++) tot += warp_cnt[w][threadIdx.x];
      run[threadIdx.x] += tot;
    }
    if (d != 255) {
      const int64_t dst = (int64_t)block_off[(size_t)blockIdx.x * n_dest + d] + pos;  // row index inside (my_rank -> d)
      if (dst >= L.cap_rows) {
        *overflow = 1;
      } else {
        uint8_t* reg = peers.base[d] + (int64_t)my_rank * L.region_bytes;
        reg[L.ops_off + dst] = ch.ops[r];
        for (int k = 0; k < ch.n_cols; k++) {
          const ColRef& c = ch.cols[k];
          uint8_t* col = reg + L.col_off[k];
          switch (c.width) {
            case 1: ((uint8_t*)col)[dst] = ((const uint8_t*)c.data)[r]; break;
            case 2: ((uint16_t*)col)[dst] = ((const uint16_t*)c.data)[r]; break;
            case 4: ((uint32_t*)col)[dst] = ((const uint32_t*)c.data)[r]; break;
            case 8: ((uint64_t*)col)[dst] = ((const uint64_t*)c.data)[r]; break;
            default: ((ulonglong2*)col)[dst] = ((const ulonglong2*)c.data)[r]; break;
          }
        }
      }
    }
    __syncthreads();
  }
}

// publish the per-destination row counts in the region headers of the peers
__global__ void p2p_publish_counts_kernel(const int64_t* counts, int n_dest, P2PLayout L, PeerBases peers, int my_rank) {
  int d = threadIdx.x;
  if (d < n_dest) {
    int64_t c = counts[d] <= L.cap_rows ? counts[d] : -1;  // -1: this (source, destination) pair overflowed its region
    *(int64_t*)(peers.base[d] + (int64_t)my_rank * L.region_bytes) = c;
    __threadfence_system();
  }
}

// receiver: W regions -> contiguous ops / columns (source-rank order, row order kept inside a source)
__global__ void __launch_bounds__(256) p2p_unpack_kernel(const uint8_t* recv, int n_src, P2PLayout L, uint8_t* out_ops, PartOut o,
                                                          int64_t* total) {
  __shared__ int64_t off[PART_MAX_DEST + 1];
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    bool bad = false;
    for (int s = 0; s < n_src; s++) {
      off[s] = acc;
      const int64_t c = *(const volatile int64_t*)(recv + (int64_t)s * L.region_bytes);
      if (c < 0) bad = true; else acc += c;
    }
    off[n_src] = acc;
    if (blockIdx.x == 0) *total = bad ? -1 : acc;
  }
  __syncthreads();
  const int64_t n = off[n_src];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int s = 0;
    while (i >= off[s + 1]) s++;
    const int64_t j = i - off[s];
    const uint8_t* reg = recv + (int64_t)s * L.region_bytes;
    out_ops[i] = reg[L.ops_off + j];
    for (int k = 0; k < L.n_cols; k++) {
      const uint8_t* col = reg + L.col_off[k];
      switch (L.col_width[k]) {
        case 1: ((uint8_t*)o.col[k])[i] = col[j]; break;
        case 2: ((uint16_t*)o.col[k])[i] = ((const uint16_t*)col)[j]; break;
        case 4: ((uint32_t*)o.col[k])[i] = ((const uint32_t*)col)[j]; break;
        case 8: ((uint64_t*)o.col[k])[i] = ((const uint64_t*)col)[j]; break;
        default: ((ulonglong2*)o.col[k])[i] = ((const ulonglong2*)col)[j]; break;
      }
    }
  }
}

// cross-rank barrier on peer-mapped flag arrays: thread t signals rank t and waits for rank t's signal.
// Everything this rank stored into its peers (earlier kernels of the stream) is ordered before the
// signal (fence + release store at system scope); the peers' data is visible once their signal is seen.
__global__ void p2p_barrier_kernel(PeerBases flags, int n, int my_rank, unsigned long long epoch) {
  const int t = threadIdx.x;
  if (t < n) {
    __threadfence_system();
    unsigned long long* remote = (unsigned long long*)flags.base[t] + my_rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(remote), "l"(epoch) : "memory");
    const unsigned long long* mine = (const unsigned long long*)flags.base[my_rank] + t;
    unsigned long long v;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory");
    } while (v < epoch);
  }
}

__global__ void p2p_total_to_host_kernel(const int64_t* total, int64_t* total_host) {
  *total_host = *total;
  __threadfence_system();
}

// ------------------------------------------------------------------ fused exchange: ONE kernel per batch
// Flat receive buffer of a rank (symmetric on every rank, two of them alternate):
//   [ header: int64 M[PART_MAX_DEST][PART_MAX_DEST], M[s][d] = rows source s sends to destination d in this batch ]
//   [ ops: cap bytes ][ column k: cap * width_k bytes ]                      (each part 256-byte aligned)
// Every source publishes its count row M[me][*] into EVERY rank's header, a cross-rank barrier makes the matrix
// complete, and each source then knows where its rows belong inside every destination's buffer:
//   first row of (s -> d) = sum over s' < s of M[s'][d]
// so the scatter stores the rows over NVLink straight into their FINAL, contiguous place (source-rank order, row order
// kept inside a source): nothing is unpacked on the receiving side, the consumer reads the buffer as it is.  A second
// barrier tells every rank that its buffer is complete.  hist -> scan -> publish -> barrier -> scatter -> barrier are the
// phases of one launch (grid-wide barriers in between, see soft_grid_sync), replacing six launches and the unpack copy.
struct FlatLayout {
  int64_t cap;  // rows a buffer can hold (the caller sizes it for world x batch rows: every batch fits)
  int64_t ops_off;
  int64_t col_off[RW_MAX_COLS];
  int64_t total_bytes;
  int n_cols;
  int col_width[RW_MAX_COLS];
};
#define FLAT_HEADER_BYTES ((int64_t)PART_MAX_DEST * PART_MAX_DEST * 8)

static int flat_layout(const int32_t* types, int n_cols, int64_t cap_rows, FlatLayout* L) {
  if (n_cols < 0 || n_cols > RW_MAX_COLS || cap_rows <= 0) return fail(RW_ERR_INVALID, "flat layout");
  auto up = [](int64_t x) { return (x + 255) / 256 * 256; };
  int64_t off = FLAT_HEADER_BYTES;
  L->cap = cap_rows;
  L->n_cols = n_cols;
  L->ops_off = off;
  off = up(off + cap_rows);
  for (int k = 0; k < n_cols; k++) {
    int w = type_width(types[k]);
    if (!w || type_is_varlen(types[k])) return fail(RW_ERR_UNSUPPORTED, "column type");
    L->col_width[k] = w;
    L->col_off[k] = off;
    off = up(off + cap_rows * w);
  }
  L->total_bytes = off;
  return RW_OK;
}

// signal every rank, wait for every rank (thread t <-> rank t); bounded: a peer that never arrives (a rank that died,
// kernels that cannot run side by side) raises bit 1 of *err instead of hanging the GPU
__device__ __forceinline__ void flat_barrier(const PeerBases& flags, int n, int my_rank, unsigned long long value, int* err) {
  const int t = threadIdx.x;
  if (t < n) {
    __threadfence_system();
    unsigned long long* remote = (unsigned long long*)flags.base[t] + my_rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(remote), "l"(value) : "memory");
    const unsigned long long* mine = (const unsigned long long*)flags.base[my_rank] + t;
    unsigned long long v;
    const long long t0 = clock64();
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory");
      if (v < value && clock64() - t0 > 20000000000ll) { atomicOr(err, 2); break; }  // ~10 s
    } while (v < value);
  }
}

// grid-wide barrier of a PLAIN launch whose grid is sized to be resident (flat_exchange_kernel): `bar` counts arrivals
// and is never reset inside a launch -- barrier number k (1, 2, ...) waits for k * gridDim.x.  A cooperative launch
// (grid.sync()) costs more per launch and cannot start before EVERY block fits; this
// one starts with the blocks that fit and the rest follow as a neighbour kernel drains.
__device__ __forceinline__ void soft_grid_sync(unsigned int* bar, unsigned int k) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    const unsigned int target = k * gridDim.x;
    while (*(volatile unsigned int*)bar < target) __nanosleep(32);
    __threadfence();
  }
  __syncthreads();
}

// STAGED (every column 8 bytes wide): a tile's rows are first partitioned into SHARED MEMORY (stable, destination by
// destination) and then written out with consecutive threads storing consecutive rows of a destination's segment -- a
// warp's store instruction covers 256 contiguous bytes of ONE peer instead of 8-byte pieces scattered over all of them
// (per-row peer stores reach a small fraction of NVLink's bandwidth).  Otherwise rows go out one by one.
#define FLAT_TILE 1024
template <bool STAGED>
__global__ void __launch_bounds__(PART_BLOCK) flat_exchange_kernel(DevChunk ch, VnodePlan p, const int32_t* vnode_to_dest, int n_dest, int my_rank,
                                                                    FlatLayout L, PeerBases peers, PeerBases flags, unsigned long long epoch,
                                                                    uint8_t* dest, uint32_t* block_hist, uint32_t* tile_cnt, int n_vblocks,
                                                                    int64_t* counts, int64_t* total_dev, int64_t* total_host, int* err,
                                                                    unsigned int* bar, int coop) {
  extern __shared__ __align__(16) uint8_t s_stage[];  // STAGED: ops[FLAT_TILE] | col k: u64[FLAT_TILE]
  __shared__ uint32_t tab[256];
  __shared__ uint32_t hist[PART_MAX_DEST];
  __shared__ uint32_t run[PART_MAX_DEST];
  __shared__ uint32_t warp_cnt[PART_BLOCK / 32][PART_MAX_DEST];
  __shared__ uint32_t s_seg[PART_MAX_DEST + 1];  // STAGED: first staged row of destination d in this tile
  __shared__ int64_t s_first[PART_MAX_DEST];     // first row of (me -> d) inside d's buffer
  const int lane = lane_id(), wid = threadIdx.x >> 5;
  constexpr int ITERS = FLAT_TILE / PART_BLOCK;
  tab[threadIdx.x] = crc_table_entry(threadIdx.x);
  // ---- phase A: destination per row + per-tile histograms
  for (int vb = blockIdx.x; vb < n_vblocks; vb += gridDim.x) {
    if (threadIdx.x < PART_MAX_DEST) hist[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)vb * FLAT_TILE;
    uint8_t dv[ITERS];
#pragma unroll
    for (int it = 0; it < ITERS; it++) {  // (the tile's loads are independent: issued together)
      const int64_t r = base + it * PART_BLOCK + threadIdx.x;
      dv[it] = 255;
      if (r < ch.n) {
        const uint8_t op = ch.ops[r];
        if (row_visible(ch, r, op)) dv[it] = (uint8_t)vnode_to_dest[row_vnode(tab, p, ch, r, true)];
      }
    }
#pragma unroll
    for (int it = 0; it < ITERS; it++) {
      const int64_t r = base + it * PART_BLOCK + threadIdx.x;
      if (r < ch.n) {
        dest[r] = dv[it];
        if (dv[it] != 255) atomicAdd(&hist[dv[it]], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x < n_dest) {
      block_hist[(size_t)vb * n_dest + threadIdx.x] = hist[threadIdx.x];
      tile_cnt[(size_t)vb * n_dest + threadIdx.x] = hist[threadIdx.x];
    }
    __syncthreads();
  }
  if (coop) cooperative_groups::this_grid().sync(); else soft_grid_sync(bar, 1u);
  // ---- phase B (block 0): exclusive scan over the tiles per destination, count row to every rank, barrier 1
  if (blockIdx.x == 0) {
    for (int d = wid; d < n_dest; d += PART_BLOCK / 32) {
      uint32_t acc = 0;
      for (int b0 = 0; b0 < n_vblocks; b0 += 32) {
        const int b = b0 + lane;
        const uint32_t v = b < n_vblocks ? block_hist[(size_t)b * n_dest + d] : 0u;
        uint32_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += t;
        }
        if (b < n_vblocks) block_hist[(size_t)b * n_dest + d] = acc + inc - v;
        acc += __shfl_sync(0xffffffffu, inc, 31);
      }
      if (lane == 0) counts[d] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_dest * n_dest; i += PART_BLOCK) {  // M[me][d] into rank q's header
      const int q = i / n_dest, d = i % n_dest;
      int64_t* M = (int64_t*)peers.base[q];
      M[(size_t)my_rank * PART_MAX_DEST + d] = counts[d];
    }
    __syncthreads();
    flat_barrier(flags, n_dest, my_rank, 2ull * epoch - 1ull, err);
  }
  if (coop) cooperative_groups::this_grid().sync(); else soft_grid_sync(bar, 2u);
  // ---- phase C: stable scatter into the final place
  {
    const volatile int64_t* M = (const volatile int64_t*)peers.base[my_rank];
    if (threadIdx.x < n_dest) {
      int64_t first = 0;
      for (int s2 = 0; s2 < my_rank; s2++) first += M[(size_t)s2 * PART_MAX_DEST + threadIdx.x];
      s_first[threadIdx.x] = first;
    }
    __syncthreads();
  }
  uint8_t* s_ops = s_stage;
  unsigned long long* s_col = (unsigned long long*)(s_stage + FLAT_TILE);
  for (int vb = blockIdx.x; vb < n_vblocks; vb += gridDim.x) {
    if (threadIdx.x < PART_MAX_DEST) run[threadIdx.x] = 0;
    if (STAGED && threadIdx.x == 0) {
      uint32_t acc = 0;
      for (int d = 0; d < n_dest; d++) { s_seg[d] = acc; acc += tile_cnt[(size_t)vb * n_dest + d]; }
      s_seg[n_dest] = acc;
    }
    __syncthreads();
    const int64_t base = (int64_t)vb * FLAT_TILE;
    for (int it = 0; it < ITERS; it++) {
      const int64_t r = base + it * PART_BLOCK + threadIdx.x;
      const uint8_t d = (r < ch.n) ? dest[r] : 255;
      const unsigned peers_m = __match_any_sync(0xffffffffu, (unsigned)d);
      const unsigned rank_in_warp = __popc(peers_m & ((1u << lane) - 1));
      for (int k = lane; k < n_dest; k += 32) warp_cnt[wid][k] = 0;
      __syncwarp();
      if (rank_in_warp == 0 && d != 255) warp_cnt[wid][d] = __popc(peers_m);
      __syncthreads();
      uint32_t pos = 0;
      if (d != 255) {
        uint32_t before = 0;
        for (int w = 0; w < wid; w++) before += warp_cnt[w][d];
        pos = run[d] + before + rank_in_warp;
      }
      __syncthreads();
      if (threadIdx.x < n_dest) {
        uint32_t tot = 0;
        for (int w = 0; w < PART_BLOCK / 32; w++) tot += warp_cnt[w][threadIdx.x];
        run[threadIdx.x] += tot;
      }
      if (d != 255) {
        if (STAGED) {
          const uint32_t at = s_seg[d] + pos;
          s_ops[at] = ch.ops[r];
          for (int k = 0; k < ch.n_cols; k++) s_col[(size_t)k * FLAT_TILE + at] = ((const unsigned long long*)ch.cols[k].data)[r];
        } else {
          const int64_t dst = s_first[d] + (int64_t)block_hist[(size_t)vb * n_dest + d] + pos;
          if (dst >= L.cap) {
            atomicOr(err, 1);
          } else {
            uint8_t* buf = peers.base[d];
            buf[L.ops_off + dst] = ch.ops[r];
            for (int k = 0; k < ch.n_cols; k++) {
              const ColRef& c = ch.cols[k];
              uint8_t* col = buf + L.col_off[k];
              switch (c.width) {
                case 1: ((uint8_t*)col)[dst] = ((const uint8_t*)c.data)[r]; break;
                case 2: ((uint16_t*)col)[dst] = ((const uint16_t*)c.data)[r]; break;
                case 4: ((uint32_t*)col)[dst] = ((const uint32_t*)c.data)[r]; break;
                case 8: ((uint64_t*)col)[dst] = ((const uint64_t*)c.data)[r]; break;
                default: ((ulonglong2*)col)[dst] = ((const ulonglong2*)c.data)[r]; break;
              }
            }
          }
        }
      }
      __syncthreads();
    }
    if (STAGED) {  // write the staged tile out: consecutive threads, consecutive rows of a destination's segment
      const uint32_t staged = s_seg[n_dest];
      for (uint32_t i = threadIdx.x; i < staged; i += PART_BLOCK) {
        int d = 0;
        while (d + 1 < n_dest && i >= s_seg[d + 1]) d++;
        const int64_t dst = s_first[d] + (int64_t)block_hist[(size_t)vb * n_dest + d] + (int64_t)(i - s_seg[d]);
        if (dst >= L.cap) { atomicOr(err, 1); continue; }
        uint8_t* buf = peers.base[d];
        buf[L.ops_off + dst] = s_ops[i];
        for (int k = 0; k < ch.n_cols; k++) ((unsigned long long*)(buf + L.col_off[k]))[dst] = s_col[(size_t)k * FLAT_TILE + i];
      }
      __syncthreads();  // the staging area is refilled by the next tile
    }
  }
  __threadfence_system();
  if (coop) cooperative_groups::this_grid().sync(); else soft_grid_sync(bar, 3u);
  // ---- phase D (block 0): barrier 2, then the received row count for the consumer
  if (blockIdx.x == 0) {
    flat_barrier(flags, n_dest, my_rank, 2ull * epoch, err);
    __syncthreads();
    if (threadIdx.x == 0) {
      const volatile int64_t* M = (const volatile int64_t*)peers.base[my_rank];
      int64_t total = 0;
      for (int s2 = 0; s2 < n_dest; s2++) total += M[(size_t)s2 * PART_MAX_DEST + my_rank];
      if (*(volatile int*)err) total = -1;
      *total_dev = total;
      if (total_host) { *total_host = total; __threadfence_system(); }
    }
  }
}

static int make_vnode_plan(const rw_chunk* c, const int32_t* keys, int n_keys, int vnode_count, VnodePlan* p) {
  if (n_keys < 1 || n_keys > RW_MAX_KEYS * 2) return fail(RW_ERR_UNSUPPORTED, "1..8 distribution key columns");
  if (vnode_count < 1 || vnode_count > 32768) return fail(RW_ERR_INVALID, "vnode_count (vnode.rs:79 MAX_COUNT = 2^15)");
  p->n_keys = n_keys;
  for (int k = 0; k < c->n_cols; k++)
    if (type_is_varlen(c->columns[k].type)) return fail(RW_ERR_UNSUPPORTED, "the hash shuffle does not carry varlen columns");
  for (int k = 0; k < n_keys; k++) {
    if (keys[k] < 0 || keys[k] >= c->n_cols) return fail(RW_ERR_INVALID, "key index");
    p->key_col[k] = keys[k];
  }
  p->vnode_count = vnode_count;
  p->serial_fast = (n_keys == 1 && c->columns[keys[0]].type == RW_T_SERIAL) ? 1 : 0;
  return RW_OK;
}

static int grid_rows(int64_t n, int block) {
  int64_t g = (n + block - 1) / block;
  return (int)std::max<int64_t>(1, std::min<int64_t>(g, RW_SMS * 8));
}

// upload a HOST rw_chunk into one temporary device allocation
int upload_chunk(const rw_chunk* c, DevBuf& buf, DevChunk* out, cudaStream_t st) {
  if (c->n_cols > RW_MAX_COLS) return fail(RW_ERR_UNSUPPORTED, "too many columns");
  int64_t n = c->n_rows;
  size_t nw = (size_t)((n + 63) / 64) * 8;
  size_t total = 256 + (size_t)n + nw;
  for (int k = 0; k < c->n_cols; k++) {
    int w = type_width(c->columns[k].type);
    if (!w) return fail(RW_ERR_UNSUPPORTED, "column type");
    total += 256 + (size_t)n * w + 256 + nw;
  }
  RW_CUDA(buf.reserve(total + 1024));
  uint8_t* d = buf.as<uint8_t>();
  size_t off = 0;
  auto put = [&](const void* src, size_t bytes) -> const void* {
    if (!src) return nullptr;
    size_t o = (off + 255) / 256 * 256;
    cudaMemcpyAsync(d + o, src, bytes, cudaMemcpyHostToDevice, st);
    off = o + bytes;
    return d + o;
  };
  memset(out, 0, sizeof(*out));
  out->n = n;
  out->n_cols = c->n_cols;
  out->ops = (const uint8_t*)put(c->ops, (size_t)n);
  out->vis_bits = (const uint64_t*)put(c->visibility, nw);
  for (int k = 0; k < c->n_cols; k++) {
    int w = type_width(c->columns[k].type);
    out->cols[k].type = c->columns[k].type;
    out->cols[k].width = w;
    // (a varlen payload column is not uploaded: no kernel behind this helper touches columns it does not reference)
    out->cols[k].data = type_is_varlen(c->columns[k].type) ? nullptr : put(c->columns[k].data, (size_t)n * w);
    out->cols[k].valid_bits = (const uint64_t*)put(c->columns[k].validity, nw);
  }
  RW_CUDA(cudaGetLastError());
  return RW_OK;
}

}  // namespace rw

using namespace rw;

extern "C" {

int32_t rwgpu_vnode_compute(const rw_chunk* c, const int32_t* keys, int32_t n_keys, int32_t vnode_count, uint16_t* out) {
  if (!c || !keys || !out) return fail(RW_ERR_INVALID, "null");
  int rc = rwgpu_device_check();
  if (rc != RW_OK) return rc;
  VnodePlan p;
  rc = make_vnode_plan(c, keys, n_keys, vnode_count, &p);
  if (rc != RW_OK) return rc;
  if (c->n_rows == 0) return RW_OK;
  DevBuf buf, dout;
  DevChunk ch;
  rc = upload_chunk(c, buf, &ch, 0);
  if (rc != RW_OK) return rc;
  RW_CUDA(dout.reserve((size_t)c->n_rows * 2));
  vnode_kernel<<<grid_rows(c->n_rows, 256), 256>>>(ch, p, dout.as<uint16_t>());
  RW_CUDA(cudaGetLastError());
  RW_CUDA(cudaMemcpy(out, dout.p, (size_t)c->n_rows * 2, cudaMemcpyDeviceToHost));
  return RW_OK;
}

int32_t rwgpu_dispatch_rewrite_ops(const rw_chunk* c, const int32_t* keys, int32_t n_keys, uint8_t* out_ops) {
  if (!c || !keys || !out_ops) return fail(RW_ERR_INVALID, "null");
  int rc = rwgpu_device_check();
  if (rc != RW_OK) return rc;
  VnodePlan p;
  rc = make_vnode_plan(c, keys, n_keys, 256, &p);
  if (rc != RW_OK) return rc;
  if (c->n_rows == 0) return RW_OK;
  DevBuf buf, dout;
  DevChunk ch;
  rc = upload_chunk(c, buf, &ch, 0);
  if (rc != RW_OK) return rc;
  RW_CUDA(dout.reserve((size_t)c->n_rows + 16));
  unsigned int* err = (unsigned int*)(dout.as<uint8_t>() + ((size_t)c->n_rows + 7) / 8 * 8);
  RW_CUDA(cudaMemset(dout.p, 0, (size_t)c->n_rows + 16));
  dispatch_rewrite_kernel<<<grid_rows(c->n_rows, 256), 256>>>(ch, p, dout.as<uint8_t>(), err);
  RW_CUDA(cudaGetLastError());
  RW_CUDA(cudaMemcpy(out_ops, dout.p, (size_t)c->n_rows, cudaMemcpyDeviceToHost));
  unsigned int e = 0;
  RW_CUDA(cudaMemcpy(&e, err, 4, cudaMemcpyDeviceToHost));
  if (e & 1u) return fail(RW_ERR_INCONSISTENT, "missing U- before U+");
  if (e & 2u) return fail(RW_ERR_INCONSISTENT, "missing U+ after U-");
  return RW_OK;
}

int32_t rwgpu_shuffle_partition_device(const rw_chunk* c, const int32_t* keys, int32_t n_keys, int32_t vnode_count,
                                       const int32_t* vnode_to_dest, int32_t n_dest, uint8_t* out_ops,
                                       void* const* out_cols, uint8_t* const* out_valid_bytes, int64_t* counts,
                                       int64_t* offsets, void* cuda_stream) {
  if (!c || !keys || !vnode_to_dest || !out_ops || !out_cols || !counts || !offsets) return fail(RW_ERR_INVALID, "null");
  if (n_dest < 1 || n_dest > PART_MAX_DEST) return fail(RW_ERR_UNSUPPORTED, "1..64 destinations");
  for (int k = 0; k < c->n_cols; k++)
    if (c->columns[k].validity && !(out_valid_bytes && out_valid_bytes[k]))
      return fail(RW_ERR_UNSUPPORTED, "a column carries a validity bitmap but no out_valid_bytes buffer was given for it");
  VnodePlan p;
  int rc = make_vnode_plan(c, keys, n_keys, vnode_count, &p);
  if (rc != RW_OK) return rc;
  DevChunk ch;
  rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  int n_blocks = (int)std::max<int64_t>(1, (c->n_rows + PART_ROWS_PER_BLOCK - 1) / PART_ROWS_PER_BLOCK);
  // scratch: dest bytes + block histograms (stream-ordered allocation)
  uint8_t* scratch = nullptr;
  size_t dest_bytes = ((size_t)c->n_rows + 255) / 256 * 256;
  size_t hist_bytes = (size_t)n_blocks * n_dest * 4;
  RW_CUDA(cudaMallocAsync((void**)&scratch, dest_bytes + hist_bytes + 256, st));
  uint8_t* dest = scratch;
  uint32_t* hist = (uint32_t*)(scratch + dest_bytes);
  part_hist_kernel<<<n_blocks, PART_BLOCK, 0, st>>>(ch, p, vnode_to_dest, n_dest, dest, hist);
  part_scan_kernel<<<1, PART_SCAN_THREADS, 0, st>>>(hist, n_blocks, n_dest, counts, offsets);
  PartOut o;
  memset(&o, 0, sizeof(o));
  o.ops = out_ops;
  for (int k = 0; k < c->n_cols; k++) {
    o.col[k] = out_cols[k];
    o.valid[k] = out_valid_bytes ? out_valid_bytes[k] : nullptr;
  }
  part_scatter_kernel<<<n_blocks, PART_BLOCK, 0, st>>>(ch, dest, hist, n_dest, offsets, o);
  RW_CUDA(cudaGetLastError());
  RW_CUDA(cudaFreeAsync(scratch, st));
  return RW_OK;
}


int32_t rwgpu_shuffle_p2p_region_bytes(const int32_t* types, int32_t n_cols, int64_t cap_rows, int64_t* region_bytes) {
  if (!types || !region_bytes) return fail(RW_ERR_INVALID, "null");
  P2PLayout L;
  int rc = p2p_layout(types, n_cols, cap_rows, &L);
  if (rc != RW_OK) return rc;
  *region_bytes = L.region_bytes;
  return RW_OK;
}

int32_t rwgpu_shuffle_partition_p2p_device(const rw_chunk* c, const int32_t* keys, int32_t n_keys, int32_t vnode_count,
                                           const int32_t* vnode_to_dest, int32_t n_dest, int32_t my_rank,
                                           void* const* peer_bases, int64_t cap_rows, int64_t* counts, int32_t* overflow,
                                           void* cuda_stream) {
  if (!c || !keys || !vnode_to_dest || !peer_bases || !counts || !overflow) return fail(RW_ERR_INVALID, "null");
  if (n_dest < 1 || n_dest > PART_MAX_DEST || my_rank < 0 || my_rank >= n_dest) return fail(RW_ERR_INVALID, "ranks");
  // the receive regions carry ops + column data only: a validity bitmap would be dropped and NULLs arrive as garbage
  for (int k = 0; k < c->n_cols; k++)
    if (c->columns[k].validity) return fail(RW_ERR_UNSUPPORTED, "the peer-memory exchange does not carry validity bitmaps");
  VnodePlan p;
  int rc = make_vnode_plan(c, keys, n_keys, vnode_count, &p);
  if (rc != RW_OK) return rc;
  DevChunk ch;
  rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  std::vector<int32_t> types(c->n_cols);
  for (int k = 0; k < c->n_cols; k++) types[k] = c->columns[k].type;
  P2PLayout L;
  rc = p2p_layout(types.data(), c->n_cols, cap_rows, &L);
  if (rc != RW_OK) return rc;
  PeerBases pb;
  memset(&pb, 0, sizeof(pb));
  for (int d = 0; d < n_dest; d++) pb.base[d] = (uint8_t*)peer_bases[d];
  cudaStream_t st = (cudaStream_t)cuda_stream;
  int n_blocks = (int)std::max<int64_t>(1, (c->n_rows + PART_ROWS_PER_BLOCK - 1) / PART_ROWS_PER_BLOCK);
  uint8_t* scratch = nullptr;
  size_t dest_bytes = ((size_t)c->n_rows + 255) / 256 * 256;
  size_t hist_bytes = (size_t)n_blocks * n_dest * 4;
  RW_CUDA(cudaMallocAsync((void**)&scratch, dest_bytes + hist_bytes + 1024, st));
  uint8_t* dest = scratch;
  uint32_t* hist = (uint32_t*)(scratch + dest_bytes);
  int64_t* offsets = (int64_t*)(scratch + dest_bytes + (hist_bytes + 255) / 256 * 256);
  part_hist_kernel<<<n_blocks, PART_BLOCK, 0, st>>>(ch, p, vnode_to_dest, n_dest, dest, hist);
  part_scan_kernel<<<1, PART_SCAN_THREADS, 0, st>>>(hist, n_blocks, n_dest, counts, offsets);
  part_scatter_p2p_kernel<<<n_blocks, PART_BLOCK, 0, st>>>(ch, dest, hist, n_dest, L, pb, my_rank, overflow);
  p2p_publish_counts_kernel<<<1, PART_MAX_DEST, 0, st>>>(counts, n_dest, L, pb, my_rank);
  RW_CUDA(cudaGetLastError());
  RW_CUDA(cudaFreeAsync(scratch, st));
  return RW_OK;
}

int32_t rwgpu_shuffle_exchange_p2p_device(const rw_chunk* c, const int32_t* keys, int32_t n_keys, int32_t vnode_count,
                                          const int32_t* vnode_to_dest, int32_t n_dest, int32_t my_rank,
                                          void* const* peer_bases, void* const* peer_flags, uint64_t epoch, int64_t cap_rows,
                                          const void* recv_base, uint8_t* out_ops, void* const* out_cols, int64_t* counts,
                                          int32_t* overflow, int64_t* total_host, void* cuda_stream) {
  if (!peer_flags || !recv_base || !out_ops || !out_cols || !total_host || !c) return fail(RW_ERR_INVALID, "null");
  int rc = rwgpu_shuffle_partition_p2p_device(c, keys, n_keys, vnode_count, vnode_to_dest, n_dest, my_rank, peer_bases, cap_rows,
                                              counts, overflow, cuda_stream);
  if (rc != RW_OK) return rc;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  PeerBases pf;
  memset(&pf, 0, sizeof(pf));
  for (int d = 0; d < n_dest; d++) pf.base[d] = (uint8_t*)peer_flags[d];
  p2p_barrier_kernel<<<1, PART_MAX_DEST, 0, st>>>(pf, n_dest, my_rank, (unsigned long long)epoch);
  RW_CUDA(cudaGetLastError());
  std::vector<int32_t> types(c->n_cols);
  for (int k = 0; k < c->n_cols; k++) types[k] = c->columns[k].type;
  // the device-side row count lives behind the flags of this rank's block: byte 512 + 8 * (epoch & 1)
  // (two slots, so that a consumer of batch e may still read its count while batch e+1 is unpacked)
  int64_t* total_dev = (int64_t*)((uint8_t*)peer_flags[my_rank] + sizeof(uint64_t) * (PART_MAX_DEST + (epoch & 1)));
  rc = rwgpu_shuffle_unpack_device(recv_base, n_dest, types.data(), c->n_cols, cap_rows, out_ops, out_cols, total_dev, cuda_stream);
  if (rc != RW_OK) return rc;
  p2p_total_to_host_kernel<<<1, 1, 0, st>>>(total_dev, total_host);
  RW_CUDA(cudaGetLastError());
  return RW_OK;
}

int32_t rwgpu_shuffle_unpack_device(const void* recv_base, int32_t n_src, const int32_t* types, int32_t n_cols, int64_t cap_rows,
                                    uint8_t* out_ops, void* const* out_cols, int64_t* total, void* cuda_stream) {
  if (!recv_base || !types || !out_ops || !out_cols || !total) return fail(RW_ERR_INVALID, "null");
  if (n_src < 1 || n_src > PART_MAX_DEST) return fail(RW_ERR_INVALID, "n_src");
  P2PLayout L;
  int rc = p2p_layout(types, n_cols, cap_rows, &L);
  if (rc != RW_OK) return rc;
  PartOut o;
  memset(&o, 0, sizeof(o));
  for (int k = 0; k < n_cols; k++) o.col[k] = out_cols[k];
  p2p_unpack_kernel<<<RW_SMS * 4, 256, 0, (cudaStream_t)cuda_stream>>>((const uint8_t*)recv_base, n_src, L, out_ops, o, total);
  RW_CUDA(cudaGetLastError());
  return RW_OK;
}

int32_t rwgpu_shuffle_flat_layout(const int32_t* types, int32_t n_cols, int64_t cap_rows, int64_t* total_bytes, int64_t* ops_off,
                                  int64_t* col_off) {
  if (!types || !total_bytes || !ops_off || !col_off) return fail(RW_ERR_INVALID, "null");
  FlatLayout L;
  int rc = flat_layout(types, n_cols, cap_rows, &L);
  if (rc != RW_OK) return rc;
  *total_bytes = L.total_bytes;
  *ops_off = L.ops_off;
  for (int k = 0; k < n_cols; k++) col_off[k] = L.col_off[k];
  return RW_OK;
}

int32_t rwgpu_shuffle_exchange_flat_device(const rw_chunk* c, const int32_t* keys, int32_t n_keys, int32_t vnode_count,
                                           const int32_t* vnode_to_dest, int32_t n_dest, int32_t my_rank, void* const* peer_bases,
                                           void* const* peer_flags, uint64_t epoch, int64_t cap_rows, int64_t* counts, int32_t* err,
                                           int64_t* total_dev, int64_t* total_host, int32_t max_blocks, void* cuda_stream) {
  if (!c || !keys || !vnode_to_dest || !peer_bases || !peer_flags || !counts || !err || !total_dev) return fail(RW_ERR_INVALID, "null");
  if (n_dest < 1 || n_dest > PART_MAX_DEST || my_rank < 0 || my_rank >= n_dest) return fail(RW_ERR_INVALID, "ranks");
  if (epoch == 0) return fail(RW_ERR_INVALID, "epochs start at 1");
  for (int k = 0; k < c->n_cols; k++)
    if (c->columns[k].validity) return fail(RW_ERR_UNSUPPORTED, "the peer-memory exchange does not carry validity bitmaps");
  VnodePlan p;
  int rc = make_vnode_plan(c, keys, n_keys, vnode_count, &p);
  if (rc != RW_OK) return rc;
  DevChunk ch;
  rc = devchunk_from_abi(c, &ch);
  if (rc != RW_OK) return rc;
  std::vector<int32_t> types(c->n_cols);
  for (int k = 0; k < c->n_cols; k++) types[k] = c->columns[k].type;
  FlatLayout L;
  rc = flat_layout(types.data(), c->n_cols, cap_rows, &L);
  if (rc != RW_OK) return rc;
  PeerBases pb, pf;
  memset(&pb, 0, sizeof(pb));
  memset(&pf, 0, sizeof(pf));
  for (int d = 0; d < n_dest; d++) { pb.base[d] = (uint8_t*)peer_bases[d]; pf.base[d] = (uint8_t*)peer_flags[d]; }
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const int n_vblocks = (int)std::max<int64_t>(1, (c->n_rows + FLAT_TILE - 1) / FLAT_TILE);
  bool staged = c->n_cols <= 12;
  for (int k = 0; k < c->n_cols; k++) staged = staged && type_width(c->columns[k].type) == 8;
  const size_t smem = staged ? (size_t)FLAT_TILE * (1 + 8 * (size_t)c->n_cols) : 0;
  // every block resident at once (the grid-wide barriers rely on it): occupancy x SMs, at most 3 blocks per SM
  static int coresident[2][13] = {{0}};
  int& cores = coresident[staged ? 1 : 0][staged ? c->n_cols : 0];
  if (!cores) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (staged) {
      if (smem > 48 * 1024) RW_CUDA(cudaFuncSetAttribute(flat_exchange_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(FLAT_TILE * (1 + 8 * 12))));
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flat_exchange_kernel<true>, PART_BLOCK, smem);
    } else {
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flat_exchange_kernel<false>, PART_BLOCK, 0);
    }
    // at most three blocks per SM, so that the join's kernel keeps SM slots beside the exchange
    cores = std::max(1, sms * std::max(1, std::min(per_sm, 3)));
  }
  int grid = std::min(n_vblocks, cores);
  if (max_blocks > 0) grid = std::min(grid, (int)max_blocks);
  uint8_t* scratch = nullptr;
  size_t dest_bytes = ((size_t)c->n_rows + 255) / 256 * 256;
  size_t hist_bytes = ((size_t)n_vblocks * n_dest * 4 + 255) / 256 * 256;
  RW_CUDA(cudaMallocAsync((void**)&scratch, dest_bytes + 2 * hist_bytes + 512, st));
  uint8_t* dest = scratch;
  uint32_t* hist = (uint32_t*)(scratch + dest_bytes);
  uint32_t* tcnt = (uint32_t*)(scratch + dest_bytes + hist_bytes);
  unsigned int* bar = (unsigned int*)(scratch + dest_bytes + 2 * hist_bytes);
  RW_CUDA(cudaMemsetAsync(bar, 0, 4, st));
  // RWGPU_EXCHANGE_COOP=1: cooperative launch (grid.sync()) instead of the software barriers -- the whole grid starts at
  // once, and the join's kernel fills in around it
  static const int coop = getenv("RWGPU_EXCHANGE_COOP") ? atoi(getenv("RWGPU_EXCHANGE_COOP")) : 0;
  int coop_arg = coop;
  unsigned long long ep = epoch;
  int* errp = (int*)err;
  int nvb = n_vblocks;
  void* args[] = {(void*)&ch, (void*)&p, (void*)&vnode_to_dest, (void*)&n_dest, (void*)&my_rank, (void*)&L, (void*)&pb, (void*)&pf, (void*)&ep,
                  (void*)&dest, (void*)&hist, (void*)&tcnt, (void*)&nvb, (void*)&counts, (void*)&total_dev, (void*)&total_host, (void*)&errp,
                  (void*)&bar, (void*)&coop_arg};
  const void* fn = staged ? (const void*)flat_exchange_kernel<true> : (const void*)flat_exchange_kernel<false>;
  if (coop) RW_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(PART_BLOCK), args, smem, st));
  else RW_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(PART_BLOCK), args, smem, st));
  RW_CUDA(cudaGetLastError());
  RW_CUDA(cudaFreeAsync(scratch, st));
  return RW_OK;
}

}  // extern "C"
