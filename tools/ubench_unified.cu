// ubench_unified.cu -- prototype of the round-2 join step: ONE table whose 64-byte bucket holds the key, the
// state words of BOTH sides and the inline record of the build side, so that a probe-side row's probe and its
// own-side insert touch the SAME line (2 random DRAM transactions per row instead of 3), with the row itself
// appended to a sequential record log.  Variants measure where the own-side chain head should live:
//   A  head+count word inside the bucket (CAS64 on the line the probe just loaded)
//   B  heads in a separate dense 4-byte array indexed by bucket number (64 MB: L2-resident?), atomicExch
//   B' same with L2 evict_last on the heads and evict_first on every stream / the bucket loads
//   C  probe + emit only (read-only floor)
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/ubench_unified tools/ubench_unified.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) { return __shfl_sync(0xffffffffu, (unsigned long long)v, src); }

__device__ __forceinline__ uint64_t mkpolicy_last() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t mkpolicy_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ ulonglong2 ld128_hint(const void* p, uint64_t pol) {
  ulonglong2 v;
  asm volatile("ld.global.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint64_t ld64_hint(const void* p, uint64_t pol) {
  uint64_t v;
  asm volatile("ld.global.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st64_hint(void* p, uint64_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st128_hint(void* p, ulonglong2 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.u64 [%0], {%1,%2}, %3;" ::"l"(p), "l"(v.x), "l"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ uint32_t exch32_hint(uint32_t* p, uint32_t v, uint64_t pol) {
  uint32_t o;
  asm volatile("atom.global.exch.L2::cache_hint.b32 %0, [%1], %2, %3;" : "=r"(o) : "l"(p), "r"(v), "l"(pol) : "memory");
  return o;
}

enum { V_A = 0, V_B, V_BH, V_C, V_A_NOREC, V_B_NOOUT, NV };

struct Args {
  const uint8_t* ops;
  const uint64_t* col[4];   // col[0] = key
  uint64_t* out[8];
  uint8_t* out_ops;
  uint8_t* out_vis;
  uint8_t* tab;             // buckets, 64 B each: key | W_R | W_L | hdr | 4 cols
  uint32_t* heads;          // variant B
  uint8_t* log;             // record log, 48 B records: {link, seq, key..} 16 B hdr + 32 B cols
  uint64_t mask;
  int64_t n;
  uint32_t log_base;
};

template <int V, int MINB>
__global__ void __launch_bounds__(256, MINB) k(Args a, unsigned long long* sink) {
  const int lane = threadIdx.x & 31, q = lane & 3, qlead = lane & ~3;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t groups = (a.n + 7) >> 3;
  const bool hint = (V == V_BH);
  uint64_t pl = 0, pf = 0;
  if (hint) { pl = mkpolicy_last(); pf = mkpolicy_first(); }
  // lanes 0,1 stream update columns (0,1)/(2,3); lanes 2,3 write matched columns
  const int ca = 2 * (q & 1), cb = ca + 1;
  const uint64_t* pa = a.col[ca];
  const uint64_t* pb = a.col[cb];
  uint64_t* po0 = a.out[(q < 2 ? 0 : 4) + ca];
  uint64_t* po1 = a.out[(q < 2 ? 0 : 4) + cb];
  unsigned long long acc = 0;
  // this warp's slice of the record log: 8 records per group, contiguous (stands for the per-warp id pools)
  for (int64_t g = warp_global; g < groups; g += nwarps) {
    const int64_t r = g * 8 + (lane >> 2);
    const bool in = r < a.n;
    uint8_t op = 0;
    uint64_t key = 0, va = 0, vb = 0;
    if (in) {
      op = a.ops[r];
      if (hint) { key = ld64_hint(a.col[0] + r, pf); va = ld64_hint(pa + r, pf); vb = ld64_hint(pb + r, pf); }
      else { key = __ldg(a.col[0] + r); va = __ldg(pa + r); vb = __ldg(pb + r); }
    }
    const uint64_t b = mix64(key) & a.mask;
    uint8_t* bp = a.tab + b * 64;
    // probe: lane q loads 16 bytes of the bucket
    ulonglong2 pv;
    if (hint) pv = ld128_hint(bp + 16 * q, pf);
    else pv = __ldcg((const ulonglong2*)(bp + 16 * q));
    const uint64_t bkey = shfl64(pv.x, qlead), WR = shfl64(pv.y, qlead);
    const uint64_t WL = shfl64(pv.x, qlead + 1);
    const uint64_t m0 = shfl64(pv.x, qlead + 2), m1 = shfl64(pv.y, qlead + 2), m2 = shfl64(pv.x, qlead + 3), m3 = shfl64(pv.y, qlead + 3);
    const uint64_t ma = q == 3 ? m2 : m0, mb = q == 3 ? m3 : m1;
    acc += bkey + WR;
    // emit (positional)
    if (V != V_B_NOOUT && in) {
      if (q == 0) a.out_ops[r] = op;
      if (q == 1) a.out_vis[r] = 1;
      if (hint) { st64_hint(po0 + r, q < 2 ? va : ma, pf); st64_hint(po1 + r, q < 2 ? vb : mb, pf); }
      else { po0[r] = q < 2 ? va : ma; po1[r] = q < 2 ? vb : mb; }
    }
    if (V == V_C) continue;
    // own-side append: record id = position in the log (sequential), link = previous head
    const uint32_t row = a.log_base + (uint32_t)r;
    uint32_t link = 0;
    if (in && q == 0) {
      if (V == V_A || V == V_A_NOREC) {
        unsigned long long cur = WL;
        while (true) {
          const unsigned long long nw = ((cur + (1ull << 32)) & ~0xffffffffull) | row;
          const unsigned long long old = atomicCAS((unsigned long long*)(bp + 16), cur, nw);
          if (old == cur) break;
          cur = old;
        }
        link = (uint32_t)cur;
      } else if (V == V_BH) {
        link = exch32_hint(a.heads + b, row, pl);
      } else {
        link = atomicExch(a.heads + b, row);
      }
    }
    link = __shfl_sync(0xffffffffu, link, qlead);
    if (V != V_A_NOREC && in && q != 0) {
      ulonglong2 v;
      if (q == 1) { v.x = link; v.y = (uint64_t)r; }
      else { v.x = va; v.y = vb; }
      uint8_t* rp = a.log + (uint64_t)row * 48 + 16 * (q - 1);
      if (hint) st128_hint(rp, v, pf);
      else *(ulonglong2*)rp = v;
    }
  }
  if (acc == 0x1234567) *sink = acc;
}

static uint64_t hmix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }

__global__ void fill_cols(uint64_t* key, uint64_t* c1, uint64_t* c2, uint64_t* c3, uint8_t* ops, int64_t n, uint64_t salt, uint64_t nkeys) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    key[i] = mix64((uint64_t)i ^ salt) % nkeys;
    c1[i] = i; c2[i] = i * 3; c3[i] = i * 7; ops[i] = 1;
  }
}

template <int V, int MINB> void run(const char* name, int grid, Args a, int nbatch, int64_t n, unsigned long long* sink, bool window, cudaStream_t st) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  // each batch: fresh inputs (different key salt) -> regenerate outside the timed region; we time kernels only
  float tot = 0;
  for (int it = 0; it < nbatch + 2; it++) {
    fill_cols<<<592, 256, 0, st>>>((uint64_t*)a.col[0], (uint64_t*)a.col[1], (uint64_t*)a.col[2], (uint64_t*)a.col[3], (uint8_t*)a.ops, n, 1000 + it, 10000000ull);
    a.log_base = (uint32_t)(it * n);
    cudaEventRecord(e0, st);
    k<V, MINB><<<grid, 256, 0, st>>>(a, sink);
    cudaEventRecord(e1, st);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (it >= 2) tot += ms;
  }
  cudaError_t e = cudaGetLastError();
  const float ms = tot / nbatch;
  printf("%-64s grid %5d  %7.1f us per 2^20 rows  (%.2f G rows/s, %.0f GB/s algorithmic)%s %s\n", name, grid, ms * 1e3 * (1 << 20) / n, n / ms / 1e6,
         194.125 * n / ms / 1e6, window ? " [persisting window]" : "", e == cudaSuccess ? "" : cudaGetErrorString(e));
}

int main(int argc, char** argv) {
  unsigned long long* sink; cudaMalloc(&sink, 8);
  const uint64_t buckets = 1ull << 24;  // 1 GB of 64-byte buckets
  const int64_t n = 1 << 20;
  const int nb = 12;
  Args a;
  uint8_t* tab; cudaMalloc(&tab, buckets * 64); cudaMemset(tab, 1, buckets * 64);
  uint32_t* heads; cudaMalloc(&heads, buckets * 4); cudaMemset(heads, 0xff, buckets * 4);
  uint8_t* log; cudaMalloc(&log, (size_t)(nb + 2) * n * 48 * 2);
  uint64_t* cols[4]; for (int c = 0; c < 4; c++) cudaMalloc(&cols[c], n * 8);
  uint8_t* ops; cudaMalloc(&ops, n);
  for (int c = 0; c < 8; c++) cudaMalloc(&a.out[c], n * 8);
  cudaMalloc(&a.out_ops, n); cudaMalloc(&a.out_vis, n);
  a.ops = ops; for (int c = 0; c < 4; c++) a.col[c] = cols[c];
  a.tab = tab; a.heads = heads; a.log = log; a.mask = buckets - 1; a.n = n; a.log_base = 0;
  cudaStream_t st; cudaStreamCreate(&st);
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  printf("L2 %d MB, persistingL2CacheMaxSize %d MB, accessPolicyMaxWindowSize %d MB\n", prop.l2CacheSize >> 20, prop.persistingL2CacheMaxSize >> 20,
         prop.accessPolicyMaxWindowSize >> 20);
  for (int grid : {132 * 4, 132 * 8}) {
    run<V_C, 4>("C  probe + emit only (no own-side insert)", grid, a, nb, n, sink, false, st);
    run<V_A, 4>("A  unified bucket: CAS64 on W_L in the probed line + log append", grid, a, nb, n, sink, false, st);
    run<V_A_NOREC, 4>("A- same without the log append", grid, a, nb, n, sink, false, st);
    run<V_B, 4>("B  heads[] 64 MB side array: atomicExch + log append", grid, a, nb, n, sink, false, st);
    run<V_BH, 4>("B' same, evict_last on heads / evict_first on streams+buckets", grid, a, nb, n, sink, false, st);
    run<V_B_NOOUT, 4>("B- heads variant without output stores", grid, a, nb, n, sink, false, st);
  }
  run<V_A, 8>("A  (8 blocks/SM, 32 regs)", 132 * 8, a, nb, n, sink, false, st);
  run<V_B, 8>("B  (8 blocks/SM, 32 regs)", 132 * 8, a, nb, n, sink, false, st);
  // persisting-L2 window on the heads array
  size_t want = (size_t)buckets * 4;
  if (prop.persistingL2CacheMaxSize > 0) {
    cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, std::min<size_t>(want, (size_t)prop.persistingL2CacheMaxSize));
    cudaStreamAttrValue attr;
    attr.accessPolicyWindow.base_ptr = heads;
    attr.accessPolicyWindow.num_bytes = std::min<size_t>(want, (size_t)prop.accessPolicyMaxWindowSize);
    attr.accessPolicyWindow.hitRatio = 1.0f;
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    cudaError_t e = cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr);
    printf("access policy window: %s\n", cudaGetErrorString(e));
    run<V_B, 4>("B  heads[] with persisting access-policy window", 132 * 4, a, nb, n, sink, true, st);
    run<V_B, 4>("B  heads[] with persisting access-policy window", 132 * 8, a, nb, n, sink, true, st);
    run<V_A, 4>("A  (window set on heads: control)", 132 * 4, a, nb, n, sink, true, st);
  }
  return 0;
}
