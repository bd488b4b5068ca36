// ubench_bucket.cu -- how should one thread (or a few lanes) touch a random 64-byte bucket in HBM?
// ubench_probe showed 4 x LDG.128 of one bucket costs 3.5x one LDG.128.  This measures the alternatives:
// 32-byte accesses (sm_90 has no 256-bit load: two 16-byte instructions on one sector), lane-cooperative access,
// and the insert-side sequences.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/ubench_bucket tools/ubench_bucket.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }
struct U4 { uint64_t a, b, c, d; };
__device__ __forceinline__ U4 ld256(const void* p) {
  U4 v;
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%4];\n\tld.global.cg.v2.u64 {%2,%3}, [%4+16];"
               : "=l"(v.a), "=l"(v.b), "=l"(v.c), "=l"(v.d) : "l"(p));
  return v;
}
__device__ __forceinline__ void st256(void* p, U4 v) {
  asm volatile("st.global.cg.v2.u64 [%0], {%1,%2};\n\tst.global.cg.v2.u64 [%0+16], {%3,%4};"
               ::"l"(p), "l"(v.a), "l"(v.b), "l"(v.c), "l"(v.d) : "memory");
}
__device__ __forceinline__ bool cas128(void* addr, ulonglong2 expect, ulonglong2 desired, ulonglong2* found) {
  asm volatile(
      "{\n\t.reg .b128 e, d, f;\n\tmov.b128 e, {%2, %3};\n\tmov.b128 d, {%4, %5};\n\t"
      "atom.global.relaxed.gpu.cas.b128 f, [%6], e, d;\n\tmov.b128 {%0, %1}, f;\n\t}"
      : "=l"(found->x), "=l"(found->y)
      : "l"(expect.x), "l"(expect.y), "l"(desired.x), "l"(desired.y), "l"(addr)
      : "memory");
  return found->x == expect.x && found->y == expect.y;
}
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) { return __shfl_sync(0xffffffffu, (unsigned long long)v, src); }

enum { L_16 = 0, L_4x16, L_2x32, L_1x32, L_PF_4x16, L_COOP4, L_COOP2, S_3x16, S_16_32, S_COOP4, S_CAS128, S_LD_CAS128, S_CAS128_ST, S_CAS128_CAS64,
       C_PROBE_INSERT, C_PROBE_INSERT_OLD, NV };

template <int V>
__global__ void __launch_bounds__(256) k(uint8_t* tab, uint8_t* tab2, uint64_t mask, int64_t n, unsigned long long* sink, uint64_t salt) {
  unsigned long long acc = 0;
  const int lane = threadIdx.x & 31;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t key = mix64((uint64_t)r ^ salt);
    uint8_t* bp = tab + (mix64(key) & mask) * 64;
    uint8_t* wp = tab2 + (mix64(key ^ 0x5555) & mask) * 64;
    if (V == L_16) { ulonglong2 a = __ldcg((const ulonglong2*)bp); acc += a.x + a.y; }
    if (V == L_4x16 || V == L_PF_4x16) {
      if (V == L_PF_4x16) asm volatile("prefetch.global.L2 [%0];" ::"l"(bp));
      ulonglong2 a = __ldcg((const ulonglong2*)bp), b = __ldcg((const ulonglong2*)bp + 1), c = __ldcg((const ulonglong2*)bp + 2), d = __ldcg((const ulonglong2*)bp + 3);
      acc += a.x + a.y + b.x + b.y + c.x + c.y + d.x + d.y;
    }
    if (V == L_2x32) { U4 a = ld256(bp), b = ld256(bp + 32); acc += a.a + a.b + a.c + a.d + b.a + b.b + b.c + b.d; }
    if (V == L_1x32) { U4 a = ld256(bp); acc += a.a + a.b + a.c + a.d; }
    if (V == L_COOP4) {
      // round t: the 8 rows owned by lanes 8t..8t+7; lane l loads piece l%4 of the bucket of owner 8t + l/4
      uint64_t w[8];
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const uint64_t obp = shfl64((uint64_t)bp, 8 * t + (lane >> 2));
        const ulonglong2 v = __ldcg((const ulonglong2*)(obp + 16 * (lane & 3)));
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const uint64_t x = shfl64(v.x, 4 * (lane & 7) + q), y = shfl64(v.y, 4 * (lane & 7) + q);
          if ((lane >> 3) == t) { w[2 * q] = x; w[2 * q + 1] = y; }
        }
      }
      acc += w[0] + w[1] + w[2] + w[3] + w[4] + w[5] + w[6] + w[7];
    }
    if (V == L_COOP2) {
      uint64_t w[8];
#pragma unroll
      for (int t = 0; t < 2; t++) {
        const uint64_t obp = shfl64((uint64_t)bp, 16 * t + (lane >> 1));
        const U4 v = ld256((const void*)(obp + 32 * (lane & 1)));
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const int src = 2 * (lane & 15) + q;
          const uint64_t a = shfl64(v.a, src), b = shfl64(v.b, src), c = shfl64(v.c, src), d = shfl64(v.d, src);
          if ((lane >> 4) == t) { w[4 * q] = a; w[4 * q + 1] = b; w[4 * q + 2] = c; w[4 * q + 3] = d; }
        }
      }
      acc += w[0] + w[1] + w[2] + w[3] + w[4] + w[5] + w[6] + w[7];
    }
    if (V == S_3x16) {
      ulonglong2 v = {key, (uint64_t)r};
      __stcg((ulonglong2*)wp + 1, v); __stcg((ulonglong2*)wp + 2, v); __stcg((ulonglong2*)wp + 3, v);
    }
    if (V == S_16_32) {
      ulonglong2 v = {key, (uint64_t)r};
      __stcg((ulonglong2*)wp + 1, v);
      st256(wp + 32, U4{key, key, key, (uint64_t)r});
    }
    if (V == S_COOP4) {
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const uint64_t obp = shfl64((uint64_t)wp, 8 * t + (lane >> 2));
        const uint64_t k2 = shfl64(key, 8 * t + (lane >> 2));
        ulonglong2 v = {k2, (uint64_t)lane};
        if ((lane & 3) != 0) __stcg((ulonglong2*)(obp + 16 * (lane & 3)), v);
      }
    }
    if (V == S_CAS128 || V == S_CAS128_ST || V == S_CAS128_CAS64) {
      ulonglong2 e = {0x0101010101010101ull, 0x0101010101010101ull}, d = {key, 1}, f;
      const bool ok = cas128(wp, e, d, &f);
      acc += f.x;
      if (V == S_CAS128_ST) {
        ulonglong2 v = {key, (uint64_t)r};
        __stcg((ulonglong2*)wp + 1, v);
        st256(wp + 32, U4{key, key, key, (uint64_t)r});
      }
      if (V == S_CAS128_CAS64) {
        acc += atomicCAS((unsigned long long*)wp + 1, (unsigned long long)f.y, (unsigned long long)(f.y + (1ull << 33)));
      }
      (void)ok;
    }
    if (V == S_LD_CAS128) {
      ulonglong2 cur = __ldcg((const ulonglong2*)wp), d = {key, 1}, f;
      cas128(wp, cur, d, &f);
      acc += f.x;
    }
    if (V == C_PROBE_INSERT) {
      // proposed: probe = 2 x 32B loads; insert = CAS128 + 16B hdr store + 32B payload store
      U4 a = ld256(bp), b = ld256(bp + 32);
      ulonglong2 e = {0x0101010101010101ull, 0x0101010101010101ull}, d = {key, 1}, f;
      cas128(wp, e, d, &f);
      ulonglong2 v = {key, (uint64_t)r};
      __stcg((ulonglong2*)wp + 1, v);
      st256(wp + 32, U4{a.a + f.x, b.b, b.c + a.c, (uint64_t)r});
    }
    if (V == C_PROBE_INSERT_OLD) {
      // current kernel: probe 4 x 16B; prefetch + 16B load + CAS128 + 3 x 16B stores
      asm volatile("prefetch.global.L2 [%0];" ::"l"(wp));
      ulonglong2 a = __ldcg((const ulonglong2*)bp), b = __ldcg((const ulonglong2*)bp + 1), c = __ldcg((const ulonglong2*)bp + 2), d4 = __ldcg((const ulonglong2*)bp + 3);
      ulonglong2 cur = __ldcg((const ulonglong2*)wp), d = {key, 1}, f;
      cas128(wp, cur, d, &f);
      ulonglong2 v = {key + a.x + b.x, (uint64_t)r + c.x + d4.x + f.x};
      __stcg((ulonglong2*)wp + 1, v); __stcg((ulonglong2*)wp + 2, v); __stcg((ulonglong2*)wp + 3, v);
    }
  }
  if (acc == 0x1234567) *sink = acc;
}

template <int V> void run(const char* name, int grid, uint8_t* tab, uint8_t* tab2, uint64_t buckets, int64_t n, unsigned long long* sink) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<V><<<grid, 256>>>(tab, tab2, buckets - 1, n, sink, 1);
  cudaEventRecord(a);
  for (int it = 0; it < 5; it++) k<V><<<grid, 256>>>(tab, tab2, buckets - 1, n, sink, 100 + it);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
  cudaError_t e = cudaGetLastError();
  printf("%-58s %7.1f us per 2^20 rows  (%.2f G rows/s) %s\n", name, ms * 1e3 * (1 << 20) / n, n / ms / 1e6, e == cudaSuccess ? "" : cudaGetErrorString(e));
}

int main() {
  unsigned long long* sink; cudaMalloc(&sink, 8);
  const uint64_t buckets = 1ull << 25;  // 2 GB of 64 B buckets, twice
  uint8_t *tab, *tab2; cudaMalloc(&tab, buckets * 64); cudaMemset(tab, 1, buckets * 64);
  cudaMalloc(&tab2, buckets * 64); cudaMemset(tab2, 1, buckets * 64);
  const int64_t n = 1 << 22;
  const int grid = 132 * 16;
  run<L_16>("L  1 x 16B load", grid, tab, tab2, buckets, n, sink);
  run<L_4x16>("L  4 x 16B loads (current probe)", grid, tab, tab2, buckets, n, sink);
  run<L_PF_4x16>("L  prefetch.L2 + 4 x 16B loads", grid, tab, tab2, buckets, n, sink);
  run<L_1x32>("L  1 x 32B load (LDG.256)", grid, tab, tab2, buckets, n, sink);
  run<L_2x32>("L  2 x 32B loads", grid, tab, tab2, buckets, n, sink);
  run<L_COOP4>("L  4 lanes x 16B cooperative + shuffles", grid, tab, tab2, buckets, n, sink);
  run<L_COOP2>("L  2 lanes x 32B cooperative + shuffles", grid, tab, tab2, buckets, n, sink);
  run<S_3x16>("S  3 x 16B stores (current record write)", grid, tab, tab2, buckets, n, sink);
  run<S_16_32>("S  16B + 32B stores", grid, tab, tab2, buckets, n, sink);
  run<S_COOP4>("S  3 of 4 lanes x 16B cooperative stores", grid, tab, tab2, buckets, n, sink);
  run<S_CAS128>("S  CAS128 alone (speculative claim)", grid, tab, tab2, buckets, n, sink);
  run<S_LD_CAS128>("S  16B load + CAS128 (current claim)", grid, tab, tab2, buckets, n, sink);
  run<S_CAS128_ST>("S  CAS128 + 16B + 32B stores (proposed insert)", grid, tab, tab2, buckets, n, sink);
  run<S_CAS128_CAS64>("S  CAS128 + CAS64 (existing key)", grid, tab, tab2, buckets, n, sink);
  run<C_PROBE_INSERT_OLD>("C  current probe + insert sequence", grid, tab, tab2, buckets, n, sink);
  run<C_PROBE_INSERT>("C  proposed probe + insert sequence", grid, tab, tab2, buckets, n, sink);
  return 0;
}
