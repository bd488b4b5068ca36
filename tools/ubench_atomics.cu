// ubench_atomics.cu -- random-access load / atomic throughput on a table much larger than L2 (H100).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/ubench_atomics tools/ubench_atomics.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }

template <int MODE>
__global__ void k(ulonglong2* tab, uint64_t mask, uint64_t n, uint64_t seed, unsigned long long* sink) {
  unsigned long long acc = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t idx = mix64(i ^ seed) & mask;
    ulonglong2* p = tab + idx;
    if (MODE == 0) { ulonglong2 v = __ldcg(p); acc += v.x + v.y; }                                     // 16B load
    if (MODE == 1) { atomicAdd((unsigned int*)p, 1u); }                                                 // RED 32
    if (MODE == 2) { acc += atomicExch((unsigned int*)p, (unsigned int)i); }                            // ATOM exch 32
    if (MODE == 3) { acc += atomicCAS((unsigned long long*)p, 0ull, (unsigned long long)i); }           // CAS 64
    if (MODE == 4) { ulonglong2 v = __ldcg(p); acc += atomicExch((unsigned int*)p + 2, (unsigned int)i) + v.x; atomicAdd((unsigned int*)p + 3, 1u); }  // load + exch + red (our insert)
    if (MODE == 5) { ulonglong2 v; v.x = i; v.y = i; *p = v; }                                           // 16B store
    if (MODE == 6) { atomicAdd((unsigned long long*)p, 1ull); atomicAdd((unsigned long long*)p + 1, i); atomicMax((long long*)p + 1, (long long)i); }  // 3 RED 64 same sector... (agg-like: 2 sectors)
    if (MODE == 7) { acc += atomicAdd((unsigned long long*)p, 1ull); }                                  // ATOM add 64 w/ return
    if (MODE == 8) { atomicAdd((unsigned long long*)p, 1ull); }                                          // RED add 64
    if (MODE == 9) {   // dependent: load, then CAS64 + CAS32 + ADD32 on the same line (current insert protocol, new key)
      ulonglong2 v = __ldcg(p);
      unsigned long long o = atomicCAS((unsigned long long*)p, v.x, v.x + 1);
      unsigned int o2 = atomicCAS((unsigned int*)p + 2, (unsigned int)v.y, (unsigned int)(v.y + (o & 1)));
      atomicAdd((unsigned int*)p + 3, 1u + (o2 & 1));
    }
    if (MODE == 10) {  // dependent: load, then ONE CAS64
      ulonglong2 v = __ldcg(p);
      acc += atomicCAS((unsigned long long*)p + 1, v.y, v.y + 1 + (v.x & 1));
    }
    if (MODE == 11) {  // dependent: load, then ONE CAS128
      ulonglong2 v = __ldcg(p);
      unsigned long long o0, o1;
      asm volatile("{\n .reg .b128 c, d, o;\n mov.b128 c, {%2, %3};\n mov.b128 d, {%4, %5};\n atom.global.cas.b128 o, [%6], c, d;\n mov.b128 {%0, %1}, o;\n}"
                   : "=l"(o0), "=l"(o1) : "l"(v.x), "l"(v.y), "l"(v.x + 1), "l"(v.y + 1), "l"(p) : "memory");
      acc += o0 + o1;
    }
    if (MODE == 12) {  // dependent: load, then plain 16B store (exclusive-owner update)
      ulonglong2 v = __ldcg(p);
      v.x += 1; v.y += 1;
      *p = v;
    }
    if (MODE == 13) {  // load16, then ONE EXCH64 of head | (count + 1) << 32; RED only when the count moved meanwhile (insert)
      ulonglong2 v = __ldcg(p);
      const unsigned int L = (unsigned int)(v.y >> 32);
      const unsigned long long old = atomicExch((unsigned long long*)p + 1, (unsigned long long)(unsigned int)i | ((unsigned long long)(L + 1u) << 32));
      const unsigned int C = (unsigned int)(old >> 32);
      if (C != L) atomicAdd((unsigned int*)p + 3, C - L);
      acc += (unsigned int)old + v.x;
    }
  }
  if (acc == 0x1234567) *sink = acc;
}

template <int MODE> void run(const char* name, ulonglong2* tab, uint64_t slots, uint64_t n, unsigned long long* sink) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<132 * 8, 256>>>(tab, slots - 1, n, 1, sink);
  cudaEventRecord(a);
  for (int it = 0; it < 3; it++) k<MODE><<<132 * 8, 256>>>(tab, slots - 1, n, 77 + it, sink);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); ms /= 3;
  printf("%-34s table %5.0f MB  %7.2f G ops/s  (%.3f ms for %llu ops)\n", name, slots * 16.0 / 1e6, n / ms / 1e6, ms, (unsigned long long)n);
}

int main() {
  unsigned long long* sink; cudaMalloc(&sink, 8);
  if (getenv("UBENCH_SWEEP")) {  // footprint sweep at the join's bucket-table sizes (1, 2, 4 GiB): TLB reach, DRAM pages
    for (uint64_t slots : {1ull << 26, 1ull << 27, 1ull << 28}) {
      ulonglong2* tab; if (cudaMalloc(&tab, slots * 16) != cudaSuccess) break; cudaMemset(tab, 0, slots * 16);
      uint64_t n = 1ull << 24;
      run<0>("16B load (ld.cg)", tab, slots, n, sink);
      run<12>("load -> store16", tab, slots, n, sink);
      run<13>("load16 + EXCH64 (+RED if moved)", tab, slots, n, sink);
      cudaFree(tab);
    }
    return 0;
  }
  for (uint64_t slots : {1ull << 22, 1ull << 26}) {   // 64 MB (L2-resident) and 1 GB
    ulonglong2* tab; cudaMalloc(&tab, slots * 16); cudaMemset(tab, 0, slots * 16);
    uint64_t n = 1ull << 24;
    run<0>("16B load (ld.cg)", tab, slots, n, sink);
    run<5>("16B store", tab, slots, n, sink);
    run<1>("RED.ADD u32", tab, slots, n, sink);
    run<8>("RED.ADD u64", tab, slots, n, sink);
    run<7>("ATOM.ADD u64 (return)", tab, slots, n, sink);
    run<2>("ATOM.EXCH u32", tab, slots, n, sink);
    run<3>("ATOM.CAS u64", tab, slots, n, sink);
    run<4>("load16 + EXCH32 + RED32 (insert)", tab, slots, n, sink);
    run<13>("load16 + EXCH64 (+RED if moved)", tab, slots, n, sink);
    run<6>("3x RED u64 one slot (agg)", tab, slots, n, sink);
    run<9>("load -> CAS64 + CAS32 + ADD32", tab, slots, n, sink);
    run<10>("load -> CAS64", tab, slots, n, sink);
    run<11>("load -> CAS128", tab, slots, n, sink);
    run<12>("load -> store16", tab, slots, n, sink);
    cudaFree(tab);
  }
  return 0;
}
