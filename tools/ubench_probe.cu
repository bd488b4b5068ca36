// ubench_probe.cu -- build the join probe up from the raw random-load baseline to find what costs time.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/ubench_probe tools/ubench_probe.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }
struct Cols { const uint64_t* c[4]; uint64_t* o[8]; uint8_t* ops; uint8_t* vis; };

// V=0: random 16B load from 64B buckets, key generated           (baseline)
// V=1: + all four 16B loads of the bucket
// V=2: + key read from a column (coalesced)
// V=3: + 4 update columns read (coalesced)
// V=4: + 8 output columns + ops + vis written (coalesced)
// V=5: like 4, 2 rows per thread interleaved
template <int V>
__global__ void __launch_bounds__(256) k(const ulonglong2* tab, uint64_t mask, int64_t n, Cols cs, unsigned long long* sink) {
  unsigned long long acc = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t key = V >= 2 ? __ldg(cs.c[0] + r) : mix64((uint64_t)r ^ 99);
    uint64_t u1 = 0, u2 = 0, u3 = 0;
    if (V >= 3) { u1 = __ldg(cs.c[1] + r); u2 = __ldg(cs.c[2] + r); u3 = __ldg(cs.c[3] + r); }
    const ulonglong2* bp = tab + (mix64(key) & mask) * 4;
    ulonglong2 a = __ldcg(bp), b = {0, 0}, c = {0, 0}, d = {0, 0};
    if (V >= 1) { b = __ldcg(bp + 1); c = __ldcg(bp + 2); d = __ldcg(bp + 3); }
    if (V >= 4) {
      cs.ops[r] = 1; cs.vis[r] = (uint8_t)(a.x & 1);
      cs.o[0][r] = key; cs.o[1][r] = u1; cs.o[2][r] = u2; cs.o[3][r] = u3;
      cs.o[4][r] = c.x; cs.o[5][r] = c.y; cs.o[6][r] = d.x; cs.o[7][r] = d.y + b.x;
    } else acc += a.x + a.y + b.x + b.y + c.x + c.y + d.x + d.y + u1 + u2 + u3;
  }
  if (acc == 0x1234567) *sink = acc;
}

template <int V> void run(const char* name, int grid, ulonglong2* tab, uint64_t buckets, int64_t n, Cols cs, unsigned long long* sink) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<V><<<grid, 256>>>(tab, buckets - 1, n, cs, sink);
  cudaEventRecord(a);
  for (int it = 0; it < 5; it++) k<V><<<grid, 256>>>(tab, buckets - 1, n, cs, sink);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
  printf("%-52s grid %5d  %7.1f us per 2^20 rows  (%.2f G rows/s)\n", name, grid, ms * 1e3 * (1 << 20) / n, n / ms / 1e6);
}

int main() {
  unsigned long long* sink; cudaMalloc(&sink, 8);
  const uint64_t buckets = 1ull << 25;  // 2 GB of 64 B buckets
  ulonglong2* tab; cudaMalloc(&tab, buckets * 64); cudaMemset(tab, 1, buckets * 64);
  const int64_t n = 1 << 22;
  Cols cs;
  for (int i = 0; i < 4; i++) { uint64_t* p; cudaMalloc(&p, n * 8); cudaMemset(p, i + 1, n * 8); cs.c[i] = p; }
  for (int i = 0; i < 8; i++) cudaMalloc(&cs.o[i], n * 8);
  cudaMalloc(&cs.ops, n); cudaMalloc(&cs.vis, n);
  // make the key column pseudo-random
  {
    uint64_t* h = (uint64_t*)malloc(n * 8);
    for (int64_t i = 0; i < n; i++) { uint64_t x = i * 0x9E3779B97F4A7C15ull; x ^= x >> 31; h[i] = x; }
    cudaMemcpy((void*)cs.c[0], h, n * 8, cudaMemcpyHostToDevice); free(h);
  }
  for (int grid : {132 * 8, 132 * 16, (int)(n / 256)}) {
    run<0>("V0 random 16B load from 64B bucket", grid, tab, buckets, n, cs, sink);
    run<1>("V1 + whole 64B bucket (4 x 16B)", grid, tab, buckets, n, cs, sink);
    run<2>("V2 + key from column", grid, tab, buckets, n, cs, sink);
    run<3>("V3 + 3 more update columns", grid, tab, buckets, n, cs, sink);
    run<4>("V4 + write 8 out cols + ops + vis", grid, tab, buckets, n, cs, sink);
  }
  return 0;
}
