// common.cuh -- shared host/device helpers for librwgpu (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/rwgpu.h"

namespace rw {

// ------------------------------------------------------------------ errors
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
const char* last_error_cstr();

#define RW_CUDA(expr)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return ::rw::fail(RW_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// streaming multiprocessors of the H100 SXM; grid-stride kernels cap their grids at RW_SMS x 8 blocks of
// 256 threads (2048 resident threads per SM)
#define RW_SMS 132

int type_width(int t);
bool type_is_float(int t);
bool type_is_varlen(int t);
bool type_supported(int t);
// the operand rule of join conditions and filter terms (api.cu): may `a cmp b` compare the two raw integers?
bool cmp_operands_ok(int a, int b);

// ------------------------------------------------------------------ device buffer (RAII)
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
  // grow-only allocation; contents are NOT preserved
  cudaError_t reserve(size_t n) {
    if (n <= bytes) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&p, n);
    if (e == cudaSuccess) bytes = n; else p = nullptr;
    return e;
  }
  template <class T> T* as() const { return (T*)p; }
};

// Device buffer that GROWS IN PLACE: a virtual address range is reserved once (cuMemAddressReserve)
// and physical memory is mapped behind it chunk by chunk (cuMemCreate / cuMemMap).  Join state
// keeps growing while the stream runs; growing a cudaMalloc'd store means allocating the doubled
// store, copying hundreds of MB and freeing the old one in the middle of the data path, growing
// this one touches no existing byte and keeps every device pointer valid.  The driver entry points
// are looked up at run time (cudaGetDriverEntryPoint), so the library has no link dependency on
// libcuda and still loads on a machine without a driver.  If the VMM API is unavailable the buffer
// degrades to allocate-copy-free.
struct VmmApi {
  bool ok = false;
  CUresult (*AddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*AddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*Create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*Release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*Map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*Unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*SetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*GetGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
};
const VmmApi& vmm_api();  // api.cu

struct GrowBuf {
  CUdeviceptr base = 0;
  size_t reserved = 0, mapped = 0, gran = 0;
  int dev = 0;
  std::vector<std::pair<CUmemGenericAllocationHandle, size_t>> chunks;
  DevBuf plain;          // fallback storage
  bool use_vmm = false, decided = false;
  GrowBuf() {}
  GrowBuf(const GrowBuf&) = delete;
  GrowBuf& operator=(const GrowBuf&) = delete;
  ~GrowBuf() { release(); }
  void swap(GrowBuf& o) {
    std::swap(base, o.base); std::swap(reserved, o.reserved); std::swap(mapped, o.mapped); std::swap(gran, o.gran);
    std::swap(dev, o.dev); chunks.swap(o.chunks); std::swap(use_vmm, o.use_vmm); std::swap(decided, o.decided);
    DevBuf t = std::move(plain); plain = std::move(o.plain); o.plain = std::move(t);
  }
  void* p() const { return use_vmm ? (void*)base : plain.p; }
  size_t bytes() const { return use_vmm ? mapped : plain.bytes; }
  template <class T> T* as() const { return (T*)p(); }
  void release() {
    if (use_vmm) {
      const VmmApi& a = vmm_api();
      size_t off = 0;
      for (auto& c : chunks) {
        a.Unmap(base + off, c.second);
        a.Release(c.first);
        off += c.second;
      }
      chunks.clear();
      if (base) a.AddressFree(base, reserved);
      base = 0; reserved = 0; mapped = 0;
    }
    plain.release();
  }
  // make at least `need` bytes usable; the first `live` bytes keep their contents (always true for
  // the VMM path; the fallback copies them on `st`).  `va_limit` bounds the address reservation.
  cudaError_t ensure(size_t need, size_t live, size_t va_limit, cudaStream_t st) {
    if (need <= bytes()) return cudaSuccess;
    if (!decided) {
      decided = true;
      const VmmApi& a = vmm_api();
      if (a.ok && cudaGetDevice(&dev) == cudaSuccess) {
        CUmemAllocationProp prop;
        memset(&prop, 0, sizeof(prop));
        prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
        prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        prop.location.id = dev;
        size_t g = 0;
        if (a.GetGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) == CUDA_SUCCESS && g) {
          gran = g;
          size_t want = (std::max(va_limit, need) + gran - 1) / gran * gran;
          if (a.AddressReserve(&base, want, 0, 0, 0) == CUDA_SUCCESS) {
            reserved = want;
            use_vmm = true;
          }
        }
      }
    }
    if (use_vmm) {
      if (need > reserved) return cudaErrorMemoryAllocation;
      const VmmApi& a = vmm_api();
      // geometric growth in mapped chunks (amortises the map calls), never below the granularity
      size_t add = std::max(need - mapped, std::max(mapped / 2, gran));
      add = std::min((add + gran - 1) / gran * gran, reserved - mapped);
      CUmemAllocationProp prop;
      memset(&prop, 0, sizeof(prop));
      prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
      prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      prop.location.id = dev;
      CUmemGenericAllocationHandle hnd;
      CUresult r = a.Create(&hnd, add, &prop, 0);
      if (r != CUDA_SUCCESS && add > (need - mapped + gran - 1) / gran * gran) {  // retry with the bare minimum
        add = (need - mapped + gran - 1) / gran * gran;
        r = a.Create(&hnd, add, &prop, 0);
      }
      if (r != CUDA_SUCCESS) return cudaErrorMemoryAllocation;
      if (a.Map(base + mapped, add, 0, hnd, 0) != CUDA_SUCCESS) { a.Release(hnd); return cudaErrorMemoryAllocation; }
      CUmemAccessDesc acc;
      memset(&acc, 0, sizeof(acc));
      acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      acc.location.id = dev;
      acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      if (a.SetAccess(base + mapped, add, &acc, 1) != CUDA_SUCCESS) {
        a.Unmap(base + mapped, add);
        a.Release(hnd);
        return cudaErrorMemoryAllocation;
      }
      chunks.emplace_back(hnd, add);
      mapped += add;
      return cudaSuccess;
    }
    // fallback: allocate, copy the live prefix, free
    size_t ncap = std::max(need, plain.bytes * 2);
    DevBuf nb;
    cudaError_t e = nb.reserve(ncap);
    if (e != cudaSuccess) {
      ncap = need;
      e = nb.reserve(ncap);
      if (e != cudaSuccess) return e;
    }
    if (live && plain.p) {
      e = cudaMemcpyAsync(nb.p, plain.p, live, cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) return e;
      e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return e;
    }
    plain = std::move(nb);
    return cudaSuccess;
  }
};

struct PinnedBuf {
  void* p = nullptr;
  size_t bytes = 0;
  PinnedBuf() {}
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  ~PinnedBuf() { release(); }
  void release() { if (p) cudaFreeHost(p); p = nullptr; bytes = 0; }
  cudaError_t reserve(size_t n) {
    if (n <= bytes) return cudaSuccess;
    release();
    cudaError_t e = cudaMallocHost(&p, n);
    if (e == cudaSuccess) bytes = n; else p = nullptr;
    return e;
  }
  template <class T> T* as() const { return (T*)p; }
};

// ------------------------------------------------------------------ CUDA-event bracket of one kernel family
struct KernelProf {
  bool on = false;
  std::vector<cudaEvent_t> ev;  // pairs
  size_t used = 0;
  double ms = 0;
  uint64_t n = 0;
  ~KernelProf() { for (auto e : ev) cudaEventDestroy(e); }
  void begin(cudaStream_t st) {
    if (!on) return;
    if (used + 2 > ev.size()) { cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); ev.push_back(a); ev.push_back(b); }
    cudaEventRecord(ev[used], st);
  }
  void end(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(ev[used + 1], st);
    used += 2;
  }
  // caller has synchronised the stream(s)
  void collect() {
    for (size_t i = 0; i + 1 < used; i += 2) {
      float t = 0;
      if (cudaEventElapsedTime(&t, ev[i], ev[i + 1]) == cudaSuccess) { ms += t; n++; }
    }
    used = 0;
  }
};

// ------------------------------------------------------------------ device-side chunk view
#define RW_MAX_COLS 24
#define RW_MAX_KEYS 4
#define RW_MAX_CALLS 16

struct ColRef {
  const void* data;
  const uint64_t* valid_bits;  // LSB-first bitmap, or nullptr
  const uint8_t* valid_bytes;  // 1 byte / row, or nullptr
  int32_t type;
  int32_t width;
};

struct DevChunk {
  int64_t n;
  const uint8_t* ops;          // RW_OP_*; 0 = invisible (host staging folds visibility in)
  const uint64_t* vis_bits;    // or nullptr
  int32_t n_cols;
  int32_t pad;
  const int64_t* n_dev;        // or nullptr: the row count lives on the device (<= n, which is then the capacity)
  ColRef cols[RW_MAX_COLS];
};

// host: build a DevChunk from an rw_chunk whose pointers are DEVICE pointers
int devchunk_from_abi(const rw_chunk* c, DevChunk* out);
// host: upload a HOST rw_chunk into one temporary device allocation (shuffle.cu)
int upload_chunk(const rw_chunk* c, DevBuf& buf, DevChunk* out, cudaStream_t st);

// ------------------------------------------------------------------ output object (host side)
struct OutColHost {
  int type = 0;
  std::vector<uint8_t> data;
  std::vector<uint64_t> valid;  // packed per chunk on demand
  bool has_null = false;
};

}  // namespace rw

// pool of pinned host blocks backing the output objects (D2H at full PCIe rate, no page faults);
// shared between a handle and the outputs it produced so either may die first
struct PinnedBlock {
  uint8_t* p = nullptr;
  size_t bytes = 0;
};
struct PinnedPool {
  std::mutex mu;
  std::vector<PinnedBlock> free_blocks;
  ~PinnedPool() { for (auto& b : free_blocks) cudaFreeHost(b.p); }
  PinnedBlock get(size_t bytes) {
    {
      std::lock_guard<std::mutex> g(mu);
      for (size_t i = 0; i < free_blocks.size(); i++)
        if (free_blocks[i].bytes >= bytes) {
          PinnedBlock b = free_blocks[i];
          free_blocks.erase(free_blocks.begin() + i);
          return b;
        }
      if (!free_blocks.empty()) {  // drop a too-small block rather than hoarding
        cudaFreeHost(free_blocks.back().p);
        free_blocks.pop_back();
      }
    }
    PinnedBlock b;
    size_t want = bytes + bytes / 4 + 4096;
    if (cudaMallocHost((void**)&b.p, want) != cudaSuccess) { b.p = nullptr; b.bytes = 0; cudaGetLastError(); return b; }
    b.bytes = want;
    return b;
  }
  void put(PinnedBlock b) {
    if (!b.p) return;
    std::lock_guard<std::mutex> g(mu);
    if (free_blocks.size() >= 4) { cudaFreeHost(b.p); return; }
    free_blocks.push_back(b);
  }
};

// C-ABI output object: one super-chunk in pinned host memory + chunk views cut from it
struct rwgpu_out {
  int64_t n_rows = 0;
  int chunk_size = 1024;
  std::vector<int> types;
  uint8_t* ops = nullptr;
  uint8_t* vis_bytes = nullptr;            // nullptr = all visible
  std::vector<uint8_t*> data;              // per column, native width (varlen: the bytes, see var_bytes)
  std::vector<uint32_t*> offsets;          // per column: varlen offsets[n_rows + 1], nullptr for fixed-width columns
  std::vector<std::unique_ptr<rw::PinnedBuf>> var_store;
  uint8_t* var_bytes(size_t k, size_t bytes);
  std::vector<uint8_t*> valid_bytes;       // per column, nullptr = no NULLs
  PinnedBlock block;
  std::shared_ptr<PinnedPool> pool;
  // chunk cutting (StreamChunkBuilder rule: a U- is never the last row of a chunk)
  std::vector<int64_t> cut;  // chunk i = rows [cut[i], cut[i+1])
  // per-chunk packed bitmaps, built by finalize()
  std::vector<std::vector<uint64_t>> chunk_vis;
  std::vector<std::vector<std::vector<uint64_t>>> chunk_valid;
  std::vector<std::vector<rw_column>> chunk_cols;
  // carve ops / column / valid / vis regions for `rows` rows out of a pool block; false on OOM
  bool layout(int64_t rows, const std::vector<int>& col_types, unsigned long long null_mask, bool with_vis,
              const std::shared_ptr<PinnedPool>& pl);
  void finalize();
  ~rwgpu_out() { if (pool) pool->put(block); else if (block.p) cudaFreeHost(block.p); }
};

#ifdef __CUDACC__
namespace rw {

// ------------------------------------------------------------------ device helpers
__device__ __forceinline__ bool bit_get(const uint64_t* w, int64_t i) {
  return w == nullptr || ((w[i >> 6] >> (i & 63)) & 1ull);
}

// a chunk whose row count lives on the device (e.g. the output of the exchange): clamp the capacity.
// A count out of range is no rows; the kernel that reads the count first reports it (JERR_BAD_COUNT / AGG_ERR_BAD_COUNT).
__device__ __forceinline__ int64_t chunk_rows(const DevChunk& ch) {
  if (!ch.n_dev) return ch.n;
  const int64_t n = *ch.n_dev;
  return (n < 0 || n > ch.n) ? 0 : n;
}

__device__ __forceinline__ bool row_visible(const DevChunk& c, int64_t r, uint8_t op) {
  return op != 0 && (c.vis_bits == nullptr || ((c.vis_bits[r >> 6] >> (r & 63)) & 1ull));
}

__device__ __forceinline__ bool col_is_null(const ColRef& c, int64_t r) {
  if (c.valid_bits != nullptr && !((c.valid_bits[r >> 6] >> (r & 63)) & 1ull)) return true;
  if (c.valid_bytes != nullptr && c.valid_bytes[r] == 0) return true;
  return false;
}

// finalizer of murmur3 / splitmix64: the table hash (values never observable, SURVEY §0.2.1)
__device__ __host__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// sortable encoding of a double (total order, NaN canonical & largest, -0 == +0):
// mirrors Ord on OrderedFloat (src/common/src/types/ordered_float.rs)
__device__ __host__ __forceinline__ int64_t f64_sortable(double f) {
  if (f != f) return INT64_MAX;
  if (f == 0.0) f = 0.0;
  int64_t b;
#ifdef __CUDA_ARCH__
  b = __double_as_longlong(f);
#else
  memcpy(&b, &f, 8);
#endif
  return b < 0 ? (b ^ 0x7fffffffffffffffLL) : b;
}
__device__ __host__ __forceinline__ double f64_unsortable(int64_t s) {
  int64_t b = s < 0 ? (s ^ 0x7fffffffffffffffLL) : s;
#ifdef __CUDA_ARCH__
  return __longlong_as_double(b);
#else
  double f; memcpy(&f, &b, 8); return f;
#endif
}

// load column value r as a 64-bit word: ints sign-extended, floats as normalised double bits
// (HashKeySer: F32/F64 `normalized()`, -0 -> +0, canonical NaN; src/common/src/hash/key.rs:400-631)
__device__ __forceinline__ int64_t load_i64(const ColRef& c, int64_t r) {
  switch (c.width) {
    case 1: return (int64_t)((const uint8_t*)c.data)[r];
    case 2: return (int64_t)((const int16_t*)c.data)[r];
    case 4: return (int64_t)((const int32_t*)c.data)[r];
    default: return ((const int64_t*)c.data)[r];
  }
}
__device__ __forceinline__ double load_f64(const ColRef& c, int64_t r) {
  return c.type == RW_T_FLOAT32 ? (double)((const float*)c.data)[r] : ((const double*)c.data)[r];
}
__device__ __forceinline__ uint64_t load_key_word(const ColRef& c, int64_t r) {
  if (c.type == RW_T_FLOAT32 || c.type == RW_T_FLOAT64) {
    double f = load_f64(c, r);
    if (f != f) return 0x7ff8000000000000ull;
    if (f == 0.0) f = 0.0;
    return (uint64_t)__double_as_longlong(f);
  }
  return (uint64_t)load_i64(c, r);
}

// store a 64-bit word into an output column of native width
__device__ __forceinline__ void store_word(void* data, int width, int type, int64_t r, uint64_t w) {
  switch (width) {
    case 1: ((uint8_t*)data)[r] = (uint8_t)w; break;
    case 2: ((int16_t*)data)[r] = (int16_t)w; break;
    case 4:
      if (type == RW_T_FLOAT32) ((float*)data)[r] = (float)__longlong_as_double((long long)w);
      else ((int32_t*)data)[r] = (int32_t)w;
      break;
    default: ((uint64_t*)data)[r] = w; break;
  }
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ int type_width_dev(int t) {
  switch (t) {
    case RW_T_BOOL: return 1;
    case RW_T_INT16: return 2;
    case RW_T_INT32: case RW_T_FLOAT32: case RW_T_DATE: return 4;
    case RW_T_DECIMAL: return 16;
    default: return 8;
  }
}

// bytes (1 = set) -> LSB-first bitmap words; thread per output word
__global__ void pack_bytes_to_bits_kernel(const uint8_t* bytes, uint64_t* words, int64_t n);

}  // namespace rw
#endif
