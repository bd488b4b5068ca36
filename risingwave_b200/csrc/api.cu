// api.cu -- host-only parts of the C ABI: errors, type table, output object, misc.
#include <stdlib.h>

#include <cstdlib>

#include "common.cuh"

namespace rw {

// driver entry points of the virtual memory management API, resolved once through the runtime
static VmmApi load_vmm_api() {
  VmmApi a;
  // opt-in: cuMemCreate + cuMemMap of a few hundred MB can take longer than cudaMalloc + device copy + cudaFree of
  // the same store
  if (!getenv("RWGPU_VMM")) return a;
  auto get = [](const char* name, void** fn) -> bool {
    cudaDriverEntryPointQueryResult q;
    *fn = nullptr;
    return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
  };
  bool ok = get("cuMemAddressReserve", (void**)&a.AddressReserve);
  ok = ok && get("cuMemAddressFree", (void**)&a.AddressFree);
  ok = ok && get("cuMemCreate", (void**)&a.Create);
  ok = ok && get("cuMemRelease", (void**)&a.Release);
  ok = ok && get("cuMemMap", (void**)&a.Map);
  ok = ok && get("cuMemUnmap", (void**)&a.Unmap);
  ok = ok && get("cuMemSetAccess", (void**)&a.SetAccess);
  ok = ok && get("cuMemGetAllocationGranularity", (void**)&a.GetGranularity);
  a.ok = ok;
  if (!ok) cudaGetLastError();  // clear the sticky-less error state of a failed lookup
  return a;
}
const VmmApi& vmm_api() {
  static const VmmApi a = load_vmm_api();
  return a;
}

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) { g_err = msg; return code; }
const char* last_error_cstr() { return g_err.c_str(); }

int type_width(int t) {
  switch (t) {
    case RW_T_BOOL: return 1;
    case RW_T_INT16: return 2;
    case RW_T_INT32: case RW_T_FLOAT32: case RW_T_DATE: return 4;
    case RW_T_INT64: case RW_T_FLOAT64: case RW_T_TIME: case RW_T_TIMESTAMP:
    case RW_T_TIMESTAMPTZ: case RW_T_SERIAL: return 8;
    case RW_T_DECIMAL: return 16;
    // varlen payload: inside the library a value is an 8-byte HANDLE (heap offset | length | heap id) into a byte heap
    // in HBM; the bytes themselves only move when a chunk enters (interned) or leaves (materialised)
    case RW_T_VARCHAR: case RW_T_BYTEA: return 8;
    default: return 0;
  }
}
bool type_is_float(int t) { return t == RW_T_FLOAT32 || t == RW_T_FLOAT64; }
bool type_is_varlen(int t) { return t == RW_T_VARCHAR || t == RW_T_BYTEA; }
bool type_supported(int t) { return type_width(t) != 0; }

int devchunk_from_abi(const rw_chunk* c, DevChunk* out) {
  if (!c || c->n_cols < 0 || c->n_cols > RW_MAX_COLS) return fail(RW_ERR_INVALID, "chunk: bad column count");
  out->n = c->n_rows;
  out->ops = c->ops;
  out->vis_bits = c->visibility;
  out->n_cols = c->n_cols;
  out->pad = 0;
  out->n_dev = nullptr;
  for (int k = 0; k < c->n_cols; k++) {
    int w = type_width(c->columns[k].type);
    if (!w) return fail(RW_ERR_UNSUPPORTED, "chunk: unsupported column type");
    out->cols[k].data = c->columns[k].data;
    out->cols[k].valid_bits = c->columns[k].validity;
    out->cols[k].valid_bytes = nullptr;
    out->cols[k].type = c->columns[k].type;
    out->cols[k].width = w;
  }
  return RW_OK;
}

}  // namespace rw

bool rwgpu_out::layout(int64_t rows, const std::vector<int>& col_types, unsigned long long null_mask, bool with_vis,
                       const std::shared_ptr<PinnedPool>& pl) {
  n_rows = rows;
  types = col_types;
  pool = pl;
  data.assign(types.size(), nullptr);
  valid_bytes.assign(types.size(), nullptr);
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  offsets.assign(types.size(), nullptr);
  auto col_bytes = [&](size_t k) {  // a varlen column's block share is its offsets array; the bytes come later (set_var_bytes)
    return rw::type_is_varlen(types[k]) ? (size_t)(rows + 1) * 4 : (size_t)rows * rw::type_width(types[k]);
  };
  size_t total = up((size_t)rows) * (1 + (with_vis ? 1 : 0));
  for (size_t k = 0; k < types.size(); k++) {
    total += up(col_bytes(k));
    if ((null_mask >> k) & 1) total += up((size_t)rows);
  }
  if (rows == 0) return true;
  block = pl ? pl->get(total) : PinnedBlock();
  if (!block.p) return false;
  size_t off = 0;
  ops = block.p + off; off += up((size_t)rows);
  if (with_vis) { vis_bytes = block.p + off; off += up((size_t)rows); }
  for (size_t k = 0; k < types.size(); k++) {
    if (rw::type_is_varlen(types[k])) offsets[k] = (uint32_t*)(block.p + off);
    else data[k] = block.p + off;
    off += up(col_bytes(k));
    if ((null_mask >> k) & 1) { valid_bytes[k] = block.p + off; off += up((size_t)rows); }
  }
  return true;
}

// pinned bytes of varlen column k (owned by the output object)
uint8_t* rwgpu_out::var_bytes(size_t k, size_t bytes) {
  var_store.emplace_back(new rw::PinnedBuf());
  if (var_store.back()->reserve(std::max<size_t>(bytes, 16)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  data[k] = var_store.back()->as<uint8_t>();
  return data[k];
}

// Cut the super-chunk into StreamChunks of <= chunk_size rows; a U- is never the last row of a
// chunk (StreamChunkBuilder::append_iter_inner, src/common/src/array/stream_chunk_builder.rs:189-219),
// and build per-chunk LSB-first bitmaps.
void rwgpu_out::finalize() {
  cut.clear();
  cut.push_back(0);
  int64_t pos = 0;
  while (pos < n_rows) {
    int64_t end = pos + chunk_size;
    if (end >= n_rows) end = n_rows;
    else if (ops[end - 1] == RW_OP_UPDATE_DELETE) end += 1;
    cut.push_back(end);
    pos = end;
  }
  size_t nch = cut.size() - 1;
  chunk_vis.assign(nch, {});
  chunk_valid.assign(nch, {});
  chunk_cols.assign(nch, {});
  for (size_t i = 0; i < nch; i++) {
    int64_t lo = cut[i], n = cut[i + 1] - cut[i];
    size_t nw = (size_t)((n + 63) / 64);
    if (vis_bytes) {
      bool all = true;
      std::vector<uint64_t> w(nw ? nw : 1, 0);
      for (int64_t r = 0; r < n; r++) {
        if (vis_bytes[lo + r]) w[r >> 6] |= 1ull << (r & 63); else all = false;
      }
      if (!all) chunk_vis[i] = std::move(w);
    }
    chunk_valid[i].assign(types.size(), {});
    chunk_cols[i].resize(types.size());
    for (size_t k = 0; k < types.size(); k++) {
      int wd = rw::type_width(types[k]);
      rw_column& c = chunk_cols[i][k];
      c.type = types[k];
      c.reserved = 0;
      c.offsets = nullptr;
      if (rw::type_is_varlen(types[k])) {  // chunk views share the column's bytes; their offsets are a slice
        c.data = data[k];
        c.offsets = offsets[k] + lo;
      } else {
        c.data = data[k] + (size_t)lo * wd;
      }
      c.validity = nullptr;
      if (valid_bytes[k]) {
        bool all = true;
        std::vector<uint64_t> w(nw ? nw : 1, 0);
        for (int64_t r = 0; r < n; r++) {
          if (valid_bytes[k][lo + r]) w[r >> 6] |= 1ull << (r & 63); else all = false;
        }
        if (!all) {
          chunk_valid[i][k] = std::move(w);
          c.validity = chunk_valid[i][k].data();
        }
      }
    }
  }
}

extern "C" {

int32_t rwgpu_type_width(int32_t type) { return rw::type_is_varlen(type) ? 0 : rw::type_width(type); }
const char* rwgpu_last_error(void) { return rw::last_error_cstr(); }
const char* rwgpu_version(void) { return "rwgpu 0.1.0 sm_90a"; }

int32_t rwgpu_device_check(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return rw::fail(RW_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e));
  }
  // Experiment knob: RWGPU_L2_FETCH=32|64|128 sets cudaLimitMaxL2FetchGranularity (the hot kernels
  // are random 64-byte bucket accesses; the driver default of 64 B matches the bucket size).
  static thread_local int applied_dev = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (applied_dev != dev) {
    size_t g = 0;  // default: leave the driver's 64 B
    if (const char* v = getenv("RWGPU_L2_FETCH")) g = (size_t)atoi(v);
    if (g == 32 || g == 64 || g == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, g);
    cudaGetLastError();
    applied_dev = dev;
  }
  return RW_OK;
}

int32_t rwgpu_out_num_chunks(const rwgpu_out* o) { return o ? (int32_t)(o->cut.size() - 1) : 0; }
int64_t rwgpu_out_num_rows(const rwgpu_out* o) { return o ? o->n_rows : 0; }
int32_t rwgpu_out_chunk(const rwgpu_out* o, int32_t idx, rw_chunk* view) {
  if (!o || !view || idx < 0 || (size_t)idx + 1 >= o->cut.size()) return rw::fail(RW_ERR_INVALID, "chunk index");
  int64_t lo = o->cut[idx];
  view->n_rows = o->cut[idx + 1] - lo;
  view->n_cols = (int32_t)o->types.size();
  view->reserved = 0;
  view->ops = o->ops + lo;
  view->visibility = o->chunk_vis[idx].empty() ? nullptr : o->chunk_vis[idx].data();
  view->columns = o->chunk_cols[idx].data();
  return RW_OK;
}
void rwgpu_out_release(rwgpu_out* o) { delete o; }

}  // extern "C"
