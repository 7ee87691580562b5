#include "host_common.h"

#include <atomic>
#include <map>
#include <mutex>
#include <utility>

namespace ce {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }
int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
const std::string& last_error() { return g_last_error; }

int register_weight(WeightMap& w, const char* fn, const char* name, const void* ptr, int dtype, int64_t numel) {
  CE_REQUIRE(name && ptr, std::string(fn) + ": null argument");
  CE_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, std::string(fn) + ": pointer must be 16-byte aligned");
  w[name] = WeightRef{ptr, dtype, numel};
  return CE_OK;
}

const void* WeightLookup::get(const std::string& name, int dtype, int64_t numel) {
  if (rc) return nullptr;
  auto it = w.find(name);
  if (it == w.end()) {
    rc = fail(CE_ERR_MISSING_WEIGHT, "missing weight: " + name);
    return nullptr;
  }
  if (dtype >= 0 && it->second.dtype != dtype) {
    rc = fail(CE_ERR_MISSING_WEIGHT, "weight " + name + " has dtype " + std::to_string(it->second.dtype) + ", expected " +
                                         std::to_string(dtype) + " (0 bf16, 1 fp32, 2 e4m3" +
                                         (dtype == 2 || it->second.dtype == 2
                                              ? "; the six block GEMM weights of every layer are either all bf16 or all e4m3)"
                                              : ")"));
    return nullptr;
  }
  if (it->second.numel != numel) {
    rc = fail(CE_ERR_MISSING_WEIGHT, "weight " + name + " has " + std::to_string(it->second.numel) + " elements, expected " +
                                         std::to_string(numel));
    return nullptr;
  }
  return it->second.ptr;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(CE_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail(CE_ERR_INVALID, "TMA base pointer not 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (gstr[i] % 16 != 0) return fail(CE_ERR_INVALID, "TMA global stride not a multiple of 16 bytes");
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(CE_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return CE_OK;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box, elem_strides);
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld * 2};
  uint32_t box[2] = {64, box_rows};
  return make_tmap_bf16(out, base, 2, dims, strides, box);
}

int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box, nullptr);
}

int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld};
  uint32_t box[2] = {128, box_rows};
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, 2, dims, strides, box, nullptr);
}

constexpr int kMaxDevices = 64;

int device_sm_count() {
  static std::atomic<int> n[kMaxDevices] = {};   // handles driven from several host threads fill it concurrently
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

int ensure_dynamic_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> done;  // (kernel, device) -> bytes already opted in
  int dev = 0;
  CE_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  auto key = std::make_pair(kernel, dev);
  auto it = done.find(key);
  if (it != done.end() && it->second >= bytes) return CE_OK;
  CE_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done[key] = bytes;
  return CE_OK;
}

int check_device() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess)
    return fail(CE_ERR_NO_DEVICE, std::string("no CUDA device (") + cudaGetErrorString(e) +
                                      "); chronoedit_b200 has no CPU fallback");
  int major = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (major != 9)
    return fail(CE_ERR_NO_DEVICE, "device compute capability " + std::to_string(major) +
                                      ".x is not sm_90; this library is built for sm_90a only");
  return CE_OK;
}

}  // namespace ce
