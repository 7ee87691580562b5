// Host-side helpers shared by all translation units: status/error plumbing of the C ABI and
// CUtensorMap construction (driver entry point fetched at run time, so the library has no
// link-time dependency on libcuda and builds on a GPU-less box).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <string>

namespace ce {

typedef __nv_bfloat16 bf16;

// ---- error plumbing ------------------------------------------------------------------------
// Every extern "C" entry point returns 0 on success or a negative code and records a message
// retrievable with ce_last_error().  No exceptions cross the ABI.
enum Status : int {
  CE_OK = 0,
  CE_ERR_INVALID = -1,      // bad argument / unsupported shape
  CE_ERR_CUDA = -2,         // CUDA runtime / driver error
  CE_ERR_NO_DEVICE = -3,    // no sm_90 device: there is NO CPU fallback
  CE_ERR_MISSING_WEIGHT = -4,
  CE_ERR_WORKSPACE = -5,
};

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);

#define CE_CHECK_CUDA(expr)                                                                       \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return ::ce::fail(::ce::CE_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));   \
  } while (0)

#define CE_REQUIRE(cond, msg)                                                        \
  do {                                                                               \
    if (!(cond)) return ::ce::fail(::ce::CE_ERR_INVALID, std::string(msg) + " [" #cond "]"); \
  } while (0)

// ---- tensor maps ---------------------------------------------------------------------------
// bf16 tensor, `rank` dims listed innermost first.  strides_bytes[i] is the byte stride of dim i+1
// (dim 0 is contiguous).  128-byte swizzle, zero OOB fill.
// elem_strides (optional): traversal stride per dim; TMA then fetches ceil(box[i] / elem_strides[i]) elements along dim i.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides = nullptr);

// 2-D row-major [rows, cols] bf16 with leading dimension `ld` (elements); box = [box_rows, 64 cols].
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);
// The same for a 1-byte element type (e4m3 GEMM operands); box = [box_rows, 128 cols], still one 128-byte swizzled row.
int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);
// A 1-byte tensor of any rank, as make_tmap_bf16 (the FP8 attention's q, k and V^T tiles).
int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);

int device_sm_count();   // of the CURRENT device (cached per device index)
int check_device();
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, and a process
// may drive several GPUs (VAE on cuda:1, DiT on cuda:0; model.to() after a first forward).
int ensure_dynamic_smem(const void* kernel, int bytes);
#define CE_ENSURE_SMEM(kernel, bytes)                                                              \
  do {                                                                                             \
    int _rc = ::ce::ensure_dynamic_smem(reinterpret_cast<const void*>(kernel), (int)(bytes));      \
    if (_rc) return _rc;                                                                           \
  } while (0)  // CE_OK iff the current device is compute capability 9.x

// ---- workspace carving and launch sizing -------------------------------------------------------
// Hands out consecutive 256-byte aligned slices of one caller-owned buffer.  With a null base it only measures: every pointer
// is null and `off` is the size so far, so one carve function serves both the size query and the forward.
struct Bump {
  uint8_t* base;
  int64_t off = 0;
  explicit Bump(void* b) : base(reinterpret_cast<uint8_t*>(b)) {}
  template <typename T>
  T* take(int64_t n) {
    off = (off + 255) & ~int64_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * (int64_t)sizeof(T);
    return p;
  }
  int64_t bytes() const { return (off + 255) & ~int64_t(255); }
};

inline int up8(int v) { return (v + 7) & ~7; }

// Blocks of TPB threads for a grid-stride loop over n elements: one per TPB elements, at most 16 per SM.
constexpr int TPB = 256;
inline int grid_for(size_t n) {
  const size_t g = (n + TPB - 1) / TPB, cap = (size_t)device_sm_count() * 16;
  return (int)(g < cap ? (g ? g : 1) : cap);
}

#define CE_TRY(expr)        \
  do {                      \
    const int _rc = (expr); \
    if (_rc) return _rc;    \
  } while (0)

// ---- weights ----------------------------------------------------------------------------------
// A weight registered with a handle: the caller's pointer, its dtype (0 bf16, 1 fp32, 2 e4m3; -1 where the handle's set_weight
// takes none) and its element count.
struct WeightRef {
  const void* ptr = nullptr;
  int dtype = -1;
  int64_t numel = 0;
};
using WeightMap = std::map<std::string, WeightRef>;

// The body of every *_set_weight entry point: `fn` names it in the error message.
int register_weight(WeightMap& w, const char* fn, const char* name, const void* ptr, int dtype, int64_t numel);

// Looks weights up one at a time, checking the element count and the dtype (unless dtype < 0: handles whose set_weight takes
// none); the first one that is missing or wrong records CE_ERR_MISSING_WEIGHT with its name, and every lookup after it returns
// null.
struct WeightLookup {
  const WeightMap& w;
  int rc = CE_OK;

  const void* get(const std::string& name, int dtype, int64_t numel);
  template <class T>
  const T* any(const std::string& name, int64_t numel) { return static_cast<const T*>(get(name, -1, numel)); }
  const bf16* b16(const std::string& name, int64_t numel) { return static_cast<const bf16*>(get(name, 0, numel)); }
  const float* f32(const std::string& name, int64_t numel) { return static_cast<const float*>(get(name, 1, numel)); }
};

// ---- launches ---------------------------------------------------------------------------------
// Every launch of the VAE, encoder and fp32 validation chains: a launch_* call, or a __global__ function launched here and
// checked with cudaGetLastError.  A launch that was enqueued is counted in *launches (when given).
struct Launcher {
  cudaStream_t s;
  int64_t* launches;

  template <class Launch>
  int operator()(Launch&& launch) {
    const int rc = launch();
    if (!rc && launches) ++*launches;
    return rc;
  }
  template <class... P, class... A>
  int kernel(void (*k)(P...), int grid, int block, A... args) {
    k<<<grid, block, 0, s>>>(args...);
    CE_CHECK_CUDA(cudaGetLastError());
    if (launches) ++*launches;
    return CE_OK;
  }
};

}  // namespace ce
