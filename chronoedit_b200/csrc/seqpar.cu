#include "seqpar.cuh"

#include <string.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <map>
#include <mutex>
#include <string>

#include "../../include/chronoedit_b200.h"

namespace ce {

namespace {

struct Ptrs8 {
  void* p[8];
};

__global__ void sp_barrier_kernel(Ptrs8 flags, int rank, int world, uint32_t epoch) {
  const int w = threadIdx.x;
  if (w >= world) return;
  __threadfence_system();
  uint32_t* remote = reinterpret_cast<uint32_t*>(flags.p[w]) + rank;   // my slot in rank w's flag array
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
  const uint32_t* mine = reinterpret_cast<const uint32_t*>(flags.p[rank]) + w;   // rank w's slot in my array
  const uint64_t t0 = global_timer_ns();
  uint32_t v = 0, spins = 0;
  do {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
    if ((++spins & 0x3FFF) == 0 && global_timer_ns() - t0 > 20000000000ull) {
      printf("[chronoedit_b200] sequence-parallel barrier timeout: rank %d waits for rank %d (epoch %u, saw %u)\n", rank, w, epoch, v);
      __trap();
    }
  } while ((int32_t)(v - epoch) < 0);
  __threadfence_system();
}

struct SpCopies {
  SpCopy c[8];
};

// blockIdx.y = job; V = uint4 when every address, pitch and size of the launch is 16-byte aligned, else one bf16 at a time
template <typename V>
__global__ void sp_copy_kernel(const __grid_constant__ SpCopies jobs) {
  const SpCopy& j = jobs.c[blockIdx.y];
  const int64_t nv = j.bytes / (int64_t)sizeof(V);
  const int64_t total = nv * j.n0 * j.n1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i % nv, p = i / nv;
    const int64_t i0 = p % j.n0, i1 = p / j.n0;
    const V* s = reinterpret_cast<const V*>(reinterpret_cast<const uint8_t*>(j.src) + i1 * j.sp1 + i0 * j.sp0) + v;
    V* d = reinterpret_cast<V*>(reinterpret_cast<uint8_t*>(j.dst) + i1 * j.dp1 + i0 * j.dp0) + v;
    *d = *s;
  }
}

}  // namespace

// The host barrier's rendezvous: one per region table (keyed on region[0]) among the handles of this process.
struct HostRendezvous {
  std::mutex mu;
  std::condition_variable cv;
  int world = 0;
  uint32_t arrived = 0;     // bit r: rank r has arrived at the current barrier
  uint32_t epoch = 0;       // the epoch of the current barrier (every rank's handle counts its barriers the same way)
  uint64_t generation = 0;  // completed barriers
  std::string poisoned;     // non-empty: a barrier timed out or a rank fell out of step; every later barrier fails with this

  int arrive(int rank, uint32_t ep, int timeout_ms) {
    std::unique_lock<std::mutex> lock(mu);
    if (!poisoned.empty()) return fail(CE_ERR_INVALID, "sequence-parallel host barrier: rank " + std::to_string(rank) + " at barrier " +
                                                           std::to_string(ep) + ": the group failed earlier (" + poisoned + ")");
    if (arrived == 0) epoch = ep;
    if (ep != epoch || (arrived >> rank & 1u)) {
      poisoned = "rank " + std::to_string(rank) + " arrived at barrier " + std::to_string(ep) + " while the group waits at barrier " +
                 std::to_string(epoch) + ((arrived >> rank & 1u) ? " (twice)" : "");
      cv.notify_all();
      return fail(CE_ERR_INVALID, "sequence-parallel host barrier: ranks out of step: " + poisoned);
    }
    arrived |= 1u << rank;
    if (arrived == (1u << world) - 1) {
      arrived = 0;
      ++generation;
      cv.notify_all();
      return CE_OK;
    }
    const uint64_t gen = generation;
    const bool done = cv.wait_for(lock, std::chrono::milliseconds(timeout_ms), [&] { return generation != gen || !poisoned.empty(); });
    if (generation != gen) return CE_OK;
    if (!done) {
      std::string missing;
      for (int w = 0; w < world; ++w)
        if (!(arrived >> w & 1u)) missing += (missing.empty() ? "" : ", ") + std::to_string(w);
      poisoned = "rank " + std::to_string(rank) + " timed out after " + std::to_string(timeout_ms) + " ms at barrier " + std::to_string(ep) +
                 " waiting for rank(s) " + missing;
      cv.notify_all();
      return fail(CE_ERR_INVALID, "sequence-parallel host barrier: " + poisoned);
    }
    return fail(CE_ERR_INVALID, "sequence-parallel host barrier: rank " + std::to_string(rank) + " at barrier " + std::to_string(ep) +
                                    ": the group failed (" + poisoned + ")");
  }
};

int sp_configure(SeqPar& sp, const char* who, int rank, int world, void* const* regions, int64_t bytes) {
  SeqPar c;
  c.host_barrier_ms = sp.host_barrier_ms;
  if (world != 1) {
    CE_REQUIRE(world >= 2 && world <= 8 && rank >= 0 && rank < world && regions && bytes > 0, std::string(who) + ": arguments");
    for (int w = 0; w < world; ++w) {
      CE_REQUIRE(regions[w] != nullptr && (reinterpret_cast<uintptr_t>(regions[w]) & 255) == 0,
                 std::string(who) + ": null region pointer or one not 256-byte aligned");
      c.region[w] = reinterpret_cast<uint8_t*>(regions[w]);
    }
    c.rank = rank;
    c.world = world;
    c.region_bytes = bytes;
  }
  sp = c;
  return CE_OK;
}

int sp_set_host_barrier(SeqPar* sp, const char* who, int timeout_ms) {
  CE_REQUIRE(sp && timeout_ms >= 0, std::string(who) + ": arguments");
  sp->host_barrier_ms = timeout_ms;
  sp->host.reset();   // the next barrier joins the rendezvous afresh
  return CE_OK;
}

static int host_barrier(SeqPar& sp, cudaStream_t stream) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CE_CHECK_CUDA(cudaStreamIsCapturing(stream, &cs));
  CE_REQUIRE(cs == cudaStreamCaptureStatusNone, "sequence-parallel host barrier: the stream is capturing (a host wait cannot be captured)");
  CE_CHECK_CUDA(cudaStreamSynchronize(stream));
  if (!sp.host) {   // join (or found) the rendezvous of this region table; it lives as long as a handle configured with it
    static std::mutex mu;
    static std::map<const void*, std::weak_ptr<HostRendezvous>> groups;
    std::lock_guard<std::mutex> lock(mu);
    for (auto it = groups.begin(); it != groups.end();) it = it->second.expired() ? groups.erase(it) : std::next(it);
    std::shared_ptr<HostRendezvous> g = groups[sp.region[0]].lock();
    if (!g) {
      g = std::make_shared<HostRendezvous>();
      g->world = sp.world;
      groups[sp.region[0]] = g;
    }
    CE_REQUIRE(g->world == sp.world, "sequence-parallel host barrier: handles share region 0 with different rank counts");
    sp.host = g;
  }
  return sp.host->arrive(sp.rank, sp.epoch, sp.host_barrier_ms);
}

int launch_sp_barrier(SeqPar& sp, int64_t flags, cudaStream_t stream) {
  Ptrs8 f;
  for (int w = 0; w < 8; ++w) f.p[w] = w < sp.world ? sp.region[w] + flags : nullptr;
  ++sp.epoch;
  if (sp.host_barrier_ms > 0) return host_barrier(sp, stream);
  sp_barrier_kernel<<<1, 32, 0, stream>>>(f, sp.rank, sp.world, sp.epoch);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

int launch_sp_copy(const SpCopy* jobs, int n, cudaStream_t stream) {
  CE_REQUIRE(n >= 1 && n <= 8, "sp copy: 1 to 8 jobs");
  SpCopies c;
  bool vec = true;
  int64_t most = 0;
  for (int i = 0; i < n; ++i) {
    const SpCopy& j = jobs[i];
    CE_REQUIRE(j.src && j.dst && j.bytes > 0 && j.bytes % 2 == 0 && j.n0 >= 1 && j.n1 >= 1, "sp copy: job");
    const uint64_t bits = reinterpret_cast<uintptr_t>(j.src) | reinterpret_cast<uintptr_t>(j.dst) | (uint64_t)j.bytes | (uint64_t)j.sp0 |
                          (uint64_t)j.sp1 | (uint64_t)j.dp0 | (uint64_t)j.dp1;
    CE_REQUIRE((bits & 1) == 0, "sp copy: bf16 alignment");
    vec = vec && (bits & 15) == 0;
    most = std::max(most, j.bytes * j.n0 * j.n1);
    c.c[i] = j;
  }
  const dim3 grid((unsigned)grid_for((size_t)(most / (vec ? 16 : 2))), (unsigned)n);
  if (vec)
    sp_copy_kernel<uint4><<<grid, 256, 0, stream>>>(c);
  else
    sp_copy_kernel<uint16_t><<<grid, 256, 0, stream>>>(c);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce

using namespace ce;

extern "C" {

// ---- CUDA IPC plumbing for the peer regions (cudaMalloc'ed here so that the IPC handle covers exactly the region)
int ce_ipc_alloc(int64_t bytes, void** ptr) {
  CE_REQUIRE(bytes > 0 && ptr, "ce_ipc_alloc: arguments");
  CE_CHECK_CUDA(cudaMalloc(ptr, (size_t)bytes));
  CE_CHECK_CUDA(cudaMemset(*ptr, 0, (size_t)bytes));
  CE_CHECK_CUDA(cudaDeviceSynchronize());
  return CE_OK;
}
int ce_ipc_free(void* ptr) {
  if (ptr) CE_CHECK_CUDA(cudaFree(ptr));
  return CE_OK;
}
int ce_ipc_get_handle(void* ptr, void* handle_out_64_bytes) {
  CE_REQUIRE(ptr && handle_out_64_bytes, "ce_ipc_get_handle: arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  CE_CHECK_CUDA(cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle_out_64_bytes), ptr));
  return CE_OK;
}
int ce_ipc_open(const void* handle_64_bytes, void** ptr) {
  CE_REQUIRE(handle_64_bytes && ptr, "ce_ipc_open: arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle_64_bytes, 64);
  CE_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return CE_OK;
}
int ce_ipc_close(void* ptr) {
  if (ptr) CE_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
  return CE_OK;
}

}  // extern "C"
