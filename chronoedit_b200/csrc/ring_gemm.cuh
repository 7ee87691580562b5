// The TMA -> shared-memory ring -> wgmma pipeline under gemm_bf16_kernel / gemm_fp8_kernel (gemm.cu) and conv3d_cl_kernel (conv.cu).
//
// Persistent, warp-specialised, one CTA per SM, 384 threads = 3 warpgroups (registers re-partitioned with setmaxnreg):
//   warpgroup 0     TMA producer (one lane of warp 0): per k-block one A tile BMxBK and one B tile BNxBK into the next stage
//                   of a STAGES-deep ring (128B swizzle); the operation supplies the coordinates.  Given epilogue_warps, its
//                   warps 1-3 are the operation's epilogue warps (the GEMM's: they take the rounded tile from the consumers
//                   through shared memory and finish it while the consumers run the next tile's main loop); otherwise they idle
//   warpgroups 1,2  consumers: 64 rows x BN columns of the tile each, 4 x wgmma (M64, N=BN, K16 bf16 / K32 e4m3) per k-block with both operands
//                   read from the ring, then the operation's epilogue from the accumulator registers
// All roles walk the same tiles (RingTiles) and ring positions, so the producer fills the ring for tile i+1 while the
// consumers run the epilogue of tile i.  A kernel calls ring.start() with its producer, then `for (int t : RingTiles{n})
// { ring.mma_tile(acc, kblocks); epilogue }` in its own body (a lambda epilogue ran the BN = 192 conv 10 % slower, H100 700 W).
#pragma once
#include "host_common.h"
#include "wgmma.cuh"

#include <type_traits>

namespace ce {

constexpr int BM = 128;          // tile rows: two consumer warpgroups of 64
constexpr int BK = 64;           // k-block: one 128-byte swizzled row of bf16
template <class T>
constexpr int BK_OF = 128 / sizeof(T);   // k-block in elements of T: 64 bf16, 128 e4m3
constexpr int RING_THREADS = 384;

// The tiles of this CTA in the order both roles walk them: blockIdx.x, blockIdx.x + gridDim.x, ... below num_tiles.
struct RingTiles {
  struct It {
    int t;
    __device__ __forceinline__ int operator*() const { return t; }
    __device__ __forceinline__ void operator++() { t += gridDim.x; }
    __device__ __forceinline__ bool operator!=(It end) const { return t < end.t; }
  };
  int num_tiles;
  __device__ __forceinline__ It begin() const { return {(int)blockIdx.x}; }
  __device__ __forceinline__ It end() const { return {num_tiles}; }
};

// This consumer thread's accumulators (wgmma.cuh layout): acc[4 j + 2 h + e] is row ring_row() + 8 h, col 8 j + ring_col() + e.
__device__ __forceinline__ int ring_row() { return ((threadIdx.x >> 5) - 4) * 16 + ((threadIdx.x & 31) >> 2); }
__device__ __forceinline__ int ring_col() { return 2 * (threadIdx.x & 3); }

// Ring::start()'s default for a kernel without epilogue warps.
struct NoEpilogueWarps {
  __device__ __forceinline__ void operator()() const {}
};

// Shared memory, from a 1024-byte aligned base (the 128B swizzle atom): A ring, B ring, then 256 bytes of barriers: full[STAGES],
// empty[STAGES] and, from empty + STAGES, room for the operation's own; the operation's shared memory starts at tail().
// `stage` / `phase` are one role's position in the ring; each role keeps its own copy and carries it from tile to tile.
template <int BN, int STAGES>
struct Ring {
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t B_BYTES = BN * BK * 2;
  static constexpr size_t SMEM_BYTES = (size_t)STAGES * (A_BYTES + B_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;

  uint8_t *sA, *sB;
  uint64_t* full;    // stage loaded: the producer's arrive + the TMA bytes
  uint64_t* empty;   // stage consumed: one arrive per consumer warpgroup
  int stage = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ Ring() {
    extern __shared__ uint8_t smem_raw[];
    sA = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    sB = sA + STAGES * A_BYTES;
    full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
    empty = full + STAGES;
  }

  __device__ __forceinline__ uint8_t* tail() const { return reinterpret_cast<uint8_t*>(full) + 256; }

  // Barrier init and role split.  Warpgroup 0 gives registers up, runs produce(t) on one lane for every tile t of this CTA and,
  // given epilogue_warps, runs it on its warps 1-3; then it returns false.  The consumer warpgroups take the registers and
  // return true.  Registers per thread: 40 / 232 / 232, or with epilogue warps, which need more than the producer,
  // 88 / 208 / 208 (the kernel itself is compiled to 168, the 384-thread bound).  The epilogue warps run in here, as the
  // producer does: when the kernel picked the role after start() returned, ptxas dropped both setmaxnreg (C7507).
  template <class Produce, class EpilogueWarps = NoEpilogueWarps>
  __device__ __forceinline__ bool start(const CUtensorMap* tma_a, const CUtensorMap* tma_b, int num_tiles, Produce&& produce,
                                        EpilogueWarps&& epilogue_warps = EpilogueWarps()) {
    constexpr bool EPI = !std::is_same<std::decay_t<EpilogueWarps>, NoEpilogueWarps>::value;
    if (threadIdx.x == 0) {
      for (int i = 0; i < STAGES; ++i) {
        mbar_init(&full[i], 1);
        mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
      }
      fence_mbar_init();
      tma_prefetch_desc(tma_a);
      tma_prefetch_desc(tma_b);
    }
    __syncthreads();
    if (threadIdx.x < 128) {
      setmaxnreg_dec<EPI ? 88 : 40>();
      if (threadIdx.x < 32 && elect_one_sync())
        for (int t : RingTiles{num_tiles}) produce(t);
      if constexpr (EPI) {
        if (threadIdx.x >= 32) epilogue_warps();
      }
      return false;
    }
    setmaxnreg_inc<EPI ? 208 : 232>();
    return true;
  }

  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  // Producer: waits until the current stage is consumed, arms `bar` for one A and one B tile (load them into a, b), moves on.
  struct Slot { uint8_t *a, *b; uint64_t* bar; };
  __device__ __forceinline__ Slot acquire() {
    const Slot s{sA + stage * A_BYTES, sB + stage * B_BYTES, &full[stage]};
    mbar_wait(&empty[stage], phase ^ 1);
    mbar_arrive_expect_tx(s.bar, A_BYTES + B_BYTES);
    advance();
    return s;
  }

  // Consumer main loop of this thread's warpgroup: acc[64 x BN] = sum over `kblocks` of A[64 x BK_OF<T>] (its 64 rows of the
  // tile) * B[BN x BK_OF<T>]^T, with T = bf16 or __nv_fp8_e4m3 (a k-block is one 128-byte row either way, 4 instructions).
  // One wgmma group stays in flight: a stage is handed back to the producer (one arrive per warpgroup on empty) when the group
  // after it has been issued, so the tensor cores never wait for the hand-back.
  template <class T = bf16>
  __device__ __forceinline__ void mma_tile(float (&acc)[BN / 2], int kblocks) {
    const int wg = (threadIdx.x >> 7) - 1;
    const uint32_t a_smem = smem_u32(sA) + wg * 64 * 128, b_smem = smem_u32(sB);
    const bool signaller = (threadIdx.x & 127) == 0;
    int prev = -1;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint64_t da = wgmma_desc_kmajor_sw128(a_smem + stage * A_BYTES);
      const uint64_t db = wgmma_desc_kmajor_sw128(b_smem + stage * B_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (sizeof(T) == 1) wgmma_ss_e4m3<BN>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        else wgmma_ss<BN, 0>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && signaller) mbar_arrive(&empty[prev]);
      prev = stage;
      advance();
    }
    wgmma_wait<0>();
    if (prev >= 0 && signaller) mbar_arrive(&empty[prev]);
  }
};

// Persistent launch of a ring kernel: min(tiles, SM count) CTAs of RING_THREADS threads, one per SM, with EXTRA bytes of
// shared memory after the ring for the operation (Ring::tail()).
template <int BN, int STAGES, size_t EXTRA = 0, class... Params>
int launch_ring_gemm(void (*kernel)(Params...), int tiles, cudaStream_t stream, Params... params) {
  constexpr size_t smem = Ring<BN, STAGES>::SMEM_BYTES + EXTRA;
  CE_ENSURE_SMEM(kernel, smem);
  const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  kernel<<<grid, RING_THREADS, smem, stream>>>(params...);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce
