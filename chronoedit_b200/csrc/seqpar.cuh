// Sequence parallelism for single-edit latency (SURVEY.md section 8(f) row 2): the tokens of ONE edit are split over the ranks of
// a node, every rank holds all weights, and the only exchange is around the self-attention (heads <-> tokens, "Ulysses" layout,
// reference: chronoedit_diffsynth/wan_video_new_chronoedit.py:330-355, 1448-1498).  Here the exchange is not a collective call:
// the kernels that PRODUCE the data store it straight into the consuming rank's memory over NVLink (peer pointers obtained with
// CUDA IPC) -- the RMSNorm+RoPE kernel scatters q | k by head, a copy kernel scatters v, the attention epilogue scatters the
// output rows back to the ranks that own the tokens -- and a flag barrier in peer memory orders the phases.
//
// Test aid (ce_dit_sp_host_barrier): `world` handles of ONE process on ONE GPU can play the ranks, with ordinary device allocations
// as regions.  The barrier is then a host rendezvous instead of the flag kernel, so no kernel ever waits for another rank's work.
#pragma once
#include <memory>

#include "host_common.h"
#include "ptx.cuh"

namespace ce {

struct HostRendezvous;

struct SeqPar {
  int rank = 0, world = 1;
  uint8_t* region[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // same layout on every rank
  int64_t region_bytes = 0;
  uint32_t epoch = 0;
  int host_barrier_ms = 0;                // > 0: launch_sp_barrier is a host rendezvous with this timeout (kept across configures)
  std::shared_ptr<HostRendezvous> host;   // the rendezvous of this region table, joined at the first host barrier
};

struct SpLayout {   // byte offsets inside a rank's region
  int64_t q, k, v;      // gathered q / k / v of the heads this rank owns: [B, L, D / world] bf16 each
  int64_t attn;         // attention output of the tokens this rank owns: [B * L / world, D] bf16
  int64_t yout;         // full head output [B * L, out_channels * 4] bf16 (every rank gets all of it)
  int64_t flags;        // uint32 [8 * 32]
  int64_t bytes;
};
SpLayout sp_layout(int64_t B, int64_t L, int64_t D, int64_t No, int world);

// all ranks: everything this rank issued so far on `stream` (incl. its peer stores) is complete and visible before any rank continues.
// The flags (uint32 [8 * 32]) lie at byte offset `flags` of every rank's region.
// With sp.host_barrier_ms > 0 no kernel is launched: the stream is synchronised and the calling thread waits for the other ranks'
// threads (same process, same region[0]); a timeout is an error naming the rank and the barrier and poisons the group, so every
// later barrier of it fails at once.  Refused while `stream` is capturing.
int launch_sp_barrier(SeqPar& sp, int64_t flags, cudaStream_t stream);
// dst[r] + ((b * dst_rows_per_batch + dst_row0 + i) * cols_per_rank + c % cols_per_rank) = src[(b * rows_per_batch + i) * ld_src + c],
// r = c / cols_per_rank   (v scatter: columns to the rank that owns the head)
int launch_sp_scatter_cols(const bf16* src, int ld_src, int B, int rows_per_batch, int ncols, bf16* const* dst, int world, int cols_per_rank,
                           int dst_rows_per_batch, int dst_row0, cudaStream_t stream);
// every rank r: dst[r] + ((b * dst_rows_per_batch + dst_row0 + i) * ncols + c) = src[(b * rows_per_batch + i) * ncols + c]   (all-gather of rows)
int launch_sp_broadcast_rows(const bf16* src, int B, int rows_per_batch, int ncols, bf16* const* dst, int world, int dst_rows_per_batch,
                             int dst_row0, cudaStream_t stream);
// One launch of up to 8 strided copies, each to local or peer memory: for i1 < n1, i0 < n0, dst + i1 * dp1 + i0 * dp0 receives the `bytes`
// bytes at src + i1 * sp1 + i0 * sp0 (byte offsets and sizes; bf16 data, so all of them even).  The VAE's band exchanges.
struct SpCopy {
  const void* src = nullptr;
  void* dst = nullptr;
  int64_t bytes = 0;
  int n0 = 1, n1 = 1;
  int64_t sp0 = 0, sp1 = 0, dp0 = 0, dp1 = 0;
};
int launch_sp_copy(const SpCopy* jobs, int n, cudaStream_t stream);
// patchify of a token range: patches[(b, i), k] for global tokens tok0 .. tok0 + ntok - 1 of every sample
int launch_patchify_range(const bf16* x, bf16* patches, int B, int C, int T, int H, int W, int tok0, int ntok, cudaStream_t stream);

}  // namespace ce
