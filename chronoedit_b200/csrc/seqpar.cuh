// The peer group of a model split over the ranks of a node (SURVEY.md section 8(f) row 2): every rank holds all weights and a peer
// region of the same layout, the kernels that produce exchanged data store it straight into the consuming rank's region over NVLink
// (peer pointers obtained with CUDA IPC), and a flag barrier in peer memory orders the phases.  What is here serves every split
// model: the handle's configuration, the barrier and a batched copy to local or peer memory.  The region layouts and the exchanges
// that use them live with their model (sp_layout and the slots of the batch split and the call pair in dit.cu, vae_sp_layout in vae.cu).
//
// Test aid (ce_dit_sp_host_barrier, ce_vae_sp_host_barrier): `world` handles of ONE process on ONE GPU can play the ranks, with
// ordinary device allocations as regions.  The barrier is then a host rendezvous instead of the flag kernel, so no kernel ever waits
// for another rank's work.
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

// Configures `sp` for rank `rank` of `world` with one region pointer per rank.  world == 1 switches the split off; any other world
// outside 2..8 is refused, and so is a null or not 256-byte aligned region pointer.  host_barrier_ms is kept.  A refusal names `who`
// and leaves `sp` unchanged.
int sp_configure(SeqPar& sp, const char* who, int rank, int world, void* const* regions, int64_t bytes);
// timeout_ms > 0: launch_sp_barrier becomes the host rendezvous with that timeout; 0: the device barrier.  `sp` may be null (refused).
int sp_set_host_barrier(SeqPar* sp, const char* who, int timeout_ms);

// all ranks: everything this rank issued so far on `stream` (incl. its peer stores) is complete and visible before any rank continues.
// The flags (uint32 [8 * 32]) lie at byte offset `flags` of every rank's region.
// With sp.host_barrier_ms > 0 no kernel is launched: the stream is synchronised and the calling thread waits for the other ranks'
// threads (same process, same region[0]); a timeout is an error naming the rank and the barrier and poisons the group, so every
// later barrier of it fails at once.  Refused while `stream` is capturing.
int launch_sp_barrier(SeqPar& sp, int64_t flags, cudaStream_t stream);
// One launch of up to 8 strided copies, each to local or peer memory: for i1 < n1, i0 < n0, dst + i1 * dp1 + i0 * dp0 receives the `bytes`
// bytes at src + i1 * sp1 + i0 * sp0 (byte offsets and sizes; bf16 data, so all of them even).  16-byte copies when every address,
// pitch and size of the launch is a multiple of 16.
struct SpCopy {
  const void* src = nullptr;
  void* dst = nullptr;
  int64_t bytes = 0;
  int n0 = 1, n1 = 1;
  int64_t sp0 = 0, sp1 = 0, dp0 = 0, dp1 = 0;
};
int launch_sp_copy(const SpCopy* jobs, int n, cudaStream_t stream);

}  // namespace ce
