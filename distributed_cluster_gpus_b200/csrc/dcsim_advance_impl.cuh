/*
 * dcsim_advance_impl.cuh — the event-loop kernel for ONE lanes-per-replica setting.
 *
 * Included once per translation unit with DCSIM_LANES (32 / 16 / 8) and DCSIM_ADV_SUFFIX (_g32 / _g16 / _g8) defined:
 * dcsim_b200.cu carries the 32-lane build (one warp per replica), dcsim_advance_g8.cu / _g16.cu the builds in which a
 * warp carries 4 / 2 replicas on aligned lane groups.  Each build exports two host functions (launch, attributes).
 */
#pragma once
#include <cuda_runtime.h>

#include "dcsim_core.cuh"

#define DCSIM_CAT2(a, b) a##b
#define DCSIM_CAT(a, b) DCSIM_CAT2(a, b)
#define DCSIM_ADV(name) DCSIM_CAT(name, DCSIM_ADV_SUFFIX)

#define DCSIM_MAX_WARPS_PER_CTA 4
#define DCSIM_REPLICAS_PER_WARP (32 / DCSIM_LANES)
#ifndef DCSIM_MIN_CTAS_PER_SM
/* 32 lanes per replica: 8 CTAs x 4 warps = 32 warps/SM -> ptxas keeps the kernel within 64 registers.  With several
 * replicas per warp shared memory allows fewer warps anyway, so the register budget per thread is wider: 8 lanes at
 * 5 CTAs (96 registers, 80 replicas per SM) — 4 CTAs leave too few replicas resident, 6 CTAs (80 registers) spill. */
#define DCSIM_MIN_CTAS_PER_SM (DCSIM_LANES == 32 ? 8 : (DCSIM_LANES == 16 ? 6 : 5))
#endif

extern __shared__ __align__(16) char dcsim_smem[];

/* CAP = the power-cap controller (algo = cap_greedy with power_cap > 0: SIM:207-338) is compiled in.  It is a
 * separate instantiation because merely inlining that cold code slows the common path (registers, code size). */
/* MODE = where the replica's state block lives during the launch (a compile-time switch: a run-time select would turn
 * every state access into a generic load/store):
 *   DCSIM_MODE_STAGED  the whole block is staged in shared memory (small blocks: 4 DC x 64 is ~5 kB, 32 warps/SM);
 *   DCSIM_MODE_HEAD    only the head [0, L.rec_off) — header, event set, per-DC arrays, list window, seq ring —
 *                      is staged; the running-job records stay at the block's home in HBM/L2 and are touched once per
 *                      job_finish (dcsim_handle_finish) and written once per start.  Picked when the whole block would
 *                      leave the SM below its 32 warps (8 DC x 256: 17 kB -> 12 warps/SM; head ~4 kB -> 32);
 *   DCSIM_MODE_INPLACE nothing is staged (even the head exceeds a CTA's shared memory): same core on the HBM copy. */
enum { DCSIM_MODE_INPLACE = 0, DCSIM_MODE_STAGED = 1, DCSIM_MODE_HEAD = 2 };
/* PP = the profile recorders (power profile, occupancy, tail latency, job resources) are compiled in (launched when any is enabled):
 * the kernels without them keep their registers, spills and code. */
template <bool CAP, int MODE, bool PP>
__global__ void __launch_bounds__(DCSIM_MAX_WARPS_PER_CTA * 32, DCSIM_MIN_CTAS_PER_SM)
DCSIM_ADV(dcsim_advance_kernel)(const __grid_constant__ dcsim_kparams_t P, unsigned long long* __restrict__ events_total) {
  /* one replica per group of DCSIM_LANES lanes: a whole warp, or an aligned quarter / half of one */
  const int grp = (int)(threadIdx.x / DCSIM_LANES), lane = (int)(threadIdx.x & (DCSIM_LANES - 1));
  const uint64_t r0 = (uint64_t)blockIdx.x * (uint64_t)(blockDim.x / DCSIM_LANES) + (uint64_t)grp;
#if DCSIM_LANES == 32
  if (r0 >= P.n_replicas) return;
  const bool ghost = false;
#else
  /* The event loop's collectives span the whole warp (dcsim_event_sync): a warp leaves only as a whole.  In the batch's
   * last warp a lane group without a replica stays as a GHOST: it runs the loop switched off next to the real ones. */
  if (r0 - (uint64_t)(grp % DCSIM_REPLICAS_PER_WARP) >= P.n_replicas) return;
  const bool ghost = r0 >= P.n_replicas;
#endif
  const uint64_t r = ghost ? P.n_replicas - 1u : r0; /* (a ghost only ever READS replica n-1's state: in place, where blk
                                                        is that replica's live block, see dcsim_ctx_t::quiet) */
  const int bytes = MODE == DCSIM_MODE_HEAD ? P.L.rec_off : P.L.total_bytes; /* what is staged */
  char* home = P.state + r * (uint64_t)P.L.total_bytes;
  char* blk = MODE != DCSIM_MODE_INPLACE ? dcsim_smem + (size_t)grp * (size_t)bytes : home;
  char* rec = MODE == DCSIM_MODE_STAGED ? blk : home;
  const bool fresh = !ghost && reinterpret_cast<const dcsim_hdr_t*>(home)->initialized == 0u;
  if (MODE != DCSIM_MODE_INPLACE && !fresh && !ghost) { /* resume: coalesced 16-byte loads of the replica's block */
    const uint4* src = reinterpret_cast<const uint4*>(home);
    uint4* dst = reinterpret_cast<uint4*>(blk);
    for (int i = lane; i < bytes / 16; i += DCSIM_LANES) dst[i] = src[i];
  }
  dcsim_warp_sync();
  const uint32_t n = dcsim_replica_step<CAP, MODE != DCSIM_MODE_STAGED, PP, MODE == DCSIM_MODE_INPLACE>(&P, r, blk, rec, fresh, ghost);
  dcsim_warp_sync();
  if (MODE != DCSIM_MODE_INPLACE && !ghost) {
    const uint4* src = reinterpret_cast<const uint4*>(blk);
    uint4* dst = reinterpret_cast<uint4*>(home);
    for (int i = lane; i < bytes / 16; i += DCSIM_LANES) dst[i] = src[i];
  }
  if (lane == 0 && n) atomicAdd(events_total, (unsigned long long)n);
}


typedef void (*DCSIM_ADV(dcsim_advance_fn))(const dcsim_kparams_t, unsigned long long*);
static DCSIM_ADV(dcsim_advance_fn) DCSIM_ADV(dcsim_pick_kernel)(bool cap, int mode, bool pp) {
  static const DCSIM_ADV(dcsim_advance_fn) table[12] = {
      DCSIM_ADV(dcsim_advance_kernel)<false, 0, false>, DCSIM_ADV(dcsim_advance_kernel)<false, 1, false>, DCSIM_ADV(dcsim_advance_kernel)<false, 2, false>,
      DCSIM_ADV(dcsim_advance_kernel)<true, 0, false>,  DCSIM_ADV(dcsim_advance_kernel)<true, 1, false>,  DCSIM_ADV(dcsim_advance_kernel)<true, 2, false>,
      DCSIM_ADV(dcsim_advance_kernel)<false, 0, true>,  DCSIM_ADV(dcsim_advance_kernel)<false, 1, true>,  DCSIM_ADV(dcsim_advance_kernel)<false, 2, true>,
      DCSIM_ADV(dcsim_advance_kernel)<true, 0, true>,   DCSIM_ADV(dcsim_advance_kernel)<true, 1, true>,   DCSIM_ADV(dcsim_advance_kernel)<true, 2, true>};
  return table[(pp ? 6 : 0) + (cap ? 3 : 0) + mode];
}

/* Resident CTAs per SM this build's register budget was chosen for (its __launch_bounds__). */
int DCSIM_ADV(dcsim_adv_min_ctas)(void) { return DCSIM_MIN_CTAS_PER_SM; }

/* Launch on `stream`: `ctas` CTAs of `threads` threads (threads / DCSIM_LANES replicas each), `smem` dynamic bytes.  The
 * instantiation with the profile recorders when P->pp, P->occ, P->tail or P->jres is set. */
cudaError_t DCSIM_ADV(dcsim_adv_launch)(const dcsim_kparams_t* P, unsigned long long* events, int cap, int mode, int ctas, int threads,
                                        int smem, cudaStream_t stream) {
  DCSIM_ADV(dcsim_pick_kernel)(cap != 0, mode, P->pp != nullptr || P->occ != nullptr || P->tail != nullptr ||
                                           P->jres != nullptr)<<<ctas, threads, smem, stream>>>(*P, events);
  return cudaGetLastError();
}

/* Registers per thread and resident CTAs per SM of the instantiation for (cap, mode) at that CTA shape (the one without
 * the profile recorders); also raises the dynamic shared-memory limit of both to `smem_optin`. */
cudaError_t DCSIM_ADV(dcsim_adv_attrs)(int cap, int mode, int threads, int smem, int smem_optin, int* regs, int* blocks_per_sm,
                                       int* min_ctas_per_sm) {
  const DCSIM_ADV(dcsim_advance_fn) kern = DCSIM_ADV(dcsim_pick_kernel)(cap != 0, mode, false);
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(DCSIM_ADV(dcsim_pick_kernel)(cap != 0, mode, true), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                smem_optin)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin)) != cudaSuccess) return e;
  cudaFuncAttributes fa;
  if ((e = cudaFuncGetAttributes(&fa, kern)) != cudaSuccess) return e;
  *regs = fa.numRegs;
  *min_ctas_per_sm = DCSIM_MIN_CTAS_PER_SM;
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, kern, threads, smem);
}
