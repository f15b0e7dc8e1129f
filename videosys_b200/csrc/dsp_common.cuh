// vsb200 -- device-side pieces shared by every kernel that talks to the DSP peer windows (dsp_p2p.cu: the signal and
// wait kernels; elementwise.cu: the producer- / consumer-fused switch).
#pragma once
#include "vsb_common.cuh"

namespace vsb {

constexpr int kMaxWorld = 16;
// Own flag array layout (uint32, 64 entries, zeroed at allocation):
//   [0, world)  epoch last published by source rank r            (written by the peers, system scope)
//   [32]        epochs this rank has SENT in this direction      (device-side counter: CUDA-graph replays advance it)
//   [33]        epochs this rank has WAITED for in this direction
constexpr int kDspSendCtr = 32, kDspWaitCtr = 33;

struct DspPeers {
  bf16* recv[kMaxWorld];
  unsigned* flags[kMaxWorld];
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// One per translation unit (no relocatable device code): kernels of one TU that publish are stream-ordered.
static __device__ unsigned g_dsp_done_ctas = 0;

// Called by EVERY thread of EVERY CTA after its last peer store.  The last CTA to arrive publishes the epoch to all
// peers (release, system scope).  epoch == 0: take the next value of the device-side send counter, so that a captured
// CUDA graph advances the epoch on every replay without the host.
__device__ __forceinline__ void dsp_publish(const DspPeers& peers, int rank, int world, unsigned epoch) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned done = atomicAdd(&g_dsp_done_ctas, 1u) + 1u;
    if (done == gridDim.x) {
      g_dsp_done_ctas = 0;
      unsigned* mine = peers.flags[rank];
      if (epoch == 0) {
        epoch = mine[kDspSendCtr] + 1u;
        mine[kDspSendCtr] = epoch;
      }
      __threadfence_system();
      for (int d = 0; d < world; ++d) st_release_sys(peers.flags[d] + rank, epoch);
    }
  }
}

}  // namespace vsb
