// vsb200 -- Dynamic Sequence Parallelism signalling and peer-window plumbing.  The switch itself is fused into its
// producer and consumer (elementwise.cu: vsb_ln_modulate_dsp stores into the peers' receive windows,
// vsb_gate_residual_dsp loads from them over NVLink).  Completion: every CTA of the producer fences (system scope); the
// last CTA to finish publishes the epoch into each peer's flag slot; vsb_dsp_wait spins (acquire, system scope) on the
// receiver's stream.
#include "dsp_common.cuh"
#include "vsb_host.h"

namespace vsb {

// Publishes the next epoch without moving data: the producer (the proj GEMM) wrote its output into this rank's own
// window and the consumers PULL their rows (vsb_gate_residual_dsp).
__global__ void dsp_signal_kernel(DspPeers peers, int rank, int world, unsigned epoch) {
  dsp_publish(peers, rank, world, epoch);
}

// epoch == 0: wait for the next value of the device-side wait counter (flags[kDspWaitCtr])
__global__ void dsp_wait_kernel(unsigned* flags, int world, unsigned epoch) {
  __shared__ unsigned s_epoch;
  if (threadIdx.x == 0) {
    if (epoch == 0) {
      epoch = flags[kDspWaitCtr] + 1u;
      flags[kDspWaitCtr] = epoch;
    }
    s_epoch = epoch;
  }
  __syncthreads();
  epoch = s_epoch;
  const int src = threadIdx.x;
  if (src < world) {
    long long t0 = clock64();
    while ((int)(ld_acquire_sys(flags + src) - epoch) < 0) {
      if (clock64() - t0 > 20000000000ll) {
        printf("vsb200: dsp_wait watchdog src=%d epoch=%u have=%u\n", src, epoch, ld_acquire_sys(flags + src));
        __trap();
      }
    }
  }
}

int dsp_fill_peers(DspPeers* peers, void* const* host_peer_recv, void* const* host_peer_flags, int world, const char* what) {
  for (int i = 0; i < world; ++i) {
    peers->recv[i] = host_peer_recv ? (bf16*)host_peer_recv[i] : nullptr;
    peers->flags[i] = host_peer_flags ? (unsigned*)host_peer_flags[i] : nullptr;
    if ((host_peer_recv && (!peers->recv[i] || !aligned16(peers->recv[i]))) || (host_peer_flags && !peers->flags[i]))
      return fail(VSB_ERR_INVALID, "%s: peer %d window", what, i);
  }
  return VSB_OK;
}

}  // namespace vsb

using namespace vsb;

extern "C" int vsb_dsp_signal(void* const* host_peer_flags, int rank, int world, unsigned epoch, void* stream) {
  if (!host_peer_flags || world < 1 || world > kMaxWorld || rank < 0 || rank >= world)
    return fail(VSB_ERR_INVALID, "dsp_signal: bad args");
  DspPeers peers;
  int rc = dsp_fill_peers(&peers, nullptr, host_peer_flags, world, "dsp_signal");
  if (rc) return rc;
  dsp_signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(peers, rank, world, epoch);
  return check_launch("dsp_signal");
}

extern "C" int vsb_dsp_wait(void* my_flags, int world, unsigned epoch, void* stream) {
  if (!my_flags || world < 1 || world > kMaxWorld) return fail(VSB_ERR_INVALID, "dsp_wait: bad args");
  dsp_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((unsigned*)my_flags, world, epoch);
  return check_launch("dsp_wait");
}

// ---- symmetric-window plumbing (CUDA IPC); windows are cudaMalloc'ed here so the handle maps the exact base ----
extern "C" int vsb_dsp_alloc(void** out, size_t bytes) {
  if (!out || bytes == 0) return fail(VSB_ERR_INVALID, "dsp_alloc: bad args");
  cudaError_t e = cudaMalloc(out, bytes);
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "dsp_alloc: %s", cudaGetErrorString(e));
  e = cudaMemset(*out, 0, bytes);
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "dsp_alloc memset: %s", cudaGetErrorString(e));
  return VSB_OK;
}
extern "C" int vsb_dsp_free(void* p) {
  cudaError_t e = cudaFree(p);
  return e == cudaSuccess ? VSB_OK : fail(VSB_ERR_CUDA, "dsp_free: %s", cudaGetErrorString(e));
}
extern "C" int vsb_ipc_get_handle(void* devptr, void* out_handle64) {
  if (!devptr || !out_handle64) return fail(VSB_ERR_INVALID, "ipc_get_handle: bad args");
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, devptr);
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
  memcpy(out_handle64, &h, sizeof(h));
  return VSB_OK;
}
extern "C" int vsb_ipc_open_handle(const void* handle64, void** out_devptr) {
  if (!handle64 || !out_devptr) return fail(VSB_ERR_INVALID, "ipc_open_handle: bad args");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  cudaError_t e = cudaIpcOpenMemHandle(out_devptr, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "cudaIpcOpenMemHandle: %s", cudaGetErrorString(e));
  return VSB_OK;
}
extern "C" int vsb_ipc_close_handle(void* devptr) {
  cudaError_t e = cudaIpcCloseMemHandle(devptr);
  return e == cudaSuccess ? VSB_OK : fail(VSB_ERR_CUDA, "cudaIpcCloseMemHandle: %s", cudaGetErrorString(e));
}
