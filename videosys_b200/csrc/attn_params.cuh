// vsb200 -- parameters shared by the two flash-attention kernels (attn_wgmma.cu: head_dim 64 / 72 on the warpgroup tensor
// cores; attn_mma.cu: the other head dims on mma.sync) and the vsb_attn_flash entry that dispatches between them.
#pragma once
#include "vsb_common.cuh"
#include "vsb_host.h"

namespace vsb {

constexpr int kAttnMaxLens = 64;  // per-batch key counts travel by value in the kernel parameters
struct AttnParams {
  bf16* out;
  // out element (b, n, h, d) at out + b*out_batch_stride + n*out_row_stride + h*D + d (elements): the temporal
  // (T >= 30) path writes straight back into the token-major activation
  long long out_row_stride, out_batch_stride;
  long long q_row_stride, q_batch_stride;
  int nb, nq, nk, H;
  float scale_log2;  // softmax scale * log2(e)
  int has_lens;
  int lens[kAttnMaxLens];
};

// attn_wgmma.cu: head_dim 64 / 72; q / k / v are strided views (element (b, n, h, d) at base + b*batch_stride +
// n*row_stride + h*D + d, strides in elements).
int attn_wgmma_launch(const bf16* q, const bf16* k, const bf16* v, long long kv_row_stride, long long kv_batch_stride,
                      const AttnParams& prm, int D, cudaStream_t st);

}  // namespace vsb
