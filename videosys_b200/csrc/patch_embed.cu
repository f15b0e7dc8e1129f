// vsb200 -- patch embedding of the latent: a (1, ph, pw)-strided convolution with Cin * ph * pw = 16 taps per token
// (OpenSora STDiT3 PatchEmbed3D, patch (1, 2, 2), 4 latent channels; Latte's 2 x 2 PatchEmbed on 4 channels), the
// position embedding add, and the sequence-parallel split -- one pass whose only real traffic is the write of the token
// tensor (332 MB at 720p), on the rank's OWN patch columns only.
//
// Replaces open_sora_transformer_3d.py:568-572 (x_embedder -> rearrange -> + pos_emb -> rearrange) and :577
// (split_sequence along S): the eager chain runs a cuDNN implicit GEMM with K = 16 plus two layout transposes, a
// transposed read-modify-write for the position add and a slicing copy, all on the FULL sequence on every rank --
// and that cost does not shrink with the number of GPUs.
//
// Mapping: a thread owns 8 consecutive output channels (one 16-byte store per token) and keeps their 16 x 8 weights in
// registers as fp32 for the whole kernel; a CTA walks tiles of 32 tokens whose 16 taps are staged in shared memory
// (broadcast reads).  128 FMAs per 16 bytes written: ~100 us of FMA-pipe time at 720p against 50 us of HBM writes.
// Rounding follows the eager chain: conv accumulates in fp32 and rounds, the bias add rounds (ATen adds the bias of a
// cuDNN convolution as a separate op), the position add rounds.
#include "vsb_common.cuh"
#include "vsb_host.h"

namespace vsb {

constexpr int kPeTaps = 16;
constexpr int kPeTile = 32;  // tokens per tile

union PeVec {
  uint4 u;
  elem2 h[4];
};

__global__ void __launch_bounds__(256, 1) patch_embed_kernel(
    const bf16* __restrict__ z, const bf16* __restrict__ w, const bf16* __restrict__ bias, const bf16* __restrict__ pos,
    bf16* __restrict__ out, int B, int Cin, int T, int H, int W, long long sb, long long sc, long long st, int ph, int pw,
    int C, int Wn, int S_total, int s0, int S_local) {
  __shared__ float taps[kPeTile][kPeTaps];
  const int cg = threadIdx.x;  // channel group: channels [8 cg, 8 cg + 8)
  const bool live = cg * 8 < C;
  float wr[kPeTaps][8];
  float br[8];
  if (live) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      br[j] = bias != nullptr ? e_to_float(bias[cg * 8 + j]) : 0.f;
#pragma unroll
      for (int k = 0; k < kPeTaps; ++k) wr[k][j] = e_to_float(w[(size_t)(cg * 8 + j) * kPeTaps + k]);
    }
  }
  const int tiles_per_row = (S_local + kPeTile - 1) / kPeTile;  // a "row" = one (batch, frame) of S_local tokens
  const long long n_tiles = (long long)B * T * tiles_per_row;
  const int pp = ph * pw;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int bt = int(tile / tiles_per_row);
    const int sl0 = int(tile - (long long)bt * tiles_per_row) * kPeTile;
    const int b = bt / T, t = bt - b * T;
    __syncthreads();  // the previous tile's taps are dead
    for (int i = threadIdx.x; i < kPeTile * kPeTaps; i += blockDim.x) {
      const int tok = i / kPeTaps, k = i - tok * kPeTaps;
      const int s = s0 + sl0 + tok;  // global patch index
      float v = 0.f;
      if (sl0 + tok < S_local && s < S_total) {
        const int c = k / pp, r = k - c * pp;
        const int y = (s / Wn) * ph + r / pw, x = (s % Wn) * pw + r % pw;
        if (y < H && x < W) v = e_to_float(z[(size_t)b * sb + (size_t)c * sc + (size_t)t * st + (size_t)y * W + x]);
      }
      taps[tok][k] = v;
    }
    __syncthreads();
    if (!live) continue;
    const int n_tok = min(kPeTile, S_local - sl0);
    for (int tok = 0; tok < n_tok; ++tok) {
      const int s = s0 + sl0 + tok;
      PeVec o;
      if (s < S_total) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
        for (int k4 = 0; k4 < kPeTaps / 4; ++k4) {
          const float4 x4 = *reinterpret_cast<const float4*>(&taps[tok][k4 * 4]);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[j] = fmaf(x4.x, wr[k4 * 4][j], acc[j]);
            acc[j] = fmaf(x4.y, wr[k4 * 4 + 1][j], acc[j]);
            acc[j] = fmaf(x4.z, wr[k4 * 4 + 2][j], acc[j]);
            acc[j] = fmaf(x4.w, wr[k4 * 4 + 3][j], acc[j]);
          }
        }
        PeVec pe;
        pe.u = make_uint4(0, 0, 0, 0);
        if (pos != nullptr) pe.u = __ldg(reinterpret_cast<const uint4*>(pos + (size_t)s * C + cg * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float v0 = rbf(acc[2 * j]), v1 = rbf(acc[2 * j + 1]);          // conv output
          if (bias != nullptr) v0 = rbf(v0 + br[2 * j]), v1 = rbf(v1 + br[2 * j + 1]);  // + bias (separate eager op)
          if (pos != nullptr) {
            const float2 p2 = e2_to_float2(pe.h[j]);
            v0 += p2.x;
            v1 += p2.y;
          }
          o.h[j] = floats_to_e2(v0, v1);
        }
      } else {
        o.u = make_uint4(0, 0, 0, 0);  // padded patch columns of the last rank (split_sequence pads zeros)
      }
      *reinterpret_cast<uint4*>(out + ((size_t)bt * S_local + sl0 + tok) * C + cg * 8) = o.u;
    }
  }
}

}  // namespace vsb

using namespace vsb;

extern "C" int VSB_API(vsb_patch_embed)(const vsb_bf16* z, const vsb_bf16* w, const vsb_bf16* bias, const vsb_bf16* pos,
                                        vsb_bf16* out, int B, int Cin, int T, int H, int W, long long batch_stride,
                                        long long chan_stride, long long frame_stride, int ph, int pw, int C, int s0,
                                        int S_local, void* stream) {
  if (!z || !w || !out || B <= 0 || Cin <= 0 || T <= 0 || H <= 0 || W <= 0 || ph <= 0 || pw <= 0 || C <= 0 || s0 < 0 ||
      S_local <= 0)
    return fail(VSB_ERR_INVALID, "patch_embed: bad args");
  if (Cin * ph * pw != kPeTaps || (C & 7) || C / 8 > 256) return 1;  // not this kernel's shape: nothing launched
  if (!aligned16(out) || (pos && !aligned16(pos))) return fail(VSB_ERR_UNSUPPORTED, "patch_embed: alignment");
  const int Hn = (H + ph - 1) / ph, Wn = (W + pw - 1) / pw;
  const long long tiles = (long long)B * T * ((S_local + kPeTile - 1) / kPeTile);
  const int threads = ((C / 8 + 31) / 32) * 32;
  long long grid = tiles < 2LL * num_sms() ? tiles : 2LL * num_sms();
  patch_embed_kernel<<<(int)grid, threads, 0, (cudaStream_t)stream>>>(
      (const bf16*)z, (const bf16*)w, (const bf16*)bias, (const bf16*)pos, (bf16*)out, B, Cin, T, H, W, batch_stride,
      chan_stride, frame_stride, ph, pw, C, Wn, Hn * Wn, s0, S_local);
  return check_launch("patch_embed");
}
