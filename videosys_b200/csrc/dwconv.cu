// vsb200 -- depth-wise convolutions of Open-Sora-Plan v1.2.0's conv down-sampler variants (downsampler="k333_s222" /
// "k33_s22"), on the token-major activation: the attention down-sampler (conv + shortcut, stored straight into the
// sub-grid regrouping), its inverse regrouping fused into the gate + residual, and the conv feed-forward's 5x5 + 3x3 + 1x1
// depth-wise sum.  HBM-bound: every kernel reads its input once from HBM and writes its output once.
//
// Thread layout of both convolutions: lane = one 16-byte vector of 8 channels (a warp covers 256 channels of one token
// row, 512 contiguous bytes), warp = one output row h of the block's 8-row tile, and every thread produces kTW = 4 outputs
// along w from a sliding register window of kTW + KW - 1 input vectors per input row.  The halo rows a warp reads are the
// rows its neighbours in the block read too, so they come from L1; zero "same" padding = out-of-range taps load zeros.
// Depth-wise weights arrive tap-major ([taps, C]: one 16-byte load per tap gives 8 channels).  fp32 accumulation, 16-bit
// rounding at the points where the reference's eager ops round.
//
// Also Open-Sora-Plan v1.1.0's KV compression (compress_kv_factor): the strided depth-wise conv + LayerNorm that makes the
// keys / values of its second-half blocks (kv_compress_kernel, one warp per output row; see its comment).
#include "vsb_common.cuh"
#include "vsb_host.h"

namespace vsb {

namespace {

constexpr int kTW = 4;     // outputs per thread along w
constexpr int kRows = 8;   // warps per block = output rows per block

union V8 {
  uint4 u;
  elem2 h[4];
};

__device__ __forceinline__ void fma8(float (&acc)[8], const V8& x, const V8& w) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = e2_to_float2(x.h[j]), b = e2_to_float2(w.h[j]);
    acc[2 * j] = fmaf(a.x, b.x, acc[2 * j]);
    acc[2 * j + 1] = fmaf(a.y, b.y, acc[2 * j + 1]);
  }
}

__device__ __forceinline__ uint4 ld_or_zero(const bf16* p, bool ok) {
  return ok ? __ldg(reinterpret_cast<const uint4*>(p)) : make_uint4(0, 0, 0, 0);
}

// Block -> (bt, row tile, w tile, channel slice); w tiles vary fastest so neighbouring blocks share halos in L2.
struct Tile {
  int bt, h, w0, cv;
  bool ok;
};
__device__ __forceinline__ Tile tile_of(int H, int W, int nvec) {
  const int wt = (W + kTW - 1) / kTW, ht = (H + kRows - 1) / kRows;
  unsigned r = blockIdx.x;
  Tile t;
  const int wi = int(r % wt);
  r /= wt;
  const int hi = int(r % ht);
  r /= ht;
  t.bt = int(r);
  t.cv = blockIdx.y * 32 + (threadIdx.x & 31);
  t.h = hi * kRows + (threadIdx.x >> 5);
  t.w0 = wi * kTW;
  t.ok = t.h < H && t.cv < nvec;
  return t;
}

}  // namespace

// Attention down-sampler (DownSampler3d / DownSampler2d): x [B, T*H*W, C] token-major, w [KT*KH*KW, C] tap-major,
// out[(b dt dh dw), (t' h' w'), C] = bf16(bf16(bf16(conv(x)) + bias) + x): torch's GPU convolution rounds the conv and
// then adds the bias as a separate 16-bit op.
template <int KT, int KH, int KW>
__global__ void __launch_bounds__(256) dwconv_shuffle_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                             const bf16* __restrict__ bias, bf16* __restrict__ out, int T,
                                                             int H, int W, int C, int dt, int dh, int dw) {
  const int nvec = C >> 3;
  const Tile tl = tile_of(H, W, nvec);
  if (!tl.ok) return;
  const int b = tl.bt / T, t = tl.bt - b * T;
  const int c = tl.cv * 8;
  float acc[kTW][8];
#pragma unroll
  for (int o = 0; o < kTW; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[o][j] = 0.f;
#pragma unroll
  for (int kt = 0; kt < KT; ++kt) {
    const int ti = t + kt - KT / 2;
    const bool tok = ti >= 0 && ti < T;
#pragma unroll
    for (int kh = 0; kh < KH; ++kh) {
      const int hi = tl.h + kh - KH / 2;
      const bool rok = tok && hi >= 0 && hi < H;
      const bf16* row = x + (((size_t)b * T + ti) * H + hi) * (size_t)W * C + c;
      V8 win[kTW + KW - 1];
#pragma unroll
      for (int i = 0; i < kTW + KW - 1; ++i) {
        const int wi = tl.w0 + i - KW / 2;
        win[i].u = ld_or_zero(row + (size_t)wi * C, rok && wi >= 0 && wi < W);
      }
#pragma unroll
      for (int kw = 0; kw < KW; ++kw) {
        V8 wt;
        wt.u = __ldg(reinterpret_cast<const uint4*>(w + (size_t)((kt * KH + kh) * KW + kw) * C + c));
#pragma unroll
        for (int o = 0; o < kTW; ++o) fma8(acc[o], win[o + kw], wt);
      }
    }
  }
  V8 bv;
  bv.u = __ldg(reinterpret_cast<const uint4*>(bias + c));
  const int Hs = H / dh, Ws = W / dw, Ns = (T / dt) * Hs * Ws;
  const int sub_th = (b * dt + t % dt) * dh + tl.h % dh;
  const int tok_th = ((t / dt) * Hs + tl.h / dh) * Ws;
  const bf16* xc = x + (((size_t)b * T + t) * H + tl.h) * (size_t)W * C + c;
#pragma unroll
  for (int o = 0; o < kTW; ++o) {
    const int wo = tl.w0 + o;
    if (wo >= W) break;
    V8 xv, r;
    xv.u = __ldg(reinterpret_cast<const uint4*>(xc + (size_t)wo * C));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 bb = e2_to_float2(bv.h[j]), xs = e2_to_float2(xv.h[j]);
      const float2 y = e2_to_float2(floats_to_e2(rbf(acc[o][2 * j]) + bb.x, rbf(acc[o][2 * j + 1]) + bb.y));  // bf16(bf16(conv) + bias)
      r.h[j] = floats_to_e2(y.x + xs.x, y.y + xs.y);                                                         // bf16(. + x)
    }
    const size_t orow = (size_t)(sub_th * dw + wo % dw) * Ns + tok_th + wo / dw;
    *reinterpret_cast<uint4*>(out + orow * C + c) = r.u;
  }
}

// Conv feed-forward (FeedForward_Conv2d, per frame): h [BT, H, W, C2], w [25 + 9 + 1, C2] tap-major (5x5 taps, then 3x3,
// then 1x1), bias [3, C2];  out = bf16(bf16(bf16(h + c5) + c3) + c1), ck = bf16(bf16(conv_k(h)) + bias_k).
__global__ void __launch_bounds__(256) dwconv_ffn_kernel(const bf16* __restrict__ hsrc, const bf16* __restrict__ w,
                                                         const bf16* __restrict__ bias, bf16* __restrict__ out, int H, int W,
                                                         int C) {
  const int nvec = C >> 3;
  const Tile tl = tile_of(H, W, nvec);
  if (!tl.ok) return;
  const int c = tl.cv * 8;
  float a5[kTW][8], a3[kTW][8];
#pragma unroll
  for (int o = 0; o < kTW; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) a5[o][j] = a3[o][j] = 0.f;
  const bf16* img = hsrc + (size_t)tl.bt * H * W * C + c;
#pragma unroll
  for (int kh = 0; kh < 5; ++kh) {
    const int hi = tl.h + kh - 2;
    const bool rok = hi >= 0 && hi < H;
    const bf16* row = img + (size_t)hi * W * C;
    V8 win[kTW + 4];
#pragma unroll
    for (int i = 0; i < kTW + 4; ++i) {
      const int wi = tl.w0 + i - 2;
      win[i].u = ld_or_zero(row + (size_t)wi * C, rok && wi >= 0 && wi < W);
    }
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      V8 wt;
      wt.u = __ldg(reinterpret_cast<const uint4*>(w + (size_t)(kh * 5 + kw) * C + c));
#pragma unroll
      for (int o = 0; o < kTW; ++o) fma8(a5[o], win[o + kw], wt);
      if (kh >= 1 && kh <= 3 && kw >= 1 && kw <= 3) {
        wt.u = __ldg(reinterpret_cast<const uint4*>(w + (size_t)(25 + (kh - 1) * 3 + (kw - 1)) * C + c));
#pragma unroll
        for (int o = 0; o < kTW; ++o) fma8(a3[o], win[o + kw], wt);
      }
    }
  }
  V8 b5, b3, b1, w1;
  b5.u = __ldg(reinterpret_cast<const uint4*>(bias + c));
  b3.u = __ldg(reinterpret_cast<const uint4*>(bias + C + c));
  b1.u = __ldg(reinterpret_cast<const uint4*>(bias + 2 * C + c));
  w1.u = __ldg(reinterpret_cast<const uint4*>(w + (size_t)34 * C + c));
  const bf16* xc = img + (size_t)tl.h * W * C;
  bf16* oc = out + ((size_t)tl.bt * H + tl.h) * W * C + c;
#pragma unroll
  for (int o = 0; o < kTW; ++o) {
    const int wo = tl.w0 + o;
    if (wo >= W) break;
    V8 xv, r;
    xv.u = __ldg(reinterpret_cast<const uint4*>(xc + (size_t)wo * C));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 xs = e2_to_float2(xv.h[j]);
      const float2 q5 = e2_to_float2(b5.h[j]), q3 = e2_to_float2(b3.h[j]), q1 = e2_to_float2(b1.h[j]);
      const float2 k1 = e2_to_float2(w1.h[j]);
      const float2 c5 = e2_to_float2(floats_to_e2(rbf(a5[o][2 * j]) + q5.x, rbf(a5[o][2 * j + 1]) + q5.y));
      const float2 c3 = e2_to_float2(floats_to_e2(rbf(a3[o][2 * j]) + q3.x, rbf(a3[o][2 * j + 1]) + q3.y));
      const float2 c1 = e2_to_float2(floats_to_e2(rbf(xs.x * k1.x) + q1.x, rbf(xs.y * k1.y) + q1.y));
      const float2 s1 = e2_to_float2(floats_to_e2(xs.x + c5.x, xs.y + c5.y));
      const float2 s2 = e2_to_float2(floats_to_e2(s1.x + c3.x, s1.y + c3.y));
      r.h[j] = floats_to_e2(s2.x + c1.x, s2.y + c1.y);
    }
    *reinterpret_cast<uint4*>(oc + (size_t)wo * C) = r.u;
  }
}

// out[b, (t h w)] = bf16(x + bf16(gate[b] * y[(b t%dt h%dh w%dw), (t/dt h/dh w/dw)])): DownSampler.reverse fused into the
// load of the gate + residual (one pass, 2 reads + 1 write).
__global__ void __launch_bounds__(256) gate_residual_unshuffle_kernel(const bf16* __restrict__ x, const bf16* __restrict__ y,
                                                                      bf16* __restrict__ out, const bf16* __restrict__ mod,
                                                                      int gate_row, int T, int H, int W, int C, int dt,
                                                                      int dh, int dw, long long nvec_total) {
  const int nvec = C >> 3;
  const int Hs = H / dh, Ws = W / dw, Ns = (T / dt) * Hs * Ws;
  const unsigned HW = (unsigned)H * W, THW = HW * T;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec_total;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned row = unsigned(i / nvec);
    const int vi = int(i - (long long)row * nvec);
    const unsigned b = row / THW, r = row - b * THW;
    const unsigned t = r / HW, hw = r - t * HW;
    const unsigned h = hw / W, wq = hw - h * W;
    const unsigned sub = ((b * dt + t % dt) * dh + h % dh) * dw + wq % dw;
    const unsigned tok = ((t / dt) * Hs + h / dh) * Ws + wq / dw;
    const bf16* gate = mod + ((size_t)b * 6 + gate_row) * C;
    V8 vx, vy, vg, o;
    vx.u = __ldg(reinterpret_cast<const uint4*>(x + i * 8));
    vy.u = __ldg(reinterpret_cast<const uint4*>(y + ((size_t)sub * Ns + tok) * C + vi * 8));
    vg.u = __ldg(reinterpret_cast<const uint4*>(gate + vi * 8));
#pragma unroll
    for (int j = 0; j < 4; ++j) o.h[j] = __hadd2_rn(vx.h[j], __hmul2_rn(vg.h[j], vy.h[j]));
    *reinterpret_cast<uint4*>(out + i * 8) = o.u;
  }
}

__device__ __forceinline__ float kvc_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// KV compression of Open-Sora-Plan v1.1.0 (attn.sr + attn.norm): x [B, T, H, W, C] token-major, window (kt, kh, kw) with
// stride = window, pad_t leading copies of frame 0; out [B, (T+pad_t)/kt, H/kh, W/kw, C] token-major.  One warp per output
// row, the row in registers (lane owns vectors lane, lane+32, ...).  Conv rounding (round_conv):
//   1: bf16(bf16(conv) + bias) -- cuDNN, which torch picks for the spatial Conv2d because the reference hands it a
//      channels-last view of the tokens (it rounds the conv, then adds the bias as a separate 16-bit op);
//   0: bf16(bias + conv), bias first in the fp32 sum -- ATen's native depthwise kernel, which the Conv1d takes (conv1d
//      makes its input contiguous).
// Then LayerNorm (two-pass fp32 statistics, affine) rounded once.
template <int kMaxVec>
__global__ void __launch_bounds__(256) kv_compress_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                          const bf16* __restrict__ bias, const bf16* __restrict__ ln_w,
                                                          const bf16* __restrict__ ln_b, bf16* __restrict__ out, int T,
                                                          int H, int W, int C, int kt, int kh, int kw, int pad_t, int Tc,
                                                          int Hc, int Wc, float eps, int round_conv, long long rows) {
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  const int taps = kt * kh * kw;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    long long r = row;
    const int wc = int(r % Wc);
    r /= Wc;
    const int hc = int(r % Hc);
    r /= Hc;
    const int tc = int(r % Tc);
    const int b = int(r / Tc);
    float acc[kMaxVec][8];
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec && !round_conv) {
        V8 bv;
        bv.u = __ldg(reinterpret_cast<const uint4*>(bias + vi * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = e2_to_float2(bv.h[j]);
          acc[i][2 * j] = f.x;
          acc[i][2 * j + 1] = f.y;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      }
    }
    // taps in (it, ih, iw) order: the order of the weight's [kt, kh, kw] extent and of ATen's native accumulation
#pragma unroll 1
    for (int tap = 0; tap < taps; ++tap) {
      const int iw = tap % kw, ih = (tap / kw) % kh, it = tap / (kw * kh);
      const int tp = tc * kt + it - pad_t;
      const int t = tp < 0 ? 0 : tp;
      const bf16* xr = x + ((((size_t)b * T + t) * H + hc * kh + ih) * W + wc * kw + iw) * C;
      const bf16* wr = w + (size_t)tap * C;
      V8 xv[kMaxVec];
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i) {
        const int vi = lane + i * 32;
        if (vi < nvec) xv[i].u = __ldg(reinterpret_cast<const uint4*>(xr + vi * 8));
      }
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i) {
        const int vi = lane + i * 32;
        if (vi < nvec) {
          V8 wv;
          wv.u = __ldg(reinterpret_cast<const uint4*>(wr + vi * 8));
          fma8(acc[i], xv[i], wv);
        }
      }
    }
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        V8 bv;
        if (round_conv) bv.u = __ldg(reinterpret_cast<const uint4*>(bias + vi * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float y0 = rbf(acc[i][2 * j]), y1 = rbf(acc[i][2 * j + 1]);
          if (round_conv) {
            const float2 f = e2_to_float2(bv.h[j]);
            y0 = rbf(y0 + f.x);
            y1 = rbf(y1 + f.y);
          }
          acc[i][2 * j] = y0;
          acc[i][2 * j + 1] = y1;
          sum += y0 + y1;
        }
      }
    }
    const float mean = kvc_warp_sum(sum) / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = acc[i][j] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(kvc_warp_sum(sq) / (float)C + eps);
    bf16* orow = out + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        V8 gv, bv, o;
        gv.u = __ldg(reinterpret_cast<const uint4*>(ln_w + vi * 8));
        bv.u = __ldg(reinterpret_cast<const uint4*>(ln_b + vi * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 g = e2_to_float2(gv.h[j]), bb = e2_to_float2(bv.h[j]);
          o.h[j] = floats_to_e2((acc[i][2 * j] - mean) * rstd * g.x + bb.x, (acc[i][2 * j + 1] - mean) * rstd * g.y + bb.y);
        }
        *reinterpret_cast<uint4*>(orow + vi * 8) = o.u;
      }
    }
  }
}

}  // namespace vsb

using namespace vsb;

static int conv_grid(long long BT, int H, int W, int C, dim3* g) {
  const long long tiles = BT * ((H + kRows - 1) / kRows) * ((W + kTW - 1) / kTW);
  if (tiles >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "dwconv: %lld tiles", tiles);
  *g = dim3((unsigned)tiles, (unsigned)((C / 8 + 31) / 32), 1);
  return VSB_OK;
}

extern "C" int VSB_API(vsb_dwconv_shuffle)(const vsb_bf16* x, const vsb_bf16* w_taps, const vsb_bf16* bias, vsb_bf16* out,
                                           int B, int T, int H, int W, int C, int kt, int kh, int kw, int dt, int dh, int dw,
                                           void* stream) {
  if (!x || !w_taps || !bias || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || dt <= 0 || dh <= 0 || dw <= 0)
    return fail(VSB_ERR_INVALID, "dwconv_shuffle: bad args");
  if (T % dt || H % dh || W % dw) return fail(VSB_ERR_INVALID, "dwconv_shuffle: grid %dx%dx%d does not divide by %dx%dx%d", T, H, W, dt, dh, dw);
  if (C % 8 || !aligned16(x) || !aligned16(w_taps) || !aligned16(bias) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "dwconv_shuffle: need C %% 8 == 0 and 16B-aligned pointers");
  if ((long long)B * T * H * W * C >= (1ll << 40)) return fail(VSB_ERR_UNSUPPORTED, "dwconv_shuffle: too large");
  dim3 g;
  int rc = conv_grid((long long)B * T, H, W, C, &g);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
#define VSB_DWS(KT, KH, KW)                                                                                            \
  if (kt == KT && kh == KH && kw == KW) {                                                                              \
    dwconv_shuffle_kernel<KT, KH, KW><<<g, 256, 0, st>>>((const bf16*)x, (const bf16*)w_taps, (const bf16*)bias,        \
                                                         (bf16*)out, T, H, W, C, dt, dh, dw);                           \
    return check_launch("dwconv_shuffle");                                                                             \
  }
  VSB_DWS(3, 3, 3)
  VSB_DWS(1, 3, 3)
  VSB_DWS(3, 5, 5)
  VSB_DWS(1, 5, 5)
  VSB_DWS(3, 3, 5)
  VSB_DWS(1, 3, 5)
  VSB_DWS(3, 5, 3)
  VSB_DWS(1, 5, 3)
#undef VSB_DWS
  return fail(VSB_ERR_UNSUPPORTED, "dwconv_shuffle: kernel %dx%dx%d (kt in {1,3}, kh and kw in {3,5})", kt, kh, kw);
}

extern "C" int VSB_API(vsb_dwconv_ffn)(const vsb_bf16* h, const vsb_bf16* w_taps, const vsb_bf16* bias, vsb_bf16* out, int BT,
                                       int H, int W, int C, void* stream) {
  if (!h || !w_taps || !bias || !out || BT <= 0 || H <= 0 || W <= 0 || C <= 0) return fail(VSB_ERR_INVALID, "dwconv_ffn: bad args");
  if (C % 8 || !aligned16(h) || !aligned16(w_taps) || !aligned16(bias) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "dwconv_ffn: need C %% 8 == 0 and 16B-aligned pointers");
  dim3 g;
  int rc = conv_grid(BT, H, W, C, &g);
  if (rc) return rc;
  dwconv_ffn_kernel<<<g, 256, 0, (cudaStream_t)stream>>>((const bf16*)h, (const bf16*)w_taps, (const bf16*)bias, (bf16*)out,
                                                         H, W, C);
  return check_launch("dwconv_ffn");
}

extern "C" int VSB_API(vsb_gate_residual_unshuffle)(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, const vsb_bf16* mod,
                                                    int gate_row, int B, int T, int H, int W, int C, int dt, int dh, int dw,
                                                    void* stream) {
  if (!x || !y || !out || !mod || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || dt <= 0 || dh <= 0 || dw <= 0 ||
      gate_row < 0 || gate_row > 5)
    return fail(VSB_ERR_INVALID, "gate_residual_unshuffle: bad args");
  if (T % dt || H % dh || W % dw) return fail(VSB_ERR_INVALID, "gate_residual_unshuffle: grid does not divide");
  if (C % 8 || !aligned16(x) || !aligned16(y) || !aligned16(out) || !aligned16(mod))
    return fail(VSB_ERR_UNSUPPORTED, "gate_residual_unshuffle: need C %% 8 == 0 and 16B-aligned pointers");
  const long long rows = (long long)B * T * H * W;
  if (rows >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "gate_residual_unshuffle: too many rows");
  const long long nvec = rows * (C / 8);
  long long blocks = (nvec + 1023) / 1024, cap = (long long)num_sms() * 8;
  gate_residual_unshuffle_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)x, (const bf16*)y, (bf16*)out, (const bf16*)mod, gate_row, T, H, W, C, dt, dh, dw, nvec);
  return check_launch("gate_residual_unshuffle");
}

extern "C" int VSB_API(vsb_kv_compress)(const vsb_bf16* x, const vsb_bf16* w_taps, const vsb_bf16* bias, const vsb_bf16* ln_w,
                                        const vsb_bf16* ln_b, vsb_bf16* out, int B, int T, int H, int W, int C, int kt, int kh,
                                        int kw, int pad_t, float eps, int round_conv, void* stream) {
  if (B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || kt <= 0 || kh <= 0 || kw <= 0 || pad_t < 0 ||
      (round_conv != 0 && round_conv != 1))
    return fail(VSB_ERR_INVALID, "kv_compress: bad args");
  const int Tc = (T + pad_t) / kt, Hc = H / kh, Wc = W / kw;
  if (Tc == 0 || Hc == 0 || Wc == 0)  // checked before the pointers: an empty output tensor has no storage
    return fail(VSB_ERR_INVALID, "kv_compress: empty output grid (%d+%d frames, %dx%d) for window %dx%dx%d", T, pad_t, H, W, kt, kh, kw);
  if (!x || !w_taps || !bias || !ln_w || !ln_b || !out) return fail(VSB_ERR_INVALID, "kv_compress: null pointer");
  if (C % 8) return fail(VSB_ERR_INVALID, "kv_compress: C %% 8 != 0 (C=%d)", C);
  if (C > 3072 || !aligned16(x) || !aligned16(w_taps) || !aligned16(bias) || !aligned16(ln_w) || !aligned16(ln_b) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "kv_compress: need C <= 3072 and 16B-aligned pointers");
  if ((long long)B * T * H * W * C >= (1ll << 40)) return fail(VSB_ERR_UNSUPPORTED, "kv_compress: too large");
  const long long rows = (long long)B * Tc * Hc * Wc;
  long long blocks = (rows + 7) / 8, cap = (long long)num_sms() * 16;
  const int grid = (int)(blocks < cap ? blocks : cap);
  cudaStream_t st = (cudaStream_t)stream;
#define VSB_KVC(MV)                                                                                                    \
  kv_compress_kernel<MV><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)w_taps, (const bf16*)bias, (const bf16*)ln_w, \
                                               (const bf16*)ln_b, (bf16*)out, T, H, W, C, kt, kh, kw, pad_t, Tc, Hc, Wc, eps, \
                                               round_conv, rows)
  if (C <= 1280)
    VSB_KVC(5);
  else
    VSB_KVC(12);
#undef VSB_KVC
  return check_launch("kv_compress");
}
