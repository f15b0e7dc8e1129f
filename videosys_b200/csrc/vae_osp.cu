// vsb200 -- the Open-Sora-Plan causal-VAE decoder (models/autoencoders/autoencoder_kl_open_sora_plan.py): the pieces that
// vae_conv.cu does not already provide.  Activations are channels-last [B, T, H, W, C] 16-bit tensors throughout.
//
//   groupnorm_act_kernel    nn.GroupNorm(32, C, eps=1e-6) with the statistics of vsb_vae_groupnorm_stats, optionally followed
//                           by the reference's nonlinearity x * torch.sigmoid(x) (two eager ops, each rounded) or by
//                           F.silu (one rounding; nn.SiLU of the OpenSora v1.2 decoders)
//   depth_to_time_kernel    OpenSora's temporal decoder: [B, T, H, W, 2C] -> [B, 2T, H, W, C], a 16-byte gather copy
//   upsample_linear_kernel  F.interpolate(mode="trilinear", align_corners=False) by 2 in H and W and / or in T over frames
//                           1.. (Spatial2xTime2x3DUpsample, TimeUpsample2x, TimeUpsampleRes2x)
//   mix_kernel              TimeUpsampleRes2x's alpha * x + (1 - alpha) * conv(x), each eager op rounded
//   attn_split_kernel       q | k | v of the attention block's fused 1x1x1 GEMM -> per-frame Q, K [P, C] and V^T [C, P]
//                           (the wgmma GEMM's K-major operands), optionally through AttnBlock3D's frame / channel mixing
//   attn_softmax_kernel     softmax(bf16(S * scale)) per row of the materialised score matrix, fp32 inside, rounded once
//   attn_merge_kernel       AttnBlock3D's output scatter back to the real frames and channels
// S = Q K^T and O = P V run on the wgmma GEMM of gemm_wgmma.cu.
#include "vsb_common.cuh"
#include "vsb_host.h"

namespace vsb {

namespace {

int grid_for(long long work) {
  const long long blocks = (work + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm (+ nonlinearity).  torch keeps a 16-bit input's mean and rstd in the input's dtype and forms
// a = rstd * gamma, b = -a * mean + beta, y = a * x + b in fp32 (group_norm_kernel.cu), rounded.  The nonlinearity is
// torch.sigmoid (1 / (1 + exp(-x)) in fp32, rounded), then the product (rounded).
// ---------------------------------------------------------------------------------------------------------------------
struct GnArgs {
  const bf16* x;       // [B, T, H, W, C]
  const float* stats;  // [B, G, 2]
  const bf16* gamma;
  const bf16* beta;
  bf16* out;           // [B, T_out, H, W, C], frames t_off .. t_off + T - 1 written
  int B, T, HW, C, G, t_off, T_out, act;
};

__global__ void __launch_bounds__(256) groupnorm_act_kernel(const GnArgs a) {
  const int nv = a.C / 8;
  const long long total = (long long)a.B * a.T * a.HW * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long long p = i / nv;
    const int px = (int)(p % a.HW);
    p /= a.HW;
    const int t = (int)(p % a.T);
    const int b = (int)(p / a.T);
    const uint4 xu = __ldg(reinterpret_cast<const uint4*>(a.x + (size_t)i * 8));
    const uint4 gu = __ldg(reinterpret_cast<const uint4*>(a.gamma + v * 8));
    const uint4 bu = __ldg(reinterpret_cast<const uint4*>(a.beta + v * 8));
    const uint32_t xw[4] = {xu.x, xu.y, xu.z, xu.w}, gw[4] = {gu.x, gu.y, gu.z, gu.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 xx = unpack_bf16x2(xw[k]), gg = unpack_bf16x2(gw[k]), bb = unpack_bf16x2(bw[k]);
      float r[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gi = (v * 8 + 2 * k + e) / (a.C / a.G);
        const float mean = rbf(a.stats[2 * (b * a.G + gi)]), rstd = rbf(a.stats[2 * (b * a.G + gi) + 1]);
        const float sc = rstd * (e ? gg.y : gg.x);
        const float sh = fmaf(-sc, mean, e ? bb.y : bb.x);
        const float n = rbf(fmaf(sc, e ? xx.y : xx.x, sh));
        if (a.act == 2)
          r[e] = n / (1.f + expf(-n));  // F.silu: x / (1 + exp(-x)) in fp32, rounded once
        else
          r[e] = a.act ? n * rbf(1.f / (1.f + expf(-n))) : n;
      }
      o[k] = pack_bf16x2(r[0], r[1]);
    }
    const size_t ooff = (((size_t)b * a.T_out + a.t_off + t) * a.HW + px) * a.C + v * 8;
    *reinterpret_cast<uint4*>(a.out + ooff) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Linear 2x interpolation, align_corners=False, scale_factor given (ATen upsample_trilinear3d: source = max(0.5 * (dst +
// 0.5) - 0.5, 0), i0 = floor, i1 = min(i0 + 1, in - 1), lambda = source - i0).  With scale 1 a dimension is a copy.
// ---------------------------------------------------------------------------------------------------------------------
struct LinTap {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ LinTap lin_tap(int dst, int in, bool up) {
  if (!up) return LinTap{dst, dst, 1.f, 0.f};
  const float src = fmaxf(0.5f * (dst + 0.5f) - 0.5f, 0.f);
  const int i0 = (int)src;
  const float l1 = src - (float)i0;
  return LinTap{i0, i0 < in - 1 ? i0 + 1 : i0, 1.f - l1, l1};
}

struct LinArgs {
  const bf16* x;  // [B, T, H, W, C]
  bf16* out;      // [B, T_out, Ho, Wo, C], frames t_off .. t_off + To - 1 written
  int B, T, H, W, C, To, Ho, Wo, t_off, T_out, spatial, temporal;
};

__global__ void __launch_bounds__(256) upsample_linear_kernel(const LinArgs a) {
  const int nv = a.C / 8;
  const long long total = (long long)a.B * a.To * a.Ho * a.Wo * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long long p = i / nv;
    const int xo = (int)(p % a.Wo);
    p /= a.Wo;
    const int yo = (int)(p % a.Ho);
    p /= a.Ho;
    const int to = (int)(p % a.To);
    const int b = (int)(p / a.To);
    LinTap tt;
    if (a.temporal && to > 0) {  // frames 1.. are interpolated on their own (x_ = x[:, :, 1:])
      tt = lin_tap(to - 1, a.T - 1, true);
      tt.i0 += 1;
      tt.i1 += 1;
    } else {
      tt = LinTap{to, to, 1.f, 0.f};
    }
    const LinTap th = lin_tap(yo, a.H, a.spatial), tw = lin_tap(xo, a.W, a.spatial);
    const bf16* xb = a.x + (size_t)b * a.T * a.H * a.W * a.C + v * 8;
    uint32_t src[8][4];
    const int ts[2] = {tt.i0, tt.i1}, hs[2] = {th.i0, th.i1}, ws[2] = {tw.i0, tw.i1};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + (((size_t)ts[c >> 2] * a.H + hs[(c >> 1) & 1]) * a.W + ws[c & 1]) * a.C));
      src[c][0] = u.x;
      src[c][1] = u.y;
      src[c][2] = u.z;
      src[c][3] = u.w;
    }
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float r[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float q[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float2 f = unpack_bf16x2(src[c][k]);
          q[c] = e ? f.y : f.x;
        }
        // the nesting of upsample_trilinear3d_out_frame: t outer, then h, then w
        r[e] = tt.l0 * (th.l0 * (tw.l0 * q[0] + tw.l1 * q[1]) + th.l1 * (tw.l0 * q[2] + tw.l1 * q[3])) +
               tt.l1 * (th.l0 * (tw.l0 * q[4] + tw.l1 * q[5]) + th.l1 * (tw.l0 * q[6] + tw.l1 * q[7]));
      }
      o[k] = pack_bf16x2(r[0], r[1]);
    }
    const size_t ooff = ((((size_t)b * a.T_out + a.t_off + to) * a.Ho + yo) * a.Wo + xo) * a.C + v * 8;
    *reinterpret_cast<uint4*>(a.out + ooff) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// out = bf16(bf16(alpha * x) + bf16(one_minus_alpha * y)); x = frames t_off .. of xbuf [B, T_x, n] (n = H*W*C)
__global__ void __launch_bounds__(256) mix_kernel(const bf16* __restrict__ xbuf, const bf16* __restrict__ y, bf16* __restrict__ out,
                                                  int B, int T, long long n, int t_off, int T_x, float alpha, float oma) {
  const long long nv = n / 8;
  const long long total = (long long)B * T * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long bt = i / nv, r = i % nv;
    const int b = (int)(bt / T), t = (int)(bt % T);
    const uint4 xu = __ldg(reinterpret_cast<const uint4*>(xbuf + (((size_t)b * T_x + t_off + t) * nv + r) * 8));
    const uint4 yu = __ldg(reinterpret_cast<const uint4*>(y + (size_t)i * 8));
    const uint32_t xw[4] = {xu.x, xu.y, xu.z, xu.w}, yw[4] = {yu.x, yu.y, yu.z, yu.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 xx = unpack_bf16x2(xw[k]), yy = unpack_bf16x2(yw[k]);
      o[k] = pack_bf16x2(rbf(alpha * xx.x) + rbf(oma * yy.x), rbf(alpha * xx.y) + rbf(oma * yy.y));
    }
    *reinterpret_cast<uint4*>(out + (size_t)i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Attention operands.  Pseudo-frame f = b * T + j, pseudo-channel ch of pixel p reads qkv[b, j, p, which * C + ch]
// (AttnBlock3DFix), or with mixed = 1 qkv[b, m % T, p, which * C + m / T], m = j * C + ch: AttnBlock3D's
// reshape(b*t, c, h*w) of a b c t h w tensor.  Q [BT, P, C]; K [BT, Pp, C] and V^T [BT, C, Pp] are zero past P.
// One CTA per 32 pixels x 32 channels of a pseudo-frame; V goes through shared memory to be stored transposed.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ size_t qkv_off(int b, int j, int p, int ch, int which, int T, int P, int C, int mixed) {
  int t = j, c = ch;
  if (mixed) {
    const long long m = (long long)j * C + ch;
    t = (int)(m % T);
    c = (int)(m / T);
  }
  return (((size_t)b * T + t) * P + p) * (3 * (size_t)C) + (size_t)which * C + c;
}

__global__ void __launch_bounds__(256) attn_split_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ q, bf16* __restrict__ k,
                                                         bf16* __restrict__ vt, int T, int P, int Pp, int C, int mixed) {
  __shared__ bf16 tile[32][33];
  const int f = blockIdx.z, b = f / T, j = f % T;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const bf16 zero = float_to_e(0.f);
  for (int r = ty; r < 32; r += 8) {
    const int p = p0 + r, ch = c0 + tx;
    bf16 qv = zero, kv = zero, vv = zero;
    if (p < P) {
      qv = qkv[qkv_off(b, j, p, ch, 0, T, P, C, mixed)];
      kv = qkv[qkv_off(b, j, p, ch, 1, T, P, C, mixed)];
      vv = qkv[qkv_off(b, j, p, ch, 2, T, P, C, mixed)];
      q[((size_t)f * P + p) * C + ch] = qv;
    }
    if (p < Pp) k[((size_t)f * Pp + p) * C + ch] = kv;
    tile[r][tx] = vv;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int ch = c0 + r, p = p0 + tx;
    if (p < Pp) vt[((size_t)f * C + ch) * Pp + p] = tile[tx][r];
  }
}

// One CTA per score row: s = bf16(S * scale) (w_ * c ** -0.5), then softmax over the P valid columns in fp32
// (exp(s - max) / sum, ATen's epilogue), rounded once; columns P .. Pp - 1 are set to zero.
constexpr int kSmThreads = 256;

__global__ void __launch_bounds__(kSmThreads) attn_softmax_kernel(bf16* __restrict__ S, int P, int Pp, float scale) {
  __shared__ float red[kSmThreads / 32];
  bf16* row = S + (size_t)blockIdx.x * Pp;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < P; c += kSmThreads) mx = fmaxf(mx, rbf(e_to_float(row[c]) * scale));
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < kSmThreads / 32; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < P; c += kSmThreads) sum += expf(rbf(e_to_float(row[c]) * scale) - mx);
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int w = 0; w < kSmThreads / 32; ++w) sum += red[w];
  for (int c = threadIdx.x; c < Pp; c += kSmThreads)
    row[c] = c < P ? float_to_e(expf(rbf(e_to_float(row[c]) * scale) - mx) / sum) : float_to_e(0.f);
}

// out[b, t, p, c] = o[b * T + m / C, p, m % C], m = c * T + t: AttnBlock3D's h_.reshape(b, c, t, h, w)
__global__ void __launch_bounds__(256) attn_merge_kernel(const bf16* __restrict__ o, bf16* __restrict__ out, int B, int T, int P, int C) {
  const long long total = (long long)B * T * P * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int p = (int)(r % P);
    r /= P;
    const int t = (int)(r % T), b = (int)(r / T);
    const long long m = (long long)c * T + t;
    out[i] = o[(((size_t)b * T + m / C) * P + p) * C + m % C];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Depth to time (OpenSora's temporal decoder, rearrange "B (C ts) T H W -> B C (T ts) H W", ts = 2): channel 2c + ts of
// input frame t is channel c of output frame 2t + ts.  One thread per 16 input channels of a pixel: two 16-byte loads,
// the even / odd halves of each 32-bit word sorted apart, one 16-byte store into each of the two output frames.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) depth_to_time_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int B, int T,
                                                            int HW, int C, int t_off, int T_out) {
  const int nv = C / 8;  // output vectors per pixel = input vectors per pixel / 2
  const long long total = (long long)B * T * HW * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long long p = i / nv;
    const int px = (int)(p % HW);
    p /= HW;
    const int t = (int)(p % T), b = (int)(p / T);
    const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)i * 16);
    const uint4 u0 = __ldg(src), u1 = __ldg(src + 1);
    const uint32_t w[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
    uint32_t ev[4], od[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ev[k] = __byte_perm(w[2 * k], w[2 * k + 1], 0x5410);  // low halves: ts = 0
      od[k] = __byte_perm(w[2 * k], w[2 * k + 1], 0x7632);  // high halves: ts = 1
    }
    const size_t o0 = (((size_t)b * T_out + t_off + 2 * t) * HW + px) * C + v * 8;
    *reinterpret_cast<uint4*>(out + o0) = make_uint4(ev[0], ev[1], ev[2], ev[3]);
    *reinterpret_cast<uint4*>(out + o0 + (size_t)HW * C) = make_uint4(od[0], od[1], od[2], od[3]);
  }
}

}  // namespace

}  // namespace vsb

using namespace vsb;

extern "C" int VSB_API(vsb_vae_depth_to_time)(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C, int t_off,
                                              int T_out, void* stream) {
  if (!x || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || t_off < 0 || t_off + 2 * T > T_out)
    return fail(VSB_ERR_INVALID, "vae_depth_to_time: bad args");
  if (C % 8 || !aligned16(x) || !aligned16(out)) return fail(VSB_ERR_UNSUPPORTED, "vae_depth_to_time: need C %% 8 == 0, 16B-aligned");
  depth_to_time_kernel<<<grid_for((long long)B * T * H * W * (C / 8)), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)out, B, T,
                                                                                                       H * W, C, t_off, T_out);
  return check_launch("vae_depth_to_time");
}

extern "C" int VSB_API(vsb_vae_groupnorm_act)(const vsb_bf16* x, const float* stats, const vsb_bf16* gamma, const vsb_bf16* beta,
                                              vsb_bf16* out, int B, int T, int H, int W, int C, int G, int t_off, int T_out,
                                              int act, void* stream) {
  if (!x || !stats || !gamma || !beta || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || G <= 0 || t_off < 0 ||
      t_off + T > T_out)
    return fail(VSB_ERR_INVALID, "vae_groupnorm_act: bad args");
  if (C % 8 || C % G) return fail(VSB_ERR_UNSUPPORTED, "vae_groupnorm_act: C=%d G=%d", C, G);
  if (!aligned16(x) || !aligned16(gamma) || !aligned16(beta) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "vae_groupnorm_act: misaligned pointer");
  GnArgs a{(const bf16*)x, stats, (const bf16*)gamma, (const bf16*)beta, (bf16*)out, B, T, H * W, C, G, t_off, T_out,
           act == 2 ? 2 : (act ? 1 : 0)};
  groupnorm_act_kernel<<<grid_for((long long)B * T * H * W * (C / 8)), 256, 0, (cudaStream_t)stream>>>(a);
  return check_launch("vae_groupnorm_act");
}

extern "C" int VSB_API(vsb_vae_upsample_linear2x)(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C, int spatial,
                                                  int temporal, int t_off, int T_out, void* stream) {
  if (!x || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || t_off < 0) return fail(VSB_ERR_INVALID, "vae_upsample_linear2x: bad args");
  const int To = (temporal && T > 1) ? 1 + 2 * (T - 1) : T;
  if (t_off + To > T_out) return fail(VSB_ERR_INVALID, "vae_upsample_linear2x: %d frames after t_off=%d exceed T_out=%d", To, t_off, T_out);
  if (C % 8 || !aligned16(x) || !aligned16(out)) return fail(VSB_ERR_UNSUPPORTED, "vae_upsample_linear2x: need C %% 8 == 0, 16B-aligned");
  const int Ho = spatial ? 2 * H : H, Wo = spatial ? 2 * W : W;
  LinArgs a{(const bf16*)x, (bf16*)out, B, T, H, W, C, To, Ho, Wo, t_off, T_out, spatial ? 1 : 0, temporal ? 1 : 0};
  upsample_linear_kernel<<<grid_for((long long)B * To * Ho * Wo * (C / 8)), 256, 0, (cudaStream_t)stream>>>(a);
  return check_launch("vae_upsample_linear2x");
}

extern "C" int VSB_API(vsb_vae_mix)(const vsb_bf16* xbuf, const vsb_bf16* y, vsb_bf16* out, int B, int T, long long n, int t_off,
                                    int T_x, float alpha, float one_minus_alpha, void* stream) {
  if (!xbuf || !y || !out || B <= 0 || T <= 0 || n <= 0 || t_off < 0 || t_off + T > T_x) return fail(VSB_ERR_INVALID, "vae_mix: bad args");
  if (n % 8 || !aligned16(xbuf) || !aligned16(y) || !aligned16(out)) return fail(VSB_ERR_UNSUPPORTED, "vae_mix: need n %% 8 == 0, 16B-aligned");
  mix_kernel<<<grid_for((long long)B * T * (n / 8)), 256, 0, (cudaStream_t)stream>>>((const bf16*)xbuf, (const bf16*)y, (bf16*)out, B, T,
                                                                                       n, t_off, T_x, alpha, one_minus_alpha);
  return check_launch("vae_mix");
}

extern "C" int VSB_API(vsb_vae_attn_split)(const vsb_bf16* qkv, vsb_bf16* q, vsb_bf16* k, vsb_bf16* vt, int B, int T, int P, int Pp,
                                           int C, int mixed, void* stream) {
  if (!qkv || !q || !k || !vt || B <= 0 || T <= 0 || P <= 0 || Pp < P || C <= 0) return fail(VSB_ERR_INVALID, "vae_attn_split: bad args");
  if (C % 32 || Pp % 8) return fail(VSB_ERR_UNSUPPORTED, "vae_attn_split: need C %% 32 == 0, Pp %% 8 == 0 (C=%d Pp=%d)", C, Pp);
  if ((long long)B * T > 65535) return fail(VSB_ERR_UNSUPPORTED, "vae_attn_split: B*T=%lld frames", (long long)B * T);
  attn_split_kernel<<<dim3((Pp + 31) / 32, C / 32, B * T), 256, 0, (cudaStream_t)stream>>>((const bf16*)qkv, (bf16*)q, (bf16*)k, (bf16*)vt,
                                                                                           T, P, Pp, C, mixed ? 1 : 0);
  return check_launch("vae_attn_split");
}

extern "C" int VSB_API(vsb_vae_attn_softmax)(vsb_bf16* S, int rows, int P, int Pp, float scale, void* stream) {
  if (!S || rows <= 0 || P <= 0 || Pp < P) return fail(VSB_ERR_INVALID, "vae_attn_softmax: bad args");
  attn_softmax_kernel<<<rows, kSmThreads, 0, (cudaStream_t)stream>>>((bf16*)S, P, Pp, scale);
  return check_launch("vae_attn_softmax");
}

extern "C" int VSB_API(vsb_vae_attn_merge)(const vsb_bf16* o, vsb_bf16* out, int B, int T, int P, int C, void* stream) {
  if (!o || !out || B <= 0 || T <= 0 || P <= 0 || C <= 0) return fail(VSB_ERR_INVALID, "vae_attn_merge: bad args");
  attn_merge_kernel<<<grid_for((long long)B * T * P * C), 256, 0, (cudaStream_t)stream>>>((const bf16*)o, (bf16*)out, B, T, P, C);
  return check_launch("vae_attn_merge");
}
