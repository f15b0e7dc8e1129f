// vsb200 -- the CogVideoX VAE decoder (models/autoencoders/autoencoder_kl_cogvideox.py): causal 3-D convolution as an
// implicit GEMM on the warpgroup tensor cores, GroupNorm statistics, the spatially conditioned norm + SiLU, and the
// nearest 2x up-sampler.  Activations are channels-last [B, T, H, W, C] 16-bit tensors throughout.
//
// vae_conv_kernel: one CTA per (sample, output frame, 8 x 16 pixel tile, BN output channels), three warpgroups as in
// gemm_wgmma.cu:
//   warpgroup 0     TMA producer (one thread).  K runs over (tap, 64-channel slice).  The A tile of a K step is one
//                   5-D TMA box (64 channels, 16 columns, 8 rows, 1 frame, 1 sample) of the channels-last input at the
//                   tap-shifted coordinates: its 128 pixel rows of 128 bytes are exactly a 128 x 64 K-major, 128B-swizzled
//                   wgmma tile.  The spatial zero padding of the reference (F.pad, :131-132) is the TMA out-of-bounds
//                   fill, and so are the missing channels when Cin = 16 (conv_in).  The W tile is a BN x 64 box of the
//                   tap-major packed weights [Cout_pad, taps * Cin_pad].
//   warpgroups 1-2  consumers: pixel rows 0..63 / 64..127, wgmma.m64nBNk16 from the swizzled stages.
//   epilogue        + bias (rounded the way torch's convolution rounds, see round_conv), optional + residual, masked
//                   stores of the valid pixels and the Cout real channels (Cout = 3 for conv_out, 4 for the OpenSora
//                   temporal decoder's).
// TAPS is the number of spatial taps per frame: 9 for the (kt, 3, 3) convolutions, 1 for the (kt, 1, 1) time-axis
// convolution of the SVD temporal decoder (vsb_vae_conv_time), where only the A box's frame coordinate moves per tap.
// MIX adds that decoder's residual and AlphaBlender to the epilogue (see vsb_vae_conv_time).
// SHW / ST are the spatial and temporal strides of the down-sampling convolutions of the OpenSora v1.2 VAE encoder
// (vsb_vae_conv_down).  SHW = 2: the A box is a 5-D TMA box with traversal strides {1, 2, 2, 1, 1} over 64 x 32 x 16
// input elements, which lands the same 128 x 64 K-major tile; the taps start at (2 w0 + dx, 2 h0 + dy), dx, dy in
// {0, 1, 2}, and the (0, 1, 0, 1) zero padding of Downsample2D is the out-of-bounds fill.  ST = 2: output frame t reads
// input frames 2t - 1 .. 2t + 1; the causal time pad (one zero frame in front) is the out-of-bounds fill of frame -1.
#include "vsb_common.cuh"
#include "vsb_host.h"
#include "wgmma.cuh"

namespace vsb {

namespace {

constexpr int kConvBH = 8, kConvBW = 16;  // pixel tile: 8 rows x 16 columns = the 128-row M tile
constexpr int kConvBK = 64;
constexpr int kConvThreads = 384;
constexpr int kConvStages = 4;

template <int BN>
struct ConvCfg {
  static constexpr int kABytes = 128 * kConvBK * 2;
  static constexpr int kStageBytes = kABytes + BN * kConvBK * 2;
  // + 1024 for manual alignment, + 256 for barriers
  static constexpr int kSmemBytes = kConvStages * kStageBytes + 1024 + 256;
};

template <int BN>
__device__ __forceinline__ void conv_wgmma(float (&d)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 128)
    wgmma_m64n128k16_ss(d, da, db, 1u);
  else
    wgmma_m64n64k16_ss(d, da, db, 1u);
}

struct ConvArgs {
  const bf16* bias;   // [Cout]
  const bf16* resid;  // [B, T, H, W, Cout] or null
  bf16* out;          // [B, T, H, W, Cout]
  int T, H, W, Cout, kt, cin_slices, tiles_h, tiles_w, tiles_n, round_conv;
  float mix_a, mix_b;  // MIX only: the AlphaBlender's weights of resid and of resid + conv
};

template <int BN, int TAPS = 9, bool MIX = false, int SHW = 1, int ST = 1>
__global__ void __launch_bounds__(kConvThreads, 1)
vae_conv_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w, const ConvArgs a) {
  static_assert(TAPS == 9 || TAPS == 1, "3x3 or 1x1 spatial taps");
  static_assert((SHW == 1 || (SHW == 2 && TAPS == 9)) && (ST == 1 || ST == 2), "strides 1 or 2 (spatial: 3x3 taps)");
  using Cfg = ConvCfg<BN>;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kConvStages * Cfg::kStageBytes);
  uint64_t* empty = full + kConvStages;

  // N tiles fastest: the CTAs that share an input tile run together and find it in L2
  int r = blockIdx.x;
  const int n0 = (r % a.tiles_n) * BN;
  r /= a.tiles_n;
  const int w0 = (r % a.tiles_w) * kConvBW;
  r /= a.tiles_w;
  const int h0 = (r % a.tiles_h) * kConvBH;
  r /= a.tiles_h;
  const int t = r % a.T, b = r / a.T;
  const int taps = a.kt * TAPS;
  const int num_kb = taps * a.cin_slices;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < kConvStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      int kb = 0;
      for (int tap = 0; tap < taps; ++tap) {
        // stride 1: centred taps (-1, 0, 1); stride 2: the padding is on the far side only, taps (0, 1, 2)
        constexpr int kLead = SHW == 1 ? 1 : 0;
        const int dz = tap / TAPS, dy = TAPS == 9 ? (tap / 3) % 3 - kLead : 0, dx = TAPS == 9 ? tap % 3 - kLead : 0;
        for (int cs = 0; cs < a.cin_slices; ++cs, ++kb) {
          const int s = kb % kConvStages;
          mbar_wait_quiet(&empty[s], ((kb / kConvStages) & 1) ^ 1);
          unsigned char* st = smem + s * Cfg::kStageBytes;
          mbar_arrive_expect_tx(&full[s], Cfg::kStageBytes);
          tma_load_5d(&tm_x, &full[s], st, cs * kConvBK, SHW * w0 + dx, SHW * h0 + dy, ST * t + dz - (ST - 1), b);
          tma_load_2d(&tm_w, &full[s], st + Cfg::kABytes, (tap * a.cin_slices + cs) * kConvBK, n0);
        }
      }
    }
    return;
  }

  const int c = wg - 1;
  const int tid = threadIdx.x & 127;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const uint32_t s0 = smem_u32(smem);
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % kConvStages;
    mbar_wait_quiet(&full[s], (kb / kConvStages) & 1);
    const uint32_t sa = s0 + s * Cfg::kStageBytes + c * (64 * 128);
    const uint32_t sw = s0 + s * Cfg::kStageBytes + Cfg::kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kConvBK / 16; ++k) conv_wgmma<BN>(acc, wgmma_desc_sw128(sa + 32 * k), wgmma_desc_sw128(sw + 32 * k));
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0 && tid == 0) mbar_arrive(&empty[(kb - 1) % kConvStages]);
  }
  wgmma_wait<0>();

  // ===================== epilogue: rows are pixels of the 8 x 16 tile, columns output channels =====================
  const int warp = tid >> 5, lane = tid & 31;
  const int rl0 = c * 64 + warp * 16 + (lane >> 2);
  long long pix[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rl = rl0 + 8 * h;
    const int y = h0 + rl / kConvBW, x = w0 + rl % kConvBW;
    pix[h] = (y < a.H && x < a.W) ? (((long long)b * a.T + t) * a.H + y) * a.W + x : -1;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + j * 8 + 2 * (lane & 3);
    if (col >= a.Cout) continue;
    const bool two = col + 1 < a.Cout;
    const float b0 = e_to_float(a.bias[col]), b1 = two ? e_to_float(a.bias[col + 1]) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (pix[h] < 0) continue;
      float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
      if (a.round_conv) {  // the convolution is rounded to 16 bits, then the bias is added
        x0 = rbf(x0);
        x1 = rbf(x1);
      }
      x0 = rbf(x0 + b0);
      x1 = rbf(x1 + b1);
      const size_t off = (size_t)pix[h] * a.Cout + col;
      if constexpr (MIX) {  // xt = xs + v, then a * xs + b * xt, each eager op rounded (Cout % 64 == 0: both columns)
        const float2 sp = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.resid + off));
        const float s0 = sp.x, s1 = sp.y;
        x0 = rbf(rbf(a.mix_a * s0) + rbf(a.mix_b * rbf(s0 + x0)));
        x1 = rbf(rbf(a.mix_a * s1) + rbf(a.mix_b * rbf(s1 + x1)));
      } else if (a.resid != nullptr) {  // ResNet sum conv2(...) + inputs (:298), its own eager rounding
        x0 += e_to_float(a.resid[off]);
        if (two) x1 += e_to_float(a.resid[off + 1]);
      }
      if (two && (a.Cout & 1) == 0) {
        *reinterpret_cast<uint32_t*>(a.out + off) = pack_bf16x2(x0, x1);
      } else {
        a.out[off] = float_to_e(x0);
        if (two) a.out[off + 1] = float_to_e(x1);
      }
    }
  }
}

template <int BN, int TAPS = 9, bool MIX = false, int SHW = 1, int ST = 1>
int launch_conv(const CUtensorMap& tx, const CUtensorMap& tw, const ConvArgs& a, int B, cudaStream_t st) {
  const char* what = SHW * ST > 1 ? "vae_conv_down" : TAPS == 9 ? "vae_conv3d" : "vae_conv_time";
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(vae_conv_kernel<BN, TAPS, MIX, SHW, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         ConvCfg<BN>::kSmemBytes);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "%s: smem attr: %s", what, cudaGetErrorString(e));
    attr = true;
  }
  const long long tiles = (long long)B * a.T * a.tiles_h * a.tiles_w * a.tiles_n;
  if (tiles >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "%s: too many tiles", what);
  vae_conv_kernel<BN, TAPS, MIX, SHW, ST><<<(unsigned)tiles, kConvThreads, ConvCfg<BN>::kSmemBytes, st>>>(tx, tw, a);
  return check_launch(what);
}

// ---------------------------------------------------------------------------------------------------------------------
// time_conv_out of the SVD temporal decoder: Conv3d 3 -> 3, kernel (3, 1, 1), zero frames at both ends, one thread per
// pixel.  Each output is the 9 products summed in fp32 (frame-major, then input channel), rounded, + bias, rounded.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) time_conv_rgb_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                            const bf16* __restrict__ bias, bf16* __restrict__ out, int B,
                                                            int T, long long P) {
  __shared__ float ws[27], bs[3];
  if (threadIdx.x < 27) ws[threadIdx.x] = e_to_float(w[threadIdx.x]);  // [Cout, Cin, kt]
  if (threadIdx.x < 3) bs[threadIdx.x] = e_to_float(bias[threadIdx.x]);
  __syncthreads();
  const long long total = (long long)B * T * P;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)((i / P) % T);
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int dz = 0; dz < 3; ++dz) {
      const int ts = t + dz - 1;
      if (ts < 0 || ts >= T) continue;
      const bf16* src = x + (i + (long long)(dz - 1) * P) * 3;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v = e_to_float(src[ci]);
#pragma unroll
        for (int co = 0; co < 3; ++co) acc[co] = fmaf(ws[(co * 3 + ci) * 3 + dz], v, acc[co]);
      }
    }
#pragma unroll
    for (int co = 0; co < 3; ++co) out[i * 3 + co] = float_to_e(rbf(acc[co]) + bs[co]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm statistics: kGnChunks CTAs per sample each sum a fixed pixel subset per channel (fp32), then one thread per
// (sample, group) adds the partials in a fixed order in fp64.  No atomics: repeated launches are bit-identical.
// The sums are of x - k and (x - k)^2 with a pivot k per (sample, channel), the sample's first pixel: on a DC offset
// large against the spread (a flat region of a frame) plain E[x^2] - mean^2 in fp32 loses the variance to cancellation.
// The finalize merges the channels' (mean, M2) into the group's in fp64 (Chan et al.).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;

__global__ void __launch_bounds__(kGnThreads) gn_partial_kernel(const bf16* __restrict__ x, float* __restrict__ part,
                                                                long long P, int C) {
  __shared__ float red[kGnThreads][17];
  const int tpp = C / 8, ppi = kGnThreads / tpp;  // threads per pixel, pixels per iteration
  const int v = threadIdx.x % tpp, pl = threadIdx.x / tpp;
  const int b = blockIdx.y, chunk = blockIdx.x;
  float s[8], q[8], k[8];
  const bf16* xb = x + (size_t)b * P * C;
  {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + v * 8));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(w[i]);
      k[2 * i] = f.x;
      k[2 * i + 1] = f.y;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = 0.f;
  for (long long p = (long long)chunk * ppi + pl; p < P; p += (long long)VSB_GN_CHUNKS * ppi) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + p * C + v * 8));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(w[i]);
      const float d0 = f.x - k[2 * i], d1 = f.y - k[2 * i + 1];
      s[2 * i] += d0;
      s[2 * i + 1] += d1;
      q[2 * i] = fmaf(d0, d0, q[2 * i]);
      q[2 * i + 1] = fmaf(d1, d1, q[2 * i + 1]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red[threadIdx.x][i] = s[i];
    red[threadIdx.x][8 + i] = q[i];
  }
  __syncthreads();
  float* pb = part + ((size_t)b * VSB_GN_CHUNKS + chunk) * C * 2;
  for (int ch = threadIdx.x; ch < C; ch += kGnThreads) {
    const int vv = ch / 8, i = ch % 8;
    float ss = 0.f, qq = 0.f;
    for (int l = 0; l < ppi; ++l) {
      ss += red[l * tpp + vv][i];
      qq += red[l * tpp + vv][8 + i];
    }
    pb[2 * ch] = ss;
    pb[2 * ch + 1] = qq;
  }
}

// one channel's pivot-shifted sums over all chunks, in fp64: s = sum(x - k), q = sum((x - k)^2)
__device__ __forceinline__ void gn_channel_sums(const float* __restrict__ part, int b, int c, int C, double& s, double& q) {
  s = q = 0.0;
  for (int k = 0; k < VSB_GN_CHUNKS; ++k) {
    const float* pk = part + ((size_t)b * VSB_GN_CHUNKS + k) * C * 2 + 2 * c;
    s += pk[0];
    q += pk[1];
  }
}

__global__ void gn_finalize_kernel(const bf16* __restrict__ x, const float* __restrict__ part, float* __restrict__ stats,
                                   long long P, int C, int G, int B, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * G) return;
  const int b = i / G, g = i % G, cg = C / G;
  const bf16* pivot = x + (size_t)b * P * C + (size_t)g * cg;
  const double np = (double)P;
  double s, q, msum = 0.0;
  for (int c = 0; c < cg; ++c) {
    gn_channel_sums(part, b, g * cg + c, C, s, q);
    msum += (double)e_to_float(pivot[c]) + s / np;
  }
  const double mean = msum / cg;
  double m2 = 0.0;  // sum over the group of (x - mean)^2: each channel's M2 plus its mean's offset from the group's
  for (int c = 0; c < cg; ++c) {
    gn_channel_sums(part, b, g * cg + c, C, s, q);
    const double dm = (double)e_to_float(pivot[c]) + s / np - mean;
    m2 += fmax(q - s * s / np, 0.0) + np * dm * dm;
  }
  const double var = m2 / (np * cg);
  stats[2 * i] = (float)mean;
  stats[2 * i + 1] = rsqrtf((float)var + eps);
}

// ---------------------------------------------------------------------------------------------------------------------
// Spatial norm + SiLU: out = silu(GroupNorm(f) * zy + zb), zy / zb = conv_y / conv_b of the latent at latent resolution,
// gathered with F.interpolate's nearest rule (CogVideoXSpatialNorm3D.forward, :165-178).  Each eager op rounds.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
  // upsample_nearest (size given): floorf(dst * (float)in / out), clamped (aten/src/ATen/native/cuda/UpSample.cuh)
  const float scale = (float)in / (float)out;
  return min((int)floorf(dst * scale), in - 1);
}

struct SnArgs {
  const bf16* f;           // [B, T, H, W, C]
  const float* stats;      // [B, G, 2] mean, rstd
  const bf16* gamma;       // [C]
  const bf16* beta;        // [C]
  const bf16* zyb;         // [B, Tz, h, w, 2C]: conv_y | conv_b
  bf16* out;               // [B, T_out, H, W, C], frames t_off .. t_off + T - 1 written
  int B, T, H, W, C, G, Tz, h, w, t_off, T_out;
};

__global__ void __launch_bounds__(256) spatial_norm_silu_kernel(const SnArgs a) {
  const int nv = a.C / 8;
  const long long total = (long long)a.B * a.T * a.H * a.W * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long long p = i / nv;
    const int x = (int)(p % a.W);
    p /= a.W;
    const int y = (int)(p % a.H);
    p /= a.H;
    const int t = (int)(p % a.T);
    const int b = (int)(p / a.T);
    int zt;
    if (a.T > 1 && (a.T & 1)) {  // odd frame count: the first frame is interpolated on its own (:166-172)
      zt = t == 0 ? 0 : 1 + nearest_src(t - 1, a.Tz - 1, a.T - 1);
    } else {
      zt = nearest_src(t, a.Tz, a.T);
    }
    const int zy = nearest_src(y, a.h, a.H), zx = nearest_src(x, a.w, a.W);
    const size_t zoff = ((((size_t)b * a.Tz + zt) * a.h + zy) * a.w + zx) * (2 * a.C) + v * 8;
    const uint4 fu = __ldg(reinterpret_cast<const uint4*>(a.f + (size_t)i * 8));
    const uint4 yu = __ldg(reinterpret_cast<const uint4*>(a.zyb + zoff));
    const uint4 bu = __ldg(reinterpret_cast<const uint4*>(a.zyb + zoff + a.C));
    const uint4 gu = __ldg(reinterpret_cast<const uint4*>(a.gamma + v * 8));
    const uint4 be = __ldg(reinterpret_cast<const uint4*>(a.beta + v * 8));
    const uint32_t fw[4] = {fu.x, fu.y, fu.z, fu.w}, yw[4] = {yu.x, yu.y, yu.z, yu.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w},
                   gw[4] = {gu.x, gu.y, gu.z, gu.w}, ew[4] = {be.x, be.y, be.z, be.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 ff = unpack_bf16x2(fw[k]), zz = unpack_bf16x2(yw[k]), zb = unpack_bf16x2(bw[k]), gg = unpack_bf16x2(gw[k]),
                   bb = unpack_bf16x2(ew[k]);
      float r[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ch = v * 8 + 2 * k + e;
        const int gi = ch / (a.C / a.G);
        // torch keeps a 16-bit input's mean and rstd in the input's dtype; group_norm_kernel.cu then forms
        // a = rstd * gamma, b = -a * mean + beta and y = a * x + b in fp32, rounded
        const float mean = rbf(a.stats[2 * (b * a.G + gi)]), rstd = rbf(a.stats[2 * (b * a.G + gi) + 1]);
        const float sc = rstd * (e ? gg.y : gg.x);
        const float sh = fmaf(-sc, mean, e ? bb.y : bb.x);
        const float n = rbf(fmaf(sc, e ? ff.y : ff.x, sh));
        const float m = rbf(n * (e ? zz.y : zz.x));
        const float s = rbf(m + (e ? zb.y : zb.x));
        r[e] = s / (1.f + expf(-s));  // torch's silu: x / (1 + exp(-x)) in fp32
      }
      o[k] = pack_bf16x2(r[0], r[1]);
    }
    const size_t ooff = ((((size_t)b * a.T_out + a.t_off + t) * a.H + y) * a.W + x) * a.C + v * 8;
    *reinterpret_cast<uint4*>(a.out + ooff) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Nearest 2x up-sampling in H and W, and in T with compress_time (CogVideoXUpsample3D.forward, upsampling.py:40-60).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) upsample2x_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int B, int T,
                                                         int H, int W, int C, int T2, int compress_time) {
  const int nv = C / 8, H2 = 2 * H, W2 = 2 * W;
  const long long total = (long long)B * T2 * H2 * W2 * nv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long long p = i / nv;
    const int xo = (int)(p % W2);
    p /= W2;
    const int yo = (int)(p % H2);
    p /= H2;
    const int to = (int)(p % T2);
    const int b = (int)(p / T2);
    int ti = to;
    if (compress_time && T > 1) ti = (T & 1) ? (to == 0 ? 0 : 1 + (to - 1) / 2) : to / 2;
    const size_t src = ((((size_t)b * T + ti) * H + (yo >> 1)) * W + (xo >> 1)) * C + v * 8;
    reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(x + src));
  }
}

int grid_for(long long work) {
  const long long blocks = (work + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

}  // namespace vsb

using namespace vsb;

namespace vsb {
namespace {
// The two TMA operands of vae_conv_kernel: x [B, Tin, H, W, Cin] as 64-channel x 16 x 8 x 1 x 1 boxes and the packed
// weight [Cout_pad, K] as 64 x BN boxes, both 128B-swizzled.  shw = 2: the x box spans 32 x 16 pixels traversed with
// stride 2 in W and H (16 x 8 pixels land).
int conv_tmaps(CUtensorMap* tx, CUtensorMap* tw, const void* x, const void* w_packed, int B, int Tin, int H, int W, int Cin,
               unsigned long long K, int cout_pad, int BN, int shw = 1) {
  unsigned long long dx[5] = {(unsigned long long)Cin, (unsigned long long)W, (unsigned long long)H, (unsigned long long)Tin,
                              (unsigned long long)B};
  unsigned long long sx[4] = {(unsigned long long)Cin * 2, (unsigned long long)W * Cin * 2,
                              (unsigned long long)H * W * Cin * 2, (unsigned long long)Tin * H * W * Cin * 2};
  unsigned bx[5] = {kConvBK, (unsigned)(kConvBW * shw), (unsigned)(kConvBH * shw), 1, 1};
  unsigned ex[5] = {1, (unsigned)shw, (unsigned)shw, 1, 1};
  int rc = make_tmap_bf16(tx, x, 5, dx, sx, bx, CU_TENSOR_MAP_SWIZZLE_128B, ex);
  if (rc) return rc;
  unsigned long long dw[2] = {K, (unsigned long long)cout_pad};
  unsigned long long sw[1] = {K * 2};
  unsigned bw[2] = {kConvBK, (unsigned)BN};
  return make_tmap_bf16(tw, w_packed, 2, dw, sw, bw, CU_TENSOR_MAP_SWIZZLE_128B);
}
}  // namespace
}  // namespace vsb

extern "C" int VSB_API(vsb_vae_conv3d)(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias, const vsb_bf16* resid,
                                       vsb_bf16* out, int B, int T, int H, int W, int Cin, int Cout, int kt, int round_conv,
                                       void* stream) {
  if (!x || !w_packed || !bias || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0)
    return fail(VSB_ERR_INVALID, "vae_conv3d: bad args");
  if (kt != 1 && kt != 3) return fail(VSB_ERR_UNSUPPORTED, "vae_conv3d: kt=%d (need 1 or 3)", kt);
  if (!(Cin == 16 || Cin % 64 == 0)) return fail(VSB_ERR_UNSUPPORTED, "vae_conv3d: Cin=%d (need 16 or a multiple of 64)", Cin);
  if (!(Cout == 3 || Cout == 4 || Cout == 8 || Cout % 64 == 0))
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv3d: Cout=%d (need 3, 4, 8 or a multiple of 64)", Cout);
  if (!aligned16(x) || !aligned16(w_packed) || (resid && ((uintptr_t)resid & 3)) || ((uintptr_t)out & 3))
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv3d: misaligned pointer");
  const int BN = Cout % 128 == 0 ? 128 : 64;
  const int cin_pad = (Cin + 63) / 64 * 64, cout_pad = (Cout + BN - 1) / BN * BN;
  CUtensorMap tx, tw;
  int rc = conv_tmaps(&tx, &tw, x, w_packed, B, T + kt - 1, H, W, Cin, (unsigned long long)kt * 9 * cin_pad, cout_pad, BN);
  if (rc) return rc;
  ConvArgs a{(const bf16*)bias, (const bf16*)resid, (bf16*)out, T, H, W, Cout, kt, cin_pad / 64,
             (H + kConvBH - 1) / kConvBH, (W + kConvBW - 1) / kConvBW, cout_pad / BN, round_conv ? 1 : 0, 0.f, 0.f};
  if (BN == 128) return launch_conv<128>(tx, tw, a, B, (cudaStream_t)stream);
  return launch_conv<64>(tx, tw, a, B, (cudaStream_t)stream);
}

extern "C" int VSB_API(vsb_vae_conv_time)(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias,
                                          const vsb_bf16* resid, vsb_bf16* out, int B, int T, int H, int W, int Cin, int Cout,
                                          int kt, int mix, float mix_a, float mix_b, int round_conv, void* stream) {
  if (!x || !w_packed || !bias || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || kt <= 0 ||
      (mix && !resid))
    return fail(VSB_ERR_INVALID, "vae_conv_time: bad args");
  if (Cin % 64 || Cout % 64)
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv_time: Cin=%d Cout=%d (need multiples of 64)", Cin, Cout);
  if (!aligned16(x) || !aligned16(w_packed) || (resid && ((uintptr_t)resid & 3)) || ((uintptr_t)out & 3))
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv_time: misaligned pointer");
  const int BN = Cout % 128 == 0 ? 128 : 64;
  CUtensorMap tx, tw;
  int rc = conv_tmaps(&tx, &tw, x, w_packed, B, T + kt - 1, H, W, Cin, (unsigned long long)kt * Cin, Cout, BN);
  if (rc) return rc;
  ConvArgs a{(const bf16*)bias, (const bf16*)resid, (bf16*)out, T, H, W, Cout, kt, Cin / 64,
             (H + kConvBH - 1) / kConvBH, (W + kConvBW - 1) / kConvBW, Cout / BN, round_conv ? 1 : 0, mix_a, mix_b};
  cudaStream_t st = (cudaStream_t)stream;
  if (BN == 128) return mix ? launch_conv<128, 1, true>(tx, tw, a, B, st) : launch_conv<128, 1, false>(tx, tw, a, B, st);
  return mix ? launch_conv<64, 1, true>(tx, tw, a, B, st) : launch_conv<64, 1, false>(tx, tw, a, B, st);
}

extern "C" int VSB_API(vsb_vae_conv_down)(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias, vsb_bf16* out,
                                          int B, int Tin, int Hin, int Win, int Cin, int Cout, int kt, int stride_t,
                                          int stride_hw, int round_conv, void* stream) {
  if (!x || !w_packed || !bias || !out || B <= 0 || Tin <= 0 || Hin <= 0 || Win <= 0 || Cin <= 0 || Cout <= 0)
    return fail(VSB_ERR_INVALID, "vae_conv_down: bad args");
  const bool spatial = kt == 1 && stride_t == 1 && stride_hw == 2, temporal = kt == 3 && stride_t == 2 && stride_hw == 1;
  if (!spatial && !temporal)
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv_down: kt=%d strides (%d, %d) (need kt 1 / (1, 2) or kt 3 / (2, 1))", kt,
                stride_t, stride_hw);
  if ((spatial && (Hin < 2 || Win < 2)) || (temporal && Tin < 2))
    return fail(VSB_ERR_INVALID, "vae_conv_down: input %dx%dx%d smaller than the padded kernel", Tin, Hin, Win);
  if (!(Cin == 16 || Cin % 64 == 0)) return fail(VSB_ERR_UNSUPPORTED, "vae_conv_down: Cin=%d (need 16 or a multiple of 64)", Cin);
  if (!(Cout == 8 || Cout % 64 == 0)) return fail(VSB_ERR_UNSUPPORTED, "vae_conv_down: Cout=%d (need 8 or a multiple of 64)", Cout);
  if (!aligned16(x) || !aligned16(w_packed) || ((uintptr_t)out & 3))
    return fail(VSB_ERR_UNSUPPORTED, "vae_conv_down: misaligned pointer");
  // F.pad(x, (0, 1, 0, 1)) then a stride-2 3x3 conv: floor((H + 1 - 3) / 2) + 1; the causal time conv over 1 + Tin
  // frames: floor((Tin + 1 - 3) / 2) + 1
  const int T = temporal ? (Tin - 2) / 2 + 1 : Tin, H = spatial ? (Hin - 2) / 2 + 1 : Hin, W = spatial ? (Win - 2) / 2 + 1 : Win;
  const int BN = Cout % 128 == 0 ? 128 : 64;
  const int cin_pad = (Cin + 63) / 64 * 64, cout_pad = (Cout + BN - 1) / BN * BN;
  CUtensorMap tx, tw;
  int rc = conv_tmaps(&tx, &tw, x, w_packed, B, Tin, Hin, Win, Cin, (unsigned long long)kt * 9 * cin_pad, cout_pad, BN,
                      stride_hw);
  if (rc) return rc;
  ConvArgs a{(const bf16*)bias, nullptr, (bf16*)out, T, H, W, Cout, kt, cin_pad / 64,
             (H + kConvBH - 1) / kConvBH, (W + kConvBW - 1) / kConvBW, cout_pad / BN, round_conv ? 1 : 0, 0.f, 0.f};
  cudaStream_t st = (cudaStream_t)stream;
  if (spatial) return BN == 128 ? launch_conv<128, 9, false, 2, 1>(tx, tw, a, B, st) : launch_conv<64, 9, false, 2, 1>(tx, tw, a, B, st);
  return BN == 128 ? launch_conv<128, 9, false, 1, 2>(tx, tw, a, B, st) : launch_conv<64, 9, false, 1, 2>(tx, tw, a, B, st);
}

extern "C" int VSB_API(vsb_vae_time_conv_rgb)(const vsb_bf16* x, const vsb_bf16* w, const vsb_bf16* bias, vsb_bf16* out,
                                              int B, int T, int H, int W, void* stream) {
  if (!x || !w || !bias || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0) return fail(VSB_ERR_INVALID, "vae_time_conv_rgb: bad args");
  const long long P = (long long)H * W;
  time_conv_rgb_kernel<<<grid_for((long long)B * T * P), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)w,
                                                                                         (const bf16*)bias, (bf16*)out, B, T, P);
  return check_launch("vae_time_conv_rgb");
}

extern "C" int VSB_API(vsb_vae_groupnorm_stats)(const vsb_bf16* x, float* stats, float* workspace, int B, long long P, int C,
                                                int G, float eps, void* stream) {
  if (!x || !stats || !workspace || B <= 0 || P <= 0 || C <= 0 || G <= 0) return fail(VSB_ERR_INVALID, "vae_groupnorm_stats: bad args");
  if (!(C == 64 || C == 128 || C == 256 || C == 512) || C % G)
    return fail(VSB_ERR_UNSUPPORTED, "vae_groupnorm_stats: C=%d G=%d (need C in {64,128,256,512}, G | C)", C, G);
  if (!aligned16(x)) return fail(VSB_ERR_UNSUPPORTED, "vae_groupnorm_stats: misaligned x");
  cudaStream_t st = (cudaStream_t)stream;
  gn_partial_kernel<<<dim3(VSB_GN_CHUNKS, B), kGnThreads, 0, st>>>((const bf16*)x, workspace, P, C);
  int rc = check_launch("vae_groupnorm_stats");
  if (rc) return rc;
  gn_finalize_kernel<<<(B * G + 127) / 128, 128, 0, st>>>((const bf16*)x, workspace, stats, P, C, G, B, eps);
  return check_launch("vae_groupnorm_stats");
}

extern "C" int VSB_API(vsb_vae_spatial_norm_silu)(const vsb_bf16* f, const float* stats, const vsb_bf16* gamma,
                                                  const vsb_bf16* beta, const vsb_bf16* zyb, vsb_bf16* out, int B, int T,
                                                  int H, int W, int C, int G, int Tz, int h, int w, int t_off, int T_out,
                                                  void* stream) {
  if (!f || !stats || !gamma || !beta || !zyb || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0 || G <= 0 ||
      Tz <= 0 || h <= 0 || w <= 0 || t_off < 0 || t_off + T > T_out)
    return fail(VSB_ERR_INVALID, "vae_spatial_norm_silu: bad args");
  if (C % 8 || C % G) return fail(VSB_ERR_UNSUPPORTED, "vae_spatial_norm_silu: C=%d G=%d", C, G);
  if (T > 1 && (T & 1) && Tz < 2) return fail(VSB_ERR_INVALID, "vae_spatial_norm_silu: odd T=%d needs Tz >= 2", T);
  if (!aligned16(f) || !aligned16(gamma) || !aligned16(beta) || !aligned16(zyb) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "vae_spatial_norm_silu: misaligned pointer");
  SnArgs a{(const bf16*)f, stats, (const bf16*)gamma, (const bf16*)beta, (const bf16*)zyb, (bf16*)out,
           B, T, H, W, C, G, Tz, h, w, t_off, T_out};
  spatial_norm_silu_kernel<<<grid_for((long long)B * T * H * W * (C / 8)), 256, 0, (cudaStream_t)stream>>>(a);
  return check_launch("vae_spatial_norm_silu");
}

extern "C" int VSB_API(vsb_vae_upsample2x)(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C,
                                           int compress_time, void* stream) {
  if (!x || !out || B <= 0 || T <= 0 || H <= 0 || W <= 0 || C <= 0) return fail(VSB_ERR_INVALID, "vae_upsample2x: bad args");
  if (C % 8 || !aligned16(x) || !aligned16(out)) return fail(VSB_ERR_UNSUPPORTED, "vae_upsample2x: need C %% 8 == 0, 16B-aligned");
  const int T2 = (compress_time && T > 1) ? ((T & 1) ? 1 + 2 * (T - 1) : 2 * T) : T;
  upsample2x_kernel<<<grid_for((long long)B * T2 * 4 * H * W * (C / 8)), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)x, (bf16*)out, B, T, H, W, C, T2, compress_time ? 1 : 0);
  return check_launch("vae_upsample2x");
}
