// vsb200 -- HBM-bound kernels of the STDiT3 block: AdaLN modulate, gate+residual, residual add, q/k RMSNorm.
// One pass over the activation each (128-bit coalesced loads/stores, fp32 math, bf16 rounding at the eager
// op boundaries so results track the reference's eager chain bit-for-bit wherever the reduction order allows).
#include <cuda_fp8.h>
#include <string.h>

#include "dsp_common.cuh"
#include "vsb_host.h"

namespace vsb {

union Vec8 {
  uint4 u;
  elem2 h[4];
};

__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- e4m3 quantization of one row held by a warp (the rule of include/vsb200.h, vsb_quant_rows_fp8) ------------------
// amax = max |x| over the row's 16-bit values; amax > 0: q = cvt.rn.satfinite.e4m3(x * s) with s = 448 / amax (both
// fp32, round to nearest even), scale = amax / 448; amax == 0: all-zero codes and scale 1.  |x * s| <= 448 (1 + 2^-23)
// rounds to at most 448, so saturation never acts and the codes are torch's x.to(float8_e4m3fn) of the same fp32 product.
template <int kMaxVec>
__device__ __forceinline__ float row_amax(const Vec8 (&v)[kMaxVec], int nvec, int lane) {
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = e2_to_float2(v[i].h[j]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
  return warp_max(m);
}

template <int kMaxVec>
__device__ __forceinline__ void store_row_e4m3(const Vec8 (&v)[kMaxVec], int nvec, int lane, float amax, uint8_t* qrow,
                                               float* scale) {
  const float s = amax > 0.f ? __fdiv_rn(448.f, amax) : 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      uint32_t w[2] = {0u, 0u};
      if (amax > 0.f) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = e2_to_float2(v[i].h[j]);
          const uint32_t c = __nv_cvt_float2_to_fp8x2(make_float2(f.x * s, f.y * s), __NV_SATFINITE, __NV_E4M3);
          w[j >> 1] |= c << (16 * (j & 1));
        }
      }
      *reinterpret_cast<uint2*>(qrow + vi * 8) = make_uint2(w[0], w[1]);
    }
  }
  if (lane == 0) *scale = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
}

// [rows, C] 16-bit -> e4m3 codes + per-row scales, a warp per row (C <= kMaxVec * 256)
template <int kMaxVec>
__global__ void __launch_bounds__(256) quant_rows_fp8_kernel(const bf16* __restrict__ x, uint8_t* __restrict__ q,
                                                             float* __restrict__ scale, int C, long long rows) {
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    Vec8 v[kMaxVec];
    const bf16* xr = x + (size_t)row * C;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i)
      if (lane + i * 32 < nvec) v[i].u = ld_stream(xr + (lane + i * 32) * 8);
    store_row_e4m3<kMaxVec>(v, nvec, lane, row_amax<kMaxVec>(v, nvec, lane), q + (size_t)row * C, scale + row);
  }
}

// ---------------------------------------------------------------------------------------------------------
// LayerNorm (no affine) + modulate + per-frame select.  One warp per token row; the row lives in registers.
// kMaxVec: max 16-byte vectors per lane (C <= kMaxVec*32*8).
// ---------------------------------------------------------------------------------------------------------
// kDsp: the DSP dimension switch fused into the store path (north_star: the reshard issued by its producer).  The
// modulated row (b, t, sl) of this rank's S-shard is stored straight into the receive window of the rank that owns
// (batch, frame) sequence tf = b*T + t after the switch -- peers.recv[tf / Tl] viewed as [Tl, Sg, C], row
// (tf % Tl, rank*S + sl) -- with 128-bit peer stores over NVLink; rows of padded frames (tf >= B*T) are written as
// zeros, padded columns (rank*S + sl >= Sg) are never sent; the last CTA publishes the epoch (dsp_publish).
struct LnDspArgs {
  DspPeers peers;
  int rank, world, Sg;
  unsigned epoch;
};

// kMinBlocks: resident 256-thread blocks per SM the register budget is sized for; 3 at hidden <= 1280 = 80 registers,
// 24 resident warps per SM (one 2.3 KB row in flight each).
// kFp8: instead of the 16-bit row, store its e4m3 codes to q and its scale to qscale (store_row_e4m3 over the 16-bit
// outputs, so the result is that of vsb_quant_rows_fp8 on the 16-bit output).
template <int kMaxVec, bool kDsp, int kMinBlocks, bool kFp8 = false>
__global__ void __launch_bounds__(256, kMinBlocks) ln_modulate_kernel(const bf16* __restrict__ x, bf16* __restrict__ out,
                                                          const bf16* __restrict__ mod,
                                                          const uint8_t* __restrict__ x_mask, int shift_row,
                                                          int scale_row, int B, int T, int S, int C, float eps,
                                                          long long rows, const bf16* __restrict__ gamma,
                                                          const bf16* __restrict__ beta,
                                                          const __grid_constant__ LnDspArgs dsp,
                                                          uint8_t* __restrict__ q, float* __restrict__ qscale) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  const long long stride = (long long)gridDim.x * warps_per_block;
  long long row = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  Vec8 nxt[kMaxVec];
  auto load_row = [&](long long r) {
    const bf16* xr = x + (size_t)r * C;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) nxt[i].u = ld_stream(xr + vi * 8);
    }
  };
  if (row < rows) load_row(row);
  for (; row < rows; row += stride) {
    Vec8 v[kMaxVec];
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) v[i].u = nxt[i].u;
    if (row + stride < rows) load_row(row + stride);  // keep the next row's 128-bit loads in flight
    const unsigned bt = (unsigned)row / (unsigned)S;  // rows < 2^31 (checked by the launcher)
    const int b = int(bt / (unsigned)T);
    const int sel = (x_mask != nullptr && x_mask[bt] == 0) ? 1 : 0;
    const bf16* shift = mod + ((size_t)(sel * B + b) * 6 + shift_row) * C;
    const bf16* scale = mod + ((size_t)(sel * B + b) * 6 + scale_row) * C;
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = e2_to_float2(v[i].h[j]);
          sum += f.x + f.y;
        }
      }
    }
    const float mean = warp_sum(sum) / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = e2_to_float2(v[i].h[j]);
          float a = f.x - mean, c = f.y - mean;
          sq += a * a + c * c;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
    const elem2 one2 = floats_to_e2(1.f, 1.f);
    bf16* orow = out + (size_t)row * C;
    bool send = true;
    if (kDsp) {
      const unsigned Tl = ((unsigned)(B * T) + dsp.world - 1) / dsp.world;
      const unsigned sl = (unsigned)row - bt * (unsigned)S;
      const unsigned col = (unsigned)dsp.rank * (unsigned)S + sl;
      const unsigned d = bt / Tl, tl = bt - d * Tl;
      send = col < (unsigned)dsp.Sg;
      orow = dsp.peers.recv[d] + ((size_t)tl * dsp.Sg + col) * C;
    }
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        Vec8 sh, sc, o;
        sh.u = __ldg(reinterpret_cast<const uint4*>(shift + vi * 8));
        sc.u = __ldg(reinterpret_cast<const uint4*>(scale + vi * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = e2_to_float2(v[i].h[j]);
          // eager chain on packed bf16 (each op = exact result rounded once, like the eager bf16 kernels):
          // n = bf16(LN(x)); g = bf16(1 + scale); m = bf16(n * g); out = bf16(m + shift)
          float n0 = (f.x - mean) * rstd, n1 = (f.y - mean) * rstd;
          if (gamma != nullptr) {  // nn.LayerNorm with affine: one rounding after weight and bias (CogVideoXLayerNormZero)
            const float2 gw = e2_to_float2(*reinterpret_cast<const elem2*>(gamma + vi * 8 + 2 * j));
            const float2 gb = e2_to_float2(*reinterpret_cast<const elem2*>(beta + vi * 8 + 2 * j));
            n0 = n0 * gw.x + gb.x;
            n1 = n1 * gw.y + gb.y;
          }
          const elem2 n2 = floats_to_e2(n0, n1);
          const elem2 g2 = __hadd2_rn(one2, sc.h[j]);
          o.h[j] = __hadd2_rn(__hmul2_rn(n2, g2), sh.h[j]);
        }
        if (kFp8)
          v[i].u = o.u;
        else if (!kDsp || send)
          st_stream(orow + vi * 8, o.u);
      }
    }
    if (kFp8) store_row_e4m3<kMaxVec>(v, nvec, lane, row_amax<kMaxVec>(v, nvec, lane), q + (size_t)row * C, qscale + row);
  }
  if (kDsp) {
    // zero rows of the padded frames [B*T, Tl*world): the receiver's attention reads them (the reference pads zeros)
    const unsigned Tf = (unsigned)(B * T), Tl = (Tf + dsp.world - 1) / dsp.world;
    const unsigned npad = (Tl * dsp.world - Tf) * (unsigned)S;
    for (unsigned pr = blockIdx.x * warps_per_block + (threadIdx.x >> 5); pr < npad; pr += (unsigned)stride) {
      const unsigned tf = Tf + pr / (unsigned)S, sl = pr % (unsigned)S;
      const unsigned col = (unsigned)dsp.rank * (unsigned)S + sl;
      if (col >= (unsigned)dsp.Sg) continue;
      const unsigned d = tf / Tl, tl = tf - d * Tl;
      bf16* orow = dsp.peers.recv[d] + ((size_t)tl * dsp.Sg + col) * C;
      for (int vi = lane; vi < nvec; vi += 32) st_stream(orow + vi * 8, make_uint4(0, 0, 0, 0));
    }
    dsp_publish(dsp.peers, dsp.rank, dsp.world, dsp.epoch);
  }
}

__global__ void modulation_table_kernel(const bf16* __restrict__ table, const bf16* __restrict__ t,
                                        const bf16* __restrict__ t0, bf16* __restrict__ mod, int B, int C, int rows) {
  // mod[s, b, r, c] = bf16(table[r, c] + (s ? t0 : t)[b, r*C + c])
  const int total = 2 * B * rows * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int c = i % C;
    int r = (i / C) % rows;
    int b = (i / (C * rows)) % B;
    int s = i / (C * rows * B);
    const bf16* src = (s == 1 && t0 != nullptr) ? t0 : t;
    float v = e_to_float(table[r * C + c]) + e_to_float(src[(size_t)b * rows * C + r * C + c]);
    mod[i] = float_to_e(v);
  }
}

// out = x + bf16(gate * y), gate row selected per frame; optional cache of the gated value.
__global__ void __launch_bounds__(256) gate_residual_kernel(const bf16* __restrict__ x, const bf16* __restrict__ y,
                                                            bf16* __restrict__ out, bf16* __restrict__ cache,
                                                            const bf16* __restrict__ mod,
                                                            const uint8_t* __restrict__ x_mask, int gate_row, int B,
                                                            int T, int S, int C, long long nvec_total) {
  const int nvec = C >> 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec_total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / nvec;
    const int vi = int(i - row * nvec);
    const unsigned bt = (unsigned)row / (unsigned)S;  // rows < 2^31 (checked by the launcher)
    const int b = int(bt / (unsigned)T);
    const int sel = (x_mask != nullptr && x_mask[bt] == 0) ? 1 : 0;
    const bf16* gate = mod + ((size_t)(sel * B + b) * 6 + gate_row) * C;
    Vec8 vx, vy, vg, o, g;
    vx.u = ld_stream(x + i * 8);
    vy.u = ld_stream(y + i * 8);
    vg.u = __ldg(reinterpret_cast<const uint4*>(gate + vi * 8));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      g.h[j] = __hmul2_rn(vg.h[j], vy.h[j]);  // bf16(gate * y)
      o.h[j] = __hadd2_rn(vx.h[j], g.h[j]);   // bf16(x + gated)
    }
    if (cache != nullptr) st_stream(cache + i * 8, g.u);
    st_stream(out + i * 8, o.u);
  }
}

__global__ void __launch_bounds__(256) residual_add_kernel(const bf16* __restrict__ x, const bf16* __restrict__ y,
                                                           bf16* __restrict__ out, long long nvec_total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec_total;
       i += (long long)gridDim.x * blockDim.x) {
    Vec8 vx, vy, o;
    vx.u = ld_stream(x + i * 8);
    vy.u = ld_stream(y + i * 8);
#pragma unroll
    for (int j = 0; j < 4; ++j) o.h[j] = __hadd2_rn(vx.h[j], vy.h[j]);
    st_stream(out + i * 8, o.u);
  }
}

// gate + residual with the DSP switch-back fused into the LOAD path: the branch output y lives T-sharded in the
// producers' own windows (the proj GEMM wrote it there); this rank PULLS the rows of its S-shard over NVLink with
// 128-bit peer loads -- row (b, t, sl) from peers.recv[tf / Tl] viewed as [Tl, Sg, C], row (tf % Tl, rank*S + sl),
// tf = b*T + t -- so the reshard costs no kernel, no staging window and no extra HBM pass.  One warp per token row
// (decode once per row), 5 x 16-byte loads of x and of y in flight per lane (NVLink round trip ~2 us).
// Padded columns (rank*S + sl >= Sg) take y = 0, as the reference's zero padding does.
template <int kMaxVec>
__global__ void __launch_bounds__(256) gate_residual_dsp_kernel(const bf16* __restrict__ x, DspPeers peers,
                                                                bf16* __restrict__ out, bf16* __restrict__ cache,
                                                                const bf16* __restrict__ mod,
                                                                const uint8_t* __restrict__ x_mask, int gate_row, int B,
                                                                int T, int S, int C, int rank, int world, int Sg,
                                                                unsigned rows) {
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
  const unsigned Tl = ((unsigned)(B * T) + world - 1) / world;
  for (unsigned row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nwarps) {
    const unsigned bt = row / (unsigned)S, sl = row - bt * (unsigned)S;
    const int b = int(bt / (unsigned)T);
    const int sel = (x_mask != nullptr && x_mask[bt] == 0) ? 1 : 0;
    const bf16* gate = mod + ((size_t)(sel * B + b) * 6 + gate_row) * C;
    const unsigned col = (unsigned)rank * (unsigned)S + sl;
    const unsigned d = bt / Tl, tl = bt - d * Tl;
    const bf16* yrow = col < (unsigned)Sg ? peers.recv[d] + ((size_t)tl * Sg + col) * C : nullptr;
    const bf16* xrow = x + (size_t)row * C;
    Vec8 vx[kMaxVec], vy[kMaxVec];
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      vy[i].u = make_uint4(0, 0, 0, 0);
      if (vi < nvec) {
        vx[i].u = ld_stream(xrow + vi * 8);
        if (yrow != nullptr) vy[i].u = ld_stream(yrow + vi * 8);
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        Vec8 vg, o, g;
        vg.u = __ldg(reinterpret_cast<const uint4*>(gate + vi * 8));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          g.h[j] = __hmul2_rn(vg.h[j], vy[i].h[j]);  // bf16(gate * y)
          o.h[j] = __hadd2_rn(vx[i].h[j], g.h[j]);   // bf16(x + gated)
        }
        if (cache != nullptr) st_stream(cache + (size_t)row * C + vi * 8, g.u);
        st_stream(out + (size_t)row * C + vi * 8, o.u);
      }
    }
  }
}

// In-place RMSNorm of the q and k heads of a packed [rows, 3, H, D] buffer.  A group of D/8 lanes owns one
// (row, q|k, head) vector of D elements (D=72 -> 9 lanes, D=64 -> 8 lanes); groups are packed 3 per warp.
template <int D>
__global__ void __launch_bounds__(256, 4) qk_rmsnorm_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ wq,
                                                         const bf16* __restrict__ wk, long long rows, int H, float eps,
                                                         const float* __restrict__ rope_cos,
                                                         const float* __restrict__ rope_sin, unsigned pos_div,
                                                         unsigned pos_mod) {
  constexpr int LPG = D / 8;     // lanes per group
  constexpr int GPW = 32 / LPG;  // groups per warp (3 for D=72, 4 for D=64)
  constexpr int U = 4;           // independent head vectors in flight per lane
  const int lane = threadIdx.x & 31;
  const int g = lane / LPG, l = lane % LPG;
  const int gs = (g < GPW ? g : 0) * LPG;  // first lane of my group (idle tail lanes shadow group 0)
  // 32-bit index arithmetic (the launcher checks rows * 2 * H < 2^31): the 64-bit divisions of the first version cost
  // more issue slots than the normalisation itself
  const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
  const unsigned ngroups = (unsigned)rows * 2u * H;  // (row, which in {q,k}, head)
  const unsigned H2 = 2u * H;
  const bool do_norm = wq != nullptr;  // NULL weights: RoPE only (attention without q/k norm: Vchitect temporal)
  Vec8 wv[2];
  wv[0].u = do_norm ? __ldg(reinterpret_cast<const uint4*>(wq + l * 8)) : make_uint4(0, 0, 0, 0);
  wv[1].u = do_norm ? __ldg(reinterpret_cast<const uint4*>(wk + l * 8)) : make_uint4(0, 0, 0, 0);
  for (unsigned base = warp * (GPW * U); base < ngroups; base += nwarps * (GPW * U)) {
    Vec8 v[U];
    bf16* p[U];
    int which[U];
    unsigned pos[U];
    bool active[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned gi = base + u * GPW + g;
      pos[u] = 0u;
      active[u] = (g < GPW) && (gi < ngroups);
      p[u] = nullptr;
      which[u] = 0;
      if (active[u]) {
        const unsigned row = gi / H2;
        const int rem = int(gi - row * H2);
        which[u] = rem >= H ? 1 : 0;
        const int h = rem - which[u] * H;
        p[u] = qkv + ((size_t)row * 3 + which[u]) * H * D + (size_t)h * D + l * 8;
        v[u].u = *reinterpret_cast<const uint4*>(p[u]);
        pos[u] = rope_cos != nullptr ? (row / pos_div) % pos_mod : 0u;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float ss = 0.f;
      if (active[u]) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = e2_to_float2(v[u].h[j]);
          ss += f.x * f.x + f.y * f.y;
        }
      }
      float tot = 0.f;  // reduce within the group; every lane takes part in the shuffles
#pragma unroll
      for (int i = 0; i < LPG; ++i) tot += __shfl_sync(0xffffffffu, ss, gs + i);
      if (active[u]) {
        const float r = rsqrtf(tot / (float)D + eps);
        Vec8 o;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 f = e2_to_float2(v[u].h[j]);
          // eager: h = bf16(x * rstd); out = bf16(w * h)
          o.h[j] = do_norm ? __hmul2_rn(wv[which[u]].h[j], floats_to_e2(f.x * r, f.y * r)) : v[u].h[j];
          if (rope_cos != nullptr) {
            // rotate_queries_or_keys (attentions.py:76-78): t*cos + rotate_half(t)*sin in fp32 on interleaved pairs
            // (2i, 2i+1), rot = (-x2, x1), cast back to bf16; position = the token's frame index
            const float2 y = e2_to_float2(o.h[j]);
            const int d = l * 8 + 2 * j;
            const float2 cs = *reinterpret_cast<const float2*>(rope_cos + (size_t)pos[u] * D + d);
            const float2 sn = *reinterpret_cast<const float2*>(rope_sin + (size_t)pos[u] * D + d);
            const float o0 = __fadd_rn(__fmul_rn(y.x, cs.x), __fmul_rn(-y.y, sn.x));
            const float o1 = __fadd_rn(__fmul_rn(y.y, cs.y), __fmul_rn(y.x, sn.y));
            o.h[j] = floats_to_e2(o0, o1);
          }
        }
        *reinterpret_cast<uint4*>(p[u]) = o.u;
      }
    }
  }
}

// Per-head LayerNorm(D, eps, affine) of q and k inside a packed [rows, 3, H, D] buffer (CogVideoX: diffusers Attention
// with qk_norm="layer_norm", cogvideox_transformer_3d.py:241-242).  Same lane grouping as qk_rmsnorm_kernel.
template <int D>
__global__ void __launch_bounds__(256) qk_layernorm_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ wq,
                                                           const bf16* __restrict__ bq, const bf16* __restrict__ wk,
                                                           const bf16* __restrict__ bk, long long rows, int H,
                                                           float eps) {
  constexpr int LPG = D / 8;
  constexpr int GPW = 32 / LPG;
  const int lane = threadIdx.x & 31;
  const int g = lane / LPG, l = lane % LPG;
  const int gs = (g < GPW ? g : 0) * LPG;
  const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long ngroups = rows * 2 * H;
  Vec8 wv[2], bv[2];
  wv[0].u = __ldg(reinterpret_cast<const uint4*>(wq + l * 8));
  wv[1].u = __ldg(reinterpret_cast<const uint4*>(wk + l * 8));
  bv[0].u = __ldg(reinterpret_cast<const uint4*>(bq + l * 8));
  bv[1].u = __ldg(reinterpret_cast<const uint4*>(bk + l * 8));
  for (long long base = warp * GPW; base < ngroups; base += nwarps * GPW) {
    const long long gi = base + g;
    const bool active = (g < GPW) && (gi < ngroups);
    Vec8 v;
    bf16* p = nullptr;
    int which = 0;
    float s1 = 0.f;
    if (active) {
      const long long row = gi / (2 * H);
      const int rem = int(gi - row * 2 * H);
      which = rem / H;
      const int h = rem - which * H;
      p = qkv + ((size_t)row * 3 + which) * H * D + (size_t)h * D + l * 8;
      v.u = *reinterpret_cast<const uint4*>(p);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = e2_to_float2(v.h[j]);
        s1 += f.x + f.y;
      }
    }
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < LPG; ++i) tot += __shfl_sync(0xffffffffu, s1, gs + i);
    const float mean = tot / (float)D;
    float s2 = 0.f;
    if (active) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = e2_to_float2(v.h[j]);
        s2 += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < LPG; ++i) var += __shfl_sync(0xffffffffu, s2, gs + i);
    if (active) {
      const float r = rsqrtf(var / (float)D + eps);
      Vec8 o;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = e2_to_float2(v.h[j]);
        float2 w = e2_to_float2(wv[which].h[j]), b = e2_to_float2(bv[which].h[j]);
        o.h[j] = floats_to_e2((f.x - mean) * r * w.x + b.x, (f.y - mean) * r * w.y + b.y);
      }
      *reinterpret_cast<uint4*>(p) = o.u;
    }
  }
}

// Half-rotation RoPE ("rotate_half" inside blocks of 2*half channels of every head) on the q and k thirds of a packed
// [rows, 3, H, D] buffer, in place: Open-Sora-Plan's RoPE1D / RoPE2D / RoPE3D
// (open_sora_plan_v110_transformer_3d.py:136-252, open_sora_plan_v120_transformer_3d.py:63-118):
//     out[d] = x[d] * cos[p, d] + rotate_half(x)[d] * sin[p, d],   evaluated in the 16-bit dtype op by op.
// One thread owns two adjacent rotation pairs (d, d + half), (d + 1, d + 1 + half): it reads and writes the same four
// elements, so the in-place update needs no ordering between threads.  The tables are fp32 copies of the 16-bit cos / sin
// the reference computes (the sign of rotate_half folded into sin), so every product is exact in fp32 before its rounding.
__global__ void __launch_bounds__(256) qk_rope_halves_kernel(bf16* __restrict__ qkv, unsigned items, unsigned per_vec,
                                                             int H, int D, int half, const float* __restrict__ cosv,
                                                             const float* __restrict__ sinv, unsigned pos_div,
                                                             unsigned pos_mod) {
  const unsigned per_head = (unsigned)D / 4u;      // thread slots per head (4 elements each)
  const unsigned per_blk = (unsigned)half / 2u;    // thread slots per rotation block
  for (unsigned it = blockIdx.x * blockDim.x + threadIdx.x; it < items; it += gridDim.x * blockDim.x) {
    const unsigned rw = it / per_vec, j = it - rw * per_vec;  // (row, q|k), slot within the H*D vector
    const unsigned row = rw >> 1, which = rw & 1u;
    const unsigned h = j / per_head, q = j - h * per_head;
    const unsigned b = q / per_blk, o2 = q - b * per_blk;
    const unsigned d1 = b * 2u * (unsigned)half + 2u * o2, d2 = d1 + (unsigned)half;
    bf16* base = qkv + ((size_t)row * 3 + which) * H * D + (size_t)h * D;
    const unsigned p = (row / pos_div) % pos_mod;
    const float* ct = cosv + (size_t)p * D;
    const float* st = sinv + (size_t)p * D;
    const float2 x1 = e2_to_float2(*reinterpret_cast<const elem2*>(base + d1));
    const float2 x2 = e2_to_float2(*reinterpret_cast<const elem2*>(base + d2));
    const float2 c1 = *reinterpret_cast<const float2*>(ct + d1), c2 = *reinterpret_cast<const float2*>(ct + d2);
    const float2 s1 = *reinterpret_cast<const float2*>(st + d1), s2 = *reinterpret_cast<const float2*>(st + d2);
    // first half: x1 * cos + (-x2) * sin (the table holds -sin there); second half: x2 * cos + x1 * sin
    const float2 a1 = e2_to_float2(floats_to_e2(__fmul_rn(x1.x, c1.x), __fmul_rn(x1.y, c1.y)));
    const float2 r1 = e2_to_float2(floats_to_e2(__fmul_rn(x2.x, s1.x), __fmul_rn(x2.y, s1.y)));
    const float2 a2 = e2_to_float2(floats_to_e2(__fmul_rn(x2.x, c2.x), __fmul_rn(x2.y, c2.y)));
    const float2 r2 = e2_to_float2(floats_to_e2(__fmul_rn(x1.x, s2.x), __fmul_rn(x1.y, s2.y)));
    *reinterpret_cast<elem2*>(base + d1) = floats_to_e2(__fadd_rn(a1.x, r1.x), __fadd_rn(a1.y, r1.y));
    *reinterpret_cast<elem2*>(base + d2) = floats_to_e2(__fadd_rn(a2.x, r2.x), __fadd_rn(a2.y, r2.y));
  }
}

static int grid_for(long long work_items, int per_block) {
  long long blocks = (work_items + per_block - 1) / per_block;
  long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace vsb

using namespace vsb;

// q != null: the e4m3 output (codes q, per-row scales qscale) instead of out; never with dsp or gamma / beta
static int ln_modulate_launch(const vsb_bf16* x, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask,
                              const vsb_bf16* gamma, const vsb_bf16* beta, int shift_row, int scale_row, int B, int T,
                              int S, int C, float eps, const LnDspArgs* dsp, void* stream, uint8_t* q = nullptr,
                              float* qscale = nullptr) {
  if ((gamma == nullptr) != (beta == nullptr)) return fail(VSB_ERR_INVALID, "ln_modulate: gamma and beta go together");
  if (!x || (!out && !dsp && !q) || !mod || B <= 0 || T <= 0 || S <= 0 || C <= 0) return fail(VSB_ERR_INVALID, "ln_modulate: bad args");
  if (q != nullptr && (qscale == nullptr || dsp || gamma)) return fail(VSB_ERR_INVALID, "ln_modulate_fp8: bad args");
  if (C % 8 || C > 3072 || (dsp && C > 2048) || !aligned16(x) || !aligned16(out) || !aligned16(mod) || !aligned16(q))
    return fail(VSB_ERR_UNSUPPORTED, "ln_modulate: need C %% 8 == 0, C <= 3072 (2048 with the fused reshard), 16B-aligned pointers (C=%d)", C);
  if (shift_row < 0 || shift_row > 5 || scale_row < 0 || scale_row > 5) return fail(VSB_ERR_INVALID, "ln_modulate: row");
  long long rows = (long long)B * T * S;
  if (rows >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "ln_modulate: %lld rows", rows);
  int grid = grid_for(rows, 8);
  cudaStream_t st = (cudaStream_t)stream;
  LnDspArgs none;
  memset(&none, 0, sizeof(none));
#define VSB_LN_LAUNCH(MV, DSP, OCC, ARGS, ...)                                                                         \
  ln_modulate_kernel<MV, DSP, OCC, ##__VA_ARGS__><<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)out, (const bf16*)mod,   \
                                                                         x_mask, shift_row, scale_row, B, T, S, C, eps, \
                                                                         rows, (const bf16*)gamma, (const bf16*)beta,   \
                                                                         ARGS, q, qscale)
  if (q != nullptr) {
    if (C <= 1280) VSB_LN_LAUNCH(5, false, 3, none, true);
    else if (C <= 2048) VSB_LN_LAUNCH(8, false, 2, none, true);
    else if (C <= 2304) VSB_LN_LAUNCH(9, false, 2, none, true);
    else VSB_LN_LAUNCH(12, false, 1, none, true);
  } else if (dsp) {
    if (C <= 1280) VSB_LN_LAUNCH(5, true, 3, *dsp); else VSB_LN_LAUNCH(8, true, 2, *dsp);
  } else if (C <= 1280) {
    VSB_LN_LAUNCH(5, false, 3, none);
  } else if (C <= 2048) {
    VSB_LN_LAUNCH(8, false, 2, none);
  } else if (C <= 2304) {  // hidden 2304 (Open-Sora-Plan v1.2.0: 24 heads x 96)
    VSB_LN_LAUNCH(9, false, 2, none);
  } else {  // hidden 3072 (CogVideoX-5b: 48 heads x 64): the row still lives in registers, one block per SM slot
    VSB_LN_LAUNCH(12, false, 1, none);
  }
#undef VSB_LN_LAUNCH
  return check_launch("ln_modulate");
}

extern "C" int VSB_API(vsb_ln_modulate_affine)(const vsb_bf16* x, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask,
                                      const vsb_bf16* gamma, const vsb_bf16* beta, int shift_row, int scale_row, int B,
                                      int T, int S, int C, float eps, void* stream) {
  return ln_modulate_launch(x, out, mod, x_mask, gamma, beta, shift_row, scale_row, B, T, S, C, eps, nullptr, stream);
}

#ifndef VSB_HALF  // the DSP-fused entries exist in the bf16 build only (sequence parallelism is an OpenSora / bf16 path)
namespace vsb {
int dsp_fill_peers(DspPeers* peers, void* const* host_peer_recv, void* const* host_peer_flags, int world, const char* what);
}

extern "C" int vsb_ln_modulate_dsp(const vsb_bf16* x, const vsb_bf16* mod, const uint8_t* x_mask, int shift_row,
                                   int scale_row, int B, int T, int Sl, int C, float eps, void* const* host_peer_recv,
                                   void* const* host_peer_flags, int rank, int world, int Sg, unsigned epoch,
                                   void* stream) {
  if (!host_peer_recv || !host_peer_flags || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || Sg <= 0)
    return fail(VSB_ERR_INVALID, "ln_modulate_dsp: bad args");
  if ((long long)Sl * world < Sg) return fail(VSB_ERR_INVALID, "ln_modulate_dsp: Sl * world < Sg");
  LnDspArgs a;
  memset(&a, 0, sizeof(a));
  int rc = dsp_fill_peers(&a.peers, host_peer_recv, host_peer_flags, world, "ln_modulate_dsp");
  if (rc) return rc;
  a.rank = rank;
  a.world = world;
  a.Sg = Sg;
  a.epoch = epoch;
  return ln_modulate_launch(x, nullptr, mod, x_mask, nullptr, nullptr, shift_row, scale_row, B, T, Sl, C, eps, &a, stream);
}

extern "C" int vsb_gate_residual_dsp(const vsb_bf16* x, void* const* host_peer_y, vsb_bf16* out, vsb_bf16* cache_out,
                                     const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int B, int T, int Sl, int C,
                                     int rank, int world, int Sg, void* stream) {
  if (!x || !host_peer_y || !out || !mod || B <= 0 || T <= 0 || Sl <= 0 || C <= 0 || world < 1 || world > kMaxWorld ||
      rank < 0 || rank >= world || Sg <= 0)
    return fail(VSB_ERR_INVALID, "gate_residual_dsp: bad args");
  if (C % 8 || C > 2048 || !aligned16(x) || !aligned16(out) || !aligned16(mod) || (cache_out && !aligned16(cache_out)))
    return fail(VSB_ERR_UNSUPPORTED, "gate_residual_dsp: need C %% 8 == 0, C <= 2048 and 16B-aligned pointers");
  long long rows = (long long)B * T * Sl;
  if (rows >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "gate_residual_dsp: too many rows");
  DspPeers peers;
  int rc = dsp_fill_peers(&peers, host_peer_y, nullptr, world, "gate_residual_dsp");
  if (rc) return rc;
  const int grid = grid_for(rows, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (C <= 1280)
    gate_residual_dsp_kernel<5><<<grid, 256, 0, st>>>((const bf16*)x, peers, (bf16*)out, (bf16*)cache_out,
                                                       (const bf16*)mod, x_mask, gate_row, B, T, Sl, C, rank, world, Sg,
                                                       (unsigned)rows);
  else
    gate_residual_dsp_kernel<8><<<grid, 256, 0, st>>>((const bf16*)x, peers, (bf16*)out, (bf16*)cache_out,
                                                       (const bf16*)mod, x_mask, gate_row, B, T, Sl, C, rank, world, Sg,
                                                       (unsigned)rows);
  return check_launch("gate_residual_dsp");
}

#endif  // !VSB_HALF

extern "C" int VSB_API(vsb_ln_modulate)(const vsb_bf16* x, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask,
                               int shift_row, int scale_row, int B, int T, int S, int C, float eps, void* stream) {
  return VSB_API(vsb_ln_modulate_affine)(x, out, mod, x_mask, nullptr, nullptr, shift_row, scale_row, B, T, S, C, eps, stream);
}

extern "C" int VSB_API(vsb_ln_modulate_fp8)(const vsb_bf16* x, uint8_t* q, float* scale, const vsb_bf16* mod,
                                            const uint8_t* x_mask, int shift_row, int scale_row, int B, int T, int S, int C,
                                            float eps, void* stream) {
  if (!q) return fail(VSB_ERR_INVALID, "ln_modulate_fp8: bad args");
  return ln_modulate_launch(x, nullptr, mod, x_mask, nullptr, nullptr, shift_row, scale_row, B, T, S, C, eps, nullptr, stream,
                            q, scale);
}

extern "C" int VSB_API(vsb_quant_rows_fp8)(const vsb_bf16* x, uint8_t* q, float* scale, int M, int K, void* stream) {
  if (!x || !q || !scale || M <= 0 || K <= 0) return fail(VSB_ERR_INVALID, "quant_rows_fp8: bad args");
  if (K % 8 || K > 4608 || !aligned16(x) || !aligned16(q))
    return fail(VSB_ERR_UNSUPPORTED, "quant_rows_fp8: need K %% 8 == 0, K <= 4608, 16B-aligned pointers (K=%d)", K);
  const int grid = grid_for(M, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (K <= 1280)
    quant_rows_fp8_kernel<5><<<grid, 256, 0, st>>>((const bf16*)x, q, scale, K, M);
  else
    quant_rows_fp8_kernel<18><<<grid, 256, 0, st>>>((const bf16*)x, q, scale, K, M);
  return check_launch("quant_rows_fp8");
}

extern "C" int VSB_API(vsb_modulation_table)(const vsb_bf16* table, const vsb_bf16* t, const vsb_bf16* t0, vsb_bf16* mod,
                                    int B, int C, int rows, void* stream) {
  if (!table || !t || !mod || B <= 0 || C <= 0 || rows <= 0) return fail(VSB_ERR_INVALID, "modulation_table: bad args");
  int total = 2 * B * rows * C;
  modulation_table_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>((const bf16*)table, (const bf16*)t,
                                                                                  (const bf16*)t0, (bf16*)mod, B, C,
                                                                                  rows);
  return check_launch("modulation_table");
}

extern "C" int VSB_API(vsb_gate_residual)(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, vsb_bf16* cache_out,
                                 const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int B, int T, int S, int C,
                                 void* stream) {
  if (!x || !y || !out || !mod || B <= 0 || T <= 0 || S <= 0 || C <= 0)
    return fail(VSB_ERR_INVALID, "gate_residual: bad args");
  if (C % 8 || !aligned16(x) || !aligned16(y) || !aligned16(out) || !aligned16(mod) || (cache_out && !aligned16(cache_out)))
    return fail(VSB_ERR_UNSUPPORTED, "gate_residual: need C %% 8 == 0 and 16B-aligned pointers");
  if ((long long)B * T * S >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "gate_residual: too many rows");
  long long nvec = (long long)B * T * S * (C / 8);
  gate_residual_kernel<<<grid_for(nvec, 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)x, (const bf16*)y, (bf16*)out, (bf16*)cache_out, (const bf16*)mod, x_mask, gate_row, B, T, S, C,
      nvec);
  return check_launch("gate_residual");
}

extern "C" int VSB_API(vsb_residual_add)(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, size_t n, void* stream) {
  if (!x || !y || !out || n == 0) return fail(VSB_ERR_INVALID, "residual_add: bad args");
  if (n % 8 || !aligned16(x) || !aligned16(y) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "residual_add: need n %% 8 == 0 and 16B-aligned pointers");
  long long nvec = (long long)(n / 8);
  residual_add_kernel<<<grid_for(nvec, 256 * 4), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)y,
                                                                                  (bf16*)out, nvec);
  return check_launch("residual_add");
}

extern "C" int VSB_API(vsb_qk_rmsnorm)(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* wk, size_t rows, int H, int D,
                              float eps, void* stream) {
  return VSB_API(vsb_qk_rmsnorm_rope)(qkv, wq, wk, rows, H, D, eps, nullptr, nullptr, 1, 1, stream);
}

extern "C" int VSB_API(vsb_qk_rmsnorm_rope)(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* wk, size_t rows, int H, int D,
                                   float eps, const float* rope_cos, const float* rope_sin, int pos_div, int pos_mod,
                                   void* stream) {
  if (!qkv || rows == 0 || H <= 0 || ((wq == nullptr) != (wk == nullptr)))
    return fail(VSB_ERR_INVALID, "qk_rmsnorm: bad args");
  if ((rope_cos == nullptr) != (rope_sin == nullptr) || pos_div <= 0 || pos_mod <= 0)
    return fail(VSB_ERR_INVALID, "qk_rmsnorm: rope tables / position map");
  if (wq == nullptr && rope_cos == nullptr) return fail(VSB_ERR_INVALID, "qk_rmsnorm: neither norm weights nor rope tables");
  if (!aligned16(qkv) || !aligned16(wq) || !aligned16(wk)) return fail(VSB_ERR_UNSUPPORTED, "qk_rmsnorm: alignment");
  long long groups = (long long)rows * 2 * H;
  if (groups >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "qk_rmsnorm: %lld head vectors", groups);
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 72)
    qk_rmsnorm_kernel<72><<<grid_for(groups, 8 * 3 * 4), 256, 0, st>>>((bf16*)qkv, (const bf16*)wq, (const bf16*)wk,
                                                                     (long long)rows, H, eps, rope_cos, rope_sin,
                                                                     (unsigned)pos_div, (unsigned)pos_mod);
  else if (D == 64)
    qk_rmsnorm_kernel<64><<<grid_for(groups, 8 * 4 * 4), 256, 0, st>>>((bf16*)qkv, (const bf16*)wq, (const bf16*)wk,
                                                                     (long long)rows, H, eps, rope_cos, rope_sin,
                                                                     (unsigned)pos_div, (unsigned)pos_mod);
  else
    return fail(VSB_ERR_UNSUPPORTED, "qk_rmsnorm: head_dim %d (72 or 64 only)", D);
  return check_launch("qk_rmsnorm");
}

extern "C" int VSB_API(vsb_qk_rope_halves)(vsb_bf16* qkv, size_t rows, int H, int D, int half, const float* rope_cos,
                                           const float* rope_sin_signed, int pos_div, int pos_mod, void* stream) {
  if (!qkv || !rope_cos || !rope_sin_signed || rows == 0 || H <= 0 || D <= 0 || pos_div <= 0 || pos_mod <= 0)
    return fail(VSB_ERR_INVALID, "qk_rope_halves: bad args");
  if (half <= 0 || (half & 1) || D % (2 * half) != 0)
    return fail(VSB_ERR_UNSUPPORTED, "qk_rope_halves: head_dim %d is not a whole number of 2 x %d rotation blocks (half even)", D, half);
  if (!aligned16(qkv) || (reinterpret_cast<uintptr_t>(rope_cos) & 7) || (reinterpret_cast<uintptr_t>(rope_sin_signed) & 7))
    return fail(VSB_ERR_UNSUPPORTED, "qk_rope_halves: alignment");
  const long long per_vec = (long long)H * D / 4;
  const long long items = (long long)rows * 2 * per_vec;
  if (items >= (1ll << 32) - (1ll << 24)) return fail(VSB_ERR_UNSUPPORTED, "qk_rope_halves: %lld thread slots", items);
  qk_rope_halves_kernel<<<grid_for(items, 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      (bf16*)qkv, (unsigned)items, (unsigned)per_vec, H, D, half, rope_cos, rope_sin_signed, (unsigned)pos_div,
      (unsigned)pos_mod);
  return check_launch("qk_rope_halves");
}

extern "C" int VSB_API(vsb_qk_layernorm)(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* bq, const vsb_bf16* wk,
                                const vsb_bf16* bk, size_t rows, int H, int D, float eps, void* stream) {
  if (!qkv || !wq || !bq || !wk || !bk || rows == 0 || H <= 0) return fail(VSB_ERR_INVALID, "qk_layernorm: bad args");
  if (!aligned16(qkv) || !aligned16(wq) || !aligned16(bq) || !aligned16(wk) || !aligned16(bk))
    return fail(VSB_ERR_UNSUPPORTED, "qk_layernorm: alignment");
  long long groups = (long long)rows * 2 * H;
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 64)
    qk_layernorm_kernel<64><<<grid_for(groups, 8 * 4), 256, 0, st>>>((bf16*)qkv, (const bf16*)wq, (const bf16*)bq,
                                                                       (const bf16*)wk, (const bf16*)bk, (long long)rows,
                                                                       H, eps);
  else if (D == 72)
    qk_layernorm_kernel<72><<<grid_for(groups, 8 * 3), 256, 0, st>>>((bf16*)qkv, (const bf16*)wq, (const bf16*)bq,
                                                                       (const bf16*)wk, (const bf16*)bk, (long long)rows,
                                                                       H, eps);
  else
    return fail(VSB_ERR_UNSUPPORTED, "qk_layernorm: head_dim %d (64 or 72 only)", D);
  return check_launch("qk_layernorm");
}
