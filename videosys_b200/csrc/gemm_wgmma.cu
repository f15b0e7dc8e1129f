// vsb200 -- 16-bit TN GEMM on the Hopper warpgroup tensor cores: out[M,N] = act(A[M,K] @ W[N,K]^T + bias), or with the
// residual branch fused into the epilogue: out = resid + [gate *] (A @ W^T + bias).
//
// One CTA per 128 x BN output tile, three warpgroups:
//   warpgroup 0     TMA producer (one thread): A tile 128x64 and W tile BNx64, SWIZZLE_128B, kStages-deep mbarrier ring
//   warpgroups 1-2  consumers: rows 0..63 / 64..127 of the tile, wgmma.m64nBNk16 straight from the swizzled stages into
//                   fp32 registers; each consumer releases a stage once the wgmma that read it has retired
//   epilogue        the consumers: + bias -> [bf16 round -> tanh-GELU | gate + residual] -> 16-bit -> 128B-swizzled
//                   staging tile -> TMA store (64-column chunks)
// Tiles are walked N-fastest so that the 128-row A panel is reused from L2 across its N tiles.  TMA zero-fills K/M/N
// tails on load and clips them on store, so any M, N % 8 == 0, K % 8 == 0 is legal.
#include "vsb_common.cuh"
#include "vsb_host.h"
#include "wgmma.cuh"

namespace vsb {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 384;

template <int BN>
struct GemmCfg {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kStageBytes = (kBM + BN) * kBK * 2;
  static constexpr int kCBytes = kBM * BN * 2;
  static constexpr int kStages = 4;
  // + 1024 for manual alignment, + 256 for barriers
  static constexpr int kSmemBytes = kStages * kStageBytes + kCBytes + 1024 + 256;
};

__device__ __forceinline__ float gelu_tanh_f(float x) {
  // torch GELU(approximate='tanh') = 0.5 x (1 + tanh(u)), u = sqrt(2/pi) (x + 0.044715 x^3), rewritten as
  //   x * sigmoid(2u) = x / (1 + 2^(-2 u log2 e)):
  // 5 ALU + 2 MUFU per element instead of ~14 + 2, and no cancellation in the negative tail.  |difference| to the tanh
  // form <= 5e-7; 99.6 % of all bf16 inputs in [-12, 12] round to the same bf16 output as torch's fp32 evaluation, the
  // rest differ below 1e-6 absolute (x < -3).
  const float kC0 = -2.f * 0.7978845608028654f * 1.4426950408889634f, kC1 = kC0 * 0.044715f;
  const float w = x * fmaf(x * x, kC1, kC0);
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fast_exp2(w) + 1.f));
  return x * r;
}

// exact GELU (F.gelu, approximate='none') as torch's CUDA kernel evaluates it: x * 0.5 * (1 + erf(x / sqrt(2))) in fp32
__device__ __forceinline__ float gelu_erf_f(float x) { return x * 0.5f * (1.f + erff(x * 0.70710678118654752440f)); }

// ACT == 2: out = resid + g, g = bf16(gate * y) (gate_row >= 0, per-frame t/t0 select) or g = y (plain residual add),
// y = bf16(acc + bias): the eager chain of open_sora_transformer_3d.py (Linear, gate multiply, residual add) in the epilogue.
struct EpiArgs {
  const bf16* resid;      // [M, N], may alias the output
  const bf16* mod;        // [2, B, 6, N] or null
  const uint8_t* x_mask;  // [B, T] or null
  int gate_row, B, T, S;
};

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 192)
    wgmma_m64n192k16_ss(d, da, db, scale_d);
  else
    wgmma_m64n128k16_ss(d, da, db, scale_d);
}

template <int BN, int ACT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                  const __grid_constant__ CUtensorMap tm_c, const bf16* __restrict__ bias, int M, int N, int K,
                  const EpiArgs ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  unsigned char* smem_ab = smem;                              // [kStages][A 16 KB | W BN*128 B]
  unsigned char* smem_c = smem + kStages * Cfg::kStageBytes;  // [BN/64][128 rows][128 B] swizzled
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_c + Cfg::kCBytes);  // [kStages]
  uint64_t* empty = full + kStages;                                     // [kStages]

  const int wg = threadIdx.x >> 7;
  const int tiles_n = (N + BN - 1) / BN;
  const int m0 = (blockIdx.x / tiles_n) * kBM, n0 = (blockIdx.x % tiles_n) * BN;
  const int num_kb = (K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_c);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % kStages;
        mbar_wait_quiet(&empty[s], ((kb / kStages) & 1) ^ 1);
        unsigned char* sa = smem_ab + s * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[s], Cfg::kStageBytes);
        tma_load_2d(&tm_a, &full[s], sa, kb * kBK, m0);
        tma_load_2d(&tm_w, &full[s], sa + Cfg::kABytes, kb * kBK, n0);
      }
    }
    return;
  }

  // ===================== consumers: warpgroup c owns rows 64 c .. 64 c + 63 =====================
  const int c = wg - 1;
  const int t = threadIdx.x & 127;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const uint32_t ab0 = smem_u32(smem_ab);
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % kStages;
    mbar_wait_quiet(&full[s], (kb / kStages) & 1);
    const uint32_t sa = ab0 + s * Cfg::kStageBytes + c * (64 * 128);
    const uint32_t sw = ab0 + s * Cfg::kStageBytes + Cfg::kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) wgmma_tile<BN>(acc, wgmma_desc_sw128(sa + 32 * k), wgmma_desc_sw128(sw + 32 * k), 1u);
    wgmma_commit();
    wgmma_wait<1>();  // the group of k-block kb - 1 has retired: its stage can be refilled
    if (kb > 0 && t == 0) mbar_arrive(&empty[(kb - 1) % kStages]);
  }
  wgmma_wait<0>();

  // ===================== epilogue =====================
  const int warp = t >> 5, lane = t & 31;
  const int rl0 = c * 64 + warp * 16 + (lane >> 2);  // tile rows of acc[.. 0/1] and (+8) acc[.. 2/3]
  const bf16* gate_vec[2] = {nullptr, nullptr};
  if (ACT == 2 && ep.gate_row >= 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long grow = (long long)m0 + rl0 + 8 * h;
      if (grow < M) {
        const long long bt = grow / ep.S;
        const int bb = int(bt / ep.T);
        const int sel = (ep.x_mask != nullptr && ep.x_mask[bt] == 0) ? 1 : 0;
        gate_vec[h] = ep.mod + ((size_t)(sel * ep.B + bb) * 6 + ep.gate_row) * N;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = j * 8 + 2 * (lane & 3);  // column inside the tile
    const int gcol = n0 + col;
    float2 b2 = make_float2(0.f, 0.f);
    if (bias != nullptr && gcol < N) b2 = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(bias + gcol)));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rl0 + 8 * h;
      float x0 = acc[4 * j + 2 * h] + b2.x, x1 = acc[4 * j + 2 * h + 1] + b2.y;
      if (ACT == 1) {
        x0 = gelu_tanh_f(rbf(x0));
        x1 = gelu_tanh_f(rbf(x1));
      }
      if (ACT == 3) {
        x0 = gelu_erf_f(rbf(x0));
        x1 = gelu_erf_f(rbf(x1));
      }
      if (ACT == 2) {
        const long long grow = (long long)m0 + row;
        if (grow < M && gcol < N) {
          float y0 = rbf(x0), y1 = rbf(x1);  // the Linear's 16-bit output
          if (gate_vec[h] != nullptr) {
            const float2 g = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(gate_vec[h] + gcol)));
            y0 = rbf(g.x * y0);  // bf16(gate * y)
            y1 = rbf(g.y * y1);
          }
          const float2 xr = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ep.resid + (size_t)grow * N + gcol));
          x0 = xr.x + y0;  // residual add (rounded by the pack below)
          x1 = xr.y + y1;
        }
      }
      // 128B swizzle of the staging chunk: conflict-free (the 8 rows of a store land in 8 different 16-byte units)
      unsigned char* dst = smem_c + (col >> 6) * (kBM * 128) + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(x0, x1);
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 256);
  if (threadIdx.x == 128) {
#pragma unroll 1
    for (int ch = 0; ch < BN / 64; ++ch)
      if (n0 + ch * 64 < N) tma_store_2d(&tm_c, smem_c + ch * (kBM * 128), n0 + ch * 64, m0);
    tma_store_commit();
    tma_store_wait0();
  }
}

template <int BN, int ACT>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tc, const bf16* bias, int M,
                       int N, int K, cudaStream_t st, const EpiArgs& ep) {
  using Cfg = GemmCfg<BN>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "gemm: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  const int tiles = ((M + kBM - 1) / kBM) * ((N + BN - 1) / BN);
  gemm_wgmma_kernel<BN, ACT><<<tiles, kGemmThreads, Cfg::kSmemBytes, st>>>(ta, tw, tc, bias, M, N, K, ep);
  return check_launch("gemm_wgmma");
}

// act: 0 none, 1 tanh-GELU, 2 fused residual (ep->resid != nullptr), 3 erf-GELU
static int gemm_dispatch(const void* A, const void* W, const void* bias, void* out, int M, int N, int K, int act,
                         cudaStream_t st, const EpiArgs& ep) {
  // tile width: 192 divides every STDiT3 / CogVideoX / Latte width (1152, 1920, 2304, 3072, 3456, 4608, 7680); narrow
  // outputs and widths that 128 divides but 192 does not take 128
  const int BN = (N % 192 == 0 || (N > 192 && N % 128 != 0)) ? 192 : 128;
  CUtensorMap ta, tw, tc;
  unsigned long long da[2] = {(unsigned long long)K, (unsigned long long)M};
  unsigned long long sa[1] = {(unsigned long long)K * 2};
  unsigned ba[2] = {kBK, kBM};
  int rc = make_tmap_bf16(&ta, A, 2, da, sa, ba, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  unsigned long long dw[2] = {(unsigned long long)K, (unsigned long long)N};
  unsigned bw[2] = {kBK, (unsigned)BN};
  rc = make_tmap_bf16(&tw, W, 2, dw, sa, bw, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  unsigned long long dc[2] = {(unsigned long long)N, (unsigned long long)M};
  unsigned long long sc[1] = {(unsigned long long)N * 2};
  unsigned bc[2] = {64, kBM};
  rc = make_tmap_bf16(&tc, out, 2, dc, sc, bc, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  const bf16* b = (const bf16*)bias;
#define VSB_GEMM_CASE(bn)                                                     \
  if (BN == bn) {                                                             \
    if (act == 3) return launch_gemm<bn, 3>(ta, tw, tc, b, M, N, K, st, ep);  \
    if (act == 2) return launch_gemm<bn, 2>(ta, tw, tc, b, M, N, K, st, ep);  \
    if (act == 1) return launch_gemm<bn, 1>(ta, tw, tc, b, M, N, K, st, ep);  \
    return launch_gemm<bn, 0>(ta, tw, tc, b, M, N, K, st, ep);                \
  }
  VSB_GEMM_CASE(192)
  VSB_GEMM_CASE(128)
#undef VSB_GEMM_CASE
  return fail(VSB_ERR_UNSUPPORTED, "gemm: no tile config");
}

}  // namespace vsb

using namespace vsb;

extern "C" int VSB_API(vsb_gemm_bias_act)(const vsb_bf16* A, const vsb_bf16* W, const vsb_bf16* bias, vsb_bf16* out, int M,
                                 int N, int K, int act, void* stream) {
  if (!A || !W || !out || M <= 0 || N <= 0 || K <= 0) return fail(VSB_ERR_INVALID, "gemm: bad args");
  if (K % 8 || N % 8 || !aligned16(A) || !aligned16(W) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "gemm: need K %% 8 == 0, N %% 8 == 0, 16B-aligned pointers (M=%d N=%d K=%d)", M, N, K);
  if (act < 0 || act > 2) return fail(VSB_ERR_INVALID, "gemm: act=%d", act);
  // public act 2 (erf-GELU) is epilogue 3: epilogue 2 is the fused residual of vsb_gemm_bias_residual
  return gemm_dispatch(A, W, bias, out, M, N, K, act == 2 ? 3 : act, (cudaStream_t)stream, EpiArgs{nullptr, nullptr, nullptr, -1, 1, 1, 1});
}

// Fused epilogue: out = resid + [gate *] (A @ W^T + bias), see include/vsb200.h.
extern "C" int VSB_API(vsb_gemm_bias_residual)(const vsb_bf16* A, const vsb_bf16* W, const vsb_bf16* bias, const vsb_bf16* resid,
                                      vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int M,
                                      int N, int K, int B, int T, int S, void* stream) {
  if (!A || !W || !resid || !out || M <= 0 || N <= 0 || K <= 0) return fail(VSB_ERR_INVALID, "gemm_residual: bad args");
  if (K % 8 || N % 8 || !aligned16(A) || !aligned16(W) || !aligned16(out) || !aligned16(resid))
    return fail(VSB_ERR_UNSUPPORTED, "gemm_residual: need K %% 8 == 0, N %% 8 == 0, 16B-aligned pointers");
  if (gate_row >= 0) {
    if (!mod || gate_row > 5 || B <= 0 || T <= 0 || S <= 0 || (long long)B * T * S != M || !aligned16(mod))
      return fail(VSB_ERR_INVALID, "gemm_residual: gate needs mod[2,B,6,N] and B*T*S == M");
  }
  EpiArgs ep{(const bf16*)resid, (const bf16*)mod, x_mask, gate_row, B, T, S};
  return gemm_dispatch(A, W, bias, out, M, N, K, 2, (cudaStream_t)stream, ep);
}
