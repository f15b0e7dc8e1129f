// vsb200 -- 16-bit TN GEMM on the Hopper warpgroup tensor cores: out[M,N] = act(A[M,K] @ W[N,K]^T + bias), or with the
// residual branch fused into the epilogue: out = resid + [gate *] (A @ W^T + bias).
//
// Three kernels, chosen in gemm_route from the epilogue, K and the tile count.  Large-M GEMMs (except the residual
// epilogue at short K) run gemm_wide_kernel (persistent, 256 x 128 tiles, below), whose K loop moves the fewest bytes
// per FLOP and whose epilogue runs under the next tile's K loop.  Of the rest, the gate + residual epilogue, and a GELU epilogue at K <= 1536, run the persistent ping-pong kernel, which
// hides the epilogue under the tensor cores; a bias-only GEMM, and a GELU GEMM at longer K, run gemm_tile_kernel (one
// CTA per 128 x 192 tile, below), whose K loop is faster.
//
// Persistent ping-pong kernel: min(tiles, SMs) CTAs, each walking the 128 x 128 output tiles blockIdx.x, + gridDim.x, ...
// N-fastest (so the 128-row A panel is reused from L2 across its N tiles), two warpgroups and one warp:
//   warp 8          TMA producer (one thread): A tile 128x64 and W tile 128x64 per k-block,
//                   SWIZZLE_128B, through a kStages-deep mbarrier ring whose position carries over from tile to tile, so
//                   the loads of the next tile are in flight while the current one is still on the tensor cores; for the
//                   fused residual also the tile's resid block, straight into the staging buffer of the consumer that owns it
//   warpgroups 0-1  consumers, taking alternate tiles of the CTA: wgmma.m64n128k16 x 2 (rows 0..63
//                   and 64..127) from the swizzled stages into 128 fp32 registers per thread.  The two mainloops take turns
//                   on the tensor cores (named barriers 1 / 2), so one consumer's epilogue -- + bias -> [bf16 round ->
//                   tanh-GELU | gate + residual] -> 16-bit -> its own 128B-swizzled staging tile -> TMA store -- runs under
//                   the other consumer's mainloop, and so does the refill of the ring between tiles
// A consumer releases a stage once the wgmma that read it has retired, and its staging tile once the TMA store has read
// it (cp.async.bulk.wait_group.read).  TMA zero-fills K/M/N tails on load and clips them on store, so any M,
// N % 8 == 0, K % 8 == 0 is legal.
//
// e4m3 operands (vsb_gemm_fp8_*): gemm_wide_kernel on WideFp8Cfg, 128 x 128 tiles, k-blocks of 128 elements -- the same
// 128-byte swizzled rows, so the producer, the stage ring and the descriptors are those of the 16-bit kernels -- with
// wgmma.m64n128k32.e4m3 and each k-block's products promoted into fp32 registers (consumer_k_loop), and y =
// bf16(acc * sa[row] * sw[col] + bias) at the start of the shared epilogue.  K % 16 == 0 (16-byte rows of codes).
#include "vsb_common.cuh"
#include "vsb_host.h"
#include "wgmma.cuh"

namespace vsb {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 64;
constexpr int kABox = kBM * kBK * 2;       // one 128-row A box of a k-block
constexpr int kPersistentGeluMaxK = 1536;  // longest K at which a GELU epilogue runs on the persistent kernel
constexpr long long kWideMinTiles = 2048;  // fewest 256 x 128 tiles at which gemm_route picks gemm_wide_kernel

// Each kernel's tile, launch and shared memory.  kStageBytes: the A boxes then the W box of one k-block.
// kBK: elements of K per k-block (one 128-byte swizzle row); kFp8: e4m3 operands.
struct GemmCfg {  // gemm_wgmma_kernel
  static constexpr int kTileM = kBM, kTileN = kBN, kBK = vsb::kBK;
  static constexpr bool kPersistent = true, kFp8 = false;
  // two consumer warpgroups + one producer warp; ptxas allots 168 registers per thread: 128 accumulators + the epilogue
  static constexpr int kThreads = 288;
  static constexpr int kABytes = kABox;
  static constexpr int kStageBytes = (kBM + kBN) * kBK * 2;
  static constexpr int kCBytes = kBM * kBN * 2;  // one staging tile: [kBN/64][128 rows][128 B] swizzled
  static constexpr int kStages = 5;
  // 5 x 32 KB ring + 2 x 32 KB staging, + 1024 for manual alignment, + 256 for barriers: 230 656 B of the 227 KB
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kCBytes + 1024 + 256;
};

template <int BN>
struct TileCfg {  // gemm_tile_kernel<BN, .>
  static constexpr int kTileM = kBM, kTileN = BN, kBK = vsb::kBK;
  static constexpr bool kPersistent = false, kFp8 = false;
  static constexpr int kThreads = 384;
  static constexpr int kABytes = kABox;
  static constexpr int kStageBytes = (kBM + BN) * kBK * 2;
  static constexpr int kCBytes = kBM * BN * 2;
  static constexpr int kStages = 4;
  // + 1024 for manual alignment, + 256 for barriers
  static constexpr int kSmemBytes = kStages * kStageBytes + kCBytes + 1024 + 256;
};

constexpr int kWideEpiThreads = 96;
// gemm_wide_kernel.  16-bit operands: 256 x 128 tiles, each consumer warpgroup 128 rows.  e4m3 operands (FP8 = true):
// 128 x 128 tiles, each consumer 64 rows -- the fp32 promotion fragment doubles the accumulators, and 2 x 64 of them
// per thread fit the 168-register budget where 2 x 128 would not; a k-block is 128 elements, the same 128-byte rows.
template <bool FP8>
struct WideCfgT {
  static constexpr int kTileM = FP8 ? kBM : 2 * kBM, kTileN = kBN, kBK = FP8 ? 128 : vsb::kBK;
  static constexpr bool kPersistent = true, kFp8 = FP8;
  static constexpr int kThreads = 384;  // two consumer warpgroups, three epilogue warps, one producer warp
  static constexpr int kCBlocks = kTileM / kBM;  // 128-row TMA boxes of A, and of the staging tile
  static constexpr int kABytes = kCBlocks * kABox;
  static constexpr int kStageBytes = kABytes + kBN * 128;
  static constexpr int kCBytes = kBM * kBN * 2;  // one 128-row block of the staging tile
  static constexpr int kStages = FP8 ? 6 : 3;
  // 16-bit: 3 x 48 KB ring + 2 x 32 KB staging; e4m3: 6 x 32 KB ring + 32 KB staging; + 1024 for manual alignment, + 256
  // for barriers: 214 272 / 230 656 B of the 227 KB
  static constexpr int kSmemBytes = kStages * kStageBytes + kCBlocks * kCBytes + 1024 + 256;
};
using WideCfg = WideCfgT<false>;
using WideFp8Cfg = WideCfgT<true>;

// ---- the epilogue's element functions: every kernel applies them to y = bf16(acc + bias), two adjacent columns -------
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

// ACT 1: tanh-GELU(y), ACT 3: erf-GELU(y)
template <int ACT>
__device__ __forceinline__ float2 gelu2(float2 y) {
  return ACT == 1 ? make_float2(gelu_tanh_f(y.x), gelu_tanh_f(y.y)) : make_float2(gelu_erf_f(y.x), gelu_erf_f(y.y));
}

// ACT == 2: out = resid + g, g = bf16(gate * y) (gate_row >= 0, per-frame t/t0 select) or g = y (plain residual add),
// y = bf16(acc + bias): the eager chain of open_sora_transformer_3d.py (Linear, gate multiply, residual add) in the epilogue.
struct EpiArgs {
  const bf16* resid;      // [M, N], may alias the output; read by TMA through its own tensor map
  const bf16* mod;        // [2, B, 6, N] or null
  const uint8_t* x_mask;  // [B, T] or null
  int gate_row, B, T, S;
  const float* sa;        // e4m3 operands: per-row scale of A [M] and per-output-channel scale of W [N]
  const float* sw;
};

// element offset in mod of output row `row`'s gate vector: row gate_row of its sample's t (or, where x_mask marks the
// row's frame 0, t0) modulation
__device__ __forceinline__ int gate_offset(const EpiArgs& ep, int row, int N) {
  const int bt = row / ep.S;
  const int bb = bt / ep.T;
  const int sel = (ep.x_mask != nullptr && ep.x_mask[bt] == 0) ? 1 : 0;
  return ((sel * ep.B + bb) * 6 + ep.gate_row) * N;
}

// resid + [bf16(gate * y)], resid and gate packed; the caller's pack rounds the residual add
__device__ __forceinline__ float2 residual_add2(float2 y, uint32_t resid, bool gated, uint32_t gate) {
  if (gated) {
    const float2 g = unpack_bf16x2(gate);
    y.x = rbf(g.x * y.x);  // bf16(gate * y)
    y.y = rbf(g.y * y.y);
  }
  const float2 r = unpack_bf16x2(resid);
  return make_float2(r.x + y.x, r.y + y.y);
}

// ---- one consumer's epilogue: HALVES 64-row halves x BN columns ----------------------------------------------------
// acc[hm] holds rows 64 hm .. 64 hm + 63 of the block whose first output element is (m0, n0); the 16-bit result goes
// to the consumer's 128B-swizzled staging rows at my_c ([BN/64][128 rows][128 B]), for the caller to TMA-store.  ACT 2
// reads resid from the same slots, where the producer's TMA load lands it (resid_full completes phase `parity`).
// FP8: acc sums e4m3 products, y = bf16(fmaf(acc * sa[row], sw[col], bias[col])) (ep.sa, ep.sw).
template <int BN, int HALVES, int ACT, bool FP8 = false>
__device__ __forceinline__ void gemm_epilogue(const float (&acc)[HALVES][BN / 2], uint32_t my_c, int m0, int n0, int M,
                                              int N, const bf16* __restrict__ bias, const EpiArgs& ep,
                                              uint64_t* resid_full, uint32_t parity, int warp, int lane) {
  // thread rows: rl + 8 h + 64 hm for acc[hm][.. 2 h / 2 h + 1].  Every row of a thread has the same row % 8, so the
  // 128B swizzle of the staging chunk is one XOR per 8-column group: conflict-free (the 8 rows of a store land in 8
  // different 16-byte units).
  const int rl = warp * 16 + (lane >> 2);
  const uint32_t c_row = my_c + rl * 128 + (lane & 3) * 4;
  int gate_off[HALVES][2];  // element offset of the row's gate vector in mod, -1: none
  float row_scale[HALVES][2];  // FP8: sa of the row
#pragma unroll
  for (int hm = 0; hm < HALVES; ++hm)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = m0 + rl + 8 * h + 64 * hm;
      gate_off[hm][h] = -1;
      if (ACT == 2 && ep.gate_row >= 0 && grow < M) gate_off[hm][h] = gate_offset(ep, grow, N);
      row_scale[hm][h] = 0.f;
      if (FP8 && grow < M) row_scale[hm][h] = __ldg(ep.sa + grow);
    }
  if (ACT == 2) mbar_wait_quiet(resid_full, parity);  // the resid block is in the staging tile
#pragma unroll
  for (int jj = 0; jj < BN / 8; ++jj) {
    const int col = jj * 8 + 2 * (lane & 3);  // column inside the tile
    const int gcol = n0 + col;
    float2 b2 = make_float2(0.f, 0.f);
    if (bias != nullptr && gcol < N) b2 = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(bias + gcol)));
    float2 sw2 = make_float2(0.f, 0.f);
    if (FP8 && gcol < N) sw2 = __ldg(reinterpret_cast<const float2*>(ep.sw + gcol));
#pragma unroll
    for (int hm = 0; hm < HALVES; ++hm)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rl + 8 * h + 64 * hm;
        const uint32_t dst = c_row + (jj >> 3) * (kBM * 128) + (8 * h + 64 * hm) * 128 + (((jj & 7) ^ (rl & 7)) << 4);
        float2 x = make_float2(acc[hm][4 * jj + 2 * h] + b2.x, acc[hm][4 * jj + 2 * h + 1] + b2.y);
        if (FP8)
          x = make_float2(fmaf(acc[hm][4 * jj + 2 * h] * row_scale[hm][h], sw2.x, b2.x),
                          fmaf(acc[hm][4 * jj + 2 * h + 1] * row_scale[hm][h], sw2.y, b2.y));
        if (ACT == 1) x = gelu2<1>(make_float2(rbf(x.x), rbf(x.y)));
        if (ACT == 2 && m0 + row < M && gcol < N) {
          const bool gated = gate_off[hm][h] >= 0;
          const uint32_t g = gated ? __ldg(reinterpret_cast<const uint32_t*>(ep.mod + gate_off[hm][h] + gcol)) : 0u;
          uint32_t r;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(dst));  // resid, landed by TMA in the same slot
          x = residual_add2(make_float2(rbf(x.x), rbf(x.y)), r, gated, g);
        }
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(pack_bf16x2(x.x, x.y)) : "memory");  // ACT 3: y, see below
      }
  }
  if (ACT == 3) {
    // erf-GELU in a second pass over the thread's own staging slots, once the accumulators are dead: erff next to the
    // live accumulators would not fit in the register budget.
#pragma unroll 8
    for (int i = 0; i < BN / 8 * HALVES * 2; ++i) {
      const int jj = i / (2 * HALVES), hm = (i >> 1) % HALVES, h = i & 1;
      const uint32_t dst = c_row + (jj >> 3) * (kBM * 128) + (8 * h + 64 * hm) * 128 + (((jj & 7) ^ (rl & 7)) << 4);
      uint32_t r;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(dst));
      const float2 v = gelu2<3>(unpack_bf16x2(r));
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(pack_bf16x2(v.x, v.y)) : "memory");
    }
  }
}

// ---- the producer's k-block and the consumers' K loop, shared by the three kernels -----------------------------------
// Loads k-block kb of the tile at (m0, n0) into ring position n once the consumers have released the slot: a_boxes
// 128-row A boxes (1 or 2) and the W box.
template <class Cfg>
__device__ __forceinline__ void load_k_block(const CUtensorMap* tm_a, const CUtensorMap* tm_w, unsigned char* smem_ab,
                                             uint64_t* full, uint64_t* empty, int n, int kb, int m0, int n0, int a_boxes) {
  const int s = n % Cfg::kStages;
  mbar_wait_quiet(&empty[s], ((n / Cfg::kStages) & 1) ^ 1);
  unsigned char* sa = smem_ab + s * Cfg::kStageBytes;
  mbar_arrive_expect_tx(&full[s], a_boxes * kABox + Cfg::kStageBytes - Cfg::kABytes);
  tma_load_2d(tm_a, &full[s], sa, kb * Cfg::kBK, m0);
  if (a_boxes == 2) tma_load_2d(tm_a, &full[s], sa + kABox, kb * Cfg::kBK, m0 + kBM);
  tma_load_2d(tm_w, &full[s], sa + Cfg::kABytes, kb * Cfg::kBK, n0);
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 192)
    wgmma_m64n192k16_ss(d, da, db, scale_d);
  else
    wgmma_m64n128k16_ss(d, da, db, scale_d);
}

// One consumer's K loop over the k-blocks at ring positions n_base .. n_base + num_kb - 1: per k16 step one
// wgmma.m64n{BN}k16 per 64-row half, A from a_off inside the stage.  Each stage is released once the wgmma that read
// it has retired, all but the last: the caller releases that after its wgmma_wait<0>.
// e4m3 (Cfg::kFp8): per k32 step one wgmma.m64n128k32.e4m3, and each k-block's chain of four runs into a fresh
// fragment that is then added to the fp32 accumulators (promotion every 128 of K: the tensor core's own accumulation
// of fp8 products keeps fewer bits than fp32, so it never sums more than one k-block).
template <class Cfg, int HALVES>
__device__ __forceinline__ void consumer_k_loop(float (&acc)[HALVES][Cfg::kTileN / 2], uint32_t ab0, uint32_t a_off,
                                                uint64_t* full, uint64_t* empty, int n_base, int num_kb, int t) {
#pragma unroll
  for (int hm = 0; hm < HALVES; ++hm)
#pragma unroll
    for (int i = 0; i < Cfg::kTileN / 2; ++i) acc[hm][i] = 0.f;
  if constexpr (Cfg::kFp8) {
    static_assert(Cfg::kTileN == 128, "the e4m3 K loop runs m64n128k32");
    float part[HALVES][Cfg::kTileN / 2];
    for (int kb = 0; kb < num_kb; ++kb) {
      const int n = n_base + kb, s = n % Cfg::kStages;
      mbar_wait_quiet(&full[s], (n / Cfg::kStages) & 1);
      const uint32_t sa = ab0 + s * Cfg::kStageBytes + a_off;
      const uint32_t sw = ab0 + s * Cfg::kStageBytes + Cfg::kABytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t dw = wgmma_desc_sw128(sw + 32 * k);
#pragma unroll
        for (int hm = 0; hm < HALVES; ++hm)
          wgmma_m64n128k32_e4m3_ss(part[hm], wgmma_desc_sw128(sa + hm * (64 * 128) + 32 * k), dw, k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (kb > 0 && t == 0) mbar_arrive(&empty[(n - 1) % Cfg::kStages]);
#pragma unroll
      for (int hm = 0; hm < HALVES; ++hm)
#pragma unroll
        for (int i = 0; i < Cfg::kTileN / 2; ++i) acc[hm][i] += part[hm][i];
    }
    return;
  }
  for (int kb = 0; kb < num_kb; ++kb) {
    const int n = n_base + kb, s = n % Cfg::kStages;
    mbar_wait_quiet(&full[s], (n / Cfg::kStages) & 1);
    const uint32_t sa = ab0 + s * Cfg::kStageBytes + a_off;
    const uint32_t sw = ab0 + s * Cfg::kStageBytes + Cfg::kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      const uint64_t dw = wgmma_desc_sw128(sw + 32 * k);
#pragma unroll
      for (int hm = 0; hm < HALVES; ++hm) wgmma_tile<Cfg::kTileN>(acc[hm], wgmma_desc_sw128(sa + hm * (64 * 128) + 32 * k), dw, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the group of k-block kb - 1 has retired: its stage can be refilled
    if (kb > 0 && t == 0) mbar_arrive(&empty[(n - 1) % Cfg::kStages]);
  }
}

// TMA store from a 32-bit shared-memory address (the consumers keep no 64-bit pointer live across the mainloop)
__device__ __forceinline__ void tma_store_2d_s(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}

// ---- one CTA per 128 x BN tile (BN = 192 where it divides N): bias only, or GELU at long K --------------------------
// Without an epilogue to hide, the persistent kernel's 128 x 128 tile loses to this one: its mainloop moves 32 KB from L2
// per 2.1 MFLOP against 40 KB per 3.1 MFLOP here, and at ~8.7 TB/s both are bound by the L2 -> SM bandwidth, so the wider
// tile runs the K loop ~20 % faster (DESIGN.md section 9).  Warpgroup 0 is the TMA producer (one thread), warpgroups 1-2
// own rows 0..63 / 64..127 of the tile; the epilogue adds the bias, [rounds and applies tanh- or erf-GELU,] and
// TMA-stores the 16-bit tile.
template <int BN, int ACT>
__global__ void __launch_bounds__(TileCfg<BN>::kThreads, 1)
gemm_tile_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                 const __grid_constant__ CUtensorMap tm_c, const __grid_constant__ CUtensorMap tm_r,
                 const bf16* __restrict__ bias, int M, int N, int K, const EpiArgs ep) {
  using Cfg = TileCfg<BN>;
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
    if (threadIdx.x == 0)
      for (int kb = 0; kb < num_kb; ++kb) load_k_block<Cfg>(&tm_a, &tm_w, smem_ab, full, empty, kb, kb, m0, n0, 1);
    return;
  }

  // consumer c: rows 64 c .. 64 c + 63 of the tile and of its staging tile
  const int c = wg - 1;
  const int t = threadIdx.x & 127;
  float acc[1][BN / 2];
  consumer_k_loop<Cfg, 1>(acc, smem_u32(smem_ab), c * (64 * 128), full, empty, 0, num_kb, t);
  wgmma_wait<0>();
  gemm_epilogue<BN, 1, ACT>(acc, smem_u32(smem_c) + c * (64 * 128), m0 + 64 * c, n0, M, N, bias, ep, nullptr, 0, t >> 5,
                            t & 31);
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

// ---- persistent ping-pong kernel: the epilogues that cost (gate + residual, GELU at short K) ------------------------
template <int ACT>
__global__ void __launch_bounds__(GemmCfg::kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                  const __grid_constant__ CUtensorMap tm_c, const __grid_constant__ CUtensorMap tm_r,
                  const bf16* __restrict__ bias, int M, int N, int K, const EpiArgs ep) {
  using Cfg = GemmCfg;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  unsigned char* smem_ab = smem;                              // [kStages][A 16 KB | W 16 KB]
  unsigned char* smem_c = smem + kStages * Cfg::kStageBytes;  // [consumer][kBN/64][128 rows][128 B] swizzled
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_c + 2 * Cfg::kCBytes);  // [kStages]
  uint64_t* empty = full + kStages;                                         // [kStages]
  uint64_t* c_full = empty + kStages;   // [2] resid block landed in the consumer's staging tile (ACT 2)
  uint64_t* c_empty = c_full + 2;       // [2] the consumer's last TMA store has read its staging tile (ACT 2)

  const int wg = threadIdx.x >> 7;
  const int tiles_n = (N + kBN - 1) / kBN;
  const int tiles = ((M + kBM - 1) / kBM) * tiles_n;
  const int num_kb = (K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_c);
    if (ACT == 2) tma_prefetch_desc(&tm_r);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 1);  // each stage is read by the one consumer that owns its tile
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&c_full[i], 1);
      mbar_init(&c_empty[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 256) {
      int n = 0;  // k-blocks loaded so far: the position in the ring, carried over between tiles
      int j = 0;  // tile of this CTA; consumer j & 1 owns it
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++j) {
        const int m0 = (tile / tiles_n) * kBM, n0 = (tile % tiles_n) * kBN;
        for (int kb = 0; kb < num_kb; ++kb, ++n) {
          load_k_block<Cfg>(&tm_a, &tm_w, smem_ab, full, empty, n, kb, m0, n0, 1);
          if (ACT == 2 && kb == min(kStages, num_kb) - 1) {
            // the resid block, once the ring holds the tile's first k-blocks: the consumer is done with its previous
            // tile's staging by the time it needs more of this tile's k-blocks
            const int c = j & 1, u = j >> 1;  // u: the consumer's tile count so far
            if (u > 0) mbar_wait_quiet(&c_empty[c], (u - 1) & 1);
            const int nch = min(kBN / 64, (N - n0 + 63) / 64);  // 64-column chunks inside N
            unsigned char* dst = smem_c + c * Cfg::kCBytes;
            mbar_arrive_expect_tx(&c_full[c], nch * kBM * 128);
            for (int ch = 0; ch < nch; ++ch) tma_load_2d(&tm_r, &c_full[c], dst + ch * (kBM * 128), n0 + ch * 64, m0);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup c takes the CTA's tiles j = c, c + 2, ... =====================
  const int c = wg;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const uint32_t my_c = smem_u32(smem_c) + c * Cfg::kCBytes;
  const uint32_t ab0 = smem_u32(smem_ab);
  int u = 0;  // this consumer's tiles so far
  for (int j = c, tile = blockIdx.x + c * gridDim.x; tile < tiles; j += 2, tile += 2 * gridDim.x, ++u) {
    const int m0 = (tile / tiles_n) * kBM, n0 = (tile % tiles_n) * kBN;
    float acc[2][64];
    if (j > 0) named_bar_sync(1 + c, 256);  // our turn: the other consumer has issued its mainloop of tile j - 1
    const int n_base = j * num_kb;          // ring position of this tile's first k-block
    consumer_k_loop<Cfg, 2>(acc, ab0, 0, full, empty, n_base, num_kb, t);
    if (tile + gridDim.x < tiles) named_bar_arrive(1 + (c ^ 1), 256);  // hand the tensor cores to tile j + 1
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&empty[(n_base + num_kb - 1) % kStages]);

    gemm_epilogue<kBN, 2, ACT>(acc, my_c, m0, n0, M, N, bias, ep, &c_full[c], u & 1, warp, lane);
    fence_proxy_async_smem();
    named_bar_sync(3 + c, 128);
    if (t == 0) {
#pragma unroll 1
      for (int ch = 0; ch < kBN / 64; ++ch)
        if (n0 + ch * 64 < N) tma_store_2d_s(&tm_c, my_c + ch * (kBM * 128), n0 + ch * 64, m0);
      tma_store_commit();
      // the staging tile is rewritten by this consumer's next tile, after the turn barrier above (or the resid load
      // the producer issues on c_empty): wait here, under the other consumer's mainloop, until the store has read it
      tma_store_wait_read0();
      if (ACT == 2) mbar_arrive(&c_empty[c]);
    }
  }
  if (t == 0) tma_store_wait0();
}

// ---- persistent cooperative kernel on 256 x 128 tiles: the large-M Linears --------------------------------------------
// min(tiles, SMs) CTAs walk the 256 x 128 output tiles with a static stride, N-fastest.  Both consumer warpgroups work on
// the same tile, warpgroup c on rows 128 c .. 128 c + 127, with the same 2 x wgmma.m64n128k16 per k16 step as a consumer
// of gemm_wgmma_kernel, and both read one W stage: a stage is A 256x64 + W 128x64 = 48 KB per 4.2 MFLOP, a quarter
// fewer L2 -> SM bytes per FLOP than the 128 x 128 tile.
// Without a second tile to ping-pong with, the epilogue is split so that little of it stays off the tensor cores.  Every
// epilogue starts from y = bf16(acc + bias): the consumers store that into their half of the staging tile (the bias-only
// gemm_epilogue) and go on to the next tile's mainloop; three epilogue warps then apply the rest in place -- tanh-GELU(y),
// erf-GELU(y), or resid + [bf16(gate * y)] with resid read from global memory -- and TMA-store the tile.
// Every step sees the same 16-bit y and calls the same element functions as gemm_wgmma_kernel, so the outputs are
// bit-identical.  Barriers per consumer c: st_full[c] (the consumer's 128 threads have written y), st_free[c] (the
// tile's TMA store has read the consumer's rows).
// With e4m3 operands (WideFp8Cfg) the tile is 128 x 128, each consumer owns 64 rows of it, and y is
// bf16(acc * sa * sw + bias) (gemm_epilogue); the epilogue warps and their element functions are the same.
template <class Cfg, int ACT>
__global__ void __launch_bounds__(Cfg::kThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                 const __grid_constant__ CUtensorMap tm_c, const __grid_constant__ CUtensorMap tm_r,
                 const bf16* __restrict__ bias, int M, int N, int K, const EpiArgs ep) {
  constexpr int kStages = Cfg::kStages;
  constexpr int kRowsC = Cfg::kTileM / 2;     // rows of a tile per consumer
  constexpr int kHalves = kRowsC / 64;        // 64-row wgmma halves per consumer
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  unsigned char* smem_ab = smem;                              // [kStages][A 32 / 16 KB | W 16 KB]
  unsigned char* smem_c = smem + kStages * Cfg::kStageBytes;  // [kCBlocks][kBN/64][128 rows][128 B] swizzled
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_c + Cfg::kCBlocks * Cfg::kCBytes);  // [kStages]
  uint64_t* empty = full + kStages;                                                      // [kStages]
  uint64_t* st_full = empty + kStages;  // [2]
  uint64_t* st_free = st_full + 2;      // [2]

  const int wg = threadIdx.x >> 7;
  const int tiles_n = (N + kBN - 1) / kBN;
  const int tiles = ((M + Cfg::kTileM - 1) / Cfg::kTileM) * tiles_n;
  const int num_kb = (K + Cfg::kBK - 1) / Cfg::kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_c);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&st_full[i], 128);
      mbar_init(&st_free[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256 + kWideEpiThreads) {
      // ===================== TMA producer (warp 11) =====================
      int n = 0;  // k-blocks loaded so far: the position in the ring, carried over between tiles
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * Cfg::kTileM, n0 = (tile % tiles_n) * kBN;
        const int a_boxes = Cfg::kCBlocks == 2 && m0 + kBM < M ? 2 : 1;  // the lower box only where it has rows inside M
        for (int kb = 0; kb < num_kb; ++kb, ++n) load_k_block<Cfg>(&tm_a, &tm_w, smem_ab, full, empty, n, kb, m0, n0, a_boxes);
      }
    } else if (threadIdx.x < 256 + kWideEpiThreads) {
      // ===================== epilogue warps 8-10: the staged y -> the output, under the next mainloop ===============
      const int e = threadIdx.x - 256;
      const uint32_t c0 = smem_u32(smem_c);
      int j = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++j) {
        const int m0 = (tile / tiles_n) * Cfg::kTileM, n0 = (tile % tiles_n) * kBN;
        mbar_wait_quiet(&st_full[0], j & 1);
        mbar_wait_quiet(&st_full[1], j & 1);
        if (ACT != 0) {
          // 16-byte unit u of the staging tile = 8 columns of one row: u = ((half * 2 + chunk) * 128 + row) * 8 + slot,
          // the slot holding column group slot ^ (row & 7) of the 128B swizzle
#pragma unroll 2
          for (int u = e; u < Cfg::kCBlocks * Cfg::kCBytes / 16; u += kWideEpiThreads) {
            const int row = (u >> 3) & (kBM - 1), hc = u >> 10;
            const int grow = m0 + (hc >> 1) * kBM + row;
            const int gcol = n0 + (hc & 1) * 64 + (((u & 7) ^ (row & 7)) << 3);
            if (ACT == 2 && (grow >= M || gcol >= N)) continue;
            const uint32_t addr = c0 + u * 16;
            uint32_t v[4];
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr));
            if (ACT == 2) {
              const uint4 r4 = *reinterpret_cast<const uint4*>(ep.resid + (size_t)grow * N + gcol);  // may alias the output
              const uint32_t r[4] = {r4.x, r4.y, r4.z, r4.w};
              uint32_t g[4] = {0, 0, 0, 0};
              if (ep.gate_row >= 0) {
                const uint4 g4 = __ldg(reinterpret_cast<const uint4*>(ep.mod + (gate_offset(ep, grow, N) + gcol)));
                g[0] = g4.x, g[1] = g4.y, g[2] = g4.z, g[3] = g4.w;
              }
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float2 x = residual_add2(unpack_bf16x2(v[i]), r[i], ep.gate_row >= 0, g[i]);
                v[i] = pack_bf16x2(x.x, x.y);
              }
            } else {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float2 x = gelu2<ACT>(unpack_bf16x2(v[i]));
                v[i] = pack_bf16x2(x.x, x.y);
              }
            }
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3])
                         : "memory");
          }
          fence_proxy_async_smem();
        }
        named_bar_sync(1, kWideEpiThreads);
        if (e == 0) {
#pragma unroll 1
          for (int h = 0; h < Cfg::kCBlocks; ++h)
            for (int ch = 0; ch < kBN / 64; ++ch)
              if (m0 + h * kBM < M && n0 + ch * 64 < N)
                tma_store_2d_s(&tm_c, c0 + h * Cfg::kCBytes + ch * (kBM * 128), n0 + ch * 64, m0 + h * kBM);
          tma_store_commit();
          tma_store_wait_read0();  // the consumers write the next tile's y into the halves after this
          mbar_arrive(&st_free[0]);
          mbar_arrive(&st_free[1]);
        }
      }
      if (e == 0) tma_store_wait0();
    }
    return;
  }

  // ===================== consumers: warpgroup c takes rows kRowsC c .. kRowsC c + kRowsC - 1 of every tile ============
  const int c = wg;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  // the consumer's first row in the staging tile: 128-row block c (16-bit), or row 64 c of the one block (e4m3)
  const uint32_t my_c = smem_u32(smem_c) + c * (kRowsC == kBM ? Cfg::kCBytes : kRowsC * 128);
  const uint32_t ab0 = smem_u32(smem_ab);
  int j = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++j) {
    const int m0 = (tile / tiles_n) * Cfg::kTileM + c * kRowsC, n0 = (tile % tiles_n) * kBN;
    float acc[kHalves][64];
    const int n_base = j * num_kb;  // ring position of this tile's first k-block
    consumer_k_loop<Cfg, kHalves>(acc, ab0, c * kRowsC * 128, full, empty, n_base, num_kb, t);
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&empty[(n_base + num_kb - 1) % kStages]);

    if (j > 0) mbar_wait_quiet(&st_free[c], (j - 1) & 1);  // the previous tile's store has read these rows
    // y = bf16(acc + bias), or bf16(acc * sa * sw + bias)
    gemm_epilogue<kBN, kHalves, 0, Cfg::kFp8>(acc, my_c, m0, n0, M, N, bias, ep, nullptr, 0, warp, lane);
    fence_proxy_async_smem();  // bias only: the TMA store reads y as written
    mbar_arrive(&st_full[c]);
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
// Tensor map of a row-major [rows, cols] 16-bit (or, fp8, 1-byte) matrix, moved in 128B-swizzled boxes of box_rows
// rows x 128 bytes.
static int make_tmap_rows(CUtensorMap* m, const void* p, int rows, int cols, int box_rows, bool fp8 = false) {
  const int esize = fp8 ? 1 : 2;
  const unsigned long long dims[2] = {(unsigned long long)cols, (unsigned long long)rows};
  const unsigned long long stride[1] = {(unsigned long long)cols * esize};
  const unsigned box[2] = {128u / esize, (unsigned)box_rows};
  return make_tmap_elem(fp8 ? kTmapDtypeU8 : VSB_TMAP_DTYPE, m, p, 2, dims, stride, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

typedef int (*GemmLaunch)(const void* A, const void* W, const bf16* bias, void* out, int M, int N, int K,
                          const EpiArgs& ep, cudaStream_t st);

// Launches one kernel instance: a CTA per tile, or min(tiles, SMs) CTAs for a persistent kernel.  The first launch of
// an instance raises its dynamic shared-memory limit.  All three kernels take the same parameters, so that this one
// launcher serves them; tm_r (read only by gemm_wgmma_kernel<2>) and ep go unused where the epilogue has no residual.
template <auto kKernel, class Cfg>
static int launch_gemm(const void* A, const void* W, const bf16* bias, void* out, int M, int N, int K,
                       const EpiArgs& ep, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "gemm: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  CUtensorMap ta, tw, tc, tr;
  int rc = make_tmap_rows(&ta, A, M, K, kBM, Cfg::kFp8);
  if (!rc) rc = make_tmap_rows(&tw, W, N, K, Cfg::kTileN, Cfg::kFp8);
  if (!rc) rc = make_tmap_rows(&tc, out, M, N, kBM);
  if (rc) return rc;
  tr = tc;  // unused without a resid
  if (ep.resid != nullptr) {
    rc = make_tmap_rows(&tr, ep.resid, M, N, kBM);
    if (rc) return rc;
  }
  const long long tiles = (long long)((M + Cfg::kTileM - 1) / Cfg::kTileM) * ((N + Cfg::kTileN - 1) / Cfg::kTileN);
  const int grid = Cfg::kPersistent && tiles > num_sms() ? num_sms() : int(tiles);
  kKernel<<<grid, Cfg::kThreads, Cfg::kSmemBytes, st>>>(ta, tw, tc, tr, bias, M, N, K, ep);
  return check_launch("gemm");
}

enum class GemmKernel { kTile128, kTile192, kPingPong, kWide };

// The instance gemm_dispatch launches and vsb_gemm_kernel_name reports, by [GemmKernel][epilogue]; an empty slot is one
// gemm_route never picks.
struct GemmInstance {
  GemmLaunch launch;
  const char* name;
};
static const GemmInstance kGemmInstances[4][4] = {
    {{launch_gemm<gemm_tile_kernel<128, 0>, TileCfg<128>>, "gemm_tile_kernel<128, 0>"},
     {launch_gemm<gemm_tile_kernel<128, 1>, TileCfg<128>>, "gemm_tile_kernel<128, 1>"},
     {},
     {launch_gemm<gemm_tile_kernel<128, 3>, TileCfg<128>>, "gemm_tile_kernel<128, 3>"}},
    {{launch_gemm<gemm_tile_kernel<192, 0>, TileCfg<192>>, "gemm_tile_kernel<192, 0>"},
     {launch_gemm<gemm_tile_kernel<192, 1>, TileCfg<192>>, "gemm_tile_kernel<192, 1>"},
     {},
     {launch_gemm<gemm_tile_kernel<192, 3>, TileCfg<192>>, "gemm_tile_kernel<192, 3>"}},
    {{},
     {launch_gemm<gemm_wgmma_kernel<1>, GemmCfg>, "gemm_wgmma_kernel<1>"},
     {launch_gemm<gemm_wgmma_kernel<2>, GemmCfg>, "gemm_wgmma_kernel<2>"},
     {launch_gemm<gemm_wgmma_kernel<3>, GemmCfg>, "gemm_wgmma_kernel<3>"}},
    {{launch_gemm<gemm_wide_kernel<WideCfg, 0>, WideCfg>, "gemm_wide_kernel<0>"},
     {launch_gemm<gemm_wide_kernel<WideCfg, 1>, WideCfg>, "gemm_wide_kernel<1>"},
     {launch_gemm<gemm_wide_kernel<WideCfg, 2>, WideCfg>, "gemm_wide_kernel<2>"},
     {launch_gemm<gemm_wide_kernel<WideCfg, 3>, WideCfg>, "gemm_wide_kernel<3>"}}};

// The e4m3 instances by epilogue (0 none, 1 tanh-GELU, 2 fused residual): gemm_route_fp8 picks one for every shape.
static const GemmInstance kGemmFp8Instances[3] = {
    {launch_gemm<gemm_wide_kernel<WideFp8Cfg, 0>, WideFp8Cfg>, "gemm_wide_kernel<fp8, 0>"},
    {launch_gemm<gemm_wide_kernel<WideFp8Cfg, 1>, WideFp8Cfg>, "gemm_wide_kernel<fp8, 1>"},
    {launch_gemm<gemm_wide_kernel<WideFp8Cfg, 2>, WideFp8Cfg>, "gemm_wide_kernel<fp8, 2>"}};

// Which kernel runs a GEMM; act: 0 none, 1 tanh-GELU, 2 fused residual, 3 erf-GELU.
static GemmKernel gemm_route(int M, int N, int K, int act) {
  // The 256 x 128 kernel against the kernel each shape ran on before (bench_gemm.py, H100 80GB HBM3, 700 W, SM clock
  // 1980 MHz, bit-identical outputs; DESIGN.md section 9):
  //   bias only (was gemm_tile_kernel<192>): K 1152 1.24x (N 3456) / 1.15x (N 1152), K 1920 1.12x, K 2304 1.07x,
  //     K 4608 1.05x
  //   tanh-GELU: K 1152 1.20x, K 1536 1.20x (both were persistent), K 1920 1.16x, K 2304 1.16x, K 3072 1.12x
  //   erf-GELU, K 2304: 1.09x;  gate + residual (was persistent): K 1152 0.55x, K 4608 1.24x
  // The residual epilogue reads resid from global memory in the epilogue warps, which a K loop of 1152 does not hide.
  // It runs at 2048 tiles or more: the fewest it was measured at (CogVideoX-2B, 2085).
  const long long wide_tiles = (long long)((M + WideCfg::kTileM - 1) / WideCfg::kTileM) * ((N + kBN - 1) / kBN);
  if (wide_tiles >= kWideMinTiles && (act != 2 || K >= 4608))
    return GemmKernel::kWide;
  // The persistent kernel's K loop is slower than the one-tile-per-CTA kernel's (0.671 against 0.521 ms per 1152 of K at
  // N 1152, H100 SXM, DESIGN.md section 9); what it saves per tile is the fill, the store and the epilogue.  The gate +
  // residual epilogue saves more than the K loop costs at every K measured (up to 4608); a bias-only epilogue never does;
  // a GELU epilogue only while K is short.
  if (act == 0 || ((act == 1 || act == 3) && K > kPersistentGeluMaxK)) {
    // tile width: 192 divides every STDiT3 / CogVideoX / Latte width (1152, 1920, 2304, 3072, 3456, 4608, 7680); narrow
    // outputs and widths that 128 divides but 192 does not take 128
    return (N % 192 == 0 || (N > 192 && N % 128 != 0)) ? GemmKernel::kTile192 : GemmKernel::kTile128;
  }
  return GemmKernel::kPingPong;
}

// act: 0 none, 1 tanh-GELU, 2 fused residual (ep->resid != nullptr), 3 erf-GELU
static int gemm_dispatch(const void* A, const void* W, const void* bias, void* out, int M, int N, int K, int act,
                         cudaStream_t st, const EpiArgs& ep) {
  if ((long long)((M + kBM - 1) / kBM) * ((N + kBN - 1) / kBN) > 0x7fffffffLL)
    return fail(VSB_ERR_UNSUPPORTED, "gemm: too many tiles (M=%d N=%d)", M, N);
  const GemmKernel kern = gemm_route(M, N, K, act);
  const GemmInstance& g = kGemmInstances[int(kern)][act];
  if (g.launch == nullptr) return fail(VSB_ERR_UNSUPPORTED, "gemm: no kernel instance for route %d, epilogue %d", int(kern), act);
  return g.launch(A, W, (const bf16*)bias, out, M, N, K, ep, st);
}

// Which e4m3 instance runs a GEMM; act: 0 none, 1 tanh-GELU, 2 fused residual.  Every shape takes the persistent
// 128 x 128 kernel: the promotion fragment rules out the 256-row tile, and no epilogue is left on the tensor cores' path.
static const GemmInstance& gemm_route_fp8(int act) { return kGemmFp8Instances[act]; }

static int gemm_fp8_dispatch(const void* A, const float* sa, const void* W, const float* sw, const void* bias, void* out,
                             int M, int N, int K, int act, cudaStream_t st, EpiArgs ep) {
  if (!A || !sa || !W || !sw || !out || M <= 0 || N <= 0 || K <= 0) return fail(VSB_ERR_INVALID, "gemm_fp8: bad args");
  if (K % 16 || N % 8 || !aligned16(A) || !aligned16(W) || !aligned16(out) || !aligned16(sw) ||
      (ep.resid != nullptr && !aligned16(ep.resid)))
    return fail(VSB_ERR_UNSUPPORTED, "gemm_fp8: need K %% 16 == 0, N %% 8 == 0, 16B-aligned pointers (M=%d N=%d K=%d)", M, N, K);
  if ((long long)((M + kBM - 1) / kBM) * ((N + kBN - 1) / kBN) > 0x7fffffffLL)
    return fail(VSB_ERR_UNSUPPORTED, "gemm_fp8: too many tiles (M=%d N=%d)", M, N);
  ep.sa = sa;
  ep.sw = sw;
  return gemm_route_fp8(act).launch(A, W, (const bf16*)bias, out, M, N, K, ep, st);
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

// e4m3 operands, see include/vsb200.h: out = act(bf16(acc * sa[m] * sw[n] + bias)).
extern "C" int VSB_API(vsb_gemm_fp8_bias_act)(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw,
                                              const vsb_bf16* bias, vsb_bf16* out, int M, int N, int K, int act, void* stream) {
  if (act < 0 || act > 1) return fail(VSB_ERR_INVALID, "gemm_fp8: act=%d", act);
  return gemm_fp8_dispatch(A, sa, W, sw, bias, out, M, N, K, act, (cudaStream_t)stream, EpiArgs{nullptr, nullptr, nullptr, -1, 1, 1, 1});
}

extern "C" int VSB_API(vsb_gemm_fp8_bias_residual)(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw,
                                                   const vsb_bf16* bias, const vsb_bf16* resid, vsb_bf16* out,
                                                   const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int M, int N,
                                                   int K, int B, int T, int S, void* stream) {
  if (!resid) return fail(VSB_ERR_INVALID, "gemm_fp8_residual: bad args");
  if (gate_row >= 0) {
    if (!mod || gate_row > 5 || B <= 0 || T <= 0 || S <= 0 || (long long)B * T * S != M || !aligned16(mod))
      return fail(VSB_ERR_INVALID, "gemm_fp8_residual: gate needs mod[2,B,6,N] and B*T*S == M");
  }
  EpiArgs ep{(const bf16*)resid, (const bf16*)mod, x_mask, gate_row, B, T, S};
  return gemm_fp8_dispatch(A, sa, W, sw, bias, out, M, N, K, 2, (cudaStream_t)stream, ep);
}

#ifndef VSB_HALF
// The kernel gemm_fp8_dispatch picks for a shape (the same for both 16-bit output types), see include/vsb200.h.
extern "C" const char* vsb_gemm_fp8_kernel_name(int M, int N, int K, int act, int residual) {
  if (M <= 0 || N <= 0 || K <= 0 || act < 0 || act > 1 || (residual && act != 0)) return "";
  return gemm_route_fp8(residual ? 2 : act).name;
}

// The kernel gemm_dispatch picks for a shape (the same for both 16-bit types), see include/vsb200.h.
extern "C" const char* vsb_gemm_kernel_name(int M, int N, int K, int act, int residual) {
  if (M <= 0 || N <= 0 || K <= 0 || act < 0 || act > 2 || (residual && act != 0)) return "";
  const int epi = residual ? 2 : (act == 2 ? 3 : act);
  const char* name = kGemmInstances[int(gemm_route(M, N, K, epi))][epi].name;
  return name != nullptr ? name : "";
}
#endif
