// vsb200 -- flash attention forward on the Hopper warpgroup tensor cores for head_dim 64 (CogVideoX, Vchitect) and 72
// (STDiT3, Latte, Open-Sora-Plan v1.1.0): the spatial, cross and joint attention of every model.
//
// CTA = 128 query rows of one (batch, head), 9 warps:
//   warps 0-3, 4-7  two consumer warpgroups, 64 query rows each
//   warp 8          TMA producer (one lane): the Q tile once, then 128-key K / V tiles through a kStages-deep mbarrier ring
// Per key tile a consumer warpgroup runs S = Q K^T as wgmma.m64n128k16 with Q and K both read from shared memory (fp32
// scores in registers), the online softmax on those registers (row max / sum across the 4 lanes that share a row), packs P
// to the 16-bit dtype straight into the register A fragments of O += P V (wgmma with A from registers, V read as an
// MN-major B operand), and releases the stage.  The two warpgroups run independently, so one's softmax overlaps the
// other's MMAs.
//
// Operand tiles are staged by TMA as a 64-column SWIZZLE_128B part and, for head_dim 72, a 16-column SWIZZLE_32B part
// (columns 64..79; the tensor map's inner extent is 72, so TMA zero-fills 72..79 and every row past the sequence): Q K^T
// takes 4 (+1) k16 steps, P V two N slices (64 and 16 columns).  Keys past the per-batch count are masked to -inf.
#include "attn_params.cuh"
#include "wgmma.cuh"

namespace vsb {

constexpr int kWaRows = 128;  // query rows per CTA
constexpr int kWaKeys = 128;  // keys per tile
constexpr int kWaStages = 2;
constexpr int kWaThreads = 288;

template <int D>
struct WaCfg {
  static constexpr bool kHas32 = D > 64;
  static constexpr int kPart128 = 128 * 128;               // 128 rows x 64 columns, SWIZZLE_128B
  static constexpr int kPart32 = kHas32 ? 128 * 32 : 0;    // 128 rows x 16 columns, SWIZZLE_32B
  static constexpr int kTile = kPart128 + kPart32;         // a Q, K or V tile
  static constexpr int kSmem = kTile * (1 + 2 * kWaStages) + 1024 + 256;
};

template <int D>
__global__ void __launch_bounds__(kWaThreads, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_q32,
                  const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_k32,
                  const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_v32,
                  const __grid_constant__ AttnParams p) {
  using Cfg = WaCfg<D>;
  constexpr bool kHas32 = Cfg::kHas32;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  unsigned char* sQ = smem;                       // [Q128 | Q32]
  unsigned char* sKV = smem + Cfg::kTile;         // [stage][K128 | K32 | V128 | V32]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + kWaStages * 2 * Cfg::kTile);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;               // [kWaStages]
  uint64_t* kv_empty = kv_full + kWaStages;   // [kWaStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kWaRows, h = blockIdx.y, b = blockIdx.z;
  const int kv_len = p.has_lens ? p.lens[b] : p.nk;
  const int n_tiles = (kv_len + kWaKeys - 1) / kWaKeys;

  if (threadIdx.x == 256) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kWaStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // =============================== TMA producer ===============================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, Cfg::kTile);
      tma_load_4d(&tm_q, q_full, sQ, 0, h, q0, b);
      if (kHas32) tma_load_4d(&tm_q32, q_full, sQ + Cfg::kPart128, 64, h, q0, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % kWaStages;
        mbar_wait_quiet(&kv_empty[s], ((j / kWaStages) & 1) ^ 1);
        unsigned char* st = sKV + s * 2 * Cfg::kTile;
        mbar_arrive_expect_tx(&kv_full[s], 2 * Cfg::kTile);
        tma_load_4d(&tm_k, &kv_full[s], st, 0, h, j * kWaKeys, b);
        if (kHas32) tma_load_4d(&tm_k32, &kv_full[s], st + Cfg::kPart128, 64, h, j * kWaKeys, b);
        tma_load_4d(&tm_v, &kv_full[s], st + Cfg::kTile, 0, h, j * kWaKeys, b);
        if (kHas32) tma_load_4d(&tm_v32, &kv_full[s], st + Cfg::kTile + Cfg::kPart128, 64, h, j * kWaKeys, b);
      }
    }
    return;
  }

  // =============================== consumer warpgroup c: query rows 64 c .. 64 c + 63 ===============================
  const int c = warp >> 2, t = threadIdx.x & 127, w = warp & 3, tq = lane & 3;
  const uint32_t qa = smem_u32(sQ) + c * (64 * 128);
  const uint32_t qa32 = smem_u32(sQ) + Cfg::kPart128 + c * (64 * 32);
  const float sl2 = p.scale_log2;
  float o[32], o2[8], sacc[64];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) o2[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g and g + 8 of this warp's 16
  mbar_wait_quiet(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j % kWaStages;
    mbar_wait_quiet(&kv_full[s], (j / kWaStages) & 1);
    const uint32_t ka = smem_u32(sKV) + s * 2 * Cfg::kTile;
    const uint32_t va = ka + Cfg::kTile;
    // ---- S = Q K^T (K-major A and B: 8-row groups 1024 B apart in the 128B-swizzled part, 256 B in the 32B one) ----
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n128k16_ss(sacc, wgmma_desc(qa + 32 * k, 16, 1024, 1), wgmma_desc(ka + 32 * k, 16, 1024, 1), k > 0 ? 1u : 0u);
    if (kHas32) wgmma_m64n128k16_ss(sacc, wgmma_desc(qa32, 16, 256, 3), wgmma_desc(ka + Cfg::kPart128, 16, 256, 3), 1u);
    wgmma_commit();
    wgmma_wait<0>();

    // ---- online softmax (base 2, scale folded); key of sacc[i] = j*128 + 8 (i / 4) + 2 tq + (i & 1), row half (i / 2) & 1 ----
    const int k0 = j * kWaKeys;
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int col = k0 + 8 * (i >> 2) + 2 * tq + (i & 1);
      const float v = col < kv_len ? sacc[i] * sl2 : -INFINITY;
      sacc[i] = v;
      if (i & 2) mx1 = fmaxf(mx1, v); else mx0 = fmaxf(mx0, v);
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // every tile holds at least one valid key, so mx0 / mx1 are finite; exp2(-inf) = 0 on the first tile
    const float a0 = fast_exp2(m0 - mx0), a1 = fast_exp2(m1 - mx1);
    m0 = mx0;
    m1 = mx1;
    float r0 = 0.f, r1 = 0.f;
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = 8 * kk + 2 * q;  // q = 0: row g, keys 16 kk + 2 tq; 1: row g + 8; 2 / 3: the same at keys + 8
        const float mm = (q & 1) ? mx1 : mx0;
        const float e0 = fast_exp2(sacc[i] - mm), e1 = fast_exp2(sacc[i + 1] - mm);
        if (q & 1) r1 += e0 + e1; else r0 += e0 + e1;
        pa[kk][q] = pack_bf16x2(e0, e1);
      }
    }
    r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
    r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
    r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
    r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
    l0 = l0 * a0 + r0;
    l1 = l1 * a1 + r1;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= (i & 2) ? a1 : a0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o2[i] *= (i & 2) ? a1 : a0;

    // ---- O += P V (V MN-major: key rows 128 B / 32 B apart, 8-key groups 1024 B / 256 B apart; +16 keys per k16 step) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      wgmma_m64n64k16_rs_t(o, pa[kk], wgmma_desc(va + kk * 2048, 1024, 1024, 1), 1u);
      if (kHas32) wgmma_m64n16k16_rs_t(o2, pa[kk], wgmma_desc(va + Cfg::kPart128 + kk * 512, 256, 256, 3), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&kv_empty[s]);  // both MMAs of this warpgroup have read the stage
  }

  // ---- O / l -> 16-bit -> out (rows g and g + 8; columns 8 (i / 4) + 2 tq) ----
  const int row0 = q0 + c * 64 + w * 16 + (lane >> 2), row1 = row0 + 8;
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  bf16* ob = p.out + (size_t)b * p.out_batch_stride + (size_t)h * D;
#pragma unroll
  for (int i = 0; i < 32; i += 4) {
    const int col = 8 * (i >> 2) + 2 * tq;
    if (row0 < p.nq) *reinterpret_cast<uint32_t*>(ob + (size_t)row0 * p.out_row_stride + col) = pack_bf16x2(o[i] * i0, o[i + 1] * i0);
    if (row1 < p.nq) *reinterpret_cast<uint32_t*>(ob + (size_t)row1 * p.out_row_stride + col) = pack_bf16x2(o[i + 2] * i1, o[i + 3] * i1);
  }
  if (kHas32) {  // columns 64..71 (o2[0..3]); 72..79 are the zero padding
    const int col = 64 + 2 * tq;
    if (row0 < p.nq) *reinterpret_cast<uint32_t*>(ob + (size_t)row0 * p.out_row_stride + col) = pack_bf16x2(o2[0] * i0, o2[1] * i0);
    if (row1 < p.nq) *reinterpret_cast<uint32_t*>(ob + (size_t)row1 * p.out_row_stride + col) = pack_bf16x2(o2[2] * i1, o2[3] * i1);
  }
}

template <int D>
static int launch_wgmma(const CUtensorMap* tm, const AttnParams& prm, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_wgmma_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, WaCfg<D>::kSmem);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "attn_wgmma: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  dim3 grid((prm.nq + kWaRows - 1) / kWaRows, prm.H, prm.nb);
  attn_wgmma_kernel<D><<<grid, kWaThreads, WaCfg<D>::kSmem, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], prm);
  return check_launch("attn_wgmma");
}

int attn_wgmma_launch(const bf16* q, const bf16* k, const bf16* v, long long kv_row_stride, long long kv_batch_stride,
                      const AttnParams& prm, int D, cudaStream_t st) {
  // Two tensor maps per operand: the 64-column SWIZZLE_128B part and (head_dim 72) the 16-column SWIZZLE_32B part.
  CUtensorMap tm[6];
  const bf16* base[3] = {q, k, v};
  for (int i = 0; i < 3; ++i) {
    const long long rs = i == 0 ? prm.q_row_stride : kv_row_stride, bs = i == 0 ? prm.q_batch_stride : kv_batch_stride;
    unsigned long long dims[4] = {(unsigned long long)D, (unsigned long long)prm.H, (unsigned long long)(i == 0 ? prm.nq : prm.nk),
                                  (unsigned long long)prm.nb};
    unsigned long long str[3] = {(unsigned long long)D * 2, (unsigned long long)rs * 2, (unsigned long long)bs * 2};
    unsigned box128[4] = {64, 1, 128, 1}, box32[4] = {16, 1, 128, 1};
    int rc = make_tmap_bf16(&tm[2 * i], base[i], 4, dims, str, box128, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    if (D == 72) {
      rc = make_tmap_bf16(&tm[2 * i + 1], base[i], 4, dims, str, box32, CU_TENSOR_MAP_SWIZZLE_32B);
      if (rc) return rc;
    } else {
      tm[2 * i + 1] = tm[2 * i];  // unused by the head_dim-64 instantiation
    }
  }
  if (D == 72) return launch_wgmma<72>(tm, prm, st);
  if (D == 64) return launch_wgmma<64>(tm, prm, st);
  return fail(VSB_ERR_UNSUPPORTED, "attn_wgmma: head_dim %d", D);
}

}  // namespace vsb
