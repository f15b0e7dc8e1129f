// vsb200 -- flash attention forward on the Hopper warpgroup tensor cores for head_dim 64 (CogVideoX, Vchitect) and 72
// (STDiT3, Latte, Open-Sora-Plan v1.1.0): the spatial, cross and joint attention of every model.
//
// Persistent CTAs (one per SM), 12 warps, each CTA walking the work items (128-row query tile, head, batch), query tile
// fastest, so the CTAs that run at the same time read the same K / V from L2:
//   warps 0-3, 4-7  two consumer warpgroups, 64 query rows each (registers raised to 240 with setmaxnreg)
//   warps 8-11      producer warpgroup (registers lowered to 24); one thread issues TMA: the item's Q tile, then its
//                   128-key K and V tiles through two separate kWaStages-deep mbarrier rings
// Per key tile a consumer warpgroup runs S = Q K^T as wgmma.m64n128k16 with Q and K both read from shared memory (fp32
// scores in registers), the online softmax on those registers (row max / sum across the 4 lanes that share a row), packs P
// to the 16-bit dtype straight into the register A fragments of O += P V (wgmma with A from registers, V read as an
// MN-major B operand).
//
// Schedule (FlashAttention-3, sections 3.1 and 3.2): a warpgroup issues S_j = Q K_j^T and O += P_{j-1} V_{j-1} back to
// back, runs the softmax of tile j while P_{j-1} V_{j-1} is still on the tensor cores, then waits for it and rescales O.
// The two warpgroups take turns issuing their MMAs (named barriers 1 and 2), so one's softmax runs under the other's
// MMAs.  Q is released after the item's last S MMA, so the producer loads the next item's Q while the consumers finish
// the last P V and store the output.  The arithmetic is the one of a plain sequential loop: scores x scale_log2, row max,
// exp2(s - m), per-thread row sums then two shuffles, O rescaled before each P V, and O / l at the end.
//
// Operand tiles are staged by TMA as a 64-column SWIZZLE_128B part and, for head_dim 72, a 16-column SWIZZLE_32B part
// (columns 64..79; the tensor map's inner extent is 72, so TMA zero-fills 72..79 and every row past the sequence): Q K^T
// takes 4 (+1) k16 steps, P V two N slices (64 and 16 columns).  Keys past the per-batch count are masked to -inf; only
// the last key tile of an item can hold such keys, so only it pays for the mask.
#include "attn_params.cuh"
#include "wgmma.cuh"

namespace vsb {

constexpr int kWaRows = 128;  // query rows per work item
constexpr int kWaKeys = 128;  // keys per tile
constexpr int kWaStages = 2;  // depth of the K ring and of the V ring
constexpr int kWaThreads = 384;
constexpr int kWaProducerRegs = 24, kWaConsumerRegs = 240;  // 24 x 128 + 240 x 256 = 168 x 384 (the launch allocation)

template <int D>
struct WaCfg {
  static constexpr bool kHas32 = D > 64;
  static constexpr int kPart128 = 128 * 128;               // 128 rows x 64 columns, SWIZZLE_128B
  static constexpr int kPart32 = kHas32 ? 128 * 32 : 0;    // 128 rows x 16 columns, SWIZZLE_32B
  static constexpr int kTile = kPart128 + kPart32;         // a Q, K or V tile
  static constexpr int kSmem = kTile * (1 + 2 * kWaStages) + 1024 + 256;
};

// Online-softmax step on one 64 x 128 score tile held as wgmma accumulators: s <- exp2(s * sl2 - m_new) in place, the new
// row maxima in m0 / m1, the rescale factors exp2(m_old - m_new) in a0 / a1, the row sums of this tile in r0 / r1.
// kMask: keys at tile column >= lim are -inf (the tile that crosses the key count).
template <bool kMask>
__device__ __forceinline__ void wa_softmax(float (&s)[64], float& m0, float& m1, float& a0, float& a1, float& r0, float& r1,
                                           float sl2, int lim, int tq) {
  float mx0 = m0, mx1 = m1;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const float v = (!kMask || 8 * (i >> 2) + 2 * tq + (i & 1) < lim) ? s[i] * sl2 : -INFINITY;
    s[i] = v;
    if (i & 2) mx1 = fmaxf(mx1, v); else mx0 = fmaxf(mx0, v);
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  // every tile holds at least one valid key, so mx0 / mx1 are finite; exp2(-inf) = 0 on the first tile
  a0 = fast_exp2(m0 - mx0);
  a1 = fast_exp2(m1 - mx1);
  m0 = mx0;
  m1 = mx1;
  r0 = 0.f;
  r1 = 0.f;
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = 8 * kk + 2 * q;  // q = 0: row g, keys 16 kk + 2 tq; 1: row g + 8; 2 / 3: the same at keys + 8
      const float mm = (q & 1) ? mx1 : mx0;
      const float e0 = fast_exp2(s[i] - mm), e1 = fast_exp2(s[i + 1] - mm);
      if (q & 1) r1 += e0 + e1; else r0 += e0 + e1;
      s[i] = e0;
      s[i + 1] = e1;
    }
  }
  r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
  r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
  r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
  r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
}

// Position of the n-th tile of a ring: stage and the parity of its use.
__device__ __forceinline__ void wa_ring(int n, int& stage, uint32_t& parity) {
  stage = n % kWaStages;
  parity = (n / kWaStages) & 1;
}

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
  unsigned char* sQ = smem;                            // [Q128 | Q32]
  unsigned char* sK = smem + Cfg::kTile;               // [stage][K128 | K32]
  unsigned char* sV = sK + kWaStages * Cfg::kTile;     // [stage][V128 | V32]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kWaStages * Cfg::kTile);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* k_full = bars + 2;                  // [kWaStages]
  uint64_t* k_empty = k_full + kWaStages;       // [kWaStages]
  uint64_t* v_full = k_empty + kWaStages;       // [kWaStages]
  uint64_t* v_empty = v_full + kWaStages;       // [kWaStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_qt = (p.nq + kWaRows - 1) / kWaRows;
  const int n_items = n_qt * p.H * p.nb;

  if (threadIdx.x == 256) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 2);  // one arrival per consumer warpgroup
    for (int i = 0; i < kWaStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 2);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // =============================== TMA producer ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWaProducerRegs));
    if (threadIdx.x == 256) {
      int n = 0;  // key tiles loaded so far (position in both rings)
      uint32_t it = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
        const int q0 = (item % n_qt) * kWaRows, h = (item / n_qt) % p.H, b = item / (n_qt * p.H);
        const int n_tiles = ((p.has_lens ? p.lens[b] : p.nk) + kWaKeys - 1) / kWaKeys;
        mbar_wait_quiet(q_empty, (it & 1) ^ 1);
        mbar_arrive_expect_tx(q_full, Cfg::kTile);
        tma_load_4d(&tm_q, q_full, sQ, 0, h, q0, b);
        if (kHas32) tma_load_4d(&tm_q32, q_full, sQ + Cfg::kPart128, 64, h, q0, b);
        for (int j = 0; j < n_tiles; ++j, ++n) {
          int s;
          uint32_t ph;
          wa_ring(n, s, ph);
          mbar_wait_quiet(&k_empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&k_full[s], Cfg::kTile);
          tma_load_4d(&tm_k, &k_full[s], sK + s * Cfg::kTile, 0, h, j * kWaKeys, b);
          if (kHas32) tma_load_4d(&tm_k32, &k_full[s], sK + s * Cfg::kTile + Cfg::kPart128, 64, h, j * kWaKeys, b);
          mbar_wait_quiet(&v_empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&v_full[s], Cfg::kTile);
          tma_load_4d(&tm_v, &v_full[s], sV + s * Cfg::kTile, 0, h, j * kWaKeys, b);
          if (kHas32) tma_load_4d(&tm_v32, &v_full[s], sV + s * Cfg::kTile + Cfg::kPart128, 64, h, j * kWaKeys, b);
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroup c: query rows 64 c .. 64 c + 63 of each item ===============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWaConsumerRegs));
  const int c = warp >> 2, t = threadIdx.x & 127, w = warp & 3, tq = lane & 3;
  // MMA turn-taking: warpgroup c waits on barrier 1 + c before issuing its MMAs and then hands the turn to the other.
  // Both warpgroups run the same items with the same tile counts, so they issue the same number of rounds; warpgroup 1
  // gives warpgroup 0 the first turn, and warpgroup 0 takes the turn warpgroup 1 hands back after its last round.
  const uint32_t my_bar = 1 + c, other_bar = 2 - c;
  if (c == 1) named_bar_arrive(1, 256);
  const uint32_t qa = smem_u32(sQ) + c * (64 * 128);
  const uint32_t qa32 = smem_u32(sQ) + Cfg::kPart128 + c * (64 * 32);
  const uint32_t ka0 = smem_u32(sK), va0 = smem_u32(sV);
  const float sl2 = p.scale_log2;
  float o[32], o2[8], sacc[64];
  uint32_t pa[8][4];
  int n = 0;  // key tiles consumed so far (position in both rings)
  uint32_t it = 0;

  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
    const int q0 = (item % n_qt) * kWaRows, h = (item / n_qt) % p.H, b = item / (n_qt * p.H);
    const int kv_len = p.has_lens ? p.lens[b] : p.nk;
    const int n_tiles = (kv_len + kWaKeys - 1) / kWaKeys;
    const int last_lim = kv_len - (n_tiles - 1) * kWaKeys;  // valid keys of the last tile
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) o2[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g and g + 8 of this warp's 16
    float a0, a1, r0, r1;

    // S = Q K^T into sacc (K-major A and B: 8-row groups 1024 B apart in the 128B-swizzled part, 256 B in the 32B one)
    auto issue_s = [&](uint32_t ka) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n128k16_ss(sacc, wgmma_desc(qa + 32 * k, 16, 1024, 1), wgmma_desc(ka + 32 * k, 16, 1024, 1), k > 0 ? 1u : 0u);
      if (kHas32) wgmma_m64n128k16_ss(sacc, wgmma_desc(qa32, 16, 256, 3), wgmma_desc(ka + Cfg::kPart128, 16, 256, 3), 1u);
      wgmma_commit();
    };
    // O += P V (V MN-major: key rows 128 B / 32 B apart, 8-key groups 1024 B / 256 B apart; +16 keys per k16 step)
    auto issue_pv = [&](uint32_t va) {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        wgmma_m64n64k16_rs_t(o, pa[kk], wgmma_desc(va + kk * 2048, 1024, 1024, 1), 1u);
        if (kHas32) wgmma_m64n16k16_rs_t(o2, pa[kk], wgmma_desc(va + Cfg::kPart128 + kk * 512, 256, 256, 3), 1u);
      }
      wgmma_commit();
    };
    // softmax of tile j (in sacc), then l and O rescaled; O must hold every P V up to tile j - 1
    auto softmax = [&](int j) {
      if (j == n_tiles - 1 && last_lim < kWaKeys)
        wa_softmax<true>(sacc, m0, m1, a0, a1, r0, r1, sl2, last_lim, tq);
      else
        wa_softmax<false>(sacc, m0, m1, a0, a1, r0, r1, sl2, kWaKeys, tq);
    };
    auto rescale_pack = [&]() {
      l0 = l0 * a0 + r0;
      l1 = l1 * a1 + r1;
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= (i & 2) ? a1 : a0;
#pragma unroll
      for (int i = 0; i < 8; ++i) o2[i] *= (i & 2) ? a1 : a0;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int q = 0; q < 4; ++q) pa[kk][q] = pack_bf16x2(sacc[8 * kk + 2 * q], sacc[8 * kk + 2 * q + 1]);
    };

    mbar_wait_quiet(q_full, it & 1);
    int s;
    uint32_t ph;
    // ---- tile 0: S_0 alone ----
    wa_ring(n, s, ph);
    mbar_wait_quiet(&k_full[s], ph);
    named_bar_sync(my_bar, 256);
    wgmma_fence();
    issue_s(ka0 + s * Cfg::kTile);
    named_bar_arrive(other_bar, 256);
    wgmma_wait<0>();
    if (t == 0) {
      mbar_arrive(&k_empty[s]);
      if (n_tiles == 1) mbar_arrive(q_empty);
    }
    softmax(0);
    rescale_pack();

    // ---- tile j: S_j and P_{j-1} V_{j-1} issued together, the softmax of j under P_{j-1} V_{j-1} ----
    for (int j = 1; j < n_tiles; ++j) {
      int sk, sv;
      uint32_t phk, phv;
      wa_ring(n + j, sk, phk);
      wa_ring(n + j - 1, sv, phv);
      mbar_wait_quiet(&k_full[sk], phk);
      mbar_wait_quiet(&v_full[sv], phv);
      named_bar_sync(my_bar, 256);
      wgmma_fence();
      issue_s(ka0 + sk * Cfg::kTile);
      issue_pv(va0 + sv * Cfg::kTile);
      named_bar_arrive(other_bar, 256);
      wgmma_wait<1>();
      if (t == 0) {
        mbar_arrive(&k_empty[sk]);
        if (j == n_tiles - 1) mbar_arrive(q_empty);
      }
      softmax(j);
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&v_empty[sv]);
      rescale_pack();
    }

    // ---- the last P V ----
    wa_ring(n + n_tiles - 1, s, ph);
    mbar_wait_quiet(&v_full[s], ph);
    named_bar_sync(my_bar, 256);
    wgmma_fence();
    issue_pv(va0 + s * Cfg::kTile);
    named_bar_arrive(other_bar, 256);
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&v_empty[s]);
    n += n_tiles;

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
  if (c == 0) named_bar_sync(1, 256);
}

template <int D>
static int launch_wgmma(const CUtensorMap* tm, const AttnParams& prm, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_wgmma_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, WaCfg<D>::kSmem);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "attn_wgmma: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "attn_wgmma: SM count: %s", cudaGetErrorString(e));
  // one persistent CTA per SM (or per item when there are fewer)
  const long long items = (long long)((prm.nq + kWaRows - 1) / kWaRows) * prm.H * prm.nb;
  if (items > INT_MAX) return fail(VSB_ERR_UNSUPPORTED, "attn_wgmma: %lld work items", items);
  const int grid = (int)(items < sms ? items : sms);
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
