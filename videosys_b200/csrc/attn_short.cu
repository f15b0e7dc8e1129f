// vsb200 -- short-sequence attention (n <= 32 tokens): the temporal self-attention of STDiT3 (n = T = 15..20).
//
// FLOPs are negligible (3.7e11 per step at 720p); the kernel should be HBM-bound on one read of q,k,v and one write
// of o.  One warp owns one (sequence, head) at a time; a CTA is 8..16 such warps (one CTA per SM, persistent):
//   1. q,k,v rows (n x D each) -> per-warp shared memory by THREE 5-D TMA box loads ({D, 1 head, 1 sequence, n tokens,
//      1 batch} of the packed token-major qkv) on the warp's own mbarrier: no address arithmetic, no registers, and
//      the load of the NEXT item is in flight as soon as the store of this one has released the Q rows;
//   2. RMSNorm (+ RoPE from a per-block smem table, q scale) in place on q and k, three lanes per row;
//   3. S = Q K^T and O = P V on the warp-level tensor path (mma.sync m16n8k16 / m16n8k8 bf16, fp32 accumulate,
//      ldmatrix fragments; P is re-packed from the S accumulators, FA2 style) -- the sequences are far too short for
//      a warpgroup MMA tile (20 keys against a 64-row x 128-key tile would waste most of the work);
//   4. O staged over the dead Q rows and written by one TMA box store.
// (Staging with per-lane 16-byte loads / stores instead costs 4800 instructions per item, half of them index arithmetic.)
// Rounding follows the reference's eager op order (attentions.py:111-120): bf16(q*scale), bf16(q@k^T),
// fp32 softmax, bf16(probs), bf16(probs@v).
#include <type_traits>

#include "vsb_common.cuh"
#include "vsb_host.h"

namespace vsb {

constexpr int kMaxN = 32;   // the OpenSora instantiation (temporal sequences of 15..20 frames; limit 32)
constexpr int kMaxN2 = 64;  // second instantiation for 33..64 tokens (Vchitect: 40 frames; OpenSora 102..204-frame videos)
constexpr int kMaxWarps = 16;

union Vec8s {
  uint4 u;
  elem2 h[4];
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x2(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x1(uint32_t& r, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x1.shared.b16 {%0}, [%1];" : "=r"(r) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];"
               : "=r"(r[0]), "=r"(r[1])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_k16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32." VSB_MMA_T "." VSB_MMA_T ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma_k8(float (&c)[4], const uint32_t (&a)[2], uint32_t b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32." VSB_MMA_T "." VSB_MMA_T ".f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(b));
}

template <int D, int MAXN = kMaxN>
__global__ void __launch_bounds__(kMaxWarps * 32, 1) attn_short_kernel(
    const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
    const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_o, const bf16* __restrict__ wq,
    const bf16* __restrict__ wk, const float* __restrict__ rope_cos, const float* __restrict__ rope_sin, int n_outer,
    int n_inner, int n, int H, float eps, float scale, int flags) {
  constexpr int VPR = D / 8;        // 16-byte vectors per head row
  constexpr int K16 = D / 16;       // full k16 steps of Q K^T
  constexpr bool K8 = (D % 16) != 0;  // one trailing k8 step (D = 72)
  constexpr int ND = D / 8;         // n8 tiles of the output
  constexpr int NT = MAXN / 8;      // key n8 tiles of a score row
  constexpr int KK = MAXN / 16;     // key k16 steps of P V = query m16 tiles
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem_raw = smem_dyn + ((128u - (smem_u32(smem_dyn) & 127u)) & 127u);  // keeps the shared address space
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwarps = blockDim.x >> 5;
  const int rq = (n + 7) & ~7;  // q / k rows per warp (TMA destinations stay 128-byte aligned: 8 rows = 9 * 128 B)
  // [mbarriers | rope cos | rope sin] (fp32, n x D each, shared by the block) then per warp q[rq] | k[rq] | v[32].
  // ldmatrix of Q rows >= rq runs on into K / V (valid memory, results unused); V rows n..31 are zero.
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  // rope table, one float4 per rotated pair (2i, 2i+1) of a position: (cos[2i], cos[2i+1], sin[2i], sin[2i+1])
  float4* s_rope = reinterpret_cast<float4*>(smem_raw + 128);
  bf16* sq = reinterpret_cast<bf16*>(s_rope + MAXN * (D / 2)) + (size_t)warp * (2 * rq + MAXN) * D;
  bf16* sk = sq + (size_t)rq * D;
  bf16* sv = sk + (size_t)rq * D;
  uint64_t* bar = &bars[warp];
  const bool has_rope = rope_cos != nullptr;
  const bool do_norm = (flags & 1) == 0;   // flag bit 0: q/k arrive un-normalised and stay so (Latte / plain MHA)
  const bool sdpa_math = (flags & 2) != 0; // flag bit 1: F.scaled_dot_product_attention rounding (fp32 scores,
                                           // scale inside the softmax) instead of native_attention's bf16 steps
  if (has_rope) {
    for (int i = threadIdx.x; i < n * (D / 2); i += blockDim.x)
      s_rope[i] = make_float4(rope_cos[2 * i], rope_cos[2 * i + 1], rope_sin[2 * i], rope_sin[2 * i + 1]);
  }
  // zero V's padding rows once (P is 0 there, but 0 * garbage could be NaN); the TMA boxes never touch them
  for (int i = lane; i < (MAXN - n) * VPR; i += 32)
    *reinterpret_cast<uint4*>(sv + (size_t)n * D + i * 8) = make_uint4(0, 0, 0, 0);
  if (lane == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const unsigned total = (unsigned)n_outer * n_inner * H;  // < 2^31 (checked by the launcher)
  const unsigned stride = gridDim.x * nwarps;
  const int nt = (n + 7) >> 3;   // key n8 tiles
  const int kk = (n + 15) >> 4;  // key k16 steps of P V
  const int g = lane >> 2, t = lane & 3;
  const uint32_t tx_bytes = 3u * n * D * sizeof(bf16);
  auto issue_loads = [&](unsigned item) {  // lane 0 only
    const unsigned seq = item / (unsigned)H;
    const int h = int(item - seq * H);
    const int ou = int(seq / (unsigned)n_inner), in = int(seq - (unsigned)ou * n_inner);
    mbar_arrive_expect_tx(bar, tx_bytes);
    tma_load_5d(&tm_q, bar, sq, 0, h, in, 0, ou);
    tma_load_5d(&tm_k, bar, sk, 0, h, in, 0, ou);
    tma_load_5d(&tm_v, bar, sv, 0, h, in, 0, ou);
  };
  unsigned item = blockIdx.x * nwarps + warp;
  if (item < total && lane == 0) issue_loads(item);
  uint32_t phase = 0;

  for (; item < total; item += stride) {
    // ---- 1. this item's q,k,v rows have landed (the loads were issued one iteration ago) ----
    mbar_wait(bar, phase);
    phase ^= 1;

    if (n == 1) {  // attentions.py:65-66: x = v
      for (int c = lane; c < VPR; c += 32)
        *reinterpret_cast<uint4*>(sq + c * 8) = *reinterpret_cast<const uint4*>(sv + c * 8);
    } else {
    // ---- 2. RMSNorm (+RoPE, q scale) in place.  LPR lanes share one row (CPL 16-byte chunks each); the n query rows,
    //         then the n key rows, are walked 32/LPR at a time (two instantiations: the q-only scale is compile-time and a
    //         pass never mixes q and k rows, so no lane diverges); the sum of squares crosses lanes by shuffle ----
    if (do_norm || has_rope || !sdpa_math) {
      constexpr int LPR = (D == 72) ? 3 : 2;  // lanes per row
      constexpr int CPL = VPR / LPR;          // chunks per lane (3 or 4)
      constexpr int RPP = 32 / LPR;           // rows per pass
      const int gi = lane / LPR, part = lane - gi * LPR;
      const int gbase = (gi < RPP ? gi : 0) * LPR;
      auto norm_rows = [&](auto is_q_c) {
        constexpr bool kIsQ = decltype(is_q_c)::value;
        const bool scale_q = kIsQ && !sdpa_math;  // q = bf16(q * scale)  (attentions.py:113)
        if (!do_norm && !has_rope && !scale_q) return;
        const bf16* wrow = (kIsQ ? wq : wk) + part * CPL * 8;
        for (int r0 = 0; r0 < n; r0 += RPP) {
          const int r = r0 + gi;
          const bool act = (gi < RPP) && (r < n);
          bf16* rowp = (kIsQ ? sq : sk) + (act ? r : 0) * D + part * CPL * 8;
          Vec8s v[CPL];
          float ss = 0.f;
          if (act) {
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
              v[c].u = *reinterpret_cast<const uint4*>(rowp + c * 8);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 f = e2_to_float2(v[c].h[j]);
                ss = fmaf(f.x, f.x, ss);
                ss = fmaf(f.y, f.y, ss);
              }
            }
          }
          float tot = 0.f;
#pragma unroll
          for (int i = 0; i < LPR; ++i) tot += __shfl_sync(0xffffffffu, ss, gbase + i);
          if (act) {
            const float rs = do_norm ? rsqrtf(tot / (float)D + eps) : 1.f;
            const float4* rp = s_rope + (size_t)r * (D / 2) + part * CPL * 4;
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
              Vec8s w, o;
              w.u = do_norm ? __ldg(reinterpret_cast<const uint4*>(wrow + c * 8)) : make_uint4(0, 0, 0, 0);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 f = e2_to_float2(v[c].h[j]);
                // normalization.py:28-33: h = bf16(x*rstd); y = bf16(w*h)
                elem2 y2 = do_norm ? __hmul2_rn(w.h[j], floats_to_e2(f.x * rs, f.y * rs)) : v[c].h[j];
                if (has_rope || scale_q) {
                  float2 y = e2_to_float2(y2);
                  if (has_rope) {
                    // rotate_queries_or_keys: t*cos + rotate_half(t)*sin in fp32, pairs (2i, 2i+1): rot = (-x2, x1)
                    const float4 cs = rp[c * 4 + j];
                    const float o0 = __fadd_rn(__fmul_rn(y.x, cs.x), __fmul_rn(-y.y, cs.z));
                    const float o1 = __fadd_rn(__fmul_rn(y.y, cs.y), __fmul_rn(y.x, cs.w));
                    y = scale_q ? e2_to_float2(floats_to_e2(o0, o1)) : make_float2(o0, o1);
                  }
                  if (scale_q) {
                    y.x *= scale;
                    y.y *= scale;
                  }
                  y2 = floats_to_e2(y.x, y.y);
                }
                o.h[j] = y2;
              }
              *reinterpret_cast<uint4*>(rowp + c * 8) = o.u;
            }
          }
        }
      };
      norm_rows(std::true_type{});
      norm_rows(std::false_type{});
    }
    __syncwarp();

    // ---- 3. S = Q K^T (bf16 out), softmax fp32, P bf16, O = P V ----
#pragma unroll 1
    for (int mt = 0; mt < KK; ++mt) {
      if (mt * 16 >= n) break;
      float sacc[NT][4];
#pragma unroll
      for (int j = 0; j < NT; ++j) sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
      const bf16* qa = sq + (size_t)(mt * 16 + (lane & 15)) * D + (lane >> 4) * 8;
#pragma unroll
      for (int ks = 0; ks < K16; ++ks) {
        uint32_t a[4];
        ldsm_x4(a, qa + ks * 16);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          if (j < nt) {
            uint32_t b[2];
            ldsm_x2(b, sk + (size_t)(j * 8 + (lane & 7)) * D + ks * 16 + ((lane >> 3) & 1) * 8);
            mma_k16(sacc[j], a, b);
          }
        }
      }
      if (K8) {
        uint32_t a[2];
        ldsm_x2(a, sq + (size_t)(mt * 16 + (lane & 15)) * D + K16 * 16);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          if (j < nt) {
            uint32_t b;
            ldsm_x1(b, sk + (size_t)(j * 8 + (lane & 7)) * D + K16 * 16);
            mma_k8(sacc[j], a, b);
          }
        }
      }
      // rows g (c0,c1) and g+8 (c2,c3) of this m-tile; columns 8j + 2t, +1
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < NT; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = j * 8 + 2 * t + (e & 1);
          // native_attention: bf16 matmul output; SDPA: fp32 scores scaled inside the softmax; pad keys masked
          const float v = (j < nt && col < n) ? (sdpa_math ? sacc[j][e] * scale : rbf(sacc[j][e])) : -INFINITY;
          sacc[j][e] = v;
          if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      float d0 = 0.f, d1 = 0.f;
      const bool rows_hi = mt * 16 + 8 < n;  // rows g + 8 of this m-tile exist (warp-uniform): else their P stays unused
#pragma unroll
      for (int j = 0; j < NT; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // exp(-inf) = 0 for masked keys; key tiles beyond the sequence and absent rows skip the exponential
          const float p = (j < nt && (e < 2 || rows_hi)) ? expf(sacc[j][e] - (e < 2 ? mx0 : mx1)) : 0.f;
          sacc[j][e] = p;
          if (e < 2) d0 += p; else d1 += p;
        }
      }
      d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
      d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
      d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
      d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
      // P (bf16) as A fragments of the two k16 steps
      // one correctly rounded reciprocal per row, then a multiply (vs p / d: <= 1.5 fp32 ulp before the bf16 rounding of P)
      const float i0 = 1.f / d0, i1 = rows_hi ? 1.f / d1 : 0.f;
      uint32_t pa[KK][4];
#pragma unroll
      for (int kb = 0; kb < KK; ++kb) {
        pa[kb][0] = pack_bf16x2(sacc[2 * kb][0] * i0, sacc[2 * kb][1] * i0);
        pa[kb][1] = pack_bf16x2(sacc[2 * kb][2] * i1, sacc[2 * kb][3] * i1);
        pa[kb][2] = pack_bf16x2(sacc[2 * kb + 1][0] * i0, sacc[2 * kb + 1][1] * i0);
        pa[kb][3] = pack_bf16x2(sacc[2 * kb + 1][2] * i1, sacc[2 * kb + 1][3] * i1);
      }
      float oacc[ND][4];
#pragma unroll
      for (int jd = 0; jd < ND; ++jd) oacc[jd][0] = oacc[jd][1] = oacc[jd][2] = oacc[jd][3] = 0.f;
#pragma unroll
      for (int kb = 0; kb < KK; ++kb) {
        if (kb < kk) {
#pragma unroll
          for (int jd = 0; jd < ND; ++jd) {
            uint32_t b[2];
            ldsm_x2_trans(b, sv + (size_t)(kb * 16 + (lane & 15)) * D + jd * 8);
            mma_k16(oacc[jd], pa[kb], b);
          }
        }
      }
      // ---- 4. O (bf16) -> smem over this m-tile's Q rows (Q is dead for these rows; rows >= n are not stored) ----
      __syncwarp();
      const int r0 = mt * 16 + g, r1 = r0 + 8;
#pragma unroll
      for (int jd = 0; jd < ND; ++jd) {
        if (r0 < n) *reinterpret_cast<uint32_t*>(sq + (size_t)r0 * D + jd * 8 + 2 * t) = pack_bf16x2(oacc[jd][0], oacc[jd][1]);
        if (r1 < n) *reinterpret_cast<uint32_t*>(sq + (size_t)r1 * D + jd * 8 + 2 * t) = pack_bf16x2(oacc[jd][2], oacc[jd][3]);
      }
    }
    }
    // ---- 5. one TMA box store of the n x D output rows; then the next item's loads (K and V are dead after the last
    //         ldmatrix above, Q's rows once the store has read them) ----
    fence_proxy_async_smem();  // my generic-proxy writes of O -> visible to the async proxy
    __syncwarp();
    if (lane == 0) {
      const unsigned seq = item / (unsigned)H;
      const int ou = int(seq / (unsigned)n_inner);
      tma_store_5d(&tm_o, sq, 0, int(item - seq * H), int(seq - (unsigned)ou * n_inner), 0, ou);
      tma_store_commit();
      tma_store_wait_read0();
      if (item + stride < total) issue_loads(item + stride);
    }
    __syncwarp();
  }
  if (lane == 0) tma_store_wait0();
}

template <int D, int MAXN>
static int launch_short(const bf16* qkv, bf16* out, const bf16* wq, const bf16* wk, const float* rc, const float* rs,
                        int n_outer, int n_inner, long long os, long long is, long long ts, int n, int H, float eps,
                        float scale, int flags, cudaStream_t st) {
  const int C = H * D;
  const int rq = (n + 7) & ~7;
  const size_t fixed = 128 + 128 + 2 * MAXN * D * sizeof(float);  // alignment slack, mbarriers, rope tables
  const size_t per_warp = (size_t)(2 * rq + MAXN) * D * sizeof(bf16);
  int warps = int((227 * 1024 - fixed) / per_warp);
  warps = warps >= kMaxWarps ? kMaxWarps : (warps & ~3);
  if (warps < 4) return fail(VSB_ERR_UNSUPPORTED, "attn_short: shared memory");
  const size_t smem = fixed + warps * per_warp;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_short_kernel<D, MAXN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "attn_short: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  // 5-D views {d, head, inner sequence index, token of the sequence, outer sequence index}; box = one head of one
  // sequence: {D, 1, 1, n, 1}.  q / k / v are the three column blocks of the packed qkv rows.
  CUtensorMap tm[4];
  const unsigned long long dims[5] = {(unsigned long long)D, (unsigned long long)H, (unsigned long long)n_inner,
                                      (unsigned long long)n, (unsigned long long)n_outer};
  const unsigned box[5] = {(unsigned)D, 1, 1, (unsigned)n, 1};
  for (int i = 0; i < 4; ++i) {
    const unsigned long long row = (unsigned long long)(i < 3 ? 3 * C : C) * sizeof(bf16);
    // a dimension of extent 1 is never stepped: give it a valid (non-zero, 16-byte multiple) stride
    const unsigned long long str[4] = {(unsigned long long)D * sizeof(bf16),
                                       (unsigned long long)(n_inner > 1 ? is : 1) * row,
                                       (unsigned long long)(n > 1 ? ts : 1) * row,
                                       (unsigned long long)(n_outer > 1 ? os : 1) * row};
    const void* base = i < 3 ? (const void*)(qkv + (size_t)i * C) : (const void*)out;
    int rc2 = make_tmap_bf16(&tm[i], base, 5, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc2) return rc2;
  }
  const long long total = (long long)n_outer * n_inner * H;
  if (total >= (1ll << 31)) return fail(VSB_ERR_UNSUPPORTED, "attn_short: %lld (sequence, head) items", total);
  long long blocks = (total + warps - 1) / warps;
  if (blocks > num_sms()) blocks = num_sms();  // persistent: one CTA per SM, each warp walks its share of the items
  attn_short_kernel<D, MAXN><<<(int)blocks, warps * 32, smem, st>>>(tm[0], tm[1], tm[2], tm[3], wq, wk, rc, rs, n_outer, n_inner,
                                                               n, H, eps, scale, flags);
  return check_launch("attn_short");
}

}  // namespace vsb

using namespace vsb;

extern "C" int VSB_API(vsb_attn_short)(const vsb_bf16* qkv, vsb_bf16* out, const vsb_bf16* wq, const vsb_bf16* wk,
                              const float* rope_cos, const float* rope_sin, int n_outer, int n_inner,
                              long long outer_stride, long long inner_stride, long long tok_stride, int n, int H,
                              int D, float eps, float scale, int flags, void* stream) {
  if (!qkv || !out || n_outer <= 0 || n_inner <= 0 || n <= 0 || H <= 0)
    return fail(VSB_ERR_INVALID, "attn_short: bad args");
  if ((flags & 1) == 0 && (!wq || !wk)) return fail(VSB_ERR_INVALID, "attn_short: q/k norm weights required (or flag 1)");
  if (n > kMaxN2) return fail(VSB_ERR_UNSUPPORTED, "attn_short: n=%d > %d (use vsb_attn_flash)", n, kMaxN2);
  if ((rope_cos == nullptr) != (rope_sin == nullptr)) return fail(VSB_ERR_INVALID, "attn_short: rope tables");
  if (!aligned16(qkv) || !aligned16(out)) return fail(VSB_ERR_UNSUPPORTED, "attn_short: alignment");
  cudaStream_t st = (cudaStream_t)stream;
#define VSB_SHORT(DD, MM)                                                                                                  \
  return launch_short<DD, MM>((const bf16*)qkv, (bf16*)out, (const bf16*)wq, (const bf16*)wk, rope_cos, rope_sin, n_outer, \
                              n_inner, outer_stride, inner_stride, tok_stride, n, H, eps, scale, flags, st)
  if (D == 72) {
    if (n <= kMaxN) VSB_SHORT(72, kMaxN);
    VSB_SHORT(72, kMaxN2);
  }
  if (D == 64) {
    if (n <= kMaxN) VSB_SHORT(64, kMaxN);
    VSB_SHORT(64, kMaxN2);
  }
#undef VSB_SHORT
  return fail(VSB_ERR_UNSUPPORTED, "attn_short: head_dim %d (72 or 64 only)", D);
}
