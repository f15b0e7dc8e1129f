// vsb200 -- flash attention forward for the head dims that attn_wgmma.cu is not laid out for (96: Open-Sora-Plan v1.2.0;
// also 32, 48, 80, 128), FlashAttention-2 schedule on the warp-level tensor cores; and the vsb_attn_flash entry points,
// which send head_dim 64 / 72 to the warpgroup kernel.  Arithmetic contract (both kernels): fp32 scores, softmax scale folded
// into exp2, P rounded to the 16-bit dtype before P V, fp32 accumulation.
//
//   CTA = 8 warps = 128 query rows of one (batch, head); a warp owns 16 rows (one m16 tile), its Q fragments live in registers.
//   Loop over 64-key tiles: K / V tile -> shared memory (cp.async into two buffers: the next tile loads while this one is
//   multiplied; rows padded by 16 bytes: conflict-free ldmatrix; B fragments fetched two tiles per ldmatrix.x4),
//   S = Q K^T (mma.sync m16n8k16, fp32), online softmax on the accumulator fragments (row max / sum across the 4 lanes of a
//   row), P re-packed as A fragments, O += P V (V fragments by ldmatrix.x4.trans).  Rows beyond the sequence are zero (Q) or
//   masked to -inf (keys); V rows beyond the key count are zero so that 0 * garbage cannot produce NaN.
#include "attn_params.cuh"

namespace vsb {


__device__ __forceinline__ void mm_ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mm_ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
// 16-byte asynchronous copy global -> shared; src_bytes = 0 writes zeros (rows past the key count)
__device__ __forceinline__ void mm_cp_async16(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void mm_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void mm_cp_async_wait0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void mm_mma_k16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32." VSB_MMA_T "." VSB_MMA_T ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

constexpr int kMmQ = 128;        // query rows per CTA (8 warps x 16): every K / V tile staged in shared memory serves 128 rows
constexpr int kMmK = 64;         // keys per tile
constexpr int kMmThreads = 256;

template <int D>
__global__ void __launch_bounds__(kMmThreads) attn_mma_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k,
                                                       const bf16* __restrict__ v, long long kv_row_stride,
                                                       long long kv_batch_stride, const __grid_constant__ AttnParams p) {
  constexpr int LD = D + 8;   // smem row pitch in elements (16 bytes of padding)
  constexpr int VPR = D / 8;  // 16-byte vectors per row
  constexpr int KS = D / 16;  // k16 steps of Q K^T
  constexpr int ND = D / 8;   // n8 tiles of O
  static_assert(ND % 2 == 0, "output tiles are loaded in pairs");
  extern __shared__ __align__(16) unsigned char mm_smem[];
  bf16* sQ = reinterpret_cast<bf16*>(mm_smem);
  bf16* sKV = sQ + kMmQ * LD;  // [2 buffers][K tile | V tile]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kMmQ, h = blockIdx.y, b = blockIdx.z;
  const int kv_len = p.has_lens ? p.lens[b] : p.nk;
  const int n_tiles = (kv_len + kMmK - 1) / kMmK;
  const bf16* qb = q + (size_t)b * p.q_batch_stride + (size_t)h * D;
  const bf16* kb = k + (size_t)b * kv_batch_stride + (size_t)h * D;
  const bf16* vb = v + (size_t)b * kv_batch_stride + (size_t)h * D;

  // ---- Q tile -> shared memory (rows past nq are zero), then this warp's A fragments -> registers ----
  for (int i = threadIdx.x; i < kMmQ * VPR; i += kMmThreads) {
    const int r = i / VPR, c = i - r * VPR;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (q0 + r < p.nq) val = *reinterpret_cast<const uint4*>(qb + (size_t)(q0 + r) * p.q_row_stride + c * 8);
    *reinterpret_cast<uint4*>(sQ + r * LD + c * 8) = val;
  }
  __syncthreads();
  uint32_t qf[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) mm_ldsm_x4(qf[ks], sQ + (warp * 16 + (lane & 15)) * LD + ks * 16 + (lane >> 4) * 8);

  float oacc[ND][4];
#pragma unroll
  for (int jd = 0; jd < ND; ++jd) oacc[jd][0] = oacc[jd][1] = oacc[jd][2] = oacc[jd][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g and g + 8 of this warp's tile
  const int t = lane & 3;

  // K / V tiles travel by cp.async into two buffers: tile kt + 1 is in flight while tile kt is multiplied
  auto prefetch = [&](int kt) {
    const int k0 = kt * kMmK;
    bf16* dK = sKV + (size_t)(kt & 1) * 2 * kMmK * LD;
    bf16* dV = dK + kMmK * LD;
    for (int i = threadIdx.x; i < kMmK * VPR; i += kMmThreads) {
      const int r = i / VPR, c = i - r * VPR;
      const bool ok = k0 + r < kv_len;
      const size_t off = (size_t)(ok ? k0 + r : 0) * kv_row_stride + c * 8;  // a valid address even when nothing is read
      mm_cp_async16(dK + r * LD + c * 8, kb + off, ok ? 16 : 0);
      mm_cp_async16(dV + r * LD + c * 8, vb + off, ok ? 16 : 0);
    }
    mm_cp_async_commit();
  };
  prefetch(0);

  for (int kt = 0; kt < n_tiles; ++kt) {
    mm_cp_async_wait0();
    __syncthreads();  // tile kt has landed for every thread; every warp is done with tile kt - 1 (the buffer refilled next)
    if (kt + 1 < n_tiles) prefetch(kt + 1);
    const int k0 = kt * kMmK;
    const bf16* sK = sKV + (size_t)(kt & 1) * 2 * kMmK * LD;
    const bf16* sV = sK + kMmK * LD;

    // ---- S = Q K^T: 16 rows x 64 keys per warp ----
    float sacc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int j = 0; j < 8; j += 2) {  // one ldmatrix.x4 = the B fragments of key tiles j and j + 1
        uint32_t bfr[4];
        mm_ldsm_x4(bfr, sK + ((j + (lane >> 4)) * 8 + (lane & 7)) * LD + ks * 16 + ((lane >> 3) & 1) * 8);
        const uint32_t b0[2] = {bfr[0], bfr[1]}, b1[2] = {bfr[2], bfr[3]};
        mm_mma_k16(sacc[j], qf[ks], b0);
        mm_mma_k16(sacc[j + 1], qf[ks], b1);
      }
    }
    // ---- online softmax (base 2, scale folded); key column of sacc[j][e] = k0 + 8j + 2t + (e & 1) ----
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = k0 + j * 8 + 2 * t + (e & 1);
        const float s = col < kv_len ? sacc[j][e] * p.scale_log2 : -INFINITY;
        sacc[j][e] = s;
        if (e < 2) mx0 = fmaxf(mx0, s); else mx1 = fmaxf(mx1, s);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // every tile holds at least one valid key (n_tiles covers kv_len >= 1), so mx0 / mx1 are finite from the first tile on
    const float a0 = exp2f(m0 - mx0), a1 = exp2f(m1 - mx1);  // exp2(-inf) = 0 on the first tile
    m0 = mx0;
    m1 = mx1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pe = exp2f(sacc[j][e] - (e < 2 ? mx0 : mx1));
        sacc[j][e] = pe;
        if (e < 2) r0 += pe; else r1 += pe;
      }
    }
    r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
    r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
    r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
    r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
    l0 = l0 * a0 + r0;
    l1 = l1 * a1 + r1;
#pragma unroll
    for (int jd = 0; jd < ND; ++jd) {
      oacc[jd][0] *= a0;
      oacc[jd][1] *= a0;
      oacc[jd][2] *= a1;
      oacc[jd][3] *= a1;
    }
    // ---- O += P V: P (16-bit) as the A fragments of four k16 steps over the 64 keys ----
#pragma unroll
    for (int kb4 = 0; kb4 < 4; ++kb4) {
      uint32_t pa[4];
      pa[0] = pack_bf16x2(sacc[2 * kb4][0], sacc[2 * kb4][1]);
      pa[1] = pack_bf16x2(sacc[2 * kb4][2], sacc[2 * kb4][3]);
      pa[2] = pack_bf16x2(sacc[2 * kb4 + 1][0], sacc[2 * kb4 + 1][1]);
      pa[3] = pack_bf16x2(sacc[2 * kb4 + 1][2], sacc[2 * kb4 + 1][3]);
#pragma unroll
      for (int jd = 0; jd < ND; jd += 2) {  // one ldmatrix.x4.trans = the B fragments of output tiles jd and jd + 1
        uint32_t bfr[4];
        mm_ldsm_x4_trans(bfr, sV + (kb4 * 16 + (lane & 15)) * LD + (jd + (lane >> 4)) * 8);
        const uint32_t b0[2] = {bfr[0], bfr[1]}, b1[2] = {bfr[2], bfr[3]};
        mm_mma_k16(oacc[jd], pa, b0);
        mm_mma_k16(oacc[jd + 1], pa, b1);
      }
    }
  }

  // ---- O / l -> out (rows g and g + 8 of the warp's tile; columns 8 jd + 2t, + 1) ----
  const int g = lane >> 2;
  const int row0 = q0 + warp * 16 + g, row1 = row0 + 8;
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  bf16* ob = p.out + (size_t)b * p.out_batch_stride + (size_t)h * D;
#pragma unroll
  for (int jd = 0; jd < ND; ++jd) {
    if (row0 < p.nq)
      *reinterpret_cast<uint32_t*>(ob + (size_t)row0 * p.out_row_stride + jd * 8 + 2 * t) = pack_bf16x2(oacc[jd][0] * i0, oacc[jd][1] * i0);
    if (row1 < p.nq)
      *reinterpret_cast<uint32_t*>(ob + (size_t)row1 * p.out_row_stride + jd * 8 + 2 * t) = pack_bf16x2(oacc[jd][2] * i1, oacc[jd][3] * i1);
  }
}

template <int D>
static int launch_mma(const bf16* q, const bf16* k, const bf16* v, long long kv_row_stride, long long kv_batch_stride,
                      const AttnParams& prm, cudaStream_t st) {
  constexpr size_t smem = (size_t)(kMmQ + 4 * kMmK) * (D + 8) * sizeof(bf16);  // Q + two (K | V) buffers
  static bool attr = false;
  if (!attr && smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(attn_mma_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "attn_mma: smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  dim3 grid((prm.nq + kMmQ - 1) / kMmQ, prm.H, prm.nb);
  attn_mma_kernel<D><<<grid, kMmThreads, smem, st>>>(q, k, v, kv_row_stride, kv_batch_stride, prm);
  return check_launch("attn_mma");
}

static int attn_mma_launch(const bf16* q, const bf16* k, const bf16* v, long long kv_row_stride, long long kv_batch_stride,
                    const AttnParams& prm, int D, cudaStream_t st) {
  switch (D) {
    case 96: return launch_mma<96>(q, k, v, kv_row_stride, kv_batch_stride, prm, st);
    case 128: return launch_mma<128>(q, k, v, kv_row_stride, kv_batch_stride, prm, st);
    case 80: return launch_mma<80>(q, k, v, kv_row_stride, kv_batch_stride, prm, st);
    case 48: return launch_mma<48>(q, k, v, kv_row_stride, kv_batch_stride, prm, st);
    case 32: return launch_mma<32>(q, k, v, kv_row_stride, kv_batch_stride, prm, st);
    default: return fail(VSB_ERR_UNSUPPORTED, "attn_flash: head_dim %d (32, 48, 64, 72, 80, 96, 128)", D);
  }
}

}  // namespace vsb

using namespace vsb;

extern "C" int VSB_API(vsb_attn_flash)(const vsb_bf16* q, const vsb_bf16* k, const vsb_bf16* v, vsb_bf16* out, int nb, int nq,
                              int nk, int H, int D, long long q_row_stride, long long q_batch_stride,
                              long long kv_row_stride, long long kv_batch_stride, const int* host_kv_lens, float scale,
                              void* stream) {
  return VSB_API(vsb_attn_flash_strided)(q, k, v, out, nb, nq, nk, H, D, q_row_stride, q_batch_stride, kv_row_stride,
                                kv_batch_stride, (long long)H * D, (long long)nq * H * D, host_kv_lens, scale, stream);
}

extern "C" int VSB_API(vsb_attn_flash_strided)(const vsb_bf16* q, const vsb_bf16* k, const vsb_bf16* v, vsb_bf16* out, int nb,
                                      int nq, int nk, int H, int D, long long q_row_stride, long long q_batch_stride,
                                      long long kv_row_stride, long long kv_batch_stride, long long out_row_stride,
                                      long long out_batch_stride, const int* host_kv_lens, float scale, void* stream) {
  if (!q || !k || !v || !out || nb <= 0 || nq <= 0 || nk <= 0 || H <= 0) return fail(VSB_ERR_INVALID, "attn_flash: bad args");
  if ((out_row_stride % 8) || (out_batch_stride % 8) || out_row_stride < (long long)H * D)
    return fail(VSB_ERR_UNSUPPORTED, "attn_flash: output strides must be multiples of 8 elements, rows >= H*D apart");
  if ((q_row_stride % 8) || (q_batch_stride % 8) || (kv_row_stride % 8) || (kv_batch_stride % 8) || !aligned16(q) ||
      !aligned16(k) || !aligned16(v) || !aligned16(out))
    return fail(VSB_ERR_UNSUPPORTED, "attn_flash: strides must be multiples of 8 elements and pointers 16B-aligned");
  if (host_kv_lens && nb > kAttnMaxLens)
    return fail(VSB_ERR_UNSUPPORTED, "attn_flash: per-batch key lengths need nb <= %d", kAttnMaxLens);
  if (nb > 65535 || H > 65535) return fail(VSB_ERR_UNSUPPORTED, "attn_flash: grid too large");
  AttnParams prm;
  prm.out = (bf16*)out;
  prm.out_row_stride = out_row_stride;
  prm.out_batch_stride = out_batch_stride;
  prm.q_row_stride = q_row_stride;
  prm.q_batch_stride = q_batch_stride;
  prm.nb = nb;
  prm.nq = nq;
  prm.nk = nk;
  prm.H = H;
  prm.scale_log2 = scale * 1.4426950408889634f;
  prm.has_lens = host_kv_lens ? 1 : 0;
  for (int i = 0; i < kAttnMaxLens; ++i) prm.lens[i] = 0;
  if (host_kv_lens)
    for (int i = 0; i < nb; ++i) {
      if (host_kv_lens[i] < 1 || host_kv_lens[i] > nk) return fail(VSB_ERR_INVALID, "attn_flash: kv_lens[%d]=%d", i, host_kv_lens[i]);
      prm.lens[i] = host_kv_lens[i];
    }
  if (D == 64 || D == 72)
    return attn_wgmma_launch((const bf16*)q, (const bf16*)k, (const bf16*)v, kv_row_stride, kv_batch_stride, prm, D,
                             (cudaStream_t)stream);
  return attn_mma_launch((const bf16*)q, (const bf16*)k, (const bf16*)v, kv_row_stride, kv_batch_stride, prm, D,
                         (cudaStream_t)stream);
}
