/* vsb200.h -- C-ABI of libvsb200.so: the H100-native (sm_90a) kernels behind the VideoSys DiT denoising hot path.
 *
 * The reference (NUS-HPC-AI-Lab/VideoSys @ 4cce4778) is pure Python and exposes no FFI/plugin boundary
 * (SURVEY.md section 8b); this header is the boundary a maintainer binds with ctypes (INTEGRATION.md shows the
 * stub).  Each entry cites the reference code it replaces (paths relative to the reference's videosys/ package).
 *
 * Conventions
 *   - plain pointers and sizes; every pointer is DEVICE memory unless named host_*; bf16 = uint16 storage.
 *   - all kernels are asynchronous on `stream` (a cudaStream_t passed as void*); no allocation, no host sync.
 *   - return 0 on success, a negative vsb_status otherwise; vsb_last_error() gives the text (per host thread).
 *   - no CPU fallback and no multi-backend dispatch: unsupported shape/alignment = VSB_ERR_UNSUPPORTED.
 *   - one process per GPU; entries are not re-entrant per device (same as one torch stream).
 */
#ifndef VSB200_H_
#define VSB200_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  VSB_OK = 0,
  VSB_ERR_INVALID = -1,     /* bad argument (null pointer, non-positive size) */
  VSB_ERR_UNSUPPORTED = -2, /* shape / alignment outside what the sm_90a kernels handle */
  VSB_ERR_CUDA = -3,        /* CUDA runtime / driver error (text in vsb_last_error) */
  VSB_ERR_NO_DEVICE = -4    /* no sm_90 device: the library never falls back to the CPU */
} vsb_status;

typedef uint16_t vsb_bf16;

int vsb_version(void);
const char* vsb_last_error(void);
/* Checks that `device` is compute capability 9.0 and loads cuTensorMapEncodeTiled. */
int vsb_init(int device);
/* Number of kernels this library has launched since load (all entries); bench.py reports the delta. */
unsigned long long vsb_launch_count(void);
/* Encoded TMA tensor maps are cached by (base, shape, strides, box, swizzle): which = 0 -> hits, 1 -> misses (host
 * cuTensorMapEncodeTiled calls actually made).  Option "tmap_cache" (default 1) turns the cache off. */
unsigned long long vsb_tmap_cache_stats(int which);
/* Run-time options.
 *   "tmap_cache" (default 1): cache of encoded TMA tensor maps. */
int vsb_set_option(const char* name, int value);

/* ---- AdaLN: LayerNorm(eps, no affine) -> x*(1+scale)+shift with per-frame t / t0 select --------------------
 * replaces norm1/norm2 + t2i_modulate + t_mask_select: models/transformers/open_sora_transformer_3d.py:47-48,
 * :152-160, :196-200, :260-264.  Rounds to bf16 at the same points as the eager chain (after LN, after 1+scale,
 * after the multiply, after the add).
 *   x, out   [B, T, S, C] bf16 (out may alias x); C % 8 == 0, C <= 3072
 *   mod      [2, B, 6, C] bf16: mod[0] = scale_shift_table + t, mod[1] = table + t0 (see vsb_modulation_table)
 *   x_mask   [B, T] uint8 (nonzero -> use mod[0]) or NULL (always mod[0])
 *   shift_row/scale_row: which of the 6 rows (0,1 for attention; 3,4 for the MLP) */
int vsb_ln_modulate(const vsb_bf16* x, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask, int shift_row,
                    int scale_row, int B, int T, int S, int C, float eps, void* stream);

/* Same with nn.LayerNorm(C, eps, elementwise_affine=True) in front (gamma, beta [C]): the video / text streams of
 * CogVideoXLayerNormZero (models/modules/normalization.py:51-57): mod = the 6-way chunk of linear(silu(temb)) laid
 * out as [1 or 2, B, 6, C]; rows (0,1) video, (3,4) text. */
int vsb_ln_modulate_affine(const vsb_bf16* x, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask,
                           const vsb_bf16* gamma, const vsb_bf16* beta, int shift_row, int scale_row, int B, int T, int S,
                           int C, float eps, void* stream);

/* mod[0,b,r,:] = bf16(table[r,:] + t[b, r*C:(r+1)*C]); mod[1] likewise from t0 (t0 may be NULL -> mod[1]=mod[0]).
 * replaces open_sora_transformer_3d.py:177-184.  table [6,C], t/t0 [B,6C], mod [2,B,6,C]. */
int vsb_modulation_table(const vsb_bf16* table, const vsb_bf16* t, const vsb_bf16* t0, vsb_bf16* mod, int B, int C,
                         int rows, void* stream);

/* ---- patch embedding of the latent + position embedding + sequence-parallel split ------------------------------
 * replaces open_sora_transformer_3d.py:568-572 (x_embedder: Conv3d kernel = stride = (1, ph, pw); rearrange; + pos_emb)
 * and :577 (split_sequence along the patch axis); the same for Latte's 2-D PatchEmbed (latte_transformer_3d.py:1245).
 *   z    latent, element (b, c, t, y, x) at b*batch_stride + c*chan_stride + t*frame_stride + y*W + x (elements);
 *        rows / columns beyond H / W read as zero (the reference pads to the patch grid)
 *   w    [C, Cin*ph*pw] (= conv.weight storage, taps ordered (c, ky, kx)); bias [C] or NULL; pos [S_total, C] or NULL
 *   out  [B, T, S_local, C]: patch columns s0 .. s0+S_local-1 of every (batch, frame); columns >= S_total are zero
 * Rounds like the eager chain: conv (fp32 accumulate) -> bf16, + bias -> bf16, + pos -> bf16.
 * Returns 1 without launching unless Cin*ph*pw == 16, C % 8 == 0 and C <= 2048. */
int vsb_patch_embed(const vsb_bf16* z, const vsb_bf16* w, const vsb_bf16* bias, const vsb_bf16* pos, vsb_bf16* out, int B,
                    int Cin, int T, int H, int W, long long batch_stride, long long chan_stride, long long frame_stride,
                    int ph, int pw, int C, int s0, int S_local, void* stream);

/* ---- gate * y (+ per-frame select) + residual, optional PAB cache write ---------------------------------------
 * replaces open_sora_transformer_3d.py:219-228 and :270-284.  gated = bf16(gate*y); out = bf16(x + gated).
 *   cache_out (nullable): receives `gated` (what the reference keeps as last_attn, :224-225). */
int vsb_gate_residual(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, vsb_bf16* cache_out, const vsb_bf16* mod,
                      const uint8_t* x_mask, int gate_row, int B, int T, int S, int C, void* stream);

/* out = bf16(x + y) over n elements: cross-attention residual (:240) and PAB replay of a cached tensor
 * (:192-193 -> :228, :234-235).  One coalesced pass: 2 reads + 1 write. */
int vsb_residual_add(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, size_t n, void* stream);

/* ---- per-head RMSNorm of q and k inside a packed qkv buffer (spatial blocks, no RoPE) -------------------------
 * replaces LlamaRMSNorm on q,k: models/modules/normalization.py:28-33 via attentions.py:75.
 *   qkv [rows, 3, H, D] bf16, normalised in place for the q and k thirds; wq, wk [D] bf16. */
int vsb_qk_rmsnorm(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* wk, size_t rows, int H, int D, float eps,
                   void* stream);
/* Same, followed by RoPE on q and k (attentions.py:76-78 -> rotary_embedding_torch rotate_queries_or_keys: interleaved
 * pairs, fp32 math, cast back): the pre-pass of TEMPORAL attention over >= 30 frames, where the reference leaves
 * native_attention for F.scaled_dot_product_attention (attentions.py:95-100).  rope_cos / rope_sin [pos_mod, D] fp32;
 * token row r sits at position (r / pos_div) % pos_mod
 * (token-major [B, T, S] activation: pos_div = S, pos_mod = T).
 * wq == wk == NULL: RoPE only (q / k stay un-normalised): the temporal attention of Vchitect beyond 64 frames
 * (attentions.py:688-701 apply_rotary_emb, complex multiply on the same interleaved pairs; no q/k norm). */
int vsb_qk_rmsnorm_rope(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* wk, size_t rows, int H, int D, float eps,
                        const float* rope_cos, const float* rope_sin, int pos_div, int pos_mod, void* stream);

/* Half-rotation RoPE on q and k in place (Open-Sora-Plan RoPE1D / RoPE2D / RoPE3D:
 * models/transformers/open_sora_plan_v110_transformer_3d.py:136-252 applied :1217-1232,
 * open_sora_plan_v120_transformer_3d.py:63-118 applied :921-925): every head is cut into D / (2*half) blocks (one per
 * position axis), inside a block out[d] = x[d]*cos + rotate_half(x)[d]*sin with rotate_half = (-second half, first half),
 * each product and the sum rounded to the 16-bit dtype as the reference's eager ops do.
 *   rope_cos, rope_sin_signed [pos_mod, D] fp32: row p holds, for every channel of a head, the reference's 16-bit cos / sin
 *   of that channel's axis position (sin negated on the first half of each block); token row r uses table row
 *   (r / pos_div) % pos_mod.  half even, D a multiple of 2*half. */
int vsb_qk_rope_halves(vsb_bf16* qkv, size_t rows, int H, int D, int half, const float* rope_cos,
                       const float* rope_sin_signed, int pos_div, int pos_mod, void* stream);
/* Per-head LayerNorm(D, eps, affine) of q and k in place (CogVideoX: diffusers Attention(qk_norm="layer_norm"),
 * models/transformers/cogvideox_transformer_3d.py:241-242 -> processor :130-133).  wq,bq,wk,bk [D] bf16. */
int vsb_qk_layernorm(vsb_bf16* qkv, const vsb_bf16* wq, const vsb_bf16* bq, const vsb_bf16* wk, const vsb_bf16* bk,
                     size_t rows, int H, int D, float eps, void* stream);

/* ---- short-sequence attention (n < 30): RMSNorm(q,k) -> [RoPE] -> native_attention, one warp per (seq, head) --
 * replaces OpenSoraAttention.forward's N<30 path: attentions.py:59-78,95-97,111-120 with the reference's op order
 * (bf16(q*scale), bf16 scores, fp32 softmax, bf16 probs).  Reads the packed qkv of the token-major activation
 * without any rearrange: sequence (o,i) token j lives at row o*outer_stride + i*inner_stride + j*tok_stride.
 *   qkv [rows,3,H,D] bf16; out [rows,H*D] bf16; rope_cos/rope_sin [n, D] fp32 or NULL; n == 1 copies v (:65-66).
 *   n <= 64: two instantiations, up to 32 tokens (OpenSora's 15 .. 20 frames) and 33 .. 64 (Vchitect's 40-frame temporal
 *   attention, models/modules/attentions.py:707-768, with flags = 3 and RoPE tables from freqs_cis).
 *   flags: bit 0 = no q/k RMSNorm (wq, wk may be NULL): diffusers Attention as used by Latte
 *          (models/transformers/latte_transformer_3d.py:259-268,611-619); bit 1 = SDPA rounding (fp32 scores, scale
 *          inside the softmax) instead of native_attention's bf16 intermediate steps. */
int vsb_attn_short(const vsb_bf16* qkv, vsb_bf16* out, const vsb_bf16* wq, const vsb_bf16* wk, const float* rope_cos,
                   const float* rope_sin, int n_outer, int n_inner, long long outer_stride, long long inner_stride,
                   long long tok_stride, int n, int H, int D, float eps, float scale, int flags, void* stream);

/* ---- GEMM on wgmma: out[M,N] = act(A[M,K] @ W[N,K]^T + bias[N]) ---------------------------------------------
 * replaces every nn.Linear on the path (attentions.py:59,107,156-157; timm Mlp fc1/fc2) and the tanh-GELU between
 * fc1 and fc2 (models/modules/activations.py:3).  bf16 in, fp32 accumulate in registers, bf16 out.
 *   act: 0 = none, 1 = gelu_tanh applied to bf16(acc+bias) (the eager rounding point), 2 = exact (erf) GELU applied to
 *   bf16(acc+bias): F.gelu after project_in of Open-Sora-Plan v1.2.0's FeedForward_Conv2d
 *   (models/transformers/open_sora_plan_v120_transformer_3d.py:1080-1082).
 *   Requirements: K % 8 == 0, N % 8 == 0, 16-byte aligned pointers, row-major contiguous. */
int vsb_gemm_bias_act(const vsb_bf16* A, const vsb_bf16* W, const vsb_bf16* bias, vsb_bf16* out, int M, int N, int K,
                      int act, void* stream);

/* Same GEMM with the residual branch of the block fused into the epilogue:
 *   y = bf16(A @ W^T + bias);  g = gate_row >= 0 ? bf16(gate * y) : y;  out = bf16(resid + g)
 * gate = mod[sel(b,t), b, gate_row, :] with the per-frame t/t0 select of x_mask (as in vsb_gate_residual); M == B*T*S.
 * replaces proj/fc2 Linear + open_sora_transformer_3d.py:219-228,:270-284 (gate_row 2 / 5) and cross proj + :240
 * (gate_row -1).  out may alias resid.  Same requirements as vsb_gemm_bias_act. */
int vsb_gemm_bias_residual(const vsb_bf16* A, const vsb_bf16* W, const vsb_bf16* bias, const vsb_bf16* resid,
                           vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int M, int N, int K,
                           int B, int T, int S, void* stream);

/* Name of the kernel instance the two GEMM entries above launch for a shape, e.g. "gemm_wide_kernel<2>" (the same for
 * bf16 and fp16): act as in vsb_gemm_bias_act, residual != 0 for vsb_gemm_bias_residual (act 0).  "" for bad arguments.
 * Benchmarks label their rows with it. */
const char* vsb_gemm_kernel_name(int M, int N, int K, int act, int residual);

/* ---- FP8 (e4m3) Linears: quantized activations and weights, fp32 scales -------------------------------------------
 * The quantization rule, one definition for the kernels below and the tests' torch restatement: a row x of 16-bit values
 * (an activation row, or a weight's output channel) has amax = max |x|.  amax > 0: q = e4m3_rn(x * s) with
 * s = 448 / amax, both fp32 round-to-nearest-even operations (PTX cvt.rn.satfinite.e4m3x2.f32; |x * s| <= 448 rounds
 * inside the finite range, where torch's x.to(torch.float8_e4m3fn) gives the same codes), scale = amax / 448 (fp32).
 * amax == 0: all-zero codes, scale = 1.
 *
 * vsb_quant_rows_fp8: x [M, K] 16-bit -> q [M, K] e4m3 codes, scale [M] fp32.  K % 8 == 0, K <= 4608. */
int vsb_quant_rows_fp8(const vsb_bf16* x, uint8_t* q, float* scale, int M, int K, void* stream);

/* vsb_ln_modulate whose output row goes out quantized: q [B*T*S, C] e4m3 and scale [B*T*S] fp32 are exactly
 * vsb_quant_rows_fp8 of the 16-bit rows vsb_ln_modulate would write (the amax is over the rounded outputs). */
int vsb_ln_modulate_fp8(const vsb_bf16* x, uint8_t* q, float* scale, const vsb_bf16* mod, const uint8_t* x_mask,
                        int shift_row, int scale_row, int B, int T, int S, int C, float eps, void* stream);

/* GEMM on e4m3 operands: A [M, K] codes with per-row scales sa [M], W [N, K] codes with per-output-channel scales sw [N].
 *   y = bf16(acc * sa[m] * sw[n] + bias[n]), evaluated as fmaf(acc * sa[m], sw[n], bias[n]) in fp32, where acc is the
 *   fp32 sum of the e4m3 products: the tensor cores sum 128 of K at a time into a fresh fragment, which is added to fp32
 *   registers.  From y on, act (0 none, 1 tanh-GELU) as in vsb_gemm_bias_act, and the gate + select + residual epilogue
 *   of vsb_gemm_bias_residual (same arguments) in vsb_gemm_fp8_bias_residual.
 *   Requirements: K % 16 == 0 (16-byte rows of codes), N % 8 == 0, 16-byte aligned A, W, sw, out and resid;
 *   otherwise VSB_ERR_UNSUPPORTED. */
int vsb_gemm_fp8_bias_act(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw, const vsb_bf16* bias,
                          vsb_bf16* out, int M, int N, int K, int act, void* stream);
int vsb_gemm_fp8_bias_residual(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw, const vsb_bf16* bias,
                               const vsb_bf16* resid, vsb_bf16* out, const vsb_bf16* mod, const uint8_t* x_mask,
                               int gate_row, int M, int N, int K, int B, int T, int S, void* stream);
/* The kernel instance the two fp8 GEMM entries launch, e.g. "gemm_wide_kernel<fp8, 2>"; as vsb_gemm_kernel_name. */
const char* vsb_gemm_fp8_kernel_name(int M, int N, int K, int act, int residual);

/* ---- flash attention (spatial self-attention and text cross-attention) -------------------------------
 * replaces F.scaled_dot_product_attention at attentions.py:100 and :268 (bool key mask = per-batch key count).
 * q/k/v are strided views: element (b, n, h, d) at base + b*batch_stride + n*row_stride + h*D + d (strides in
 * elements, multiples of 8).  out [nb, nq, H*D] contiguous.  kv_lens (host int array, nullable) = valid keys per
 * batch (<= nk, nb <= 64 when given).  head_dim 64 / 72 run on the warpgroup tensor cores (TMA + wgmma,
 * csrc/attn_wgmma.cu); 32, 48, 80, 96 (Open-Sora-Plan v1.2.0, open_sora_plan_v120_transformer_3d.py:929-931) and 128 on
 * the warp-level tensor cores (mma.sync, FlashAttention-2 schedule, csrc/attn_mma.cu). */
int vsb_attn_flash(const vsb_bf16* q, const vsb_bf16* k, const vsb_bf16* v, vsb_bf16* out, int nb, int nq, int nk,
                   int H, int D, long long q_row_stride, long long q_batch_stride, long long kv_row_stride,
                   long long kv_batch_stride, const int* host_kv_lens, float scale, void* stream);
/* Same with a strided OUTPUT view: element (b, n, h, d) at out + b*out_batch_stride + n*out_row_stride + h*D + d.
 * Temporal attention over >= 30 frames runs on the token-major activation with batch = patch s, row = frame t:
 * q/k/v row stride S*3C, batch stride 3C; out row stride S*C, batch stride C (one call per CFG sample). */
int vsb_attn_flash_strided(const vsb_bf16* q, const vsb_bf16* k, const vsb_bf16* v, vsb_bf16* out, int nb, int nq, int nk,
                           int H, int D, long long q_row_stride, long long q_batch_stride, long long kv_row_stride,
                           long long kv_batch_stride, long long out_row_stride, long long out_batch_stride,
                           const int* host_kv_lens, float scale, void* stream);

/* ---- Open-Sora-Plan v1.2.0 conv down-sampler variants (downsampler = "k333_s222" / "k33_s22") ------------------------
 * Depth-wise attention down-sampler: replaces DownSampler3d / DownSampler2d.forward
 * (models/transformers/open_sora_plan_v120_transformer_3d.py:735-834, called at :872-874): rearrange to NCDHW, depth-wise
 * Conv3d / Conv2d (zero "same" padding, bias) + shortcut, rearrange into dt*dh*dw interleaved sub-grids.
 *   x      [B, T*H*W, C] token-major;  w_taps [kt*kh*kw, C] (conv.weight [C, 1, kt, kh, kw] transposed tap-major);  bias [C]
 *   out    [(B dt dh dw), (T/dt H/dh W/dw), C]: token (b, t, h, w) lands in sub-grid ((b*dt + t%dt)*dh + h%dh)*dw + w%dw
 *          at position ((t/dt)*(H/dh) + h/dh)*(W/dw) + w/dw.  Rounds as torch's eager GPU chain: bf16(conv), + bias,
 *          + x, each rounded to 16 bits.
 *   kt in {1, 3}, kh and kw in {3, 5}; dt, dh, dw divide T, H, W.  Otherwise VSB_ERR_UNSUPPORTED / VSB_ERR_INVALID. */
int vsb_dwconv_shuffle(const vsb_bf16* x, const vsb_bf16* w_taps, const vsb_bf16* bias, vsb_bf16* out, int B, int T, int H,
                       int W, int C, int kt, int kh, int kw, int dt, int dh, int dw, void* stream);
/* DownSampler.reverse (:787-790, :829-833, applied at :959-960) fused into the gate + residual of the attention branch:
 *   out[b, (t h w)] = bf16(x + bf16(gate * y[sub-grid row of (b, t, h, w)])), gate = mod[0, b, gate_row, :];
 *   x, out [B, T*H*W, C] (out may alias x); y [(B dt dh dw), (T/dt H/dh W/dw), C] as vsb_dwconv_shuffle lays it out. */
int vsb_gate_residual_unshuffle(const vsb_bf16* x, const vsb_bf16* y, vsb_bf16* out, const vsb_bf16* mod, int gate_row, int B,
                                int T, int H, int W, int C, int dt, int dh, int dw, void* stream);
/* Depth-wise part of FeedForward_Conv2d (:1033-1088): per frame, out = h + dw5x5(h) + dw3x3(h) + dw1x1(h) with the eager
 * rounding bf16(bf16(bf16(h + c5) + c3) + c1), ck = bf16(bf16(conv_k(h)) + bias_k), zero "same" padding.
 *   h, out [BT, H, W, C] token-major (C = the 2 x hidden width);  w_taps [25 + 9 + 1, C]: the 5x5 taps, then the 3x3
 *   taps, then the 1x1 tap, each tap-major;  bias [3, C] (5x5, 3x3, 1x1). */
int vsb_dwconv_ffn(const vsb_bf16* h, const vsb_bf16* w_taps, const vsb_bf16* bias, vsb_bf16* out, int BT, int H, int W, int C,
                   void* stream);

/* ---- Open-Sora-Plan v1.1.0 KV compression (compress_kv_factor = k > 1, second-half blocks) ----------------------------
 * replaces Attention.sr + Attention.norm and the rearranges around them in AttnProcessor2_0.__call__
 * (models/transformers/open_sora_plan_v110_transformer_3d.py:1181-1197; layers built by _init_compress :1101-1122):
 * depth-wise Conv2d / Conv1d with stride = kernel (floors), + bias, then nn.LayerNorm(C) (affine).
 *   x     [B, T, H, W, C] token-major;  window (kt, kh, kw): spatial (1, k, k) per frame, temporal (k, 1, 1) per patch;
 *   pad_t leading copies of frame 0 (the reference prepends k - 1 of them when T is odd, :1190-1192);
 *   w_taps [kt*kh*kw, C] (sr.weight transposed tap-major);  bias, ln_w, ln_b [C];  eps = norm.eps (1e-5);
 *   out   [B, (T+pad_t)/kt, H/kh, W/kw, C] token-major (the layout of the queries).
 *   round_conv = 1: bf16(bf16(conv) + bias), what cuDNN gives for the spatial Conv2d on the reference's channels-last view;
 *   round_conv = 0: bf16(bias + conv) rounded once, ATen's native depthwise kernel, which the Conv1d takes.
 *   The LayerNorm rounds once at its output.  VSB_ERR_INVALID for an empty output grid or C % 8 != 0; C <= 3072. */
int vsb_kv_compress(const vsb_bf16* x, const vsb_bf16* w_taps, const vsb_bf16* bias, const vsb_bf16* ln_w, const vsb_bf16* ln_b,
                    vsb_bf16* out, int B, int T, int H, int W, int C, int kt, int kh, int kw, int pad_t, float eps, int round_conv,
                    void* stream);

/* ---- Pyramid Attention Broadcast gate (host integer logic, bit-exact) -------------------------------------------
 * replaces PABManager.if_broadcast_{spatial,temporal,cross}: core/pab/pab_mgr.py:54-91.
 * Returns 1 (reuse the cached tensor) or 0; *count advances on every call and wraps modulo steps.
 * has_timestep = 0 models `timestep is None`. */
int vsb_pab_gate(int broadcast_on, int has_timestep, int timestep, int* count, int range, int lo, int hi, int steps);

/* ---- DSP dimension switch over NVLink peer memory ---------------------------------------------------------------
 * replaces STDiT3Block.dynamic_switch -> all_to_all_with_pad -> _all_to_all_func:
 * open_sora_transformer_3d.py:288-315, core/distributed/comm.py:282-304,104-108.
 * The switch is fused into its producer and its consumer (north_star: "in-kernel sequence-dim all-to-all issuing P2P
 * stores fused with the preceding [producer]"; in STDiT3 the producer of the S-shard -> T-shard switch is the AdaLN
 * modulate, open_sora_transformer_3d.py:196-216, and the consumer of the switch back is the gate + residual, :213-228):
 *
 * vsb_ln_modulate_dsp = vsb_ln_modulate whose store path IS the switch: row (b, t, sl) goes to peer (b*T+t) / Tl,
 *   window viewed as [Tl, Sg, C], row ((b*T+t) % Tl, rank*Sl + sl), Tl = ceil(B*T / world) ((batch, frame) sequences
 *   are scattered, not frames: 2*20 = 40 split 8 ways exactly); zero rows for padded sequences, padded columns never
 *   sent; the last CTA to finish publishes the epoch into every peer's flag array.  Follow with vsb_dsp_wait on the
 *   same flag array.
 *     host_peer_recv[r]   device pointer (peer-mapped) to rank r's receive window
 *     host_peer_flags[r]  device pointer (peer-mapped) to rank r's flag array (uint32 epoch counters)
 * vsb_dsp_signal publishes the next epoch without moving data (the proj GEMM wrote into this rank's OWN window).
 * vsb_dsp_wait blocks the stream until all `world` peers have published epoch `epoch` into my_flags.
 * vsb_gate_residual_dsp = vsb_gate_residual whose y operand is PULLED with 128-bit peer loads from the producers'
 *   windows host_peer_y[r] (each viewed as [Tl, Sg, C]); call after vsb_dsp_wait on the signalled flag array.
 * epoch == 0: take the next value of a DEVICE-side counter kept in the flag array (slots 32 = sent, 33 = waited), so a
 * captured CUDA graph of a whole denoising step advances the epochs on every replay without host involvement.  Do not
 * mix explicit and device-side epochs on one flag array. */
int vsb_ln_modulate_dsp(const vsb_bf16* x, const vsb_bf16* mod, const uint8_t* x_mask, int shift_row, int scale_row,
                        int B, int T, int Sl, int C, float eps, void* const* host_peer_recv, void* const* host_peer_flags,
                        int rank, int world, int Sg, unsigned epoch, void* stream);
int vsb_dsp_signal(void* const* host_peer_flags, int rank, int world, unsigned epoch, void* stream);
int vsb_dsp_wait(void* my_flags, int world, unsigned epoch, void* stream);
int vsb_gate_residual_dsp(const vsb_bf16* x, void* const* host_peer_y, vsb_bf16* out, vsb_bf16* cache_out,
                          const vsb_bf16* mod, const uint8_t* x_mask, int gate_row, int B, int T, int Sl, int C, int rank,
                          int world, int Sg, void* stream);

/* Symmetric receive windows for the reshard: cudaMalloc'ed (zeroed) here so that a CUDA IPC handle maps the exact
 * base address; handles (64 bytes) are exchanged once at initialize() over the process group's store.
 * replaces nothing in the reference (NCCL owns its buffers); this is the native plumbing for P2P stores. */
int vsb_dsp_alloc(void** out, size_t bytes);
int vsb_dsp_free(void* p);
int vsb_ipc_get_handle(void* devptr, void* out_handle64);
int vsb_ipc_open_handle(const void* handle64, void** out_devptr);
int vsb_ipc_close_handle(void* devptr);

/* ---- CogVideoX VAE decoder (models/autoencoders/autoencoder_kl_cogvideox.py) -------------------------------------
 * Activations are channels-last [B, T, H, W, C] 16-bit tensors.
 *
 * vsb_vae_conv3d: CogVideoXCausalConv3d (:59-135, kernel (kt, 3, 3), kt = 3) and the up-sampler's Conv2d (kt = 1,
 *   modules/upsampling.py:36,62-65) as an implicit GEMM on wgmma.  x [B, kt-1+T, H, W, Cin] holds the kt-1 causal context
 *   frames first (copies of frame 0 or the carried conv_cache, :112-117); out [B, T, H, W, Cout].  The spatial zero
 *   padding (:131-132) is not materialised.  w_packed [Cout_pad, kt*9, Cin_pad] is the weight packed tap-major (tap =
 *   (dt*3 + dy)*3 + dx), Cin_pad / Cout_pad = Cin / Cout rounded up to a multiple of 64,
 *   zero padded.  out = bf16(conv + bias) [+ resid, rounded again: the ResNet sum of :298]; round_conv = 1 rounds the
 *   convolution to 16 bits before the bias is added.  Cin = 16 or a multiple of 64; Cout = 3, 4, 8 or a multiple of 64
 *   (4: the OpenSora v1.2 temporal decoder's conv_out; 8: the SDXL image encoder's conv_out).
 * vsb_vae_groupnorm_stats: mean and rstd = rsqrt(var + eps) (fp32, stats [B, G, 2]) of nn.GroupNorm over x [B, P, C]
 *   (P = T*H*W pixels).  workspace: B * VSB_GN_CHUNKS * C * 2 floats.  The sums are shifted by each channel's value at
 *   the sample's first pixel, so a DC offset large against the spread does not cancel the variance away.  Fixed-order
 *   reduction, no atomics: repeated launches are bit-identical.  C in {64, 128, 256, 512}, G | C.
 * vsb_vae_spatial_norm_silu: silu(GroupNorm(f) * conv_y(zq) + conv_b(zq)) (CogVideoXSpatialNorm3D :165-178, then the
 *   ResNet's nonlinearity :280,:291 or conv_act :867), each eager op rounded.  zyb [B, Tz, h, w, 2C] holds conv_y | conv_b
 *   at latent resolution, gathered with F.interpolate's nearest rule (the odd frame count split of :166-174).  The result
 *   goes to frames t_off .. t_off+T-1 of out [B, T_out, H, W, C] (the next convolution's input after its context).
 * vsb_vae_upsample2x: nearest 2x in H and W, and in T when compress_time (with the odd-frame rule of upsampling.py:40-60):
 *   x [B, T, H, W, C] -> out [B, T2, 2H, 2W, C], T2 = T, 2T (even T > 1) or 2T - 1 (odd T > 1). */
#define VSB_GN_CHUNKS 256
int vsb_vae_conv3d(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias, const vsb_bf16* resid, vsb_bf16* out,
                   int B, int T, int H, int W, int Cin, int Cout, int kt, int round_conv, void* stream);
int vsb_vae_groupnorm_stats(const vsb_bf16* x, float* stats, float* workspace, int B, long long P, int C, int G, float eps,
                            void* stream);
int vsb_vae_spatial_norm_silu(const vsb_bf16* f, const float* stats, const vsb_bf16* gamma, const vsb_bf16* beta,
                              const vsb_bf16* zyb, vsb_bf16* out, int B, int T, int H, int W, int C, int G, int Tz, int h,
                              int w, int t_off, int T_out, void* stream);
int vsb_vae_upsample2x(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C, int compress_time, void* stream);

/* ---- Open-Sora-Plan causal-VAE decoder (models/autoencoders/autoencoder_kl_open_sora_plan.py) ---------------------
 * Channels-last [B, T, H, W, C] 16-bit activations; the causal convolutions run on vsb_vae_conv3d, the 1x1x1 ones and
 * the attention's S = Q K^T and O = P V on vsb_gemm_bias_act / vsb_gemm_bias_residual.
 *
 * vsb_vae_groupnorm_act: Normalize = nn.GroupNorm(G, C, eps=1e-6) of x (stats from vsb_vae_groupnorm_stats, kept in the
 *   16-bit dtype as torch does), then with act = 1 the nonlinearity x * torch.sigmoid(x) (v1.2.0 :100-101, v1.1.0
 *   :1255-1256), each eager op rounded, or with act = 2 F.silu (nn.SiLU of the OpenSora v1.2 temporal and spatial
 *   decoders): x / (1 + exp(-x)) in fp32, rounded once.  Writes frames t_off .. t_off+T-1 of out [B, T_out, H, W, C].
 *   C % 8 == 0, G | C.
 * vsb_vae_upsample_linear2x: F.interpolate(mode="trilinear", align_corners=False) of x [B, T, H, W, C] by 2 in H and W
 *   (spatial) and by 2 in T over frames 1.. with frame 0 kept (temporal; Spatial2xTime2x3DUpsample v1.2.0 :349-357,
 *   TimeUpsample2x / TimeUpsampleRes2x v1.1.0 :1549-1596), fp32, rounded once.  To = 1 + 2 (T - 1) frames when temporal
 *   and T > 1, else T, written to frames t_off .. t_off+To-1 of out [B, T_out, Ho, Wo, C].  C % 8 == 0.
 * vsb_vae_mix: out = alpha * x + one_minus_alpha * y with each product and the sum rounded (TimeUpsampleRes2x :1596);
 *   x = frames t_off .. t_off+T-1 of xbuf [B, T_x, n], y and out [B, T, n], n = H*W*C, n % 8 == 0.
 * vsb_vae_attn_split: the attention block's fused q | k | v (qkv [B, T, P, 3C], P = H*W) to per-frame GEMM operands
 *   q [B*T, P, C], k [B*T, Pp, C] and vt [B*T, C, Pp] (V transposed), zero past P (Pp = P rounded up to 8).  mixed = 0:
 *   AttnBlock3DFix (frames as they are); mixed = 1: AttnBlock3D's reshape(b*t, c, h*w) of a b c t h w tensor
 *   (v1.1.0 :921-929): pseudo-frame j, channel ch reads channel (j*C + ch) / T of frame (j*C + ch) % T.  C % 32 == 0.
 * vsb_vae_attn_softmax: in place on S [rows, Pp]: softmax over the first P columns of bf16(S * scale) in fp32, rounded
 *   once (torch.nn.functional.softmax of w_ * c ** -0.5); columns P .. Pp-1 become zero.
 * vsb_vae_attn_merge: AttnBlock3D's output h_.reshape(b, c, t, h, w) (:932): out [B, T, P, C] channel c, frame t =
 *   o [B*T, P, C] pseudo-frame (c*T + t) / C, channel (c*T + t) % C. */
int vsb_vae_groupnorm_act(const vsb_bf16* x, const float* stats, const vsb_bf16* gamma, const vsb_bf16* beta, vsb_bf16* out,
                          int B, int T, int H, int W, int C, int G, int t_off, int T_out, int act, void* stream);
int vsb_vae_upsample_linear2x(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C, int spatial, int temporal,
                              int t_off, int T_out, void* stream);
int vsb_vae_mix(const vsb_bf16* xbuf, const vsb_bf16* y, vsb_bf16* out, int B, int T, long long n, int t_off, int T_x,
                float alpha, float one_minus_alpha, void* stream);
int vsb_vae_attn_split(const vsb_bf16* qkv, vsb_bf16* q, vsb_bf16* k, vsb_bf16* vt, int B, int T, int P, int Pp, int C,
                       int mixed, void* stream);
int vsb_vae_attn_softmax(vsb_bf16* S, int rows, int P, int Pp, float scale, void* stream);
int vsb_vae_attn_merge(const vsb_bf16* o, vsb_bf16* out, int B, int T, int P, int C, void* stream);

/* ---- OpenSora v1.2 VAE decoder (models/autoencoders/autoencoder_kl_open_sora.py) ------------------------------------
 * The temporal decoder and the SDXL image decoder run on the entries above (vsb_vae_groupnorm_act with act = 2,
 * vsb_vae_conv3d with Cout = 4, the attention split / softmax and the GEMM) plus:
 * vsb_vae_depth_to_time: rearrange "B (C ts) T H W -> B C (T ts) H W" with ts = 2 on channels-last tensors: channel
 *   2c + ts of frame t of x [B, T, H, W, 2C] is channel c of frame t_off + 2t + ts of out [B, T_out, H, W, C].  Pure data
 *   movement (bit exact).  C % 8 == 0, 16-byte aligned pointers. */
int vsb_vae_depth_to_time(const vsb_bf16* x, vsb_bf16* out, int B, int T, int H, int W, int C, int t_off, int T_out,
                          void* stream);

/* ---- OpenSora v1.2 VAE encoder (models/autoencoders/autoencoder_kl_open_sora.py, OpenSoraVAEEncoder) ----------------
 * The temporal encoder (reference Encoder :177-272) and the SDXL image encoder (diffusers' Encoder) run on the decoder's
 * entries above (vsb_vae_conv3d with Cout = 8 for the image encoder's conv_out; RGB and the 4-channel latent zero
 * padded to 16 channels on the host) plus:
 * vsb_vae_conv_down: the two down-sampling convolutions on the implicit GEMM of vsb_vae_conv3d, x [B, Tin, Hin, Win, Cin]
 *   -> out [B, T, H, W, Cout] = bf16(conv + bias) (round_conv as in vsb_vae_conv3d), w_packed as for vsb_vae_conv3d:
 *   - kt = 1, stride_t = 1, stride_hw = 2: Downsample2D, F.pad(x, (0, 1, 0, 1)) then a 3x3 conv with stride 2 (T = Tin,
 *     H = (Hin - 2) / 2 + 1, W likewise).  The A tile is a TMA box with traversal strides 2 in W and H; the right and
 *     bottom zero padding is its out-of-bounds fill.  Hin, Win >= 2.
 *   - kt = 3, stride_t = 2, stride_hw = 1: CausalConv3d(k=3, strides=(2, 1, 1)) (:107-124), whose time_pad is one zero
 *     frame in front: x holds the Tin real frames only, and output frame t reads frames 2t - 1 .. 2t + 1 of x, frame -1
 *     being the TMA out-of-bounds zero fill (T = (Tin - 2) / 2 + 1, Tin >= 2).  Spatial zero padding 1 as
 *     vsb_vae_conv3d.
 *   Cin = 16 or a multiple of 64; Cout = 8 or a multiple of 64. */
int vsb_vae_conv_down(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias, vsb_bf16* out, int B, int Tin,
                      int Hin, int Win, int Cin, int Cout, int kt, int stride_t, int stride_hw, int round_conv, void* stream);

/* ---- SVD temporal decoder (Latte's vae_temporal_decoder, models/autoencoders/autoencoder_kl_temporal_decoder.py) -----
 * The per-frame ResnetBlock2D halves, the mid-block attention and the up-samplers run on the entries above; the
 * TemporalResnetBlock halves and time_conv_out run on:
 * vsb_vae_conv_time: a (kt, 1, 1) convolution of x [B, kt-1+T, H, W, Cin] (channels-last; a zero-padded input with
 *   padding (1, 0, 0) is frames 1 .. T of a buffer whose frames 0 and T+1 are zero) on the implicit GEMM of
 *   vsb_vae_conv3d with one spatial tap: K = kt * Cin, the A box only moves in time.  w_packed [Cout, kt, Cin] (tap-major,
 *   kernels.pack_conv_weight of a [Cout, Cin, kt, 1, 1] weight).  v = bf16(bf16(conv) + bias) with round_conv (else
 *   bf16(conv + bias)); mix = 0: out = v [+ resid, rounded]; mix = 1 (TemporalResnetBlock.conv2 + AlphaBlender):
 *   xt = bf16(resid + v), out = bf16(bf16(mix_a * resid) + bf16(mix_b * xt)), resid [B, T, H, W, Cout] being the spatial
 *   block's output and mix_a / mix_b 16-bit values (1 - sigmoid(mix_factor) and 1 - that, rounded on the host).
 *   Cin and Cout multiples of 64.
 * vsb_vae_time_conv_rgb: time_conv_out, Conv3d 3 -> 3 with kernel (3, 1, 1), padding (1, 0, 0) and bias, of x [B, T, H,
 *   W, 3] -> out [B, T, H, W, 3]; w is the Conv3d weight [3, 3, 3, 1, 1] as stored.  Each output: the 9 products summed
 *   in fp32, rounded, + bias, rounded (as vsb_vae_conv3d with round_conv). */
int vsb_vae_conv_time(const vsb_bf16* x, const vsb_bf16* w_packed, const vsb_bf16* bias, const vsb_bf16* resid, vsb_bf16* out,
                      int B, int T, int H, int W, int Cin, int Cout, int kt, int mix, float mix_a, float mix_b, int round_conv,
                      void* stream);
int vsb_vae_time_conv_rgb(const vsb_bf16* x, const vsb_bf16* w, const vsb_bf16* bias, vsb_bf16* out, int B, int T, int H,
                          int W, void* stream);

/* ---- IEEE fp16 twins ----------------------------------------------------------------------------------------------
 * The reference runs CogVideoX-2b and Latte in torch.float16 (pipelines/cogvideox/pipeline_cogvideox.py:138-139,
 * pipelines/latte/pipeline_latte.py:201).  Every kernel entry above that touches activations exists a second time with
 * the suffix _f16: same arguments, same tile schedules, fp32 accumulation and rounding points, the 16-bit storage type
 * being IEEE half instead of bfloat16 (each kernel source is compiled twice: csrc/vsb_common.cuh, -DVSB_HALF).  The
 * DSP entries are bf16 only (sequence parallelism is an OpenSora path). */
typedef uint16_t vsb_f16;
int vsb_ln_modulate_f16(const vsb_f16* x, vsb_f16* out, const vsb_f16* mod, const uint8_t* x_mask, int shift_row,
                    int scale_row, int B, int T, int S, int C, float eps, void* stream);
int vsb_ln_modulate_affine_f16(const vsb_f16* x, vsb_f16* out, const vsb_f16* mod, const uint8_t* x_mask,
                           const vsb_f16* gamma, const vsb_f16* beta, int shift_row, int scale_row, int B, int T, int S,
                           int C, float eps, void* stream);
int vsb_modulation_table_f16(const vsb_f16* table, const vsb_f16* t, const vsb_f16* t0, vsb_f16* mod, int B, int C,
                         int rows, void* stream);
int vsb_patch_embed_f16(const vsb_f16* z, const vsb_f16* w, const vsb_f16* bias, const vsb_f16* pos, vsb_f16* out, int B,
                    int Cin, int T, int H, int W, long long batch_stride, long long chan_stride, long long frame_stride,
                    int ph, int pw, int C, int s0, int S_local, void* stream);
int vsb_gate_residual_f16(const vsb_f16* x, const vsb_f16* y, vsb_f16* out, vsb_f16* cache_out, const vsb_f16* mod,
                      const uint8_t* x_mask, int gate_row, int B, int T, int S, int C, void* stream);
int vsb_residual_add_f16(const vsb_f16* x, const vsb_f16* y, vsb_f16* out, size_t n, void* stream);
int vsb_qk_rmsnorm_f16(vsb_f16* qkv, const vsb_f16* wq, const vsb_f16* wk, size_t rows, int H, int D, float eps,
                   void* stream);
int vsb_qk_rmsnorm_rope_f16(vsb_f16* qkv, const vsb_f16* wq, const vsb_f16* wk, size_t rows, int H, int D, float eps,
                        const float* rope_cos, const float* rope_sin, int pos_div, int pos_mod, void* stream);
int vsb_qk_rope_halves_f16(vsb_f16* qkv, size_t rows, int H, int D, int half, const float* rope_cos,
                           const float* rope_sin_signed, int pos_div, int pos_mod, void* stream);
int vsb_qk_layernorm_f16(vsb_f16* qkv, const vsb_f16* wq, const vsb_f16* bq, const vsb_f16* wk, const vsb_f16* bk,
                     size_t rows, int H, int D, float eps, void* stream);
int vsb_attn_short_f16(const vsb_f16* qkv, vsb_f16* out, const vsb_f16* wq, const vsb_f16* wk, const float* rope_cos,
                   const float* rope_sin, int n_outer, int n_inner, long long outer_stride, long long inner_stride,
                   long long tok_stride, int n, int H, int D, float eps, float scale, int flags, void* stream);
int vsb_gemm_bias_act_f16(const vsb_f16* A, const vsb_f16* W, const vsb_f16* bias, vsb_f16* out, int M, int N, int K,
                      int act, void* stream);
int vsb_quant_rows_fp8_f16(const vsb_f16* x, uint8_t* q, float* scale, int M, int K, void* stream);
int vsb_ln_modulate_fp8_f16(const vsb_f16* x, uint8_t* q, float* scale, const vsb_f16* mod, const uint8_t* x_mask,
                            int shift_row, int scale_row, int B, int T, int S, int C, float eps, void* stream);
int vsb_gemm_fp8_bias_act_f16(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw, const vsb_f16* bias,
                              vsb_f16* out, int M, int N, int K, int act, void* stream);
int vsb_gemm_fp8_bias_residual_f16(const uint8_t* A, const float* sa, const uint8_t* W, const float* sw,
                                   const vsb_f16* bias, const vsb_f16* resid, vsb_f16* out, const vsb_f16* mod,
                                   const uint8_t* x_mask, int gate_row, int M, int N, int K, int B, int T, int S,
                                   void* stream);
int vsb_gemm_bias_residual_f16(const vsb_f16* A, const vsb_f16* W, const vsb_f16* bias, const vsb_f16* resid,
                           vsb_f16* out, const vsb_f16* mod, const uint8_t* x_mask, int gate_row, int M, int N, int K,
                           int B, int T, int S, void* stream);
int vsb_attn_flash_f16(const vsb_f16* q, const vsb_f16* k, const vsb_f16* v, vsb_f16* out, int nb, int nq, int nk,
                   int H, int D, long long q_row_stride, long long q_batch_stride, long long kv_row_stride,
                   long long kv_batch_stride, const int* host_kv_lens, float scale, void* stream);
int vsb_attn_flash_strided_f16(const vsb_f16* q, const vsb_f16* k, const vsb_f16* v, vsb_f16* out, int nb, int nq, int nk,
                           int H, int D, long long q_row_stride, long long q_batch_stride, long long kv_row_stride,
                           long long kv_batch_stride, long long out_row_stride, long long out_batch_stride,
                           const int* host_kv_lens, float scale, void* stream);
int vsb_dwconv_shuffle_f16(const vsb_f16* x, const vsb_f16* w_taps, const vsb_f16* bias, vsb_f16* out, int B, int T, int H,
                           int W, int C, int kt, int kh, int kw, int dt, int dh, int dw, void* stream);
int vsb_gate_residual_unshuffle_f16(const vsb_f16* x, const vsb_f16* y, vsb_f16* out, const vsb_f16* mod, int gate_row, int B,
                                    int T, int H, int W, int C, int dt, int dh, int dw, void* stream);
int vsb_dwconv_ffn_f16(const vsb_f16* h, const vsb_f16* w_taps, const vsb_f16* bias, vsb_f16* out, int BT, int H, int W, int C,
                       void* stream);
int vsb_kv_compress_f16(const vsb_f16* x, const vsb_f16* w_taps, const vsb_f16* bias, const vsb_f16* ln_w, const vsb_f16* ln_b,
                        vsb_f16* out, int B, int T, int H, int W, int C, int kt, int kh, int kw, int pad_t, float eps,
                        int round_conv, void* stream);
int vsb_vae_conv3d_f16(const vsb_f16* x, const vsb_f16* w_packed, const vsb_f16* bias, const vsb_f16* resid, vsb_f16* out,
                       int B, int T, int H, int W, int Cin, int Cout, int kt, int round_conv, void* stream);
int vsb_vae_groupnorm_stats_f16(const vsb_f16* x, float* stats, float* workspace, int B, long long P, int C, int G,
                                float eps, void* stream);
int vsb_vae_spatial_norm_silu_f16(const vsb_f16* f, const float* stats, const vsb_f16* gamma, const vsb_f16* beta,
                                  const vsb_f16* zyb, vsb_f16* out, int B, int T, int H, int W, int C, int G, int Tz, int h,
                                  int w, int t_off, int T_out, void* stream);
int vsb_vae_upsample2x_f16(const vsb_f16* x, vsb_f16* out, int B, int T, int H, int W, int C, int compress_time,
                           void* stream);
int vsb_vae_groupnorm_act_f16(const vsb_f16* x, const float* stats, const vsb_f16* gamma, const vsb_f16* beta, vsb_f16* out,
                              int B, int T, int H, int W, int C, int G, int t_off, int T_out, int act, void* stream);
int vsb_vae_upsample_linear2x_f16(const vsb_f16* x, vsb_f16* out, int B, int T, int H, int W, int C, int spatial,
                                  int temporal, int t_off, int T_out, void* stream);
int vsb_vae_mix_f16(const vsb_f16* xbuf, const vsb_f16* y, vsb_f16* out, int B, int T, long long n, int t_off, int T_x,
                    float alpha, float one_minus_alpha, void* stream);
int vsb_vae_attn_split_f16(const vsb_f16* qkv, vsb_f16* q, vsb_f16* k, vsb_f16* vt, int B, int T, int P, int Pp, int C,
                           int mixed, void* stream);
int vsb_vae_attn_softmax_f16(vsb_f16* S, int rows, int P, int Pp, float scale, void* stream);
int vsb_vae_attn_merge_f16(const vsb_f16* o, vsb_f16* out, int B, int T, int P, int C, void* stream);
int vsb_vae_depth_to_time_f16(const vsb_f16* x, vsb_f16* out, int B, int T, int H, int W, int C, int t_off, int T_out,
                              void* stream);
int vsb_vae_conv_time_f16(const vsb_f16* x, const vsb_f16* w_packed, const vsb_f16* bias, const vsb_f16* resid, vsb_f16* out,
                          int B, int T, int H, int W, int Cin, int Cout, int kt, int mix, float mix_a, float mix_b,
                          int round_conv, void* stream);
int vsb_vae_time_conv_rgb_f16(const vsb_f16* x, const vsb_f16* w, const vsb_f16* bias, vsb_f16* out, int B, int T, int H,
                              int W, void* stream);
int vsb_vae_conv_down_f16(const vsb_f16* x, const vsb_f16* w_packed, const vsb_f16* bias, vsb_f16* out, int B, int Tin,
                          int Hin, int Win, int Cin, int Cout, int kt, int stride_t, int stride_hw, int round_conv,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VSB200_H_ */
