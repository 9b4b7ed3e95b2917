/*
 * megatts2_b200.h - C ABI of libmegatts2_b200.so (sm_90a).
 *
 * The reference (LSimon95/megatts2 @ 2ab81a1) has no FFI layer: its replaceable surface
 * is the Python nn.Module API (SURVEY.md §8b).  This library is what those modules bind
 * through ctypes; every entry point names the reference function it replaces
 * (file:line relative to the reference repo).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless the name ends in _host; fp32 unless stated
 *  - activations are channels-last: (B, T, C) with an explicit row stride `ld` (elements)
 *    and batch stride; the Python layer converts from/to the reference's (B, C, T)
 *  - the caller owns every buffer (inputs, outputs, workspace); the library never
 *    allocates device memory and keeps no pointer after return
 *  - work is enqueued on `stream` (a cudaStream_t passed as void*); no hidden device sync
 *  - every function returns 0 on success or a negative mtts_status; mtts_last_error()
 *    returns a thread-local message.  There is NO CPU fallback anywhere.
 */
#ifndef MEGATTS2_B200_H
#define MEGATTS2_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MTTS_ABI_VERSION 3

typedef enum {
  MTTS_OK = 0,
  MTTS_ERR_BAD_ARG = -1,
  MTTS_ERR_UNSUPPORTED = -2,
  MTTS_ERR_CUDA = -3,
  MTTS_ERR_WORKSPACE = -4
} mtts_status;

int mtts_abi_version(void);
const char* mtts_last_error(void);
/* number of kernels this library has launched in this process (bench.py gpu_launches) */
int64_t mtts_launch_count(void);
/* measurement aid (bench.py roofline leg; off by default): between begin and end every
 * tap-GEMM launch is bracketed by CUDA events on its stream; end() synchronises and returns
 * the summed kernel time, the summed algorithmic FLOPs (2*M*N*Cin*k) and the launch count. */
int mtts_profile_begin(void);
int mtts_profile_end(double* gemm_ms, double* gemm_flops, int64_t* gemm_launches);
/* per-engine split of the last profile_end: {ffma_ms, ffma_flops, ffma_launches, tc_ms, tc_flops, tc_launches} */
int mtts_profile_split(double* out6);
/* diagnostics: per-launcher CUDA-event trace of everything enqueued between begin and end (single stream);
 * end synchronises and writes a text table "launcher launches total_ms share" into buf */
int mtts_trace_begin(void* stream);
int mtts_trace_end(char* buf, int32_t buf_len);

/* Tensor-core operand formats.  BF16X3 and F16X2 give fp32-grade results (the tests hold them to the same bars):
 *   BF16X3: x = x1 + x2 + x3 (bf16), products x1w1 + x1w2 + x2w1 + x2w2 + x1w3 + x3w1  -> 6 MMAs, fp32 range
 *   F16X2 : x = x1 + x2' * 2^-11 (fp16, residual stored scaled so it stays in the normal range), products
 *           x1w1 + (x1w2' + x2'w1) * 2^-11 -> 3 MMAs, 22 significant bits per operand; |x| must be <= 65504.
 *           At the low end x1 is an fp16 subnormal below 2^-14 and both planes are zero below about 2^-35, so
 *           the representation error is |x - x^| <= 2^-22 |x| + 2^-36, not 2^-22 |x|: tiny operands (training
 *           gradients) lose their precision, and below 2^-36 they vanish.  BF16X3 has neither edge.
 * F16 is the opt-in half-precision inference format, NOT fp32-grade:
 *   F16   : x ~ x1 = fp16(x) (round-to-nearest, one plane), product x1w1 -> 1 MMA into an fp32 accumulator,
 *           11 significant bits per operand; |x| must be <= 65504.
 * A format has 3 - fmt planes.  An activation outside the fp16 range (F16X2, F16) poisons its result (inf/NaN) and sets
 * the int32 flag registered here for the current device (the caller owns the 4 bytes; NULL unbinds).  The Python layer
 * checks it once per synthesis and reruns the batch on BF16X3. */
enum { MTTS_TC_BF16X3 = 0, MTTS_TC_F16X2 = 1, MTTS_TC_F16 = 2 };
int mtts_tc_overflow_bind(int32_t* flag_dev);
/* SM budget of the calling host thread's subsequent launches (0 = the whole device): the persistent tensor-core kernels
 * size their grids from it, so work enqueued on two streams can share the device (the prompt re-vocode of Megatts.forward
 * runs beside the latency-bound AR loops). */
int mtts_set_sm_limit(int32_t n_sms);
/* Launch policy of the calling host thread while two streams share the device: SM budget (as above), allow_pairs (0 keeps
 * the tap-GEMM on single CTAs instead of 2-CTA clusters, which need two free SMs of one GPC), and whether launches carry the
 * programmatic-dependent-launch attribute (a long kernel's successor would otherwise be scheduled early onto the SMs left
 * free for the other stream).  (0, 1, 1) restores the defaults.  Megatts.synthesize uses it to re-vocode the prompt
 * (models/megatts2.py:371-372 of the reference) beside the MRTE + ADM stages. */
int mtts_set_launch_policy(int32_t sm_limit, int32_t allow_pairs, int32_t allow_pdl);
/* Diagnostics (host only, no CUDA call): the launch plan the tap-GEMM dispatcher picks for a stride-1 layer of this shape
 * (B x T output rows, k taps) on n_sms SMs, with partial_bytes of split-K partial-sum space and, if ln_rides, a LayerNorm
 * that the split's reduction can carry.  out5 = {N-tile width, K splits, CTA pair (always 0),
 * halo form (0 | 1), K-slab bytes}. */
int mtts_tc_plan_query(int32_t n_sms, int32_t B, int32_t T, int32_t Cin, int32_t Cout, int32_t k, int32_t dil, int32_t fmt,
                       int64_t partial_bytes, int32_t ln_rides, int32_t* out5);
/* As mtts_tc_plan_query, for a thread whose launch policy allows 2-CTA clusters (allow_pairs) or not.  out7 = out5, then
 * CTAs per cluster (2: the CTAs of a cluster share the weight tile through TMA multicast; 1: single CTAs) and the CTAs of
 * the grid (even when clustered; a clustered launch is further capped at the clusters the device can hold at once). */
int mtts_tc_plan_query_ex(int32_t n_sms, int32_t B, int32_t T, int32_t Cin, int32_t Cout, int32_t k, int32_t dil,
                          int32_t fmt, int64_t partial_bytes, int32_t ln_rides, int32_t allow_pairs, int32_t* out7);

/* activation / padding codes */
enum { MTTS_ACT_NONE = 0, MTTS_ACT_RELU = 1, MTTS_ACT_LEAKY = 2, MTTS_ACT_TANH = 3 };
enum { MTTS_PAD_ZERO = 0, MTTS_PAD_REFLECT = 1, MTTS_PAD_REPLICATE = 2 };

/* ------------------------------------------------------------------------------------------
 * Tap-GEMM: the one dense contraction of the path.  Covers nn.Linear (k = 1), nn.Conv1d
 * (modules/convnet.py:13-18,88-94; modules/transformer.py:76-78; modules/mrte.py:101-107
 * stride 16), dilated HiFi-GAN convs and ConvTranspose1d (as a 2-tap conv with s*Cout
 * columns):
 *   acc[b,t,n] = sum_{j<k} sum_{c<Cin} pre(X[b, t*stride + j*dil - pad, c]) * W[j][c][n]
 *   v = post(acc + bias[n]);  v += R[b,t,n];  v *= out_scale;  v += Y_old (accumulate)
 *   Y[b, t*ldy + n + out_shift] = v        (skipped when outside [0, y_batch_elems))
 * W is PRE-PACKED as (k, Cin, Cout) row-major (mtts_pack_* on the host side does that once).
 */
typedef struct {
  const float* x; int64_t x_batch_stride; int32_t ldx;
  const float* w;
  const float* bias;                       /* (Cout) or NULL */
  const float* res; int64_t res_batch_stride; int32_t ldr;   /* optional */
  float* y; int64_t y_batch_stride; int32_t ldy;
  int32_t B, Tin, Tout, Cin, Cout;
  int32_t k, stride, dil, pad;
  int32_t pad_mode;                        /* MTTS_PAD_* */
  int32_t pre_act; float pre_slope;        /* applied to X on load */
  int32_t post_act; float post_slope;
  float out_scale;
  int32_t accumulate;
  int64_t out_shift;                       /* 0 for ordinary convs */
  int64_t y_batch_elems;                   /* 0 -> Tout*ldy */
  const int32_t* in_lens;                  /* optional (B): item b's input is its first len = min(in_lens[b], Tin) rows;
                                              a row index ti outside [0, len) reads as zero (MTTS_PAD_ZERO, or len <= 0),
                                              as row 0 / len - 1 (MTTS_PAD_REPLICATE) or, MTTS_PAD_REFLECT, as its one
                                              reflection about row 0 (-ti) or row len - 1 (2 (len - 1) - ti), and as zero
                                              when that reflection is still outside (a len shorter than the halo) */
  /* tensor-core engine (optional): the same weights as three bf16 planes (3, k, Cout, Cin) and a scratch
   * buffer for the padded activation planes (>= 6*B*(Tout + dil*(k-1))*Cin + 2048 bytes).  Used when the
   * shape is eligible (stride 1, Cin % 8 == 0, Cin >= 32, Cout in {32, 64, >= 128 and % 32 == 0}). */
  const void* w_tc;
  void* tc_scratch; int64_t tc_scratch_bytes;
  int64_t tc_rows_cap;                     /* k == 1 only: row capacity of the scratch planes (>= B*Tin, 0 -> B*Tin);
                                              a stable capacity keeps the cached TMA descriptors valid across AR steps */
  /* plane fusion (tensor-core engine only).  tc_presplit = 1: the activation planes already sit in tc_scratch
   * (three planes of (B, Tout + dil*(k-1), Cin) bf16, padding materialised, pre-activation applied) - x is not
   * read.  tc_out_planes != NULL: the epilogue additionally writes act(result) as three bf16 planes for the next
   * tensor-core layer (row (b*tc_out_tp + tc_out_hl + t), stride tc_out_ld); y may then be NULL. */
  int32_t tc_presplit;
  void* tc_out_planes; int64_t tc_out_plane_stride;
  int32_t tc_out_ld, tc_out_tp, tc_out_hl, tc_out_act; float tc_out_slope;
  /* optional room for split-K partial sums (tensor-core engine, k == 1): when a dense layer has too few output tiles to
   * fill the GPU, K is split across CTAs into fp32 partials here and a second kernel reduces them in a fixed order and
   * applies the epilogue.  >= splits * B*Tout * Cout * 4 bytes; NULL -> never split. */
  void* tc_partial; int64_t tc_partial_bytes;
  /* operand format of w_tc / the activation planes: MTTS_TC_BF16X3 (three bf16 planes, 6 MMAs per product),
   * MTTS_TC_F16X2 (two fp16 planes, residual scaled by 2^11, 3 MMAs per product; see mtts_tc_overflow_bind) or
   * MTTS_TC_F16 (one fp16 plane, 1 MMA per product, not fp32-grade) */
  int32_t tc_fmt;
  /* tc_presplit only: the planes in tc_scratch may be a SHARED buffer with a larger halo than this conv needs -
   * tc_in_tp rows per batch item (0 -> Tout + dil*(k-1)) and this conv's first padded row at tc_in_row0 (HiFi-GAN: the
   * three ResBlocks of a stage read one split of the up-sampled signal, each at its own row offset) */
  int32_t tc_in_tp, tc_in_row0;
} mtts_conv_params;

int mtts_conv1d_f32(const mtts_conv_params* p, void* stream);
/* Diagnostics (host only, no CUDA call; of the pointers in *p only the alignment of x, w, y and res, whether res, in_lens
 * and tc_scratch are NULL, and tc_scratch_bytes are read): the kernel mtts_conv1d_f32 launches for *p on the exact-fp32
 * FFMA engine (the calls the tensor-core engine does not take) with n_sms SMs.  A K split (MTTS_FFMA_SPLITK) writes fp32
 * partial sums into tc_scratch and reduces them in a fixed order.  out8 = {kernel (MTTS_FFMA_*; NONE: no output rows),
 * rows BM and columns BN of a CTA's output tile (256 x 1 for the Cout = 1 kernels), K splits (1: unsplit), 16-channel
 * K slices per split (0: unsplit), 16-byte loads of x (1) or scalar ones (0), the same for w, the same for the y / res
 * epilogue}.  The argument checks and error codes are those of the launch. */
enum { MTTS_FFMA_NONE = -1, MTTS_FFMA_TILE = 0, MTTS_FFMA_SPLITK = 1, MTTS_FFMA_COUT1 = 2, MTTS_FFMA_COUT1_TILED = 3 };
int mtts_ffma_plan_query(const mtts_conv_params* p, int32_t n_sms, int32_t* out8);

/* Tensor-core linear layer (wgmma, sm_90a): Y[M,N] = post(pre(X)[M,K] . W[N,K]^T + bias) (+ R) with
 * fp32-grade accuracy from split operands (fp32 accumulation in registers).  w_planes: (3, N, K) bf16 [BF16X3],
 * (2, N, K) fp16 [F16X2] or (1, N, K) fp16 [F16, half precision] row-major; scratch receives the activation planes
 * (mtts_linear_tc_scratch_bytes(rows_cap, K), rows_cap >= M).  K %% 8 == 0. */
int64_t mtts_linear_tc_scratch_bytes(int64_t rows_cap, int32_t K);
int mtts_linear_tc_f32(const float* x, int32_t ldx, int64_t M, int32_t K, const void* w_planes, int32_t N,
                       const float* bias, const float* res, int32_t ldr, float* y, int32_t ldy,
                       int32_t pre_act, float pre_slope, int32_t post_act,
                       void* scratch, int64_t scratch_bytes, int64_t rows_cap, int32_t fmt, void* stream);
/* fp32 (rows, C) with row stride ldx -> operand planes (3 | 2 | 1, rows, C) of `fmt` (the split the kernels apply to
 * activations; the host side uses it to pack weights once).  C %% 4 == 0, x 16-byte aligned. */
int mtts_split_planes_f32(const float* x, int32_t ldx, int64_t rows, int32_t C, void* planes, int32_t fmt, void* stream);

/* One HiFi-GAN ResBlock1 dilation step in one launch (the C = 32 / 64 vocoder stages; x, y (B, T, C) contiguous):
 *   y = (x + conv2(leaky(conv1_dil(leaky(x)) + b1)) + b2) * out_scale (+ y_old if accumulate)
 * leaky slope 0.1, both convs "same" with reflect padding, conv1 at dilation `dil`, conv2 at dilation 1.  w1_tc / w2_tc are
 * the (3 - fmt, k, C, C) operand planes of the (C, C, k) conv weights (the layout pack_conv_tc_planes writes); fmt is
 * MTTS_TC_F16X2 or MTTS_TC_F16, and the fp16 range flag of mtts_tc_overflow_bind is raised when an element of leaky(x) or of
 * leaky(conv1 + b1) at a position t in [0, T) is beyond 65504.  x and y must not alias; x, y, b1, b2 16-byte aligned.  MTTS_ERR_UNSUPPORTED outside
 * mtts_resblock_step_eligible. */
int mtts_resblock_step_f32(const float* x, float* y, const void* w1_tc, const float* b1, const void* w2_tc, const float* b2,
                           int32_t B, int32_t T, int32_t C, int32_t k, int32_t dil, float out_scale, int32_t accumulate,
                           int32_t fmt, void* stream);
/* Host only (no CUDA call): 1 if mtts_resblock_step_f32 accepts the shape - fmt f16x2 | f16, C 32 | 64, odd k >= 3 with
 * h2 = (k - 1) / 2 <= 31 and h1 = dil * h2 <= 32, T > h1 + h2, B * T >= 128 - else 0. */
int mtts_resblock_step_eligible(int32_t B, int32_t T, int32_t C, int32_t k, int32_t dil, int32_t fmt);

/* LayerNorm over the last dim (nn.LayerNorm, eps 1e-5; modules/convnet.py:28-30,
 * modules/transformer.py:67-68, modules/mrte.py:136):
 *   v = LN(x[row]) * gamma + beta;  v = post(v);  v += res[row];  v += y_old (accumulate) */
int mtts_layernorm_f32(const float* x, int32_t ldx, const float* gamma, const float* beta,
                       const float* res, int32_t ldr, float* y, int32_t ldy,
                       int64_t rows, int32_t C, float eps, int32_t post_act, int32_t accumulate,
                       void* stream);

/* Timbre interpolation: MRTE's LayerNorm -> ReLU (modules/mrte.py:168-169) applied to a weighted mix of K sources'
 * pre-norm attention outputs, one per timbre prompt (Megatts.synthesize(timbre_mels=...)).  Rows r = b*T + t,
 * 0 <= r < rows; row r of source k is the C floats at y + k*y_ks + r*ldy, and its weight row is the K floats at
 * weights + b*w_sb + t*w_st ((K,) weights: strides (0, 0); (B, K): (K, 0); (B, T, K): (T*K, K)).  For each row:
 *   1. wsum = the sum of the positive weights of the row in fp32, in k order; w^_k = w_k / wsum;
 *   2. m = w^_k0 * y_k0 for the first positive weight k0, then m = fmaf(w^_k, y_k, m) for the later positive weights in
 *      k order, element by element (the rule of mtts_adm_readout_mix_f32).  Sources with a zero, negative or NaN weight
 *      are skipped and never read, so non-finite values in them cannot reach the result;
 *   3. out[r] = post(LN(m) * gamma + beta), with mtts_layernorm_f32's arithmetic for this C, operation for operation.
 * With exactly one positive weight w^ = 1, so m is that source's row bit for bit and out[r] is what mtts_layernorm_f32
 * writes for it (res NULL, accumulate 0).  A row without a positive weight normalises the zero row (out = post(beta)).
 * Since MRTE's out-projection is affine, the mix of its outputs is the attention output under the w^-weighted mixture
 * of the per-prompt attention distributions.  K in 1..8 and C in {384, 512, 768, 1024} (MTTS_ERR_UNSUPPORTED outside);
 * post_act none, relu or tanh; y, out, gamma, beta 16-byte aligned, ldy, ldo and y_ks multiples of 4, T >= 1, strides
 * >= 0; out must not overlap the sources.  Every argument is checked before anything is enqueued; rows = 0 does
 * nothing. */
int mtts_mix_layernorm_f32(const float* y, int64_t y_ks, int32_t ldy, int32_t K, const float* weights, int64_t w_sb,
                           int64_t w_st, int32_t T, const float* gamma, const float* beta, float* out, int32_t ldo,
                           int64_t rows, int32_t C, float eps, int32_t post_act, void* stream);

/* softmax(Q K^T * scale + mask) V  (F.scaled_dot_product_attention at
 * modules/transformer.py:52-53).  q/k/v/o are (B, T, H, dh) views given by strides;
 * mask is additive fp32 with element strides (mask_sb, mask_sh, mask_sq, 1) or NULL.
 * dh in {64, 96, 128, 256, 512}.  q_row0/n_q select a row range of the queries. */
typedef struct {
  const float* q; int64_t q_sb; int32_t q_st;
  const float* k; int64_t k_sb; int32_t k_st;
  const float* v; int64_t v_sb; int32_t v_st;
  float* o; int64_t o_sb; int32_t o_st;
  const float* mask; int64_t mask_sb, mask_sh, mask_sq;
  int32_t B, H, Tq, Tk, dh;
  float scale;
  /* optional: write the output as three bf16 planes (row b*Tq + t, stride o_planes_ld) for a following
   * tensor-core GEMM; o may then be NULL */
  void* o_planes; int64_t o_plane_stride; int32_t o_planes_ld;
  int32_t o_planes_fmt;                    /* MTTS_TC_BF16X3 | MTTS_TC_F16X2 | MTTS_TC_F16 */
} mtts_attn_params;
/* fp32 kernel for every shape: q, k and v may use the full fp32 range (the BF16X3 and FFMA engines). */
int mtts_attention_f32(const mtts_attn_params* p, void* stream);
/* The same operation for callers whose engine accepts fp16-range operands (F16X2, F16): sequences of at least 65 queries
 * with dh in {64, 96, 128}, and the opt-in AR steps below, run on the tensor-core kernel, which splits q, k and v into
 * F16X2 planes - |x| must be <= 65504 (an element beyond it poisons the result and sets the flag of
 * mtts_tc_overflow_bind); every other shape runs as mtts_attention_f32. */
int mtts_attention_tc_f32(const mtts_attn_params* p, void* stream);
/* Opt-in, mtts_attention_tc_f32 only: AR-step attention (Tq == Tk <= 64, even head count, dh 64 | 96) with at least
 * `min_len` rows runs on the tensor-core kernel (one 64-row tile per head) instead of the fp32 kernel; min_len <= 0 switches it off (the default: it is slower
 * inside the synthesis step, see csrc/ops.cu).  Returns the previous setting. */
int mtts_set_attention_pair_min(int32_t min_len);
/* Diagnostics (host only, no CUDA call; only the alignment of the pointers in *p is read): the kernel mtts_attention_f32
 * (allow_f16_operands = 0) or mtts_attention_tc_f32 (1) launches for *p when mtts_set_attention_pair_min is set to
 * pair_min.  out6 = {kernel (MTTS_ATTN_*), dh, then for MTTS_ATTN_FP32 its instantiation: query rows per warp RW, warps
 * per CTA NW, keys per lane and tile KPL (0 otherwise), 16-byte loads (1) or scalar ones (0)}.  The argument checks and
 * error codes are those of the launches. */
enum { MTTS_ATTN_NONE = -1, MTTS_ATTN_FP32 = 0, MTTS_ATTN_TC = 1, MTTS_ATTN_TC_PAIR = 2 };
int mtts_attention_plan_query(const mtts_attn_params* p, int32_t allow_f16_operands, int32_t pair_min, int32_t* out6);

/* EuclideanCodebook.quantize (modules/quantization/core_vq.py:175-183): first index of
 * max_k -(|x|^2 - 2 x.e_k + |e_k|^2).  x (N, D) ld = ldx, embed (K, D) -> idx (N) int64 */
int mtts_vq_argmin_f32(const float* x, int32_t ldx, const float* embed, int64_t N, int32_t D, int32_t K,
                       int64_t* idx, void* stream);
/* EuclideanCodebook.dequantize / ResidualVectorQuantizer.decode (core_vq.py:188-190, 360-367)
 * with an optional time-repeat (vqpe.py:60-61, models/megatts2.py:362-364):
 *   y[b, t, :] = embed[idx[b, t / repeat], :]  for t < T_out;  y is (B, T_out, ldy) */
int mtts_vq_gather_f32(const int64_t* idx, int32_t idx_ld, const float* embed, int32_t D, int32_t K,
                       int32_t B, int32_t T_out, int32_t repeat, float* y, int64_t y_sb, int32_t ldy,
                       void* stream);

/* extract_mel_spec (modules/tokenizer.py:107-125; SURVEY.md Appendix B): reflect-padded
 * 1024-point STFT (hop 256, window table given), magnitude, banded mel filterbank,
 * log(max(., clamp)).  wav (B, L) -> out[b*out_sb + m*out_sm + f*out_sf], f < 1 + L/256.
 * The filterbank is passed in GROUPED banded form (the host packs it once, like a weight plane;
 * megatts2_b200/modules/tokenizer.py:pack_grouped_filterbank).  Mels are taken in groups of 4, G = ceil(n_mels / 4):
 *   fb_start[4 G]  first bin read for each mel, a multiple of 4 (slots past n_mels: 0)
 *   fb_off[G + 1]  float offset of each group's block in fb_w; a block holds 4 * len_g floats, len_g a multiple of 4
 *                  covering the longest (aligned) band of the group
 *   fb_w           16-byte aligned; block g, element i * len_g + t = weight of mel 4 g + i at bin fb_start[4 g + i] + t
 *                  (0 outside its band); fb_start[m] + len_g <= 516 for every mel (bins 513..515 read as zero).
 * n_fft must be 1024, hop 256, n_mels <= 128. */
int mtts_mel_spectrogram_f32(const float* wav, int64_t wav_sb, int32_t B, int32_t L,
                             const float* window, const float* fb_w, const int32_t* fb_off,
                             const int32_t* fb_start, int32_t n_mels, float clamp_min,
                             float* out, int64_t out_sb, int64_t out_sm, int64_t out_sf, void* stream);
/* Ragged batch for bulk extraction (MelSpecExtractor.extract over a corpus, modules/tokenizer.py:139-155,
 * prepare_ds.py:211-217; SURVEY.md 8f-2): clip b holds lens[b] <= L_max valid samples (device int32); its reflect
 * padding and frame count 1 + lens[b]/256 follow its own length; frames past that are not written. lens[b] > 512. */
int mtts_mel_spectrogram_ragged_f32(const float* wav, int64_t wav_sb, int32_t B, int32_t L_max, const int32_t* lens,
                                    const float* window, const float* fb_w, const int32_t* fb_off,
                                    const int32_t* fb_start, int32_t n_mels, float clamp_min,
                                    float* out, int64_t out_sb, int64_t out_sm, int64_t out_sf, void* stream);

/* nn.MaxPool1d(k, ceil_mode=True) over time, channels-last (modules/vqpe.py:38,
 * models/megatts2.py:357-358).  x (B, T, C) -> y (B, ceil(T/k), C) */
int mtts_maxpool_time_f32(const float* x, int64_t x_sb, int32_t ldx, float* y, int64_t y_sb, int32_t ldy,
                          int32_t B, int32_t T, int32_t C, int32_t k, void* stream);

/* TokenEmbedding + SinePositionalEmbedding (modules/embedding.py:41-47, 94-98):
 *   y[b,t,:] = table[ids[b,t],:] + alpha * pe[t + pe_offset,:]    (pe may be NULL) */
int mtts_embed_pe_f32(const int64_t* ids, int32_t ids_ld, const float* table, int32_t vocab, int32_t D,
                      const float* pe, float alpha, int32_t pe_offset, int32_t B, int32_t T,
                      float* y, int64_t y_sb, int32_t ldy, void* stream);
/* y = x + alpha * pe[t,:]  (SinePositionalEmbedding.forward on an existing tensor) */
int mtts_add_pe_f32(const float* x, int64_t x_sb, int32_t ldx, const float* pe, float alpha,
                    int32_t B, int32_t T, int32_t D, float* y, int64_t y_sb, int32_t ldy, void* stream);

/* LengthRegulator.forward (modules/mrte.py:23-31, 42-60) as a gather:
 *   y[b, sum_{j<i} d[b,j] + r, :] = x[b,i,:]; rows >= sum(d[b]) are zero.
 * totals (B) int32 receives sum(d[b]) (pass NULL to skip). y is (B, L_out, ldy). */
int mtts_length_regulate_f32(const float* x, int64_t x_sb, int32_t ldx, const int32_t* dur, int32_t dur_ld,
                             int32_t B, int32_t Tp, int32_t D, int32_t L_out,
                             float* y, int64_t y_sb, int32_t ldy, int32_t* totals, void* stream);

/* strided 2-D copy / transpose helpers used at the (B,C,T) <-> (B,T,C) module boundary:
 *   y[b, t, c] = x[b*x_sb + t*x_st + c*x_sc]   with optional replicate padding of `pad`
 *   rows at both ends of t (HiFi-GAN inference_padding) */
int mtts_copy_strided_f32(const float* x, int64_t x_sb, int64_t x_st, int64_t x_sc,
                          float* y, int64_t y_sb, int64_t y_st, int64_t y_sc,
                          int32_t B, int32_t T, int32_t C, int32_t pad_rep, void* stream);

/* ------------------------------------------------------------------------------------------
 * Audio front / back ends of Megatts.forward on the device (SURVEY.md 8f-3).
 *
 * mtts_resample_f32 - librosa.load(path, sr=16000) at models/megatts2.py:335 (and prepare_ds.py:113), the resampling
 * part: band-limited polyphase FIR, y[i*up + p] = sum_k xpad[i*down + k] * h[p][k] with xpad = x preceded by `width`
 * zeros; h is the (up, taps) filter table of torchaudio.functional.resample (built on the host in fp64:
 * megatts2_b200/audio.py).  x (B, L_in) with optional per-clip lengths; y (B, L_out), samples past lens_out[b] are zero.
 * mtts_peak_normalize_f32 - librosa.util.normalize(y) (:336): x[b] /= max|x[b]| in place (unchanged if the peak is below
 * FLT_MIN); scratch: B x 4 bytes.
 * mtts_pcm16_f32 - the integer encoding of the wav writer behind torchaudio.save (:375): round-to-nearest of x * 32768,
 * saturated. */
int mtts_resample_f32(const float* x, int64_t x_sb, int32_t B, int32_t L_in, const int32_t* lens_in, const float* h,
                      int32_t up, int32_t down, int32_t width, int32_t taps, float* y, int64_t y_sb, int32_t L_out,
                      const int32_t* lens_out, void* stream);
int mtts_peak_normalize_f32(float* x, int64_t x_sb, int32_t B, int32_t L, const int32_t* lens, void* scratch, void* stream);
int mtts_pcm16_f32(const float* x, int64_t n, int16_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training-mode / backward kernels (SURVEY.md 8f-4): what autograd needs so that MegaPLMTrainer / MegaADMTrainer
 * .training_step (models/trainer.py:243-268, 334-355) run through the drop-in modules.  The dense contractions of the
 * backward pass (dX = dY W, dW = dY^T X) use mtts_linear_tc_f32 / mtts_conv1d_f32 like the forward; these are the rest.
 *
 * mtts_bmm_f32: C[z1,z2][m,n] = alpha * sum_k A[z1,z2][m,k] * B[z1,z2][k,n] (+ C), every operand given by element strides
 *   (transposes and (B,T,H,dh) head views are free) - the attention products Q K^T, P V and their gradients.
 * mtts_softmax_fwd_f32: rows of S (B,H,Tq,Tk) -> P = softmax(S + mask) and Pd = P * keep (keep = dropout keep-scale or
 *   NULL); mtts_softmax_bwd_f32: dS = P * (dPd * keep - <dPd * keep, P>)   (F.scaled_dot_product_attention with dropout,
 *   modules/transformer.py:52-53, unfused for training).
 * mtts_layernorm_bwd_f32: dx (rows, C) and per-CTA partials (ceil(rows / 8), 2, C) of d-gamma | d-beta
 *   (reduce with mtts_colsum_f32).  mtts_colsum_f32: out[c] (+)= sum_r in[r*ld + c], fixed row order.
 * mtts_relu_bwd_f32: dx = dy * (y > 0).  mtts_embedding_bwd_f32: dW[ids[r]] += dy[r] (nn.Embedding).
 * mtts_rowdot_f32: out[r] = <a[r, :], b[r % period, :]> (d-alpha of SinePositionalEmbedding). */
int mtts_bmm_f32(const float* a, int64_t a_s1, int64_t a_s2, int64_t a_sm, int64_t a_sk, const float* b, int64_t b_s1,
                 int64_t b_s2, int64_t b_sk, int64_t b_sn, float* c, int64_t c_s1, int64_t c_s2, int64_t c_sm, int64_t c_sn,
                 int32_t Z1, int32_t Z2, int32_t M, int32_t N, int32_t K, float alpha, int32_t accumulate, void* stream);
int mtts_softmax_fwd_f32(const float* S, const float* mask, int64_t m_sb, int64_t m_sh, int64_t m_sq, int32_t B, int32_t H,
                         int32_t Tq, int32_t Tk, const float* keep, float* P, float* Pd, void* stream);
int mtts_softmax_bwd_f32(const float* P, const float* dPd, const float* keep, float* dS, int32_t Tk, int64_t rows, void* stream);
int mtts_layernorm_bwd_f32(const float* x, const float* gamma, const float* dy, float* dx, float* partial, int64_t rows, int32_t C,
                           float eps, void* stream);
int mtts_colsum_f32(const float* in, int64_t ld, int64_t rows, int32_t C, float* out, int32_t accumulate, void* stream);
int mtts_relu_bwd_f32(const float* y, const float* dy, float* dx, int64_t n, void* stream);
int mtts_embedding_bwd_f32(const int64_t* ids, const float* dy, int64_t rows, int32_t D, int32_t vocab, float* dW, void* stream);
int mtts_rowdot_f32(const float* a, const float* b, int64_t rows, int32_t C, int32_t period, float* out, void* stream);

/* Training-only pieces of the VQ codebook (SURVEY.md 8f-4): EuclideanCodebook.forward in train mode and the
 * straight-through / commitment step of VectorQuantization.forward.
 * mtts_kmeans_assign_f32: idx[n] = first argmin_k sum_d (x[n,d] - means[k,d])^2 - the bucket step of kmeans()
 *   (modules/quantization/core_vq.py:81-86; direct differences, not the expanded form of quantize).  D <= 512.
 * mtts_vq_cluster_sum_f32: sum[k,:] = sum_{n: idx[n]=k} x[n,:] accumulated in sample order, cnt[k] = bucket size as
 *   float - bincount + scatter_add_ of kmeans (:87-92) and embed_onehot.sum(0) / x.t() @ embed_onehot of the EMA step
 *   (:220-222).
 * mtts_kmeans_update_f32: means[k] = cnt[k] > 0 ? sum[k] / cnt[k] : means[k]   (:88-95).
 * mtts_vq_ema_update_f32: cluster_size <- decay cs + (1-decay) cnt; embed_avg <- decay ea + (1-decay) sum;
 *   embed = embed_avg / ((cs + eps) / (sum(cs) + K eps) * sum(cs))   (ema_inplace, laplace_smoothing; :217-229).
 *   scratch: K floats.
 * mtts_vq_replace_rows_f32: embed[k] = samples[pick[k]] where cluster_size[k] < thr   (expire_codes_ / replace_, :151-169;
 *   the caller draws pick = sample_vectors' indices).
 * mtts_vq_ste_commit_f32: out = x + (q - x) (the straight-through value as the reference rounds it) and
 *   loss[0] = mean((out - x)^2) (F.mse_loss(quantize.detach(), x), :303-311); partials: 256 floats of scratch.
 * mtts_vq_ste_commit_bwd_f32: dx = g_out + g_loss[0] * scale * (x - out), scale = commitment_weight * 2 / numel;
 *   g_out or g_loss may be NULL. */
int mtts_kmeans_assign_f32(const float* x, const float* means, int32_t N, int32_t K, int32_t D, int64_t* idx, void* stream);
int mtts_vq_cluster_sum_f32(const float* x, const int64_t* idx, int32_t N, int32_t K, int32_t D, float* sum, float* cnt,
                            void* stream);
int mtts_kmeans_update_f32(float* means, const float* sum, const float* cnt, int32_t K, int32_t D, void* stream);
int mtts_vq_ema_update_f32(float* cluster_size, float* embed_avg, float* embed, const float* sum, const float* cnt,
                           int32_t K, int32_t D, float decay, float eps, float* scratch, void* stream);
int mtts_vq_replace_rows_f32(float* embed, const float* samples, const int64_t* pick, const float* cluster_size, float thr,
                             int32_t K, int32_t D, int32_t N, void* stream);
int mtts_vq_ste_commit_f32(const float* x, const float* q, int64_t n, float* out, float* partials, float* loss, void* stream);
int mtts_vq_ste_commit_bwd_f32(const float* x, const float* out, const float* g_out, const float* g_loss, float scale,
                               int64_t n, float* dx, void* stream);

/* x (B, rows, L) contiguous: x[b, r, keep[b]:] = 0 in place - speechbrain HIFIGAN.mask_noise behind
 * decode_batch(mel, mel_lens, hop_len) (reference call site models/megatts2.py:370). */
int mtts_mask_tail_f32(float* x, int32_t B, int32_t rows, int32_t L, const int32_t* keep, void* stream);

/* Ragged row copy, one launch for B batch rows (long-form synthesis joins sentences with it: the prosody LM's context
 * history, its window, and the passage mel).  A buffer holds B batch rows of `*_rows` logical rows of row_bytes bytes;
 * logical row r of batch row b starts at byte b*sb + r*st.  For b < B and 0 <= r < min(n[b], n_max):
 *   dst[b, dst_off[b] + r] = src ? src[b, src_off[b] + r] : row_bytes / 4 copies of fill_word,
 * and only for the r with 0 <= dst_off[b] + r < dst_rows and (with src) 0 <= src_off[b] + r < src_rows: entries of the
 * tables that would run past either buffer, or below row 0, copy only the rows inside it, so no table value can reach
 * memory outside the two buffers.  Nothing else of dst is written.  The tables src_off, dst_off and n are (B,) int32 in
 * device memory; src_off may be NULL when src is (fill mode).  row_bytes is a positive multiple of 4 (so one entry serves
 * fp32 rows and int64 codes); strides are byte counts, multiples of 4, row strides >= row_bytes, batch strides >= 0
 * (src_sb = 0 broadcasts one src batch row), and dst's batch rows must not overlap.  16-byte accesses are used when
 * both bases, every stride and row_bytes are multiples of 16, 4-byte words otherwise.  src and dst must differ and must
 * not overlap.  B <= 65535.  Every argument is checked before anything is enqueued; B, n_max or dst_rows = 0 does
 * nothing. */
int mtts_copy_row_segments(const void* src, int64_t src_sb, int64_t src_st, int64_t src_rows, void* dst, int64_t dst_sb,
                           int64_t dst_st, int64_t dst_rows, int32_t row_bytes, const int32_t* src_off,
                           const int32_t* dst_off, const int32_t* n, int32_t B, int32_t n_max, uint32_t fill_word,
                           void* stream);

/* ------------------------------------------------------------------------------------------
 * Composite drivers: whole sub-networks enqueued by one call (C++ launch loop, no Python
 * per-kernel overhead).  Weight pointers refer to PRE-PACKED device buffers owned by the
 * caller.
 */
typedef struct {
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  const float *w_qkv, *b_qkv;          /* (1, D, 3D) packed, (3D) */
  const float *w_o, *b_o;              /* (1, D, D), (D) */
  const float *w_ff1, *b_ff1;          /* linear: (1, D, F); conv-FF: (5, D, F) */
  const float *w_ff2, *b_ff2;          /* linear: (1, F, D); conv-FF: (5, F, D) */
  /* tensor-core engine (optional, linear layers only): the same weights as THREE bf16 planes
   * (3, N, K) row-major (w = w1 + w2 + w3, see mtts_linear_tc_f32); NULL -> exact FFMA engine */
  const void *w_qkv_tc, *w_o_tc, *w_ff1_tc, *w_ff2_tc;
} mtts_encoder_layer;

typedef struct {
  int32_t n_layers, d_model, n_heads, ff_dim, conv_ff;
  int32_t engine;                      /* 0: fp32 FFMA everywhere; wgmma for GEMMs with M >= 128: 1 = BF16X3, 2 = F16X2, 3 = F16 operands */
  const mtts_encoder_layer* layers;    /* HOST array of n_layers entries */
} mtts_encoder;

/* TransformerEncoder.forward (modules/transformer.py:119-133).  x (B,T,D) -> y (B,T,D);
 * mask: optional additive (B,H,T,T) fp32 (utils/utils.py:21-39) given by strides.
 * last_row_only != 0: y is (B,1,D) = the last position's output (exact pruning of the final
 * layer; what MegaPLM.infer / MegaADM.infer consume, models/megatts2.py:178, 272). */
int64_t mtts_encoder_workspace_bytes(const mtts_encoder* enc, int32_t B, int32_t T);
int mtts_encoder_forward_f32(const mtts_encoder* enc, const float* x, float* y, int32_t B, int32_t T,
                             const float* mask, int64_t mask_sb, int64_t mask_sh, int64_t mask_sq,
                             int32_t last_row_only, void* workspace, int64_t workspace_bytes, void* stream);

/* MegaPLM.infer (models/megatts2.py:165-181): greedy AR decode, BOS = vq_bins, exactly T
 * steps, NON-causal full recompute per step (reference-faithful).  tc_latent (B,T,tc_dim);
 * codes_out (B,T) int64; logits_out optional (B,T,vq_bins) = last-position logits per step. */
typedef struct {
  mtts_encoder enc;
  const float* pc_embedding;   /* (vq_bins+2, vq_dim) */
  const float* w_predict;      /* packed (1, D, vq_bins) */
  const float* pe;             /* (>=T, D) sine table (modules/embedding.py:66-92) */
  float pe_alpha;
  int32_t vq_bins, vq_dim, tc_dim;
} mtts_plm;
int64_t mtts_plm_infer_workspace_bytes(const mtts_plm* m, int32_t B, int32_t T);
int mtts_plm_infer_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                       int32_t B, int32_t T, int64_t* codes_out, float* logits_out,
                       void* workspace, int64_t workspace_bytes, void* stream);

/* MegaADM.infer (models/megatts2.py:257-275): AR duration regression, raw float feedback,
 * final (p + 0.5) -> int32 -> clamp(1,128).  dur_out (B,T) int32; raw_out optional (B,T). */
typedef struct {
  mtts_encoder enc;
  const float* w_dt;           /* (emb_dim)   dt_linear_emb.weight[:,0] */
  const float* w_tc;           /* packed (1, tc_dim, tc_emb_dim) */
  const float* w_predict;      /* (D) predict_layer.weight[0,:] */
  const float* pe; float pe_alpha;
  int32_t emb_dim, tc_dim, tc_emb_dim;
} mtts_adm;
int64_t mtts_adm_infer_workspace_bytes(const mtts_adm* m, int32_t B, int32_t T);
int mtts_adm_infer_f32(const mtts_adm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                       int32_t B, int32_t T, int32_t* dur_out, float* raw_out,
                       void* workspace, int64_t workspace_bytes, void* stream);

/* Opt-in causal KV-cache decode (SURVEY.md 8f-1; NOT what the reference's infer() computes).  Follows the TRAINING
 * semantics of MegaPLM.forward / MegaADM.forward (causal=True, models/megatts2.py:158, 244): row t attends to rows <= t,
 * so a step computes one row per utterance and appends its K/V to per-layer caches - O(T) instead of the O(T^2) full
 * recompute.  Same arguments and outputs as the *_infer_f32 entry points; linear feed-forward encoders only. */
int64_t mtts_plm_decode_causal_workspace_bytes(const mtts_plm* m, int32_t B, int32_t T);
int mtts_plm_decode_causal_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                               int32_t B, int32_t T, int64_t* codes_out, float* logits_out,
                               void* workspace, int64_t workspace_bytes, void* stream);
int64_t mtts_adm_decode_causal_workspace_bytes(const mtts_adm* m, int32_t B, int32_t T);
int mtts_adm_decode_causal_f32(const mtts_adm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                               int32_t B, int32_t T, int32_t* dur_out, float* raw_out,
                               void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Opt-in sampled PLM decode: temperature, top-k and top-p, with a device-side Gumbel-max draw (the greedy entry points
 * above are unchanged and stay the reference-faithful path).  For one logits row z[0..V) (fp32) at AR step t of a row
 * whose key is kappa:
 *   1. temperature == 0 or top_k == 1: exactly the greedy argmax (lowest index on ties).
 *   2. y_i = z_i / temperature (fp32 division); NaN and -inf are never candidates.
 *   3. top_k > 0 and < V: keep the top_k largest y, ordered by (value descending, index ascending).
 *   4. top_p < 1: over the kept tokens in that order, keep the shortest prefix whose softmax mass is >= top_p (>= 1 token).
 *   5. pick = argmax over kept i of y_i - log(-log u_i), lowest index on ties, with u_i = ((w_i >> 8) + 0.5) * 2^-24 and
 *      w_i = word (i & 3) of Philox4x32-10 with key (seed_lo, seed_hi) and counter (i >> 2, t, kappa_lo, kappa_hi).
 *   6. a row with a +inf y returns its lowest +inf index; a row without a candidate returns 0.
 * A draw depends only on (row, parameters, seed, kappa, t): not on the batch size, the row's position or the launch, and
 * a replayed CUDA graph picks up new seed / key values from device memory.  V <= 4096 (MTTS_ERR_UNSUPPORTED above). */
typedef struct {
  float temperature;         /* finite, >= 0 */
  int32_t top_k;             /* >= 0; 0 = off (as is top_k >= V) */
  float top_p;               /* in (0, 1]; 1 = off */
  int32_t reserved;          /* must be 0 */
  const uint64_t* seed;      /* device, 1 element */
  const uint64_t* keys;      /* device, one element per row */
} mtts_sampling;
/* out[r * ld_out] = the pick of row r of logits (rows, V), row stride ld (0: every row reads the same logits) */
int mtts_sample_rows_f32(const float* logits, int64_t ld, int32_t V, int32_t rows, int32_t step, const mtts_sampling* s,
                         int64_t* out, int64_t ld_out, void* stream);
/* The sampler's generator on its own: out[4 i .. 4 i + 3] = Philox4x32-10(counter ctr[4 i .. 4 i + 3], key key[2 i, 2 i + 1])
 * (uint32 words), for callers that reproduce or audit its noise. */
int mtts_philox4x32_10_u32(const uint32_t* ctr, const uint32_t* key, uint32_t* out, int64_t n, void* stream);
/* mtts_plm_infer_f32 / mtts_plm_decode_causal_f32 with step t's codes drawn by the sampler above (row b keyed by
 * s->keys[b]) instead of the argmax; the drawn codes are what the next step consumes.  logits_out keeps the raw,
 * untempered logits.  Same arguments plus `s` (non-NULL), and the same workspace sizes: mtts_plm_infer_workspace_bytes and
 * mtts_plm_decode_causal_workspace_bytes. */
int mtts_plm_infer_sample_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                              int32_t B, int32_t T, int64_t* codes_out, float* logits_out, const mtts_sampling* s,
                              void* workspace, int64_t workspace_bytes, void* stream);
int mtts_plm_decode_causal_sample_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                                      int32_t B, int32_t T, int64_t* codes_out, float* logits_out, const mtts_sampling* s,
                                      void* workspace, int64_t workspace_bytes, void* stream);

/* Resumable MegaPLM.infer (greedy / sampled): runs AR steps [t0, t1) of the T-step decode, 0 <= t0 <= t1 <= T, against a
 * caller-owned code state `code_state` (B, T+1) int64, row stride T+1: column 0 holds BOS (vq_bins) and columns 1..t0 the
 * codes of steps < t0; step t writes column t+1.  codes_out (B,T) and logits_out (optional, (B,T,vq_bins)) are laid out as
 * in mtts_plm_infer_f32; only columns [t0, t1) are written.  Step t reads only tc_latent[:, :t+1] and codes < t, and a
 * sampled draw is keyed by (seed, key, t), so any split of [0, T) into consecutive ranges yields the codes and logits of
 * one mtts_plm_infer_f32 / mtts_plm_infer_sample_f32 call.  Same workspace size: mtts_plm_infer_workspace_bytes(m, B, T);
 * the workspace holds nothing between ranges. */
int mtts_plm_infer_range_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                             int32_t B, int32_t T, int32_t t0, int32_t t1, int64_t* code_state,
                             int64_t* codes_out, float* logits_out, void* workspace, int64_t workspace_bytes, void* stream);
int mtts_plm_infer_range_sample_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                                    int32_t B, int32_t T, int32_t t0, int32_t t1, int64_t* code_state,
                                    int64_t* codes_out, float* logits_out, const mtts_sampling* s,
                                    void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Prosody interpolation: the PLM decoded from a weighted mixture of K prompts' code distributions (Mega-TTS 2,
 * arXiv 2307.07218).  Utterance b has K >= 1 sources; source k is a latent tc^(k)[b] (T, tc_dim), all with the same T, and
 * b has a weight row w[b, 0..K) (fp32, every weight >= 0 and finite, row sum > 0; normalised on the device: w^ = w / sum).
 * All K sources share one code history, BOS then c_0 .. c_{t-1}.  At step t:
 *   1. each source runs the reference-faithful step (mtts_plm_infer_f32's non-causal full recompute) over its own latent
 *      and the shared history -> logits z^(k);
 *   2. l_i = log sum_k w^_k softmax(z^(k))_i, a log-sum-exp over the sources in fp32.  NaN and -inf have zero mass in
 *      their source; a source with a +inf logit puts all its mass on its lowest +inf index; a source with no candidate
 *      contributes nothing; without any candidate l is -inf everywhere (and the pick is 0);
 *   3. if exactly one weight of the row is positive, l is that source's raw logits row, copied bit for bit (so a one-hot
 *      row decodes exactly what mtts_plm_infer_f32 decodes from that source alone);
 *   4. c_t is picked from l by the greedy argmax or, with `s`, by the sampler (mtts_sampling) keyed by (seed, keys[b], t),
 *      and appended to the shared history.
 * A weight row without a positive weight gives l = -inf.  K <= 8 and vq_bins <= 4096 (MTTS_ERR_UNSUPPORTED above). */

/* l (B, V) into out (row stride ld_out) from logits rows (row stride ld): source k of utterance b is row k * B + b;
 * weights (B, K) contiguous, device. */
int mtts_mix_logprob_rows_f32(const float* logits, int64_t ld, int32_t V, int32_t K, int32_t B, const float* weights,
                              float* out, int64_t ld_out, void* stream);
/* The mixed decode.  tc_latent is the (K*B, T, tc_dim) stack of the sources, row k*B + b = source k of utterance b (batch
 * stride tc_sb, row stride tc_ld); weights (B, K) device; codes_out (B, T); logits_out optional, (K*B, T, vq_bins), the
 * raw per-source logits; s NULL = greedy.  Each step runs the encoder and the predict layer once over the K*B rows.  The
 * weights, the seed and the keys are read from device memory at every step, so a replayed CUDA graph picks up new values.
 * With K = 1 the codes and logits equal mtts_plm_infer_f32 / mtts_plm_infer_sample_f32 bit for bit. */
int64_t mtts_plm_infer_mix_workspace_bytes(const mtts_plm* m, int32_t K, int32_t B, int32_t T);
int mtts_plm_infer_mix_f32(const mtts_plm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                           int32_t B, int32_t T, const float* weights, int64_t* codes_out, float* logits_out,
                           const mtts_sampling* s, void* workspace, int64_t workspace_bytes, void* stream);
/* Steps [t0, t1) of the mixed decode against the shared (B, T+1) code state, as mtts_plm_infer_range_f32: any split of
 * [0, T) into consecutive ranges yields the codes and logits of one mtts_plm_infer_mix_f32 call.  Same workspace size. */
int mtts_plm_infer_mix_range_f32(const mtts_plm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                                 int32_t B, int32_t T, const float* weights, int32_t t0, int32_t t1, int64_t* code_state,
                                 int64_t* codes_out, float* logits_out, const mtts_sampling* s,
                                 void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Prosody and duration schedules: mix weights that change along the utterance.  The weights are an array W (B, T, K) fp32
 * on the device, row (b, t) at W + b*w_sb + t*w_st (K contiguous floats; w_sb, w_st >= 0).  Target step t of utterance b
 * runs the mix above with row (b, t) in place of the utterance's one row: the PLM picks c_t from
 * l = log sum_k w^_{b,t,k} softmax(z^(k)), the ADM feeds back r = sum_k w^_{b,t,k} y^(k), each row normalised, checked
 * and applied exactly as the per-utterance row is (a row with one positive weight gives that source's raw logits row or
 * readout, bit for bit).  w_st = 0 and w_sb = K is the (B, K) mix: the per-utterance entries are these with those
 * strides, and their launch sequences are the same.  Same workspace sizes as the per-utterance entries.
 *
 * Per-phone weights (B, Tp, K) become PLM step weights by mtts_mix_step_weights_f32, with the phone durations that the
 * length regulator uses (negative durations count as 0).  PLM step t covers the mel frames [8t, 8t+8) of [0, L_b),
 * L_b = sum of b's durations, and takes the weight row of the phone that owns the most of those frames, the earlier
 * phone on a tie; zero-duration phones own no frames.  A step at or past L_b (the steps of a shorter utterance in a batch
 * of T = ceil(max L_b / 8) steps) takes the row of b's last phone with a positive duration, or phone 0 if none has one.
 * So prosody changes are quantised to the PLM's 8-frame steps (128 ms at 16 kHz, hop 256).  The rule is integer-only and
 * the rows are copied as bits, so the expansion is exact.  The ADM's steps are the phones themselves: per-phone duration
 * weights go to mtts_adm_infer_mix_steps_f32 as they are, T = Tp. */

/* mtts_plm_infer_mix_f32 / mtts_plm_infer_mix_range_f32 with weights (B, T, K) at strides (w_sb, w_st).  In a range,
 * target step j reads row j, so any split of [0, T) into consecutive ranges yields the codes and logits of the whole
 * decode.  K in 1..8 (MTTS_ERR_UNSUPPORTED above 8); weights must not be NULL. */
int mtts_plm_infer_mix_steps_f32(const mtts_plm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                                 int32_t B, int32_t T, const float* weights, int64_t w_sb, int64_t w_st,
                                 int64_t* codes_out, float* logits_out, const mtts_sampling* s,
                                 void* workspace, int64_t workspace_bytes, void* stream);
int mtts_plm_infer_mix_steps_range_f32(const mtts_plm* m, int32_t K, const float* tc_latent, int64_t tc_sb,
                                       int32_t tc_ld, int32_t B, int32_t T, const float* weights, int64_t w_sb,
                                       int64_t w_st, int32_t t0, int32_t t1, int64_t* code_state, int64_t* codes_out,
                                       float* logits_out, const mtts_sampling* s, void* workspace,
                                       int64_t workspace_bytes, void* stream);
/* The phone -> PLM step rule above: phone_w (B, Tp, K) device, utterance b at phone_w + b*pw_sb, phone rows K floats
 * apart; durations (B, Tp) int32 device, utterance b at durations + b*dur_sb; out (B, T, K) contiguous.  One CTA per
 * utterance.  1 <= K <= 8 and 1 <= Tp <= 8192 (MTTS_ERR_UNSUPPORTED above the bounds); B <= 0 or T <= 0 does nothing. */
int mtts_mix_step_weights_f32(const float* phone_w, int64_t pw_sb, int32_t Tp, int32_t K, int32_t B,
                              const int32_t* durations, int64_t dur_sb, int32_t T, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * In-context prompting: the PLM decodes the target's codes as the continuation of prompt utterances' latents and codes,
 * the sequences it is trained on (the reference's MegaPLMDataset prepends up to ten same-speaker cuts to every target).
 * A context is P >= 0 rows: latents ctx_tc (Bc, P, tc_dim) and codes ctx_codes (Bc, P) int64 in [0, vq_bins), with Bc = 1
 * (one context for every utterance: batch strides ctx_sb = ctx_codes_sb = 0) or B.  P is the same for every utterance of a
 * call: there is no padding, since the encoder is unmasked and padding rows would change the result.  Target step j
 * (0 <= j < T) is the reference loop's step P + j over the concatenated sequence:
 *   latents [ctx_tc; tc[:, :j+1]] at positions 0 .. P+j of the sinusoidal table, codes [BOS, ctx_codes, c_0 .. c_{j-1}],
 *   and the logits of the last row.
 * That is MegaPLM.infer on cat(ctx_tc, tc) with the first P codes teacher-forced and only the last T steps decoded; P = 0
 * is mtts_plm_infer_f32.  The causal form is the same under the causal mask: the teacher-forced MegaPLM.forward over the
 * concatenation evaluated on its own output, which is what training optimises.  A sampled draw at target step j is keyed by
 * (seed, keys[b], j), not P + j, so the same seed and key give the same noise with and without a context.  codes_out (B, T)
 * and logits_out (optional, (B, T, vq_bins)) hold the target steps only.  The context latents and codes are read from
 * device memory at every call, so a replayed CUDA graph picks up a new context of the same (Bc, P). */
int64_t mtts_plm_infer_ctx_workspace_bytes(const mtts_plm* m, int32_t B, int32_t P, int32_t T);
/* The non-causal decode with a context (s NULL = greedy).  The pe table of m must have >= P + T rows. */
int mtts_plm_infer_ctx_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld, int32_t B, int32_t T,
                           const float* ctx_tc, int64_t ctx_sb, int32_t ctx_ld, const int64_t* ctx_codes, int64_t ctx_codes_sb,
                           int32_t P, int64_t* codes_out, float* logits_out, const mtts_sampling* s, void* workspace,
                           int64_t workspace_bytes, void* stream);
/* Target steps [j0, j1) of it against a caller-owned code state (B, P + T + 1) int64: column 0 holds BOS, columns 1..P the
 * context codes (written by this call when j0 = 0), column P + 1 + j the code of target step j.  Any split of [0, T) into
 * consecutive ranges yields the codes and logits of one mtts_plm_infer_ctx_f32 call.  Same workspace size. */
int mtts_plm_infer_ctx_range_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld, int32_t B,
                                 int32_t T, const float* ctx_tc, int64_t ctx_sb, int32_t ctx_ld, const int64_t* ctx_codes,
                                 int64_t ctx_codes_sb, int32_t P, int32_t j0, int32_t j1, int64_t* code_state,
                                 int64_t* codes_out, float* logits_out, const mtts_sampling* s, void* workspace,
                                 int64_t workspace_bytes, void* stream);
/* Code pins: the range decode with some of its picks fixed, the prosody half of speech editing.  pinned (B, T) int32
 * device, utterance b at pinned + b*pin_sb (NULL pins nothing).  A pin in [0, vq_bins) is written into state column
 * P + 1 + j and into codes_out[b, j] in place of target step j's pick (greedy or sampled: a pinned row draws nothing, and
 * the other rows' draws, keyed by (seed, keys[b], j), do not change); any other value, conventionally -1, leaves the step
 * free, so no out-of-range code can reach the embedding lookup.  Step j reads state columns <= P + j and writes column
 * P + 1 + j only, so a caller may leave out steps at which every utterance is pinned, provided their pins are already in
 * its state: steps below j0 must already be in the caller's state, pinned steps it never enqueues included.  The pins are
 * read from device memory at every call, so a replayed CUDA graph picks up new values.  With every pin free (or pinned
 * NULL) the outputs and launch sequence equal mtts_plm_infer_ctx_range_f32's; P = 0 with NULL context pointers is the
 * plain range decode (mtts_plm_infer_range_f32, or mtts_plm_infer_range_sample_f32 when s is given).  logits_out, when
 * given, holds the model's logits at every enqueued step, pinned ones included: at a pinned step they score the pinned
 * history, i.e. teacher forcing.  Workspace: mtts_plm_infer_ctx_workspace_bytes.  There is no mixed or causal variant. */
int mtts_plm_infer_pinned_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld, int32_t B,
                              int32_t T, const float* ctx_tc, int64_t ctx_sb, int32_t ctx_ld, const int64_t* ctx_codes,
                              int64_t ctx_codes_sb, int32_t P, int32_t j0, int32_t j1, int64_t* code_state,
                              int64_t* codes_out, float* logits_out, const mtts_sampling* s, const int32_t* pinned,
                              int64_t pin_sb, void* workspace, int64_t workspace_bytes, void* stream);
/* The causal decode with a context.  The P context rows run through the stack once, as one teacher-forced causal pass of
 * B*P rows per layer that fills the K/V caches of positions 0..P-1; T single-row steps from position P follow. */
int64_t mtts_plm_decode_causal_ctx_workspace_bytes(const mtts_plm* m, int32_t B, int32_t P, int32_t T);
int mtts_plm_decode_causal_ctx_f32(const mtts_plm* m, const float* tc_latent, int64_t tc_sb, int32_t tc_ld, int32_t B,
                                   int32_t T, const float* ctx_tc, int64_t ctx_sb, int32_t ctx_ld, const int64_t* ctx_codes,
                                   int64_t ctx_codes_sb, int32_t P, int64_t* codes_out, float* logits_out,
                                   const mtts_sampling* s, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Duration interpolation: the ADM decoded from a weighted mean of K prompts' duration predictions, the rhythm half of
 * Mega-TTS 2's prosody (the PLM mix above is the pitch and energy half).  Utterance b has K >= 1 sources; source k is a
 * latent tc^(k)[b] (T, tc_dim), source 0 conventionally the target prompt's, all with the same T, and b has a weight row
 * w[b, 0..K) (fp32, every weight >= 0 and finite, row sum > 0; the host never reads it, callers validate it).  All K
 * sources share one raw-duration history p[b, 0..T], p[b, 0] = 0.  At step t:
 *   1. each source runs the reference-faithful step (mtts_adm_infer_f32's non-causal full recompute over t+1 positions,
 *      the last layer pruned to the last row) over its own latent and the shared history -> readout y^(k);
 *   2. w^_k = w_k / sum_k w_k, the sum in fp32 in k order; sources with w_k = 0 are skipped, even when y^(k) is not finite;
 *   3. r = w^_k0 * y^(k0) for the first positive weight k0, then r = fmaf(w^_k, y^(k), r) for the later positive weights in
 *      k order, all in fp32.  With exactly one positive weight w^ = w / w = 1, so r is that source's y bit for bit
 *      (-0 included: starting from fmaf(1, y, 0) would turn -0 into +0), and a one-hot row decodes exactly what
 *      mtts_adm_infer_f32 decodes from that source alone.  A row without a positive weight gives r = 0, the empty sum;
 *   4. p[b, t+1] = r: the mixed value is what the next step reads back, as the single-source decode feeds back its own raw
 *      prediction.
 * The durations are mtts_adm_infer_f32's, from the mixed raw values: (r + 0.5) -> int32 -> clamp(1, 128).
 * Why the mean: the ADM is trained with an MSE loss, so each y^(k) estimates the conditional mean of the next duration
 * given source k; the weighted mean of the sources' means is the mean of their mixture.  K <= 8 (MTTS_ERR_UNSUPPORTED
 * above). */

/* The mix readout of one step: xl (K*B, D) contiguous, row k*B + b = the last encoder row of source k of utterance b;
 * w_predict (D); weights (B, K) contiguous, device (NULL only when K = 1: weight 1).  out[b * ld_out] = r_b; y_out
 * optional, y_out[(k*B + b) * ld_y] = y^(k)_b for every source, weighted or not.  y is the dot product of
 * mtts_adm_infer_f32's readout, computed the same way, so y_out equals what that readout writes for the same row. */
int mtts_adm_readout_mix_f32(const float* xl, int32_t D, const float* w_predict, int32_t K, int32_t B, const float* weights,
                             float* out, int64_t ld_out, float* y_out, int64_t ld_y, void* stream);
/* The mixed decode.  tc_latent is the (K*B, T, tc_dim) stack of the sources, row k*B + b = source k of utterance b (batch
 * stride tc_sb, row stride tc_ld); weights (B, K) device (NULL only when K = 1); dur_out (B, T) int32; raw_out optional
 * (B, T), the mixed raw values; raw_src_out optional (K, B, T), every source's readout y^(k) at every step.  Each step
 * runs the encoder once over the K*B rows, then the mix readout.  The weights are read from device memory at every step,
 * so a replayed CUDA graph picks up new values.  With K = 1 and weights NULL the launch sequence is mtts_adm_infer_f32's
 * (raw_src_out NULL) and the outputs equal it bit for bit. */
int64_t mtts_adm_infer_mix_workspace_bytes(const mtts_adm* m, int32_t K, int32_t B, int32_t T);
int mtts_adm_infer_mix_f32(const mtts_adm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                           int32_t B, int32_t T, const float* weights, int32_t* dur_out, float* raw_out,
                           float* raw_src_out, void* workspace, int64_t workspace_bytes, void* stream);
/* mtts_adm_infer_mix_f32 with weights (B, T, K) at strides (w_sb, w_st), T = Tp: step t, the duration of phone t, mixes
 * by row t (the schedule section above states the rule).  weights must not be NULL. */
int mtts_adm_infer_mix_steps_f32(const mtts_adm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                                 int32_t B, int32_t T, const float* weights, int64_t w_sb, int64_t w_st,
                                 int32_t* dur_out, float* raw_out, float* raw_src_out, void* workspace,
                                 int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Duration control: phone durations pinned inside the ADM loop, and durations fitted to a speaking rate and a target
 * length.
 *
 * Pins.  pinned (B, T) int32 device, utterance b at pinned + b*pin_sb; pinned[b, t] >= 1 pins phone t of b to that many
 * frames, a value < 1 (conventionally -1) leaves it free.  At step t the value written into the raw history p[b, t+1] is
 * (float)pinned[b, t] for a pinned phone and the readout (plain, mixed or scheduled) otherwise, so the rest of the
 * utterance is decoded after the pinned values.  The reference trains the ADM teacher-forced on integer frame counts cast
 * to float and skips cuts with a duration >= 128, so a pin in 1..127 is the kind of history the model was trained on.
 * The durations follow from the history as before; for p in 1..127, (p + 0.5) truncates to p, so a pinned phone comes
 * out exactly p, and raw_out holds p there.  raw_src_out keeps every source's own readout, pinned or not.
 * mtts_adm_infer_pinned_f32 takes mtts_adm_infer_mix_steps_f32's arguments (weights NULL only when K = 1: then with
 * raw_src_out NULL it is the plain decode; (B, K) weights are w_sb = K, w_st = 0) and the pins; pinned NULL pins
 * nothing.  The pins are read from device memory at every call, so a replayed CUDA graph picks up new pins.  With every
 * pin < 1 the outputs equal the unpinned entry's bit for bit, with the same launch sequence.  Workspace:
 * mtts_adm_infer_mix_workspace_bytes.  The causal decode takes no pins. */
int mtts_adm_infer_pinned_f32(const mtts_adm* m, int32_t K, const float* tc_latent, int64_t tc_sb, int32_t tc_ld,
                              int32_t B, int32_t T, const float* weights, int64_t w_sb, int64_t w_st, int32_t* dur_out,
                              float* raw_out, float* raw_src_out, const int32_t* pinned, int64_t pin_sb, void* workspace,
                              int64_t workspace_bytes, void* stream);
/* The fit.  raw (B, Tp) fp32 device, utterance b at raw + b*raw_sb: the ADM's raw values.  scale optional (NULL = 1):
 * c[b, i] at scale + b*scale_sb + i*scale_st, so strides (0, 0) give one scalar, (1, 0) one value per utterance and
 * (Tp, 1) one per phone.  pinned optional, as above (pinned phones get their pin).  total optional (B,) int32 device.
 * dur_out (B, Tp) int32, utterance b at dur_out + b*dur_sb.  For utterance b, F is its set of free phones and
 * w_i = fl32(raw_i * c_i), a non-finite w or a w <= 0 counting as 0.
 *   No total: free phone i gets clamp(trunc(fl32(w_i + 0.5)), 1, 128), the ADM's own rounding applied to w; with c = 1
 *   that is mtts_adm_infer_f32's dur_out, bit for bit.  For finite w the fp32 add never moves the truncation across an
 *   integer, so this is clamp(floor(w_i + 1/2), 1, 128) exactly.
 *   Total L_b: N = L_b - sum of pins - |F| frames above one per free phone, 0 <= N <= 127 |F| (the feasible totals are
 *   [|F| + sum pins, 128 |F| + sum pins]; the host validates them, the device clamps N into that range).  The candidates
 *   are v_ik = w_i / (k + 1/2), i in F, k = 1..127; the N largest are taken, ordered by value descending, then phone
 *   index ascending, and free phone i gets 1 + (the number of its candidates taken).  This is Sainte-Lague apportionment
 *   with per-phone bounds 1 and 128: the same as rounding w_i / theta for one common theta, so theta = 1 is the no-total
 *   rule and durations that already sum to L_b come back unchanged.  Candidates compare exactly, as w_i (2m+1) against
 *   w_j (2k+1).
 * One CTA per utterance; 1 <= Tp <= 8192 (MTTS_ERR_UNSUPPORTED above); B <= 0 does nothing.  Device-only, so it can be
 * captured in a CUDA graph. */
int mtts_fit_durations_f32(const float* raw, int64_t raw_sb, int32_t Tp, int32_t B, const float* scale, int64_t scale_sb,
                           int64_t scale_st, const int32_t* pinned, int64_t pin_sb, const int32_t* total, int32_t* dur_out,
                           int64_t dur_sb, void* stream);

/* ConvNet family (modules/convnet.py).  One ConvBlock = ReLU -> Conv1d(C,C,k,same) -> LN(C). */
typedef struct { const float *w, *b, *ln_g, *ln_b; const void* w_tc; } mtts_conv_block;   /* w packed (k,C,C); w_tc (3,k,C,C) bf16 or NULL */

typedef struct {
  int32_t in_channels, out_channels, hidden, k, n_stacks, n_blocks;
  int32_t engine;                      /* 0: fp32 FFMA; wgmma for the eligible convs: 1 = BF16X3, 2 = F16X2, 3 = F16 */
  const float *w_first, *b_first;      /* packed (k, Cin, hidden) */
  const float *w_last, *b_last;        /* packed (k, hidden, Cout) */
  const mtts_conv_block* blocks;       /* HOST array [n_stacks*n_blocks] */
} mtts_convnet;
/* ConvNet.forward (convnet.py:115-119): x (B,T,Cin) -> y (B,T,Cout), channels-last */
int64_t mtts_convnet_workspace_bytes(const mtts_convnet* n, int32_t B, int32_t T);
int mtts_convnet_forward_f32(const mtts_convnet* n, const float* x, int64_t x_sb, int32_t ldx,
                             float* y, int64_t y_sb, int32_t ldy, int32_t B, int32_t T,
                             void* workspace, int64_t workspace_bytes, void* stream);

typedef struct {
  int32_t in_channels, out_channels, hidden, k, n_layers, n_stacks, n_blocks;
  int32_t engine;
  int32_t middle_kind;                 /* 0: MaxPool1d(middle_k, ceil) ; 1: strided Conv1d(k=middle_k, stride, pad) */
  int32_t middle_k, middle_stride, middle_pad;
  const float *w_middle, *b_middle;    /* packed (middle_k, hidden, hidden) when middle_kind == 1 */
  const float *w_first, *b_first, *w_last, *b_last;
  const mtts_conv_block* blocks;       /* HOST array [n_layers][2][n_stacks*n_blocks] */
} mtts_convnet_double;
/* ConvNetDouble.forward (convnet.py:202-210): x (B,T,Cin) -> y (B,T_mid,Cout) */
int32_t mtts_convnet_double_out_len(const mtts_convnet_double* n, int32_t T);
int64_t mtts_convnet_double_workspace_bytes(const mtts_convnet_double* n, int32_t B, int32_t T);
int mtts_convnet_double_forward_f32(const mtts_convnet_double* n, const float* x, int64_t x_sb, int32_t ldx,
                                    float* y, int64_t y_sb, int32_t ldy, int32_t B, int32_t T,
                                    void* workspace, int64_t workspace_bytes, void* stream);

/* HiFi-GAN V1 generator (speechbrain HIFIGAN.decode_batch, called at
 * models/megatts2.py:370-372).  mel (B, T, 80) channels-last -> wav (B, 256*(T+2*pad)). */
typedef struct {
  const float *w1[3], *b1[3], *w2[3], *b2[3]; int32_t k; int32_t dil[3];
  const void *w1_tc[3], *w2_tc[3];     /* (3, k, C, C) bf16 planes or NULL */
} mtts_hifigan_resblock;
typedef struct {
  int32_t in_channels, ch0, n_ups, n_kernels, inference_padding;
  int32_t engine;
  int32_t up_factor[4], up_kernel[4];
  const float *w_pre, *b_pre;          /* packed (7, 80, ch0) */
  const float *w_up[4], *b_up[4];      /* packed (2, Cin, s*Cout), bias expanded to (s*Cout) */
  const void* w_up_tc[4];              /* (3, 2, s*Cout, Cin) bf16 planes or NULL */
  const mtts_hifigan_resblock* resblocks;  /* HOST array [n_ups*n_kernels] */
  const float *w_post, *b_post;        /* packed (7, C_last, 1) */
} mtts_hifigan;
int64_t mtts_hifigan_workspace_bytes(const mtts_hifigan* h, int32_t B, int32_t T);
int mtts_hifigan_forward_f32(const mtts_hifigan* h, const float* mel, int64_t mel_sb, int32_t mel_ld,
                             int32_t B, int32_t T, float* wav, int64_t wav_sb,
                             void* workspace, int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MEGATTS2_B200_H */
