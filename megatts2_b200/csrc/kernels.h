// Internal (C++) entry points shared by the drivers and the C ABI.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace mtts {
// Tensor-core operand formats ("planes": 2-byte elements in the activation's own (B, Tp, C) layout):
//   fmt 0  bf16x3: x = p0 + p1 + p2 (three bf16 terms, to ~2^-24); six MMAs per product
//   fmt 1  f16x2 : x = p0 + p1 * 2^-11 (two fp16 terms, the residual stored SCALED by 2^11 so it keeps the
//                  magnitude - and the normal range - of x; 22 significant bits); three MMAs per product
//                  (x0w0 | x0w1' + x1'w0, the second accumulator scaled by 2^-11 in the epilogue).  fp16 range:
//                  |x| > 65504 cannot be represented - the split then poisons the value (inf/NaN propagate to the
//                  output) and raises the caller-registered overflow flag (mtts_tc_overflow_bind).  At the low
//                  end p0 is subnormal below 2^-14 and both terms are zero below about 2^-35: the representation
//                  error is |x - x^| <= 2^-22 |x| + 2^-36, so tiny operands lose precision (training gradients run
//                  on bf16x3 for that reason).
//   fmt 2  f16   : x ~ p0 = fp16(x) (one fp16 plane, round-to-nearest; 11 significant bits); ONE MMA per product.
//                  Not fp32-grade: the opt-in half-precision inference engine.  Same fp16 range and flag as f16x2.
// The number of planes of fmt is 3 - fmt.
enum { MTTS_TC_BF16X3 = 0, MTTS_TC_F16X2 = 1, MTTS_TC_F16 = 2 };
constexpr float F16X2_SCALE = 2048.0f;           // 2^11
constexpr float F16X2_INV_SCALE = 1.0f / 2048.0f;

// optional plane output of a producer kernel (feeds the tensor-core engine without a split pass)
struct PlanesOut {
  __nv_bfloat16* p;      // plane 0; planes 1 (, 2) follow at +stride (, +2*stride) elements; 2-byte elements of `fmt`
  int64_t stride;
  int ld;                // row stride (elements)
  int act;               // activation applied to the planes copy (the consumer's pre-activation)
  float slope;
  int fmt;               // MTTS_TC_BF16X3 | MTTS_TC_F16X2 | MTTS_TC_F16
  int32_t* ovf;          // fp16 range flag (device, may be null)
};

// 4 consecutive elements -> one 8-byte store per plane
__device__ __forceinline__ void store_planes4(__nv_bfloat16* planes, int64_t plane_stride, int64_t off, const float* v,
                                              int fmt = MTTS_TC_BF16X3, int32_t* ovf = nullptr) {
  if (fmt == MTTS_TC_F16X2 || fmt == MTTS_TC_F16) {
    // two elements per conversion instruction (cvt.rn.f16x2.f32); the range check is one NaN-propagating max per element
    const __half2 h01 = __floats2half2_rn(v[0], v[1]), h23 = __floats2half2_rn(v[2], v[3]);   // +-inf beyond the fp16 range
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&h01);
    o.y = *reinterpret_cast<const uint32_t*>(&h23);
    *reinterpret_cast<uint2*>(planes + off) = o;
    if (fmt == MTTS_TC_F16X2) {
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      const __half2 l01 = __floats2half2_rn((v[0] - f01.x) * F16X2_SCALE, (v[1] - f01.y) * F16X2_SCALE);   // exact difference,
      const __half2 l23 = __floats2half2_rn((v[2] - f23.x) * F16X2_SCALE, (v[3] - f23.y) * F16X2_SCALE);   // exact scaling
      o.x = *reinterpret_cast<const uint32_t*>(&l01);
      o.y = *reinterpret_cast<const uint32_t*>(&l23);
      *reinterpret_cast<uint2*>(planes + plane_stride + off) = o;
    }
    if (ovf) {
      float m;
      asm("{\n\t.reg .f32 t0, t1, t2, t3;\n\tabs.f32 t0, %1;\n\tabs.f32 t1, %2;\n\tabs.f32 t2, %3;\n\tabs.f32 t3, %4;\n\t"
          "max.NaN.f32 t0, t0, t1;\n\tmax.NaN.f32 t2, t2, t3;\n\tmax.NaN.f32 %0, t0, t2;\n\t}"
          : "=f"(m) : "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]));
      if (!(m <= 65504.0f)) *ovf = 1;                                  // also NaN
    }
    return;
  }
  // bf16x3: round-to-nearest at every step
  __nv_bfloat16 p[3][4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float a = v[e];
    p[0][e] = __float2bfloat16_rn(a);
    a -= __bfloat162float(p[0][e]);
    p[1][e] = __float2bfloat16_rn(a);
    a -= __bfloat162float(p[1][e]);
    p[2][e] = __float2bfloat16_rn(a);
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    uint2 o;
    o.x = (uint32_t)__bfloat16_as_ushort(p[q][0]) | ((uint32_t)__bfloat16_as_ushort(p[q][1]) << 16);
    o.y = (uint32_t)__bfloat16_as_ushort(p[q][2]) | ((uint32_t)__bfloat16_as_ushort(p[q][3]) << 16);
    *reinterpret_cast<uint2*>(planes + q * plane_stride + off) = o;
  }
}
// the overflow flag registered for the current device (null if none) and the current device's id / SM count
int32_t* tc_ovf_ptr();
int cur_device();
int cur_device_sms();
int set_sm_limit(int n);
int set_launch_policy(int sm_limit, int allow_pairs, int allow_pdl);
int tc_plan_query(int sms, int B, int T, int Cin, int Cout, int k, int dil, int fmt, int64_t partial_bytes, int ln_rides, int32_t* out5);
int tc_plan_query_ex(int sms, int B, int T, int Cin, int Cout, int k, int dil, int fmt, int64_t partial_bytes, int ln_rides,
                     int allow_pairs, int32_t* out7);
// engine 1 | 2 | 3 (bf16x3 | f16x2 | f16) -> operand format; the one place that maps engines to formats
static inline int tc_fmt_of_engine(int engine) {
  return engine == 3 ? MTTS_TC_F16 : engine == 2 ? MTTS_TC_F16X2 : MTTS_TC_BF16X3;
}
// engines whose operands are limited to the fp16 range (f16x2, f16): the only ones whose attention may use attn_tc.cu
static inline int engine_allows_f16_operands(int engine) { return engine == 2 || engine == 3; }
int layernorm_ex(const float* x, int ldx, const float* gamma, const float* beta, const float* res, int ldr, float* y,
                 int ldy, int64_t rows, int C, float eps, int post_act, int accumulate, PlanesOut po, cudaStream_t st);
int conv1d_ffma(const mtts_conv_params& p, cudaStream_t st);
// conv1d_ffma()'s routing as a pure host function: ffma_check holds the argument checks, ffma_plan picks the kernel
// (MTTS_FFMA_*) for an SM budget of `sms`: its output tile (BM x BN; 256 x 1 for the Cout = 1 kernels), the K split
// (splits, 16-channel slices per split; 1, 0 unsplit), the 16-byte load / store paths and the dynamic shared memory
struct FfmaPlan { int kernel, bm, bn, splits, kk_per_split, vec_a, vec_b, vec_y; size_t smem; };
int ffma_check(const mtts_conv_params& p);
FfmaPlan ffma_plan(const mtts_conv_params& p, int sms);
int ffma_plan_query(const mtts_conv_params* p, int sms, int32_t* out8);
int conv1d(const mtts_conv_params& p, cudaStream_t st);   // engine dispatch (FFMA today)
bool conv_tc_eligible(const mtts_conv_params& p);
// Optional LayerNorm of the rows a split-K tap-GEMM has just reduced (the dense layers of the AR loops' early steps): the
// reduction kernel then also normalises each finished row and writes the next layer's operand planes, which saves the
// separate LayerNorm launch.  `done` is set when the fused kernel ran; the caller launches LayerNorm itself otherwise.
struct LnFuse {
  const float* gamma; const float* beta; float eps;
  PlanesOut po;
  int done;
};
int conv_tc(const mtts_conv_params& p, cudaStream_t st, LnFuse* ln = nullptr);
// launch plumbing shared by the tensor-core kernels (conv_tc.cu): the cached TMA descriptor of a 2-byte-element tensor
// (d2, d1, d0) with box (1, b1, b0) and SWB-byte swizzle (rank 2 when d2 == 0), and the max-dynamic-shared-memory
// attribute of a kernel, raised once per device (slot: a bit of the per-device table, < 32)
int cmap_get(const void* p, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1, int swb, int fmt, CUtensorMap* out);
int tc_smem_attr(const void* kernel, int slot, int bytes);
// One HiFi-GAN ResBlock1 dilation step y = (x + conv2(leaky(conv1_dil(leaky(x))))) * out_scale (+ y if accumulate), reflect
// padding, in one launch (resblock_tc.cu); w1_tc / w2_tc are the convs' packed planes of `fmt`.  Bit-identical to the
// two-launch tap-GEMM flow.  Only where resblock_tc_eligible holds: C 32 | 64, f16x2 | f16, T > the two halos, B*T >= 128.
bool resblock_tc_eligible(int B, int T, int C, int k, int dil, int fmt);
int resblock_pair_tc(const float* x, float* y, const void* w1_tc, const float* b1, const void* w2_tc, const float* b2,
                     int B, int T, int C, int k, int dil, float out_scale, int accumulate, int fmt, cudaStream_t st);
int halo_fill(void* planes_base, int B, int T, int C, int hl, int hr, int pad_mode, int fmt, cudaStream_t st);
int64_t linear_tc_scratch_bytes(int64_t rows_cap, int K);
int linear_tc(const float* x, int ldx, int64_t M, int K, const void* w_planes, int N, const float* bias,
              const float* res, int ldr, float* y, int ldy, int pre_act, float pre_slope, int post_act,
              float out_scale, void* scratch, int64_t scratch_bytes, int64_t rows_cap, int fmt, cudaStream_t st);
int split_planes(const float* x, int ldx, int64_t rows, int C, void* planes, int fmt, cudaStream_t st);
int split_pad(const float* x, int64_t x_sb, int ldx, int B, int T, int C, int hl, int hr, int pad_mode, int act, float slope,
              void* planes_base, int fmt, cudaStream_t st);
int tc_overflow_bind(int32_t* flag);
int mask_tail(float* x, int B, int rows, int L, const int32_t* keep, cudaStream_t st);
// ragged row copy / fill, one launch for B batch rows (mtts_copy_row_segments)
int copy_row_segments(const void* src, int64_t src_sb, int64_t src_st, int64_t src_rows, void* dst, int64_t dst_sb,
                      int64_t dst_st, int64_t dst_rows, int row_bytes, const int32_t* src_off, const int32_t* dst_off,
                      const int32_t* n, int B, int n_max, uint32_t fill_word, cudaStream_t st);
int layernorm(const float* x, int ldx, const float* gamma, const float* beta, const float* res, int ldr, float* y,
              int ldy, int64_t rows, int C, float eps, int post_act, int accumulate, cudaStream_t st);
// timbre mix: rows r = b T + t of K sources y + k y_ks mixed by the weight rows w + b w_sb + t w_st, then LayerNorm +
// post_act into out (mtts_mix_layernorm_f32)
int mix_layernorm(const float* y, int64_t y_ks, int ldy, int K, const float* w, int64_t w_sb, int64_t w_st, int T,
                  const float* gamma, const float* beta, float* out, int ldo, int64_t rows, int C, float eps, int post_act,
                  cudaStream_t st);
// allow_f16_operands: the caller's engine accepts fp16-range operands, so long sequences may use attn_tc.cu (f16x2 planes)
int attention(const mtts_attn_params& p, bool allow_f16_operands, cudaStream_t st);
// attention()'s routing as a pure host function: attn_check holds the argument checks, attn_plan picks the kernel
// (MTTS_ATTN_*, or ATTN_UNSUPPORTED for a head dim without one), and for the fp32 kernel its attn_kernel<dh / 32, RW, NW,
// KPL> instantiation and whether it takes the 16-byte load path (vec); pair_min: shortest AR step routed to the tensor
// cores (1 << 30: off)
constexpr int ATTN_UNSUPPORTED = -2;
struct AttnPlan { int kernel, dh, rw, nw, kpl, vec; };
int attn_check(const mtts_attn_params& p);
AttnPlan attn_plan(const mtts_attn_params& p, bool allow_f16_operands, int pair_min);
int attention_plan_query(const mtts_attn_params* p, int allow_f16_operands, int pair_min, int32_t* out6);
bool attention_tc_eligible(const mtts_attn_params& p);
int attention_tc(const mtts_attn_params& p, cudaStream_t st);
bool attention_tc_pair_eligible(const mtts_attn_params& p);
int attention_tc_pair(const mtts_attn_params& p, cudaStream_t st);
int set_attention_pair_min(int n);   // AR-step routing to attention_tc_pair (attn_tc.cu)
int vq_argmin(const float* x, int ldx, const float* embed, int64_t N, int D, int K, int64_t* idx, cudaStream_t st);
int vq_gather(const int64_t* idx, int idx_ld, const float* embed, int D, int K, int B, int T_out, int repeat, float* y,
              int64_t y_sb, int ldy, cudaStream_t st);
int maxpool_time(const float* x, int64_t x_sb, int ldx, float* y, int64_t y_sb, int ldy, int B, int T, int C, int k,
                 cudaStream_t st);
int embed_pe(const int64_t* ids, int ids_ld, const float* table, int vocab, int D, const float* pe, float alpha,
             int pe_offset, int B, int T, float* y, int64_t y_sb, int ldy, cudaStream_t st);
int add_pe(const float* x, int64_t x_sb, int ldx, const float* pe, float alpha, int B, int T, int D, float* y,
           int64_t y_sb, int ldy, cudaStream_t st);
int length_regulate(const float* x, int64_t x_sb, int ldx, const int32_t* dur, int dur_ld, int B, int Tp, int D,
                    int L_out, float* y, int64_t y_sb, int ldy, int32_t* totals, cudaStream_t st);
int copy_strided(const float* x, int64_t x_sb, int64_t x_st, int64_t x_sc, float* y, int64_t y_sb, int64_t y_st,
                 int64_t y_sc, int B, int T, int C, int pad_rep, cudaStream_t st);
int mel_spectrogram(const float* wav, int64_t wav_sb, int B, int L, const int32_t* lens, const float* window,
                    const float* fb_w, const int32_t* fb_off, const int32_t* fb_start, int n_mels, float clamp_min,
                    float* out, int64_t out_sb, int64_t out_sm, int64_t out_sf, cudaStream_t st);
// AR-loop helpers
// latent row r reads code row r % B_codes (B_codes = B: one code row per latent row; fewer: sources sharing a history).
// With a context (P > 0), positions s < P read their latent from ctx (batch stride ctx_sb, 0 = one context for every row,
// row stride ctx_ld) and positions s >= P read tc row s - P.
int plm_build_input(const float* tc, int64_t tc_sb, int tc_ld, int tc_dim, const int64_t* codes, int codes_ld,
                    int B_codes, const float* emb, int vq_dim, int vocab, const float* pe, float alpha, int B, int S,
                    float* X, cudaStream_t st, const float* ctx = nullptr, int64_t ctx_sb = 0, int ctx_ld = 0, int P = 0);
// y[b * ldy + p] = x[b * x_sb + p], p < n (int64 codes; x_sb = 0 broadcasts one row)
int copy_codes(const int64_t* x, int64_t x_sb, int64_t* y, int64_t ldy, int B, int n, cudaStream_t st);
// additive causal mask (T, T): 0 where key <= query, -inf above the diagonal
int causal_mask(float* m, int T, cudaStream_t st);
// pin (optional, code pins of the PLM decode): row r writes pin[r * pin_sb] instead of its pick when that value is in
// [0, V); any other value leaves the row free
int argmax_rows(const float* x, int64_t ldx, int V, int rows, int64_t* out_a, int64_t lda, int64_t* out_b, int64_t ldb,
                cudaStream_t st, const int32_t* pin = nullptr, int64_t pin_sb = 0);
// opt-in sampler (sample.cu): validates s against V, then draws one code per row (argmax_rows when temperature == 0 or
// top_k == 1); sampling_check alone lets a driver reject bad parameters before it enqueues anything.  pin as argmax_rows';
// a pinned row draws nothing and leaves the other rows' draws unchanged
int sampling_check(const mtts_sampling* s, int V);
int sample_rows(const float* x, int64_t ldx, int V, int rows, int step, const mtts_sampling& s, int64_t* out_a,
                int64_t lda, int64_t* out_b, int64_t ldb, cudaStream_t st, const int32_t* pin = nullptr,
                int64_t pin_sb = 0);
int philox4x32_10_words(const uint32_t* ctr, const uint32_t* key, uint32_t* out, int64_t n, cudaStream_t st);
// prosody mix (sample.cu): l (B, V) from K source rows per utterance and the weight rows w + b ldw; mix_logprob_check
// validates (V, K) before a driver enqueues anything
int mix_logprob_check(int V, int K);
int mix_logprob_rows(const float* x, int64_t ldx, int V, int K, int B, const float* w, int64_t ldw, float* out,
                     int64_t ldo, cudaStream_t st);
int fill_i64(int64_t* p, int64_t stride, int n, int64_t v, cudaStream_t st);
int fill_f32(float* p, int64_t stride, int n, float v, cudaStream_t st);
// latent row r reads history row r % B_hist (B_hist = B: one history per latent row; fewer: sources sharing a history)
int adm_build_input(const float* tc_emb, int64_t te_sb, int te_ld, int tc_emb_dim, const float* praw, int p_ld,
                    int B_hist, const float* w_dt, int emb_dim, const float* pe, float alpha, int B, int S, float* X,
                    cudaStream_t st);
// pin (optional): the pins of this step's phone, utterance b at pin[b * pin_sb]; a pin >= 1 is fed back in place of the
// readout (mtts_adm_infer_pinned_f32)
int adm_readout(const float* xl, int D, const float* w, int B, float* praw, int p_ld, int s_next, cudaStream_t st,
                const int32_t* pin = nullptr, int64_t pin_sb = 0);
// duration mix: r_b from the K rows k*B + b of xl and the weight rows weights + b ldw into out[b * ld_out]; y_out
// (optional) gets every source's readout.  adm_mix_check validates K before a driver enqueues anything.
int adm_mix_check(int K);
int adm_readout_mix(const float* xl, int D, const float* w, int K, int B, const float* weights, int64_t ldw, float* out,
                    int64_t ld_out, float* y_out, int64_t ld_y, cudaStream_t st, const int32_t* pin = nullptr,
                    int64_t pin_sb = 0);
// per-phone mix weights (B, Tp, K) -> per-PLM-step weights (B, T, K) by the durations (mtts_mix_step_weights_f32)
int mix_step_weights(const float* pw, int64_t pw_sb, int Tp, int K, int B, const int32_t* dur, int64_t dur_sb, int T,
                     float* out, cudaStream_t st);
int adm_finalize(const float* praw, int p_ld, int B, int T, int32_t* dur, float* raw_out, cudaStream_t st);
// raw ADM values -> durations fitted to a scale, pins and a target total (mtts_fit_durations_f32)
int fit_durations(const float* raw, int64_t raw_sb, int Tp, int B, const float* scale, int64_t sc_sb, int64_t sc_st,
                  const int32_t* pin, int64_t pin_sb, const int32_t* total, int32_t* dur, int64_t dur_sb, cudaStream_t st);

// convenience: dense linear layer  Y[M,N] = act(X[M,K] W + b) (+ res)
inline mtts_conv_params linear_params(const float* x, int ldx, const float* w, const float* bias, float* y, int ldy,
                                      int64_t M, int K, int N) {
  mtts_conv_params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.ldx = ldx; p.x_batch_stride = 0;
  p.w = w; p.bias = bias;
  p.y = y; p.ldy = ldy; p.y_batch_stride = 0;
  p.B = 1; p.Tin = (int32_t)M; p.Tout = (int32_t)M; p.Cin = K; p.Cout = N;
  p.k = 1; p.stride = 1; p.dil = 1; p.pad = 0; p.pad_mode = MTTS_PAD_ZERO;
  p.out_scale = 1.0f;
  return p;
}
// "same" stride-1 conv over (B, T, Cin) -> (B, T, Cout), contiguous buffers
inline mtts_conv_params conv_same_params(const float* x, const float* w, const float* bias, float* y, int B, int T,
                                         int Cin, int Cout, int k, int dil, int pad_mode) {
  mtts_conv_params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.ldx = Cin; p.x_batch_stride = (int64_t)T * Cin;
  p.w = w; p.bias = bias;
  p.y = y; p.ldy = Cout; p.y_batch_stride = (int64_t)T * Cout;
  p.B = B; p.Tin = T; p.Tout = T; p.Cin = Cin; p.Cout = Cout;
  p.k = k; p.stride = 1; p.dil = dil; p.pad = dil * (k - 1) / 2; p.pad_mode = pad_mode;
  p.out_scale = 1.0f;
  return p;
}
}  // namespace mtts
