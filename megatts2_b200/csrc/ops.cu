// HBM-bound and small kernels of the synthesis path: LayerNorm, attention (fp32),
// VQ search / gather, max-pool, embeddings + sine PE, length regulator, layout copies,
// and the per-step helpers of the PLM / ADM autoregressive loops.
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include <atomic>

#include "kernels.h"

namespace mtts {

// ------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, three passes over a row that stays in L1 (C <= 4096 floats).
// x / res may alias y (same element is read then written by the same lane only).
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* x, int ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
                 const float* res, int ldr, float* y, int ldy, int64_t rows, int C, float eps,
                 int post_act, int accumulate, int vec, const PlanesOut po) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * ldx;
  float s = 0.f;
  if (vec) {
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(xr + c);
      s += (v.x + v.y) + (v.z + v.w);
    }
  } else {
    for (int c = lane; c < C; c += 32) s += xr[c];
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
  if (vec) {
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(xr + c);
      const float a = v.x - mean, b = v.y - mean, d = v.z - mean, e = v.w - mean;
      q += (a * a + b * b) + (d * d + e * e);
    }
  } else {
    for (int c = lane; c < C; c += 32) {
      const float a = xr[c] - mean;
      q += a * a;
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
  float* yr = y ? y + row * ldy : nullptr;
  const float* rr = res ? res + row * ldr : nullptr;
  if (vec) {
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(xr + c);
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c));
      float o[4] = {(v.x - mean) * rstd * g.x + bb.x, (v.y - mean) * rstd * g.y + bb.y,
                    (v.z - mean) * rstd * g.z + bb.z, (v.w - mean) * rstd * g.w + bb.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = act_apply(o[e], post_act, 0.f);
      if (rr) {
        const float4 r = *reinterpret_cast<const float4*>(rr + c);
        o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
      }
      if (accumulate) {
        const float4 r = *reinterpret_cast<const float4*>(yr + c);
        o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
      }
      if (yr) *reinterpret_cast<float4*>(yr + c) = make_float4(o[0], o[1], o[2], o[3]);
      if (po.p) {
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = act_apply(o[e], po.act, po.slope);
        store_planes4(po.p, po.stride, row * po.ld + c, o, po.fmt, po.ovf);
      }
    }
  } else {
    for (int c = lane; c < C; c += 32) {
      float o = act_apply((xr[c] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c), post_act, 0.f);
      if (rr) o += rr[c];
      if (accumulate) o += yr[c];
      if (yr) yr[c] = o;
    }
  }
}

// LayerNorm of one register-resident row v (C = 128*NV, lane l holds elements i*128 + 4l .. +3) and what follows it:
// post-activation, + res, + y_old, the y store and the operand planes.  Every register-resident LayerNorm calls this one
// function, so a row that reaches it by another path (mix_layernorm_kernel) is normalised with the same arithmetic.
template <int NV>
__device__ __forceinline__ void layernorm_row(const float4 (&v)[NV], int lane, int64_t row, const float* __restrict__ gamma,
                                              const float* __restrict__ beta, const float* res, int ldr, float* y, int ldy,
                                              float eps, int post_act, int accumulate, const PlanesOut& po) {
  constexpr int C = 128 * NV;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, d = v[i].z - mean, e = v[i].w - mean;
    q += (a * a + b * b) + (d * d + e * e);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
  float* yr = y ? y + row * ldy : nullptr;
  const float* rr = res ? res + row * ldr : nullptr;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * 128 + lane * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c));
    float o[4] = {(v[i].x - mean) * rstd * g.x + bb.x, (v[i].y - mean) * rstd * g.y + bb.y,
                  (v[i].z - mean) * rstd * g.z + bb.z, (v[i].w - mean) * rstd * g.w + bb.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = act_apply(o[e], post_act, 0.f);
    if (rr) {
      const float4 r = *reinterpret_cast<const float4*>(rr + c);
      o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
    }
    if (accumulate) {
      const float4 r = *reinterpret_cast<const float4*>(yr + c);
      o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
    }
    if (yr) *reinterpret_cast<float4*>(yr + c) = make_float4(o[0], o[1], o[2], o[3]);
    if (po.p) {
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = act_apply(o[e], po.act, po.slope);
      store_planes4(po.p, po.stride, row * po.ld + c, o, po.fmt, po.ovf);
    }
  }
}

// Register-resident variant for the row widths of the path (C = 128*NV, NV float4 per lane): one global read
// of the row (NV independent 128-bit loads in flight), two shuffle reductions, one write.
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_reg_kernel(const float* x, int ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const float* res, int ldr, float* y, int ldy, int64_t rows, float eps, int post_act,
                     int accumulate, const PlanesOut po) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * ldx;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(xr + i * 128 + lane * 4);
  layernorm_row<NV>(v, lane, row, gamma, beta, res, ldr, y, ldy, eps, post_act, accumulate, po);
}

// Timbre mix (the contract is stated with mtts_mix_layernorm_f32 in include/megatts2_b200.h): one warp per row r = b T + t
// of K sources y + k y_ks, whose weight row is W + b w_sb + t w_st.  The row is mixed by adm_readout_mix_kernel's rule,
// element by element (the first positive term w^ y, the later ones fmaf(w^, y, acc) in k order; sources without a
// positive weight are never read), then normalised by layernorm_row: a one-hot row is layernorm_reg_kernel's bit for bit.
constexpr int LN_MIX_MAX_K = 8;
template <int NV>
__global__ void __launch_bounds__(256)
mix_layernorm_kernel(const float* __restrict__ y, int64_t y_ks, int ldy, int K, const float* __restrict__ W,
                     int64_t w_sb, int64_t w_st, int T, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* out, int ldo, int64_t rows, float eps, int post_act) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int64_t b = row / T, t = row - b * T;
  const float* wr = W + b * w_sb + t * w_st;
  float wk[LN_MIX_MAX_K];
  float wsum = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MIX_MAX_K; ++k) {
    wk[k] = k < K ? __ldg(wr + k) : 0.f;
    if (wk[k] > 0.f) wsum += wk[k];             // zero weights add nothing; NaN or negative ones are skipped throughout
  }
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  bool first = true;
#pragma unroll
  for (int k = 0; k < LN_MIX_MAX_K; ++k) {
    if (k >= K) break;
    if (!(wk[k] > 0.f)) continue;
    const float wn = wk[k] / wsum;
    const float* yr = y + k * y_ks + row * ldy;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 a = *reinterpret_cast<const float4*>(yr + i * 128 + lane * 4);
      v[i] = first ? make_float4(wn * a.x, wn * a.y, wn * a.z, wn * a.w)
                   : make_float4(fmaf(wn, a.x, v[i].x), fmaf(wn, a.y, v[i].y), fmaf(wn, a.z, v[i].z),
                                 fmaf(wn, a.w, v[i].w));
    }
    first = false;
  }
  const PlanesOut no_planes{nullptr, 0, 0, 0, 0.f, 0, nullptr};
  layernorm_row<NV>(v, lane, row, gamma, beta, nullptr, 0, out, ldo, eps, post_act, 0, no_planes);
}

static inline bool al16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

int layernorm_ex(const float* x, int ldx, const float* gamma, const float* beta, const float* res, int ldr,
                 float* y, int ldy, int64_t rows, int C, float eps, int post_act, int accumulate, PlanesOut po,
                 cudaStream_t st) {
  MTTS_REQUIRE(x && gamma && beta && (y || po.p), "null pointer");
  MTTS_REQUIRE(C > 0 && ldx >= C && (!y || ldy >= C), "bad dims");
  MTTS_REQUIRE(!(accumulate && !y), "accumulate needs a y buffer");
  MTTS_REQUIRE(post_act != MTTS_ACT_LEAKY, "leaky post-activation is not supported by LayerNorm (no slope argument)");
  if (rows <= 0) return 0;
  const int vec = (C % 4 == 0) && (ldx % 4 == 0) && (!y || ((ldy % 4 == 0) && al16(y))) && al16(x) && al16(gamma) &&
                  al16(beta) && (!res || ((ldr % 4 == 0) && al16(res)));
  MTTS_REQUIRE(!po.p || (vec && po.ld % 4 == 0 && po.stride % 4 == 0), "plane output needs the vector path");
  const int wpb = 8;
  const unsigned grid = (unsigned)cdiv64(rows, wpb);
#define MTTS_LN_REG(NV)                                                                                          \
  launch_k(layernorm_reg_kernel<NV>, grid, wpb * 32, 0, st, x, ldx, gamma, beta, res, ldr, y, ldy, rows, eps, post_act, \
                                                      accumulate, po)
  if (vec && C == 1024) MTTS_LN_REG(8);
  else if (vec && C == 768) MTTS_LN_REG(6);
  else if (vec && C == 512) MTTS_LN_REG(4);
  else if (vec && C == 384) MTTS_LN_REG(3);
  else
    launch_k(layernorm_kernel, grid, wpb * 32, 0, st, x, ldx, gamma, beta, res, ldr, y, ldy, rows, C, eps, post_act,
                                                accumulate, vec, po);
#undef MTTS_LN_REG
  MTTS_CHECK_LAUNCH();
  return 0;
}

int layernorm(const float* x, int ldx, const float* gamma, const float* beta, const float* res, int ldr,
              float* y, int ldy, int64_t rows, int C, float eps, int post_act, int accumulate,
              cudaStream_t st) {
  MTTS_REQUIRE(y, "null pointer");
  PlanesOut po{nullptr, 0, 0, 0, 0.f, 0, nullptr};
  return layernorm_ex(x, ldx, gamma, beta, res, ldr, y, ldy, rows, C, eps, post_act, accumulate, po, st);
}

int mix_layernorm(const float* y, int64_t y_ks, int ldy, int K, const float* w, int64_t w_sb, int64_t w_st, int T,
                  const float* gamma, const float* beta, float* out, int ldo, int64_t rows, int C, float eps, int post_act,
                  cudaStream_t st) {
  MTTS_REQUIRE(K >= 1, "K must be >= 1");
  if (K > LN_MIX_MAX_K)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: K = %lld sources is above the bound of %lld", "mix_layernorm", (long long)K,
                (long long)LN_MIX_MAX_K);
  if (C != 384 && C != 512 && C != 768 && C != 1024)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: C = %lld, expected 384, 512, 768 or 1024", "mix_layernorm", (long long)C);
  MTTS_REQUIRE(rows >= 0, "rows must be >= 0");
  MTTS_REQUIRE(y && w && gamma && beta && out, "null pointer");
  MTTS_REQUIRE(T >= 1 && y_ks >= 0 && w_sb >= 0 && w_st >= 0 && ldy >= C && ldo >= C, "bad T, strides or row strides");
  MTTS_REQUIRE(post_act == MTTS_ACT_NONE || post_act == MTTS_ACT_RELU || post_act == MTTS_ACT_TANH,
               "post_act must be none, relu or tanh");
  MTTS_REQUIRE(al16(y) && al16(out) && al16(gamma) && al16(beta) && ldy % 4 == 0 && ldo % 4 == 0 && y_ks % 4 == 0,
               "y, out, gamma and beta must be 16-byte aligned, with ldy, ldo and y_ks multiples of 4");
  if (rows == 0) return 0;
  const int wpb = 8;
  const unsigned grid = (unsigned)cdiv64(rows, wpb);
#define MTTS_LN_MIX(NV) \
  launch_k(mix_layernorm_kernel<NV>, grid, wpb * 32, 0, st, y, y_ks, ldy, K, w, w_sb, w_st, T, gamma, beta, out, ldo, rows, \
           eps, post_act)
  if (C == 1024) MTTS_LN_MIX(8);
  else if (C == 768) MTTS_LN_MIX(6);
  else if (C == 512) MTTS_LN_MIX(4);
  else MTTS_LN_MIX(3);
#undef MTTS_LN_MIX
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Attention, fp32, online softmax.  CTA = NW warps x RW query rows of one (b, h); K/V stream through
// shared memory 32*KPL keys at a time (float4 global loads when aligned); lane l scores keys l (+32 when KPL = 2:
// the broadcast Q loads of the score loop are then shared by two keys - that loop is shared-memory-bound), then owns
// output dims l + 32*i.  Head dims on the path: 64 (PLM), 96 (ADM), 256 (phone encoder), 512 (MRTE
// cross-attention, Tk ~ 32).  For dh <= 128 a CTA covers 64 query rows, i.e. a whole AR-step sequence:
// K and V are read once per (b, h).
// dh = 64 (NI = 2): capped at 80 registers so that three CTAs share an SM; the wider heads spill too much under that cap
// and keep two CTAs
template <int NI, int RW, int NW, int KPL>
__global__ void __launch_bounds__(NW * 32, (NI == 2 ? 3 : 2)) attn_kernel(const mtts_attn_params p, const int vec, int32_t* ovf) {
  pdl_entry();
  constexpr int DH = 32 * NI;
  constexpr int BQ = RW * NW, BKV = 32 * KPL, NT = NW * 32;
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;                        // [BQ][DH]
  constexpr int KS = DH + 4;             // K row stride: 16-byte aligned rows, conflict-free 128-bit reads (lane stride 4 banks)
  float* Ks = Qs + BQ * DH;              // [BKV][KS]
  float* Vs = Ks + BKV * KS;             // [BKV][DH]
  float* Ps = Vs + BKV * DH;             // [NW][RW][BKV]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const float* qb = p.q + (int64_t)b * p.q_sb + (int64_t)h * DH;
  const float* kb = p.k + (int64_t)b * p.k_sb + (int64_t)h * DH;
  const float* vb = p.v + (int64_t)b * p.v_sb + (int64_t)h * DH;

  if (vec) {
    for (int i = tid; i < BQ * (DH / 4); i += NT) {
      const int r = i / (DH / 4), d = (i - r * (DH / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + r < p.Tq) v = *reinterpret_cast<const float4*>(qb + (int64_t)(q0 + r) * p.q_st + d);
      *reinterpret_cast<float4*>(Qs + r * DH + d) = v;
    }
  } else {
    for (int i = tid; i < BQ * DH; i += NT) {
      const int r = i / DH, d = i - r * DH;
      Qs[i] = (q0 + r < p.Tq) ? qb[(int64_t)(q0 + r) * p.q_st + d] : 0.f;
    }
  }
  float m_run[RW], l_run[RW], acc[RW][NI];
#pragma unroll
  for (int i = 0; i < RW; ++i) {
    m_run[i] = -INFINITY;
    l_run[i] = 0.f;
#pragma unroll
    for (int j = 0; j < NI; ++j) acc[i][j] = 0.f;
  }
  const float* mrow[RW];
#pragma unroll
  for (int i = 0; i < RW; ++i) {
    const int qr = min(q0 + w * RW + i, p.Tq - 1);
    mrow[i] = p.mask ? p.mask + (int64_t)b * p.mask_sb + (int64_t)h * p.mask_sh + (int64_t)qr * p.mask_sq : nullptr;
  }
  const bool warp_live = (q0 + w * RW) < p.Tq;   // warp-uniform: this warp owns at least one real query row

  for (int k0 = 0; k0 < p.Tk; k0 += BKV) {
    __syncthreads();   // previous tile fully consumed (also orders the Q fill)
    if (vec) {
      for (int i = tid; i < BKV * (DH / 4); i += NT) {
        const int r = i / (DH / 4), d = (i - r * (DH / 4)) * 4;
        float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
        if (k0 + r < p.Tk) {
          kv = *reinterpret_cast<const float4*>(kb + (int64_t)(k0 + r) * p.k_st + d);
          vv = *reinterpret_cast<const float4*>(vb + (int64_t)(k0 + r) * p.v_st + d);
        }
        *reinterpret_cast<float4*>(Ks + r * KS + d) = kv;
        *reinterpret_cast<float4*>(Vs + r * DH + d) = vv;
      }
    } else {
      for (int i = tid; i < BKV * DH; i += NT) {
        const int r = i / DH, d = i - r * DH;
        const bool ok = k0 + r < p.Tk;
        Ks[r * KS + d] = ok ? kb[(int64_t)(k0 + r) * p.k_st + d] : 0.f;
        Vs[r * DH + d] = ok ? vb[(int64_t)(k0 + r) * p.v_st + d] : 0.f;
      }
    }
    __syncthreads();
    if (!warp_live) continue;
    float s[RW][KPL];
#pragma unroll
    for (int i = 0; i < RW; ++i)
#pragma unroll
      for (int c = 0; c < KPL; ++c) s[i][c] = 0.f;
    // 128-bit shared loads: KPL key chunks per lane + RW broadcast Q chunks feed 4 * RW * KPL FMAs (the scalar form
    // issued 9 loads per 8 FMAs and was load-issue bound); the d order of every dot product is unchanged
    const float* kr = Ks + lane * KS;
    const float* qr = Qs + (w * RW) * DH;
#pragma unroll 4
    for (int d = 0; d < DH; d += 4) {
      float4 kv[KPL];
#pragma unroll
      for (int c = 0; c < KPL; ++c) kv[c] = *reinterpret_cast<const float4*>(kr + c * 32 * KS + d);
#pragma unroll
      for (int i = 0; i < RW; ++i) {
        const float4 qv = *reinterpret_cast<const float4*>(qr + i * DH + d);
#pragma unroll
        for (int c = 0; c < KPL; ++c) {
          s[i][c] = fmaf(qv.x, kv[c].x, s[i][c]);
          s[i][c] = fmaf(qv.y, kv[c].y, s[i][c]);
          s[i][c] = fmaf(qv.z, kv[c].z, s[i][c]);
          s[i][c] = fmaf(qv.w, kv[c].w, s[i][c]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < RW; ++i) {
      float v[KPL];
      float vmax = -INFINITY;
#pragma unroll
      for (int c = 0; c < KPL; ++c) {
        const int key = k0 + lane + 32 * c;
        const bool kvalid = key < p.Tk;
        float x = s[i][c] * p.scale;
        if (mrow[i]) x += kvalid ? mrow[i][key] : 0.f;
        v[c] = kvalid ? x : -INFINITY;
        vmax = fmaxf(vmax, v[c]);
      }
      const float m_new = fmaxf(m_run[i], warp_max(vmax));
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      float psum = 0.f;
#pragma unroll
      for (int c = 0; c < KPL; ++c) {
        const float pr = expf(v[c] - m_use);
        Ps[(w * RW + i) * BKV + lane + 32 * c] = pr;
        psum += pr;
      }
      const float alpha = expf(m_run[i] - m_use);
      l_run[i] = l_run[i] * alpha + warp_sum(psum);
      m_run[i] = m_new;
#pragma unroll
      for (int j = 0; j < NI; ++j) acc[i][j] *= alpha;
    }
    __syncwarp();
    const float* pw = Ps + (w * RW) * BKV;
#pragma unroll 2
    for (int j = 0; j < BKV; j += 4) {
      float4 pj[RW];
#pragma unroll
      for (int i = 0; i < RW; ++i) pj[i] = *reinterpret_cast<const float4*>(pw + i * BKV + j);
#pragma unroll
      for (int ii = 0; ii < NI; ++ii) {
        const float v0 = Vs[(j + 0) * DH + lane + 32 * ii], v1 = Vs[(j + 1) * DH + lane + 32 * ii];
        const float v2 = Vs[(j + 2) * DH + lane + 32 * ii], v3 = Vs[(j + 3) * DH + lane + 32 * ii];
#pragma unroll
        for (int i = 0; i < RW; ++i) {
          acc[i][ii] = fmaf(pj[i].x, v0, acc[i][ii]);
          acc[i][ii] = fmaf(pj[i].y, v1, acc[i][ii]);
          acc[i][ii] = fmaf(pj[i].z, v2, acc[i][ii]);
          acc[i][ii] = fmaf(pj[i].w, v3, acc[i][ii]);
        }
      }
    }
    __syncwarp();
  }
  if (p.o) {
#pragma unroll
    for (int i = 0; i < RW; ++i) {
      const int qr = q0 + w * RW + i;
      if (qr >= p.Tq) continue;
      float* o = p.o + (int64_t)b * p.o_sb + (int64_t)qr * p.o_st + (int64_t)h * DH;
      const float inv = 1.0f / l_run[i];
#pragma unroll
      for (int ii = 0; ii < NI; ++ii) o[lane + 32 * ii] = acc[i][ii] * inv;
    }
  }
  if (p.o_planes) {
    // bf16x3 planes for the following tensor-core GEMM: stage this warp's rows in its (now dead) Q rows so
    // that every lane can split 4 CONSECUTIVE dims and store 8 bytes per plane
    __syncwarp();
    float* stg = Qs + (w * RW) * DH;
#pragma unroll
    for (int i = 0; i < RW; ++i) {
      const float inv = 1.0f / l_run[i];
#pragma unroll
      for (int ii = 0; ii < NI; ++ii) stg[i * DH + lane + 32 * ii] = acc[i][ii] * inv;
    }
    __syncwarp();
    __nv_bfloat16* pl = reinterpret_cast<__nv_bfloat16*>(p.o_planes);
    for (int e = lane; e < RW * (DH / 4); e += 32) {
      const int i = e / (DH / 4), d = (e - i * (DH / 4)) * 4;
      const int qr = q0 + w * RW + i;
      if (qr >= p.Tq) continue;
      const float4 v = *reinterpret_cast<const float4*>(stg + i * DH + d);
      const float vv[4] = {v.x, v.y, v.z, v.w};
      store_planes4(pl, p.o_plane_stride, ((int64_t)b * p.Tq + qr) * p.o_planes_ld + (int64_t)h * DH + d, vv, p.o_planes_fmt, ovf);
    }
  }
}

template <int NI, int RW, int NW, int KPL = 1>
static int attn_launch(const mtts_attn_params& p, int vec, cudaStream_t st) {
  constexpr int DH = 32 * NI;
  constexpr int BQ = RW * NW, BKV = 32 * KPL;
  const size_t smem = sizeof(float) * (BQ * DH + BKV * (DH + 4) + BKV * DH + NW * RW * BKV);
  // the max-dynamic-shared-memory attribute is per device: one flag per (instantiation, device)
  static std::atomic<uint64_t> configured{0};
  const int dev = cur_device();
  if (!(configured.load(std::memory_order_relaxed) & (1ull << dev))) {
    cudaError_t e = cudaFuncSetAttribute(attn_kernel<NI, RW, NW, KPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(MTTS_ERR_CUDA, "%s: cudaFuncSetAttribute failed: %lld", "attention", (long long)e);
    configured.fetch_or(1ull << dev, std::memory_order_relaxed);
  }
  dim3 grid((unsigned)cdiv64(p.Tq, BQ), (unsigned)p.H, (unsigned)p.B);
  launch_k(attn_kernel<NI, RW, NW, KPL>, grid, NW * 32, smem, st, p, vec, p.o_planes ? tc_ovf_ptr() : nullptr);
  MTTS_CHECK_LAUNCH();
  return 0;
}

static std::atomic<int> g_attn_pair_min{[] {
  const char* m = getenv("MEGATTS2_ATTN_PAIR_MIN");
  return m ? atoi(m) : (1 << 30);
}()};
int set_attention_pair_min(int n) { return g_attn_pair_min.exchange(n > 0 ? n : (1 << 30), std::memory_order_relaxed); }

int attn_check(const mtts_attn_params& p) {
  MTTS_REQUIRE(p.q && p.k && p.v && (p.o || p.o_planes), "null pointer");
  MTTS_REQUIRE(!p.o_planes || (p.o_planes_ld % 4 == 0 && p.o_plane_stride % 4 == 0), "plane output alignment");
  MTTS_REQUIRE(p.B >= 0 && p.H > 0 && p.Tq >= 0 && p.Tk > 0, "bad dims");
  MTTS_REQUIRE(p.H <= 65535 && p.B <= 65535, "grid too large");
  return 0;
}

AttnPlan attn_plan(const mtts_attn_params& p, bool allow_f16_operands, int pair_min) {
  AttnPlan pl{MTTS_ATTN_NONE, (int)p.dh, 0, 0, 0, 0};
  if (p.B == 0 || p.Tq == 0) return pl;
  pl.vec = al16(p.q) && al16(p.k) && al16(p.v) && p.q_st % 4 == 0 && p.k_st % 4 == 0 && p.v_st % 4 == 0 && p.q_sb % 4 == 0 &&
           p.k_sb % 4 == 0 && p.v_sb % 4 == 0;
  // tensor-core path (attn_tc.cu): the head dims of the AR stacks once a sequence has more than 64 queries.  At the C4 step
  // shapes (Tq = Tk <= 64) a head is a 64 x 64 x 64 problem, all latency, so the AR steps of the benchmark stay on this fp32
  // kernel; longer sequences (teacher-forced forwards, config C3) go to the tensor cores.
  // That kernel splits Q, K and V into f16x2 planes, so only callers on an fp16-range engine take it; the bf16x3 and
  // FFMA engines keep the full fp32 range here.
  if (allow_f16_operands) {
    constexpr int tc_min = 65;
    if (p.Tq >= tc_min && attention_tc_eligible(p)) { pl.kernel = MTTS_ATTN_TC; return pl; }
    // AR steps (Tq == Tk <= 64) on the tensor cores: one 64-row tile per head.  The operand conversions, not the MMAs, are
    // what a 64 x 64 x 64 head costs, so it is opt-in (mtts_set_attention_pair_min / MEGATTS2_ATTN_PAIR_MIN: shortest
    // sequence that takes it), off by default.
    if (p.Tq >= pair_min && attention_tc_pair_eligible(p)) { pl.kernel = MTTS_ATTN_TC_PAIR; return pl; }
  }
  // dh <= 128: one CTA of 8 warps covers a whole AR-step sequence (Tq <= 64), so K and V are read once per (b, h);
  // the rows are dealt evenly to the warps (RW = ceil(Tq / 8) rows each) - with a fixed 8 rows per warp a 35-row
  // step left three of the eight warps idle.  Row results do not depend on RW (each row's sums keep their order).
  // KPL = 2 (Tk > 32): two keys per lane, one 64-key tile instead of two 32-key tiles.
  if (p.dh == 64 || p.dh == 96 || p.dh == 128) {
    pl.kernel = MTTS_ATTN_FP32;
    pl.rw = p.Tq >= 64 ? 8 : (p.Tq + 7) / 8;
    pl.nw = 8;
    pl.kpl = p.Tk > 32 ? 2 : 1;
  } else if (p.dh == 256 || p.dh == 512) {
    pl.kernel = MTTS_ATTN_FP32;
    pl.rw = 4;
    pl.nw = 4;
    pl.kpl = 1;
  } else {
    pl.kernel = ATTN_UNSUPPORTED;
  }
  return pl;
}

template <int NI>
static int attn_launch_rw(const mtts_attn_params& p, const AttnPlan& pl, cudaStream_t st) {
  const bool two = pl.kpl == 2;
  const int vec = pl.vec;
  switch (pl.rw) {
    case 1: return two ? attn_launch<NI, 1, 8, 2>(p, vec, st) : attn_launch<NI, 1, 8>(p, vec, st);
    case 2: return two ? attn_launch<NI, 2, 8, 2>(p, vec, st) : attn_launch<NI, 2, 8>(p, vec, st);
    case 3: return two ? attn_launch<NI, 3, 8, 2>(p, vec, st) : attn_launch<NI, 3, 8>(p, vec, st);
    case 4: return two ? attn_launch<NI, 4, 8, 2>(p, vec, st) : attn_launch<NI, 4, 8>(p, vec, st);
    case 5: return two ? attn_launch<NI, 5, 8, 2>(p, vec, st) : attn_launch<NI, 5, 8>(p, vec, st);
    case 6: return two ? attn_launch<NI, 6, 8, 2>(p, vec, st) : attn_launch<NI, 6, 8>(p, vec, st);
    case 7: return two ? attn_launch<NI, 7, 8, 2>(p, vec, st) : attn_launch<NI, 7, 8>(p, vec, st);
    default: return two ? attn_launch<NI, 8, 8, 2>(p, vec, st) : attn_launch<NI, 8, 8>(p, vec, st);
  }
}

int attention(const mtts_attn_params& p, bool allow_f16_operands, cudaStream_t st) {
  MTTS_TRY(attn_check(p));
  const AttnPlan pl = attn_plan(p, allow_f16_operands, g_attn_pair_min.load(std::memory_order_relaxed));
  switch (pl.kernel) {
    case MTTS_ATTN_NONE: return 0;
    case MTTS_ATTN_TC: return attention_tc(p, st);
    case MTTS_ATTN_TC_PAIR: return attention_tc_pair(p, st);
    case MTTS_ATTN_FP32: break;
    default: return fail(MTTS_ERR_UNSUPPORTED, "%s: head dim %lld not in {64,96,128,256,512}", "attention", (long long)p.dh);
  }
  switch (pl.dh) {
    case 64: return attn_launch_rw<2>(p, pl, st);
    case 96: return attn_launch_rw<3>(p, pl, st);
    case 128: return attn_launch_rw<4>(p, pl, st);
    case 256: return attn_launch<8, 4, 4>(p, pl.vec, st);
    default: return attn_launch<16, 4, 4>(p, pl.vec, st);
  }
}

// diagnostics: the plan attention() would launch for these parameters with `pair_min` as the AR-step routing threshold
// (<= 0: off); out6 = {kernel (MTTS_ATTN_*), dh, RW, NW, KPL, vec}
int attention_plan_query(const mtts_attn_params* p, int allow_f16_operands, int pair_min, int32_t* out6) {
  MTTS_REQUIRE(p && out6, "null params");
  MTTS_TRY(attn_check(*p));
  const AttnPlan pl = attn_plan(*p, allow_f16_operands != 0, pair_min > 0 ? pair_min : (1 << 30));
  if (pl.kernel == ATTN_UNSUPPORTED)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: head dim %lld not in {64,96,128,256,512}", "attention", (long long)p->dh);
  out6[0] = pl.kernel; out6[1] = pl.dh; out6[2] = pl.rw; out6[3] = pl.nw; out6[4] = pl.kpl; out6[5] = pl.vec;
  return 0;
}

// ------------------------------------------------------------------------------------------
// VQ nearest-code search.  CTA = 8 rows x all K codes; warp w scans codes w, w+8, ...; lanes
// split D (float4 chunks) and butterfly-reduce; strict '<' keeps the first index on ties,
// matching torch.max(-dist) on CPU (core_vq.py:175-183).
template <int CH>   // D = 128 * CH
__global__ void __launch_bounds__(256)
vq_argmin_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ embed, int64_t N, int K,
                 int64_t* __restrict__ idx) {
  pdl_entry();
  constexpr int R = 8, D = 128 * CH;
  __shared__ float sd[8][R];
  __shared__ int sk[8][R];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * R;
  float4 xv[R][CH];
  float xx[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      xv[r][c] = (r0 + r < N) ? *reinterpret_cast<const float4*>(x + (r0 + r) * ldx + c * 128 + lane * 4)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (xv[r][c].x * xv[r][c].x + xv[r][c].y * xv[r][c].y) + (xv[r][c].z * xv[r][c].z + xv[r][c].w * xv[r][c].w);
    }
    xx[r] = warp_sum(s);
  }
  float best[R];
  int bestk[R];
#pragma unroll
  for (int r = 0; r < R; ++r) { best[r] = INFINITY; bestk[r] = 0x7fffffff; }
  for (int k = w; k < K; k += 8) {
    float4 ev[CH];
    float ee = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      ev[c] = __ldg(reinterpret_cast<const float4*>(embed + (int64_t)k * D + c * 128 + lane * 4));
      ee += (ev[c].x * ev[c].x + ev[c].y * ev[c].y) + (ev[c].z * ev[c].z + ev[c].w * ev[c].w);
    }
    ee = warp_sum(ee);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < CH; ++c)
        d += (xv[r][c].x * ev[c].x + xv[r][c].y * ev[c].y) + (xv[r][c].z * ev[c].z + xv[r][c].w * ev[c].w);
      d = warp_sum(d);
      const float dist = (xx[r] - 2.0f * d) + ee;
      if (dist < best[r]) { best[r] = dist; bestk[r] = k; }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < R; ++r) { sd[w][r] = best[r]; sk[w][r] = bestk[r]; }
  }
  __syncthreads();
  if (threadIdx.x < R && r0 + threadIdx.x < N) {
    float bd = sd[0][threadIdx.x];
    int bk = sk[0][threadIdx.x];
    for (int ww = 1; ww < 8; ++ww) {
      const float d = sd[ww][threadIdx.x];
      const int k = sk[ww][threadIdx.x];
      if (d < bd || (d == bd && k < bk)) { bd = d; bk = k; }
    }
    idx[r0 + threadIdx.x] = (int64_t)bk;
  }
}

int vq_argmin(const float* x, int ldx, const float* embed, int64_t N, int D, int K, int64_t* idx, cudaStream_t st) {
  MTTS_REQUIRE(x && embed && idx, "null pointer");
  MTTS_REQUIRE(K > 0 && D > 0 && ldx >= D, "bad dims");
  MTTS_REQUIRE(ldx % 4 == 0 && al16(x) && al16(embed), "x / embed must be 16-byte aligned with ldx % 4 == 0");
  if (N <= 0) return 0;
  const unsigned grid = (unsigned)cdiv64(N, 8);
  switch (D) {
    case 128: launch_k(vq_argmin_kernel<1>, grid, 256, 0, st, x, ldx, embed, N, K, idx); break;
    case 256: launch_k(vq_argmin_kernel<2>, grid, 256, 0, st, x, ldx, embed, N, K, idx); break;
    case 512: launch_k(vq_argmin_kernel<4>, grid, 256, 0, st, x, ldx, embed, N, K, idx); break;
    default: return fail(MTTS_ERR_UNSUPPORTED, "%s: codebook dim %lld not in {128,256,512}", "vq_argmin", D);
  }
  MTTS_CHECK_LAUNCH();
  return 0;
}

__global__ void vq_gather_kernel(const int64_t* __restrict__ idx, int idx_ld, const float* __restrict__ embed, int D,
                                 int K, int T_out, int repeat, float* __restrict__ y, int64_t y_sb, int ldy,
                                 int64_t total) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i % D);
  const int64_t bt = i / D;
  const int t = (int)(bt % T_out);
  const int b = (int)(bt / T_out);
  int64_t code = idx[(int64_t)b * idx_ld + t / repeat];
  code = code < 0 ? 0 : (code >= K ? K - 1 : code);
  y[(int64_t)b * y_sb + (int64_t)t * ldy + d] = __ldg(embed + code * D + d);
}

int vq_gather(const int64_t* idx, int idx_ld, const float* embed, int D, int K, int B, int T_out, int repeat,
              float* y, int64_t y_sb, int ldy, cudaStream_t st) {
  MTTS_REQUIRE(idx && embed && y && repeat >= 1 && D > 0 && K > 0, "bad arguments");
  const int64_t total = (int64_t)B * T_out * D;
  if (total <= 0) return 0;
  launch_k(vq_gather_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, idx, idx_ld, embed, D, K, T_out, repeat, y, y_sb, ldy, total);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------
__global__ void maxpool_time_kernel(const float* __restrict__ x, int64_t x_sb, int ldx, float* __restrict__ y,
                                    int64_t y_sb, int ldy, int T, int To, int C, int k, int64_t total) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int64_t bt = i / C;
  const int to = (int)(bt % To);
  const int b = (int)(bt / To);
  const float* src = x + (int64_t)b * x_sb + c;
  float m = -INFINITY;
  for (int r = 0; r < k; ++r) {
    const int t = to * k + r;
    if (t < T) m = fmaxf(m, src[(int64_t)t * ldx]);
  }
  y[(int64_t)b * y_sb + (int64_t)to * ldy + c] = m;
}

int maxpool_time(const float* x, int64_t x_sb, int ldx, float* y, int64_t y_sb, int ldy, int B, int T, int C, int k,
                 cudaStream_t st) {
  MTTS_REQUIRE(x && y && k >= 1 && C > 0, "bad arguments");
  const int To = (T + k - 1) / k;
  const int64_t total = (int64_t)B * To * C;
  if (total <= 0) return 0;
  launch_k(maxpool_time_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, x, x_sb, ldx, y, y_sb, ldy, T, To, C, k, total);
  MTTS_CHECK_LAUNCH();
  return 0;
}

__global__ void embed_pe_kernel(const int64_t* __restrict__ ids, int ids_ld, const float* __restrict__ table,
                                int vocab, int D, const float* __restrict__ pe, float alpha, int pe_offset, int T,
                                float* __restrict__ y, int64_t y_sb, int ldy, int64_t total) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i % D);
  const int64_t bt = i / D;
  const int t = (int)(bt % T);
  const int b = (int)(bt / T);
  int64_t id = ids[(int64_t)b * ids_ld + t];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  float v = __ldg(table + id * D + d);
  if (pe) v = v * 1.0f + alpha * __ldg(pe + (int64_t)(t + pe_offset) * D + d);
  y[(int64_t)b * y_sb + (int64_t)t * ldy + d] = v;
}

int embed_pe(const int64_t* ids, int ids_ld, const float* table, int vocab, int D, const float* pe, float alpha,
             int pe_offset, int B, int T, float* y, int64_t y_sb, int ldy, cudaStream_t st) {
  MTTS_REQUIRE(ids && table && y && D > 0 && vocab > 0, "bad arguments");
  const int64_t total = (int64_t)B * T * D;
  if (total <= 0) return 0;
  launch_k(embed_pe_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, ids, ids_ld, table, vocab, D, pe, alpha, pe_offset, T, y, y_sb, ldy, total);
  MTTS_CHECK_LAUNCH();
  return 0;
}

__global__ void add_pe_kernel(const float* __restrict__ x, int64_t x_sb, int ldx, const float* __restrict__ pe,
                              float alpha, int T, int D, float* __restrict__ y, int64_t y_sb, int ldy, int64_t total) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i % D);
  const int64_t bt = i / D;
  const int t = (int)(bt % T);
  const int b = (int)(bt / T);
  y[(int64_t)b * y_sb + (int64_t)t * ldy + d] =
      x[(int64_t)b * x_sb + (int64_t)t * ldx + d] * 1.0f + alpha * __ldg(pe + (int64_t)t * D + d);
}

int add_pe(const float* x, int64_t x_sb, int ldx, const float* pe, float alpha, int B, int T, int D, float* y,
           int64_t y_sb, int ldy, cudaStream_t st) {
  MTTS_REQUIRE(x && pe && y && D > 0, "bad arguments");
  const int64_t total = (int64_t)B * T * D;
  if (total <= 0) return 0;
  launch_k(add_pe_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, x, x_sb, ldx, pe, alpha, T, D, y, y_sb, ldy, total);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// LengthRegulator: CTA = 32 output rows of one utterance; thread 0 scans the durations of
// that utterance into shared memory, each warp binary-searches its rows.
__global__ void __launch_bounds__(256)
length_regulate_kernel(const float* __restrict__ x, int64_t x_sb, int ldx, const int32_t* __restrict__ dur, int dur_ld,
                       int Tp, int D, int L_out, float* __restrict__ y, int64_t y_sb, int ldy,
                       int32_t* __restrict__ totals) {
  pdl_entry();
  extern __shared__ int cum[];   // Tp + 1
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    int s = 0;
    cum[0] = 0;
    for (int i = 0; i < Tp; ++i) {
      s += max(dur[(int64_t)b * dur_ld + i], 0);
      cum[i + 1] = s;
    }
    if (totals && blockIdx.x == 0) totals[b] = s;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int total = cum[Tp];
  for (int rr = w; rr < 32; rr += 8) {
    const int r = blockIdx.x * 32 + rr;
    if (r >= L_out) break;
    float* dst = y + (int64_t)b * y_sb + (int64_t)r * ldy;
    if (r >= total) {
      for (int d = lane; d < D; d += 32) dst[d] = 0.f;
      continue;
    }
    int lo = 0, hi = Tp;   // largest i with cum[i] <= r
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (cum[mid] <= r) lo = mid; else hi = mid;
    }
    const float* src = x + (int64_t)b * x_sb + (int64_t)lo * ldx;
    for (int d = lane; d < D; d += 32) dst[d] = src[d];
  }
}

int length_regulate(const float* x, int64_t x_sb, int ldx, const int32_t* dur, int dur_ld, int B, int Tp, int D,
                    int L_out, float* y, int64_t y_sb, int ldy, int32_t* totals, cudaStream_t st) {
  MTTS_REQUIRE(x && dur && D > 0 && Tp > 0 && B >= 0 && L_out >= 0, "bad arguments");
  MTTS_REQUIRE(Tp <= 8192, "Tp too large");
  if (B == 0) return 0;
  MTTS_REQUIRE(y || L_out == 0, "null output");
  dim3 grid((unsigned)(L_out > 0 ? cdiv64(L_out, 32) : 1), (unsigned)B);
  launch_k(length_regulate_kernel, grid, 256, (Tp + 1) * sizeof(int), st, x, x_sb, ldx, dur, dur_ld, Tp, D, L_out, y, y_sb, ldy, totals);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// Generic strided (B,T,C) copy through a 32x32 shared tile so that both the read and the
// write are coalesced whichever of (t, c) is the unit-stride dim on each side.
__global__ void __launch_bounds__(256)
copy_strided_kernel(const float* __restrict__ x, int64_t x_sb, int64_t x_st, int64_t x_sc, float* __restrict__ y,
                    int64_t y_sb, int64_t y_st, int64_t y_sc, int T, int C, int pad_rep) {
  pdl_entry();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int To = T + 2 * pad_rep;
  const int fx = threadIdx.x & 31, sy = threadIdx.x >> 5;   // 32 x 8
  const bool src_c_fast = (x_sc <= x_st);
  const bool dst_c_fast = (y_sc <= y_st);
  for (int s = sy; s < 32; s += 8) {
    const int tl = src_c_fast ? s : fx, cl = src_c_fast ? fx : s;
    const int t = t0 + tl, c = c0 + cl;
    if (t < To && c < C) {
      int ts = t - pad_rep;
      ts = ts < 0 ? 0 : (ts >= T ? T - 1 : ts);
      tile[tl][cl] = x[(int64_t)b * x_sb + (int64_t)ts * x_st + (int64_t)c * x_sc];
    }
  }
  __syncthreads();
  for (int s = sy; s < 32; s += 8) {
    const int tl = dst_c_fast ? s : fx, cl = dst_c_fast ? fx : s;
    const int t = t0 + tl, c = c0 + cl;
    if (t < To && c < C) y[(int64_t)b * y_sb + (int64_t)t * y_st + (int64_t)c * y_sc] = tile[tl][cl];
  }
}

int copy_strided(const float* x, int64_t x_sb, int64_t x_st, int64_t x_sc, float* y, int64_t y_sb, int64_t y_st,
                 int64_t y_sc, int B, int T, int C, int pad_rep, cudaStream_t st) {
  MTTS_REQUIRE(x && y && pad_rep >= 0, "bad arguments");
  if (B <= 0 || T <= 0 || C <= 0) return 0;
  MTTS_REQUIRE(B <= 65535 && cdiv64(C, 32) <= 65535, "grid too large");
  dim3 grid((unsigned)cdiv64(T + 2 * pad_rep, 32), (unsigned)cdiv64(C, 32), (unsigned)B);
  launch_k(copy_strided_kernel, grid, 256, 0, st, x, x_sb, x_st, x_sc, y, y_sb, y_st, y_sc, T, C, pad_rep);
  MTTS_CHECK_LAUNCH();
  return 0;
}

__global__ void mask_tail_kernel(float* __restrict__ x, int rows, int L, const int32_t* __restrict__ keep) {
  pdl_entry();
  const int b = blockIdx.z, r = blockIdx.y;
  const int k0 = max(keep[b], 0);
  float* xr = x + ((int64_t)b * rows + r) * L;
  for (int i = k0 + blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) xr[i] = 0.f;
}
int mask_tail(float* x, int B, int rows, int L, const int32_t* keep, cudaStream_t st) {
  MTTS_REQUIRE(x && keep && B >= 0 && rows >= 0 && L >= 0, "bad arguments");
  if (B == 0 || rows == 0 || L == 0) return 0;
  MTTS_REQUIRE(B <= 65535 && rows <= 65535, "grid too large");
  dim3 grid((unsigned)(cdiv64(L, 1024) < 64 ? cdiv64(L, 1024) : 64), (unsigned)rows, (unsigned)B);
  launch_k(mask_tail_kernel, grid, 256, 0, st, x, rows, L, keep);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// Ragged row copy (the contract is stated with mtts_copy_row_segments in include/megatts2_b200.h): CTA row y = batch row
// b, the x CTAs stride over the (row, word) pairs of b's segment.  The segment is clipped on the device to the rows that
// lie inside both buffers, so no table value can move an access outside them.  W is uint4 when every address is 16-byte
// aligned, else uint32_t.
template <typename W>
__global__ void copy_row_segments_kernel(const char* __restrict__ src, int64_t src_sb, int64_t src_st, int64_t src_rows,
                                         char* __restrict__ dst, int64_t dst_sb, int64_t dst_st, int64_t dst_rows,
                                         int words, const int32_t* __restrict__ src_off,
                                         const int32_t* __restrict__ dst_off, const int32_t* __restrict__ n, int n_max,
                                         uint32_t fill_word) {
  pdl_entry();
  const int b = blockIdx.y;
  const int64_t d0 = dst_off[b];
  const int64_t s0 = src ? (int64_t)src_off[b] : 0;
  int64_t r0 = d0 < 0 ? -d0 : 0;
  int64_t r1 = min(min((int64_t)n[b], (int64_t)n_max), dst_rows - d0);
  if (src) {
    r0 = max(r0, -s0);
    r1 = min(r1, src_rows - s0);
  }
  if (r1 <= r0) return;
  W fill;
  const uint32_t* fw = &fill_word;
  if constexpr (sizeof(W) == 16) fill = make_uint4(*fw, *fw, *fw, *fw);
  else fill = *fw;
  const int64_t total = (r1 - r0) * words;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = r0 + i / words;
    const int w = (int)(i % words);
    W* dp = reinterpret_cast<W*>(dst + b * dst_sb + (d0 + r) * dst_st) + w;
    *dp = src ? reinterpret_cast<const W*>(src + b * src_sb + (s0 + r) * src_st)[w] : fill;
  }
}

int copy_row_segments(const void* src, int64_t src_sb, int64_t src_st, int64_t src_rows, void* dst, int64_t dst_sb,
                      int64_t dst_st, int64_t dst_rows, int row_bytes, const int32_t* src_off, const int32_t* dst_off,
                      const int32_t* n, int B, int n_max, uint32_t fill_word, cudaStream_t st) {
  MTTS_REQUIRE(dst && dst_off && n && (!src || src_off), "null pointer (dst, dst_off and n always; src_off with src)");
  MTTS_REQUIRE(src != dst, "src and dst must differ");
  MTTS_REQUIRE(row_bytes > 0 && row_bytes % 4 == 0, "row_bytes must be a positive multiple of 4");
  MTTS_REQUIRE(B >= 0 && B <= 65535, "B must be in 0..65535");
  MTTS_REQUIRE(n_max >= 0, "n_max must be >= 0");
  MTTS_REQUIRE(src_rows >= 0 && dst_rows >= 0, "src_rows and dst_rows must be >= 0");
  MTTS_REQUIRE(src_sb >= 0 && src_st >= row_bytes && dst_sb >= 0 && dst_st >= row_bytes &&
                   (src_sb | src_st | dst_sb | dst_st) % 4 == 0,
               "strides must be multiples of 4 bytes, row strides >= row_bytes and batch strides >= 0");
  MTTS_REQUIRE(B <= 1 || dst_rows == 0 || dst_sb >= dst_rows * dst_st, "dst's batch rows must not overlap");
  MTTS_REQUIRE((((uintptr_t)src) & 3) == 0 && (((uintptr_t)dst) & 3) == 0, "src and dst must be 4-byte aligned");
  if (B == 0 || n_max == 0 || dst_rows == 0) return 0;
  const bool v16 = (((uintptr_t)src | (uintptr_t)dst) & 15) == 0 && row_bytes % 16 == 0 &&
                   (src_sb | src_st | dst_sb | dst_st) % 16 == 0;
  const int words = row_bytes / (v16 ? 16 : 4);
  const int64_t per_b = (int64_t)n_max * words;
  const dim3 grid((unsigned)(cdiv64(per_b, 256) < 128 ? cdiv64(per_b, 256) : 128), (unsigned)B);
  if (v16)
    launch_k(copy_row_segments_kernel<uint4>, grid, 256, 0, st, (const char*)src, src_sb, src_st, src_rows, (char*)dst,
             dst_sb, dst_st, dst_rows, words, src_off, dst_off, n, n_max, fill_word);
  else
    launch_k(copy_row_segments_kernel<uint32_t>, grid, 256, 0, st, (const char*)src, src_sb, src_st, src_rows,
             (char*)dst, dst_sb, dst_st, dst_rows, words, src_off, dst_off, n, n_max, fill_word);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Autoregressive-loop helpers (device-resident state: no host sync inside the loops).

// PLM step input (models/megatts2.py:173-175): X[b,s,:] = cat(lat[b,s,:], emb[codes[b,s]]) + alpha*pe[s], where the latent
// row lat[b,s] is ctx[b,s] for s < P (a prompt context) and tc[b,s-P] after it
__global__ void plm_build_input_kernel(const float* __restrict__ tc, int64_t tc_sb, int tc_ld, int tc_dim,
                                       const int64_t* __restrict__ codes, int codes_ld, int B_codes,
                                       const float* __restrict__ emb, int vq_dim, int vocab,
                                       const float* __restrict__ pe, float alpha, int S, float* __restrict__ X,
                                       int64_t total, const float* __restrict__ ctx, int64_t ctx_sb, int ctx_ld, int P) {
  pdl_entry();
  const int D = tc_dim + vq_dim;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i % D);
  const int64_t bs = i / D;
  const int s = (int)(bs % S);
  const int b = (int)(bs / S);
  float v;
  if (d < tc_dim) {
    v = s < P ? ctx[(int64_t)b * ctx_sb + (int64_t)s * ctx_ld + d] : tc[(int64_t)b * tc_sb + (int64_t)(s - P) * tc_ld + d];
  } else {
    int64_t id = codes[(int64_t)(b % B_codes) * codes_ld + s];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    v = __ldg(emb + id * vq_dim + (d - tc_dim));
  }
  X[i] = v * 1.0f + alpha * __ldg(pe + (int64_t)s * D + d);
}

int plm_build_input(const float* tc, int64_t tc_sb, int tc_ld, int tc_dim, const int64_t* codes, int codes_ld,
                    int B_codes, const float* emb, int vq_dim, int vocab, const float* pe, float alpha, int B, int S,
                    float* X, cudaStream_t st, const float* ctx, int64_t ctx_sb, int ctx_ld, int P) {
  const int64_t total = (int64_t)B * S * (tc_dim + vq_dim);
  if (total <= 0) return 0;
  MTTS_REQUIRE(B_codes >= 1, "B_codes must be >= 1");
  MTTS_REQUIRE(P >= 0 && (P == 0 || ctx), "context rows without a context latent");
  launch_k(plm_build_input_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, tc, tc_sb, tc_ld, tc_dim, codes, codes_ld,
           B_codes, emb, vq_dim, vocab, pe, alpha, S, X, total, ctx, ctx_sb, ctx_ld, P);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// argmax over the last dim, first index on ties (torch.argmax on CPU); one warp per row.
// writes out_a[row*lda] and (optionally) out_b[row*ldb].  pin (optional): a row whose pin[row*pin_sb] is in [0, V) writes
// that value instead of its argmax; any other pin value leaves the row free.
__global__ void argmax_rows_kernel(const float* __restrict__ x, int64_t ldx, int V, int rows, int64_t* out_a,
                                   int64_t lda, int64_t* out_b, int64_t ldb, const int32_t* __restrict__ pin,
                                   int64_t pin_sb) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  if (pin) {
    const int32_t p = pin[(int64_t)row * pin_sb];
    if (p >= 0 && p < V) {
      if (lane == 0) {
        out_a[(int64_t)row * lda] = p;
        if (out_b) out_b[(int64_t)row * ldb] = p;
      }
      return;
    }
  }
  const float* xr = x + (int64_t)row * ldx;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = lane; i < V; i += 32) {
    const float v = xr[i];
    if (v > best) { best = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) {
    if (bi == 0x7fffffff) bi = 0;
    out_a[(int64_t)row * lda] = bi;
    if (out_b) out_b[(int64_t)row * ldb] = bi;
  }
}

int argmax_rows(const float* x, int64_t ldx, int V, int rows, int64_t* out_a, int64_t lda, int64_t* out_b, int64_t ldb,
                cudaStream_t st, const int32_t* pin, int64_t pin_sb) {
  if (rows <= 0) return 0;
  launch_k(argmax_rows_kernel, (unsigned)cdiv64(rows, 4), 128, 0, st, x, ldx, V, rows, out_a, lda, out_b, ldb, pin,
           pin_sb);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// y[b * ldy + p] = x[b * x_sb + p] for p < n: the context codes into a code state (x_sb = 0: one row for every b)
__global__ void copy_codes_kernel(const int64_t* __restrict__ x, int64_t x_sb, int64_t* __restrict__ y, int64_t ldy, int B,
                                  int n) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * n) return;
  const int b = (int)(i / n), p = (int)(i % n);
  y[(int64_t)b * ldy + p] = x[(int64_t)b * x_sb + p];
}
int copy_codes(const int64_t* x, int64_t x_sb, int64_t* y, int64_t ldy, int B, int n, cudaStream_t st) {
  if (B <= 0 || n <= 0) return 0;
  launch_k(copy_codes_kernel, (unsigned)cdiv64((int64_t)B * n, 256), 256, 0, st, x, x_sb, y, ldy, B, n);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// m (T, T): 0 on and below the diagonal, -inf above it (make_attn_mask's causal part, utils/utils.py:21-39)
__global__ void causal_mask_kernel(float* m, int T) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)T * T) return;
  m[i] = (int)(i % T) > (int)(i / T) ? -INFINITY : 0.0f;
}
int causal_mask(float* m, int T, cudaStream_t st) {
  if (T <= 0) return 0;
  launch_k(causal_mask_kernel, (unsigned)cdiv64((int64_t)T * T, 256), 256, 0, st, m, T);
  MTTS_CHECK_LAUNCH();
  return 0;
}

__global__ void fill_i64_kernel(int64_t* p, int64_t stride, int n, int64_t v) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[(int64_t)i * stride] = v;
}
int fill_i64(int64_t* p, int64_t stride, int n, int64_t v, cudaStream_t st) {
  if (n <= 0) return 0;
  launch_k(fill_i64_kernel, (unsigned)cdiv64(n, 256), 256, 0, st, p, stride, n, v);
  MTTS_CHECK_LAUNCH();
  return 0;
}
__global__ void fill_f32_kernel(float* p, int64_t stride, int n, float v) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[(int64_t)i * stride] = v;
}
int fill_f32(float* p, int64_t stride, int n, float v, cudaStream_t st) {
  if (n <= 0) return 0;
  launch_k(fill_f32_kernel, (unsigned)cdiv64(n, 256), 256, 0, st, p, stride, n, v);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ADM step input (models/megatts2.py:265-269): X[b,s,:] = cat(tc_emb[b,s,:], p[b,s]*w_dt[:]) + alpha*pe[s]
__global__ void adm_build_input_kernel(const float* __restrict__ tc_emb, int64_t te_sb, int te_ld, int tc_emb_dim,
                                       const float* __restrict__ praw, int p_ld, int B_hist,
                                       const float* __restrict__ w_dt, int emb_dim, const float* __restrict__ pe,
                                       float alpha, int S, float* __restrict__ X, int64_t total) {
  pdl_entry();
  const int D = tc_emb_dim + emb_dim;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i % D);
  const int64_t bs = i / D;
  const int s = (int)(bs % S);
  const int b = (int)(bs / S);
  float v;
  if (d < tc_emb_dim) v = tc_emb[(int64_t)b * te_sb + (int64_t)s * te_ld + d];
  else v = praw[(int64_t)(b % B_hist) * p_ld + s] * __ldg(w_dt + (d - tc_emb_dim));
  X[i] = v * 1.0f + alpha * __ldg(pe + (int64_t)s * D + d);
}

int adm_build_input(const float* tc_emb, int64_t te_sb, int te_ld, int tc_emb_dim, const float* praw, int p_ld,
                    int B_hist, const float* w_dt, int emb_dim, const float* pe, float alpha, int B, int S, float* X,
                    cudaStream_t st) {
  const int64_t total = (int64_t)B * S * (tc_emb_dim + emb_dim);
  if (total <= 0) return 0;
  MTTS_REQUIRE(B_hist >= 1, "B_hist must be >= 1");
  launch_k(adm_build_input_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, tc_emb, te_sb, te_ld, tc_emb_dim, praw, p_ld,
           B_hist, w_dt, emb_dim, pe, alpha, S, X, total);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// x_last . w_predict of one row (models/megatts2.py:272-273), by one warp; every lane returns the sum.  Both readouts
// call it, so a mixed row with one weighted source reproduces the plain readout bit for bit.
__device__ __forceinline__ float adm_readout_dot(const float* __restrict__ xl, int64_t row, int D,
                                                 const float* __restrict__ w, int lane) {
  float s = 0.f;
  for (int d = lane; d < D; d += 32) s = fmaf(xl[row * D + d], __ldg(w + d), s);
  return warp_sum(s);
}

// The value a step feeds back: a pinned phone (pin[b pin_sb] >= 1, pin already at this step's phone) its frame count,
// any other phone the readout r.
__device__ __forceinline__ float adm_pinned(float r, const int32_t* __restrict__ pin, int64_t pin_sb, int b) {
  if (!pin) return r;
  const int32_t p = pin[(int64_t)b * pin_sb];
  return p >= 1 ? (float)p : r;
}

// ADM readout (models/megatts2.py:272-273): p[b, s_next] = x_last[b,:] . w_predict ; one warp per b
__global__ void adm_readout_kernel(const float* __restrict__ xl, int D, const float* __restrict__ w, int B,
                                   float* __restrict__ praw, int p_ld, int s_next, const int32_t* __restrict__ pin,
                                   int64_t pin_sb) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float s = adm_readout_dot(xl, b, D, w, lane);
  if (lane == 0) praw[(int64_t)b * p_ld + s_next] = adm_pinned(s, pin, pin_sb, b);
}
int adm_readout(const float* xl, int D, const float* w, int B, float* praw, int p_ld, int s_next, cudaStream_t st,
                const int32_t* pin, int64_t pin_sb) {
  if (B <= 0) return 0;
  launch_k(adm_readout_kernel, (unsigned)cdiv64(B, 4), 128, 0, st, xl, D, w, B, praw, p_ld, s_next, pin, pin_sb);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// Duration mix readout (the contract is stated with mtts_adm_readout_mix_f32 in include/megatts2_b200.h): one warp per
// utterance b, whose weight row is weights + b ldw.  The warp computes y of each weighted source (of every source when y_out is given) and folds the weighted
// ones into r in k order: the first term is w^ y, the later ones fmaf(w^, y, r).
constexpr int ADM_MIX_MAX_K = 8;
__global__ void adm_readout_mix_kernel(const float* __restrict__ xl, int D, const float* __restrict__ w, int K, int B,
                                       const float* __restrict__ weights, int64_t ldw, float* __restrict__ out,
                                       int64_t ld_out, float* __restrict__ y_out, int64_t ld_y,
                                       const int32_t* __restrict__ pin, int64_t pin_sb) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  float wk[ADM_MIX_MAX_K];
  float wsum = 0.f;
#pragma unroll
  for (int k = 0; k < ADM_MIX_MAX_K; ++k) {
    wk[k] = k < K ? (weights ? weights[(int64_t)b * ldw + k] : 1.f) : 0.f;
    if (wk[k] > 0.f) wsum += wk[k];             // zero weights add nothing; NaN or negative ones are skipped throughout
  }
  float r = 0.f;
  bool first = true;
#pragma unroll
  for (int k = 0; k < ADM_MIX_MAX_K; ++k) {
    if (k >= K) break;
    const bool on = wk[k] > 0.f;
    if (!on && !y_out) continue;
    const int64_t row = (int64_t)k * B + b;
    const float y = adm_readout_dot(xl, row, D, w, lane);
    if (y_out && lane == 0) y_out[row * ld_y] = y;
    if (!on) continue;
    const float wn = wk[k] / wsum;
    r = first ? wn * y : fmaf(wn, y, r);
    first = false;
  }
  if (lane == 0) out[(int64_t)b * ld_out] = adm_pinned(r, pin, pin_sb, b);
}

int adm_mix_check(int K) {
  MTTS_REQUIRE(K >= 1, "K must be >= 1");
  if (K > ADM_MIX_MAX_K)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: K = %lld sources is above the bound of %lld", "adm_readout_mix", K, ADM_MIX_MAX_K);
  return 0;
}

int adm_readout_mix(const float* xl, int D, const float* w, int K, int B, const float* weights, int64_t ldw, float* out,
                    int64_t ld_out, float* y_out, int64_t ld_y, cudaStream_t st, const int32_t* pin, int64_t pin_sb) {
  MTTS_TRY(adm_mix_check(K));
  MTTS_REQUIRE(weights || K == 1, "K > 1 sources need weights");
  MTTS_REQUIRE(D >= 1 && ldw >= 0 && ld_out >= 0 && ld_y >= 0, "D must be >= 1 and ld >= 0");
  if (B <= 0) return 0;
  MTTS_REQUIRE(xl && w && out, "null pointer");
  launch_k(adm_readout_mix_kernel, (unsigned)cdiv64(B, 4), 128, 0, st, xl, D, w, K, B, weights, ldw, out, ld_out, y_out,
           ld_y, pin, pin_sb);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// Phone -> PLM step weights (the contract is stated with mtts_mix_step_weights_f32 in include/megatts2_b200.h): one CTA
// per utterance.  The CTA scans the durations into cum[0..Tp] (cum[i] = frames of the phones before i, negative durations
// counted as 0, as length_regulate_kernel counts them); then each thread takes steps t: the phone owning frame 8t by
// length_regulate_kernel's search, then the phones after it while they start before the step's end, keeping the first
// with the most frames.  Integer arithmetic only, and the K weights are copied as bits.
constexpr int STEPW_THREADS = 256;
constexpr int STEPW_MAX_TP = 8192;
__device__ __forceinline__ int stepw_owner(const int* cum, int Tp, int r) {   // largest i < Tp with cum[i] <= r
  int lo = 0, hi = Tp;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cum[mid] <= r) lo = mid; else hi = mid;
  }
  return lo;
}
__global__ void __launch_bounds__(STEPW_THREADS)
mix_step_weights_kernel(const float* __restrict__ pw, int64_t pw_sb, int Tp, int K, const int32_t* __restrict__ dur,
                        int64_t dur_sb, int T, float* __restrict__ out) {
  extern __shared__ int cum[];   // Tp + 1
  __shared__ int s_warp[STEPW_THREADS / 32];
  pdl_entry();
  const int b = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int32_t* d = dur + (int64_t)b * dur_sb;
  const int per = (Tp + STEPW_THREADS - 1) / STEPW_THREADS;
  const int i0 = min((int)threadIdx.x * per, Tp), i1 = min(i0 + per, Tp);
  int own = 0;
  for (int i = i0; i < i1; ++i) own += max(d[i], 0);
  int incl = own;                                            // block scan: warp shuffles, then the warp totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[wp] = incl;
  __syncthreads();
  if (wp == 0) {
    int v = lane < STEPW_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    if (lane < STEPW_THREADS / 32) s_warp[lane] = v;
  }
  __syncthreads();
  int c = incl - own + (wp ? s_warp[wp - 1] : 0);
  for (int i = i0; i < i1; ++i) {
    cum[i] = c;
    c += max(d[i], 0);
  }
  if (threadIdx.x == 0) cum[Tp] = s_warp[STEPW_THREADS / 32 - 1];
  __syncthreads();
  const int L = cum[Tp];
  const int last = L > 0 ? stepw_owner(cum, Tp, L - 1) : 0;   // the last phone with a positive duration
  const uint32_t* src = reinterpret_cast<const uint32_t*>(pw + (int64_t)b * pw_sb);
  uint32_t* dst = reinterpret_cast<uint32_t*>(out + (int64_t)b * T * K);
  for (int t = threadIdx.x; t < T; t += STEPW_THREADS) {
    int p = last;
    if ((int64_t)t * 8 < L) {
      const int s0 = 8 * t, e = min(s0 + 8, L);
      int best = 0;
      for (int i = stepw_owner(cum, Tp, s0); i < Tp && cum[i] < e; ++i) {
        const int n = min(cum[i + 1], e) - max(cum[i], s0);
        if (n > best) { best = n; p = i; }
      }
    }
    for (int k = 0; k < K; ++k) dst[(int64_t)t * K + k] = src[(int64_t)p * K + k];
  }
}

int mix_step_weights(const float* pw, int64_t pw_sb, int Tp, int K, int B, const int32_t* dur, int64_t dur_sb, int T,
                     float* out, cudaStream_t st) {
  MTTS_REQUIRE(K >= 1, "K must be >= 1");
  if (K > ADM_MIX_MAX_K)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: K = %lld sources is above the bound of %lld", "mix_step_weights", K,
                ADM_MIX_MAX_K);
  MTTS_REQUIRE(Tp >= 1, "Tp must be >= 1");
  if (Tp > STEPW_MAX_TP)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: Tp = %lld phones is above the bound of %lld", "mix_step_weights", Tp,
                STEPW_MAX_TP);
  MTTS_REQUIRE(pw_sb >= 0 && dur_sb >= 0, "strides must be >= 0");
  if (B <= 0 || T <= 0) return 0;
  MTTS_REQUIRE(pw && dur && out, "null pointer");
  launch_k(mix_step_weights_kernel, (unsigned)B, STEPW_THREADS, (size_t)(Tp + 1) * sizeof(int), st, pw, pw_sb, Tp, K,
           dur, dur_sb, T, out);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// (p + 0.5).to(int32).clamp(1, 128)  (models/megatts2.py:275); praw row b holds [0, p_1..p_T]
__global__ void adm_finalize_kernel(const float* __restrict__ praw, int p_ld, int B, int T, int32_t* __restrict__ dur,
                                    float* __restrict__ raw_out) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T) return;
  const int b = i / T, t = i - b * T;
  const float p = praw[(int64_t)b * p_ld + t + 1];
  int v = (int)(p + 0.5f);             // truncation toward zero, like Tensor.to(int32)
  v = v < 1 ? 1 : (v > 128 ? 128 : v);
  dur[i] = v;
  if (raw_out) raw_out[i] = p;
}
int adm_finalize(const float* praw, int p_ld, int B, int T, int32_t* dur, float* raw_out, cudaStream_t st) {
  if (B * T <= 0) return 0;
  launch_k(adm_finalize_kernel, (unsigned)cdiv64((int64_t)B * T, 256), 256, 0, st, praw, p_ld, B, T, dur, raw_out);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// Duration fit (the contract is stated with mtts_fit_durations_f32 in include/megatts2_b200.h): one CTA per utterance,
// each thread a contiguous run of phones.  Free phone i with weight w_i >= 0 has the candidates v_ik = fl64(w_i / (k + ½)),
// k = 1..FIT_EXTRA.  fp64 division is correctly rounded and two different candidates differ by at least 2^-33 of their
// size (w_i (2k+1) vs w_j (2m+1) are fp32 values times integers <= 255), so the fp64 values order and tie exactly as the
// rationals do.  The CTA bisects the bit pattern of a threshold th >= 0 for the largest th with N candidates >= th (the
// N-th largest candidate), then gives each phone its candidates > th and hands the N - #(> th) candidates equal to th to
// the phones in index order by a block scan.
constexpr int FIT_THREADS = 256;
constexpr int FIT_MAX_TP = 8192;
constexpr int FIT_EXTRA = 127;            // frames above the first that a free phone can take (durations 1..128)

// #{k in 1..FIT_EXTRA : fl64(w / (k + 0.5)) >= th} for w >= 0, th >= 0: an estimate, then exact steps to the boundary
__device__ __forceinline__ int fit_count_ge(float w, double th) {
  if (th <= 0.0) return FIT_EXTRA;
  if (w <= 0.f) return 0;
  const double wd = w;
  const double e = wd / th - 0.5;
  int k = e >= (double)FIT_EXTRA ? FIT_EXTRA : (e < 1.0 ? 0 : (int)e);
  while (k < FIT_EXTRA && wd / (k + 1.5) >= th) ++k;
  while (k > 0 && wd / (k + 0.5) < th) --k;
  return k;
}

// block-wide sums of two ints; every thread gets them.  s holds 2 * (FIT_THREADS / 32) ints.
__device__ __forceinline__ int2 fit_block_sum2(int a, int c, int* s) {
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  __syncthreads();                                           // s is free: the previous call's readers are done
  if (lane == 0) { s[wp] = a; s[FIT_THREADS / 32 + wp] = c; }
  __syncthreads();
  int2 r = make_int2(0, 0);
#pragma unroll
  for (int i = 0; i < FIT_THREADS / 32; ++i) { r.x += s[i]; r.y += s[FIT_THREADS / 32 + i]; }
  return r;
}

__global__ void __launch_bounds__(FIT_THREADS)
fit_durations_kernel(const float* __restrict__ raw, int64_t raw_sb, int Tp, const float* __restrict__ scale,
                     int64_t sc_sb, int64_t sc_st, const int32_t* __restrict__ pin, int64_t pin_sb,
                     const int32_t* __restrict__ total, int32_t* __restrict__ dur, int64_t dur_sb) {
  extern __shared__ float w_s[];                              // Tp: w_i of a free phone, -1 for a pinned one
  __shared__ int s_red[2 * (FIT_THREADS / 32)];
  pdl_entry();
  const int b = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int per = (Tp + FIT_THREADS - 1) / FIT_THREADS;
  const int i0 = min((int)threadIdx.x * per, Tp), i1 = min(i0 + per, Tp);
  int32_t* d = dur + (int64_t)b * dur_sb;
  int n_free = 0, pinned = 0;
  for (int i = i0; i < i1; ++i) {
    const int32_t p = pin ? pin[(int64_t)b * pin_sb + i] : -1;
    if (p >= 1) {
      w_s[i] = -1.f;
      pinned += p;
      d[i] = p;
      continue;
    }
    const float c = scale ? scale[(int64_t)b * sc_sb + (int64_t)i * sc_st] : 1.f;
    float w = __fmul_rn(raw[(int64_t)b * raw_sb + i], c);
    if (!(w > 0.f) || isinf(w)) w = 0.f;                      // NaN, +-inf and w <= 0 count as 0
    w_s[i] = w;
    ++n_free;
    if (!total) {                                             // adm_finalize's rounding of w
      const int v = (int)(w + 0.5f);
      d[i] = v < 1 ? 1 : (v > FIT_EXTRA + 1 ? FIT_EXTRA + 1 : v);
    }
  }
  if (!total) return;
  const int2 fp = fit_block_sum2(n_free, pinned, s_red);
  // frames above one per free phone; the host checks feasibility, the device clamps to the feasible range
  const int N = max(0, min(total[b] - fp.y - fp.x, FIT_EXTRA * fp.x));
  // the largest th (as fp64 bits) with F(th) = #{candidates >= th} >= N: F(0) = FIT_EXTRA |F| >= N, F(+inf) = 0 < N
  unsigned long long lo = 0ull, hi = 0x7FF0000000000000ull;
  while (N > 0 && hi - lo > 1) {
    const unsigned long long mid = lo + ((hi - lo) >> 1);
    const double th = __longlong_as_double((long long)mid);
    int cnt = 0;
    for (int i = i0; i < i1; ++i)
      if (w_s[i] >= 0.f) cnt += fit_count_ge(w_s[i], th);
    if (fit_block_sum2(cnt, 0, s_red).x >= N) lo = mid; else hi = mid;
  }
  // each free phone: g candidates > th (>= the next double), e == th; the N - G ties go to the lowest phone indices
  const double th = __longlong_as_double((long long)lo), th_up = __longlong_as_double((long long)hi);
  int g_own = 0, e_own = 0;
  for (int i = i0; i < i1; ++i)
    if (N > 0 && w_s[i] >= 0.f) {
      const int g = fit_count_ge(w_s[i], th_up);
      g_own += g;
      e_own += fit_count_ge(w_s[i], th) - g;
    }
  const int G = fit_block_sum2(g_own, 0, s_red).x;
  int incl = e_own;                                          // block scan of the ties: warp shuffles, then warp totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  __syncthreads();
  if (lane == 31) s_red[wp] = incl;
  __syncthreads();
  int before = incl - e_own;
  for (int j = 0; j < wp; ++j) before += s_red[j];
  int left = N - G - before;                                 // ties still to hand out when this thread's run starts
  for (int i = i0; i < i1; ++i) {
    if (w_s[i] < 0.f) continue;
    int g = 0, t = 0;
    if (N > 0) {
      g = fit_count_ge(w_s[i], th_up);
      const int e = fit_count_ge(w_s[i], th) - g;
      t = max(0, min(left, e));
      left -= e;
    }
    d[i] = 1 + g + t;
  }
}

int fit_durations(const float* raw, int64_t raw_sb, int Tp, int B, const float* scale, int64_t sc_sb, int64_t sc_st,
                  const int32_t* pin, int64_t pin_sb, const int32_t* total, int32_t* dur, int64_t dur_sb, cudaStream_t st) {
  MTTS_REQUIRE(Tp >= 1, "Tp must be >= 1");
  if (Tp > FIT_MAX_TP)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: Tp = %lld phones is above the bound of %lld", "fit_durations", Tp, FIT_MAX_TP);
  MTTS_REQUIRE(raw_sb >= 0 && sc_sb >= 0 && sc_st >= 0 && pin_sb >= 0 && dur_sb >= 0, "strides must be >= 0");
  if (B <= 0) return 0;
  MTTS_REQUIRE(raw && dur, "null pointer");
  launch_k(fit_durations_kernel, (unsigned)B, FIT_THREADS, (size_t)Tp * sizeof(float), st, raw, raw_sb, Tp, scale, sc_sb,
           sc_st, pin, pin_sb, total, dur, dur_sb);
  MTTS_CHECK_LAUNCH();
  return 0;
}

}  // namespace mtts
