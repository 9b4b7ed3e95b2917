// Backward / training-mode kernels (SURVEY.md 8f-4): what autograd needs around the tensor-core GEMMs so that
// MegaPLMTrainer / MegaADMTrainer.training_step (models/trainer.py:243-268, 334-355) run forward AND backward through the
// drop-in modules.  The dense contractions of the backward pass (dX = dY W, dW = dY^T X) go through the same wgmma
// tap-GEMM as the forward (megatts2_b200/autograd.py); this file holds the rest:
//   bmm_kernel            strided batched matmul (fp32 FFMA) for the attention products and for shapes the tensor-core
//                         engine does not take (K = 1 embeddings of the ADM, ragged row counts)
//   softmax_fwd / _bwd    training attention: P = softmax(S + mask) materialised (dropout needs it), dS = P (dP - <dP, P>)
//   layernorm_bwd         dx per row + per-CTA partial d-gamma / d-beta (reduced by colsum: fixed order, deterministic)
//   colsum, relu_bwd, embedding_bwd, rowdot
// All fp32; rows are reduced with warp shuffles; HBM-bound except bmm.
#include <float.h>
#include <math.h>

#include "kernels.h"

namespace mtts {

// ------------------------------------------------------------------------------------------ strided batched matmul
// C[z][m, n] = alpha * sum_k A[z][m, k] * B[z][k, n] (+ C) with z = (z1, z2) and arbitrary element strides, so transposed
// operands and (B, T, H, dh) head views need no copies.  64 x 64 tile, 16-wide k step, 4 x 4 micro-tile per thread.
struct BmmArgs {
  const float* a; int64_t a_s1, a_s2, a_sm, a_sk;
  const float* b; int64_t b_s1, b_s2, b_sk, b_sn;
  float* c; int64_t c_s1, c_s2, c_sm, c_sn;
  int Z2, M, N, K;
  float alpha; int accumulate;
};

__global__ void __launch_bounds__(256)
bmm_kernel(const BmmArgs g) {
  pdl_entry();
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int z = blockIdx.z, z1 = z / g.Z2, z2 = z - z1 * g.Z2;
  const float* A = g.a + z1 * g.a_s1 + z2 * g.a_s2;
  const float* B = g.b + z1 * g.b_s1 + z2 * g.b_s2;
  float* Cp = g.c + z1 * g.c_s1 + z2 * g.c_s2;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < g.K; k0 += 16) {
    // 64 x 16 of A and 16 x 64 of B: 1024 elements each, 4 per thread; the faster-varying index follows the smaller stride
    for (int e = tid; e < 1024; e += 256) {
      int m, k;
      if (g.a_sk <= g.a_sm) { k = e & 15; m = e >> 4; } else { m = e & 63; k = e >> 6; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < g.M && gk < g.K) ? A[(int64_t)gm * g.a_sm + (int64_t)gk * g.a_sk] : 0.f;
      int n, kk;
      if (g.b_sn <= g.b_sk) { n = e & 63; kk = e >> 6; } else { kk = e & 15; n = e >> 4; }
      const int gn = n0 + n, gk2 = k0 + kk;
      Bs[kk][n] = (gn < g.N && gk2 < g.K) ? B[(int64_t)gk2 * g.b_sk + (int64_t)gn * g.b_sn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= g.N) continue;
      float* dst = Cp + (int64_t)gm * g.c_sm + (int64_t)gn * g.c_sn;
      const float v = g.alpha * acc[i][j];
      *dst = g.accumulate ? *dst + v : v;
    }
  }
}

int bmm(const BmmArgs& g, int Z1, cudaStream_t st) {
  MTTS_REQUIRE(g.a && g.b && g.c && g.M >= 0 && g.N >= 0 && g.K >= 0 && Z1 >= 0 && g.Z2 >= 1, "bad arguments");
  if (g.M == 0 || g.N == 0 || Z1 == 0) return 0;
  MTTS_REQUIRE((int64_t)Z1 * g.Z2 <= 65535 && cdiv64(g.M, 64) <= 65535, "grid too large");
  dim3 grid((unsigned)cdiv64(g.N, 64), (unsigned)cdiv64(g.M, 64), (unsigned)(Z1 * g.Z2));
  launch_k(bmm_kernel, grid, 256, 0, st, g);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------ training softmax
// rows of S (R, Tk): p = softmax(s + mask_row); P <- p (saved for the backward), Pd <- p * keep (keep: 0 or 1 / (1 - p_drop),
// may be null -> Pd = P and may alias it).  mask row of global row r = (b, h, q): mask + b*sb + h*sh + q*sq.
__global__ void __launch_bounds__(256)
softmax_fwd_kernel(const float* __restrict__ S, const float* __restrict__ mask, int64_t m_sb, int64_t m_sh, int64_t m_sq, int H,
                   int Tq, int Tk, const float* __restrict__ keep, float* P, float* Pd, int64_t rows) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int q = (int)(r % Tq);
  const int64_t bh = r / Tq;
  const int h = (int)(bh % H), b = (int)(bh / H);
  const float* s = S + r * Tk;
  const float* mr = mask ? mask + b * m_sb + h * m_sh + q * m_sq : nullptr;
  float mx = -INFINITY;
  for (int j = lane; j < Tk; j += 32) mx = fmaxf(mx, s[j] + (mr ? mr[j] : 0.f));
  mx = warp_max(mx);
  const float mu = (mx == -INFINITY) ? 0.f : mx;
  float sum = 0.f;
  for (int j = lane; j < Tk; j += 32) sum += expf(s[j] + (mr ? mr[j] : 0.f) - mu);
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  for (int j = lane; j < Tk; j += 32) {
    const float p = expf(s[j] + (mr ? mr[j] : 0.f) - mu) * inv;
    P[r * Tk + j] = p;
    if (Pd != P || keep) Pd[r * Tk + j] = keep ? p * keep[r * Tk + j] : p;
  }
}
// dS = P * (dP - sum_j dP_j P_j),  dP = dPd * keep
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const float* __restrict__ P, const float* __restrict__ dPd, const float* __restrict__ keep, float* __restrict__ dS,
                   int Tk, int64_t rows) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* p = P + r * Tk;
  const float* d = dPd + r * Tk;
  const float* kp = keep ? keep + r * Tk : nullptr;
  float t = 0.f;
  for (int j = lane; j < Tk; j += 32) t = fmaf(d[j] * (kp ? kp[j] : 1.f), p[j], t);
  t = warp_sum(t);
  for (int j = lane; j < Tk; j += 32) dS[r * Tk + j] = p[j] * (d[j] * (kp ? kp[j] : 1.f) - t);
}
int softmax_fwd(const float* S, const float* mask, int64_t m_sb, int64_t m_sh, int64_t m_sq, int B, int H, int Tq, int Tk,
                const float* keep, float* P, float* Pd, cudaStream_t st) {
  MTTS_REQUIRE(S && P && Pd && Tk > 0, "bad arguments");
  const int64_t rows = (int64_t)B * H * Tq;
  if (rows <= 0) return 0;
  launch_k(softmax_fwd_kernel, (unsigned)cdiv64(rows, 8), 256, 0, st, S, mask, m_sb, m_sh, m_sq, H, Tq, Tk, keep, P, Pd, rows);
  MTTS_CHECK_LAUNCH();
  return 0;
}
int softmax_bwd(const float* P, const float* dPd, const float* keep, float* dS, int Tk, int64_t rows, cudaStream_t st) {
  MTTS_REQUIRE(P && dPd && dS && Tk > 0, "bad arguments");
  if (rows <= 0) return 0;
  launch_k(softmax_bwd_kernel, (unsigned)cdiv64(rows, 8), 256, 0, st, P, dPd, keep, dS, Tk, rows);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------ LayerNorm backward
// one warp per row (8 rows per CTA): recompute mean / rstd, dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma;
// the CTA's 8 rows are summed into partial[blockIdx.x][0 | 1][C] (d-gamma | d-beta) in a fixed order.
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ dy, float* __restrict__ dx,
                     float* __restrict__ partial, int64_t rows, int C, float eps) {
  pdl_entry();
  extern __shared__ float sm[];                      // [8][2][C]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * 8 + w;
  float* mine = sm + (size_t)w * 2 * C;
  if (r < rows) {
    const float* xr = x + r * C;
    const float* dr = dy + r * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += xr[c];
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
    for (int c = lane; c < C; c += 32) { const float a = xr[c] - mean; q += a * a; }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
    float m1 = 0.f, m2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * rstd, gg = dr[c] * __ldg(gamma + c);
      m1 += gg;
      m2 = fmaf(gg, xh, m2);
      mine[c] = dr[c] * xh;                          // d-gamma contribution
      mine[C + c] = dr[c];                           // d-beta contribution
    }
    m1 = warp_sum(m1) / (float)C;
    m2 = warp_sum(m2) / (float)C;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * rstd, gg = dr[c] * __ldg(gamma + c);
      dx[r * C + c] = rstd * (gg - m1 - xh * m2);
    }
  } else {
    for (int c = lane; c < 2 * C; c += 32) mine[c] = 0.f;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += 256) {
    float t = 0.f;
#pragma unroll
    for (int ww = 0; ww < 8; ++ww) t += sm[(size_t)ww * 2 * C + c];
    partial[(int64_t)blockIdx.x * 2 * C + c] = t;
  }
}
int layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx, float* partial, int64_t rows, int C, float eps,
                  cudaStream_t st) {
  MTTS_REQUIRE(x && gamma && dy && dx && partial && C > 0 && C <= 3072, "bad arguments (C <= 3072: 8 rows x 2 x C floats of shared memory)");
  if (rows <= 0) return 0;
  const size_t smem = sizeof(float) * 16 * (size_t)C;
  static std::atomic<uint64_t> configured{0};
  const int dev = cur_device();
  if (smem > 48 * 1024 && !(configured.load(std::memory_order_relaxed) & (1ull << dev))) {
    cudaError_t e = cudaFuncSetAttribute(layernorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * 3072 * 4);
    if (e != cudaSuccess) {
      cudaGetLastError();      // do not leave the error for the next launch check
      return fail(MTTS_ERR_CUDA, "%s: cudaFuncSetAttribute failed: %lld", "layernorm_bwd", (long long)e);
    }
    configured.fetch_or(1ull << dev, std::memory_order_relaxed);
  }
  launch_k(layernorm_bwd_kernel, (unsigned)cdiv64(rows, 8), 256, smem, st, x, gamma, dy, dx, partial, rows, C, eps);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// out[c] = sum_r in[r * ld + c] in row order (deterministic); one thread per column, coalesced across the warp
__global__ void colsum_kernel(const float* __restrict__ in, int64_t ld, int64_t rows, int C, float* __restrict__ out, int accumulate) {
  pdl_entry();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int64_t r = 0;
  for (; r + 4 <= rows; r += 4) {
    a0 += in[r * ld + c]; a1 += in[(r + 1) * ld + c]; a2 += in[(r + 2) * ld + c]; a3 += in[(r + 3) * ld + c];
  }
  for (; r < rows; ++r) a0 += in[r * ld + c];
  const float t = (a0 + a1) + (a2 + a3);
  out[c] = accumulate ? out[c] + t : t;
}
int colsum(const float* in, int64_t ld, int64_t rows, int C, float* out, int accumulate, cudaStream_t st) {
  MTTS_REQUIRE(in && out && C > 0 && rows >= 0, "bad arguments");
  launch_k(colsum_kernel, (unsigned)cdiv64(C, 128), 128, 0, st, in, ld, rows, C, out, accumulate);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// dx = dy where y > 0 else 0 (ReLU backward from the saved OUTPUT)
__global__ void relu_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx, int64_t n) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dx[i] = y[i] > 0.f ? dy[i] : 0.f;
}
int relu_bwd(const float* y, const float* dy, float* dx, int64_t n, cudaStream_t st) {
  MTTS_REQUIRE(y && dy && dx && n >= 0, "bad arguments");
  if (n == 0) return 0;
  launch_k(relu_bwd_kernel, (unsigned)cdiv64(n, 256), 256, 0, st, y, dy, dx, n);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// dW[ids[r], :] += dy[r, :]   (nn.Embedding backward; dW zeroed by the caller)
__global__ void embedding_bwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dy, int64_t rows, int D, int vocab,
                                     float* __restrict__ dW) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * D) return;
  const int64_t r = i / D;
  const int d = (int)(i - r * D);
  int64_t id = ids[r];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  atomicAdd(dW + id * D + d, dy[i]);
}
int embedding_bwd(const int64_t* ids, const float* dy, int64_t rows, int D, int vocab, float* dW, cudaStream_t st) {
  MTTS_REQUIRE(ids && dy && dW && D > 0 && vocab > 0, "bad arguments");
  if (rows <= 0) return 0;
  launch_k(embedding_bwd_kernel, (unsigned)cdiv64(rows * D, 256), 256, 0, st, ids, dy, rows, D, vocab, dW);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// out[r] = sum_c a[r, c] * b[(r % period), c]   (d-alpha of the sine positional embedding: rows of dy against pe rows)
__global__ void rowdot_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t rows, int C, int period,
                              float* __restrict__ out) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* ar = a + r * C;
  const float* br = b + (r % period) * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(ar[c], br[c], s);
  s = warp_sum(s);
  if (lane == 0) out[r] = s;
}
int rowdot(const float* a, const float* b, int64_t rows, int C, int period, float* out, cudaStream_t st) {
  MTTS_REQUIRE(a && b && out && C > 0 && period > 0, "bad arguments");
  if (rows <= 0) return 0;
  launch_k(rowdot_kernel, (unsigned)cdiv64(rows, 8), 256, 0, st, a, b, rows, C, period, out);
  MTTS_CHECK_LAUNCH();
  return 0;
}

}  // namespace mtts

using namespace mtts;
extern "C" {
int mtts_bmm_f32(const float* a, int64_t a_s1, int64_t a_s2, int64_t a_sm, int64_t a_sk, const float* b, int64_t b_s1,
                 int64_t b_s2, int64_t b_sk, int64_t b_sn, float* c, int64_t c_s1, int64_t c_s2, int64_t c_sm, int64_t c_sn,
                 int32_t Z1, int32_t Z2, int32_t M, int32_t N, int32_t K, float alpha, int32_t accumulate, void* stream) {
  BmmArgs g{a, a_s1, a_s2, a_sm, a_sk, b, b_s1, b_s2, b_sk, b_sn, c, c_s1, c_s2, c_sm, c_sn, Z2, M, N, K, alpha, accumulate};
  return bmm(g, Z1, (cudaStream_t)stream);
}
int mtts_softmax_fwd_f32(const float* S, const float* mask, int64_t m_sb, int64_t m_sh, int64_t m_sq, int32_t B, int32_t H,
                         int32_t Tq, int32_t Tk, const float* keep, float* P, float* Pd, void* stream) {
  return softmax_fwd(S, mask, m_sb, m_sh, m_sq, B, H, Tq, Tk, keep, P, Pd, (cudaStream_t)stream);
}
int mtts_softmax_bwd_f32(const float* P, const float* dPd, const float* keep, float* dS, int32_t Tk, int64_t rows, void* stream) {
  return softmax_bwd(P, dPd, keep, dS, Tk, rows, (cudaStream_t)stream);
}
int mtts_layernorm_bwd_f32(const float* x, const float* gamma, const float* dy, float* dx, float* partial, int64_t rows, int32_t C,
                           float eps, void* stream) {
  return layernorm_bwd(x, gamma, dy, dx, partial, rows, C, eps, (cudaStream_t)stream);
}
int mtts_colsum_f32(const float* in, int64_t ld, int64_t rows, int32_t C, float* out, int32_t accumulate, void* stream) {
  return colsum(in, ld, rows, C, out, accumulate, (cudaStream_t)stream);
}
int mtts_relu_bwd_f32(const float* y, const float* dy, float* dx, int64_t n, void* stream) {
  return relu_bwd(y, dy, dx, n, (cudaStream_t)stream);
}
int mtts_embedding_bwd_f32(const int64_t* ids, const float* dy, int64_t rows, int32_t D, int32_t vocab, float* dW, void* stream) {
  return embedding_bwd(ids, dy, rows, D, vocab, dW, (cudaStream_t)stream);
}
int mtts_rowdot_f32(const float* a, const float* b, int64_t rows, int32_t C, int32_t period, float* out, void* stream) {
  return rowdot(a, b, rows, C, period, out, (cudaStream_t)stream);
}
}
