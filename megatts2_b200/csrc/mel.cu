// Mel front end: reflect-padded STFT (n_fft = win = 1024, hop 256) -> |.| -> banded slaney
// filterbank -> log(max(., clamp)).  Replaces extract_mel_spec (modules/tokenizer.py:107-125,
// speechbrain mel_spectogram -> torchaudio MelSpectrogram; SURVEY.md Appendix B).
//
// One warp per frame: the 1024 real samples are packed as 512 complex points and transformed
// by three register-resident radix-8 Stockham passes (8*8*8) that exchange data through a
// per-warp padded shared buffer (__syncwarp only), then untangled to the 513 one-sided bins,
// whose magnitudes overwrite the exchange buffer.  A CTA owns 16 consecutive frames of one clip
// (two rounds of 8, one frame per warp), stages their 4864-sample span once (each sample is
// needed by 4 frames), applies the banded filterbank CTA-wide per round (lanes = 8 frames x 4
// tap phases of one mel: conflict-free magnitude reads, broadcast tap reads) and writes an
// 80 x 16 output tile coalesced.
#include <math.h>
#include <mutex>

#include "common.cuh"

namespace mtts {

constexpr int MEL_NFFT = 1024, MEL_HOP = 256, MEL_NZ = 512;
constexpr int MEL_WARPS = 8, MEL_ROUNDS = 2, MEL_FPB = MEL_WARPS * MEL_ROUNDS;   // 16 frames per CTA, 8 at a time
// float2 slots of one warp's exchange buffer: slot(i) = i + (i >> 4) (one pad per 16) up to slot(512) = 544, rounded
// so that the float view of the buffer (the frame's 513 magnitudes, written over it after the untangle) has a frame
// stride of 4 mod 32 banks and 16-byte aligned rows
constexpr int MEL_ZPAD = 546;
constexpr int MEL_FBW = 1536;                   // grouped filterbank floats staged in shared memory (slaney 80: 1344, slaney 128: 1584)
constexpr int MEL_MAXG = 32;                    // groups of 4 mels
constexpr int MEL_SPAN = MEL_NFFT + (MEL_FPB - 1) * MEL_HOP;   // 4864 samples cover the CTA's 16 frames

__device__ float2 g_tw1024[1024];   // exp(-2*pi*i*k/1024), filled once per process in fp64
// per-lane twiddles of the second and third radix-8 passes, laid out so that a warp's fetch of one is one 256-byte
// row: [r - 1][lane] = w^(16 r (lane & 7)) for rows 0..6, w^(2 r lane) for rows 7..13
__device__ float2 g_tw_pass[14][32];

__global__ void mel_init_twiddle_kernel() {
  pdl_entry();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < 1024) {
    double s, c;
    sincospi(2.0 * (double)k / 1024.0, &s, &c);
    g_tw1024[k] = make_float2((float)c, (float)(-s));
  }
  if (k < 14 * 32) {
    const int row = k >> 5, lane = k & 31, r = (row % 7) + 1;
    const int e = (row < 7) ? 16 * r * (lane & 7) : 2 * r * lane;
    double s, c;
    sincospi(2.0 * (double)e / 1024.0, &s, &c);
    g_tw_pass[row][lane] = make_float2((float)c, (float)(-s));
  }
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ void bf2(float2& a, float2& b) {
  const float2 t = a;
  a = make_float2(t.x + b.x, t.y + b.y);
  b = make_float2(t.x - b.x, t.y - b.y);
}
__device__ __forceinline__ void fft4_inplace(float2& a0, float2& a1, float2& a2, float2& a3) {
  bf2(a0, a2);
  bf2(a1, a3);
  a3 = make_float2(a3.y, -a3.x);   // * (-i)
  bf2(a0, a1);
  bf2(a2, a3);
}
// forward 8-point DFT; natural-order result is (v0,v4,v2,v6,v1,v5,v3,v7)
__device__ __forceinline__ void fft8_inplace(float2* v) {
  const float s = 0.70710678118654752440f;
  bf2(v[0], v[4]);
  bf2(v[1], v[5]);
  bf2(v[2], v[6]);
  bf2(v[3], v[7]);
  v[5] = make_float2((v[5].x + v[5].y) * s, (v[5].y - v[5].x) * s);
  v[6] = make_float2(v[6].y, -v[6].x);
  v[7] = make_float2((-v[7].x + v[7].y) * s, (-v[7].x - v[7].y) * s);
  fft4_inplace(v[0], v[1], v[2], v[3]);
  fft4_inplace(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ int zpad(int i) { return i + (i >> 3); }

__device__ __forceinline__ float sqrt_approx(float x) {   // one MUFU.SQRT: max relative error 2^-23, sqrt(0) = 0
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(MEL_WARPS * 32, 3)
mel_kernel(const float* __restrict__ wav, int64_t wav_sb, int L_max, const int32_t* __restrict__ lens,
           const float* __restrict__ window,
           const float* __restrict__ fb_w, const int32_t* __restrict__ fb_off, const int32_t* __restrict__ fb_start,
           int n_mels, float clamp_min, float* __restrict__ out, int64_t out_sb, int64_t out_sm, int64_t out_sf,
           int vec_ok) {
  pdl_entry();
  constexpr int NT = MEL_WARPS * 32;
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                                  // [SPAN]
  float* win = xs + MEL_SPAN;                        // [1024]
  float2* zb = reinterpret_cast<float2*>(win + MEL_NFFT);   // [WARPS][ZPAD]; the frame's magnitudes overwrite it
  float* otile = reinterpret_cast<float*>(zb + MEL_WARPS * MEL_ZPAD);   // [128][FPB]
  float* fbw_s = otile + 128 * MEL_FPB;              // [MEL_FBW] grouped filterbank blocks
  int4* s_desc = reinterpret_cast<int4*>(fbw_s + MEL_FBW);   // [4 * MAXG] per (group, mel in group): first bin,
                                                             // weight offset, taps / 4, mel index or -1

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * MEL_FPB;
  // ragged batches (bulk extraction): clip b holds lens[b] <= L_max valid samples; its reflection and frame
  // count follow ITS length.  CTA-uniform exit for the frames past a short clip's end.
  const int L = lens ? min(lens[b], L_max) : L_max;
  const int F = 1 + L / MEL_HOP;
  if (f0 >= F || L <= MEL_NFFT / 2) return;
  const float* wv = wav + (int64_t)b * wav_sb;
  const int g0 = f0 * MEL_HOP - MEL_NFFT / 2;
  // stage the CTA's sample span once (each sample is needed by 4 frames).  Interior tiles (no reflection, 16-byte
  // aligned) use batched float4 loads so that all of a thread's global requests are in flight together; edge
  // tiles take the scalar reflect path.
  const bool interior = vec_ok && g0 >= 0 && (g0 + MEL_SPAN) <= L;
  if (interior) {
    constexpr int NV = MEL_SPAN / 4;                           // 1216 float4
    constexpr int PER = (NV + NT - 1) / NT;
    const float4* src = reinterpret_cast<const float4*>(wv + g0);
    float4 v[PER];
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int i = tid + q * NT;
      if (i < NV) v[q] = __ldg(src + i);
    }
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int i = tid + q * NT;
      if (i < NV) *reinterpret_cast<float4*>(xs + 4 * i) = v[q];
    }
  } else {
    const int need = min(MEL_SPAN, (F - f0 - 1) * MEL_HOP + MEL_NFFT);   // frames past the clip's end are never read
    for (int i = tid; i < need; i += NT) {
      int g = g0 + i;
      if (g < 0) g = -g;
      if (g >= L) g = 2 * (L - 1) - g;
      xs[i] = (g >= 0 && g < L) ? __ldg(wv + g) : 0.f;
    }
  }
  {
    // the packed-real untangle yields 2 X[k]; the factor 1/2 rides on the window (exact)
    const float4* wsrc = reinterpret_cast<const float4*>(window);   // 1024 floats, 16-byte aligned (checked on host)
    float4 wq = __ldg(wsrc + tid);                                  // 256 threads x float4 = 1024
    wq.x *= 0.5f; wq.y *= 0.5f; wq.z *= 0.5f; wq.w *= 0.5f;
    *reinterpret_cast<float4*>(win + 4 * tid) = wq;
  }
  const int ngroups = (n_mels + 3) >> 2;
  const int n_fbw = fb_off[ngroups];
  const bool staged = n_fbw <= MEL_FBW;              // otherwise the blocks are read from global memory
  if (staged)
    for (int i = tid; i < n_fbw; i += NT) fbw_s[i] = __ldg(fb_w + i);
  if (tid < 4 * ngroups) {
    const int g = tid >> 2, o = fb_off[g], len = (fb_off[g + 1] - o) >> 2;   // taps per mel, a multiple of 4
    s_desc[tid] = make_int4(fb_start[tid], o + (tid & 3) * len, len >> 2, tid < n_mels ? tid : -1);
  }
  // twiddles of the second pass (k = lane & 7) and the third (k = lane; its upper half is this times a constant)
  // stay in registers across the warp's frames
  float2 tw1[8], tw2[8];
#pragma unroll
  for (int r = 1; r < 8; ++r) {
    tw1[r] = g_tw_pass[r - 1][lane];
    tw2[r] = g_tw_pass[6 + r][lane];
  }
  __syncthreads();

  // every shared-memory address of the transform is one of these per-lane bases plus a compile-time constant:
  // slot(i) = i + (i >> 4) (one pad per 16 float2) is additive over multiples of 16.  Conflict-free (16 lanes x 8
  // bytes per wavefront) for every access but the second pass's stores (2-way on 4 of 16 lanes).
  float2* z = zb + w * MEL_ZPAD;
  float2* z_nat = z + lane + (lane >> 4);                    // slot(lane + 32h + 64r) = z_nat + 34h + 68r
  float2* z_st0 = z + 8 * lane + (lane >> 1);                // slot(8j + q), j = lane + 32h: z_st0 + 272h + q
  float2* z_st1 = z + 68 * (lane >> 3) + (lane & 7);         // slot((j/8)*64 + (j&7) + 8q) = z_st1 + 272h + 8q + (q>>1)
  const float2* z_rev = z + (512 - lane) + ((512 - lane) >> 4);   // slot(512 - lane - 32i) = z_rev - 34i

  for (int rd = 0; rd < MEL_ROUNDS; ++rd) {
    const int fl = rd * MEL_WARPS + w;
    if (f0 + fl < F) {   // warp-uniform
      const float2* xf2 = reinterpret_cast<const float2*>(xs + fl * MEL_HOP) + lane;
      const float2* wn2 = reinterpret_cast<const float2*>(win) + lane;
      float2 v[2][8];
      // ---- pass 0 (Ns = 1): no twiddles; inputs straight from the windowed samples
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float2 xv = xf2[32 * h + 64 * r];
          const float2 wv2 = wn2[32 * h + 64 * r];
          v[h][r] = make_float2(xv.x * wv2.x, xv.y * wv2.y);
        }
        fft8_inplace(v[h]);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2* zs = z_st0 + 272 * h;
        zs[0] = v[h][0]; zs[1] = v[h][4]; zs[2] = v[h][2]; zs[3] = v[h][6];
        zs[4] = v[h][1]; zs[5] = v[h][5]; zs[6] = v[h][3]; zs[7] = v[h][7];
      }
      __syncwarp();
      // ---- pass 1 (Ns = 8): twiddle w^(r*k), k = j & 7 (both halves of a lane share it)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float2 a = z_nat[34 * h + 68 * r];
          v[h][r] = (r > 0) ? cmul(a, tw1[r]) : a;
        }
        fft8_inplace(v[h]);
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2* zs = z_st1 + 272 * h;
        zs[0] = v[h][0]; zs[8] = v[h][4]; zs[17] = v[h][2]; zs[25] = v[h][6];
        zs[34] = v[h][1]; zs[42] = v[h][5]; zs[51] = v[h][3]; zs[59] = v[h][7];
      }
      __syncwarp();
      // ---- pass 2 (Ns = 64): twiddle w^(r*k), k = j; the upper half's is the lower half's times exp(-2 pi i r/16)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float2 a = z_nat[34 * h + 68 * r];
          if (r > 0) {
            float2 t = tw2[r];
            if (h == 1) {
              constexpr float C16[8] = {1.f, 0.92387953251128674f, 0.70710678118654752f, 0.38268343236508977f, 0.f,
                                        -0.38268343236508977f, -0.70710678118654752f, -0.92387953251128674f};
              constexpr float S16[8] = {0.f, -0.38268343236508977f, -0.70710678118654752f, -0.92387953251128674f, -1.f,
                                        -0.92387953251128674f, -0.70710678118654752f, -0.38268343236508977f};
              t = cmul(t, make_float2(C16[r], S16[r]));
            }
            v[h][r] = cmul(a, t);
          } else {
            v[h][r] = a;
          }
        }
        fft8_inplace(v[h]);
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2* zs = z_nat + 34 * h;
        zs[0] = v[h][0]; zs[68] = v[h][4]; zs[136] = v[h][2]; zs[204] = v[h][6];
        zs[272] = v[h][1]; zs[340] = v[h][5]; zs[408] = v[h][3]; zs[476] = v[h][7];
      }
      if (lane == 0) z[512 + 32] = v[0][0];   // Z[512] := Z[0] (slot(512)), so that bin 0 needs no special case
      __syncwarp();
      // ---- untangle the packed real transform: bins k and 512-k from Z[k], Z[512-k].  All of the lane's bins are
      // formed in registers first; the magnitudes then overwrite the exchange buffer (as floats [0, 513)).
      //   X[k] = (a + conj c) + w^k (a - conj c) / i,   X[512-k] = conj((a + conj c) - w^k (a - conj c) / i)
      // (the 1/2 of the even / odd split is already in the window)
      float mlo[9], mhi[8];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        // i < 8: k = lane + 32 i (k = 0 pairs with the copy of Z[0] at 512); i = 8: k = 256 for every lane
        const float2 a = (i < 8) ? z_nat[34 * i] : z[256 + 16];
        const float2 c = (i < 8) ? z_rev[-34 * i] : a;
        const float2 tw = (i < 8) ? g_tw1024[lane + 32 * i] : make_float2(0.f, -1.f);
        const float ex = a.x + c.x, ey = a.y - c.y;
        const float ox = a.y + c.y, oy = c.x - a.x;
        const float tx = tw.x * ox - tw.y * oy, ty = tw.x * oy + tw.y * ox;
        const float pr = ex + tx, pi = ey + ty;
        mlo[i] = sqrt_approx(pr * pr + pi * pi);
        if (i < 8) {
          const float qr = ex - tx, qi = ey - ty;
          mhi[i] = sqrt_approx(qr * qr + qi * qi);
        }
      }
      __syncwarp();
      float* mg = reinterpret_cast<float*>(z);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mg[lane + 32 * i] = mlo[i];
        mg[512 - lane - 32 * i] = mhi[i];
      }
      if (lane == 0) mg[256] = mlo[8];
      if (lane < 3) mg[513 + lane] = 0.f;   // a group's 4-aligned band may read up to bin 515 (with zero weights)
    }
    __syncthreads();
    // ---- grouped banded filterbank over the round's 8 frames, CTA-wide.  A warp takes groups of 4 mels in a snake
    // order (longest first, then shortest, ...) so that the warps' tap counts even out; its lanes are
    // (mel in group, frame).  A group's bands start on a multiple of 4 bins and are zero-padded to a common
    // multiple-of-4 tap count, so the loop is uniform: per 4 taps one 128-bit magnitude read (8 frames x 16 bytes
    // per quarter warp: conflict-free), one 128-bit broadcast weight read and 4 FMAs.
    {
      const int fr = lane & 7, mi = lane >> 3;
      const float* mgf = reinterpret_cast<const float*>(zb + fr * MEL_ZPAD);
      for (int r = 0; r * MEL_WARPS < ngroups; ++r) {
        const int pos = r * MEL_WARPS + ((r & 1) ? (MEL_WARPS - 1 - w) : w);
        const int g = ngroups - 1 - pos;
        if (g < 0) continue;
        const int4 d = s_desc[4 * g + mi];
        const float4* mp = reinterpret_cast<const float4*>(mgf + d.x);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        if (staged) {
          const float4* wp = reinterpret_cast<const float4*>(fbw_s + d.y);
#pragma unroll 2
          for (int t = 0; t < d.z; ++t) {
            const float4 x4 = mp[t], w4 = wp[t];
            a0 = fmaf(x4.x, w4.x, a0); a1 = fmaf(x4.y, w4.y, a1); a2 = fmaf(x4.z, w4.z, a2); a3 = fmaf(x4.w, w4.w, a3);
          }
        } else {
          const float4* wp = reinterpret_cast<const float4*>(fb_w + d.y);
          for (int t = 0; t < d.z; ++t) {
            const float4 x4 = mp[t], w4 = __ldg(wp + t);
            a0 = fmaf(x4.x, w4.x, a0); a1 = fmaf(x4.y, w4.y, a1); a2 = fmaf(x4.z, w4.z, a2); a3 = fmaf(x4.w, w4.w, a3);
          }
        }
        const float acc = (a0 + a1) + (a2 + a3);
        // MUFU.LG2-based log: absolute error ~1e-7 on values in [-11.6, 10], far inside the 1e-4 mel tolerance
        if (d.w >= 0) otile[d.w * MEL_FPB + rd * MEL_WARPS + fr] = __logf(fmaxf(acc, clamp_min));
      }
    }
    __syncthreads();   // the next round's transforms overwrite the magnitudes
  }
  const int nf = min(MEL_FPB, F - f0);
  float* ob = out + (int64_t)b * out_sb;
  if (out_sf <= out_sm) {   // frame index is the fast output dim
    for (int i = tid; i < n_mels * MEL_FPB; i += NT) {
      const int m = i / MEL_FPB, fl = i - m * MEL_FPB;
      if (fl < nf) ob[(int64_t)m * out_sm + (int64_t)(f0 + fl) * out_sf] = otile[i];
    }
  } else {
    for (int i = tid; i < n_mels * MEL_FPB; i += NT) {
      const int fl = i / n_mels, m = i - fl * n_mels;
      if (fl < nf) ob[(int64_t)m * out_sm + (int64_t)(f0 + fl) * out_sf] = otile[m * MEL_FPB + fl];
    }
  }
}

static std::mutex g_mel_mu;
static bool g_mel_ready[64] = {false};

int mel_spectrogram(const float* wav, int64_t wav_sb, int B, int L, const int32_t* lens, const float* window,
                    const float* fb_w, const int32_t* fb_off, const int32_t* fb_start, int n_mels, float clamp_min,
                    float* out, int64_t out_sb, int64_t out_sm, int64_t out_sf, cudaStream_t st) {
  MTTS_REQUIRE(wav && window && fb_w && fb_off && fb_start && out, "null pointer");
  MTTS_REQUIRE(L > MEL_NFFT / 2, "reflect padding needs L > n_fft/2 (torch.stft center=True)");
  MTTS_REQUIRE(n_mels > 0 && n_mels <= 4 * MEL_MAXG, "n_mels out of range");
  MTTS_REQUIRE(B >= 0 && B <= 65535 * 32, "bad batch");
  MTTS_REQUIRE((((uintptr_t)window) & 15) == 0, "window table must be 16-byte aligned");
  MTTS_REQUIRE((((uintptr_t)fb_w) & 15) == 0, "filterbank blocks must be 16-byte aligned");
  const int vec_ok = ((((uintptr_t)wav) & 15) == 0) && (wav_sb % 4 == 0);
  if (B == 0) return 0;
  const int F = 1 + L / MEL_HOP;
  const size_t smem = sizeof(float) * (MEL_SPAN + MEL_NFFT + 2 * MEL_WARPS * MEL_ZPAD + 128 * MEL_FPB + MEL_FBW + 16 * MEL_MAXG);
  {
    std::lock_guard<std::mutex> lk(g_mel_mu);
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return fail(MTTS_ERR_UNSUPPORTED, "%s: device ordinal %lld out of range", "mel", dev);
    if (!g_mel_ready[dev]) {
      cudaError_t e = cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return fail(MTTS_ERR_CUDA, "%s: cudaFuncSetAttribute failed: %lld", "mel", (long long)e);
      launch_k(mel_init_twiddle_kernel, 4, 256, 0, st);
      MTTS_CHECK_LAUNCH();
      cudaStreamSynchronize(st);   // one-time table init only; never on the steady-state path
      g_mel_ready[dev] = true;
    }
  }
  // grid.y is limited to 65535: fold larger batches over several launches
  for (int b0 = 0; b0 < B; b0 += 65535) {
    const int nb = (B - b0 < 65535) ? (B - b0) : 65535;
    dim3 grid((unsigned)cdiv64(F, MEL_FPB), (unsigned)nb);
    launch_k(mel_kernel, grid, MEL_WARPS * 32, smem, st, wav + (int64_t)b0 * wav_sb, wav_sb, L, lens ? lens + b0 : nullptr, window, fb_w,
                                               fb_off, fb_start, n_mels, clamp_min, out + (int64_t)b0 * out_sb, out_sb, out_sm,
                                               out_sf, vec_ok);
    MTTS_CHECK_LAUNCH();
  }
  return 0;
}

}  // namespace mtts
