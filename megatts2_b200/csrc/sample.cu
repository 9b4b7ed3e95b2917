// Opt-in sampled decode of the PLM loops: temperature, top-k and top-p over one logits row, then a Gumbel-max draw
// whose noise is a pure function of (seed, row key, step, token index) through Philox4x32-10.  The contract is stated
// with mtts_sampling in include/megatts2_b200.h.
#include <float.h>
#include <limits.h>
#include <math.h>

#include "kernels.h"

namespace mtts {

constexpr int SAMPLE_THREADS = 256;
constexpr int SAMPLE_WARPS = SAMPLE_THREADS / 32;
constexpr int SAMPLE_MAX_V = 4096;      // a filtered row is staged as 8-byte keys: at most 32 KB of shared memory
constexpr int MIX_MAX_K = SAMPLE_WARPS; // the mix reduces one source per warp

// Philox4x32-10 (Salmon et al., SC'11, with the Random123 / cuRAND constants)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ uint32_t word_of(const uint4& r, int e) {
  return e == 0 ? r.x : e == 1 ? r.y : e == 2 ? r.z : r.w;
}

// -log(-log u) for u = ((w >> 8) + 0.5) * 2^-24 in (0, 1).  Above 1/2, u has 25 significant bits and is no fp32 number, so
// -log u is taken there as -log1p(-(1 - u)) with 1 - u exact: no u rounds to 1, and the tail keeps its relative precision.
__device__ __forceinline__ float gumbel_of(uint32_t w) {
  const uint32_t m = w >> 8;
  const float e = m < (1u << 23) ? -logf(((float)m + 0.5f) * 0x1p-24f)
                                 : -log1pf(-(((float)(0xFFFFFFu - m) + 0.5f) * 0x1p-24f));
  return -logf(e);
}

// float -> unsigned with the same order, and back (the filtered path sorts 64-bit keys ~order(y) << 32 | index)
__device__ __forceinline__ uint32_t f2ord(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint64_t key) {
  const uint32_t o = ~(uint32_t)(key >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__device__ __forceinline__ void better(float& s, int& i, float os, int oi) {
  if (os > s || (os == s && oi < i)) { s = os; i = oi; }
}

// CTA-wide: the (score, index) maximum with the lowest index on ties and the lowest +inf index -> the row's pick
// (thread 0 only): the +inf index if there is one, else the best index, else 0 (no candidate)
__device__ int block_pick(float s, int i, int inf_i) {
  __shared__ float ws[SAMPLE_WARPS];
  __shared__ int wi[SAMPLE_WARPS], winf[SAMPLE_WARPS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    better(s, i, __shfl_xor_sync(0xffffffffu, s, o), __shfl_xor_sync(0xffffffffu, i, o));
    inf_i = min(inf_i, __shfl_xor_sync(0xffffffffu, inf_i, o));
  }
  if (lane == 0) { ws[w] = s; wi[w] = i; winf[w] = inf_i; }
  __syncthreads();
  if (threadIdx.x != 0) return 0;
  for (int k = 1; k < SAMPLE_WARPS; ++k) {
    better(s, i, ws[k], wi[k]);
    inf_i = min(inf_i, winf[k]);
  }
  return inf_i != INT_MAX ? inf_i : (i != INT_MAX ? i : 0);
}

// CTA-wide inclusive prefix sum; *total is the same value in every thread
__device__ double block_scan(double v, double* total) {
  __shared__ double wsum[SAMPLE_WARPS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  if (lane == 31) wsum[w] = v;
  __syncthreads();
  double off = 0.0, tot = 0.0;
  for (int k = 0; k < SAMPLE_WARPS; ++k) {
    if (k < w) off += wsum[k];
    tot += wsum[k];
  }
  *total = tot;
  return v + off;
}

// One CTA per row.  filter == 0: one Gumbel-max pass over the row.  filter != 0: the row's candidates (y not NaN, not -inf)
// are staged as keys and bitonic-sorted (value descending, index ascending); top-k keeps the first k, top-p the shortest
// prefix of those whose softmax mass reaches p (fp64 sums), and the Gumbel-max runs over the kept prefix.
__global__ void __launch_bounds__(SAMPLE_THREADS)
sample_rows_kernel(const float* __restrict__ x, int64_t ldx, int V, int step, float temperature, int top_k, float top_p,
                   int filter, int n_sort, const uint64_t* __restrict__ seed, const uint64_t* __restrict__ keys,
                   int64_t* out_a, int64_t lda, int64_t* out_b, int64_t ldb, const int32_t* __restrict__ pin,
                   int64_t pin_sb) {
  extern __shared__ uint64_t s_key[];
  __shared__ int s_n, s_cut;
  pdl_entry();
  const int row = blockIdx.x;
  if (pin) {                                               // a pinned row: the whole CTA leaves before any barrier
    const int32_t p = pin[(int64_t)row * pin_sb];
    if (p >= 0 && p < V) {
      if (threadIdx.x == 0) {
        out_a[(int64_t)row * lda] = p;
        if (out_b) out_b[(int64_t)row * ldb] = p;
      }
      return;
    }
  }
  const float* xr = x + (int64_t)row * ldx;
  const uint64_t sd = seed[0], kr = keys[row];
  const uint2 pkey = make_uint2((uint32_t)sd, (uint32_t)(sd >> 32));      // Philox key (seed_lo, seed_hi)
  const uint32_t c2 = (uint32_t)kr, c3 = (uint32_t)(kr >> 32);           // counter (i >> 2, step, key_lo, key_hi)
  float best = -INFINITY;
  int bi = INT_MAX, inf_i = INT_MAX;
  if (!filter) {
    for (int i0 = threadIdx.x * 4; i0 < V; i0 += SAMPLE_THREADS * 4) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)i0 >> 2, (uint32_t)step, c2, c3), pkey);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = i0 + e;
        if (i >= V) break;
        const float y = xr[i] / temperature;
        if (y == INFINITY) inf_i = min(inf_i, i);
        else if (isfinite(y)) better(best, bi, y + gumbel_of(word_of(r, e)), i);
      }
    }
  } else {
    if (threadIdx.x == 0) { s_n = 0; s_cut = INT_MAX; }
    __syncthreads();
    int cnt = 0;
    for (int i = threadIdx.x; i < n_sort; i += SAMPLE_THREADS) {
      uint64_t k = ~0ull;                                  // padding and non-candidates sort last
      if (i < V) {
        float y = xr[i] / temperature;
        if (y == 0.f) y = 0.f;                             // -0 ties with +0 on the index
        if (!isnan(y) && y != -INFINITY) { k = ((uint64_t)~f2ord(y) << 32) | (uint32_t)i; ++cnt; }
      }
      s_key[i] = k;
    }
    if (cnt) atomicAdd(&s_n, cnt);
    for (int k = 2; k <= n_sort; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        __syncthreads();
        for (int i = threadIdx.x; i < n_sort; i += SAMPLE_THREADS) {
          const int p = i ^ j;
          if (p > i) {
            const uint64_t a = s_key[i], b = s_key[p];
            if ((a > b) == ((i & k) == 0)) { s_key[i] = b; s_key[p] = a; }
          }
        }
      }
    }
    __syncthreads();
    const int n = s_n;
    int kept = (top_k > 0 && top_k < n) ? top_k : n;
    const float y0 = n > 0 ? key_value(s_key[0]) : 0.f;
    if (y0 == INFINITY) {
      inf_i = (int)(uint32_t)s_key[0];                     // the lowest +inf index sorts first
    } else if (n > 0) {
      if (top_p < 1.f) {
        // thread t owns sorted positions [t * per, (t + 1) * per): n_sort >= SAMPLE_THREADS, both powers of two
        const int per = n_sort / SAMPLE_THREADS, j0 = threadIdx.x * per, j1 = min(j0 + per, kept);
        double loc = 0.0;
        for (int j = j0; j < j1; ++j) loc += exp((double)key_value(s_key[j]) - (double)y0);
        double total;
        double run = block_scan(loc, &total) - loc;
        const double thr = (double)top_p * total;
        for (int j = j0; j < j1; ++j) {
          run += exp((double)key_value(s_key[j]) - (double)y0);
          if (run >= thr) { atomicMin(&s_cut, j + 1); break; }
        }
        __syncthreads();
        kept = min(kept, s_cut);
      }
      for (int j = threadIdx.x; j < kept; j += SAMPLE_THREADS) {
        const uint64_t key = s_key[j];
        const int i = (int)(uint32_t)key;
        const uint4 r = philox4x32_10(make_uint4((uint32_t)i >> 2, (uint32_t)step, c2, c3), pkey);
        better(best, bi, key_value(key) + gumbel_of(word_of(r, i & 3)), i);
      }
    }
  }
  const int pick = block_pick(best, bi, inf_i);
  if (threadIdx.x == 0) {
    out_a[(int64_t)row * lda] = pick;
    if (out_b) out_b[(int64_t)row * ldb] = pick;
  }
}

// (max, sum of exp(z - max)) of two parts of a row; (-inf, 0) is the empty part
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  if (om == -INFINITY) return;
  if (m == -INFINITY) { m = om; s = os; return; }
  if (om > m) { s = s * expf(m - om) + os; m = om; }
  else s += os * expf(om - m);
}

// One CTA per utterance b: l_i = log sum_k w^_k softmax(z_k)_i over the K rows z_k = x[(k B + b) ldx ..] (the contract is
// stated with mtts_mix_logprob_rows_f32 in include/megatts2_b200.h), with the weight row w + b ldw.  Warp k reduces source k's (max, sum of exps) and its
// lowest +inf index with shuffles; then every thread combines the sources for its tokens as a log-sum-exp in fp32.  The
// rows were just written by the predict layer and are read from L2: each lane issues MIX_CHUNK loads before it uses one,
// so a row costs V / (32 MIX_CHUNK) load latencies instead of V / 32.
constexpr int MIX_CHUNK = 16;
__global__ void __launch_bounds__(SAMPLE_THREADS)
mix_logprob_rows_kernel(const float* __restrict__ x, int64_t ldx, int V, int K, int B, const float* __restrict__ w,
                        int64_t ldw, float* __restrict__ out, int64_t ldo) {
  __shared__ float s_lw[MIX_MAX_K], s_m[MIX_MAX_K];          // log w^_k - log sum_k, max_k
  __shared__ int s_inf[MIX_MAX_K], s_on[MIX_MAX_K];
  pdl_entry();
  const int b = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const float* wr = w + (int64_t)b * ldw;
  float wk[MIX_MAX_K];
#pragma unroll
  for (int k = 0; k < MIX_MAX_K; ++k) wk[k] = k < K ? wr[k] : 0.f;
  float wsum = 0.f;
  int npos = 0, kpos = 0;
#pragma unroll
  for (int k = 0; k < MIX_MAX_K; ++k)
    if (wk[k] > 0.f) { wsum += wk[k]; ++npos; kpos = k; }
  float* orow = out + (int64_t)b * ldo;
  if (npos == 1) {                                           // one weighted source: its raw row, bit for bit
    const float* z = x + ((int64_t)kpos * B + b) * ldx;
#pragma unroll 4
    for (int i = threadIdx.x; i < V; i += SAMPLE_THREADS) orow[i] = z[i];
    return;
  }
  if (wp < K) {
    const float* z = x + ((int64_t)wp * B + b) * ldx;
    float m = -INFINITY, s = 0.f;
    int inf_i = INT_MAX;
    for (int i0 = lane; i0 < V; i0 += 32 * MIX_CHUNK) {
      float v[MIX_CHUNK];
#pragma unroll
      for (int j = 0; j < MIX_CHUNK; ++j) v[j] = i0 + 32 * j < V ? z[i0 + 32 * j] : -INFINITY;
      float cm = -INFINITY, cs = 0.f;
#pragma unroll
      for (int j = 0; j < MIX_CHUNK; ++j) {
        if (v[j] == INFINITY) inf_i = min(inf_i, i0 + 32 * j);
        else if (isfinite(v[j])) cm = fmaxf(cm, v[j]);
      }
      if (cm != -INFINITY) {
#pragma unroll
        for (int j = 0; j < MIX_CHUNK; ++j)
          if (isfinite(v[j])) cs += expf(v[j] - cm);
      }
      lse_merge(m, s, cm, cs);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
      inf_i = min(inf_i, __shfl_xor_sync(0xffffffffu, inf_i, o));
    }
    if (lane == 0) {
      const float v = wr[wp];
      s_inf[wp] = inf_i;
      s_m[wp] = m;
      // NaN weights fail v > 0 and, like a source without a candidate, contribute nothing
      s_on[wp] = v > 0.f && (inf_i != INT_MAX || m != -INFINITY);
      s_lw[wp] = logf(v / wsum) - (inf_i != INT_MAX ? 0.f : logf(s));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < V; i += SAMPLE_THREADS) {
    float v[MIX_MAX_K];
#pragma unroll
    for (int k = 0; k < MIX_MAX_K; ++k) v[k] = k < K ? x[((int64_t)k * B + b) * ldx + i] : 0.f;
    float m = -INFINITY, s = 0.f;
#pragma unroll
    for (int k = 0; k < MIX_MAX_K; ++k) {
      if (k >= K || !s_on[k]) continue;
      float t;
      if (s_inf[k] != INT_MAX) {
        if (i != s_inf[k]) continue;
        t = s_lw[k];
      } else {
        if (!isfinite(v[k])) continue;                       // NaN or -inf: zero mass in its source
        t = (v[k] - s_m[k]) + s_lw[k];
      }
      lse_merge(m, s, t, 1.f);
    }
    orow[i] = m == -INFINITY ? -INFINITY : m + logf(s);
  }
}

__global__ void philox_kernel(const uint32_t* __restrict__ ctr, const uint32_t* __restrict__ key, uint32_t* __restrict__ out,
                              int64_t n) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 r = philox4x32_10(make_uint4(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]),
                                make_uint2(key[2 * i], key[2 * i + 1]));
  out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
}

int sampling_check(const mtts_sampling* s, int V) {
  MTTS_REQUIRE(s, "null sampling parameters");
  MTTS_REQUIRE(isfinite(s->temperature) && s->temperature >= 0.f, "temperature must be finite and >= 0");
  MTTS_REQUIRE(s->top_k >= 0, "top_k must be >= 0");
  MTTS_REQUIRE(s->top_p > 0.f && s->top_p <= 1.f, "top_p must be in (0, 1]");
  MTTS_REQUIRE(s->reserved == 0, "reserved must be 0");
  MTTS_REQUIRE(s->seed && s->keys, "null seed or keys");
  MTTS_REQUIRE(V >= 1, "V must be >= 1");
  if (V > SAMPLE_MAX_V)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: V = %lld is above the sampler's shared-memory bound of %lld tokens", "sample_rows",
                V, SAMPLE_MAX_V);
  return 0;
}

int sample_rows(const float* x, int64_t ldx, int V, int rows, int step, const mtts_sampling& s, int64_t* out_a,
                int64_t lda, int64_t* out_b, int64_t ldb, cudaStream_t st, const int32_t* pin, int64_t pin_sb) {
  MTTS_TRY(sampling_check(&s, V));
  MTTS_REQUIRE(x && out_a, "null pointer");
  MTTS_REQUIRE(step >= 0 && ldx >= 0, "step and ld must be >= 0");
  if (rows <= 0) return 0;
  if (s.temperature == 0.f || s.top_k == 1)
    return argmax_rows(x, ldx, V, rows, out_a, lda, out_b, ldb, st, pin, pin_sb);
  const int filter = (s.top_k > 0 && s.top_k < V) || s.top_p < 1.f;
  int n_sort = SAMPLE_THREADS;
  while (n_sort < V) n_sort <<= 1;
  launch_k(sample_rows_kernel, (unsigned)rows, SAMPLE_THREADS, filter ? (size_t)n_sort * 8 : 0, st, x, ldx, V, step,
           s.temperature, s.top_k, s.top_p, filter, n_sort, s.seed, s.keys, out_a, lda, out_b, ldb, pin, pin_sb);
  MTTS_CHECK_LAUNCH();
  return 0;
}

int mix_logprob_check(int V, int K) {
  MTTS_REQUIRE(K >= 1, "K must be >= 1");
  MTTS_REQUIRE(V >= 1, "V must be >= 1");
  if (K > MIX_MAX_K)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: K = %lld sources is above the bound of %lld", "mix_logprob_rows", K, MIX_MAX_K);
  if (V > SAMPLE_MAX_V)
    return fail(MTTS_ERR_UNSUPPORTED, "%s: V = %lld is above the bound of %lld tokens", "mix_logprob_rows", V, SAMPLE_MAX_V);
  return 0;
}

int mix_logprob_rows(const float* x, int64_t ldx, int V, int K, int B, const float* w, int64_t ldw, float* out,
                     int64_t ldo, cudaStream_t st) {
  MTTS_TRY(mix_logprob_check(V, K));
  MTTS_REQUIRE(ldx >= 0 && ldw >= 0 && ldo >= 0, "ld must be >= 0");
  if (B <= 0) return 0;
  MTTS_REQUIRE(x && w && out, "null pointer");
  launch_k(mix_logprob_rows_kernel, (unsigned)B, SAMPLE_THREADS, 0, st, x, ldx, V, K, B, w, ldw, out, ldo);
  MTTS_CHECK_LAUNCH();
  return 0;
}

int philox4x32_10_words(const uint32_t* ctr, const uint32_t* key, uint32_t* out, int64_t n, cudaStream_t st) {
  MTTS_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return 0;
  MTTS_REQUIRE(ctr && key && out, "null pointer");
  launch_k(philox_kernel, (unsigned)cdiv64(n, 256), 256, 0, st, ctr, key, out, n);
  MTTS_CHECK_LAUNCH();
  return 0;
}

}  // namespace mtts
