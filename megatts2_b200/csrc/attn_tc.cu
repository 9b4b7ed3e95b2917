// Tensor-core attention (wgmma): softmax(Q K^T * scale + mask) V with fp32-grade accuracy from f16x2 split operands
// (kernels.h: x = x1 + x2' * 2^-11, three MMAs per product: x1*y1 | x1*y2' + x2'*y1, the correction accumulator scaled by
// 2^-11 when it is read back).  Replaces F.scaled_dot_product_attention at modules/transformer.py:52-53 for the head dims
// of the autoregressive stacks (PLM: 16 x 64, ADM: 8 x 96).
//
// One CTA = one warpgroup (128 threads) = one (batch item, head, 64-query tile); the accumulators live in registers in the
// wgmma fragment layout (tc_ptx.cuh), so the four lanes of a quad share a query row:
//   stage   Q (64 x dh) once, then per 64-key tile K (64 x dh) and V^T (dh x 64): fp32 global -> f16x2 planes in shared
//           memory, written directly in the K-major 64-byte-swizzle layout (what a TMA load with SWIZZLE_64B would
//           produce: 16-byte chunk c of row r lands at chunk c ^ ((r >> 1) & 3)); fence.proxy.async hands them to the MMA
//   S       3 * dh/16 MMAs (M 64, N 64) into two register accumulators (main | correction)
//   softmax scale, mask, running max / sum of the online softmax per row (quad shuffles), P (unnormalised, f16x2 planes)
//           written to shared memory as the A operand of the second product
//   O       3 * 4 MMAs (M 64, N dh, K 64 keys) accumulated into the output accumulators, which are rescaled by
//           exp(m_old - m_new) first
//   out     (main + correction) / l  ->  fp32 rows and / or operand planes (bf16x3 | f16x2) for the out-projection GEMM
// Shared memory: 64 KB (dh 64) / 88 KB (dh 96) / 112 KB (dh 128).
#include "kernels.h"
#include "tc_ptx.cuh"

namespace mtts {

namespace {

constexpr int ATC_NK = 64;     // keys per tile
constexpr int ATC_NQ = 64;     // queries per CTA

// 8 consecutive fp32 values -> one 16-byte chunk per f16x2 plane
__device__ __forceinline__ void split8_f16x2(const float* v, uint4& p0, uint4& p1, bool& bad) {
  uint32_t a[4], b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint16_t h0[2], h1[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float x = v[2 * i + e];
      const __half x1 = __float2half_rn(x);
      const __half x2 = __float2half_rn((x - __half2float(x1)) * F16X2_SCALE);
      h0[e] = __half_as_ushort(x1);
      h1[e] = __half_as_ushort(x2);
      bad |= !(fabsf(x) <= 65504.0f);
    }
    a[i] = (uint32_t)h0[0] | ((uint32_t)h0[1] << 16);
    b[i] = (uint32_t)h1[0] | ((uint32_t)h1[1] << 16);
  }
  p0 = make_uint4(a[0], a[1], a[2], a[3]);
  p1 = make_uint4(b[0], b[1], b[2], b[3]);
}

// byte offset of 16-byte chunk `c` (0..3) of row `r` inside a K-major slab of 64-byte rows with the 64-byte swizzle
__device__ __forceinline__ uint32_t sw64_off(int r, int c) { return (uint32_t)r * 64u + (uint32_t)((c ^ ((r >> 1) & 3)) << 4); }

template <int DH>
struct AtcCfg {
  static constexpr int NS = DH / 32;                      // 32-element (64-byte) K-slabs along dh
  static constexpr int Q_SLAB = ATC_NQ * 64;              // bytes: 64 rows x 64 B
  static constexpr int K_SLAB = ATC_NK * 64;
  static constexpr int V_SLAB = DH * 64;                  // V^T: dh rows, one slab per 32 keys
  static constexpr int P_SLAB = ATC_NQ * 64;
  static constexpr int Q_PLANE = NS * Q_SLAB, K_PLANE = NS * K_SLAB, V_PLANE = 2 * V_SLAB, P_PLANE = 2 * P_SLAB;
  static constexpr int OFF_Q = 0, OFF_K = OFF_Q + 2 * Q_PLANE, OFF_V = OFF_K + 2 * K_PLANE, OFF_P = OFF_V + 2 * V_PLANE;
  static constexpr int SMEM = OFF_P + 2 * P_PLANE + 1024;      // + alignment slack
};

template <int DH>
__global__ void __launch_bounds__(128)
attn_tc_kernel(const mtts_attn_params p, int32_t* ovf) {
  using Cfg = AtcCfg<DH>;
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - smem_u32(smem_raw));

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * ATC_NQ, h = blockIdx.y, b = blockIdx.z;
  // fragment rows of this thread: r0 = 16 warp + lane / 4 and r0 + 8; fragment columns 8 j + 2 (lane % 4) + {0, 1}
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
  int qrow[2];
  bool qvalid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    qrow[i] = q0 + r0 + 8 * i;
    qvalid[i] = qrow[i] < p.Tq;
  }

  pdl_wait();
  bool bad = false;
  // ---- stage Q (two threads per query row; rows past Tq are zero)
  {
    const int row = tid >> 1, half = tid & 1;
    const bool valid = q0 + row < p.Tq;
    const float* src = p.q + (int64_t)b * p.q_sb + (int64_t)(valid ? q0 + row : 0) * p.q_st + (int64_t)h * DH + half * (DH / 2);
#pragma unroll
    for (int i = 0; i < DH / 16; ++i) {
      float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (valid) {
        const float4 a = *reinterpret_cast<const float4*>(src + i * 8);
        const float4 c = *reinterpret_cast<const float4*>(src + i * 8 + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
      }
      uint4 p0, p1;
      split8_f16x2(v, p0, p1, bad);
      const int c8 = half * (DH / 16) + i;
      const uint32_t off = (uint32_t)(c8 >> 2) * Cfg::Q_SLAB + sw64_off(row, c8 & 3);
      *reinterpret_cast<uint4*>(sm + Cfg::OFF_Q + off) = p0;
      *reinterpret_cast<uint4*>(sm + Cfg::OFF_Q + Cfg::Q_PLANE + off) = p1;
    }
  }

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};    // l_run: this thread's share of the row sum
  float om[DH / 2], oc[DH / 2];                                       // O accumulators: main | correction
#pragma unroll
  for (int d = 0; d < DH / 2; ++d) { om[d] = 0.f; oc[d] = 0.f; }
  const float* mrow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
    mrow[i] = p.mask ? p.mask + (int64_t)b * p.mask_sb + (int64_t)h * p.mask_sh + (int64_t)(qvalid[i] ? qrow[i] : 0) * p.mask_sq
                     : nullptr;
  const float* kb = p.k + (int64_t)b * p.k_sb + (int64_t)h * DH;
  const float* vb = p.v + (int64_t)b * p.v_sb + (int64_t)h * DH;
  const uint64_t desc_hi = wgmma_desc<64>(0u);

  for (int k0 = 0; k0 < p.Tk; k0 += ATC_NK) {
    __syncthreads();         // the previous tile's MMAs (which read K, V and P) have retired in every warp
    // ---- stage the K tile (two threads per key row) and the V^T tile (lanes = consecutive keys, so that a warp fills
    //      one 64-byte row of V^T with 2-byte stores); keys past Tk are zero
    {
      const int key = tid >> 1, half = tid & 1;
      const bool kvalid = k0 + key < p.Tk;
      const float* src = kb + (int64_t)(kvalid ? k0 + key : 0) * p.k_st + half * (DH / 2);
#pragma unroll
      for (int i = 0; i < DH / 16; ++i) {
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (kvalid) {
          const float4 a = *reinterpret_cast<const float4*>(src + i * 8);
          const float4 c = *reinterpret_cast<const float4*>(src + i * 8 + 4);
          v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
        }
        uint4 p0, p1;
        split8_f16x2(v, p0, p1, bad);
        const int c8 = half * (DH / 16) + i;              // 16-byte chunk index along dh
        const uint32_t off = (uint32_t)(c8 >> 2) * Cfg::K_SLAB + sw64_off(key, c8 & 3);
        *reinterpret_cast<uint4*>(sm + Cfg::OFF_K + off) = p0;
        *reinterpret_cast<uint4*>(sm + Cfg::OFF_K + Cfg::K_PLANE + off) = p1;
      }
    }
    {
      const int key = tid & 63, dg = tid >> 6;            // dg: which half of dh this thread transposes
      const bool kvalid = k0 + key < p.Tk;
      const float* src = vb + (int64_t)(kvalid ? k0 + key : 0) * p.v_st + dg * (DH / 2);
      uint8_t* vt0 = sm + Cfg::OFF_V + (key >> 5) * Cfg::V_SLAB;
      const int kk = key & 31;
#pragma unroll
      for (int i = 0; i < DH / 8; ++i) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kvalid) a = *reinterpret_cast<const float4*>(src + i * 4);
        const float vv[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int d = dg * (DH / 2) + i * 4 + e;
          const __half x1 = __float2half_rn(vv[e]);
          const __half x2 = __float2half_rn((vv[e] - __half2float(x1)) * F16X2_SCALE);
          bad |= !(fabsf(vv[e]) <= 65504.0f);
          const uint32_t off = sw64_off(d, kk >> 3) + (uint32_t)(kk & 7) * 2u;
          *reinterpret_cast<uint16_t*>(vt0 + off) = __half_as_ushort(x1);
          *reinterpret_cast<uint16_t*>(vt0 + Cfg::V_PLANE + off) = __half_as_ushort(x2);
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- S = Q K^T
    float sm_[ATC_NK / 2], sc_[ATC_NK / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < DH / 16; ++ks) {
      const uint32_t qa = base + Cfg::OFF_Q + (ks >> 1) * Cfg::Q_SLAB + (ks & 1) * 32;
      const uint32_t ka = base + Cfg::OFF_K + (ks >> 1) * Cfg::K_SLAB + (ks & 1) * 32;
      const uint64_t a1 = desc_hi | (uint64_t)((qa >> 4) & 0x3FFF), a2 = desc_hi | (uint64_t)(((qa + Cfg::Q_PLANE) >> 4) & 0x3FFF);
      const uint64_t b1 = desc_hi | (uint64_t)((ka >> 4) & 0x3FFF), b2 = desc_hi | (uint64_t)(((ka + Cfg::K_PLANE) >> 4) & 0x3FFF);
      Wgmma<ATC_NK>::template mma<false>(sc_, a1, b2, ks ? 1u : 0u);      // correction: q1 k2' + q2' k1
      Wgmma<ATC_NK>::template mma<false>(sc_, a2, b1, 1u);
      Wgmma<ATC_NK>::template mma<false>(sm_, a1, b1, ks ? 1u : 0u);      // main: q1 k1
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sm_);
    wgmma_fence_regs(sc_);
    // ---- online softmax on this thread's two rows (a row is spread over the four lanes of a quad)
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float tmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < ATC_NK / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = 4 * j + 2 * i + e, key = k0 + 8 * j + cq + e;
          float x = fmaf(sc_[r], F16X2_INV_SCALE, sm_[r]) * p.scale;
          if (mrow[i] && key < p.Tk) x += mrow[i][key];
          x = key < p.Tk ? x : -INFINITY;
          sm_[r] = x;
          tmax = fmaxf(tmax, x);
        }
      }
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
      const float m_new = fmaxf(m_run[i], tmax);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[i] = expf(m_run[i] - m_use);
      float psum = 0.f;
#pragma unroll
      for (int j = 0; j < ATC_NK / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = 4 * j + 2 * i + e;
          sm_[r] = expf(sm_[r] - m_use);
          psum += sm_[r];
        }
      }
      l_run[i] = l_run[i] * alpha[i] + psum;
      m_run[i] = m_new;
    }
    // P (f16x2 planes, p in [0, 1]: never out of range): row r0 + 8 i, keys 8 j + cq + {0, 1} -> one 4-byte store per plane
#pragma unroll
    for (int j = 0; j < ATC_NK / 8; ++j) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float x0 = sm_[4 * j + 2 * i], x1 = sm_[4 * j + 2 * i + 1];
        const __half2 hi = __floats2half2_rn(x0, x1);
        const float2 hf = __half22float2(hi);
        const __half2 lo = __floats2half2_rn((x0 - hf.x) * F16X2_SCALE, (x1 - hf.y) * F16X2_SCALE);
        const int key = 8 * j + cq;
        const uint32_t off = (uint32_t)(key >> 5) * Cfg::P_SLAB + sw64_off(r0 + 8 * i, (key >> 3) & 3) + (uint32_t)(key & 7) * 2u;
        *reinterpret_cast<__half2*>(sm + Cfg::OFF_P + off) = hi;
        *reinterpret_cast<__half2*>(sm + Cfg::OFF_P + Cfg::P_PLANE + off) = lo;
      }
    }
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        om[4 * j + e] *= alpha[e >> 1];
        oc[4 * j + e] *= alpha[e >> 1];
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- O += P V   (K = the tile's 64 keys: 4 k-steps)
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < ATC_NK / 16; ++ks) {
      const uint32_t pa = base + Cfg::OFF_P + (ks >> 1) * Cfg::P_SLAB + (ks & 1) * 32;
      const uint32_t va = base + Cfg::OFF_V + (ks >> 1) * Cfg::V_SLAB + (ks & 1) * 32;
      const uint64_t a1 = desc_hi | (uint64_t)((pa >> 4) & 0x3FFF), a2 = desc_hi | (uint64_t)(((pa + Cfg::P_PLANE) >> 4) & 0x3FFF);
      const uint64_t b1 = desc_hi | (uint64_t)((va >> 4) & 0x3FFF), b2 = desc_hi | (uint64_t)(((va + Cfg::V_PLANE) >> 4) & 0x3FFF);
      Wgmma<DH>::template mma<false>(oc, a1, b2, 1u);
      Wgmma<DH>::template mma<false>(oc, a2, b1, 1u);
      Wgmma<DH>::template mma<false>(om, a1, b1, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(om);
    wgmma_fence_regs(oc);
  }
  if (bad && ovf) *ovf = 1;

  // ---- output.  Lane pairs (l, l ^ 1) swap halves so that each lane holds 4 consecutive columns of ONE row: the even
  // lane columns 8 j + cq .. + 3 of row r0, the odd lane columns 8 j + cq - 2 .. + 1 of row r0 + 8.
  float inv[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[i] = 1.0f / l;
  }
  const bool odd = lane & 1;
  const int orow = odd ? qrow[1] : qrow[0];
  const bool ovalid = odd ? qvalid[1] : qvalid[0];
  float* o = p.o ? p.o + (int64_t)b * p.o_sb + (int64_t)(ovalid ? orow : 0) * p.o_st + (int64_t)h * DH : nullptr;
  __nv_bfloat16* pl = reinterpret_cast<__nv_bfloat16*>(p.o_planes);
  const int64_t poff = ((int64_t)b * p.Tq + (ovalid ? orow : 0)) * p.o_planes_ld + (int64_t)h * DH;
#pragma unroll
  for (int j = 0; j < DH / 8; ++j) {
    float f[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) f[e] = fmaf(oc[4 * j + e], F16X2_INV_SCALE, om[4 * j + e]) * inv[e >> 1];
    const float s0 = __shfl_xor_sync(0xffffffffu, odd ? f[0] : f[2], 1);
    const float s1 = __shfl_xor_sync(0xffffffffu, odd ? f[1] : f[3], 1);
    const float v[4] = {odd ? s0 : f[0], odd ? s1 : f[1], odd ? f[2] : s0, odd ? f[3] : s1};
    const int col = 8 * j + cq - (odd ? 2 : 0);
    if (ovalid) {
      if (o) *reinterpret_cast<float4*>(o + col) = make_float4(v[0], v[1], v[2], v[3]);
      if (pl) store_planes4(pl, p.o_plane_stride, poff + col, v, p.o_planes_fmt, ovf);
    }
  }
}

template <int DH>
int attn_tc_launch(const mtts_attn_params& p, cudaStream_t st) {
  using Cfg = AtcCfg<DH>;
  static std::atomic<uint64_t> configured{0};
  const int dev = cur_device();
  if (!(configured.load(std::memory_order_relaxed) & (1ull << dev))) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return fail(MTTS_ERR_CUDA, "%s: cudaFuncSetAttribute failed: %lld", "attention_tc", (long long)e);
    configured.fetch_or(1ull << dev, std::memory_order_relaxed);
  }
  dim3 grid((unsigned)cdiv64(p.Tq, ATC_NQ), (unsigned)p.H, (unsigned)p.B);
  launch_k(attn_tc_kernel<DH>, grid, 128, Cfg::SMEM, st, p, tc_ovf_ptr());
  MTTS_CHECK_LAUNCH();
  return 0;
}

}  // namespace

// eligible: head dims of the AR stacks, 16-byte aligned fp32 views, output rows aligned for float4 / plane stores
bool attention_tc_eligible(const mtts_attn_params& p) {
  if (!(p.dh == 64 || p.dh == 96 || p.dh == 128)) return false;
  auto al = [](const void* q) { return (((uintptr_t)q) & 15) == 0; };
  if (!(al(p.q) && al(p.k) && al(p.v) && p.q_st % 4 == 0 && p.k_st % 4 == 0 && p.v_st % 4 == 0 && p.q_sb % 4 == 0 &&
        p.k_sb % 4 == 0 && p.v_sb % 4 == 0))
    return false;
  if (p.o && !(al(p.o) && p.o_st % 4 == 0 && p.o_sb % 4 == 0)) return false;
  if (p.o_planes && (p.o_planes_ld % 4 != 0 || p.o_plane_stride % 4 != 0)) return false;
  return p.B > 0 && p.H > 0 && p.Tq > 0 && p.Tk > 0 && p.H <= 65535 && p.B <= 65535;
}

// an AR step (every query sees every key of an equally long sequence of at most 64 rows): one 64-row tile per head, the
// whole sequence in one key tile.  The same kernel as attention_tc; the entry point is kept for the opt-in routing of the
// AR steps (mtts_set_attention_pair_min).
bool attention_tc_pair_eligible(const mtts_attn_params& p) {
  return (p.dh == 64 || p.dh == 96) && p.Tq == p.Tk && p.Tk <= 64 && (p.H % 2) == 0 && attention_tc_eligible(p);
}

int attention_tc_pair(const mtts_attn_params& p, cudaStream_t st) {
  MTTS_REQUIRE(attention_tc_pair_eligible(p), "shape / alignment not eligible for the AR-step tensor-core attention");
  return p.dh == 64 ? attn_tc_launch<64>(p, st) : attn_tc_launch<96>(p, st);
}

int attention_tc(const mtts_attn_params& p, cudaStream_t st) {
  MTTS_REQUIRE(attention_tc_eligible(p), "shape / alignment not eligible for the tensor-core attention");
  if (p.dh == 64) return attn_tc_launch<64>(p, st);
  if (p.dh == 96) return attn_tc_launch<96>(p, st);
  return attn_tc_launch<128>(p, st);
}

}  // namespace mtts
