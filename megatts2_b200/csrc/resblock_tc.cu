// One HiFi-GAN ResBlock1 dilation step in ONE wgmma launch, for the C = 32 / 64 stages of the vocoder:
//   y = (x + conv2(leaky(conv1_d(leaky(x))))) * out_scale (+ y)
// Both convolutions are "same" convolutions with reflect padding; conv1 has k taps at dilation d, conv2 k taps at
// dilation 1.  The unfused flow (drivers.cu) runs them as two tap-GEMM launches with the intermediate activation going
// through HBM as operand planes (plus a halo_fill launch for its reflect rows); here the intermediate of a tile never
// leaves shared memory, and the fp32 input is split into operand planes by the kernel itself.
//
// Work item = R = 128 - 2 h2 output rows of one batch item (h1 = d (k - 1) / 2, h2 = (k - 1) / 2):
//   1. the loader warps copy fp32 x rows [r0 - h1 - h2, r0 + 128 + h1 - h2) (reflected about the sequence ends exactly
//      like split_pad_kernel) into a staging buffer with cp.async, apply leaky 0.1 and write the operand planes into an
//      x buffer in the K-major swizzled layout a TMA load would produce;
//   2. conv1 over 128 rows (positions [r0 - h2, r0 - h2 + 128)): tap j reads the planes through a descriptor shifted by
//      j d rows, as the halo form of conv_tc_kernel does;
//   3. epilogue 1 writes leaky(conv1 + bias) as operand planes over the x planes (the same buffer), then the rows at
//      positions outside [0, T) are replaced by their reflections - what halo_fill does to the unfused flow's planes;
//   4. conv2 over 128 rows of the intermediate (its last 2 h2 rows are discarded);
//   5. epilogue 2: bias, the fp32 residual (x, re-read from global / L2), out_scale and the accumulate form.
// Every output element sees the same MMAs on the same operands in the same order, and the same epilogue arithmetic, as
// under the two conv_tc_kernel halo-form launches it replaces, so the result is bit-identical to them.
//
// One CTA = 2 consumer warpgroups (each owns its items' conv1, epilogue 1, conv2 and epilogue 2) + the producer
// warpgroup: warp 8 streams the per-tap weight tiles with TMA into one ring PER WARPGROUP, warps 9-11 (the loader) do
// step 1 for every item of the CTA, in the order the warpgroups take them, into a ring of XBUFS x buffers (item li of
// the CTA in buffer li % XBUFS), so the x traffic of the next items runs under the MMAs and epilogues of the current
// ones.  A buffer is handed over through two mbarriers: xfull (the loader's planes are in place) and xempty (conv2's
// MMAs of the buffer's item have retired; epilogue 2 reads the residual from global memory, not from the buffer).
// Each warpgroup consumes only its own weight ring, strictly in order, so when it waits for a slab every earlier slab of
// that slot has landed and been consumed: the parity of the full barrier is never ambiguous, whatever the ring depth and
// however far the warpgroups drift apart.  The x ring is filled and drained in item order, and the fill of item li waits
// only for item li - XBUFS (<= li - 2, the same warpgroup's previous item or an earlier one), so its parities are
// unambiguous too.  The producer fills the weight rings in the order conv1 of the first item of a pair, conv1 of the
// second, conv2 of the first, conv2 of the second, so the two warpgroups take turns on the tensor pipe: one runs its MMAs
// while the other runs an epilogue.  Formats: f16x2 (NP = 2) and f16 (NP = 1); bf16x3 keeps the unfused flow.
#include "kernels.h"
#include "tc_ptx.cuh"

namespace mtts {

struct RbTcMaps {
  CUtensorMap w1[2], w2[2];   // 2-D (C, k * C) weight planes of conv1 / conv2
};

struct RbTcArgs {
  int32_t B, T, k, dil;         // batch items, rows per item, taps, dilation of conv1
  const float* x;               // (B, T, C) fp32: conv1's input and the residual
  const float* b1; const float* b2;
  float* y;                     // (B, T, C) fp32 output, must not alias x
  float out_scale; int32_t accumulate;
  int32_t* ovf;                 // f16 range flag (may be null)
};

constexpr int RB_XROWS = 192;           // rows of an x buffer: 128 + 2 h1 <= 192
constexpr int RB_LOADER_THREADS = 96;   // warps 9-11
// barrier area: the weight rings' full / empty barriers (2 rings x 2 x 8 bytes x STAGES <= 256 bytes), then the x ring's
// xfull / xempty barriers (2 x 8 bytes x XBUFS <= 64 bytes)
constexpr int RB_BAR_BYTES = 256 + 64;

template <int C, int NP>
struct RbTcCfg {
  static constexpr int SWB = 2 * C;                      // one 16-bit activation row = one swizzled row (64 or 128 bytes)
  static constexpr int XPLANE = RB_XROWS * SWB;
  static constexpr int XBUF = NP * XPLANE;               // one x buffer (24 KB, or 48 KB at C = 64, f16x2)
  // two buffers per warpgroup where they are 24 KB, so the loader can run a whole item ahead of each warpgroup
  static constexpr int XBUFS = XBUF <= 24 * 1024 ? 4 : 2;
  // fp32 staging of one item's x rows, which cp.async fills.  Two at C = 32, where an item's MMAs take less time than
  // one round trip to memory, so the copies of the next item are in flight while the loader converts the current one
  static constexpr int XSTAGE = RB_XROWS * C * 4;
  static constexpr int SBUFS = C == 32 ? 2 : 1;
  static constexpr int W_PLANE = C * SWB;                // one tap's weight tile (C x C), one plane
  static constexpr int STAGE = NP * W_PLANE;
  static constexpr int EPI_STAGE = 8 * 16 * 20 * 4;
  static constexpr int STAGES_RAW =
      (227 * 1024 - 1024 - RB_BAR_BYTES - EPI_STAGE - XBUFS * XBUF - SBUFS * XSTAGE) / (2 * STAGE);
  // stages of EACH warpgroup's ring.  A warpgroup holds at most two slabs unreleased (the one whose MMAs run and the one
  // it waits for), so 2 stages cannot deadlock; 3 keep the next tap's weights in flight during the current tap's MMAs
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM = XBUFS * XBUF + SBUFS * XSTAGE + 2 * STAGES * STAGE + 1024 + RB_BAR_BYTES + EPI_STAGE;
  static_assert(STAGES >= 2 && SMEM <= 227 * 1024, "shared-memory budget");
  static_assert(XBUFS >= 2 && 2 * 8 * XBUFS <= 64, "x ring");
  static_assert(XPLANE % 1024 == 0 && XSTAGE % 1024 == 0 && STAGE % 1024 == 0, "swizzle-atom alignment");
};

// element offset of column c (a multiple of 4) of row r in a K-major plane of SWB-byte rows with the SWB-byte swizzle
// (16-byte chunk q of row r sits at chunk q ^ (r & 7) for 128-byte rows, q ^ ((r >> 1) & 3) for 64-byte rows)
template <int SWB>
__device__ __forceinline__ int sw_elem(int r, int c) {
  const int q = c >> 3, sw = SWB == 128 ? (r & 7) : ((r >> 1) & 3);
  return r * (SWB / 2) + ((q ^ sw) << 3) + (c & 7);
}

// one tap of a 128-row tap-GEMM: A = planes at a_addr (128 rows), B = the weight tile at b_addr; the product order of
// conv_tc_kernel (f16x2: x1 w2', x2' w1 into the correction accumulator, x1 w1 into the main one)
template <int C, int NP>
__device__ __forceinline__ void rb_tap(float (&acc)[2][C / 2], float (&cor)[2][NP == 1 ? 1 : C / 2], uint32_t a_addr,
                                       uint32_t b_addr, uint32_t first) {
  using Cfg = RbTcCfg<C, NP>;
  const uint64_t desc_base = wgmma_desc<Cfg::SWB>(0u);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < C / 16; ++ks) {
    const uint32_t bb = b_addr + ks * 32;
    const uint64_t b1 = desc_base | (uint64_t)((bb >> 4) & 0x3FFF), b2 = desc_base | (uint64_t)(((bb + Cfg::W_PLANE) >> 4) & 0x3FFF);
    const uint32_t f = ks == 0 ? first : 1u;
#pragma unroll
    for (int hv = 0; hv < 2; ++hv) {
      const uint32_t aa = a_addr + hv * 64 * Cfg::SWB + ks * 32;
      const uint64_t a1 = wgmma_desc_shifted(desc_base, aa);
      if constexpr (NP == 1) {
        Wgmma<C>::template mma<false>(acc[hv], a1, b1, f);
      } else {
        const uint64_t a2 = wgmma_desc_shifted(desc_base, aa + Cfg::XPLANE);
        Wgmma<C>::template mma<false>(cor[hv], a1, b2, f);
        Wgmma<C>::template mma<false>(cor[hv], a2, b1, 1u);
        Wgmma<C>::template mma<false>(acc[hv], a1, b1, f);
      }
    }
  }
  wgmma_commit();
}

template <int C, int NP>
__global__ void __launch_bounds__(CTC_THREADS, 1)
resblock_pair_tc_kernel(const __grid_constant__ RbTcMaps maps, const RbTcArgs g) {
  using Cfg = RbTcCfg<C, NP>;
  pdl_trigger();
  constexpr int STAGES = Cfg::STAGES, SWB = Cfg::SWB, XBUFS = Cfg::XBUFS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t smem_x = (raw + 1023u) & ~1023u;                  // the x ring: buffer s at smem_x + s * XBUF
  const uint32_t smem_s = smem_x + XBUFS * Cfg::XBUF;              // fp32 staging: buffer u at smem_s + u * XSTAGE
  const uint32_t smem_w = smem_s + Cfg::SBUFS * Cfg::XSTAGE;       // the two weight rings (warpgroup 0, warpgroup 1)
  const uint32_t bars = smem_w + 2 * STAGES * Cfg::STAGE;
  // ring w: slot s at ring(w) + s * STAGE, its barriers at full_bar(w) + 8 s / empty_bar(w) + 8 s
  auto ring = [&](int w) { return smem_w + (uint32_t)(w * STAGES * Cfg::STAGE); };
  auto full_bar = [&](int w) { return bars + (uint32_t)(w * 16 * STAGES); };
  auto empty_bar = [&](int w) { return bars + (uint32_t)(w * 16 * STAGES + 8 * STAGES); };
  auto xfull_bar = [&](int s) { return bars + 256u + (uint32_t)(8 * s); };
  auto xempty_bar = [&](int s) { return bars + 256u + (uint32_t)(8 * (XBUFS + s)); };
  float* epi_stage = reinterpret_cast<float*>(smem_raw + (bars + RB_BAR_BYTES - raw));

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int k = g.k, T = g.T;
  const int h1 = g.dil * (k - 1) / 2, h2 = (k - 1) / 2;
  const int R = 128 - 2 * h2;                                       // output rows of a work item
  const int num_t = (T + R - 1) / R;
  const int num_items = g.B * num_t;
  const int n_items = num_items > (int)blockIdx.x ? (num_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  if (warp == 8 && lane == 0) {
#pragma unroll
    for (int q = 0; q < NP; ++q) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w1[q]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w2[q]) : "memory");
    }
    for (int w = 0; w < 2; ++w)
      for (int s = 0; s < STAGES; ++s) {
        mbar_init(full_bar(w) + 8 * s, 1);
        mbar_init(empty_bar(w) + 8 * s, 4);     // one arrive per warp of the ring's warpgroup
      }
    for (int s = 0; s < XBUFS; ++s) {
      mbar_init(xfull_bar(s), RB_LOADER_THREADS);
      mbar_init(xempty_bar(s), 4);              // one arrive per warp of the item's warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  constexpr int PL = Cfg::XPLANE / 2;                  // plane stride (elements)
  constexpr int fmt = 3 - NP;

  if (warp >= 8) {
    setmaxnreg_dec<CTC_PRODUCER_REGS>();
    if (warp > 8) {
      // ================= x loader: the fp32 rows of item li of the CTA -> cp.async -> staging buffer li % SBUFS; then
      // leaky -> operand planes of x buffer li % XBUFS.  Each thread converts exactly the float4s it copied, so its own
      // cp.async.wait_group is all the ordering the staging buffer needs
      constexpr int CQ = C / 4, SB = Cfg::SBUFS;
      const int lt = threadIdx.x - 9 * 32;
      const int total = (128 + 2 * h1) * CQ;
      for (int li = 0; li < n_items + SB - 1; ++li) {
        if (li < n_items) {
          const int item = blockIdx.x + li * gridDim.x;
          const int tb = item % num_t, b = item / num_t;
          const float* xb = g.x + (int64_t)b * T * C;
          const int t0 = tb * R - h1 - h2;
          const uint32_t st = smem_s + (li % SB) * Cfg::XSTAGE;
          for (int i = lt; i < total; i += RB_LOADER_THREADS) {
            int t = t0 + i / CQ;
            if (t < 0) t = -t;
            if (t >= T) t = 2 * (T - 1) - t;
            const bool in = t >= 0 && t < T;           // a row outside the sequence after the reflection: zeros
            cp_async16(st + 16 * i, in ? xb + (int64_t)t * C + (i % CQ) * 4 : xb, in ? 16u : 0u);
          }
        }
        cp_async_commit();                             // (an empty group past the last item)
        const int lc = li - (SB - 1);                  // the item converted now: its copies were committed SB - 1 groups ago
        if (lc < 0) continue;
        cp_async_wait<SB - 1>();
        const int s = lc % XBUFS;
        mbar_wait(xempty_bar(s), ((lc / XBUFS) & 1) ^ 1);
        const float4* sv = reinterpret_cast<const float4*>(smem_raw + (smem_s + (lc % SB) * Cfg::XSTAGE - raw));
        __nv_bfloat16* xg = reinterpret_cast<__nv_bfloat16*>(smem_raw + (smem_x + s * Cfg::XBUF - raw));
        for (int i = lt; i < total; i += RB_LOADER_THREADS) {
          const float4 v = sv[i];
          float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) f[e] = act_apply(f[e], MTTS_ACT_LEAKY, 0.1f);
          store_planes4(xg, PL, sw_elem<SWB>(i / CQ, (i % CQ) * 4), f, fmt, g.ovf);
        }
        fence_proxy_async_smem();
        mbar_arrive(xfull_bar(s));
      }
      return;
    }
    // ================= weight producer: per pair of items conv1 | conv1 | conv2 | conv2, k tap tiles each, item 2p + e
    // (owned by warpgroup e) into ring e.  Waiting on ring e's empty slot cannot deadlock: before warpgroup e waits for
    // its slab n it has released every slab up to n - 2, and the producer needs slab n - STAGES (STAGES >= 2) released
    const bool leader = elect_one();
    int stage[2] = {0, 0}, phase[2] = {0, 0};
    for (int p = 0; 2 * p < n_items; ++p) {
      const int ne = 2 * p + 1 < n_items ? 2 : 1;
      for (int cv = 0; cv < 2; ++cv)
#pragma unroll
        for (int e = 0; e < 2; ++e)            // unrolled: stage[] / phase[] stay in registers
          for (int j = 0; j < k && e < ne; ++j) {
            mbar_wait(empty_bar(e) + 8 * stage[e], phase[e] ^ 1);
            if (leader) {
              const uint32_t sb = ring(e) + stage[e] * Cfg::STAGE, fb = full_bar(e) + 8 * stage[e];
              mbar_expect_tx(fb, Cfg::STAGE);
#pragma unroll
              for (int q = 0; q < NP; ++q) tma_load_2d(sb + q * Cfg::W_PLANE, cv ? &maps.w2[q] : &maps.w1[q], fb, 0, j * C);
            }
            if (++stage[e] == STAGES) { stage[e] = 0; phase[e] ^= 1; }
          }
    }
    return;
  }

  // ================= consumers: warpgroup wg owns the CTA's items wg, wg + 2, ... =================
  setmaxnreg_inc<CTC_CONSUMER_REGS>();
  constexpr float CS = NP == 2 ? F16X2_INV_SCALE : 1.0f;
  constexpr int NCOR = NP == 1 ? 1 : C / 2;
  const int wg = warp >> 2, w4 = warp & 3, tid = threadIdx.x & 127;
  const int chunk = lane & 3, rsub = lane >> 2;
  float* stg = epi_stage + warp * (16 * 20);
  float acc[2][C / 2], cor[2][NCOR];

  const uint32_t my_ring = ring(wg), my_full = full_bar(wg), my_empty = empty_bar(wg);
  // k taps of one conv from this warpgroup's ring, whose n-th slab (n = (2 m + cv) k + j for conv cv of the warpgroup's
  // m-th item) sits in slot n % STAGES; the MMAs of the previous tap retire before its slab is released
  auto run_conv = [&](int s0, uint32_t a_base, int dil) {
    for (int j = 0; j < k; ++j) {
      const int s = s0 + j;
      mbar_wait(my_full + 8 * (s % STAGES), (s / STAGES) & 1);
      rb_tap<C, NP>(acc, cor, a_base + (uint32_t)(j * dil) * SWB, my_ring + (s % STAGES) * Cfg::STAGE, j == 0 ? 0u : 1u);
      wgmma_wait<1>();
      if (j > 0 && lane == 0) mbar_arrive(my_empty + 8 * ((s - 1) % STAGES));
    }
    wgmma_wait<0>();
#pragma unroll
    for (int hv = 0; hv < 2; ++hv) {
      wgmma_fence_regs(acc[hv]);
      if constexpr (NP > 1) wgmma_fence_regs(cor[hv]);
    }
    if (lane == 0) mbar_arrive(my_empty + 8 * ((s0 + k - 1) % STAGES));
  };
  // main + 2^-11 correction of 16 x 16 unit u of half hv, transposed through this warp's staging buffer
  auto stage_unit = [&](int hv, int u) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = 2 * u + h, c = 8 * h + 2 * chunk;
      if constexpr (NP == 1) {
        *reinterpret_cast<float2*>(stg + rsub * 20 + c) = make_float2(acc[hv][4 * j + 0], acc[hv][4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (rsub + 8) * 20 + c) = make_float2(acc[hv][4 * j + 2], acc[hv][4 * j + 3]);
      } else {
        *reinterpret_cast<float2*>(stg + rsub * 20 + c) =
            make_float2(fmaf(cor[hv][4 * j + 0], CS, acc[hv][4 * j + 0]), fmaf(cor[hv][4 * j + 1], CS, acc[hv][4 * j + 1]));
        *reinterpret_cast<float2*>(stg + (rsub + 8) * 20 + c) =
            make_float2(fmaf(cor[hv][4 * j + 2], CS, acc[hv][4 * j + 2]), fmaf(cor[hv][4 * j + 3], CS, acc[hv][4 * j + 3]));
      }
    }
    __syncwarp();
  };

  for (int li = wg; li < n_items; li += 2) {
    const int item = blockIdx.x + li * gridDim.x;
    const int tb = item % num_t, b = item / num_t;
    const int r0 = tb * R;
    const float* xb = g.x + (int64_t)b * T * C;
    const int s = li % XBUFS;
    const uint32_t xs = smem_x + s * Cfg::XBUF;
    __nv_bfloat16* xg = reinterpret_cast<__nv_bfloat16*>(smem_raw + (xs - raw));

    // ---- 1. the loader's x planes of this item
    mbar_wait(xfull_bar(s), (li / XBUFS) & 1);

    // ---- 2. conv1: intermediate row i = position r0 - h2 + i reads x plane rows i + j d
    run_conv((2 * (li >> 1)) * k, xs, g.dil);
    named_bar_sync(1 + wg, 128);                       // every warp's MMAs have retired: the buffer may be overwritten

    // ---- 3. epilogue 1: leaky(conv1 + b1) -> intermediate planes (same buffer); the range flag only for rows in [0, T)
#pragma unroll
    for (int hv = 0; hv < 2; ++hv) {
#pragma unroll
      for (int u = 0; u < C / 16; ++u) {
        stage_unit(hv, u);
        const int n = u * 16 + chunk * 4;
        const float4 bvec = __ldg(reinterpret_cast<const float4*>(g.b1 + n));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = hv * 64 + w4 * 16 + i * 8 + rsub;
          const int t = r0 - h2 + row;
          const float4 a4 = *reinterpret_cast<const float4*>(stg + (i * 8 + rsub) * 20 + chunk * 4);
          float v[4] = {a4.x + bvec.x, a4.y + bvec.y, a4.z + bvec.z, a4.w + bvec.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e] + 0.f, MTTS_ACT_LEAKY, 0.1f);   // (+ 0: the unfused epilogue's zero residual)
          store_planes4(xg, PL, sw_elem<SWB>(row, n), v, fmt, (t >= 0 && t < T) ? g.ovf : nullptr);
        }
        __syncwarp();
      }
    }
    named_bar_sync(1 + wg, 128);
    {
      // rows at positions in [-h2, 0) and [T, T + h2) take the planes of their reflection (a position inside this tile)
      constexpr int NCH = SWB / 16;
      const int ns = r0 < h2 ? h2 - r0 : 0;
      const int e0 = T - r0 + h2;
      const int e1 = e0 + h2 < 128 ? e0 + h2 : 128;
      const int ne = e1 > e0 ? e1 - e0 : 0;
      const int total = (ns + ne) * NCH * NP;
      for (int i = tid; i < total; i += 128) {
        const int rr = i / (NCH * NP), rem = i - rr * (NCH * NP);
        const int q = rem / NCH, ch = rem - q * NCH;
        const int row = rr < ns ? rr : e0 + (rr - ns);
        const int t = r0 - h2 + row;
        const int src = (t < 0 ? -t : 2 * (T - 1) - t) - r0 + h2;
        const __nv_bfloat16* pl = xg + q * PL;
        const uint4 v = *reinterpret_cast<const uint4*>(pl + sw_elem<SWB>(src, ch * 8));
        *reinterpret_cast<uint4*>(const_cast<__nv_bfloat16*>(pl) + sw_elem<SWB>(row, ch * 8)) = v;
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1 + wg, 128);

    // ---- 4. conv2: output row i reads intermediate rows i + j; once its MMAs have retired the buffer goes back to the
    // loader
    run_conv((2 * (li >> 1) + 1) * k, xs, 1);
    if (lane == 0) mbar_arrive(xempty_bar(s));

    // ---- 5. epilogue 2: bias -> residual -> scale -> accumulate -> fp32 (the arithmetic of conv_tc_kernel's epilogue)
    float* yb = g.y + (int64_t)b * T * C;
#pragma unroll
    for (int hv = 0; hv < 2; ++hv) {
      // this lane's residual vectors of the half, all requested before the first is used
      float4 rvs[C / 16][2];
#pragma unroll
      for (int u = 0; u < C / 16; ++u)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = hv * 64 + w4 * 16 + i * 8 + rsub, t = r0 + row;
          rvs[u][i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (row < R && t < T) rvs[u][i] = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)t * C + u * 16 + chunk * 4));
        }
#pragma unroll
      for (int u = 0; u < C / 16; ++u) {
        stage_unit(hv, u);
        const int n = u * 16 + chunk * 4;
        const float4 bvec = __ldg(reinterpret_cast<const float4*>(g.b2 + n));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = hv * 64 + w4 * 16 + i * 8 + rsub;
          const int t = r0 + row;
          if (row >= R || t >= T) continue;
          const float4 a4 = *reinterpret_cast<const float4*>(stg + (i * 8 + rsub) * 20 + chunk * 4);
          const float4 rv = rvs[u][i];
          float4 ov = make_float4(0.f, 0.f, 0.f, 0.f);
          if (g.accumulate) ov = *reinterpret_cast<const float4*>(yb + (int64_t)t * C + n);
          float v[4] = {a4.x + bvec.x, a4.y + bvec.y, a4.z + bvec.z, a4.w + bvec.w};
          v[0] = (v[0] + rv.x) * g.out_scale + ov.x;
          v[1] = (v[1] + rv.y) * g.out_scale + ov.y;
          v[2] = (v[2] + rv.z) * g.out_scale + ov.z;
          v[3] = (v[3] + rv.w) * g.out_scale + ov.w;
          *reinterpret_cast<float4*>(yb + (int64_t)t * C + n) = make_float4(v[0], v[1], v[2], v[3]);
        }
        __syncwarp();
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
bool resblock_tc_eligible(int B, int T, int C, int k, int dil, int fmt) {
  if (fmt != MTTS_TC_F16X2 && fmt != MTTS_TC_F16) return false;
  if (C != 32 && C != 64) return false;
  if (k < 3 || k % 2 == 0 || dil < 1) return false;
  const int h1 = dil * (k - 1) / 2, h2 = (k - 1) / 2;
  if (128 + 2 * h1 > RB_XROWS || 2 * h2 >= 64) return false;
  // one reflection maps every padded row of both convolutions into the sequence (the unfused flow's rule then agrees)
  if (T <= h1 + h2) return false;
  return (int64_t)B * T >= 128;
}

template <int C, int NP>
static int rb_launch(const RbTcMaps& maps, const RbTcArgs& a, cudaStream_t st) {
  using Cfg = RbTcCfg<C, NP>;
  MTTS_TRY(tc_smem_attr((const void*)resblock_pair_tc_kernel<C, NP>, 24 + (C == 64 ? 1 : 0) + 2 * (NP - 1), Cfg::SMEM));
  const int R = 128 - (a.k - 1);
  const int64_t items = (int64_t)a.B * cdiv64(a.T, R);
  const int sms = cur_device_sms();
  const int grid = (int)(items < sms ? items : sms);
  launch_k(resblock_pair_tc_kernel<C, NP>, grid, CTC_THREADS, Cfg::SMEM, st, maps, a);
  MTTS_CHECK_LAUNCH();
  return 0;
}

int resblock_pair_tc(const float* x, float* y, const void* w1_tc, const float* b1, const void* w2_tc, const float* b2,
                     int B, int T, int C, int k, int dil, float out_scale, int accumulate, int fmt, cudaStream_t st) {
  MTTS_REQUIRE(x && y && w1_tc && b1 && w2_tc && b2 && x != y, "bad arguments");
  MTTS_REQUIRE(((((uintptr_t)x) | ((uintptr_t)y) | ((uintptr_t)b1) | ((uintptr_t)b2)) & 15) == 0, "unaligned buffers");
  if (!resblock_tc_eligible(B, T, C, k, dil, fmt))
    return fail(MTTS_ERR_UNSUPPORTED, "%s: shape not eligible (C=%lld T=%lld)", "resblock_tc", (long long)C, (long long)T);
  const int np = 3 - fmt, swb = 2 * C;
  RbTcMaps maps;
  for (int q = 0; q < np; ++q) {
    MTTS_TRY(cmap_get((const __nv_bfloat16*)w1_tc + (int64_t)q * k * C * C, (uint64_t)C, (uint64_t)k * C, 0, C, C, swb, fmt, &maps.w1[q]));
    MTTS_TRY(cmap_get((const __nv_bfloat16*)w2_tc + (int64_t)q * k * C * C, (uint64_t)C, (uint64_t)k * C, 0, C, C, swb, fmt, &maps.w2[q]));
  }
  if (np == 1) { maps.w1[1] = maps.w1[0]; maps.w2[1] = maps.w2[0]; }   // unused
  RbTcArgs a;
  a.B = B; a.T = T; a.k = k; a.dil = dil;
  a.x = x; a.b1 = b1; a.b2 = b2; a.y = y;
  a.out_scale = out_scale; a.accumulate = accumulate;
  a.ovf = tc_ovf_ptr();
  if (C == 64) return np == 2 ? rb_launch<64, 2>(maps, a, st) : rb_launch<64, 1>(maps, a, st);
  return np == 2 ? rb_launch<32, 2>(maps, a, st) : rb_launch<32, 1>(maps, a, st);
}

}  // namespace mtts
