// Tensor-core tap-GEMM: every stride-1 Conv1d / ConvTranspose1d (2-tap form) / Linear (k = 1) on wgmma with fp32-grade
// accuracy from split operands and two register accumulators (leading product | corrections):
//   NP = 3 (bf16x3): x = x1 + x2 + x3 in bf16 (to 2^-24); the six products whose weight is >= 2^-16 are issued.
//   NP = 2 (f16x2):  x = x1 + x2' * 2^-11 in fp16 (the residual is stored scaled by 2^11, so it stays a normal fp16 number
//                    whenever x is); three products x1*w1 | x1*w2' + x2'*w1, the correction accumulator is scaled by 2^-11
//                    in the epilogue.  22 significant bits per operand: the dropped x2*w2 term is 2^-22 relative, below
//                    the rounding noise of an fp32 dot product; half the MMAs and two thirds of the operand bytes.
//   NP = 1 (f16):    x ~ fp16(x), ONE product x1*w1 into one accumulator - the opt-in half-precision inference engine, not
//                    fp32-grade (11 significant bits per operand, fp32 accumulation); a sixth of bf16x3's MMAs.
// Eligible wherever Cin % 8 == 0, Cin >= 32, Cout in {32, 64, >= 128 and % 32 == 0} and B*T >= 128; everything else
// stays on the exact FFMA engine (tapconv.cu).  Reference layers: modules/convnet.py:13-18, modules/transformer.py:16-102,
// the speechbrain HiFi-GAN generator (ResBlock1 convs, ConvTranspose1d upsamplers).
//
// Data flow:  activation planes (B, T + halo, C) bf16 x 3 with the padding MATERIALISED (zero / reflect / replicate)
// and the pre-activation applied - written by the producing kernel (LayerNorm, attention, the previous tap-GEMM's
// epilogue) or, failing that, by split_pad_bf16x3_kernel - so that the conv is a "valid" conv over the planes and tap j
// of an output tile is simply the same 128-row tile shifted by j*dil rows: one 3-D TMA box load per (tap, channel
// slab, plane), no im2col, the k-fold re-reads are served by L2.  Weights are packed per tap as (k, Cout, Cin) bf16
// planes (K-major B).  Variants: tile width BN 128 / 64 / 32, split-K with a fixed-order reduction kernel for
// under-filled dense layers.  DESIGN.md section 4 has the anatomy.
#include <algorithm>
#include <mutex>
#include <unordered_map>

#include <stdlib.h>

#include "kernels.h"
#include "tc_ptx.cuh"

namespace mtts {

struct ConvTcMaps {
  CUtensorMap a[3];   // 3-D: (C, Tp, B)
  CUtensorMap b[3];   // 2-D: (Cin, k*Cout)
};

struct ConvTcArgs {
  int32_t B, T, Cin, Cout, k, dil;
  const float* bias;
  const float* res; int64_t res_sb; int32_t ldr;
  float* y; int64_t y_sb; int32_t ldy;
  int32_t post_act; float post_slope; float out_scale; int32_t accumulate;
  int64_t out_shift, ybe;      // transposed-conv form: element offset of the output and valid range per batch item
  // optional bf16x3 copy of the result for the next tensor-core layer
  __nv_bfloat16* op; int64_t op_stride; int32_t op_ld, op_tp, op_hl, op_act; float op_slope;
  // split-K (dense layers with too few tiles): work item = (tile, split); partial sums go to `partial`
  int32_t splits; float* partial;
  int32_t fmt; int32_t* ovf;   // operand format of the plane output (== the kernel's own NP) and the f16 range flag
  int32_t row0;                // first padded row of this conv inside a shared plane buffer (0 for its own planes)
};

// One CTA = 2 consumer warpgroups + 1 TMA producer warpgroup, persistent over the work items, a STAGES-deep ring of
// operand stages between them.  Ping-pong schedule: the consumer warpgroups take the CTA's work items alternately, each
// item whole (mainloop, then its own epilogue, accumulators in registers throughout), and take turns on the tensor pipe
// through a pair of named barriers: warpgroup A issues the MMAs of its item while warpgroup B runs the epilogue of its
// previous one, so every epilogue hides under the other warpgroup's MMAs.  An item is ROWS x BN with at most 128
// accumulator registers per thread: 64 x 128 (one m64 MMA per product) at BN = 128, 128 x BN (two m64 halves) below.
// The producer warpgroup hands its registers to the consumers (setmaxnreg); one elected lane issues the loads, in the
// order the consumers take the items.
// HALO = 1 (convolutions whose input channels fit ONE K-slab, Cin <= SWB / 2): the activation tile of an output tile -
// its 128 rows plus the dil * (k - 1) halo rows - is loaded ONCE into a multi-buffered region and every tap reads it
// through a row-shifted wgmma descriptor; only the (tiny) per-tap weight tiles stream through the stage ring.  The plain
// form re-reads the tile once per tap (k-fold L2 -> SM traffic), which is what bounds the C = 32 / 64 HiFi-GAN stages.
// CL = 2 (plain form, no K split): 2-CTA clusters share the weight tile.  A cluster walks pair items (row-tile pair, N tile);
// rank 0 takes row tile 2p, rank 1 row tile 2p + 1 (past the last row tile: a dummy item on row tile 2p that runs the whole
// barrier protocol and stores nothing).  Each CTA loads its own activation tile and half of the weight rows, multicast into
// both CTAs at the same offset, so a stage moves NP * (A_PLANE + B_PLANE / 2) bytes from L2 into each SM instead of
// NP * (A_PLANE + B_PLANE).  Either CTA's producer writes a stage slot of both, so a slot is refilled only once the owning
// warpgroups of BOTH CTAs have released it (each consumer warp arrives on the local and the peer's empty barrier).
constexpr int CTC_HALO_ROWS = 192;     // rows of a halo tile buffer: 128 + dil * (k - 1) <= 192, a multiple of 8
template <int BN, int SWB, int NP = 3, int HALO = 0>
struct ConvTcCfg {
  // output rows of a work item.  NP = 1 keeps 64 rows at BN = 128 although its single accumulator would fit a 128-row item:
  // the 64-row item measured faster over the PLM / ADM / vocoder shapes (DESIGN.md section 4)
  static constexpr int ROWS = BN == 128 ? 64 : 128;
  static constexpr int HALVES = ROWS / 64;                 // m64 MMAs per product
  static_assert(!HALO || ROWS == 128, "the halo form keeps 128-row tiles");
  static constexpr int BK = SWB / 2;                       // bf16 elements per swizzled row
  static constexpr int A_PLANE = (HALO ? CTC_HALO_ROWS : ROWS) * SWB;
  static constexpr int B_PLANE = BN * SWB;
  static constexpr int STAGE = HALO ? NP * B_PLANE : NP * (A_PLANE + B_PLANE);
  // halo-tile buffers: a tile's rows are requested when the buffer of the tile A_BUFS back is released, i.e. A_BUFS - 1 tiles
  // ahead, so the next tiles' rows are in flight while this one's MMAs and epilogue run
  static constexpr int A_BUFS = HALO ? ((SWB == 64 || NP == 1) ? 4 : (NP == 2 ? 3 : 2)) : 0;
  static constexpr int A_REGION = A_BUFS * NP * A_PLANE;
  static constexpr int EPI_STAGE = 8 * 16 * 20 * 4;          // epilogue transpose buffers: 8 warps x [16 rows][20 floats]
  static constexpr int STAGES_RAW = (227 * 1024 - 1024 - 256 - EPI_STAGE - A_REGION) / STAGE;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : (STAGES_RAW < 2 ? 2 : STAGES_RAW);
  static constexpr int SMEM = A_REGION + STAGES * STAGE + 1024 + 256 + EPI_STAGE;
  static_assert(SMEM <= 227 * 1024 && STAGES_RAW >= 2, "shared-memory budget");
};

template <int BN, int SWB, int NP, int HALO, int CL>
__global__ void __launch_bounds__(CTC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ ConvTcMaps maps, const ConvTcArgs g) {
  using Cfg = ConvTcCfg<BN, SWB, NP, HALO>;
  static_assert(CL == 1 || (CL == 2 && !HALO), "clusters run the plain form");
  pdl_trigger();                                           // the next kernel may be scheduled; it waits for this grid itself
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_a = (smem_u32(smem_raw) + 1023u) & ~1023u;      // HALO: the halo-tile buffers come first
  const uint32_t smem_base = smem_a + Cfg::A_REGION;                   // the stage ring
  const uint32_t bars = smem_base + STAGES * Cfg::STAGE;
  const uint32_t full_bar = bars, empty_bar = bars + 8 * STAGES;
  const uint32_t afull_bar = bars + 16 * STAGES, aempty_bar = afull_bar + 32;   // HALO only (16 * STAGES + 64 <= 256)
  float* epi_stage = reinterpret_cast<float*>(smem_raw + (bars + 256 - smem_u32(smem_raw)));   // 16-byte aligned

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform as far as the compiler can tell
  const int lane = threadIdx.x & 31;
  constexpr int ROWS = Cfg::ROWS, HALVES = Cfg::HALVES;
  const int num_t = (g.T + ROWS - 1) / ROWS, num_n = (g.Cout + BN - 1) / BN;
  const int num_rt = g.B * num_t;                            // row tiles
  const int splits = (HALO || CL == 2) ? 1 : g.splits;
  // work items: (row tile, N tile, K split), N fastest; under CL = 2 (row-tile pair, N tile), walked by the cluster
  const int num_tiles = CL == 2 ? (num_rt + 1) / 2 * num_n : num_rt * num_n * splits;
  const int rank = CL == 2 ? (int)cluster_ctarank() : 0;
  const int item0 = (int)blockIdx.x / CL, istride = (int)gridDim.x / CL;   // CL = 2: the cluster's index and count
  const int ncb = (g.Cin + Cfg::BK - 1) / Cfg::BK;
  const int num_k = g.k * ncb;

  if (warp == 8 && lane == 0) {
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.a[i]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.b[i]) : "memory");
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 4 * CL);     // one arrive per warp of the owning consumer warpgroup of each CTA
    }
    if constexpr (HALO) {
      for (int s = 0; s < Cfg::A_BUFS; ++s) {
        mbar_init(afull_bar + 8 * s, 1);
        mbar_init(aempty_bar + 8 * s, 4);
      }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // CL = 2: the peer's barriers are initialised before any multicast or remote arrive reaches them.  The exits below meet in
  // a second cluster barrier, so that no CTA leaves while its peer can still multicast into it or arrive on its barriers.
  if constexpr (CL == 2) cluster_sync();
  else __syncthreads();
  pdl_wait();        // everything above (barriers, descriptor prefetch) overlapped the previous kernel's tail

  if (warp >= 8) {
    // ================= TMA producer (warp 8 walks the loops, one elected lane issues) =================
    setmaxnreg_dec<CTC_PRODUCER_REGS>();
    if (warp != 8) {
      if constexpr (CL == 2) cluster_sync();
      return;
    }
    const bool leader = elect_one();
    int stage = 0, phase = 0;
    [[maybe_unused]] int ait = 0;
    for (int item = item0; item < num_tiles; item += istride) {
      const int sp = item % splits, tile = item / splits;
      const int kb0 = (int)((int64_t)sp * num_k / splits), kb1 = (int)((int64_t)(sp + 1) * num_k / splits);
      const int nb = tile % num_n;
      int r = tile / num_n;
      if constexpr (CL == 2) r = min(2 * r + rank, num_rt - 1);     // a dummy item loads row tile 2p (valid rows)
      const int tb = r % num_t, b = r / num_t;
      const int trow = tb * ROWS + g.row0;     // the item's first (padded) input row
      if constexpr (HALO) {
        // the tile's activation rows [trow, trow + 128 + dil * (k - 1)) once, then one weight tile per tap
        const int ab = ait % Cfg::A_BUFS, aph = (ait / Cfg::A_BUFS) & 1;
        ++ait;
        mbar_wait(aempty_bar + 8 * ab, aph ^ 1);
        if (leader) {
          mbar_expect_tx(afull_bar + 8 * ab, (uint32_t)(NP * (128 + g.dil * (g.k - 1)) * SWB));
#pragma unroll
          for (int q = 0; q < NP; ++q)
            tma_load_3d(smem_a + (ab * NP + q) * Cfg::A_PLANE, &maps.a[q], afull_bar + 8 * ab, 0, trow, b);
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar + 8 * stage, phase ^ 1);
          const uint32_t sb = smem_base + stage * Cfg::STAGE;
          const uint32_t fb = full_bar + 8 * stage;
          if (leader) {
            mbar_expect_tx(fb, Cfg::STAGE);
#pragma unroll
            for (int q = 0; q < NP; ++q) tma_load_2d(sb + q * Cfg::B_PLANE, &maps.b[q], fb, 0, kb * g.Cout + nb * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      } else {
        for (int kb = kb0; kb < kb1; ++kb) {
          const int j = kb / ncb, cb = kb - j * ncb;
          mbar_wait(empty_bar + 8 * stage, phase ^ 1);
          const uint32_t sa = smem_base + stage * Cfg::STAGE;
          const uint32_t sb = sa + NP * Cfg::A_PLANE;
          const uint32_t fb = full_bar + 8 * stage;
          if (leader) {
            mbar_expect_tx(fb, Cfg::STAGE);
#pragma unroll
            for (int q = 0; q < NP; ++q) tma_load_3d(sa + q * Cfg::A_PLANE, &maps.a[q], fb, cb * Cfg::BK, trow + j * g.dil, b);
            if constexpr (CL == 2) {
              // weight rows [rank * BN / 2, (rank + 1) * BN / 2) of the tile into both CTAs (whole 8-row swizzle atoms);
              // the peer's half completes the other BN / 2 rows' bytes on this CTA's full barrier
              const uint32_t ho = (uint32_t)(rank * (BN / 2) * SWB);
#pragma unroll
              for (int q = 0; q < NP; ++q)
                tma_load_2d_mc(sb + q * Cfg::B_PLANE + ho, &maps.b[q], fb, cb * Cfg::BK, j * g.Cout + nb * BN + rank * (BN / 2),
                               (uint16_t)0x3);
            } else {
#pragma unroll
              for (int q = 0; q < NP; ++q) tma_load_2d(sb + q * Cfg::B_PLANE, &maps.b[q], fb, cb * Cfg::BK, j * g.Cout + nb * BN);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    if constexpr (CL == 2) cluster_sync();
    return;
  }

  // ================= consumers: warpgroup wg owns the CTA's work items wg, wg + 2, wg + 4, ... =================
  setmaxnreg_inc<CTC_CONSUMER_REGS>();
  constexpr float CS = NP == 2 ? F16X2_INV_SCALE : 1.0f;   // weight of the correction accumulator (exact: a power of two)
  constexpr bool BF16 = NP == 3;
  constexpr int NCOR = NP == 1 ? 1 : BN / 2;               // NP = 1: no correction accumulator
  const int wg = warp >> 2, w4 = warp & 3;
  const int chunk = lane & 3, rsub = lane >> 2;
  const int64_t out_shift = HALO ? (int64_t)0 : g.out_shift;
  const bool partial_out = splits > 1;          // raw partial sums; bias / activation / residual run in the reduction kernel
  const bool has_bias = g.bias != nullptr && !partial_out;
  const bool has_res = g.res != nullptr && out_shift == 0 && !partial_out;
  const bool has_acc = g.accumulate != 0 && out_shift == 0 && !partial_out;
  const bool has_y = g.y != nullptr, has_op = g.op != nullptr;
  const int64_t ystep = 8 * (int64_t)g.ldy, rstep = 8 * (int64_t)g.ldr, ostep = 8 * (int64_t)g.op_ld;
  const int64_t pstep = 8 * (int64_t)g.Cout;
  const uint64_t desc_base = wgmma_desc<SWB>(0u);      // everything except the start address
  // Each unit = this warp's 16 rows x 16 columns.  The fragment holds two rows x two columns per lane; writing them out
  // like that would make every global instruction touch 16 different lines, so the unit is transposed through a padded
  // shared buffer and ALL global traffic of the epilogue (y, residual, accumulate, operand planes) is issued as 8 rows x
  // 64 contiguous bytes per instruction.
  float* stg = epi_stage + warp * (16 * 20);
  float acc[HALVES][BN / 2], cor[HALVES][NCOR];
  // Turns on the tensor pipe: warpgroup wg waits on barrier 1 + wg before it issues the MMAs of its item li (li > 0); the
  // other warpgroup arrives there once it has issued all MMAs of item li - 1.  Arrivals are made only for an item that
  // exists, so no barrier is left half-arrived when the CTA exits.
  // The two CTAs of a cluster walk the same items, so their stages, phases and warpgroup turns match.
  const int n_items = num_tiles > item0 ? (num_tiles - item0 + istride - 1) / istride : 0;
  // release of a stage: CL = 2 on this CTA's empty barrier and the peer's, whose producer also writes this slot
  auto release = [&](int s) {
    if constexpr (CL == 2) {
      mbar_arrive_cluster(empty_bar + 8 * s, 0);
      mbar_arrive_cluster(empty_bar + 8 * s, 1);
    } else {
      mbar_arrive(empty_bar + 8 * s);
    }
  };
  int stage = 0, phase = 0;
  for (int li = 0; li < n_items; ++li) {
    const int item = item0 + li * istride;
    const int sp = item % splits, tile = item / splits;
    const int kb0 = (int)((int64_t)sp * num_k / splits), kb1 = (int)((int64_t)(sp + 1) * num_k / splits);
    if ((li & 1) != wg) {                       // the other warpgroup's item: step over its stages of the ring
      const int s = stage + (kb1 - kb0);
      phase ^= (s / STAGES) & 1;
      stage = s % STAGES;
      continue;
    }
    const int nb = tile % num_n;
    int r = tile / num_n;
    bool dummy = false;
    if constexpr (CL == 2) {
      r = 2 * r + rank;
      dummy = r >= num_rt;
    }
    const int tb = r % num_t, b = r / num_t;
    [[maybe_unused]] int ab = 0;
    if (li > 0) named_bar_sync(1 + wg, 256);
    if constexpr (HALO) {
      ab = li % Cfg::A_BUFS;
      mbar_wait(afull_bar + 8 * ab, (li / Cfg::A_BUFS) & 1);
    }
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar + 8 * stage, phase);
      // HALO: A is the halo tile shifted by kb * dil rows (kb == tap: one K-slab per tap).  The swizzle is a function of the
      // shared-memory ADDRESS bits (the TMA wrote with them, the MMA reads with them), so a start address that is a whole
      // number of rows into the tile needs nothing else.
      const uint32_t a_addr = HALO ? smem_a + ab * NP * Cfg::A_PLANE + (uint32_t)(kb * g.dil) * SWB
                                   : smem_base + stage * Cfg::STAGE;
      const uint32_t b_addr = smem_base + stage * Cfg::STAGE + (HALO ? 0 : NP * Cfg::A_PLANE);
      const uint32_t first = (kb == kb0) ? 0u : 1u;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < Cfg::BK / 16; ++ks) {
        const uint32_t bb = b_addr + ks * 32;
        const uint64_t b1 = desc_base | (uint64_t)((bb >> 4) & 0x3FFF), b2 = desc_base | (uint64_t)(((bb + Cfg::B_PLANE) >> 4) & 0x3FFF);
        const uint32_t f = (ks == 0) ? first : 1u;
#pragma unroll
        for (int hv = 0; hv < HALVES; ++hv) {                  // rows [64 hv, 64 hv + 64) of the item
          const uint32_t aa = a_addr + hv * 64 * SWB + ks * 32;
          const uint64_t a1 = wgmma_desc_shifted(desc_base, aa);
          const uint64_t a2 = wgmma_desc_shifted(desc_base, aa + Cfg::A_PLANE);
          if constexpr (NP == 1) {
            Wgmma<BN>::template mma<BF16>(acc[hv], a1, b1, f);       // x1 w1: the only product
          } else if constexpr (NP == 2) {
            Wgmma<BN>::template mma<BF16>(cor[hv], a1, b2, f);       // x1 w2'
            Wgmma<BN>::template mma<BF16>(cor[hv], a2, b1, 1u);      // x2' w1
            Wgmma<BN>::template mma<BF16>(acc[hv], a1, b1, f);       // x1 w1
          } else {
            const uint64_t a3 = wgmma_desc_shifted(desc_base, aa + 2 * Cfg::A_PLANE);
            const uint64_t b3 = desc_base | (uint64_t)(((bb + 2 * Cfg::B_PLANE) >> 4) & 0x3FFF);
            Wgmma<BN>::template mma<BF16>(cor[hv], a2, b2, f);       // x2 w2   (smallest terms first)
            Wgmma<BN>::template mma<BF16>(cor[hv], a1, b3, 1u);      // x1 w3
            Wgmma<BN>::template mma<BF16>(cor[hv], a3, b1, 1u);      // x3 w1
            Wgmma<BN>::template mma<BF16>(cor[hv], a1, b2, 1u);      // x1 w2
            Wgmma<BN>::template mma<BF16>(cor[hv], a2, b1, 1u);      // x2 w1
            Wgmma<BN>::template mma<BF16>(acc[hv], a1, b1, f);       // x1 w1
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                         // the previous stage's MMAs have retired: release it
      if (prev >= 0 && lane == 0) release(prev);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if (li + 1 < n_items) named_bar_arrive(2 - wg, 256);      // all MMAs of this item issued: the other warpgroup's turn
    wgmma_wait<0>();
#pragma unroll
    for (int hv = 0; hv < HALVES; ++hv) {
      wgmma_fence_regs(acc[hv]);
      if constexpr (NP > 1) wgmma_fence_regs(cor[hv]);
    }
    if (lane == 0) {
      if (prev >= 0) release(prev);
      if constexpr (HALO) mbar_arrive(aempty_bar + 8 * ab);     // the halo tile is free once this tile's MMAs have retired
    }
    if (dummy) continue;

    // ---- epilogue of this warp's 16 rows of each 64-row half
#pragma unroll
    for (int hv = 0; hv < HALVES; ++hv) {
      const int t0 = tb * ROWS + hv * 64 + w4 * 16 + rsub;         // this lane's rows: t0 + 8 i
      const int nbase = nb * BN + chunk * 4;
      const int64_t yo = (int64_t)t0 * g.ldy + nbase;                // within batch item b
      const int64_t yb = (int64_t)b * g.y_sb;
      const int64_t ro = (int64_t)b * g.res_sb + (int64_t)t0 * g.ldr + nbase;
      const int64_t oo = ((int64_t)b * g.op_tp + g.op_hl + t0) * g.op_ld + nbase;
      const int64_t po = (((int64_t)sp * g.B + b) * g.T + t0) * g.Cout + nbase;
#pragma unroll
      for (int u = 0; u < BN / 16; ++u) {
        const int n = nbase + u * 16;
        const bool ncol = n < g.Cout;                 // Cout % 4 == 0: a 4-wide chunk is all-in or all-out
#pragma unroll
        for (int h = 0; h < 2; ++h) {                 // fragment columns 8 (2u + h) + 2 (lane % 4) + {0, 1}, rows lane / 4 + {0, 8}
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
        float4 bvec = make_float4(0.f, 0.f, 0.f, 0.f);
        if (has_bias && ncol) bvec = __ldg(reinterpret_cast<const float4*>(g.bias + n));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (!(ncol && (t0 + 8 * i) < g.T)) continue;
          const float4 a4 = *reinterpret_cast<const float4*>(stg + (i * 8 + rsub) * 20 + chunk * 4);
          if (partial_out) {
            *reinterpret_cast<float4*>(g.partial + po + i * pstep + u * 16) = a4;
            continue;
          }
          float4 rv = make_float4(0.f, 0.f, 0.f, 0.f), ov = rv;
          if (has_res) rv = *reinterpret_cast<const float4*>(g.res + ro + i * rstep + u * 16);
          if (has_acc) ov = *reinterpret_cast<const float4*>(g.y + yb + yo + i * ystep + u * 16);
          float v[4] = {a4.x + bvec.x, a4.y + bvec.y, a4.z + bvec.z, a4.w + bvec.w};
          if (g.post_act != MTTS_ACT_NONE) {
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e], g.post_act, g.post_slope);
          }
          v[0] = (v[0] + rv.x) * g.out_scale + ov.x;
          v[1] = (v[1] + rv.y) * g.out_scale + ov.y;
          v[2] = (v[2] + rv.z) * g.out_scale + ov.z;
          v[3] = (v[3] + rv.w) * g.out_scale + ov.w;
          if (has_y) {
            const int64_t flat = yo + i * ystep + u * 16 + out_shift;      // out_shift % 4 == 0: all-in or all-out
            if (HALO || (flat >= 0 && flat + 4 <= g.ybe))
              *reinterpret_cast<float4*>(g.y + yb + flat) = make_float4(v[0], v[1], v[2], v[3]);
          }
          if (has_op) {
            if (g.op_act != MTTS_ACT_NONE) {
#pragma unroll
              for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e], g.op_act, g.op_slope);
            }
            store_planes4(g.op, g.op_stride, oo + i * ostep + u * 16, v, 3 - NP, g.ovf);   // the format of this kernel's NP
          }
        }
        __syncwarp();   // the staging buffer is reused by the next unit
      }
    }
  }
  if constexpr (CL == 2) cluster_sync();
}

// split-K reduction: sums the partial tiles in a FIXED order (bit-reproducible) and applies the tap-GEMM epilogue
// (bias -> activation -> residual -> scale -> accumulate -> fp32 and/or bf16x3 plane store)
__global__ void __launch_bounds__(256)
tc_splitk_reduce_kernel(const ConvTcArgs g, int64_t total4) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int c4 = g.Cout / 4;
  const int n = (int)(i % c4) * 4;
  const int64_t row = i / c4;                 // b * T + t
  const int b = (int)(row / g.T), tt = (int)(row - (int64_t)b * g.T);
  const int64_t stride = (int64_t)g.B * g.T * g.Cout;
  float4 a = *reinterpret_cast<const float4*>(g.partial + row * g.Cout + n);
  for (int sp = 1; sp < g.splits; ++sp) {
    const float4 q = *reinterpret_cast<const float4*>(g.partial + sp * stride + row * g.Cout + n);
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  float v[4] = {a.x, a.y, a.z, a.w};
  if (g.bias) {
    const float4 bv = __ldg(reinterpret_cast<const float4*>(g.bias + n));
    v[0] += bv.x; v[1] += bv.y; v[2] += bv.z; v[3] += bv.w;
  }
  if (g.post_act != MTTS_ACT_NONE) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e], g.post_act, g.post_slope);
  }
  float4 rv = make_float4(0.f, 0.f, 0.f, 0.f), ov = rv;
  if (g.res) rv = *reinterpret_cast<const float4*>(g.res + (int64_t)b * g.res_sb + (int64_t)tt * g.ldr + n);
  if (g.accumulate) ov = *reinterpret_cast<const float4*>(g.y + (int64_t)b * g.y_sb + (int64_t)tt * g.ldy + n);
  v[0] = (v[0] + rv.x) * g.out_scale + ov.x;
  v[1] = (v[1] + rv.y) * g.out_scale + ov.y;
  v[2] = (v[2] + rv.z) * g.out_scale + ov.z;
  v[3] = (v[3] + rv.w) * g.out_scale + ov.w;
  if (g.y) *reinterpret_cast<float4*>(g.y + (int64_t)b * g.y_sb + (int64_t)tt * g.ldy + n) = make_float4(v[0], v[1], v[2], v[3]);
  if (g.op) {
    if (g.op_act != MTTS_ACT_NONE) {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e], g.op_act, g.op_slope);
    }
    store_planes4(g.op, g.op_stride, ((int64_t)b * g.op_tp + g.op_hl + tt) * g.op_ld + n, v, g.fmt, g.ovf);
  }
}

// split-K reduction + LayerNorm of the finished rows (one warp per row, Cout = 128 * NV): the row is reduced exactly like
// tc_splitk_reduce_kernel does (same order of the partial sums, bias -> activation -> residual -> scale -> accumulate), stored
// as fp32, and - still in registers - normalised exactly like layernorm_reg_kernel (ops.cu) and written as operand planes.
// Bit-identical to the two separate launches it replaces.
template <int NV>
__global__ void __launch_bounds__(256)
tc_splitk_reduce_ln_kernel(const ConvTcArgs g, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                           const PlanesOut po) {
  pdl_entry();
  constexpr int C = 128 * NV;
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // b * T + t
  if (row >= (int64_t)g.B * g.T) return;
  const int b = (int)(row / g.T), tt = (int)(row - (int64_t)b * g.T);
  const int64_t stride = (int64_t)g.B * g.T * C;
  float4 v[NV];
  // partial sums: split 0, then + split 1, + split 2 ... per element (the order of tc_splitk_reduce_kernel); the NV loads of
  // one split are independent and in flight together
  const float* pr = g.partial + row * C + lane * 4;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(pr + i * 128);
  for (int sp = 1; sp < g.splits; ++sp) {
    float4 q[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) q[i] = *reinterpret_cast<const float4*>(pr + sp * stride + i * 128);
#pragma unroll
    for (int i = 0; i < NV; ++i) { v[i].x += q[i].x; v[i].y += q[i].y; v[i].z += q[i].z; v[i].w += q[i].w; }
  }
  {
    float4 bvv[NV], rvv[NV], ovv[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int n = i * 128 + lane * 4;
      bvv[i] = g.bias ? __ldg(reinterpret_cast<const float4*>(g.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
      rvv[i] = g.res ? *reinterpret_cast<const float4*>(g.res + (int64_t)b * g.res_sb + (int64_t)tt * g.ldr + n) : make_float4(0.f, 0.f, 0.f, 0.f);
      ovv[i] = g.accumulate ? *reinterpret_cast<const float4*>(g.y + (int64_t)b * g.y_sb + (int64_t)tt * g.ldy + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int n = i * 128 + lane * 4;
      float w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
      if (g.bias) { w[0] += bvv[i].x; w[1] += bvv[i].y; w[2] += bvv[i].z; w[3] += bvv[i].w; }
      if (g.post_act != MTTS_ACT_NONE) {
#pragma unroll
        for (int e = 0; e < 4; ++e) w[e] = act_apply(w[e], g.post_act, g.post_slope);
      }
      v[i] = make_float4((w[0] + rvv[i].x) * g.out_scale + ovv[i].x, (w[1] + rvv[i].y) * g.out_scale + ovv[i].y,
                         (w[2] + rvv[i].z) * g.out_scale + ovv[i].z, (w[3] + rvv[i].w) * g.out_scale + ovv[i].w);
      *reinterpret_cast<float4*>(g.y + (int64_t)b * g.y_sb + (int64_t)tt * g.ldy + n) = v[i];
    }
  }
  // ---- LayerNorm of the row (the arithmetic of layernorm_reg_kernel, operation for operation)
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, d = v[i].z - mean, e = v[i].w - mean;
    q += (a * a + bb * bb) + (d * d + e * e);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * 128 + lane * 4;
    const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + c));
    float o[4] = {(v[i].x - mean) * rstd * gm.x + bt.x, (v[i].y - mean) * rstd * gm.y + bt.y,
                  (v[i].z - mean) * rstd * gm.z + bt.z, (v[i].w - mean) * rstd * gm.w + bt.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = act_apply(o[e], po.act, po.slope);
    store_planes4(po.p, po.stride, row * po.ld + c, o, po.fmt, po.ovf);
  }
}

// fp32 (B,T,C) -> operand planes (B, Tp = T + hl + hr, C): padding materialised, pre-activation applied
__global__ void __launch_bounds__(256)
split_pad_kernel(const float* __restrict__ x, int64_t x_sb, int ldx, int T, int C, int hl, int Tp, int pad_mode,
                 int pre_act, float slope, __nv_bfloat16* __restrict__ planes, int64_t plane_stride,
                 int64_t total4, int fmt, int32_t* ovf) {
  pdl_entry();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int cq = C >> 2;
  const int c = (int)(i % cq) * 4;
  const int64_t bu = i / cq;
  const int u = (int)(bu % Tp);
  const int b = (int)(bu / Tp);
  int ti = u - hl;
  if (ti < 0 || ti >= T) {
    if (pad_mode == MTTS_PAD_ZERO) ti = -1;
    else if (pad_mode == MTTS_PAD_REPLICATE) ti = ti < 0 ? 0 : T - 1;
    else {
      if (ti < 0) ti = -ti;
      if (ti >= T) ti = 2 * (T - 1) - ti;
      if (ti < 0 || ti >= T) ti = -1;
    }
  }
  float f[4] = {0.f, 0.f, 0.f, 0.f};
  if (ti >= 0) {
    const float4 v = *reinterpret_cast<const float4*>(x + (int64_t)b * x_sb + (int64_t)ti * ldx + c);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) f[e] = act_apply(f[e], pre_act, slope);
  store_planes4(planes, plane_stride, ((int64_t)b * Tp + u) * C + c, f, fmt, ovf);
}

// Materialise the padding rows of plane buffers whose interior rows were written by a producer epilogue:
// planes (3 | 2 | 1, B, Tp, C) of `fmt` (one plane per gridDim.z) with hl leading halo rows; reflect / replicate / zero
// about the T interior rows.
__global__ void __launch_bounds__(256)
halo_fill_kernel(__nv_bfloat16* __restrict__ planes, int64_t plane_stride, int T, int C, int hl, int Tp, int pad_mode) {
  pdl_entry();
  const int b = blockIdx.y, q = blockIdx.z;
  const int nh = Tp - T;                     // halo rows in total (hl leading, the rest trailing)
  const int c8 = C / 8;                      // 16-byte chunks per row
  __nv_bfloat16* base = planes + q * plane_stride + (int64_t)b * Tp * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nh * c8; i += gridDim.x * blockDim.x) {
    const int hr = i / c8, ch = i - hr * c8;
    const int u = hr < hl ? hr : T + hr;     // padded row index of this halo row
    int ti = u - hl;
    if (pad_mode == MTTS_PAD_REPLICATE) ti = ti < 0 ? 0 : T - 1;
    else if (pad_mode == MTTS_PAD_REFLECT) {
      if (ti < 0) ti = -ti;
      if (ti >= T) ti = 2 * (T - 1) - ti;
      if (ti < 0 || ti >= T) ti = -1;
    } else ti = -1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (ti >= 0) v = *reinterpret_cast<const uint4*>(base + (int64_t)(hl + ti) * C + ch * 8);
    *reinterpret_cast<uint4*>(base + (int64_t)u * C + ch * 8) = v;
  }
}

int halo_fill(void* planes_base, int B, int T, int C, int hl, int hr, int pad_mode, int fmt, cudaStream_t st) {
  MTTS_REQUIRE(planes_base && C % 8 == 0 && hl >= 0 && hr >= 0, "bad arguments");
  MTTS_REQUIRE(fmt == MTTS_TC_BF16X3 || fmt == MTTS_TC_F16X2 || fmt == MTTS_TC_F16, "unknown operand format");
  if (hl + hr == 0 || B <= 0) return 0;
  __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>((((uintptr_t)planes_base) + 1023) & ~(uintptr_t)1023);
  const int Tp = T + hl + hr;
  const int64_t plane_stride = (int64_t)B * Tp * C;
  const int work = (hl + hr) * (C / 8);
  dim3 grid((unsigned)cdiv64(work, 256), (unsigned)B, (unsigned)(3 - fmt));
  launch_k(halo_fill_kernel, grid, 256, 0, st, planes, plane_stride, T, C, hl, Tp, pad_mode);
  MTTS_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_enc = nullptr;
static std::mutex g_ctc_mu;          // guards g_enc, the descriptor cache and the per-device table (not the launches)

// per-device state: SM count, which kernel instantiations have had their shared-memory attribute raised (the attribute
// is per device), how many 2-CTA clusters of each clustered instantiation can be resident at once, and the
// caller-registered f16 range flag
constexpr int MAX_DEV = 64;
struct DevState { int sms = 0; uint64_t attr_done = 0; int max_clusters[12] = {}; int32_t* ovf = nullptr; };
static DevState g_dev[MAX_DEV];

int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev < 0 || dev >= MAX_DEV ? 0 : dev;
}
// SM budget of the calling host thread's launches (0 = the whole device).  The persistent tensor-core kernels size their
// grids from it, so two streams can share the device: the vocoder pass that re-vocodes the prompt runs on a side stream
// with a reduced budget while the latency-bound AR loops use the SMs it leaves free (models/megatts2.py).
static thread_local int g_sm_limit = 0;
int set_sm_limit(int n) {
  g_sm_limit = n > 0 ? n : 0;
  return 0;
}
// Launch policy of the calling host thread while two streams share the device (models/megatts2.py, the prompt re-vocode beside
// the MRTE + ADM stages).  Two rules make the sharing work; without either of them the short launches of one stream queue
// behind long persistent CTAs of the other:
//  * the budgets of the two streams add up to the device (a persistent grid sized for all SMs waits for the other stream's CTAs);
//  * no programmatic dependent launch on the stream with the long kernels: its NEXT kernel's CTAs would be scheduled early onto
//    the SMs left free for the other stream and sit there in griddepcontrol.wait until the current kernel has finished.
// `allow_pairs` = 0 keeps the tap-GEMM on single CTAs: a 2-CTA cluster needs two free SMs of one GPC at once, which a
// stream sharing the device with long persistent kernels of another may not find.
static thread_local bool g_allow_pairs = true;
int set_launch_policy(int sm_limit, int allow_pairs, int allow_pdl) {
  g_allow_pairs = allow_pairs != 0;
  g_sm_limit = sm_limit > 0 ? sm_limit : 0;
  set_thread_pdl(allow_pdl != 0);
  return 0;
}
int cur_device_sms() {
  const int dev = cur_device();
  if (!g_dev[dev].sms) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    g_dev[dev].sms = n > 0 ? n : 1;
  }
  const int all = g_dev[dev].sms;
  return g_sm_limit > 0 && g_sm_limit < all ? g_sm_limit : all;
}
int tc_smem_attr(const void* kernel, int slot, int bytes) {
  const int dev = cur_device();
  if (g_dev[dev].attr_done & (1ull << slot)) return 0;
  std::lock_guard<std::mutex> lk(g_ctc_mu);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return fail(MTTS_ERR_CUDA, "%s: cudaFuncSetAttribute failed: %lld", "conv_tc", (long long)e);
  g_dev[dev].attr_done |= (1ull << slot);
  return 0;
}
// 2-CTA clusters of a clustered tap-GEMM instantiation (index idx < 12) that the device can hold at once; queried once per
// device after the shared-memory attribute is set.  On H100 this may be fewer than SMs / 2: a cluster's CTAs share a GPC.
static int tc_max_clusters(const void* kernel, int idx, int smem, int* out) {
  int& mc = g_dev[cur_device()].max_clusters[idx];
  *out = mc;
  if (mc > 0) return 0;
  std::lock_guard<std::mutex> lk(g_ctc_mu);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2); cfg.blockDim = dim3(CTC_THREADS); cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeClusterDimension;
  at.val.clusterDim.x = 2; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
  cfg.attrs = &at; cfg.numAttrs = 1;
  int n = 0;
  const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg);
  if (e != cudaSuccess || n < 1)
    return fail(MTTS_ERR_CUDA, "%s: no 2-CTA cluster fits (cudaOccupancyMaxActiveClusters: error %lld, %lld clusters)",
                "conv_tc", (long long)e, (long long)n);
  mc = n;
  *out = n;
  return 0;
}
int32_t* tc_ovf_ptr() { return g_dev[cur_device()].ovf; }
int tc_overflow_bind(int32_t* flag) {
  g_dev[cur_device()].ovf = flag;
  return 0;
}

struct CMapKey {
  const void* p; uint64_t d0, d1, d2, b0, b1; int swb, dt;
  bool operator==(const CMapKey& o) const {
    return p == o.p && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && b0 == o.b0 && b1 == o.b1 && swb == o.swb && dt == o.dt;
  }
};
struct CMapKeyHash {
  size_t operator()(const CMapKey& k) const {
    uint64_t h = (uint64_t)k.p;
    h = h * 0x9E3779B97F4A7C15ull + k.d0; h = h * 0x9E3779B97F4A7C15ull + k.d1; h = h * 0x9E3779B97F4A7C15ull + k.d2;
    h = h * 0x9E3779B97F4A7C15ull + k.b0 * 131 + k.b1 * 7 + k.swb + 1000 * k.dt;
    return (size_t)h;
  }
};
// Descriptor cache: keyed by (pointer, dims, box, swizzle, dtype); a descriptor holds nothing but those, so a stale entry
// for a freed-and-reused address is still correct.  Bounded: when full, the older half (by insertion order) is dropped.
static std::unordered_map<CMapKey, std::pair<CUtensorMap, uint64_t>, CMapKeyHash> g_cmaps;
static uint64_t g_cmap_tick = 0;
constexpr size_t CMAP_CAP = 16384;

static int ctc_init_locked() {
  if (g_enc) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
    return fail(MTTS_ERR_CUDA, "%s: cuTensorMapEncodeTiled not available", "conv_tc");
  g_enc = (EncodeTiledFn)fn;
  return 0;
}

// 2-byte-element tensor (d2, d1, d0) row-major, box (1, b1, b0), SWB-byte swizzle; rank 2 when d2 == 0
int cmap_get(const void* p, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1, int swb, int fmt,
                    CUtensorMap* out) {
  std::lock_guard<std::mutex> lk(g_ctc_mu);
  MTTS_TRY(ctc_init_locked());
  CMapKey key{p, d0, d1, d2, b0, b1, swb, fmt};
  auto itf = g_cmaps.find(key);
  if (itf != g_cmaps.end()) { *out = itf->second.first; return 0; }
  const int rank = d2 ? 3 : 2;
  cuuint64_t dims[3] = {d0, d1, d2 ? d2 : 1};
  cuuint64_t strides[2] = {d0 * 2, d0 * d1 * 2};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  CUresult r = g_enc(&m, fmt != MTTS_TC_BF16X3 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank,
                     const_cast<void*>(p), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MTTS_ERR_CUDA, "%s: cuTensorMapEncodeTiled failed: %lld", "conv_tc", (long long)r);
  if (g_cmaps.size() >= CMAP_CAP) {
    const uint64_t cut = g_cmap_tick - CMAP_CAP / 2;
    for (auto it = g_cmaps.begin(); it != g_cmaps.end();) it = it->second.second < cut ? g_cmaps.erase(it) : ++it;
  }
  g_cmaps[key] = {m, g_cmap_tick++};
  *out = m;
  return 0;
}

// `ctas`: the plan's grid (TcPlan::ctas); a clustered launch is further capped at the clusters the device can hold at once
template <int BN, int SWB, int NP, int HALO = 0, int CL = 1>
static int conv_tc_launch(const ConvTcMaps& maps, const ConvTcArgs& a, int ctas, cudaStream_t st) {
  using Cfg = ConvTcCfg<BN, SWB, NP, HALO>;
  static_assert(SWB == 128 || BN == 32, "64-byte K-slabs run at BN = 32 only");
  // one bit per instantiation in the per-device table (the max-dynamic-shared-memory attribute is per device)
  constexpr int plain = (BN == 128 ? 0 : BN == 64 ? 1 : SWB == 128 ? 2 : 3) + 4 * (3 - NP);
  constexpr int slot = HALO ? 12 + (BN == 64 ? 0 : 1) + 2 * (3 - NP) : CL == 2 ? 32 + plain : plain;
  static_assert(slot < 24 || slot >= 32, "attribute slots (24-31: resblock_tc.cu)");
  const void* kern = (const void*)conv_tc_kernel<BN, SWB, NP, HALO, CL>;
  MTTS_TRY(tc_smem_attr(kern, slot, Cfg::SMEM));
  int grid = ctas;
  if constexpr (CL == 2) {
    int mc = 0;
    MTTS_TRY(tc_max_clusters(kern, plain, Cfg::SMEM, &mc));
    if (grid > 2 * mc) grid = 2 * mc;
  }
  launch_kc(CL, conv_tc_kernel<BN, SWB, NP, HALO, CL>, grid, CTC_THREADS, Cfg::SMEM, st, maps, a);
  MTTS_CHECK_LAUNCH();
  return 0;
}

template <int NP, int CL>
static int conv_tc_dispatch(const ConvTcMaps& maps, const ConvTcArgs& a, int BN, int SWB, int ctas, cudaStream_t st) {
  if (SWB == 64) {
    MTTS_REQUIRE(BN == 32 && a.splits == 1, "a plan with 64-byte K-slabs runs at BN = 32 without a K split");
    return conv_tc_launch<32, 64, NP, 0, CL>(maps, a, ctas, st);
  }
  if (BN == 128) return conv_tc_launch<128, 128, NP, 0, CL>(maps, a, ctas, st);
  if (BN == 64) return conv_tc_launch<64, 128, NP, 0, CL>(maps, a, ctas, st);
  return conv_tc_launch<32, 128, NP, 0, CL>(maps, a, ctas, st);
}

bool conv_tc_eligible(const mtts_conv_params& p) {
  if (!p.w_tc || !p.tc_scratch) return false;
  if (p.tc_fmt != MTTS_TC_BF16X3 && p.tc_fmt != MTTS_TC_F16X2 && p.tc_fmt != MTTS_TC_F16) return false;
  if (p.stride != 1 || p.in_lens) return false;
  if (p.out_shift != 0 && (p.out_shift % 4 != 0 || p.y_batch_elems % 4 != 0 || p.res || p.accumulate || p.tc_out_planes || !p.y))
    return false;
  if (p.Cin % 8 != 0 || p.Cin < 32) return false;
  if (!p.tc_presplit && (p.ldx % 4 != 0 || (p.x_batch_stride % 4) != 0 || (((uintptr_t)p.x) & 15) != 0)) return false;
  if (!(p.Cout == 32 || p.Cout == 64 || (p.Cout >= 128 && p.Cout % 32 == 0))) return false;
  if (p.Cin < 64 && p.Cout != 32) return false;          // Cin < 64 (64-byte K-slabs) is planned at BN = 32 only
  if (p.y && (p.ldy % 4 != 0 || p.y_batch_stride % 4 != 0 || (((uintptr_t)p.y) & 15) != 0)) return false;
  if (!p.y && (!p.tc_out_planes || p.accumulate)) return false;
  if (p.tc_out_planes && (p.Cout % 32 != 0 || p.tc_out_ld % 4 != 0 || p.tc_out_plane_stride % 4 != 0)) return false;
  if (p.res && (p.ldr % 4 != 0 || p.res_batch_stride % 4 != 0 || (((uintptr_t)p.res) & 15) != 0)) return false;
  if (p.Tout != p.Tin + 2 * p.pad - p.dil * (p.k - 1)) return false;
  // tiny problems stay on the exact FFMA engine - except rows that already sit in a plane buffer of >= 128 rows (the last
  // rows of an AR step: one half-filled tile, K split across the SMs)
  if ((int64_t)p.B * p.Tout < ((p.tc_presplit && p.tc_rows_cap >= 128) ? 32 : 128)) return false;
  int64_t Tp = p.Tout + p.dil * (p.k - 1);
  if (p.tc_in_tp > 0 || p.tc_in_row0 != 0) {      // shared plane buffer: this conv's rows must lie inside it
    if (!p.tc_presplit || p.tc_rows_cap > 0 || p.tc_in_row0 < 0 || p.tc_in_tp < p.tc_in_row0 + Tp) return false;
    Tp = p.tc_in_tp;
  }
  int64_t rows = (int64_t)p.B * Tp;
  if (p.tc_rows_cap > 0) {
    if (p.k != 1 || p.B != 1 || p.tc_rows_cap < rows) return false;
    rows = p.tc_rows_cap;
  }
  return 3 * rows * p.Cin * 2 + 2048 <= p.tc_scratch_bytes;
}

// Split-K cost model of tc_plan: at most CTC_SPLITK_MAX splits, taken when the split launch models below
// CTC_SPLITK_MARGIN of the unsplit one.  CTC_SPLITK_LN_RED: modelled cycles of a reduction that REPLACES the LayerNorm
// launch that would follow anyway (tc_splitk_reduce_ln_kernel), against 9000 for a reduction in a launch of its own.
constexpr int CTC_SPLITK_MAX = 8;
constexpr double CTC_SPLITK_MARGIN = 0.85;
constexpr double CTC_SPLITK_LN_RED = 2000.0;

// The launch plan of one tap-GEMM: K-slab width, N-tile width, K splits, halo form, CTAs per cluster (1 | 2) and grid.  A
// pure function of the shape, the SM budget, the operand format, the partial-sum space, whether a LayerNorm rides on the
// reduction and whether clusters are allowed, so the policy can be queried and tested without a GPU (mtts_tc_plan_query_ex,
// tests/test_abi_and_host.py, tests/test_gpu_tc_cluster.py).
struct TcPlan { int SWB, BN, splits; bool halo_form; int cluster, ctas; };
static TcPlan tc_plan(int sms, const mtts_conv_params& p, int np, bool ln_rides, bool pairs) {
  const int halo = p.dil * (p.k - 1);
  const int SWB = p.Cin >= 64 ? 128 : 64;
  int BN = 32;             // Cin < 64 (64-byte K-slabs): conv_tc_eligible admits Cout = 32 only
  int splits = 1;
  // N-tile width.  A persistent CTA walks ceil(tiles / SMs) tiles of nk K-slabs, so the width with the cheapest walk wins
  // (modelled cycles per MMA: 65 at N = 128, 55, the per-instruction floor, at N <= 64) and ties go to the narrower tile
  // (under-filled grids are latency-bound: more SMs stream the weights).  The fill rule (the widest tile that still gives
  // 80 % of the SMs a tile) would e.g. run the PLM FF2 layer of steps 19 ... 28 as two waves of N = 64 tiles where one wave
  // of N = 128 tiles does.  Convolutions (k > 1) keep the fill rule: their grids are hundreds of waves deep and the halo
  // form wants BN == Cout.
  if (SWB == 128) {
    const int64_t mt = (int64_t)p.B * cdiv64(p.Tout, 128);
    const int cands[3] = {128, 64, 32};
    if (p.k == 1) {
      int64_t best = INT64_MAX;
      for (int i = 0; i < 3; ++i) {
        if (cands[i] > p.Cout) continue;
        const int64_t c = cdiv64(mt * cdiv64(p.Cout, cands[i]), sms) * (cands[i] == 128 ? 65 : 55);
        if (c <= best) { best = c; BN = cands[i]; }
      }
    } else {
      for (int i = 0; i < 3; ++i) {
        if (cands[i] > p.Cout) continue;
        BN = cands[i];
        if (mt * cdiv64(p.Cout, cands[i]) >= (int64_t)(sms * 4) / 5) break;
      }
    }
  }
  // split-K for dense layers with too few output tiles to fill the GPU (the early steps of the AR loops, the N = 1024
  // layers up to ~30 steps): narrow tiles would pay the per-MMA minimum on every k-step, so K is split across CTAs at full
  // tile width instead and a second kernel reduces the partials
  {
    const int64_t rows = (int64_t)p.B * p.Tout;
    const int64_t t128 = (int64_t)p.B * cdiv64(p.Tout, 128) * cdiv64(p.Cout, 128);
    const int nk = (p.Cin + 63) / 64;
    if (SWB == 128 && p.k == 1 && p.out_shift == 0 && p.tc_partial && p.Cout >= 128 && t128 < (int64_t)(sms * 4) / 5) {
      int sk = (int)(sms / t128);
      if (sk > CTC_SPLITK_MAX) sk = CTC_SPLITK_MAX;
      if (sk > nk / 2) sk = nk / 2;
      if (sk >= 2 && (int64_t)sk * rows * p.Cout * 4 <= p.tc_partial_bytes) {
        const int64_t tiles_bn = (int64_t)p.B * cdiv64(p.Tout, 128) * cdiv64(p.Cout, BN);
        const double waves = (double)cdiv64(tiles_bn, sms);
        const double mmas = 4.0 * (np == 1 ? 1 : 2 * np);                                   // MMAs per 64-wide K-slab (modelled)
        const double cost_now = waves * nk * mmas * (BN == 128 ? 65.0 : 55.0);                // cycles per CTA
        const double cost_split = (double)cdiv64(nk, sk) * mmas * 65.0 + (ln_rides ? CTC_SPLITK_LN_RED : 9000.0);   // + reduction kernel
        if (cost_split < CTC_SPLITK_MARGIN * cost_now) { splits = sk; BN = 128; }
      }
    }
  }
  // halo form: one K-slab per tap (Cin <= SWB / 2), the activation tile + halo fits the 192-row buffer
  const bool halo_form = splits == 1 && p.out_shift == 0 && p.k > 1 && p.Cin <= SWB / 2 &&
                         halo + 128 <= CTC_HALO_ROWS &&   // (the halo kernel's epilogue has no K-split / transposed-conv paths)
                         ((SWB == 64 && BN == 32) || (SWB == 128 && BN == 64)) && p.Cout == BN;
  // 2-CTA clusters sharing the weight tile: the plain form without a K split, at least one row-tile pair and two SMs.
  // Split launches (the early, latency-bound AR steps) and the halo form (its weight tiles are small) stay single CTAs.
  const int64_t row_tiles = (int64_t)p.B * cdiv64(p.Tout, (BN == 128 && !halo_form) ? 64 : 128);
  const int64_t n_tiles = cdiv64(p.Cout, BN);
  const int cluster = (pairs && !halo_form && splits == 1 && row_tiles >= 2 && sms >= 2) ? 2 : 1;
  int64_t ctas;
  if (cluster == 2) {
    const int64_t pair_items = cdiv64(row_tiles, 2) * n_tiles;
    ctas = 2 * std::min<int64_t>(pair_items, sms / 2);          // an odd SM budget leaves one SM unused
  } else {
    ctas = std::min<int64_t>(row_tiles * n_tiles * splits, sms);
  }
  TcPlan pl;
  pl.SWB = SWB; pl.BN = BN; pl.splits = splits; pl.halo_form = halo_form; pl.cluster = cluster; pl.ctas = (int)ctas;
  return pl;
}

// MEGATTS2_LN_FUSE=0: the LayerNorm a split-K reduction could carry runs as its own launch instead (read once).  The launch
// plan does not change with it, so the two forms sum the same partials in the same order and agree bit for bit.
static bool ln_fuse() {
  static const bool on = [] {
    const char* e = getenv("MEGATTS2_LN_FUSE");
    return !(e && e[0] == '0');
  }();
  return on;
}

int conv_tc(const mtts_conv_params& p, cudaStream_t st, LnFuse* ln) {
  if (ln) ln->done = 0;
  const int sms = cur_device_sms();
  const int fmt = p.tc_fmt;
  const int np = 3 - fmt;                                     // operand planes
  int32_t* ovf = tc_ovf_ptr();
  const int halo = p.dil * (p.k - 1);
  const int hl = p.pad, Tp = p.Tout + halo;
  const int64_t Tp_map = p.tc_rows_cap > 0 ? p.tc_rows_cap : (p.tc_in_tp > 0 ? p.tc_in_tp : Tp);     // descriptor rows (>= Tp)
  __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>((((uintptr_t)p.tc_scratch) + 1023) & ~(uintptr_t)1023);
  const int64_t plane_stride = (int64_t)p.B * Tp_map * p.Cin;
  if (!p.tc_presplit) {
    const int64_t total4 = (int64_t)p.B * Tp * p.Cin / 4;
    launch_k(split_pad_kernel, (unsigned)cdiv64(total4, 256), 256, 0, st, p.x, p.x_batch_stride, p.ldx, p.Tin, p.Cin, hl, Tp,
                                                                   p.pad_mode, p.pre_act, p.pre_slope, planes, plane_stride,
                                                                   total4, fmt, ovf);
    MTTS_CHECK_LAUNCH();
  }
  // the reduction of a split launch can carry the LayerNorm the caller asked for when a row is 3 / 4 / 6 / 8 x 128 wide
  const bool ln_rides = ln && ln->po.p && p.y && !p.tc_out_planes && (p.Cout == 1024 || p.Cout == 768 || p.Cout == 512 || p.Cout == 384);
  const TcPlan pl = tc_plan(sms, p, np, ln_rides, g_allow_pairs);
  const int SWB = pl.SWB, BN = pl.BN, splits = pl.splits, ctas = pl.ctas;
  const bool halo_form = pl.halo_form;
  // activation box: the work item's rows (ConvTcCfg::ROWS: 64 at BN = 128, else 128), the halo form adds the halo rows
  const int a_rows = halo_form ? 128 + halo : (BN == 128 ? 64 : 128);
  ConvTcMaps maps;
  for (int q = 0; q < np; ++q) {
    MTTS_TRY(cmap_get(planes + q * plane_stride, (uint64_t)p.Cin, (uint64_t)Tp_map, (uint64_t)p.B, SWB / 2,
                      a_rows, SWB, fmt, &maps.a[q]));
    // weight box: the N tile, or the half of it that each CTA of a 2-CTA cluster loads
    MTTS_TRY(cmap_get((const __nv_bfloat16*)p.w_tc + (int64_t)q * p.k * p.Cout * p.Cin, (uint64_t)p.Cin,
                      (uint64_t)p.k * p.Cout, 0, SWB / 2, BN / pl.cluster, SWB, fmt, &maps.b[q]));
  }
  for (int q = np; q < 3; ++q) { maps.a[q] = maps.a[np - 1]; maps.b[q] = maps.b[np - 1]; }   // unused
  ConvTcArgs a;
  a.B = p.B; a.T = p.Tout; a.Cin = p.Cin; a.Cout = p.Cout; a.k = p.k; a.dil = p.dil;
  a.bias = p.bias; a.res = p.res; a.res_sb = p.res_batch_stride; a.ldr = p.ldr;
  a.y = p.y; a.y_sb = p.y_batch_stride; a.ldy = p.ldy;
  a.post_act = p.post_act; a.post_slope = p.post_slope; a.out_scale = p.out_scale; a.accumulate = p.accumulate;
  a.out_shift = p.out_shift; a.ybe = p.y_batch_elems ? p.y_batch_elems : (int64_t)p.Tout * p.ldy;
  a.op = reinterpret_cast<__nv_bfloat16*>(p.tc_out_planes); a.op_stride = p.tc_out_plane_stride; a.op_ld = p.tc_out_ld;
  a.op_tp = p.tc_out_tp; a.op_hl = p.tc_out_hl; a.op_act = p.tc_out_act; a.op_slope = p.tc_out_slope;
  a.splits = splits; a.partial = reinterpret_cast<float*>(p.tc_partial);
  a.fmt = fmt; a.ovf = ovf; a.row0 = p.tc_in_row0;
  if (halo_form) {
    if (SWB == 64)
      return np == 1 ? conv_tc_launch<32, 64, 1, 1>(maps, a, ctas, st)
           : np == 2 ? conv_tc_launch<32, 64, 2, 1>(maps, a, ctas, st) : conv_tc_launch<32, 64, 3, 1>(maps, a, ctas, st);
    return np == 1 ? conv_tc_launch<64, 128, 1, 1>(maps, a, ctas, st)
         : np == 2 ? conv_tc_launch<64, 128, 2, 1>(maps, a, ctas, st) : conv_tc_launch<64, 128, 3, 1>(maps, a, ctas, st);
  }
  if (splits > 1) {
    // a split launch runs at BN = 128 on the plan's K-slab width: the kernel's stage size must match the boxes the
    // descriptors above were encoded with
    MTTS_TRY((np == 1 ? conv_tc_dispatch<1, 1>(maps, a, 128, SWB, ctas, st)
            : np == 2 ? conv_tc_dispatch<2, 1>(maps, a, 128, SWB, ctas, st) : conv_tc_dispatch<3, 1>(maps, a, 128, SWB, ctas, st)));
    // the rows' LayerNorm rides on the reduction when the caller asked for it and a row is 3 / 4 / 6 / 8 x 128 wide
    if (ln_fuse() && ln && ln->po.p && a.y && !a.op && a.out_shift == 0 && (p.Cout == 1024 || p.Cout == 768 || p.Cout == 512 || p.Cout == 384) &&
        p.ldy % 4 == 0 && ln->po.ld % 4 == 0 && ln->po.stride % 4 == 0) {
      const unsigned grid = (unsigned)cdiv64((int64_t)p.B * p.Tout, 4);      // 4 rows (warps) per CTA
      if (p.Cout == 1024) launch_k(tc_splitk_reduce_ln_kernel<8>, grid, 128, 0, st, a, ln->gamma, ln->beta, ln->eps, ln->po);
      else if (p.Cout == 768) launch_k(tc_splitk_reduce_ln_kernel<6>, grid, 128, 0, st, a, ln->gamma, ln->beta, ln->eps, ln->po);
      else if (p.Cout == 512) launch_k(tc_splitk_reduce_ln_kernel<4>, grid, 128, 0, st, a, ln->gamma, ln->beta, ln->eps, ln->po);
      else launch_k(tc_splitk_reduce_ln_kernel<3>, grid, 128, 0, st, a, ln->gamma, ln->beta, ln->eps, ln->po);
      MTTS_CHECK_LAUNCH();
      ln->done = 1;
      return 0;
    }
    const int64_t total4 = (int64_t)p.B * p.Tout * p.Cout / 4;
    launch_k(tc_splitk_reduce_kernel, (unsigned)cdiv64(total4, 256), 256, 0, st, a, total4);
    MTTS_CHECK_LAUNCH();
    return 0;
  }
  if (pl.cluster == 2)
    return np == 1 ? conv_tc_dispatch<1, 2>(maps, a, BN, SWB, ctas, st)
         : np == 2 ? conv_tc_dispatch<2, 2>(maps, a, BN, SWB, ctas, st) : conv_tc_dispatch<3, 2>(maps, a, BN, SWB, ctas, st);
  return np == 1 ? conv_tc_dispatch<1, 1>(maps, a, BN, SWB, ctas, st)
       : np == 2 ? conv_tc_dispatch<2, 1>(maps, a, BN, SWB, ctas, st) : conv_tc_dispatch<3, 1>(maps, a, BN, SWB, ctas, st);
}

// diagnostics: the plan conv_tc() would pick for a stride-1 tap-GEMM of this shape on `sms` SMs; out7 = {BN, splits, CTA
// pair (always 0: no CTA-pair MMA kernels on sm_90), halo form (0 | 1), K-slab bytes, CTAs per cluster (1 | 2), CTAs of the
// grid (before a clustered launch is capped at the clusters the device can hold)}
int tc_plan_query_ex(int sms, int B, int T, int Cin, int Cout, int k, int dil, int fmt, int64_t partial_bytes, int ln_rides,
                     int allow_pairs, int32_t* out7) {
  MTTS_REQUIRE(out7 && sms > 0 && B > 0 && T > 0 && Cin > 0 && Cout > 0 && k > 0 && dil > 0, "bad arguments");
  MTTS_REQUIRE(fmt == MTTS_TC_BF16X3 || fmt == MTTS_TC_F16X2 || fmt == MTTS_TC_F16, "unknown operand format");
  mtts_conv_params p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.Tin = T + dil * (k - 1); p.Tout = T; p.Cin = Cin; p.Cout = Cout; p.k = k; p.stride = 1; p.dil = dil;
  static float dummy;
  p.y = &dummy;
  if (partial_bytes > 0) { p.tc_partial = &dummy; p.tc_partial_bytes = partial_bytes; }
  const TcPlan pl = tc_plan(sms, p, 3 - fmt, ln_rides != 0, allow_pairs != 0);
  out7[0] = pl.BN; out7[1] = pl.splits; out7[2] = 0; out7[3] = pl.halo_form ? 1 : 0; out7[4] = pl.SWB;
  out7[5] = pl.cluster; out7[6] = pl.ctas;
  return 0;
}
// the first five fields of tc_plan_query_ex with clusters allowed
int tc_plan_query(int sms, int B, int T, int Cin, int Cout, int k, int dil, int fmt, int64_t partial_bytes, int ln_rides, int32_t* out5) {
  MTTS_REQUIRE(out5, "bad arguments");
  int32_t out7[7];
  MTTS_TRY(tc_plan_query_ex(sms, B, T, Cin, Cout, k, dil, fmt, partial_bytes, ln_rides, 1, out7));
  memcpy(out5, out7, 5 * sizeof(int32_t));
  return 0;
}

// fp32 (B, T, C) -> padded operand planes (B, hl + T + hr, C) at the 1024-byte-aligned start of `planes_base`
int split_pad(const float* x, int64_t x_sb, int ldx, int B, int T, int C, int hl, int hr, int pad_mode, int act, float slope,
              void* planes_base, int fmt, cudaStream_t st) {
  MTTS_REQUIRE(x && planes_base && C % 4 == 0 && ldx % 4 == 0 && x_sb % 4 == 0 && ((((uintptr_t)x) & 15) == 0), "bad arguments");
  if (B <= 0 || T <= 0) return 0;
  __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>((((uintptr_t)planes_base) + 1023) & ~(uintptr_t)1023);
  const int Tp = T + hl + hr;
  const int64_t total4 = (int64_t)B * Tp * C / 4;
  launch_k(split_pad_kernel, (unsigned)cdiv64(total4, 256), 256, 0, st, x, x_sb, ldx, T, C, hl, Tp, pad_mode, act, slope, planes,
           (int64_t)B * Tp * C, total4, fmt, tc_ovf_ptr());
  MTTS_CHECK_LAUNCH();
  return 0;
}

// fp32 (rows, C) -> operand planes (3 | 2 | 1, rows, C): the activation split, exposed for packing weights on the device
int split_planes(const float* x, int ldx, int64_t rows, int C, void* planes, int fmt, cudaStream_t st) {
  MTTS_REQUIRE(x && planes && C > 0 && C % 4 == 0 && ldx % 4 == 0 && ((((uintptr_t)x) | ((uintptr_t)planes)) & 15) == 0, "bad arguments");
  MTTS_REQUIRE(fmt == MTTS_TC_BF16X3 || fmt == MTTS_TC_F16X2 || fmt == MTTS_TC_F16, "unknown operand format");
  if (rows <= 0) return 0;
  MTTS_REQUIRE(rows < (int64_t)1 << 31, "too many rows");
  const int64_t total4 = rows * C / 4;
  launch_k(split_pad_kernel, (unsigned)cdiv64(total4, 256), 256, 0, st, x, 0, ldx, (int)rows, C, 0, (int)rows, MTTS_PAD_ZERO, MTTS_ACT_NONE, 0.f,
                                                                 reinterpret_cast<__nv_bfloat16*>(planes), rows * (int64_t)C, total4,
                                                                 fmt, tc_ovf_ptr());
  MTTS_CHECK_LAUNCH();
  return 0;
}

// nn.Linear on the tensor-core engine = the k = 1 case of the tap-GEMM
int64_t linear_tc_scratch_bytes(int64_t rows_cap, int K) { return 3 * rows_cap * (int64_t)K * 2 + 4096; }

int linear_tc(const float* x, int ldx, int64_t M, int K, const void* w_planes, int N, const float* bias,
              const float* res, int ldr, float* y, int ldy, int pre_act, float pre_slope, int post_act,
              float out_scale, void* scratch, int64_t scratch_bytes, int64_t rows_cap, int fmt, cudaStream_t st) {
  MTTS_REQUIRE(x && w_planes && y && scratch, "null pointer");
  mtts_conv_params p = linear_params(x, ldx, nullptr, bias, y, ldy, M, K, N);
  p.w = reinterpret_cast<const float*>(w_planes);     // unused on this path (non-null for validation only)
  p.res = res; p.ldr = ldr; p.pre_act = pre_act; p.pre_slope = pre_slope; p.post_act = post_act; p.out_scale = out_scale;
  p.w_tc = w_planes; p.tc_scratch = scratch; p.tc_scratch_bytes = scratch_bytes; p.tc_rows_cap = rows_cap; p.tc_fmt = fmt;
  if (!conv_tc_eligible(p))
    return fail(MTTS_ERR_UNSUPPORTED, "%s: shape not eligible for the tensor-core engine (M=%lld N=%lld)", "linear_tc", M, N);
  return conv_tc(p, st);
}

}  // namespace mtts
