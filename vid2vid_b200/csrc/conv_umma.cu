// Implicit-GEMM convolution on Hopper tensor cores (sm_90a wgmma), persistent and warp-specialised.
//
//   D[128 pixels x BN channels] (fp32, registers) = sum over (tap, K block of kc = 16/32/64 channels) A[128 x kc] * B[BN x kc]^T
//
// A tiles are boxes of the halo-padded NHWC bf16 activation buffer fetched by TMA (5-D tiled map,
// 128-byte swizzle): a box of TH x TW pixels x 64 channels lands in shared memory as 128 rows of
// 128 bytes -- exactly the K-major SWIZZLE_128B operand layout wgmma reads.  That box *is*
// the im2col slice for one filter tap; for stride-1 filters on row tiles (TH == 1) one box of
// TW + R - 1 pixels serves R horizontally adjacent taps, each tap's operand being the same smem
// patch with its start address advanced by one 128-byte row.  B tiles come from the packed weight
// matrix [Cout][tap * Cp + c] (2-D tiled map); when all B tiles of one (phase, N tile) fit in shared
// memory they are loaded once and stay resident while the CTA walks its M tiles.
// Reference op being replaced: nn.Conv2d / nn.ConvTranspose2d (+ ReflectionPad2d) at
// models/networks.py:132-183,247-279,571,586,685-706.
//
// One CTA per SM walks tiles t = blockIdx.x, += gridDim.x (M fastest, so co-running CTAs share weights in L2).
//   warps 0-7   two consumer warpgroups: warpgroup h issues the m64nBNk16 wgmmas of rows [64 h, 64 h + 64) of every M tile
//               (MG tiles side by side, accumulators in registers), keeping one commit group in flight and handing each
//               operand slot back to the producer as soon as the MMAs that read it have retired.  Both then drain the
//               accumulators through a 128 x 64 fp32 shared-memory staging tile, so that in the epilogue thread
//               (warp q = 0..3, lane) owns pixel row 32 q + lane and warps q / q + 4 take alternate 32-channel chunks:
//     EPI_RAW_STATS : bf16 NHWC raw output + per-channel (sum, sumsq) of the tile for the following
//                     Batch/InstanceNorm (deterministic fixed-point atomics)
//     EPI_HEAD_F32  : bias + tanh/sigmoid/scale -> fp32 NCHW planes (the 7x7 image/flow/weight heads)
//     EPI_ACT_BF16  : bias + (leaky)ReLU -> interior of the next layer's padded NHWC buffer
//   warp 8      TMA producer (one elected lane)
#include <cstdlib>
#include "ptx.cuh"
#include "wgmma.cuh"
#include "v2v_internal.h"
#include "finalize.cuh"

namespace v2v {

static constexpr int kConsumerThreads = 256;              // two warpgroups
static constexpr int kThreads = kConsumerThreads + 32;    // + the producer warp
static constexpr int kStgStride = 65;                     // floats per staging row: row-wise and column-wise walks are conflict free
static constexpr int kStgFloats = 128 * kStgStride;       // 128 pixel rows x 64 accumulator columns
static constexpr int kRedFloats = 4 * 2 * 128;            // [warp quarter][sum|sumsq][128 columns] running column sums

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_LRELU: return v > 0.f ? v : v * slope;
    case ACT_TANH: return tanhf(v);
    case ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    default: return v;
  }
}

// kx-GEMM heads: acc[j] = sum_kx (value of accumulator column kx * COUT + j held by lane + kx)
template <int COUT>
__device__ __forceinline__ void head_shift_sum(const uint32_t (&r)[32], int kw, float (&acc)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j] = 0.f;
#pragma unroll
  for (int kx = 0; kx < 8; ++kx) {
    if (kx * COUT + COUT <= 32) {
#pragma unroll
      for (int j = 0; j < COUT; ++j) {
        const float v = __shfl_down_sync(0xffffffffu, __uint_as_float(r[kx * COUT + j]), kx);
        if (kx < kw) acc[j] += v;
      }
    }
  }
}

// Work units (MG consecutive M tiles of one tile row, of one (phase, N tile) "key"; M fastest) are walked by every role as u = first, first + step, ...
// The iterator keeps (key, N tile, phase, image, tile row, tile column) as a mixed-radix number and advances it by the
// pre-split step with carries, so the integer divisions (~150 cycles of dependent SASS each) happen once per kernel
// instead of once per unit on the issuing threads.
struct UnitIter {
  int u, key, nt, phase, img, ty, txi;
  int s_img, s_ty, s_tx, step;
  __device__ __forceinline__ void init(const ConvKernelParams& p, int first, int step_) {
    const int txu = p.tiles_x / p.MG;                   // units per tile row (MG consecutive x tiles share a weight pass)
    const int per_img = txu * p.tiles_y;
    u = first; step = step_;
    key = first / p.m_total;
    const int m = first - key * p.m_total;
    phase = key / p.n_tiles; nt = key - phase * p.n_tiles;
    img = m / per_img;
    const int r = m - img * per_img;
    ty = r / txu; txi = r - ty * txu;
    s_tx = step_ % txu;
    const int q = step_ / txu;
    s_ty = q % p.tiles_y; s_img = q / p.tiles_y;
  }
  __device__ __forceinline__ bool valid(const ConvKernelParams& p) const { return u < p.total_units; }
  __device__ __forceinline__ void next(const ConvKernelParams& p) {
    u += step;
    const int txu = p.tiles_x / p.MG;
    txi += s_tx; if (txi >= txu) { txi -= txu; ++ty; }
    ty += s_ty;  if (ty >= p.tiles_y) { ty -= p.tiles_y; ++img; }
    img += s_img;
    while (img >= p.N) { img -= p.N; ++key; if (++nt == p.n_tiles) { nt = 0; ++phase; } }
  }
  __device__ __forceinline__ int n0(const ConvKernelParams& p) const { return nt * p.BN; }
  __device__ __forceinline__ int x0(const ConvKernelParams& p) const { return txi * p.MG * p.tile_dx; }   // first tile of the unit
  __device__ __forceinline__ int y0(const ConvKernelParams& p) const { return ty * p.TH; }
};


// All MMAs of one (tap, K block) for the MG accumulators: KMMA K=16 steps x the operand passes of the arithmetic mode
// (precise plans: A_hi*B_hi + A_lo*B_hi + A_hi*B_lo, the lo halves a_half / b_half bytes further in the same slots).
template <int BN, int MG>
__device__ __forceinline__ void mma_tap(float (&acc)[MG][BN / 2], uint64_t ad, uint64_t bd, uint32_t a_tile16, int kmma, int ps_step,
                                        uint32_t a_half16, uint32_t b_half16, uint32_t first) {
#pragma unroll
  for (int j = 0; j < MG; ++j) {
    uint32_t f = first;
    for (int ps = 0; ps < 3; ps += ps_step) {
      const uint64_t a = ad + (uint64_t)j * a_tile16 + (ps == 1 ? a_half16 : 0u), b = bd + (ps == 2 ? b_half16 : 0u);
      for (int k = 0; k < kmma; ++k) {
        Wgmma<BN>::template mma<0, 0>(acc[j], a + 2 * k, b + 2 * k, f);      // +32 bytes along K per MMA
        f = 1u;
      }
    }
  }
}

template <int BN, int MG>
__global__ void __launch_bounds__(kThreads, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ ConvKernelParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // group slots: [SG][ CG activation patches | CG streamed weight slots ], then the resident weight set (if any)
  // ring2: [SG patch slots of MG tiles][SBr weight slots]
  const int slot_b = (p.b_resident || p.ring2) ? 0 : p.b_slot_bytes;
  const int group_bytes = p.CG * (p.MG * p.a_slot_bytes + slot_b);
  uint8_t* sG = smem;
  uint8_t* sBres = sG + (size_t)p.SG * group_bytes;
  float* stg = reinterpret_cast<float*>(sBres + (p.ring2 ? (size_t)p.SBr * p.b_slot_bytes : (p.b_resident ? (size_t)p.SB * p.b_slot_bytes : 0)));
  float* racc = stg + kStgFloats;
  uint64_t* bars = reinterpret_cast<uint64_t*>(racc + kRedFloats);
  uint64_t* g_full = bars;
  uint64_t* g_empty = g_full + p.SG;
  uint64_t* bres_full = g_empty + p.SG;
  uint64_t* bres_empty = bres_full + 1;
  uint64_t* b_full = bres_empty + 1;        // ring2: weight ring barriers [8] + [8]
  uint64_t* b_empty = b_full + 8;
  uint32_t* ticket = reinterpret_cast<uint32_t*>(b_empty + 8);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // (warp-uniform to the compiler)
  const int n_consumer_warps = kConsumerThreads / 32;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < p.SG; ++i) { mbar_init(&g_full[i], 1); mbar_init(&g_empty[i], n_consumer_warps); }
    mbar_init(bres_full, 1); mbar_init(bres_empty, n_consumer_warps);
    if (p.ring2) for (int i = 0; i < p.SBr; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], n_consumer_warps); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue();          // everything above overlaps the previous kernel's tail; nothing above touches global memory

  const int a_tx = p.PW * p.PH * p.row_bytes;
  const int b_tx = p.BN * p.row_bytes;
  const int t_first = blockIdx.x, t_step = gridDim.x;

  if (warp == n_consumer_warps) {
    if (elect_one_sync()) {
      // ---------------------------------------------------------- TMA producer (single elected lane)
      // The K loop of a tile is a sequence of steps (tap group g, K block cb); CG consecutive steps share one
      // full/empty barrier pair ("group slot"), so a barrier round trip and a wgmma commit group are paid once per CG
      // steps.
      int gs = 0;
      uint32_t gpar = 0, gen = 0;
      int prev_key = -1;
      const int nhalf = p.split ? 2 : 1;                       // weight halves
      const int nhalfA = (p.split && !p.a_exact) ? 2 : 1;      // activation halves (an exact-in-bf16 input has no lo half)
      UnitIter un;
      un.init(p, t_first, t_step);
      if (p.ring2) {
        int as = 0, bs = 0;
        uint32_t apar = 0, bpar = 0;
        for (; un.valid(p); un.next(p)) {
          const ConvPhase ph = p.phases[un.phase];
          const int x0 = un.x0(p), y0 = un.y0(p), n0 = un.n0(p);
          for (int g = ph.group_begin; g < ph.group_end; ++g) {
            const ConvGroup grp = p.groups[g];
            for (int cb = 0; cb < p.cblocks; ++cb) {
              uint8_t* abase = sG + (size_t)as * p.MG * p.a_slot_bytes;
              mbar_wait(&g_empty[as], apar ^ 1);
              mbar_expect_tx(&g_full[as], (uint32_t)(nhalfA * p.MG * a_tx));
              for (int j = 0; j < p.MG; ++j)
                for (int hf = 0; hf < nhalfA; ++hf)
                  tma_load_5d(abase + (size_t)j * p.a_slot_bytes + (size_t)hf * p.a_half_bytes, &tmA, &g_full[as], hf * p.Cp + cb * p.kc,
                              x0 + j * p.TW + grp.dx, y0 + grp.dy, grp.plane, un.img);
              if (++as == p.SG) { as = 0; apar ^= 1; }
              for (int t0 = 0; t0 < p.R; t0 += p.TB) {
                uint8_t* bbase = sBres + (size_t)bs * p.b_slot_bytes;
                const int nt = min(p.TB, p.R - t0);
                mbar_wait(&b_empty[bs], bpar ^ 1);
                mbar_expect_tx(&b_full[bs], (uint32_t)(nhalf * nt * b_tx));
                for (int hf = 0; hf < nhalf; ++hf)
                  for (int t = 0; t < nt; ++t)
                    tma_load_2d(bbase + (size_t)hf * p.b_half_bytes + (size_t)t * b_tx, &tmB, &b_full[bs],
                                hf * p.Khalf + (grp.tap0 + t0 + t) * p.Cp + cb * p.kc, n0);
                if (++bs == p.SBr) { bs = 0; bpar ^= 1; }
              }
            }
          }
        }
      } else
      for (; un.valid(p); un.next(p)) {
        const ConvPhase ph = p.phases[un.phase];
        const int x0 = un.x0(p), y0 = un.y0(p), n0 = un.n0(p);
        const int nsteps = (ph.group_end - ph.group_begin) * p.cblocks;
        if (p.b_resident && un.key != prev_key) {
          if (prev_key >= 0) gen ^= 1;
          mbar_wait(bres_empty, gen ^ 1);                      // all MMAs that read the previous weight set retired
          mbar_expect_tx(bres_full, (uint32_t)nsteps * p.R * b_tx * nhalf);
          int sidx = 0;
          for (int g = ph.group_begin; g < ph.group_end; ++g)
            for (int cb = 0; cb < p.cblocks; ++cb, ++sidx)
              for (int hf = 0; hf < nhalf; ++hf)
                for (int r = 0; r < p.R; ++r)
                  tma_load_2d(sBres + (size_t)sidx * p.b_slot_bytes + (size_t)hf * p.b_half_bytes + (size_t)r * b_tx, &tmB,
                              bres_full, hf * p.Khalf + (p.groups[g].tap0 + r) * p.Cp + cb * p.kc, n0);
        }
        prev_key = un.key;
        int g = ph.group_begin, cb = 0;
        for (int s0 = 0; s0 < nsteps; s0 += p.CG) {
          const int n = min(p.CG, nsteps - s0);
          uint8_t* base = sG + (size_t)gs * group_bytes;
          mbar_wait(&g_empty[gs], gpar ^ 1);
          mbar_expect_tx(&g_full[gs], (uint32_t)n * (nhalfA * p.MG * a_tx + (p.b_resident ? 0 : nhalf * p.R * b_tx)));
          for (int i = 0; i < n; ++i) {
            const ConvGroup grp = p.groups[g];
            for (int j = 0; j < p.MG; ++j)
              for (int hf = 0; hf < nhalfA; ++hf)     // lo half: channels [Cp, 2 Cp) of the pixel
                tma_load_5d(base + (size_t)(i * p.MG + j) * p.a_slot_bytes + (size_t)hf * p.a_half_bytes, &tmA, &g_full[gs],
                            hf * p.Cp + cb * p.kc, x0 + j * p.TW + grp.dx, y0 + grp.dy, grp.plane, un.img);
            if (!p.b_resident) {
              uint8_t* bb = base + (size_t)p.CG * p.MG * p.a_slot_bytes + (size_t)i * p.b_slot_bytes;
              for (int hf = 0; hf < nhalf; ++hf)
                for (int r = 0; r < p.R; ++r)
                  tma_load_2d(bb + (size_t)hf * p.b_half_bytes + (size_t)r * b_tx, &tmB, &g_full[gs],
                              hf * p.Khalf + (grp.tap0 + r) * p.Cp + cb * p.kc, n0);
            }
            if (++cb == p.cblocks) { cb = 0; ++g; }
          }
          if (++gs == p.SG) { gs = 0; gpar ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: wgmma issue + epilogue
    const int wg = warp >> 2;                             // M half of the tile this warpgroup multiplies
    const int q = warp & 3, hc = wg;                      // epilogue: pixel rows 32 q .. 32 q + 31, chunk parity hc
    const int row = q * 32 + lane;
    const int ps_step = p.split ? (p.a_exact ? 2 : 1) : 3;    // 3 = one pass (fast), 1 = three passes, 2 = {hi*hi, hi*lo}
    const uint32_t a_half16 = (uint32_t)(p.a_half_bytes >> 4), b_half16 = (uint32_t)(p.b_half_bytes >> 4);
    const uint32_t a_tile16 = (uint32_t)(p.a_slot_bytes >> 4);
    // rows 64.. of an M tile are eight 8-row core-matrix groups further on
    const uint64_t a_d0 = make_kmajor_desc(0, p.sbo_a_bytes, p.layout_type) + (uint64_t)((wg * 8 * p.sbo_a_bytes) >> 4);
    const uint64_t b_d0 = make_kmajor_desc(0, p.sbo_bytes, p.layout_type);
    // tap r of a patch: next pixel (horizontal reuse) or, for kx-GEMM heads, next patch ROW (TW pixels further)
    const uint32_t a_step = (uint32_t)(((p.headkx ? p.TW : 1) * p.row_bytes) >> 4), b_step = (uint32_t)(b_tx >> 4);
    const uint32_t a_wrap = (uint32_t)(((p.PW - p.RW) * p.row_bytes) >> 4);     // to the next patch row
    const uint32_t row16 = (uint32_t)(p.row_bytes >> 4), prow16 = (uint32_t)((p.PW * p.row_bytes) >> 4);
    const uint32_t sB_u32 = smem_u32(sBres);
    const bool do_stats = (p.epi == EPI_RAW_STATS) && (p.stats != nullptr) && !(p.dbg & 1);
    const int nchunks = p.BN / 32;
    const int tw_shift = __ffs(p.TW) - 1;                 // TW is a power of two
    const int ry = row >> tw_shift, rx = row & (p.TW - 1);

    float acc[MG][BN / 2];
    // Operand slots retire one commit group late: after committing group k the warpgroup waits for group k - 1 only, so
    // the tensor core always has the next group queued.  Each warp then arrives once on the slot barriers (count 8).
    int pend_g = -1, pend_b = -1;
    auto retire = [&](int g, int b) {
      __syncwarp();
      mbar_arrive_if(&g_empty[g < 0 ? 0 : g], lane == 0 && g >= 0);
      mbar_arrive_if(&b_empty[b < 0 ? 0 : b], lane == 0 && b >= 0);
    };
    auto commit_and_retire_previous = [&](int g, int b) {
      wgmma_commit();
      wgmma_wait<1>();
      retire(pend_g, pend_b);
      pend_g = g; pend_b = b;
    };
    auto drain = [&]() {
      wgmma_wait<0>();
      retire(pend_g, pend_b);
      pend_g = pend_b = -1;
#pragma unroll
      for (int j = 0; j < MG; ++j) wgmma_fence_operands(acc[j]);
    };
    // Statistics: running (sum, sumsq) per (warp quarter, column of the current N tile) in shared memory, flushed onto the
    // image's statistics row when (phase, N tile, image) changes.  Every (quarter, column) has one writer warp.
    int acc_key = -1, acc_img = -1, acc_n0 = 0;
    // flush() publishes the running sums and zeroes them again: thread c owns column c of every quarter.
    auto flush = [&]() {
      named_bar_sync(1, kConsumerThreads);                // every warp has added its last tile
      const int etid = threadIdx.x;
      if (etid < p.BN) {
        float s = 0.f, qq = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          s += racc[(w * 2 + 0) * 128 + etid];
          qq += racc[(w * 2 + 1) * 128 + etid];
          racc[(w * 2 + 0) * 128 + etid] = 0.f;
          racc[(w * 2 + 1) * 128 + etid] = 0.f;
        }
        // 64-bit fixed-point integer atomics onto the image's single statistics row: order independent (deterministic)
        if (acc_n0 + etid < p.stats_C) {
          atomicAdd(&p.stats[((size_t)acc_img * 2 + 0) * p.stats_C + acc_n0 + etid], (stat_t)__float2ll_rn(s * V2V_STAT_SUM_SCALE));
          atomicAdd(&p.stats[((size_t)acc_img * 2 + 1) * p.stats_C + acc_n0 + etid], (stat_t)__float2ll_rn(qq * V2V_STAT_SQ_SCALE));
        }
      }
      named_bar_sync(1, kConsumerThreads);                // every column is zero again
    };
    for (int i = threadIdx.x; i < kRedFloats; i += kConsumerThreads) racc[i] = 0.f;    // (ordered by the first stage())
    // accumulator columns [c0, c0 + 64) of tile jt -> staging rows (the wgmma fragment layout, see wgmma.cuh)
    auto stage = [&](int jt, int c0) {
#pragma unroll
      for (int j = 0; j < MG; ++j) {
        if (j != jt) continue;
#pragma unroll
        for (int b = 0; b < BN / 8; ++b) {
          if (b * 8 < c0 || b * 8 >= c0 + 64) continue;
          const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), col = b * 8 + 2 * (lane & 3) - c0;
          stg[r0 * kStgStride + col] = acc[j][b * 4 + 0];
          stg[r0 * kStgStride + col + 1] = acc[j][b * 4 + 1];
          stg[(r0 + 8) * kStgStride + col] = acc[j][b * 4 + 2];
          stg[(r0 + 8) * kStgStride + col + 1] = acc[j][b * 4 + 3];
        }
      }
      named_bar_sync(1, kConsumerThreads);
    };

    int gs = 0, as = 0, bs = 0;
    uint32_t gpar = 0, gen = 0, apar = 0, bpar = 0;
    int prev_key = -1;
    UnitIter un;
    un.init(p, t_first, t_step);
    for (; un.valid(p);) {
      const ConvPhase ph = p.phases[un.phase];
      const int key = un.key;
      const bool first_of_key = key != prev_key;
      if (p.b_resident && first_of_key && prev_key >= 0) gen ^= 1;
      prev_key = key;
      // everything the epilogue needs from the iterator, captured before it advances
      const int y0 = un.y0(p), x0 = un.x0(p), n0 = un.n0(p), n_img = un.img;
      un.next(p);
      const bool last_of_key = !un.valid(p) || un.key != key;
      const int nsteps = (ph.group_end - ph.group_begin) * p.cblocks;

      // ---------------- MMAs
      if (p.b_resident && first_of_key) mbar_wait_converged(bres_full, gen);
#pragma unroll
      for (int j = 0; j < MG; ++j) wgmma_fence_operands(acc[j]);
      wgmma_fence();
      uint32_t first = 0;
      if (p.ring2) {
        // K loop: steps (tap group, K block); per step ONE patch slot (MG tiles) from the A ring and ceil(R / TB) weight
        // chunks from the B ring; tap r of the step reads the patch advanced by (r / RW) * PW + (r % RW) rows.
        const int RH = p.R / p.RW;
        for (int st = 0; st < nsteps; ++st) {
          mbar_wait_converged(&g_full[as], apar);
          const uint32_t a_base16 = (smem_u32(sG + (size_t)as * p.MG * p.a_slot_bytes) & 0x3FFFF) >> 4;
          uint32_t bchunk16 = 0;
          int tin = 0, r = 0;
          for (int ky = 0; ky < RH; ++ky) {
            for (int kx = 0; kx < p.RW; ++kx, ++r) {
              if (tin == 0) {
                mbar_wait_converged(&b_full[bs], bpar);
                bchunk16 = ((sB_u32 + (uint32_t)bs * (uint32_t)p.b_slot_bytes) & 0x3FFFF) >> 4;
              }
              mma_tap<BN, MG>(acc, a_d0 + a_base16 + (uint32_t)ky * prow16 + (uint32_t)kx * row16, b_d0 + bchunk16 + (uint32_t)tin * b_step,
                              a_tile16, p.kmma, ps_step, a_half16, b_half16, first);
              first = 1u;
              if (++tin == p.TB || r == p.R - 1) {             // chunks hold TB taps; the last one of a step may be short
                tin = 0;
                commit_and_retire_previous(r == p.R - 1 ? as : -1, bs);      // the patch slot retires with the step's last chunk
                if (++bs == p.SBr) { bs = 0; bpar ^= 1; }
                wgmma_fence();
              }
            }
          }
          if (++as == p.SG) { as = 0; apar ^= 1; }
        }
      } else {
        for (int s0 = 0; s0 < nsteps; s0 += p.CG) {
          const int n = min(p.CG, nsteps - s0);
          mbar_wait_converged(&g_full[gs], gpar);
          const uint32_t base = smem_u32(sG + (size_t)gs * group_bytes);
          for (int i = 0; i < n; ++i) {
            const uint32_t b_base = p.b_resident ? sB_u32 + (s0 + i) * p.b_slot_bytes
                                                 : base + p.CG * p.MG * p.a_slot_bytes + i * p.b_slot_bytes;
            const uint32_t a_base = base + i * p.MG * p.a_slot_bytes;
            uint32_t al = (a_base & 0x3FFFF) >> 4, bl = (b_base & 0x3FFFF) >> 4;
            // tap r reads the patch shifted by (r / RW) patch rows and (r % RW) pixels
            for (int r0 = 0; r0 < p.R; r0 += p.RW, al += a_wrap) {
              for (int r = 0; r < p.RW; ++r, al += a_step, bl += b_step) {
                mma_tap<BN, MG>(acc, a_d0 + al, b_d0 + bl, a_tile16, p.kmma, ps_step, a_half16, b_half16, first);
                first = 1u;
              }
            }
          }
          commit_and_retire_previous(gs, -1);              // the whole group slot retires with these MMAs
          if (++gs == p.SG) { gs = 0; gpar ^= 1; }
          wgmma_fence();
        }
      }
      drain();
      __syncwarp();
      mbar_arrive_if(bres_empty, lane == 0 && p.b_resident && last_of_key);

      // ---------------- epilogue
      const int gy = y0 + ry, gx0 = x0 + rx;
      const int oy = gy * p.oy_mul + ph.oy_add;
#pragma unroll
      for (int jt = 0; jt < MG; ++jt) {                   // the unit's MG tiles sit side by side along x
        const int gx = gx0 + jt * p.TW;
        const bool valid = (gy < p.grid_h) && (gx < p.grid_w);
        const int ox = gx * p.ox_mul + ph.ox_add;
        bf16* dst = nullptr;
        float* dstf = nullptr;
        if (valid && p.epi != EPI_HEAD_F32) {
          const size_t pix_off = (((size_t)n_img * p.out_H + oy) * p.out_W + ox) * p.out_C;
          if (p.epi == EPI_RAW_STATS) {
            if (p.out_f32) dstf = reinterpret_cast<float*>(p.out) + pix_off;
            else dst = reinterpret_cast<bf16*>(p.out) + pix_off;
          } else {
            dst = p.out_act.base + p.out_act.offset(n_img, oy, ox);
          }
        }
        const float* srow = stg + row * kStgStride;

        if (p.epi == EPI_HEAD_F32 && p.headkx) {
          // kx-GEMM head.  Tile = 4 rows x 32 INPUT pixels: warp quarter q = tile row, lane = pixel, accumulator column
          // kx * Cout + c.  out(x)[c] = sum_kx D[x + kx][kx * Cout + c] is a sum over the NEXT kw - 1 lanes of the same
          // warp: warp shuffles.  Lanes 32 - (kw - 1) .. 31 only feed their left neighbours (tiles advance by
          // tile_dx = 32 - (kw - 1) pixels).
          stage(jt, 0);
          if (hc == 0) {
            uint32_t r[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(srow[j]);
            float hacc[4];
            switch (p.Cout) {
              case 1: head_shift_sum<1>(r, p.headkx, hacc); break;
              case 2: head_shift_sum<2>(r, p.headkx, hacc); break;
              case 3: head_shift_sum<3>(r, p.headkx, hacc); break;
              default: head_shift_sum<4>(r, p.headkx, hacc); break;
            }
            if (valid && rx < p.tile_dx) {
              const size_t pix = (size_t)oy * p.out_W + ox;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (j < p.Cout) {
                  float v = hacc[j];
                  if (p.bias) v += (p.bias2 && j >= p.Cout1) ? __ldg(p.bias2 + j - p.Cout1) : __ldg(p.bias + j);
                  v = apply_act(v, p.head_act[j], p.lrelu_slope) * p.head_scale[j];
                  reinterpret_cast<float*>(p.io[p.head_slot[j]])[p.head_off[j] + (size_t)n_img * p.head_bstride[j] + pix] = v;
                }
              }
            }
          }
          named_bar_sync(1, kConsumerThreads);
          continue;
        }
        if (p.epi == EPI_HEAD_F32) {
          stage(jt, 0);
          if (hc == 0 && valid) {
            const size_t pix = (size_t)oy * p.out_W + ox;
#pragma unroll
            for (int j = 0; j < V2V_MAX_HEAD; ++j) {
              if (j < p.Cout) {
                float v = srow[j];
                if (p.bias) v += (p.bias2 && j >= p.Cout1) ? __ldg(p.bias2 + j - p.Cout1) : __ldg(p.bias + j);
                v = apply_act(v, p.head_act[j], p.lrelu_slope) * p.head_scale[j];
                reinterpret_cast<float*>(p.io[p.head_slot[j]])[p.head_off[j] + (size_t)n_img * p.head_bstride[j] + pix] = v;
              }
            }
          }
          named_bar_sync(1, kConsumerThreads);
          continue;
        }

        if (do_stats && (key != acc_key || n_img != acc_img)) {
          if (acc_key >= 0) flush();
          acc_key = key; acc_img = n_img; acc_n0 = n0;
        }
        for (int c0 = 0; c0 < nchunks; c0 += 2) {
          stage(jt, c0 * 32);
          const int c = c0 + hc;
          if (c < nchunks) {
            float v[32];
            const int col0 = n0 + c * 32;
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = valid ? srow[hc * 32 + j] : 0.f;
            if (p.epi == EPI_ACT_BF16) {
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                float b = (p.bias && col0 + j < p.Cout) ? __ldg(p.bias + col0 + j) : 0.f;
                v[j] = (col0 + j < p.Cout) ? apply_act(v[j] + b, p.act, p.lrelu_slope) : 0.f;
              }
            }
            if (valid && !(p.dbg & 2)) {
              if (dstf) {                                // precise plan: fp32 raw output
#pragma unroll
                for (int qv = 0; qv < 8; ++qv)
                  if (col0 + qv * 4 < p.out_C)
                    *reinterpret_cast<float4*>(dstf + col0 + qv * 4) = make_float4(v[qv * 4], v[qv * 4 + 1], v[qv * 4 + 2], v[qv * 4 + 3]);
              } else if (p.epi == EPI_ACT_BF16 && p.out_act.split) {
#pragma unroll
                for (int qv = 0; qv < 4; ++qv) {
                  if (col0 + qv * 8 < p.out_C) {
                    float lo[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) lo[j] = v[qv * 8 + j] - __bfloat162float(__float2bfloat16_rn(v[qv * 8 + j]));
                    uint4 pk, pl;
                    pk.x = pack_bf16x2(v[qv * 8 + 0], v[qv * 8 + 1]); pl.x = pack_bf16x2(lo[0], lo[1]);
                    pk.y = pack_bf16x2(v[qv * 8 + 2], v[qv * 8 + 3]); pl.y = pack_bf16x2(lo[2], lo[3]);
                    pk.z = pack_bf16x2(v[qv * 8 + 4], v[qv * 8 + 5]); pl.z = pack_bf16x2(lo[4], lo[5]);
                    pk.w = pack_bf16x2(v[qv * 8 + 6], v[qv * 8 + 7]); pl.w = pack_bf16x2(lo[6], lo[7]);
                    *reinterpret_cast<uint4*>(dst + col0 + qv * 8) = pk;
                    *reinterpret_cast<uint4*>(dst + p.out_act.C + col0 + qv * 8) = pl;
                  }
                }
              } else {
#pragma unroll
                for (int qv = 0; qv < 4; ++qv) {
                  if (col0 + qv * 8 < p.out_C) {
                    uint4 pk;
                    pk.x = pack_bf16x2(v[qv * 8 + 0], v[qv * 8 + 1]);
                    pk.y = pack_bf16x2(v[qv * 8 + 2], v[qv * 8 + 3]);
                    pk.z = pack_bf16x2(v[qv * 8 + 4], v[qv * 8 + 5]);
                    pk.w = pack_bf16x2(v[qv * 8 + 6], v[qv * 8 + 7]);
                    *reinterpret_cast<uint4*>(dst + col0 + qv * 8) = pk;
                  }
                }
              }
            }
            if (do_stats) {
              // column sums over this warp's 32 rows: each lane writes its (masked) row back into the staging tile, then
              // lane l walks column l down the 32 rows (banks (r + l) mod 32: conflict free)
              float* sw = stg + hc * 32;
#pragma unroll
              for (int j = 0; j < 32; ++j) sw[row * kStgStride + j] = v[j];
              __syncwarp();
              float s = 0.f, qq = 0.f;
#pragma unroll
              for (int r2 = 0; r2 < 32; ++r2) {
                const float x = sw[(q * 32 + r2) * kStgStride + lane];
                s += x;
                qq = fmaf(x, x, qq);
              }
              racc[(q * 2 + 0) * 128 + c * 32 + lane] += s;
              racc[(q * 2 + 1) * 128 + c * 32 + lane] += qq;
            }
          }
          named_bar_sync(1, kConsumerThreads);             // the staging tile may be overwritten
        }
      }
    }
    if (do_stats && acc_key >= 0) flush();
  }

  __threadfence();                                  // this thread's statistics atomics are visible device-wide
  __syncthreads();
  if (p.n_fin > 0) {
    // Statistics finalisation by the LAST CTA to get here (ticket counter, zeroed with the statistics rows before every run):
    // all rows are complete then; every other CTA has exited, nobody waits.
    if (threadIdx.x == 0) *ticket = atomicAdd(p.fin_counter, 1u);
    __syncthreads();
    if (*ticket == gridDim.x - 1) {
      __threadfence();
      for (int f = 0; f < p.n_fin; ++f)
        for (int c = threadIdx.x; c < p.fin[f].C; c += blockDim.x) channel_side_effects(p.fin[f], c);
    }
  }
}

bool pdl_enabled() {
  // opt-in (V2V_PDL=1): the early-launched blocks of the elementwise kernels sit in griddepcontrol.wait holding thread slots
  // the persistent conv CTAs then wait for
  static const bool on = [] { const char* e = getenv("V2V_PDL"); return e && e[0] == '1'; }();
  return on;
}

int device_sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, int MG>
static cudaError_t launch_bn_mg(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvKernelParams& p, size_t smem, cudaStream_t stream) {
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(conv_umma_kernel<BN, MG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = smem;
  }
  return launch_pdl(conv_umma_kernel<BN, MG>, dim3(p.grid), dim3(kThreads), smem, stream, tmA, tmB, p);
}

size_t conv_umma_smem_bytes(const ConvKernelParams& p) {
  const size_t operands = p.ring2 ? (size_t)p.SG * p.MG * p.a_slot_bytes + (size_t)p.SBr * p.b_slot_bytes
                                  : (size_t)p.SG * p.CG * ((size_t)p.MG * p.a_slot_bytes + (p.b_resident ? 0 : p.b_slot_bytes)) +
                                        (p.b_resident ? (size_t)p.SB * p.b_slot_bytes : 0);
  return operands + 1024 /*align*/ + (size_t)(kStgFloats + kRedFloats) * sizeof(float) + (2 * p.SG + 2 + 16 + 1) * sizeof(uint64_t);
}

cudaError_t launch_conv_umma(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvKernelParams& p,
                             cudaStream_t stream) {
  const size_t smem = conv_umma_smem_bytes(p);
  // the N tile and the M blocking fix the accumulator registers: one instantiation per plan choice (V2V_MAX_ACC_COLS)
  switch (p.BN * 4 + p.MG) {
    case 16 * 4 + 1: return launch_bn_mg<16, 1>(tmA, tmB, p, smem, stream);
    case 32 * 4 + 1: return launch_bn_mg<32, 1>(tmA, tmB, p, smem, stream);
    case 32 * 4 + 2: return launch_bn_mg<32, 2>(tmA, tmB, p, smem, stream);
    case 64 * 4 + 1: return launch_bn_mg<64, 1>(tmA, tmB, p, smem, stream);
    case 64 * 4 + 2: return launch_bn_mg<64, 2>(tmA, tmB, p, smem, stream);
    case 96 * 4 + 1: return launch_bn_mg<96, 1>(tmA, tmB, p, smem, stream);
    case 128 * 4 + 1: return launch_bn_mg<128, 1>(tmA, tmB, p, smem, stream);
    default: return cudaErrorInvalidConfiguration;
  }
}

}  // namespace v2v
