// Weight gradient of a convolution on Hopper tensor cores (sm_90a wgmma): a GEMM whose K dimension is the PIXEL index,
//
//   G[tap][m][n] = sum over grid pixels (img, y, x) of OUT[img][y][x][m] * IN[img][(y, x) @ tap][n]
//
// where OUT is the gradient of the conv output and IN the conv input (train.py:83-90 back-propagates through every
// nn.Conv2d / nn.ConvTranspose2d of models/networks.py; for a transposed conv the roles of "input" and "output gradient"
// swap, see plan_backward.cu).  Both operands are read where the forward pass left them: halo-padded NHWC activation buffers, a
// pixel being [hi C | lo C] bf16.  A TMA box of KP pixels x 64 channels lands in shared memory as KP rows of 128 bytes with
// the 128-byte swizzle -- the canonical *MN-major* SWIZZLE_128B operand layout (64 contiguous M / N elements per K index,
// 8-K groups 1024 bytes apart, 64-element blocks one box apart), so no transposed copy of any tensor is made: the same
// bytes serve the forward conv K-major and this kernel MN-major (wgmma's transpose flags).
//
// One CTA per work unit (tap, M tile of 128 channels of one tensor, N tile of 16 .. 128 channels of the other, K split);
// the K loop walks row segments of KP pixels through a ring of shared-memory stages.
//   warps 0-7  two consumer warpgroups: warpgroup h accumulates rows [64 h, 64 h + 64) of the M tile (its 64-channel A
//              block) in registers; precise plans accumulate OUT_hi*IN_hi + OUT_lo*IN_hi + OUT_hi*IN_lo like the forward
//              kernel.  At the end each thread adds its accumulator fragment to the staging buffer G (vector atomics: the
//              K splits of one (tap, tile) meet there); unstage_wgrad_kernel then adds G into the caller's gradient tensor
//              in the parameter's own layout [M][N][kh][kw].
//   warp 8     TMA producer (one elected lane)
#include <cstdlib>
#include "ptx.cuh"
#include "wgmma.cuh"
#include "v2v_internal.h"
#include "backward.h"

namespace v2v {

static constexpr int kWgConsumers = 256;
static constexpr int kWgThreads = kWgConsumers + 32;

__device__ __forceinline__ uint64_t make_mnmajor_desc(uint32_t smem_addr, int lbo_bytes, int sbo_bytes, int layout_type) {
  // MN-major, swizzled: one K index = one shared-memory row of 128 / 64 / 32 bytes (64 / 32 / 16 contiguous M or N elements,
  // layout type 2 / 4 / 6 as in make_kmajor_desc); SBO = distance between groups of 8 K indices (8 rows), LBO = distance
  // between row-wide blocks
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout_type) << 61;
  return d;
}

template <int BN>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_umma_kernel(const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmIn,
                  const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // A operand (M side, 128 rows of the accumulator): two 64-channel blocks of 128-byte rows.  B operand (N side): Nblocks
  // blocks of b_row bytes per pixel (128: 64 channels; 64 / 32: a 32- / 16-channel tensor in one block).
  const int boxA = p.KP * 128, boxB = p.KP * p.b_row;              // bytes one TMA box delivers
  const int blkA = (boxA + 1023) & ~1023, blkB = (boxB + 1023) & ~1023;      // block strides in shared memory (TMA destinations 1024-byte aligned)
  const int nh = p.split ? 2 : 1;
  const int a_half = 2 * blkA, b_half = p.Nblocks * blkB;
  const int a_bytes = nh * a_half, b_bytes = nh * b_half;
  const int stage_bytes = a_bytes + b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.stages;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // (warp-uniform to the compiler)
  const int n_consumer_warps = kWgConsumers / 32;

  // unit -> (K split, tap, M tile, N tile), tiles fastest: the CTAs running together walk the same pixel range, so every
  // operand row is fetched from HBM once and then served by L2 to the other (tap, tile) units
  int u = blockIdx.x;
  const int nt = u % p.n_tiles; u /= p.n_tiles;
  const int mt = u % p.m_tiles; u /= p.m_tiles;
  const int tap = u % p.ntaps;
  const int ks = u / p.ntaps;
  const int c_begin = ks * p.chunks_per_unit;
  const int c_end = min(p.chunks_total, c_begin + p.chunks_per_unit);
  const int nchunks = c_end - c_begin;                           // >= 1 by construction (launcher)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmOut);
    tma_prefetch_desc(&tmIn);
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], n_consumer_warps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == n_consumer_warps) {
    if (elect_one_sync()) {
      const WgradTap t = p.taps[tap];
      // swap == 0: A = OUT (gradient side, grid pixel itself), B = IN (activation side, shifted by the tap); swap == 1: the
      // other way round (a narrow gradient tensor -- heads, the discriminators' last layer -- sits on the N side)
      const CUtensorMap* tmA = p.swap ? &tmIn : &tmOut;
      const CUtensorMap* tmB = p.swap ? &tmOut : &tmIn;
      const int ax = p.swap ? t.dx : p.out_padl, ay = p.swap ? t.dy : p.out_padt, apl = p.swap ? t.plane : 0;
      const int bx = p.swap ? p.out_padl : t.dx, by = p.swap ? p.out_padt : t.dy, bpl = p.swap ? 0 : t.plane;
      int xs = c_begin % p.xsegs;
      int row = c_begin / p.xsegs;                               // img * gh + y
      int y = row % p.gh, img = row / p.gh;
      int s = 0; uint32_t par = 0;
      for (int c = 0; c < nchunks; ++c) {
        uint8_t* st = smem + (size_t)s * stage_bytes;
        mbar_wait(&empty[s], par ^ 1);
        mbar_expect_tx(&full[s], (uint32_t)(nh * (2 * boxA + p.Nblocks * boxB)));      // (what the boxes deliver, not the padded slots)
        for (int hf = 0; hf < nh; ++hf)
          for (int mb = 0; mb < 2; ++mb) {
            // a 64-channel A tensor fills both halves of the M = 128 tile with the same block (rows 64.. are not stored)
            const int blk = p.Mblocks == 2 ? mt * 2 + mb : mt;
            tma_load_5d(st + (size_t)hf * a_half + (size_t)mb * blkA, tmA, &full[s], hf * p.a_C + blk * 64, xs * p.KP + ax, y + ay, apl, img);
          }
        for (int hf = 0; hf < nh; ++hf)
          for (int nb = 0; nb < p.Nblocks; ++nb)
            tma_load_5d(st + a_bytes + (size_t)hf * b_half + (size_t)nb * blkB, tmB, &full[s], hf * p.b_C + (nt * p.Nblocks + nb) * 64,
                        xs * p.KP + bx, y + by, bpl, img);
        if (++s == p.stages) { s = 0; par ^= 1; }
        if (++xs == p.xsegs) { xs = 0; if (++y == p.gh) { y = 0; ++img; } }
      }
    }
  } else {
    const int wg = warp >> 2;                                     // A block (M half) of this warpgroup
    const bool active = p.Mblocks == 2 || wg == 0;               // a 64-channel A tensor has no second half
    const int ps_step = p.split ? 1 : 3;
    const int b_layout = p.b_row == 128 ? 2 : (p.b_row == 64 ? 4 : 6);
    const int b_kstep = 16 * p.b_row, b_sbo = 8 * p.b_row;        // 16 pixels per MMA = two 8-row groups
    float acc[BN / 2];
    int s = 0; uint32_t par = 0;
    uint32_t first = 0;
    int pend = -1;                                                // stage whose MMAs are still in flight
    for (int c = 0; c < nchunks; ++c) {
      mbar_wait(&full[s], par);
      if (active) {
        wgmma_fence_operands(acc);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem + (size_t)s * stage_bytes) + wg * blkA, b0 = smem_u32(smem + (size_t)s * stage_bytes) + a_bytes;
        for (int ps = 0; ps < 3; ps += ps_step) {
          const uint32_t a = a0 + (ps == 1 ? a_half : 0), b = b0 + (ps == 2 ? b_half : 0);
          for (int k = 0; k < p.kmma; ++k) {
            Wgmma<BN>::template mma<1, 1>(acc, make_mnmajor_desc(a + k * 2048, blkA, 1024, 2), make_mnmajor_desc(b + k * b_kstep, blkB, b_sbo, b_layout),
                                          first);
            first = 1u;
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                          // the previous stage's MMAs have retired
      }
      __syncwarp();
      mbar_arrive_if(&empty[pend < 0 ? 0 : pend], lane == 0 && pend >= 0);
      pend = s;
      if (++s == p.stages) { s = 0; par ^= 1; }
    }
    if (active) {
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
    }
    __syncwarp();
    mbar_arrive_if(&empty[pend < 0 ? 0 : pend], lane == 0 && pend >= 0);
    if (active) {
      // fragment (see wgmma.cuh): rows w * 16 + lane / 4 (+ 8) of this half, column pairs b * 8 + 2 (lane % 4)
      const int n0 = nt * BN;
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int m = mt * (p.Mblocks * 64) + r0 + 8 * i;
        if (m >= p.Mp) continue;
        float* dst = p.stage + ((size_t)tap * p.Mp + m) * p.Np + n0;
#pragma unroll
        for (int b = 0; b < BN / 8; ++b) {
          const int col = b * 8 + 2 * (lane & 3);
          if (n0 + col < p.Np) atomicAdd(reinterpret_cast<float2*>(dst + col), make_float2(acc[b * 4 + i * 2], acc[b * 4 + i * 2 + 1]));
        }
      }
    }
  }
}

// G[tap][m][n] -> parameter gradient [R][Cc][taps] (+=) with (row, column) = (m, n), or (n, m) when the operands were swapped;
// rows >= R1 go to the second weight set of a fused unit
__global__ void __launch_bounds__(256) unstage_wgrad_kernel(const float* __restrict__ stage, int Mp, int Np, int swap, int R, int R1, int Cc,
                                                            int taps, float* __restrict__ dw, float* __restrict__ dw2) {
  const long long total = (long long)R * Cc * taps;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(idx % taps);
    const long long r = idx / taps;
    const int col = (int)(r % Cc), row = (int)(r / Cc);
    const int m = swap ? col : row, n = swap ? row : col;
    const float v = stage[((size_t)t * Mp + m) * Np + n];
    if (row < R1) { if (dw) dw[idx] += v; }
    else if (dw2) dw2[((size_t)(row - R1) * Cc + col) * taps + t] += v;
  }
}

template <int BN>
static cudaError_t launch_wgrad_bn(const CUtensorMap& tmOut, const CUtensorMap& tmIn, const WgradParams& p, int units, size_t smem, cudaStream_t s) {
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_umma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = smem;
  }
  wgrad_umma_kernel<BN><<<units, kWgThreads, smem, s>>>(tmOut, tmIn, p);
  return cudaGetLastError();
}

size_t wgrad_stage_bytes(const WgradParams& p) { return (size_t)p.ntaps * p.Mp * p.Np * sizeof(float); }

// shared memory of one pipeline stage (must match the kernel's layout)
size_t wgrad_stage_smem_bytes(const WgradParams& p) {
  const size_t blkA = ((size_t)p.KP * 128 + 1023) & ~(size_t)1023, blkB = ((size_t)p.KP * p.b_row + 1023) & ~(size_t)1023;
  return (size_t)(p.split ? 2 : 1) * (2 * blkA + p.Nblocks * blkB);
}

cudaError_t launch_wgrad_umma(const CUtensorMap& tmOut, const CUtensorMap& tmIn, const WgradParams& p, int R, int R1, int Cc,
                              float* dw, float* dw2, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(p.stage, 0, wgrad_stage_bytes(p), s);
  if (e != cudaSuccess) return e;
  const size_t stage_bytes = wgrad_stage_smem_bytes(p);
  const size_t smem = (size_t)p.stages * stage_bytes + 1024 + 2 * p.stages * sizeof(uint64_t);
  const int units = p.ntaps * p.m_tiles * p.n_tiles * p.ksplit;
  static const bool log = getenv("V2V_WG_LOG") != nullptr;        // one line per launch, to pair with a profiler's kernel list
  if (log) fprintf(stderr, "wgrad grid %dx%dx%d taps %d aC %d bC %d BN %d swap %d KP %d units %d (ksplit %d x %d chunks) R %d Cc %d\n", p.N, p.gh, p.gw,
                   p.ntaps, p.a_C, p.b_C, p.BN, p.swap, p.KP, units, p.ksplit, p.chunks_per_unit, R, Cc);
  switch (p.BN) {
    case 16: e = launch_wgrad_bn<16>(tmOut, tmIn, p, units, smem, s); break;
    case 32: e = launch_wgrad_bn<32>(tmOut, tmIn, p, units, smem, s); break;
    case 64: e = launch_wgrad_bn<64>(tmOut, tmIn, p, units, smem, s); break;
    case 128: e = launch_wgrad_bn<128>(tmOut, tmIn, p, units, smem, s); break;
    default: return cudaErrorInvalidConfiguration;
  }
  if (e != cudaSuccess) return e;
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const long long total = (long long)R * Cc * p.ntaps;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 132 * 16);
  unstage_wgrad_kernel<<<blocks, 256, 0, s>>>(p.stage, p.Mp, p.Np, p.swap, R, R1, Cc, p.ntaps, dw, dw2);
  return cudaGetLastError();
}

// dX[n][y][x][c] += sum of the padded-extent gradient over the padded positions that mirror onto (y, x) (reflect halo) or
// the interior position alone (zero halo / no halo): gather form, deterministic.  src: dense NHWC fp32 (N, PH, PW, stride Cs)
// whose pixel (pad, pad) is input pixel (0, 0); rows / columns beyond H + 2 pad are ignored (cropped).
__global__ void __launch_bounds__(256) fold_add_kernel(const float* __restrict__ src, int Cs, int PH, int PW, float* __restrict__ dx, int N,
                                                       int H, int W, int C, int pad, int reflect) {
  const size_t total = (size_t)N * H * W * C;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    size_t t = idx / C;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H);
    const int n = (int)(t / H);
    int ys[3], xs[3], ny = 0, nx = 0;
    ys[ny++] = y + pad; xs[nx++] = x + pad;
    if (reflect) {
      if (y >= 1 && y <= pad) ys[ny++] = pad - y;
      if (y <= H - 2 && y >= H - 1 - pad) ys[ny++] = pad + 2 * (H - 1) - y;
      if (x >= 1 && x <= pad) xs[nx++] = pad - x;
      if (x <= W - 2 && x >= W - 1 - pad) xs[nx++] = pad + 2 * (W - 1) - x;
    }
    float s = 0.f;
    for (int a = 0; a < ny; ++a)
      for (int b = 0; b < nx; ++b) s += src[(((size_t)n * PH + ys[a]) * PW + xs[b]) * Cs + c];
    dx[idx] += s;
  }
}

cudaError_t launch_fold_add(const FoldParams& p, cudaStream_t s) {
  const size_t total = (size_t)p.N * p.H * p.W * p.C;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 16);
  fold_add_kernel<<<blocks, 256, 0, s>>>(p.src, p.Cs, p.PH, p.PW, p.dx, p.N, p.H, p.W, p.C, p.pad, p.reflect);
  return cudaGetLastError();
}

}  // namespace v2v
