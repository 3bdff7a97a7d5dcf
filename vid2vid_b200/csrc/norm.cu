// Batch/Instance-norm statistics finalisation and the fused
//   normalise * gamma + beta -> activation -> (+ residual / skip addends) -> write next layer's
//   halo-padded NHWC bf16 buffer (reflect or zero halo, optional stride-2 parity split)
// pass.  HBM-bound: reads 2 B/elem raw (+2 B per addend), writes 2 B/elem.
// Reference ops replaced: nn.BatchNorm2d (train-mode statistics, SURVEY App. B #1) /
// nn.InstanceNorm2d, nn.ReLU / LeakyReLU, nn.ReflectionPad2d and the residual adds at
// models/networks.py:23-30,126,204,298-305,559-593,687-703.
#include <algorithm>

#include <cstdlib>
#include "ptx.cuh"
#include "v2v_internal.h"
#include "finalize.cuh"

namespace v2v {

// Stand-alone finalisation (one thread per channel): writes scale / shift and the train-mode side effects of the norm slices
// whose producing conv launch does not finalise them in its tail (the SIMT conv implementation, a third slice of one raw).
// Both normalise kernels only read the scale / shift arrays.
__global__ void __launch_bounds__(128) stats_finalize_kernel(FinalizeParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.C) return;
  channel_side_effects(p, c);
}

__device__ __forceinline__ int reflect_idx(int i, int n) {   // nn.ReflectionPad2d index map
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

__device__ __forceinline__ void bf16x8_to_float(const uint4& r, float (&f)[8]) {
  const __nv_bfloat162* rp = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) { float2 a = __bfloat1622float2(rp[j]); f[2 * j] = a.x; f[2 * j + 1] = a.y; }
}
__device__ __forceinline__ void bf16x8_add(const uint4& r, float (&f)[8]) {
  const __nv_bfloat162* rp = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) { float2 a = __bfloat1622float2(rp[j]); f[2 * j] += a.x; f[2 * j + 1] += a.y; }
}


// Grid-stride over (padded pixel, 8-channel vector) items (2-D-grid and multi-item-per-thread variants measured slower).
// 32-bit index arithmetic throughout: with 64-bit div/mod this kernel was instruction bound (~4 x 100-instruction
// divisions per 16-byte item), not bandwidth bound.
__device__ __forceinline__ void apply_item(const ApplyParams& p, int vecs, int Wpad, int Hpad, unsigned idx) {
  const unsigned t0 = idx / (unsigned)vecs;
  const int v = (int)(idx - t0 * (unsigned)vecs);
  const unsigned t1 = t0 / (unsigned)Wpad;
  const int xp = (int)(t0 - t1 * (unsigned)Wpad);
  const int n = (int)(t1 / (unsigned)Hpad);
  const int yp = (int)(t1 - (unsigned)n * (unsigned)Hpad);
  int y = yp - p.out.pad_t, x = xp - p.out.pad_l;
  const bool halo = (y < 0 || y >= p.out.H || x < 0 || x >= p.out.W);
  uint4 o = make_uint4(0, 0, 0, 0);
  const int c0 = v * 8;
  bool zero = (c0 >= p.raw.Cvalid);
  if (halo) {
    if (p.pad_mode == PAD_REFLECT) { y = reflect_idx(y, p.out.H); x = reflect_idx(x, p.out.W); }
    else zero = true;
  }
  uint4 ol = make_uint4(0, 0, 0, 0);
  if (!zero) {
    const size_t ri = (((size_t)n * p.raw.H + y) * p.raw.W + x) * p.raw.C + c0;
    float f[8];
    if (p.raw.f32) {
      const float4* rp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.raw.base) + ri);
      const float4 f0 = rp[0], f1 = rp[1];
      f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
    } else {
      bf16x8_to_float(*reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(p.raw.base) + ri), f);
    }
    if (p.scale) {
      const float* sc = p.scale + (size_t)n * p.scale_stride + c0;
      const float* sh = p.shift + (size_t)n * p.scale_stride + c0;
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = (c0 + j < p.raw.Cvalid) ? fmaf(f[j], sc[j], sh[j]) : 0.f;
    }
    if (p.act == ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
    } else if (p.act == ACT_LRELU) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = f[j] > 0.f ? f[j] : f[j] * p.slope;
    }
    for (int a = 0; a < p.n_add; ++a) {
      const ActDesc& ad = p.add[a];
      if (c0 < ad.C) {
        const bf16* ap = ad.base + ad.offset(n, y, x) + c0;
        bf16x8_add(*reinterpret_cast<const uint4*>(ap), f);
        if (ad.split) bf16x8_add(*reinterpret_cast<const uint4*>(ap + ad.C), f);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) if (c0 + j >= p.raw.Cvalid) f[j] = 0.f;
    o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
    o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
    if (p.out.split) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] -= __bfloat162float(__float2bfloat16_rn(f[j]));
      ol.x = pack_bf16x2(f[0], f[1]); ol.y = pack_bf16x2(f[2], f[3]);
      ol.z = pack_bf16x2(f[4], f[5]); ol.w = pack_bf16x2(f[6], f[7]);
    }
  }
  bf16* op = p.out.base + p.out.offset(n, yp - p.out.pad_t, xp - p.out.pad_l) + c0;
  *reinterpret_cast<uint4*>(op) = o;
  if (p.out.split) *reinterpret_cast<uint4*>(op + p.out.C) = ol;
}

__global__ void __launch_bounds__(256) norm_apply_kernel(ApplyParams p) {
  const int vecs = p.out.C / 8;
  const int Hpad = p.out.H + p.out.pad_t + p.out.pad_b, Wpad = p.out.W + p.out.pad_l + p.out.pad_r;
  const unsigned total = (unsigned)p.out.N * Hpad * Wpad * vecs;        // < 2^31 checked by the launcher
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) apply_item(p, vecs, Wpad, Hpad, idx);
}

// Row-segment variant (default).  A block owns one padded output row (n, yp) and a segment of it; a thread keeps ONE
// 8-channel vector v = t % vecs for its whole life, so scale / shift live in registers and there is no division or
// 64-bit index arithmetic per item: the grid-stride kernel above issues ~260 instructions per 16-byte item and is
// instruction bound, this one ~45.
// Consecutive threads cover the C * 2 contiguous bytes of a pixel, then the next pixel: loads and stores are coalesced.
struct RowAddr { size_t base; int xs; size_t plane; int parity, C, pad_l; };   // C = bf16 elements per pixel
__device__ __forceinline__ RowAddr row_addr(const ActDesc& a, int n, int y) {     // y relative to the interior
  RowAddr r;
  const int yp = y + a.pad_t;
  r.parity = a.parity; r.C = a.Cs(); r.pad_l = a.pad_l;
  if (a.parity) {
    r.base = (((size_t)n * 4 + ((yp & 1) << 1)) * a.Hp + (yp >> 1)) * a.Wp * (size_t)a.Cs();
    r.plane = (size_t)a.Hp * a.Wp * a.Cs();
  } else {
    r.base = ((size_t)n * a.Hp + yp) * a.Wp * (size_t)a.Cs();
    r.plane = 0;
  }
  return r;
}
__device__ __forceinline__ size_t row_off(const RowAddr& r, int x) {               // x relative to the interior
  const int xp = x + r.pad_l;
  return r.parity ? r.base + (xp & 1) * r.plane + (size_t)(xp >> 1) * r.C : r.base + (size_t)xp * r.C;
}

// PREC (precise plans): raw is fp32 (two 16-byte loads per item), addends and the output are [hi | lo] bf16 pairs
// (two 16-byte loads / stores per item, C elements apart); batches of 2 items instead of 4 keep the same bytes in flight.
template <int NADD, bool PREC>
__global__ void __launch_bounds__(256) norm_apply_rows_kernel(ApplyParams p, int xt, int ppb) {
  constexpr int NB = PREC ? 2 : 4;          // items per batch
  constexpr int NW = PREC ? 2 : 1;          // 16-byte words per item and tensor
  const int vecs = p.out.C >> 3;
  const int t = threadIdx.x;
  const bool idle = t >= ppb * vecs;                 // (idle threads still take part in the prologue barrier)
  const int pl = idle ? 0 : t / vecs, v = idle ? 0 : t - pl * vecs;
  const int Hpad = p.out.H + p.out.pad_t + p.out.pad_b, Wpad = p.out.W + p.out.pad_l + p.out.pad_r;
  const int n = blockIdx.y / Hpad, yp = blockIdx.y - n * Hpad;
  const int c0 = v * 8;
  const bool reflect = p.pad_mode == PAD_REFLECT;
  int y = yp - p.out.pad_t;
  const bool yhalo = (y < 0 || y >= p.out.H);
  if (reflect) y = reflect_idx(y, p.out.H);
  const bool zero_row = (c0 >= p.raw.Cvalid) || (yhalo && !reflect);
  // per-thread constants: scale / shift of its 8 channels (0 beyond the valid channels: those outputs are 0)
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const bool cv = c0 + j < p.raw.Cvalid;
    sc[j] = cv ? (p.scale ? __ldg(p.scale + (size_t)n * p.scale_stride + c0 + j) : 1.f) : 0.f;
    sh[j] = (cv && p.scale) ? __ldg(p.shift + (size_t)n * p.scale_stride + c0 + j) : 0.f;
  }
  if (idle) return;
  const size_t eb = PREC ? 4 : 2;
  const char* raw_row = reinterpret_cast<const char*>(p.raw.base) +
                        (((size_t)n * p.raw.H + (zero_row ? 0 : y)) * p.raw.W * (size_t)p.raw.C + c0) * eb;
  const size_t raw_px = (size_t)p.raw.C * eb;
  const RowAddr out_row = row_addr(p.out, n, yp - p.out.pad_t);
  RowAddr add_row[2];
  bool add_on[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    add_on[a] = a < NADD && c0 < p.add[a].C && !zero_row;
    if (add_on[a]) add_row[a] = row_addr(p.add[a], n, y);
  }
  const int x_end = min(Wpad, (int)(blockIdx.x + 1) * xt);
  // Batches of NB items: all loads of a batch are issued before the first use, so a thread keeps several 16-byte loads
  // in flight -- one load per thread leaves the kernel latency bound.
  for (int xb = blockIdx.x * xt + pl; xb < x_end; xb += NB * ppb) {
    uint4 r[NB][NW], q0[NADD > 0 ? NB : 1][NW], q1[NADD > 1 ? NB : 1][NW];
    bool live[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int xp = xb + b * ppb;
      int x = xp - p.out.pad_l;
      const bool xhalo = (x < 0 || x >= p.out.W);
      live[b] = xp < x_end && !(zero_row || (xhalo && !reflect));
      if (reflect) x = reflect_idx(x, p.out.W);
      if (live[b]) {
        const uint4* rp = reinterpret_cast<const uint4*>(raw_row + (size_t)x * raw_px);
#pragma unroll
        for (int w = 0; w < NW; ++w) r[b][w] = rp[w];
        if (NADD > 0 && add_on[0]) {
          const bf16* ap = p.add[0].base + row_off(add_row[0], x) + c0;
          q0[NADD > 0 ? b : 0][0] = *reinterpret_cast<const uint4*>(ap);
          if (PREC) q0[NADD > 0 ? b : 0][NW - 1] = *reinterpret_cast<const uint4*>(ap + p.add[0].C);
        }
        if (NADD > 1 && add_on[1]) {
          const bf16* ap = p.add[1].base + row_off(add_row[1], x) + c0;
          q1[NADD > 1 ? b : 0][0] = *reinterpret_cast<const uint4*>(ap);
          if (PREC) q1[NADD > 1 ? b : 0][NW - 1] = *reinterpret_cast<const uint4*>(ap + p.add[1].C);
        }
      }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int xp = xb + b * ppb;
      if (xp >= x_end) break;
      uint4 o = make_uint4(0, 0, 0, 0), ol = make_uint4(0, 0, 0, 0);
      if (live[b]) {
        float f[8];
        if (PREC) {
          const float4 f0 = *reinterpret_cast<const float4*>(&r[b][0]), f1 = *reinterpret_cast<const float4*>(&r[b][NW - 1]);
          f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
        } else {
          bf16x8_to_float(r[b][0], f);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], sc[j], sh[j]);
        if (p.act == ACT_RELU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
        } else if (p.act == ACT_LRELU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = f[j] > 0.f ? f[j] : f[j] * p.slope;
        }
        if (NADD > 0 && add_on[0]) {
          bf16x8_add(q0[NADD > 0 ? b : 0][0], f);
          if (PREC) bf16x8_add(q0[NADD > 0 ? b : 0][NW - 1], f);
        }
        if (NADD > 1 && add_on[1]) {
          bf16x8_add(q1[NADD > 1 ? b : 0][0], f);
          if (PREC) bf16x8_add(q1[NADD > 1 ? b : 0][NW - 1], f);
        }
        if (NADD > 0) {        // addends may carry values in channels the raw tensor does not have: keep the padding zero
#pragma unroll
          for (int j = 0; j < 8; ++j) if (c0 + j >= p.raw.Cvalid) f[j] = 0.f;
        }
        o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
        o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
        if (PREC) {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] -= __bfloat162float(__float2bfloat16_rn(f[j]));
          ol.x = pack_bf16x2(f[0], f[1]); ol.y = pack_bf16x2(f[2], f[3]);
          ol.z = pack_bf16x2(f[4], f[5]); ol.w = pack_bf16x2(f[6], f[7]);
        }
      }
      bf16* op = p.out.base + row_off(out_row, xp - p.out.pad_l) + c0;
      *reinterpret_cast<uint4*>(op) = o;
      if (PREC) *reinterpret_cast<uint4*>(op + p.out.C) = ol;
    }
  }
}

static inline int grid_for(long long total, int block) {
  long long b = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

cudaError_t launch_stats_finalize(const FinalizeParams& p, cudaStream_t stream) {
  stats_finalize_kernel<<<(p.C + 127) / 128, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

// Row-segment kernel while a block can hold one vector per thread of a padded row (vecs <= 256) and the rows fit grid.y;
// the grid-stride kernel otherwise.  v2v_plan_describe reports the same choice.
NormApplyLaunch norm_apply_launch(const ApplyParams& p) {
  NormApplyLaunch l{};
  const long long total = (long long)p.out.N * (p.out.H + p.out.pad_t + p.out.pad_b) *
                          (p.out.W + p.out.pad_l + p.out.pad_r) * (p.out.C / 8);
  const int Wpad = p.out.W + p.out.pad_l + p.out.pad_r, Hpad = p.out.H + p.out.pad_t + p.out.pad_b;
  l.vecs = p.out.C / 8;
  l.rows = l.vecs <= 256 && (long long)p.out.N * Hpad <= 65535;
  if (l.rows) {
    l.ppb = 256 / l.vecs;                           // pixels per block pass
    l.xt = l.ppb * 8;                               // 8 items per thread
    l.grid[0] = (Wpad + l.xt - 1) / l.xt; l.grid[1] = p.out.N * Hpad;
  } else {
    l.grid[0] = grid_for(total, 256); l.grid[1] = 1;
  }
  return l;
}

cudaError_t launch_norm_apply(const ApplyParams& p, cudaStream_t stream) {
  const long long total = (long long)p.out.N * (p.out.H + p.out.pad_t + p.out.pad_b) *
                          (p.out.W + p.out.pad_l + p.out.pad_r) * (p.out.C / 8);
  if (total >= (1LL << 31)) return cudaErrorInvalidValue;
  const bool prec = p.raw.f32 != 0;
  if (prec != (p.out.split != 0)) return cudaErrorInvalidValue;      // precise plans: fp32 raw <-> split activations
  const NormApplyLaunch l = norm_apply_launch(p);
  if (l.rows) {
    const dim3 grid(l.grid[0], l.grid[1]);
    const int xt = l.xt, ppb = l.ppb;
    if (prec) {
      if (p.n_add == 0) norm_apply_rows_kernel<0, true><<<grid, 256, 0, stream>>>(p, xt, ppb);
      else if (p.n_add == 1) norm_apply_rows_kernel<1, true><<<grid, 256, 0, stream>>>(p, xt, ppb);
      else norm_apply_rows_kernel<2, true><<<grid, 256, 0, stream>>>(p, xt, ppb);
    } else {
      if (p.n_add == 0) norm_apply_rows_kernel<0, false><<<grid, 256, 0, stream>>>(p, xt, ppb);
      else if (p.n_add == 1) norm_apply_rows_kernel<1, false><<<grid, 256, 0, stream>>>(p, xt, ppb);
      else norm_apply_rows_kernel<2, false><<<grid, 256, 0, stream>>>(p, xt, ppb);
    }
  } else {
    norm_apply_kernel<<<l.grid[0], 256, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

}  // namespace v2v
