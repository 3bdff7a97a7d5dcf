// Plain SIMT (CUDA-core, fp32-accumulate) evaluation of the same convolution plan the wgmma kernel
// runs: same halo-padded NHWC bf16 input, same packed bf16 weights, same tap groups, same epilogues.
// It exists to cross-check the tensor-core kernel on the device (tests, V2V_CONV_IMPL=simt) -- it is a
// CUDA kernel, not a CPU fallback, and is never selected by default.
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

__device__ __forceinline__ float simt_act(float v, int act, float slope) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_LRELU: return v > 0.f ? v : v * slope;
    case ACT_TANH: return tanhf(v);
    case ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    default: return v;
  }
}

// one thread per (phase, n, gy, gx, co); co fastest so weight rows differ per lane and the
// activation vector is broadcast.
__global__ void conv_simt_kernel(ActDesc in, const bf16* __restrict__ w, int Ktotal, ConvKernelParams p) {
  const long long total = (long long)p.num_phases * p.N * p.grid_h * p.grid_w * p.Cout;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    long long t = idx;
    const int co = (int)(t % p.Cout); t /= p.Cout;
    const int gx = (int)(t % p.grid_w); t /= p.grid_w;
    const int gy = (int)(t % p.grid_h); t /= p.grid_h;
    const int n = (int)(t % p.N); t /= p.N;
    const int phi = (int)t;
    const ConvPhase ph = p.phases[phi];
    float acc = 0.f;
    for (int g = ph.group_begin; g < ph.group_end; ++g) {
      const ConvGroup grp = p.groups[g];
      for (int r = 0; r < p.R; ++r) {
        const int yy = gy + grp.dy + r / p.RW, xx = gx + grp.dx + r % p.RW;
        if (yy < 0 || yy >= in.Hp || xx < 0 || xx >= in.Wp) continue;   // TMA zero fill
        const bf16* a = in.base + ((((size_t)n * in.P + grp.plane) * in.Hp + yy) * in.Wp + xx) * in.Cs();
        const bf16* b = w + (size_t)co * Ktotal * (p.split ? 2 : 1) + (size_t)(grp.tap0 + r) * p.Cp;
        for (int c = 0; c < p.Cp; c += 2) {
          float2 av = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a + c));
          float2 bv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(b + c));
          if (p.split) {     // precise plans: the same three products the tensor-core kernel accumulates
            const float2 al = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a + in.C + c));
            const float2 bl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(b + Ktotal + c));
            acc = fmaf(al.x, bv.x, acc); acc = fmaf(av.x, bl.x, acc);
            acc = fmaf(al.y, bv.y, acc); acc = fmaf(av.y, bl.y, acc);
          }
          acc = fmaf(av.x, bv.x, acc);
          acc = fmaf(av.y, bv.y, acc);
        }
      }
    }
    const int oy = gy * p.oy_mul + ph.oy_add, ox = gx * p.ox_mul + ph.ox_add;
    if (p.epi == EPI_HEAD_F32) {
      float v = acc + (p.bias ? ((p.bias2 && co >= p.Cout1) ? p.bias2[co - p.Cout1] : p.bias[co]) : 0.f);
      v = simt_act(v, p.head_act[co], p.lrelu_slope) * p.head_scale[co];
      reinterpret_cast<float*>(p.io[p.head_slot[co]])[p.head_off[co] + (size_t)n * p.head_bstride[co] + (size_t)oy * p.out_W + ox] = v;
    } else if (p.epi == EPI_RAW_STATS) {
      const size_t oi = (((size_t)n * p.out_H + oy) * p.out_W + ox) * p.out_C + co;
      if (p.out_f32) reinterpret_cast<float*>(p.out)[oi] = acc;
      else reinterpret_cast<bf16*>(p.out)[oi] = __float2bfloat16_rn(acc);
    } else {
      float v = simt_act(acc + (p.bias ? p.bias[co] : 0.f), p.act, p.lrelu_slope);
      const size_t oi = p.out_act.offset(n, oy, ox) + co;
      if (p.out_act.split) split_bf16(v, p.out_act.base[oi], p.out_act.base[oi + p.out_act.C]);
      else p.out_act.base[oi] = __float2bfloat16_rn(v);
    }
  }
}

// Per-channel (sum, sumsq) of a raw NHWC bf16 tensor, one partial row per image:
// stats[(n*2 + {0,1}) * C + c].  Used with the SIMT conv (the wgmma kernel's epilogue produces these itself).
__global__ void raw_stats_kernel(const void* __restrict__ raw_, int f32, int HW, int C, int Cs, stat_t* __restrict__ stats) {
  const int n = blockIdx.y, c = blockIdx.x;
  float s = 0.f, q = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const size_t e = ((size_t)n * HW + i) * C + c;
    float v = f32 ? reinterpret_cast<const float*>(raw_)[e] : __bfloat162float(reinterpret_cast<const bf16*>(raw_)[e]);
    s += v; q += v * v;
  }
  __shared__ float ss[256], sq[256];
  ss[threadIdx.x] = s; sq[threadIdx.x] = q;
  __syncthreads();
  for (int k = blockDim.x / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) { ss[threadIdx.x] += ss[threadIdx.x + k]; sq[threadIdx.x] += sq[threadIdx.x + k]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    stats[((size_t)n * 2 + 0) * Cs + c] = (stat_t)__float2ll_rn(ss[0] * V2V_STAT_SUM_SCALE);
    stats[((size_t)n * 2 + 1) * Cs + c] = (stat_t)__float2ll_rn(sq[0] * V2V_STAT_SQ_SCALE);
  }
}

cudaError_t launch_conv_simt(const ActDesc& in, const bf16* wpacked, int Ktotal, const ConvKernelParams& p,
                             cudaStream_t stream) {
  const long long total = (long long)p.num_phases * p.N * p.grid_h * p.grid_w * p.Cout;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  conv_simt_kernel<<<blocks, 256, 0, stream>>>(in, wpacked, Ktotal, p);
  return cudaGetLastError();
}

cudaError_t launch_raw_stats(const RawDesc& raw, stat_t* stats, int stats_C, cudaStream_t stream) {
  dim3 grid(raw.Cvalid, raw.N);
  raw_stats_kernel<<<grid, 256, 0, stream>>>(raw.base, raw.f32, raw.H * raw.W, raw.C, stats_C, stats);
  return cudaGetLastError();
}

}  // namespace v2v
