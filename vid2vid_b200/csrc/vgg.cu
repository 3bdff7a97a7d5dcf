// Kernels of the VGG19 perceptual loss (VGGLoss / Vgg19, models/networks.py:776-791,840-869) that are not convolutions:
//   maxpool2      nn.MaxPool2d(2, stride 2) between two plan activation buffers, and its backward (gradient to the FIRST
//                 maximum of each window in row-major order, as PyTorch routes it)
//   feature_l1    mean |x - y| of two plan values into one element of a caller fp32 tensor: a per-block partial sum in
//                 double, then one warp adds the partials in a fixed order (no float atomics: the same inputs give the
//                 same bits on every run and every graph replay); backward adds g / numel * sign(x - y) into x's gradient
//   avgpool2      nn.AvgPool2d(2, stride 2, count_include_pad=False) on fp32 NCHW planes (the `while x.size(3) > 1024`
//                 downsample in front of the network) and its backward
#include "v2v_internal.h"

namespace v2v {

static inline int grid1d(size_t total, int threads = 256) {
  const size_t b = (total + threads - 1) / threads, cap = (size_t)device_sm_count() * 8;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

// one value of a (possibly split) activation: hi + lo
__device__ __forceinline__ float act_val(const ActDesc& a, size_t off) {
  float v = __bfloat162float(a.base[off]);
  if (a.split) v += __bfloat162float(a.base[off + a.C]);
  return v;
}

// 8 consecutive channels of one pixel, hi and lo halves (lo is zero in bf16 plans)
struct Px8 { bf16 hi[8], lo[8]; };
__device__ __forceinline__ Px8 load8(const ActDesc& a, size_t off) {
  Px8 r;
  *reinterpret_cast<uint4*>(r.hi) = *reinterpret_cast<const uint4*>(a.base + off);
  if (a.split) *reinterpret_cast<uint4*>(r.lo) = *reinterpret_cast<const uint4*>(a.base + off + a.C);
  else *reinterpret_cast<uint4*>(r.lo) = make_uint4(0, 0, 0, 0);
  return r;
}

// ------------------------------------------------------------------------------ max-pool 2x2 / stride 2
// One thread per (output pixel, 8 channels).  Windows are scanned row-major and a later element wins only when it is
// strictly greater (or NaN), as in PyTorch's max_pool2d; the winner's hi / lo pair is copied unchanged, so the pooled value
// is exactly one of the inputs in either precision.  Padded channels are zero in the input and stay zero.
__global__ void __launch_bounds__(256) maxpool2_kernel(PoolParams p) {
  const int C8 = p.in.C / 8, Ho = p.out.H, Wo = p.out.W;
  const size_t total = (size_t)p.out.N * Ho * Wo * C8;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % C8) * 8;
    size_t t = idx / C8;
    const int xo = (int)(t % Wo); t /= Wo;
    const int yo = (int)(t % Ho);
    const int n = (int)(t / Ho);
    Px8 best = load8(p.in, p.in.offset(n, 2 * yo, 2 * xo) + c0);
    float bv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bv[j] = __bfloat162float(best.hi[j]) + __bfloat162float(best.lo[j]);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const Px8 c = load8(p.in, p.in.offset(n, 2 * yo + (k >> 1), 2 * xo + (k & 1)) + c0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = __bfloat162float(c.hi[j]) + __bfloat162float(c.lo[j]);
        if (v > bv[j] || isnan(v)) { bv[j] = v; best.hi[j] = c.hi[j]; best.lo[j] = c.lo[j]; }
      }
    }
    const size_t o = p.out.offset(n, yo, xo) + c0;
    *reinterpret_cast<uint4*>(p.out.base + o) = *reinterpret_cast<const uint4*>(best.hi);
    if (p.out.split) *reinterpret_cast<uint4*>(p.out.base + o + p.out.C) = *reinterpret_cast<const uint4*>(best.lo);
  }
}

// The argmax is recomputed from the saved input (the plan still holds it), with the forward's comparison.  Windows do not
// overlap, so every input element receives from at most one output: plain read-modify-write, no atomics.
__global__ void __launch_bounds__(256) maxpool2_bwd_kernel(PoolParams p, const float* __restrict__ gout, float* __restrict__ gin) {
  const int C = p.in.Cvalid, Ho = p.out.H, Wo = p.out.W, H = p.in.H, W = p.in.W;
  const size_t total = (size_t)p.out.N * Ho * Wo * C;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    size_t t = idx / C;
    const int xo = (int)(t % Wo); t /= Wo;
    const int yo = (int)(t % Ho);
    const int n = (int)(t / Ho);
    int arg = 0;
    float bv = act_val(p.in, p.in.offset(n, 2 * yo, 2 * xo) + c);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const float v = act_val(p.in, p.in.offset(n, 2 * yo + (k >> 1), 2 * xo + (k & 1)) + c);
      if (v > bv || isnan(v)) { bv = v; arg = k; }
    }
    const int y = 2 * yo + (arg >> 1), x = 2 * xo + (arg & 1);
    gin[(((size_t)n * H + y) * W + x) * C + c] += gout[idx];
  }
}

cudaError_t launch_maxpool2(const PoolParams& p, cudaStream_t s) {
  const size_t total = (size_t)p.out.N * p.out.H * p.out.W * (p.in.C / 8);
  maxpool2_kernel<<<grid1d(total), 256, 0, s>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_maxpool2_bwd(const PoolParams& p, const float* gout, float* gin, cudaStream_t s) {
  const size_t total = (size_t)p.out.N * p.out.H * p.out.W * p.in.Cvalid;
  maxpool2_bwd_kernel<<<grid1d(total), 256, 0, s>>>(p, gout, gin);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------ feature L1
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// partials[block] = sum over this block's fixed share of the elements of |x - y|.  The grid is fixed at plan build time
// (feature_l1_blocks), so which elements a thread adds, and in which order, never changes.
__global__ void __launch_bounds__(256) feature_l1_partial_kernel(FeatL1Params p) {
  const int C8 = p.x.C / 8, H = p.x.H, W = p.x.W;
  const size_t total = (size_t)p.x.N * H * W * C8;
  double s = 0.0;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % C8) * 8;
    size_t t = idx / C8;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H);
    const int n = (int)(t / H);
    const Px8 a = load8(p.x, p.x.offset(n, y, x) + c0), b = load8(p.y, p.y.offset(n, y, x) + c0);
    float r = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {        // channels >= Cvalid are zero in both operands
      const float d = (__bfloat162float(a.hi[j]) + __bfloat162float(a.lo[j])) - (__bfloat162float(b.hi[j]) + __bfloat162float(b.lo[j]));
      r += fabsf(d);
    }
    s += (double)r;
  }
  __shared__ double sh[8];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += sh[w];
    p.partials[blockIdx.x] = b;
  }
}

// one warp: lane l adds partials l, l + 32, ... in order, then a fixed butterfly; io[slot][index] = sum / numel
__global__ void feature_l1_final_kernel(FeatL1Params p, double numel) {
  double s = 0.0;
  for (int i = threadIdx.x; i < p.blocks; i += 32) s += p.partials[i];
  s = warp_sum_d(s);
  if (threadIdx.x == 0) reinterpret_cast<float*>(p.io[p.slot])[p.index] = (float)(s / numel);
}

__global__ void __launch_bounds__(256) feature_l1_bwd_kernel(FeatL1Params p, const float* __restrict__ g, float* __restrict__ gx) {
  const int C = p.Cvalid, H = p.x.H, W = p.x.W;
  const size_t total = (size_t)p.x.N * H * W * C;
  const float gs = g[p.index] / (float)total;          // mean backward (grad / numel), then sign: PyTorch's order
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    size_t t = idx / C;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H);
    const int n = (int)(t / H);
    const float d = act_val(p.x, p.x.offset(n, y, x) + c) - act_val(p.y, p.y.offset(n, y, x) + c);
    gx[idx] += d > 0.f ? gs : (d < 0.f ? -gs : 0.f);
  }
}

int feature_l1_blocks(const ActDesc& x) {
  return grid1d((size_t)x.N * x.H * x.W * (x.C / 8));
}

cudaError_t launch_feature_l1(const FeatL1Params& p, cudaStream_t s) {
  feature_l1_partial_kernel<<<p.blocks, 256, 0, s>>>(p);
  feature_l1_final_kernel<<<1, 32, 0, s>>>(p, (double)p.x.N * p.x.H * p.x.W * p.Cvalid);
  return cudaGetLastError();
}
cudaError_t launch_feature_l1_bwd(const FeatL1Params& p, const float* g, float* gx, cudaStream_t s) {
  feature_l1_bwd_kernel<<<grid1d((size_t)p.x.N * p.x.H * p.x.W * p.Cvalid), 256, 0, s>>>(p, g, gx);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------ avg-pool 2x2 / stride 2 (fp32 NCHW planes)
// out = (((a00 + a01) + a10) + a11) / 4 -- PyTorch's summation order; rows / columns past 2 * (H / 2) are dropped (floor).
__global__ void __launch_bounds__(256) avgpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int P, int H, int W, int Ho,
                                                       int Wo) {
  const size_t total = (size_t)P * Ho * Wo;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int xo = (int)(idx % Wo);
    const size_t r = idx / Wo;                       // plane * Ho + yo
    const int yo = (int)(r % Ho);
    const float* ip = in + (r / Ho) * H * W + (size_t)(2 * yo) * W + 2 * xo;
    out[idx] = (((__ldg(ip) + __ldg(ip + 1)) + __ldg(ip + W)) + __ldg(ip + W + 1)) / 4.f;
  }
}
// W % 4 == 0: a thread produces two adjacent outputs from one 16-byte load per input row (same summation order)
__global__ void __launch_bounds__(256) avgpool2_vec_kernel(const float* __restrict__ in, float* __restrict__ out, int P, int H, int W, int Ho,
                                                           int Wo) {
  const int Wq = Wo / 2;
  const size_t total = (size_t)P * Ho * Wq;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(idx % Wq);
    const size_t r = idx / Wq;
    const int yo = (int)(r % Ho);
    const float* ip = in + (r / Ho) * H * W + (size_t)(2 * yo) * W + 4 * k;
    const float4 a = __ldg(reinterpret_cast<const float4*>(ip)), b = __ldg(reinterpret_cast<const float4*>(ip + W));
    *reinterpret_cast<float2*>(out + r * Wo + 2 * k) =
        make_float2((((a.x + a.y) + b.x) + b.y) / 4.f, (((a.z + a.w) + b.z) + b.w) / 4.f);
  }
}
// gin (P, H, W) = gout / 4 at the window each element belongs to; 0 on the rows / columns the floor dropped
__global__ void __launch_bounds__(256) avgpool2_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gin, int P, int H, int W, int Ho,
                                                           int Wo) {
  const size_t total = (size_t)P * H * W;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W);
    const size_t r = idx / W;
    const int y = (int)(r % H);
    const int yo = y >> 1, xo = x >> 1;
    gin[idx] = (yo < Ho && xo < Wo) ? __ldg(gout + ((r / H) * Ho + yo) * Wo + xo) / 4.f : 0.f;
  }
}
// W % 4 == 0 and H even: one 16-byte store per thread from one 8-byte load
__global__ void __launch_bounds__(256) avgpool2_bwd_vec_kernel(const float* __restrict__ gout, float* __restrict__ gin, int P, int H, int W,
                                                               int Wo) {
  const int Wq = W / 4;
  const size_t total = (size_t)P * H * Wq;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(idx % Wq);
    const size_t r = idx / Wq;                       // plane * H + y
    const int y = (int)(r % H);
    const float2 g = __ldg(reinterpret_cast<const float2*>(gout + ((r / H) * (H / 2) + (y >> 1)) * Wo + 2 * k));
    const float a = g.x / 4.f, b = g.y / 4.f;
    *reinterpret_cast<float4*>(gin + r * W + 4 * k) = make_float4(a, a, b, b);
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

cudaError_t launch_avgpool2(const float* in, float* out, int P, int H, int W, cudaStream_t s) {
  const int Ho = H / 2, Wo = W / 2;
  if (W % 4 == 0 && aligned16(in) && aligned16(out)) avgpool2_vec_kernel<<<grid1d((size_t)P * Ho * (Wo / 2)), 256, 0, s>>>(in, out, P, H, W, Ho, Wo);
  else avgpool2_kernel<<<grid1d((size_t)P * Ho * Wo), 256, 0, s>>>(in, out, P, H, W, Ho, Wo);
  return cudaGetLastError();
}
cudaError_t launch_avgpool2_bwd(const float* gout, float* gin, int P, int H, int W, cudaStream_t s) {
  const int Ho = H / 2, Wo = W / 2;
  if (W % 4 == 0 && H % 2 == 0 && aligned16(gout) && aligned16(gin)) avgpool2_bwd_vec_kernel<<<grid1d((size_t)P * H * (W / 4)), 256, 0, s>>>(gout, gin, P, H, W, Wo);
  else avgpool2_bwd_kernel<<<grid1d((size_t)P * H * W), 256, 0, s>>>(gout, gin, P, H, W, Ho, Wo);
  return cudaGetLastError();
}

}  // namespace v2v
