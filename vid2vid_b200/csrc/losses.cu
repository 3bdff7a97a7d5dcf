// Loss reductions of the training step and the backward of the two HBM helpers the losses differentiate through
// (SURVEY 8 row a13; models/vid2vid_model_D.py:117-140,199-213, models/networks.py:731-812):
//   l1_loss      mean |a*m - b*m|  (MaskedL1Loss with a (N,1,H,W) mask broadcast over channels; plain L1 with m == NULL:
//                criterionFeat) -- forward sum and backward in one pass each
//   mse_const    mean (x - t)^2 against a constant label (GANLoss with use_lsgan, networks.py:764-774)
//   avgpool3s2_bwd, resample_bwd  (gradients wrt image and flow of BaseModel.resample, base_model.py:189-196)
//   face_region  the face bounding box the face discriminator crops (vid2vid_model_D.py:149-162,215-230)
#include <climits>

#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float sh[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  v = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

// sum[0] += sum |a*m - b*m|   (double accumulator: the mean over up to 2^25 elements must not depend on the block order)
__global__ void __launch_bounds__(256) l1_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ m,
                                                     size_t total, size_t HW, int C, double* sum) {
  float s = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float d;
    if (m) { const float mv = m[(i / (HW * C)) * HW + i % HW]; d = a[i] * mv - (b ? b[i] * mv : 0.f); }
    else d = a[i] - (b ? b[i] : 0.f);
    s += fabsf(d);
  }
  s = block_sum(s);
  if (threadIdx.x == 0) atomicAdd(sum, (double)s);
}
// ga = sign(a*m - b*m) * m * g / numel ; gb = -ga   (either may be NULL)
__global__ void __launch_bounds__(256) l1_bwd_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ m,
                                                     size_t total, size_t HW, int C, const float* __restrict__ g, float inv_numel,
                                                     float* __restrict__ ga, float* __restrict__ gb) {
  const float gs = g[0] * inv_numel;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float mv = 1.f;
    if (m) mv = m[(i / (HW * C)) * HW + i % HW];
    const float d = a[i] * mv - (b ? b[i] * mv : 0.f);
    const float r = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * mv * gs;
    if (ga) ga[i] = r;
    if (gb) gb[i] = -r;
  }
}
__global__ void __launch_bounds__(256) mse_const_fwd_kernel(const float* __restrict__ x, size_t total, float t, double* sum) {
  float s = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const float d = x[i] - t;
    s += d * d;
  }
  s = block_sum(s);
  if (threadIdx.x == 0) atomicAdd(sum, (double)s);
}
__global__ void mse_const_bwd_kernel(const float* __restrict__ x, size_t total, float t, const float* __restrict__ g, float inv_numel,
                                     float* __restrict__ gx) {
  const float gs = 2.f * g[0] * inv_numel;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    gx[i] = (x[i] - t) * gs;
}
__global__ void sum_to_mean_kernel(const double* sum, float inv_numel, float* out) { out[0] = (float)(sum[0] * (double)inv_numel); }

// gin[y][x] = sum over the <= 4 output windows containing (y, x) of gout / count(window)
__global__ void avgpool3s2_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gin, int P, int H, int W, int Ho, int Wo) {
  const size_t total = (size_t)P * H * W;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W), y = (int)((idx / W) % H);
    const size_t pl = idx / ((size_t)W * H);
    float s = 0.f;
    for (int oy = (y - 1 + 1) / 2; oy <= (y + 1) / 2; ++oy) {      // 2*oy - 1 <= y <= 2*oy + 1
      if (oy < 0 || oy >= Ho || 2 * oy - 1 > y) continue;
      const int cy = min(2 * oy + 1, H - 1) - max(2 * oy - 1, 0) + 1;
      for (int ox = x / 2; ox <= (x + 1) / 2; ++ox) {
        if (ox < 0 || ox >= Wo || 2 * ox - 1 > x) continue;
        const int cx = min(2 * ox + 1, W - 1) - max(2 * ox - 1, 0) + 1;
        s += gout[(pl * Ho + oy) * Wo + ox] / (float)(cy * cx);
      }
    }
    gin[idx] = s;
  }
}

// backward of resample(image, flow): gimage (atomicAdd scatter, zero-filled by the caller), gflow (written)
__device__ __forceinline__ float lin_m1p1(int i, int n) {
  const float step = 2.0f / (float)(n - 1);
  return (i < n / 2) ? (-1.0f + step * (float)i) : (1.0f - step * (float)(n - 1 - i));
}
__global__ void resample_bwd_kernel(const float* __restrict__ img, const float* __restrict__ flow, const float* __restrict__ gout,
                                    float* __restrict__ gimg, float* __restrict__ gflow, int N, int C, int H, int W, int ac) {
  const size_t HW = (size_t)H * W, total = (size_t)N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    const int y = (int)(pix / W), x = (int)(pix - (size_t)y * W);
    const float gx = lin_m1p1(x, W) + flow[((size_t)n * 2) * HW + pix] / (((float)W - 1.0f) / 2.0f);
    const float gy = lin_m1p1(y, H) + flow[((size_t)n * 2 + 1) * HW + pix] / (((float)H - 1.0f) / 2.0f);
    float sx = ac ? ((gx + 1.f) / 2.f) * (float)(W - 1) : ((gx + 1.f) * (float)W - 1.f) / 2.f;
    float sy = ac ? ((gy + 1.f) / 2.f) * (float)(H - 1) : ((gy + 1.f) * (float)H - 1.f) / 2.f;
    float dsx = (ac ? (float)(W - 1) / 2.f : (float)W / 2.f) / (((float)W - 1.0f) / 2.0f);
    float dsy = (ac ? (float)(H - 1) / 2.f : (float)H / 2.f) / (((float)H - 1.0f) / 2.0f);
    if (sx <= 0.f || sx >= (float)(W - 1)) dsx = 0.f;
    if (sy <= 0.f || sy >= (float)(H - 1)) dsy = 0.f;
    sx = fminf((float)(W - 1), fmaxf(sx, 0.f)); sy = fminf((float)(H - 1), fmaxf(sy, 0.f));
    const float x0f = floorf(sx), y0f = floorf(sy);
    const int x0 = (int)x0f, y0 = (int)y0f, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float wx = sx - x0f, wy = sy - y0f;
    float dfx = 0.f, dfy = 0.f;
    for (int c = 0; c < C; ++c) {
      const float g = gout[((size_t)n * C + c) * HW + pix];
      const float* pl = img + ((size_t)n * C + c) * HW;
      const float v00 = pl[(size_t)y0 * W + x0], v01 = pl[(size_t)y0 * W + x1], v10 = pl[(size_t)y1 * W + x0], v11 = pl[(size_t)y1 * W + x1];
      dfx += g * ((v01 - v00) * (1.f - wy) + (v11 - v10) * wy) * dsx;
      dfy += g * ((v10 - v00) * (1.f - wx) + (v11 - v01) * wx) * dsy;
      if (gimg) {
        float* gp = gimg + ((size_t)n * C + c) * HW;
        atomicAdd(gp + (size_t)y0 * W + x0, g * (1.f - wx) * (1.f - wy));
        atomicAdd(gp + (size_t)y0 * W + x1, g * wx * (1.f - wy));
        atomicAdd(gp + (size_t)y1 * W + x0, g * (1.f - wx) * wy);
        atomicAdd(gp + (size_t)y1 * W + x1, g * wx * wy);
      }
    }
    if (gflow) { gflow[((size_t)n * 2) * HW + pix] = dfx; gflow[((size_t)n * 2 + 1) * HW + pix] = dfy; }
  }
}

// Face region of the pose demo's face discriminator (Vid2VidModelD.get_face_region, vid2vid_model_D.py:215-230): the bounding
// box of the pixels of the whole batch that satisfy the face predicate, box = {found, ymin, ymax, xmin, xmax}.  The predicate
// compares in fp32 against the fp32-rounded constants, as PyTorch compares an fp32 tensor with a Python float.  Each warp
// reduces its pixels, each block combines its warps in shared memory, and one thread per block merges the block's box into
// `box` with integer atomics: min / max / or, so the result does not depend on the order.
__device__ __forceinline__ bool face_pixel(const float* p, size_t HW, int openpose_only) {
  if (!openpose_only) return p[2 * HW] > 0.9f;
  const float c0 = p[0], c1 = p[HW], c2 = p[2 * HW];
  return c0 > 0.19f && c0 < 0.21f && c1 < -0.99f && c2 > -0.61f && c2 < -0.59f;
}
__global__ void face_region_reset_kernel(int* box) {
  box[0] = 0; box[1] = INT_MAX; box[2] = -1; box[3] = INT_MAX; box[4] = -1;
}
__global__ void __launch_bounds__(256) face_region_kernel(const float* __restrict__ a, int N, int C, int H, int W, int openpose_only,
                                                          int* box) {
  __shared__ int s_box[5];
  if (threadIdx.x == 0) { s_box[0] = 0; s_box[1] = INT_MAX; s_box[2] = -1; s_box[3] = INT_MAX; s_box[4] = -1; }
  __syncthreads();
  const size_t HW = (size_t)H * W, total = (size_t)N * HW;
  int ymin = INT_MAX, ymax = -1, xmin = INT_MAX, xmax = -1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t n = i / HW, pix = i - n * HW;
    if (face_pixel(a + n * C * HW + pix, HW, openpose_only)) {
      const int y = (int)(pix / W), x = (int)(pix - (size_t)y * W);
      ymin = min(ymin, y); ymax = max(ymax, y); xmin = min(xmin, x); xmax = max(xmax, x);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
    xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
  }
  if ((threadIdx.x & 31) == 0 && ymax >= 0) {
    s_box[0] = 1;
    atomicMin(s_box + 1, ymin); atomicMax(s_box + 2, ymax); atomicMin(s_box + 3, xmin); atomicMax(s_box + 4, xmax);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_box[0]) {
    atomicOr(box, 1);
    atomicMin(box + 1, s_box[1]); atomicMax(box + 2, s_box[2]); atomicMin(box + 3, s_box[3]); atomicMax(box + 4, s_box[4]);
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 8;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_face_region(const float* real_A, int N, int C, int H, int W, int openpose_only, int* box, cudaStream_t s) {
  face_region_reset_kernel<<<1, 1, 0, s>>>(box);
  face_region_kernel<<<grid1d((size_t)N * H * W), 256, 0, s>>>(real_A, N, C, H, W, openpose_only, box);
  return cudaGetLastError();
}

cudaError_t launch_l1_fwd(const float* a, const float* b, const float* m, int N, int C, int H, int W, double* sum_ws, float* out,
                          cudaStream_t s) {
  const size_t total = (size_t)N * C * H * W;
  cudaError_t e = cudaMemsetAsync(sum_ws, 0, sizeof(double), s);
  if (e != cudaSuccess) return e;
  l1_fwd_kernel<<<grid1d(total), 256, 0, s>>>(a, b, m, total, (size_t)H * W, C, sum_ws);
  sum_to_mean_kernel<<<1, 1, 0, s>>>(sum_ws, 1.f / (float)total, out);
  return cudaGetLastError();
}
cudaError_t launch_l1_bwd(const float* a, const float* b, const float* m, int N, int C, int H, int W, const float* g, float* ga, float* gb,
                          cudaStream_t s) {
  const size_t total = (size_t)N * C * H * W;
  l1_bwd_kernel<<<grid1d(total), 256, 0, s>>>(a, b, m, total, (size_t)H * W, C, g, 1.f / (float)total, ga, gb);
  return cudaGetLastError();
}
cudaError_t launch_mse_const_fwd(const float* x, long long total, float t, double* sum_ws, float* out, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(sum_ws, 0, sizeof(double), s);
  if (e != cudaSuccess) return e;
  mse_const_fwd_kernel<<<grid1d((size_t)total), 256, 0, s>>>(x, (size_t)total, t, sum_ws);
  sum_to_mean_kernel<<<1, 1, 0, s>>>(sum_ws, 1.f / (float)total, out);
  return cudaGetLastError();
}
cudaError_t launch_mse_const_bwd(const float* x, long long total, float t, const float* g, float* gx, cudaStream_t s) {
  mse_const_bwd_kernel<<<grid1d((size_t)total), 256, 0, s>>>(x, (size_t)total, t, g, 1.f / (float)total, gx);
  return cudaGetLastError();
}
cudaError_t launch_avgpool3s2_bwd(const float* gout, float* gin, int P, int H, int W, cudaStream_t s) {
  avgpool3s2_bwd_kernel<<<grid1d((size_t)P * H * W), 256, 0, s>>>(gout, gin, P, H, W, (H - 1) / 2 + 1, (W - 1) / 2 + 1);
  return cudaGetLastError();
}
cudaError_t launch_resample_bwd(const float* img, const float* flow, const float* gout, float* gimg, float* gflow, int N, int C, int H,
                                int W, int ac, cudaStream_t s) {
  resample_bwd_kernel<<<grid1d((size_t)N * H * W), 256, 0, s>>>(img, flow, gout, gimg, gflow, N, C, H, W, ac);
  return cudaGetLastError();
}

}  // namespace v2v
