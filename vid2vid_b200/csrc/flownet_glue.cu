// HBM-bound glue of the FlowNet2 cascade between its convolutional sub-networks (fp32 NCHW, coalesced along x):
//   flownet_prep   : per-sample per-colour mean over both frames, subtract, /rgb_max, (B,3,2,H,W) -> (B,6,H,W)
//                    (FlowNet2.forward, models/flownet2_pytorch/models.py:97-103)
//   resize         : F.interpolate bilinear (align_corners=False) / nearest, optional pre-multiplier and a second
//                    output divided by a constant: the x4 flow upsampling between the stages (models.py:50,59,104-143:
//                    upsample1/2 bilinear, upsample3/4 nearest; `* div_flow` before, `/ div_flow` for the next stack) and
//                    the resize-to-multiple-of-64 of the vid2vid wrapper (models/flownet.py:46-58)
//   sub_channels   : a[:, c_off:c_off+C] - b   (brightness error input, models.py:113-116)
//   flow_conf      : conf = (sum_c (im1 - warp)^2 < 0.02)  (models/flownet.py:52-54 `norm`)
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

// one block per (b, c): fp64 sum over the 2*H*W values of colour c in both frames.  Frame f of sample b, colour c is the
// plane f{0,1} + b * bstride + c * cstride (stacked (B,3,2,H,W) input: f1 = f0 + HW, bstride 6 HW, cstride 2 HW; two separate
// (B,3,H,W) images: bstride 3 HW, cstride HW).
__global__ void __launch_bounds__(256) flownet_mean_kernel(const float* __restrict__ f0, const float* __restrict__ f1, size_t bstride,
                                                           size_t cstride, float* __restrict__ mean, size_t HW) {
  const int b = blockIdx.x / 3, c = blockIdx.x - 3 * b;
  const float* p0 = f0 + b * bstride + c * cstride;
  const float* p1 = f1 + b * bstride + c * cstride;
  double s = 0.0;
  for (size_t i = threadIdx.x; i < HW; i += blockDim.x) s += (double)p0[i] + (double)p1[i];
  __shared__ double sh[256];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[blockIdx.x] = (float)(sh[0] / (double)(2 * HW));
}

// -> x (B,6,H,W): channel f*3 + c = (frame f colour c - mean[b,c]) / rgb_max; x1 (B,3,H,W) = the frame-1 half, contiguous
__global__ void flownet_center_kernel(const float* __restrict__ f0, const float* __restrict__ f1, size_t bstride, size_t cstride,
                                      const float* __restrict__ mean, float* __restrict__ x, float* __restrict__ x1, int B, size_t HW,
                                      float rgb_max) {
  const size_t total = (size_t)B * 6 * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = idx % HW;
    const int ch = (int)((idx / HW) % 6), b = (int)(idx / (6 * HW));
    const int f = ch / 3, c = ch - 3 * f;
    const float v = (f ? f1 : f0)[b * bstride + c * cstride + pix];
    const float r = __fdiv_rn(__fsub_rn(v, mean[b * 3 + c]), rgb_max);
    x[idx] = r;
    if (f && x1) x1[((size_t)b * 3 + c) * HW + pix] = r;
  }
}

// ATen upsample_bilinear2d / upsample_nearest2d index rules (align_corners = False); scale = in / out (or 1 / scale_factor)
// value read = in * mul, or in / pre_div when pre_div != 1 (FlowNetSD's flow is DIVIDED by div_flow, models.py:142-143)
__global__ void resize_kernel(const float* __restrict__ in, float* __restrict__ out, float* __restrict__ out_div, int planes,
                              int h, int w, int H, int W, float sh, float sw, float mul, float pre_div, float div, int nearest) {
  const size_t total = (size_t)planes * H * W;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int X = (int)(idx % W), Y = (int)((idx / W) % H);
    const size_t pl = idx / ((size_t)W * H);
    const float* p = in + pl * (size_t)h * w;
    float v;
    if (nearest) {
      const int ys = min((int)floorf(__fmul_rn((float)Y, sh)), h - 1), xs = min((int)floorf(__fmul_rn((float)X, sw)), w - 1);
      v = pre_div != 1.f ? __fdiv_rn(p[(size_t)ys * w + xs], pre_div) : __fmul_rn(p[(size_t)ys * w + xs], mul);
    } else {
      float fy = __fsub_rn(__fmul_rn(sh, (float)Y + 0.5f), 0.5f), fx = __fsub_rn(__fmul_rn(sw, (float)X + 0.5f), 0.5f);
      if (fy < 0.f) fy = 0.f;
      if (fx < 0.f) fx = 0.f;
      const int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
      const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
      const float ly = __fsub_rn(fy, (float)y0), lx = __fsub_rn(fx, (float)x0);
      const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
      float v00 = p[(size_t)y0 * w + x0], v01 = p[(size_t)y0 * w + x1], v10 = p[(size_t)y1 * w + x0], v11 = p[(size_t)y1 * w + x1];
      if (pre_div != 1.f) { v00 = __fdiv_rn(v00, pre_div); v01 = __fdiv_rn(v01, pre_div); v10 = __fdiv_rn(v10, pre_div); v11 = __fdiv_rn(v11, pre_div); }
      else { v00 = __fmul_rn(v00, mul); v01 = __fmul_rn(v01, mul); v10 = __fmul_rn(v10, mul); v11 = __fmul_rn(v11, mul); }
      // h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11), unfused
      const float top = __fadd_rn(__fmul_rn(hx, v00), __fmul_rn(lx, v01));
      const float bot = __fadd_rn(__fmul_rn(hx, v10), __fmul_rn(lx, v11));
      v = __fadd_rn(__fmul_rn(hy, top), __fmul_rn(ly, bot));
    }
    out[idx] = v;
    if (out_div) out_div[idx] = __fdiv_rn(v, div);
  }
}

__global__ void sub_channels_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int N,
                                    int Ca, int c_off, int C, size_t HW) {
  const size_t total = (size_t)N * C * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = idx % HW;
    const int c = (int)((idx / HW) % C), n = (int)(idx / ((size_t)C * HW));
    out[idx] = __fsub_rn(a[((size_t)n * Ca + c_off + c) * HW + pix], b[idx]);
  }
}

__global__ void flow_conf_kernel(const float* __restrict__ im1, const float* __restrict__ warp, float* __restrict__ conf, int N,
                                 int C, size_t HW, float thresh) {
  const size_t total = (size_t)N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    float s = 0.f;
    for (int c = 0; c < C; ++c) {
      const float d = __fsub_rn(im1[((size_t)n * C + c) * HW + pix], warp[((size_t)n * C + c) * HW + pix]);
      s = __fadd_rn(s, __fmul_rn(d, d));
    }
    conf[idx] = s < thresh ? 1.f : 0.f;
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_flownet_prep(const float* f0, const float* f1, long long bstride, long long cstride, float* x, float* x1,
                                float* mean_ws, int B, int H, int W, float rgb_max, cudaStream_t s) {
  const size_t HW = (size_t)H * W;
  flownet_mean_kernel<<<B * 3, 256, 0, s>>>(f0, f1, (size_t)bstride, (size_t)cstride, mean_ws, HW);
  flownet_center_kernel<<<grid1d((size_t)B * 6 * HW), 256, 0, s>>>(f0, f1, (size_t)bstride, (size_t)cstride, mean_ws, x, x1, B, HW, rgb_max);
  return cudaGetLastError();
}

cudaError_t launch_resize(const float* in, float* out, float* out_div, int planes, int h, int w, int H, int W, float sh, float sw,
                          float mul, float pre_div, float div, int nearest, cudaStream_t s) {
  resize_kernel<<<grid1d((size_t)planes * H * W), 256, 0, s>>>(in, out, out_div, planes, h, w, H, W, sh, sw, mul, pre_div, div, nearest);
  return cudaGetLastError();
}

cudaError_t launch_sub_channels(const float* a, const float* b, float* out, int N, int Ca, int c_off, int C, int H, int W,
                                cudaStream_t s) {
  sub_channels_kernel<<<grid1d((size_t)N * C * H * W), 256, 0, s>>>(a, b, out, N, Ca, c_off, C, (size_t)H * W);
  return cudaGetLastError();
}

cudaError_t launch_flow_conf(const float* im1, const float* warp, float* conf, int N, int C, int H, int W, float thresh,
                             cudaStream_t s) {
  flow_conf_kernel<<<grid1d((size_t)N * H * W), 256, 0, s>>>(im1, warp, conf, N, C, (size_t)H * W, thresh);
  return cudaGetLastError();
}

}  // namespace v2v
