// sm_90a replacements for the three native FlowNet2 operators of the reference
// (models/flownet2_pytorch/networks/{correlation,resample2d,channelnorm}_package/*.cu).
// All three are fp32, NCHW, HBM/L2-bound; outputs are caller-owned (C-ABI in include/v2v_b200.h).
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

// ---------------------------------------------------------------------------------------------
// Correlation (correlation_cuda_kernel.cu:73-147, kernel_size == 1):
//   out[n][(tj+dr)*D + (ti+dr)][y][x] = (1/C) * sum_c f1[n][c][y1][x1] * f2[n][c][y1 + tj*s2][x1 + ti*s2]
// with (y1, x1) = (y*s1 + max_disp - pad, x*s1 + max_disp - pad) in unpadded coordinates and zero
// outside the image.  Block = one output row segment of 32 pixels; f1 / f2 row patches are staged in
// shared memory channel-chunk by channel-chunk ([c][x], so lanes read consecutive words); each of the
// 32 x 7 threads keeps 3 displacement accumulators per displacement row.
static constexpr int CORR_TX = 32;     // output pixels per block
static constexpr int CORR_CC = 32;     // channels per smem chunk
static constexpr int CORR_MAXD = 21;   // displacement window (2*dr+1) supported by the register blocking

__global__ void __launch_bounds__(CORR_TX * 7)
correlation_kernel(const float* __restrict__ f1, const float* __restrict__ f2, float* __restrict__ out, int C, int H,
                   int W, int outH, int outW, int pad, int max_disp, int s1, int s2) {
  extern __shared__ float sm[];
  const int dr = max_disp / s2, D = 2 * dr + 1;
  const int PW = (CORR_TX - 1) * s1 + 2 * dr * s2 + 1;        // f2 patch width
  float* s_f1 = sm;                                          // [CC][TX]
  float* s_f2 = sm + CORR_CC * CORR_TX;                      // [CC][PW]
  const int n = blockIdx.z, yo = blockIdx.y, xo0 = blockIdx.x * CORR_TX;
  const int px = threadIdx.x % CORR_TX, tg = threadIdx.x / CORR_TX;   // tg in [0,7)
  const int y1 = yo * s1 + max_disp - pad;
  const int x1_0 = xo0 * s1 + max_disp - pad;                // x1 of pixel 0 of the tile
  const size_t HW = (size_t)H * W;
  const float inv = 1.0f / (float)C;
  for (int tj = -dr; tj <= dr; ++tj) {
    const int y2 = y1 + tj * s2;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int c0 = 0; c0 < C; c0 += CORR_CC) {
      __syncthreads();
      for (int i = threadIdx.x; i < CORR_CC * CORR_TX; i += blockDim.x) {
        const int c = i / CORR_TX, x = i % CORR_TX;
        const int xx = x1_0 + x * s1;
        float v = 0.f;
        if (c0 + c < C && y1 >= 0 && y1 < H && xx >= 0 && xx < W) v = f1[((size_t)n * C + c0 + c) * HW + (size_t)y1 * W + xx];
        s_f1[c * CORR_TX + x] = v;
      }
      for (int i = threadIdx.x; i < CORR_CC * PW; i += blockDim.x) {
        const int c = i / PW, x = i % PW;
        const int xx = x1_0 - dr * s2 + x;
        float v = 0.f;
        if (c0 + c < C && y2 >= 0 && y2 < H && xx >= 0 && xx < W) v = f2[((size_t)n * C + c0 + c) * HW + (size_t)y2 * W + xx];
        s_f2[c * PW + x] = v;
      }
      __syncthreads();
#pragma unroll 4
      for (int c = 0; c < CORR_CC; ++c) {
        const float a = s_f1[c * CORR_TX + px];
        const float* row = s_f2 + c * PW + px * s1;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int ti = tg + 7 * k;                         // displacement index 0..D-1
          if (ti < D) acc[k] = fmaf(a, row[ti * s2], acc[k]);
        }
      }
    }
    const int xo = xo0 + px;
    if (xo < outW) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int ti = tg + 7 * k;
        if (ti < D) {
          const int tc = (tj + dr) * D + ti;
          out[(((size_t)n * D * D + tc) * outH + yo) * outW + xo] = acc[k] * inv;
        }
      }
    }
  }
}

cudaError_t launch_correlation(const float* f1, const float* f2, float* out, int N, int C, int H, int W, int pad,
                               int kernel_size, int max_disp, int s1, int s2, cudaStream_t stream) {
  if (kernel_size != 1 || s2 < 1 || s1 < 1) return cudaErrorInvalidValue;
  const int dr = max_disp / s2, D = 2 * dr + 1;
  if (D > CORR_MAXD) return cudaErrorInvalidValue;
  const int border = max_disp;   // kernel_radius == 0
  const int outH = (int)ceilf((float)(H + 2 * pad - 2 * border) / (float)s1);
  const int outW = (int)ceilf((float)(W + 2 * pad - 2 * border) / (float)s1);
  const int PW = (CORR_TX - 1) * s1 + 2 * dr * s2 + 1;
  const size_t smem = sizeof(float) * CORR_CC * (CORR_TX + PW);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(correlation_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  dim3 grid((outW + CORR_TX - 1) / CORR_TX, outH, N);
  correlation_kernel<<<grid, CORR_TX * 7, smem, stream>>>(f1, f2, out, C, H, W, outH, outW, pad, max_disp, s1, s2);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Resample2d (resample2d_kernel.cu:15-64, kernel_size == 1): backward bilinear warp with the
// reference's own floor/clamp rule; one thread per pixel, channels looped (flow read once).
__global__ void resample2d_kernel(const float* __restrict__ in1, const float* __restrict__ flow, float* __restrict__ out,
                                  int N, int C, int H, int W, int inH, int inW) {
  const size_t HW = (size_t)H * W, total = (size_t)N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    const int y = (int)(pix / W), x = (int)(pix - (size_t)y * W);
    const float dx = flow[((size_t)n * 2 + 0) * HW + pix], dy = flow[((size_t)n * 2 + 1) * HW + pix];
    const float xf = (float)x + dx, yf = (float)y + dy;
    const float alpha = xf - floorf(xf), beta = yf - floorf(yf);
    // the reference clamps against the OUTPUT extent (dim_w/dim_h of `output`), :48-51
    const int xL = max(min((int)floorf(xf), W - 1), 0), xR = max(min((int)floorf(xf) + 1, W - 1), 0);
    const int yT = max(min((int)floorf(yf), H - 1), 0), yB = max(min((int)floorf(yf) + 1, H - 1), 0);
    // weights as the reference forms them (:55-58): the three terms containing `1.` are promoted to double,
    // `(alpha)*(beta) * v` stays in float; explicit _rn intrinsics keep ptxas from fusing (the oracle is unfused C)
    const double w00 = __dmul_rn(1. - alpha, 1. - beta), w01 = __dmul_rn((double)alpha, 1. - beta);
    const double w10 = __dmul_rn(1. - alpha, (double)beta);
    const float w11 = __fmul_rn(alpha, beta);
    const size_t inHW = (size_t)inH * inW;
    for (int c = 0; c < C; ++c) {
      const float* pl = in1 + ((size_t)n * C + c) * inHW;
      float val = 0.f;
      val = __fadd_rn(val, (float)__dmul_rn(w00, (double)pl[(size_t)yT * inW + xL]));
      val = __fadd_rn(val, (float)__dmul_rn(w01, (double)pl[(size_t)yT * inW + xR]));
      val = __fadd_rn(val, (float)__dmul_rn(w10, (double)pl[(size_t)yB * inW + xL]));
      val = __fadd_rn(val, __fmul_rn(w11, pl[(size_t)yB * inW + xR]));
      out[((size_t)n * C + c) * HW + pix] = val;
    }
  }
}

// ChannelNorm (channelnorm_kernel.cu:18-60): out[n][0][y][x] = sqrt(sum_c in[n][c][y][x]^2)
__global__ void channelnorm_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int C, size_t HW) {
  const size_t total = (size_t)N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    float r = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = in[((size_t)n * C + c) * HW + pix];
      r = __fadd_rn(r, __fmul_rn(v, v));      // unfused, like the C restatement
    }
    out[idx] = sqrtf(r);
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_resample2d(const float* in1, const float* flow, float* out, int N, int C, int H, int W, int inH,
                              int inW, int kernel_size, cudaStream_t stream) {
  if (kernel_size != 1) return cudaErrorInvalidValue;
  resample2d_kernel<<<grid1d((size_t)N * H * W), 256, 0, stream>>>(in1, flow, out, N, C, H, W, inH, inW);
  return cudaGetLastError();
}

cudaError_t launch_channelnorm(const float* in, float* out, int N, int C, int H, int W, int norm_deg,
                               cudaStream_t stream) {
  if (norm_deg != 2) return cudaErrorInvalidValue;
  channelnorm_kernel<<<grid1d((size_t)N * H * W), 256, 0, stream>>>(in, out, N, C, (size_t)H * W);
  return cudaGetLastError();
}

}  // namespace v2v
