// Bilinear flow warp of the previous frame, soft occlusion-mask blend and fg/bg composite, fused
// into one HBM pass (fp32 NCHW in / out, 76 B per pixel algorithmic):
//   img_warp  = grid_sample(img_prev[:, -3:], grid + flow / ((dim-1)/2), bilinear, border)
//   img_final = img_raw * w + img_warp * (1 - w)                      models/networks.py:219-221
//   img_final = img_fg * m + img_final * (1 - m) ; img_raw = img_fg * m + img_raw * (1 - m)   :228-230
// plus the stand-alone `resample` (BaseModel.resample, models/base_model.py:189-196) used by the losses.
// The reference omits align_corners (PyTorch 0.4 == True, installed torch == False, SURVEY App. B #2):
// the flag is explicit.  Coordinate arithmetic mirrors get_grid (networks.py:79-93: torch.linspace)
// and ATen's grid_sampler unnormalise / clip so results agree with the oracle to ~1e-6.
#include <cstdlib>
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

// torch.linspace(-1, 1, n)[i] as ATen's CPU kernel computes it (symmetric halves)
__device__ __forceinline__ float linspace_m1p1(int i, int n) {
  const float step = 2.0f / (float)(n - 1);
  return (i < n / 2) ? (-1.0f + step * (float)i) : (1.0f - step * (float)(n - 1 - i));
}

__device__ __forceinline__ float unnormalize(float g, int size, int align_corners) {
  return align_corners ? ((g + 1.f) / 2.f) * (float)(size - 1) : ((g + 1.f) * (float)size - 1.f) / 2.f;
}

struct Bilerp { int x0, x1, y0, y1; float wx, wy; };

__device__ __forceinline__ Bilerp warp_coords(int x, int y, float fx, float fy, int W, int H, int ac) {
  float gx = linspace_m1p1(x, W) + fx / (((float)W - 1.0f) / 2.0f);
  float gy = linspace_m1p1(y, H) + fy / (((float)H - 1.0f) / 2.0f);
  float ix = unnormalize(gx, W, ac), iy = unnormalize(gy, H, ac);
  ix = fminf((float)(W - 1), fmaxf(ix, 0.f));     // padding_mode='border'
  iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  const float x0f = floorf(ix), y0f = floorf(iy);
  Bilerp b;
  b.x0 = (int)x0f; b.y0 = (int)y0f;
  b.x1 = min(b.x0 + 1, W - 1); b.y1 = min(b.y0 + 1, H - 1);
  b.wx = ix - x0f; b.wy = iy - y0f;
  return b;
}

__device__ __forceinline__ float bilerp(const float* pl, const Bilerp& b, int W) {
  const float v00 = __ldg(pl + (size_t)b.y0 * W + b.x0), v01 = __ldg(pl + (size_t)b.y0 * W + b.x1);
  const float v10 = __ldg(pl + (size_t)b.y1 * W + b.x0), v11 = __ldg(pl + (size_t)b.y1 * W + b.x1);
  // same association as ATen: nw*(1-wx)(1-wy) + ne*wx(1-wy) + sw*(1-wx)wy + se*wx*wy
  return v00 * ((1.f - b.wx) * (1.f - b.wy)) + v01 * (b.wx * (1.f - b.wy)) + v10 * ((1.f - b.wx) * b.wy) +
         v11 * (b.wx * b.wy);
}

__global__ void composite_kernel(CompositeParams p) {
  pdl_prologue();
  const size_t HW = (size_t)p.H * p.W;
  const size_t total = (size_t)p.N * HW;
  float* raw = reinterpret_cast<float*>(p.io[p.s_raw]);          // in: tanh head output; out: composited
  float* fin = reinterpret_cast<float*>(p.io[p.s_final]);
  float* raw_out = p.s_raw_out >= 0 ? reinterpret_cast<float*>(p.io[p.s_raw_out]) : raw;
  const float* flow = p.s_flow >= 0 ? reinterpret_cast<const float*>(p.io[p.s_flow]) : nullptr;
  const float* wgt = p.s_weight >= 0 ? reinterpret_cast<const float*>(p.io[p.s_weight]) : nullptr;
  const float* prev = p.s_prev >= 0 ? reinterpret_cast<const float*>(p.io[p.s_prev]) : nullptr;
  const float* fg = p.s_fg >= 0 ? reinterpret_cast<const float*>(p.io[p.s_fg]) : nullptr;
  const float* mask = p.s_mask >= 0 ? reinterpret_cast<const float*>(p.io[p.s_mask]) : nullptr;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    const int y = (int)(pix / p.W), x = (int)(pix - (size_t)y * p.W);
    float r[3], f[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = raw[((size_t)n * 3 + c) * HW + pix];
    if (p.use_warp) {
      const float fx = flow[((size_t)n * 2 + 0) * HW + pix], fy = flow[((size_t)n * 2 + 1) * HW + pix];
      const float w = wgt[(size_t)n * HW + pix];
      const Bilerp b = warp_coords(x, y, fx, fy, p.W, p.H, p.align_corners);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float wv = bilerp(prev + ((size_t)n * p.prev_C + (p.prev_C - 3) + c) * HW, b, p.W);
        f[c] = r[c] * w + wv * (1.f - w);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) f[c] = r[c];
    }
    if (fg) {
      const float m = mask[(size_t)n * HW + pix];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float g = fg[((size_t)n * 3 + c) * HW + pix];
        f[c] = g * m + f[c] * (1.f - m);
        r[c] = g * m + r[c] * (1.f - m);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      fin[((size_t)n * 3 + c) * HW + pix] = f[c];
      if (fg || raw_out != raw) raw_out[((size_t)n * 3 + c) * HW + pix] = r[c];
    }
  }
}

// Vectorised form (W % 4 == 0): a thread owns 4 consecutive pixels of one row, so every streamed tensor moves as 16-byte
// loads / stores with no per-pixel index division (grid = x blocks, rows, images); the warp gathers stay scalar (they hit
// L2: neighbouring pixels sample neighbouring texels).  Same per-pixel arithmetic as composite_kernel -> identical results.
__global__ void __launch_bounds__(128) composite_vec4_kernel(CompositeParams p) {
  pdl_prologue();
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y, n = blockIdx.z;
  if (x0 >= p.W) return;
  const size_t HW = (size_t)p.H * p.W, pix = (size_t)y * p.W + x0;
  float* raw = reinterpret_cast<float*>(p.io[p.s_raw]);
  float* fin = reinterpret_cast<float*>(p.io[p.s_final]);
  float* raw_out = p.s_raw_out >= 0 ? reinterpret_cast<float*>(p.io[p.s_raw_out]) : raw;
  const float* fg = p.s_fg >= 0 ? reinterpret_cast<const float*>(p.io[p.s_fg]) : nullptr;
  auto ld4 = [&](const float* base, int c, int C) { return *reinterpret_cast<const float4*>(base + ((size_t)n * C + c) * HW + pix); };
  float4 r[3], f[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) r[c] = ld4(raw, c, 3);
  if (p.use_warp) {
    const float* flow = reinterpret_cast<const float*>(p.io[p.s_flow]);
    const float* prev = reinterpret_cast<const float*>(p.io[p.s_prev]);
    const float4 fx = ld4(flow, 0, 2), fy = ld4(flow, 1, 2);
    const float4 w = ld4(reinterpret_cast<const float*>(p.io[p.s_weight]), 0, 1);
    const float fxs[4] = {fx.x, fx.y, fx.z, fx.w}, fys[4] = {fy.x, fy.y, fy.z, fy.w}, ws[4] = {w.x, w.y, w.z, w.w};
    float o[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const Bilerp b = warp_coords(x0 + j, y, fxs[j], fys[j], p.W, p.H, p.align_corners);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float wv = bilerp(prev + ((size_t)n * p.prev_C + (p.prev_C - 3) + c) * HW, b, p.W);
        const float rc = reinterpret_cast<const float*>(&r[c])[j];
        o[c][j] = rc * ws[j] + wv * (1.f - ws[j]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) f[c] = make_float4(o[c][0], o[c][1], o[c][2], o[c][3]);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) f[c] = r[c];
  }
  if (fg) {
    const float4 m = ld4(reinterpret_cast<const float*>(p.io[p.s_mask]), 0, 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4 g = ld4(fg, c, 3);
      f[c] = make_float4(g.x * m.x + f[c].x * (1.f - m.x), g.y * m.y + f[c].y * (1.f - m.y), g.z * m.z + f[c].z * (1.f - m.z),
                         g.w * m.w + f[c].w * (1.f - m.w));
      r[c] = make_float4(g.x * m.x + r[c].x * (1.f - m.x), g.y * m.y + r[c].y * (1.f - m.y), g.z * m.z + r[c].z * (1.f - m.z),
                         g.w * m.w + r[c].w * (1.f - m.w));
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    *reinterpret_cast<float4*>(fin + ((size_t)n * 3 + c) * HW + pix) = f[c];
    if (fg || raw_out != raw) *reinterpret_cast<float4*>(raw_out + ((size_t)n * 3 + c) * HW + pix) = r[c];
  }
}

// stand-alone resample(image, flow): image (N,C,H,W), flow (N,2,H,W) in pixels -> (N,C,H,W)
__global__ void resample_kernel(const float* __restrict__ img, const float* __restrict__ flow, float* __restrict__ out,
                                int N, int C, int H, int W, int align_corners) {
  const size_t HW = (size_t)H * W, total = (size_t)N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    const int y = (int)(pix / W), x = (int)(pix - (size_t)y * W);
    const Bilerp b = warp_coords(x, y, flow[((size_t)n * 2) * HW + pix], flow[((size_t)n * 2 + 1) * HW + pix], W, H,
                                 align_corners);
    for (int c = 0; c < C; ++c) out[((size_t)n * C + c) * HW + pix] = bilerp(img + ((size_t)n * C + c) * HW, b, W);
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_composite(const CompositeParams& p, cudaStream_t stream) {
  static const bool vec_ok = [] { const char* e = getenv("V2V_COMPOSITE_VEC"); return !(e && e[0] == '0'); }();
  if (vec_ok && p.W % 4 == 0 && p.H <= 65535 && p.N <= 65535)
    return launch_pdl(composite_vec4_kernel, dim3((p.W / 4 + 127) / 128, p.H, p.N), dim3(128), 0, stream, p);
  return launch_pdl(composite_kernel, dim3(grid1d((size_t)p.N * p.H * p.W)), dim3(256), 0, stream, p);
  return cudaGetLastError();
}

cudaError_t launch_resample(const float* img, const float* flow, float* out, int N, int C, int H, int W,
                            int align_corners, cudaStream_t stream) {
  resample_kernel<<<grid1d((size_t)N * H * W), 256, 0, stream>>>(img, flow, out, N, C, H, W, align_corners);
  return cudaGetLastError();
}

}  // namespace v2v
