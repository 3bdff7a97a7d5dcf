// HBM-bound helpers of the Vid2VidModelG level (fp32 NCHW, coalesced along x):
//   onehot_edges : label ids + instance ids -> one-hot(+edge) input tensor
//                  (Vid2VidModelG.encode_input, models/vid2vid_model_G.py:86-112; BaseModel.get_edges,
//                   models/base_model.py:146-152)
//   avgpool3s2   : AvgPool2d(3, stride 2, pad 1, count_include_pad=False) pyramid level
//                  (BaseModel.build_pyr, models/base_model.py:122-134; networks.py:400,652)
//   fg_mask      : clamp(sum of fg label channels, 0, 1)  (compute_mask, vid2vid_model_G.py:322-330)
#include "../../include/v2v_b200.h"
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

// out (F, label_nc + use_inst, H, W) ; labels / inst (F, H, W) float ids ; F = b * t frames
__global__ void onehot_edges_kernel(const float* __restrict__ labels, const float* __restrict__ inst,
                                    float* __restrict__ out, int F, int label_nc, int use_inst, int H, int W) {
  const size_t HW = (size_t)H * W;
  const int Cout = label_nc + (use_inst ? 1 : 0);
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;   // grid = (x blocks, row, frame)
  if (x < W) {
    const size_t pix = (size_t)y * W + x;
    const size_t idx = (size_t)f * HW + pix;
    const int lab = (int)labels[idx];
    float* o = out + (size_t)f * Cout * HW + pix;
    for (int c = 0; c < label_nc; ++c) o[(size_t)c * HW] = (c == lab) ? 1.f : 0.f;
    if (use_inst) {
      const float* ip = inst + (size_t)f * HW;
      const float v = ip[pix];
      bool e = false;
      if (x > 0) e |= (ip[pix - 1] != v);
      if (x < W - 1) e |= (ip[pix + 1] != v);
      if (y > 0) e |= (ip[pix - W] != v);
      if (y < H - 1) e |= (ip[pix + W] != v);
      o[(size_t)label_nc * HW] = e ? 1.f : 0.f;
    }
  }
}

// in (P, H, W) -> out (P, H/2, W/2) planes; grid = (x blocks, output row, plane): no per-element divisions
__global__ void __launch_bounds__(256) avgpool3s2_kernel(const float* __restrict__ in, float* __restrict__ out, int P, int H, int W,
                                                         int Ho, int Wo) {
  const int xo = blockIdx.x * blockDim.x + threadIdx.x;
  if (xo >= Wo) return;
  const int yo = blockIdx.y;
  for (int pl = blockIdx.z; pl < P; pl += gridDim.z) {
    const float* ip = in + (size_t)pl * H * W;
    float s = 0.f;
    int cnt = 0;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const int y = 2 * yo + dy;
      if (y < 0 || y >= H) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int x = 2 * xo + dx;
        if (x < 0 || x >= W) continue;
        s += __ldg(ip + (size_t)y * W + x);
        ++cnt;
      }
    }
    out[((size_t)pl * Ho + yo) * Wo + xo] = s / (float)cnt;
  }
}

// W % 4 == 0: a thread produces two adjacent outputs from one 16-byte load (+ one scalar) per input row: 3x fewer load
// instructions and twice the bytes in flight per thread (the scalar kernel above is latency bound).  Same summation order ->
// same results.
__global__ void __launch_bounds__(128) avgpool3s2_vec_kernel(const float* __restrict__ in, float* __restrict__ out, int P, int H, int W,
                                                             int Ho, int Wo) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;      // output pair index: outputs 2k, 2k + 1 read input columns 4k-1 .. 4k+3
  if (4 * k >= W) return;
  const int yo = blockIdx.y;
  for (int pl = blockIdx.z; pl < P; pl += gridDim.z) {
    const float* ip = in + (size_t)pl * H * W;
    float s0 = 0.f, s1 = 0.f;
    int rows = 0;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const int y = 2 * yo + dy;
      if (y < 0 || y >= H) continue;
      ++rows;
      const float* rp = ip + (size_t)y * W + 4 * k;
      const float4 v = *reinterpret_cast<const float4*>(rp);
      if (k > 0) s0 += __ldg(rp - 1);
      s0 += v.x; s0 += v.y;
      s1 += v.y; s1 += v.z; s1 += v.w;
    }
    const int c0 = (k > 0 ? 3 : 2), c1 = 3;                  // 4k + 3 <= W - 1 always when W % 4 == 0
    *reinterpret_cast<float2*>(out + ((size_t)pl * Ho + yo) * Wo + 2 * k) = make_float2(s0 / (float)(rows * c0), s1 / (float)(rows * c1));
  }
}

// real_A (B, T, C, H, W) -> mask (B, 1, H, W) for frame index t
struct FgLabels { int v[16]; };
__global__ void fg_mask_kernel(const float* __restrict__ real_A, float* __restrict__ mask, int B, int T, int C, int H,
                               int W, int t, FgLabels labels, int n_labels) {
  const size_t HW = (size_t)H * W, total = (size_t)B * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / HW);
    const size_t pix = idx - (size_t)b * HW;
    float s = 0.f;
    for (int i = 0; i < n_labels; ++i) s += real_A[(((size_t)b * T + t) * C + labels.v[i]) * HW + pix];
    mask[idx] = fminf(fmaxf(s, 0.f), 1.f);
  }
}

// Streaming input: B windows (B, T, HW) float ids, oldest frame first; drop each window's oldest frame, append its clip's
// new frame (B, HW) converted from uint8 / int32 / float (dtype 0 / 1 / 2).  One thread per (clip, pixel) walks the frames,
// so the in-place shift has no hazard.
__global__ void ids_window_push_kernel(float* __restrict__ window, const void* __restrict__ frame, int dtype, int T, size_t HW,
                                       size_t total) {
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t b = idx / HW, pix = idx - b * HW;
    float* win = window + b * T * HW;
    for (int t = 0; t + 1 < T; ++t) win[(size_t)t * HW + pix] = win[(size_t)(t + 1) * HW + pix];
    float v;
    if (dtype == 0) v = (float)reinterpret_cast<const uint8_t*>(frame)[idx];
    else if (dtype == 1) v = (float)reinterpret_cast<const int*>(frame)[idx];
    else v = reinterpret_cast<const float*>(frame)[idx];
    win[(size_t)(T - 1) * HW + pix] = v;
  }
}

// Slot streams: window (B, T, C*HW) float, frames (B, C*HW) uint8 / int32 / float (dtype 0 / 1 / 2).  Each slot's op
// (V2V_SLOT_*) travels by value; one thread per (slot, element) walks the frames, so the in-place shift has no hazard.
struct SlotOps { int v[V2V_MAX_SLOTS]; };
__global__ void slots_window_push_kernel(float* __restrict__ window, const void* __restrict__ frames, int dtype, int T, size_t E,
                                         size_t total, SlotOps ops) {
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t b = idx / E, e = idx - b * E;
    const int op = ops.v[b];
    if (op == V2V_SLOT_KEEP) continue;
    float* win = window + b * T * E;
    if (op == V2V_SLOT_PUSH)
      for (int t = 0; t + 1 < T; ++t) win[(size_t)t * E + e] = win[(size_t)(t + 1) * E + e];
    else
      for (int t = 0; t + 1 < T; ++t) win[(size_t)t * E + e] = 0.f;
    float v = 0.f;
    if (op != V2V_SLOT_CLEAR) {
      if (dtype == 0) v = (float)reinterpret_cast<const uint8_t*>(frames)[idx];
      else if (dtype == 1) v = (float)reinterpret_cast<const int*>(frames)[idx];
      else v = reinterpret_cast<const float*>(frames)[idx];
    }
    win[(size_t)(T - 1) * E + e] = v;
  }
}

// util.tensor2im (util/util.py:48-71) per image: (B,C,H,W) float in [-1,1] -> (B,H,W,C) uint8 = clip((x + 1) / 2 * 255, 0, 255)
// truncated
__global__ void tensor2im_u8_kernel(const float* __restrict__ img, uint8_t* __restrict__ out, int C, size_t HW, size_t total) {
  for (size_t pix = blockIdx.x * (size_t)blockDim.x + threadIdx.x; pix < total; pix += (size_t)gridDim.x * blockDim.x) {
    const size_t b = pix / HW, p = pix - b * HW;
    for (int c = 0; c < C; ++c) {
      float v = __fmul_rn(__fdiv_rn(__fadd_rn(img[(b * C + c) * HW + p], 1.f), 2.0f), 255.0f);
      v = fminf(fmaxf(v, 0.f), 255.f);
      out[pix * C + c] = (uint8_t)v;
    }
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_onehot_edges(const float* labels, const float* inst, float* out, int F, int label_nc, int use_inst,
                                int H, int W, cudaStream_t s) {
  dim3 grid((W + 255) / 256, H, F);
  onehot_edges_kernel<<<grid, 256, 0, s>>>(labels, inst, out, F, label_nc, use_inst, H, W);
  return cudaGetLastError();
}
cudaError_t launch_avgpool3s2(const float* in, float* out, int P, int H, int W, cudaStream_t s) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  // the vector kernel loads float4 rows and stores float2 pairs: a caller's view at an odd float offset takes the scalar one
  const bool aligned = (reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
  if (W % 4 == 0 && W >= 4 && aligned) {
    dim3 grid((W / 4 + 127) / 128, Ho, P < 64 ? P : 64);
    avgpool3s2_vec_kernel<<<grid, 128, 0, s>>>(in, out, P, H, W, Ho, Wo);
    return cudaGetLastError();
  }
  dim3 grid((Wo + 255) / 256, Ho, P < 64 ? P : 64);
  avgpool3s2_kernel<<<grid, 256, 0, s>>>(in, out, P, H, W, Ho, Wo);
  return cudaGetLastError();
}
cudaError_t launch_ids_window_push(float* window, const void* frame, int dtype, int B, int T, int H, int W, cudaStream_t s) {
  ids_window_push_kernel<<<grid1d((size_t)B * H * W), 256, 0, s>>>(window, frame, dtype, T, (size_t)H * W, (size_t)B * H * W);
  return cudaGetLastError();
}
cudaError_t launch_slots_window_push(float* window, const void* frames, int dtype, int B, int T, int C, int H, int W, const int* ops,
                                    cudaStream_t s) {
  SlotOps o{};
  for (int b = 0; b < B; ++b) o.v[b] = ops[b];
  const size_t E = (size_t)C * H * W;
  slots_window_push_kernel<<<grid1d((size_t)B * E), 256, 0, s>>>(window, frames, dtype, T, E, (size_t)B * E, o);
  return cudaGetLastError();
}
cudaError_t launch_tensor2im_u8(const float* img, uint8_t* out, int B, int C, int H, int W, cudaStream_t s) {
  tensor2im_u8_kernel<<<grid1d((size_t)B * H * W), 256, 0, s>>>(img, out, C, (size_t)H * W, (size_t)B * H * W);
  return cudaGetLastError();
}
cudaError_t launch_fg_mask(const float* real_A, float* mask, int B, int T, int C, int H, int W, int t,
                           FgLabels labels, int n_labels, cudaStream_t s) {
  fg_mask_kernel<<<grid1d((size_t)B * H * W), 256, 0, s>>>(real_A, mask, B, T, C, H, W, t, labels, n_labels);
  return cudaGetLastError();
}

}  // namespace v2v
