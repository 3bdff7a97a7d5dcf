// Backward kernels of the training step (SURVEY 8 row T; reference: autograd through models/networks.py:203-232,296-325,
// 663-725 as driven by train.py:50-93).  First correct CUDA path: fp32 SIMT, shared-memory tiled implicit GEMMs that read the
// forward plan's own buffers (halo-padded NHWC activations, fp32 / bf16 raw conv outputs, saved batch statistics) and
// dense NHWC fp32 gradient buffers.  The forward pass stays on the wgmma kernel.
//   conv_dgrad   dXpad[n][py][px][ci] = sum_{taps, co} dY[n][oy][ox][co] * W      (padded input extent; reflect / zero halo
//                                                                                   folded back by fold_pad_kernel)
//   conv_wgrad   dW[co][ci][ky][kx]  += sum_{n, oy, ox} dY[n][oy][ox][co] * Xpad[n][oy*s+ky][ox*s+kx][ci]   (split over pixels)
//   norm_bwd     train-mode BatchNorm + (Leaky)ReLU backward (two passes: per-channel sums, then apply) and the norm-less
//                bias + activation unit; residual / skip addends receive the incoming gradient
//   head_bwd     tanh / sigmoid / scale heads: caller gradient planes (fp32 NCHW) -> dense NHWC dz
//   composite_bwd  warp + blend + fg composite (networks.py:219-221,228-230): grads of raw, flow, weight, fg and, when the
//                caller asks for it, of the warped previous frame (grid_sample's input gradient, scattered with fp32 atomics)
//   grad import / export between caller fp32 NCHW gradient tensors and the dense NHWC gradient buffers
#include "ptx.cuh"
#include "v2v_internal.h"
#include "backward.h"

namespace v2v {

__device__ __forceinline__ float act_load(const ActDesc& a, size_t off) {      // one value of a (possibly split) activation
  float v = __bfloat162float(a.base[off]);
  if (a.split) v += __bfloat162float(a.base[off + a.C]);
  return v;
}

__device__ __forceinline__ float w_fwd(const BwdConv& p, int co, int ci, int ky, int kx) {
  // forward weight of (output channel co, input channel ci): conv [Cout][Cin][kh][kw]; transposed conv [Cin][Cout][kh][kw]
  if (p.transposed) return p.w[(((size_t)ci * p.Cout + co) * p.kh + ky) * p.kw + kx];
  if (p.w2 && co >= p.Cout1) return p.w2[(((size_t)(co - p.Cout1) * p.Cin + ci) * p.kh + ky) * p.kw + kx];
  return p.w[(((size_t)co * p.Cin + ci) * p.kh + ky) * p.kw + kx];
}

// ---------------------------------------------------------------------------------------------------- data gradient
// Block: 16 positions x 64 input channels; thread (tx = ci lane 0..63, ty = 0..3) owns 4 positions x 1 channel.
// For every tap the block stages W[32 co][64 ci] and dY[16 positions][32 co] in shared memory.
// conv:        position = padded input pixel (py, px); tap (ky, kx) contributes when (py - ky) % s == 0, oy = (py - ky) / s
// transposed:  position = input pixel (iy, ix); tap contributes dY[iy * 2 - pad + ky][ix * 2 - pad + kx]
__global__ void __launch_bounds__(256) conv_dgrad_kernel(BwdConv p) {
  __shared__ float sW[32][65];
  __shared__ float sY[16][33];
  __shared__ int sOff[16];      // per position: dY pixel offset for the current tap, or -1
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int PH = p.transposed ? p.H : p.H + 2 * p.pad, PW = p.transposed ? p.W : p.W + 2 * p.pad;
  const long long npos = (long long)p.N * PH * PW;
  const long long pos0 = (long long)blockIdx.x * 16;
  const int ci = blockIdx.y * 64 + tx;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ky = 0; ky < p.kh; ++ky)
    for (int kx = 0; kx < p.kw; ++kx) {
      __syncthreads();
      if (threadIdx.x < 16) {
        const long long pos = pos0 + threadIdx.x;
        int off = -1;
        if (pos < npos) {
          const int px = (int)(pos % PW), py = (int)((pos / PW) % PH), n = (int)(pos / ((long long)PW * PH));
          int oy, ox;
          bool ok;
          if (p.transposed) { oy = py * p.stride - p.pad + ky; ox = px * p.stride - p.pad + kx; ok = true; }
          else {
            const int ry = py - ky, rx = px - kx;
            ok = ry >= 0 && rx >= 0 && (ry % p.stride) == 0 && (rx % p.stride) == 0;
            oy = ry / p.stride; ox = rx / p.stride;
          }
          if (ok && oy >= 0 && oy < p.oh && ox >= 0 && ox < p.ow) off = (n * p.oh + oy) * p.ow + ox;
        }
        sOff[threadIdx.x] = off;
      }
      for (int co0 = 0; co0 < p.Cout; co0 += 32) {
        __syncthreads();
        for (int r = ty; r < 32; r += 4) {
          const int co = co0 + r;
          sW[r][tx] = (co < p.Cout && ci < p.Cin) ? w_fwd(p, co, ci, ky, kx) : 0.f;
        }
        for (int i = threadIdx.x; i < 16 * 32; i += 256) {
          const int ps = i >> 5, c = i & 31;
          const int off = sOff[ps];
          sY[ps][c] = (off >= 0 && co0 + c < p.Cout) ? p.dy[(size_t)off * p.dy_C + co0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int c = 0; c < 32; ++c) {
          const float w = sW[c][tx];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j] = fmaf(sY[ty * 4 + j][c], w, acc[j]);
        }
      }
    }
  if (ci >= p.Cin) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long pos = pos0 + ty * 4 + j;
    if (pos >= npos) continue;
    if (p.transposed) {
      p.dx[(size_t)pos * p.Cin + ci] += acc[j];                       // positions are interior pixels of the dense grad buffer
    } else {
      // fold the padded position back into the interior: reflect halo mirrors, zero halo is dropped
      const int px = (int)(pos % PW) - p.pad, py = (int)((pos / PW) % PH) - p.pad, n = (int)(pos / ((long long)PW * PH));
      int y = py, x = px;
      const bool halo = (y < 0 || y >= p.H || x < 0 || x >= p.W);
      if (halo) {
        if (p.pad_mode != PAD_REFLECT) continue;
        if (y < 0) y = -y; if (y >= p.H) y = 2 * (p.H - 1) - y;
        if (x < 0) x = -x; if (x >= p.W) x = 2 * (p.W - 1) - x;
      }
      atomicAdd(&p.dx[(((size_t)n * p.H + y) * p.W + x) * p.Cin + ci], acc[j]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- weight gradient
// Block: tile of 32 co x 32 ci for one tap over a range of output pixels (split-K); 256 threads = 16 x 16, 2 x 2 outputs each.
__global__ void __launch_bounds__(256) conv_wgrad_kernel(BwdConv p, int ksplit) {
  __shared__ float sY[32][33];      // [pixel][co]
  __shared__ float sX[32][33];      // [pixel][ci]
  const int tiles_ci = (p.Cin + 31) / 32;
  const int co0 = (blockIdx.x / tiles_ci) * 32, ci0 = (blockIdx.x % tiles_ci) * 32;
  const int tap = blockIdx.y, ky = tap / p.kw, kx = tap % p.kw;
  // pixels of the "driving" grid: conv -> output pixels; transposed conv -> input pixels
  const int gh = p.transposed ? p.H : p.oh, gw = p.transposed ? p.W : p.ow;
  const long long npix = (long long)p.N * gh * gw;
  const long long per = (npix + ksplit - 1) / ksplit;
  const long long k_begin = (long long)blockIdx.z * per, k_end = min(npix, k_begin + per);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (long long k0 = k_begin; k0 < k_end; k0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 32; i += 256) {
      const int ps = i >> 5, c = i & 31;
      const long long pix = k0 + ps;
      float vy = 0.f, vx = 0.f;
      if (pix < k_end) {
        const int gx = (int)(pix % gw), gy = (int)((pix / gw) % gh), n = (int)(pix / ((long long)gw * gh));
        if (!p.transposed) {
          if (co0 + c < p.Cout) vy = p.dy[(size_t)pix * p.dy_C + co0 + c];
          if (ci0 + c < p.Cin) vx = act_load(p.x, p.x.offset(n, gy * p.stride + ky - p.pad, gx * p.stride + kx - p.pad) + ci0 + c);
        } else {
          const int oy = gy * p.stride - p.pad + ky, ox = gx * p.stride - p.pad + kx;
          if (oy >= 0 && oy < p.oh && ox >= 0 && ox < p.ow) {
            if (co0 + c < p.Cout) vy = p.dy[(((size_t)n * p.oh + oy) * p.ow + ox) * p.dy_C + co0 + c];
            if (ci0 + c < p.Cin) vx = act_load(p.x, p.x.offset(n, gy, gx) + ci0 + c);
          }
        }
      }
      sY[ps][c] = vy;
      sX[ps][c] = vx;
    }
    __syncthreads();
#pragma unroll 8
    for (int ps = 0; ps < 32; ++ps) {
      const float y0 = sY[ps][ty * 2], y1 = sY[ps][ty * 2 + 1], x0 = sX[ps][tx * 2], x1 = sX[ps][tx * 2 + 1];
      acc[0][0] = fmaf(y0, x0, acc[0][0]); acc[0][1] = fmaf(y0, x1, acc[0][1]);
      acc[1][0] = fmaf(y1, x0, acc[1][0]); acc[1][1] = fmaf(y1, x1, acc[1][1]);
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int co = co0 + ty * 2 + a, ci = ci0 + tx * 2 + b;
      if (co >= p.Cout || ci >= p.Cin) continue;
      float* dst;
      if (p.transposed) dst = p.dw + (((size_t)ci * p.Cout + co) * p.kh + ky) * p.kw + kx;
      else if (p.w2 && co >= p.Cout1) dst = p.dw2 ? p.dw2 + (((size_t)(co - p.Cout1) * p.Cin + ci) * p.kh + ky) * p.kw + kx : nullptr;
      else dst = p.dw ? p.dw + (((size_t)co * p.Cin + ci) * p.kh + ky) * p.kw + kx : nullptr;
      if (dst) atomicAdd(dst, acc[a][b]);
    }
}

// per-channel sum of a dense NHWC gradient: dbias[c] += sum_p dy[p][c]
__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ dy, int dy_C, long long npix, int C, float* dbias,
                                                        float* dbias2, int C1) {
  const int c = blockIdx.x;
  float s = 0.f;
  for (long long i = blockIdx.y * (long long)blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.y * blockDim.x)
    s += dy[(size_t)i * dy_C + c];
  __shared__ float sh[256];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float* d = (dbias2 && c >= C1) ? dbias2 + (c - C1) : (dbias ? dbias + c : nullptr);
    if (d) atomicAdd(d, sh[0]);
  }
}

// ---------------------------------------------------------------------------------------------------- norm + activation
__device__ __forceinline__ float raw_load(const RawDesc& r, size_t i) {
  return r.f32 ? reinterpret_cast<const float*>(r.base)[i] : __bfloat162float(reinterpret_cast<const bf16*>(r.base)[i]);
}

// z = raw * scale + shift (pre-activation), dz = dy * act'(z).  sums[0][n][c] += dz, sums[1][n][c] += dz * xhat.
__global__ void __launch_bounds__(256) norm_bwd_reduce_kernel(NormBwd p) {
  const int c = blockIdx.x, n = blockIdx.y;
  const long long HW = (long long)p.H * p.W;
  const float sc = p.scale[(size_t)n * p.stat_stride + c], sh = p.shift[(size_t)n * p.stat_stride + c];
  const float mean = p.mean ? p.mean[(size_t)n * p.stat_stride + c] : 0.f, rstd = p.rstd ? p.rstd[(size_t)n * p.stat_stride + c] : 1.f;
  float s1 = 0.f, s2 = 0.f;
  for (long long i = blockIdx.z * (long long)blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.z * blockDim.x) {
    const size_t pix = (size_t)n * HW + i;
    const float raw = raw_load(p.raw, pix * p.raw.C + p.c_off + c);
    const float z = fmaf(raw, sc, sh);
    float dz = p.dy[pix * p.C + c];
    if (p.act == ACT_RELU) dz = z > 0.f ? dz : 0.f;
    else if (p.act == ACT_LRELU) dz = z > 0.f ? dz : dz * p.slope;
    s1 += dz;
    s2 += dz * (raw - mean) * rstd;
  }
  __shared__ float a1[256], a2[256];
  a1[threadIdx.x] = s1; a2[threadIdx.x] = s2;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) { a1[threadIdx.x] += a1[threadIdx.x + k]; a2[threadIdx.x] += a2[threadIdx.x + k]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int row = p.batch_stats ? 0 : n;        // BatchNorm: one statistic over the batch
    atomicAdd(&p.sums[(size_t)row * p.C + c], a1[0]);
    atomicAdd(&p.sums[((size_t)p.N + row) * p.C + c], a2[0]);
  }
}

// Coalesced form of norm_bwd_reduce_kernel for C % 4 == 0, C <= 1024: a thread owns 4 consecutive channels (one float4 of the
// NHWC rows) and strides over the pixels of its block's chunk; per-block partial sums meet in shared memory, one global atomic
// per channel and block.
__global__ void __launch_bounds__(256) norm_bwd_reduce_vec_kernel(NormBwd p, int chunk) {
  extern __shared__ float sred[];                  // [2][C]
  const int vec = p.C >> 2, ppb = 256 / vec;
  const int n = blockIdx.y;
  const long long HW = (long long)p.H * p.W;
  for (int i = threadIdx.x; i < 2 * p.C; i += 256) sred[i] = 0.f;
  __syncthreads();
  const int c4 = threadIdx.x % vec, pl = threadIdx.x / vec;
  if (pl < ppb) {
    const int c = c4 * 4;
    float sc[4], sh[4], mean[4], rstd[4], s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      sc[j] = p.scale[(size_t)n * p.stat_stride + c + j]; sh[j] = p.shift[(size_t)n * p.stat_stride + c + j];
      mean[j] = p.mean ? p.mean[(size_t)n * p.stat_stride + c + j] : 0.f; rstd[j] = p.rstd ? p.rstd[(size_t)n * p.stat_stride + c + j] : 1.f;
    }
    const long long begin = (long long)blockIdx.x * chunk, end = min(HW, begin + chunk);
    for (long long i = begin + pl; i < end; i += ppb) {
      const size_t pix = (size_t)n * HW + i;
      float raw[4];
      if (p.raw.f32) {
        const float4 r4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.raw.base) + pix * p.raw.C + p.c_off + c);
        raw[0] = r4.x; raw[1] = r4.y; raw[2] = r4.z; raw[3] = r4.w;
      } else {
        const bf16* rp = reinterpret_cast<const bf16*>(p.raw.base) + pix * p.raw.C + p.c_off + c;
#pragma unroll
        for (int j = 0; j < 4; ++j) raw[j] = __bfloat162float(rp[j]);
      }
      const float4 d4 = *reinterpret_cast<const float4*>(p.dy + pix * p.C + c);
      const float dy[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float z = fmaf(raw[j], sc[j], sh[j]);
        float dz = dy[j];
        if (p.act == ACT_RELU) dz = z > 0.f ? dz : 0.f;
        else if (p.act == ACT_LRELU) dz = z > 0.f ? dz : dz * p.slope;
        s1[j] += dz;
        s2[j] += dz * (raw[j] - mean[j]) * rstd[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { atomicAdd(&sred[c + j], s1[j]); atomicAdd(&sred[p.C + c + j], s2[j]); }
  }
  __syncthreads();
  const int row = p.batch_stats ? 0 : n;
  for (int i = threadIdx.x; i < p.C; i += 256) {
    atomicAdd(&p.sums[(size_t)row * p.C + i], sred[i]);
    atomicAdd(&p.sums[((size_t)p.N + row) * p.C + i], sred[p.C + i]);
  }
}

// draw = gamma * rstd * (dz - mean(dz) - xhat * mean(dz * xhat))   (train-mode norm)   or   draw = dz (norm-less unit);
// the addends of the unit (residual / skip inputs) receive dy unchanged.
__global__ void __launch_bounds__(256) norm_bwd_apply_kernel(NormBwd p) {
  const long long total = (long long)p.N * p.H * p.W * p.C;
  const long long HW = (long long)p.H * p.W;
  const float inv_m = 1.f / (float)((p.batch_stats ? p.N : 1) * HW);
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % p.C);
    const size_t pix = (size_t)(idx / p.C);
    const int n = (int)(pix / HW);
    const float sc = p.scale[(size_t)n * p.stat_stride + c], sh = p.shift[(size_t)n * p.stat_stride + c];
    const float raw = raw_load(p.raw, pix * p.raw.C + p.c_off + c);
    const float z = fmaf(raw, sc, sh);
    const float dy = p.dy[idx];
    float dz = dy;
    if (p.act == ACT_RELU) dz = z > 0.f ? dz : 0.f;
    else if (p.act == ACT_LRELU) dz = z > 0.f ? dz : dz * p.slope;
    float dr = dz;
    if (p.has_norm) {
      const int row = p.batch_stats ? 0 : n;
      const float mean = p.mean[(size_t)n * p.stat_stride + c], rstd = p.rstd[(size_t)n * p.stat_stride + c];
      const float s1 = p.sums[(size_t)row * p.C + c], s2 = p.sums[((size_t)p.N + row) * p.C + c];
      const float xhat = (raw - mean) * rstd;
      dr = sc * (dz - s1 * inv_m - xhat * s2 * inv_m);      // sc = gamma * rstd
    }
    p.draw[pix * p.draw_C + p.c_off + c] += dr;        // += : the same raw slice may feed several normalise passes (defer_last)
    if (p.dadd0) p.dadd0[idx] += dy;
    if (p.dadd1) p.dadd1[idx] += dy;
  }
}

// dgamma[c] += sum_n sums[1][n][c] / ... : gamma-gradient = sum dz * xhat, beta-gradient = sum dz (already reduced)
__global__ void norm_param_grad_kernel(NormBwd p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.C) return;
  const int rows = p.batch_stats ? 1 : p.N;
  float s1 = 0.f, s2 = 0.f;
  for (int r = 0; r < rows; ++r) { s1 += p.sums[(size_t)r * p.C + c]; s2 += p.sums[((size_t)p.N + r) * p.C + c]; }
  if (p.has_norm) {
    if (p.dgamma) p.dgamma[c] += s2;
    if (p.dbeta) p.dbeta[c] += s1;
  } else if (p.dbeta) {
    p.dbeta[c] += s1;                                         // norm-less unit: dbeta is the conv bias gradient
  }
}

// ---------------------------------------------------------------------------------------------------- heads
// dz[p][j] = (g_ext + g_int)[j][p] * scale_j * act'(out_j[p]);  out = the head's forward output planes (caller tensors)
__global__ void __launch_bounds__(256) head_bwd_kernel(HeadBwd p) {
  const long long HW = (long long)p.H * p.W, total = (long long)p.N * HW;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const long long pix = idx - (long long)n * HW;
    for (int j = 0; j < p.Cout; ++j) {
      const size_t o = (size_t)p.off[j] + (size_t)n * p.bstride[j] + pix;
      float g = 0.f;
      if (p.g_ext[j]) g += p.g_ext[j][o];
      if (p.g_int[j]) g += p.g_int[j][o];
      float d = g * p.scale[j];
      if (p.act[j] == ACT_TANH) { const float t = p.out[j][o] / p.scale[j]; d *= 1.f - t * t; }
      else if (p.act[j] == ACT_SIGMOID) { const float t = p.out[j][o] / p.scale[j]; d *= t * (1.f - t); }
      p.dz[(size_t)idx * p.dz_C + j] = d;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- composite
struct Bil { int x0, y0, x1, y1; float wx, wy; float dsx, dsy; };
__device__ __forceinline__ float linspace_m1p1_b(int i, int n) {            // as csrc/warp.cu
  const float step = 2.0f / (float)(n - 1);
  return (i < n / 2) ? (-1.0f + step * (float)i) : (1.0f - step * (float)(n - 1 - i));
}
__device__ __forceinline__ Bil warp_coords_bwd(int x, int y, float fx, float fy, int W, int H, int ac) {
  // same coordinate arithmetic as csrc/warp.cu:warp_coords (ATen grid_sampler, border padding);
  // dsx / dsy = d(sample coordinate) / d(flow), zero where the coordinate is clipped (ATen clip_coordinates_set_grad)
  const float gx = linspace_m1p1_b(x, W) + fx / (((float)W - 1.0f) / 2.0f);
  const float gy = linspace_m1p1_b(y, H) + fy / (((float)H - 1.0f) / 2.0f);
  float sx = ac ? ((gx + 1.f) / 2.f) * (float)(W - 1) : ((gx + 1.f) * (float)W - 1.f) / 2.f;
  float sy = ac ? ((gy + 1.f) / 2.f) * (float)(H - 1) : ((gy + 1.f) * (float)H - 1.f) / 2.f;
  Bil b;
  b.dsx = (ac ? (float)(W - 1) / 2.f : (float)W / 2.f) / (((float)W - 1.0f) / 2.0f);
  b.dsy = (ac ? (float)(H - 1) / 2.f : (float)H / 2.f) / (((float)H - 1.0f) / 2.0f);
  if (sx <= 0.f || sx >= (float)(W - 1)) b.dsx = 0.f;
  if (sy <= 0.f || sy >= (float)(H - 1)) b.dsy = 0.f;
  sx = fminf((float)(W - 1), fmaxf(sx, 0.f)); sy = fminf((float)(H - 1), fmaxf(sy, 0.f));
  const float x0f = floorf(sx), y0f = floorf(sy);
  b.x0 = (int)x0f; b.y0 = (int)y0f; b.x1 = min(b.x0 + 1, W - 1); b.y1 = min(b.y0 + 1, H - 1);
  b.wx = sx - x0f; b.wy = sy - y0f;
  return b;
}

// PREV: also accumulate the gradient of the warped previous frame, grid_sample's input gradient of
// g_final * (1 - mask) * (1 - weight), into the last three channels of d_prev.  Several pixels may sample the same source
// pixel (all of them, at the border, when a flow leaves the frame) and there is no inverse map, so the four corner updates
// are fp32 atomics: d_prev is reproducible to ~1e-7 relative, not bit for bit.  As ATen's safe_add_2d, a corner whose
// contribution is zero (the clamped x1 / y1 at the border carry weight 0) issues no update.  Plans that need no img_prev
// gradient run PREV = false, which is the kernel without that code.
template <bool PREV>
__global__ void __launch_bounds__(256) composite_bwd_kernel(CompositeBwd p) {
  const size_t HW = (size_t)p.H * p.W, total = (size_t)p.N * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / HW);
    const size_t pix = idx - (size_t)n * HW;
    const int y = (int)(pix / p.W), x = (int)(pix - (size_t)y * p.W);
    const float m = p.mask ? p.mask[(size_t)n * HW + pix] : 0.f;
    float gf[3], gr[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gf[c] = p.g_final ? p.g_final[((size_t)n * 3 + c) * HW + pix] : 0.f;
      gr[c] = p.g_rawout ? p.g_rawout[((size_t)n * 3 + c) * HW + pix] : 0.f;
    }
    if (p.d_fg) {
#pragma unroll
      for (int c = 0; c < 3; ++c) p.d_fg[((size_t)n * 3 + c) * HW + pix] = (gf[c] + gr[c]) * m;
    }
    const float om = p.mask ? 1.f - m : 1.f;
    if (p.use_warp) {
      const float fx = p.flow[((size_t)n * 2) * HW + pix], fy = p.flow[((size_t)n * 2 + 1) * HW + pix];
      const float w = p.weight[(size_t)n * HW + pix];
      const Bil b = warp_coords_bwd(x, y, fx, fy, p.W, p.H, p.align_corners);
      float dw = 0.f, dfx = 0.f, dfy = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* pl = p.prev + ((size_t)n * p.prev_C + (p.prev_C - 3) + c) * HW;
        const float v00 = pl[(size_t)b.y0 * p.W + b.x0], v01 = pl[(size_t)b.y0 * p.W + b.x1];
        const float v10 = pl[(size_t)b.y1 * p.W + b.x0], v11 = pl[(size_t)b.y1 * p.W + b.x1];
        const float warp = v00 * (1.f - b.wx) * (1.f - b.wy) + v01 * b.wx * (1.f - b.wy) + v10 * (1.f - b.wx) * b.wy + v11 * b.wx * b.wy;
        const float dwarp_dx = (v01 - v00) * (1.f - b.wy) + (v11 - v10) * b.wy;
        const float dwarp_dy = (v10 - v00) * (1.f - b.wx) + (v11 - v01) * b.wx;
        const float raw = p.raw[((size_t)n * 3 + c) * HW + pix];
        const float g = gf[c] * om;                     // gradient reaching img_raw * w + warp * (1 - w)
        dw += g * (raw - warp);
        dfx += g * (1.f - w) * dwarp_dx * b.dsx;
        dfy += g * (1.f - w) * dwarp_dy * b.dsy;
        p.d_raw[((size_t)n * 3 + c) * HW + pix] = g * w + gr[c] * om;
        if (PREV) {
          float* dp = p.d_prev + ((size_t)n * p.prev_C + (p.prev_C - 3) + c) * HW;
          const float gp = g * (1.f - w);
          const float u00 = gp * ((1.f - b.wx) * (1.f - b.wy)), u01 = gp * (b.wx * (1.f - b.wy));
          const float u10 = gp * ((1.f - b.wx) * b.wy), u11 = gp * (b.wx * b.wy);
          if (u00 != 0.f) atomicAdd(dp + (size_t)b.y0 * p.W + b.x0, u00);
          if (u01 != 0.f) atomicAdd(dp + (size_t)b.y0 * p.W + b.x1, u01);
          if (u10 != 0.f) atomicAdd(dp + (size_t)b.y1 * p.W + b.x0, u10);
          if (u11 != 0.f) atomicAdd(dp + (size_t)b.y1 * p.W + b.x1, u11);
        }
      }
      p.d_weight[(size_t)n * HW + pix] = dw;
      p.d_flow[((size_t)n * 2) * HW + pix] = dfx;
      p.d_flow[((size_t)n * 2 + 1) * HW + pix] = dfy;
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) p.d_raw[((size_t)n * 3 + c) * HW + pix] = (gf[c] + gr[c]) * om;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- layout of gradients
// caller gradient (fp32 NCHW, channel window [c_off, c_off + C) of C_src) -> dense NHWC gradient buffer (accumulate)
__global__ void grad_import_kernel(const float* __restrict__ g, float* __restrict__ dst, int N, int C_src, int c_off, int C, size_t HW) {
  const size_t total = (size_t)N * C * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = idx % HW;
    const int c = (int)((idx / HW) % C), n = (int)(idx / ((size_t)C * HW));
    dst[((size_t)n * HW + pix) * C + c] += g[((size_t)n * C_src + c_off + c) * HW + pix];
  }
}
// dense NHWC gradient buffer -> caller gradient tensor (fp32 NCHW window), written (the caller zero-fills)
__global__ void grad_export_kernel(const float* __restrict__ src, float* __restrict__ g, int N, int C_src, int c_off, int C, size_t HW) {
  const size_t total = (size_t)N * C * HW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = idx % HW;
    const int c = (int)((idx / HW) % C), n = (int)(idx / ((size_t)C * HW));
    g[((size_t)n * C_src + c_off + c) * HW + pix] += src[((size_t)n * HW + pix) * C + c];
  }
}
// 32 x 32 tiles through shared memory: both the NCHW side (pixel-contiguous) and the NHWC side (channel-contiguous) are
// accessed coalesced.  IMPORT: dst(NHWC) += g(NCHW window); EXPORT: g(NCHW window) += src(NHWC).
template <bool IMPORT>
__global__ void __launch_bounds__(256) grad_layout_tiled_kernel(float* __restrict__ nchw, float* __restrict__ nhwc, int C_src, int c_off, int C,
                                                                size_t HW) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const size_t pix0 = (size_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32, n = blockIdx.z;
  if (IMPORT) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + ty + 8 * j;
      const size_t pix = pix0 + tx;
      tile[ty + 8 * j][tx] = (c < C && pix < HW) ? nchw[((size_t)n * C_src + c_off + c) * HW + pix] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t pix = pix0 + ty + 8 * j;
      const int c = c0 + tx;
      if (c < C && pix < HW) nhwc[((size_t)n * HW + pix) * C + c] += tile[tx][ty + 8 * j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t pix = pix0 + ty + 8 * j;
      const int c = c0 + tx;
      tile[ty + 8 * j][tx] = (c < C && pix < HW) ? nhwc[((size_t)n * HW + pix) * C + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + ty + 8 * j;
      const size_t pix = pix0 + tx;
      if (c < C && pix < HW) nchw[((size_t)n * C_src + c_off + c) * HW + pix] += tile[tx][ty + 8 * j];
    }
  }
}

// dz = dy * act'(out) for a bias + activation conv epilogue unit (EPI_ACT_BF16): out = the forward activation buffer
__global__ void convact_bwd_kernel(const float* __restrict__ dy, ActDesc out, int act, float slope, float* __restrict__ dz, int C, int dz_C) {
  const size_t total = (size_t)out.N * out.H * out.W * C;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    size_t t = idx / C;
    const int x = (int)(t % out.W); t /= out.W;
    const int y = (int)(t % out.H);
    const int n = (int)(t / out.H);
    const float o = act_load(out, out.offset(n, y, x) + c);
    float d = dy[idx];
    if (act == ACT_RELU) d = o > 0.f ? d : 0.f;
    else if (act == ACT_LRELU) d = o > 0.f ? d : d * slope;
    dz[(idx / C) * dz_C + c] = d;
  }
}

static inline int grid1d(size_t total) {
  size_t b = (total + 255) / 256;
  const size_t cap = 132 * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

cudaError_t launch_conv_bwd(const BwdConv& p, cudaStream_t s) {
  if (p.dx) {
    const int PH = p.transposed ? p.H : p.H + 2 * p.pad, PW = p.transposed ? p.W : p.W + 2 * p.pad;
    const long long npos = (long long)p.N * PH * PW;
    dim3 grid((unsigned)((npos + 15) / 16), (p.Cin + 63) / 64);
    conv_dgrad_kernel<<<grid, 256, 0, s>>>(p);
  }
  if (p.dw || p.dw2) {
    const int gh = p.transposed ? p.H : p.oh, gw = p.transposed ? p.W : p.ow;
    const long long npix = (long long)p.N * gh * gw;
    const int tiles = ((p.Cin + 31) / 32) * ((p.Cout + 31) / 32), taps = p.kh * p.kw;
    long long ks = (132LL * 8 + (long long)tiles * taps - 1) / ((long long)tiles * taps);
    ks = std::max(1LL, std::min(ks, (npix + 255) / 256));
    dim3 grid(tiles, taps, (unsigned)ks);
    conv_wgrad_kernel<<<grid, 256, 0, s>>>(p, (int)ks);
  }
  if (p.dbias || p.dbias2) {
    const long long npix = (long long)p.N * p.oh * p.ow;
    dim3 grid(p.Cout, (unsigned)bias_grad_blocks(npix));
    bias_grad_kernel<<<grid, 256, 0, s>>>(p.dy, p.dy_C, npix, p.Cout, p.dbias, p.dbias2, p.w2 ? p.Cout1 : p.Cout);
  }
  return cudaGetLastError();
}

int bias_grad_blocks(long long npix) { return (int)std::max(1LL, std::min(64LL, npix / 4096)); }

// The vectorised reduce aims at 4 blocks per SM of the H100 SXM (132 SMs) over the batch, each block summing at least 8
// pixel rows per thread; the scalar kernel takes one block per channel and image, split over up to 32 slices of 8192 pixels.
NormBwdLaunch norm_bwd_launch(const NormBwd& p) {
  NormBwdLaunch l{};
  const long long HW = (long long)p.H * p.W;
  l.param = (p.dgamma || p.dbeta) ? 1 : 0;
  l.grid[0] = l.grid[1] = l.grid[2] = 1;
  if (!p.has_norm && !l.param) return l;           // norm-less unit without a bias gradient: draw = dz needs no sums
  if (p.C % 4 == 0 && p.C <= 1024 && p.raw.C % 4 == 0 && p.c_off % 4 == 0) {
    l.reduce = 1;
    l.ppb = 256 / (p.C / 4);
    const long long want_blocks = std::max(1LL, (4LL * 132) / p.N);
    l.chunk = std::max<long long>((long long)l.ppb * 8, (HW + want_blocks - 1) / want_blocks);
    l.grid[0] = (int)((HW + l.chunk - 1) / l.chunk); l.grid[1] = p.N;
  } else {
    l.reduce = 2;
    l.grid[0] = p.C; l.grid[1] = p.N; l.grid[2] = (int)std::max(1LL, std::min(32LL, HW / 8192));
  }
  return l;
}

cudaError_t launch_norm_bwd(const NormBwd& p, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(p.sums, 0, sizeof(float) * 2 * p.N * p.C, s);
  if (e != cudaSuccess) return e;
  const NormBwdLaunch l = norm_bwd_launch(p);
  const dim3 grid(l.grid[0], l.grid[1], l.grid[2]);
  if (l.reduce == 1) norm_bwd_reduce_vec_kernel<<<grid, 256, 2 * p.C * sizeof(float), s>>>(p, (int)l.chunk);
  else if (l.reduce == 2) norm_bwd_reduce_kernel<<<grid, 256, 0, s>>>(p);
  norm_bwd_apply_kernel<<<grid1d((size_t)p.N * p.H * p.W * p.C), 256, 0, s>>>(p);
  if (l.param) norm_param_grad_kernel<<<(p.C + 127) / 128, 128, 0, s>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_head_bwd(const HeadBwd& p, cudaStream_t s) {
  head_bwd_kernel<<<grid1d((size_t)p.N * p.H * p.W), 256, 0, s>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_composite_bwd(const CompositeBwd& p, cudaStream_t s) {
  if (p.d_prev && p.use_warp) composite_bwd_kernel<true><<<grid1d((size_t)p.N * p.H * p.W), 256, 0, s>>>(p);
  else composite_bwd_kernel<false><<<grid1d((size_t)p.N * p.H * p.W), 256, 0, s>>>(p);
  return cudaGetLastError();
}
// The gradient import / export transposes through 32 x 32 shared-memory tiles (grad_layout_tiled_kernel) when a tile row of
// channels is worth it and the grid fits; narrow tensors (C < 8: the 3-channel images) take the elementwise kernels.
int grad_layout_tiled(const GradLayout& p) { return p.C >= 8 && ((long long)p.H * p.W + 31) / 32 <= 0x7fffffffLL && p.N <= 65535; }

cudaError_t launch_grad_import(const GradLayout& p, cudaStream_t s) {
  const size_t HW = (size_t)p.H * p.W;
  if (grad_layout_tiled(p)) {
    dim3 grid((unsigned)((HW + 31) / 32), (p.C + 31) / 32, p.N);
    grad_layout_tiled_kernel<true><<<grid, 256, 0, s>>>(p.g, p.v, p.C_src, p.c_off, p.C, HW);
    return cudaGetLastError();
  }
  grad_import_kernel<<<grid1d((size_t)p.N * p.C * HW), 256, 0, s>>>(p.g, p.v, p.N, p.C_src, p.c_off, p.C, HW);
  return cudaGetLastError();
}
cudaError_t launch_grad_export(const GradLayout& p, cudaStream_t s) {
  const size_t HW = (size_t)p.H * p.W;
  if (grad_layout_tiled(p)) {
    dim3 grid((unsigned)((HW + 31) / 32), (p.C + 31) / 32, p.N);
    grad_layout_tiled_kernel<false><<<grid, 256, 0, s>>>(p.g, p.v, p.C_src, p.c_off, p.C, HW);
    return cudaGetLastError();
  }
  grad_export_kernel<<<grid1d((size_t)p.N * p.C * HW), 256, 0, s>>>(p.v, p.g, p.N, p.C_src, p.c_off, p.C, HW);
  return cudaGetLastError();
}
cudaError_t launch_convact_bwd(const float* dy, const ActDesc& out, int act, float slope, float* dz, int C, int dz_C, cudaStream_t s) {
  convact_bwd_kernel<<<grid1d((size_t)out.N * out.H * out.W * C), 256, 0, s>>>(dy, out, act, slope, dz, C, dz_C);
  return cudaGetLastError();
}

}  // namespace v2v
