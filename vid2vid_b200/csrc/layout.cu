// Layout conversion at the module boundary and weight packing.
//   import : caller fp32 NCHW tensor  -> halo-padded NHWC bf16 activation buffer (reflect/zero halo)
//   export : activation buffer interior -> caller fp32 NCHW tensor
//   pack   : torch conv / transposed-conv weights (fp32) -> bf16 GEMM B matrix [Cout][tap*Cp + c]
// The boundary tensors are the ones Vid2VidModelG passes to netG.forward
// (models/vid2vid_model_G.py:225-226); caller pointers are read from a small device-side IO
// table so the captured CUDA graph stays valid when PyTorch hands us new tensors every frame.
#include <cstdlib>
#include <algorithm>
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

__device__ __forceinline__ int reflect_i(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// block (32, 8): tile of 128 padded-x positions x CT channels at one (n, yp); CT = 64, or 16 for narrow tensors.
// Loads are coalesced along x (4 independent 128-byte rows per channel per warp), stores along channels.
template <int CT>
__global__ void __launch_bounds__(256) import_nchw_kernel(ImportParams p) {
  __shared__ float tile[CT][129];
  pdl_prologue();
  const float* src = p.direct ? p.direct : reinterpret_cast<const float*>(p.io[p.slot]);
  const ActDesc& o = p.out;
  const int Wpad = o.W + o.pad_l + o.pad_r, Hpad = o.H + o.pad_t + o.pad_b;
  const int xt = blockIdx.x * 128;
  const int yp = blockIdx.y % Hpad, n = blockIdx.y / Hpad;
  const int cblk = blockIdx.z * CT;
  int y = yp - o.pad_t;
  const bool yhalo = (y < 0 || y >= o.H);
  if (p.pad_mode == PAD_REFLECT) y = reflect_i(y, o.H);
  int xs[4];
  bool zero_px[4];
#pragma unroll
  for (int sx = 0; sx < 4; ++sx) {
    const int xp = xt + sx * 32 + threadIdx.x;
    int x = xp - o.pad_l;
    const bool xhalo = (x < 0 || x >= o.W);
    if (p.pad_mode == PAD_REFLECT) x = reflect_i(x, o.W);
    xs[sx] = x;
    zero_px[sx] = (xp >= Wpad) || ((yhalo || xhalo) && p.pad_mode != PAD_REFLECT);
  }
  // two channels per pass: 8 independent 4-byte loads in flight per thread (one channel per pass left the kernel
  // latency bound at ~50 % of the HBM rate)
  for (int cc = threadIdx.y; cc < CT; cc += 16) {
    float v[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = cblk + cc + 8 * h;
      const bool cv = (cc + 8 * h < CT) && c < o.Cvalid;
      const float* row = src + (((size_t)n * p.C_src + p.c_off + (cv ? c : 0)) * o.H + y) * o.W;
#pragma unroll
      for (int sx = 0; sx < 4; ++sx) {
        float t = (cv && !zero_px[sx]) ? __ldg(row + xs[sx]) : 0.f;
        if (p.act == ACT_LRELU) t = t > 0.f ? t : t * p.slope;
        v[h][sx] = t;
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (cc + 8 * h < CT) {
#pragma unroll
        for (int sx = 0; sx < 4; ++sx) tile[cc + 8 * h][sx * 32 + threadIdx.x] = v[h][sx];
      }
  }
  __syncthreads();
  // write: lane -> channel pair (CT = 64) or (pixel parity, channel pair) (CT = 16)
  if (CT == 64) {
    for (int px = threadIdx.y; px < 128; px += 8) {
      const int xo = xt + px;
      if (xo >= Wpad) break;
      if (cblk + 2 * (int)threadIdx.x >= o.C) continue;
      const float f0 = tile[2 * threadIdx.x][px], f1 = tile[2 * threadIdx.x + 1][px];
      bf16* d = o.base + o.offset(n, yp - o.pad_t, xo - o.pad_l) + cblk + 2 * threadIdx.x;
      *reinterpret_cast<uint32_t*>(d) = pack_bf16x2(f0, f1);
      if (o.split && !p.skip_lo) *reinterpret_cast<uint32_t*>(d + o.C) = pack_bf16x2(f0 - __bfloat162float(__float2bfloat16_rn(f0)),
                                                                      f1 - __bfloat162float(__float2bfloat16_rn(f1)));
    }
  } else {
    const int cp = threadIdx.x & 7, sub = threadIdx.x >> 3;         // 8 channel pairs x 4 pixels per warp row
    for (int px = threadIdx.y * 4 + sub; px < 128; px += 32) {
      const int xo = xt + px;
      if (xo >= Wpad || cblk + 2 * cp >= o.C) continue;
      const float f0 = tile[2 * cp][px], f1 = tile[2 * cp + 1][px];
      bf16* d = o.base + o.offset(n, yp - o.pad_t, xo - o.pad_l) + cblk + 2 * cp;
      *reinterpret_cast<uint32_t*>(d) = pack_bf16x2(f0, f1);
      if (o.split && !p.skip_lo) *reinterpret_cast<uint32_t*>(d + o.C) = pack_bf16x2(f0 - __bfloat162float(__float2bfloat16_rn(f0)),
                                                                      f1 - __bfloat162float(__float2bfloat16_rn(f1)));
    }
  }
}

// block (32, 8): tile of 128 x positions x 32 channels at one (n, y).
__global__ void __launch_bounds__(256) export_nchw_kernel(ExportParams p) {
  __shared__ float tile[32][129];
  pdl_prologue();
  float* dst = p.direct ? p.direct : reinterpret_cast<float*>(p.io[p.slot]);
  const ActDesc& a = p.in;
  const int xt = blockIdx.x * 128;
  const int y = blockIdx.y % a.H, n = blockIdx.y / a.H;
  const int cblk = blockIdx.z * 32;
  // read: lane -> channel pair (16 pairs) x 2 pixels
  const int cp = threadIdx.x & 15, sub = threadIdx.x >> 4;
#pragma unroll
  for (int px = threadIdx.y * 2 + sub; px < 128; px += 16) {
    const int x = xt + px, c = cblk + 2 * cp;
    float2 v = make_float2(0.f, 0.f);
    if (x < a.W && c < a.C) {
      const bf16* sp = a.base + a.offset(n, y, x) + c;
      v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sp));
      if (a.split) {
        const float2 l = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sp + a.C));
        v.x += l.x; v.y += l.y;
      }
    }
    tile[2 * cp][px] = v.x;
    tile[2 * cp + 1][px] = v.y;
  }
  __syncthreads();
  for (int cc = threadIdx.y; cc < 32; cc += 8) {
    const int c = cblk + cc;
    if (c >= a.Cvalid) continue;
    float* row = dst + (((size_t)n * a.Cvalid + c) * a.H + y) * a.W;
#pragma unroll
    for (int sx = 0; sx < 4; ++sx) {
      const int x = xt + sx * 32 + threadIdx.x;
      if (x < a.W) row[x] = tile[cc][sx * 32 + threadIdx.x];
    }
  }
}

__global__ void pack_weights_kernel(PackParams p) {
  const int K = p.ntaps * p.Cp;
  const int rows = p.headkx ? p.headkx * p.Cout : p.Cout;
  const long long total = (long long)rows * K;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % K), row = (int)(idx / K);
    const int t = k / p.Cp, c = k - t * p.Cp;
    int co = row, ky, kx;
    if (p.headkx) { kx = row / p.Cout; co = row - kx * p.Cout; ky = t; }        // kx-GEMM head: one tap per filter ROW
    else { ky = p.tap_ky[t]; kx = p.tap_kx[t]; }
    float v = 0.f;
    if (p.dgrad) {
      // data-gradient form of a stride-1 conv: rows = forward INPUT channels, K columns = forward OUTPUT channels, taps flipped;
      // the forward tensors are [Cout_f = p.Cin][Cin_f = p.Cout][kh][kw], the second set starting at forward output channel Cout1
      if (c < p.Cin) {
        const int fy = p.kh - 1 - ky, fx = p.kw - 1 - kx;
        if (p.w2 && c >= p.Cout1) v = p.w2[((((size_t)(c - p.Cout1)) * p.Cout + co) * p.kh + fy) * p.kw + fx];
        else v = p.w[((((size_t)c) * p.Cout + co) * p.kh + fy) * p.kw + fx];
      }
    } else if (c < p.Cin) {
      if (p.w2 && co >= p.Cout1) {
        v = p.w2[((((size_t)(co - p.Cout1)) * p.Cin + c) * p.kh + ky) * p.kw + kx];
      } else {
        const int co1 = p.w2 ? p.Cout1 : p.Cout;
        const size_t wi = p.transposed ? ((((size_t)c * co1 + co) * p.kh + ky) * p.kw + kx)
                                       : ((((size_t)co * p.Cin + c) * p.kh + ky) * p.kw + kx);
        v = p.w[wi];
      }
    }
    if (p.split) split_bf16(v, p.out[(size_t)row * 2 * K + k], p.out[(size_t)row * 2 * K + K + k]);
    else p.out[idx] = __float2bfloat16_rn(v);
  }
}

// torch.cat along channels: one thread per (padded pixel of out, source channel), channel fastest.
__global__ void __launch_bounds__(256) act_copy_kernel(CopyParams p) {
  pdl_prologue();
  const ActDesc& o = p.out;
  const ActDesc& a = p.in;
  const int Wpad = o.W + o.pad_l + o.pad_r, Hpad = o.H + o.pad_t + o.pad_b, C = a.Cvalid;
  const size_t total = (size_t)o.N * Hpad * Wpad * C;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    size_t t = idx / C;
    const int xp = (int)(t % Wpad); t /= Wpad;
    const int yp = (int)(t % Hpad);
    const int n = (int)(t / Hpad);
    int y = yp - o.pad_t, x = xp - o.pad_l;
    const bool halo = (y < 0 || y >= o.H || x < 0 || x >= o.W);
    bf16 hi = __float2bfloat16_rn(0.f), lo = hi;
    if (!halo || p.pad_mode == PAD_REFLECT) {
      if (halo) { y = reflect_i(y, o.H); x = reflect_i(x, o.W); }
      const bf16* sp = a.base + a.offset(n, y, x) + c;
      hi = sp[0];
      if (a.split) lo = sp[a.C];
    }
    bf16* dp = o.base + o.offset(n, yp - o.pad_t, xp - o.pad_l) + p.c_off + c;
    dp[0] = hi;
    if (o.split) dp[o.C] = lo;
  }
}

// scale = 1, shift = bias for the normalise pass of a norm-less biased convolution
__global__ void bias_affine_kernel(float* scale, float* shift, const float* bias, int N, int C, int stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  scale[(size_t)n * stride + c] = 1.f;
  shift[(size_t)n * stride + c] = bias ? bias[c] : 0.f;
}

cudaError_t launch_act_copy(const CopyParams& p, cudaStream_t stream) {
  const size_t total = (size_t)p.out.N * (p.out.H + p.out.pad_t + p.out.pad_b) * (p.out.W + p.out.pad_l + p.out.pad_r) * p.in.Cvalid;
  size_t b = (total + 255) / 256;
  if (b > 132 * 16) b = 132 * 16;
  return launch_pdl(act_copy_kernel, dim3((unsigned)(b ? b : 1)), dim3(256), 0, stream, p);
}

cudaError_t launch_bias_affine(float* scale, float* shift, const float* bias, int N, int C, int stride, cudaStream_t stream) {
  bias_affine_kernel<<<(N * C + 255) / 256, 256, 0, stream>>>(scale, shift, bias, N, C, stride);
  return cudaGetLastError();
}

cudaError_t launch_import_nchw(const ImportParams& p, cudaStream_t stream) {
  const ActDesc& o = p.out;
  const int Wpad = o.W + o.pad_l + o.pad_r, Hpad = o.H + o.pad_t + o.pad_b;
  dim3 block(32, 8);
  if (o.C <= 16) {
    dim3 grid((Wpad + 127) / 128, Hpad * o.N, 1);
    return launch_pdl(import_nchw_kernel<16>, grid, block, 0, stream, p);
  } else {
    dim3 grid((Wpad + 127) / 128, Hpad * o.N, (o.C + 63) / 64);
    return launch_pdl(import_nchw_kernel<64>, grid, block, 0, stream, p);
  }
  return cudaGetLastError();
}

cudaError_t launch_export_nchw(const ExportParams& p, cudaStream_t stream) {
  const ActDesc& a = p.in;
  dim3 grid((a.W + 127) / 128, a.H * a.N, (a.Cvalid + 31) / 32), block(32, 8);
  return launch_pdl(export_nchw_kernel, grid, block, 0, stream, p);
}

// Tiled variant for plain convs (forward packing and the data-gradient packing of stride-1 convs): a block stages a
// [TC output channels][32 input channels][taps] tile of the torch-layout tensor through shared memory, so both the fp32 reads
// (32 * taps contiguous floats per output channel) and the bf16 writes (32 / TC contiguous K columns per row and tap) are
// coalesced; the elementwise kernel above reads with a stride of kh * kw floats.  Every optimiser step re-packs every weight of
// the forward plans and of the backward sub-plans (~0.9 G parameters at cfg3), which made this kernel 4 % of a training step.
__global__ void __launch_bounds__(256) pack_weights_tiled_kernel(PackParams p, int TC) {
  extern __shared__ float wt[];                       // [TC][32][tstride] with odd strides (conflict-free along either channel axis)
  const int taps = p.kh * p.kw, tstride = taps | 1, astride = 32 * tstride + 1;
  // forward tensors: [Cf_out][Cf_in][taps]; dgrad packing sees them as [p.Cin][p.Cout][taps], plain packing as [p.Cout][p.Cin][taps]
  const int f_out = p.dgrad ? p.Cin : p.Cout, f_in = p.dgrad ? p.Cout : p.Cin;
  const int co0 = blockIdx.y * TC, ci0 = blockIdx.x * 32;
  for (int i = threadIdx.x; i < TC * 32 * taps; i += 256) {
    const int a = i / (32 * taps), r = i - a * (32 * taps);
    const int b = r / taps, t = r - b * taps;
    const int co = co0 + a, ci = ci0 + b;
    float v = 0.f;
    if (co < f_out && ci < f_in) {
      if (p.w2 && co >= p.Cout1) v = p.w2[((size_t)(co - p.Cout1) * f_in + ci) * taps + t];
      else v = p.w[((size_t)co * f_in + ci) * taps + t];
    }
    wt[a * astride + b * tstride + t] = v;
  }
  __syncthreads();
  const int K = p.ntaps * p.Cp;
  if (!p.dgrad) {
    // out[co][t * Cp + ci]: ci fastest
    for (int i = threadIdx.x; i < TC * taps * 32; i += 256) {
      const int b = i & 31, r = i >> 5;
      const int t = r % taps, a = r / taps;
      const int co = co0 + a, ci = ci0 + b;
      if (co >= p.Cout || ci >= p.Cp) continue;
      const float v = wt[a * astride + b * tstride + t];
      const size_t k = (size_t)t * p.Cp + ci;
      if (p.split) split_bf16(v, p.out[(size_t)co * 2 * K + k], p.out[(size_t)co * 2 * K + K + k]);
      else p.out[(size_t)co * K + k] = __float2bfloat16_rn(v);
    }
  } else {
    // out[ci_f][t' * Cp + co_f] with t' the flipped tap: co_f fastest
    for (int i = threadIdx.x; i < 32 * taps * TC; i += 256) {
      const int a = i % TC, r = i / TC;
      const int t = r % taps, b = r / taps;
      const int co = co0 + a, ci = ci0 + b;                  // forward output / input channel
      if (ci >= p.Cout || co >= p.Cp) continue;              // rows = forward input channels (p.Cout of this conv), K channels padded to Cp
      const float v = wt[a * astride + b * tstride + (taps - 1 - t)];
      const size_t k = (size_t)t * p.Cp + co;
      if (p.split) split_bf16(v, p.out[(size_t)ci * 2 * K + k], p.out[(size_t)ci * 2 * K + K + k]);
      else p.out[(size_t)ci * K + k] = __float2bfloat16_rn(v);
    }
  }
}

cudaError_t launch_pack_weights(const PackParams& p, cudaStream_t stream) {
  const int taps = p.kh * p.kw;
  bool natural = !p.transposed && !p.headkx && p.ntaps == taps;
  for (int t = 0; t < taps && natural; ++t) natural = (p.tap_ky[t] * p.kw + p.tap_kx[t] == t);
  static const bool tiled_ok = [] { const char* e = getenv("V2V_PACK_TILED"); return !(e && e[0] == '0'); }();
  if (natural && tiled_ok) {
    const int tstride = taps | 1;
    int TC = 32;
    while (TC > 4 && (size_t)TC * (32 * tstride + 1) * sizeof(float) > 40 * 1024) TC >>= 1;
    if ((size_t)TC * (32 * tstride + 1) * sizeof(float) <= 48 * 1024) {
      // grid: x over the 32-wide tiles of the forward INPUT channel axis, y over TC-wide tiles of the forward OUTPUT channel axis;
      // each axis covers the padded extent where it is the K axis of the packed matrix (zero fill)
      const int f_out = p.dgrad ? std::max(p.Cin, p.Cp) : p.Cout, f_in = p.dgrad ? p.Cout : std::max(p.Cin, p.Cp);
      dim3 grid((f_in + 31) / 32, (f_out + TC - 1) / TC);
      pack_weights_tiled_kernel<<<grid, 256, (size_t)TC * (32 * tstride + 1) * sizeof(float), stream>>>(p, TC);
      return cudaGetLastError();
    }
  }
  const long long total = (long long)(p.headkx ? p.headkx * p.Cout : p.Cout) * p.ntaps * p.Cp;
  long long b = (total + 255) / 256;
  if (b > 132 * 16) b = 132 * 16;
  pack_weights_kernel<<<(int)b, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace v2v
