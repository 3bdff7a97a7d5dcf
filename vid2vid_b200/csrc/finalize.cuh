// Batch / instance-norm affine of ONE channel from the fixed-point statistics rows (see FinalizeParams): the few
// double-precision operations sit in the mean / variance subtraction only.  Shared by the stand-alone stats_finalize_kernel
// (csrc/norm.cu) and the tail of conv_umma_kernel, which must stay call-free: the divisions are div_rn_normal (ptx.cuh),
// whose operands here are counts and fixed-point sums, never near underflow.
#pragma once
#include "../../include/v2v_b200.h"
#include "ptx.cuh"
#include "v2v_internal.h"

namespace v2v {

struct ChannelAffine { float scale, shift, mean, rstd; double var_unbiased; };

// statistics of image n (instance norm) or of the whole batch (n ignored)
__device__ __forceinline__ ChannelAffine channel_affine(const FinalizeParams& p, int n, int c) {
  long long s = 0, q = 0;
  const int n0 = p.instance ? n : 0, n1 = p.instance ? n + 1 : p.N;
  for (int i = n0; i < n1; ++i) {
    s += (long long)__ldcg(p.stats + ((size_t)i * 2 + 0) * p.Cs + p.c_off + c);
    q += (long long)__ldcg(p.stats + ((size_t)i * 2 + 1) * p.Cs + p.c_off + c);
  }
  const double cnt = p.count * (n1 - n0);
  const double mean = div_rn_normal((double)s * (1.0 / (double)V2V_STAT_SUM_SCALE), cnt);
  double var = div_rn_normal((double)q * (1.0 / (double)V2V_STAT_SQ_SCALE), cnt) - mean * mean;
  if (var < 0) var = 0;
  ChannelAffine a;
  a.rstd = rsqrtf((float)var + p.eps);
  a.rstd = a.rstd * (1.5f - 0.5f * ((float)var + p.eps) * a.rstd * a.rstd);      // one Newton step: full fp32 accuracy
  const float g = p.gamma ? p.gamma[c] : 1.f, b = p.beta ? p.beta[c] : 0.f;
  a.scale = g * a.rstd;
  a.mean = (float)mean;
  a.shift = b - a.mean * a.scale;
  a.var_unbiased = var * div_rn_normal(cnt, cnt > 1 ? cnt - 1 : 1);
  return a;
}

// nn.BatchNorm2d's train-mode running-statistics update from the statistics of n images (mean sum rm, unbiased variance sum rv)
__device__ __forceinline__ void running_update(const FinalizeParams& p, int c, double rm, double rv, int n) {
  const float bias = p.conv_bias ? p.conv_bias[c] : 0.f;
  p.running_mean[c] = (1.f - p.momentum) * p.running_mean[c] + p.momentum * ((float)div_rn_normal(rm, n) + bias);
  p.running_var[c] = (1.f - p.momentum) * p.running_var[c] + p.momentum * (float)div_rn_normal(rv, n);
}

// side effects of a train-mode norm layer for channel c: running statistics, and the per-image arrays the backward reads.
// Per-sample plans (p.sample_running) update the running statistics once per image, in image order, with the expression a
// one-image plan evaluates: N images leave them exactly as N one-image forwards in that order would.  With per-image flags
// (p.flags_slot >= 0, per-sample plans only) an image without V2V_IMAGE_ACTIVE is skipped, so the running statistics end as
// the one-image forwards of the active images in image order would leave them.
__device__ __forceinline__ void channel_side_effects(const FinalizeParams& p, int c) {
  const int* flags = p.flags_slot >= 0 ? reinterpret_cast<const int*>(p.io[p.flags_slot]) : nullptr;
  double rm = 0.0, rv = 0.0;
  int active = 0;
  for (int n = 0; n < p.N; ++n) {
    const ChannelAffine a = channel_affine(p, n, c);
    if (p.scale) {
      p.scale[(size_t)n * p.scale_stride + p.c_off + c] = a.scale;
      p.shift[(size_t)n * p.scale_stride + p.c_off + c] = a.shift;
    }
    if (p.mean_out) {
      p.mean_out[(size_t)n * p.scale_stride + p.c_off + c] = a.mean;
      p.rstd_out[(size_t)n * p.scale_stride + p.c_off + c] = a.rstd;
    }
    if (p.sample_running) {
      if (flags && !(__ldcg(flags + n) & V2V_IMAGE_ACTIVE)) continue;
      ++active;
      if (p.running_mean) running_update(p, c, 0.0 + (double)a.mean, 0.0 + a.var_unbiased, 1);
      continue;
    }
    rm += a.mean; rv += a.var_unbiased;
    if (!p.instance && !p.scale && !p.mean_out) { rm *= p.N; rv *= p.N; break; }       // batch statistics: identical for all n
  }
  if (p.running_mean) {
    if (!p.sample_running) running_update(p, c, rm, rv, p.N);
    if (c == 0 && p.num_batches_tracked) *p.num_batches_tracked += p.sample_running ? active : 1;
  }
}

}  // namespace v2v
