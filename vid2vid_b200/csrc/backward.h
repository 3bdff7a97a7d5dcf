// Parameter blocks of the backward kernels (csrc/backward.cu); internal, not part of the C ABI.
#pragma once
#include "v2v_internal.h"

namespace v2v {

struct BwdConv {
  int N, H, W;                 // forward input extent (unpadded)
  int oh, ow;                  // forward output extent
  int Cin, Cout, kh, kw, stride, pad, transposed, pad_mode;
  ActDesc x;                   // forward input buffer (halo-padded NHWC, bf16 or split)        [weight gradient]
  const float* dy; int dy_C;   // gradient of the conv output, dense NHWC fp32, channel stride dy_C
  const float* w; const float* w2; int Cout1;   // forward weights, torch layout (second set for stacked convs)
  float* dx;                   // gradient of the conv input, dense NHWC fp32 [N][H][W][Cin], accumulated; may be null
  float* dw; float* dw2;       // weight gradients, torch layout, accumulated; may be null
  float* dbias; float* dbias2; // bias gradients; may be null
};

struct NormBwd {
  int N, H, W, C;              // value extent; C = channels of this unit (slice of the raw tensor)
  RawDesc raw; int c_off;      // forward raw conv output (full tensor) and the slice offset
  const float* scale; const float* shift; const float* mean; const float* rstd; int stat_stride;   // [N][stat_stride], slice-offset applied
  int has_norm, batch_stats;   // 0: norm-less bias unit; batch_stats: BatchNorm (one statistic over N)
  int act; float slope;
  const float* dy;             // gradient of the unit output, dense NHWC [.][C]
  float* draw; int draw_C;     // gradient of the raw tensor (full channel stride draw_C), written at c_off
  float* dadd0; float* dadd1;  // gradients of the addends (accumulated); may be null
  float* sums;                 // scratch [2][N][C]
  float* dgamma; float* dbeta; // accumulated; may be null
};

struct HeadBwd {
  int N, H, W, Cout;
  const float* out[V2V_MAX_HEAD];     // forward output plane base (caller tensor) per head channel
  const float* g_ext[V2V_MAX_HEAD];   // caller gradient tensor base per channel (may be null)
  const float* g_int[V2V_MAX_HEAD];   // plan-internal gradient (composite backward) base per channel (may be null)
  long long off[V2V_MAX_HEAD], bstride[V2V_MAX_HEAD];
  int act[V2V_MAX_HEAD]; float scale[V2V_MAX_HEAD];
  float* dz; int dz_C;                // dense NHWC fp32 [N][H][W][dz_C]
};

struct CompositeBwd {
  int N, H, W, prev_C, use_warp, align_corners;
  const float* raw; const float* flow; const float* weight; const float* prev; const float* mask;   // forward tensors (raw = head output)
  const float* g_final; const float* g_rawout;                                                      // incoming gradients (may be null)
  float* d_raw; float* d_flow; float* d_weight; float* d_fg;                                          // written
  float* d_prev;   // img_prev gradient (fp32 NCHW, prev_C channels), accumulated into its last 3 channels; may be null
};

// Tensor-core weight gradient (csrc/wgrad_umma.cu): G[tap][m][n] = sum_pixels OUT[pixel][m] * IN[pixel @ tap][n]
struct WgradTap { int8_t plane, dy, dx, pad_; };      // IN buffer coordinate of grid pixel (y, x): plane, (y + dy, x + dx)
struct WgradParams {
  int N, gh, gw;               // driving grid = pixels of OUT
  int KP, kmma;                // pixels per K chunk (64 / 32 / 16), MMAs (16 pixels each) per chunk
  int xsegs;                   // ceil(gw / KP) chunks per grid row
  int out_padt, out_padl;      // OUT buffer halo: buffer coordinate of grid pixel (0, 0)
  int swap;                    // 0: A (M side) = OUT, B (N side) = IN;  1: A = IN, B = OUT (narrow gradient tensors)
  int a_C, b_C;                // padded channel counts of the A / B tensors: the lo half starts at channel coordinate C
  int Mblocks, Nblocks;        // A: 64-channel blocks per M tile (2, or 1 for a 64-channel tensor); B: blocks per N tile
  int b_row, BN;               // B: bytes per pixel row of one block (128 / 64 / 32) and channels per N tile (16 / 32 / 64 / 128)
  int m_tiles, n_tiles, ntaps, ksplit;
  int chunks_total, chunks_per_unit;
  int split;                   // 1: [hi | lo] operands, three MMAs per K step
  int stages;
  WgradTap taps[V2V_MAX_TAPS];
  float* stage;                // [ntaps][Mp][Np] fp32, zeroed by the launcher
  int Mp, Np;                  // = a_C, b_C
};
size_t wgrad_stage_bytes(const WgradParams& p);
size_t wgrad_stage_smem_bytes(const WgradParams& p);
cudaError_t launch_wgrad_umma(const CUtensorMap& tmOut, const CUtensorMap& tmIn, const WgradParams& p, int R, int R1, int Cc,
                              float* dw, float* dw2, cudaStream_t s);
// dx [N][H][W][C] += the data gradient over the padded extent, src: dense NHWC fp32 (N, PH, PW, channel stride Cs) whose pixel
// (pad, pad) is input pixel (0, 0); reflect: the halo mirrors back onto the interior (fold_add_kernel)
struct FoldParams {
  const float* src; int Cs, PH, PW;
  float* dx; int N, H, W, C;
  int pad, reflect;
};
cudaError_t launch_fold_add(const FoldParams& p, cudaStream_t s);

// Launch shape of launch_norm_bwd, chosen on the host from the unit's parameters alone (v2v_plan_describe reports the same).
// param: norm_param_grad_kernel runs, i.e. the unit has gamma / beta (or, norm-less, a bias) whose gradient is requested.
struct NormBwdLaunch {
  int reduce;                  // per-channel sums: 0 none (norm-less unit without a bias gradient), 1 vectorised, 2 scalar kernel
  int ppb;                     // vectorised: pixel rows per block pass (256 threads / (C / 4))
  long long chunk;             // vectorised: pixels per block and image
  int grid[3];                 // reduce grid (vectorised: chunks x N x 1; scalar: C x N x pixel slices)
  int param;                   // norm_param_grad_kernel runs (norm_bwd_apply_kernel always does)
};
NormBwdLaunch norm_bwd_launch(const NormBwd& p);
int bias_grad_blocks(long long npix);          // bias_grad_kernel: blocks per channel (grid.y)

// A caller's fp32 NCHW gradient tensor g (channels [c_off, c_off + C) of C_src) and a plan's dense NHWC fp32 gradient buffer
// v [N][H][W][C]: launch_grad_import adds g onto v, launch_grad_export adds v onto g.
struct GradLayout {
  float* g; float* v;
  int N, C_src, c_off, C, H, W;
};
int grad_layout_tiled(const GradLayout& p);   // 1: launch_grad_import / launch_grad_export take the tiled kernel

cudaError_t launch_conv_bwd(const BwdConv& p, cudaStream_t s);
cudaError_t launch_norm_bwd(const NormBwd& p, cudaStream_t s);
cudaError_t launch_head_bwd(const HeadBwd& p, cudaStream_t s);
cudaError_t launch_composite_bwd(const CompositeBwd& p, cudaStream_t s);
cudaError_t launch_grad_import(const GradLayout& p, cudaStream_t s);
cudaError_t launch_grad_export(const GradLayout& p, cudaStream_t s);
cudaError_t launch_convact_bwd(const float* dy, const ActDesc& out, int act, float slope, float* dz, int C, int dz_C, cudaStream_t s);

}  // namespace v2v
