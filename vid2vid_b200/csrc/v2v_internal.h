// Internal (non-ABI) declarations shared by the kernels and the plan runtime.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace v2v {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------
// Activation buffer: NHWC bf16 with a materialised halo, optionally split into the four
// (row parity, column parity) planes so that a stride-2 consumer reads unit-stride boxes.
//   padded coords  yp = y + pad_t, xp = x + pad_l   (y, x may lie in the halo)
//   parity == 0 :  [n][0][yp][xp][c]          plane dims Hp x Wp
//   parity == 1 :  [n][(yp&1)*2 + (xp&1)][yp>>1][xp>>1][c]   plane dims Hp x Wp (= ceil(padded/2))
// C is the padded channel count (16, 32, or a multiple of 64; channels >= Cvalid are zero): one K block of the
// implicit GEMM is min(C, 64) channels = one shared-memory row of 32 / 64 / 128 bytes (TMA swizzle 32B / 64B / 128B).
//
// Precise plans (split == 1, "bf16x3"): every value x is stored as the bf16 pair hi = bf16(x), lo = bf16(x - hi)
// (16 mantissa bits together), a pixel holding [hi channels 0..C) | lo channels 0..C)]: 2*C bf16 per pixel.  The conv
// kernel then accumulates A_hi*B_hi + A_lo*B_hi + A_hi*B_lo in fp32 (three wgmma per K block; the dropped lo*lo
// term is 2^-18 relative), which makes the conv stack fp32-class while staying on the bf16 tensor pipe.
struct ActDesc {
  bf16* base;
  int N, H, W;          // logical (unpadded) extent
  int C;                // padded channels (16 / 32 / multiple of 64)
  int Cvalid;
  int pad_t, pad_l, pad_b, pad_r;
  int parity;           // 0 / 1
  int P, Hp, Wp;        // planes and plane extent
  int split;            // 1: [hi | lo] bf16 pair per value (precise plans)
  __host__ __device__ int Cs() const { return C << split; }        // bf16 elements per pixel
  __host__ __device__ size_t elems() const { return (size_t)N * P * Hp * Wp * Cs(); }
  __host__ __device__ size_t offset(int n, int y, int x) const {   // element offset of channel 0 (hi half)
    int yp = y + pad_t, xp = x + pad_l;
    if (parity) {
      int pl = ((yp & 1) << 1) | (xp & 1);
      return ((((size_t)n * 4 + pl) * Hp + (yp >> 1)) * Wp + (xp >> 1)) * Cs();
    }
    return (((size_t)n * Hp + yp) * Wp + xp) * Cs();
  }
};

// Raw conv output: dense NHWC, C = channel stride (multiple of 8); bf16, or fp32 in precise plans.
struct RawDesc {
  void* base;
  int N, H, W, C, Cvalid;
  int f32;              // element type: 0 bf16, 1 fp32
  __host__ __device__ size_t elems() const { return (size_t)N * H * W * C; }
  __host__ __device__ size_t elem_bytes() const { return f32 ? 4 : 2; }
};

enum PadMode { PAD_NONE = 0, PAD_ZERO = 1, PAD_REFLECT = 2 };
enum ActKind { ACT_NONE = 0, ACT_RELU = 1, ACT_LRELU = 2, ACT_TANH = 3, ACT_SIGMOID = 4 };
enum EpiMode { EPI_RAW_STATS = 0, EPI_HEAD_F32 = 1, EPI_ACT_BF16 = 2 };

#define V2V_MAX_TAPS 64
#define V2V_MAX_PHASES 4
#define V2V_MAX_HEAD 16
// widest accumulator of one conv work unit (MG * BN fp32 columns; conv_umma.cu keeps it in registers, two warpgroups
// x 64 rows): wider units spill
#define V2V_MAX_ACC_COLS 128

// One "patch group": an A box (plane, dy, dx) that serves `R` consecutive taps (shifted by one
// pixel = one 128-byte smem row each).  tap0 = index of the first tap in the packed weight matrix.
struct ConvGroup {
  int8_t plane, dy, dx, pad_;
  int16_t tap0, pad2_;
};

struct ConvPhase {
  int group_begin, group_end;   // range in ConvKernelParams::groups
  int oy_add, ox_add;           // output coordinate offset (transposed-conv sub-pixel phase)
};

// Norm statistics of a raw conv output: ONE row per image, stats[n][0][c] = sum, stats[n][1][c] = sum of squares, as 64-bit
// fixed point (sum * 2^20, sumsq * 2^16) accumulated with integer atomics by the conv epilogue: integer addition is
// associative, so the result does not depend on the CTA order (deterministic) and needs no second reduction pass.
typedef unsigned long long stat_t;
#define V2V_STAT_SUM_SCALE 1048576.0f
#define V2V_STAT_SQ_SCALE 65536.0f

struct FinalizeParams {
  const stat_t* stats;     // [N][2][Cs]
  int Cs, C;               // stats channel stride, channels
  int N, tiles_per_img, num_phases;
  double count;            // elements per channel per image
  int instance;            // 0 = batch statistics over N, 1 = per-image statistics
  const float* gamma;      // may be null (-> 1)
  const float* beta;       // may be null (-> 0)
  const float* conv_bias;  // folded into running_mean only (cancels in the normalised output)
  float* running_mean;     // may be null
  float* running_var;
  long long* num_batches_tracked;
  float momentum, eps;
  float* scale;            // [N][scale_stride], written at column c_off + c
  float* shift;
  float* mean_out;         // training plans: batch / instance mean and 1/sqrt(var + eps), same indexing; may be null
  float* rstd_out;
  int c_off, scale_stride; // channel slice of the raw tensor this norm layer covers
};

struct ConvKernelParams {
  // problem
  int N, tiles_x, tiles_y, TH, TW;   // M tile = TH x TW output-grid pixels (TH*TW == 128)
  int grid_h, grid_w;                // extent of the output grid this launch iterates over
  int Cout, BN;                      // valid output channels, N tile (16/32/64/128)
  int Cp, cblocks;                   // padded input channels, K blocks per tap (Cp / kc)
  int kc, row_bytes, kmma;           // channels per K block (16/32/64), smem row bytes (2*kc), MMAs per row (kc/16)
  int layout_type, sbo_bytes;        // smem-descriptor swizzle code (6/4/2: 32B/64B/128B) and 8-row group stride (8*row_bytes)
  int R, RW;                         // taps served per A patch (1 = none); taps per patch row (tap r: row r / RW, column r % RW)
  int PW, PH;                        // patch extent in pixels (TMA box)
  int sbo_a_bytes;                   // A operand 8-row group stride: 8*row_bytes (row tiles) or PW*row_bytes (2-D patch)
  int a_slot_bytes, b_slot_bytes, SA, SB;
  int b_resident;                    // 1: SB == B tiles of one (phase, n-tile): loaded once per key, kept in smem
  int n_tiles, m_total, total_tiles; // N tiles, M tiles (N * tiles_x * tiles_y), all tiles incl. phases
  int CG, SG;                        // K-loop steps per barrier / commit group, group slots in the ring
  int MG, mg_total, total_units;     // M tiles accumulated side by side per weight pass (work unit), units per key, all units
  int num_phases;
  int split;                         // precise plan: A and B slots hold a hi and a lo half; 3 MMAs per (tap, K block)
  int a_half_bytes, b_half_bytes;    // byte offset of the lo half inside an A / B slot
  int Khalf;                         // taps * Cp: column offset of the lo half in the packed weight matrix
  int out_f32;                       // EPI_RAW_STATS: raw output element type (1 = fp32)
  // Decoupled operand rings (ring2): the activation patch of a K-loop step (MG tiles) and its weights travel through separate
  // rings -- SG patch slots, SBr weight slots of TB taps each (b_slot_bytes per slot) -- so a step's R taps need not fit in
  // shared memory next to the patch: 64-channel K blocks (128-byte rows, the efficient TMA / MMA operand) and 128-wide N
  // tiles stay available to streamed-weight layers and to precise (hi/lo) plans.
  int ring2, TB, SBr;
  int tile_dx;                       // x distance between consecutive M tiles (TW, or TW - (kw - 1) for kx-GEMM heads)
  int headkx;                        // > 0: small-Cout head as a GEMM over (kx, channel) columns: N = kw * Cout accumulator
                                     // columns per INPUT pixel, taps over ky only; the epilogue sums the kw shifted columns
  // Statistics finalisation in the tail of the launch: the CTA that takes the last ticket of a counter (zeroed with the
  // statistics rows before every run) turns the completed rows of up to two norm slices into scale / shift (and the
  // train-mode side effects).  No grid barrier: every other CTA has already exited.
  int n_fin;
  FinalizeParams fin[2];
  unsigned int* fin_counter;
  int a_exact;                       // precise plans: the input values are exact in bf16 (one-hot labels, edge maps): the lo
                                     // half of A is all zero, so it is neither fetched nor multiplied (2 MMAs per K block)

  ConvPhase phases[V2V_MAX_PHASES];
  ConvGroup groups[V2V_MAX_TAPS];
  // epilogue
  int epi;                           // EpiMode
  int oy_mul, ox_mul;                // output coord = grid coord * mul + phase add
  int out_H, out_W, out_C;           // destination extent / channel stride
  void* out;                         // EPI_RAW_STATS: bf16 NHWC raw; EPI_ACT_BF16: ActDesc base (see out_act)
  ActDesc out_act;                   // EPI_ACT_BF16 destination
  stat_t* stats;                     // [N][2][stats_C] fixed-point (sum, sumsq), see FinalizeParams; may be null
  int stats_C;
  const float* bias;                 // may be null
  const float* bias2; int Cout1;     // fused heads: channels >= Cout1 take bias2[j - Cout1]
  int dbg;                           // timing experiments only (V2V_DBG): bit0 skip stats, bit1 skip output stores
  int EG;                            // epilogue groups (always 1: both consumer warpgroups drain every tile)
  int grid;                          // CTAs launched (persistent); also the stats partial rows per (phase, image)
  // EPI_HEAD_F32: per output channel destination = io[head_slot] + head_off (+ n * head_bstride),
  // activation and scale.  Caller pointers are read from the device IO table at run time.
  void* const* io;
  int head_slot[V2V_MAX_HEAD];
  long long head_off[V2V_MAX_HEAD];
  long long head_bstride[V2V_MAX_HEAD];
  int head_act[V2V_MAX_HEAD];
  float head_scale[V2V_MAX_HEAD];
  float lrelu_slope;
  int act;                           // EPI_ACT_BF16 activation
};

// kernel launchers (defined in the .cu files); all enqueue on `stream` and return cudaError_t
cudaError_t launch_conv_umma(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvKernelParams& p,
                             cudaStream_t stream);
cudaError_t launch_conv_simt(const ActDesc& in, const bf16* wpacked, int Ktotal, const ConvKernelParams& p,
                             cudaStream_t stream);


// ---------------------------------------------------------------------------------------

struct ApplyParams {
  RawDesc raw;
  const float* scale;      // [N][scale_stride], already offset to the slice  (null -> identity)
  const float* shift;
  int scale_stride;
  int act; float slope;
  int n_add;
  ActDesc add[2];          // interior is read (any padding / parity)
  ActDesc out;
  int pad_mode;            // PadMode of out's halo
  int fused;               // (unused: a block-prologue variant was slower than reading the arrays)
  int update_running;
  FinalizeParams fin;
};

// fp32 NCHW (caller tensor, read through the IO table) -> halo-padded NHWC bf16
struct ImportParams {
  const void* const* io;   // device IO pointer table
  int slot;
  const float* direct;     // non-null: read this plan-internal fp32 NCHW scratch tensor instead of io[slot]
  int act; float slope;    // activation applied on the way in (LeakyReLU after the correlation, FlowNetC.py:83-84)
  int c_off, C_src;        // channel window [c_off, c_off + out.Cvalid) of a tensor with C_src channels
  ActDesc out;
  int pad_mode;
  int skip_lo;             // the caller promised values exact in bf16 (one-hot labels, edges): the lo half stays at the zeros the
                           // arena was initialised with
};
// halo-padded NHWC bf16 interior -> fp32 NCHW (caller tensor)
struct ExportParams {
  void* const* io;
  int slot;
  float* direct;           // non-null: write this plan-internal fp32 NCHW scratch tensor instead of io[slot]
  ActDesc in;
};

// channel-window copy between activation buffers (torch.cat along channels): out[:, c_off : c_off + in.Cvalid] = in
struct CopyParams {
  ActDesc in, out;
  int c_off;
  int pad_mode;            // PadMode of out's halo
};

// correlation_cuda.forward on plan-internal fp32 NCHW scratch tensors (FlowNetC.py:30-31,79-81)
struct CorrParams {
  const float* in1; const float* in2; float* out;
  int N, C, H, W, pad, k, max_disp, s1, s2;
};

struct PackParams {
  const float* w;          // torch layout: conv [Cout][Cin][kh][kw]; transposed conv [Cin][Cout][kh][kw]
  const float* w2; int Cout1;   // optional second source for output channels >= Cout1
  int transposed;
  int Cout, Cin, kh, kw;
  int Cp, ntaps;
  int8_t tap_ky[V2V_MAX_TAPS], tap_kx[V2V_MAX_TAPS];   // filter coordinates of packed tap t
  int split;               // 1: [Cout][2][ntaps * Cp] (hi row half, then lo row half)
  int headkx;              // > 0 (= kw): rows are (kx * Cout + co), taps are the kh filter rows: out[kx * Cout + co][ky * Cp + c]
  int dgrad;               // 1: w is the FORWARD tensor [Cin][Cout][kh][kw] of a stride-1 conv whose data gradient this conv computes
                           //    (rows = forward input channels, K = forward output channels, taps flipped; w2 from K index Cout1 on)
  bf16* out;               // [Cout][ntaps * Cp]
};

// fused warp + soft-mask blend + fg composite (models/networks.py:219-221,228-230)
struct CompositeParams {
  void* const* io;
  int s_raw, s_flow, s_weight, s_prev, s_fg, s_mask, s_final;   // IO slots; -1 = absent
  int s_raw_out;           // >= 0: the composited raw image goes to this slot and s_raw keeps the head output (training plans)
  int prev_C;              // img_prev channel count (last 3 are warped)
  int N, H, W;
  int align_corners;
  int use_warp;            // 0: img_final = img_raw (use_raw_only / no_flow)
};

cudaError_t launch_raw_stats(const RawDesc& raw, stat_t* stats, int stats_C, cudaStream_t stream);

// x = hi + lo with hi = bf16(x), lo = bf16(x - hi)
__device__ __forceinline__ void split_bf16(float x, bf16& hi, bf16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
cudaError_t launch_stats_finalize(const FinalizeParams& p, cudaStream_t stream);
cudaError_t launch_norm_apply(const ApplyParams& p, cudaStream_t stream);
bool norm_apply_uses_rows(const ApplyParams& p);
cudaError_t launch_import_nchw(const ImportParams& p, cudaStream_t stream);
cudaError_t launch_export_nchw(const ExportParams& p, cudaStream_t stream);
cudaError_t launch_pack_weights(const PackParams& p, cudaStream_t stream);
cudaError_t launch_act_copy(const CopyParams& p, cudaStream_t stream);
cudaError_t launch_bias_affine(float* scale, float* shift, const float* bias, int N, int C, int stride, cudaStream_t stream);
cudaError_t launch_correlation(const float*, const float*, float*, int, int, int, int, int, int, int, int, int, cudaStream_t);
cudaError_t launch_composite(const CompositeParams& p, cudaStream_t stream);
int device_sm_count();


// Host side of PDL: launch with the programmatic-stream-serialization attribute (captured into the CUDA graph as a
// programmatic dependency) when V2V_PDL=1; plain serialised launches otherwise (the default, see pdl_enabled()).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace v2v
