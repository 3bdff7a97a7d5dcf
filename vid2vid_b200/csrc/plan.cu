// Plan runtime: lowers a graph of logical values / convolution units (described through the C ABI in
// include/v2v_b200.h) to halo-padded NHWC bf16 buffers, TMA tensor maps, packed weight matrices and a
// flat kernel sequence, captures the sequence in a CUDA graph and replays it per frame.
// This is the H100-native counterpart of the nn.Module surface the reference's Vid2VidModelG calls
// (netG.forward, models/vid2vid_model_G.py:225-226; module bodies models/networks.py:117-419,634-725).
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/v2v_b200.h"
#include "v2v_internal.h"
#include "backward.h"
#include <unordered_map>

namespace v2v {

thread_local std::string g_last_error;
void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
}

#define V2V_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e__ = (expr);                                                                   \
    if (e__ != cudaSuccess) {                                                                   \
      set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__);   \
      return (int)e__;                                                                          \
    }                                                                                           \
  } while (0)
#define V2V_REQUIRE(cond, code, ...) \
  do {                               \
    if (!(cond)) {                   \
      set_error(__VA_ARGS__);        \
      return code;                   \
    }                                \
  } while (0)

// Makes the plan's device current for the duration of an entry point and restores the caller's device afterwards (the
// reference supports several GPUs per process: models/vid2vid_model_G.py:126-133; PyTorch's current device must not change
// behind the caller's back).
struct DeviceGuard {
  int prev = -1; bool changed = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) changed = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() { if (changed) cudaSetDevice(prev); }
};

static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
static inline size_t round_up_sz(size_t a, size_t b) { return (a + b - 1) / b * b; }
// padded channel count of an activation buffer: one K block of min(C,64) channels per shared-memory row
static thread_local int g_pad_min = 0;     // a backward sub-plan's pad_min while it is built, lowered or described (PadScope)
static inline int pad_channels(int c) {
  const int r = c <= 16 ? 16 : (c <= 32 ? 32 : round_up(c, 64));
  return std::max(r, g_pad_min);
}
struct PadScope {
  int prev;
  explicit PadScope(int m) : prev(g_pad_min) { g_pad_min = m; }
  ~PadScope() { g_pad_min = prev; }
};

// ------------------------------------------------------------------------------ conv geometry
struct ConvGeom {
  int pads[4];            // top, left, bottom, right of the input buffer
  int parity;
  int grid_h, grid_w;     // grid the kernel iterates over
  int out_h, out_w;       // conv output extent
  int mul;                // output coord = grid coord * mul + phase add
  int TH, TW, R;
  int RW;                 // taps per patch row: tap r of a group reads the patch shifted by (r / RW) rows, (r % RW) columns
  int patch2d_kc;         // > 0: 16x8 pixel tiles, ONE activation patch of (16+kh-1) x (8+kw-1) pixels serves all kh*kw taps;
  int patch2d_bn;         //      K block / N tile chosen together with the geometry (they decide the fit)
  int headkx;             // > 0 (= kw): small-Cout head evaluated as a GEMM over (kx, channel) columns (taps over ky only)
  int n_groups, n_phases;
  ConvGroup groups[V2V_MAX_TAPS];
  ConvPhase phases[V2V_MAX_PHASES];
};


static const int kSmemBudget = 188 * 1024;      // operand slots + resident weights (227 KB - 36.5 KB epilogue staging - alignment - barriers)
static const int kResidentMax = 150 * 1024;

// Bytes of one shared-memory operand slot, each of its sp halves 1 KB aligned: the activation patch of `pixels` pixels for
// one K block of kc channels (A), and the weights of `taps` taps x an N tile of bn x kc (B).
static inline int a_slot_bytes(int sp, int pixels, int kc) { return sp * round_up(pixels * kc * 2, 1024); }
static inline int b_slot_bytes(int sp, int taps, int bn, int kc) { return sp * round_up(taps * bn * kc * 2, 1024); }

// 2-D patch mode (stride-1 filters): a tile of 16 rows x 8 pixels makes every 8-row core-matrix group of the A operand
// one tile row, so the operand of tap (ky, kx) is the SAME shared-memory patch of (16+kh-1) x (8+kw-1) pixels read with
// start address advanced by (ky * PW + kx) rows and a group stride (SBO) of PW rows.  Each input pixel is then fetched
// ~1.4x (3x3) instead of 3x (row tiles with horizontal reuse) or 9x (one box per tap).  Feasible when a step's weights
// (all taps of one K block) fit next to the patch, double buffered, or the whole (phase, N tile) weight set stays resident.
// sp = 2 for precise plans: every operand slot holds a hi and a lo half, so all byte counts double.
static bool choose_patch2d(const v2v_conv_desc& c, bool head, int N, int grid_h, int grid_w, int sp, int* kc_out, int* bn_out) {
  if (c.transposed || c.stride != 1 || c.kh * c.kw == 1 || grid_w < 8) return false;
  const long long tiles = (long long)((grid_w + 7) / 8) * ((grid_h + 15) / 16);
  if (tiles * 128 * 4 > (long long)grid_h * grid_w * 5) return false;          // > 25 % masked rows: keep row tiles
  const int Cp = pad_channels(c.Cin), taps = c.kh * c.kw, patch_px = (16 + c.kh - 1) * (8 + c.kw - 1);
  const int bn0 = head ? 16 : std::min(128, round_up(c.Cout, 32));
  const long long m_total = tiles * N;
  const int sms = device_sm_count();
  const int kc_max = std::min(Cp, 64);
  // resident weights with the natural N tile, when a CTA walks several M tiles
  if (m_total > sms) {
    // precise plans also try 32-channel K blocks: the resident weight set is the same size, the two patch stages halve
    for (int kc = kc_max; kc >= (sp == 2 ? 32 : kc_max); kc >>= 1) {
      const long long res_bytes = (long long)(Cp / kc) * b_slot_bytes(sp, taps, bn0, kc);
      if (res_bytes <= kResidentMax && kSmemBudget - res_bytes >= 2 * a_slot_bytes(sp, patch_px, kc)) {
        *kc_out = kc; *bn_out = bn0;
        return true;
      }
    }
  }
  // Streamed weights: only when a CTA sees few M tiles (the weights pass through once per unit either way, and the
  // patch saves the activation re-reads of one box per tap).  With many M tiles per CTA the row-tile path with M
  // blocking shares each weight tile between tiles instead, and K blocks below 32 channels would turn the 49 taps of a
  // 7x7 filter into 1 KB TMA boxes.
  if (m_total >= 4LL * sms) return false;
  // (precise plans: halve the N tile before going below 32-channel K blocks; 32-byte rows ingest badly)
  for (int bn = bn0; bn >= (sp == 2 && !head ? std::min(bn0, 64) : bn0); bn >>= 1)
    for (int kc = kc_max; kc >= 32; kc >>= 1)
      if (2 * (a_slot_bytes(sp, patch_px, kc) + b_slot_bytes(sp, taps, bn, kc)) <= kSmemBudget) {
        *kc_out = kc; *bn_out = bn;
        return true;
      }
  return false;
}

// head: 0 = no, 1 = small-Cout head, 2 = head that may use the kx-GEMM form (tensor-core implementation only)
static int conv_geometry(const v2v_conv_desc& c, int head, int N, int H, int W, bool allow_reuse, int sp, ConvGeom* g) {
  memset(g, 0, sizeof(*g));
  V2V_REQUIRE(c.kh >= 1 && c.kw >= 1 && c.kh * c.kw <= V2V_MAX_TAPS, V2V_ERR_UNSUPPORTED, "kernel %dx%d unsupported",
              c.kh, c.kw);
  V2V_REQUIRE(c.stride == 1 || c.stride == 2, V2V_ERR_UNSUPPORTED, "stride %d unsupported", c.stride);
  if (!c.transposed) {
    g->out_h = (H + 2 * c.pad - c.kh) / c.stride + 1;
    g->out_w = (W + 2 * c.pad - c.kw) / c.stride + 1;
    V2V_REQUIRE(g->out_h > 0 && g->out_w > 0, V2V_ERR_INVALID, "empty conv output");
    g->grid_h = g->out_h; g->grid_w = g->out_w; g->mul = 1;
    g->pads[0] = g->pads[1] = g->pads[2] = g->pads[3] = c.pad;
    g->parity = (c.stride == 2);
  } else {
    V2V_REQUIRE(c.stride == 2, V2V_ERR_UNSUPPORTED, "transposed conv needs stride 2");
    g->out_h = (H - 1) * 2 - 2 * c.pad + c.kh + c.output_padding;
    g->out_w = (W - 1) * 2 - 2 * c.pad + c.kw + c.output_padding;
    V2V_REQUIRE(g->out_h == 2 * H && g->out_w == 2 * W, V2V_ERR_UNSUPPORTED,
                "transposed conv must exactly double the extent (got %dx%d from %dx%d)", g->out_h, g->out_w, H, W);
    g->grid_h = H; g->grid_w = W; g->mul = 2; g->parity = 0;
  }
  g->TW = g->grid_w > 64 ? 128 : 8;
  while (g->TW < g->grid_w && g->TW < 128) g->TW *= 2;
  g->TH = 128 / g->TW;
  g->R = 1;
  int ng = 0;
  if (head == 2 && !c.transposed && c.stride == 1 && c.kw >= 3 && c.kw <= 8 && c.Cout <= 4 && c.kw * c.Cout <= 32 &&
      c.kh <= 8 && g->grid_w >= 32) {
    // Small-Cout heads (7x7, 2-3 channels) are MMA-issue bound as N = 16 convolutions: 49 taps x K blocks of ~40-cycle MMAs per
    // 128 pixels.  As a GEMM with N = kw * Cout columns per INPUT pixel and taps over the kh filter rows only, a tile issues
    // kh x K-block MMAs (7x fewer) and the epilogue sums the kw horizontally shifted columns (warp shuffles).  Tile = 4 rows x
    // 32 input pixels; ONE patch of (4 + kh - 1) rows x 32 pixels serves all kh taps (operand of tap ky = the patch advanced
    // by ky rows: contiguous in shared memory, so the canonical 8-row group stride applies); tiles advance by 32 - (kw - 1)
    // pixels.  (One box per filter row on 1x128 tiles was TMA-request bound: 1792 smem rows per 122 outputs against 640 per
    // 104 here.)
    g->n_phases = 1;
    g->TW = 32; g->TH = 4; g->R = c.kh; g->RW = c.kh;
    g->headkx = c.kw;
    g->groups[ng++] = ConvGroup{0, 0, 0, 0, 0, 0};
    g->phases[0] = ConvPhase{0, ng, 0, 0};
  } else if (allow_reuse && choose_patch2d(c, head != 0, N, g->grid_h, g->grid_w, sp, &g->patch2d_kc, &g->patch2d_bn)) {
    g->n_phases = 1;
    g->TH = 16; g->TW = 8;
    g->R = c.kh * c.kw; g->RW = c.kw;
    g->groups[ng++] = ConvGroup{0, 0, 0, 0, 0, 0};
    g->phases[0] = ConvPhase{0, ng, 0, 0};
  } else if (!c.transposed && c.stride == 1) {
    g->n_phases = 1;
    if (allow_reuse && g->TH == 1 && c.kw > 1) {
      g->R = c.kw;
      for (int ky = 0; ky < c.kh; ++ky) g->groups[ng++] = ConvGroup{0, (int8_t)ky, 0, 0, (int16_t)(ky * c.kw), 0};
    } else {
      for (int ky = 0; ky < c.kh; ++ky)
        for (int kx = 0; kx < c.kw; ++kx)
          g->groups[ng++] = ConvGroup{0, (int8_t)ky, (int8_t)kx, 0, (int16_t)(ky * c.kw + kx), 0};
    }
    g->phases[0] = ConvPhase{0, ng, 0, 0};
  } else if (!c.transposed) {   // stride 2: parity-split planes, tap (ky,kx) -> plane (ky&1, kx&1), offset (ky>>1, kx>>1)
    g->n_phases = 1;
    for (int ky = 0; ky < c.kh; ++ky)
      for (int kx = 0; kx < c.kw; ++kx)
        g->groups[ng++] = ConvGroup{(int8_t)(((ky & 1) << 1) | (kx & 1)), (int8_t)(ky >> 1), (int8_t)(kx >> 1), 0,
                                    (int16_t)(ky * c.kw + kx), 0};
    g->phases[0] = ConvPhase{0, ng, 0, 0};
  } else {
    // sub-pixel phases of the stride-2 transposed conv: out(2i+a, 2j+b) gathers input (i+dy, j+dx) for the
    // taps with (a + pad - ky) even, dy = (a + pad - ky) / 2 (same in x)
    int dmin = 0, dmax = 0;
    for (int a = 0; a < 2; ++a)
      for (int k = 0; k < std::max(c.kh, c.kw); ++k)
        if (((a + c.pad - k) % 2) == 0) { int d = (a + c.pad - k) / 2; dmin = std::min(dmin, d); dmax = std::max(dmax, d); }
    g->pads[0] = g->pads[1] = -dmin; g->pads[2] = g->pads[3] = dmax;
    g->n_phases = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int begin = ng;
        for (int ky = 0; ky < c.kh; ++ky) {
          if ((a + c.pad - ky) % 2 != 0) continue;
          for (int kx = 0; kx < c.kw; ++kx) {
            if ((b + c.pad - kx) % 2 != 0) continue;
            const int dy = (a + c.pad - ky) / 2 - dmin, dx = (b + c.pad - kx) / 2 - dmin;
            V2V_REQUIRE(ng < V2V_MAX_TAPS, V2V_ERR_UNSUPPORTED, "too many taps");
            g->groups[ng++] = ConvGroup{0, (int8_t)dy, (int8_t)dx, 0, (int16_t)(ky * c.kw + kx), 0};
          }
        }
        g->phases[a * 2 + b] = ConvPhase{begin, ng, a, b};
      }
  }
  g->n_groups = ng;
  if (!g->patch2d_kc) g->RW = g->R;
  return 0;
}

// ------------------------------------------------------------------------------ graph description
struct Req { int mode, pads[4], parity; };
static bool same_req(const Req& a, const Req& b) {
  return a.mode == b.mode && a.parity == b.parity && !memcmp(a.pads, b.pads, sizeof(a.pads));
}

struct Value {
  int N, H, W, C;
  std::vector<Req> reqs;
  std::vector<int> bufs;     // index into Plan::acts, one per req
  bool interior_use = false;
  float* gval = nullptr;     // training plans: gradient of the value, dense NHWC fp32 [N][H][W][C]
  int input_slot = -1;       // >= 0: the value is an import of that IO slot (data gradient only on request)
  bool exact_bf16 = false;   // caller promise: every element is exactly representable in bf16 (one-hot labels, edge maps)
  bool detached = false;     // every consumer is a detached operand (or skipped in the backward): no gradient buffer
};
struct Raw {
  int N, H, W, C;
  int conv_op = -1;          // index of producing graph op
  RawDesc desc{};
  stat_t* stats = nullptr;           // [N][2][C] fixed-point statistics rows (zeroed at the start of every run)
  float* scale = nullptr; float* shift = nullptr;
  int tiles_per_img = 0, num_phases = 1;
  std::vector<int> running_done;   // channel offsets whose running stats already have an updating launch
  float* mean = nullptr; float* rstd = nullptr;   // training plans: saved statistics [N][C]
  float* graw = nullptr;           // training plans: gradient of the raw tensor, dense NHWC fp32 (channel stride desc.C)
  bool no_stats = false;           // backward sub-plans: the conv output feeds no norm layer
};

enum GKind { G_INPUT, G_CONV, G_NORM_ACT, G_CONV_ACT, G_HEAD, G_EXPORT, G_COMPOSITE, G_CONCAT, G_CORR, G_RAWIN, G_MAXPOOL, G_FEATL1 };
struct GOp {
  GKind kind;
  // input
  int slot = -1, C_src = 0, c_off = 0;
  int value_in = -1, value_out = -1, raw = -1;
  v2v_conv_desc conv{};
  ConvGeom geom{};
  int req_index = -1;        // which materialisation of value_in this conv reads
  v2v_norm_desc norm{};
  int act = 0; float slope = 0.f;
  int add[2] = {-1, -1};
  int n_off = 0, cC = 0;     // G_NORM_ACT: channel slice [n_off, n_off + cC) of the raw
  v2v_head_channel head[V2V_MAX_HEAD];
  CompositeParams comp{};
  std::vector<int> cat_in;   // G_CONCAT: source values in channel order
  int value_in2 = -1;        // G_CORR: second operand; G_FEATL1: the (detached) target operand
  int l1_index = 0;          // G_FEATL1: element of the output slot
  int corr[5] = {0, 0, 0, 0, 0};   // pad, kernel, max_disp, stride1, stride2
  const float* ext_raw = nullptr; int ext_C = 0;   // G_RAWIN: dense NHWC fp32 tensor owned by the parent plan (a gradient buffer)
  // backward sub-plans: pack the forward weights [Cout_f][Cin_f][kh][kw] (+ second set from output channel dg_Cout1 on) transposed
  // and flipped, so that this forward conv computes the data gradient of that conv
  int pack_dgrad = 0; const float* dg_w2 = nullptr; int dg_Cout1 = 0;
  // lowered
  bf16* wpacked = nullptr; int Ktotal = 0, Cp = 0;
  float* gdz = nullptr;      // training plans: G_HEAD / G_CONV_ACT pre-activation gradient, dense NHWC fp32 [.][Cout]
  double macs = 0.0;
  CUtensorMap tmA{}, tmB{};
  ConvKernelParams kp{};
};

enum XKind { X_IMPORT, X_CONV, X_RAWSTATS, X_FINALIZE, X_APPLY, X_EXPORT, X_COMPOSITE, X_MEMSET, X_COPY, X_CORR, X_MAXPOOL, X_FEATL1 };
struct XOp {
  XKind kind;
  int gop = -1;
  ImportParams imp{};
  ExportParams exp{};
  FinalizeParams fin{};
  ApplyParams app{};
  CompositeParams comp{};
  CopyParams copy{};
  CorrParams corr{};
  PoolParams pool{};
  FeatL1Params fl1{};
  RawDesc rawd{}; stat_t* stats = nullptr; int stats_C = 0;
  void* ms_ptr = nullptr; size_t ms_bytes = 0;
};

}  // namespace v2v

using namespace v2v;

// Tensor-core backward of one conv op of a training plan (precise plans, tensor-core implementation):
//   data gradient   = a FORWARD conv of the output gradient, run by a sub-plan on conv_umma_kernel:
//                       mode 1  stride-1 conv          -> stride-1 conv, zero pad k-1, weights transposed + flipped; the result covers
//                                                         the padded input extent and fold_add folds the (reflect) halo back
//                       mode 2  transposed conv (s 2)  -> stride-2 conv of dY with the same weight tensor
//                       mode 3  stride-2 conv          -> transposed conv of dY with the same weight tensor
//   weight gradient = wgrad_umma_kernel over the two activation buffers the passes above left in place
// Mode 0: the fp32 SIMT backward (backward.cu) does all of the conv, `simt` says why; wgrad false with mode > 0: it does the
// weight gradient, `wg_simt` says why.
struct BwdUnit {
  int gop = -1, mode = 0;
  v2v_plan* child = nullptr;
  int child_raw = -1;
  bool wgrad = false;
  std::string simt, wg_simt;
  CUtensorMap tmOut{}, tmIn{};
  WgradParams wg{};
  int M = 0, M1 = 0, Nv = 0;
};

struct v2v_plan {
  std::vector<BwdUnit> bwd;     // one per live conv op of a training plan, in graph order
  std::vector<int> bwd_of;      // per graph op: its unit in bwd when that runs on the tensor cores (mode > 0), else -1
  float* wg_stage = nullptr;    // staging buffer of the weight-gradient kernel (largest unit)
  int pad_min = 0;              // minimum padded channel count of every buffer (a backward sub-plan's dY: see choose_backward_unit)

  int device = 0;
  int impl = V2V_IMPL_UMMA;
  int precise = 0;            // V2V_PREC_BF16X3: split activations / weights, fp32 raw tensors, 3 MMAs per K block
  int sp() const { return precise ? 2 : 1; }
  bool lowered = false, finalized = false;
  bool train = false;          // keep what the backward needs (batch statistics) and allocate gradient buffers
  void* garena = nullptr; size_t garena_bytes = 0;
  std::vector<float*> gslot;   // per IO slot: plan-internal gradient of a head output produced by the composite backward
  float* gsums = nullptr;      // scratch of the norm backward [2][N][Cmax]
  float* train_stats = nullptr;
  std::vector<Value> values;
  std::vector<Raw> raws;
  std::vector<GOp> gops;
  std::vector<ActDesc> acts;
  std::vector<int> act_pad_mode;
  std::vector<char> op_live;    // per graph op: visited by the backward (0: all its outputs only feed detached operands)
  std::vector<XOp> xops;
  int n_slots = 0;
  double conv_macs = 0.0;
  struct BiasAffine { float* scale; float* shift; const float* bias; int N, C, stride; };
  std::vector<BiasAffine> bias_affines;   // norm-less biased convs routed through the normalise pass (scale 1, shift bias)
  // arena layout (size_arena) and device memory
  struct RawOff { size_t raw = 0, stats = 0, scale = 0, shift = 0; };
  bool sized = false, arena_owned = true;
  std::vector<size_t> act_off, w_off, corr_off, l1_off;
  std::vector<RawOff> raw_off;
  size_t stats_begin = 0, stats_end = 0;
  void* arena = nullptr; size_t arena_bytes = 0;
  void** io_dev = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  cudaStream_t graph_stream = nullptr;
};


extern "C" int v2v_plan_create(int device, int conv_impl, v2v_plan** out);
extern "C" int v2v_g_conv(v2v_plan* p, int value_in, const v2v_conv_desc* c, int* raw_out);
extern "C" int v2v_plan_finalize(v2v_plan* P, v2v_stream_t stream_);
extern "C" { static int new_value(v2v_plan* p, int N, int H, int W, int C); static int size_arena(v2v_plan* P); }

namespace v2v {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

static CUtensorMapSwizzle swizzle_for(int kc) {
  return kc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

static int make_tmap_act(CUtensorMap* tm, const ActDesc& a, int box_w, int box_h, int kc) {
  EncodeTiledFn fn = get_encode_fn();
  V2V_REQUIRE(fn, V2V_ERR_STATE, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t cs = (cuuint64_t)a.Cs();      // precise plans: [hi | lo] halves, the lo half at channel coordinate C
  cuuint64_t dims[5] = {cs, (cuuint64_t)a.Wp, (cuuint64_t)a.Hp, (cuuint64_t)a.P, (cuuint64_t)a.N};
  cuuint64_t strides[4] = {cs * 2, (cuuint64_t)a.Wp * cs * 2, (cuuint64_t)a.Hp * a.Wp * cs * 2,
                           (cuuint64_t)a.P * a.Hp * a.Wp * cs * 2};
  cuuint32_t box[5] = {(cuuint32_t)kc, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, a.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_for(kc), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  V2V_REQUIRE(r == CUDA_SUCCESS, V2V_ERR_STATE, "cuTensorMapEncodeTiled(A) failed: %d (C=%d Wp=%d Hp=%d P=%d N=%d box %dx%d)",
              (int)r, a.C, a.Wp, a.Hp, a.P, a.N, box_w, box_h);
  return 0;
}

static int make_tmap_w(CUtensorMap* tm, bf16* w, int Ktotal /* columns, both halves */, int Cout, int BN, int kc) {
  EncodeTiledFn fn = get_encode_fn();
  V2V_REQUIRE(fn, V2V_ERR_STATE, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)Ktotal, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)Ktotal * 2};
  cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)BN};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_for(kc), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  V2V_REQUIRE(r == CUDA_SUCCESS, V2V_ERR_STATE, "cuTensorMapEncodeTiled(B) failed: %d (K=%d Cout=%d BN=%d)", (int)r, Ktotal,
              Cout, BN);
  return 0;
}

static ActDesc make_act(const Value& v, const Req& r, int split) {
  ActDesc a{};
  a.split = split;
  a.base = nullptr;
  a.N = v.N; a.H = v.H; a.W = v.W; a.Cvalid = v.C; a.C = pad_channels(v.C);
  a.pad_t = r.pads[0]; a.pad_l = r.pads[1]; a.pad_b = r.pads[2]; a.pad_r = r.pads[3];
  a.parity = r.parity;
  const int Hpad = v.H + a.pad_t + a.pad_b, Wpad = v.W + a.pad_l + a.pad_r;
  if (a.parity) { a.P = 4; a.Hp = (Hpad + 1) / 2; a.Wp = (Wpad + 1) / 2; }
  else { a.P = 1; a.Hp = Hpad; a.Wp = Wpad; }
  return a;
}

static int add_req(Value& v, const Req& r) {
  for (size_t i = 0; i < v.reqs.size(); ++i)
    if (same_req(v.reqs[i], r)) return (int)i;
  v.reqs.push_back(r);
  return (int)v.reqs.size() - 1;
}

static Req conv_req(const v2v_conv_desc& c, const ConvGeom& g) {
  Req r{};
  r.mode = c.transposed ? PAD_ZERO : (c.pad == 0 ? PAD_ZERO : c.pad_mode);
  memcpy(r.pads, g.pads, sizeof(r.pads));
  r.parity = g.parity;
  return r;
}

// Backward liveness.  A value all of whose consumers are detached operands (the target side of a feature L1), or ops that
// are themselves skipped, gets no gradient buffer, and an op all of whose outputs are such values is skipped by the
// backward (no data-gradient conv, no dY buffer).  Ops are in execution order, so walking them backwards sees every
// consumer of a value before its producer.  Heads, exports, composites and feature L1 nodes feed outputs and always run.
// A value that has no consumer at all keeps its gradient buffer: in a plan without feature L1 nodes every op stays live.
static void mark_backward_liveness(v2v_plan* P) {
  const size_t nv = P->values.size(), nr = P->raws.size();
  std::vector<int> uses(nv, 0), raw_uses(nr, 0);
  std::vector<char> live(nv, 0), raw_live(nr, 0);
  auto dead = [&](int v) { return uses[v] > 0 && !live[v]; };
  auto use = [&](int v, bool l) { if (v < 0) return; ++uses[v]; if (l) live[v] = 1; };
  P->op_live.assign(P->gops.size(), 1);
  for (int i = (int)P->gops.size() - 1; i >= 0; --i) {
    const GOp& op = P->gops[i];
    bool ol = true;
    switch (op.kind) {
      case G_INPUT: case G_RAWIN: case G_NORM_ACT: case G_CONV_ACT: case G_CONCAT: case G_CORR: case G_MAXPOOL:
        ol = !dead(op.value_out); break;
      case G_CONV: ol = !(raw_uses[op.raw] > 0 && !raw_live[op.raw]); break;
      default: break;
    }
    P->op_live[i] = ol;
    switch (op.kind) {
      case G_CONV: case G_CONV_ACT: case G_HEAD: case G_EXPORT: case G_MAXPOOL: use(op.value_in, ol); break;
      case G_NORM_ACT: ++raw_uses[op.raw]; if (ol) raw_live[op.raw] = 1; use(op.add[0], ol); use(op.add[1], ol); break;
      case G_CONCAT: for (int v : op.cat_in) use(v, ol); break;
      case G_CORR: use(op.value_in, ol); use(op.value_in2, ol); break;
      case G_FEATL1: use(op.value_in, true); use(op.value_in2, false); break;
      default: break;
    }
  }
  for (size_t v = 0; v < nv; ++v) P->values[v].detached = dead((int)v);
}

// Host-only lowering: requirements, buffer descriptors (no addresses), kernel parameter skeletons.
static int lower(v2v_plan* P) {
  if (P->lowered) return 0;
  // pass 1: consumer requirements
  for (auto& op : P->gops) {
    if (op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD) {
      Value& vin = P->values[op.value_in];
      int rc = conv_geometry(op.conv, op.kind == G_HEAD ? (P->impl == V2V_IMPL_UMMA ? 2 : 1) : 0, vin.N, vin.H, vin.W, true,
                             P->sp(), &op.geom);
      if (rc) return rc;
      op.req_index = add_req(vin, conv_req(op.conv, op.geom));
      const v2v_conv_desc& c = op.conv;
      const double px = op.conv.transposed ? (double)vin.N * vin.H * vin.W : (double)vin.N * op.geom.out_h * op.geom.out_w;
      op.macs = px * c.Cin * c.Cout * c.kh * c.kw;
      P->conv_macs += op.macs;
    } else if (op.kind == G_NORM_ACT) {
      for (int k = 0; k < 2; ++k) if (op.add[k] >= 0) P->values[op.add[k]].interior_use = true;
    } else if (op.kind == G_EXPORT) {
      P->values[op.value_in].interior_use = true;
    } else if (op.kind == G_CONCAT) {
      for (int v : op.cat_in) P->values[v].interior_use = true;
    } else if (op.kind == G_CORR || op.kind == G_FEATL1) {
      P->values[op.value_in].interior_use = true;
      P->values[op.value_in2].interior_use = true;
    } else if (op.kind == G_MAXPOOL) {
      P->values[op.value_in].interior_use = true;
    }
  }
  mark_backward_liveness(P);
  for (auto& v : P->values) {
    if (v.reqs.empty()) { Req r{}; r.mode = PAD_NONE; v.reqs.push_back(r); }
    v.bufs.clear();
    for (auto& r : v.reqs) {
      P->acts.push_back(make_act(v, r, P->precise));
      P->act_pad_mode.push_back(r.mode);
      v.bufs.push_back((int)P->acts.size() - 1);
    }
  }
  P->lowered = true;
  return 0;
}

static int max_phase_groups(const ConvGeom& g) {
  int m = 0;
  for (int i = 0; i < g.n_phases; ++i) m = std::max(m, g.phases[i].group_end - g.phases[i].group_begin);
  return m;
}

// The configuration of one conv_umma_kernel launch that fill_conv_params derives every other kernel parameter from.
struct ConvTiling {
  int kc, BN, MG;          // K block, N tile, M tiles accumulated side by side per weight pass
  int b_resident;          // the weights of one (phase, N tile) stay in shared memory
  int ring2, TB, SBr;      // decoupled operand rings: taps per weight chunk, weight slots
  int CG, SG;              // K-loop steps per commit group, group slots
};

// Chooses the tiling from the conv, its geometry and the tile grid / patch extent already in kp.  The rules apply in order;
// each later rule refines what the earlier ones chose.
static ConvTiling choose_tiling(const v2v_plan* P, const GOp& op, const ConvKernelParams& kp) {
  const ConvGeom& g = op.geom;
  const v2v_conv_desc& c = op.conv;
  const bool head = op.kind == G_HEAD, p2d = g.patch2d_kc > 0;
  const int sp = P->sp(), sms = device_sm_count(), budget = kSmemBudget;
  const int Cp = kp.Cp, kc_nat = std::min(Cp, 64), bn_nat = std::min(128, round_up(c.Cout, 32));
  const int m_tiles = kp.N * kp.tiles_x * kp.tiles_y;
  auto a_slot = [&](int kc) { return a_slot_bytes(sp, kp.PW * kp.PH, kc); };
  ConvTiling t{};
  t.kc = kc_nat; t.BN = head ? (g.headkx ? 32 : 16) : bn_nat; t.MG = 1;
  if (p2d) { t.kc = g.patch2d_kc; if (!head) t.BN = g.patch2d_bn; }
  if (g.headkx) {
    // K block of a kx-GEMM head: the largest whose patch ring (2 stages) fits next to the resident weight set, or, failing
    // that, whose two streamed stages fit
    for (; t.kc > 16; t.kc >>= 1) {
      const int a_sl = a_slot(t.kc), b_sl = b_slot_bytes(sp, g.R, t.BN, t.kc);
      const long long res = (long long)(Cp / t.kc) * b_sl;
      if ((res <= kResidentMax && budget - res >= 2 * a_sl) || 2 * (a_sl + b_sl) <= budget) break;
    }
  }
  // M blocking for row-tile filters whose weights must be streamed (the 7x7 stems over the 108-channel label input):
  // per M tile such a layer pulls taps*Cp*BN*2 bytes of weights through L2 -> SM (802 KB for 108->48, 13 GB per launch at
  // 2048x1024), more than an SM ingests at the full MMA rate.  MG = 2 consecutive x tiles accumulate side by side in
  // registers and share every weight tile, within the accumulator budget V2V_MAX_ACC_COLS.  64-byte rows (32-channel K
  // blocks) cost TMA request rate, so they are used only where they buy an exact N tile (Cout = 96).
  bool mblock = false;
  if (!p2d && !c.transposed && c.stride == 1 && g.R >= 5 && g.n_phases == 1 && !head && m_tiles >= 4 * sms &&
      (long long)sp * c.kh * c.kw * Cp * std::min(64, t.BN) * 2 > kResidentMax) {   // cannot stay resident
    int c_kc = kc_nat, c_bn = std::min(64, round_up(c.Cout, 32));
    if (round_up(c.Cout, 32) == 96 && Cp % 32 == 0) { c_kc = 32; c_bn = 96; }
    const int c_mg = std::min(2, V2V_MAX_ACC_COLS / c_bn);      // (the exact 96-wide N tile leaves room for one tile)
    // precise plans double every slot: fall back through smaller K blocks / N tiles until two stages fit
    const int cand[4][3] = {{c_kc, c_bn, c_mg}, {32, c_bn, c_mg}, {32, 64, c_mg}, {32, 64, 1}};
    for (int ci = 0; ci < (sp == 2 ? 4 : 1) && !mblock; ++ci) {
      const int t_kc = cand[ci][0], t_bn = cand[ci][1], t_mg = cand[ci][2];
      if (Cp % t_kc || kp.tiles_x % t_mg) continue;
      if (2 * (t_mg * a_slot(t_kc) + b_slot_bytes(sp, g.R, t_bn, t_kc)) <= budget) { t.kc = t_kc; t.BN = t_bn; t.MG = t_mg; mblock = true; }
    }
  }
  if (!p2d && !mblock && g.R > 1) {
    // a weight slot holds the R taps served by one activation patch; keep >= 2 slots + 3 patches in the budget
    auto fits = [&](int kc, int bn) { return 2 * sp * g.R * bn * kc * 2 + 3 * a_slot(kc) <= budget; };
    if (sp == 2 && !g.headkx) {
      // precise plans: every slot doubles.  N tiles below 64 make the (3x) MMAs issue bound, so try (K block, N tile) in the
      // order (kc, BN), (kc, BN/2 >= 64), (32, BN), (32, BN/2 >= 64) before falling through to the generic halving
      const int bn0 = t.BN, kc0 = t.kc;
      for (int i = 0; i < 4; ++i) {
        const int t_kc = (i & 2) ? 32 : kc0, t_bn = (i & 1) ? bn0 / 2 : bn0;
        if (t_kc > kc0 || ((i & 1) && (t_bn < 64 || t_bn % 32))) continue;
        if (fits(t_kc, t_bn)) { t.kc = t_kc; t.BN = t_bn; break; }
      }
    }
    while (t.BN > 32 && !fits(t.kc, t.BN)) t.BN = std::max(32, t.BN / 2 / 32 * 32);
  }
  // Precise convs whose 128-wide N tile gives at most one work unit per SM (the 512->512 and 1024->1024 3x3 convs at 32x64,
  // 64 and 128 units of one M tile each) take a 64-wide tile instead.  Each unit then streams 48 instead of 64 KB per K step,
  // so three stages fit where two did, and the stage pipeline, not the MMA rate, is what bounds these layers: one round of
  // half-width units fills the SMs the 64-unit layers left idle, and two rounds of them beat one round of full-width units
  // (1024->1024: 0.278 against 0.348 ms on an H100 SXM).  Splitting N changes no output's sum, and a CTA's units belong to
  // different (N tile) keys, so it still adds the statistics of exactly one M tile per channel and flush.
  if (sp == 2 && !p2d && !mblock && !head && g.n_phases == 1 && t.BN == 128 && c.Cout % 128 == 0 &&
      (long long)m_tiles * (c.Cout / 128) <= sms)
    t.BN = 64;
  // resident weights pay off when a CTA walks several M tiles with the same weights
  const int nB = max_phase_groups(g) * (Cp / t.kc);            // weight slots of one (phase, N tile)
  const int b_slot = b_slot_bytes(sp, g.R, t.BN, t.kc);
  t.b_resident = (t.MG == 1 && m_tiles > sms && (long long)nB * b_slot <= kResidentMax &&
                  budget - nB * b_slot >= 2 * a_slot(t.kc)) ? 1 : 0;
  if (p2d && !t.b_resident && 2 * (a_slot(t.kc) + b_slot) > budget)
    set_error("internal: 2-D patch conv does not fit (a %d b %d)", a_slot(t.kc), b_slot);
  // Decoupled operand rings for streamed-weight layers whose coupled stages forced a narrow K block or N tile (see
  // ConvKernelParams::ring2): 64-byte rows cost TMA request rate and narrow N tiles cost MMA issue slots.
  // Precise plans only: bf16 plans and the exact-input finest stem keep the coupled stages (fewer barrier round trips
  // per MMA).
  if (sp == 2 && !kp.a_exact && P->impl == V2V_IMPL_UMMA && !t.b_resident && g.R >= 3 && !g.headkx && g.n_phases == 1 &&
      !head && (t.kc < kc_nat || t.BN < bn_nat)) {
    // N tile: the natural one unless that leaves SMs idle (512->512 @32x64: 64 tiles of 128 columns)
    const long long units_nat = (long long)m_tiles * ((c.Cout + bn_nat - 1) / bn_nat);
    const int bns[2] = {bn_nat, bn_nat / 2}, mgs[2] = {t.MG, 1};
    const bool too_few = units_nat * 5 < (long long)sms * 3;      // then the coupled path with a halved N tile fills the SMs
    for (int bi = 0; bi < 2 && !t.ring2 && !too_few; ++bi) {
      const int bn = bns[bi];
      if (bi == 1 && (bn < 64 || bn % 32)) continue;
      for (int mi = 0; mi < 2 && !t.ring2; ++mi) {
        const int mg = mgs[mi];
        if (kp.tiles_x % mg || mg * std::max(32, bn) > V2V_MAX_ACC_COLS || (mi == 1 && mgs[0] == 1)) continue;
        // taps per weight chunk: as many as leave >= 3 chunks in flight (every chunk costs a commit group and a barrier
        // round trip: fewer, longer chunks)
        for (int tb = std::min(g.R, 4); tb >= 1 && !t.ring2; --tb) {
          const int sbr = (budget - 2 * mg * a_slot(kc_nat)) / b_slot_bytes(sp, tb, bn, kc_nat);
          if (sbr >= 3) { t.ring2 = 1; t.kc = kc_nat; t.BN = bn; t.MG = mg; t.TB = tb; t.SBr = std::min(8, sbr); t.CG = 1; t.SG = 2; }
        }
      }
    }
  }
  // Commit groups: CG consecutive K-loop steps share one barrier pair and one wgmma commit group, so that the barrier
  // round trips are paid once per group; `est` is a step's MMA work in cycle-like units (small-N MMAs are floored).
  if (!t.ring2) {
    const int slot = t.MG * a_slot(t.kc) + (t.b_resident ? 0 : b_slot);
    const int avail = budget - (t.b_resident ? nB * b_slot : 0);
    const int nslots = std::max(2, avail / slot);
    const int steps = nB;
    const int est = (sp == 2 ? (kp.a_exact ? 2 : 3) : 1) * t.MG * g.R * (t.kc / 16) * std::max(40, t.BN / 2);
    if (steps * est <= 6000 && 2 * steps <= nslots) t.CG = steps;           // one group per tile, double buffered
    else {
      t.CG = std::max(1, std::min({(1500 + est - 1) / est, steps, nslots / 2}));
      if (nslots / t.CG < 3 && t.CG > 1) t.CG = std::max(1, nslots / 3);
    }
    t.SG = std::max(2, std::min(8, nslots / t.CG));
  }
  return t;
}

static void fill_conv_params(v2v_plan* P, GOp& op) {
  const Value& vin = P->values[op.value_in];
  const ConvGeom& g = op.geom;
  const v2v_conv_desc& c = op.conv;
  const bool p2d = g.patch2d_kc > 0;
  const int sp = P->sp();
  ConvKernelParams& kp = op.kp;
  memset(&kp, 0, sizeof(kp));
  // geometry: the tile grid and the A patch extent in pixels
  kp.N = vin.N; kp.TH = g.TH; kp.TW = g.TW;
  kp.headkx = g.headkx;
  kp.tile_dx = g.headkx ? g.TW - (g.headkx - 1) : g.TW;
  kp.tiles_x = (g.grid_w + kp.tile_dx - 1) / kp.tile_dx; kp.tiles_y = (g.grid_h + g.TH - 1) / g.TH;
  kp.grid_h = g.grid_h; kp.grid_w = g.grid_w;
  kp.Cout = c.Cout;
  kp.Cp = pad_channels(c.Cin);
  kp.R = g.R; kp.RW = g.RW;
  kp.PW = p2d ? g.TW + c.kw - 1 : (g.headkx ? g.TW : g.TW + g.R - 1);
  kp.PH = p2d || g.headkx ? g.TH + c.kh - 1 : g.TH;
  kp.split = P->precise;
  kp.a_exact = (P->precise && vin.exact_bf16) ? 1 : 0;
  kp.num_phases = g.n_phases;
  memcpy(kp.phases, g.phases, sizeof(kp.phases));
  memcpy(kp.groups, g.groups, sizeof(kp.groups));
  // the choice, and every field that follows from it
  const ConvTiling t = choose_tiling(P, op, kp);
  kp.kc = t.kc; kp.BN = t.BN; kp.MG = t.MG; kp.b_resident = t.b_resident;
  kp.ring2 = t.ring2; kp.TB = t.TB; kp.SBr = t.SBr; kp.CG = t.CG; kp.SG = t.SG;
  kp.cblocks = kp.Cp / kp.kc;
  kp.row_bytes = kp.kc * 2; kp.kmma = kp.kc / 16;
  kp.layout_type = kp.kc == 64 ? 2 : (kp.kc == 32 ? 4 : 6);
  // 8-row core-matrix groups of the A operand are SBO bytes apart: the canonical 8 rows for row tiles, one patch row (PW
  // pixels) in 2-D patch mode
  kp.sbo_bytes = 8 * kp.row_bytes;
  kp.sbo_a_bytes = p2d ? kp.PW * kp.row_bytes : 8 * kp.row_bytes;
  kp.a_half_bytes = a_slot_bytes(1, kp.PW * kp.PH, kp.kc);
  kp.a_slot_bytes = sp * kp.a_half_bytes;
  kp.b_half_bytes = b_slot_bytes(1, kp.ring2 ? kp.TB : g.R, kp.BN, kp.kc);   // a ring2 weight slot holds TB taps
  kp.b_slot_bytes = sp * kp.b_half_bytes;
  kp.SB = kp.b_resident ? max_phase_groups(g) * kp.cblocks : 0;
  kp.n_tiles = (kp.Cout + kp.BN - 1) / kp.BN;
  kp.kmma_last = std::min(kp.kmma, std::max(1, (c.Cin - (kp.cblocks - 1) * kp.kc + 15) / 16));
  kp.BNt = conv_umma_tail_width(kp);
  kp.m_total = kp.N * (kp.tiles_x / kp.MG) * kp.tiles_y;       // M units: MG consecutive x tiles each
  kp.total_units = kp.m_total * kp.n_tiles * g.n_phases;
  kp.grid = std::min(kp.total_units, device_sm_count());
  kp.oy_mul = kp.ox_mul = g.mul;
  kp.out_H = g.out_h; kp.out_W = g.out_w;
  kp.bias = c.bias;
  kp.lrelu_slope = op.slope;
  kp.act = op.act;
  op.Cp = kp.Cp; op.Ktotal = (g.headkx ? c.kh : c.kh * c.kw) * kp.Cp;
  kp.Khalf = op.Ktotal;
}

static int pack_one(const GOp& op, cudaStream_t stream) {
  PackParams pp{};
  pp.w = op.conv.weight; pp.transposed = op.conv.transposed;
  pp.w2 = op.conv.Cout2 > 0 ? op.conv.weight2 : nullptr; pp.Cout1 = op.conv.Cout - op.conv.Cout2;
  pp.Cout = op.conv.Cout; pp.Cin = op.conv.Cin; pp.kh = op.conv.kh; pp.kw = op.conv.kw;
  pp.Cp = op.Cp; pp.ntaps = op.geom.headkx ? op.conv.kh : op.conv.kh * op.conv.kw; pp.split = op.kp.split; pp.headkx = op.geom.headkx;
  for (int ky = 0; ky < op.conv.kh; ++ky)
    for (int kx = 0; kx < op.conv.kw; ++kx) { pp.tap_ky[ky * op.conv.kw + kx] = (int8_t)ky; pp.tap_kx[ky * op.conv.kw + kx] = (int8_t)kx; }
  pp.out = op.wpacked;
  if (op.pack_dgrad) { pp.dgrad = 1; pp.w2 = op.dg_w2; pp.Cout1 = op.dg_Cout1; }
  V2V_CUDA(launch_pack_weights(pp, stream));
  return 0;
}

static int run_xop(v2v_plan* P, const XOp& x, cudaStream_t s) {
  switch (x.kind) {
    case X_IMPORT: V2V_CUDA(launch_import_nchw(x.imp, s)); break;
    case X_EXPORT: V2V_CUDA(launch_export_nchw(x.exp, s)); break;
    case X_FINALIZE: V2V_CUDA(launch_stats_finalize(x.fin, s)); break;
    case X_APPLY: V2V_CUDA(launch_norm_apply(x.app, s)); break;
    case X_COMPOSITE: V2V_CUDA(launch_composite(x.comp, s)); break;
    case X_RAWSTATS: V2V_CUDA(launch_raw_stats(x.rawd, x.stats, x.stats_C, s)); break;
    case X_MEMSET: V2V_CUDA(cudaMemsetAsync(x.ms_ptr, 0, x.ms_bytes, s)); break;
    case X_COPY: V2V_CUDA(launch_act_copy(x.copy, s)); break;
    case X_CORR:
      V2V_CUDA(launch_correlation(x.corr.in1, x.corr.in2, x.corr.out, x.corr.N, x.corr.C, x.corr.H, x.corr.W, x.corr.pad, x.corr.k,
                                  x.corr.max_disp, x.corr.s1, x.corr.s2, s));
      break;
    case X_MAXPOOL: V2V_CUDA(launch_maxpool2(x.pool, s)); break;
    case X_FEATL1: V2V_CUDA(launch_feature_l1(x.fl1, s)); break;
    case X_CONV: {
      const GOp& op = P->gops[x.gop];
      if (P->impl == V2V_IMPL_UMMA) V2V_CUDA(launch_conv_umma(op.tmA, op.tmB, op.kp, s));
      else V2V_CUDA(launch_conv_simt(P->acts[P->values[op.value_in].bufs[op.req_index]], op.wpacked, op.Ktotal, op.kp, s));
      break;
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------ training: gradient buffers
static int alloc_training(v2v_plan* P, cudaStream_t stream) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = round_up_sz(off + bytes, 256); return o; };
  std::vector<size_t> vo(P->values.size()), ro(P->raws.size()), go(P->gops.size(), 0), so(P->n_slots, (size_t)-1);
  int cmax = 1, nmax = 1;
  // (values and ops the backward skips, mark_backward_liveness, get no buffer)
  const size_t none = (size_t)-1;
  for (size_t i = 0; i < P->values.size(); ++i) {
    const Value& v = P->values[i];
    vo[i] = v.detached ? none : take((size_t)v.N * v.H * v.W * v.C * 4);
    nmax = std::max(nmax, v.N);
  }
  for (size_t i = 0; i < P->raws.size(); ++i) {
    const Raw& r = P->raws[i];
    ro[i] = (r.conv_op >= 0 && !P->op_live[r.conv_op]) ? none : take(r.desc.elems() * 4);
    cmax = std::max(cmax, r.C);
  }
  std::vector<char> has_gdz(P->gops.size(), 0);
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (!P->op_live[i]) continue;
    if (op.kind == G_HEAD || op.kind == G_CONV_ACT) {
      has_gdz[i] = 1;
      const Value& vin = P->values[op.value_in];
      go[i] = take((size_t)vin.N * op.geom.out_h * op.geom.out_w * round_up(op.conv.Cout, 8) * 4);   // channel stride: multiple of 8
      cmax = std::max(cmax, op.conv.Cout);
    } else if (op.kind == G_COMPOSITE) {
      const CompositeParams& c = op.comp;
      const size_t px = (size_t)c.N * c.H * c.W * 4;
      so[c.s_raw] = take(3 * px);
      if (c.s_flow >= 0) so[c.s_flow] = take(2 * px);
      if (c.s_weight >= 0) so[c.s_weight] = take(px);
      if (c.s_fg >= 0) so[c.s_fg] = take(3 * px);
    }
  }
  const size_t sums_off = take((size_t)2 * nmax * cmax * 4);
  P->garena_bytes = off;
  V2V_CUDA(cudaMalloc(&P->garena, P->garena_bytes));
  V2V_CUDA(cudaMemsetAsync(P->garena, 0, P->garena_bytes, stream));
  uint8_t* b = reinterpret_cast<uint8_t*>(P->garena);
  for (size_t i = 0; i < P->values.size(); ++i) P->values[i].gval = vo[i] == none ? nullptr : reinterpret_cast<float*>(b + vo[i]);
  for (size_t i = 0; i < P->raws.size(); ++i) P->raws[i].graw = ro[i] == none ? nullptr : reinterpret_cast<float*>(b + ro[i]);
  for (size_t i = 0; i < P->gops.size(); ++i) if (has_gdz[i]) P->gops[i].gdz = reinterpret_cast<float*>(b + go[i]);
  P->gslot.assign(P->n_slots, nullptr);
  for (int sidx = 0; sidx < P->n_slots; ++sidx) if (so[sidx] != (size_t)-1) P->gslot[sidx] = reinterpret_cast<float*>(b + so[sidx]);
  P->gsums = reinterpret_cast<float*>(b + sums_off);
  return 0;
}


// ------------------------------------------------------------------------------ training: tensor-core backward units
static bool bwd_tensor_enabled() {      // read per plan, so that one process can build both variants (tests)
  const char* e = getenv("V2V_BWD");
  return !(e && !strcmp(e, "simt"));
}

// The weight gradient's operands: OUT is the gradient side, IN the activation side.  A transposed conv's data gradient is a
// stride-2 conv of dY, so there the roles of the forward input x and of dY swap.
static void wgrad_operands(const v2v_plan* P, const BwdUnit& u, const ActDesc** out, const ActDesc** in) {
  const v2v_plan* C = u.child;
  const GOp& op = P->gops[u.gop];
  const ActDesc* a_dy = &C->acts[C->values[C->gops[0].value_out].bufs[0]];
  const ActDesc* a_x = &P->acts[P->values[op.value_in].bufs[op.req_index]];
  *out = u.mode == 2 ? a_x : a_dy;
  *in = u.mode == 2 ? a_dy : a_x;
}

// Host-only half of the backward of live conv op i: the data-gradient mode and its sub-plan (built and lowered, no device
// memory), and the weight-gradient launch or the reason it stays on the SIMT kernel.  u.child, when set, belongs to the
// caller.  The device half is build_backward_units; v2v_plan_describe reports the same choice without a device.
static int choose_backward_unit(v2v_plan* P, int i, BwdUnit& u) {
  const GOp& op = P->gops[i];
  const v2v_conv_desc& c = op.conv;
  const Value& vin = P->values[op.value_in];
  const int oh = op.geom.out_h, ow = op.geom.out_w;
  char why[200];
  u.gop = i;
  if (!P->precise) { u.simt = "bf16 plan"; return 0; }
  if (P->impl != V2V_IMPL_UMMA) { u.simt = "SIMT conv implementation"; return 0; }
  if (!bwd_tensor_enabled()) { u.simt = "V2V_BWD=simt"; return 0; }
  v2v_conv_desc cd{};
  cd.Cin = c.Cout; cd.Cout = c.Cin; cd.kh = c.kh; cd.kw = c.kw; cd.pad_mode = V2V_PAD_ZERO; cd.weight = c.weight;
  if (!c.transposed && c.stride == 1 && c.kh == c.kw && c.pad <= c.kh - 1 && (c.pad_mode != V2V_PAD_REFLECT || c.pad < std::min(vin.H, vin.W))) {
    u.mode = 1; cd.stride = 1; cd.pad = c.kh - 1;
  } else if (c.transposed && c.Cout2 == 0) {
    u.mode = 2; cd.stride = 2; cd.pad = c.pad;
  } else if (!c.transposed && c.stride == 2 && c.Cout2 == 0 && c.kh == c.kw && 2 + 2 * c.pad - c.kh >= 0 && 2 * oh >= vin.H && 2 * ow >= vin.W) {
    // the transposed conv is asked for exactly 2 oh x 2 ow outputs (output_padding 2 + 2 pad - k; for 4x4 / pad 2 that is one
    // row more than nn.ConvTranspose2d would accept, the extra rows are simply cropped by fold_add)
    u.mode = 3; cd.stride = 2; cd.pad = c.pad; cd.transposed = 1; cd.output_padding = 2 + 2 * c.pad - c.kh;
  } else {
    snprintf(why, sizeof(why), "no data-gradient mode for k %dx%d stride %d pad %d (mode %d) transposed %d Cout2 %d on %dx%d -> %dx%d",
             c.kh, c.kw, c.stride, c.pad, c.pad_mode, c.transposed, c.Cout2, vin.H, vin.W, oh, ow);
    u.simt = why;
    return 0;
  }
  // ---- sub-plan: dY (dense fp32 NHWC, channel stride round_up(Cout, 8)) -> halo-padded split activation -> conv
  // the weight-gradient GEMM needs >= 64 channels on one side: when the forward input AND output are narrow (the 32 -> 3
  // foreground head), the sub-plan carries dY padded to 64 channels
  const int pad_min = (pad_channels(c.Cout) < 64 && pad_channels(c.Cin) < 64) ? 64 : 0;
  v2v_plan* C = nullptr;
  int rc = v2v_plan_create(P->device, P->impl, &C); if (rc) return rc;
  C->precise = P->precise; C->pad_min = pad_min;
  u.child = C;
  PadScope scope(pad_min);
  GOp gi; gi.kind = G_RAWIN; gi.ext_raw = op.kind == G_CONV ? P->raws[op.raw].graw : op.gdz; gi.ext_C = round_up(c.Cout, 8);
  gi.value_out = new_value(C, vin.N, oh, ow, c.Cout);
  C->gops.push_back(gi);
  rc = v2v_g_conv(C, gi.value_out, &cd, &u.child_raw); if (rc) return rc;
  C->raws[u.child_raw].no_stats = true;
  if (u.mode == 1) { GOp& co = C->gops.back(); co.pack_dgrad = 1; co.dg_w2 = c.Cout2 > 0 ? c.weight2 : nullptr; co.dg_Cout1 = c.Cout - c.Cout2; }
  rc = size_arena(C); if (rc) return rc;
  {
    const Raw& cr = C->raws[u.child_raw];
    const int eh = u.mode == 1 ? vin.H + 2 * c.pad : vin.H, ew = u.mode == 1 ? vin.W + 2 * c.pad : vin.W;
    V2V_REQUIRE(cr.H >= eh && cr.W >= ew && (u.mode == 3 || (cr.H == eh && cr.W == ew)) && cr.C == c.Cin, V2V_ERR_STATE,
                "internal: data-gradient conv of op %d yields %dx%dx%d, expected %dx%dx%d", i, cr.H, cr.W, cr.C, eh, ew, c.Cin);
  }
  // ---- weight gradient on the tensor cores: OUT (gradient side) x IN (activation side) over the driving grid
  const ActDesc *pa_out, *pa_in;
  wgrad_operands(P, u, &pa_out, &pa_in);
  const ActDesc& a_out = *pa_out, &a_in = *pa_in;
  const int wmin = std::min(a_out.Wp, a_in.Wp);
  const int kp = wmin >= 64 ? 64 : (wmin >= 32 ? 32 : (wmin >= 16 ? 16 : 0));
  const bool wide_out = a_out.C % 64 == 0, wide_in = a_in.C % 64 == 0;
  const bool narrow_ok_out = a_out.C == 16 || a_out.C == 32, narrow_ok_in = a_in.C == 16 || a_in.C == 32;
  if (kp == 0) snprintf(why, sizeof(why), "operand rows of %d pixels (< 16)", wmin);
  else if (!((wide_out && (wide_in || narrow_ok_in)) || (wide_in && narrow_ok_out)))
    snprintf(why, sizeof(why), "padded channels %d (gradient) x %d (activation): neither 64-wide with the other 16 / 32 / 64-wide", a_out.C, a_in.C);
  else if (a_out.parity) snprintf(why, sizeof(why), "gradient operand in parity planes");
  else if (a_out.split != a_in.split) snprintf(why, sizeof(why), "operands differ in split");
  else if (c.kh * c.kw > V2V_MAX_TAPS) snprintf(why, sizeof(why), "%d taps (> %d)", c.kh * c.kw, V2V_MAX_TAPS);
  else why[0] = 0;
  if (why[0]) { u.wg_simt = why; return 0; }
  WgradParams& w = u.wg;
  w.N = vin.N; w.gh = u.mode == 2 ? vin.H : oh; w.gw = u.mode == 2 ? vin.W : ow;
  w.KP = kp; w.kmma = kp / 16; w.xsegs = (w.gw + kp - 1) / kp;
  w.out_padt = a_out.pad_t; w.out_padl = a_out.pad_l;
  w.swap = wide_out ? 0 : 1;                          // the narrow tensor (16 / 32 channels) always sits on the N side
  const ActDesc& aA = w.swap ? a_in : a_out;
  const ActDesc& aB = w.swap ? a_out : a_in;
  w.a_C = aA.C; w.b_C = aB.C;
  w.Mblocks = aA.C >= 128 ? 2 : 1;
  w.b_row = aB.C >= 64 ? 128 : aB.C * 2;
  w.Nblocks = aB.C >= 128 ? 2 : 1;
  w.BN = aB.C >= 128 ? 128 : aB.C;
  w.m_tiles = (aA.C + w.Mblocks * 64 - 1) / (w.Mblocks * 64); w.n_tiles = (aB.C + w.BN - 1) / w.BN;
  w.ntaps = c.kh * c.kw; w.split = a_out.split; w.Mp = aA.C; w.Np = aB.C;
  // taps: IN buffer coordinate of grid pixel (y, x).  Stride 1: (y + ky, x + kx); stride 2 (IN in parity planes):
  // plane (ky & 1, kx & 1), (y + ky / 2, x + kx / 2) -- as conv_geometry lays the forward taps out
  const bool s2 = (u.mode != 1);
  for (int ky = 0; ky < c.kh; ++ky)
    for (int kx = 0; kx < c.kw; ++kx)
      w.taps[ky * c.kw + kx] = s2 ? WgradTap{(int8_t)(((ky & 1) << 1) | (kx & 1)), (int8_t)(ky >> 1), (int8_t)(kx >> 1), 0}
                                  : WgradTap{0, (int8_t)ky, (int8_t)kx, 0};
  V2V_REQUIRE(!s2 || a_in.parity, V2V_ERR_STATE, "internal: stride-2 weight gradient needs a parity-plane operand");
  const int stage_bytes = (int)wgrad_stage_smem_bytes(w);
  w.stages = std::max(2, std::min(6, kSmemBudget / stage_bytes));
  w.chunks_total = w.N * w.gh * w.xsegs;
  const int base_units = w.ntaps * w.m_tiles * w.n_tiles;
  const int want = std::max(1, (2 * device_sm_count() + base_units - 1) / base_units);
  w.chunks_per_unit = std::max(std::min(8, w.chunks_total), (w.chunks_total + want - 1) / want);
  w.ksplit = (w.chunks_total + w.chunks_per_unit - 1) / w.chunks_per_unit;
  // parameter gradient [R][Cc][taps]: rows = channels of OUT, columns = channels of IN
  u.M = u.mode == 2 ? c.Cin : c.Cout; u.M1 = u.mode == 2 ? c.Cin : c.Cout - c.Cout2; u.Nv = u.mode == 2 ? c.Cout : c.Cin;
  u.wgrad = true;
  return 0;
}

// Device half: finalizes each unit's sub-plan, encodes the weight gradient's tensor maps and allocates its stage buffer.
static int build_backward_units(v2v_plan* P, cudaStream_t stream) {
  P->bwd_of.assign(P->gops.size(), -1);
  size_t stage_max = 0;
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (op.kind != G_CONV && op.kind != G_CONV_ACT && op.kind != G_HEAD) continue;
    if (!P->op_live[i]) continue;                 // forward-only branch: no backward
    P->bwd.emplace_back();                        // owns the sub-plan from here on, also when a step below fails
    BwdUnit& u = P->bwd.back();
    int rc = choose_backward_unit(P, (int)i, u); if (rc) return rc;
    if (!u.mode) continue;
    {
      PadScope scope(u.child->pad_min);
      rc = v2v_plan_finalize(u.child, reinterpret_cast<v2v_stream_t>(stream)); if (rc) return rc;
    }
    if (u.wgrad) {
      const ActDesc *a_out, *a_in;
      wgrad_operands(P, u, &a_out, &a_in);
      rc = make_tmap_act(&u.tmOut, *a_out, u.wg.KP, 1, std::min(a_out->C, 64)); if (rc) return rc;
      rc = make_tmap_act(&u.tmIn, *a_in, u.wg.KP, 1, std::min(a_in->C, 64)); if (rc) return rc;
      stage_max = std::max(stage_max, wgrad_stage_bytes(u.wg));
    }
    P->bwd_of[i] = (int)P->bwd.size() - 1;
  }
  if (stage_max) {
    V2V_CUDA(cudaMalloc(reinterpret_cast<void**>(&P->wg_stage), stage_max));
    for (auto& u : P->bwd) u.wg.stage = P->wg_stage;
  }
  return 0;
}

static FeatL1Params featl1_params(const v2v_plan* P, const GOp& op) {
  FeatL1Params f{};
  f.x = P->acts[P->values[op.value_in].bufs[0]]; f.y = P->acts[P->values[op.value_in2].bufs[0]];
  f.Cvalid = P->values[op.value_in].C;
  f.io = P->io_dev; f.slot = op.slot; f.index = op.l1_index;
  f.blocks = feature_l1_blocks(f.x);
  return f;
}

// Backward of one recorded forward (the plan's buffers still hold it).  Walks the graph ops in reverse.
static int run_backward(v2v_plan* P, void* const* io, void* const* gio, const std::unordered_map<const void*, void*>& pg,
                        cudaStream_t s) {
  auto grad_of = [&](const void* param) -> float* {
    if (!param) return nullptr;
    auto it = pg.find(param);
    return it == pg.end() ? nullptr : reinterpret_cast<float*>(it->second);
  };
  V2V_CUDA(cudaMemsetAsync(P->garena, 0, P->garena_bytes, s));
  auto conv_bwd = [&](const GOp& op, const float* dy, int dy_C, bool bias_grad) -> int {
    const Value& vin = P->values[op.value_in];
    BwdConv b{};
    b.N = vin.N; b.H = vin.H; b.W = vin.W; b.oh = op.geom.out_h; b.ow = op.geom.out_w;
    b.Cin = op.conv.Cin; b.Cout = op.conv.Cout; b.kh = op.conv.kh; b.kw = op.conv.kw; b.stride = op.conv.stride;
    b.pad = op.conv.pad; b.transposed = op.conv.transposed; b.pad_mode = op.conv.pad_mode;
    b.x = P->acts[vin.bufs[op.req_index]];
    b.dy = dy; b.dy_C = dy_C;
    b.w = op.conv.weight; b.w2 = op.conv.Cout2 > 0 ? op.conv.weight2 : nullptr; b.Cout1 = op.conv.Cout - op.conv.Cout2;
    const bool input_needs = vin.input_slot < 0 || (gio && gio[vin.input_slot] != nullptr);
    b.dx = input_needs ? vin.gval : nullptr;
    b.dw = grad_of(op.conv.weight); b.dw2 = b.w2 ? grad_of(op.conv.weight2) : nullptr;
    if (bias_grad) { b.dbias = grad_of(op.conv.bias); b.dbias2 = b.w2 ? grad_of(op.conv.bias2) : nullptr; }
    const int ui = P->bwd_of.empty() ? -1 : P->bwd_of[&op - P->gops.data()];
    if (ui >= 0) {
      // tensor-core path: dY -> the sub-plan's halo-padded split activation; data gradient = its conv (+ fold); weight gradient
      // = wgrad_umma over the two activation buffers
      const BwdUnit& u = P->bwd[ui];
      v2v_plan* C = u.child;
      const bool need_w = (b.dw || b.dw2);
      if (b.dx || (need_w && u.wgrad)) {
        for (const XOp& x : C->xops) {
          if (x.kind == X_CONV && !b.dx) continue;
          int rc = run_xop(C, x, s); if (rc) return rc;
        }
      }
      if (b.dx) {
        const Raw& cr = C->raws[u.child_raw];
        const int pad = u.mode == 1 ? op.conv.pad : 0;
        V2V_CUDA(launch_fold_add(reinterpret_cast<const float*>(cr.desc.base), cr.desc.C, cr.H, cr.W, b.dx, vin.N, vin.H, vin.W, op.conv.Cin, pad,
                                 (op.conv.pad_mode == V2V_PAD_REFLECT && pad > 0) ? 1 : 0, s));
      }
      if (need_w && u.wgrad) {
        V2V_CUDA(launch_wgrad_umma(u.tmOut, u.tmIn, u.wg, u.M, u.M1, u.Nv, b.dw, b.dw2, s));
        b.dw = nullptr; b.dw2 = nullptr;
      }
      b.dx = nullptr;
      if (!b.dw && !b.dw2 && !b.dbias && !b.dbias2) return 0;
    }
    V2V_CUDA(launch_conv_bwd(b, s));
    return 0;
  };
  for (int i = (int)P->gops.size() - 1; i >= 0; --i) {
    const GOp& op = P->gops[i];
    if (!P->op_live[i]) continue;
    switch (op.kind) {
      case G_FEATL1: {
        if (gio[op.slot]) {
          const FeatL1Params fp = featl1_params(P, op);
          V2V_CUDA(launch_feature_l1_bwd(fp, reinterpret_cast<const float*>(gio[op.slot]), P->values[op.value_in].gval, s));
        }
        break;
      }
      case G_MAXPOOL: {
        PoolParams pp{P->acts[P->values[op.value_in].bufs[0]], P->acts[P->values[op.value_out].bufs[0]]};
        V2V_CUDA(launch_maxpool2_bwd(pp, P->values[op.value_out].gval, P->values[op.value_in].gval, s));
        break;
      }
      case G_EXPORT: {
        const Value& v = P->values[op.value_in];
        if (gio[op.slot]) V2V_CUDA(launch_grad_import(reinterpret_cast<const float*>(gio[op.slot]), v.gval, v.N, v.C, 0, v.C, v.H, v.W, s));
        break;
      }
      case G_COMPOSITE: {
        const CompositeParams& c = op.comp;
        CompositeBwd b{};
        b.N = c.N; b.H = c.H; b.W = c.W; b.prev_C = c.prev_C; b.use_warp = c.use_warp; b.align_corners = c.align_corners;
        auto f = [&](int slot) { return slot >= 0 ? reinterpret_cast<const float*>(io[slot]) : nullptr; };
        b.raw = f(c.s_raw); b.flow = f(c.s_flow); b.weight = f(c.s_weight); b.prev = f(c.s_prev); b.mask = f(c.s_mask);
        V2V_REQUIRE(c.s_fg < 0 || c.s_raw_out >= 0, V2V_ERR_STATE, "training needs the composited raw image in its own slot");
        b.g_final = reinterpret_cast<const float*>(gio[c.s_final]);
        b.g_rawout = c.s_raw_out >= 0 ? reinterpret_cast<const float*>(gio[c.s_raw_out]) : nullptr;
        b.d_raw = P->gslot[c.s_raw]; b.d_flow = c.s_flow >= 0 ? P->gslot[c.s_flow] : nullptr;
        b.d_weight = c.s_weight >= 0 ? P->gslot[c.s_weight] : nullptr; b.d_fg = c.s_fg >= 0 ? P->gslot[c.s_fg] : nullptr;
        // img_prev's gradient through the warp goes straight into the caller's (zero-filled) gradient tensor.  The slot's
        // G_INPUT op precedes the composite in the graph, so this walk reaches it afterwards; its export of the stem's data
        // gradient adds (+=) onto the warp term and must never overwrite it.
        b.d_prev = (c.use_warp && c.s_prev >= 0) ? reinterpret_cast<float*>(gio[c.s_prev]) : nullptr;
        V2V_CUDA(launch_composite_bwd(b, s));
        break;
      }
      case G_HEAD: {
        const Value& vin = P->values[op.value_in];
        HeadBwd h{};
        h.N = vin.N; h.H = op.geom.out_h; h.W = op.geom.out_w; h.Cout = op.conv.Cout; h.dz = op.gdz; h.dz_C = round_up(op.conv.Cout, 8);
        for (int j = 0; j < op.conv.Cout; ++j) {
          const int slot = op.head[j].slot;
          h.out[j] = reinterpret_cast<const float*>(io[slot]);
          h.g_ext[j] = reinterpret_cast<const float*>(gio[slot]);
          h.g_int[j] = slot < (int)P->gslot.size() ? P->gslot[slot] : nullptr;
          h.off[j] = op.kp.head_off[j]; h.bstride[j] = op.kp.head_bstride[j];
          h.act[j] = op.head[j].act; h.scale[j] = op.head[j].scale;
        }
        V2V_CUDA(launch_head_bwd(h, s));
        int rc = conv_bwd(op, op.gdz, round_up(op.conv.Cout, 8), true); if (rc) return rc;
        break;
      }
      case G_NORM_ACT: {
        const Raw& r = P->raws[op.raw];
        const GOp& cop = P->gops[r.conv_op];
        const Value& vo = P->values[op.value_out];
        NormBwd n{};
        n.N = vo.N; n.H = vo.H; n.W = vo.W; n.C = op.cC; n.raw = r.desc; n.c_off = op.n_off;
        n.has_norm = op.norm.kind != V2V_NORM_NONE; n.batch_stats = op.norm.kind == V2V_NORM_BATCH;
        V2V_REQUIRE(n.has_norm || cop.conv.bias || true, V2V_ERR_STATE, "unreachable");
        n.scale = r.scale + op.n_off; n.shift = r.shift + op.n_off; n.stat_stride = r.C;
        n.mean = n.has_norm ? r.mean + op.n_off : nullptr; n.rstd = n.has_norm ? r.rstd + op.n_off : nullptr;
        if (!n.has_norm && !cop.conv.bias) {   // plain activation of a bias-less conv: scale / shift arrays are unset
          v2v_plan::BiasAffine ba{r.scale, r.shift, nullptr, r.N, r.C, r.C};
          V2V_CUDA(launch_bias_affine(ba.scale, ba.shift, nullptr, ba.N, ba.C, ba.stride, s));
        }
        n.act = op.act; n.slope = op.slope; n.dy = vo.gval; n.draw = r.graw; n.draw_C = r.desc.C;
        n.dadd0 = op.add[0] >= 0 ? P->values[op.add[0]].gval : nullptr;
        n.dadd1 = op.add[1] >= 0 ? P->values[op.add[1]].gval : nullptr;
        n.sums = P->gsums;
        if (n.has_norm) { n.dgamma = grad_of(op.norm.gamma); n.dbeta = grad_of(op.norm.beta); }
        else { n.dgamma = nullptr; n.dbeta = grad_of(op.n_off == 0 ? cop.conv.bias : cop.conv.bias2); }
        V2V_CUDA(launch_norm_bwd(n, s));
        break;
      }
      case G_CONV: {
        const Raw& r = P->raws[op.raw];
        int rc = conv_bwd(op, r.graw, r.desc.C, false); if (rc) return rc;    // a bias in front of a norm has zero gradient
        break;
      }
      case G_CONV_ACT: {
        const Value& vo = P->values[op.value_out];
        V2V_CUDA(launch_convact_bwd(vo.gval, P->acts[vo.bufs[0]], op.act, op.slope, op.gdz, op.conv.Cout, round_up(op.conv.Cout, 8), s));
        int rc = conv_bwd(op, op.gdz, round_up(op.conv.Cout, 8), true); if (rc) return rc;
        break;
      }
      case G_INPUT: {
        const Value& v = P->values[op.value_out];
        if (gio[op.slot]) V2V_CUDA(launch_grad_export(v.gval, reinterpret_cast<float*>(gio[op.slot]), v.N, op.C_src, op.c_off, v.C, v.H, v.W, s));
        break;
      }
      case G_RAWIN: break;
      case G_CONCAT: case G_CORR:
        set_error("backward through concat / correlation is not implemented (FlowNet2 runs under no_grad, models/flownet.py:26)");
        return V2V_ERR_UNSUPPORTED;
    }
  }
  return 0;
}

}  // namespace v2v

// =============================================================================================== C ABI
extern "C" {

int v2v_version(void) { return 100; }
const char* v2v_last_error(void) { return g_last_error.c_str(); }

int v2v_plan_create(int device, int conv_impl, v2v_plan** out) {
  V2V_REQUIRE(out, V2V_ERR_INVALID, "null out");
  v2v_plan* p = new v2v_plan();
  p->device = device;
  p->impl = conv_impl;
  *out = p;
  return 0;
}

int v2v_plan_set_precision(v2v_plan* p, int precision) {
  V2V_REQUIRE(p && !p->lowered && p->gops.empty(), V2V_ERR_STATE, "set the precision before describing the plan");
  V2V_REQUIRE(precision == V2V_PREC_BF16 || precision == V2V_PREC_BF16X3, V2V_ERR_INVALID, "unknown precision %d", precision);
  p->precise = (precision == V2V_PREC_BF16X3);
  return 0;
}

int v2v_plan_set_training(v2v_plan* p, int on) {
  V2V_REQUIRE(p && !p->finalized, V2V_ERR_STATE, "set the training flag before finalize");
  p->train = on != 0;
  return 0;
}

int v2v_plan_backward(v2v_plan* P, void* const* io_ptrs, void* const* grad_io_ptrs, int n_io, const void* const* params,
                      void* const* param_grads, int n_params, v2v_stream_t stream_) {
  V2V_REQUIRE(P && P->finalized && P->train, V2V_ERR_STATE, "plan not finalized in training mode");
  V2V_REQUIRE(n_io >= P->n_slots && io_ptrs && grad_io_ptrs, V2V_ERR_INVALID, "need %d io / gradient pointers", P->n_slots);
  DeviceGuard guard(P->device);
  std::unordered_map<const void*, void*> pg;
  for (int i = 0; i < n_params; ++i) if (params[i] && param_grads[i]) pg[params[i]] = param_grads[i];
  return run_backward(P, io_ptrs, grad_io_ptrs, pg, reinterpret_cast<cudaStream_t>(stream_));
}

int v2v_plan_destroy(v2v_plan* p) {
  if (!p) return 0;
  if (p->graph_exec) cudaGraphExecDestroy(p->graph_exec);
  if (p->graph_stream) cudaStreamDestroy(p->graph_stream);
  if (p->arena && p->arena_owned) cudaFree(p->arena);
  if (p->garena) cudaFree(p->garena);
  if (p->train_stats) cudaFree(p->train_stats);
  if (p->io_dev) cudaFree(p->io_dev);
  if (p->wg_stage) cudaFree(p->wg_stage);
  for (auto& u : p->bwd) if (u.child) v2v_plan_destroy(u.child);
  delete p;
  return 0;
}

static int new_value(v2v_plan* p, int N, int H, int W, int C) {
  Value v; v.N = N; v.H = H; v.W = W; v.C = C;
  p->values.push_back(v);
  return (int)p->values.size() - 1;
}

int v2v_g_input_ex(v2v_plan* p, int slot, int N, int C_src, int c_off, int C, int H, int W, int flags, int* value_out) {
  int rc = v2v_g_input(p, slot, N, C_src, c_off, C, H, W, value_out);
  if (rc) return rc;
  p->values[*value_out].exact_bf16 = (flags & V2V_INPUT_EXACT_BF16) != 0;
  return 0;
}

int v2v_g_input(v2v_plan* p, int slot, int N, int C_src, int c_off, int C, int H, int W, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && value_out, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(slot >= 0 && N > 0 && C > 0 && c_off >= 0 && c_off + C <= C_src && H > 0 && W > 0, V2V_ERR_INVALID,
              "bad input description");
  GOp op; op.kind = G_INPUT; op.slot = slot; op.C_src = C_src; op.c_off = c_off;
  op.value_out = new_value(p, N, H, W, C);
  p->values[op.value_out].input_slot = slot;
  p->n_slots = std::max(p->n_slots, slot + 1);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

static int check_conv(v2v_plan* p, int value_in, const v2v_conv_desc* c) {
  V2V_REQUIRE(p && !p->lowered && c, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(value_in >= 0 && value_in < (int)p->values.size(), V2V_ERR_INVALID, "bad value id %d", value_in);
  V2V_REQUIRE(c->Cin == p->values[value_in].C, V2V_ERR_INVALID, "conv Cin %d != value channels %d", c->Cin,
              p->values[value_in].C);
  V2V_REQUIRE(c->Cout > 0, V2V_ERR_INVALID, "bad Cout");
  return 0;
}

int v2v_g_conv(v2v_plan* p, int value_in, const v2v_conv_desc* c, int* raw_out) {
  int rc = check_conv(p, value_in, c); if (rc) return rc;
  V2V_REQUIRE(raw_out, V2V_ERR_INVALID, "null raw_out");
  ConvGeom g; rc = conv_geometry(*c, 0, p->values[value_in].N, p->values[value_in].H, p->values[value_in].W, true, p->sp(), &g); if (rc) return rc;
  GOp op; op.kind = G_CONV; op.value_in = value_in; op.conv = *c;
  Raw r{}; r.N = p->values[value_in].N; r.H = g.out_h; r.W = g.out_w; r.C = c->Cout; r.conv_op = (int)p->gops.size();
  p->raws.push_back(r);
  op.raw = (int)p->raws.size() - 1;
  p->gops.push_back(op);
  *raw_out = op.raw;
  return 0;
}

int v2v_g_norm_act_slice(v2v_plan* p, int raw_in, int c_off, int C, const v2v_norm_desc* norm, int act, float slope,
                         int add0, int add1, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && norm && value_out, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(raw_in >= 0 && raw_in < (int)p->raws.size(), V2V_ERR_INVALID, "bad raw id");
  const Raw& r = p->raws[raw_in];
  V2V_REQUIRE(c_off >= 0 && C > 0 && c_off + C <= r.C && (c_off % 8) == 0, V2V_ERR_INVALID,
              "bad channel slice [%d, %d) of %d", c_off, c_off + C, r.C);
  GOp op; op.kind = G_NORM_ACT; op.raw = raw_in; op.norm = *norm; op.act = act; op.slope = slope;
  op.add[0] = add0; op.add[1] = add1; op.n_off = c_off; op.cC = C;
  for (int k = 0; k < 2; ++k)
    if (op.add[k] >= 0) {
      V2V_REQUIRE(op.add[k] < (int)p->values.size(), V2V_ERR_INVALID, "bad addend id");
      const Value& a = p->values[op.add[k]];
      V2V_REQUIRE(a.N == r.N && a.H == r.H && a.W == r.W && a.C == C, V2V_ERR_INVALID,
                  "addend shape (%d,%d,%d,%d) != raw shape (%d,%d,%d,%d)", a.N, a.C, a.H, a.W, r.N, C, r.H, r.W);
    }
  op.value_out = new_value(p, r.N, r.H, r.W, C);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

int v2v_g_norm_act(v2v_plan* p, int raw_in, const v2v_norm_desc* norm, int act, float slope, int add0, int add1,
                   int* value_out) {
  V2V_REQUIRE(p && raw_in >= 0 && raw_in < (int)p->raws.size(), V2V_ERR_INVALID, "bad raw id");
  return v2v_g_norm_act_slice(p, raw_in, 0, p->raws[raw_in].C, norm, act, slope, add0, add1, value_out);
}

int v2v_g_conv_act(v2v_plan* p, int value_in, const v2v_conv_desc* c, int act, float slope, int* value_out) {
  int rc = check_conv(p, value_in, c); if (rc) return rc;
  V2V_REQUIRE(value_out, V2V_ERR_INVALID, "null value_out");
  ConvGeom g; rc = conv_geometry(*c, 0, p->values[value_in].N, p->values[value_in].H, p->values[value_in].W, true, p->sp(), &g); if (rc) return rc;
  GOp op; op.kind = G_CONV_ACT; op.value_in = value_in; op.conv = *c; op.act = act; op.slope = slope;
  op.value_out = new_value(p, p->values[value_in].N, g.out_h, g.out_w, c->Cout);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

int v2v_g_head(v2v_plan* p, int value_in, const v2v_conv_desc* c, const v2v_head_channel* ch) {
  int rc = check_conv(p, value_in, c); if (rc) return rc;
  V2V_REQUIRE(ch && c->Cout <= V2V_MAX_HEAD && !c->transposed && c->stride == 1, V2V_ERR_UNSUPPORTED,
              "head conv must be stride-1 with Cout <= %d", V2V_MAX_HEAD);
  GOp op; op.kind = G_HEAD; op.value_in = value_in; op.conv = *c;
  for (int j = 0; j < c->Cout; ++j) { op.head[j] = ch[j]; p->n_slots = std::max(p->n_slots, ch[j].slot + 1); }
  p->gops.push_back(op);
  return 0;
}

int v2v_g_concat(v2v_plan* p, const int* values, int n, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && values && n >= 1 && value_out, V2V_ERR_STATE, "plan already lowered or null");
  GOp op; op.kind = G_CONCAT;
  int C = 0;
  for (int i = 0; i < n; ++i) {
    V2V_REQUIRE(values[i] >= 0 && values[i] < (int)p->values.size(), V2V_ERR_INVALID, "bad value id %d", values[i]);
    const Value& a = p->values[values[i]], &a0 = p->values[values[0]];
    V2V_REQUIRE(a.N == a0.N && a.H == a0.H && a.W == a0.W, V2V_ERR_INVALID, "concat operands differ in extent");
    C += a.C;
    op.cat_in.push_back(values[i]);
  }
  const int N0 = p->values[values[0]].N, H0 = p->values[values[0]].H, W0 = p->values[values[0]].W;
  op.value_out = new_value(p, N0, H0, W0, C);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

int v2v_g_correlation(v2v_plan* p, int value_a, int value_b, int pad_size, int kernel_size, int max_displacement, int stride1,
                      int stride2, int act, float slope, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && value_out, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(value_a >= 0 && value_a < (int)p->values.size() && value_b >= 0 && value_b < (int)p->values.size(), V2V_ERR_INVALID,
              "bad value id");
  const Value a = p->values[value_a], b = p->values[value_b];
  V2V_REQUIRE(a.N == b.N && a.C == b.C && a.H == b.H && a.W == b.W, V2V_ERR_INVALID, "correlation operands differ in shape");
  V2V_REQUIRE(kernel_size == 1 && stride1 == 1 && pad_size == max_displacement, V2V_ERR_UNSUPPORTED,
              "correlation: only kernel 1, stride1 1, pad == max displacement (FlowNetC.py:31)");
  V2V_REQUIRE(act == V2V_ACT_NONE || act == V2V_ACT_LRELU, V2V_ERR_UNSUPPORTED, "correlation: activation must be none / LeakyReLU");
  int oc, oh, ow;
  int rc = v2v_correlation_out_shape(a.H, a.W, pad_size, kernel_size, max_displacement, stride1, stride2, &oc, &oh, &ow);
  if (rc) return rc;
  GOp op; op.kind = G_CORR; op.value_in = value_a; op.value_in2 = value_b; op.act = act; op.slope = slope;
  op.corr[0] = pad_size; op.corr[1] = kernel_size; op.corr[2] = max_displacement; op.corr[3] = stride1; op.corr[4] = stride2;
  op.value_out = new_value(p, a.N, oh, ow, oc);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

int v2v_g_maxpool2(v2v_plan* p, int value_in, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && value_out, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(value_in >= 0 && value_in < (int)p->values.size(), V2V_ERR_INVALID, "bad value id %d", value_in);
  const Value a = p->values[value_in];
  V2V_REQUIRE(a.H >= 2 && a.W >= 2, V2V_ERR_INVALID, "max-pool input %dx%d is smaller than its window", a.H, a.W);
  GOp op; op.kind = G_MAXPOOL; op.value_in = value_in;
  op.value_out = new_value(p, a.N, a.H / 2, a.W / 2, a.C);
  p->gops.push_back(op);
  *value_out = op.value_out;
  return 0;
}

int v2v_g_feature_l1(v2v_plan* p, int value_x, int value_y, int slot, int index) {
  V2V_REQUIRE(p && !p->lowered, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(value_x >= 0 && value_x < (int)p->values.size() && value_y >= 0 && value_y < (int)p->values.size() && value_x != value_y,
              V2V_ERR_INVALID, "bad value ids %d, %d", value_x, value_y);
  V2V_REQUIRE(slot >= 0 && index >= 0, V2V_ERR_INVALID, "bad output slot %d / index %d", slot, index);
  const Value a = p->values[value_x], b = p->values[value_y];
  V2V_REQUIRE(a.N == b.N && a.C == b.C && a.H == b.H && a.W == b.W, V2V_ERR_INVALID, "feature L1 operands differ in shape");
  GOp op; op.kind = G_FEATL1; op.value_in = value_x; op.value_in2 = value_y; op.slot = slot; op.l1_index = index;
  p->n_slots = std::max(p->n_slots, slot + 1);
  p->gops.push_back(op);
  return 0;
}

int v2v_g_export(v2v_plan* p, int value, int slot) {
  V2V_REQUIRE(p && !p->lowered, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(value >= 0 && value < (int)p->values.size() && slot >= 0, V2V_ERR_INVALID, "bad export");
  GOp op; op.kind = G_EXPORT; op.value_in = value; op.slot = slot;
  p->n_slots = std::max(p->n_slots, slot + 1);
  p->gops.push_back(op);
  return 0;
}

int v2v_g_composite(v2v_plan* p, int s_raw, int s_flow, int s_weight, int s_prev, int prev_C, int s_fg, int s_mask,
                    int s_final, int N, int H, int W, int use_warp, int align_corners) {
  return v2v_g_composite_ex(p, s_raw, s_flow, s_weight, s_prev, prev_C, s_fg, s_mask, s_final, -1, N, H, W, use_warp, align_corners);
}

int v2v_g_composite_ex(v2v_plan* p, int s_raw, int s_flow, int s_weight, int s_prev, int prev_C, int s_fg, int s_mask,
                       int s_final, int s_raw_out, int N, int H, int W, int use_warp, int align_corners) {
  V2V_REQUIRE(p && !p->lowered, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(s_raw >= 0 && s_final >= 0, V2V_ERR_INVALID, "composite needs raw and final slots");
  V2V_REQUIRE(!use_warp || (s_flow >= 0 && s_weight >= 0 && s_prev >= 0 && prev_C >= 3), V2V_ERR_INVALID,
              "warp needs flow, weight and prev");
  V2V_REQUIRE((s_fg >= 0) == (s_mask >= 0), V2V_ERR_INVALID, "fg and mask go together");
  GOp op; op.kind = G_COMPOSITE;
  CompositeParams& c = op.comp;
  c.s_raw = s_raw; c.s_flow = s_flow; c.s_weight = s_weight; c.s_prev = s_prev; c.s_fg = s_fg; c.s_mask = s_mask;
  c.s_raw_out = s_raw_out;
  p->n_slots = std::max(p->n_slots, s_raw_out + 1);
  c.s_final = s_final; c.prev_C = prev_C; c.N = N; c.H = H; c.W = W; c.align_corners = align_corners; c.use_warp = use_warp;
  int m = std::max({s_raw, s_flow, s_weight, s_prev, s_fg, s_mask, s_final});
  p->n_slots = std::max(p->n_slots, m + 1);
  p->gops.push_back(op);
  return 0;
}

// Host-only: lower the graph, choose every conv's tiling and lay the arena out (offsets only).  Idempotent.
static int size_arena(v2v_plan* P) {
  if (P->sized) return 0;
  int rc = lower(P); if (rc) return rc;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = round_up_sz(off + bytes, 1024); return o; };
  P->act_off.assign(P->acts.size(), 0);
  for (size_t i = 0; i < P->acts.size(); ++i) P->act_off[i] = take(P->acts[i].elems() * sizeof(bf16));
  P->raw_off.assign(P->raws.size(), v2v_plan::RawOff{});
  P->w_off.assign(P->gops.size(), 0);
  for (size_t i = 0; i < P->gops.size(); ++i) {
    GOp& op = P->gops[i];
    if (op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD) {
      fill_conv_params(P, op);
      P->w_off[i] = take((size_t)P->sp() * (op.geom.headkx ? op.geom.headkx * op.conv.Cout : op.conv.Cout) * op.Ktotal * sizeof(bf16));
      if (op.kind == G_CONV) {
        Raw& r = P->raws[op.raw];
        r.desc.N = r.N; r.desc.H = r.H; r.desc.W = r.W; r.desc.Cvalid = r.C; r.desc.C = round_up(r.C, 8);
        r.desc.f32 = P->precise;
        if (P->impl == V2V_IMPL_UMMA) { r.tiles_per_img = op.kp.grid; r.num_phases = op.kp.num_phases; }
        else { r.tiles_per_img = 1; r.num_phases = 1; }
        P->raw_off[op.raw].raw = take(r.desc.elems() * r.desc.elem_bytes());
        P->raw_off[op.raw].scale = take((size_t)r.N * r.C * sizeof(float));
        P->raw_off[op.raw].shift = take((size_t)r.N * r.C * sizeof(float));
      }
    }
  }
  P->corr_off.assign(P->gops.size(), 0);
  for (size_t i = 0; i < P->gops.size(); ++i)
    if (P->gops[i].kind == G_CORR) {
      const Value& a = P->values[P->gops[i].value_in], &o = P->values[P->gops[i].value_out];
      P->corr_off[i] = take((2 * (size_t)a.N * a.C * a.H * a.W + (size_t)o.N * o.C * o.H * o.W) * sizeof(float));
    }
  P->l1_off.assign(P->gops.size(), 0);
  for (size_t i = 0; i < P->gops.size(); ++i)
    if (P->gops[i].kind == G_FEATL1) {
      const Value& x = P->values[P->gops[i].value_in];
      P->l1_off[i] = take((size_t)feature_l1_blocks(make_act(x, x.reqs[0], P->precise)) * sizeof(double));
    }
  // all norm-statistics rows live in one contiguous region that is zeroed at the start of every run
  P->stats_begin = off;
  for (size_t i = 0; i < P->raws.size(); ++i)
    if (P->raws[i].conv_op >= 0 && !P->raws[i].no_stats) P->raw_off[i].stats = take((size_t)P->raws[i].N * 2 * P->raws[i].C * sizeof(stat_t) + 64);   // + ticket counter
  P->stats_end = off;
  P->arena_bytes = off;
  P->sized = true;
  return 0;
}

static int finalize_impl(v2v_plan* P, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  V2V_REQUIRE(P && !P->finalized, V2V_ERR_STATE, "plan null or already finalized");
  int rc = size_arena(P); if (rc) return rc;
  DeviceGuard guard(P->device);
  const std::vector<size_t>& act_off = P->act_off;
  const std::vector<v2v_plan::RawOff>& raw_off = P->raw_off;
  const std::vector<size_t>& w_off = P->w_off;
  const std::vector<size_t>& corr_off = P->corr_off;
  const size_t stats_begin = P->stats_begin, stats_end = P->stats_end;
  if (workspace) {
    // caller-owned arena (v2v_plan_workspace_bytes before this call): not freed by v2v_plan_destroy
    V2V_REQUIRE(workspace_bytes >= P->arena_bytes && (reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, V2V_ERR_INVALID,
                "workspace of %zu bytes (1024-byte aligned) needed, got %zu at %p", P->arena_bytes, workspace_bytes, workspace);
    P->arena = workspace; P->arena_owned = false;
  } else {
    V2V_CUDA(cudaMalloc(&P->arena, P->arena_bytes));
  }
  V2V_CUDA(cudaMemsetAsync(P->arena, 0, P->arena_bytes, stream));
  V2V_CUDA(cudaMalloc(reinterpret_cast<void**>(&P->io_dev), sizeof(void*) * std::max(1, P->n_slots)));
  uint8_t* base = reinterpret_cast<uint8_t*>(P->arena);
  for (size_t i = 0; i < P->acts.size(); ++i) P->acts[i].base = reinterpret_cast<bf16*>(base + act_off[i]);
  for (size_t i = 0; i < P->raws.size(); ++i) {
    Raw& r = P->raws[i];
    r.desc.base = base + raw_off[i].raw;
    r.stats = reinterpret_cast<stat_t*>(base + raw_off[i].stats);
    r.scale = reinterpret_cast<float*>(base + raw_off[i].scale);
    r.shift = reinterpret_cast<float*>(base + raw_off[i].shift);
  }

  if (P->train) {                       // saved batch statistics (the finalize launches below write them)
    size_t tot = 0;
    for (auto& r : P->raws) tot += 2 * (size_t)r.N * r.C;
    float* st = nullptr;
    V2V_CUDA(cudaMalloc(reinterpret_cast<void**>(&st), std::max<size_t>(tot, 1) * sizeof(float)));
    V2V_CUDA(cudaMemsetAsync(st, 0, std::max<size_t>(tot, 1) * sizeof(float), stream));
    P->train_stats = st;
    for (auto& r : P->raws) { r.mean = st; st += (size_t)r.N * r.C; r.rstd = st; st += (size_t)r.N * r.C; }
  }
  // ---- emit executable ops
  if (stats_end > stats_begin) {
    XOp m; m.kind = X_MEMSET; m.ms_ptr = base + stats_begin; m.ms_bytes = stats_end - stats_begin;
    P->xops.push_back(m);
  }
  for (size_t i = 0; i < P->gops.size(); ++i) {
    GOp& op = P->gops[i];
    switch (op.kind) {
      case G_INPUT: {
        const Value& v = P->values[op.value_out];
        for (size_t m = 0; m < v.bufs.size(); ++m) {
          XOp x; x.kind = X_IMPORT; x.gop = (int)i;
          x.imp.io = reinterpret_cast<const void* const*>(P->io_dev); x.imp.slot = op.slot;
          x.imp.c_off = op.c_off; x.imp.C_src = op.C_src;
          x.imp.out = P->acts[v.bufs[m]]; x.imp.pad_mode = P->act_pad_mode[v.bufs[m]];
          x.imp.skip_lo = v.exact_bf16 ? 1 : 0;
          P->xops.push_back(x);
        }
        break;
      }
      case G_CONV: case G_CONV_ACT: case G_HEAD: {
        const Value& vin = P->values[op.value_in];
        const ActDesc& ain = P->acts[vin.bufs[op.req_index]];
        op.wpacked = reinterpret_cast<bf16*>(base + w_off[i]);
        ConvKernelParams& kp = op.kp;
        kp.io = P->io_dev;
        if (op.kind == G_CONV) {
          Raw& r = P->raws[op.raw];
          kp.epi = EPI_RAW_STATS; kp.out = r.desc.base; kp.out_C = r.desc.C; kp.out_f32 = r.desc.f32;
          kp.stats = r.no_stats ? nullptr : r.stats; kp.stats_C = r.C; kp.bias = nullptr;
        } else if (op.kind == G_CONV_ACT) {
          const Value& vo = P->values[op.value_out];
          V2V_REQUIRE(vo.bufs.size() == 1 && P->act_pad_mode[vo.bufs[0]] != PAD_REFLECT, V2V_ERR_UNSUPPORTED,
                      "conv_act output needs a single zero/none-padded consumer layout");
          kp.epi = EPI_ACT_BF16; kp.out_act = P->acts[vo.bufs[0]]; kp.out_C = kp.out_act.C;
        } else {
          kp.epi = EPI_HEAD_F32;
          kp.bias2 = op.conv.Cout2 > 0 ? op.conv.bias2 : nullptr; kp.Cout1 = op.conv.Cout - op.conv.Cout2;
          for (int j = 0; j < op.conv.Cout; ++j) {
            kp.head_slot[j] = op.head[j].slot;
            kp.head_off[j] = (long long)op.head[j].channel * op.geom.out_h * op.geom.out_w;
            kp.head_bstride[j] = (long long)op.head[j].dst_C * op.geom.out_h * op.geom.out_w;
            kp.head_act[j] = op.head[j].act; kp.head_scale[j] = op.head[j].scale;
          }
        }
        if (P->impl == V2V_IMPL_UMMA) {
          rc = make_tmap_act(&op.tmA, ain, kp.PW, kp.PH, kp.kc); if (rc) return rc;
          rc = make_tmap_w(&op.tmB, op.wpacked, P->sp() * op.Ktotal, op.geom.headkx ? op.geom.headkx * op.conv.Cout : op.conv.Cout, kp.BN,
                           kp.kc); if (rc) return rc;
        }
        rc = pack_one(op, stream); if (rc) return rc;
        XOp x; x.kind = X_CONV; x.gop = (int)i;
        P->xops.push_back(x);
        if (op.kind == G_CONV && P->impl == V2V_IMPL_SIMT) {
          XOp s; s.kind = X_RAWSTATS; s.rawd = P->raws[op.raw].desc; s.stats = P->raws[op.raw].stats; s.stats_C = P->raws[op.raw].C;
          P->xops.push_back(s);
        }
        break;
      }
      case G_NORM_ACT: {
        Raw& r = P->raws[op.raw];
        const GOp& cop = P->gops[r.conv_op];
        FinalizeParams fp{};
        const bool has_norm = op.norm.kind != V2V_NORM_NONE;
        if (has_norm) {
          fp.stats = r.stats; fp.Cs = r.C; fp.C = op.cC; fp.c_off = op.n_off; fp.scale_stride = r.C;
          fp.N = r.N; fp.tiles_per_img = 1; fp.num_phases = 1;
          fp.count = (double)r.H * r.W; fp.instance = (op.norm.kind == V2V_NORM_INSTANCE);
          const int cout1 = cop.conv.Cout - cop.conv.Cout2;
          V2V_REQUIRE(op.n_off == 0 || (cop.conv.Cout2 > 0 && op.n_off == cout1), V2V_ERR_UNSUPPORTED,
                      "a raw slice must start at channel 0 or at the second weight set");
          fp.gamma = op.norm.gamma; fp.beta = op.norm.beta; fp.conv_bias = op.n_off == 0 ? cop.conv.bias : cop.conv.bias2;
          fp.momentum = op.norm.momentum; fp.eps = op.norm.eps;
        } else if (cop.conv.bias != nullptr) {
          // norm-less biased conv (FlowNet2's conv / deconv / predict_flow units): the normalise pass runs with scale 1 and
          // shift = bias, written here and after every repack
          V2V_REQUIRE(op.n_off == 0 && cop.conv.Cout2 == 0, V2V_ERR_UNSUPPORTED, "biased norm-less conv cannot be sliced");
          v2v_plan::BiasAffine ba{r.scale, r.shift, cop.conv.bias, r.N, r.C, r.C};
          P->bias_affines.push_back(ba);
          V2V_CUDA(launch_bias_affine(ba.scale, ba.shift, ba.bias, ba.N, ba.C, ba.stride, stream));
        }
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          XOp a; a.kind = X_APPLY;
          ApplyParams& ap = a.app;
          ap.raw = r.desc;
          ap.raw.base = reinterpret_cast<uint8_t*>(r.desc.base) + (size_t)op.n_off * r.desc.elem_bytes();
          ap.raw.Cvalid = op.cC;                                               // channel slice, full row stride
          ap.scale = (has_norm || cop.conv.bias != nullptr) ? r.scale + op.n_off : nullptr;
          ap.shift = r.shift + op.n_off;
          ap.scale_stride = r.C;
          ap.act = op.act; ap.slope = op.slope;
          ap.n_add = 0;
          for (int k = 0; k < 2; ++k) if (op.add[k] >= 0) ap.add[ap.n_add++] = P->acts[P->values[op.add[k]].bufs[0]];
          ap.out = P->acts[vo.bufs[m]]; ap.pad_mode = P->act_pad_mode[vo.bufs[m]];
          ap.fin = fp;
          if (has_norm) {
            // Train-mode side effects (running statistics; the scale / shift / mean / rstd arrays the backward and the
            // grid-stride fallback read) happen ONCE per (raw, slice), however many normalise passes read it (two output
            // layouts; defer_last emits the same slice twice).
            const bool first = std::find(r.running_done.begin(), r.running_done.end(), op.n_off) == r.running_done.end();
            FinalizeParams side = fp;
            side.running_mean = op.norm.running_mean; side.running_var = op.norm.running_var;
            side.num_batches_tracked = reinterpret_cast<long long*>(op.norm.num_batches_tracked);
            side.scale = r.scale; side.shift = r.shift; side.mean_out = r.mean; side.rstd_out = r.rstd;
            if (first) {
              // scale / shift come from the tail of the producing tensor-core launch (last-CTA finalisation, conv_umma.cu); the
              // SIMT cross-check implementation and a third slice of one raw use a stats_finalize launch instead
              GOp& prod = P->gops[r.conv_op];
              if (P->impl == V2V_IMPL_UMMA && prod.kp.n_fin < 2) {
                prod.kp.fin[prod.kp.n_fin++] = side;
                prod.kp.fin_counter = reinterpret_cast<unsigned int*>(reinterpret_cast<uint8_t*>(r.stats) + (size_t)r.N * 2 * r.C * sizeof(stat_t));
              } else {
                XOp f; f.kind = X_FINALIZE; f.fin = side; P->xops.push_back(f);
              }
              r.running_done.push_back(op.n_off);
            }
          }
          P->xops.push_back(a);
        }
        break;
      }
      case G_RAWIN: {
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          XOp a; a.kind = X_APPLY;
          ApplyParams& ap = a.app;
          ap.raw.base = const_cast<float*>(op.ext_raw); ap.raw.N = vo.N; ap.raw.H = vo.H; ap.raw.W = vo.W; ap.raw.C = op.ext_C;
          ap.raw.Cvalid = vo.C; ap.raw.f32 = 1;
          ap.scale = nullptr; ap.shift = nullptr; ap.scale_stride = 0; ap.act = ACT_NONE; ap.slope = 0.f; ap.n_add = 0;
          ap.out = P->acts[vo.bufs[m]]; ap.pad_mode = P->act_pad_mode[vo.bufs[m]];
          P->xops.push_back(a);
        }
        break;
      }
      case G_EXPORT: {
        XOp x; x.kind = X_EXPORT; x.exp.io = P->io_dev; x.exp.slot = op.slot; x.exp.in = P->acts[P->values[op.value_in].bufs[0]];
        P->xops.push_back(x);
        break;
      }
      case G_COMPOSITE: {
        XOp x; x.kind = X_COMPOSITE; x.comp = op.comp; x.comp.io = P->io_dev;
        P->xops.push_back(x);
        break;
      }
      case G_CONCAT: {
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          int c_off = 0;
          for (int src : op.cat_in) {
            XOp x; x.kind = X_COPY;
            x.copy.in = P->acts[P->values[src].bufs[0]];
            x.copy.out = P->acts[vo.bufs[m]];
            x.copy.c_off = c_off; x.copy.pad_mode = P->act_pad_mode[vo.bufs[m]];
            c_off += P->values[src].C;
            P->xops.push_back(x);
          }
        }
        break;
      }
      case G_MAXPOOL: {
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          V2V_REQUIRE(P->act_pad_mode[vo.bufs[m]] != PAD_REFLECT, V2V_ERR_UNSUPPORTED, "max-pool output needs a zero / no halo");
          XOp x; x.kind = X_MAXPOOL; x.gop = (int)i;
          x.pool.in = P->acts[P->values[op.value_in].bufs[0]]; x.pool.out = P->acts[vo.bufs[m]];
          P->xops.push_back(x);
        }
        break;
      }
      case G_FEATL1: {
        XOp x; x.kind = X_FEATL1; x.gop = (int)i;
        x.fl1 = featl1_params(P, op);
        x.fl1.partials = reinterpret_cast<double*>(base + P->l1_off[i]);
        P->xops.push_back(x);
        break;
      }
      case G_CORR: {
        const Value& va = P->values[op.value_in], &vb = P->values[op.value_in2], &vo = P->values[op.value_out];
        float* sa = reinterpret_cast<float*>(base + corr_off[i]);
        float* sb = sa + (size_t)va.N * va.C * va.H * va.W;
        float* so = sb + (size_t)va.N * va.C * va.H * va.W;
        XOp ea; ea.kind = X_EXPORT; ea.exp.io = P->io_dev; ea.exp.slot = 0; ea.exp.direct = sa; ea.exp.in = P->acts[va.bufs[0]];
        XOp eb = ea; eb.exp.direct = sb; eb.exp.in = P->acts[vb.bufs[0]];
        P->xops.push_back(ea); P->xops.push_back(eb);
        XOp c; c.kind = X_CORR;
        c.corr = CorrParams{sa, sb, so, va.N, va.C, va.H, va.W, op.corr[0], op.corr[1], op.corr[2], op.corr[3], op.corr[4]};
        P->xops.push_back(c);
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          XOp x; x.kind = X_IMPORT; x.gop = (int)i;
          x.imp.io = reinterpret_cast<const void* const*>(P->io_dev); x.imp.slot = 0; x.imp.direct = so;
          x.imp.c_off = 0; x.imp.C_src = vo.C; x.imp.act = op.act; x.imp.slope = op.slope;
          x.imp.out = P->acts[vo.bufs[m]]; x.imp.pad_mode = P->act_pad_mode[vo.bufs[m]];
          P->xops.push_back(x);
        }
        break;
      }
    }
  }
  if (P->train) {
    rc = alloc_training(P, stream); if (rc) return rc;
    rc = build_backward_units(P, stream); if (rc) return rc;
  }
  V2V_CUDA(cudaStreamSynchronize(stream));
  P->finalized = true;
  return 0;
}

int v2v_plan_finalize(v2v_plan* P, v2v_stream_t stream_) {
  return finalize_impl(P, nullptr, 0, reinterpret_cast<cudaStream_t>(stream_));
}

int v2v_plan_finalize_ws(v2v_plan* P, void* workspace, int64_t workspace_bytes, v2v_stream_t stream_) {
  V2V_REQUIRE(workspace && workspace_bytes > 0, V2V_ERR_INVALID, "null workspace");
  return finalize_impl(P, workspace, (size_t)workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

int v2v_plan_repack(v2v_plan* P, v2v_stream_t stream_) {
  V2V_REQUIRE(P && P->finalized, V2V_ERR_STATE, "plan not finalized");
  DeviceGuard guard(P->device);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  for (auto& op : P->gops)
    if (op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD) { int rc = pack_one(op, stream); if (rc) return rc; }
  for (const auto& ba : P->bias_affines) V2V_CUDA(launch_bias_affine(ba.scale, ba.shift, ba.bias, ba.N, ba.C, ba.stride, stream));
  for (auto& u : P->bwd) if (u.child) { int rc = v2v_plan_repack(u.child, stream_); if (rc) return rc; }
  return 0;
}

int v2v_plan_run(v2v_plan* P, void* const* io_ptrs, int n_io, int use_graph, v2v_stream_t stream_) {
  V2V_REQUIRE(P && P->finalized, V2V_ERR_STATE, "plan not finalized");
  V2V_REQUIRE(n_io >= P->n_slots && io_ptrs, V2V_ERR_INVALID, "need %d io pointers, got %d", P->n_slots, n_io);
  DeviceGuard guard(P->device);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  V2V_CUDA(cudaMemcpyAsync(P->io_dev, io_ptrs, sizeof(void*) * P->n_slots, cudaMemcpyHostToDevice, stream));
  if (use_graph & 2) {        // recomputation before a backward: same results, no running-statistics side effect
    for (const XOp& x : P->xops) {
      if (x.kind == X_FINALIZE) {
        XOp y = x; y.fin.running_mean = nullptr; y.fin.running_var = nullptr; y.fin.num_batches_tracked = nullptr;
        int rc = run_xop(P, y, stream); if (rc) return rc;
      } else if (x.kind == X_CONV && P->impl == V2V_IMPL_UMMA && P->gops[x.gop].kp.n_fin > 0) {
        const GOp& op = P->gops[x.gop];
        ConvKernelParams kp = op.kp;
        for (int q = 0; q < kp.n_fin; ++q) { kp.fin[q].running_mean = nullptr; kp.fin[q].running_var = nullptr; kp.fin[q].num_batches_tracked = nullptr; }
        V2V_CUDA(launch_conv_umma(op.tmA, op.tmB, kp, stream));
      } else { int rc = run_xop(P, x, stream); if (rc) return rc; }
    }
    return 0;
  }
  if (!use_graph) {
    for (const XOp& x : P->xops) { int rc = run_xop(P, x, stream); if (rc) return rc; }
    return 0;
  }
  if (!P->graph_exec) {
    // capture on a plan-owned stream: the caller's stream may be the legacy default stream (PyTorch's
    // default), which cannot be captured; the instantiated graph is then launched on the caller's stream
    cudaGraph_t graph;
    if (!P->graph_stream) V2V_CUDA(cudaStreamCreateWithFlags(&P->graph_stream, cudaStreamNonBlocking));
    V2V_CUDA(cudaStreamBeginCapture(P->graph_stream, cudaStreamCaptureModeThreadLocal));
    int rc = 0;
    for (const XOp& x : P->xops) { rc = run_xop(P, x, P->graph_stream); if (rc) break; }
    cudaError_t e = cudaStreamEndCapture(P->graph_stream, &graph);
    if (rc) return rc;
    V2V_CUDA(e);
    V2V_CUDA(cudaGraphInstantiate(&P->graph_exec, graph, 0));
    V2V_CUDA(cudaGraphDestroy(graph));
  }
  V2V_CUDA(cudaGraphLaunch(P->graph_exec, stream));
  return 0;
}

int v2v_plan_profile(v2v_plan* P, void* const* io_ptrs, int n_io, v2v_stream_t stream_, int max_ops, int* kinds,
                     float* ms, double* macs, int* n_ops) {
  V2V_REQUIRE(P && P->finalized, V2V_ERR_STATE, "plan not finalized");
  V2V_REQUIRE(n_io >= P->n_slots && io_ptrs && kinds && ms && macs && n_ops, V2V_ERR_INVALID, "bad profile arguments");
  DeviceGuard guard(P->device);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  V2V_CUDA(cudaMemcpyAsync(P->io_dev, io_ptrs, sizeof(void*) * P->n_slots, cudaMemcpyHostToDevice, stream));
  const int n = std::min<int>(max_ops, (int)P->xops.size());
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) V2V_CUDA(cudaEventCreate(&e));
  V2V_CUDA(cudaEventRecord(ev[0], stream));
  for (int i = 0; i < (int)P->xops.size(); ++i) {
    int rc = run_xop(P, P->xops[i], stream);
    if (rc) return rc;
    if (i < n) V2V_CUDA(cudaEventRecord(ev[i + 1], stream));
  }
  V2V_CUDA(cudaStreamSynchronize(stream));
  for (int i = 0; i < n; ++i) {
    V2V_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    kinds[i] = (int)P->xops[i].kind;
    macs[i] = (P->xops[i].kind == X_CONV) ? P->gops[P->xops[i].gop].macs : 0.0;
  }
  for (auto& e : ev) cudaEventDestroy(e);
  *n_ops = n;
  return 0;
}

int v2v_plan_num_kernels(const v2v_plan* P) { return P ? (int)P->xops.size() : 0; }
double v2v_plan_conv_macs(const v2v_plan* P) {
  if (!P) return 0.0;
  if (!P->lowered) lower(const_cast<v2v_plan*>(P));
  return P->conv_macs;
}
int64_t v2v_plan_workspace_bytes(const v2v_plan* P_) {
  // valid before v2v_plan_finalize(_ws): lowers the graph and lays the arena out on the host (no GPU work)
  v2v_plan* P = const_cast<v2v_plan*>(P_);
  if (!P) return 0;
  if (!P->sized && size_arena(P)) return -1;
  return (int64_t)P->arena_bytes;
}

}  // extern "C"

// One conv record of v2v_plan_describe: the conv, its geometry and the kernel configuration fill_conv_params chooses (host-only
// logic; no device state needed).
static void describe_conv(v2v_plan* P, const GOp& op, std::string& s) {
  char t[512];
  const ConvGeom& g = op.geom;
  GOp tmp = op;                                  // kernel configuration (host-only logic; no device state needed)
  fill_conv_params(const_cast<v2v_plan*>(P), tmp);
  const ConvKernelParams& kp = tmp.kp;
  // EG: epilogue groups per tile, always 1 (one 256-thread epilogue stores every tile; async_epi: which threads run it)
  snprintf(t, sizeof(t),
           "{\"kind\":%d,\"Cin\":%d,\"Cout\":%d,\"k\":[%d,%d],\"stride\":%d,\"transposed\":%d,\"in\":%d,\"TH\":%d,\"TW\":%d,"
           "\"R\":%d,\"groups\":%d,\"phases\":%d,\"grid\":[%d,%d],\"out\":[%d,%d],"
           "\"BN\":%d,\"kc\":%d,\"MG\":%d,\"CG\":%d,\"SG\":%d,\"resident\":%d,\"EG\":1,\"units\":%d,\"split\":%d,\"ring2\":%d,\"TB\":%d,\"SBr\":%d,"
           "\"p2d\":%d,\"a_exact\":%d,\"headkx\":%d,\"grad\":%d,",
           (int)op.kind, op.conv.Cin, op.conv.Cout, op.conv.kh, op.conv.kw, op.conv.stride, op.conv.transposed,
           op.value_in, g.TH, g.TW, g.R, g.n_groups, g.n_phases, g.grid_h, g.grid_w, g.out_h, g.out_w,
           kp.BN, kp.kc, kp.MG, kp.CG, kp.SG, kp.b_resident, kp.total_units, kp.split, kp.ring2, kp.TB, kp.SBr,
           g.patch2d_kc > 0 ? 1 : 0, kp.a_exact, kp.headkx, (int)P->op_live[&op - P->gops.data()]);
  s += t;
  // the derived launch parameters the kernel reads (ctas: persistent CTAs launched; smem: dynamic shared memory)
  snprintf(t, sizeof(t),
           "\"tiles_x\":%d,\"tiles_y\":%d,\"tile_dx\":%d,\"Cp\":%d,\"cblocks\":%d,\"row_bytes\":%d,\"kmma\":%d,\"kmma_last\":%d,\"BNt\":%d,\"layout_type\":%d,"
           "\"sbo_bytes\":%d,\"sbo_a_bytes\":%d,\"RW\":%d,\"PW\":%d,\"PH\":%d,\"a_half_bytes\":%d,\"a_slot_bytes\":%d,"
           "\"b_half_bytes\":%d,\"b_slot_bytes\":%d,\"SB\":%d,\"n_tiles\":%d,\"m_total\":%d,\"ctas\":%d,\"Khalf\":%d,\"smem\":%zu,\"async_epi\":%d}",
           kp.tiles_x, kp.tiles_y, kp.tile_dx, kp.Cp, kp.cblocks, kp.row_bytes, kp.kmma, kp.kmma_last, kp.BNt, kp.layout_type, kp.sbo_bytes,
           kp.sbo_a_bytes, kp.RW, kp.PW, kp.PH, kp.a_half_bytes, kp.a_slot_bytes, kp.b_half_bytes, kp.b_slot_bytes, kp.SB,
           kp.n_tiles, kp.m_total, kp.grid, kp.Khalf, conv_umma_smem_bytes(kp), conv_umma_async_epilogue(kp));
  s += t;
}

// One backward record: the data-gradient mode (0: SIMT, "simt" says why), the sub-plan's conv as a conv record, and the
// weight-gradient launch (null: SIMT, "wgrad_simt" says why).
static void describe_backward_unit(const BwdUnit& u, std::string& s) {
  char t[640];
  snprintf(t, sizeof(t), "{\"gop\":%d,\"mode\":%d,\"simt\":\"%s\",\"wgrad_simt\":\"%s\",\"conv\":", u.gop, u.mode, u.simt.c_str(),
           u.wg_simt.c_str());
  s += t;
  if (u.mode) {
    PadScope scope(u.child->pad_min);
    describe_conv(u.child, u.child->gops[1], s);
  } else {
    s += "null";
  }
  s += ",\"wgrad\":";
  if (u.wgrad) {
    const WgradParams& w = u.wg;
    snprintf(t, sizeof(t),
             "{\"swap\":%d,\"KP\":%d,\"BN\":%d,\"Mblocks\":%d,\"Nblocks\":%d,\"b_row\":%d,\"m_tiles\":%d,\"n_tiles\":%d,\"ntaps\":%d,"
             "\"ksplit\":%d,\"chunks_per_unit\":%d,\"chunks_total\":%d,\"xsegs\":%d,\"gh\":%d,\"gw\":%d,\"stages\":%d,\"split\":%d,"
             "\"Mp\":%d,\"Np\":%d}}",
             w.swap, w.KP, w.BN, w.Mblocks, w.Nblocks, w.b_row, w.m_tiles, w.n_tiles, w.ntaps, w.ksplit, w.chunks_per_unit,
             w.chunks_total, w.xsegs, w.gh, w.gw, w.stages, w.split, w.Mp, w.Np);
    s += t;
  } else {
    s += "null}";
  }
}

extern "C" {

int64_t v2v_plan_describe(const v2v_plan* P_, char* buf, int64_t cap) {
  v2v_plan* P = const_cast<v2v_plan*>(P_);
  if (!P) return 0;
  if (!P->lowered && lower(P)) return -1;
  std::string s = "{\"values\":[";
  char t[512];
  for (size_t i = 0; i < P->values.size(); ++i) {
    const Value& v = P->values[i];
    snprintf(t, sizeof(t), "%s{\"id\":%zu,\"N\":%d,\"C\":%d,\"H\":%d,\"W\":%d,\"layouts\":[", i ? "," : "", i, v.N, v.C, v.H, v.W);
    s += t;
    for (size_t m = 0; m < v.reqs.size(); ++m) {
      const Req& r = v.reqs[m];
      snprintf(t, sizeof(t), "%s{\"mode\":%d,\"pads\":[%d,%d,%d,%d],\"parity\":%d}", m ? "," : "", r.mode, r.pads[0], r.pads[1],
               r.pads[2], r.pads[3], r.parity);
      s += t;
    }
    s += "]}";
  }
  s += "],\"convs\":[";
  bool first = true;
  for (const GOp& op : P->gops) {
    if (!(op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD)) continue;
    if (!first) s += ",";
    describe_conv(P, op, s);
    first = false;
  }
  // training plans: the backward of every live conv, as finalize built it, or as it would build it (same host-only choice)
  if (P->train) {
    s += "],\"backward\":[";
    first = true;
    if (P->finalized) {
      for (const BwdUnit& u : P->bwd) { if (!first) s += ","; describe_backward_unit(u, s); first = false; }
    } else {
      for (size_t i = 0; i < P->gops.size(); ++i) {
        const GOp& op = P->gops[i];
        if (!(op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD) || !P->op_live[i]) continue;
        BwdUnit u;
        const int rc = choose_backward_unit(P, (int)i, u);
        if (!rc) { if (!first) s += ","; describe_backward_unit(u, s); first = false; }
        if (u.child) v2v_plan_destroy(u.child);
        if (rc) return -1;
      }
    }
  }
  // ops the backward visits (0 for the forward-only branch of a feature L1 target) and values without a gradient buffer
  int bwd_ops = 0, detached = 0;
  for (char l : P->op_live) bwd_ops += l;
  for (const Value& v : P->values) detached += v.detached;
  snprintf(t, sizeof(t), "],\"conv_macs\":%.0f,\"n_slots\":%d,\"ops\":%zu,\"backward_ops\":%d,\"detached_values\":%d}", P->conv_macs,
           P->n_slots, P->gops.size(), bwd_ops, detached);
  s += t;
  if (buf && cap > 0) {
    size_t n = std::min((size_t)cap - 1, s.size());
    memcpy(buf, s.data(), n);
    buf[n] = 0;
  }
  return (int64_t)s.size() + 1;
}

int v2v_conv_tap_table(const v2v_conv_desc* conv, int H, int W, int allow_reuse, int* n_groups, int* R, int* plane,
                       int* dy, int* dx, int* tap0, int* n_phases, int* phase_begin, int* oy_add, int* ox_add,
                       int* pads, int* parity, int* grid_hw, int* out_hw, int* mul) {
  V2V_REQUIRE(conv, V2V_ERR_INVALID, "null conv");
  ConvGeom g;
  int rc = conv_geometry(*conv, 0, 1, H, W, allow_reuse != 0, 1, &g);
  if (rc) return rc;
  *n_groups = g.n_groups; R[0] = g.R; R[1] = g.RW; *n_phases = g.n_phases; *parity = g.parity; *mul = g.mul;
  for (int i = 0; i < g.n_groups; ++i) { plane[i] = g.groups[i].plane; dy[i] = g.groups[i].dy; dx[i] = g.groups[i].dx; tap0[i] = g.groups[i].tap0; }
  for (int i = 0; i < g.n_phases; ++i) { phase_begin[i] = g.phases[i].group_begin; oy_add[i] = g.phases[i].oy_add; ox_add[i] = g.phases[i].ox_add; }
  phase_begin[g.n_phases] = g.n_groups;
  memcpy(pads, g.pads, sizeof(g.pads));
  grid_hw[0] = g.grid_h; grid_hw[1] = g.grid_w; out_hw[0] = g.out_h; out_hw[1] = g.out_w;
  return 0;
}

}  // extern "C"
