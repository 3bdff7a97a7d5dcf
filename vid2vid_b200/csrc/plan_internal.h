// Internal declarations of the plan runtime: the graph, its lowering and the plan object, shared by plan.cu (graph
// builders, lowering, arena layout, finalize, run / profile / repack), conv_lower.cu (conv geometry, tiling, tensor maps
// and weight packing) and plan_backward.cu (gradient buffers and the tensor-core backward).
#pragma once
#include <iomanip>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/v2v_b200.h"
#include "v2v_internal.h"
#include "backward.h"

namespace v2v {

void set_error(const char* fmt, ...);

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

static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
static inline size_t round_up_sz(size_t a, size_t b) { return (a + b - 1) / b * b; }
// padded channel count of an activation buffer: one K block of min(C,64) channels per shared-memory row (a plan's buffers
// may be padded further: Value::Cp)
static inline int pad_channels(int c) { return c <= 16 ? 16 : (c <= 32 ? 32 : round_up(c, 64)); }

// The JSON writer of v2v_plan_describe: appends to s, placing every separator itself.  obj() / arr() open a container (as a
// value: after key(), inside an array or at the top), end() closes the innermost one.  Integers print in full, a double as
// %.0f, a string escaped.
class Json {
 public:
  explicit Json(std::string& s) : s_(s) {}
  Json& obj() { value(); s_ += '{'; open_.push_back('}'); first_ = true; return *this; }
  Json& arr() { value(); s_ += '['; open_.push_back(']'); first_ = true; return *this; }
  Json& end() { s_ += open_.back(); open_.pop_back(); first_ = false; return *this; }
  Json& key(const char* k) { value(); str(k); s_ += ':'; keyed_ = true; return *this; }
  Json& val(int v) { value(); s_ += std::to_string(v); return *this; }
  Json& val(long long v) { value(); s_ += std::to_string(v); return *this; }
  Json& val(size_t v) { value(); s_ += std::to_string(v); return *this; }
  Json& val(double v) { value(); std::ostringstream o; o << std::fixed << std::setprecision(0) << v; s_ += o.str(); return *this; }
  Json& val(const char* v) { value(); str(v); return *this; }
  Json& val(const std::string& v) { return val(v.c_str()); }
  Json& null() { value(); s_ += "null"; return *this; }
  Json& val(std::initializer_list<int> v) { arr(); for (int x : v) val(x); return end(); }
  template <class T> Json& kv(const char* k, const T& v) { return key(k).val(v); }
  Json& kv(const char* k, std::initializer_list<int> v) { return key(k).val(v); }

 private:
  void value() {               // the separator in front of a key, or of a value that follows no key
    if (!keyed_ && !first_) s_ += ',';
    keyed_ = false; first_ = false;
  }
  void str(const char* v) {
    s_ += '"';
    for (; *v; ++v) { if (*v == '"' || *v == '\\') s_ += '\\'; s_ += *v; }
    s_ += '"';
  }
  std::string& s_;
  std::vector<char> open_;
  bool first_ = true, keyed_ = false;
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

// ------------------------------------------------------------------------------ graph description
struct Req { int mode, pads[4], parity; };

struct Value {
  int N, H, W, C;
  int Cp;                    // padded channels of every buffer of the value (ActDesc::C) and of a conv reading it (kp.Cp):
                             // pad_channels(C), at least the plan's pad_min
  std::vector<Req> reqs;
  std::vector<int> bufs;     // index into Plan::acts, one per req
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
  ConvKernelParams kp{};     // fill_conv_params: every parameter without an arena address (the launch's XOp::kp adds those)
};

enum XKind { X_IMPORT, X_CONV, X_RAWSTATS, X_FINALIZE, X_APPLY, X_EXPORT, X_COMPOSITE, X_MEMSET, X_COPY, X_CORR, X_MAXPOOL, X_FEATL1 };
// One launch of the forward list (emit_forward).  Besides its parameters it keeps what v2v_plan_describe reports and the
// parameters do not say.
struct XOp {
  XKind kind;
  int gop = -1;              // the graph op the launch belongs to (-1: the statistics memset)
  int buf = -1;              // import, copy, apply: the activation buffer written; export: the buffer read
  int in_buf = -1;           // copy: the buffer read
  bool repeat = false;       // apply: an earlier normalise pass read the same raw slice
  int fin_gop[2] = {-1, -1};   // conv: the normalising op each tail finalisation kp.fin[q] serves
  ConvKernelParams kp{};
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

using namespace v2v;     // the plan object is the C ABI's opaque v2v_plan, outside the namespace

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
  int pad_min = 0;              // minimum padded channel count of every buffer (a backward sub-plan's dY: see choose_backward_unit);
                                // set before the first value (new_value reads it into Value::Cp)

  int device = 0;
  int impl = V2V_IMPL_UMMA;
  int precise = 0;            // V2V_PREC_BF16X3: split activations / weights, fp32 raw tensors, 3 MMAs per K block
  int sp() const { return precise ? 2 : 1; }
  bool lowered = false, finalized = false;
  bool train = false;          // keep what the backward needs (batch statistics) and allocate gradient buffers
  // Per-sample statistics (v2v_plan_set_sample_stats): every norm layer normalises image n with the statistics of image n.
  // Such a plan also configures each conv as the plan of ONE image would (tiling_n): the configuration fixes the order in
  // which a pixel's products are accumulated, so each image's outputs equal its one-image plan's bit for bit, and the N
  // images only add work units.
  bool sample_stats = false;
  int tiling_n(int N) const { return sample_stats ? 1 : N; }
  int flags_slot = -1;         // v2v_plan_set_image_flags: IO slot of the per-image flags read by the finalisations and composites
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

namespace v2v {

// conv_lower.cu
extern const int kSmemBudget;      // dynamic shared memory of a kernel's operand slots + resident weights
int conv_geometry(const v2v_conv_desc& c, int Cp, int head, int N, int H, int W, bool allow_reuse, int sp, ConvGeom* g);
void fill_conv_params(v2v_plan* P, GOp& op);
int make_tmap_act(CUtensorMap* tm, const ActDesc& a, int box_w, int box_h, int kc);
int make_tmap_w(CUtensorMap* tm, bf16* w, int Ktotal, int Cout, int BN, int kc);
PackParams pack_params(const GOp& op);
int pack_one(const GOp& op, cudaStream_t stream);
void describe_conv(const v2v_plan* P, const GOp& op, Json& j);
void describe_pack(const v2v_plan* P, size_t i, Json& j);

// plan.cu
int new_value(v2v_plan* p, int N, int H, int W, int C);
int size_arena(v2v_plan* P);
int run_xop(v2v_plan* P, const XOp& x, cudaStream_t s);
FeatL1Params featl1_params(const v2v_plan* P, const GOp& op);

// plan_backward.cu
int alloc_training(v2v_plan* P, cudaStream_t stream);
// the host half of the backward unit of every live conv, in graph order (build_backward_units finalizes them, v2v_plan_describe
// reports them); units own their sub-plans, also after an error
int choose_backward_units(v2v_plan* P, std::vector<BwdUnit>& units);
int build_backward_units(v2v_plan* P, cudaStream_t stream);
int run_backward(v2v_plan* P, void* const* io, void* const* gio, const std::unordered_map<const void*, void*>& pg,
                 cudaStream_t s);
void describe_backward_unit(const BwdUnit& u, Json& j);
void describe_epilogue_backward(const v2v_plan* P, Json& j);
void describe_backward_layout(const v2v_plan* P, const std::vector<BwdUnit>& units, Json& j);

}  // namespace v2v
