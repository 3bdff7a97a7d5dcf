// Training plans: the gradient buffers and the backward pass.  Each live conv gets a tensor-core backward unit where it can
// (precise plans): a sub-plan whose forward conv computes the data gradient, and a wgrad_umma_kernel launch for the weight
// gradient; the fp32 SIMT kernels (backward.cu) do the rest.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "plan_internal.h"

namespace v2v {

// ------------------------------------------------------------------------------ training: gradient buffers
int alloc_training(v2v_plan* P, cudaStream_t stream) {
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
// caller.
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
  } else if (!c.transposed && c.stride == 2 && c.pad_mode == V2V_PAD_REFLECT && c.pad > 0) {
    // mode 3 crops the transposed conv's output to the interior: the gradient of the reflected halo rows and columns would be
    // dropped instead of mirrored back (the SIMT data gradient folds it)
    u.simt = "stride-2 conv behind a reflect halo: the cropped transposed conv cannot fold the mirrored halo";
    return 0;
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
  const int pad_min = (pad_channels(c.Cout) < 64 && vin.Cp < 64) ? 64 : 0;
  v2v_plan* C = nullptr;
  int rc = v2v_plan_create(P->device, P->impl, &C); if (rc) return rc;
  C->precise = P->precise; C->pad_min = pad_min;
  u.child = C;
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

int choose_backward_units(v2v_plan* P, std::vector<BwdUnit>& units) {
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (op.kind != G_CONV && op.kind != G_CONV_ACT && op.kind != G_HEAD) continue;
    if (!P->op_live[i]) continue;                 // forward-only branch: no backward
    units.emplace_back();                         // owns the sub-plan from here on, also when the choice fails
    int rc = choose_backward_unit(P, (int)i, units.back()); if (rc) return rc;
  }
  return 0;
}

// Device half: finalizes each unit's sub-plan, encodes the weight gradient's tensor maps and allocates its stage buffer.
int build_backward_units(v2v_plan* P, cudaStream_t stream) {
  int rc = choose_backward_units(P, P->bwd); if (rc) return rc;
  P->bwd_of.assign(P->gops.size(), -1);
  size_t stage_max = 0;
  for (size_t k = 0; k < P->bwd.size(); ++k) {
    BwdUnit& u = P->bwd[k];
    if (!u.mode) continue;
    rc = v2v_plan_finalize(u.child, reinterpret_cast<v2v_stream_t>(stream)); if (rc) return rc;
    if (u.wgrad) {
      const ActDesc *a_out, *a_in;
      wgrad_operands(P, u, &a_out, &a_in);
      rc = make_tmap_act(&u.tmOut, *a_out, u.wg.KP, 1, std::min(a_out->C, 64)); if (rc) return rc;
      rc = make_tmap_act(&u.tmIn, *a_in, u.wg.KP, 1, std::min(a_in->C, 64)); if (rc) return rc;
      stage_max = std::max(stage_max, wgrad_stage_bytes(u.wg));
    }
    P->bwd_of[u.gop] = (int)k;
  }
  if (stage_max) {
    V2V_CUDA(cudaMalloc(reinterpret_cast<void**>(&P->wg_stage), stage_max));
    for (auto& u : P->bwd) u.wg.stage = P->wg_stage;
  }
  return 0;
}

// ------------------------------------------------------------------------------ training: launch parameters of the backward
// What one backward is asked for: io and gio, the caller's tensors and gradient tensors per IO slot (a null gradient tensor
// asks for none), and pg, each parameter's gradient buffer (a parameter it lacks asks for none).  kEveryGradient asks for
// every gradient, as v2v_plan_describe reports the launches: the gradient pointers it yields stand for requested buffers and
// are never launched.
static float g_requested;
struct BwdRequest {
  void* const* io;
  void* const* gio;
  const std::unordered_map<const void*, void*>* pg;     // null: every gradient
  float* grad_io(int slot) const { return pg ? reinterpret_cast<float*>(gio[slot]) : &g_requested; }
  float* grad(const void* param) const {
    if (!param || !pg) return param ? &g_requested : nullptr;
    auto it = pg->find(param);
    return it == pg->end() ? nullptr : reinterpret_cast<float*>(it->second);
  }
};
static const BwdRequest kEveryGradient{nullptr, nullptr, nullptr};

// The fp32 SIMT backward of a conv op: data, weight and bias gradients (a bias in front of a norm, G_CONV, has zero gradient).
// A tensor-core unit takes the data and weight gradients over.
static BwdConv conv_bwd_params(const v2v_plan* P, const GOp& op, const BwdRequest& q) {
  const Value& vin = P->values[op.value_in];
  const v2v_conv_desc& c = op.conv;
  BwdConv b{};
  b.N = vin.N; b.H = vin.H; b.W = vin.W; b.oh = op.geom.out_h; b.ow = op.geom.out_w;
  b.Cin = c.Cin; b.Cout = c.Cout; b.kh = c.kh; b.kw = c.kw; b.stride = c.stride;
  b.pad = c.pad; b.transposed = c.transposed; b.pad_mode = c.pad_mode;
  b.x = P->acts[vin.bufs[op.req_index]];
  if (op.kind == G_CONV) { b.dy = P->raws[op.raw].graw; b.dy_C = P->raws[op.raw].desc.C; }
  else { b.dy = op.gdz; b.dy_C = round_up(c.Cout, 8); }
  b.w = c.weight; b.w2 = c.Cout2 > 0 ? c.weight2 : nullptr; b.Cout1 = c.Cout - c.Cout2;
  b.dx = (vin.input_slot < 0 || q.grad_io(vin.input_slot)) ? vin.gval : nullptr;
  b.dw = q.grad(c.weight); b.dw2 = b.w2 ? q.grad(c.weight2) : nullptr;
  if (op.kind != G_CONV) { b.dbias = q.grad(c.bias); b.dbias2 = b.w2 ? q.grad(c.bias2) : nullptr; }
  return b;
}

// The head backward: dz of each head channel from the gradients of its IO slot (the caller's and the composite backward's)
static HeadBwd head_bwd_params(const v2v_plan* P, const GOp& op, const BwdRequest& q) {
  HeadBwd h{};
  h.N = P->values[op.value_in].N; h.H = op.geom.out_h; h.W = op.geom.out_w; h.Cout = op.conv.Cout;
  h.dz = op.gdz; h.dz_C = round_up(op.conv.Cout, 8);
  for (int j = 0; j < op.conv.Cout; ++j) {
    const int slot = op.head[j].slot;
    h.out[j] = q.io ? reinterpret_cast<const float*>(q.io[slot]) : nullptr;
    h.g_ext[j] = q.grad_io(slot);
    h.g_int[j] = slot < (int)P->gslot.size() ? P->gslot[slot] : nullptr;
    h.off[j] = op.kp.head_off[j]; h.bstride[j] = op.kp.head_bstride[j];
    h.act[j] = op.head[j].act; h.scale[j] = op.head[j].scale;
  }
  return h;
}

// The norm backward of a G_NORM_ACT op: its slice of the raw tensor's saved statistics (set at finalize) and gradients
static NormBwd norm_bwd_params(const v2v_plan* P, const GOp& op, const BwdRequest& q) {
  const Raw& r = P->raws[op.raw];
  const Value& vo = P->values[op.value_out];
  auto slice = [&](const float* rows) { return rows ? rows + op.n_off : nullptr; };
  NormBwd n{};
  n.N = vo.N; n.H = vo.H; n.W = vo.W; n.C = op.cC; n.raw = r.desc; n.c_off = op.n_off;
  n.has_norm = op.norm.kind != V2V_NORM_NONE; n.batch_stats = op.norm.kind == V2V_NORM_BATCH;
  n.scale = slice(r.scale); n.shift = slice(r.shift); n.stat_stride = r.C;
  n.mean = n.has_norm ? slice(r.mean) : nullptr; n.rstd = n.has_norm ? slice(r.rstd) : nullptr;
  n.act = op.act; n.slope = op.slope; n.dy = vo.gval; n.draw = r.graw; n.draw_C = r.desc.C;
  n.dadd0 = op.add[0] >= 0 ? P->values[op.add[0]].gval : nullptr;
  n.dadd1 = op.add[1] >= 0 ? P->values[op.add[1]].gval : nullptr;
  n.sums = P->gsums;
  const v2v_conv_desc& c = P->gops[r.conv_op].conv;
  if (n.has_norm) { n.dgamma = q.grad(op.norm.gamma); n.dbeta = q.grad(op.norm.beta); }
  else { n.dgamma = nullptr; n.dbeta = q.grad(op.n_off == 0 ? c.bias : c.bias2); }
  return n;
}

// The fold of a tensor-core unit's data gradient (its sub-plan's raw output) into dx
static FoldParams fold_params(const v2v_plan* P, const BwdUnit& u, float* dx) {
  const GOp& op = P->gops[u.gop];
  const Value& vin = P->values[op.value_in];
  const Raw& cr = u.child->raws[u.child_raw];
  const int pad = u.mode == 1 ? op.conv.pad : 0;
  return FoldParams{reinterpret_cast<const float*>(cr.desc.base), cr.desc.C, cr.H, cr.W, dx, vin.N, vin.H, vin.W, op.conv.Cin,
                    pad, (op.conv.pad_mode == V2V_PAD_REFLECT && pad > 0) ? 1 : 0};
}

// The gradient import of a G_EXPORT (the caller's gradient of the output onto the value's) or the gradient export of a
// G_INPUT (the value's gradient onto the caller's gradient of the input); g null: not requested
static GradLayout grad_layout_params(const v2v_plan* P, const GOp& op, const BwdRequest& q) {
  if (op.kind == G_EXPORT) {
    const Value& v = P->values[op.value_in];
    return GradLayout{q.grad_io(op.slot), v.gval, v.N, v.C, 0, v.C, v.H, v.W};
  }
  const Value& v = P->values[op.value_out];
  return GradLayout{q.grad_io(op.slot), v.gval, v.N, op.C_src, op.c_off, v.C, v.H, v.W};
}

// Backward of one recorded forward (the plan's buffers still hold it).  Walks the graph ops in reverse.
int run_backward(v2v_plan* P, void* const* io, void* const* gio, const std::unordered_map<const void*, void*>& pg,
                        cudaStream_t s) {
  const BwdRequest q{io, gio, &pg};
  V2V_CUDA(cudaMemsetAsync(P->garena, 0, P->garena_bytes, s));
  auto conv_bwd = [&](const GOp& op) -> int {
    BwdConv b = conv_bwd_params(P, op, q);
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
      if (b.dx) V2V_CUDA(launch_fold_add(fold_params(P, u, b.dx), s));
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
        const GradLayout g = grad_layout_params(P, op, q);
        if (g.g) V2V_CUDA(launch_grad_import(g, s));
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
        V2V_CUDA(launch_head_bwd(head_bwd_params(P, op, q), s));
        int rc = conv_bwd(op); if (rc) return rc;
        break;
      }
      case G_NORM_ACT: {
        const Raw& r = P->raws[op.raw];
        const NormBwd n = norm_bwd_params(P, op, q);
        if (!n.has_norm && !P->gops[r.conv_op].conv.bias)     // plain activation of a bias-less conv: scale / shift arrays are unset
          V2V_CUDA(launch_bias_affine(r.scale, r.shift, nullptr, r.N, r.C, r.C, s));
        V2V_CUDA(launch_norm_bwd(n, s));
        break;
      }
      case G_CONV: {
        int rc = conv_bwd(op); if (rc) return rc;
        break;
      }
      case G_CONV_ACT: {
        const Value& vo = P->values[op.value_out];
        V2V_CUDA(launch_convact_bwd(vo.gval, P->acts[vo.bufs[0]], op.act, op.slope, op.gdz, op.conv.Cout, round_up(op.conv.Cout, 8), s));
        int rc = conv_bwd(op); if (rc) return rc;
        break;
      }
      case G_INPUT: {
        const GradLayout g = grad_layout_params(P, op, q);
        if (g.g) V2V_CUDA(launch_grad_export(g, s));
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

// One backward record: the data-gradient mode (0: SIMT, "simt" says why), the sub-plan's conv as a conv record, and the
// weight-gradient launch (null: SIMT, "wgrad_simt" says why).
void describe_backward_unit(const BwdUnit& u, Json& j) {
  j.obj().kv("gop", u.gop).kv("mode", u.mode).kv("simt", u.simt).kv("wgrad_simt", u.wg_simt).key("conv");
  if (u.mode) describe_conv(u.child, u.child->gops[1], j);
  else j.null();
  j.key("wgrad");
  if (u.wgrad) {
    const WgradParams& w = u.wg;
    j.obj().kv("swap", w.swap).kv("KP", w.KP).kv("BN", w.BN).kv("Mblocks", w.Mblocks).kv("Nblocks", w.Nblocks).kv("b_row", w.b_row)
        .kv("m_tiles", w.m_tiles).kv("n_tiles", w.n_tiles).kv("ntaps", w.ntaps).kv("ksplit", w.ksplit)
        .kv("chunks_per_unit", w.chunks_per_unit).kv("chunks_total", w.chunks_total).kv("xsegs", w.xsegs).kv("gh", w.gh)
        .kv("gw", w.gw).kv("stages", w.stages).kv("split", w.split).kv("Mp", w.Mp).kv("Np", w.Np).end();
  } else {
    j.null();
  }
  j.end();
}

// The layout launches of the backward as run_backward makes them, assuming the caller passes every gradient: the gradient
// import of every export and the gradient export of every input, then per tensor-core unit the packing of its sub-plan's
// weights (the dgrad packing in mode 1), the fold of the data gradient into dX (crop: the sub-plan's output extends past the
// padded input; overlap: a reflect halo so deep that the top and bottom, or left and right, mirrors reach the same pixel)
// and the unstage of the weight gradient.
void describe_backward_layout(const v2v_plan* P, const std::vector<BwdUnit>& units, Json& j) {
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (!P->op_live[i] || (op.kind != G_EXPORT && op.kind != G_INPUT)) continue;
    const GradLayout g = grad_layout_params(P, op, kEveryGradient);
    j.obj().kv("kind", op.kind == G_EXPORT ? "grad_import" : "grad_export").kv("gop", i).kv("N", g.N).kv("C", g.C).kv("H", g.H)
        .kv("W", g.W).kv("C_src", g.C_src).kv("c_off", g.c_off).kv("tiled", grad_layout_tiled(g)).end();
  }
  for (const BwdUnit& u : units) {
    if (!u.mode) continue;
    describe_pack(u.child, 1, j);
    const FoldParams f = fold_params(P, u, nullptr);
    j.obj().kv("kind", "fold").kv("gop", u.gop).kv("mode", u.mode).kv("pad", f.pad).kv("reflect", f.reflect)
        .kv("crop", f.PH > f.H + 2 * f.pad || f.PW > f.W + 2 * f.pad)
        .kv("overlap", f.reflect && (f.pad >= f.H - 1 - f.pad || f.pad >= f.W - 1 - f.pad)).kv("N", f.N).kv("H", f.H)
        .kv("W", f.W).kv("C", f.C).kv("PH", f.PH).kv("PW", f.PW).kv("Cs", f.Cs).end();
    if (u.wgrad)
      j.obj().kv("kind", "unstage").kv("gop", u.gop).kv("swap", u.wg.swap).kv("R", u.M).kv("R1", u.M1).kv("Cc", u.Nv)
          .kv("taps", u.wg.ntaps).kv("Mp", u.wg.Mp).kv("Np", u.wg.Np).end();
  }
}

// One record per live G_NORM_ACT / G_CONV_ACT / G_HEAD: the launches of its epilogue backward as run_backward makes them,
// assuming every parameter gradient (gamma, beta, bias) is requested.  Norm units: the norm_bwd_launch choice; conv_act and
// head units: the dense dz buffer's channel stride, the stacked second bias (channels from C1 on go to dbias2) and the
// bias_grad grid.
void describe_epilogue_backward(const v2v_plan* P, Json& j) {
  j.key("epilogue_backward").arr();
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (!P->op_live[i] || !(op.kind == G_NORM_ACT || op.kind == G_CONV_ACT || op.kind == G_HEAD)) continue;
    if (op.kind == G_NORM_ACT) {
      const NormBwd n = norm_bwd_params(P, op, kEveryGradient);
      const NormBwdLaunch l = norm_bwd_launch(n);
      j.obj().kv("kind", "norm_act").kv("gop", i).kv("raw", op.raw).kv("C", n.C).kv("N", n.N).kv("H", n.H).kv("W", n.W)
          .kv("c_off", n.c_off).kv("raw_C", n.raw.C).kv("raw_f32", n.raw.f32).kv("has_norm", n.has_norm)
          .kv("batch_stats", n.batch_stats).kv("act", n.act).kv("adds", (op.add[0] >= 0) + (op.add[1] >= 0))
          .kv("reduce", l.reduce == 1 ? "vec" : (l.reduce == 2 ? "scalar" : "none")).kv("ppb", l.ppb).kv("chunk", l.chunk)
          .kv("grid", {l.grid[0], l.grid[1], l.grid[2]}).kv("param", l.param).end();
      continue;
    }
    const BwdConv b = conv_bwd_params(P, op, kEveryGradient);
    const bool bias = b.dbias || b.dbias2;
    j.obj().kv("kind", op.kind == G_HEAD ? "head" : "conv_act").kv("gop", i).kv("C", b.Cout).kv("N", b.N).kv("H", b.oh)
        .kv("W", b.ow).kv("dz_C", b.dy_C).kv("bias", bias).kv("C1", b.w2 ? b.Cout1 : b.Cout)
        .kv("bias_grid", {bias ? b.Cout : 0, bias ? bias_grad_blocks((long long)b.N * b.oh * b.ow) : 0}).key("acts").arr();
    if (op.kind == G_HEAD) {
      const HeadBwd h = head_bwd_params(P, op, kEveryGradient);
      for (int c = 0; c < h.Cout; ++c) j.val(h.act[c]);
    } else {
      j.val(op.act);
    }
    j.end().end();
  }
  j.end();
}

}  // namespace v2v
