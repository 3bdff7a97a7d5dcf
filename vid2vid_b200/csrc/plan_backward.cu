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
// caller.  The device half is build_backward_units; v2v_plan_describe reports the same choice without a device.
int choose_backward_unit(v2v_plan* P, int i, BwdUnit& u) {
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

// Device half: finalizes each unit's sub-plan, encodes the weight gradient's tensor maps and allocates its stage buffer.
int build_backward_units(v2v_plan* P, cudaStream_t stream) {
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
    rc = v2v_plan_finalize(u.child, reinterpret_cast<v2v_stream_t>(stream)); if (rc) return rc;
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

// Backward of one recorded forward (the plan's buffers still hold it).  Walks the graph ops in reverse.
int run_backward(v2v_plan* P, void* const* io, void* const* gio, const std::unordered_map<const void*, void*>& pg,
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
        n.scale = r.scale + op.n_off; n.shift = r.shift + op.n_off; n.stat_stride = r.C;
        n.mean = n.has_norm ? r.mean + op.n_off : nullptr; n.rstd = n.has_norm ? r.rstd + op.n_off : nullptr;
        if (!n.has_norm && !cop.conv.bias)     // plain activation of a bias-less conv: scale / shift arrays are unset
          V2V_CUDA(launch_bias_affine(r.scale, r.shift, nullptr, r.N, r.C, r.C, s));
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

// One backward record: the data-gradient mode (0: SIMT, "simt" says why), the sub-plan's conv as a conv record, and the
// weight-gradient launch (null: SIMT, "wgrad_simt" says why).
void describe_backward_unit(const BwdUnit& u, std::string& s) {
  char t[640];
  snprintf(t, sizeof(t), "{\"gop\":%d,\"mode\":%d,\"simt\":\"%s\",\"wgrad_simt\":\"%s\",\"conv\":", u.gop, u.mode, u.simt.c_str(),
           u.wg_simt.c_str());
  s += t;
  if (u.mode) describe_conv(u.child, u.child->gops[1], s);
  else s += "null";
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

// The layout launches of one tensor-core backward unit as run_backward makes them (each record with a leading comma): the
// packing of the sub-plan's weights (the dgrad packing in mode 1), the fold of the data gradient into dX (crop: the sub-plan's
// output extends past the padded input; overlap: a reflect halo so deep that the top and bottom, or left and right, mirrors
// reach the same pixel) and the unstage of the weight gradient.
void describe_backward_layout(const v2v_plan* P, const BwdUnit& u, std::string& s) {
  if (!u.mode) return;
  char t[512];
  s += ",";
  describe_pack(u.child, 1, s);
  const GOp& op = P->gops[u.gop];
  const Value& vin = P->values[op.value_in];
  const Raw& cr = u.child->raws[u.child_raw];
  const int pad = u.mode == 1 ? op.conv.pad : 0;
  const int reflect = (op.conv.pad_mode == V2V_PAD_REFLECT && pad > 0) ? 1 : 0;
  const int crop = cr.H > vin.H + 2 * pad || cr.W > vin.W + 2 * pad;
  const int overlap = reflect && (pad >= vin.H - 1 - pad || pad >= vin.W - 1 - pad);
  snprintf(t, sizeof(t),
           ",{\"kind\":\"fold\",\"gop\":%d,\"mode\":%d,\"pad\":%d,\"reflect\":%d,\"crop\":%d,\"overlap\":%d,\"N\":%d,\"H\":%d,\"W\":%d,"
           "\"C\":%d,\"PH\":%d,\"PW\":%d,\"Cs\":%d}",
           u.gop, u.mode, pad, reflect, crop, overlap, vin.N, vin.H, vin.W, op.conv.Cin, cr.H, cr.W, cr.desc.C);
  s += t;
  if (u.wgrad) {
    snprintf(t, sizeof(t), ",{\"kind\":\"unstage\",\"gop\":%d,\"swap\":%d,\"R\":%d,\"R1\":%d,\"Cc\":%d,\"taps\":%d,\"Mp\":%d,\"Np\":%d}",
             u.gop, u.wg.swap, u.M, u.M1, u.Nv, u.wg.ntaps, u.wg.Mp, u.wg.Np);
    s += t;
  }
}

// One record per live G_NORM_ACT / G_CONV_ACT / G_HEAD: the launches of its epilogue backward as run_backward makes them,
// assuming every parameter gradient (gamma, beta, bias) is requested.  Norm units: the norm_bwd_launch choice; conv_act and
// head units: the dense dz buffer's channel stride, the stacked second bias (channels from C1 on go to dbias2) and the
// bias_grad grid.
void describe_epilogue_backward(const v2v_plan* P, std::string& s) {
  char t[640];
  bool first = true;
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (!P->op_live[i] || !(op.kind == G_NORM_ACT || op.kind == G_CONV_ACT || op.kind == G_HEAD)) continue;
    if (!first) s += ",";
    first = false;
    if (op.kind == G_NORM_ACT) {
      const Raw& r = P->raws[op.raw];
      const GOp& cop = P->gops[r.conv_op];
      const Value& vo = P->values[op.value_out];
      const int has_norm = op.norm.kind != V2V_NORM_NONE;
      const int param = has_norm ? (op.norm.gamma || op.norm.beta) : ((op.n_off == 0 ? cop.conv.bias : cop.conv.bias2) != nullptr);
      const NormBwdLaunch l = norm_bwd_launch(vo.N, vo.H, vo.W, op.cC, r.desc.C, op.n_off, has_norm, param);
      snprintf(t, sizeof(t),
               "{\"kind\":\"norm_act\",\"gop\":%zu,\"raw\":%d,\"C\":%d,\"N\":%d,\"H\":%d,\"W\":%d,\"c_off\":%d,\"raw_C\":%d,\"raw_f32\":%d,"
               "\"has_norm\":%d,\"batch_stats\":%d,\"act\":%d,\"adds\":%d,\"reduce\":\"%s\",\"ppb\":%d,\"chunk\":%lld,\"grid\":[%d,%d,%d],"
               "\"param\":%d}",
               i, op.raw, op.cC, vo.N, vo.H, vo.W, op.n_off, r.desc.C, r.desc.f32, has_norm, op.norm.kind == V2V_NORM_BATCH ? 1 : 0,
               op.act, (op.add[0] >= 0) + (op.add[1] >= 0), l.reduce == 1 ? "vec" : (l.reduce == 2 ? "scalar" : "none"), l.ppb,
               l.chunk, l.grid[0], l.grid[1], l.grid[2], l.param);
      s += t;
      continue;
    }
    const v2v_conv_desc& c = op.conv;
    const Value& vin = P->values[op.value_in];
    const long long npix = (long long)vin.N * op.geom.out_h * op.geom.out_w;
    const int has_bias = c.bias != nullptr || (c.Cout2 > 0 && c.bias2 != nullptr);
    snprintf(t, sizeof(t),
             "{\"kind\":\"%s\",\"gop\":%zu,\"C\":%d,\"N\":%d,\"H\":%d,\"W\":%d,\"dz_C\":%d,\"bias\":%d,\"C1\":%d,\"bias_grid\":[%d,%d],"
             "\"acts\":[",
             op.kind == G_HEAD ? "head" : "conv_act", i, c.Cout, vin.N, op.geom.out_h, op.geom.out_w, round_up(c.Cout, 8), has_bias,
             c.Cout2 > 0 ? c.Cout - c.Cout2 : c.Cout, has_bias ? c.Cout : 0, has_bias ? bias_grad_blocks(npix) : 0);
    s += t;
    const int nch = op.kind == G_HEAD ? c.Cout : 1;
    for (int j = 0; j < nch; ++j) {
      snprintf(t, sizeof(t), "%s%d", j ? "," : "", op.kind == G_HEAD ? op.head[j].act : op.act);
      s += t;
    }
    s += "]}";
  }
}

}  // namespace v2v
