// Plan runtime: lowers a graph of logical values / convolution units (described through the C ABI in
// include/v2v_b200.h) to halo-padded NHWC bf16 buffers, TMA tensor maps, packed weight matrices and a
// flat kernel sequence, captures the sequence in a CUDA graph and replays it per frame.  Each conv's geometry, tiling and
// tensor maps come from conv_lower.cu; training plans' gradient buffers and backward pass from plan_backward.cu.
// This is the H100-native counterpart of the nn.Module surface the reference's Vid2VidModelG calls
// (netG.forward, models/vid2vid_model_G.py:225-226; module bodies models/networks.py:117-419,634-725).
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "plan_internal.h"

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

static ActDesc make_act(const Value& v, const Req& r, int split) {
  ActDesc a{};
  a.split = split;
  a.base = nullptr;
  a.N = v.N; a.H = v.H; a.W = v.W; a.Cvalid = v.C; a.C = v.Cp;
  a.pad_t = r.pads[0]; a.pad_l = r.pads[1]; a.pad_b = r.pads[2]; a.pad_r = r.pads[3];
  a.parity = r.parity;
  const int Hpad = v.H + a.pad_t + a.pad_b, Wpad = v.W + a.pad_l + a.pad_r;
  if (a.parity) { a.P = 4; a.Hp = (Hpad + 1) / 2; a.Wp = (Wpad + 1) / 2; }
  else { a.P = 1; a.Hp = Hpad; a.Wp = Wpad; }
  return a;
}

static bool same_req(const Req& a, const Req& b) {
  return a.mode == b.mode && a.parity == b.parity && !memcmp(a.pads, b.pads, sizeof(a.pads));
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
      int rc = conv_geometry(op.conv, vin.Cp, op.kind == G_HEAD ? (P->impl == V2V_IMPL_UMMA ? 2 : 1) : 0, P->tiling_n(vin.N), vin.H,
                             vin.W, true, P->sp(), &op.geom);
      if (rc) return rc;
      op.req_index = add_req(vin, conv_req(op.conv, op.geom));
      const v2v_conv_desc& c = op.conv;
      const double px = op.conv.transposed ? (double)vin.N * vin.H * vin.W : (double)vin.N * op.geom.out_h * op.geom.out_w;
      op.macs = px * c.Cin * c.Cout * c.kh * c.kw;
      P->conv_macs += op.macs;
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

int new_value(v2v_plan* p, int N, int H, int W, int C) {
  Value v; v.N = N; v.H = H; v.W = W; v.C = C; v.Cp = std::max(pad_channels(C), p->pad_min);
  p->values.push_back(v);
  return (int)p->values.size() - 1;
}

// Host-only: lower the graph, choose every conv's tiling and lay the arena out (offsets only).  Idempotent.
int size_arena(v2v_plan* P) {
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

int run_xop(v2v_plan* P, const XOp& x, cudaStream_t s) {
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
      if (P->impl == V2V_IMPL_UMMA) V2V_CUDA(launch_conv_umma(op.tmA, op.tmB, x.kp, s));
      else V2V_CUDA(launch_conv_simt(P->acts[P->values[op.value_in].bufs[op.req_index]], op.wpacked, op.Ktotal, x.kp, s));
      break;
    }
  }
  return 0;
}

FeatL1Params featl1_params(const v2v_plan* P, const GOp& op) {
  FeatL1Params f{};
  f.x = P->acts[P->values[op.value_in].bufs[0]]; f.y = P->acts[P->values[op.value_in2].bufs[0]];
  f.Cvalid = P->values[op.value_in].C;
  f.io = P->io_dev; f.slot = op.slot; f.index = op.l1_index;
  f.blocks = feature_l1_blocks(f.x);
  return f;
}

// Address `off` bytes into the plan's arena.  Integer arithmetic: before finalize binds the arena (null) an address is its
// offset, so the host-only emission never offsets a null pointer.
template <class T> static T* arena_at(const v2v_plan* P, size_t off) {
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(P->arena) + off);
}

// The finalisation of the slice a normalising G_NORM_ACT reads, with its train-mode side effects (running statistics; the
// scale / shift / mean / rstd arrays the normalise passes and the backward read).
static int finalize_params(const v2v_plan* P, const GOp& op, FinalizeParams& fp) {
  const Raw& r = P->raws[op.raw];
  const GOp& cop = P->gops[r.conv_op];
  fp.stats = r.stats; fp.Cs = r.C; fp.C = op.cC; fp.c_off = op.n_off; fp.scale_stride = r.C;
  fp.N = r.N;
  fp.count = (double)r.H * r.W; fp.instance = (op.norm.kind == V2V_NORM_INSTANCE) || P->sample_stats;
  fp.sample_running = P->sample_stats;
  fp.io = P->io_dev; fp.flags_slot = P->flags_slot;
  const int cout1 = cop.conv.Cout - cop.conv.Cout2;
  V2V_REQUIRE(op.n_off == 0 || (cop.conv.Cout2 > 0 && op.n_off == cout1), V2V_ERR_UNSUPPORTED,
              "a raw slice must start at channel 0 or at the second weight set");
  fp.gamma = op.norm.gamma; fp.beta = op.norm.beta; fp.conv_bias = op.n_off == 0 ? cop.conv.bias : cop.conv.bias2;
  fp.momentum = op.norm.momentum; fp.eps = op.norm.eps;
  fp.running_mean = op.norm.running_mean; fp.running_var = op.norm.running_var;
  fp.num_batches_tracked = reinterpret_cast<long long*>(op.norm.num_batches_tracked);
  fp.scale = r.scale; fp.shift = r.shift; fp.mean_out = r.mean; fp.rstd_out = r.rstd;
  return 0;
}

// The normalise pass of a G_NORM_ACT (or the plain conversion of a G_RAWIN) into output layout m of its value.  The raw is
// read through the op's channel slice at the full row stride; scale / shift are the slice's (null: identity, G_RAWIN and
// norm-less unbiased convs).  The launch shape depends on the layouts only.
static ApplyParams apply_params(const v2v_plan* P, const GOp& op, size_t m) {
  const Value& vo = P->values[op.value_out];
  ApplyParams ap{};
  if (op.kind == G_RAWIN) {
    ap.raw.base = const_cast<float*>(op.ext_raw); ap.raw.N = vo.N; ap.raw.H = vo.H; ap.raw.W = vo.W; ap.raw.C = op.ext_C;
    ap.raw.Cvalid = vo.C; ap.raw.f32 = 1;
    ap.scale = nullptr; ap.shift = nullptr; ap.scale_stride = 0; ap.act = ACT_NONE; ap.slope = 0.f; ap.n_add = 0;
  } else {
    const Raw& r = P->raws[op.raw];
    const v2v_plan::RawOff& o = P->raw_off[op.raw];
    const GOp& cop = P->gops[r.conv_op];
    ap.raw = r.desc;
    ap.raw.base = arena_at<void>(P, o.raw + (size_t)op.n_off * r.desc.elem_bytes());
    ap.raw.Cvalid = op.cC;                                               // channel slice, full row stride
    const bool scaled = op.norm.kind != V2V_NORM_NONE || cop.conv.bias != nullptr;
    ap.scale = scaled ? arena_at<float>(P, o.scale + op.n_off * sizeof(float)) : nullptr;
    ap.shift = arena_at<float>(P, o.shift + op.n_off * sizeof(float));
    ap.scale_stride = r.C;
    ap.act = op.act; ap.slope = op.slope;
    ap.n_add = 0;
    for (int k = 0; k < 2; ++k) if (op.add[k] >= 0) ap.add[ap.n_add++] = P->acts[P->values[op.add[k]].bufs[0]];
  }
  ap.out = P->acts[vo.bufs[m]]; ap.pad_mode = P->act_pad_mode[vo.bufs[m]];
  return ap;
}

// Host-only: the forward launch list of a sized plan, in launch order, with every launch's parameters.  Arena addresses come
// from the buffers finalize binds and from arena_at, so on an unbound plan the list differs from the finalized one in its
// addresses only.  v2v_plan_finalize runs this list and v2v_plan_describe reports it: both refuse the same plans.
static int emit_forward(const v2v_plan* P, std::vector<XOp>& xops) {
  if (P->stats_end > P->stats_begin) {
    XOp m; m.kind = X_MEMSET; m.ms_ptr = arena_at<void>(P, P->stats_begin); m.ms_bytes = P->stats_end - P->stats_begin;
    xops.push_back(m);
  }
  std::vector<int> conv_x(P->gops.size(), -1);                 // per conv op: its launch in xops
  std::vector<std::vector<int>> read(P->raws.size()), fin(P->raws.size());   // per raw: the slices normalised / finalised so far
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    switch (op.kind) {
      case G_INPUT: {
        const Value& v = P->values[op.value_out];
        for (size_t m = 0; m < v.bufs.size(); ++m) {
          XOp x; x.kind = X_IMPORT; x.gop = (int)i; x.buf = v.bufs[m];
          x.imp.io = reinterpret_cast<const void* const*>(P->io_dev); x.imp.slot = op.slot;
          x.imp.c_off = op.c_off; x.imp.C_src = op.C_src;
          x.imp.out = P->acts[v.bufs[m]]; x.imp.pad_mode = P->act_pad_mode[v.bufs[m]];
          x.imp.skip_lo = v.exact_bf16 ? 1 : 0;
          xops.push_back(x);
        }
        break;
      }
      case G_CONV: case G_CONV_ACT: case G_HEAD: {
        const ActDesc& ain = P->acts[P->values[op.value_in].bufs[op.req_index]];
        XOp x; x.kind = X_CONV; x.gop = (int)i;
        ConvKernelParams& kp = x.kp;
        kp = op.kp;
        // the kernel addresses the lo half of the input at channel coordinate Cp: the buffer must be padded to exactly that
        V2V_REQUIRE(kp.Cp == ain.C, V2V_ERR_STATE, "internal: conv of op %zu reads %d padded channels from a %d-channel buffer", i,
                    kp.Cp, ain.C);
        kp.io = P->io_dev;
        if (op.kind == G_CONV) {
          const Raw& r = P->raws[op.raw];
          kp.epi = EPI_RAW_STATS; kp.out = r.desc.base; kp.out_C = r.desc.C; kp.out_f32 = r.desc.f32;
          kp.stats = r.no_stats ? nullptr : r.stats; kp.stats_C = r.C; kp.bias = nullptr;
        } else if (op.kind == G_CONV_ACT) {
          const Value& vo = P->values[op.value_out];
          V2V_REQUIRE(vo.bufs.size() == 1 && P->act_pad_mode[vo.bufs[0]] != PAD_REFLECT, V2V_ERR_UNSUPPORTED,
                      "conv_act output needs a single zero/none-padded consumer layout");
          kp.epi = EPI_ACT_BF16; kp.out_act = P->acts[vo.bufs[0]]; kp.out_C = kp.out_act.C;
        }
        conv_x[i] = (int)xops.size();
        xops.push_back(x);
        if (op.kind == G_CONV && P->impl == V2V_IMPL_SIMT) {
          XOp s; s.kind = X_RAWSTATS; s.gop = (int)i;
          s.rawd = P->raws[op.raw].desc; s.stats = P->raws[op.raw].stats; s.stats_C = P->raws[op.raw].C;
          xops.push_back(s);
        }
        break;
      }
      case G_NORM_ACT: case G_RAWIN: {      // normalise passes (of a G_RAWIN: a plain conversion)
        bool repeat = false;
        if (op.kind == G_NORM_ACT) {
          const Raw& r = P->raws[op.raw];
          const GOp& cop = P->gops[r.conv_op];
          const bool has_norm = op.norm.kind != V2V_NORM_NONE;
          // a norm-less biased conv (FlowNet2's conv / deconv / predict_flow units) is normalised with scale 1 and shift =
          // bias (finalize's bias affines), which cover the whole raw
          V2V_REQUIRE(has_norm || cop.conv.bias == nullptr || (op.n_off == 0 && cop.conv.Cout2 == 0), V2V_ERR_UNSUPPORTED,
                      "biased norm-less conv cannot be sliced");
          std::vector<int>& rd = read[op.raw], &fd = fin[op.raw];
          repeat = std::find(rd.begin(), rd.end(), op.n_off) != rd.end();
          if (!repeat) rd.push_back(op.n_off);
          if (has_norm && std::find(fd.begin(), fd.end(), op.n_off) == fd.end()) {
            // the slice's first normalising pass finalises its statistics, with the side effects, once however many passes
            // read it: in a tail slot of the producing tensor-core conv launch (the CTA that takes its last ticket,
            // conv_umma.cu) while one is free, else in a stand-alone stats_finalize launch (the SIMT implementation, a third
            // slice of one raw)
            fd.push_back(op.n_off);
            XOp f; f.kind = X_FINALIZE; f.gop = (int)i;
            int rc = finalize_params(P, op, f.fin); if (rc) return rc;
            ConvKernelParams& ckp = xops[conv_x[r.conv_op]].kp;
            if (P->impl == V2V_IMPL_UMMA && ckp.n_fin < 2) {
              xops[conv_x[r.conv_op]].fin_gop[ckp.n_fin] = (int)i;
              ckp.fin[ckp.n_fin++] = f.fin;
              ckp.fin_counter = arena_at<unsigned int>(P, P->raw_off[op.raw].stats + (size_t)r.N * 2 * r.C * sizeof(stat_t));
            } else {
              xops.push_back(f);
            }
          }
        }
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          XOp a; a.kind = X_APPLY; a.gop = (int)i; a.buf = vo.bufs[m]; a.repeat = repeat; a.app = apply_params(P, op, m);
          xops.push_back(a);
        }
        break;
      }
      case G_EXPORT: {
        XOp x; x.kind = X_EXPORT; x.gop = (int)i; x.buf = P->values[op.value_in].bufs[0];
        x.exp.io = P->io_dev; x.exp.slot = op.slot; x.exp.in = P->acts[x.buf];
        xops.push_back(x);
        break;
      }
      case G_COMPOSITE: {
        XOp x; x.kind = X_COMPOSITE; x.gop = (int)i; x.comp = op.comp; x.comp.io = P->io_dev; x.comp.s_flags = P->flags_slot;
        xops.push_back(x);
        break;
      }
      case G_CONCAT: {
        const Value& vo = P->values[op.value_out];
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          int c_off = 0;
          for (int src : op.cat_in) {
            XOp x; x.kind = X_COPY; x.gop = (int)i; x.buf = vo.bufs[m]; x.in_buf = P->values[src].bufs[0];
            x.copy.in = P->acts[x.in_buf];
            x.copy.out = P->acts[x.buf];
            x.copy.c_off = c_off; x.copy.pad_mode = P->act_pad_mode[x.buf];
            c_off += P->values[src].C;
            xops.push_back(x);
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
          xops.push_back(x);
        }
        break;
      }
      case G_FEATL1: {
        XOp x; x.kind = X_FEATL1; x.gop = (int)i;
        x.fl1 = featl1_params(P, op);
        x.fl1.partials = arena_at<double>(P, P->l1_off[i]);
        xops.push_back(x);
        break;
      }
      case G_CORR: {
        const Value& va = P->values[op.value_in], &vb = P->values[op.value_in2], &vo = P->values[op.value_out];
        const size_t bytes = (size_t)va.N * va.C * va.H * va.W * sizeof(float);
        float* sa = arena_at<float>(P, P->corr_off[i]);
        float* sb = arena_at<float>(P, P->corr_off[i] + bytes);
        float* so = arena_at<float>(P, P->corr_off[i] + 2 * bytes);
        XOp ea; ea.kind = X_EXPORT; ea.gop = (int)i; ea.buf = va.bufs[0];
        ea.exp.io = P->io_dev; ea.exp.slot = 0; ea.exp.direct = sa; ea.exp.in = P->acts[va.bufs[0]];
        XOp eb = ea; eb.buf = vb.bufs[0]; eb.exp.direct = sb; eb.exp.in = P->acts[vb.bufs[0]];
        xops.push_back(ea); xops.push_back(eb);
        XOp c; c.kind = X_CORR; c.gop = (int)i;
        c.corr = CorrParams{sa, sb, so, va.N, va.C, va.H, va.W, op.corr[0], op.corr[1], op.corr[2], op.corr[3], op.corr[4]};
        xops.push_back(c);
        for (size_t m = 0; m < vo.bufs.size(); ++m) {
          XOp x; x.kind = X_IMPORT; x.gop = (int)i; x.buf = vo.bufs[m];
          x.imp.io = reinterpret_cast<const void* const*>(P->io_dev); x.imp.slot = 0; x.imp.direct = so;
          x.imp.c_off = 0; x.imp.C_src = vo.C; x.imp.act = op.act; x.imp.slope = op.slope;
          x.imp.out = P->acts[vo.bufs[m]]; x.imp.pad_mode = P->act_pad_mode[vo.bufs[m]];
          xops.push_back(x);
        }
        break;
      }
    }
  }
  return 0;
}

// The arena layout of v2v_plan_describe (host-only: needs the arena sized): one "buffers" record per activation buffer (its byte
// offset in the arena and the ActDesc fields that place element (n, c, y, x)), and one "scratch" record per correlation's fp32
// scratch [in1 | in2 | out], each NCHW.  A caller that finalizes into its own workspace can decode every buffer from these.
static void describe_buffers(const v2v_plan* P, Json& j) {
  j.key("buffers").arr();
  for (size_t v = 0; v < P->values.size(); ++v)
    for (int b : P->values[v].bufs) {
      const ActDesc& a = P->acts[b];
      j.obj().kv("value", v).kv("buf", b).kv("off", P->act_off[b]).kv("N", a.N).kv("H", a.H).kv("W", a.W).kv("C", a.C)
          .kv("Cvalid", a.Cvalid).kv("pads", {a.pad_t, a.pad_l, a.pad_b, a.pad_r}).kv("parity", a.parity).kv("P", a.P)
          .kv("Hp", a.Hp).kv("Wp", a.Wp).kv("split", a.split).kv("mode", P->act_pad_mode[b]).end();
    }
  j.end().key("scratch").arr();
  for (size_t i = 0; i < P->gops.size(); ++i) {
    const GOp& op = P->gops[i];
    if (op.kind != G_CORR) continue;
    const Value& a = P->values[op.value_in], &o = P->values[op.value_out];
    j.obj().kv("gop", i).kv("off", P->corr_off[i]).kv("N", a.N).kv("C", a.C).kv("H", a.H).kv("W", a.W).kv("C_out", o.C)
        .kv("H_out", o.H).kv("W_out", o.W).end();
  }
  j.end();
}

// The record writers of the forward launch list, one per launch kind.  An import or export of a correlation (direct) moves its
// fp32 scratch instead of a caller tensor.
static void describe_import(const v2v_plan* P, const XOp& x, Json& j) {
  const ImportParams& p = x.imp;
  const ActDesc& o = p.out;
  j.obj().kv("kind", "import").kv("gop", x.gop).kv("buf", x.buf).kv("slot", p.slot).kv("direct", P->gops[x.gop].kind == G_CORR)
      .kv("C_src", p.C_src).kv("c_off", p.c_off).kv("act", p.act).kv("pad_mode", p.pad_mode).kv("skip_lo", p.skip_lo)
      .kv("split", o.split).kv("parity", o.parity).kv("N", o.N).kv("H", o.H).kv("W", o.W).kv("C", o.C).kv("Cvalid", o.Cvalid)
      .kv("Wpad", o.W + o.pad_l + o.pad_r).kv("CT", import_tile_channels(o)).end();
}

static void describe_export(const v2v_plan* P, const XOp& x, Json& j) {
  const ActDesc& a = x.exp.in;
  j.obj().kv("kind", "export").kv("gop", x.gop).kv("buf", x.buf).kv("direct", P->gops[x.gop].kind == G_CORR).kv("split", a.split)
      .kv("N", a.N).kv("H", a.H).kv("W", a.W).kv("C", a.C).kv("Cvalid", a.Cvalid).end();
}

static void describe_copy(const XOp& x, Json& j) {
  const CopyParams& p = x.copy;
  j.obj().kv("kind", "copy").kv("gop", x.gop).kv("in_buf", x.in_buf).kv("buf", x.buf).kv("c_off", p.c_off).kv("Cvalid", p.in.Cvalid)
      .kv("pad_mode", p.pad_mode).kv("in_split", p.in.split).kv("split", p.out.split).kv("parity", p.out.parity).end();
}

static const char* kFinSite[] = {"tail0", "tail1", "standalone"};
struct FinRecord { int gop, site; const FinalizeParams* fp; };

// stats: how conv_umma_kernel accumulates the statistics rows of a conv whose raw a norm layer reads (async_epi, MG, BN,
// phases, units over ctas persistent CTAs) or raw_stats_kernel (SIMT), and where each of its slices is finalised
static void describe_stats(const v2v_plan* P, const XOp& x, const std::vector<int>& sites, Json& j) {
  const GOp& op = P->gops[x.gop];
  const Raw& r = P->raws[op.raw];
  const ConvKernelParams& kp = x.kp;
  j.obj().kv("kind", "stats").kv("gop", x.gop).kv("raw", op.raw).kv("N", r.N).kv("C", r.C).kv("H", r.H).kv("W", r.W)
      .kv("raw_f32", r.desc.f32).kv("impl", P->impl == V2V_IMPL_UMMA ? "umma" : "simt").kv("async_epi", conv_umma_async_epilogue(kp))
      .kv("MG", kp.MG).kv("BN", kp.BN).kv("phases", kp.num_phases).kv("n_tiles", kp.n_tiles).kv("m_total", kp.m_total)
      .kv("units", kp.total_units).kv("ctas", kp.grid).key("fin").arr();
  for (int q : sites) j.val(kFinSite[q]);
  j.end().end();
}

// finalize: batch / instance / per-sample statistics, image flags, running buffers, conv bias, the saved mean / rstd of training
// plans, the slice
static void describe_finalize(const v2v_plan* P, const FinRecord& f, Json& j) {
  const FinalizeParams& fp = *f.fp;
  j.obj().kv("kind", "finalize").kv("gop", f.gop).kv("raw", P->gops[f.gop].raw).kv("site", kFinSite[f.site])
      .kv("stats", fp.sample_running ? "sample" : (fp.instance ? "instance" : "batch")).kv("N", fp.N).kv("flags", fp.flags_slot >= 0)
      .kv("running", fp.running_mean != nullptr).kv("bias", fp.conv_bias != nullptr).kv("mean_rstd", P->train).kv("c_off", fp.c_off)
      .kv("C", fp.C).end();
}

// apply: the norm_apply_launch choice of one normalise pass into one output layout, and what the kernel reads and writes
static void describe_apply(const v2v_plan* P, const XOp& x, Json& j) {
  const GOp& op = P->gops[x.gop];
  const std::vector<int>& bufs = P->values[op.value_out].bufs;
  const size_t layout = std::find(bufs.begin(), bufs.end(), x.buf) - bufs.begin();
  const char* scale = op.kind == G_RAWIN ? "none" : (op.norm.kind != V2V_NORM_NONE ? "norm" :
                      (P->gops[P->raws[op.raw].conv_op].conv.bias != nullptr ? "bias" : "none"));
  const ApplyParams& ap = x.app;
  const NormApplyLaunch l = norm_apply_launch(ap);
  const ActDesc& o = ap.out;
  const int Wpad = o.W + o.pad_l + o.pad_r;
  j.obj().kv("kind", "apply").kv("gop", x.gop).kv("op", op.kind == G_RAWIN ? "rawin" : "norm_act").kv("raw", op.raw)
      .kv("layout", layout).kv("repeat", x.repeat).kv("kernel", l.rows ? "rows" : "grid_stride").kv("prec", ap.raw.f32)
      .kv("nadd", ap.n_add).kv("vecs", l.vecs).kv("ppb", l.ppb).kv("xt", l.xt).kv("grid", {l.grid[0], l.grid[1]})
      .kv("idle", l.rows && 256 % l.vecs != 0).kv("ragged", l.rows && Wpad % l.xt != 0).kv("N", o.N).kv("H", o.H).kv("W", o.W)
      .kv("C", o.C).kv("Cvalid", ap.raw.Cvalid).kv("raw_C", ap.raw.C).kv("c_off", op.kind == G_RAWIN ? 0 : op.n_off)
      .kv("pad_mode", ap.pad_mode).kv("pads", {o.pad_t, o.pad_l, o.pad_b, o.pad_r}).kv("parity", o.parity).kv("split", o.split)
      .kv("scale", scale).kv("act", ap.act).key("adds").arr();
  for (int a = 0; a < ap.n_add; ++a)
    j.obj().kv("parity", ap.add[a].parity).kv("split", ap.add[a].split).kv("C", ap.add[a].C).end();
  j.end().end();
}

// The "layout" records of v2v_plan_describe, in launch order: every import (caller tensor or correlation scratch), export,
// concat copy and the weight pack of every conv launch, with the fields that select its code path; training plans add their
// backward's layout launches (describe_backward_layout).
static void describe_layout(const v2v_plan* P, const std::vector<XOp>& xops, const std::vector<BwdUnit>& units, Json& j) {
  j.key("layout").arr();
  for (const XOp& x : xops) {
    switch (x.kind) {
      case X_IMPORT: describe_import(P, x, j); break;
      case X_CONV: describe_pack(P, x.gop, j); break;
      case X_EXPORT: describe_export(P, x, j); break;
      case X_COPY: describe_copy(x, j); break;
      default: break;
    }
  }
  if (P->train) describe_backward_layout(P, units, j);
  j.end();
}

// The "epilogue_forward" records of v2v_plan_describe: every stats record (in launch order), every finalize record (in the
// order of the passes they serve) and every apply record (in launch order).
static void describe_epilogue_forward(const v2v_plan* P, const std::vector<XOp>& xops, Json& j) {
  std::vector<FinRecord> fins;
  for (const XOp& x : xops) {
    if (x.kind == X_CONV) for (int q = 0; q < x.kp.n_fin; ++q) fins.push_back({x.fin_gop[q], q, &x.kp.fin[q]});
    if (x.kind == X_FINALIZE) fins.push_back({x.gop, 2, &x.fin});
  }
  std::sort(fins.begin(), fins.end(), [](const FinRecord& a, const FinRecord& b) { return a.gop < b.gop; });
  std::vector<std::vector<int>> sites(P->raws.size());      // per raw: the sites of its slices, as its stats record lists them
  for (const FinRecord& f : fins) sites[P->gops[f.gop].raw].push_back(f.site);
  j.key("epilogue_forward").arr();
  for (const XOp& x : xops) {
    if (x.kind != X_CONV || P->gops[x.gop].kind != G_CONV || sites[P->gops[x.gop].raw].empty()) continue;
    describe_stats(P, x, sites[P->gops[x.gop].raw], j);
  }
  for (const FinRecord& f : fins) describe_finalize(P, f, j);
  for (const XOp& x : xops) if (x.kind == X_APPLY) describe_apply(P, x, j);
  j.end();
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
  V2V_REQUIRE(!(on && p->sample_stats), V2V_ERR_STATE,
              "a per-sample-statistics plan cannot train: training normalises with the statistics of the whole batch");
  p->train = on != 0;
  return 0;
}

int v2v_plan_set_sample_stats(v2v_plan* p, int on) {
  V2V_REQUIRE(p && !p->lowered, V2V_ERR_STATE, "set per-sample statistics before the plan is lowered");
  V2V_REQUIRE(on || p->flags_slot < 0, V2V_ERR_STATE, "a plan with per-image flags keeps per-sample statistics");
  V2V_REQUIRE(!(on && p->train), V2V_ERR_STATE,
              "per-sample statistics are for inference plans: a training plan normalises with the statistics of the whole batch");
  p->sample_stats = on != 0;
  return 0;
}

int v2v_plan_set_image_flags(v2v_plan* p, int slot) {
  V2V_REQUIRE(p && !p->finalized, V2V_ERR_STATE, "set the image flags before finalize");
  V2V_REQUIRE(!p->train, V2V_ERR_STATE, "per-image flags are for inference plans: a training plan cannot skip images");
  V2V_REQUIRE(p->sample_stats, V2V_ERR_STATE,
              "per-image flags need a per-sample-statistics plan: batch statistics mix the images, so none can be skipped");
  V2V_REQUIRE(slot >= 0, V2V_ERR_INVALID, "bad flags slot %d", slot);
  p->flags_slot = slot;
  p->n_slots = std::max(p->n_slots, slot + 1);
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

int v2v_g_input(v2v_plan* p, int slot, int N, int C_src, int c_off, int C, int H, int W, int flags, int* value_out) {
  V2V_REQUIRE(p && !p->lowered && value_out, V2V_ERR_STATE, "plan already lowered or null");
  V2V_REQUIRE(slot >= 0 && N > 0 && C > 0 && c_off >= 0 && c_off + C <= C_src && H > 0 && W > 0, V2V_ERR_INVALID,
              "bad input description");
  GOp op; op.kind = G_INPUT; op.slot = slot; op.C_src = C_src; op.c_off = c_off;
  op.value_out = new_value(p, N, H, W, C);
  p->values[op.value_out].exact_bf16 = (flags & V2V_INPUT_EXACT_BF16) != 0;
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
  ConvGeom g; rc = conv_geometry(*c, p->values[value_in].Cp, 0, p->values[value_in].N, p->values[value_in].H, p->values[value_in].W, true, p->sp(), &g); if (rc) return rc;
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
  ConvGeom g; rc = conv_geometry(*c, p->values[value_in].Cp, 0, p->values[value_in].N, p->values[value_in].H, p->values[value_in].W, true, p->sp(), &g); if (rc) return rc;
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

static int finalize_impl(v2v_plan* P, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  V2V_REQUIRE(P && !P->finalized, V2V_ERR_STATE, "plan null or already finalized");
  int rc = size_arena(P); if (rc) return rc;
  DeviceGuard guard(P->device);
  // ---- allocate
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
  if (P->train) {                       // saved batch statistics (the finalize launches write them)
    size_t tot = 0;
    for (auto& r : P->raws) tot += 2 * (size_t)r.N * r.C;
    float* st = nullptr;
    V2V_CUDA(cudaMalloc(reinterpret_cast<void**>(&st), std::max<size_t>(tot, 1) * sizeof(float)));
    V2V_CUDA(cudaMemsetAsync(st, 0, std::max<size_t>(tot, 1) * sizeof(float), stream));
    P->train_stats = st;
    for (auto& r : P->raws) { r.mean = st; st += (size_t)r.N * r.C; r.rstd = st; st += (size_t)r.N * r.C; }
  }
  // ---- bind: the arena addresses of the buffers the launches and the backward read
  for (size_t i = 0; i < P->acts.size(); ++i) P->acts[i].base = arena_at<bf16>(P, P->act_off[i]);
  for (size_t i = 0; i < P->raws.size(); ++i) {
    Raw& r = P->raws[i];
    r.desc.base = arena_at<void>(P, P->raw_off[i].raw);
    r.stats = arena_at<stat_t>(P, P->raw_off[i].stats);
    r.scale = arena_at<float>(P, P->raw_off[i].scale);
    r.shift = arena_at<float>(P, P->raw_off[i].shift);
  }
  // ---- emit
  rc = emit_forward(P, P->xops); if (rc) return rc;
  // ---- device work: every conv launch's packed weights and tensor maps
  for (const XOp& x : P->xops) {
    if (x.kind != X_CONV) continue;
    GOp& op = P->gops[x.gop];
    op.wpacked = arena_at<bf16>(P, P->w_off[x.gop]);
    if (P->impl == V2V_IMPL_UMMA) {
      const ActDesc& ain = P->acts[P->values[op.value_in].bufs[op.req_index]];
      rc = make_tmap_act(&op.tmA, ain, x.kp.PW, x.kp.PH, x.kp.kc); if (rc) return rc;
      rc = make_tmap_w(&op.tmB, op.wpacked, P->sp() * op.Ktotal, op.geom.headkx ? op.geom.headkx * op.conv.Cout : op.conv.Cout,
                       x.kp.BN, x.kp.kc); if (rc) return rc;
    }
    rc = pack_one(op, stream); if (rc) return rc;
  }
  // a norm-less biased conv (FlowNet2's conv / deconv / predict_flow units) is normalised with scale 1 and shift = bias, written
  // here and after every repack
  for (const GOp& op : P->gops) {
    if (op.kind != G_NORM_ACT || op.norm.kind != V2V_NORM_NONE) continue;
    const Raw& r = P->raws[op.raw];
    const float* bias = P->gops[r.conv_op].conv.bias;
    if (bias) P->bias_affines.push_back(v2v_plan::BiasAffine{r.scale, r.shift, bias, r.N, r.C, r.C});
  }
  for (const auto& ba : P->bias_affines) V2V_CUDA(launch_bias_affine(ba.scale, ba.shift, ba.bias, ba.N, ba.C, ba.stride, stream));
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

// The vectorised composite moves its streamed slots as float4: refuse caller tensors that are not 16-byte aligned (a view
// at an odd float offset) on the host, before anything is launched.
static int check_composite_alignment(const v2v_plan* P, void* const* io_ptrs) {
  for (const XOp& x : P->xops)
    if (x.kind == X_COMPOSITE && composite_vec4(x.comp))
      V2V_REQUIRE(composite_slots_aligned(x.comp, io_ptrs), V2V_ERR_INVALID,
                  "composite (W %% 4 == 0) needs 16-byte aligned raw / final / flow / weight / fg / mask tensors");
  return 0;
}

// A launch without the running-statistics updates of its finalisations (stand-alone, or in a conv launch's tail).
static XOp without_running_stats(XOp x) {
  auto strip = [](FinalizeParams& f) { f.running_mean = nullptr; f.running_var = nullptr; f.num_batches_tracked = nullptr; };
  if (x.kind == X_FINALIZE) strip(x.fin);
  if (x.kind == X_CONV) for (int q = 0; q < x.kp.n_fin; ++q) strip(x.kp.fin[q]);
  return x;
}

int v2v_plan_run(v2v_plan* P, void* const* io_ptrs, int n_io, int use_graph, v2v_stream_t stream_) {
  V2V_REQUIRE(P && P->finalized, V2V_ERR_STATE, "plan not finalized");
  V2V_REQUIRE(n_io >= P->n_slots && io_ptrs, V2V_ERR_INVALID, "need %d io pointers, got %d", P->n_slots, n_io);
  if (int rc = check_composite_alignment(P, io_ptrs)) return rc;
  DeviceGuard guard(P->device);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  V2V_CUDA(cudaMemcpyAsync(P->io_dev, io_ptrs, sizeof(void*) * P->n_slots, cudaMemcpyHostToDevice, stream));
  if (use_graph & 2) {        // recomputation before a backward: same results, no running-statistics side effect
    for (const XOp& x : P->xops) { int rc = run_xop(P, without_running_stats(x), stream); if (rc) return rc; }
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
  if (int rc = check_composite_alignment(P, io_ptrs)) return rc;
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

extern "C" {

int64_t v2v_plan_describe(const v2v_plan* P_, char* buf, int64_t cap) {
  v2v_plan* P = const_cast<v2v_plan*>(P_);
  if (!P) return 0;
  if (!P->sized && size_arena(P)) return -1;          // lowers the graph and chooses every conv's kernel parameters
  std::vector<XOp> emitted;                           // an unfinalized plan: the launch list finalize would run
  if (!P->finalized && emit_forward(P, emitted)) return -1;
  const std::vector<XOp>& xops = P->finalized ? P->xops : emitted;
  // training plans: the backward unit of every live conv, as finalize built it, or as it would build it (the same host-only
  // choice; the sub-plans chosen here are destroyed on return)
  struct Chosen {
    std::vector<BwdUnit> units;
    ~Chosen() { for (BwdUnit& u : units) v2v_plan_destroy(u.child); }
  } chosen;
  if (P->train && !P->finalized && choose_backward_units(P, chosen.units)) return -1;
  const std::vector<BwdUnit>& units = P->finalized ? P->bwd : chosen.units;
  std::string s;
  Json j(s);
  j.obj().key("values").arr();
  for (size_t i = 0; i < P->values.size(); ++i) {
    const Value& v = P->values[i];
    j.obj().kv("id", i).kv("N", v.N).kv("C", v.C).kv("H", v.H).kv("W", v.W).key("layouts").arr();
    for (const Req& r : v.reqs)
      j.obj().kv("mode", r.mode).kv("pads", {r.pads[0], r.pads[1], r.pads[2], r.pads[3]}).kv("parity", r.parity).end();
    j.end().end();
  }
  j.end().key("convs").arr();
  for (const GOp& op : P->gops)
    if (op.kind == G_CONV || op.kind == G_CONV_ACT || op.kind == G_HEAD) describe_conv(P, op, j);
  j.end();
  if (P->train) {
    j.key("backward").arr();
    for (const BwdUnit& u : units) describe_backward_unit(u, j);
    j.end();
    describe_epilogue_backward(P, j);
  }
  describe_epilogue_forward(P, xops, j);
  describe_buffers(P, j);
  describe_layout(P, xops, units, j);
  // ops the backward visits (0 for the forward-only branch of a feature L1 target) and values without a gradient buffer
  int bwd_ops = 0, detached = 0;
  for (char l : P->op_live) bwd_ops += l;
  for (const Value& v : P->values) detached += v.detached;
  j.kv("conv_macs", P->conv_macs).kv("n_slots", P->n_slots).kv("ops", P->gops.size()).kv("backward_ops", bwd_ops)
      .kv("detached_values", detached).kv("sample_stats", P->sample_stats).kv("image_flags", P->flags_slot >= 0).end();
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
  int rc = conv_geometry(*conv, pad_channels(conv->Cin), 0, 1, H, W, allow_reuse != 0, 1, &g);
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
