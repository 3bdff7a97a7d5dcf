// Conv lowering: the geometry of one convolution (tap groups, sub-pixel phases, 2-D patches, kx-GEMM heads), the
// conv_umma_kernel tiling chosen for it and every kernel parameter derived from that choice, its TMA tensor maps, the weight
// packing launch and the describe record of the choice.  All of it but the two tensor maps and pack_one runs without a device.
#include <algorithm>
#include <cstdio>
#include <cstring>

#include "plan_internal.h"

namespace v2v {

const int kSmemBudget = 188 * 1024;             // operand slots + resident weights (227 KB - 36.5 KB epilogue staging - alignment - barriers)
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
// sp = 2 for precise plans: every operand slot holds a hi and a lo half, so all byte counts double.  Cp: padded input channels.
static bool choose_patch2d(const v2v_conv_desc& c, int Cp, bool head, int N, int grid_h, int grid_w, int sp, int* kc_out, int* bn_out) {
  if (c.transposed || c.stride != 1 || c.kh * c.kw == 1 || grid_w < 8) return false;
  const long long tiles = (long long)((grid_w + 7) / 8) * ((grid_h + 15) / 16);
  if (tiles * 128 * 4 > (long long)grid_h * grid_w * 5) return false;          // > 25 % masked rows: keep row tiles
  const int taps = c.kh * c.kw, patch_px = (16 + c.kh - 1) * (8 + c.kw - 1);
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

// Cp: padded input channels (Value::Cp); head: 0 = no, 1 = small-Cout head, 2 = head that may use the kx-GEMM form (tensor-core
// implementation only)
int conv_geometry(const v2v_conv_desc& c, int Cp, int head, int N, int H, int W, bool allow_reuse, int sp, ConvGeom* g) {
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
  } else if (allow_reuse && choose_patch2d(c, Cp, head != 0, N, g->grid_h, g->grid_w, sp, &g->patch2d_kc, &g->patch2d_bn)) {
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

int make_tmap_act(CUtensorMap* tm, const ActDesc& a, int box_w, int box_h, int kc) {
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

int make_tmap_w(CUtensorMap* tm, bf16* w, int Ktotal /* columns, both halves */, int Cout, int BN, int kc) {
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
  const int m_tiles = P->tiling_n(kp.N) * kp.tiles_x * kp.tiles_y;
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

void fill_conv_params(v2v_plan* P, GOp& op) {
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
  kp.Cp = vin.Cp;
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
  if (op.kind == G_HEAD) {          // each channel's destination in its IO slot (the head backward reads the same offsets)
    kp.epi = EPI_HEAD_F32;
    kp.bias2 = c.Cout2 > 0 ? c.bias2 : nullptr; kp.Cout1 = c.Cout - c.Cout2;
    for (int j = 0; j < c.Cout; ++j) {
      kp.head_slot[j] = op.head[j].slot;
      kp.head_off[j] = (long long)op.head[j].channel * g.out_h * g.out_w;
      kp.head_bstride[j] = (long long)op.head[j].dst_C * g.out_h * g.out_w;
      kp.head_act[j] = op.head[j].act; kp.head_scale[j] = op.head[j].scale;
    }
  }
  op.Cp = kp.Cp; op.Ktotal = (g.headkx ? c.kh : c.kh * c.kw) * kp.Cp;
  kp.Khalf = op.Ktotal;
}

// The packing of a lowered conv op's weights (out: op.wpacked, null before finalize)
PackParams pack_params(const GOp& op) {
  PackParams pp{};
  pp.w = op.conv.weight; pp.transposed = op.conv.transposed;
  pp.w2 = op.conv.Cout2 > 0 ? op.conv.weight2 : nullptr; pp.Cout1 = op.conv.Cout - op.conv.Cout2;
  pp.Cout = op.conv.Cout; pp.Cin = op.conv.Cin; pp.kh = op.conv.kh; pp.kw = op.conv.kw;
  pp.Cp = op.Cp; pp.ntaps = op.geom.headkx ? op.conv.kh : op.conv.kh * op.conv.kw; pp.split = op.kp.split; pp.headkx = op.geom.headkx;
  for (int ky = 0; ky < op.conv.kh; ++ky)
    for (int kx = 0; kx < op.conv.kw; ++kx) { pp.tap_ky[ky * op.conv.kw + kx] = (int8_t)ky; pp.tap_kx[ky * op.conv.kw + kx] = (int8_t)kx; }
  pp.out = op.wpacked;
  if (op.pack_dgrad) { pp.dgrad = 1; pp.w2 = op.dg_w2; pp.Cout1 = op.dg_Cout1; }
  return pp;
}

int pack_one(const GOp& op, cudaStream_t stream) {
  V2V_CUDA(launch_pack_weights(pack_params(op), stream));
  return 0;
}

// One "pack" layout record: the packed matrix [rows][split + 1][Ktotal] at arena offset w_off and the path that writes it
// (TC of the tiled kernel, 0 for the elementwise one).  Needs the op lowered and the arena sized.
void describe_pack(const v2v_plan* P, size_t i, Json& j) {
  const GOp& op = P->gops[i];
  const PackParams pp = pack_params(op);
  j.obj().kv("kind", "pack").kv("gop", i).kv("w_off", P->w_off[i]).kv("rows", pp.headkx ? pp.headkx * pp.Cout : pp.Cout)
      .kv("Ktotal", op.Ktotal).kv("Cout", pp.Cout).kv("Cin", pp.Cin).kv("k", {pp.kh, pp.kw}).kv("ntaps", pp.ntaps).kv("Cp", pp.Cp)
      .kv("split", pp.split).kv("transposed", pp.transposed).kv("headkx", pp.headkx).kv("dgrad", pp.dgrad)
      .kv("w2", pp.w2 != nullptr).kv("Cout1", pp.Cout1).kv("TC", pack_weights_tiling(pp)).end();
}

// One conv record of v2v_plan_describe: the conv, its geometry and the kernel configuration fill_conv_params chose (needs the
// arena sized).
void describe_conv(const v2v_plan* P, const GOp& op, Json& j) {
  const ConvGeom& g = op.geom;
  const ConvKernelParams& kp = op.kp;
  // EG: epilogue groups per tile, always 1 (one 256-thread epilogue stores every tile; async_epi: which threads run it)
  j.obj().kv("kind", (int)op.kind).kv("Cin", op.conv.Cin).kv("Cout", op.conv.Cout).kv("k", {op.conv.kh, op.conv.kw})
      .kv("stride", op.conv.stride).kv("transposed", op.conv.transposed).kv("in", op.value_in).kv("TH", g.TH).kv("TW", g.TW)
      .kv("R", g.R).kv("groups", g.n_groups).kv("phases", g.n_phases).kv("grid", {g.grid_h, g.grid_w}).kv("out", {g.out_h, g.out_w})
      .kv("BN", kp.BN).kv("kc", kp.kc).kv("MG", kp.MG).kv("CG", kp.CG).kv("SG", kp.SG).kv("resident", kp.b_resident).kv("EG", 1)
      .kv("units", kp.total_units).kv("split", kp.split).kv("ring2", kp.ring2).kv("TB", kp.TB).kv("SBr", kp.SBr)
      .kv("p2d", g.patch2d_kc > 0).kv("a_exact", kp.a_exact).kv("headkx", kp.headkx).kv("grad", (int)P->op_live[&op - P->gops.data()]);
  // the derived launch parameters the kernel reads (ctas: persistent CTAs launched; smem: dynamic shared memory)
  j.kv("tiles_x", kp.tiles_x).kv("tiles_y", kp.tiles_y).kv("tile_dx", kp.tile_dx).kv("Cp", kp.Cp).kv("cblocks", kp.cblocks)
      .kv("row_bytes", kp.row_bytes).kv("kmma", kp.kmma).kv("kmma_last", kp.kmma_last).kv("BNt", kp.BNt)
      .kv("layout_type", kp.layout_type).kv("sbo_bytes", kp.sbo_bytes).kv("sbo_a_bytes", kp.sbo_a_bytes).kv("RW", kp.RW)
      .kv("PW", kp.PW).kv("PH", kp.PH).kv("a_half_bytes", kp.a_half_bytes).kv("a_slot_bytes", kp.a_slot_bytes)
      .kv("b_half_bytes", kp.b_half_bytes).kv("b_slot_bytes", kp.b_slot_bytes).kv("SB", kp.SB).kv("n_tiles", kp.n_tiles)
      .kv("m_total", kp.m_total).kv("ctas", kp.grid).kv("Khalf", kp.Khalf).kv("smem", conv_umma_smem_bytes(kp))
      .kv("async_epi", conv_umma_async_epilogue(kp)).end();
}

}  // namespace v2v
