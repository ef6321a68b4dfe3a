// Model-level C ABI (include/acnn_model.h): handle = layer plan (model_plan.cu) + launch records resolved
// against the caller's device buffers.  Every launch record is a closure over raw pointers and integers
// that calls one op-level entry point of this library (include/acnn.h); running a phase is a loop over
// its records -- no lookups, no allocation, nothing but kernel launches on the given stream.
#include <string.h>

#include <memory>

#include "common.h"
#include "model_plan.h"

using namespace acnn;
using namespace acnn::model;

struct acnn_model {
  Plan plan;
  // bound device buffers (caller-owned)
  float *params = nullptr, *grads = nullptr, *momentum = nullptr, *state = nullptr;
  char *w_fprop = nullptr, *w_dgrad = nullptr, *ws = nullptr;
  bool bound = false;
  // workspace layout (bytes)
  int64_t hp_off = 0, descs_off = 0, flags_off = 0, zero_off = 0, work_off = 0, ws_bytes = 0;
  int n_descs = 0;
  // settings read at enqueue time
  double loss_scale = 1.0;
  uint64_t dropblock_seed = 0x5EED5EEDull;
  int dropblock_feed = 0;
  int det = 0, planes = 1, adt = ACNN_BF16;
  // host images of the one-time initialisation (kept alive: cudaMemcpyAsync sources)
  std::vector<acnn_weight_desc> descs;
  std::vector<uint8_t> flags;
  std::vector<float> ones;   // max C of the identity-BN scale vectors
  float hp_init[8] = {0.1f, 0.9f, 0.0f, 1.0f, 1.0f, 0.0f, 0.0f, 0.0f};
  using Launch = std::function<int(void*)>;
  std::vector<Launch> fwd, bwd, upd;
};

namespace {

constexpr int64_t kWsAlign = 1024;
int64_t ws_round(int64_t b) { return (std::max<int64_t>(b, 256) + kWsAlign - 1) / kWsAlign * kWsAlign; }

void layout(acnn_model* m) {
  Plan& p = m->plan;
  m->planes = p.cfg.fp32 ? 3 : 1;
  m->adt = p.cfg.fp32 ? ACNN_F32 : ACNN_BF16;
  m->det = p.cfg.deterministic < 0 ? (p.cfg.fp32 ? 1 : 0) : (p.cfg.deterministic ? 1 : 0);
  m->loss_scale = p.cfg.loss_scale;
  // weight descriptor table + weight-decay flags (one byte per 256 elements)
  m->flags.assign(std::max<int64_t>(p.param_elems / 256, 1), 0);
  for (const auto& v : p.vars) {
    if (v.buffer != ACNN_BUF_PARAMS) continue;
    if (v.decay)
      for (int64_t i = v.offset / 256; i < (v.offset + v.size + 255) / 256; ++i) m->flags[i] = 1;
    if ((v.kind == "conv_kernel" || v.kind == "dense_kernel") && v.store_shape.size() == 4 &&
        v.store_shape[3] % 16 == 0 && v.store_shape[0] % 32 == 0) {
      acnn_weight_desc d{};
      d.master_off = d.fprop_off = v.offset;
      d.dgrad_off = v.dgrad_off;
      d.Cout = (int)v.store_shape[0];
      d.taps = (int)(v.store_shape[1] * v.store_shape[2]);
      d.Cin = (int)v.store_shape[3];
      m->descs.push_back(d);
    }
  }
  m->n_descs = (int)m->descs.size();
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = off;
    off += ws_round(bytes);
    return o;
  };
  m->hp_off = take(8 * 4);
  m->descs_off = take((int64_t)m->descs.size() * sizeof(acnn_weight_desc));
  m->flags_off = take((int64_t)m->flags.size());
  m->zero_off = take(p.zero_elems * 4);
  m->work_off = take(p.work_elems * 4);
  for (auto& t : p.tensors) t.ws_offset = take(t.bytes());
  m->ws_bytes = off;
}

// ---- op -> launch record ----------------------------------------------------------------------------
struct Resolver {
  acnn_model* m;
  const Op& op;
  const Plan& p;
  Resolver(acnn_model* m_, const Op& op_) : m(m_), op(op_), p(m_->plan) {}

  int64_t I(const char* k, int64_t dflt = 0) const {
    const Val* v = op.find(k);
    return v ? v->i : dflt;
  }
  double F(const char* k, double dflt = 0) const {
    const Val* v = op.find(k);
    return v ? (v->kind == Val::FLT ? v->f : (double)v->i) : dflt;
  }
  bool has(const char* k) const { return op.find(k) != nullptr; }
  void* Tn(const char* k) const {   // tensor pointer (NULL when absent)
    const Val* v = op.find(k);
    return (v && v->kind == Val::TENSOR) ? m->ws + p.tensors[v->i].ws_offset : nullptr;
  }
  int64_t Tnumel(const char* k) const { return numel(p.tensors[op.find(k)->i].shape); }
  const Variable& var(const char* k) const { return p.vars[op.find(k)->i]; }
  float* base_of(const Variable& v) const { return v.buffer == ACNN_BUF_PARAMS ? m->params : m->state; }
  float* P(const char* k) const {   // variable in the fp32 master / state buffer
    const Val* v = op.find(k);
    return (v && v->kind == Val::VAR) ? base_of(p.vars[v->i]) + p.vars[v->i].offset : nullptr;
  }
  float* Pv(int id) const { return id >= 0 ? base_of(p.vars[id]) + p.vars[id].offset : nullptr; }
  float* Gv(int id) const { return (id >= 0 && m->grads) ? m->grads + p.vars[id].offset : nullptr; }
  float* G(const char* k) const {
    const Val* v = op.find(k);
    return (v && v->kind == Val::VAR) ? Gv((int)v->i) : nullptr;
  }
  char* WF(const char* k) const { return m->w_fprop + 2 * var(k).offset; }
  char* WD(const char* k) const { return m->w_dgrad + 2 * var(k).dgrad_off; }
  float* S(const Slot& s, int64_t extra = 0) const {
    if (s.buf == BUF_NONE) return nullptr;
    return reinterpret_cast<float*>(m->ws + (s.buf == BUF_ZERO ? m->zero_off : m->work_off)) + s.offset + extra;
  }
  float* S(const char* k, int64_t extra = 0) const {
    const Val* v = op.find(k);
    return v ? S(v->slot, extra) : nullptr;
  }
  Slot slot(const char* k) const {
    const Val* v = op.find(k);
    return v ? v->slot : Slot();
  }
  const BatchNorm& bn(const char* k) const { return p.bns[op.find(k)->i]; }
  // ConvGeom for the op level.  With x_wpad = (lo, hi) the input is the W-padded space-to-depth image:
  // the k2 horizontal taps become channels of one wide pixel (x_pix_stride < Cin)
  acnn_conv_geom geom() const {
    const Geom& g = op.find("geom")->g;
    acnn_conv_geom c{};
    const Val* wp = op.find("x_wpad");
    if (!wp) {
      c.B = g.B; c.H = g.H; c.W = g.W; c.Cin = g.Cin; c.Cout = g.Cout; c.kh = g.kh; c.kw = g.kw;
      c.stride = g.stride; c.pad_h_lo = g.pad_h_lo; c.pad_h_hi = g.pad_h_hi; c.pad_w_lo = g.pad_w_lo;
      c.pad_w_hi = g.pad_w_hi;
    } else {
      const int lo = (int)wp->v[0], hi = (int)wp->v[1];
      const int row = (g.W + lo + hi) * g.Cin;
      c.B = g.B; c.H = g.H; c.W = g.W; c.Cin = g.Cin * g.kw; c.Cout = g.Cout; c.kh = g.kh; c.kw = 1;
      c.stride = 1; c.pad_h_lo = g.pad_h_lo; c.pad_h_hi = g.pad_h_hi;
      c.x_pix_stride = g.Cin; c.x_row_pitch = row; c.x_img_pitch = g.H * row;
    }
    return c;
  }
};

#define REQUIRE_BIND(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      set_error(__VA_ARGS__);            \
      return acnn_model::Launch();       \
    }                                    \
  } while (0)

acnn_model::Launch resolve(acnn_model* m, const Op& op) {
  const Resolver r(m, op);
  const Plan& p = m->plan;
  const std::string& k = op.kind;
  const int adt = m->adt, det = m->det, training = p.cfg.training ? 1 : 0;
  const bool fp32 = p.cfg.fp32;
  const float bn_mom = (float)p.cfg.bn_momentum, eps = (float)p.cfg.bn_epsilon;
  float* hp = reinterpret_cast<float*>(m->ws + m->hp_off);

  if (k == "prep_weights") {
    if (!m->n_descs) return [](void*) { return ACNN_OK; };
    float* master = m->params;
    auto* descs = reinterpret_cast<acnn_weight_desc*>(m->ws + m->descs_off);
    const int n = m->n_descs, planes = m->planes;
    void *wf = m->w_fprop, *wd = m->w_dgrad;
    const int64_t fs = p.param_elems, ds = std::max<int64_t>(p.dgrad_elems, 1);
    return [=](void* st) { return acnn_prep_weights(master, descs, n, wf, wd, planes, fs, ds, st); };
  }
  if (k == "split3") {
    void *src = r.Tn("src"), *dst = r.Tn("dst");
    const int64_t n = r.I("n");
    return [=](void* st) { return acnn_split3((const float*)src, dst, n, st); };
  }
  if (k == "pack_input") {
    void *img = r.Tn("images"), *l1 = r.Tn("lam1"), *l2 = r.Tn("lam2"), *out = r.Tn("out");
    const int mode = (int)r.I("mode"), Bin = (int)r.I("Bin"), H = (int)r.I("H"), W = (int)r.I("W");
    const int lo = (int)op.find("wpad")->v[0], hi = (int)op.find("wpad")->v[1];
    return [=](void* st) {
      return acnn_pack_input((const float*)img, (const float*)l1, (const float*)l2, mode, out, Bin, H, W, lo,
                             hi, adt, st);
    };
  }
  if (k == "mix_labels") {
    void *lab = r.Tn("labels"), *l1 = r.Tn("lam1"), *l2 = r.Tn("lam2"), *y = r.Tn("y");
    const int mode = (int)r.I("mode"), Bin = (int)r.I("Bin"), NC = (int)r.I("NC");
    return [=](void* st) {
      return acnn_mix_labels((const int32_t*)lab, (const float*)l1, (const float*)l2, mode, (float*)y, Bin,
                             NC, st);
    };
  }
  if (k == "s2d_weight_pack") {
    float* w = r.P("w");
    void* w2 = r.Tn("w2");
    const int cout = (int)r.I("cout"), kk = (int)r.I("k"), pad = (int)r.I("pad"), k2 = (int)r.I("k2"),
              pad2 = (int)r.I("pad2");
    return [=](void* st) { return acnn_s2d_weight_pack(w, w2, cout, kk, pad, k2, pad2, adt, st); };
  }
  if (k == "conv") {
    const bool is_t = r.has("w_is_tensor");
    const acnn_conv_geom g = r.geom();
    void *x, *w;
    int64_t wstride = 0;
    if (fp32) {
      x = r.Tn("xp");
      w = is_t ? r.Tn("wp") : (void*)r.WF("w");
      wstride = is_t ? r.Tnumel("wp") / 3 : p.param_elems;
    } else {
      x = r.Tn("x");
      w = is_t ? r.Tn("w") : (void*)r.WF("w");
    }
    const Slot stats = r.slot("stats");
    if (stats.buf != BUF_NONE) {
      const int n = acnn_conv_stats_parts(&g);
      REQUIRE_BIND(n >= 1 && (int64_t)n * 2 * g.Cout <= stats.size,
                   "conv statistics: %d partial rows do not fit the plan's slot (%lld floats)", n,
                   (long long)stats.size);
    }
    void* y = r.Tn("y");
    float* st_p = r.S(stats);
    float* bias = r.P("bias");
    const int out_f32 = (r.I("out_f32") || fp32) ? 1 : 0;
    return [=](void* st) {
      return acnn_conv_fprop(&g, x, w, y, st_p, nullptr, nullptr, bias, out_f32, adt, wstride, st);
    };
  }
  if (k == "bn_stats") {
    void* x = r.Tn("x");
    float* s = r.S(r.bn("bn").stats);
    const int64_t M = r.I("M");
    const int C = (int)r.I("C");
    return [=](void* st) { return acnn_bn_stats(x, s, M, C, adt, st); };
  }
  if (k == "bn_finalize") {
    const BatchNorm& bn = r.bn("bn");
    const int C = bn.C, mode = (int)r.I("stats_mode");
    int nparts = 1;
    if (training && mode == 0) {
      const acnn_conv_geom g = r.geom();
      nparts = acnn_conv_stats_parts(&g);
      REQUIRE_BIND(nparts >= 1, "acnn_conv_stats_parts failed");
    }
    float *stats = r.S(bn.stats), *gamma = r.Pv(bn.gamma), *beta = r.Pv(bn.beta), *mm = r.Pv(bn.mm),
          *mv = r.Pv(bn.mv), *w0 = r.S(bn.work), *w1 = r.S(bn.work, C), *w2 = r.S(bn.work, 2 * C),
          *w3 = r.S(bn.work, 3 * C);
    const int64_t count = bn.count;
    return [=](void* st) {
      return acnn_bn_finalize(stats, nparts, mode, count, gamma, beta, mm, mv, bn_mom, eps, training, w0, w1,
                              w2, w3, C, st);
    };
  }
  if (k == "bn_act") {
    const auto& sh = op.find("shape")->v;
    const int B = (int)sh[0], H = (int)sh[1], W = (int)sh[2], C = (int)sh[3];
    const BatchNorm& a = r.bn("bn_a");
    const BatchNorm* b = r.has("bn_b") ? &r.bn("bn_b") : nullptr;
    void *at = r.Tn("a"), *bt = r.Tn("b"), *out = r.Tn("out");
    float *sa = r.S(a.work), *ha = r.S(a.work, C), *sb = b ? r.S(b->work) : nullptr,
          *hb = b ? r.S(b->work, C) : nullptr, *gate = r.S("gate");
    const int b_mode = (int)r.I("b_mode"), relu = (int)r.I("relu");
    return [=](void* st) {
      return acnn_bn_act(at, sa, ha, bt, sb, hb, b_mode, gate, relu, out, B, H, W, C, adt, st);
    };
  }
  if (k == "sk_gap" || k == "sk_combine" || k == "sk_bwd_gate") {
    const BatchNorm& bn = r.bn("bn");
    void* y = r.Tn("y");
    float *sc = r.S(bn.work), *sh = r.S(bn.work, bn.C);
    const int B = (int)r.I("B"), HW = (int)r.I("HW"), f = (int)r.I("f");
    if (k == "sk_gap") {
      float* s = r.S("s");
      return [=](void* st) { return acnn_sk_gap(y, sc, sh, s, B, HW, f, adt, st); };
    }
    if (k == "sk_combine") {
      float* att = r.S("att");
      void* v = r.Tn("v");
      return [=](void* st) { return acnn_sk_combine(y, sc, sh, att, v, B, HW, f, adt, st); };
    }
    void* dv = r.Tn("dv");
    float* dA = r.S("dA");
    return [=](void* st) { return acnn_sk_bwd_gate(dv, y, sc, sh, dA, B, HW, f, adt, st); };
  }
  if (k == "sk_fc" || k == "sk_fc_bwd") {
    const BatchNorm& bn = r.bn("bn");
    const int B = (int)r.I("B"), f = (int)r.I("f"), d = (int)r.I("d");
    REQUIRE_BIND(r.slot("scratch").size >= acnn_sk_fc_scratch_floats(B, f, d), "sk_fc scratch too small");
    float *s = r.S("s"), *w1 = r.P("w1"), *w2 = r.P("w2"), *gamma = r.Pv(bn.gamma), *beta = r.Pv(bn.beta),
          *mm = r.Pv(bn.mm), *mv = r.Pv(bn.mv), *zpre = r.S("zpre"), *bw = r.S(bn.work), *z = r.S("z"),
          *att = r.S("att"), *scratch = r.S("scratch");
    if (k == "sk_fc")
      return [=](void* st) {
        return acnn_sk_fc_fwd(s, w1, gamma, beta, mm, mv, bn_mom, eps, training, w2, zpre, bw, z, att,
                              scratch, B, f, d, det, st);
      };
    float *dA = r.S("dA"), *ds = r.S("ds"), *dw1 = r.G("w1"), *dw2 = r.G("w2"), *dg = r.Gv(bn.gamma),
          *db = r.Gv(bn.beta);
    return [=](void* st) {
      return acnn_sk_fc_bwd(dA, att, z, zpre, bw, gamma, s, w1, w2, dw1, dw2, dg, db, ds, scratch, B, f, d,
                            det, st);
    };
  }
  if (k == "se_gap" || k == "se_bwd_gate") {
    const BatchNorm& bn = r.bn("bn");
    void* y = r.Tn("y");
    float *sc = r.S(bn.work), *sh = r.S(bn.work, bn.C);
    const int B = (int)r.I("B"), HW = (int)r.I("HW"), C = (int)r.I("C");
    if (k == "se_gap") {
      float* q = r.S("q");
      return [=](void* st) { return acnn_se_gap(y, sc, sh, q, B, HW, C, adt, st); };
    }
    void* g = r.Tn("g");
    float* de = r.S("de");
    return [=](void* st) { return acnn_se_bwd_gate(g, y, sc, sh, de, B, HW, C, adt, st); };
  }
  if (k == "se_fc") {
    float *q = r.S("q"), *w1 = r.P("w1"), *w2 = r.P("w2"), *h = r.S("h"), *e = r.S("e");
    const int B = (int)r.I("B"), C = (int)r.I("C"), rr = (int)r.I("r");
    return [=](void* st) { return acnn_se_fc_fwd(q, w1, w2, h, e, B, C, rr, det, st); };
  }
  if (k == "se_fc_bwd") {
    float *de = r.S("de"), *e = r.S("e"), *h = r.S("h"), *q = r.S("q"), *w1 = r.P("w1"), *w2 = r.P("w2"),
          *dw1 = r.G("w1"), *dw2 = r.G("w2"), *dq = r.S("dq"), *scratch = r.S("scratch");
    const int B = (int)r.I("B"), C = (int)r.I("C"), rr = (int)r.I("r"), HW = (int)r.I("HW");
    return [=](void* st) {
      return acnn_se_fc_bwd(de, e, h, q, w1, w2, dw1, dw2, dq, scratch, B, C, rr, HW, det, st);
    };
  }
  if (k == "blurpool" || k == "blurpool_bwd") {
    const int B = (int)r.I("B"), H = (int)r.I("H"), W = (int)r.I("W"), C = (int)r.I("C"),
              filt = (int)r.I("filt"), stride = (int)r.I("stride");
    if (k == "blurpool") {
      void *x = r.Tn("x"), *out = r.Tn("out");
      return [=](void* st) { return acnn_blurpool_fwd(x, out, B, H, W, C, filt, stride, adt, st); };
    }
    void *dout = r.Tn("dout"), *dx = r.Tn("dx"), *add = r.Tn("add_src"), *mask = r.Tn("mask_src");
    return [=](void* st) { return acnn_blurpool_bwd(dout, dx, add, mask, B, H, W, C, filt, stride, adt, st); };
  }
  if (k == "avgpool" || k == "avgpool_bwd" || k == "maxpool" || k == "maxpool_bwd") {
    const int B = (int)r.I("B"), H = (int)r.I("H"), W = (int)r.I("W"), C = (int)r.I("C"), kk = (int)r.I("k"),
              stride = (int)r.I("stride"), pad_lo = (int)r.I("pad_lo"), Ho = (int)r.I("Ho"),
              Wo = (int)r.I("Wo"), count_pad = (int)r.I("count_pad");
    void *x = r.Tn("x"), *out = r.Tn("out"), *dout = r.Tn("dout"), *dx = r.Tn("dx"), *add = r.Tn("add_src"),
         *mask = r.Tn("mask_src");
    if (k == "avgpool")
      return [=](void* st) {
        return acnn_avgpool_fwd(x, out, B, H, W, C, kk, stride, pad_lo, Ho, Wo, count_pad, adt, st);
      };
    if (k == "avgpool_bwd")
      return [=](void* st) {
        return acnn_avgpool_bwd(dout, dx, add, mask, B, H, W, C, kk, stride, pad_lo, Ho, Wo, count_pad, adt, st);
      };
    if (k == "maxpool")
      return [=](void* st) { return acnn_maxpool_fwd(x, out, B, H, W, C, kk, stride, pad_lo, Ho, Wo, adt, st); };
    return [=](void* st) {
      return acnn_maxpool_bwd(dout, x, dx, add, mask, B, H, W, C, kk, stride, pad_lo, Ho, Wo, adt, st);
    };
  }
  if (k == "gem" || k == "gem_bwd" || k == "gap" || k == "gap_bwd") {
    const int B = (int)r.I("B"), HW = (int)r.I("HW"), C = (int)r.I("C");
    void *x = r.Tn("x"), *out = r.Tn("out"), *dp = r.Tn("dpooled"), *dx = r.Tn("dx"), *mask = r.Tn("mask_src");
    float* ssum = r.S("ssum");
    if (k == "gem") return [=](void* st) { return acnn_gem_fwd(x, out, ssum, B, HW, C, adt, st); };
    if (k == "gem_bwd") return [=](void* st) { return acnn_gem_bwd(dp, ssum, x, dx, B, HW, C, adt, st); };
    if (k == "gap") return [=](void* st) { return acnn_gap_fwd(x, out, B, HW, C, adt, st); };
    return [=](void* st) { return acnn_gap_bwd(dp, mask, dx, B, HW, C, adt, st); };
  }
  if (k == "dropblock_mask") {
    const int H = (int)r.I("H"), W = (int)r.I("W"), C = (int)r.I("C"), bs = (int)r.I("block_size");
    const int need = acnn_dropblock_scratch_floats(H, W, C, bs);
    REQUIRE_BIND(need > 0 && need <= r.slot("scratch").size, "dropblock scratch too small");
    float* u = (float*)r.Tn("u");
    float *keep = r.S("keep"), *scale = r.S("scale"), *scratch = r.S("scratch");
    const float gamma_scale = (float)r.F("gamma_scale");
    const uint64_t index = (uint64_t)r.I("index");
    return [=](void* st) {
      // one Philox key per call site: the masks of different layers are independent
      const uint64_t seed = m->dropblock_seed + 0x9E3779B97F4A7C15ull * (index + 1);
      return acnn_dropblock_mask(m->dropblock_feed ? u : nullptr, hp + 4, reinterpret_cast<uint32_t*>(hp + 5),
                                 seed, gamma_scale, bs, keep, scale, scratch, H, W, C, st);
    };
  }
  if (k == "dropblock_apply") {
    void *x = r.Tn("x"), *out = r.Tn("out");
    float *keep = r.S("keep"), *scale = r.S("scale");
    const int relu = (int)r.I("relu"), B = (int)r.I("B"), HW = (int)r.I("HW"), C = (int)r.I("C");
    return [=](void* st) { return acnn_dropblock_apply(x, keep, scale, relu, out, B, HW, C, adt, st); };
  }
  if (k == "kd_teacher") {
    void *tl = r.Tn("teacher_logits"), *lab = r.Tn("labels"), *l1 = r.Tn("lam1"), *l2 = r.Tn("lam2"),
         *yt = r.Tn("yt");
    const int mode = (int)r.I("mode"), Bin = (int)r.I("Bin"), NC = (int)r.I("NC");
    const float T = (float)r.F("kd_temp");
    return [=](void* st) {
      return acnn_kd_teacher_labels((const float*)tl, (const int32_t*)lab, (const float*)l1, (const float*)l2,
                                    mode, T, (float*)yt, Bin, NC, st);
    };
  }
  if (k == "softmax_ce") {
    void *logits = r.Tn("logits"), *y = r.Tn("y"), *yt = r.Tn("yt"), *dl = r.Tn("dlogits");
    const float T = (float)r.F("kd_temp"), ls = (float)r.F("label_smoothing");
    const int B = (int)r.I("B"), NC = (int)r.I("NC"), ld = (int)r.I("ld");
    float *loss = r.S("loss"), *dbias = r.G("dbias"), *work = r.S("work");
    return [=](void* st) {
      return acnn_softmax_ce((const float*)logits, (const float*)y, (const float*)yt, T, B, NC, ld, ls,
                             (float)m->loss_scale, loss, dl, dbias, work, adt, st);
    };
  }
  if (k == "conv_wgrad") {
    const acnn_conv_geom g = r.geom();
    float* dw = r.has("dw_slot") ? r.S("dw_slot") : r.G("w");
    void *x = fp32 ? r.Tn("xp") : r.Tn("x"), *dy = fp32 ? r.Tn("dyp") : r.Tn("dy");
    REQUIRE_BIND(dw, "conv_wgrad without a gradient buffer (bind grads)");
    return [=](void* st) { return acnn_conv_wgrad(&g, x, dy, dw, adt, det, st); };
  }
  if (k == "conv_dgrad") {
    const acnn_conv_geom g = r.geom();
    void *dy = fp32 ? r.Tn("dyp") : r.Tn("dy"), *dx = r.Tn("dx"), *add = r.Tn("add_src"),
         *mask = r.Tn("mask_src");
    REQUIRE_BIND(m->w_dgrad && r.var("w").dgrad_off >= 0, "conv_dgrad without dgrad-layout weights");
    void* w = r.WD("w");
    const int64_t ds = std::max<int64_t>(p.dgrad_elems, 1);
    return [=](void* st) { return acnn_conv_dgrad(&g, dy, w, dx, add, mask, adt, ds, st); };
  }
  if (k == "zero_insert") {
    void *dy = r.Tn("dy"), *out = r.Tn("out");
    const int B = (int)r.I("B"), Ho = (int)r.I("Ho"), Wo = (int)r.I("Wo"), H = (int)r.I("H"),
              W = (int)r.I("W"), C = (int)r.I("C");
    return [=](void* st) { return acnn_zero_insert2x(dy, out, B, Ho, Wo, H, W, C, adt, st); };
  }
  if (k == "s2d_wgrad_unpack") {
    float *dw2 = r.S("dw2"), *dw = r.G("w");
    const int cout = (int)r.I("cout"), kk = (int)r.I("k"), pad = (int)r.I("pad"), k2 = (int)r.I("k2"),
              pad2 = (int)r.I("pad2");
    return [=](void* st) { return acnn_s2d_wgrad_unpack(dw2, dw, cout, kk, pad, k2, pad2, st); };
  }
  if (k == "bn_bwd_reduce" || k == "bn_bwd_apply") {
    const auto& sh = op.find("shape")->v;
    const int B = (int)sh[0], HW = (int)(sh[1] * sh[2]), C = (int)sh[3];
    void *g = r.Tn("g"), *y = r.Tn("y");
    float *gate = r.S("gate"), *addbc = r.S("addbc");
    if (k == "bn_bwd_reduce") {
      const BatchNorm& bn = r.bn("bn");
      const int n = acnn_bn_bwd_reduce_parts(B, HW, C);
      REQUIRE_BIND(n >= 1 && (int64_t)n * 2 * C <= r.slot("sums").size, "bn_bwd_reduce partial rows");
      float *mean = r.S(bn.work, 2 * C), *rstd = r.S(bn.work, 3 * C), *sums = r.S("sums");
      return [=](void* st) { return acnn_bn_bwd_reduce(g, y, mean, rstd, gate, addbc, sums, B, HW, C, adt, st); };
    }
    float* coef = r.S("coef");
    void* dy = r.Tn("dy");
    return [=](void* st) { return acnn_bn_bwd_apply(g, y, coef, gate, addbc, dy, B, HW, C, adt, st); };
  }
  if (k == "bn_bwd_reduce2" || k == "bn_bwd_apply2") {
    const auto& sh = op.find("shape")->v;
    const int B = (int)sh[0], HW = (int)(sh[1] * sh[2]), C = (int)sh[3];
    void *g = r.Tn("g"), *y = r.Tn("y"), *y2 = r.Tn("y2");
    if (k == "bn_bwd_reduce2") {
      const BatchNorm &a = r.bn("bn"), &b = r.bn("bn2");
      const int n = acnn_bn_bwd_reduce_parts(B, HW, C);
      REQUIRE_BIND(n >= 1 && (int64_t)n * 2 * C <= r.slot("sums").size &&
                       (int64_t)n * 2 * C <= r.slot("sums2").size, "bn_bwd_reduce2 partial rows");
      float *ma = r.S(a.work, 2 * C), *ra = r.S(a.work, 3 * C), *mb = r.S(b.work, 2 * C),
            *rb = r.S(b.work, 3 * C), *sa = r.S("sums"), *sb = r.S("sums2");
      return [=](void* st) { return acnn_bn_bwd_reduce2(g, y, y2, ma, ra, mb, rb, sa, sb, B, HW, C, adt, st); };
    }
    float *ca = r.S("coef"), *cb = r.S("coef2");
    void *dy = r.Tn("dy"), *dy2 = r.Tn("dy2");
    return [=](void* st) { return acnn_bn_bwd_apply2(g, y, y2, ca, cb, dy, dy2, B, HW, C, adt, st); };
  }
  if (k == "bn_bwd_finalize") {
    // rows of `sums`: written by the reduce op that precedes this one (same slot)
    const BatchNorm& bn = r.bn("bn");
    const int C = bn.C;
    int n = -1;
    const Slot sums = r.slot("sums");
    for (const Op& o : p.backward) {
      if (&o == &op) break;
      for (const char* key : {"sums", "sums2"}) {
        const Val* s = o.find(key);
        if (!s || s->slot.buf != sums.buf || s->slot.offset != sums.offset) continue;
        if (o.kind == "bn_bwd_reduce" || o.kind == "bn_bwd_reduce2") {
          const auto& sh = o.find("shape")->v;
          n = acnn_bn_bwd_reduce_parts((int)sh[0], (int)(sh[1] * sh[2]), (int)sh[3]);
        } else if (o.kind == "sk_bn_bwd_reduce") {
          n = acnn_sk_bn_bwd_reduce_parts((int)o.find("B")->i, (int)o.find("HW")->i, (int)o.find("f")->i);
        }
      }
    }
    REQUIRE_BIND(n >= 1, "bn_bwd_finalize without a preceding reduce");
    float *s = r.S("sums"), *gamma = r.Pv(bn.gamma), *mean = r.S(bn.work, 2 * C), *rstd = r.S(bn.work, 3 * C),
          *coef = r.S("coef"), *dg = r.Gv(bn.gamma), *db = r.Gv(bn.beta);
    const int64_t count = bn.count;
    return [=](void* st) { return acnn_bn_bwd_finalize(s, n, gamma, mean, rstd, count, coef, dg, db, C, st); };
  }
  if (k == "sk_bn_bwd_reduce" || k == "sk_bn_bwd_apply") {
    const BatchNorm& bn = r.bn("bn");
    const int C = bn.C, B = (int)r.I("B"), HW = (int)r.I("HW"), f = (int)r.I("f");
    void *dv = r.Tn("dv"), *y = r.Tn("y");
    float *sc = r.S(bn.work), *sh = r.S(bn.work, C), *att = r.S("att"), *ds = r.S("ds");
    if (k == "sk_bn_bwd_reduce") {
      const int n = acnn_sk_bn_bwd_reduce_parts(B, HW, f);
      REQUIRE_BIND(n >= 1 && (int64_t)n * 2 * C <= r.slot("sums").size, "sk_bn_bwd_reduce partial rows");
      float *mean = r.S(bn.work, 2 * C), *rstd = r.S(bn.work, 3 * C), *sums = r.S("sums");
      return [=](void* st) {
        return acnn_sk_bn_bwd_reduce(dv, y, sc, sh, mean, rstd, att, ds, sums, B, HW, f, adt, st);
      };
    }
    float* coef = r.S("coef");
    void* dy = r.Tn("dy");
    return [=](void* st) { return acnn_sk_bn_bwd_apply(dv, y, sc, sh, att, ds, coef, dy, B, HW, f, adt, st); };
  }
  if (k == "upsample2x_bwd") {
    void *dout = r.Tn("dout"), *dx = r.Tn("dx"), *add = r.Tn("add_src"), *mask = r.Tn("mask_src");
    const int B = (int)r.I("B"), H = (int)r.I("H"), W = (int)r.I("W"), C = (int)r.I("C");
    return [=](void* st) { return acnn_upsample2x_bwd(dout, dx, add, mask, B, H, W, C, adt, st); };
  }
  if (k == "grad_combine") {
    void *a = r.Tn("a"), *add = r.Tn("add_src"), *mask = r.Tn("mask_src"), *out = r.Tn("out");
    const int64_t n = numel(op.find("shape")->v);
    return [=](void* st) { return acnn_grad_combine(a, add, mask, out, n, adt, st); };
  }
  if (k == "sgd") {
    REQUIRE_BIND(m->grads && m->momentum, "sgd without grads / momentum buffers");
    float *w = m->params, *g = m->grads, *acc = m->momentum, *l2 = r.S("loss", 1), *scratch = r.S("scratch");
    const int64_t n = p.param_elems;
    const uint8_t* flags = reinterpret_cast<const uint8_t*>(m->ws + m->flags_off);
    return [=](void* st) { return acnn_sgd_momentum(w, g, acc, n, flags, hp, l2, scratch, st); };
  }
  set_error("acnn_bind: unknown op kind '%s'", k.c_str());
  return acnn_model::Launch();
}

int resolve_all(acnn_model* m, const std::vector<Op>& ops, std::vector<acnn_model::Launch>* out) {
  out->clear();
  for (const Op& op : ops) {
    acnn_model::Launch l = resolve(m, op);
    if (!l) return ACNN_ERR_INVALID;
    out->push_back(std::move(l));
  }
  return ACNN_OK;
}

int run_range(acnn_model* m, const std::vector<acnn_model::Launch>& l, int first, int last, void* stream) {
  ACNN_REQUIRE(m && m->bound, "acnn_model: not bound (acnn_bind first)");
  ACNN_REQUIRE(first >= 0 && last <= (int)l.size() && first <= last, "op range [%d, %d) outside [0, %d)", first,
               last, (int)l.size());
  for (int i = first; i < last; ++i) {
    const int rc = l[i](stream);
    if (rc != ACNN_OK) return rc;
  }
  return ACNN_OK;
}

void copy_str(char* dst, size_t cap, const std::string& s) {
  strncpy(dst, s.c_str(), cap - 1);
  dst[cap - 1] = 0;
}

int memcpy_async(void* dst, const void* src, int64_t bytes, void* stream, const char* what) {
  const cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

}  // namespace

extern "C" {

void acnn_model_config_init(acnn_model_config* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->struct_size = (int32_t)sizeof(*c);
  c->resnet_size = 50;
  c->num_classes = 1001;
  c->resnet_version = 1;
  c->bl_alpha = 2;
  c->bl_beta = 4;
  strcpy(c->pool_type, "gap");
  strcpy(c->loss_type, "softmax");
  c->bn_momentum = 0.997;
  c->bn_epsilon = 1e-5;
  c->batch = 32;
  c->height = c->width = 224;
  c->training = 1;
  c->with_loss = 1;
  c->dtype = ACNN_BF16;
  c->deterministic = -1;
  c->fuse_bn_pairs = 1;
  c->loss_scale = 1.0;
}

int acnn_create(const acnn_model_config* c, acnn_model** out) {
  ACNN_REQUIRE(c && out, "acnn_create: null argument");
  ACNN_REQUIRE(c->struct_size == (int32_t)sizeof(acnn_model_config),
               "acnn_create: acnn_model_config.struct_size %d != %d (header / library mismatch)", c->struct_size,
               (int)sizeof(acnn_model_config));
  ACNN_REQUIRE(c->dtype == ACNN_BF16 || c->dtype == ACNN_F32, "dtype must be one of: ('bf16', 'fp32')");
  auto term = [](const char* s, size_t n) { return std::string(s, strnlen(s, n)); };
  Config k;
  k.resnet_size = c->resnet_size;
  k.num_classes = c->num_classes;
  k.resnet_version = c->resnet_version;
  k.no_downsample = c->no_downsample;
  k.zero_gamma = c->zero_gamma;
  k.use_se_block = c->use_se_block;
  k.use_sk_block = c->use_sk_block;
  k.bn_momentum = c->bn_momentum;
  k.bn_epsilon = c->bn_epsilon;
  k.embedding_size = c->embedding_size;
  k.anti_alias_filter_size = c->anti_alias_filter_size;
  k.anti_alias_type = term(c->anti_alias_type, sizeof(c->anti_alias_type));
  k.pool_type = term(c->pool_type, sizeof(c->pool_type));
  k.loss_type = term(c->loss_type, sizeof(c->loss_type));
  k.bl_alpha = c->bl_alpha;
  k.bl_beta = c->bl_beta;
  k.use_resnet_d = c->use_resnet_d;
  k.batch = c->batch;
  k.height = c->height;
  k.width = c->width;
  k.training = c->training;
  k.mixup_type = c->mixup_type;
  k.with_loss = c->with_loss;
  k.fp32 = c->dtype == ACNN_F32;
  k.use_dropblock = c->use_dropblock;
  k.deterministic = c->deterministic;
  k.fuse_bn_pairs = c->fuse_bn_pairs;
  k.label_smoothing = c->label_smoothing;
  k.kd_temp = c->kd_temp;
  k.loss_scale = c->loss_scale > 0 ? c->loss_scale : 1.0;
  ACNN_REQUIRE(k.bl_alpha >= 1 && k.bl_beta >= 1, "bl_alpha / bl_beta must be positive");
  std::unique_ptr<acnn_model> m(new (std::nothrow) acnn_model());
  ACNN_REQUIRE(m, "acnn_create: out of host memory");
  const int rc = build_plan(k, &m->plan);
  if (rc != ACNN_OK) return rc;
  layout(m.get());
  *out = m.release();
  return ACNN_OK;
}

void acnn_destroy(acnn_model* m) { delete m; }

int acnn_model_get_sizes(const acnn_model* m, acnn_model_sizes* o) {
  ACNN_REQUIRE(m && o, "acnn_model_get_sizes: null argument");
  const Plan& p = m->plan;
  memset(o, 0, sizeof(*o));
  o->param_elems = p.param_elems;
  o->state_elems = p.state_elems;
  o->dgrad_elems = p.dgrad_elems;
  o->w_fprop_elems = m->planes * p.param_elems;
  o->w_dgrad_elems = p.cfg.training ? m->planes * std::max<int64_t>(p.dgrad_elems, 1) : 0;
  o->workspace_bytes = m->ws_bytes;
  o->hp_offset = m->hp_off;
  o->loss_offset = p.loss.buf == BUF_NONE ? -1 : m->zero_off + 4 * p.loss.offset;
  o->decay_flags_offset = m->flags_off;
  o->zero_offset = m->zero_off;
  o->zero_bytes = p.zero_elems * 4;
  o->work_offset = m->work_off;
  o->work_bytes = p.work_elems * 4;
  o->n_variables = (int32_t)p.vars.size();
  o->n_tensors = (int32_t)p.tensors.size();
  o->n_forward = (int32_t)p.forward.size();
  o->n_loss_first = p.n_loss_first;
  o->n_backward = (int32_t)p.backward.size();
  o->n_update = (int32_t)p.update.size();
  o->input_batch = p.input_batch;
  o->ld_logits = p.ld_logits;
  return ACNN_OK;
}

int acnn_variable_count(const acnn_model* m) { return m ? (int)m->plan.vars.size() : -1; }

int acnn_variable_info_get(const acnn_model* m, int i, acnn_variable_info* o) {
  ACNN_REQUIRE(m && o && i >= 0 && i < (int)m->plan.vars.size(), "acnn_variable_info_get: bad index %d", i);
  const Variable& v = m->plan.vars[i];
  memset(o, 0, sizeof(*o));
  ACNN_REQUIRE(v.name.size() < sizeof(o->name), "variable name too long: %s", v.name.c_str());
  copy_str(o->name, sizeof(o->name), v.name);
  copy_str(o->kind, sizeof(o->kind), v.kind);
  o->buffer = v.buffer;
  o->tf_rank = (int32_t)v.tf_shape.size();
  o->store_rank = (int32_t)v.store_shape.size();
  for (size_t d = 0; d < v.tf_shape.size(); ++d) o->tf_shape[d] = v.tf_shape[d];
  for (size_t d = 0; d < v.store_shape.size(); ++d) o->store_shape[d] = v.store_shape[d];
  o->offset = v.offset;
  o->size = v.size;
  o->dgrad_off = v.dgrad_off;
  o->decay = v.decay;
  o->zero_init = v.zero_init;
  o->grad_ready_op = v.grad_ready_op;
  return ACNN_OK;
}

static int convert_variable(const acnn_model* m, int i, const float* tf, float* st, float* tf_out,
                            const float* st_in) {
  ACNN_REQUIRE(m && i >= 0 && i < (int)m->plan.vars.size(), "acnn_variable_pack/unpack: bad index %d", i);
  const Variable& v = m->plan.vars[i];
  const bool pack = st != nullptr;
  ACNN_REQUIRE(pack ? (tf != nullptr) : (tf_out != nullptr && st_in != nullptr), "null array");
  if (v.kind == "conv_kernel") {   // HWIO <-> OHWI
    const int64_t kh = v.tf_shape[0], kw = v.tf_shape[1], ci = v.tf_shape[2], co = v.tf_shape[3];
    for (int64_t o = 0; o < co; ++o)
      for (int64_t r = 0; r < kh; ++r)
        for (int64_t c = 0; c < kw; ++c)
          for (int64_t k = 0; k < ci; ++k) {
            const int64_t a = ((r * kw + c) * ci + k) * co + o, b = ((o * kh + r) * kw + c) * ci + k;
            if (pack) st[b] = tf[a]; else tf_out[a] = st_in[b];
          }
  } else if (v.kind == "dense_kernel") {   // [in, classes] <-> [ld_logits][in], padded rows zero
    const int64_t in = v.tf_shape[0], nc = v.tf_shape[1];
    if (pack) memset(st, 0, sizeof(float) * (size_t)v.size);
    for (int64_t k = 0; k < in; ++k)
      for (int64_t o = 0; o < nc; ++o) {
        if (pack) st[o * in + k] = tf[k * nc + o]; else tf_out[k * nc + o] = st_in[o * in + k];
      }
  } else {   // vectors; the dense bias is zero-padded to ld_logits
    const int64_t n = numel(v.tf_shape);
    if (pack) {
      memset(st, 0, sizeof(float) * (size_t)v.size);
      memcpy(st, tf, sizeof(float) * (size_t)n);
    } else {
      memcpy(tf_out, st_in, sizeof(float) * (size_t)n);
    }
  }
  return ACNN_OK;
}

int acnn_variable_pack(const acnn_model* m, int i, const float* tf_values, float* stored) {
  ACNN_REQUIRE(stored, "acnn_variable_pack: null destination");
  return convert_variable(m, i, tf_values, stored, nullptr, nullptr);
}
int acnn_variable_unpack(const acnn_model* m, int i, const float* stored, float* tf_values) {
  return convert_variable(m, i, nullptr, nullptr, tf_values, stored);
}

int acnn_tensor_count(const acnn_model* m) { return m ? (int)m->plan.tensors.size() : -1; }

int acnn_tensor_info_get(const acnn_model* m, int i, acnn_tensor_info* o) {
  ACNN_REQUIRE(m && o && i >= 0 && i < (int)m->plan.tensors.size(), "acnn_tensor_info_get: bad index %d", i);
  const Tensor& t = m->plan.tensors[i];
  memset(o, 0, sizeof(*o));
  copy_str(o->name, sizeof(o->name), t.name);
  o->dtype = t.dtype;
  o->rank = (int32_t)t.shape.size();
  ACNN_REQUIRE(t.shape.size() <= 5, "tensor rank");
  for (size_t d = 0; d < t.shape.size(); ++d) o->shape[d] = t.shape[d];
  o->offset = t.ws_offset;
  return ACNN_OK;
}

int acnn_find_tensor(const acnn_model* m, const char* role, int index) {
  if (!m || !role) return -1;
  const Plan& p = m->plan;
  const std::string r = role;
  if (r == "dropblock_u") return (index >= 0 && index < (int)p.dropblock_u.size()) ? p.dropblock_u[index] : -1;
  if (index != 0) return -1;
  if (r == "images") return p.images;
  if (r == "labels") return p.labels;
  if (r == "lam1") return p.lam1;
  if (r == "lam2") return p.lam2;
  if (r == "teacher_logits") return p.teacher_logits;
  if (r == "logits") return p.logits;
  if (r == "pooled") return p.pooled;
  if (r == "embedding") return p.embedding;
  if (r == "ysoft") return p.ysoft;
  return -1;
}

int acnn_bind(acnn_model* m, float* params, float* grads, float* momentum, float* state, void* w_fprop,
              void* w_dgrad, void* workspace, void* stream) {
  ACNN_REQUIRE(m && params && state && w_fprop && workspace, "acnn_bind: null buffer");
  const Plan& p = m->plan;
  ACNN_REQUIRE(!p.cfg.training || (grads && momentum && w_dgrad),
               "acnn_bind: a training handle needs grads, momentum and w_dgrad");
  ACNN_REQUIRE(((uintptr_t)workspace & 255) == 0 && ((uintptr_t)w_fprop & 255) == 0 &&
                   ((uintptr_t)params & 255) == 0, "acnn_bind: buffers must be 256-byte aligned");
  m->params = params;
  m->grads = grads;
  m->momentum = momentum;
  m->state = state;
  m->w_fprop = (char*)w_fprop;
  m->w_dgrad = (char*)w_dgrad;
  m->ws = (char*)workspace;
  m->bound = false;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(m->ws, 0, (size_t)m->ws_bytes, st);
  if (e != cudaSuccess) {
    set_error("acnn_bind: clearing the workspace: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  int rc = memcpy_async(m->ws + m->hp_off, m->hp_init, sizeof(m->hp_init), stream, "acnn_bind: hp");
  if (rc == ACNN_OK && !m->descs.empty())
    rc = memcpy_async(m->ws + m->descs_off, m->descs.data(), (int64_t)m->descs.size() * sizeof(acnn_weight_desc),
                      stream, "acnn_bind: weight descriptors");
  if (rc == ACNN_OK)
    rc = memcpy_async(m->ws + m->flags_off, m->flags.data(), (int64_t)m->flags.size(), stream,
                      "acnn_bind: decay flags");
  for (const auto& o : p.ones) {   // identity-BN scale vectors (DropBlock tails)
    if (rc != ACNN_OK) break;
    if ((int64_t)m->ones.size() < o.second) m->ones.assign((size_t)o.second, 1.0f);
    rc = memcpy_async(m->ws + m->work_off + 4 * o.first, m->ones.data(), 4 * o.second, stream, "acnn_bind: ones");
  }
  if (rc != ACNN_OK) return rc;
  if ((rc = resolve_all(m, p.forward, &m->fwd)) != ACNN_OK) return rc;
  if ((rc = resolve_all(m, p.backward, &m->bwd)) != ACNN_OK) return rc;
  if ((rc = resolve_all(m, p.update, &m->upd)) != ACNN_OK) return rc;
  m->bound = true;
  return ACNN_OK;
}

int acnn_validate(acnn_model* m) {
  ACNN_REQUIRE(m, "acnn_validate: null model");
  // synthetic, suitably aligned, non-null addresses: resolve() only does pointer arithmetic on them
  struct Saved {
    float *params, *grads, *momentum, *state;
    char *w_fprop, *w_dgrad, *ws;
  } saved{m->params, m->grads, m->momentum, m->state, m->w_fprop, m->w_dgrad, m->ws};
  char* const base = reinterpret_cast<char*>(uintptr_t(1) << 40);
  const int64_t span = int64_t(1) << 36;
  m->params = reinterpret_cast<float*>(base);
  m->state = reinterpret_cast<float*>(base + span);
  m->w_fprop = base + 2 * span;
  m->ws = base + 3 * span;
  if (m->plan.cfg.training) {
    m->grads = reinterpret_cast<float*>(base + 4 * span);
    m->momentum = reinterpret_cast<float*>(base + 5 * span);
    m->w_dgrad = base + 6 * span;
  } else {
    m->grads = m->momentum = nullptr;
    m->w_dgrad = nullptr;
  }
  std::vector<acnn_model::Launch> tmp;
  int rc = resolve_all(m, m->plan.forward, &tmp);
  if (rc == ACNN_OK) rc = resolve_all(m, m->plan.backward, &tmp);
  if (rc == ACNN_OK) rc = resolve_all(m, m->plan.update, &tmp);
  m->params = saved.params;
  m->grads = saved.grads;
  m->momentum = saved.momentum;
  m->state = saved.state;
  m->w_fprop = saved.w_fprop;
  m->w_dgrad = saved.w_dgrad;
  m->ws = saved.ws;
  return rc;
}

int acnn_set_loss_scale(acnn_model* m, double loss_scale) {
  ACNN_REQUIRE(m && loss_scale > 0, "acnn_set_loss_scale: bad argument");
  m->loss_scale = loss_scale;
  return ACNN_OK;
}

int acnn_set_dropblock(acnn_model* m, uint64_t seed, int feed_uniforms) {
  ACNN_REQUIRE(m, "acnn_set_dropblock: null model");
  m->dropblock_seed = seed;
  m->dropblock_feed = feed_uniforms ? 1 : 0;
  return ACNN_OK;
}

int acnn_set_inputs(acnn_model* m, const float* images, const int32_t* labels, const float* lam1,
                    const float* lam2, const float* teacher_logits, void* stream) {
  ACNN_REQUIRE(m && m->bound, "acnn_set_inputs: not bound");
  const Plan& p = m->plan;
  const std::pair<const void*, int> in[] = {
      {images, p.images}, {labels, p.labels}, {lam1, p.lam1}, {lam2, p.lam2}, {teacher_logits, p.teacher_logits}};
  for (const auto& i : in) {
    if (!i.first) continue;
    ACNN_REQUIRE(i.second >= 0, "acnn_set_inputs: this model has no such input");
    const Tensor& t = p.tensors[i.second];
    const int rc = memcpy_async(m->ws + t.ws_offset, i.first, t.bytes(), stream, "acnn_set_inputs");
    if (rc != ACNN_OK) return rc;
  }
  return ACNN_OK;
}

int acnn_set_images_u8(acnn_model* m, const uint8_t* images_dev, const float* mean3, void* stream) {
  ACNN_REQUIRE(m && m->bound && images_dev && mean3, "acnn_set_images_u8: not bound / null");
  const Plan& p = m->plan;
  cudaPointerAttributes at{};
  const cudaError_t e = cudaPointerGetAttributes(&at, images_dev);
  if (e != cudaSuccess) {
    set_error("acnn_set_images_u8: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  ACNN_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
               "acnn_set_images_u8: images_dev must be device memory (stage host images in a device buffer)");
  const Tensor& t = p.tensors[p.images];
  return acnn_images_from_u8(images_dev, mean3, (float*)(m->ws + t.ws_offset), (int)t.shape[0], (int)t.shape[1],
                             (int)t.shape[2], stream);
}

int acnn_set_images_resized(acnn_model* m, const acnn_resize_desc* desc_dev, int n_valid, const float* mean3,
                            void* stream) {
  ACNN_REQUIRE(m && m->bound && desc_dev && mean3, "acnn_set_images_resized: not bound / null");
  const Plan& p = m->plan;
  const Tensor& t = p.tensors[p.images];
  ACNN_REQUIRE(t.shape[1] == t.shape[2], "acnn_set_images_resized: the plan's input is %lldx%lld, not square",
               (long long)t.shape[1], (long long)t.shape[2]);
  cudaPointerAttributes at{};
  const cudaError_t e = cudaPointerGetAttributes(&at, desc_dev);
  if (e != cudaSuccess) {
    set_error("acnn_set_images_resized: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  ACNN_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
               "acnn_set_images_resized: desc_dev must be device memory");
  return acnn_resize_crop_u8(desc_dev, (int)t.shape[0], n_valid, (int)t.shape[1], mean3,
                             (float*)(m->ws + t.ws_offset), stream);
}

int acnn_set_images_cropped(acnn_model* m, const acnn_crop_desc* desc_dev, const float* mean3, void* stream) {
  ACNN_REQUIRE(m && m->bound && desc_dev && mean3, "acnn_set_images_cropped: not bound / null");
  const Plan& p = m->plan;
  const Tensor& t = p.tensors[p.images];
  ACNN_REQUIRE(t.shape[1] == t.shape[2], "acnn_set_images_cropped: the plan's input is %lldx%lld, not square",
               (long long)t.shape[1], (long long)t.shape[2]);
  cudaPointerAttributes at{};
  const cudaError_t e = cudaPointerGetAttributes(&at, desc_dev);
  if (e != cudaSuccess) {
    set_error("acnn_set_images_cropped: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  ACNN_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
               "acnn_set_images_cropped: desc_dev must be device memory");
  return acnn_crop_resize_u8(desc_dev, (int)t.shape[0], (int)t.shape[0], (int)t.shape[1], mean3,
                             (float*)(m->ws + t.ws_offset), stream);
}

int acnn_set_hparams(acnn_model* m, const float* hp, void* stream) {
  ACNN_REQUIRE(m && m->bound && hp, "acnn_set_hparams: not bound / null");
  return memcpy_async(m->ws + m->hp_off, hp, 32, stream, "acnn_set_hparams");
}

int acnn_get_logits(acnn_model* m, float* out, void* stream) {
  ACNN_REQUIRE(m && m->bound && out, "acnn_get_logits: not bound / null");
  const Plan& p = m->plan;
  const cudaError_t e = cudaMemcpy2DAsync(out, (size_t)p.cfg.num_classes * 4, m->ws + p.tensors[p.logits].ws_offset,
                                          (size_t)p.ld_logits * 4, (size_t)p.cfg.num_classes * 4, (size_t)p.cfg.batch,
                                          cudaMemcpyDefault, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("acnn_get_logits: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

int acnn_get_loss(acnn_model* m, float* out, void* stream) {
  ACNN_REQUIRE(m && m->bound && out, "acnn_get_loss: not bound / null");
  ACNN_REQUIRE(m->plan.loss.buf != BUF_NONE, "acnn_get_loss: this model has no loss ops");
  return memcpy_async(out, m->ws + m->zero_off + 4 * m->plan.loss.offset, 16, stream, "acnn_get_loss");
}

int acnn_clear_step_buffers(acnn_model* m, void* stream) {
  ACNN_REQUIRE(m && m->bound, "acnn_clear_step_buffers: not bound");
  const Plan& p = m->plan;
  int rc = acnn_fill_zero(m->ws + m->zero_off, std::max<int64_t>(p.zero_elems, 1) * 4, stream);
  if (rc == ACNN_OK && m->grads) rc = acnn_fill_zero(m->grads, p.param_elems * 4, stream);
  return rc;
}

int acnn_forward(acnn_model* m, void* stream) {
  const int rc = acnn_clear_step_buffers(m, stream);
  return rc != ACNN_OK ? rc : run_range(m, m->fwd, 0, m->plan.n_loss_first, stream);
}
int acnn_loss(acnn_model* m, void* stream) {
  ACNN_REQUIRE(m, "acnn_loss: null model");
  return run_range(m, m->fwd, m->plan.n_loss_first, (int)m->fwd.size(), stream);
}
int acnn_backward_range(acnn_model* m, int first, int last, void* stream) {
  ACNN_REQUIRE(m, "acnn_backward_range: null model");
  return run_range(m, m->bwd, first, last, stream);
}
int acnn_backward(acnn_model* m, void* stream) {
  ACNN_REQUIRE(m, "acnn_backward: null model");
  return run_range(m, m->bwd, 0, (int)m->bwd.size(), stream);
}
int acnn_sgd_step(acnn_model* m, void* stream) {
  ACNN_REQUIRE(m, "acnn_sgd_step: null model");
  return run_range(m, m->upd, 0, (int)m->upd.size(), stream);
}
int acnn_step(acnn_model* m, void* stream) {
  int rc = acnn_forward(m, stream);
  if (rc == ACNN_OK) rc = acnn_loss(m, stream);
  if (rc == ACNN_OK) rc = acnn_backward(m, stream);
  if (rc == ACNN_OK) rc = acnn_sgd_step(m, stream);
  return rc;
}
int acnn_run_ops(acnn_model* m, int phase, int first, int last, void* stream) {
  ACNN_REQUIRE(m && phase >= 0 && phase <= 2, "acnn_run_ops: bad phase %d", phase);
  return run_range(m, phase == 0 ? m->fwd : (phase == 1 ? m->bwd : m->upd), first, last, stream);
}

const char* acnn_op_kind(const acnn_model* m, int phase, int index) {
  if (!m || phase < 0 || phase > 2) return nullptr;
  const std::vector<Op>& l = phase == 0 ? m->plan.forward : (phase == 1 ? m->plan.backward : m->plan.update);
  return (index >= 0 && index < (int)l.size()) ? l[index].kind.c_str() : nullptr;
}

int acnn_op_conv_info(const acnn_model* m, int phase, int index, acnn_conv_geom* g, int64_t* alg_macs,
                      int* aux_tiles) {
  ACNN_REQUIRE(m && g && phase >= 0 && phase <= 2, "acnn_op_conv_info: bad argument");
  const std::vector<Op>& l = phase == 0 ? m->plan.forward : (phase == 1 ? m->plan.backward : m->plan.update);
  ACNN_REQUIRE(index >= 0 && index < (int)l.size(), "acnn_op_conv_info: op index %d out of range", index);
  const Op& op = l[index];
  const Val* gv = op.find("geom");
  ACNN_REQUIRE(gv && (op.kind == "conv" || op.kind == "conv_dgrad" || op.kind == "conv_wgrad"),
               "acnn_op_conv_info: op '%s' is not a GEMM", op.kind.c_str());
  const Geom& s = gv->g;
  memset(g, 0, sizeof(*g));
  g->B = s.B; g->H = s.H; g->W = s.W; g->Cin = s.Cin; g->Cout = s.Cout; g->kh = s.kh; g->kw = s.kw;
  g->stride = s.stride; g->pad_h_lo = s.pad_h_lo; g->pad_h_hi = s.pad_h_hi; g->pad_w_lo = s.pad_w_lo;
  g->pad_w_hi = s.pad_w_hi;
  const Val* am = op.find("alg_macs");
  if (alg_macs)
    *alg_macs = am ? am->i : (int64_t)s.B * s.Ho() * s.Wo() * s.Cout * s.kh * s.kw * s.Cin;
  if (aux_tiles) *aux_tiles = (op.find("add_src") ? 1 : 0) + (op.find("mask_src") ? 1 : 0);
  return ACNN_OK;
}

int64_t acnn_plan_dump(const acnn_model* m, char* buf, int64_t cap) {
  if (!m) return -1;
  const std::string s = m->plan.dump();
  if (buf && cap > 0) {
    const int64_t n = std::min<int64_t>(cap - 1, (int64_t)s.size());
    memcpy(buf, s.data(), (size_t)n);
    buf[n] = 0;
  }
  return (int64_t)s.size() + 1;
}

}  // extern "C"
