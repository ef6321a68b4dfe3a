// Layer-plan builder of the model-level C ABI (see model_plan.h).  Host code only.
#include "model_plan.h"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>

#include <algorithm>

#include "common.h"

namespace acnn {
namespace model {

namespace {

struct PlanError {
  int code;
  std::string msg;
};

[[noreturn]] void fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw PlanError{code, buf};
}

#define PLAN_ASSERT(cond, ...) \
  do {                         \
    if (!(cond)) fail(ACNN_ERR_INVALID, __VA_ARGS__); \
  } while (0)

// functions/model_fns.py:113-127
const std::vector<int>* block_sizes(int version, int size) {
  static const std::map<int, std::vector<int>> v1 = {
      {50, {3, 4, 6, 3}}, {101, {3, 4, 23, 3}}, {152, {3, 8, 36, 3}}, {200, {3, 24, 36, 3}}};
  static const std::map<int, std::vector<int>> v2 = {
      {50, {3, 4, 6, 3}}, {101, {4, 8, 18, 3}}, {152, {5, 12, 30, 3}}};
  const auto& m = version == 1 ? v1 : v2;
  auto it = m.find(size);
  return it == m.end() ? nullptr : &it->second;
}

struct Stem {   // space-to-depth stem bookkeeping
  int k = 0, pad = 0, k2 = 0, pad2 = 0, hi2 = 0;
  int w2 = -1;
  Slot dw2;
  int64_t alg_macs = 0;
};

struct ConvOut {
  int x = -1, y = -1;
  Geom geom;
  int w = -1;    // variable id
  int bn = -1;
  bool has_stem = false;
  Stem stem;
};

struct DbMask {   // one DropBlock call of the reference: a mask [H,W,C] shared by the batch + its scale
  Slot keep, scale, scratch;
  int H = 0, W = 0, C = 0, block_size = 7, u = -1, index = 0;
  double gamma_scale = 0;
};

struct SeGate {
  bool on = false;
  Slot q, h, e, scratch;
  int w1 = -1, w2 = -1, r = 0;
};

using KV = std::pair<const char*, Val>;
using EmitFn = std::function<void(int out, int add, int mask)>;

class Builder {
 public:
  Builder(const Config& cfg, Plan* plan) : cfg_(cfg), p_(*plan) {}
  void run();

 private:
  const Config& cfg_;
  Plan& p_;
  bool training_ = false, fp32_ = false, use_dropblock_ = false, with_loss_ = false;
  int mixup_type_ = 0, adt_ = ACNN_BF16, B_ = 0;
  double kd_temp_ = 0;
  std::vector<Op>* ops_ = nullptr;
  std::vector<std::function<void()>> tape_;
  std::vector<std::string> scope_{"resnet_model"};
  std::map<std::pair<std::string, std::string>, int> counters_;
  std::map<int, int> planes_;        // tensor -> its (hi, mid, lo) plane tensor
  std::map<int, int> identity_bns_;  // C -> bn id

  // ------------------------------------------------------------------ naming (TF-1.x style)
  std::string joined() const {
    std::string s;
    for (size_t i = 0; i < scope_.size(); ++i) s += (i ? "/" : "") + scope_[i];
    return s;
  }
  std::string unique(const std::string& base) {
    int& n = counters_[{joined(), base}];
    const int cur = n++;
    return cur == 0 ? base : base + "_" + std::to_string(cur);
  }
  struct Scope {
    Builder& b;
    Scope(Builder& b_, const std::string& name) : b(b_) { b.scope_.push_back(b.unique(name)); }
    ~Scope() { b.scope_.pop_back(); }
  };
  std::string full(const std::string& name) const { return joined() + "/" + name; }

  // ------------------------------------------------------------------ allocation helpers
  int tensor(const std::string& base, const Shape& shape, int dtype = -1, bool relu = false) {
    Tensor t;
    t.name = base + "#" + std::to_string(p_.tensors.size() + 1);
    t.shape = shape;
    t.dtype = dtype < 0 ? adt_ : dtype;
    t.relu = relu;
    p_.tensors.push_back(t);
    return (int)p_.tensors.size() - 1;
  }
  Tensor& T(int id) { return p_.tensors[id]; }
  std::string base_of(int id) { return T(id).name.substr(0, T(id).name.find('#')); }

  int variable(const std::string& name, const Shape& tf_shape, const char* kind, const Shape& store_shape,
               bool trainable = true, bool decay = false, bool zero_init = false, bool need_dgrad = false) {
    Variable v;
    v.name = name;
    v.kind = kind;
    v.tf_shape = tf_shape;
    v.store_shape = store_shape;
    v.size = numel(store_shape);
    for (const auto& o : p_.vars) PLAN_ASSERT(o.name != name, "duplicate variable %s", name.c_str());
    if (trainable) {
      v.buffer = ACNN_BUF_PARAMS;
      v.offset = p_.param_elems;
      v.decay = decay;
      v.zero_init = zero_init;
      p_.param_elems += round_up(v.size);
      if (need_dgrad) {
        v.dgrad_off = p_.dgrad_elems;
        p_.dgrad_elems += round_up(v.size);
      }
    } else {
      v.buffer = ACNN_BUF_STATE;
      v.offset = p_.state_elems;
      p_.state_elems += round_up(v.size);
    }
    p_.vars.push_back(v);
    return (int)p_.vars.size() - 1;
  }

  Slot slot(int buf, int64_t size) {
    Slot s;
    s.buf = buf;
    s.size = size;
    int64_t& top = buf == BUF_ZERO ? p_.zero_elems : p_.work_elems;
    s.offset = top;
    top += round_up(size, 32);
    return s;
  }

  void emit(const char* kind, std::initializer_list<KV> a) {
    Op op;
    op.kind = kind;
    for (const auto& kv : a) op.a.emplace_back(kv.first, kv.second);
    ops_->push_back(std::move(op));
  }

  // fp32 mode: the (hi, mid, lo) bf16 operand planes of a GEMM operand tensor, split once right before
  // its first consumer and reused by later ones (fprop + wgrad)
  int planes(int t) {
    if (!fp32_) return -1;
    auto it = planes_.find(t);
    if (it != planes_.end()) return it->second;
    Shape s{3};
    s.insert(s.end(), T(t).shape.begin(), T(t).shape.end());
    const int64_t n = numel(T(t).shape);
    const int pt = tensor("planes", s, ACNN_BF16);
    emit("split3", {{"src", vten(t)}, {"dst", vten(pt)}, {"n", vint(n)}});
    planes_[t] = pt;
    return pt;
  }

  // ------------------------------------------------------------------ gradient accumulation
  int use(int t) {
    T(t).consumers++;
    return t;
  }
  // fn(out, add_src, mask_src) must emit one op writing the new running sum
  void contribute(int t, const EmitFn& fn) {
    T(t).contribs++;
    const bool last = T(t).contribs == T(t).consumers;
    PLAN_ASSERT(T(t).contribs <= T(t).consumers, "too many gradient contributions to %s", T(t).name.c_str());
    const int out = tensor("d_" + base_of(t), T(t).shape);
    fn(out, T(t).grad, (last && T(t).relu) ? t : -1);
    T(t).grad = out;
  }
  // the gradient flowing into t is an existing buffer (identity shortcut)
  void contribute_alias(int t, int buf) {
    T(t).contribs++;
    const bool last = T(t).contribs == T(t).consumers;
    if (T(t).grad < 0 && !(last && T(t).relu)) {
      T(t).grad = buf;
      return;
    }
    const int out = tensor("d_" + base_of(t), T(t).shape);
    emit("grad_combine", {{"a", vten(buf)}, {"add_src", vten(T(t).grad)},
                          {"mask_src", vten((last && T(t).relu) ? t : -1)}, {"out", vten(out)},
                          {"shape", vints(T(t).shape)}});
    T(t).grad = out;
  }
  int grad_of(int t) {
    PLAN_ASSERT(T(t).contribs == T(t).consumers && T(t).grad >= 0, "gradient of %s incomplete (%d/%d)",
                T(t).name.c_str(), T(t).contribs, T(t).consumers);
    return T(t).grad;
  }

  // ------------------------------------------------------------------ layers
  Geom geom_of(int x, int cout, int k, int stride) {
    const Shape& s = T(x).shape;
    const int lo = (k - 1) / 2, hi = k - 1 - lo;
    Geom g;
    g.B = (int)s[0]; g.H = (int)s[1]; g.W = (int)s[2]; g.Cin = (int)s[3];
    g.Cout = cout; g.kh = g.kw = k; g.stride = stride;
    g.pad_h_lo = g.pad_w_lo = lo; g.pad_h_hi = g.pad_w_hi = hi;
    return g;
  }

  int bn_layer(int C, int64_t count, bool zero_gamma = false, const char* layer_name = nullptr) {
    const std::string layer = layer_name ? layer_name : unique("batch_normalization");
    BatchNorm bn;
    bn.C = C;
    bn.count = count;
    bn.gamma = variable(full(layer + "/gamma"), {C}, "gamma", {C}, true, false, zero_gamma);
    bn.beta = variable(full(layer + "/beta"), {C}, "beta", {C});
    bn.mm = variable(full(layer + "/moving_mean"), {C}, "moving_mean", {C}, false);
    bn.mv = variable(full(layer + "/moving_variance"), {C}, "moving_variance", {C}, false);
    if (training_) bn.stats = slot(BUF_WORK, fp32_ ? 2 * C : kStatsPartsCap * 2 * C);
    bn.work = slot(BUF_WORK, 4 * C);
    p_.bns.push_back(bn);
    return (int)p_.bns.size() - 1;
  }
  Val stats_of(int bn) { return (bn >= 0 && training_ && !fp32_) ? vslot(p_.bns[bn].stats) : Val(); }

  // conv2d_fixed_padding (+ the batch norm that always follows it in the reference)
  ConvOut conv(int x, int filters, int k, int stride, bool with_bn = true, bool zero_gamma = false,
               bool need_dgrad = true) {
    const Shape xs = T(x).shape;
    if (filters % 32 || xs[3] % 16)   // e.g. bl_alpha=4: the little branches would have 16 channels
      fail(ACNN_ERR_UNSUPPORTED, "conv %d -> %d channels: the tensor-core tiles need input channels in "
           "multiples of 16 and output channels in multiples of 32", (int)xs[3], filters);
    const std::string layer = unique("conv2d");
    ConvOut co;
    co.x = x;
    co.geom = geom_of(x, filters, k, stride);
    co.w = variable(full(layer + "/kernel"), {k, k, xs[3], filters}, "conv_kernel", {filters, k, k, xs[3]},
                    true, true, false, need_dgrad && training_);
    co.y = tensor("y", {xs[0], co.geom.Ho(), co.geom.Wo(), filters});
    if (with_bn) co.bn = bn_layer(filters, xs[0] * co.geom.Ho() * co.geom.Wo(), zero_gamma);
    const int xp = planes(x);
    emit("conv", {{"x", vten(x)}, {"xp", vten(xp)}, {"w", vvar(co.w)}, {"y", vten(co.y)},
                  {"geom", vgeom(co.geom)}, {"stats", stats_of(co.bn)}, {"out_f32", vint(0)}});
    if (co.bn >= 0) emit_bn_finalize(co.bn, co.y, co.geom);
    if (need_dgrad) use(x);
    return co;
  }

  // batch statistics -> scale / shift / mean / rstd (+ moving statistics).  bf16 mode: the conv epilogue
  // left partial (sum, sumsq) rows (stats_mode 0); fp32 mode: a separate two-pass kernel (stats_mode 1)
  void emit_bn_finalize(int bn, int y, const Geom& g, const std::vector<int64_t>* x_wpad = nullptr) {
    int mode = 0;
    if (training_ && fp32_) {
      emit("bn_stats", {{"x", vten(y)}, {"bn", vbn(bn)}, {"M", vint(p_.bns[bn].count)},
                        {"C", vint(p_.bns[bn].C)}});
      mode = 1;
    }
    emit("bn_finalize", {{"bn", vbn(bn)}, {"stats_mode", vint(mode)}, {"geom", vgeom(g)},
                         {"x_wpad", x_wpad ? vints(*x_wpad) : Val()}});
  }

  // k x k stride-2 conv with padding (k-1)/2 == k2 x k2 stride-1 conv on the space-to-depth(2) image
  // with padding (lo2, hi2): input offset u - p = 2*r + a
  static void stem_s2d_taps(int k, int* p, int* k2, int* lo2, int* hi2) {
    *p = (k - 1) / 2;
    const int rmin = (int)floor(-(double)*p / 2), rmax = (int)floor((double)(k - 1 - *p) / 2);
    *k2 = rmax - rmin + 1;
    *lo2 = -rmin;
    *hi2 = rmax;
  }

  // first conv (k x k, stride 2, 3 input channels) as a stride-1 conv on the packed input
  ConvOut stem_conv(int x0, int filters, int k) {
    const Shape xs = T(x0).shape;   // [B, H2, Wp, 16]
    const std::string layer = unique("conv2d");
    int p, k2, lo2, hi2;
    stem_s2d_taps(k, &p, &k2, &lo2, &hi2);
    const int H2 = (int)xs[1], W2 = (int)xs[2] - lo2 - hi2;
    ConvOut co;
    co.x = x0;
    co.w = variable(full(layer + "/kernel"), {k, k, 3, filters}, "conv_kernel", {filters, k, k, 3}, true,
                    true);
    Geom g;
    g.B = (int)xs[0]; g.H = H2; g.W = W2; g.Cin = 16; g.Cout = filters; g.kh = g.kw = k2; g.stride = 1;
    g.pad_h_lo = g.pad_w_lo = lo2; g.pad_h_hi = g.pad_w_hi = hi2;
    PLAN_ASSERT(g.Ho() == H2 && g.Wo() == W2, "stem geometry");
    co.geom = g;
    co.y = tensor("y", {xs[0], H2, W2, filters});
    co.bn = bn_layer(filters, xs[0] * H2 * W2);
    co.has_stem = true;
    Stem& st = co.stem;
    st.k = k; st.pad = p; st.k2 = k2; st.pad2 = lo2; st.hi2 = hi2;
    st.w2 = tensor("w_stem", {filters, k2, k2, 16});
    if (training_) st.dw2 = slot(BUF_ZERO, (int64_t)filters * k2 * k2 * 16);
    // the k x k x 3 conv, not its zero-padded k2 x k2 x 16 space-to-depth form
    st.alg_macs = xs[0] * H2 * W2 * filters * k * k * 3;
    emit("s2d_weight_pack", {{"w", vvar(co.w)}, {"w2", vten(st.w2)}, {"cout", vint(filters)},
                             {"k", vint(k)}, {"pad", vint(p)}, {"k2", vint(k2)}, {"pad2", vint(lo2)}});
    const int xp = planes(x0);
    const int wp = planes(st.w2);
    const std::vector<int64_t> wpad{lo2, hi2};
    emit("conv", {{"x", vten(x0)}, {"xp", vten(xp)}, {"w", vten(st.w2)}, {"wp", vten(wp)},
                  {"y", vten(co.y)}, {"geom", vgeom(g)}, {"stats", stats_of(co.bn)}, {"out_f32", vint(0)},
                  {"w_is_tensor", vint(1)}, {"x_wpad", vints(wpad)}, {"alg_macs", vint(st.alg_macs)}});
    emit_bn_finalize(co.bn, co.y, g, &wpad);
    return co;
  }

  // out = relu?( bn_a(a) [* gate] + R ); b_mode 1: R = bn_b(b), 2: R = b, 3: R = upsample2x(b)
  int bn_act(const ConvOut& co, bool relu, int b = -1, int bn_b = -1, int b_mode = 0, Slot gate = Slot(),
             const char* name = "u") {
    const int out = tensor(name, T(co.y).shape, -1, relu);
    emit("bn_act", {{"a", vten(co.y)}, {"bn_a", vbn(co.bn)}, {"b", vten(b)}, {"bn_b", vbn(bn_b)},
                    {"b_mode", vint(b_mode)}, {"gate", vslot(gate)}, {"relu", vint(relu)},
                    {"out", vten(out)}, {"shape", vints(T(co.y).shape)}});
    return out;
  }

  // -- DropBlock ---------------------------------------------------------------------------------------
  int identity_bn(int C) {   // scale = 1, shift = 0: lets bn_act consume an already-normalised tensor
    auto it = identity_bns_.find(C);
    if (it != identity_bns_.end()) return it->second;
    BatchNorm bn;
    bn.C = C;
    bn.work = slot(BUF_WORK, 4 * C);
    p_.ones.emplace_back(bn.work.offset, C);
    p_.bns.push_back(bn);
    return identity_bns_[C] = (int)p_.bns.size() - 1;
  }

  DbMask dropblock_mask(int H, int W, int C, double gamma_scale, int block_size = 7) {
    if (H < block_size || W < block_size)
      fail(ACNN_ERR_INVALID, "dropblock: feature map %dx%d smaller than block_size %d (the reference fails "
           "the same way: nets/blocks.py:222-229)", H, W, block_size);
    const int hs = H - block_size + 1, ws = W - block_size + 1;
    DbMask m;
    m.u = tensor("dropblock_u", {hs, ws, C}, ACNN_F32);
    m.index = (int)p_.dropblock_u.size();
    p_.dropblock_u.push_back(m.u);
    m.keep = slot(BUF_WORK, (int64_t)H * W * C);
    m.scale = slot(BUF_WORK, 1);
    m.scratch = slot(BUF_WORK, (int64_t)hs * ws * C + ((int64_t)H * W * C + 255) / 256);
    m.H = H; m.W = W; m.C = C; m.gamma_scale = gamma_scale; m.block_size = block_size;
    emit("dropblock_mask", {{"keep", vslot(m.keep)}, {"scale", vslot(m.scale)}, {"scratch", vslot(m.scratch)},
                            {"H", vint(H)}, {"W", vint(W)}, {"C", vint(C)}, {"gamma_scale", vflt(gamma_scale)},
                            {"block_size", vint(block_size)}, {"u", vten(m.u)}, {"index", vint(m.index)}});
    return m;
  }
  void emit_db_apply(int x, const DbMask& m, bool relu, int out, const Shape& s) {
    emit("dropblock_apply", {{"x", vten(x)}, {"keep", vslot(m.keep)}, {"scale", vslot(m.scale)},
                             {"relu", vint(relu)}, {"out", vten(out)}, {"B", vint(s[0])},
                             {"HW", vint(s[1] * s[2])}, {"C", vint(s[3])}});
  }
  // out = relu?(x * keep * scale)
  int dropblock_apply(int x, const DbMask& m, bool relu, const char* name) {
    const Shape s = T(x).shape;
    const int out = tensor(name, s, -1, relu);
    emit_db_apply(x, m, relu, out, s);
    return out;
  }
  int dropblock_bwd(int g, const DbMask& m, const Shape& shape) {   // same kernel on gradients, no relu
    const int dt = tensor("d_db", shape);
    emit_db_apply(g, m, false, dt, shape);
    return dt;
  }
  // conv -> BN -> dropblock -> ReLU (nets/resnet_model.py:49-56,65-72)
  int cbr_db(int x, int filters, int k, int stride, double gamma_scale) {
    const ConvOut co = conv(x, filters, k, stride);
    const int t = bn_act(co, false, -1, -1, 0, Slot(), "t");
    const Shape ts = T(t).shape;
    const DbMask m = dropblock_mask((int)ts[1], (int)ts[2], (int)ts[3], gamma_scale);
    const int u = dropblock_apply(t, m, true, "u");
    tape_.push_back([=] { conv_backward(co, bn_backward(co, dropblock_bwd(grad_of(u), m, ts))); });
    return u;
  }

  // -- backward helpers --------------------------------------------------------------------------------
  int bn_backward(const ConvOut& co, int g, Slot gate = Slot(), Slot addbc = Slot()) {
    const BatchNorm& bn = p_.bns[co.bn];
    const Slot sums = slot(BUF_WORK, kBwdPartsCap * 2 * bn.C);   // per-CTA partial rows
    const Slot coef = slot(BUF_WORK, 3 * bn.C);
    const Shape ys = T(co.y).shape;
    const int dy = tensor("dy", ys);
    emit("bn_bwd_reduce", {{"g", vten(g)}, {"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"gate", vslot(gate)},
                           {"addbc", vslot(addbc)}, {"sums", vslot(sums)}, {"shape", vints(ys)}});
    emit("bn_bwd_finalize", {{"bn", vbn(co.bn)}, {"sums", vslot(sums)}, {"coef", vslot(coef)}});
    emit("bn_bwd_apply", {{"g", vten(g)}, {"y", vten(co.y)}, {"coef", vslot(coef)}, {"gate", vslot(gate)},
                          {"addbc", vslot(addbc)}, {"dy", vten(dy)}, {"shape", vints(ys)}});
    return dy;
  }
  // backward of the two batch norms summed into one residual output (block-final BN and projection-
  // shortcut BN, same gradient g): g is read once per pass instead of twice
  std::pair<int, int> bn_backward2(const ConvOut& a, const ConvOut& b, int g) {
    PLAN_ASSERT(T(a.y).shape == T(b.y).shape, "bn_backward2 shapes");
    const Shape ys = T(a.y).shape;
    const Slot sa = slot(BUF_WORK, kBwdPartsCap * 2 * p_.bns[a.bn].C);
    const Slot ca = slot(BUF_WORK, 3 * p_.bns[a.bn].C);
    const int da = tensor("dy", ys);
    const Slot sb = slot(BUF_WORK, kBwdPartsCap * 2 * p_.bns[b.bn].C);
    const Slot cb = slot(BUF_WORK, 3 * p_.bns[b.bn].C);
    const int db = tensor("dy", ys);
    emit("bn_bwd_reduce2", {{"g", vten(g)}, {"y", vten(a.y)}, {"bn", vbn(a.bn)}, {"sums", vslot(sa)},
                            {"y2", vten(b.y)}, {"bn2", vbn(b.bn)}, {"sums2", vslot(sb)}, {"shape", vints(ys)}});
    emit("bn_bwd_finalize", {{"bn", vbn(a.bn)}, {"sums", vslot(sa)}, {"coef", vslot(ca)}});
    emit("bn_bwd_finalize", {{"bn", vbn(b.bn)}, {"sums", vslot(sb)}, {"coef", vslot(cb)}});
    emit("bn_bwd_apply2", {{"g", vten(g)}, {"y", vten(a.y)}, {"coef", vslot(ca)}, {"dy", vten(da)},
                           {"y2", vten(b.y)}, {"coef2", vslot(cb)}, {"dy2", vten(db)}, {"shape", vints(ys)}});
    return {da, db};
  }

  void conv_backward(const ConvOut& co, int dy, bool need_dgrad = true) {
    const Geom g = co.geom;
    const int dyp = planes(dy);
    if (co.has_stem) {
      const Stem& st = co.stem;
      const int xp = planes(co.x);
      emit("conv_wgrad", {{"x", vten(co.x)}, {"xp", vten(xp)}, {"dy", vten(dy)}, {"dyp", vten(dyp)},
                          {"geom", vgeom(g)}, {"dw_slot", vslot(st.dw2)},
                          {"x_wpad", vints({st.pad2, st.hi2})}, {"alg_macs", vint(st.alg_macs)}});
      emit("s2d_wgrad_unpack", {{"dw2", vslot(st.dw2)}, {"w", vvar(co.w)}, {"cout", vint(g.Cout)},
                                {"k", vint(st.k)}, {"pad", vint(st.pad)}, {"k2", vint(st.k2)},
                                {"pad2", vint(st.pad2)}});
      return;
    }
    const int xp = planes(co.x);
    emit("conv_wgrad", {{"x", vten(co.x)}, {"xp", vten(xp)}, {"dy", vten(dy)}, {"dyp", vten(dyp)},
                        {"geom", vgeom(g)}, {"w", vvar(co.w)}});
    if (!need_dgrad) return;
    const int w = co.w;
    if (g.stride == 1) {
      contribute(co.x, [=](int out, int add, int mask) { emit_dgrad(dy, w, out, g, add, mask, -1); });
      return;
    }
    PLAN_ASSERT(g.stride == 2, "conv stride %d", g.stride);
    const int dyz = tensor("dyz", {g.B, g.H, g.W, g.Cout});
    emit("zero_insert", {{"dy", vten(dy)}, {"out", vten(dyz)}, {"B", vint(g.B)}, {"Ho", vint(g.Ho())},
                         {"Wo", vint(g.Wo())}, {"H", vint(g.H)}, {"W", vint(g.W)}, {"C", vint(g.Cout)}});
    Geom g1 = g;
    g1.stride = 1;
    g1.pad_h_hi = g.kh - 1 - g.pad_h_lo;
    g1.pad_w_hi = g.kw - 1 - g.pad_w_lo;
    // executed on the zero-inserted dy (4x the MACs of the stride-2 transposed conv)
    const int64_t alg = (int64_t)g.B * g.Ho() * g.Wo() * g.Cout * g.kh * g.kw * g.Cin;
    contribute(co.x, [=](int out, int add, int mask) { emit_dgrad(dyz, w, out, g1, add, mask, alg); });
  }

  // dx = conv_transpose(dy) (+ add_src) (* relu mask).  bf16 mode fuses the accumulate / mask into the
  // GEMM epilogue; fp32 mode (fp32 output straight from the accumulators) runs them as one extra elementwise pass
  void emit_dgrad(int dy, int w, int out, const Geom& g, int add, int mask, int64_t alg_macs) {
    const Val alg = alg_macs >= 0 ? vint(alg_macs) : Val();
    if (fp32_ && (add >= 0 || mask >= 0)) {
      const Shape shape = T(out).shape;
      const int tmp = tensor("dx_raw", shape);
      const int dyp = planes(dy);
      emit("conv_dgrad", {{"dy", vten(dy)}, {"dyp", vten(dyp)}, {"w", vvar(w)}, {"dx", vten(tmp)},
                          {"geom", vgeom(g)}, {"alg_macs", alg}});
      emit("grad_combine", {{"a", vten(tmp)}, {"add_src", vten(add)}, {"mask_src", vten(mask)},
                            {"out", vten(out)}, {"shape", vints(shape)}});
    } else {
      const int dyp = planes(dy);
      emit("conv_dgrad", {{"dy", vten(dy)}, {"dyp", vten(dyp)}, {"w", vvar(w)}, {"dx", vten(out)},
                          {"geom", vgeom(g)}, {"add_src", vten(add)}, {"mask_src", vten(mask)},
                          {"alg_macs", alg}});
    }
  }

  // -- composite modules -------------------------------------------------------------------------------
  int cbr(int x, int filters, int k, int stride, bool need_dgrad = true) {   // conv -> BN -> ReLU
    const ConvOut co = conv(x, filters, k, stride, true, false, need_dgrad);
    const int u = bn_act(co, true);
    tape_.push_back([=] { conv_backward(co, bn_backward(co, grad_of(u)), need_dgrad); });
    return u;
  }

  int sk(int t, int filters, int stride) {   // nets/blocks.py:110-154
    const int B = (int)T(t).shape[0];
    const ConvOut co = conv(t, 2 * filters, 3, stride);
    const int H = (int)T(co.y).shape[1], W = (int)T(co.y).shape[2];
    const int f = filters, d = std::max(filters / 2, 32);
    int w1, w2, bnz;
    {
      Scope s(*this, "sk_block");
      w1 = variable(full("sk_fc_1/kernel"), {1, 1, f, d}, "conv_kernel", {d, 1, 1, f}, true, true);
      bnz = bn_layer(d, B, false, "batch_normalization");
      w2 = variable(full("sk_fc_2/kernel"), {1, 1, d, 2 * f}, "conv_kernel", {2 * f, 1, 1, d}, true, true);
    }
    const Slot s = slot(BUF_WORK, (int64_t)B * f), zpre = slot(BUF_WORK, (int64_t)B * d),
               z = slot(BUF_WORK, (int64_t)B * d), att = slot(BUF_WORK, (int64_t)B * f),
               scratch = slot(BUF_WORK, acnn_sk_fc_scratch_floats(B, f, d));
    const int v = tensor("v", {B, H, W, f});
    const int HW = H * W;
#define SK_DIMS {"B", vint(B)}, {"HW", vint(HW)}, {"f", vint(f)}, {"d", vint(d)}
    emit("sk_gap", {{"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"s", vslot(s)}, SK_DIMS});
    emit("sk_fc", {{"s", vslot(s)}, {"w1", vvar(w1)}, {"bn", vbn(bnz)}, {"w2", vvar(w2)},
                   {"zpre", vslot(zpre)}, {"z", vslot(z)}, {"att", vslot(att)}, {"scratch", vslot(scratch)},
                   SK_DIMS});
    emit("sk_combine", {{"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"att", vslot(att)}, {"v", vten(v)}, SK_DIMS});
    tape_.push_back([=] {
      const int gv = grad_of(v);
      const Slot dA = slot(BUF_WORK, (int64_t)B * f), ds = slot(BUF_WORK, (int64_t)B * f),
                 sums = slot(BUF_WORK, (kBwdPartsCap + B) * 4 * f), coef = slot(BUF_WORK, 6 * f);
      const int dy = tensor("dy", T(co.y).shape);
      emit("sk_bwd_gate", {{"dv", vten(gv)}, {"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"dA", vslot(dA)}, SK_DIMS});
      emit("sk_fc_bwd", {{"dA", vslot(dA)}, {"att", vslot(att)}, {"z", vslot(z)}, {"zpre", vslot(zpre)},
                         {"bn", vbn(bnz)}, {"s", vslot(s)}, {"w1", vvar(w1)}, {"w2", vvar(w2)},
                         {"ds", vslot(ds)}, {"scratch", vslot(scratch)}, SK_DIMS});
      emit("sk_bn_bwd_reduce", {{"dv", vten(gv)}, {"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"att", vslot(att)},
                                {"ds", vslot(ds)}, {"sums", vslot(sums)}, SK_DIMS});
      emit("bn_bwd_finalize", {{"bn", vbn(co.bn)}, {"sums", vslot(sums)}, {"coef", vslot(coef)}});
      emit("sk_bn_bwd_apply", {{"dv", vten(gv)}, {"y", vten(co.y)}, {"bn", vbn(co.bn)}, {"att", vslot(att)},
                               {"ds", vslot(ds)}, {"coef", vslot(coef)}, {"dy", vten(dy)}, SK_DIMS});
      conv_backward(co, dy);
    });
#undef SK_DIMS
    return v;
  }

  int blurpool(int x, int filt, int stride) {
    const Shape s = T(x).shape;
    const int B = (int)s[0], H = (int)s[1], W = (int)s[2], C = (int)s[3], pad = (filt - 1) / 2;
    if (pad >= H || pad >= W)
      fail(ACNN_ERR_INVALID, "anti-alias filter %d on a %dx%d feature map: REFLECT padding of %d needs a larger "
           "map (tf.pad fails the same way, nets/blocks.py:70-75)", filt, H, W, pad);
    const int Ho = (H + 2 * pad - filt) / stride + 1, Wo = (W + 2 * pad - filt) / stride + 1;
    const int out = tensor("blur", {B, Ho, Wo, C});
#define BLUR_A {"B", vint(B)}, {"H", vint(H)}, {"W", vint(W)}, {"C", vint(C)}, {"filt", vint(filt)}, \
               {"stride", vint(stride)}
    emit("blurpool", {{"x", vten(x)}, {"out", vten(out)}, BLUR_A});
    use(x);
    tape_.push_back([=] {
      contribute(x, [=](int o, int add, int mask) {
        emit("blurpool_bwd", {{"dout", vten(grad_of(out))}, {"dx", vten(o)}, {"add_src", vten(add)},
                              {"mask_src", vten(mask)}, BLUR_A});
      });
    });
#undef BLUR_A
    return out;
  }

  int avgpool(int x, int k, int stride, int pad_lo, int Ho, int Wo, int count_pad) {
    const Shape s = T(x).shape;
    const int B = (int)s[0], H = (int)s[1], W = (int)s[2], C = (int)s[3];
    const int out = tensor("avgp", {B, Ho, Wo, C});
#define AVG_A {"B", vint(B)}, {"H", vint(H)}, {"W", vint(W)}, {"C", vint(C)}, {"k", vint(k)},          \
              {"stride", vint(stride)}, {"pad_lo", vint(pad_lo)}, {"Ho", vint(Ho)}, {"Wo", vint(Wo)}, \
              {"count_pad", vint(count_pad)}
    emit("avgpool", {{"x", vten(x)}, {"out", vten(out)}, AVG_A});
    use(x);
    tape_.push_back([=] {
      contribute(x, [=](int o, int add, int mask) {
        emit("avgpool_bwd", {{"dout", vten(grad_of(out))}, {"dx", vten(o)}, {"add_src", vten(add)},
                             {"mask_src", vten(mask)}, AVG_A});
      });
    });
#undef AVG_A
    return out;
  }

  int maxpool(int x, int k, int stride) {
    const Shape s = T(x).shape;
    const int B = (int)s[0], H = (int)s[1], W = (int)s[2], C = (int)s[3];
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    const int total = std::max((Ho - 1) * stride + k - H, 0);
    const int pad_lo = total / 2;   // TF SAME: the odd cell goes after
    const int out = tensor("maxp", {B, Ho, Wo, C});
#define MAX_A {"B", vint(B)}, {"H", vint(H)}, {"W", vint(W)}, {"C", vint(C)}, {"k", vint(k)},          \
              {"stride", vint(stride)}, {"pad_lo", vint(pad_lo)}, {"Ho", vint(Ho)}, {"Wo", vint(Wo)}
    emit("maxpool", {{"x", vten(x)}, {"out", vten(out)}, MAX_A});
    use(x);
    tape_.push_back([=] {
      contribute(x, [=](int o, int add, int mask) {
        emit("maxpool_bwd", {{"dout", vten(grad_of(out))}, {"x", vten(x)}, {"dx", vten(o)},
                             {"add_src", vten(add)}, {"mask_src", vten(mask)}, MAX_A});
      });
    });
#undef MAX_A
    return out;
  }

  // block tail with DropBlock (nets/resnet_model.py:42-47,84-95): out = act(db(bn(y3)) + R), R =
  // db(bn(shortcut conv)) for a projection shortcut (mode_bn), x for an identity shortcut
  int residual_tail_db(const ConvOut& co3, const ConvOut* sc, int x_ident, bool relu, double gamma_scale,
                       const DbMask& ms) {
    const Shape ys = T(co3.y).shape;
    const int C = (int)ys[3];
    const int t3 = bn_act(co3, false, -1, -1, 0, Slot(), "t3");
    const DbMask m3 = dropblock_mask((int)ys[1], (int)ys[2], C, gamma_scale);
    const int t3d = dropblock_apply(t3, m3, false, "t3d");
    const bool mode_bn = sc != nullptr;
    int r;
    if (mode_bn) {
      // ms: the shortcut's mask, drawn by the caller where the reference draws it (first in the block)
      const int ts = bn_act(*sc, false, -1, -1, 0, Slot(), "ts");
      r = dropblock_apply(ts, ms, false, "tsd");
    } else {
      r = x_ident;
      use(x_ident);
    }
    ConvOut ident;
    ident.y = t3d;
    ident.bn = identity_bn(C);
    const int out = bn_act(ident, relu, r, -1, 2, Slot(), "out");
    const ConvOut scv = sc ? *sc : ConvOut();
    tape_.push_back([=] {
      const int g = grad_of(out);
      conv_backward(co3, bn_backward(co3, dropblock_bwd(g, m3, ys)));
      if (mode_bn)
        conv_backward(scv, bn_backward(scv, dropblock_bwd(g, ms, ys)));
      else
        contribute_alias(x_ident, g);
    });
    return out;
  }

  // out = act(bn(y3) [*gate] + R); mode 1: R = bn(shortcut conv), 2: identity, 3: 2x upsample (tensor)
  int residual_tail(const ConvOut& co3, const ConvOut* sc, int sc_tensor, int b_mode, bool relu,
                    const SeGate& se = SeGate()) {
    const int out = b_mode == 1
                        ? bn_act(co3, relu, sc->y, sc->bn, 1, se.on ? se.e : Slot(), "out")
                        : bn_act(co3, relu, sc_tensor, -1, b_mode, se.on ? se.e : Slot(), "out");
    if (b_mode == 2 || b_mode == 3) use(sc_tensor);
    const ConvOut scv = sc ? *sc : ConvOut();
    tape_.push_back([=] {
      const int g = grad_of(out);
      int dy3;
      if (se.on) {
        const Shape ys = T(co3.y).shape;
        const int B = (int)ys[0], HW = (int)(ys[1] * ys[2]), C = (int)ys[3];
        const Slot de = slot(BUF_WORK, (int64_t)B * C), dq = slot(BUF_WORK, (int64_t)B * C);
        emit("se_bwd_gate", {{"g", vten(g)}, {"y", vten(co3.y)}, {"bn", vbn(co3.bn)}, {"de", vslot(de)},
                             {"B", vint(B)}, {"HW", vint(HW)}, {"C", vint(C)}, {"r", vint(se.r)}});
        emit("se_fc_bwd", {{"de", vslot(de)}, {"e", vslot(se.e)}, {"h", vslot(se.h)}, {"q", vslot(se.q)},
                           {"w1", vvar(se.w1)}, {"w2", vvar(se.w2)}, {"dq", vslot(dq)},
                           {"scratch", vslot(se.scratch)}, {"B", vint(B)}, {"HW", vint(HW)}, {"C", vint(C)},
                           {"r", vint(se.r)}});
        dy3 = bn_backward(co3, g, se.e, dq);
      } else if (b_mode == 1 && cfg_.fuse_bn_pairs) {
        const auto d = bn_backward2(co3, scv, g);
        conv_backward(co3, d.first);
        conv_backward(scv, d.second);
        return;
      } else {
        dy3 = bn_backward(co3, g);
      }
      conv_backward(co3, dy3);
      if (b_mode == 1) {
        conv_backward(scv, bn_backward(scv, g));
      } else if (b_mode == 2) {
        contribute_alias(sc_tensor, g);
      } else if (b_mode == 3) {
        const Shape s = T(sc_tensor).shape;
        contribute(sc_tensor, [=](int o, int add, int mask) {
          emit("upsample2x_bwd", {{"dout", vten(g)}, {"dx", vten(o)}, {"add_src", vten(add)},
                                  {"mask_src", vten(mask)}, {"B", vint(s[0])}, {"H", vint(s[1])},
                                  {"W", vint(s[2])}, {"C", vint(s[3])}});
        });
      }
    });
    return out;
  }

  SeGate se(const ConvOut& co3) {   // nets/blocks.py:156-184 on t = bn(y3)
    const Shape ys = T(co3.y).shape;
    const int B = (int)ys[0], HW = (int)(ys[1] * ys[2]), C = (int)ys[3], r = C / 16;
    SeGate g;
    g.on = true;
    g.r = r;
    {
      Scope s(*this, "se_block");
      g.w1 = variable(full("seblock_dense_1/kernel"), {1, 1, C, r}, "conv_kernel", {r, 1, 1, C}, true, true);
      g.w2 = variable(full("seblock_dense_2/kernel"), {1, 1, r, C}, "conv_kernel", {C, 1, 1, r}, true, true);
    }
    g.q = slot(BUF_WORK, (int64_t)B * C);
    g.h = slot(BUF_WORK, (int64_t)B * r);
    g.e = slot(BUF_WORK, (int64_t)B * C);
    g.scratch = slot(BUF_WORK, (int64_t)B * (C + r));
    emit("se_gap", {{"y", vten(co3.y)}, {"bn", vbn(co3.bn)}, {"q", vslot(g.q)}, {"B", vint(B)},
                    {"HW", vint(HW)}, {"C", vint(C)}, {"r", vint(r)}});
    emit("se_fc", {{"q", vslot(g.q)}, {"w1", vvar(g.w1)}, {"w2", vvar(g.w2)}, {"h", vslot(g.h)},
                   {"e", vslot(g.e)}, {"B", vint(B)}, {"HW", vint(HW)}, {"C", vint(C)}, {"r", vint(r)}});
    return g;
  }

  enum Shortcut { SC_NONE, SC_PROJ, SC_RESNET_D, SC_BL };
  static bool contains(const std::string& s, const char* sub) { return s.find(sub) != std::string::npos; }

  // nets/resnet_model.py:35-97 (_bottleneck_block_v1); db = DropBlock gamma_scale of this stage (< 0: off)
  int bottleneck(int x, int filters, Shortcut kind, int strides, bool last_relu = true, double db = -1) {
    if (!use_dropblock_) db = -1;
    const bool sconv = contains(cfg_.anti_alias_type, "sconv");
    ConvOut sc;
    bool has_sc = false;
    if (kind != SC_NONE) {
      int xs = x, k_s = 1;
      const Shape s = T(x).shape;
      const int H = (int)s[1], W = (int)s[2];
      if (kind == SC_PROJ) {
        if (contains(cfg_.anti_alias_type, "proj") && strides != 1)
          xs = blurpool(x, cfg_.anti_alias_filter_size, strides);
        else
          k_s = strides;
      } else if (kind == SC_RESNET_D) {
        xs = strides > 1 ? avgpool(x, 2, strides, 0, H / strides, W / strides, 1)
                         : avgpool(x, 2, 1, 0, H, W, 0);
      } else if (kind == SC_BL) {
        if (strides > 1)
          xs = avgpool(x, 3, strides, 1, (H + 2 - 3) / strides + 1, (W + 2 - 3) / strides + 1, 1);
      }
      sc = conv(xs, filters * 4, 1, k_s);
      has_sc = true;
    }
    DbMask ms;
    if (db >= 0 && has_sc) {
      const Shape s = T(sc.y).shape;
      ms = dropblock_mask((int)s[1], (int)s[2], (int)s[3], db);
    }
    int t = db < 0 ? cbr(x, filters, 1, 1) : cbr_db(x, filters, 1, 1, db);
    const int s3 = sconv ? 1 : strides;
    if (cfg_.use_sk_block) {
      t = sk(t, filters, s3);
      if (db >= 0) {   // :57-63 dropblock on the SK output
        const int v = t;
        const Shape vs = T(v).shape;
        const DbMask m = dropblock_mask((int)vs[1], (int)vs[2], (int)vs[3], db);
        t = dropblock_apply(v, m, false, "vd");
        use(v);
        const int td = t;
        tape_.push_back([=] {
          contribute(v, [=](int out, int add, int mask) {
            PLAN_ASSERT(add < 0 && mask < 0, "dropblock contribution with epilogue");
            emit_db_apply(grad_of(td), m, false, out, vs);
          });
        });
      }
    } else {
      t = db < 0 ? cbr(t, filters, 3, s3) : cbr_db(t, filters, 3, s3, db);
    }
    if (sconv && strides != 1) t = blurpool(t, cfg_.anti_alias_filter_size, strides);
    const ConvOut co3 = conv(t, filters * 4, 1, 1, true, cfg_.zero_gamma);
    if (db >= 0) return residual_tail_db(co3, has_sc ? &sc : nullptr, x, last_relu, db, ms);
    const SeGate g = cfg_.use_se_block ? se(co3) : SeGate();
    if (has_sc) return residual_tail(co3, &sc, -1, 1, last_relu, g);
    return residual_tail(co3, nullptr, x, 2, last_relu, g);
  }

  // nets/resnet_model.py:99-163: the first block always projects and never sees last_relu
  int block_layer(int x, int filters, int num_blocks, int strides, bool use_resnet_d = false,
                  bool use_bl = false, bool last_relu = true, double db = -1) {
    const Shortcut kind = use_resnet_d ? SC_RESNET_D : (use_bl ? SC_BL : SC_PROJ);
    x = bottleneck(x, filters, kind, strides, true, db);
    for (int i = 1; i < num_blocks; ++i)
      x = bottleneck(x, filters, SC_NONE, 1, i == num_blocks - 1 ? last_relu : true, db);
    return x;
  }

  void attach_bn(ConvOut& co) {   // BN created after a with_bn=False conv
    for (auto it = ops_->rbegin(); it != ops_->rend(); ++it) {
      const Val* y = it->find("y");
      if (it->kind == "conv" && y && y->i == co.y) {
        Val* st = it->find_mut("stats");
        *st = stats_of(co.bn);
        break;
      }
    }
    emit_bn_finalize(co.bn, co.y, co.geom);
  }

  void build(int H, int W);
};

void Builder::run() {
  const Config& c = cfg_;
  // nets/resnet_model.py:201-215 / functions/model_fns.py:131-135 argument checks
  if (c.resnet_version != 1 && c.resnet_version != 2)
    fail(ACNN_ERR_INVALID, "Resnet version should be 1 or 2. See README for citations.");
  if (c.resnet_size < 50)
    fail(ACNN_ERR_UNSUPPORTED, "non-bottleneck ResNets (nets/resnet_model.py:211-212)");
  if (!block_sizes(c.resnet_version, c.resnet_size))
    fail(ACNN_ERR_INVALID, "Could not find layers for selected Resnet size. Size received: %d", c.resnet_size);
  if (c.pool_type != "gap" && c.pool_type != "gem" && c.pool_type != "flatten")
    fail(ACNN_ERR_UNSUPPORTED, "pool_type='%s' (nets/resnet_model.py:560-573)", c.pool_type.c_str());
  if (c.embedding_size && (c.embedding_size < 32 || c.embedding_size > 2048 ||
                           (c.embedding_size & (c.embedding_size - 1))))
    fail(ACNN_ERR_INVALID, "embedding_size must be a power of two between 32 and 2048 (tensor-core N tile, "
         "channel groups of the batch-norm kernels)");
  if (c.loss_type != "softmax")
    fail(ACNN_ERR_UNSUPPORTED, "only the softmax loss is on the hot path");
  if (!c.anti_alias_type.empty() && (c.anti_alias_filter_size < 1 || c.anti_alias_filter_size > 7))
    fail(ACNN_ERR_INVALID, "anti_alias_filter_size must be in 1..7");
  if (c.resnet_version == 2 && (c.bl_alpha < 1 || c.bl_beta < 1 || (64 / c.bl_alpha) % 32))
    fail(ACNN_ERR_UNSUPPORTED, "bl_alpha=%d: the little branches would have %d channels, below the 32-channel "
         "tensor-core tile (bl_alpha 1 or 2)", c.bl_alpha, 64 / std::max(c.bl_alpha, 1));
  training_ = c.training;
  use_dropblock_ = c.use_dropblock && training_;
  if (use_dropblock_ && c.use_se_block) fail(ACNN_ERR_UNSUPPORTED, "use_dropblock together with use_se_block");
  kd_temp_ = training_ ? c.kd_temp : 0.0;
  fp32_ = c.fp32;
  adt_ = fp32_ ? ACNN_F32 : ACNN_BF16;
  if (c.height % 32 || c.width % 32 || c.height <= 0 || c.width <= 0)
    fail(ACNN_ERR_INVALID, "input size must be a multiple of 32 (got %dx%d)", c.height, c.width);
  if (c.mixup_type < 0 || c.mixup_type > 2) fail(ACNN_ERR_INVALID, "mixup_type must be 0, 1 or 2");
  if (c.batch < 1 || c.num_classes < 1) fail(ACNN_ERR_INVALID, "batch and num_classes must be positive");
  B_ = c.batch;
  mixup_type_ = training_ ? c.mixup_type : 0;
  with_loss_ = c.with_loss || training_;
  ops_ = &p_.forward;
  p_.cfg = c;
  p_.ld_logits = (int)round_up(c.num_classes, 128);
  p_.input_batch = mixup_type_ == 1 ? 2 * B_ : B_;
  build(c.height, c.width);
  // gradient readiness (assembled_cnn_b200/dp.py grad_buckets): the backward op after which the
  // gradient of a variable is final
  for (size_t i = 0; i < p_.backward.size(); ++i) {
    const Op& op = p_.backward[i];
    if (op.kind == "conv_wgrad" || op.kind == "sk_fc_bwd" || op.kind == "se_fc_bwd" ||
        op.kind == "s2d_wgrad_unpack")
      for (const char* key : {"w", "w1", "w2"}) {
        const Val* v = op.find(key);
        if (v && v->kind == Val::VAR) p_.vars[v->i].grad_ready_op = (int)i;
      }
    if (op.kind == "bn_bwd_finalize" || op.kind == "sk_fc_bwd") {
      const Val* b = op.find("bn");
      if (b && p_.bns[b->i].gamma >= 0) {
        p_.vars[p_.bns[b->i].gamma].grad_ready_op = (int)i;
        p_.vars[p_.bns[b->i].beta].grad_ready_op = (int)i;
      }
    }
  }
}

void Builder::build(int H, int W) {
  const Config& cfg = cfg_;
  const int B = B_, nf = 64, Bin = p_.input_batch;
  p_.images = tensor("images", {Bin, H, W, 3}, ACNN_F32);
  // the W axis of the packed input is physically zero-padded for the stem's taps
  int sp, sk2, wlo, whi;
  stem_s2d_taps(cfg.use_resnet_d ? 3 : 7, &sp, &sk2, &wlo, &whi);
  const int x0 = tensor("x0", {B, H / 2, W / 2 + wlo + whi, 16});
  emit("prep_weights", {});
  if (mixup_type_) {
    p_.lam1 = tensor("lam1", {Bin / 2}, ACNN_F32);
    if (mixup_type_ == 2) p_.lam2 = tensor("lam2", {Bin / 2}, ACNN_F32);
  }
  emit("pack_input", {{"images", vten(p_.images)}, {"lam1", vten(p_.lam1)}, {"lam2", vten(p_.lam2)},
                      {"mode", vint(mixup_type_)}, {"out", vten(x0)}, {"Bin", vint(Bin)}, {"H", vint(H)},
                      {"W", vint(W)}, {"wpad", vints({wlo, whi})}});

  const bool d = cfg.use_resnet_d;
  ConvOut co;
  int x;
  auto stem_cbr = [&](int xin, int filters, int k) {
    const ConvOut c = stem_conv(xin, filters, k);
    const int u = bn_act(c, true);
    tape_.push_back([=] { conv_backward(c, bn_backward(c, grad_of(u))); });
    return u;
  };
  if (d && cfg.resnet_version == 1) {
    x = stem_cbr(x0, nf / 2, 3);
    x = cbr(x, nf / 2, 3, 1);
    co = conv(x, nf, 3, 1, false);
    co.bn = bn_layer(nf, (int64_t)B * (H / 2) * (W / 2));
    attach_bn(co);
  } else if (d) {
    {
      Scope s(*this, "stage0");
      x = stem_cbr(x0, nf / 2, 3);
      x = cbr(x, nf / 2, 3, 1);
      co = conv(x, nf, 3, 1, false);
    }
    {
      Scope s(*this, "stage0");
      co.bn = bn_layer(nf, (int64_t)B * (H / 2) * (W / 2));
      attach_bn(co);
    }
  } else if (cfg.resnet_version == 2) {
    {
      Scope s(*this, "stage0");
      co = stem_conv(x0, nf, 7);
      // the BN after the first conv lives in a second 'stage0' scope (nets/resnet_model.py:359-381), so
      // its variable names differ from the conv's scope: give the name counter back ...
      counters_[{joined(), "batch_normalization"}] -= 1;
    }
    {
      Scope s(*this, "stage0");   // ... and rename its four variables (the last four created)
      const std::string layer = unique("batch_normalization");
      const BatchNorm& bn = p_.bns[co.bn];
      for (int id : {bn.gamma, bn.beta, bn.mm, bn.mv}) {
        Variable& v = p_.vars[id];
        v.name = full(layer + "/" + v.name.substr(v.name.rfind('/') + 1));
      }
    }
  } else {
    co = stem_conv(x0, nf, 7);
  }
  x = bn_act(co, true);
  {
    const ConvOut c = co;
    const int u = x;
    tape_.push_back([=] { conv_backward(c, bn_backward(c, grad_of(u))); });
  }

  if (cfg.resnet_version == 1) {
    x = maxpool(x, 3, 2);
  } else {
    Scope s(*this, "stage0/pool");   // BL module 0, resnet_model.py:385-419
    const ConvOut big0 = conv(x, nf, 3, 2);
    int l0 = cbr(x, nf / cfg.bl_alpha, 3, 1);
    l0 = cbr(l0, nf / cfg.bl_alpha, 3, 2);
    const ConvOut l0c = conv(l0, nf, 1, 1);
    x = residual_tail(big0, &l0c, -1, 1, true);
    x = cbr(x, nf, 1, 1);
  }

  const std::vector<int>& sizes = *block_sizes(cfg.resnet_version, cfg.resnet_size);
  int strides[4] = {1, 2, 2, 2};
  if (cfg.resnet_version == 2) { strides[0] = 2; strides[1] = 2; strides[2] = 1; strides[3] = 2; }
  if (cfg.no_downsample) strides[3] = 1;
  for (int i = 0; i < 4; ++i) {
    const int nb = sizes[i], f = nf << i;
    // dropblock_for_group3 (gamma_scale 0.25) / group4 (1.0): nets/resnet_model.py:432-453
    const double db = i == 2 ? 0.25 : (i == 3 ? 1.0 : -1.0);
    if (cfg.resnet_version == 2 && i < 3) {
      Scope s(*this, "stage" + std::to_string(i + 1));
      int big, le_x;
      ConvOut le;
      {
        Scope sb(*this, "big" + std::to_string(i + 1));
        big = block_layer(x, f, nb - 1, 2, false, true, false, db);
      }
      {
        Scope sl(*this, "little" + std::to_string(i + 1));
        le_x = block_layer(x, f / cfg.bl_alpha, std::max(1, nb / cfg.bl_beta - 1), 1, false, true, true, db);
        le = conv(le_x, f * 4, 1, 1);
      }
      {
        Scope sm(*this, "merge" + std::to_string(i + 1));
        x = residual_tail(le, nullptr, big, 3, true);
        x = block_layer(x, f, 1, strides[i], false, true, true, db);
      }
    } else if (cfg.resnet_version == 2) {
      Scope s(*this, "stage" + std::to_string(i + 1));
      x = block_layer(x, f, nb, strides[i], d, true, true, db);
    } else {
      x = block_layer(x, f, nb, strides[i], d, false, true, db);
    }
  }

  // head: pool -> [embedding conv + BN] -> dense (nets/resnet_model.py:552-599)
  const Shape xs = T(x).shape;
  const int Hx = (int)xs[1], Wx = (int)xs[2], Cx = (int)xs[3];
  const int nc = cfg.num_classes, ld = p_.ld_logits;
  use(x);
  int pooled;
  Slot gem_s;
  if (cfg.pool_type == "gap") {
    pooled = tensor("pooled", {B, Cx});
    emit("gap", {{"x", vten(x)}, {"out", vten(pooled)}, {"B", vint(B)}, {"HW", vint(Hx * Wx)}, {"C", vint(Cx)}});
  } else if (cfg.pool_type == "gem") {
    pooled = tensor("pooled", {B, Cx});
    gem_s = slot(BUF_WORK, (int64_t)B * Cx);
    emit("gem", {{"x", vten(x)}, {"out", vten(pooled)}, {"ssum", vslot(gem_s)}, {"B", vint(B)},
                 {"HW", vint(Hx * Wx)}, {"C", vint(Cx)}});
  } else {   // flatten, NHWC order (:568-571)
    pooled = tensor("pooled", {B, (int64_t)Hx * Wx * Cx});
    emit("grad_combine", {{"a", vten(x)}, {"out", vten(pooled)}, {"shape", vints(xs)}});
  }
  int Cf = (int)T(pooled).shape[1];
  int feat = pooled;
  ConvOut emb_co;
  bool has_emb = false;
  if (cfg.embedding_size > 0) {
    // 1x1 conv 'embedding_dense' (no bias) + BN 'embedding_dense_batch_normalization' on the [B,1,1,Cf]
    // pooled tensor (:575-584); return_embedding = the BN output; ReLU before dense
    const int E = cfg.embedding_size;
    const int we = variable("resnet_model/embedding_dense/kernel", {1, 1, Cf, E}, "conv_kernel",
                            {E, 1, 1, Cf}, true, true, false, training_);
    Geom ge;
    ge.B = B; ge.H = ge.W = 1; ge.Cin = Cf; ge.Cout = E; ge.kh = ge.kw = 1; ge.stride = 1;
    const int ye = tensor("y", {B, 1, 1, E});
    const int bne = bn_layer(E, B, false, "embedding_dense_batch_normalization");
    const int xp = planes(pooled);
    emit("conv", {{"x", vten(pooled)}, {"xp", vten(xp)}, {"w", vvar(we)}, {"y", vten(ye)},
                  {"geom", vgeom(ge)}, {"stats", stats_of(bne)}, {"out_f32", vint(0)}});
    emit_bn_finalize(bne, ye, ge);
    use(pooled);
    emb_co.x = pooled; emb_co.y = ye; emb_co.geom = ge; emb_co.w = we; emb_co.bn = bne;
    has_emb = true;
    p_.embedding = bn_act(emb_co, false, -1, -1, 0, Slot(), "embedding");
    feat = bn_act(emb_co, true, -1, -1, 0, Slot(), "embedding_relu");
    Cf = E;
  }
  const int wk = variable("resnet_model/dense/kernel", {Cf, nc}, "dense_kernel", {ld, 1, 1, Cf}, true, true,
                          false, training_);
  const int bk = variable("resnet_model/dense/bias", {nc}, "dense_bias", {ld}, true, true);
  const int logits = tensor("logits", {B, ld}, ACNN_F32);
  Geom gd;
  gd.B = B; gd.H = gd.W = 1; gd.Cin = Cf; gd.Cout = ld; gd.kh = gd.kw = 1; gd.stride = 1;
  {
    const int xp = planes(feat);
    emit("conv", {{"x", vten(feat)}, {"xp", vten(xp)}, {"w", vvar(wk)}, {"y", vten(logits)},
                  {"geom", vgeom(gd)}, {"bias", vvar(bk)}, {"out_f32", vint(1)}});
  }
  use(feat);
  p_.logits = logits;
  p_.pooled = pooled;
  p_.feature_shape = xs;
  p_.n_loss_first = (int)p_.forward.size();
  if (!with_loss_) return;
  p_.labels = tensor("labels", {Bin}, ACNN_I32);
  p_.ysoft = tensor("ysoft", {B, nc}, ACNN_F32);
  emit("mix_labels", {{"labels", vten(p_.labels)}, {"mode", vint(mixup_type_)}, {"y", vten(p_.ysoft)},
                      {"Bin", vint(Bin)}, {"NC", vint(nc)}, {"lam1", vten(p_.lam1)}, {"lam2", vten(p_.lam2)}});
  int yt = -1;
  if (kd_temp_ > 0) {
    // knowledge distillation (nets/run_loop_classification.py:86-96): the labels carry the teacher's
    // logits; teacher labels = softmax(. / T), mixed like the supervised labels
    p_.teacher_logits = tensor("teacher_logits", {Bin, nc}, ACNN_F32);
    yt = tensor("yteacher", {B, nc}, ACNN_F32);
    emit("kd_teacher", {{"teacher_logits", vten(p_.teacher_logits)}, {"labels", vten(p_.labels)},
                        {"mode", vint(mixup_type_)}, {"kd_temp", vflt(kd_temp_)}, {"yt", vten(yt)},
                        {"Bin", vint(Bin)}, {"NC", vint(nc)}, {"lam1", vten(p_.lam1)},
                        {"lam2", vten(p_.lam2)}});
  }
  p_.loss = slot(BUF_ZERO, 4);   // [cross_entropy, l2_loss, kd_loss, -]
  const int dlogits = tensor("dlogits", {B, ld});
  const Slot ce_work = slot(BUF_WORK, 2 * round_up(B, 32) + (int64_t)B * ld);
  emit("softmax_ce", {{"logits", vten(logits)}, {"y", vten(p_.ysoft)}, {"yt", vten(yt)},
                      {"kd_temp", vflt(kd_temp_)}, {"B", vint(B)}, {"NC", vint(nc)}, {"ld", vint(ld)},
                      {"label_smoothing", vflt(cfg.label_smoothing)}, {"loss", vslot(p_.loss)},
                      {"dlogits", vten(dlogits)}, {"dbias", training_ ? vvar(bk) : Val()},
                      {"work", vslot(ce_work)}});
  if (!training_) return;

  // ---------------- backward ----------------
  ops_ = &p_.backward;
  {
    const int xp = planes(feat);
    const int dyp = planes(dlogits);
    emit("conv_wgrad", {{"x", vten(feat)}, {"xp", vten(xp)}, {"dy", vten(dlogits)}, {"dyp", vten(dyp)},
                        {"geom", vgeom(gd)}, {"w", vvar(wk)}});
  }
  contribute(feat, [=](int out, int add, int mask) { emit_dgrad(dlogits, wk, out, gd, add, mask, -1); });
  if (has_emb) conv_backward(emb_co, bn_backward(emb_co, grad_of(feat)));
  const int dpooled = grad_of(pooled);
  contribute(x, [=](int out, int add, int mask) {
    PLAN_ASSERT(add < 0, "pool backward with an accumulated gradient");
    if (cfg_.pool_type == "gap") {
      emit("gap_bwd", {{"dpooled", vten(dpooled)}, {"mask_src", vten(mask)}, {"dx", vten(out)}, {"B", vint(B)},
                       {"HW", vint(Hx * Wx)}, {"C", vint(Cx)}});
    } else if (cfg_.pool_type == "gem") {   // x <= 0 is outside GeM's clip range: the ReLU mask is implied
      emit("gem_bwd", {{"dpooled", vten(dpooled)}, {"ssum", vslot(gem_s)}, {"x", vten(x)}, {"dx", vten(out)},
                       {"B", vint(B)}, {"HW", vint(Hx * Wx)}, {"C", vint(Cx)}});
    } else {
      emit("grad_combine", {{"a", vten(dpooled)}, {"mask_src", vten(mask)}, {"out", vten(out)},
                            {"shape", vints(xs)}});
    }
  });
  for (auto it = tape_.rbegin(); it != tape_.rend(); ++it) (*it)();
  // ---------------- update ----------------
  ops_ = &p_.update;
  emit("sgd", {{"loss", vslot(p_.loss)}, {"scratch", vslot(slot(BUF_WORK, kSgdScratch))}});
  for (size_t i = 0; i < p_.tensors.size(); ++i)
    PLAN_ASSERT(p_.tensors[i].contribs == p_.tensors[i].consumers || (int)i == x0,
                "gradient bookkeeping of %s: %d/%d", p_.tensors[i].name.c_str(), p_.tensors[i].contribs,
                p_.tensors[i].consumers);
}

// ---------------------------------------------------------------------------------------------- dump
std::string fmt_int(int64_t i) { return std::to_string(i); }
std::string fmt_flt(double f) {
  char b[64];
  snprintf(b, sizeof(b), "%.9g", f);
  return b;
}
std::string fmt_ints(const std::vector<int64_t>& v) {
  std::string s = "(";
  for (size_t i = 0; i < v.size(); ++i) s += (i ? "," : "") + std::to_string(v[i]);
  return s + ")";
}
std::string fmt_slot(const Slot& s) {
  if (s.buf == BUF_NONE) return "-";
  return std::string(s.buf == BUF_ZERO ? "zero" : "work") + ":" + std::to_string(s.offset) + ":" +
         std::to_string(s.size);
}

}  // namespace

std::string Plan::dump() const {
  auto vname = [&](int id) { return id >= 0 ? vars[id].name : std::string("-"); };
  auto fmt_bn = [&](const BatchNorm& b) {
    return "bn(C=" + fmt_int(b.C) + ",count=" + fmt_int(b.count) + ",gamma=" + vname(b.gamma) +
           ",beta=" + vname(b.beta) + ",mm=" + vname(b.mm) + ",mv=" + vname(b.mv) +
           ",stats=" + fmt_slot(b.stats) + ",work=" + fmt_slot(b.work) + ")";
  };
  auto fmt_val = [&](const Val& v) -> std::string {
    switch (v.kind) {
      case Val::INT: return fmt_int(v.i);
      case Val::FLT: return fmt_flt(v.f);
      case Val::STR: return v.s;
      case Val::TENSOR: return tensors[v.i].name;
      case Val::VAR: return vars[v.i].name;
      case Val::SLOT: return fmt_slot(v.slot);
      case Val::BN: return fmt_bn(bns[v.i]);
      case Val::GEOM: {
        const Geom& g = v.g;
        return "g" + fmt_ints({g.B, g.H, g.W, g.Cin, g.Cout, g.kh, g.kw, g.stride, g.pad_h_lo, g.pad_h_hi,
                               g.pad_w_lo, g.pad_w_hi});
      }
      case Val::INTS: return fmt_ints(v.v);
      default: return "-";
    }
  };
  std::string out;
  out += "sizes param_elems=" + fmt_int(param_elems) + " state_elems=" + fmt_int(state_elems) +
         " dgrad_elems=" + fmt_int(dgrad_elems) + " zero_elems=" + fmt_int(zero_elems) +
         " work_elems=" + fmt_int(work_elems) + "\n";
  std::map<std::string, std::string> meta;
  auto tname = [&](int id) { return tensors[id].name; };
  meta["batch"] = fmt_int(cfg.batch);
  meta["height"] = fmt_int(cfg.height);
  meta["width"] = fmt_int(cfg.width);
  meta["training"] = fmt_int(cfg.training);
  meta["mixup_type"] = fmt_int(cfg.training ? cfg.mixup_type : 0);
  meta["label_smoothing"] = fmt_flt(cfg.label_smoothing);
  meta["num_classes"] = fmt_int(cfg.num_classes);
  meta["ld_logits"] = fmt_int(ld_logits);
  meta["bn_momentum"] = fmt_flt(cfg.bn_momentum);
  meta["dtype"] = cfg.fp32 ? "fp32" : "bf16";
  meta["use_dropblock"] = fmt_int(cfg.use_dropblock && cfg.training);
  meta["kd_temp"] = fmt_flt(cfg.training ? cfg.kd_temp : 0.0);
  meta["input_batch"] = fmt_int(input_batch);
  meta["images"] = tname(images);
  if (lam1 >= 0) meta["lam1"] = tname(lam1);
  if (lam2 >= 0) meta["lam2"] = tname(lam2);
  meta["logits"] = tname(logits);
  meta["pooled"] = tname(pooled);
  meta["feature_shape"] = fmt_ints(feature_shape);
  if (embedding >= 0) meta["embedding"] = tname(embedding);
  if (labels >= 0) meta["labels"] = tname(labels);
  if (ysoft >= 0) meta["ysoft"] = tname(ysoft);
  if (loss.buf != BUF_NONE) meta["loss"] = fmt_slot(loss);
  if (teacher_logits >= 0) meta["teacher_logits"] = tname(teacher_logits);
  {
    std::string s = "(";
    for (size_t i = 0; i < dropblock_u.size(); ++i) s += (i ? "," : "") + tname(dropblock_u[i]);
    meta["dropblock_u"] = s + ")";
    s = "(";
    for (size_t i = 0; i < ones.size(); ++i)
      s += (i ? "," : "") + fmt_ints({ones[i].first, ones[i].second});
    meta["ones"] = s + ")";
  }
  for (const auto& kv : meta) out += "meta " + kv.first + "=" + kv.second + "\n";
  for (int buffer : {ACNN_BUF_PARAMS, ACNN_BUF_STATE})
    for (const auto& v : vars) {
      if (v.buffer != buffer) continue;
      out += "var " + v.name + " buffer=" + (buffer == ACNN_BUF_PARAMS ? "params" : "state") +
             " kind=" + v.kind + " tf_shape=" + fmt_ints(v.tf_shape) + " store_shape=" +
             fmt_ints(v.store_shape) + " offset=" + fmt_int(v.offset) + " size=" + fmt_int(v.size) +
             " decay=" + fmt_int(v.decay) + " zero_init=" + fmt_int(v.zero_init) + " dgrad_off=" +
             fmt_int(v.dgrad_off) + "\n";
    }
  for (const auto& t : tensors)
    out += "tensor " + t.name + " shape=" + fmt_ints(t.shape) + " dtype=" +
           (t.dtype == ACNN_BF16 ? "bf16" : (t.dtype == ACNN_F32 ? "f32" : "i32")) + " relu=" +
           fmt_int(t.relu) + "\n";
  const std::pair<const char*, const std::vector<Op>*> lists[] = {
      {"F", &forward}, {"B", &backward}, {"U", &update}};
  for (const auto& l : lists)
    for (size_t i = 0; i < l.second->size(); ++i) {
      const Op& op = (*l.second)[i];
      std::map<std::string, std::string> kv;
      for (const auto& a : op.a)
        if (a.second.kind != Val::NONE) kv[a.first] = fmt_val(a.second);
      out += std::string("op ") + l.first + " " + fmt_int((int64_t)i) + " " + op.kind;
      for (const auto& e : kv) out += " " + e.first + "=" + e.second;
      out += "\n";
    }
  return out;
}

int build_plan(const Config& cfg, Plan* out) {
  try {
    *out = Plan();
    Builder b(cfg, out);
    b.run();
    return ACNN_OK;
  } catch (const PlanError& e) {
    set_error("%s", e.msg.c_str());
    return e.code;
  } catch (const std::exception& e) {
    set_error("acnn_create: %s", e.what());
    return ACNN_ERR_INVALID;
  }
}

}  // namespace model
}  // namespace acnn
