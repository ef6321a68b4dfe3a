// Layer plan of the assembled-ResNet step (host logic, no CUDA): the C++ side of the model-level C ABI
// (include/acnn_model.h).  Walks the topology of nets/resnet_model.py:305-599 /
// functions/model_fns.py:98-198 once and records
//   * the variables in the reference's creation order with TF names (the weights ABI),
//   * the statically shaped buffers of one step,
//   * forward / backward / update op lists over them (the backward is emitted explicitly: each forward
//     module pushes a closure on a tape, closures run in reverse; a tensor read by several ops
//     accumulates its gradient through the consumers' fused epilogues, the last contribution applying the
//     ReLU mask, so a gradient buffer always holds dL/d(pre-ReLU)).
// model_exec.cu resolves the ops into launch records over bound device pointers.
#pragma once
#include <stdint.h>

#include "common.h"

#include <functional>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/acnn_model.h"

namespace acnn {
namespace model {

constexpr int64_t kAlign = 256;   // every tensor of a flat buffer starts at a multiple of 256 elements
// capacities (rows) of the per-CTA partial-sum buffers the reductions write
constexpr int64_t kStatsPartsCap = kMaxSms;
constexpr int64_t kBwdPartsCap = 2 * kMaxSms;
constexpr int64_t kSgdScratch = kMaxSms * 8 + 1;

inline int64_t round_up(int64_t n, int64_t a = kAlign) { return (n + a - 1) / a * a; }

enum { BUF_NONE = 0, BUF_ZERO = 1, BUF_WORK = 2 };
struct Slot {   // a small fp32 vector inside the "zero" (cleared every step) or "work" buffer
  int buf = BUF_NONE;
  int64_t offset = 0, size = 0;
};

struct Geom {
  int B = 0, H = 0, W = 0, Cin = 0, Cout = 0, kh = 0, kw = 0, stride = 1;
  int pad_h_lo = 0, pad_h_hi = 0, pad_w_lo = 0, pad_w_hi = 0;
  int Ho() const { return (H + pad_h_lo + pad_h_hi - kh) / stride + 1; }
  int Wo() const { return (W + pad_w_lo + pad_w_hi - kw) / stride + 1; }
};

using Shape = std::vector<int64_t>;
inline int64_t numel(const Shape& s) {
  int64_t n = 1;
  for (int64_t d : s) n *= d;
  return n;
}

struct Tensor {
  std::string name;
  Shape shape;
  int dtype = ACNN_BF16;   // ACNN_BF16 | ACNN_F32 | ACNN_F16 | ACNN_I32
  bool relu = false;       // output of a ReLU: its gradient gets masked by (t > 0)
  int consumers = 0;       // forward readers that will send a gradient back
  int contribs = 0;
  int grad = -1;           // tensor holding the accumulated gradient so far
  int64_t ws_offset = 0;   // bytes inside the workspace (set by layout())
  int64_t bytes() const { return numel(shape) * (dtype == ACNN_BF16 || dtype == ACNN_F16 ? 2 : 4); }
};

struct Variable {
  std::string name, kind;
  Shape tf_shape, store_shape;
  int buffer = ACNN_BUF_PARAMS;
  int64_t offset = 0, size = 0;
  bool decay = false, zero_init = false;
  int64_t dgrad_off = -1;
  int grad_ready_op = -1;
};

struct BatchNorm {   // a batch-norm layer instance: variables + per-step work slots
  int C = 0;
  int gamma = -1, beta = -1, mm = -1, mv = -1;   // variable ids (-1: identity BN of a DropBlock tail)
  int64_t count = 0;
  Slot stats;   // bf16 mode: [parts][sum | sumsq] rows of the conv epilogue; fp32 mode: [mean | var]
  Slot work;    // [scale | shift | mean | rstd]
};

struct Val {
  enum Kind { NONE, INT, FLT, STR, TENSOR, VAR, SLOT, BN, GEOM, INTS } kind = NONE;
  int64_t i = 0;
  double f = 0;
  std::string s;
  Slot slot;
  Geom g;
  std::vector<int64_t> v;
};
inline Val vint(int64_t i) { Val v; v.kind = Val::INT; v.i = i; return v; }
inline Val vflt(double f) { Val v; v.kind = Val::FLT; v.f = f; return v; }
inline Val vten(int id) { Val v; if (id >= 0) { v.kind = Val::TENSOR; v.i = id; } return v; }
inline Val vvar(int id) { Val v; if (id >= 0) { v.kind = Val::VAR; v.i = id; } return v; }
inline Val vslot(const Slot& s) { Val v; if (s.buf != BUF_NONE) { v.kind = Val::SLOT; v.slot = s; } return v; }
inline Val vbn(int id) { Val v; if (id >= 0) { v.kind = Val::BN; v.i = id; } return v; }
inline Val vgeom(const Geom& g) { Val v; v.kind = Val::GEOM; v.g = g; return v; }
inline Val vints(std::vector<int64_t> l) { Val v; v.kind = Val::INTS; v.v = std::move(l); return v; }

struct Op {
  std::string kind;
  std::vector<std::pair<std::string, Val>> a;
  const Val* find(const char* key) const {
    for (const auto& kv : a)
      if (kv.first == key) return kv.second.kind == Val::NONE ? nullptr : &kv.second;
    return nullptr;
  }
  Val* find_mut(const char* key) {
    for (auto& kv : a)
      if (kv.first == key) return &kv.second;
    return nullptr;
  }
};

struct Config {
  int resnet_size = 50, num_classes = 1001, resnet_version = 1;
  bool no_downsample = false, zero_gamma = false, use_se_block = false, use_sk_block = false;
  double bn_momentum = 0.997, bn_epsilon = 1e-5;
  int embedding_size = 0, anti_alias_filter_size = 0;
  std::string anti_alias_type, pool_type = "gap", loss_type = "softmax";
  int bl_alpha = 2, bl_beta = 4;
  bool use_resnet_d = false;
  int batch = 32, height = 224, width = 224;
  bool training = true;
  int mixup_type = 0;
  bool with_loss = true;
  bool fp32 = false, use_dropblock = false;
  bool fp16 = false;   // the bf16 plan with fp16 activation storage (ACNN_F16); exclusive with fp32
  int deterministic = -1;
  bool fuse_bn_pairs = true;
  double label_smoothing = 0, kd_temp = 0, loss_scale = 1;
};

struct Plan {
  Config cfg;
  std::vector<Tensor> tensors;
  std::vector<Variable> vars;   // creation order, trainables and moving statistics interleaved
  std::vector<BatchNorm> bns;
  std::vector<Op> forward, backward, update;
  int64_t param_elems = 0, state_elems = 0, dgrad_elems = 0, zero_elems = 0, work_elems = 0;
  int n_loss_first = 0;
  // roles
  int images = -1, lam1 = -1, lam2 = -1, logits = -1, pooled = -1, embedding = -1, labels = -1,
      ysoft = -1, teacher_logits = -1;
  std::vector<int> dropblock_u;
  std::vector<std::pair<int64_t, int64_t>> ones;   // identity-BN scale vectors: (work offset, C)
  Slot loss;
  Shape feature_shape;
  int input_batch = 0, ld_logits = 0;
  std::string dump() const;
};

// Returns ACNN_OK or an error code with acnn::set_error() text.
int build_plan(const Config& cfg, Plan* out);

}  // namespace model
}  // namespace acnn
