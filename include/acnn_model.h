/*
 * acnn_model.h -- MODEL-LEVEL C ABI of libacnn.so: the whole assembled-ResNet training /
 * inference step behind one handle.  acnn.h is the op level (one entry point per TF graph op the
 * reference emits); this header is the level a host in any language binds when it wants the reference's
 * `Model(...)` + `model(inputs, training)` + `resnet_model_fn` TRAIN branch as a drop-in:
 *
 *   reference (Python / TF 1.14)                                   here
 *   ------------------------------------------------------------   ---------------------------------
 *   functions/model_fns.py:141-198   Model.__init__ (flags)         acnn_model_config + acnn_create
 *   nets/resnet_model.py:305-599     Model.__call__ (graph build)   acnn_create (layer plan, C++)
 *   tf.global_variables() in creation order, scope resnet_model/    acnn_variable_count / _info
 *   utils/data_util.py:97-158        mixup                          acnn_forward (pack_input op)
 *   losses/cls_losses.py:28-33, run_loop_classification.py:141-179  acnn_loss
 *   nets/optimizer_setting.py:30     tf.gradients                   acnn_backward(_range)
 *   nets/optimizer_setting.py:23-38  MomentumOptimizer.apply        acnn_sgd_step
 *   session.run(train_op)                                           acnn_step (or a CUDA graph of it)
 *
 * Ownership: the library never allocates device memory.  The caller owns the flat fp32 variable
 * buffers (params / grads / momentum / state), the bf16 operand copies of the weights and ONE
 * workspace of acnn_model_sizes.workspace_bytes; acnn_bind() records the pointers and lays the step's
 * statically shaped buffers out inside the workspace.  The handle owns host memory only (the layer plan
 * and the resolved launch records).
 *
 * Every call returns 0 or an ACNN_ERR_* code (acnn_last_error() has the text), never throws across
 * the ABI, only ENQUEUES on `stream` (a cudaStream_t passed as void*), performs no hidden
 * synchronisation after acnn_bind(), allocates nothing but the stream-ordered split-K scratch of the
 * wgrad / small GEMM launches (cudaMallocAsync / cudaFreeAsync on `stream`: per stream, and graph
 * memory nodes under capture), and is CUDA-graph capturable (inputs are read from
 * the static input buffers inside the workspace; hyper-parameters from the device vector `hp`).
 * One host thread per handle; the calling thread's current CUDA device must be the one that owns the
 * bound buffers (one process per GPU sets it once).  acnn_create() needs no GPU (the layer plan is host
 * logic).
 */
#ifndef ACNN_MODEL_H_
#define ACNN_MODEL_H_

#include <stdint.h>

#include "acnn.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct acnn_model acnn_model;

/* Constructor flags of functions/model_fns.py:141-157 (+ the call-time use_resnet_d of
 * nets/resnet_model.py:308) and the static shape / mode of the step this handle executes. */
typedef struct acnn_model_config {
  int32_t struct_size;            /* = sizeof(acnn_model_config): ABI version check */
  int32_t resnet_size;            /* 50 | 101 | 152 | 200 */
  int32_t num_classes;            /* 1001 for ImageNet (class 0 = background) */
  int32_t resnet_version;         /* 1 | 2 (2 = Big-Little "assemble" topology) */
  int32_t no_downsample, zero_gamma, use_se_block, use_sk_block;
  int32_t embedding_size;         /* 0 = off */
  int32_t anti_alias_filter_size; /* 1..7 when anti_alias_type is set */
  int32_t bl_alpha, bl_beta;
  int32_t use_resnet_d;
  char anti_alias_type[32];       /* "", "sconv", "proj", "sconv,proj" ... (substring tests) */
  char pool_type[16];             /* "gap" | "gem" | "flatten" */
  char loss_type[16];             /* "softmax" */
  double bn_momentum;             /* 0.997 */
  double bn_epsilon;              /* 1e-5 (nets/model_helper.py:23) */
  /* step shape and mode */
  int32_t batch, height, width;   /* per-replica batch of the step; H, W multiples of 32 */
  int32_t training;               /* 1: batch statistics + backward + SGD; 0: moving statistics */
  int32_t mixup_type;             /* 0 | 1 (input batch = 2*batch) | 2 */
  int32_t with_loss;              /* eval: also run the loss ops */
  int32_t dtype;                  /* ACNN_BF16 | ACNN_F32 (parity mode) | ACNN_F16 (the reference's fp16) */
  int32_t use_dropblock;
  int32_t deterministic;          /* -1: only in the fp32 mode; 0 / 1 */
  int32_t fuse_bn_pairs;          /* 1 (default): one backward pass for the two BNs of a projection block */
  double label_smoothing;
  double kd_temp;                 /* > 0: knowledge-distillation term */
  double loss_scale;              /* nets/optimizer_setting.py:30-33; 1 = off */
} acnn_model_config;

/* config -> defaults of the reference's flags (resnet_size 50, version 1, 224 x 224, batch 32 ...). */
void acnn_model_config_init(acnn_model_config* cfg);

int acnn_create(const acnn_model_config* cfg, acnn_model** out);
void acnn_destroy(acnn_model* m);

typedef struct acnn_model_sizes {
  int64_t param_elems;     /* fp32 elements of params / grads / momentum (tensors 256-aligned) */
  int64_t state_elems;     /* fp32 elements of the BN moving statistics buffer */
  int64_t dgrad_elems;     /* 16-bit elements of one plane of the dgrad-layout weight copies */
  int64_t w_fprop_elems;   /* 16-bit (bf16, fp16 in ACNN_F16) elements the caller allocates for w_fprop
                              (planes * param_elems) */
  int64_t w_dgrad_elems;   /* 16-bit elements the caller allocates for w_dgrad (training only) */
  int64_t workspace_bytes;
  /* byte offsets inside the workspace of the pieces a host reads or writes directly */
  int64_t hp_offset;          /* float[8]: lr, momentum, weight_decay, grad_scale, dropblock keep_prob,
                                 global step (uint32 bits), 2 spare */
  int64_t loss_offset;        /* float[4]: cross_entropy, l2_loss, kd_loss, - ; -1 without loss ops */
  int64_t decay_flags_offset; /* uint8 per 256 elements of params: weight decay applies */
  int64_t zero_offset, zero_bytes;   /* cleared at the start of every step */
  int64_t work_offset, work_bytes;
  int32_t n_variables, n_tensors;
  int32_t n_forward, n_loss_first;   /* forward ops; index of the first loss op (= n_forward if none) */
  int32_t n_backward, n_update;
  int32_t input_batch;        /* examples the input pipeline delivers per step (2*batch for mixup 1) */
  int32_t ld_logits;          /* leading dimension of the logits buffer (num_classes rounded to 128) */
} acnn_model_sizes;
int acnn_model_get_sizes(const acnn_model* m, acnn_model_sizes* out);

/* Variables in the reference's creation order, TF names ("resnet_model/stage1/big1/conv2d/kernel").
 * tf_shape is the reference's layout (HWIO kernels, [in,out] dense); store_shape how the flat buffer
 * holds it (OHWI kernels, dense rows padded to ld_logits). */
#define ACNN_BUF_PARAMS 0
#define ACNN_BUF_STATE 1
typedef struct acnn_variable_info {
  char name[160];
  char kind[24];           /* conv_kernel | dense_kernel | dense_bias | gamma | beta | moving_mean | moving_variance */
  int32_t buffer;          /* ACNN_BUF_PARAMS (trainable) | ACNN_BUF_STATE */
  int32_t tf_rank, store_rank;
  int64_t tf_shape[4], store_shape[4];
  int64_t offset, size;    /* elements, inside its buffer */
  int64_t dgrad_off;       /* element offset of the dgrad-layout bf16 copy, -1 if none */
  int32_t decay;           /* weight decay applies (run_loop_classification.py:166-177) */
  int32_t zero_init;       /* gamma initialised to 0 (zero_gamma) */
  int32_t grad_ready_op;   /* index of the backward op after which its gradient is final, -1 if none */
  int32_t reserved_;
} acnn_variable_info;
int acnn_variable_count(const acnn_model* m);
int acnn_variable_info_get(const acnn_model* m, int i, acnn_variable_info* out);

/* Layout conversion of variable i between the reference's layout (`tf_values`: prod(tf_shape) floats --
 * HWIO conv kernels, [in,out] dense kernel, [classes] bias: what a TF checkpoint holds, utils/
 * checkpoint_utils.py) and the stored one (`stored`: info.size floats at info.offset of its buffer --
 * OHWI kernels, dense rows / bias zero-padded to ld_logits).  Host arrays, no GPU: a C host converts a
 * checkpoint tensor and copies it to params + offset (or state + offset) itself. */
int acnn_variable_pack(const acnn_model* m, int i, const float* tf_values, float* stored);
int acnn_variable_unpack(const acnn_model* m, int i, const float* stored, float* tf_values);

/* The statically shaped activation / gradient / input buffers of the step (inside the workspace). */
#define ACNN_I32 2
typedef struct acnn_tensor_info {
  char name[64];
  int32_t dtype;           /* ACNN_BF16 | ACNN_F32 | ACNN_F16 | ACNN_I32 */
  int32_t rank;
  int64_t shape[5];
  int64_t offset;          /* bytes, inside the workspace */
} acnn_tensor_info;
int acnn_tensor_count(const acnn_model* m);
int acnn_tensor_info_get(const acnn_model* m, int i, acnn_tensor_info* out);
/* role: "images" [input_batch,H,W,3] f32 | "labels" [input_batch] i32 | "lam1" | "lam2" |
 * "teacher_logits" | "logits" [batch, ld_logits] f32 | "pooled" | "embedding" | "ysoft" |
 * "dropblock_u" (index = DropBlock call in the reference's order).  Returns the tensor id or -1. */
int acnn_find_tensor(const acnn_model* m, const char* role, int index);

/* Records the caller-owned device buffers, lays the workspace out and enqueues its one-time
 * initialisation on `stream` (memset, weight descriptor table, decay flags, default hp).  grads /
 * momentum / w_dgrad may be NULL for an inference handle.  Variables are NOT initialised here (the
 * caller loads a checkpoint or draws the reference's initializers); moving variances must be set.
 * The row counts of the partial-statistics buffers (acnn_conv_stats_parts() ...) are resolved here: set
 * the tuning knobs of acnn.h that change them (acnn_set_conv_cta_pairs / _halo / _mtiles ...) BEFORE
 * binding, or bind again after changing one. */
int acnn_bind(acnn_model* m, float* params, float* grads, float* momentum, float* state,
              void* w_fprop, void* w_dgrad, void* workspace, void* stream);

/* Host-only self-check, no GPU: resolves every op of the plan against synthetic buffer addresses exactly as
 * acnn_bind would (same launch-record construction, nothing is launched or copied) and reports the first
 * op that cannot be resolved -- a partial-statistics slot or scratch area of the plan smaller than the row
 * count / scratch size the op level asks for (acnn_conv_stats_parts, acnn_bn_bwd_reduce_parts,
 * acnn_sk_fc_scratch_floats, acnn_dropblock_scratch_floats ...), a missing weight layout, an unknown op.
 * Leaves the handle as it was (bound or not). */
int acnn_validate(acnn_model* m);

/* Mutable step settings (read at enqueue time, not captured values of a CUDA graph's kernels: the
 * loss scale is a kernel argument, so re-capture after changing it). */
int acnn_set_loss_scale(acnn_model* m, double loss_scale);
/* Dynamic loss scaling (the rules at acnn_loss_scale_state in acnn.h) on a bound training handle.  state_dev:
 * caller-owned DEVICE memory of one acnn_loss_scale_state, initialised here on `stream` to {initial_scale, 0,
 * 0, 0, initial_scale}; the caller may overwrite it between steps (a resumed run).  growth_interval >= 1;
 * grad_divisor: the data-parallel replicas the gradient buffer sums (world * replicas per device; 1 for one
 * model on one device).  From then on the loss op seeds scale / B from the state, and acnn_sgd_step (so
 * acnn_step) runs acnn_grads_nonfinite over the gradients, the skip-aware SGD and acnn_loss_scale_update:
 * no host read, capturable.  hp[3] is not read and acnn_set_loss_scale's value is not used.  NULL state_dev
 * returns the handle to its static scale.  Read at enqueue time: re-capture after a change. */
int acnn_set_dynamic_loss_scale(acnn_model* m, acnn_loss_scale_state* state_dev, double initial_scale,
                                int growth_interval, int grad_divisor, void* stream);
/* Copies the dynamic loss-scale state (32 bytes) to a host or device `out` on `stream`;
 * ACNN_ERR_INVALID when dynamic scaling is not enabled. */
int acnn_get_loss_scale_state(acnn_model* m, acnn_loss_scale_state* out, void* stream);
/* DropBlock randomness: Philox key, and feed != 0 takes the uniforms from the "dropblock_u" tensors. */
int acnn_set_dropblock(acnn_model* m, uint64_t seed, int feed_uniforms);

/* Copies host OR device arrays (cudaMemcpyDefault) into the static input buffers; NULL skips one. */
int acnn_set_inputs(acnn_model* m, const float* images, const int32_t* labels, const float* lam1,
                    const float* lam2, const float* teacher_logits, void* stream);
/* "images" = (float)images_dev - mean3[c] (acnn_images_from_u8) from uint8 NHWC [input_batch,H,W,3]:
 * a quarter of the bytes of the fp32 input to copy to the device, one extra pass on it.  images_dev
 * must be a DEVICE array (the caller stages its own buffer; a host pointer is ACNN_ERR_INVALID);
 * mean3: float[3], host or device. */
int acnn_set_images_u8(acnn_model* m, const uint8_t* images_dev, const float* mean3, void* stream);
/* "images" [input_batch,S,S,3] from a batch of decoded uint8 images of any sizes through
 * acnn_resize_crop_u8 (resize, central crop, - mean3[c]), S = the plan's H = W.  desc_dev: a DEVICE
 * array of input_batch acnn_resize_desc (checked by the caller, see acnn_resize_crop_u8); rows >=
 * n_valid are not written; mean3: float[3], host or device. */
int acnn_set_images_resized(acnn_model* m, const acnn_resize_desc* desc_dev, int n_valid, const float* mean3,
                            void* stream);
/* "images" [input_batch,S,S,3] from a batch of training crop windows through acnn_crop_resize_u8 (flip,
 * resize to S x S, - mean3[c]), S = the plan's H = W.  Every one of the input_batch rows is written (a
 * training batch has no padding).  desc_dev: a DEVICE array of input_batch acnn_crop_desc (checked by
 * the caller, see acnn_crop_resize_u8; a host pointer is ACNN_ERR_INVALID); mean3: float[3], host or
 * device. */
int acnn_set_images_cropped(acnn_model* m, const acnn_crop_desc* desc_dev, const float* mean3, void* stream);
/* acnn_set_images_cropped with AutoAugment: every row through acnn_crop_resize_autoaugment_u8 (flip, resize,
 * clip and truncate to uint8, the two operations of aug_dev[b], - mean3[c]).  desc_dev, aug_dev: DEVICE
 * arrays of input_batch descriptors, work_dev a DEVICE buffer of acnn_autoaugment_work_bytes(input_batch, S)
 * bytes (host pointers are ACNN_ERR_INVALID); mean3: float[3], host or device. */
int acnn_set_images_augmented(acnn_model* m, const acnn_crop_desc* desc_dev, const acnn_autoaugment_desc* aug_dev,
                              uint8_t* work_dev, const float* mean3, void* stream);
/* float hp[8] as in acnn_model_sizes.hp_offset. */
int acnn_set_hparams(acnn_model* m, const float* hp, void* stream);
/* logits [batch, num_classes] fp32 (dense, ld = num_classes) / loss float[4] to a host or device array. */
int acnn_get_logits(acnn_model* m, float* out, void* stream);
int acnn_get_loss(acnn_model* m, float* out, void* stream);

/* The step, piecewise (each only enqueues): */
int acnn_forward(acnn_model* m, void* stream);   /* clear step buffers, weights -> bf16, mixup, network */
int acnn_loss(acnn_model* m, void* stream);      /* label mixup, (KD teacher), softmax CE + dlogits */
int acnn_backward(acnn_model* m, void* stream);  /* all gradients into the flat buffer */
/* Backward ops [first, last): lets a data-parallel host all-reduce a gradient bucket as soon as
 * acnn_variable_info.grad_ready_op of all its variables has run. */
int acnn_backward_range(acnn_model* m, int first, int last, void* stream);
/* weight decay + momentum + L2 loss, from hp; with dynamic loss scaling also the finiteness check before and
 * the scale update after (acnn_set_dynamic_loss_scale) */
int acnn_sgd_step(acnn_model* m, void* stream);
int acnn_step(acnn_model* m, void* stream);      /* forward + loss + backward + sgd_step */
/* Several data-parallel replicas per device (acnn_replica_accumulate of acnn.h over this handle's grads,
 * state and loss): a global step of R = `replicas` replicas is
 *   SAVE; for r in 0 .. R-1: forward, loss, backward, then FIRST (r = 0) | MIDDLE | LAST (r = R-1); sgd_step
 * with hp[3] (grad_scale) = 1 / (R * loss_scale).  The gradient part covers [lo, hi) of grads; the moving
 * statistics and the loss go with the call whose range starts at lo = 0, so a data-parallel host can close
 * each gradient bucket right before its all-reduce.  After LAST: grads = g0 + g1 + ... in replica order, state
 * and loss = the mean of the R copies (sum in replica order, times 1/R in fp32).  SAVE ignores lo / hi.
 * Caller-owned device accumulators: acc_grads param_elems floats (same offsets as grads), state_base
 * state_elems floats, acc_state state_elems + ACNN_REPLICA_LOSS_FLOATS floats (the tail sums the loss).
 * They hold nothing between global steps. */
#define ACNN_REPLICA_LOSS_FLOATS 4
int acnn_replica_accumulate_model(acnn_model* m, int phase, float* acc_grads, float* state_base, float* acc_state,
                                  int64_t lo, int64_t hi, int replicas, void* stream);
/* Any op range of a phase (0 forward incl. loss ops, 1 backward, 2 update): profiling / tests.
 * Does not clear the step buffers (acnn_clear_step_buffers does). */
int acnn_run_ops(acnn_model* m, int phase, int first, int last, void* stream);
int acnn_clear_step_buffers(acnn_model* m, void* stream);
/* Kind name of an op ("conv", "bn_act", ...), NULL when out of range. */
const char* acnn_op_kind(const acnn_model* m, int phase, int index);

/* Geometry of a GEMM op (kind "conv" | "conv_dgrad" | "conv_wgrad") as the plan states it, its
 * algorithmic multiply-accumulates (the stem's k x k x 3 conv, not its space-to-depth form; the
 * stride-2 transposed conv, not its zero-inserted stride-1 form) and the number of extra tiles its
 * epilogue reads (add_src / mask_src): what a roofline needs.  ACNN_ERR_INVALID for other ops. */
int acnn_op_conv_info(const acnn_model* m, int phase, int index, acnn_conv_geom* g, int64_t* alg_macs,
                      int* aux_tiles);

/* Canonical text of the layer plan (sizes, meta, variables, tensors, ops): returns the byte count
 * needed (including the terminator); writes at most cap bytes.  Test / debugging aid. */
int64_t acnn_plan_dump(const acnn_model* m, char* buf, int64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* ACNN_MODEL_H_ */
