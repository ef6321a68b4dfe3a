"""CPU oracle, part 2: the assembled-ResNet forward pass, loss and SGD step (torch CPU, fp32/fp64).

TEST INFRASTRUCTURE ONLY (see oracle/tf_ops.py header).  PINNED against the reference's own code:
the reference's nets/resnet_model.py + nets/blocks.py + nets/model_helper.py are executed through
a TF-1.14 API stand-in (tests/golden/tf1_shim) to produce tests/golden/reference_shim_golden.json;
tests/test_reference_shim_golden_cpu.py checks this file's variable inventory (names, shapes,
initializers, creation order: 11 configurations up to ResNet-152) and, in float64 to 1e-6, its logits
(inference and training mode), BN moving statistics, loss and gradient digests against it -- plus
DropBlock through the whole model, the knowledge-distillation branches and BASELINE config 3 as the
reference composes it (mixup -> model -> smoothed cross-entropy -> gradients).  The stand-in's kernels
are not this package's: 'SAME' padding is Hugging Face's TF port, batch norm / convolution / pooling are
ATen's (it does not import oracle/).  What stays unpinned is TensorFlow 1.14 itself (not installable).

Restates nets/resnet_model.py:35-599 (Model.__call__, block_layer, _bottleneck_block_v1),
functions/model_fns.py:98-198 (topology constants), nets/run_loop_classification.py:86-179 (loss
assembly) and nets/optimizer_setting.py:23-38 (momentum step) on top of oracle/tf_ops.py.
Gradients come from torch autograd over this forward.

Variables are created in the reference's program order with TF-style names; kernels
are HWIO, dense kernel [in, out] -- the "TF layout" that the product's set_weights() consumes.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

from . import tf_ops as T

BLOCK_SIZES = {   # functions/model_fns.py:113-127
    1: {50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3], 200: [3, 24, 36, 3]},
    2: {50: [3, 4, 6, 3], 101: [4, 8, 18, 3], 152: [5, 12, 30, 3]},
}


class VarStore:
    """Ordered variable store with TF-1.x style scoping / auto-uniquified layer names."""

    def __init__(self, seed=42, dtype=torch.float32):
        self.vars = OrderedDict()       # name -> tensor (trainable and not)
        self.trainable = OrderedDict()  # name -> bool
        self.kind = OrderedDict()
        self.gen = torch.Generator().manual_seed(seed)
        self.dtype = dtype
        self.creating = True
        self._scope = ["resnet_model"]
        self._counters = {}

    # -- scoping ---------------------------------------------------------------------------
    def _unique(self, base):
        key = ("/".join(self._scope), base)
        n = self._counters.get(key, 0)
        self._counters[key] = n + 1
        return base if n == 0 else "%s_%d" % (base, n)

    def scope(self, default_name):
        store = self

        class _Ctx:
            def __enter__(self_inner):
                store._scope.append(store._unique(default_name))

            def __exit__(self_inner, *a):
                store._scope.pop()
        return _Ctx()

    def reset_walk(self):
        self._scope = ["resnet_model"]
        self._counters = {}
        self.creating = False

    # -- variables -------------------------------------------------------------------------
    def _get(self, name, shape, kind, trainable, init):
        full = "/".join(self._scope + [name])
        if self.creating:
            assert full not in self.vars, full
            self.vars[full] = init().to(self.dtype)
            self.trainable[full] = trainable
            self.kind[full] = kind
        v = self.vars[full]
        assert tuple(v.shape) == tuple(shape), (full, v.shape, shape)
        return full, v

    def conv_kernel(self, layer, k, cin, cout, var="kernel"):
        """tf.variance_scaling_initializer(): truncated normal, std = sqrt(1/fan_in)/.8796."""
        fan_in = k * k * cin
        std = math.sqrt(1.0 / fan_in) / 0.87962566103423978

        def init():
            w = torch.empty(k, k, cin, cout)
            torch.nn.init.trunc_normal_(w, 0.0, std, -2 * std, 2 * std, generator=self.gen)
            return w
        return self._get("%s/%s" % (layer, var), (k, k, cin, cout), "conv_kernel", True, init)

    def dense(self, layer, cin, cout):
        lim = math.sqrt(6.0 / (cin + cout))   # glorot_uniform

        def init_k():
            return (torch.rand(cin, cout, generator=self.gen) * 2 - 1) * lim
        k = self._get(layer + "/kernel", (cin, cout), "dense_kernel", True, init_k)
        b = self._get(layer + "/bias", (cout,), "dense_bias", True, lambda: torch.zeros(cout))
        return k, b

    def bn(self, layer, c, zero_gamma=False):
        g = self._get(layer + "/gamma", (c,), "gamma", True,
                      lambda: torch.zeros(c) if zero_gamma else torch.ones(c))
        b = self._get(layer + "/beta", (c,), "beta", True, lambda: torch.zeros(c))
        mm = self._get(layer + "/moving_mean", (c,), "moving_mean", False, lambda: torch.zeros(c))
        mv = self._get(layer + "/moving_variance", (c,), "moving_variance", False,
                       lambda: torch.ones(c))
        return g, b, mm, mv


class OracleModel:
    """functions/model_fns.py:138-198 Model + nets/resnet_model.py:166-599."""

    def __init__(self, resnet_size, num_classes=1001, resnet_version=1, no_downsample=False,
                 zero_gamma=False, use_se_block=False, use_sk_block=False, bn_momentum=0.997,
                 embedding_size=0, anti_alias_filter_size=0, anti_alias_type="", pool_type="gap",
                 bl_alpha=2, bl_beta=4):
        if resnet_version not in (1, 2):
            raise ValueError("Resnet version should be 1 or 2. See README for citations.")
        if resnet_size < 50:
            raise NotImplementedError("non-bottleneck blocks (nets/resnet_model.py:211-212)")
        try:
            self.block_sizes = BLOCK_SIZES[resnet_version][resnet_size]
        except KeyError:
            raise ValueError("Could not find layers for selected Resnet size.")
        self.block_strides = [2, 2, 1, 2] if resnet_version == 2 else [1, 2, 2, 2]
        if no_downsample:
            self.block_strides[-1] = 1
        self.num_classes = num_classes
        self.rv = resnet_version
        self.zero_gamma = zero_gamma
        self.use_se = use_se_block
        self.use_sk = use_sk_block
        self.bn_momentum = bn_momentum
        self.embedding_size = embedding_size
        self.aa_size = anti_alias_filter_size
        self.aa_type = anti_alias_type
        self.pool_type = pool_type
        self.alpha, self.beta = bl_alpha, bl_beta
        self.num_filters = 64

    # -- layer helpers (each consumes variables from the store in program order) -------------
    def _conv(self, vs, x, filters, k, s):
        name, w = vs.conv_kernel(vs._unique("conv2d"), k, x.shape[-1], filters)
        return T.conv2d_fixed_padding(x, w, s)

    def _bn(self, vs, x, training, zero_gamma=False, layer=None):
        layer = layer or vs._unique("batch_normalization")
        (gn, g), (bn_, b), (mmn, mm), (mvn, mv) = vs.bn(layer, x.shape[-1], zero_gamma)
        y, nmm, nmv = T.batch_norm(x, g, b, mm, mv, training, self.bn_momentum)
        if training:
            self.bn_updates[mmn] = nmm
            self.bn_updates[mvn] = nmv
        return y

    def _sk(self, vs, x, filters, strides, training):
        """nets/blocks.py:110-154."""
        y = torch.relu(self._bn(vs, self._conv(vs, x, filters * 2, 3, strides), training))
        d = max(int(filters / 2), 32)
        with vs.scope("sk_block"):
            _, w1 = vs.conv_kernel("sk_fc_1", 1, filters, d)
            (gn, g), (bn_, b), (mmn, mm), (mvn, mv) = vs.bn("batch_normalization", d)
            _, w2 = vs.conv_kernel("sk_fc_2", 1, d, filters * 2)
            v, nmm, nmv = T.sk_attention(y, w1[0, 0], g, b, mm, mv, w2[0, 0], training,
                                         self.bn_momentum)
            if training:
                self.bn_updates[mmn] = nmm
                self.bn_updates[mvn] = nmv
        return v

    def _se(self, vs, x):
        c = x.shape[-1]
        with vs.scope("se_block"):
            _, w1 = vs.conv_kernel("seblock_dense_1", 1, c, c // 16)
            _, w2 = vs.conv_kernel("seblock_dense_2", 1, c // 16, c)
        return T.se_block(x, w1[0, 0], w2[0, 0])

    def _dropblock(self, x, training, gamma_scale):
        """blocks.dropblock(block_size=7) with the uniform draws taken from self.dropblock_u (a
        callable shape -> tensor, or a list consumed in call order): nets/resnet_model.py:432-438."""
        if gamma_scale is None or not training:
            return x
        kp = self.keep_prob
        if isinstance(kp, float) and kp == 1:
            return x
        _, h, w, c = x.shape
        shape = (1, h - 7 + 1, w - 7 + 1, c)
        if shape[1] < 1 or shape[2] < 1:
            raise ValueError("dropblock: feature map %dx%d smaller than block_size 7" % (h, w))
        u = self.dropblock_u(shape) if callable(self.dropblock_u) else self.dropblock_u.pop(0)
        assert tuple(u.shape) == shape, (u.shape, shape)
        self.dropblock_shapes.append(shape)
        return T.dropblock(x, kp, 7, gamma_scale, u)

    def _bottleneck(self, vs, x, filters, training, shortcut_fn, strides, last_relu=True, db=None):
        """nets/resnet_model.py:35-97 _bottleneck_block_v1; db = dropblock gamma_scale or None."""
        shortcut = x
        if shortcut_fn is not None:
            shortcut = self._bn(vs, shortcut_fn(x), training)
            shortcut = self._dropblock(shortcut, training, db)
        sconv = "sconv" in self.aa_type
        y = self._dropblock(self._bn(vs, self._conv(vs, x, filters, 1, 1), training), training, db)
        y = torch.relu(y)
        s3 = 1 if sconv else strides
        if self.use_sk:
            y = self._dropblock(self._sk(vs, y, filters, s3, training), training, db)
        else:
            y = self._dropblock(self._bn(vs, self._conv(vs, y, filters, 3, s3), training), training,
                                db)
            y = torch.relu(y)
        if sconv and strides != 1:
            y = T.anti_aliased_downsample(y, self.aa_size, strides)
        y = self._bn(vs, self._conv(vs, y, 4 * filters, 1, 1), training, self.zero_gamma)
        y = self._dropblock(y, training, db)
        if self.use_se:
            y = self._se(vs, y)
        y = y + shortcut
        return torch.relu(y) if last_relu else y

    def _block_layer(self, vs, x, filters, num_blocks, strides, training, use_resnet_d=False,
                     use_bl=False, last_relu=True, db=None):
        """nets/resnet_model.py:99-163."""
        filters_out = filters * 4

        def projection_shortcut(inp):
            if "proj" in self.aa_type and strides != 1:
                inp = T.anti_aliased_downsample(inp, self.aa_size, strides)
                return self._conv(vs, inp, filters_out, 1, 1)
            return self._conv(vs, inp, filters_out, 1, strides)

        def resnet_d_shortcut(inp):
            return self._conv(vs, T.avg_pool_resnet_d(inp, strides), filters_out, 1, 1)

        def bl_shortcut(inp):
            return self._conv(vs, T.avg_pool_bl(inp, strides), filters_out, 1, 1)

        fn = resnet_d_shortcut if use_resnet_d else (bl_shortcut if use_bl else projection_shortcut)
        # NB: the first block never receives last_relu (reference :151-155)
        x = self._bottleneck(vs, x, filters, training, fn, strides, db=db)
        for i in range(1, num_blocks):
            x = self._bottleneck(vs, x, filters, training, None, 1,
                                 last_relu=last_relu if i == num_blocks - 1 else True, db=db)
        return x

    # -- the network ---------------------------------------------------------------------------
    def forward(self, vs, x, training, use_resnet_d=False, return_embedding=False, keep_prob=1.0,
                dropblock_u=None):
        """nets/resnet_model.py:305-599.  x: [B,H,W,3] NHWC.  Returns logits [B,num_classes].
        keep_prob / dropblock_u: DropBlock keep probability and the source of its uniform draws."""
        self.bn_updates = OrderedDict()
        self.keep_prob = keep_prob
        self.dropblock_u = dropblock_u
        self.dropblock_shapes = []
        nf = self.num_filters
        if use_resnet_d and self.rv == 1:
            x = torch.relu(self._bn(vs, self._conv(vs, x, nf // 2, 3, 2), training))
            x = torch.relu(self._bn(vs, self._conv(vs, x, nf // 2, 3, 1), training))
            x = self._conv(vs, x, nf, 3, 1)
        elif use_resnet_d and self.rv == 2:
            with vs.scope("stage0"):
                x = torch.relu(self._bn(vs, self._conv(vs, x, nf // 2, 3, 2), training))
                x = torch.relu(self._bn(vs, self._conv(vs, x, nf // 2, 3, 1), training))
                x = self._conv(vs, x, nf, 3, 1)
        elif self.rv == 2:
            with vs.scope("stage0"):
                x = self._conv(vs, x, nf, 7, 2)
        else:
            x = self._conv(vs, x, nf, 7, 2)

        if self.rv == 1:
            x = torch.relu(self._bn(vs, x, training))
            x = T.max_pool_same(x, 3, 2)
        else:
            with vs.scope("stage0"):
                x = torch.relu(self._bn(vs, x, training))
            with vs.scope("stage0/pool"):                      # BL module 0 (:385-419)
                big0 = self._bn(vs, self._conv(vs, x, nf, 3, 2), training)
                l0 = torch.relu(self._bn(vs, self._conv(vs, x, nf // self.alpha, 3, 1), training))
                l0 = torch.relu(self._bn(vs, self._conv(vs, l0, nf // self.alpha, 3, 2), training))
                l0 = self._bn(vs, self._conv(vs, l0, nf, 1, 1), training)
                x = torch.relu(big0 + l0)
                x = torch.relu(self._bn(vs, self._conv(vs, x, nf, 1, 1), training))

        for i, nb in enumerate(self.block_sizes):
            f = nf * (2 ** i)
            # dropblock_for_group3 (gamma_scale 0.25) / group4 (1.0): nets/resnet_model.py:432-453
            db = {2: 0.25, 3: 1.0}.get(i)
            if self.rv == 2 and i < 3:
                with vs.scope("stage%d" % (i + 1)):
                    with vs.scope("big%d" % (i + 1)):
                        big = self._block_layer(vs, x, f, nb - 1, 2, training, use_bl=True,
                                                last_relu=False, db=db)
                    with vs.scope("little%d" % (i + 1)):
                        little = self._block_layer(vs, x, f // self.alpha,
                                                   max(1, nb // self.beta - 1), 1, training,
                                                   use_bl=True, db=db)
                        little_e = self._bn(vs, self._conv(vs, little, f * 4, 1, 1), training)
                    with vs.scope("merge%d" % (i + 1)):
                        x = torch.relu(little_e + T.upsample2x(big))
                        x = self._block_layer(vs, x, f, 1, self.block_strides[i], training,
                                              use_bl=True, db=db)
            elif self.rv == 2:
                with vs.scope("stage%d" % (i + 1)):
                    x = self._block_layer(vs, x, f, nb, self.block_strides[i], training,
                                          use_resnet_d=use_resnet_d, use_bl=True, db=db)
            else:
                x = self._block_layer(vs, x, f, nb, self.block_strides[i], training,
                                      use_resnet_d=use_resnet_d, db=db)

        # head: nets/resnet_model.py:552-599
        if self.pool_type == "gap":
            pooled = T.global_avg_pool(x)                      # [B, C]
        elif self.pool_type == "gem":
            pooled = T.generalized_mean_pooling(x)
        elif self.pool_type == "flatten":
            pooled = x.reshape(x.shape[0], -1)                 # NHWC flatten order
        else:
            raise NotImplementedError
        if self.embedding_size > 0:
            _, w = vs.conv_kernel("embedding_dense", 1, pooled.shape[-1], self.embedding_size)
            emb = pooled[:, None, None, :] @ w[0, 0]
            emb = self._bn(vs, emb, training, layer="embedding_dense_batch_normalization")
            pooled = emb[:, 0, 0, :]
        if return_embedding:
            return pooled
        if self.embedding_size > 0:
            pooled = torch.relu(pooled)
        (kn, k), (bn_, b) = vs.dense("dense", pooled.shape[-1], self.num_classes)
        return pooled @ k + b


def build(seed=42, dtype=torch.float32, input_hw=64, use_resnet_d=False, **model_kwargs):
    """Create the model and its variables (one throw-away forward in creation mode)."""
    model = OracleModel(**model_kwargs)
    vs = VarStore(seed=seed, dtype=dtype)
    with torch.no_grad():
        model.forward(vs, torch.zeros(2, input_hw, input_hw, 3, dtype=dtype), True,
                      use_resnet_d=use_resnet_d)
    vs.reset_walk()
    return model, vs


def forward(model, vs, x, training, use_resnet_d=False, **kw):
    vs.reset_walk()
    return model.forward(vs, x, training, use_resnet_d=use_resnet_d, **kw)


def decayed(name):
    """run_loop_classification.py:166-177: every trainable whose name lacks 'batch_normalization'."""
    return "batch_normalization" not in name


def loss_fn(model, vs, images, onehot, *, training=True, use_resnet_d=False, label_smoothing=0.0,
            weight_decay=0.0, teacher_labels=None, kd_temp=0.0, keep_prob=1.0, dropblock_u=None):
    """resnet_model_fn (run_loop_classification.py:121-179): returns (loss, cross_entropy, l2_loss,
    logits); with kd_temp > 0 the knowledge-distillation term T^2 * CE(logits / T, teacher_labels)
    (:156-162) is added to the loss and left in `loss_fn.last_kd`."""
    logits = forward(model, vs, images, training, use_resnet_d, keep_prob=keep_prob,
                     dropblock_u=dropblock_u).float()
    ce = T.softmax_cross_entropy(logits, onehot, label_smoothing)
    l2 = weight_decay * sum(T.l2_loss(v) for n, v in vs.vars.items()
                            if vs.trainable[n] and decayed(n))
    kd = T.kd_loss(logits, teacher_labels.float(), kd_temp) if kd_temp > 0 else 0.0
    loss_fn.last_kd = kd
    return ce + l2 + kd, ce, l2, logits


def train_step(model, vs, momentum_buf, images, onehot, *, lr, momentum=0.9, use_resnet_d=False,
               label_smoothing=0.0, weight_decay=0.0, n_replicas=1, teacher_labels=None,
               kd_temp=0.0, keep_prob=1.0, dropblock_u=None):
    """One full training step on one replica (or the average over `n_replicas` shards of the batch,
    each with its own BN statistics: MirroredStrategy semantics).  Updates vs.vars and
    momentum_buf in place; returns dict(loss, cross_entropy, l2_loss, logits, grads)."""
    names = [n for n in vs.vars if vs.trainable[n]]
    shards = images.shape[0] // n_replicas
    grads = None
    outs = []
    updates = []
    for r in range(n_replicas):
        for n in names:
            vs.vars[n].requires_grad_(True)
        sl = slice(r * shards, (r + 1) * shards)
        loss, ce, l2, logits = loss_fn(model, vs, images[sl], onehot[sl], training=True,
                                       use_resnet_d=use_resnet_d, label_smoothing=label_smoothing,
                                       weight_decay=weight_decay,
                                       teacher_labels=None if teacher_labels is None
                                       else teacher_labels[sl], kd_temp=kd_temp,
                                       keep_prob=keep_prob, dropblock_u=dropblock_u)
        kd_val = loss_fn.last_kd
        g = torch.autograd.grad(loss, [vs.vars[n] for n in names])
        grads = [gi / n_replicas for gi in g] if grads is None else \
            [a + gi / n_replicas for a, gi in zip(grads, g)]
        outs.append((loss.detach(), ce.detach(), l2.detach(), logits.detach()))
        updates.append(dict(model.bn_updates))
        for n in names:
            vs.vars[n].requires_grad_(False)
    with torch.no_grad():
        for n, g in zip(names, grads):
            w, acc = T.momentum_step(vs.vars[n], momentum_buf[n], g, lr, momentum)
            vs.vars[n].copy_(w)
            momentum_buf[n].copy_(acc)
        for n in updates[0]:
            vs.vars[n].copy_(sum(u[n] for u in updates) / n_replicas)
    return {
        "loss": sum(o[0] for o in outs) / n_replicas,
        "cross_entropy": sum(o[1] for o in outs) / n_replicas,
        "l2_loss": outs[0][2],
        "kd_loss": kd_val.detach() if torch.is_tensor(kd_val) else kd_val,
        "logits": torch.cat([o[3] for o in outs], 0),
        "grads": OrderedDict(zip(names, grads)),
    }
