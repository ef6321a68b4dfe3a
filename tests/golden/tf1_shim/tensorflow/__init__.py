"""A minimal eager stand-in for the TensorFlow 1.14 API surface that the reference's model-building
code touches (nets/resnet_model.py, nets/blocks.py, nets/model_helper.py), backed by torch on CPU.

TEST INFRASTRUCTURE ONLY (used by tests/golden/make_reference_shim_golden.py with a checkout of the
original project).  TensorFlow 1.14 has no Python 3.12 wheel, so the reference's own Python — topology, scopes, variable names, padding
choices, block order — is EXECUTED through this shim to produce golden vectors that pin the oracle.
What the shim pins and what it does not:
  * pinned: everything the reference's Python decides (which ops, in which order, with which
    arguments; variable names / shapes / creation order through a faithful re-implementation of
    the TF1 variable_scope / tf.layers naming rules; initializer kinds);
  * the numerical semantics of the individual TF kernels are NOT taken from the oracle: the kernels of
    this stand-in are other people's code -- 'SAME' padding (convolutions and pools) is Hugging Face's
    `DynamicPad2d` (transformers.models.bit, the port of Google's TF BiT checkpoints), fused batch
    norm is ATen's `torch.nn.functional.batch_norm` (biased variance to normalise, unbiased variance
    into the moving average), convolution / pooling arithmetic is ATen's -- so the golden vectors pin
    oracle/tf_ops.py against implementations it shares no code with.  Still not TensorFlow itself.
Layout: NHWC only (`tf.test.is_built_with_cuda()` is False, so the reference picks channels_last).
"""
import contextlib
import os
import sys

import numpy as np
import torch

_REPO = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "..", ".."))
sys.path.insert(0, _REPO)
__version__ = "1.14.0-shim"
# TF_SHIM_FLOAT64=1: the stand-in's tf.float32 computes in float64, so that golden vectors of
# ill-conditioned quantities (training-mode logits of deep nets on a batch of 2) do not depend on the
# summation order of whichever kernels produced them
_F32 = torch.float64 if os.environ.get("TF_SHIM_FLOAT64") == "1" else torch.float32
_NPF32 = np.float64 if _F32 == torch.float64 else np.float32
import torch.nn.functional as _F  # noqa: E402
from transformers.models.bit.modeling_bit import DynamicPad2d as _TFSamePad  # noqa: E402


# ----------------------------------------------------------------------------- generic TF kernels
# (deliberately NOT oracle/tf_ops.py: see the module docstring)
def _same_pad(x_nchw, k, s, value=0.0):
    """TF 'SAME' padding of an NCHW tensor by Hugging Face's port of the rule."""
    return _TFSamePad(k, s, 1, value=value)(x_nchw)


def _conv2d(x_nhwc, w_hwio, stride, padding):
    """tf.nn.conv2d / tf.layers.conv2d (no bias) on NHWC input with an HWIO kernel."""
    x = x_nhwc.permute(0, 3, 1, 2)
    if padding == "SAME":
        x = _same_pad(x, (w_hwio.shape[0], w_hwio.shape[1]), stride)
    else:
        assert padding == "VALID", padding
    return _F.conv2d(x, w_hwio.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def _batch_norm(x, gamma, beta, mm, mv, training, momentum, eps):
    """tf.layers.batch_normalization(fused=True) by ATen's kernel (torch's momentum is 1 - TF's).
    Returns (y, new_moving_mean, new_moving_variance)."""
    rm, rv = mm.detach().clone(), mv.detach().clone()
    y = _F.batch_norm(x.permute(0, 3, 1, 2), rm, rv, gamma, beta, bool(training), 1.0 - momentum, eps)
    return y.permute(0, 2, 3, 1), rm, rv


def _max_pool(t, k, s, padding):
    """tf.nn.max_pool: SAME pads with -inf, the odd cell after."""
    x = t.permute(0, 3, 1, 2)
    if padding == "SAME":
        x = _same_pad(x, k, s, value=float("-inf"))
    return _F.max_pool2d(x, k, s).permute(0, 2, 3, 1)


def _avg_pool(t, k, s, padding):
    """tf.nn.avg_pool: VALID divides by k*k; SAME divides by the number of in-bounds cells."""
    x = t.permute(0, 3, 1, 2)
    if padding != "SAME":
        return _F.avg_pool2d(x, k, s).permute(0, 2, 3, 1)
    ssum = _F.avg_pool2d(_same_pad(x, k, s), k, s) * float(k * k)
    ones = _same_pad(torch.ones(1, 1, t.shape[1], t.shape[2], dtype=t.dtype), k, s)
    cnt = _F.avg_pool2d(ones, k, s) * float(k * k)
    return (ssum / cnt).permute(0, 2, 3, 1)


def _depthwise(t, w_hw1c, stride, padding):
    """Grouped convolution with one input channel per group (filter [kh, kw, 1, C])."""
    assert padding == "VALID"
    c = t.shape[3]
    w = w_hw1c.permute(3, 2, 0, 1)                   # [C, 1, kh, kw]
    return _F.conv2d(t.permute(0, 3, 1, 2), w, stride=stride, groups=c).permute(0, 2, 3, 1)


def _reflect_pad(t, t0, t1, l0, l1):
    return _F.pad(t.permute(0, 3, 1, 2), (l0, l1, t0, t1), mode="reflect").permute(0, 2, 3, 1)


# ----------------------------------------------------------------------------- dtypes / tensors
class DType:
    def __init__(self, name, torch_dtype, floating=True):
        self.name, self.torch, self.is_floating = name, torch_dtype, floating

    def __repr__(self):
        return "tf." + self.name


float32 = DType("float32", _F32)
float16 = DType("float16", torch.float16)
int32 = DType("int32", torch.int32, False)
_BY_TORCH = {torch.float32: float32, torch.float16: float16, torch.int32: int32,
             torch.float64: float32, torch.int64: int32}


class TensorShape(list):
    def as_list(self):
        return list(self)


def _raw(x):
    if isinstance(x, Tensor):
        return x.t
    if isinstance(x, (list, tuple)) and x and isinstance(x[0], Tensor):
        return torch.stack([e.t for e in x], 0)        # a Python list of tensors converts by stacking
    if isinstance(x, (list, tuple, np.ndarray)):
        return torch.as_tensor(np.asarray(x, dtype=_NPF32))
    return x


class Tensor:
    """Eager tensor with the handful of members the reference uses."""

    def __init__(self, t, name=None):
        if _F32 is torch.float64 and torch.is_tensor(t) and t.dtype == torch.float32:
            t = t.double()                 # float64 override: "tf.float32" data computes in float64
        self.t = t
        self.name = name

    @property
    def shape(self):
        return TensorShape(self.t.shape)

    @property
    def dtype(self):
        return _BY_TORCH[self.t.dtype]

    def _bin(self, other, fn, swap=False):
        o = _raw(other)
        return Tensor(fn(o, self.t) if swap else fn(self.t, o))

    def __add__(self, o): return self._bin(o, torch.add)
    def __radd__(self, o): return self._bin(o, torch.add, True)
    def __sub__(self, o): return self._bin(o, torch.sub)
    def __rsub__(self, o): return self._bin(o, lambda a, b: a - b, True)
    def __mul__(self, o): return self._bin(o, torch.mul)
    def __rmul__(self, o): return self._bin(o, torch.mul, True)
    def __truediv__(self, o): return self._bin(o, torch.div)
    def __rtruediv__(self, o): return self._bin(o, lambda a, b: a / b, True)
    def __neg__(self): return Tensor(-self.t)
    def __getitem__(self, idx): return Tensor(self.t[idx])


# ----------------------------------------------------------------------------- variable scopes
class _ScopeStore:
    def __init__(self):
        self.reset()

    def reset(self):
        self.stack = [_VarScope("", None, None)]
        self.counts = {}

    @property
    def current(self):
        return self.stack[-1]


class _VarScope:
    def __init__(self, name, reuse, custom_getter):
        self.name, self.reuse, self.custom_getter = name, reuse, custom_getter


_store = _ScopeStore()


class _Variables:
    """Creation-ordered record of every variable the model asked for, and where values come from."""

    def __init__(self):
        self.reset()

    def reset(self, values=None, requires_grad=False):
        self.order = []          # [(full name, shape, initializer kind, trainable)]
        self.values = values     # dict name -> torch tensor, or None (initializer defaults)
        self.requires_grad = requires_grad   # leaves for torch autograd through the reference graph
        self.vars = {}


variables = _Variables()


def get_variable_scope():
    return _store.current


def _unique_scope(prefix):
    cur = _store.current.name
    full = cur + "/" + prefix if cur else prefix
    if _store.counts.get(full, 0) == 0:
        return prefix
    idx = 1
    while _store.counts.get(full + "_%d" % idx, 0) > 0:
        idx += 1
    return prefix + "_%d" % idx


@contextlib.contextmanager
def variable_scope(name_or_scope, default_name=None, values=None, reuse=None, custom_getter=None,
                   auxiliary_name_scope=True):
    """TF 1.14 python/ops/variable_scope.py semantics for the cases the reference exercises: named
    scopes nest by '/', an unnamed scope takes `default_name` made unique inside the current scope
    (suffix _1, _2, ...), a scope's use count survives its exit but the counts of its sub-scopes are
    cleared when it exits."""
    if isinstance(name_or_scope, _VarScope):                      # re-entering a captured scope
        scope = _VarScope(name_or_scope.name, reuse if reuse is not None else name_or_scope.reuse,
                          name_or_scope.custom_getter)
        saved = dict(_store.counts)
        _store.stack.append(scope)
        try:
            yield scope
        finally:
            _store.stack.pop()
            _store.counts = saved
        return
    name = name_or_scope if name_or_scope is not None else _unique_scope(default_name)
    cur = _store.current
    full = cur.name + "/" + name if cur.name else name
    scope = _VarScope(full, reuse if reuse is not None else cur.reuse,
                      custom_getter if custom_getter is not None else cur.custom_getter)
    _store.counts[full] = _store.counts.get(full, 0) + 1
    _store.stack.append(scope)
    try:
        yield scope
    finally:
        _store.stack.pop()
        for k in list(_store.counts):
            if k.startswith(full + "/"):
                _store.counts[k] = 0


@contextlib.contextmanager
def name_scope(name, default_name=None, values=None):
    yield name or default_name


class _Init:
    def __init__(self, kind, value=None):
        self.kind, self.value = kind, value


def variance_scaling_initializer(*a, **k): return _Init("variance_scaling")
def zeros_initializer(*a, **k): return _Init("zeros")
def ones_initializer(*a, **k): return _Init("ones")
def constant_initializer(value=0, *a, **k): return _Init("constant", float(value))
def glorot_uniform_initializer(*a, **k): return _Init("glorot_uniform")


def _base_getter(name, shape=None, dtype=float32, initializer=None, trainable=True, **kwargs):
    if name in variables.vars:
        return variables.vars[name]
    shape = tuple(int(s) for s in shape)
    kind = initializer.kind if initializer is not None else "glorot_uniform"
    if variables.values is not None:
        v = variables.values[name]
        assert tuple(v.shape) == shape, (name, tuple(v.shape), shape)
        v = v.clone().to(_F32)
    elif kind == "ones":
        v = torch.ones(shape, dtype=_F32)
    elif kind == "constant":
        v = torch.full(shape, initializer.value, dtype=_F32)
    else:
        v = torch.zeros(shape, dtype=_F32)
    variables.order.append((name, shape, kind, bool(trainable)))
    if variables.requires_grad and trainable:
        v.requires_grad_(True)
    variables.vars[name] = Tensor(v, name=name)
    return variables.vars[name]


def get_variable(name, shape=None, dtype=float32, initializer=None, trainable=True, **kwargs):
    scope = _store.current
    full = scope.name + "/" + name if scope.name else name
    if scope.custom_getter is not None:
        return scope.custom_getter(_base_getter, full, shape, dtype, initializer=initializer,
                                   trainable=trainable)
    return _base_getter(full, shape, dtype, initializer=initializer, trainable=trainable)


# ----------------------------------------------------------------------------- tf.layers
class _Layers:
    @staticmethod
    @contextlib.contextmanager
    def _scope(name, base):
        # python/layers/base.py: a named layer opens variable_scope(name); an unnamed one opens
        # variable_scope(None, default_name=<snake-cased class name>)
        with variable_scope(name, default_name=base) as s:
            yield s

    def conv2d(self, inputs, filters, kernel_size, strides=1, padding="valid", data_format="channels_last",
               use_bias=True, kernel_initializer=None, name=None, **kw):
        assert data_format == "channels_last"
        k = kernel_size if isinstance(kernel_size, (tuple, list)) else (kernel_size, kernel_size)
        cin = inputs.shape[-1]
        with self._scope(name, "conv2d"):
            w = get_variable("kernel", (k[0], k[1], cin, filters), initializer=kernel_initializer)
            y = _conv2d(inputs.t, w.t, strides, padding.upper())
            if use_bias:
                y = y + get_variable("bias", (filters,), initializer=zeros_initializer()).t
        return Tensor(y)

    def batch_normalization(self, inputs, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True,
                            training=False, fused=None, gamma_initializer=None, name=None, **kw):
        assert axis in (3, -1)
        c = inputs.shape[-1]
        with self._scope(name, "batch_normalization"):
            gamma = get_variable("gamma", (c,), initializer=gamma_initializer or ones_initializer())
            beta = get_variable("beta", (c,), initializer=zeros_initializer())
            mm = get_variable("moving_mean", (c,), initializer=zeros_initializer(), trainable=False)
            mv = get_variable("moving_variance", (c,), initializer=ones_initializer(), trainable=False)
        y, new_mm, new_mv = _batch_norm(inputs.t, gamma.t, beta.t, mm.t, mv.t, bool(training),
                                        momentum, epsilon)
        if training:                       # the UPDATE_OPS the reference's train op depends on
            mm.t, mv.t = new_mm.detach(), new_mv.detach()
        return Tensor(y)

    def dense(self, inputs, units, bias_initializer=None, name=None, **kw):
        with self._scope(name, "dense"):
            w = get_variable("kernel", (inputs.shape[-1], units), initializer=glorot_uniform_initializer())
            b = get_variable("bias", (units,), initializer=bias_initializer or zeros_initializer())
        return Tensor(inputs.t @ w.t + b.t)

    def max_pooling2d(self, inputs, pool_size, strides, padding="valid", data_format="channels_last", **kw):
        assert data_format == "channels_last"
        return Tensor(_max_pool(inputs.t, pool_size, strides, padding.upper()))

    def average_pooling2d(self, inputs, pool_size, strides, padding="valid", data_format="channels_last", **kw):
        assert data_format == "channels_last"
        return Tensor(_avg_pool(inputs.t, pool_size, strides, padding.upper()))

    def flatten(self, inputs, **kw):
        return Tensor(inputs.t.reshape(inputs.t.shape[0], -1))


layers = _Layers()


class _UpSampling2D:
    def __init__(self, size=(2, 2), data_format=None):
        assert tuple(size) == (2, 2) and data_format in (None, "channels_last")

    def __call__(self, x):
        return Tensor(x.t.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))


class _NS:
    pass


keras = _NS()
keras.layers = _NS()
keras.layers.UpSampling2D = _UpSampling2D


# ----------------------------------------------------------------------------- tf.nn / math
class _NN:
    @staticmethod
    def relu(x, name=None): return Tensor(torch.relu(_raw(x)))
    @staticmethod
    def sigmoid(x, name=None): return Tensor(torch.sigmoid(_raw(x)))
    @staticmethod
    def softmax(x, axis=-1, name=None): return Tensor(torch.softmax(_raw(x), dim=axis))

    @staticmethod
    def conv2d(inp, filt, strides, padding, data_format="NHWC", **kw):
        assert data_format == "NHWC" and strides[0] == 1 and strides[3] == 1 and strides[1] == strides[2]
        x, w = _raw(inp), _raw(filt)
        if w.shape[2] != x.shape[3]:
            # filter depth 1 against C input channels: the grouped (depthwise) convolution the
            # reference's anti-alias filter relies on
            assert w.shape[2] == 1 and w.shape[3] == x.shape[3]
            return Tensor(_depthwise(x, w, strides[1], padding))
        return Tensor(_conv2d(x, w, strides[1], padding))


nn = _NN()
nn.l2_loss = staticmethod(lambda t, name=None: Tensor((_raw(t).to(_F32) ** 2).sum() / 2))


def _axes(axis):
    return tuple(axis) if isinstance(axis, (list, tuple)) else axis


def reduce_sum(x, axis=None, keepdims=False, keep_dims=None, name=None):
    kd = keepdims if keep_dims is None else keep_dims
    t = _raw(x)
    return Tensor(t.sum() if axis is None else t.sum(dim=_axes(axis), keepdim=bool(kd)))


def reduce_mean(x, axis=None, keepdims=False, keep_dims=None, name=None):
    kd = keepdims if keep_dims is None else keep_dims
    t = _raw(x)
    return Tensor(t.mean() if axis is None else t.mean(dim=_axes(axis), keepdim=bool(kd)))


def argmax(x, axis=None, name=None, **kw):
    return Tensor(torch.argmax(_raw(x), dim=axis))


def split(x, num_or_size_splits, axis=0, name=None):
    t = _raw(x)
    assert isinstance(num_or_size_splits, int)
    return [Tensor(p) for p in torch.chunk(t, num_or_size_splits, dim=axis)]


def concat(xs, axis, name=None): return Tensor(torch.cat([_raw(x) for x in xs], dim=axis))
def stack(xs, axis=0, name=None): return Tensor(torch.stack([torch.as_tensor(_raw(x)) for x in xs], dim=axis))
def identity(x, name=None): return x
def cast(x, dtype, name=None): return Tensor(torch.as_tensor(_raw(x)).to(dtype.torch))
def to_float(x): return Tensor(torch.as_tensor(_raw(x), dtype=_F32))
def multiply(a, b, name=None):
    r = torch.as_tensor(_raw(a)) * torch.as_tensor(_raw(b))
    return Tensor(r)
def pow(x, p, name=None): return Tensor(torch.pow(torch.as_tensor(_raw(x), dtype=_F32), _raw(p)))
def maximum(a, b, name=None): return Tensor(torch.maximum(_raw(a), torch.as_tensor(_raw(b), dtype=_F32)))
def clip_by_value(x, lo, hi, name=None): return Tensor(torch.clamp(_raw(x), lo, hi))
def sign(x, name=None): return Tensor(torch.sign(_raw(x)))
def size(x, name=None): return Tensor(torch.tensor(_raw(x).numel()))
def reshape(x, shape, name=None): return Tensor(_raw(x).reshape([int(s) for s in shape]))
def tile(x, multiples, name=None): return Tensor(_raw(x).repeat([int(m) for m in multiples]))
def transpose(x, perm, name=None): return Tensor(_raw(x).permute(*perm))
def squeeze(x, axis=None, name=None):
    t = _raw(x)
    for a in sorted(_axes(axis) if isinstance(axis, (list, tuple)) else [axis], reverse=True):
        t = t.squeeze(a)
    return Tensor(t)
def expand_dims(x, axis, name=None): return Tensor(_raw(x).unsqueeze(axis))
def constant(value, dtype=None, name=None):
    return Tensor(torch.as_tensor(np.asarray(value), dtype=(dtype or float32).torch))



def pad(x, paddings, mode="CONSTANT", name=None):
    t = _raw(x)
    assert t.dim() == 4 and paddings[0] == [0, 0] and paddings[3] == [0, 0]
    (t0, t1), (l0, l1) = paddings[1], paddings[2]
    if mode.upper() == "REFLECT":
        return Tensor(_reflect_pad(t, t0, t1, l0, l1))
    return Tensor(torch.nn.functional.pad(t, (0, 0, l0, l1, t0, t1)))


uniform_fn = None      # shape -> tensor: the source of tf.random_uniform draws (set by the generator)


def random_uniform(shape, minval=0, maxval=1, dtype=float32, seed=None):
    """DropBlock's _bernoulli draws (nets/blocks.py:187-188): TF's RNG is not reproducible, so the
    golden generator installs a seeded source; the oracle test replays the same sequence."""
    if uniform_fn is None:
        raise NotImplementedError("tf.random_uniform without an installed uniform_fn")
    shp = [int(v) for v in (_raw(shape).tolist() if hasattr(_raw(shape), "tolist") else shape)]
    return Tensor(uniform_fn(tuple(shp)).to(dtype.torch) * (maxval - minval) + minval)


class _Logging:
    @staticmethod
    def info(*a, **k): pass
    warn = warning = debug = info
    error = info


logging = _Logging()


class _Test:
    @staticmethod
    def is_built_with_cuda(): return False


test = _Test()


# ----------------------------------------------------------------------------- utils/data_util.mixup
VERSION = "1.14.0"


def shape(x, name=None):
    return list(_raw(x).shape)


def reverse(x, axis, name=None): return Tensor(torch.flip(_raw(x), dims=list(axis)))
def stop_gradient(x, name=None): return Tensor(_raw(x).detach())


Tensor.get_shape = lambda self: self.shape


class _Beta:
    """tf.contrib.distributions.Beta: samples come from the queue the golden generator fills
    (`beta_samples`), so that the reference code and the oracle see the same lambdas."""
    queue = []

    def __init__(self, a, b):
        self.a, self.b = a, b

    def sample(self, shape):
        n = int(shape[0])
        v = _Beta.queue.pop(0)
        assert v.numel() == n, (v.numel(), n)
        return Tensor(v.clone())


beta_samples = _Beta.queue


class _Dummy:
    """Anything else the reference's modules touch at import time (summaries, estimators, ...)."""

    def __init__(self, name="tf"):
        self._n = name

    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return _Dummy(self._n + "." + k)

    def __call__(self, *a, **k):
        raise NotImplementedError("%s is outside the pinned path" % self._n)


class _Summary:
    """tf.summary.*: logging side effects, no value on the pinned path."""

    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return lambda *a, **kw: None


summary = _Summary()


# ----------------------------------------------------------------------------- tf.train / tf.losses
def _f(x):
    return float(_raw(x)) if isinstance(x, Tensor) else float(x)


class _Train:
    """Learning-rate schedules as documented for TF 1.14 (python/training/learning_rate_decay*.py)."""

    @staticmethod
    def exponential_decay(lr, global_step, decay_steps, decay_rate, staircase=False, name=None):
        p = _f(global_step) / decay_steps
        return Tensor(torch.tensor(lr * decay_rate ** (np.floor(p) if staircase else p)))

    @staticmethod
    def polynomial_decay(lr, global_step, decay_steps, end_learning_rate=0.0001, power=1.0,
                         cycle=False, name=None):
        g = min(_f(global_step), decay_steps)
        return Tensor(torch.tensor((lr - end_learning_rate) * (1 - g / decay_steps) ** power
                                   + end_learning_rate))

    @staticmethod
    def piecewise_constant(x, boundaries, values, name=None):
        # values[0] for x <= boundaries[0], values[i] for boundaries[i-1] < x <= boundaries[i]
        return Tensor(torch.tensor(values[sum(1 for b in boundaries if _f(x) > b)]))

    @staticmethod
    def cosine_decay(lr, global_step, decay_steps, alpha=0.0, name=None):
        g = min(_f(global_step), decay_steps)
        cos = 0.5 * (1 + np.cos(np.pi * g / decay_steps))
        return Tensor(torch.tensor(lr * ((1 - alpha) * cos + alpha)))


train = _Train()


def cond(pred, true_fn, false_fn, name=None):
    return true_fn() if bool(_raw(pred)) else false_fn()


Tensor.__lt__ = lambda self, o: Tensor(self.t < _raw(o))


class _Losses:
    @staticmethod
    def softmax_cross_entropy(onehot_labels, logits, weights=1.0, label_smoothing=0, **kw):
        """tf.losses.softmax_cross_entropy: labels smoothed towards 1/num_classes, per-example
        cross entropy, reduction SUM_BY_NONZERO_WEIGHTS (= batch mean for a scalar weight)."""
        y, z = _raw(onehot_labels).to(_F32), _raw(logits).to(_F32)
        if label_smoothing > 0:
            n = y.shape[1]
            y = y * (1 - label_smoothing) + label_smoothing / n
        per = -(y * torch.log_softmax(z, dim=1)).sum(dim=1)
        return Tensor((per * weights).sum() / per.numel())


losses = _Losses()

contrib = _NS()
contrib.distributions = _NS()
contrib.distributions.Beta = _Beta


def __getattr__(name):          # PEP 562: unknown tf.<name>
    if name.startswith("__"):
        raise AttributeError(name)
    return _Dummy("tf." + name)


def reset(values=None, requires_grad=False):
    """Start a fresh 'graph': empty scope counts, empty variable record; `values` (name -> tensor)
    supplies the variable values, else the initializers' trivial defaults are used.  With
    requires_grad the trainable variables are autograd leaves (gradients of the reference's graph)."""
    _store.reset()
    variables.reset(values, requires_grad)
