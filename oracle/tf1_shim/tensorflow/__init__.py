"""A minimal ``tensorflow`` (1.14 API surface) stand-in -- TEST INFRASTRUCTURE ONLY.

Purpose: TensorFlow 1.14 cannot be installed in this image (no cp312 wheel, no network), so the reference's own
files could not be *executed*.  This module implements exactly the part of the TF1 API that the reference's learner
files touch (``agent/{impala,apex,r2d2}.py``, ``model/{impala_actor_critic,apex_value,r2d2_lstm}.py``,
``optimizer/{vtrace,dqn,burn_in}.py``, ``utils.py``, ``distributed_queue/buffer_queue.py``) as a deferred graph
over torch-CPU tensors, so that the UNMODIFIED reference files run here (``oracle/ref_exec.py`` puts this directory
and ``/root/reference`` on ``sys.path``).  Every slice, window, loss, stop_gradient, variable-scope/reuse and
optimizer-call decision is then the reference's own code; what is restated here is only TF's *op semantics*
(third-party, documented behaviour of tensorflow==1.14.0, the version pinned by the reference's README.md:14 /
Dockerfile:2):

  tf.layers.conv2d        NHWC, HWIO kernel, cross-correlation, VALID padding, glorot_uniform kernel, zero bias
  tf.layers.dense         [in, out] kernel, glorot_uniform, zero bias
  tf.nn.rnn_cell.LSTMCell kernel [in+h, 4h], gate order i, j, f, o, forget_bias 1.0 added inside the sigmoid, state (c, h)
  tf.nn.dynamic_rnn       loop over axis 1, variables under ``rnn/lstm_cell``
  tf.scan                 sequential fold over axis 0 (``reverse`` honoured), ``back_prop=False`` => no gradient
  tf.train.RMSPropOptimizer  ms0 = 1, ms += (1-decay)(g^2 - ms), mom = momentum*mom + lr*g*rsqrt(ms+eps), var -= mom
  tf.train.AdamOptimizer  lr_t = lr*sqrt(1-b2^t)/(1-b1^t), var -= lr_t*m/(sqrt(v)+eps); beta powers updated after apply
  tf.clip_by_global_norm  scale = clip*min(1/norm, 1/clip) + (norm - norm) (NaN for a non-finite norm); None gradients ignored
  tf.train.polynomial_decay  (lr-end)*(1-min(step,decay)/decay)^power + end
  variable_scope          default-name uniquification counters that are RESET for the sub-scopes when a scope is left
                          (``close_variable_subscopes``) -- this is what makes the reference's repeated
                          ``with tf.variable_scope('impala', reuse=tf.AUTO_REUSE)`` share ``conv2d .. dense_7``
  Session.run             tensor fetches are evaluated on the pre-update variables, then the ops' assignments commit

Floating dtype: ``tensorflow._shim.FLOAT`` (torch.float64 by default = "truth"; set to torch.float32 to mimic TF's
arithmetic type).  Nothing here is imported by the product package.
"""
import contextlib
import math as _pymath
import operator
import re
import sys

import numpy as np
import torch
import torch.nn.functional as F

__version__ = "1.14.0-shim"
sys.setrecursionlimit(max(sys.getrecursionlimit(), 100000))     # node evaluation is recursive (deep unrolls)


class _Shim:
    FLOAT = torch.float64
    seed = 0


_shim = _Shim()


# --------------------------------------------------------------------------------------------- dtypes
class DType:
    def __init__(self, name, kind, np_dtype):
        self.name, self.kind, self.as_numpy_dtype = name, kind, np_dtype

    @property
    def base_dtype(self):
        return self

    def torch(self):
        if self.kind == "f":
            return _shim.FLOAT
        return {"int32": torch.int64, "int64": torch.int64, "bool": torch.bool, "uint8": torch.uint8}[self.name]

    def __repr__(self):
        return "tf." + self.name


float32 = DType("float32", "f", np.float32)
float64 = DType("float64", "f", np.float64)
int32 = DType("int32", "i", np.int32)
int64 = DType("int64", "i", np.int64)
uint8 = DType("uint8", "u", np.uint8)
bool = DType("bool", "b", np.bool_)   # noqa: A001  (the reference spells it tf.bool)
_pybool = type(True)


def _dtype_of_value(v):
    if v.dtype == torch.bool:
        return bool
    if v.dtype == torch.uint8:
        return uint8
    if v.dtype in (torch.int64, torch.int32):
        return int32
    return float32


# --------------------------------------------------------------------------------------------- graph
class Dimension:
    def __init__(self, value):
        self.value = value

    def __int__(self):
        return int(self.value)

    def __repr__(self):
        return "Dimension(%r)" % (self.value,)

    def __eq__(self, o):
        return self.value == (o.value if isinstance(o, Dimension) else o)

    def __hash__(self):
        return hash(self.value)


class TensorShape:
    def __init__(self, dims):
        self.dims = [d if isinstance(d, Dimension) else Dimension(d) for d in dims]

    def __iter__(self):
        return iter(self.dims)

    def __len__(self):
        return len(self.dims)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return TensorShape(self.dims[i])
        return self.dims[i]

    def as_list(self):
        return [d.value for d in self.dims]

    @property
    def ndims(self):
        return len(self.dims)

    def __repr__(self):
        return "TensorShape(%r)" % (self.as_list(),)


class Graph:
    def __init__(self):
        self.variables = []                # creation order == tf.global_variables()
        self.var_by_name = {}
        self.scope_counts = {}             # variable_scope_count of TF's _VariableScopeStore
        self.scope_stack = [("", None)]    # (full name, reuse)
        self.placeholders = []
        self.global_step = None
        self.queues = {}
        self.shape_ctx = {}                # persistent dummy-evaluation caches for static shapes
        self.rng = torch.Generator().manual_seed(_shim.seed)


_graph = Graph()


def reset_default_graph():
    global _graph
    _graph = Graph()


def get_default_graph():
    return _graph


class GraphKeys:
    TRAINABLE_VARIABLES = "trainable_variables"
    GLOBAL_VARIABLES = "variables"
    GLOBAL_STEP = "global_step"


AUTO_REUSE = "AUTO_REUSE"


class _Ctx:
    """One evaluation: feed values + memo of node values + assignments staged by ops."""

    def __init__(self, feeds=None, dummy=None):
        self.feeds = feeds or {}
        self.memo = {}
        self.dummy = dummy           # None, or the size substituted for unknown (None) dimensions
        self.staged = []             # (Variable, new torch value)
        self.side_effects = []       # callables run at commit (queues)


class Tensor:
    _is_op = False
    nondiff = False     # gradient does not flow through this node (stop_gradient, argmax, scan without back_prop, ...)

    def __init__(self, fn, inputs=(), dtype=None, name=None, nondiff=False):
        self._fn = fn
        self._inputs = tuple(inputs)
        self._dtype = dtype
        self.name = name
        self.nondiff = nondiff

    # ---- evaluation
    def _eval(self, ctx):
        k = id(self)
        if k not in ctx.memo:            # the entry keeps the node alive, so ids cannot be recycled within a ctx
            ctx.memo[k] = (self, self._fn(ctx, *[i._eval(ctx) for i in self._inputs]))
        return ctx.memo[k][1]

    # ---- static information (by dummy evaluation: unknown dims are substituted by 2 and by 3)
    def _dummy_value(self, size):
        ctx = _graph.shape_ctx.setdefault(size, _Ctx(dummy=size))
        with torch.no_grad():
            return self._eval(ctx)

    def get_shape(self):
        a, b = self._dummy_value(2), self._dummy_value(3)
        return TensorShape([x if x == y else None for x, y in zip(a.shape, b.shape)])

    @property
    def shape(self):
        return self.get_shape()

    @property
    def dtype(self):
        if self._dtype is None:
            self._dtype = _dtype_of_value(self._dummy_value(2))
        return self._dtype

    # ---- operators the reference uses on tensors
    def __add__(self, o): return _binary(operator.add, self, o)
    def __radd__(self, o): return _binary(operator.add, o, self)
    def __sub__(self, o): return _binary(operator.sub, self, o)
    def __rsub__(self, o): return _binary(operator.sub, o, self)
    def __mul__(self, o): return _binary(operator.mul, self, o)
    def __rmul__(self, o): return _binary(operator.mul, o, self)
    def __truediv__(self, o): return _binary(operator.truediv, self, o)
    def __rtruediv__(self, o): return _binary(operator.truediv, o, self)
    def __pow__(self, o): return _binary(operator.pow, self, o)
    def __neg__(self): return _unary(torch.neg, self)
    def __lt__(self, o): return _binary(operator.lt, self, o, nondiff=True)
    def __gt__(self, o): return _binary(operator.gt, self, o, nondiff=True)
    def __le__(self, o): return _binary(operator.le, self, o, nondiff=True)
    def __ge__(self, o): return _binary(operator.ge, self, o, nondiff=True)
    def __invert__(self): return _unary(torch.logical_not, self, nondiff=True)
    __hash__ = object.__hash__

    def __getitem__(self, idx):
        return Tensor(lambda ctx, v: v[idx], [self], self._dtype)

    def __iter__(self):
        raise TypeError("Tensor objects are only iterable when eager execution is enabled.")

    def __bool__(self):
        raise TypeError("Using a tf.Tensor as a Python bool is not allowed.")

    def __repr__(self):
        return "<shim tf.Tensor %s>" % (self.name or hex(id(self)))


def _as_tensor(x, like=None):
    """Tensors/variables pass; numpy arrays become constants (floats in the shim's float type); Python scalars stay
    Python scalars so that torch's own scalar type promotion applies (tensor dtype wins)."""
    if isinstance(x, Tensor):
        return x
    if isinstance(x, Variable):
        return x._tensor
    if isinstance(x, torch.Tensor):
        return Tensor(lambda ctx: x)
    if isinstance(x, (int, float, _pybool)):
        return Tensor(lambda ctx: x)
    arr = np.asarray(x)
    if arr.dtype.kind == "f":
        return Tensor(lambda ctx: torch.as_tensor(arr.astype(np.float64)).to(_shim.FLOAT), dtype=float32)
    if arr.dtype.kind == "b":
        return Tensor(lambda ctx: torch.as_tensor(arr), dtype=bool)
    return Tensor(lambda ctx: torch.as_tensor(arr.astype(np.int64)), dtype=int32)


def _binary(f, a, b, nondiff=False):
    return Tensor(lambda ctx, x, y: f(x, y), [_as_tensor(a), _as_tensor(b)], nondiff=nondiff)


def _unary(f, a, nondiff=False, dtype=None):
    a = _as_tensor(a)
    return Tensor(lambda ctx, x: f(x), [a], dtype, nondiff=nondiff)


def convert_to_tensor(x, dtype=None):
    return _as_tensor(x)


def constant(x, dtype=None):
    return _as_tensor(x)


# --------------------------------------------------------------------------------------------- placeholders
def placeholder(dtype, shape=None, name=None):
    shape = None if shape is None else [None if s is None else int(s) for s in shape]

    def fn(ctx):
        if ctx.dummy is not None:
            return torch.zeros([ctx.dummy if s is None else s for s in shape], dtype=dtype.torch())
        if id(t) not in ctx.feeds:
            raise RuntimeError("You must feed a value for placeholder tensor %r" % (name,))
        v = np.asarray(ctx.feeds[id(t)])
        if shape is not None and (v.ndim != len(shape) or
                                  any(s is not None and s != d for s, d in zip(shape, v.shape))):
            raise ValueError("Cannot feed value of shape %r for Tensor %r, which has shape %r"
                             % (v.shape, name, tuple(shape)))
        if dtype.kind == "f":
            # a float64 feed of a float32 placeholder is cast to float32 first (what the TF feed does), then lifted
            return torch.as_tensor(v.astype(np.float32)).to(_shim.FLOAT)
        if dtype.kind == "b":
            return torch.as_tensor(v.astype(np.bool_))
        if dtype.kind == "u":
            return torch.as_tensor(v.astype(np.uint8))
        return torch.as_tensor(v.astype(np.int64))

    t = Tensor(fn, (), dtype, name or "Placeholder")
    t._static_shape = shape
    t.get_shape = lambda: TensorShape(shape)
    _graph.placeholders.append(t)
    return t


# --------------------------------------------------------------------------------------------- scopes / variables
@contextlib.contextmanager
def device(_name):
    yield


@contextlib.contextmanager
def name_scope(_name, *a, **k):
    yield


def _cur_scope():
    return _graph.scope_stack[-1]


def _unique_scope(default_name):
    """variable_scope(None, default_name=...) -> TF's _get_unique_variable_scope."""
    cur = _cur_scope()[0]
    full = cur + "/" + default_name if cur else default_name
    if _graph.scope_counts.get(full, 0) == 0:
        return default_name
    idx = 1
    while _graph.scope_counts.get(full + "_%d" % idx, 0) > 0:
        idx += 1
    return default_name + "_%d" % idx


class VariableScope:
    def __init__(self, name, reuse):
        self.name, self.reuse = name, reuse


@contextlib.contextmanager
def variable_scope(name_or_scope=None, default_name=None, reuse=None, **_kw):
    if isinstance(name_or_scope, VariableScope):
        full, inherit = name_or_scope.name, name_or_scope.reuse
    else:
        name = name_or_scope if name_or_scope is not None else _unique_scope(default_name)
        cur = _cur_scope()[0]
        full = cur + "/" + name if cur else name
        inherit = None
    if reuse is None:                      # reuse is inherited by sub-scopes
        reuse = inherit if inherit is not None else _cur_scope()[1]
    _graph.scope_counts[full] = _graph.scope_counts.get(full, 0) + 1
    _graph.scope_stack.append((full, reuse))
    try:
        yield VariableScope(full, reuse)
    finally:
        _graph.scope_stack.pop()
        for k in list(_graph.scope_counts):          # close_variable_subscopes(full)
            if k.startswith(full + "/"):
                _graph.scope_counts[k] = 0


def get_variable_scope():
    return VariableScope(*_cur_scope())


class Operation:
    _is_op = True

    def __init__(self, run, name=None, deps=()):
        self._run = run
        self.name = name
        self._deps = deps

    def _eval(self, ctx):
        k = id(self)
        if k not in ctx.memo:
            ctx.memo[k] = (self, None)
            for d in self._deps:
                d._eval(ctx)
            self._run(ctx)
        return None


class Variable:
    store_float32 = False     # keep a float32-rounded value even when the shim computes in float64

    def __init__(self, name, shape, dtype, initializer, trainable=True):
        self.name = name + ":0"
        self.op_name = name
        self._shape = [int(s) for s in shape]
        self._dtype = dtype
        self._initializer = initializer
        self.trainable = trainable
        self.value = None
        self.initialize()
        self._tensor = Tensor(lambda ctx: self.value, (), dtype, self.name)
        self._tensor._variable = self

    def initialize(self):
        v = self._initializer(self._shape, self._dtype)
        if self.store_float32:
            v = v.to(torch.float32).to(v.dtype)
        self.value = v.requires_grad_(self._dtype.kind == "f" and self.trainable)

    @property
    def dtype(self):
        return self._dtype

    def get_shape(self):
        return TensorShape(self._shape)

    shape = property(get_shape)

    def assign(self, value):
        value = _as_tensor(value)

        def run(ctx):
            ctx.staged.append((self, value._eval(ctx)))
        return Operation(run, "Assign")

    def load(self, value, session=None):
        self.set(value)

    def set(self, value):
        """test helper: overwrite the value (numpy or torch), keeping dtype and leaf-ness."""
        v = value.detach() if isinstance(value, torch.Tensor) else torch.as_tensor(np.asarray(value))
        if self.store_float32:
            v = v.to(torch.float32)
        v = v.to(self._dtype.torch()).reshape(self._shape).clone()
        self.value = v.requires_grad_(self._dtype.kind == "f" and self.trainable)

    def numpy(self):
        return self.value.detach().numpy().copy()

    def eval(self, session=None):
        return self.numpy()

    # arithmetic on variables goes through the read tensor
    def __getattr__(self, item):
        if (item.startswith("__") and item.endswith("__")) or "_tensor" not in self.__dict__:
            raise AttributeError(item)
        return getattr(self.__dict__["_tensor"], item)

    def __mul__(self, o): return self._tensor * o
    def __rmul__(self, o): return o * self._tensor
    def __add__(self, o): return self._tensor + o
    def __radd__(self, o): return o + self._tensor
    def __sub__(self, o): return self._tensor - o
    def __rsub__(self, o): return o - self._tensor
    def __truediv__(self, o): return self._tensor / o

    def __repr__(self):
        return "<shim tf.Variable %s shape=%s>" % (self.name, tuple(self._shape))


def _glorot_uniform(shape, dtype):
    if len(shape) == 4:
        rf = shape[0] * shape[1]
        fan_in, fan_out = rf * shape[2], rf * shape[3]
    elif len(shape) == 2:
        fan_in, fan_out = shape
    else:
        fan_in = fan_out = int(np.prod(shape))
    lim = _pymath.sqrt(6.0 / (fan_in + fan_out))
    u = torch.rand(shape, generator=_graph.rng, dtype=torch.float32)
    return ((u * 2.0 - 1.0) * lim).to(dtype.torch())


def _zeros(shape, dtype):
    return torch.zeros(shape, dtype=dtype.torch())


def _ones(shape, dtype):
    return torch.ones(shape, dtype=dtype.torch())


def _const_init(c):
    return lambda shape, dtype: torch.full(shape, c, dtype=dtype.torch())


def zeros_initializer():
    return _zeros


def ones_initializer():
    return _ones


def glorot_uniform_initializer():
    return _glorot_uniform


def get_variable(name, shape=None, dtype=float32, initializer=None, trainable=True, **_kw):
    scope, reuse = _cur_scope()
    full = scope + "/" + name if scope else name
    if full in _graph.var_by_name:
        if reuse in (True, AUTO_REUSE):
            v = _graph.var_by_name[full]
            if shape is not None and [int(s) for s in shape] != v._shape:
                raise ValueError("Trying to share variable %s, but specified shape %r and found shape %r"
                                 % (full, tuple(shape), tuple(v._shape)))
            return v
        raise ValueError("Variable %s already exists, disallowed. Did you mean to set reuse=True or "
                         "reuse=tf.AUTO_REUSE in VarScope?" % full)
    if reuse is True:
        raise ValueError("Variable %s does not exist, or was not created with tf.get_variable()." % full)
    if initializer is None:
        initializer = _glorot_uniform if dtype.kind == "f" else _zeros      # TF1 get_variable default
    v = Variable(full, shape, dtype, initializer, trainable)
    _graph.variables.append(v)
    _graph.var_by_name[full] = v
    return v


def global_variables():
    return list(_graph.variables)


def trainable_variables(scope=None):
    return get_collection(GraphKeys.TRAINABLE_VARIABLES, scope)


def get_collection(key, scope=None):
    if key == GraphKeys.TRAINABLE_VARIABLES:
        items = [v for v in _graph.variables if v.trainable]
    elif key == GraphKeys.GLOBAL_VARIABLES:
        items = list(_graph.variables)
    elif key == GraphKeys.GLOBAL_STEP:
        items = [_graph.global_step] if _graph.global_step is not None else []
    else:
        items = []
    if scope is not None:
        rx = re.compile(scope)
        items = [v for v in items if rx.match(v.name)]        # TF: re.match(scope, item.name)
    return items


def global_variables_initializer():
    def run(ctx):
        for v in _graph.variables:
            v.initialize()
    return Operation(run, "init")


def assign(ref, value):
    return ref.assign(value)


def group(*inputs, **_kw):
    ops = []
    for i in inputs:
        ops.extend(i if isinstance(i, (list, tuple)) else [i])
    return Operation(lambda ctx: None, "group", deps=ops)


def no_op():
    return Operation(lambda ctx: None, "no_op")


# --------------------------------------------------------------------------------------------- element-wise / shape ops
def _f(x):
    return _as_tensor(x)


def to_float(x):
    return _unary(lambda v: v.to(_shim.FLOAT), x, dtype=float32)


def cast(x, dtype):
    return _unary(lambda v: v.to(dtype.torch()), x, dtype=dtype)


def clip_by_value(t, lo, hi):
    return _unary(lambda v: torch.clamp(v, lo, hi), t)


def tanh(x): return _unary(torch.tanh, x)
def exp(x): return _unary(torch.exp, x)
def log(x): return _unary(torch.log, x)
def square(x): return _unary(torch.square, x)
def sqrt(x): return _unary(torch.sqrt, x)
def sign(x): return _unary(torch.sign, x)
def sigmoid(x): return _unary(torch.sigmoid, x)


def abs(x): return _unary(torch.abs, x)   # noqa: A001


def add(a, b, name=None): return _binary(operator.add, a, b)
def subtract(a, b, name=None): return _binary(operator.sub, a, b)
def multiply(a, b, name=None): return _binary(operator.mul, a, b)


def _minmax(which):
    def op(a, b, name=None):
        def run(ctx, x, y):
            if not isinstance(x, torch.Tensor):
                x, y = y, x
            if not isinstance(y, torch.Tensor):
                return torch.clamp(x, max=y) if which == "min" else torch.clamp(x, min=y)
            return torch.minimum(x, y) if which == "min" else torch.maximum(x, y)
        return Tensor(run, [_as_tensor(a), _as_tensor(b)])
    return op


minimum = _minmax("min")
maximum = _minmax("max")


def where(cond, x, y):
    cond, x, y = _f(cond), _f(x), _f(y)
    return Tensor(lambda ctx, c, a, b: torch.where(c, a, b), [cond, x, y])


def stop_gradient(x, name=None):
    return Tensor(lambda ctx, v: v.detach(), [_f(x)], nondiff=True)


def zeros_like(x, **_kw):
    return _unary(torch.zeros_like, x, nondiff=True)


def ones_like(x, **_kw):
    return _unary(torch.ones_like, x, nondiff=True)


def reduce_sum(x, axis=None, keepdims=False, **_kw):
    if axis is None:
        return _unary(torch.sum, x)
    return _unary(lambda v: torch.sum(v, dim=axis, keepdim=keepdims), x)


def reduce_mean(x, axis=None, keepdims=False, **_kw):
    if axis is None:
        return _unary(torch.mean, x)
    return _unary(lambda v: torch.mean(v, dim=axis, keepdim=keepdims), x)


def reduce_max(x, axis=None, keepdims=False, **_kw):
    if axis is None:
        return _unary(torch.max, x)
    return _unary(lambda v: torch.max(v, dim=axis, keepdim=keepdims).values, x)


def argmax(x, axis=None, **_kw):
    def f(v):                                                   # tf.argmax: smallest index among ties, int64
        m = v.max(dim=axis, keepdim=True).values
        shape = [1] * v.dim()
        shape[axis] = v.shape[axis]
        idx = torch.arange(v.shape[axis]).reshape(shape).expand_as(v)
        return torch.where(v == m, idx, torch.full_like(idx, v.shape[axis])).min(dim=axis).values
    return _unary(f, x, nondiff=True, dtype=int64)


def one_hot(indices, depth, **_kw):
    def f(v):                                                   # out-of-range indices select nothing
        return (v.to(torch.int64).unsqueeze(-1) == torch.arange(int(depth))).to(_shim.FLOAT)
    return _unary(f, indices, nondiff=True, dtype=float32)


def concat(values, axis, name=None):
    vals = [_f(v) for v in values]
    return Tensor(lambda ctx, *vs: torch.cat(vs, dim=axis), vals)


def stack(values, axis=0, name=None):
    vals = [_f(v) for v in values]
    return Tensor(lambda ctx, *vs: torch.stack(vs, dim=axis), vals)


def expand_dims(x, axis, **_kw):
    return _unary(lambda v: v.unsqueeze(axis), x)


def squeeze(x, axis=None, **_kw):
    if axis is None:
        return _unary(torch.squeeze, x)
    ax = axis if isinstance(axis, int) else tuple(axis)
    return _unary(lambda v: v.squeeze(ax), x)


def transpose(x, perm=None, **_kw):
    if perm is None:
        return _unary(lambda v: v.permute(*reversed(range(v.dim()))), x)
    return _unary(lambda v: v.permute(*perm), x)


def reshape(x, shape, **_kw):
    return _unary(lambda v: v.reshape([int(s) for s in shape]), x)


def split(value, num_or_size_splits, axis=0, **_kw):
    v = _f(value)
    n = int(num_or_size_splits)
    return [Tensor(lambda ctx, t, k=k: torch.chunk(t, n, dim=axis)[k], [v]) for k in range(n)]


def matmul(a, b, **_kw):
    return _binary(torch.matmul, a, b)


def scan(fn, elems, initializer=None, parallel_iterations=10, back_prop=True, swap_memory=False,
         infer_shape=True, reverse=False, name=None):
    """tf.scan over axis 0 of every tensor in ``elems`` (a tensor or a (nested) tuple); ``fn(acc, item)`` is the
    caller's own Python function and is called with shim tensors, once per step, at evaluation time."""
    is_seq = isinstance(elems, (list, tuple))
    elems_l = [_f(e) for e in (elems if is_seq else [elems])]
    if initializer is None:
        raise NotImplementedError("shim tf.scan needs an initializer")
    init = _f(initializer)

    def run(ctx, acc, *es):
        if not back_prop:
            acc, es = acc.detach(), [e.detach() for e in es]
        n = es[0].shape[0]
        order = range(n - 1, -1, -1) if reverse else range(n)
        outs = [None] * n
        for t in order:
            items = [Tensor(lambda c, v=e[t]: v) for e in es]
            r = fn(Tensor(lambda c, v=acc: v), type(elems)(items) if is_seq else items[0])
            acc = _f(r)._eval(_Ctx(ctx.feeds, ctx.dummy))
            outs[t] = acc
        out = torch.stack(outs, dim=0)
        return out if back_prop else out.detach()

    return Tensor(run, [init] + elems_l, nondiff=not back_prop)


def clip_by_global_norm(t_list, clip_norm, use_norm=None, name=None):
    present = [(_f(t) if t is not None else None) for t in t_list]
    live = [t for t in present if t is not None]
    gnorm = Tensor(lambda ctx, *ts: torch.sqrt(sum(torch.sum(t * t) for t in ts)), live)
    # TF 1.14 clip_ops: scale_for_finite + (norm - norm), so a NaN or infinite norm makes every clipped gradient NaN
    scale = Tensor(lambda ctx, n: clip_norm * torch.minimum(1.0 / n, torch.ones_like(n) / clip_norm) + (n - n), [gnorm])
    return [None if t is None else Tensor(lambda ctx, v, s: v * s, [t, scale]) for t in present], gnorm


def global_norm(t_list):
    live = [_f(t) for t in t_list if t is not None]
    return Tensor(lambda ctx, *ts: torch.sqrt(sum(torch.sum(t * t) for t in ts)), live)


class _Math:
    sqrt = staticmethod(sqrt)
    sign = staticmethod(sign)
    abs = staticmethod(abs)
    square = staticmethod(square)
    exp = staticmethod(exp)
    log = staticmethod(log)
    tanh = staticmethod(tanh)
    sigmoid = staticmethod(sigmoid)
    minimum = staticmethod(minimum)
    maximum = staticmethod(maximum)
    reduce_sum = staticmethod(reduce_sum)
    reduce_mean = staticmethod(reduce_mean)
    argmax = staticmethod(argmax)


math = _Math   # tf.math (the stdlib module is bound as _pymath)


# --------------------------------------------------------------------------------------------- tf.nn / tf.layers
class _LSTMStateTuple(tuple):
    def __new__(cls, c, h):
        return tuple.__new__(cls, (c, h))

    c = property(lambda self: self[0])
    h = property(lambda self: self[1])


class _LSTMCell:
    """tf.nn.rnn_cell.LSTMCell(num_units): no peepholes, no projection, forget_bias=1.0, tanh, state_is_tuple."""

    def __init__(self, num_units, forget_bias=1.0, **_kw):
        self._num_units = int(num_units)
        self._forget_bias = forget_bias
        self._scope_name = None

    def _vars(self, input_depth):
        if self._scope_name is None:                       # Layer._set_scope: default_name = 'lstm_cell'
            with variable_scope(None, default_name="lstm_cell") as s:
                self._scope_name = s
        with variable_scope(self._scope_name):
            k = get_variable("kernel", [input_depth + self._num_units, 4 * self._num_units])
            b = get_variable("bias", [4 * self._num_units], initializer=_zeros)
        return k, b

    def step(self, x, c_prev, h_prev, kernel, bias):
        z = torch.cat([x, h_prev], dim=1) @ kernel + bias
        i, j, f, o = torch.chunk(z, 4, dim=1)              # TF order: input, new input, forget, output
        c = torch.sigmoid(f + self._forget_bias) * c_prev + torch.sigmoid(i) * torch.tanh(j)
        h = torch.sigmoid(o) * torch.tanh(c)
        return h, c


def _dynamic_rnn(cell, inputs, sequence_length=None, initial_state=None, dtype=None, scope=None, **_kw):
    inputs = _f(inputs)
    depth = inputs.get_shape()[2].value
    with variable_scope(scope or "rnn"):
        kernel, bias = cell._vars(depth)
    c0, h0 = _f(initial_state[0]), _f(initial_state[1])

    def run(ctx, x, c, h, k, b):
        outs = []
        for t in range(x.shape[1]):
            h, c = cell.step(x[:, t], c, h, k, b)
            outs.append(h)
        return torch.stack(outs, dim=1), c, h

    packed = Tensor(run, [inputs, c0, h0, kernel._tensor, bias._tensor])
    out = Tensor(lambda ctx, p: p[0], [packed], float32)
    c = Tensor(lambda ctx, p: p[1], [packed], float32)
    h = Tensor(lambda ctx, p: p[2], [packed], float32)
    return out, _LSTMStateTuple(c, h)


class _RnnCell:
    LSTMStateTuple = _LSTMStateTuple
    LSTMCell = _LSTMCell


def _relu(x, name=None):
    return _unary(torch.relu, x)


def _softmax(x, axis=-1, name=None):
    return _unary(lambda v: torch.softmax(v, dim=axis), x)


class _NN:
    relu = staticmethod(_relu)
    softmax = staticmethod(_softmax)
    tanh = staticmethod(tanh)
    sigmoid = staticmethod(sigmoid)
    rnn_cell = _RnnCell
    dynamic_rnn = staticmethod(_dynamic_rnn)


nn = _NN


def _conv2d(inputs, filters, kernel_size, strides=(1, 1), padding="valid", activation=None, use_bias=True,
            name=None, **_kw):
    if str(padding).upper() != "VALID":
        raise NotImplementedError("shim conv2d: VALID padding only (all the reference uses)")
    x = _f(inputs)
    cin = x.get_shape()[3].value
    kh, kw = (kernel_size, kernel_size) if isinstance(kernel_size, int) else kernel_size
    st = (strides, strides) if isinstance(strides, int) else tuple(strides)
    with variable_scope(name, default_name="conv2d"):
        k = get_variable("kernel", [kh, kw, cin, filters])
        b = get_variable("bias", [filters], initializer=_zeros) if use_bias else None

    def run(ctx, v, kv, *bv):
        y = F.conv2d(v.permute(0, 3, 1, 2), kv.permute(3, 2, 0, 1), bv[0] if bv else None, stride=st)
        return y.permute(0, 2, 3, 1)

    y = Tensor(run, [x, k._tensor] + ([b._tensor] if b is not None else []), float32)
    return activation(y) if activation is not None else y


def _dense(inputs, units, activation=None, use_bias=True, name=None, **_kw):
    x = _f(inputs)
    cin = x.get_shape()[-1].value
    with variable_scope(name, default_name="dense"):
        k = get_variable("kernel", [cin, units])
        b = get_variable("bias", [units], initializer=_zeros) if use_bias else None
    y = Tensor(lambda ctx, v, kv, *bv: (v @ kv + bv[0]) if bv else v @ kv,
               [x, k._tensor] + ([b._tensor] if b is not None else []), float32)
    return activation(y) if activation is not None else y


def _flatten(inputs, name=None):
    return _unary(lambda v: v.reshape(v.shape[0], -1), inputs)


class _Layers:
    conv2d = staticmethod(_conv2d)
    dense = staticmethod(_dense)
    flatten = staticmethod(_flatten)


layers = _Layers


# --------------------------------------------------------------------------------------------- tf.train
def _reachable_variables(loss):
    """Variables the gradient of ``loss`` can reach (stop_gradient & co. block the walk, like tf.gradients)."""
    seen, out, stack = set(), set(), [loss]
    while stack:
        n = stack.pop()
        if id(n) in seen:
            continue
        seen.add(id(n))
        if getattr(n, "_variable", None) is not None:
            out.add(id(n._variable))
        if n.nondiff:
            continue
        stack.extend(n._inputs)
    return out


def gradients(ys, xs, **_kw):
    ys = _f(ys)
    xs = list(xs)
    tens = [_f(x) for x in xs]
    reach = _reachable_variables(ys)

    def run(ctx, y, *vals):
        g = torch.autograd.grad(y, list(vals), allow_unused=True, retain_graph=True)
        return [None if gi is None else gi.detach() for gi in g]

    live = [(i, t) for i, t in enumerate(tens) if getattr(t, "_variable", None) is None or id(t._variable) in reach]
    bundle = Tensor(run, [ys] + [t for _, t in live], nondiff=True)
    out = [None] * len(xs)
    for pos, (i, t) in enumerate(live):
        out[i] = Tensor(lambda ctx, b, pos=pos, t=t: b[pos] if b[pos] is not None else torch.zeros_like(t._eval(ctx)),
                        [bundle], float32, nondiff=True)
    return out


class _Optimizer:
    def compute_gradients(self, loss, var_list=None, **_kw):
        var_list = list(var_list) if var_list is not None else trainable_variables()
        grads = gradients(loss, var_list)
        return list(zip(grads, var_list))

    def minimize(self, loss, global_step=None, var_list=None, **_kw):
        return self.apply_gradients(self.compute_gradients(loss, var_list), global_step=global_step)

    def apply_gradients(self, grads_and_vars, global_step=None, name=None):
        gv = [(g, v) for g, v in grads_and_vars if g is not None]
        if not gv:
            raise ValueError("No gradients provided for any variable")
        self._create_slots([v for _, v in gv])
        lr = _f(self._lr)

        def run(ctx):
            lr_v = lr._eval(ctx)
            lr_v = lr_v.detach() if isinstance(lr_v, torch.Tensor) else lr_v
            self._prepare(ctx)
            for g, v in gv:
                self._apply(ctx, g._eval(ctx).detach(), v, lr_v)
            self._finish(ctx)
            if global_step is not None:
                ctx.staged.append((global_step, global_step.value + 1))

        return Operation(run, name or type(self).__name__)

    def _prepare(self, ctx): pass
    def _finish(self, ctx): pass


class RMSPropOptimizer(_Optimizer):
    """tf.train.RMSPropOptimizer (not centered): slots ``<var>/RMSProp`` (ms, ones) and ``<var>/RMSProp_1`` (momentum)."""
    _name = "RMSProp"
    _name_in_slot = True

    def __init__(self, learning_rate, decay=0.9, momentum=0.0, epsilon=1e-10, use_locking=False, centered=False,
                 name="RMSProp"):
        if centered:
            raise NotImplementedError
        self._lr, self._decay, self._momentum, self._epsilon = learning_rate, decay, momentum, epsilon
        self._slots = {}

    def _create_slots(self, var_list):
        for v in var_list:
            ms = self._slot_named(v, "RMSProp", _ones)
            mom = self._slot_named(v, "RMSProp_1", _zeros)
            self._slots[id(v)] = (ms, mom)

    @staticmethod
    def _slot_named(var, suffix, init):
        name = var.op_name + "/" + suffix
        if name not in _graph.var_by_name:
            v = Variable(name, var._shape, var._dtype, init, trainable=False)
            _graph.variables.append(v)
            _graph.var_by_name[name] = v
        return _graph.var_by_name[name]

    def get_slot(self, var, name):
        ms, mom = self._slots[id(var)]
        return {"rms": ms, "momentum": mom}[name]

    def _apply(self, ctx, g, var, lr):
        ms, mom = self._slots[id(var)]
        ms_new = ms.value + (g * g - ms.value) * (1.0 - self._decay)
        mom_new = mom.value * self._momentum + lr * g * torch.rsqrt(ms_new + self._epsilon)
        ctx.staged += [(ms, ms_new), (mom, mom_new), (var, var.value.detach() - mom_new)]


class AdamOptimizer(_Optimizer):
    """tf.train.AdamOptimizer: slots ``<var>/Adam`` (m), ``<var>/Adam_1`` (v); non-slot beta1_power / beta2_power."""
    _name = "Adam"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, use_locking=False, name="Adam"):
        self._lr, self._b1, self._b2, self._epsilon = learning_rate, beta1, beta2, epsilon
        self._slots = {}
        self._powers = None

    def _create_slots(self, var_list):
        first = min(var_list, key=lambda v: v.name)
        if self._powers is None:
            scope = first.op_name.rsplit("/", 1)[0] if "/" in first.op_name else ""
            mk = lambda nm, c: Variable((scope + "/" if scope else "") + nm, [], float32, _const_init(c), trainable=False)
            self._powers = (mk("beta1_power", self._b1), mk("beta2_power", self._b2))
            for p in self._powers:
                # TF keeps the beta powers as float32 variables; their rounding is visible in the first Adam steps
                # (1 - 0.999 loses 1.3e-5 relative), so they stay float32-rounded even when FLOAT is float64
                p.store_float32 = True
                p.set(p.value)
                _graph.variables.append(p)
                _graph.var_by_name.setdefault(p.op_name, p)
        for v in var_list:
            self._slots[id(v)] = (RMSPropOptimizer._slot_named(v, "Adam", _zeros),
                                  RMSPropOptimizer._slot_named(v, "Adam_1", _zeros))

    def get_slot(self, var, name):
        m, v = self._slots[id(var)]
        return {"m": m, "v": v}[name]

    def _apply(self, ctx, g, var, lr):
        m, v = self._slots[id(var)]
        b1p, b2p = self._powers[0].value, self._powers[1].value
        lr_t = lr * torch.sqrt(1.0 - b2p) / (1.0 - b1p)
        m_new = m.value + (g - m.value) * (1.0 - self._b1)
        v_new = v.value + (g * g - v.value) * (1.0 - self._b2)
        ctx.staged += [(m, m_new), (v, v_new),
                       (var, var.value.detach() - lr_t * m_new / (torch.sqrt(v_new) + self._epsilon))]

    def _finish(self, ctx):
        # float32 variable times float32 constant, rounded to float32 by Variable.set (store_float32)
        ctx.staged += [(self._powers[0], self._powers[0].value * float(np.float32(self._b1))),
                       (self._powers[1], self._powers[1].value * float(np.float32(self._b2)))]


class GradientDescentOptimizer(_Optimizer):
    _name = "GradientDescent"

    def __init__(self, learning_rate, **_kw):
        self._lr = learning_rate

    def _create_slots(self, var_list): pass

    def _apply(self, ctx, g, var, lr):
        ctx.staged.append((var, var.value.detach() - lr * g))


def _get_or_create_global_step(graph=None):
    if _graph.global_step is None:
        v = Variable("global_step", [], int64, _zeros, trainable=False)
        _graph.variables.append(v)
        _graph.var_by_name["global_step"] = v
        _graph.global_step = v
    return _graph.global_step


def _polynomial_decay(learning_rate, global_step, decay_steps, end_learning_rate=0.0001, power=1.0, cycle=False,
                      name=None):
    if cycle:
        raise NotImplementedError
    gs = _f(global_step)

    def run(ctx, step):
        # the learning rate is a float32 tensor in the TF graph whatever the model's arithmetic: evaluate the op
        # sequence of tf.train.polynomial_decay in float32, then lift
        f = torch.float32
        s = torch.minimum(step.to(f), torch.tensor(float(decay_steps), dtype=f))
        p = s / torch.tensor(float(decay_steps), dtype=f)
        lr = (torch.tensor(learning_rate, dtype=f) - torch.tensor(end_learning_rate, dtype=f)) * \
            torch.pow(torch.tensor(1.0, dtype=f) - p, torch.tensor(power, dtype=f)) + torch.tensor(end_learning_rate, dtype=f)
        return lr.to(_shim.FLOAT)

    return Tensor(run, [gs], float32, nondiff=True)


class _Saver:
    """tf.train.Saver(): every global variable by name, one .npz (enough for save_weights/load_weights round trips)."""

    def __init__(self, var_list=None, **_kw):
        self._vars = list(var_list) if var_list is not None else None

    def _all(self):
        return self._vars if self._vars is not None else list(_graph.variables)

    def save(self, sess, path, **_kw):
        np.savez(path + ".shim.npz", **{v.op_name: v.numpy() for v in self._all()})
        return path

    def restore(self, sess, path):
        with np.load(path + ".shim.npz") as z:
            for v in self._all():
                v.set(z[v.op_name])


class _Server:
    def __init__(self, *a, **k):
        self.target = "shim"

    def join(self):
        raise RuntimeError("shim tf.train.Server cannot serve")


class _Train:
    RMSPropOptimizer = RMSPropOptimizer
    AdamOptimizer = AdamOptimizer
    GradientDescentOptimizer = GradientDescentOptimizer
    get_or_create_global_step = staticmethod(_get_or_create_global_step)
    get_global_step = staticmethod(lambda graph=None: _graph.global_step)
    polynomial_decay = staticmethod(_polynomial_decay)
    Saver = _Saver
    Server = _Server
    ClusterSpec = staticmethod(lambda *a, **k: None)


train = _Train


# --------------------------------------------------------------------------------------------- queues
class FIFOQueue:
    """tf.FIFOQueue(capacity, dtypes, shared_name=...): in-process; queues with the same shared_name share storage.
    (Blocking on full/empty needs a second thread in TF as well; here a dequeue from an empty queue raises.)"""

    def __init__(self, capacity, dtypes, shapes=None, names=None, shared_name=None, name="fifo_queue"):
        import collections
        self._capacity = capacity
        self._dtypes = list(dtypes)
        key = shared_name or id(self)
        self._items = _graph.queues.setdefault(key, collections.deque())

    def size(self, name=None):
        return Tensor(lambda ctx: torch.tensor(len(self._items), dtype=torch.int64), (), int32, nondiff=True)

    def enqueue(self, vals, name=None):
        vals = [_f(v) for v in vals]

        def run(ctx):
            if len(self._items) >= self._capacity:
                raise RuntimeError("shim FIFOQueue is full (a TF enqueue would block)")
            self._items.append([v._eval(ctx) for v in vals])
        return Operation(run, "enqueue")

    def dequeue(self, name=None):
        n = len(self._dtypes)

        class _Dequeue(Tensor):
            def _eval(s, ctx):        # not memoised across runs; once per run
                k = id(s)
                if k not in ctx.memo:
                    if ctx.dummy is not None:
                        raise RuntimeError("static shape of a dequeue is unknown")
                    if not self._items:
                        raise RuntimeError("shim FIFOQueue is empty (a TF dequeue would block)")
                    ctx.memo[k] = (s, self._items.popleft())
                return ctx.memo[k][1]

        bundle = _Dequeue(None, ())
        return [Tensor(lambda ctx, b, i=i: b[i], [bundle], self._dtypes[i], nondiff=True) for i in range(n)]


# --------------------------------------------------------------------------------------------- session
def _to_numpy(v, dtype):
    if isinstance(v, (list, tuple)):
        return [_to_numpy(x, None) for x in v]
    a = v.detach().numpy()
    if a.dtype == np.float64 and _shim.FLOAT == torch.float64:
        return a.copy() if a.ndim else np.float64(a)
    if a.dtype.kind == "f":
        return a.astype(np.float32) if a.ndim else np.float32(a)
    if a.dtype == np.int64 and dtype is not None and dtype.name == "int32":
        a = a.astype(np.int32)
    return a.copy() if a.ndim else a[()]


class Session:
    def __init__(self, target="", graph=None, config=None):
        self.target = target

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def close(self):
        pass

    def run(self, fetches, feed_dict=None, **_kw):
        _graph.shape_ctx.clear()                       # construction-time caches are not needed any more
        feeds = {}
        for k, v in (feed_dict or {}).items():
            feeds[id(k)] = v
        ctx = _Ctx(feeds)

        tensors, ops = [], []

        def collect(f):
            if isinstance(f, (list, tuple)):
                for x in f:
                    collect(x)
            elif isinstance(f, Variable):
                tensors.append(f._tensor)
            elif getattr(f, "_is_op", False):
                ops.append(f)
            elif isinstance(f, Tensor):
                tensors.append(f)
            else:
                raise TypeError("Fetch argument %r has invalid type %r" % (f, type(f)))

        collect(fetches)
        for t in tensors:          # 1) every tensor fetch on the pre-update variables
            t._eval(ctx)
        for o in ops:              # 2) ops compute their new values from the same evaluation
            o._eval(ctx)
        with torch.no_grad():      # 3) commit
            for var, val in ctx.staged:
                var.set(val.detach() if isinstance(val, torch.Tensor) else val)

        def result(f):
            if isinstance(f, (list, tuple)):
                return [result(x) for x in f]
            if isinstance(f, Variable):
                return f.numpy()
            if getattr(f, "_is_op", False):
                return None
            return _to_numpy(ctx.memo[id(f)][1], f._dtype)

        return result(fetches)


InteractiveSession = Session


class ConfigProto:
    def __init__(self, *a, **k):
        pass


class _Flags:
    def __getattr__(self, item):
        raise AttributeError(item)


class _App:
    class flags:
        FLAGS = _Flags()

        @staticmethod
        def DEFINE_string(*a, **k): pass

        @staticmethod
        def DEFINE_integer(*a, **k): pass

    @staticmethod
    def run(main=None, argv=None):
        raise RuntimeError("shim tf.app.run is not supported")


app = _App
