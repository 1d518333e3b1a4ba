"""A NumPy stand-in for the handful of TensorFlow 1.14 primitives the reference's
interaction-layer files call (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Purpose: TF 1.14 cannot be installed here (Python 3.12, no wheel, no network), but the
reference's layer files are plain Python that only *compose* TF primitives.  Putting this
package first on ``sys.path`` lets ``oracle/make_golden.py`` import and run

    DCN/cross_layer.py, xDeepFM/cin_layer.py, DIN/din_attention.py,
    FiBiNET/senet.py, FiBiNET/bilinear_interaction_layer.py

*verbatim from the reference checkout* (nothing is copied), eagerly, on injected weights, so the
reference's own control flow -- loop bounds, pair enumeration, mask/where/scale order,
reshape index order, variable shapes -- is what produces the golden vectors.  What is NOT
pinned by this is the arithmetic inside each TF primitive (Eigen summation order etc.);
each primitive below states the public TF 1.14 semantics it implements.

The same shim also runs the INLINE interaction blocks of DeepFM/NFM/FwFM/AFM model_fns: make_golden.py reads the
cited line ranges from the reference checkout at generation time and exec()s them with a stand-in ``fc.input_layer``.

Only what those files touch is implemented.  Everything evaluates eagerly on
``numpy`` arrays in ``_STATE.dtype`` (float32 like the reference, or float64 for the
high-precision anchor).
"""
from __future__ import annotations

import contextlib

import numpy as _np

float32 = _np.float32
float64 = _np.float64
int32 = _np.int32
int64 = _np.int64
AUTO_REUSE = object()


class _State:
    dtype = _np.float32
    scope: list = []
    variables: dict = {}     # full name -> ndarray (injected by the caller, or created + recorded)
    created: dict = {}       # name -> shape, for every get_variable call (so tests can check shapes)
    uniq: dict = {}          # scope-name counters for layers that uniquify their scope (LayerNorm, LayerNorm_1, ...)
    rng = _np.random.default_rng(0)


_STATE = _State()


def reset(dtype=_np.float32, variables=None, seed=0):
    _STATE.dtype = dtype
    _STATE.scope = []
    _STATE.variables = dict(variables or {})
    _STATE.created = {}
    _STATE.uniq = {}
    _STATE.rng = _np.random.default_rng(seed)


def created_variables():
    return dict(_STATE.created)


class Dimension:
    """tf.Dimension: supports int(), .value, arithmetic and use as a range() bound."""

    def __init__(self, v):
        self.value = int(v)

    def __int__(self):
        return self.value

    __index__ = __int__

    def _b(self, o):
        return int(o)

    def __sub__(self, o): return Dimension(self.value - self._b(o))
    def __add__(self, o): return Dimension(self.value + self._b(o))
    def __mul__(self, o): return Dimension(self.value * self._b(o))
    def __rmul__(self, o): return Dimension(self.value * self._b(o))
    def __floordiv__(self, o): return Dimension(self.value // self._b(o))
    def __eq__(self, o): return self.value == int(o)
    def __lt__(self, o): return self.value < int(o)
    def __hash__(self): return hash(self.value)
    def __repr__(self): return f"Dimension({self.value})"


class TensorShape:
    def __init__(self, shape):
        self._s = tuple(int(s) for s in shape)

    def __getitem__(self, i):
        return Dimension(self._s[i])

    def __len__(self):
        return len(self._s)

    def as_list(self):
        return list(self._s)


def _arr(x):
    if isinstance(x, Tensor):
        return x.a
    if isinstance(x, (Dimension,)):
        return int(x)
    return x


class Tensor:
    __array_priority__ = 1000

    def __init__(self, a):
        self.a = _np.asarray(a)

    @property
    def shape(self):
        return TensorShape(self.a.shape)

    @property
    def dtype(self):
        return self.a.dtype

    def get_shape(self):
        return TensorShape(self.a.shape)

    def numpy(self):
        return self.a

    def __getitem__(self, idx):
        return Tensor(self.a[idx])

    def _bin(self, o, f, rev=False):
        b = _arr(o)
        if not isinstance(b, _np.ndarray) and self.a.dtype.kind == 'f':
            b = self.a.dtype.type(b)          # python scalar takes the tensor's dtype (TF semantics)
        return Tensor(f(b, self.a) if rev else f(self.a, b))

    def __add__(self, o): return self._bin(o, _np.add)
    def __radd__(self, o): return self._bin(o, _np.add, True)
    def __sub__(self, o): return self._bin(o, _np.subtract)
    def __rsub__(self, o): return self._bin(o, _np.subtract, True)
    def __mul__(self, o): return self._bin(o, _np.multiply)
    def __rmul__(self, o): return self._bin(o, _np.multiply, True)
    def __truediv__(self, o): return self._bin(o, _np.divide)
    def __neg__(self): return Tensor(-self.a)


def _t(x):
    return x if isinstance(x, Tensor) else Tensor(_np.asarray(x))


# ---- variables / scopes -------------------------------------------------------------

@contextlib.contextmanager
def variable_scope(name, reuse=None):
    _STATE.scope.append(name)
    try:
        yield
    finally:
        _STATE.scope.pop()


def _full_name(name):
    return "/".join(_STATE.scope + [name])


def get_variable(name, shape=None, dtype=None, initializer=None):
    """tf.get_variable: looked up by scoped name among the injected variables; if absent it is
    created with a glorot-uniform draw (the TF1 default initializer) and recorded."""
    full = _full_name(name)
    shp = (int(shape),) if isinstance(shape, (int, _np.integer, Dimension)) else tuple(int(s) for s in shape)   # `shape=n` is legal TF
    _STATE.created[full] = shp
    if full not in _STATE.variables:
        fan_in = shp[0] if len(shp) < 3 else int(_np.prod(shp[:-2])) * shp[-2]
        fan_out = shp[-1] if len(shp) < 3 else int(_np.prod(shp[:-2])) * shp[-1]
        lim = (6.0 / (fan_in + fan_out)) ** 0.5
        _STATE.variables[full] = _STATE.rng.uniform(-lim, lim, size=shp)
    v = _np.asarray(_STATE.variables[full])
    assert v.shape == shp, f"variable {full}: injected {v.shape} but reference asks for {shp}"
    return Tensor(v.astype(_STATE.dtype))


# ---- ops ---------------------------------------------------------------------------

def matmul(a, b, transpose_a=False, transpose_b=False):
    """tf.matmul: (batched) matrix product over the last two axes."""
    A, B = _arr(a), _arr(b)
    if transpose_a:
        A = _np.swapaxes(A, -1, -2)
    if transpose_b:
        B = _np.swapaxes(B, -1, -2)
    return Tensor(_np.matmul(A, B))


def multiply(a, b): return Tensor(_np.multiply(_arr(a), _arr(b)))
def add(a, b): return Tensor(_np.add(_arr(a), _arr(b)))
def square(a): return Tensor(_np.square(_arr(a)))


def scalar_mul(scalar, x):
    """tf.scalar_mul(scalar, x) = scalar * x (scalar is a 0-d tensor)."""
    return Tensor(_arr(scalar) * _arr(x))


def add_n(xs):
    """tf.add_n: accumulates in list order."""
    acc = _arr(xs[0])
    for x in xs[1:]:
        acc = acc + _arr(x)
    return Tensor(acc)


def transpose(a, perm=None): return Tensor(_np.transpose(_arr(a), perm))
def reshape(a, shape): return Tensor(_np.reshape(_arr(a), tuple(int(_arr(s)) for s in shape)))
def expand_dims(a, axis): return Tensor(_np.expand_dims(_arr(a), axis))
def squeeze(a, axis=None): return Tensor(_np.squeeze(_arr(a), axis))
def concat(xs, axis): return Tensor(_np.concatenate([_arr(x) for x in xs], axis=axis))
def stack(xs, axis=0): return Tensor(_np.stack([_arr(x) for x in xs], axis=axis))
def tile(a, multiples): return Tensor(_np.tile(_arr(a), tuple(int(_arr(m)) for m in multiples)))
def ones_like(a): return Tensor(_np.ones_like(_arr(a)))
def reduce_mean(a, axis=None, keepdims=False): return Tensor(_np.mean(_arr(a), axis=axis, keepdims=keepdims))
def reduce_sum(a, axis=None, keepdims=False): return Tensor(_np.sum(_arr(a), axis=axis, keepdims=keepdims))
def where(c, x, y): return Tensor(_np.where(_arr(c), _arr(x), _arr(y)))
def constant(v, dtype=None): return Tensor(_np.asarray(v, dtype=dtype))


def cast(a, dtype):
    d = _STATE.dtype if dtype in (float32, float64) else dtype
    return Tensor(_arr(a).astype(d))


def shape(a):
    """tf.shape: here an eager tuple of ints."""
    return tuple(_arr(a).shape)


def einsum(eq, *ops):
    """tf.einsum; the reference writes the equation with spaces around '->'."""
    return Tensor(_np.einsum(eq.replace(" ", ""), *[_arr(o) for o in ops]))


def sequence_mask(lengths, maxlen, dtype=None):
    """tf.sequence_mask(len, T)[b, t] = t < len[b]  (bool, or cast to `dtype` -- an EXPLICIT tf.float32 stays float32 even in
    the float64 anchor run, as it would in TF)."""
    L = _arr(lengths)
    m = _np.arange(int(_arr(maxlen)))[None, :] < L[:, None]
    return Tensor(m if dtype is None else m.astype(dtype))


def range(n):                                  # noqa: A001  (tf.range)
    return Tensor(_np.arange(int(_arr(n))))


def abs(a):                                    # noqa: A001  (tf.abs)
    return Tensor(_np.abs(_arr(a)))


def random_normal(shape, seed=None):
    return Tensor(_STATE.rng.standard_normal(tuple(shape)).astype(_STATE.dtype))


class _NN:
    @staticmethod
    def relu(a):
        return Tensor(_np.maximum(_arr(a), 0))

    @staticmethod
    def softmax(a, axis=-1):
        x = _arr(a)
        x = x - x.max(axis=axis, keepdims=True)
        e = _np.exp(x)
        return Tensor(e / e.sum(axis=axis, keepdims=True))

    @staticmethod
    def embedding_lookup(params, ids):
        """tf.nn.embedding_lookup(table, ids) = table[ids] (single dense table)."""
        return Tensor(_arr(params)[_arr(ids)])

    @staticmethod
    def safe_embedding_lookup_sparse(embedding_weights, sparse_ids, sparse_weights=None, combiner="mean"):
        """tf.nn.safe_embedding_lookup_sparse for ONE id per row, the only way FFM/ffm.py:156-157 uses it (its sparse ids come
        from a one-hot row): here `sparse_ids` is the (B,) id vector itself, -1 = empty row -> zero vector (the 'safe' part)."""
        w, ids = _arr(embedding_weights), _np.asarray(_arr(sparse_ids))
        out = w[_np.maximum(ids, 0)]
        return Tensor(_np.where((ids >= 0)[:, None], out, 0).astype(w.dtype))

    @staticmethod
    def conv1d(value, filters, stride, padding):
        """tf.nn.conv1d(x:(B,W,C), filters:(fw,C,O), stride, padding).  Only the reference's use is
        supported: fw == 1, stride 1, VALID  ==  x @ filters[0] at every position."""
        f = _arr(filters)
        assert f.shape[0] == 1 and stride == 1 and padding == "VALID"
        return Tensor(_np.matmul(_arr(value), f[0]))


nn = _NN()


class _Layers:
    @staticmethod
    def dense(inputs, units, activation=None, use_bias=True, name=None, reuse=None):
        """tf.layers.dense: variables <name>/kernel (in, units) and <name>/bias (units,);
        out = activation(x @ kernel + bias) over the last axis."""
        x = _arr(inputs)
        with variable_scope(name or "dense"):
            k = get_variable("kernel", shape=(x.shape[-1], units))
            y = _np.matmul(x, k.a)
            if use_bias:
                if _full_name("bias") not in _STATE.variables:
                    _STATE.variables[_full_name("bias")] = _np.zeros((units,))   # zeros_initializer
                y = y + get_variable("bias", shape=(units,)).a
        out = Tensor(y)
        return activation(out) if activation is not None else out


layers = _Layers()


class _ContribLayers:
    @staticmethod
    def layer_norm(inputs, center=True, scale=True, begin_norm_axis=1, begin_params_axis=-1, scope=None):
        """tf.contrib.layers.layer_norm (TF 1.14 defaults): moments over axes [begin_norm_axis:] -- for a (B,T,d) input that
        is T AND d together --, beta (zeros) / gamma (ones) of shape inputs.shape[begin_params_axis:] in variable scope
        'LayerNorm' (uniquified 'LayerNorm_1', ... on later calls in the same scope), then
        tf.nn.batch_normalization(x, mean, var, beta, gamma, variance_epsilon=1e-12):
        inv = rsqrt(var + eps) * gamma;  y = x * inv + (beta - mean * inv)."""
        x = _arr(inputs)
        base = _full_name(scope or "LayerNorm")
        n = _STATE.uniq.get(base, 0)
        _STATE.uniq[base] = n + 1
        with variable_scope((scope or "LayerNorm") + (f"_{n}" if n else "")):
            pshape = x.shape[begin_params_axis:]
            for nm, init in (("beta", _np.zeros), ("gamma", _np.ones)):
                if _full_name(nm) not in _STATE.variables:
                    _STATE.variables[_full_name(nm)] = init(pshape)
            beta, gamma = get_variable("beta", shape=pshape).a, get_variable("gamma", shape=pshape).a
        axes = tuple(_np.arange(begin_norm_axis, x.ndim))
        mean = x.mean(axis=axes, keepdims=True)
        var = _np.mean(_np.square(x - mean), axis=axes, keepdims=True)
        inv = (1.0 / _np.sqrt(var + x.dtype.type(1e-12))) * gamma
        return Tensor(x * inv + (beta - mean * inv))


class _Contrib:
    layers = _ContribLayers()


contrib = _Contrib()


class _KerasBackend:
    @staticmethod
    def batch_dot(x, y, axes=None):
        """tf.keras.backend.batch_dot for the reference's only use (FwFM/fwfm.py:156): two (B, K) tensors, axes=1
        -> (B, 1) (Keras keeps a trailing unit axis when the result would be rank 1)."""
        X, Y = _arr(x), _arr(y)
        assert X.ndim == 2 and Y.ndim == 2 and axes == 1
        return Tensor(_np.sum(X * Y, axis=1, keepdims=True))


class _Keras:
    backend = _KerasBackend()


keras = _Keras()
