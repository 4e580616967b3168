"""oracle/sec_layers.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (the in-place runs need the reference mounted).

Runs the reference's OWN SeedLossLayer and ExpandLossLayer (pylayers/pylayers/pylayers.py:95-118, :183-233)
in place, the way oracle/ref_layers.py runs the other layers: their ``ClassDef`` nodes are pulled out with ``ast``
and executed against a Theano stand-in.  The stand-in here extends oracle/theano_shim.py (left as it is, so the
goldens it pins cannot move) with what these two class bodies use:

* ``T.sort`` (torch.sort: the gradient of a sorted position goes to the element argsort put there, SortOp.grad),
* ``.max(axis=)`` / ``T.max`` with Theano's tie gradient: MaxAndArgmax.grad is ``eq(xmax, x) * g_max``, so EVERY
  element equal to the maximum gets the full gradient (torch.amax splits it between ties), and 0 * NaN stays NaN,
* ``.reshape()``, ``theano.shared``, ``>`` giving int8 like Theano (torch cannot subtract a bool tensor), integer
  ``T.sum`` (int64, as Theano sums int8),
* Theano's upcast of float32 with int32/int64 operands to float64 (the division by the integer class counts).

Theano itself is absent here; its gradient rules above are restated from Theano 0.8.2's source, so the NaN /
tie behaviour is not pinned against a Theano run.
"""
import ast
import os
import types

import numpy as np
import torch

from . import ref_layers, theano_shim

WANTED = ("SeedLossLayer", "ExpandLossLayer")
_NS = None


def _promote(x, y):
    """Theano's upcast: float32 with an int32/int64 tensor is float64 (torch keeps float32)."""
    if torch.is_tensor(x) and torch.is_tensor(y) and x.is_floating_point() != y.is_floating_point():
        f, i = (x, y) if x.is_floating_point() else (y, x)
        if f.dtype == torch.float32 and i.dtype in (torch.int32, torch.int64):
            f = f.double()
            return (f, i) if x.is_floating_point() else (i, f)
    return x, y


def _lift(x):
    return x if isinstance(x, theano_shim.Sym) else Sym(lambda env, v=x: v)


class Sym(theano_shim.Sym):
    """theano_shim.Sym with the methods and dtype rules of the SEC layers' graphs."""

    def __array_ufunc__(self, ufunc, method, *inputs, **kw):
        if method != "__call__":
            return NotImplemented
        table = {np.exp: exp, np.log: log, np.add: lambda a, b: _lift(a) + b, np.subtract: lambda a, b: _lift(a) - b,
                 np.multiply: lambda a, b: _lift(a) * b, np.true_divide: lambda a, b: _lift(a) / b,
                 np.negative: lambda a: -_lift(a)}
        if ufunc not in table:
            return NotImplemented
        return table[ufunc](*inputs)

    def _bin(self, other, op, swap=False):
        o = _lift(other)
        a, b = (o, self) if swap else (self, o)
        return Sym(lambda env: op(*_promote(a.ev(env), b.ev(env))))

    def __neg__(self):
        return Sym(lambda env: -self.ev(env))

    def __getitem__(self, idx):
        return Sym(lambda env: self.ev(env)[idx])

    def __gt__(self, o):
        return self._bin(o, lambda x, y: (x > y).to(torch.int8))

    def max(self, axis=None):
        return max(self, axis)

    def reshape(self, shape):
        return Sym(lambda env: self.ev(env).reshape(shape))


class Placeholder(Sym):
    def __init__(self):
        Sym.__init__(self, lambda env: env[id(self)])


def ftensor4():
    return Placeholder()


class _TieMax(torch.autograd.Function):
    """max over one axis whose backward is Theano's eq(xmax, x) * g_max."""

    @staticmethod
    def forward(ctx, x, dim):
        m = torch.amax(x, dim=dim)
        ctx.save_for_backward(x, m)
        ctx.dim = dim
        return m

    @staticmethod
    def backward(ctx, g):
        x, m = ctx.saved_tensors
        eq = (x == m.unsqueeze(ctx.dim)).to(g.dtype)
        return eq * g.unsqueeze(ctx.dim), None


def tie_max(x, dim):
    return _TieMax.apply(x, dim)


def max(x, axis=None):  # noqa: A001 (Theano's name)
    x = _lift(x)
    if axis is None:
        return Sym(lambda env: tie_max(x.ev(env).reshape(-1), 0))
    return Sym(lambda env: tie_max(x.ev(env), axis))


def sort(x, axis=-1):
    x = _lift(x)
    return Sym(lambda env: torch.sort(x.ev(env), dim=axis).values)


def sum(x, axis=None, keepdims=False):  # noqa: A001
    x = _lift(x)
    ax = theano_shim._axes(axis)
    return Sym(lambda env: torch.sum(x.ev(env)) if ax is None else torch.sum(x.ev(env), dim=ax, keepdim=keepdims))


def mean(x, axis=None, keepdims=False):
    x = _lift(x)
    ax = theano_shim._axes(axis)
    return Sym(lambda env: torch.mean(x.ev(env)) if ax is None else torch.mean(x.ev(env), dim=ax, keepdim=keepdims))


def log(x):
    x = _lift(x)
    return Sym(lambda env: torch.log(x.ev(env)))


def exp(x):
    x = _lift(x)
    return Sym(lambda env: torch.exp(x.ev(env)))


def addbroadcast(x, *axes):
    return x


def shared(value):
    t = torch.as_tensor(np.asarray(value))
    return Sym(lambda env: t)


def install():
    """(theano, T) stand-ins for the SEC layers' class bodies."""
    T = types.ModuleType("theano.tensor")
    for name in ("ftensor4", "sum", "mean", "max", "sort", "addbroadcast", "log", "exp"):
        setattr(T, name, globals()[name])
    T.grad = theano_shim.grad
    theano = types.ModuleType("theano")
    theano.function = theano_shim.function
    theano.shared = shared
    theano.tensor = T
    return theano, T


def available():
    return ref_layers.available()


def namespace():
    """The reference's SeedLossLayer and ExpandLossLayer, defined by executing their own source in place."""
    global _NS
    if _NS is None:
        with open(ref_layers.REF_FILE) as fh:
            tree = ast.parse(fh.read())
        keep = [n for n in tree.body
                if (isinstance(n, ast.ClassDef) and n.name in WANTED) or
                (isinstance(n, ast.Assign) and all(isinstance(t, ast.Name) for t in n.targets))]
        theano, T = install()
        caffe = types.ModuleType("caffe")
        caffe.Layer = type("Layer", (object,), {"param_str": ""})
        ns = {"np": np, "caffe": caffe, "theano": theano, "T": T, "osp": os.path}
        exec(compile(ast.Module(body=keep, type_ignores=[]), ref_layers.REF_FILE, "exec"), ns)
        _NS = ns
    return _NS


def _run(name, bottoms, dtype):
    """setup -> reshape -> forward -> backward of the reference layer `name`; returns (loss, d bottom[0])."""
    theano_shim.set_dtype(torch.float64 if dtype == "float64" else torch.float32)
    try:
        layer = namespace()[name]()
        np_dt = np.float64 if dtype == "float64" else np.float32
        bottom = [ref_layers.Blob(b) for b in bottoms]
        for bl, b in zip(bottom, bottoms):   # float64: keep the inputs exact
            bl.data = np.array(b, np_dt)
            bl.diff = np.zeros_like(bl.data)
        top = [ref_layers.Blob()]
        layer.setup(bottom, top)
        layer.reshape(bottom, top)
        top[0].data = top[0].data.astype(np_dt)
        top[0].diff = top[0].diff.astype(np_dt)
        layer.forward(bottom, top)
        layer.backward(top, [True, False], bottom)
        return np.array(top[0].data).reshape(-1)[0], np.array(bottom[0].diff)
    finally:
        theano_shim.set_dtype(torch.float32)


def seed_loss_layer(probs, labels, dtype="float64"):
    """(loss, d probs): pylayers.py:95-118."""
    return _run("SeedLossLayer", [probs, labels], dtype)


def expand_loss_layer(probs, labels, dtype="float64"):
    """(loss, d probs): pylayers.py:183-233 (probs (N, 21, 41, 41), labels (N, 1, 1, 21))."""
    return _run("ExpandLossLayer", [probs, labels], dtype)
