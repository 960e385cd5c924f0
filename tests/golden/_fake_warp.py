"""Minimal stand-in for `warp-lang==0.10.1` (GOLDEN-VECTOR TOOLING, not product code).

The reference's MPM arithmetic is written as `@wp.kernel` / `@wp.func` Python functions
(third_party/PhysGaussian/mpm_solver_warp/mpm_utils.py, and the BC closures of
mpm_solver_warp.py:749-1179).  Warp itself is not installed and cannot be (no network), but those
functions are plain Python syntax: with this module registered as `warp`, the REFERENCE'S OWN SOURCE is
imported and executed statement by statement on the CPU, one "thread" after another, in float32.
`tests/golden/make_mpm_golden.py` uses that to write the fixtures that pin oracle/mpm_ref.c and the CUDA path.

What is emulated (Warp 0.10 semantics the reference relies on):
  * vec2/vec3/mat33 value types in float32; `mat33(v0, v1, v2)` builds the matrix from COLUMN vectors;
    `mat33(9 scalars)` is row-major; `*` is matrix product for mat*mat and mat*vec, scaling otherwise;
  * `wp.array` (1-D and 3-D; float / int / vec3 / mat33 element types) that reads and writes by value;
  * `wp.launch` as a serial loop over `wp.tid()`; `wp.atomic_add` as a plain += (serial, so deterministic);
  * scalar kernel arguments annotated `float` are rounded to float32 at launch (so the host's double-precision
    clock is compared as float32, as in the Warp kernels); struct fields annotated `float` likewise;
  * `wp.int` truncates toward zero; float literals act as float32 (numpy NEP-50 weak scalars);
  * `wp.svd3`: numpy float64 SVD, then the output convention of Warp's native svd3 (McAdams et al.):
    U, V proper rotations, |sigma| descending, a negative determinant carried by the LAST singular value.
    Every use in the reference has the form U f(Sigma) V^T, which is invariant under the remaining freedom.
  * struct / kernel decorators, ScopedTimer, torch interop (`from_torch`, `to_torch`, `warp.types.array(ptr=...)`
    aliasing CPU tensor memory, as warp_utils.torch2warp_* does on the GPU).
"""
from __future__ import annotations

import ctypes
import math
import sys
import types as _pytypes

import builtins as _b

import numpy as np

f32 = np.float32
_F, _I = _b.float, _b.int  # the module defines wp.float / wp.int further down


def _s(x):
    """Scalar -> float32."""
    return f32(x)


# --------------------------------------------------------------------------------------------- value types
class _Vec:
    N = 3
    __slots__ = ("a",)
    __array_ufunc__ = None      # numpy scalars must defer to __rmul__ / __radd__ instead of broadcasting

    def __init__(self, *args):
        n = self.N
        if len(args) == 0:
            self.a = np.zeros(n, f32)
        elif len(args) == 1:
            x = args[0]
            if isinstance(x, _Vec):
                self.a = x.a.copy()
            elif isinstance(x, (list, tuple, np.ndarray)):
                self.a = np.asarray(x, dtype=f32).reshape(n).copy()
            else:
                self.a = np.full(n, f32(x), f32)
        else:
            assert len(args) == n, args
            self.a = np.array([f32(v) for v in args], f32)

    def __getitem__(self, i):
        # inside a kernel a component is a float32 value; at Python scope Warp hands back a Python float
        # (this matters for the host-side `modify` closure of set_velocity_on_cuboid, which advances the box in
        # double precision and rounds to float32 when the vec3 is rebuilt, mpm_solver_warp.py:899-905)
        return self.a[i] if _tid is not None else _F(self.a[i])

    def __setitem__(self, i, v):
        self.a[i] = f32(v)

    def __iter__(self):
        return iter(self.a)

    def __len__(self):
        return self.N

    def _wrap(self, arr):
        o = type(self).__new__(type(self))
        o.a = arr.astype(f32, copy=False)
        return o

    def __add__(self, o):
        return self._wrap(self.a + o.a)

    def __sub__(self, o):
        return self._wrap(self.a - o.a)

    def __neg__(self):
        return self._wrap(-self.a)

    def __mul__(self, s):
        assert not isinstance(s, (_Vec, mat33)), "vec*vec is not defined in Warp; use cw_mul/dot"
        return self._wrap(self.a * f32(s))

    __rmul__ = __mul__

    def __truediv__(self, s):
        return self._wrap(self.a / f32(s))

    def __repr__(self):
        return f"{type(self).__name__}{tuple(self.a.tolist())}"


class vec3(_Vec):
    N = 3
    __slots__ = ()


class vec2(_Vec):
    N = 2
    __slots__ = ()


class quat(_Vec):
    N = 4
    __slots__ = ()


class mat33:
    __slots__ = ("a",)
    __array_ufunc__ = None

    def __init__(self, *args):
        if len(args) == 0:
            self.a = np.zeros((3, 3), f32)
        elif len(args) == 1:
            x = args[0]
            if isinstance(x, mat33):
                self.a = x.a.copy()
            elif isinstance(x, np.ndarray):
                self.a = x.astype(f32).reshape(3, 3).copy()
            else:
                self.a = np.full((3, 3), f32(x), f32)
        elif len(args) == 3:  # column vectors (Warp 0.10)
            self.a = np.stack([vec3(c).a for c in args], axis=1).astype(f32)
        else:
            assert len(args) == 9, args
            self.a = np.array([f32(v) for v in args], f32).reshape(3, 3)

    @staticmethod
    def _wrap(arr):
        o = mat33.__new__(mat33)
        o.a = arr.astype(f32, copy=False)
        return o

    def __getitem__(self, ij):
        if isinstance(ij, tuple):
            return self.a[ij[0], ij[1]]
        return vec3(self.a[ij])  # row

    def __setitem__(self, ij, v):
        self.a[ij[0], ij[1]] = f32(v)

    def __add__(self, o):
        return mat33._wrap(self.a + o.a)

    def __sub__(self, o):
        return mat33._wrap(self.a - o.a)

    def __neg__(self):
        return mat33._wrap(-self.a)

    def __mul__(self, o):
        if isinstance(o, mat33):
            return mat33._wrap(_matmul(self.a, o.a))
        if isinstance(o, vec3):
            return vec3._wrap(vec3(), _matvec(self.a, o.a))
        return mat33._wrap(self.a * f32(o))

    def __rmul__(self, s):
        return mat33._wrap(self.a * f32(s))

    def __truediv__(self, s):
        return mat33._wrap(self.a / f32(s))

    def __repr__(self):
        return f"mat33({self.a.tolist()})"


def _matmul(a, b):
    # float32 products summed in k order, rounding after every operation (no fused multiply-add)
    out = np.zeros((3, 3), f32)
    for k in range(3):
        out = (out + np.outer(a[:, k], b[k, :]).astype(f32)).astype(f32)
    return out


def _matvec(a, v):
    out = np.zeros(3, f32)
    for k in range(3):
        out = (out + a[:, k] * v[k]).astype(f32)
    return out


float32 = f32
int32 = np.int32


# --------------------------------------------------------------------------------------------------- arrays
def _elem_shape(dtype):
    if dtype is vec3:
        return (3,), f32
    if dtype is vec2:
        return (2,), f32
    if dtype is quat:
        return (4,), f32
    if dtype is mat33:
        return (3, 3), f32
    if dtype in (_F, f32):
        return (), f32
    if dtype in (_I, np.int32):
        return (), np.int32
    raise TypeError(f"fake warp: unsupported array dtype {dtype}")


class array:
    """Doubles as the annotation object (`wp.array(dtype=float)`) and as the storage class."""

    def __init__(self, data=None, dtype=_F, ndim=1, shape=None, ptr=None, copy=False, owner=False,
                 requires_grad=False, device=None, length=None):
        self.dtype = dtype
        self.ndim = ndim
        self.data = None
        self.tensor = None
        es, nt = _elem_shape(dtype)
        if ptr is not None:  # alias foreign (torch CPU) memory, like warp_utils.torch2warp_*
            shp = (shape,) if np.isscalar(shape) else tuple(shape)
            count = _I(np.prod(shp + es))
            ctype = ctypes.c_float if nt is f32 else ctypes.c_int32
            buf = (ctype * count).from_address(ptr)
            self.data = np.ctypeslib.as_array(buf).reshape(shp + es)
            self.ndim = len(shp)
        elif data is not None:
            self.data = data
            self.ndim = data.ndim - len(es)

    @property
    def shape(self):
        es, _ = _elem_shape(self.dtype)
        return self.data.shape[: self.data.ndim - len(es)]

    def numpy(self):
        return self.data

    def _idx(self, i):
        return i if isinstance(i, tuple) else (i,)

    def __getitem__(self, i):
        v = self.data[self._idx(i)]
        if self.dtype is vec3:
            return vec3._wrap(vec3(), v.copy())
        if self.dtype is mat33:
            return mat33._wrap(v.copy())
        if self.dtype is vec2:
            return vec2._wrap(vec2(), v.copy())
        return v  # numpy scalar (float32 / int32)

    def __setitem__(self, i, v):
        if isinstance(v, (_Vec, mat33)):
            self.data[self._idx(i)] = v.a
        else:
            self.data[self._idx(i)] = v


def _alloc(shape, dtype, fill=0):
    shp = (shape,) if np.isscalar(shape) else tuple(shape)
    es, nt = _elem_shape(dtype)
    return array(data=np.full(shp + es, fill, nt), dtype=dtype)


def zeros(shape=None, dtype=_F, device=None, **kw):
    return _alloc(shape, dtype, 0)


def empty(shape=None, dtype=_F, device=None, **kw):
    return _alloc(shape, dtype, 0)


def from_numpy(arr, dtype=_F, device=None, **kw):
    es, nt = _elem_shape(dtype)
    a = np.ascontiguousarray(np.asarray(arr), dtype=nt)
    if es and a.shape[-len(es):] != es:
        a = a.reshape((-1,) + es)
    return array(data=a.copy(), dtype=dtype)


def from_torch(t, dtype=None, **kw):
    import torch
    a = t.detach().cpu().numpy() if t.device.type != "cpu" else t.detach().numpy()
    if dtype is None:
        dtype = _F if t.dtype == torch.float32 else _I
    out = array(data=a, dtype=dtype)
    out.tensor = t
    return out


def to_torch(a):
    import torch
    return torch.from_numpy(a.data)


# ------------------------------------------------------------------------------------------- struct / kernel
def _default_for(ann):
    if isinstance(ann, array):
        return None
    if ann is _F:
        return f32(0.0)
    if ann is _I:
        return 0
    if ann in (vec3, vec2, mat33):
        return ann()
    return None


def struct(cls):
    ann = dict(getattr(cls, "__annotations__", {}))

    def __init__(self):
        object.__setattr__(self, "_ann", ann)
        for k, t in ann.items():
            object.__setattr__(self, k, _default_for(t))

    def __setattr__(self, k, v):
        t = self._ann.get(k)
        if t is _F and not isinstance(v, (_Vec, mat33, array)):
            v = f32(v)
        elif t is _I and isinstance(v, (bool, _I, np.integer, _F)):
            v = _I(v)
        object.__setattr__(self, k, v)

    cls.__init__ = __init__
    cls.__setattr__ = __setattr__
    return cls


_tid = None


def tid():
    return _tid


class _Kernel:
    def __init__(self, fn):
        self.fn = fn
        self.ann = [fn.__annotations__.get(n) for n in fn.__code__.co_varnames[: fn.__code__.co_argcount]]
        self.__name__ = fn.__name__

    def __call__(self, *a):
        return self.fn(*a)


def kernel(fn):
    return _Kernel(fn)


def func(fn):
    return fn


def launch(kernel=None, dim=None, inputs=(), device=None, **kw):
    global _tid
    args = []
    for t, v in zip(kernel.ann, inputs):
        if t is _F and not isinstance(v, (_Vec, mat33, array)):
            v = f32(v)
        elif t is _I and isinstance(v, (bool, _I, np.integer)):
            v = _I(v)
        args.append(v)
    if np.isscalar(dim):
        for i in range(_I(dim)):
            _tid = i
            kernel.fn(*args)
    else:
        dims = tuple(_I(d) for d in dim)
        for idx in np.ndindex(*dims):
            _tid = idx if len(dims) > 1 else idx[0]
            kernel.fn(*args)
    _tid = None


class ScopedTimer:
    def __init__(self, *a, **kw):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def synchronize():
    pass


def init():
    pass


# ------------------------------------------------------------------------------------------------- builtins
def atomic_add(arr, *args):
    *idx, v = args
    idx = tuple(idx)
    if isinstance(v, (_Vec, mat33)):
        arr.data[idx] = (arr.data[idx] + v.a).astype(f32)
    else:
        arr.data[idx] = f32(arr.data[idx] + f32(v))


def transpose(m):
    return mat33._wrap(m.a.T.copy())


def determinant(m):
    a = m.a
    return f32(
        a[0, 0] * f32(a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1])
        - a[0, 1] * f32(a[1, 0] * a[2, 2] - a[1, 2] * a[2, 0])
        + a[0, 2] * f32(a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0])
    )


def svd3(A, U, sig, V):
    u, s, vt = np.linalg.svd(A.a.astype(np.float64))
    v = vt.T
    if np.linalg.det(u) < 0:
        u[:, 2] = -u[:, 2]
        s[2] = -s[2]
    if np.linalg.det(v) < 0:
        v[:, 2] = -v[:, 2]
        s[2] = -s[2]
    U.a[...] = u.astype(f32)
    V.a[...] = v.astype(f32)
    sig.a[...] = s.astype(f32)


def cw_mul(a, b):
    return a._wrap(a.a * b.a)


def dot(a, b):
    acc = f32(0.0)
    for k in range(len(a.a)):
        acc = f32(acc + a.a[k] * b.a[k])
    return acc


def length(a):
    return f32(np.sqrt(dot(a, a)))


def normalize(a):
    return a / length(a)


def cross(a, b):
    return vec3._wrap(vec3(), np.cross(a.a, b.a))


def outer(a, b):
    return mat33._wrap(np.outer(a.a, b.a))


def diag(v):
    return mat33._wrap(np.diag(v.a))


def add(a, b):
    return a + b


def sub(a, b):
    return a - b


def _un(npf):
    def g(x):
        return f32(npf(f32(x)))
    return g


log, exp, sqrt, sin, cos, acos = (_un(np.log), _un(np.exp), _un(np.sqrt), _un(np.sin), _un(np.cos), _un(np.arccos))


def abs(x):  # noqa: A001
    return f32(np.abs(f32(x)))


def pow(x, y):  # noqa: A001
    return f32(np.power(f32(x), f32(y)))


def max(a, b):  # noqa: A001
    a, b = f32(a), f32(b)
    return a if a > b else b


def min(a, b):  # noqa: A001
    a, b = f32(a), f32(b)
    return a if a < b else b


def int(x):  # noqa: A001   (wp.int: truncation toward zero)
    return _I(x)   # Python int() of a float truncates toward zero


def float(x=0.0):  # noqa: A001
    return f32(x)


# `wp.int` / `wp.float` shadow the builtins inside this module only; annotations in the reference use the
# Python builtins `float` / `int`, which is what `struct` / `launch` compare against.


def install():
    """Register this module as `warp` (+ `warp.torch`, `warp.types`) in sys.modules."""
    me = sys.modules[__name__]
    sys.modules["warp"] = me
    t = _pytypes.ModuleType("warp.torch")
    t.from_torch, t.to_torch = from_torch, to_torch
    sys.modules["warp.torch"] = t
    ty = _pytypes.ModuleType("warp.types")
    ty.array, ty.float32, ty.int32 = array, f32, np.int32
    sys.modules["warp.types"] = ty
    me.torch = t
    me.types = ty
    return me


