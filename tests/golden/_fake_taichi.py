"""A serial float32 / int32 stand-in for the part of `taichi` that PG/particle_filling/filling.py uses, so that its kernels
(densify_grids, fill_dense_grids, collision_search, collision_times, internal_filling, fill_particles) can be exec'd as they
are written. Used by make_filling_golden.py only.

Arithmetic follows Taichi's default precision: every float is float32 (Python float literals and `float` kernel arguments
are rounded to float32 first), every int int32, and vector / matrix products are summed left to right in float32, one
rounding per operation. What a serial interpreter cannot do by itself:
  * `ti.atomic_add(x, v)` must update its first argument; `rewrite_atomics` turns `ti.atomic_add(x, v)` statements into
    `x += v` and `t = ti.atomic_add(x, v)` into `t = x; x += v` while the source is still an `ast` (this also covers the
    kernel-scope scalar `new_start_idx`);
  * `ti.sym_eig` is numpy's float64 `eigh` of the float32 matrix, rounded to float32 (eigenvalues ascending, with sign);
  * `ti.random` draws float32 in [0, 1) from a seeded numpy generator (`seed`).
Struct-for over a field iterates its cells in C order.
"""
import ast

import numpy as np
import torch

F32, I32 = np.float32, np.int32


def _scalar(x):
    if isinstance(x, (bool, np.bool_)):
        return x
    if isinstance(x, (float, np.floating)):
        return F32(x)
    if isinstance(x, (int, np.integer)):
        return int(x)
    return x


def _bin(a, b, op):
    """Scalar op in Taichi's promotion: int op int -> int, anything with a float -> float32."""
    a, b = _scalar(a), _scalar(b)
    if isinstance(a, F32) or isinstance(b, F32):
        return F32(op(F32(a), F32(b)))
    return op(a, b)


class Vector:
    """ti.Vector value: a short list of float32 or int scalars."""

    def __init__(self, vals):
        self.v = [_scalar(x) for x in vals]

    def __len__(self):
        return len(self.v)

    def __iter__(self):
        return iter(self.v)

    def __getitem__(self, i):
        return self.v[i]

    def __setitem__(self, i, x):
        self.v[i] = F32(x) if isinstance(self.v[i], F32) else _scalar(x)

    def _ew(self, o, op):
        if isinstance(o, Vector):
            return Vector([_bin(a, b, op) for a, b in zip(self.v, o.v)])
        return Vector([_bin(a, o, op) for a in self.v])

    def __add__(self, o):
        return self._ew(o, lambda a, b: a + b)

    def __sub__(self, o):
        return self._ew(o, lambda a, b: a - b)

    def __mul__(self, o):
        return self._ew(o, lambda a, b: a * b)

    __rmul__ = __mul__

    def dot(self, o):
        s = _bin(self.v[0], o.v[0], lambda a, b: a * b)
        for a, b in zip(self.v[1:], o.v[1:]):
            s = _bin(s, _bin(a, b, lambda x, y: x * y), lambda x, y: x + y)
        return s

    def idx(self):
        return tuple(int(x) for x in self.v)


class Matrix:
    """ti.Matrix value: rows of float32 scalars."""

    def __init__(self, rows):
        self.m = [[F32(x) for x in r] for r in rows]

    def transpose(self):
        return Matrix([[self.m[j][i] for j in range(3)] for i in range(3)])

    def __matmul__(self, o):
        if isinstance(o, Vector):
            return Vector([Vector(r).dot(o) for r in self.m])
        cols = [Vector([o.m[k][j] for k in range(3)]) for j in range(3)]
        return Matrix([[Vector(r).dot(c) for c in cols] for r in self.m])


class Field:
    def __init__(self, dtype, shape, n=None):
        shp = (shape,) if np.isscalar(shape) else tuple(shape)
        self.a = np.zeros(shp + ((n,) if n else ()), F32 if dtype is float else I32)
        self.shape, self.n = shp, n

    def _key(self, idx):
        if isinstance(idx, Vector):
            idx = idx.idx()
        if isinstance(idx, tuple):
            idx = tuple(int(i) for i in idx)
            assert all(0 <= i < s for i, s in zip(idx, self.shape)), ("out-of-range field access", idx, self.shape)
        else:
            idx = int(idx)
            assert 0 <= idx < self.shape[0], ("out-of-range field access", idx, self.shape)
        return idx

    def __getitem__(self, idx):
        x = self.a[self._key(idx)]
        return Vector(list(x)) if self.n else _scalar(x)

    def __setitem__(self, idx, v):
        self.a[self._key(idx)] = list(v) if isinstance(v, Vector) else v

    def __iter__(self):                      # struct-for over the field's cells, C order
        return iter(np.ndindex(*self.shape))

    def from_torch(self, t):
        self.a[...] = t.detach().cpu().numpy().reshape(self.a.shape)

    def to_torch(self):
        return torch.from_numpy(self.a.copy())

    def to_numpy(self):
        return self.a.copy()


def _sym_eig(A):
    w, V = np.linalg.eigh(np.array(A.m, np.float64))
    return Vector([F32(x) for x in w]), Matrix(V.astype(F32))


class _VectorNS:
    def __call__(self, vals):
        return Vector(vals)

    @staticmethod
    def field(n, dtype, shape):
        return Field(dtype, shape, n)


def make_ti(seed):
    """A fresh `ti` namespace whose ti.random() stream starts at `seed`."""
    rng = np.random.default_rng(seed)
    ns = type("ti", (), {})()
    ns.kernel = lambda fn: (lambda *a, **kw: fn(*[_scalar(x) for x in a], **{k: _scalar(v) for k, v in kw.items()}))
    ns.func = lambda fn: fn
    ns.template = lambda: None
    ns.static = lambda x: x
    ns.field = lambda dtype, shape: Field(dtype, shape)
    ns.Vector = _VectorNS()
    ns.Matrix = Matrix
    ns.floor = lambda x, dtype=int: int(np.floor(F32(x)))
    ns.ceil = lambda x, dtype=int: int(np.ceil(F32(x)))
    ns.sqrt = lambda x: F32(np.sqrt(F32(x)))
    ns.exp = lambda x: F32(np.exp(F32(x)))
    ns.max = lambda *a: F32(max(F32(x) for x in a)) if any(isinstance(_scalar(x), F32) for x in a) else max(a)
    ns.min = lambda *a: F32(min(F32(x) for x in a)) if any(isinstance(_scalar(x), F32) for x in a) else min(a)
    ns.sym_eig = _sym_eig
    ns.random = lambda: F32(rng.random(dtype=np.float32))
    ns.math = type("math", (), {"mod": staticmethod(lambda a, b: a % b)})()

    def atomic_add(*a):
        raise AssertionError("ti.atomic_add must be rewritten by rewrite_atomics before exec")
    ns.atomic_add = atomic_add
    return ns


class _Atomics(ast.NodeTransformer):
    @staticmethod
    def _is_atomic(node):
        return (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "atomic_add"
                and isinstance(node.func.value, ast.Name) and node.func.value.id == "ti")

    def _aug(self, call):
        return ast.AugAssign(target=_store(call.args[0]), op=ast.Add(), value=call.args[1])

    def visit_Expr(self, node):
        if self._is_atomic(node.value):
            return ast.copy_location(self._aug(node.value), node)
        return node

    def visit_Assign(self, node):
        if self._is_atomic(node.value):
            call = node.value
            keep = ast.Assign(targets=node.targets, value=call.args[0])
            return [ast.copy_location(keep, node), ast.copy_location(self._aug(call), node)]
        return node


def _store(expr):
    e = ast.parse(ast.unparse(expr), mode="eval").body
    e.ctx = ast.Store()
    return e


def rewrite_atomics(tree):
    """`ti.atomic_add(x, v)` -> `x += v`; `t = ti.atomic_add(x, v)` -> `t = x; x += v` (serial execution)."""
    return ast.fix_missing_locations(_Atomics().visit(tree))
