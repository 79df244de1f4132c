"""Rank-local dense operators: the role third-party ``pylops`` operators play
inside MPIBlockDiag / MPIVStack in the reference (BlockDiag.py:127-129,
VStack.py:129-131 call ``oper.matvec`` on a slice of the local array).

Any object with ``shape``, ``dtype``, ``matvec(x)``, ``rmatvec(x)`` acting on
1-D device tensors can be used; :class:`MatrixMult` is the dense block every
reference test / BASELINE config uses, applied by the b2_gemv kernels.
"""
from __future__ import annotations

import copy
import ctypes as C
import math

import numpy as np
import torch

from . import _lib

__all__ = ["MatrixMult", "LocalOperator", "apply_into"]

_REAL_OF = {torch.complex64: torch.float32, torch.complex128: torch.float64}
_CPLX_OF = {torch.float32: torch.complex64, torch.float64: torch.complex128}


def apply_into(oper, x: torch.Tensor, out: torch.Tensor, adjoint: bool) -> None:
    """``out[...] = oper(x)`` / ``oper^H(x)`` for a rank-local operator: a kernel operator of this package (or the
    ``.H`` of one) writes into ``out`` itself, any other operator through a temporary (cast to ``out``'s dtype)."""
    while isinstance(oper, _LocalAdjoint):
        oper, adjoint = oper.op, not adjoint
    fn = oper.rmatvec if adjoint else oper.matvec
    if isinstance(oper, _KernelOperator):
        fn(x, out=out)
    else:
        _store(out, fn(x))


def _store(out: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """out <- y with NumPy ``__setitem__`` casting, as the reference's ``y[a:b] = oper.matvec(...)``
    (BlockDiag.py:127-129): complex into real keeps the real part and warns"""
    if y.dtype.is_complex and not out.dtype.is_complex:
        import warnings
        warnings.warn("Casting complex values to real discards the imaginary part", np.exceptions.ComplexWarning,
                      stacklevel=3)
        y = y.real
    out.copy_(y.reshape(out.shape))
    return out


class LocalOperator:
    """minimal rank-local linear operator interface.  ``A.H`` is the adjoint; ``A @ B`` and ``A * B`` between local
    operators are the product (applied right to left), in which ``T.H @ X @ T`` with ``T`` a :class:`Transpose` and
    ``X`` an axis operator on ``T``'s output dims is folded into ``X`` along the matching axis of ``T``'s input"""
    shape = (0, 0)
    dtype = np.float64

    def matvec(self, x: torch.Tensor) -> torch.Tensor:
        return self._matvec(x)

    def rmatvec(self, x: torch.Tensor) -> torch.Tensor:
        return self._rmatvec(x)

    # pylops-style aliases (MPILinearOperator(Op=...) calls Op._matvec)
    def _matvec(self, x):
        raise NotImplementedError

    def _rmatvec(self, x):
        raise NotImplementedError

    @property
    def H(self) -> "LocalOperator":
        return _LocalAdjoint(self)

    def __matmul__(self, other):
        if not isinstance(other, LocalOperator):
            return NotImplemented
        return _product(self, other)

    __mul__ = __matmul__


class _LocalAdjoint(LocalOperator):
    """``A.H`` of a rank-local operator: its matvec is ``A.rmatvec`` and the reverse"""

    def __init__(self, op: LocalOperator):
        self.op = op
        self.shape = (op.shape[1], op.shape[0])
        self.dtype = op.dtype

    @property
    def H(self) -> LocalOperator:
        return self.op

    def _matvec(self, x):
        return self.op.rmatvec(x)

    def _rmatvec(self, x):
        return self.op.matvec(x)


class _LocalProduct(LocalOperator):
    """``ops[0] @ ops[1] @ ... @ ops[-1]`` applied right to left, one operator at a time (eager)"""

    def __init__(self, ops):
        for a, b in zip(ops[:-1], ops[1:]):
            if a.shape[1] != b.shape[0]:
                raise ValueError(f"dimension mismatch in product: {a.shape} @ {b.shape}")
        self.ops = list(ops)
        self.shape = (ops[0].shape[0], ops[-1].shape[1])
        self.dtype = np.result_type(*[op.dtype for op in ops])

    @property
    def H(self) -> LocalOperator:
        return _product(*[op.H for op in reversed(self.ops)])

    def _matvec(self, x):
        for op in reversed(self.ops):
            x = op.matvec(x)
        return x

    def _rmatvec(self, x):
        for op in self.ops:
            x = op.rmatvec(x)
        return x


def _fold(t_inv, op, t) -> "LocalOperator | None":
    """``T.H @ X @ T`` as one operator: ``X`` along axis ``T.axes[X.axis]`` of ``T.dims`` (no transposes), when
    ``t`` is a Transpose, ``t_inv`` its inverse and ``op`` an axis operator on ``t``'s output dims; else None"""
    if not (isinstance(t, Transpose) and isinstance(t_inv, Transpose) and isinstance(op, _AxisOperator)):
        return None
    if t_inv.dims != t.dimsd or t_inv.axes != tuple(int(a) for a in np.argsort(t.axes)) or op.dims != t.dimsd:
        return None
    return op._along(t.dims, t.axes[op.axis])


def _product(*ops) -> LocalOperator:
    """product of rank-local operators, flattened, with every ``T.H @ X @ T`` folded"""
    flat = []
    for op in ops:
        flat.extend(op.ops if isinstance(op, _LocalProduct) else [op])
    i = 0
    while i + 2 < len(flat):
        f = _fold(*flat[i:i + 3])
        if f is None:
            i += 1
        else:
            flat[i:i + 3] = [f]
            i = max(i - 2, 0)
    return flat[0] if len(flat) == 1 else _LocalProduct(flat)


class _KernelOperator(LocalOperator):
    """A rank-local operator applied by this package's kernels.  Each apply is a fixed sequence of launches with no
    per-call host state (so ``CGLS.run`` may replay it in a CUDA graph), and ``matvec`` / ``rmatvec`` take ``out=``:
    ``x`` or ``out`` of the wrong length raises ``ValueError``; the result is written into ``out`` directly when it
    is contiguous, has the compute dtype and is not ``x``, else through a temporary with NumPy's assignment casting.
    A subclass provides ``_launch`` and, when its dtype rule is not "compute in the operator's dtype",
    ``_compute_dtype``."""

    def _compute_dtype(self, xdt: torch.dtype) -> torch.dtype:
        """the dtype data of dtype ``xdt`` are applied in; a real dtype for complex data means that the real and
        imaginary parts are applied one after the other"""
        return self._tdtype

    def _launch(self, x: torch.Tensor, y: torch.Tensor, dt: torch.dtype, adjoint: int) -> None:
        """``y = A x`` (adjoint 0) or ``y = A^H x`` (adjoint 1) on contiguous ``x``, ``y`` of the compute dtype ``dt``"""
        raise NotImplementedError

    def _apply(self, x: torch.Tensor, adjoint: int, out=None) -> torch.Tensor:
        x = x.reshape(-1)
        nout, nin = self.shape[::-1] if adjoint else self.shape
        if x.numel() != nin:
            raise ValueError(f"dimension mismatch: operator {self.shape}, vector {x.numel()}")
        if out is not None and out.numel() != nout:
            raise ValueError(f"dimension mismatch: operator {self.shape}, out {out.numel()}")
        dt = self._compute_dtype(x.dtype)
        if x.dtype.is_complex and not dt.is_complex:
            # real operator, complex data: result_type(op, x) is complex (the reference's NumPy promotion) --
            # apply to the real and imaginary parts instead of dropping the imaginary one
            rdt = torch.promote_types(dt, _REAL_OF[x.dtype])
            y = torch.complex(self._apply(x.real.contiguous(), adjoint).to(rdt),
                              self._apply(x.imag.contiguous(), adjoint).to(rdt))
            return y if out is None else _store(out, y)
        if x.dtype != dt:
            x = x.to(dt)
        if not x.is_contiguous():
            x = x.contiguous()
        direct = out is not None and out.dtype == dt and out.is_contiguous() and out.data_ptr() != x.data_ptr()
        y = out if direct else torch.empty(nout, dtype=dt, device=x.device)
        self._launch(x, y, dt, adjoint)
        if out is not None and not direct:       # caller's buffer has another dtype (e.g. mixed-dtype BlockDiag)
            return _store(out, y)
        return y

    def matvec(self, x, out=None):
        return self._apply(x, 0, out)

    def rmatvec(self, x, out=None):
        return self._apply(x, 1, out)

    _matvec, _rmatvec = matvec, rmatvec


class _RealTapsOperator(_KernelOperator):
    """A kernel operator with real taps: complex data are applied in one launch, their (re, im) pairs as the innermost
    dimension, in the complex dtype of the operator's and the data's real dtypes promoted"""

    def _compute_dtype(self, xdt):
        if xdt.is_complex and not self._tdtype.is_complex:
            return _CPLX_OF[torch.promote_types(self._tdtype, _REAL_OF[xdt])]
        return self._tdtype


class _AxisOperator(_RealTapsOperator):
    """A square operator applied line by line along ``axis`` of a C-ordered ``dims`` block"""

    def __init__(self, dims, axis: int, dtype):
        self.dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        self.axis = axis % len(self.dims)
        n = int(np.prod(self.dims))
        self.shape = (n, n)
        self._tdtype = _lib.torch_dtype(dtype)
        self.dtype = _lib.numpy_dtype(self._tdtype)
        _lib.ctx()

    def _along(self, dims, axis):
        """the same operator on a ``dims`` block along ``axis`` (``prod(dims)`` unchanged)"""
        new = copy.copy(self)
        new.dims = tuple(int(d) for d in dims)
        new.axis = int(axis) % len(new.dims)
        return new

    def _lines(self, dt):
        """``(n_outer, n_axis, n_inner, real dtype)`` of a launch on data of dtype ``dt``"""
        n_inner = math.prod(self.dims[self.axis + 1:]) * (2 if dt.is_complex else 1)
        return math.prod(self.dims[:self.axis]), self.dims[self.axis], n_inner, _REAL_OF.get(dt, dt)


class MatrixMult(_KernelOperator):
    """Dense block ``y = A x`` / ``y = A^H x`` (pylops.MatrixMult for a single
    right-hand side).  ``A`` may be a NumPy array (uploaded once) or a device
    tensor; dtype float32/float64/complex64/complex128, or bfloat16 with
    float32 vectors.  HBM-bound GEMV kernels (csrc/gemv.cu)."""

    def __init__(self, A, dtype=None):
        if not isinstance(A, torch.Tensor):
            A = torch.as_tensor(np.asarray(A))
        if dtype is not None:
            A = A.to(_lib.torch_dtype(dtype))
        if A.dim() != 2:
            raise ValueError("MatrixMult expects a 2-D array")
        _lib.ctx()
        self.A = A.to("cuda").contiguous()
        self.shape = (int(A.shape[0]), int(A.shape[1]))
        self._tdtype = torch.float32 if self.A.dtype is torch.bfloat16 else self.A.dtype
        self.dtype = _lib.numpy_dtype(self._tdtype)

    def _launch(self, x, y, dt, adjoint):
        m, n = self.shape
        _lib.check(_lib.lib.b2_gemv(_lib.ctx(), self.A.data_ptr(), n, m, n, x.data_ptr(), y.data_ptr(),
                                    _lib.OP_H if adjoint else _lib.OP_N, _lib.code(self.A.dtype), _lib.code(dt),
                                    _lib.stream()), "b2_gemv")


class _AxisDerivative(_AxisOperator):
    """Rank-local derivative along one axis of a C-ordered ``dims`` block (the role of
    pylops.FirstDerivative / pylops.SecondDerivative inside MPIBlockDiag in MPILaplacian / MPIGradient,
    Laplacian.py:97-126, Gradient.py:101-119).  One batched stencil launch (b2_derivative_axis)."""
    _deriv = 1

    def __init__(self, dims, axis: int = 0, sampling: float = 1.0, kind: str = "centered", edge: bool = False,
                 order: int = 3, dtype=np.float64):
        super().__init__(dims, axis, dtype)
        self.sampling, self.edge, self.order = float(sampling), bool(edge), int(order)
        kinds = {"forward": _lib.FD_FORWARD, "backward": _lib.FD_BACKWARD, "centered": _lib.FD_CENTERED}
        if kind not in kinds:
            raise NotImplementedError("'kind' must be 'forward', 'centered', or 'backward'")
        if self._deriv == 1 and kind == "centered" and order not in (3, 5):
            raise NotImplementedError("'order' must be '3, or '5'")
        self._kind = kinds[kind]

    def _launch(self, x, y, dt, adjoint):
        n_outer, n_axis, n_inner, real = self._lines(dt)
        _lib.check(_lib.lib.b2_derivative_axis(_lib.ctx(), x.data_ptr(), y.data_ptr(), n_outer, n_axis, n_inner,
                                               self._deriv, self._kind, self.order, int(self.edge), self.sampling,
                                               adjoint, _lib.code(real), _lib.stream()), "b2_derivative_axis")


class FirstDerivative(_AxisDerivative):
    _deriv = 1


class SecondDerivative(_AxisDerivative):
    _deriv = 2

    def __init__(self, dims, axis: int = 0, sampling: float = 1.0, kind: str = "centered", edge: bool = False,
                 dtype=np.float64):
        super().__init__(dims, axis=axis, sampling=sampling, kind=kind, edge=edge, order=3, dtype=dtype)


def _real_filters(h):
    """``(host array, {real dtype: device copy})`` of real taps or of a bank of real filters, given as a NumPy array
    or a torch tensor of any real dtype: uploaded once, in both real precisions"""
    h = h.detach().cpu().numpy() if isinstance(h, torch.Tensor) else np.asarray(h)
    if np.iscomplexobj(h):
        raise NotImplementedError("complex filters are not supported")
    return h, {t: torch.as_tensor(np.ascontiguousarray(h, dtype=_lib.numpy_dtype(t))).to("cuda")
               for t in (torch.float32, torch.float64)}


class _StationaryTaps:
    """One real filter of ``nh`` taps on the device: ``y[i] = sum_k h[k] x[i + offset - k]`` along the axis of
    ``lines`` (an axis operator's ``_lines``), optionally fused with the first derivative ``kind`` (``C D``; adjoint
    ``D^T C^T``).  csrc/convolve.cu."""

    def __init__(self, bank, offset):
        if bank[torch.float64].dim() != 1:
            raise NotImplementedError("only stationary (1-D) filters are supported")
        self.nh, self.offset = bank[torch.float64].numel(), int(offset)
        if self.nh < 1 or not 0 <= self.offset <= self.nh - 1:
            raise ValueError(f"offset must be in [0, nh - 1] = [0, {self.nh - 1}], got {offset}")
        self._bank = bank

    def launch(self, x, y, lines, adjoint, kind=None):
        n_outer, n_axis, n_inner, real = lines
        head = (_lib.ctx(), x.data_ptr(), y.data_ptr(), n_outer, n_axis, n_inner, self._bank[real].data_ptr(),
                self.nh, self.offset)
        tail = (adjoint, _lib.code(real), _lib.stream())
        if kind is None:
            _lib.check(_lib.lib.b2_convolve_axis(*head, *tail), "b2_convolve_axis")
        else:
            _lib.check(_lib.lib.b2_poststack_axis(*head, kind, *tail), "b2_poststack_axis")


class _FilterBank:
    """``nfilt`` real filters of ``nh`` taps (centre ``hc``) at the axis samples ``oh, oh + dh, ...`` on the device:
    ``y[i] = sum_j h_j[hc + i - j] x[j]`` with ``h_j`` interpolated between the filters around sample ``j``,
    optionally fused with the first derivative ``kind``, as :class:`_StationaryTaps`.  csrc/nsconvolve.cu."""

    def __init__(self, bank, hc, oh, dh):
        self.nfilt, self.nh = (int(n) for n in bank[torch.float64].shape)
        self.hc, self.oh, self.dh = int(hc), int(oh), int(dh)
        self._bank = bank

    def launch(self, x, y, lines, adjoint, kind=None):
        n_outer, n_axis, n_inner, real = lines
        head = (_lib.ctx(), x.data_ptr(), y.data_ptr(), n_outer, n_axis, n_inner, self._bank[real].data_ptr(),
                self.nfilt, self.nh, self.hc, self.oh, self.dh)
        tail = (adjoint, _lib.code(real), _lib.stream())
        if kind is None:
            _lib.check(_lib.lib.b2_nsconvolve_axis(*head, *tail), "b2_nsconvolve_axis")
        else:
            _lib.check(_lib.lib.b2_nspoststack_axis(*head, kind, *tail), "b2_nspoststack_axis")


class Convolve1D(_AxisOperator):
    """Rank-local 1-D convolution along ``axis`` of a C-ordered ``dims`` block with a stationary real filter ``h``:
    the role of pylops.signalprocessing.Convolve1D inside MPIBlockDiag (tutorials/reflectivity.py:74-76).  For each
    line ``x`` of length ``n`` along ``axis``::

        y[i] = sum_k h[k] x[i + offset - k]  ==  np.convolve(x, h, "full")[offset:offset + n]

    and the adjoint is the exact transpose (the same kernel with ``h`` reversed and offset ``nh - 1 - offset``).
    One b2_convolve_axis launch per apply (csrc/convolve.cu).  ``method="fft"`` is accepted and computed by the
    direct kernel: it is the same linear map, equal within rounding."""

    def __init__(self, dims, h, offset: int = 0, axis: int = -1, method=None, dtype="float64"):
        if method not in (None, "direct", "fft"):
            raise ValueError("method must be None, 'direct' or 'fft'")
        self._conv = _StationaryTaps(_real_filters(h)[1], offset)
        super().__init__(dims, axis, dtype)
        self.nh, self.offset, self.method = self._conv.nh, self._conv.offset, method

    def _launch(self, x, y, dt, adjoint):
        self._conv.launch(x, y, self._lines(dt), adjoint)


class NonStationaryConvolve1D(_AxisOperator):
    """Rank-local non-stationary 1-D convolution along ``axis`` of a C-ordered ``dims`` block,
    pylops.signalprocessing.NonStationaryConvolve1D (pylops 2.x) inside MPIBlockDiag.  ``hs`` holds ``nfilt`` real
    filters of odd length ``nh`` at the regularly spaced axis samples ``ih``; sample ``j`` uses ``h_j``, linearly
    interpolated between the two filters around it (the first / last filter before ``ih[0]`` / after ``ih[-1]``)::

        y[i] = sum_j h_j[nh // 2 + i - j] x[j]

    and the adjoint is the exact transpose.  One b2_nsconvolve_axis launch per apply (csrc/nsconvolve.cu), whose
    interpolated filters are pylops' bits.  ``ValueError`` for an even ``nh``, irregular or decreasing ``ih``, ``ih``
    outside ``[0, dims[axis])`` and ``len(ih) != hs.shape[0]``; complex filters are not provided."""

    def __init__(self, dims, hs, ih, axis: int = -1, dtype="float64"):
        hs, bank = _real_filters(hs)
        if hs.ndim != 2:
            raise ValueError(f"hs must be a 2-D array of filters (nfilt, nh); got shape {hs.shape}")
        if hs.shape[1] % 2 == 0:
            raise ValueError("filters hs must have odd length")
        super().__init__(dims, axis, dtype)
        oh, dh = _regular_nodes("ih", ih, hs.shape[0], self.dims[self.axis])
        self._conv = c = _FilterBank(bank, hs.shape[1] // 2, oh, dh)
        self.nfilt, self.nh, self.hc, self.oh, self.dh = c.nfilt, c.nh, c.hc, c.oh, c.dh

    def _launch(self, x, y, dt, adjoint):
        self._conv.launch(x, y, self._lines(dt), adjoint)


def _regular_nodes(name, ih, nfilt, n):
    """``(origin, step)`` of the filter indices ``ih`` along an axis of ``n`` samples holding ``nfilt`` filters, with
    pylops' ``ValueError``s and ours (count, decreasing); one filter has step 1"""
    ih = np.asarray(ih).ravel()
    if len(ih) != nfilt:
        raise ValueError(f"{name} has {len(ih)} indices for {nfilt} filters")
    if len(np.unique(np.diff(ih))) > 1:
        raise ValueError(f"the indices of filters '{name}' must be regularly sampled")
    if min(ih) < 0 or max(ih) >= n:
        raise ValueError(f"the indices of filters '{name}' must be larger than 0 and smaller than `dims`")
    dh = int(ih[1] - ih[0]) if len(ih) > 1 else 1
    if dh < 1:
        raise ValueError(f"the indices of filters '{name}' must be increasing")
    return int(ih[0]), dh


def _bank_nodes(names, ihs, nfilt, dims, nh):
    """``(oh, dh)``, one entry per axis, of a bank of ``nfilt`` filters of sizes ``nh`` at the indices ``ihs`` of a
    ``dims`` block: ``ValueError`` for an even size, and :func:`_regular_nodes`' per axis"""
    if any(int(n) % 2 == 0 for n in nh):
        raise ValueError("filters hs must have odd length")
    nodes = [_regular_nodes(*a) for a in zip(names, ihs, nfilt, dims)]
    return tuple(o for o, _ in nodes), tuple(d for _, d in nodes)


class _NonStationaryConvolve(_RealTapsOperator):
    """The shared part of :class:`NonStationaryConvolve2D` / :class:`NonStationaryConvolve3D` on the axes ``_axes``
    (``"xz"`` / ``"xyz"``): the argument checks, the bank (uploaded once, in both real precisions), the geometry
    tuples and one ``_entry`` launch per apply"""

    def __init__(self, dims, hs, ihs, engine, num_threads_per_blocks, dtype):
        hs = hs.detach().cpu().numpy() if isinstance(hs, torch.Tensor) else np.asarray(hs)
        if np.iscomplexobj(hs):
            raise NotImplementedError("complex filters are not supported")
        ax, nd = self._axes, len(self._axes)
        dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        if len(dims) != nd:
            raise ValueError(f"dims must hold {('two', 'three')[nd - 2]} entries ({', '.join('n' + a for a in ax)}); "
                             f"got {dims}")
        if hs.ndim != 2 * nd:
            shape = ", ".join([f"nf{a}" for a in ax] + [f"nh{a}" for a in ax])
            raise ValueError(f"hs must be a {2 * nd}-D array of filters ({shape}); got shape {hs.shape}")
        self.oh, self.dh = _bank_nodes([f"ih{a}" for a in ax], ihs, hs.shape[:nd], dims, hs.shape[nd:])
        self.dims = self.dimsd = dims
        n = math.prod(dims)
        self.shape = (n, n)
        self._tdtype = _lib.torch_dtype(dtype)
        self.dtype = _lib.numpy_dtype(self._tdtype)
        self.engine, self.num_threads_per_blocks = engine, num_threads_per_blocks
        _lib.ctx()
        self._bank = _real_filters(hs)[1]
        self.nfilt = tuple(int(v) for v in hs.shape[:nd])
        self.nh = tuple(int(v) for v in hs.shape[nd:])
        self.hc = tuple(v // 2 for v in self.nh)
        self._geom = (*self.nfilt, *self.nh, *(v for od in zip(self.oh, self.dh) for v in od))

    def _launch(self, x, y, dt, adjoint):
        real = _REAL_OF.get(dt, dt)
        _lib.check(getattr(_lib.lib, self._entry)(_lib.ctx(), x.data_ptr(), y.data_ptr(), *self.dims,
                                                  2 if dt.is_complex else 1, self._bank[real].data_ptr(), *self._geom,
                                                  adjoint, _lib.code(real), _lib.stream()), self._entry)


class NonStationaryConvolve2D(_NonStationaryConvolve):
    """Rank-local non-stationary 2-D convolution of a C-ordered ``dims = (nx, nz)`` image,
    pylops.signalprocessing.NonStationaryConvolve2D (pylops 2.x) inside MPIBlockDiag: image-domain least-squares
    migration, with point-spread functions for filters.  ``hs`` of shape ``(nfx, nfz, nhx, nhz)`` holds real filters
    of odd sizes at the regularly spaced image points ``(ihx[a], ihz[b])``; point ``j`` uses ``h_j``, bilinear in the
    four filters around it (per axis, the first / last filter outside the nodes)::

        y[i] = sum_j h_j[nhx // 2 + ix - jx, nhz // 2 + iz - jz] x[j]

    and the adjoint is the exact transpose.  One b2_nsconvolve2d launch per apply (csrc/nsconvolve2d.cu), complex data
    included.  The operator dtype is ``dtype``; data are promoted and ``out=`` is handled as in
    :class:`NonStationaryConvolve1D`, and float32 data of a float32 operator use the bank rounded to float32.
    ``ValueError`` for even filter sizes, irregular or decreasing indices, indices outside ``[0, dims)``,
    ``len(ihx) != nfx``, ``len(ihz) != nfz``, an ``hs`` that is not 4-D and ``dims`` without two entries; complex
    filters are not provided.  ``engine`` and ``num_threads_per_blocks`` are accepted and ignored."""
    _axes, _entry = "xz", "b2_nsconvolve2d"

    def __init__(self, dims, hs, ihx, ihz, engine="numpy", num_threads_per_blocks=(32, 32), dtype="float64"):
        super().__init__(dims, hs, (ihx, ihz), engine, num_threads_per_blocks, dtype)
        (self.ohx, self.ohz), (self.dhx, self.dhz) = self.oh, self.dh


class NonStationaryConvolve3D(_NonStationaryConvolve):
    """Rank-local non-stationary 3-D convolution of a C-ordered volume of shape ``dims`` (three entries),
    pylops.signalprocessing.NonStationaryConvolve3D (pylops 2.x as remembered: pylops is not installed here to check
    the signature, defaults or weight clamp) inside MPIBlockDiag: image-domain least-squares migration in 3-D, with
    point-spread functions for filters.  ``hs`` of shape ``(nfx, nfy, nfz, nhx, nhy, nhz)`` holds real filters of odd
    sizes at the regularly spaced points ``(ihx[a], ihy[b], ihz[e])``; point ``j`` uses ``h_j``, trilinear in the
    eight filters around it (per axis, the first / last filter outside the nodes)::

        y[i] = sum_j h_j[nhx // 2 + ix - jx, nhy // 2 + iy - jy, nhz // 2 + iz - jz] x[j]

    and the adjoint is the exact transpose.  ``x``, ``y`` and ``z`` are pylops' labels for the positions 0, 1 and 2 of
    ``dims``: a 3-D :class:`Kirchhoff` image is ``(ny, nx, nz)``, so the operator for its PSFs is
    ``NonStationaryConvolve3D((ny, nx, nz), hs, i_first_axis, i_second_axis, iz)``.  One b2_nsconvolve3d launch per
    apply (csrc/nsconvolve3d.cu), complex data included.  The operator dtype is ``dtype``; data are promoted and
    ``out=`` is handled as in :class:`NonStationaryConvolve2D`, and float32 data of a float32 operator use the bank
    rounded to float32.  ``ValueError`` for even filter sizes, irregular or decreasing indices, indices outside
    ``[0, dims)``, ``len(ihx) != nfx`` (and for y, z), an ``hs`` that is not 6-D and ``dims`` without three entries;
    complex filters are not provided.  ``engine`` and ``num_threads_per_blocks`` are accepted and ignored."""
    _axes, _entry = "xyz", "b2_nsconvolve3d"

    def __init__(self, dims, hs, ihx, ihy, ihz, engine="numpy", num_threads_per_blocks=(2, 16, 16),
                 dtype="float64"):
        super().__init__(dims, hs, (ihx, ihy, ihz), engine, num_threads_per_blocks, dtype)


class _NonStationaryFilters(_KernelOperator):
    """The shared part of :class:`NonStationaryFilters1D` / :class:`NonStationaryFilters2D`: the fixed real input
    ``inp`` (uploaded once, in both real precisions), the shape ``(nx, nz, nfx, nfz, nhx, nhz, ohx, dhx, ohz, dhz)``
    of the 2-D adjoint (a 1-D operator has a singleton x axis), its workspace, sized once here so that no apply has
    to allocate, and the adjoint launch.  The kernels are real: complex data are applied part by part, and an operator
    of a complex dtype computes in its real dtype and returns complex results, as a complex NumPy operator would."""

    @staticmethod
    def _host_input(inp, ndim):
        """``inp`` on the host, checked: real (``NotImplementedError``) and of rank ``ndim`` (``ValueError``)"""
        inp = inp.detach().cpu().numpy() if isinstance(inp, torch.Tensor) else np.asarray(inp)
        if np.iscomplexobj(inp):
            raise NotImplementedError("complex inp is not supported")
        if inp.ndim != ndim:
            raise ValueError(f"inp must have {ndim} dimension(s); got shape {inp.shape}")
        return inp

    def _setup(self, inp, dims, dimsd, geom, dtype):
        self.dims, self.dimsd = tuple(dims), tuple(dimsd)
        self.shape = (math.prod(self.dimsd), math.prod(self.dims))
        tdt = _lib.torch_dtype(dtype)
        self._tdtype = _REAL_OF.get(tdt, tdt)       # the kernels' dtype: a complex operator applies data by parts
        self.dtype = _lib.numpy_dtype(tdt)
        _lib.ctx()
        self._inp, self._geom = _real_filters(inp)[1], tuple(int(v) for v in geom)
        nbytes = C.c_size_t(0)
        _lib.check(_lib.lib.b2_nsfilters2d_work_bytes(*self._geom, _lib.code(torch.float64), C.byref(nbytes)),
                   "b2_nsfilters2d_work_bytes")
        self._work = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda") if nbytes.value else None

    def _complex_data(self, x):
        """real data of a complex operator as complex data, so that the result is complex"""
        return x.to(_CPLX_OF[x.dtype]) if self.dtype.kind == "c" and x.dtype in _CPLX_OF else x

    def matvec(self, x, out=None):
        return self._apply(self._complex_data(x), 0, out)

    def rmatvec(self, x, out=None):
        return self._apply(self._complex_data(x), 1, out)

    _matvec, _rmatvec = matvec, rmatvec

    def _adjoint(self, x, y, dt):
        work, nbytes = (self._work.data_ptr(), self._work.numel()) if self._work is not None else (None, 0)
        _lib.check(_lib.lib.b2_nsfilters2d_adjoint(_lib.ctx(), x.data_ptr(), self._inp[dt].data_ptr(), y.data_ptr(),
                                                   *self._geom, work, nbytes, _lib.code(dt), _lib.stream()),
                   "b2_nsfilters2d_adjoint")


class NonStationaryFilters1D(_NonStationaryFilters):
    """Rank-local non-stationary 1-D filter estimation, pylops.signalprocessing.NonStationaryFilters1D (pylops 2.x as
    remembered: pylops is not installed here to check the signature) inside MPIVStack: time-varying wavelet
    estimation.  The model is the bank ``(nfilt = len(ih), hsize)`` of filters of odd length at the regularly spaced
    samples ``ih`` of the fixed real 1-D signal ``inp`` of ``n`` samples; the data are ``(n,)``::

        y[i] = sum_j h_j[hsize // 2 + i - j] inp[j]

    with ``h_j`` interpolated from the model bank as :class:`NonStationaryConvolve1D` interpolates its filters, so
    ``NonStationaryFilters1D(inp, hsize, ih) @ hs == NonStationaryConvolve1D(n, hs, ih) @ inp``.  The forward is one
    b2_nsconvolve_axis launch with ``inp`` for the data and the model for the bank; the adjoint, the exact transpose,
    is one b2_nsfilters2d_adjoint call with a singleton x axis (csrc/nsfilters.cu).  A float32 operator uses ``inp``
    rounded to float32; complex data are applied to their real and imaginary parts.  ``ValueError`` for an even
    ``hsize``, irregular or decreasing ``ih``, ``ih`` outside ``[0, n)`` and an ``inp`` that is not 1-D; a complex
    ``inp`` raises ``NotImplementedError``."""

    def __init__(self, inp, hsize, ih, dtype="float64", name="C"):
        inp = self._host_input(inp, 1)
        self.hsize, self.name = int(hsize), name
        self.n, self.nfilt = int(inp.shape[0]), len(np.ravel(ih))
        (self.oh,), (self.dh,) = _bank_nodes(("ih",), (ih,), (self.nfilt,), (self.n,), (self.hsize,))
        self.hc = self.hsize // 2
        self._setup(inp, (self.nfilt, self.hsize), (self.n,),
                    (1, self.n, 1, self.nfilt, 1, self.hsize, 0, 1, self.oh, self.dh), dtype)

    def _launch(self, x, y, dt, adjoint):
        if adjoint:
            self._adjoint(x, y, dt)
            return
        _lib.check(_lib.lib.b2_nsconvolve_axis(_lib.ctx(), self._inp[dt].data_ptr(), y.data_ptr(), 1, self.n, 1,
                                               x.data_ptr(), self.nfilt, self.hsize, self.hc, self.oh, self.dh, 0,
                                               _lib.code(dt), _lib.stream()), "b2_nsconvolve_axis")


class NonStationaryFilters2D(_NonStationaryFilters):
    """Rank-local non-stationary 2-D filter estimation, pylops.signalprocessing.NonStationaryFilters2D (pylops 2.x as
    remembered: pylops is not installed here to check the signature) inside MPIVStack: estimating a bank of
    point-spread or deblurring filters.  The model is the bank ``(nfx, nfz, nhx, nhz)`` (``hshape = (nhx, nhz)``,
    odd) at the regularly spaced points ``(ihx[a], ihz[b])`` of the fixed real image ``inp`` of shape ``(nx, nz)``;
    the data are ``(nx, nz)``::

        y[i] = sum_j h_j[nhx // 2 + ix - jx, nhz // 2 + iz - jz] inp[j]

    with ``h_j`` bilinear in the model bank as in :class:`NonStationaryConvolve2D`, so
    ``NonStationaryFilters2D(inp, hshape, ihx, ihz) @ hs == NonStationaryConvolve2D(inp.shape, hs, ihx, ihz) @ inp``.
    The forward is one b2_nsconvolve2d launch with ``inp`` for the image and the model for the bank; the adjoint,
    the exact transpose, is b2_nsfilters2d_adjoint (csrc/nsfilters.cu).  A float32 operator uses ``inp`` rounded to
    float32; complex data are applied to their real and imaginary parts.  ``ValueError`` for even ``hshape`` entries,
    irregular or decreasing indices, indices outside ``[0, inp.shape)`` and an ``inp`` that is not 2-D; a complex
    ``inp`` raises ``NotImplementedError``.  ``engine`` and ``num_threads_per_blocks`` are accepted and ignored."""

    def __init__(self, inp, hshape, ihx, ihz, engine="numpy", num_threads_per_blocks=(32, 32), dtype="float64",
                 name="C"):
        inp = self._host_input(inp, 2)
        self.hshape = self.nh = tuple(int(h) for h in hshape)
        if len(self.nh) != 2:
            raise ValueError(f"hshape must hold two entries (nhx, nhz); got {hshape}")
        nx, nz = (int(v) for v in inp.shape)
        self.nfilt = (len(np.ravel(ihx)), len(np.ravel(ihz)))
        self.oh, self.dh = _bank_nodes(("ihx", "ihz"), (ihx, ihz), self.nfilt, (nx, nz), self.nh)
        (self.ohx, self.ohz), (self.dhx, self.dhz) = self.oh, self.dh
        self.hc = (self.nh[0] // 2, self.nh[1] // 2)
        self.engine, self.num_threads_per_blocks, self.name = engine, num_threads_per_blocks, name
        self._setup(inp, self.nfilt + self.nh, (nx, nz),
                    (nx, nz, *self.nfilt, *self.nh, self.ohx, self.dhx, self.ohz, self.dhz), dtype)

    def _launch(self, x, y, dt, adjoint):
        if adjoint:
            self._adjoint(x, y, dt)
            return
        _lib.check(_lib.lib.b2_nsconvolve2d(_lib.ctx(), self._inp[dt].data_ptr(), y.data_ptr(), *self.dimsd, 1,
                                            x.data_ptr(), *self.nfilt, *self.nh, self.ohx, self.dhx, self.ohz,
                                            self.dhz, 0, _lib.code(dt), _lib.stream()), "b2_nsconvolve2d")


class PoststackLinearModelling(_AxisOperator):
    """Rank-local post-stack seismic modelling, pylops.avo.poststack.PoststackLinearModelling (pylops 2.x) for a
    real wavelet, as tutorials/poststack.py uses it inside MPIBlockDiag::

        PoststackLinearModelling(wav, nt0, spatdims) == Convolve1D(dims, wav, offset=len(wav) // 2, axis=0)
                                                        * FirstDerivative(dims, axis=0, sampling=1.0, kind=kind)

    on ``dims = (nt0,) + spatdims``; the adjoint is ``D^T C^T``.  A 2-D wavelet of shape ``(nt0, nwav)`` holds one
    wavelet per time sample (non-stationary): ``C[i, j] = wav[j, nwav // 2 + i - j]``, pylops'
    ``nonstationary_convmtx(wav, nt0, hc=nwav // 2, pad=(nt0, nt0))`` applied matrix-free (any ``nwav``).  The
    operator dtype is ``wav.dtype``; data are promoted and ``out=`` is handled as in :class:`Convolve1D`.  Each
    apply is ONE launch with the derivative fused into the convolution kernel (b2_poststack_axis, csrc/convolve.cu;
    2-D: b2_nspoststack_axis, csrc/nsconvolve.cu), equal bit for bit to the two-launch chain.  ``explicit`` /
    ``sparse`` matrices, complex wavelets and 2-D wavelets whose first dimension is not ``nt0`` are not provided."""

    def __init__(self, wav, nt0: int, spatdims=None, explicit: bool = False, sparse: bool = False,
                 kind: str = "centered"):
        if explicit or sparse:
            raise NotImplementedError("explicit / sparse matrices are not provided: use the matrix-free operator")
        if kind not in ("forward", "centered"):
            raise NotImplementedError(f"{kind} not an available derivative kind...")
        wav, bank = _real_filters(wav)
        if spatdims is None:
            dims = (int(nt0),)
        elif np.ndim(spatdims) == 0:
            dims = (int(nt0), int(spatdims))
        else:
            dims = (int(nt0),) + tuple(int(d) for d in spatdims)
        self.nonstationary = wav.ndim == 2 and wav.shape[0] == int(nt0)
        if self.nonstationary:       # the bank of nt0 wavelets at samples 0, 1, ..., nt0 - 1
            self._conv = _FilterBank(bank, wav.shape[1] // 2, 0, 1)
        else:
            self._conv = _StationaryTaps(bank, len(wav) // 2)
        super().__init__(dims, 0, np.result_type(wav.dtype, np.float32))
        self.nh, self.offset = self._conv.nh, self._conv.nh // 2
        self.kind = kind
        self._kind = _lib.FD_CENTERED if kind == "centered" else _lib.FD_FORWARD

    def _launch(self, x, y, dt, adjoint):
        self._conv.launch(x, y, self._lines(dt), adjoint, self._kind)


class Transpose(LocalOperator):
    """pylops.basicoperators.Transpose: ``y = x.reshape(dims).transpose(axes).ravel()``; the adjoint applies the
    inverse permutation.  A strided copy through torch (plumbing, not a hot path: inside ``T.H @ X @ T`` it is
    folded away, see :class:`LocalOperator`).  ``T.H`` is the inverse Transpose."""

    def __init__(self, dims, axes, dtype="float64"):
        self.dims = tuple(int(d) for d in (dims if np.ndim(dims) else (dims,)))
        self.axes = tuple(int(a) for a in (axes if np.ndim(axes) else (axes,)))
        if sorted(self.axes) != list(range(len(self.dims))):
            raise ValueError(f"axes {axes} is not a permutation of the {len(self.dims)} axes of dims {self.dims}")
        self.dimsd = tuple(self.dims[a] for a in self.axes)
        n = int(np.prod(self.dims))
        self.shape = (n, n)
        self.dtype = np.dtype(dtype)

    @property
    def H(self) -> "Transpose":
        return Transpose(self.dimsd, tuple(int(a) for a in np.argsort(self.axes)), dtype=self.dtype)

    def _matvec(self, x):
        return x.reshape(self.dims).permute(self.axes).contiguous().reshape(-1)

    def _rmatvec(self, x):
        return x.reshape(self.dimsd).permute(tuple(int(a) for a in np.argsort(self.axes))).contiguous().reshape(-1)


def _traveltime_tables(z, x, srcs, recs, vel, y=None):
    """analytic (constant-velocity) traveltime tables of pylops.waveeqprocessing.Kirchhoff, in float64, computed on
    the host with pylops' NumPy expressions: ``trav_srcs[ii, isrc] = sqrt((X - sx)**2 + (Z - sz)**2) / vel`` on the
    raveled ``meshgrid(x, z, indexing="ij")`` grid (``ii = ix * nz + iz``), and the same for the receivers.  With
    ``y`` (3-D): the grid ``meshgrid(y, x, z, indexing="ij")`` (``ii = (iy * nx + ix) * nz + iz``), points with rows
    ``(y, x, z)``, and ``(Y - sy)**2`` added last.  :class:`Kirchhoff` builds the same tables on the device
    (b2_kirchhoff_tables); this is their host reference."""
    srcs, recs = np.asarray(srcs), np.asarray(recs)
    if y is None:
        X, Z = np.meshgrid(x, z, indexing="ij")
        X, Z = X.ravel(), Z.ravel()
        trav_srcs = np.sqrt((X[:, None] - srcs[0][None]) ** 2 + (Z[:, None] - srcs[1][None]) ** 2) / vel
        trav_recs = np.sqrt((X[:, None] - recs[0][None]) ** 2 + (Z[:, None] - recs[1][None]) ** 2) / vel
        return trav_srcs.astype(np.float64), trav_recs.astype(np.float64)
    Y, X, Z = np.meshgrid(y, x, z, indexing="ij")
    Y, X, Z = Y.ravel(), X.ravel(), Z.ravel()

    def table(pts):
        dist2 = (X[:, None] - pts[1][None]) ** 2 + (Z[:, None] - pts[2][None]) ** 2
        dist2 += (Y[:, None] - pts[0][None]) ** 2
        return (np.sqrt(dist2) / vel).astype(np.float64)

    return table(srcs), table(recs)


# Device memory the resident traveltime tables of one Kirchhoff operator may take, (ns + nr) * ni * 8 bytes.  Above
# it an analytic operator keeps one chunk of image points' tables (a multiple of 32 points within the budget) and
# rebuilds them for each chunk on every apply; eikonal and byot operators raise ValueError (with mode="eikonal" the
# solver's work buffer counts too).  Read when an operator is constructed.
KIRCHHOFF_TABLE_BYTES = 4 << 30


def _uniform_spacing(name, a):
    """the sampling of a uniform, increasing axis (1.0 for a one-point axis), else ValueError"""
    if a.size < 2:
        return 1.0
    d = float(a[1] - a[0])
    if not (d > 0.0 and np.isfinite(d)) or not np.allclose(np.diff(a), d, rtol=1e-6, atol=0.0):
        raise ValueError(f"Kirchhoff: mode='eikonal' needs uniform, increasing axes; {name} is not")
    return d


def _user_table(name, tab, ni, n):
    """one byot table, pylops' shape (ni, n), in any real dtype -> the kernel layout (n, ni), float64, on the device"""
    tab = tab if isinstance(tab, torch.Tensor) else torch.as_tensor(np.asarray(tab))
    if tab.is_complex() or tab.dtype == torch.bool or tab.dim() != 2 or tuple(tab.shape) != (ni, n):
        raise ValueError(f"Kirchhoff: mode='byot' needs {name} as a real array of shape ({ni}, {n}); got "
                         f"{tab.dtype} {tuple(tab.shape)}")
    return tab.to(device="cuda", dtype=torch.float64).t().contiguous()


class Kirchhoff(_KernelOperator):
    """Rank-local Kirchhoff demigration, pylops.waveeqprocessing.Kirchhoff (pylops 2.x) in 2-D or, with ``y``, 3-D:
    the ``Demop`` of tutorials/lsm.py inside MPIVStack.  The model is the image ``(nx, nz)`` (3-D: ``(ny, nx, nz)``,
    with ``srcs`` / ``recs`` of shape ``(3, n)``, rows ``(y, x, z)``), the data the traces ``(ns, nr, nt)``.  For
    every (image point, trace) pair the traveltime ``trav`` indexes the trace at ``it = int(trav / dt)`` with weights
    ``1 - d`` and ``d`` on samples ``it`` and ``it + 1`` (``d = trav / dt - it``, pairs with ``it >= nt - 1`` are
    dropped); the traces are then convolved with ``wav`` (``Convolve1D`` with ``offset=wavcenter`` along time).

    The float64 traveltime tables come from ``mode``:

    - ``"analytic"``: constant velocity, scalar ``vel``.  Built on the device (b2_kirchhoff_tables), equal bit for
      bit to pylops' NumPy tables.  While ``(ns + nr) * ni * 8`` bytes fit in :data:`KIRCHHOFF_TABLE_BYTES` they are
      built once at construction and stay resident; above it (``chunked``) the operator holds one chunk of image
      points' tables and each apply builds and applies them chunk by chunk (b2_kirchhoff_chunk), with the same
      result bit for bit.
    - ``"eikonal"``: ``vel`` a finite, positive velocity model of the image's shape on uniform axes.  Each source and
      receiver is snapped to its nearest grid node (half to even) and its first-arrival times are solved on the
      device (b2_eikonal_tables, a first-order Godunov upwind scheme iterated to its fixed point, ``max_iter = ni``),
      once at construction.  pylops uses scikit-fmm here, whose second-order scheme puts the zero level set half a
      cell from the node: the tables differ from pylops' by O(h / v), most near the source.  Pass scikit-fmm's
      tables through ``"byot"`` to reproduce pylops exactly.
    - ``"byot"``: ``trav=(trav_srcs, trav_recs)`` of pylops' shapes ``(ni, ns)`` / ``(ni, nr)``, NumPy arrays or
      torch tensors of any real dtype, converted to float64 once; ``vel`` is ignored.

    ``trav_srcs`` / ``trav_recs`` are ``(ni, ns)`` / ``(ni, nr)`` views of the resident device tables (not of a
    chunked analytic operator).  A workspace of ``ns * nr * nt`` samples holds the traces between the two stages.
    Forward: spreading into the workspace, then b2_convolve_axis into the output; adjoint: the reverse
    (csrc/kirchhoff.cu, csrc/convolve.cu).  Only the static (``dynamic=False``) operator without wavelet filtering
    or apertures is provided; ``engine`` is accepted and ignored."""

    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, mode="eikonal", wavfilter=False,
                 dynamic=False, trav=None, amp=None, aperture=None, angleaperture=90, snell=None, engine="numpy",
                 dtype="float64", name="K"):
        for opt, val, default in (("wavfilter", wavfilter, False), ("dynamic", dynamic, False),
                                  ("amp", amp, None), ("aperture", aperture, None),
                                  ("angleaperture", angleaperture, 90), ("snell", snell, None)):
            if not (val is default or (default is not None and np.ndim(val) == 0 and val == default)):
                raise NotImplementedError(f"Kirchhoff: {opt}={val!r} is not supported (only its default {default!r})")
        if mode not in ("analytic", "eikonal", "byot"):
            raise NotImplementedError(f"Kirchhoff: mode={mode!r} is not supported (analytic, eikonal or byot)")
        if trav is not None and mode != "byot":
            raise NotImplementedError(f"Kirchhoff: trav is only used with mode='byot' (mode={mode!r})")
        if mode == "analytic" and np.ndim(vel) != 0:
            raise ValueError("vel must be scalar for mode=analytical")
        if mode == "eikonal" and np.ndim(vel) == 0:
            raise NotImplementedError("Kirchhoff: mode='eikonal' needs a velocity model of the image's shape; a "
                                      "scalar vel (constant velocity) is mode='analytic'")
        if mode == "byot":
            if trav is None:
                raise NotImplementedError("Kirchhoff: mode='byot' needs trav=(trav_srcs, trav_recs)")
            if isinstance(trav, (np.ndarray, torch.Tensor)) or len(trav) != 2:
                raise NotImplementedError("Kirchhoff: trav as one (ni, ns * nr) table is not supported: pass "
                                          "trav=(trav_srcs, trav_recs) of shapes (ni, ns) and (ni, nr)")
        z, x, t = (np.asarray(a) for a in (z, x, t))
        srcs, recs = np.asarray(srcs), np.asarray(recs)
        nd = 2 if y is None else 3
        if srcs.ndim != 2 or recs.ndim != 2 or srcs.shape[0] != nd or recs.shape[0] != nd:
            raise NotImplementedError(
                f"Kirchhoff: y={'None' if y is None else 'given'} needs srcs and recs of shape ({nd}, n) with rows "
                f"{'(x, z)' if y is None else '(y, x, z)'} (y=None: 2-D, shape (2, n); y given: 3-D, shape "
                f"(3, n)); got srcs {srcs.shape}, recs {recs.shape}")
        self._wav = _StationaryTaps(_real_filters(wav)[1], wavcenter)   # a real 1-D wavelet, or NotImplementedError
        self.mode = mode
        self.ny = 1 if y is None else np.asarray(y).size
        self.nx, self.nz, self.nt = x.size, z.size, t.size
        self.ns, self.nr = srcs.shape[1], recs.shape[1]
        self.ni = self.ny * self.nx * self.nz
        self.dt = float(t[1] - t[0])
        self.dims = (self.nx, self.nz) if y is None else (self.ny, self.nx, self.nz)
        self.dimsd = (self.ns, self.nr, self.nt)
        self.shape = (self.ns * self.nr * self.nt, self.ni)
        self.engine = engine
        self._tdtype = _lib.torch_dtype(dtype)
        self.dtype = _lib.numpy_dtype(self._tdtype)
        if self._tdtype not in (torch.float32, torch.float64):
            raise NotImplementedError(f"Kirchhoff: dtype {dtype} is not supported (float32 or float64)")
        _lib.ctx()
        table_bytes = (self.ns + self.nr) * self.ni * 8
        if mode == "analytic":
            self._analytic(y, x, z, srcs, recs, vel)
        else:
            if mode == "byot":
                self._check_budget(table_bytes, "")
                self._ts = _user_table("trav_srcs", trav[0], self.ni, self.ns)
                self._tr = _user_table("trav_recs", trav[1], self.ni, self.nr)
            else:
                self._eikonal(y, x, z, srcs, recs, vel, table_bytes)
            self._nc, self.chunked = self.ni, False
        self._ws = {self._tdtype: torch.empty(self.shape[0], dtype=self._tdtype, device="cuda")}

    @staticmethod
    def _check_budget(need, what):
        if need > KIRCHHOFF_TABLE_BYTES:
            raise ValueError(f"Kirchhoff: the resident traveltime tables{what} need {need} bytes, more than "
                             f"KIRCHHOFF_TABLE_BYTES = {KIRCHHOFF_TABLE_BYTES}; only mode='analytic' can rebuild "
                             f"its tables in chunks")

    def _analytic(self, y, x, z, srcs, recs, vel):
        def dev(a):
            return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).to("cuda")

        # axes and point coordinates in float64 (the table builder's inputs), points as rows ((y,) x, z)
        self._axes = (None if y is None else dev(y), dev(x), dev(z))
        self._srcs, self._recs = dev(srcs), dev(recs)
        self._vel = float(vel)
        # image points per chunk: all of them while the tables fit in the budget, else a multiple of 32 that fits
        per_point = (self.ns + self.nr) * 8
        nc = self.ni if per_point * self.ni <= KIRCHHOFF_TABLE_BYTES else KIRCHHOFF_TABLE_BYTES // per_point // 32 * 32
        self._nc = min(self.ni, max(32, nc))
        self.chunked = self._nc < self.ni
        # kernel layout: (ns, nc) and (nr, nc), a trace reads contiguous image points
        self._ts = torch.empty((self.ns, self._nc), dtype=torch.float64, device="cuda")
        self._tr = torch.empty((self.nr, self._nc), dtype=torch.float64, device="cuda")
        if not self.chunked:
            self._tables(0, self.ni)

    def _eikonal(self, y, x, z, srcs, recs, vel, table_bytes):
        """the eikonal tables, solved on the device in batches of points whose work buffer fits the budget"""
        vel = vel.detach().cpu().numpy() if isinstance(vel, torch.Tensor) else np.asarray(vel)
        if tuple(vel.shape) != self.dims:
            raise ValueError(f"Kirchhoff: mode='eikonal' needs vel of the image shape {self.dims}; got {vel.shape}")
        if not (np.issubdtype(vel.dtype, np.integer) or np.issubdtype(vel.dtype, np.floating)):
            raise ValueError(f"Kirchhoff: mode='eikonal' needs a real vel; got {vel.dtype}")
        vel = np.ascontiguousarray(vel, dtype=np.float64)
        if not (np.all(np.isfinite(vel)) and np.all(vel > 0)):
            raise ValueError("Kirchhoff: mode='eikonal' needs a finite, positive vel")
        axes = ((("y", np.asarray(y, dtype=np.float64)),) if y is not None else ()) + \
            (("x", np.asarray(x, dtype=np.float64)), ("z", np.asarray(z, dtype=np.float64)))
        h = [_uniform_spacing(nm, a) for nm, a in axes]
        h = [1.0] * (3 - len(h)) + h
        full = (self.ny, self.nx, self.nz)

        def nodes(name, pts):
            """grid nodes (n, 3) of the points: round((p - axis[0]) / d), half to even, as pylops"""
            cols = [np.round((np.asarray(p, dtype=np.float64) - a[0]) / d).astype(np.int64)
                    for p, (_, a), d in zip(pts, axes, h[3 - len(axes):])]
            if len(cols) == 2:
                cols.insert(0, np.zeros_like(cols[0]))
            nd = np.ascontiguousarray(np.stack(cols, axis=1), dtype=np.int64)
            bad = np.any((nd < 0) | (nd >= np.asarray(full)), axis=1)
            if bad.any():
                raise ValueError(f"Kirchhoff: {name} {np.flatnonzero(bad).tolist()} lie outside the image grid")
            return nd

        idx_s, idx_r = nodes("sources", srcs), nodes("receivers", recs)
        wb = _lib.lib.b2_eikonal_work_bytes
        if table_bytes + wb(*full, 1) > KIRCHHOFF_TABLE_BYTES:
            self._check_budget(table_bytes + wb(*full, 1), " with the eikonal solver's work buffer")
        nb = max(self.ns, self.nr)                       # points per solve: as many as the budget allows
        while table_bytes + wb(*full, nb) > KIRCHHOFF_TABLE_BYTES:
            nb = max(1, nb // 2)
        self._ts = torch.empty((self.ns, self.ni), dtype=torch.float64, device="cuda")
        self._tr = torch.empty((self.nr, self.ni), dtype=torch.float64, device="cuda")
        dvel = torch.as_tensor(vel).to("cuda")
        work = torch.empty(wb(*full, nb), dtype=torch.uint8, device="cuda")
        info = (C.c_longlong * 4)()
        self.eikonal_info = {"iterations": 0, "passes": 0, "blocks": 0, "blocks_all": 0}
        for idx, tab in ((idx_s, self._ts), (idx_r, self._tr)):
            for p0 in range(0, len(idx), nb):
                part = np.ascontiguousarray(idx[p0:p0 + nb])
                _lib.check(_lib.lib.b2_eikonal_tables(_lib.ctx(), dvel.data_ptr(), *full, *h, part.ctypes.data,
                                                      len(part), self.ni, tab[p0].data_ptr(), work.data_ptr(),
                                                      info, _lib.stream()), "b2_eikonal_tables")
                for k, v in zip(("iterations", "passes", "blocks", "blocks_all"), info):
                    self.eikonal_info[k] = max(self.eikonal_info[k], v) if k == "iterations" else \
                        self.eikonal_info[k] + v

    @property
    def trav_srcs(self) -> torch.Tensor:
        """(ni, ns) float64 device view of the resident source tables (pylops' layout)"""
        if self.chunked:
            raise AttributeError("Kirchhoff: a chunked analytic operator keeps no resident trav_srcs")
        return self._ts.t()

    @property
    def trav_recs(self) -> torch.Tensor:
        """(ni, nr) float64 device view of the resident receiver tables (pylops' layout)"""
        if self.chunked:
            raise AttributeError("Kirchhoff: a chunked analytic operator keeps no resident trav_recs")
        return self._tr.t()

    def _compute_dtype(self, xdt):
        """float32 / float64 data are applied in ``promote(dtype, xdt)``; complex data part by part"""
        return torch.promote_types(self._tdtype, xdt) if xdt in (torch.float32, torch.float64) else self._tdtype

    def _tables(self, i0, nc):
        """the tables of image points [i0, i0 + nc) into ``_ts`` / ``_tr``, rows of nc points"""
        ay, ax, az = self._axes
        for pts, tab in ((self._srcs, self._ts), (self._recs, self._tr)):
            _lib.check(_lib.lib.b2_kirchhoff_tables(_lib.ctx(), _lib.ptr(ay), ax.data_ptr(), az.data_ptr(), self.ny,
                                                    self.nx, self.nz, pts.data_ptr(), pts.shape[1], self._vel, i0, nc,
                                                    tab.data_ptr(), _lib.stream()), "b2_kirchhoff_tables")

    def _kirch(self, x, y, real, adjoint):
        if not self.chunked:
            _lib.check(_lib.lib.b2_kirchhoff(_lib.ctx(), x.data_ptr(), y.data_ptr(), self._ts.data_ptr(),
                                             self._tr.data_ptr(), self.ni, self.ns, self.nr, self.nt, self.dt,
                                             adjoint, _lib.code(real), _lib.stream()), "b2_kirchhoff")
            return
        for i0 in range(0, self.ni, self._nc):
            nc = min(self._nc, self.ni - i0)
            self._tables(i0, nc)
            _lib.check(_lib.lib.b2_kirchhoff_chunk(_lib.ctx(), x.data_ptr(), y.data_ptr(), self._ts.data_ptr(),
                                                   self._tr.data_ptr(), self.ni, i0, nc, self.ns, self.nr, self.nt,
                                                   self.dt, adjoint, int(i0 > 0 and not adjoint), _lib.code(real),
                                                   _lib.stream()), "b2_kirchhoff_chunk")

    def _launch(self, x, y, dt, adjoint):
        ws = self._ws.get(dt)
        if ws is None:                          # data of the other precision: one more workspace, kept
            ws = self._ws[dt] = torch.empty(self.shape[0], dtype=dt, device="cuda")
        traces = (self.ns * self.nr, self.nt, 1, dt)      # the wavelet runs along time
        if adjoint:
            self._wav.launch(x, ws, traces, 1)
            self._kirch(ws, y, dt, 1)
        else:
            self._kirch(x, ws, dt, 0)
            self._wav.launch(ws, y, traces, 0)


class LSM:
    """pylops.waveeqprocessing.LSM (pylops 2.x) for ``kind="kirchhoff"``: builds the demigration operator ``Demop``, a
    :class:`Kirchhoff` with ``kwargs_mod`` passed through -- the only part tutorials/lsm.py uses (each rank's
    ``lsm.Demop`` goes into MPIVStack) -- and ``solve``, which inverts this rank's sources on their own."""

    def __init__(self, z, x, t, srcs, recs, vel, wav, wavcenter, y=None, kind="kirchhoff", dottest=False,
                 **kwargs_mod):
        if kind != "kirchhoff":
            raise NotImplementedError(f"LSM: kind={kind!r} is not supported (only 'kirchhoff')")
        if dottest:
            raise NotImplementedError("LSM: dottest=True is not supported (run utils.dottest on Demop)")
        self.y, self.x, self.z, self.t = y, x, z, t
        self.Demop = Kirchhoff(z, x, t, srcs, recs, vel, wav, wavcenter, y=y, **kwargs_mod)

    def solve(self, d, solver=None, **kwargs_solver):
        """pylops' ``LSM.solve``: invert the data ``d`` (``ns * nr * nt`` values, NumPy or torch) of this rank's
        sources, rank-local as in pylops.  ``Demop`` runs inside ``MPIVStack`` on a one-rank communicator with a
        BROADCAST model from ``x0 = 0``, through this package's ``lsqr`` (``solver=None``) or ``cgls``, with
        ``kwargs_solver`` passed on.  Returns the image, a device tensor of shape ``Demop.dims``."""
        from . import comm as _comm
        from .basicoperators.VStack import MPIVStack
        from .DistributedArray import DistributedArray, Partition
        from .optimization.basic import cgls, lsqr
        if solver is None:
            solver = lsqr
        if solver is not lsqr and solver is not cgls:
            raise NotImplementedError(f"LSM.solve: solver={solver!r} is not supported (lsqr or cgls of this package)")
        one = _comm.Comm(rank=0, size=1)
        Op = MPIVStack([self.Demop], base_comm=one)
        dt = _lib.torch_dtype(self.Demop.dtype)
        dev = torch.device("cuda", torch.cuda.current_device())
        dloc = torch.as_tensor(d).to(device=dev, dtype=dt).reshape(-1)
        if dloc.numel() != Op.shape[0]:
            raise ValueError(f"LSM.solve: d has {dloc.numel()} values, Demop has {Op.shape[0]} rows")
        dd = DistributedArray(global_shape=Op.shape[0], base_comm=one, dtype=dt)
        dd.local_array[:] = dloc
        x0 = DistributedArray(global_shape=Op.shape[1], base_comm=one, partition=Partition.BROADCAST, dtype=dt)
        x0.local_array.zero_()
        x = solver(Op, dd, x0=x0, **kwargs_solver)[0]
        return x.local_array.reshape(self.Demop.dims)


_RADON_KINDS = {"linear": _lib.RADON_LINEAR, "parabolic": _lib.RADON_PARABOLIC, "hyperbolic": _lib.RADON_HYPERBOLIC}


def _radon_sampling(name, axis):
    """``|axis[1] - axis[0]|`` of a float64 axis, or ValueError for one too short to have a sampling"""
    if axis.size < 2:
        raise ValueError(f"{name} needs at least 2 samples to define its sampling; got {axis.size}")
    return abs(axis[1] - axis[0])


class _Radon(_RealTapsOperator):
    """The shared part of :class:`Radon2D` / :class:`Radon3D`: the unitless axes (computed here in float64 and
    uploaded once) and one b2_radon launch per apply.  ``haxes`` / ``paxes`` hold one axis (2-D) or the (y, x) pair
    (3-D).  The unit conventions (pylops 2.x as remembered: pylops is not installed here to check them) all live in
    this constructor:

    - ``dt = |taxis[1] - taxis[0]|``, ``dh = |haxis[1] - haxis[0]|`` per spatial axis;
    - offsets: ``centeredh`` gives ``arange(nh) - nh // 2 + ((nh + 1) % 2) / 2``, else ``haxis / dh``;
    - slownesses: linear ``paxis * (dh / dt)``, parabolic ``paxis * (dh * dh / dt)``, hyperbolic (a velocity)
      ``paxis * (dt / dh)``."""

    def __init__(self, taxis, haxes, paxes, kind, centeredh, interp, onthefly, engine, dtype, name):
        if engine not in ("numpy", "numba", "cuda"):
            raise KeyError("engine must be numpy or numba or cuda")
        if kind not in _RADON_KINDS:
            raise NotImplementedError(f"kind={kind!r} is not supported (linear, parabolic or hyperbolic)")
        self._tdtype = _lib.torch_dtype(dtype)
        if self._tdtype not in (torch.float32, torch.float64):
            raise NotImplementedError(f"dtype={dtype!r} is not supported (float32 or float64; complex data are "
                                      f"applied by a real operator)")
        self.dtype = _lib.numpy_dtype(self._tdtype)
        self.kind, self.centeredh, self.interp = kind, bool(centeredh), bool(interp)
        self.onthefly, self.engine, self.name = onthefly, engine, name
        taxis = np.asarray(taxis, dtype=np.float64).ravel()
        dt = _radon_sampling("taxis", taxis)
        hs, ps = [], []
        for hname, haxis, paxis in zip(("haxis",) if len(haxes) == 1 else ("hyaxis", "hxaxis"), haxes, paxes):
            haxis = np.asarray(haxis, dtype=np.float64).ravel()
            paxis = np.asarray(paxis, dtype=np.float64).ravel()
            dh = _radon_sampling(hname, haxis)
            nh = haxis.size
            hs.append(np.arange(nh) - nh // 2 + ((nh + 1) % 2) / 2 if self.centeredh else haxis / dh)
            ps.append(paxis * {"linear": dh / dt, "parabolic": dh * dh / dt, "hyperbolic": dt / dh}[kind])
        self._nt = taxis.size
        nh, npp = tuple(h.size for h in hs), tuple(p.size for p in ps)
        self.dims, self.dimsd = npp + (self._nt,), nh + (self._nt,)
        self.shape = (math.prod(self.dimsd), math.prod(self.dims))
        _lib.ctx()
        self._axes = [torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).to("cuda") for a in hs + ps]
        if len(hs) == 1:
            hy, hx, py, px = None, self._axes[0], None, self._axes[1]
        else:
            hy, hx, py, px = self._axes
        nhy, nhx = (1,) + nh if len(nh) == 1 else nh
        npy, npx = (1,) + npp if len(npp) == 1 else npp
        self._geom = (nhy, nhx, npy, npx, _lib.ptr(hy), hx.data_ptr(), _lib.ptr(py), px.data_ptr(),
                      _RADON_KINDS[kind], int(self.interp))

    def _launch(self, x, y, dt, adjoint):
        real = _REAL_OF.get(dt, dt)
        _lib.check(_lib.lib.b2_radon(_lib.ctx(), x.data_ptr(), y.data_ptr(), self._nt, 2 if dt.is_complex else 1,
                                     *self._geom, adjoint, _lib.code(real), _lib.stream()), "b2_radon")


class Radon2D(_Radon):
    """Rank-local 2-D Radon transform of one gather, pylops.signalprocessing.Radon2D (pylops 2.x as remembered) inside
    MPIBlockDiag: each CMP gather is one block.  The model is ``dims = (npx, nt)``, the data ``dimsd = (nh, nt)``.
    On the unitless axes of :class:`_Radon`, model sample ``(p, t0)`` (``t0`` an integer sample index) reaches trace
    ``h`` at ``tdec`` = ``t0 + p*h`` (linear), ``t0 + p*(h*h)`` (parabolic) or ``sqrt(t0*t0 + (h/p)*(h/p))``
    (hyperbolic), in float64.  With ``interp`` the pair is used iff ``0 <= tdec < nt - 1`` and spreads onto samples
    ``it = trunc(tdec)`` and ``it + 1`` with weights ``1 - d`` and ``d`` (``d = tdec - it``); without, iff
    ``0 <= tdec < nt`` onto sample ``it``.  The adjoint is the exact transpose.

    One b2_radon launch per apply (csrc/radon.cu), complex data included (applied in the complex dtype of the
    operator's and the data's real dtypes promoted).  Index and weights are float64 and every sum is float64,
    rounded once to the data's dtype.  ``dtype`` is float32 or float64: a complex dtype, or a ``kind`` other than
    linear / parabolic / hyperbolic, raises ``NotImplementedError``; an axis with fewer than 2 samples (taxis, haxis)
    ``ValueError``; an ``engine`` other than numpy / numba / cuda ``KeyError``.  ``onthefly`` and ``engine`` do not
    change the values and are otherwise ignored."""

    def __init__(self, taxis, haxis, pxaxis, kind="linear", centeredh=True, interp=True, onthefly=False,
                 engine="numpy", dtype="float64", name="R"):
        super().__init__(taxis, (haxis,), (pxaxis,), kind, centeredh, interp, onthefly, engine, dtype, name)


class Radon3D(_Radon):
    """Rank-local 3-D Radon transform of one gather, pylops.signalprocessing.Radon3D (pylops 2.x as remembered) inside
    MPIBlockDiag.  The model is ``dims = (npy, npx, nt)``, the data ``dimsd = (nhy, nhx, nt)``.  As :class:`Radon2D`
    with the y term added last: ``tdec`` = ``(t0 + px*hx) + py*hy`` (linear), ``(t0 + px*(hx*hx)) + py*(hy*hy)``
    (parabolic) or ``sqrt((t0*t0 + (hx/px)*(hx/px)) + (hy/py)*(hy/py))`` (hyperbolic), each spatial axis made
    unitless with its own sampling.  Same launch, dtypes and errors as :class:`Radon2D` (hyaxis and hxaxis need 2
    samples each)."""

    def __init__(self, taxis, hyaxis, hxaxis, pyaxis, pxaxis, kind="linear", centeredh=True, interp=True,
                 onthefly=False, engine="numpy", dtype="float64", name="R"):
        super().__init__(taxis, (hyaxis, hxaxis), (pyaxis, pxaxis), kind, centeredh, interp, onthefly, engine, dtype,
                         name)


def _taper(nmask, ntap, tapertype):
    """pylops.utils.tapers.taper (pylops 2.x as remembered), float64: ``nmask`` samples rising over the first
    ``ntap`` and falling over the last ``ntap`` (hanning: the first ``ntap`` samples of ``np.hanning(2 * ntap - 1)``;
    cosine / cosinesquare: of ``(0.5 * (cos((k - c) * pi / c) + 1)) ** e``, ``c = ntap - 1``), ones between; ones
    for ``None``.  ``ValueError`` for a hanning ``ntap`` above ``nmask / 2``."""
    if tapertype is None:
        return np.ones(nmask)
    if tapertype == "hanning":
        if ntap > 0 and nmask // ntap < 2:
            raise ValueError(f"ntap={ntap} must be smaller or equal than {nmask // 2}")
        rise = np.hanning(2 * ntap - 1)[:ntap]
    elif tapertype in ("cosine", "cosinesquare"):
        ntap = 0 if ntap == 1 else ntap
        c = (2 * ntap - 2) / 2
        with np.errstate(divide="ignore", invalid="ignore"):
            rise = ((0.5 * (np.cos((np.arange(2 * ntap - 1) - c) * np.pi / c) + 1.0))
                    ** (2 if tapertype == "cosinesquare" else 1))[:ntap]
    else:
        raise ValueError(f"tapertype={tapertype!r} is not supported (hanning, cosine, cosinesquare or None)")
    return np.concatenate([rise, np.ones(nmask - 2 * ntap), rise[::-1]])


def _slidingsteps(n, nwin, nover):
    """the first trace of every window of ``nwin`` traces, one every ``nwin - nover``, along an axis of ``n``"""
    if nwin > n:
        raise ValueError(f"nwin={nwin} is bigger than ntr={n}...")
    if not 0 <= nover < nwin:
        raise ValueError(f"nover={nover} must be in [0, nwin) = [0, {nwin})")
    return np.arange(0, n - nwin + 1, nwin - nover, dtype=int)


def _axis_tapers(nwins, nwin, nover, tapertype, edge):
    """``(nwins, nwin)`` float64: each window's taper along one axis, the first window's leading ``nover`` samples
    and the last window's trailing ``nover`` set to ``edge(taper)`` (one window: the trailing ones only)"""
    tap = _taper(nwin, nover, tapertype)
    taps = np.tile(tap, (nwins, 1))
    if nwins > 1:
        taps[0, :nover] = edge(tap)
    taps[-1, nwin - nover:] = edge(tap)
    return taps


def sliding2d_design(dimsd, nwin, nover, nop, verb=False):
    """pylops.signalprocessing.sliding2d_design: ``(nwins, dims, mwins_inends, dwins_inends)`` of a
    :class:`Sliding2D` on data ``dimsd = (n, nt)`` with windows of ``nwin`` traces overlapping by ``nover`` and an
    inner operator of model ``nop``: ``dims = (nwins * nop[0], nop[1])``.  Host only."""
    starts = _slidingsteps(int(dimsd[0]), int(nwin), int(nover))
    nwins = len(starts)
    dims = (nwins * int(nop[0]), int(nop[1]))
    mstarts = np.arange(nwins) * int(nop[0])
    if verb:
        print(f"{nwins} windows of {nwin} traces, model {dims}, data {tuple(dimsd)}")
    return (nwins, dims, ((mstarts, mstarts + int(nop[0])), (0, dims[1])),
            ((starts, starts + int(nwin)), (0, int(dimsd[-1]))))


def sliding3d_design(dimsd, nwin, nover, nop, verb=False):
    """pylops.signalprocessing.sliding3d_design: ``(nwins, dims, mwins_inends, dwins_inends)`` of a
    :class:`Sliding3D` on data ``dimsd = (n0, n1, nt)`` with windows ``nwin = (nwin0, nwin1)`` overlapping by
    ``nover`` and an inner operator of model ``nop``: ``nwins = (nwins0, nwins1)``,
    ``dims = (nwins0 * nop[0], nwins1 * nop[1], nop[2])``.  Host only."""
    st = [_slidingsteps(int(dimsd[a]), int(nwin[a]), int(nover[a])) for a in (0, 1)]
    nwins = (len(st[0]), len(st[1]))
    dims = (nwins[0] * int(nop[0]), nwins[1] * int(nop[1]), int(nop[2]))
    m = [np.arange(nwins[a]) * int(nop[a]) for a in (0, 1)]
    if verb:
        print(f"{nwins[0]} x {nwins[1]} windows of {tuple(nwin)} traces, model {dims}, data {tuple(dimsd)}")
    return (nwins, dims, ((m[0], m[0] + int(nop[0])), (m[1], m[1] + int(nop[1])), (0, dims[2])),
            ((st[0], st[0] + int(nwin[0])), (st[1], st[1] + int(nwin[1])), (0, int(dimsd[2]))))


class _Windowed(_KernelOperator):
    """The shared part of the window operators (:class:`Sliding1D`, :class:`Sliding2D`, :class:`Sliding3D`,
    :class:`Patch2D`, :class:`Patch3D`): ``Op``, the chosen apply path and the apply:

    - ``self._fused`` a :class:`Radon2D` / :class:`Radon3D` whose data are a window's: one fused launch
      (``_fused_launch``);
    - any other kernel operator: ``Op``'s own launch per window into a workspace (allocated once per compute dtype),
      and one overlap-add launch (``_fold``) to overlap-add (forward) or cut out (adjoint) the windows."""

    def _check_op(self, Op):
        if not isinstance(Op, _KernelOperator):
            raise TypeError(f"{type(self).__name__}: Op must be a rank-local kernel operator of this package (not a "
                            f"product or an adjoint), got {type(Op).__name__}")

    def _setup(self, Op, dims, dimsd, count, tapertype, name):
        self.Op, self.dims, self.dimsd = Op, dims, dimsd
        self.tapertype, self.name = tapertype, name
        self.shape = (math.prod(dimsd), math.prod(dims))
        self.dtype = Op.dtype
        self._count = count
        self._work = {}
        self._fused = None
        _lib.ctx()

    def _compute_dtype(self, xdt):
        return self.Op._compute_dtype(xdt)

    def _workspace(self, dt):
        if dt not in self._work:
            self._work[dt] = torch.empty(self._count * self.Op.shape[0], dtype=dt, device="cuda")
        return self._work[dt]

    def _launch(self, x, y, dt, adjoint):
        real = _REAL_OF.get(dt, dt)
        cplx = 2 if dt.is_complex else 1
        if self._fused is not None:
            self._fused_launch(x, y, real, cplx, adjoint)
            return
        work = self._workspace(dt)
        nm, nd = self.Op.shape[1], self.Op.shape[0]
        if adjoint:
            self._fold(x, work, real, cplx, 1)
        for w in range(self._count):
            if adjoint:
                self.Op._launch(work[w * nd:(w + 1) * nd], y[w * nm:(w + 1) * nm], dt, 1)
            else:
                self.Op._launch(x[w * nm:(w + 1) * nm], work[w * nd:(w + 1) * nd], dt, 0)
        if not adjoint:
            self._fold(work, y, real, cplx, 0)


class _Sliding(_Windowed):
    """The shared part of :class:`Sliding2D` / :class:`Sliding3D`: a section ``(n0, n1, inner)`` holding the grid of
    ``nwins0 x nwins1`` windows of ``nwin0 x nwin1`` traces (Sliding2D: ``n0 = nwin0 = 1``), the per-window taper
    table ``[nwins][nwin0][nwin1]`` (uploaded once per real dtype, rounded to the inner operator's dtype as pylops'
    ``Diagonal(taper, dtype=Op.dtype)`` rounds it); the fused launch is b2_radon_windows, the overlap-add
    b2_sliding."""

    def _setup(self, Op, dims, dimsd, section, nwins, nwin, steps, t0, t1, tapertype, name):
        super()._setup(Op, dims, dimsd, nwins[0] * nwins[1], tapertype, name)
        self._section, self._nwins, self._nwin, self._steps = section, nwins, nwin, steps
        self._taps = None
        if tapertype is not None:
            real = np.finfo(np.dtype(Op.dtype)).dtype
            table = (t0[:, None, :, None] * t1[None, :, None, :]).reshape(self._count, *nwin).astype(real)
            self._taps = {t: torch.as_tensor(np.ascontiguousarray(table, dtype=_lib.numpy_dtype(t))).to("cuda")
                          for t in (torch.float32, torch.float64)}
        if isinstance(Op, _Radon):
            nhy, nhx, npy, npx = Op._geom[:4]
            if (nhy, nhx) == tuple(nwin) and section[2] == Op._nt:
                self._fused = Op

    def _tap_ptr(self, real):
        return None if self._taps is None else self._taps[real].data_ptr()

    def _fused_launch(self, x, y, real, cplx, adjoint):
        (n0, n1, _), (nw0, nw1), (s0, s1) = self._section, self._nwins, self._steps
        R = self._fused
        nhy, nhx, npy, npx, hy, hx, py, px, kind, interp = R._geom
        _lib.check(_lib.lib.b2_radon_windows(_lib.ctx(), x.data_ptr(), y.data_ptr(), R._nt, cplx, n0, n1, nhy, nhx,
                                             npy, npx, hy, hx, py, px, kind, interp, nw0, nw1, s0, s1,
                                             self._tap_ptr(real), adjoint, _lib.code(real), _lib.stream()),
                   "b2_radon_windows")

    def _fold(self, src, dst, real, cplx, adjoint):
        (n0, n1, inner), (nw0, nw1), (l0, l1), (s0, s1) = self._section, self._nwins, self._nwin, self._steps
        _lib.check(_lib.lib.b2_sliding(_lib.ctx(), src.data_ptr(), dst.data_ptr(), n0, n1, inner, cplx, nw0, nw1, l0,
                                       l1, s0, s1, self._tap_ptr(real), adjoint, _lib.code(real), _lib.stream()),
                   "b2_sliding")


class Sliding2D(_Sliding):
    """Rank-local sliding windows along axis 0 of a section, pylops.signalprocessing.Sliding2D (pylops 2.x as
    remembered: pylops is not installed here to check it) inside MPIBlockDiag: local slant-stack denoising, slope
    decomposition and interpolation with ``Op`` a :class:`Radon2D` applied to every window.  The data are
    ``dimsd = (n, nt)``; windows of ``nwin`` traces start every ``nwin - nover`` traces (``arange(0, n - nwin + 1,
    nwin - nover)``, so traces past the last window are 0 in the forward and ignored in the adjoint).  ``Op`` maps a
    window's model of ``nop`` values to its ``(nwin, nt)`` data; the model is ``dims = (nwins * nop[0], nop[1])``,
    window ``w``'s block contiguous (:func:`sliding2d_design` sizes it)::

        y = sum over w ascending of R_w^T (tap_w * Op x_w),     x_w = Op^H (tap_w * R_w d)

    with ``tap_w`` pylops' ``taper2d(nt, nwin, nover, tapertype)`` (hanning, cosine, cosinesquare or None), the first
    window's leading and the last window's trailing ``nover`` samples set to 1 (one window: the trailing ones only),
    rounded to ``Op``'s dtype.  Every product and sum of the overlap-add is in the data's type, in that order.

    ``Op`` is a kernel operator of this package; a :class:`Radon2D` whose ``(nh, nt)`` data are a window's is applied
    to every window in one b2_radon_windows launch (csrc/radon.cu), equal bit for bit to the per-window route; any other runs
    its own launch per window, then one b2_sliding launch (csrc/sliding.cu).  Dtype rules, ``out=`` and complex data
    are ``Op``'s.  ``TypeError`` for any other ``Op`` (products and ``.H`` included); ``ValueError`` for ``nwin > n``,
    ``nover`` outside ``[0, nwin)``, ``dims`` other than ``(nwins * nop[0], nop[1])``, an ``Op`` whose data are not
    ``nwin * nt`` values and a hanning ``nover`` above ``nwin / 2``."""

    def __init__(self, Op, dims, dimsd, nwin, nover, tapertype="hanning", name="S"):
        self._check_op(Op)
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        if len(dims) != 2 or len(dimsd) != 2:
            raise ValueError(f"dims and dimsd must hold two entries; got {dims}, {dimsd}")
        self.nwin, self.nover = int(nwin), int(nover)
        starts = _slidingsteps(dimsd[0], self.nwin, self.nover)
        nwins = len(starts)
        if nwins * Op.shape[1] // dims[1] != dims[0]:
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                             f"sliding2d_design to identify the correct number of windows for the current model size...")
        if Op.shape[0] != self.nwin * dimsd[1]:
            raise ValueError(f"Op has {Op.shape[0]} data values; a window has {self.nwin} x {dimsd[1]}")
        t1 = _axis_tapers(nwins, self.nwin, self.nover, tapertype, lambda t: 1.0)
        self._setup(Op, dims, dimsd, (1, dimsd[0], dimsd[1]), (1, nwins), (1, self.nwin),
                    (1, self.nwin - self.nover), np.ones((1, 1)), t1, tapertype, name)


class Sliding3D(_Sliding):
    """Rank-local sliding windows over axes 0 and 1 of a volume, pylops.signalprocessing.Sliding3D (pylops 2.x as
    remembered) inside MPIBlockDiag: local 3-D slant-stack processing with ``Op`` a :class:`Radon3D`.  The data are
    ``dimsd = (n0, n1, nt)``; windows of ``nwin = (nwin0, nwin1)`` traces overlap by ``nover = (nover0, nover1)`` and
    form a grid, window ``w = i0 * nwins1 + i1``.  ``Op`` maps ``nop`` model values to a window's
    ``(nwin0, nwin1, nt)`` data; the model is ``dims = (nwins0 * nop[0], nwins1 * nop[1], nop[2])`` stored
    window-major, as BlockDiag orders its blocks (:func:`sliding3d_design` sizes it).  Each trace sums, for each i0
    ascending, the sum over i1 ascending of its windows' ``tap_w * Op x_w``; the tapers are pylops'
    ``taper3d(nt, nwin, nover, tapertype)``, with the outer ``nover`` rows / columns of the edge windows set to the
    taper's middle value (one window along an axis: the trailing ones only).  Apply paths, dtypes and errors as in
    :class:`Sliding2D` (a :class:`Radon3D` whose traces are a window's takes one b2_radon_windows launch), plus
    ``ValueError`` for ``dims`` other than the above; ``nproc`` is accepted and ignored."""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", nproc=1, name="P"):
        self._check_op(Op)
        dims, dimsd = tuple(int(d) for d in dims), tuple(int(d) for d in dimsd)
        self.nwin, self.nover = tuple(int(v) for v in nwin), tuple(int(v) for v in nover)
        self.nop, self.nproc = tuple(int(v) for v in nop), nproc
        if len(dims) != 3 or len(dimsd) != 3 or len(self.nwin) != 2 or len(self.nover) != 2 or len(self.nop) != 3:
            raise ValueError(f"dims, dimsd and nop must hold three entries, nwin and nover two; got {dims}, {dimsd}, "
                             f"{nop}, {nwin}, {nover}")
        st = [_slidingsteps(dimsd[a], self.nwin[a], self.nover[a]) for a in (0, 1)]
        nwins = (len(st[0]), len(st[1]))
        if nwins[0] * self.nop[0] != dims[0] or nwins[1] * self.nop[1] != dims[1] or self.nop[2] != dims[2]:
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                             f"sliding3d_design to identify the correct number of windows for the current model size...")
        if Op.shape[1] != math.prod(self.nop):
            raise ValueError(f"Op has {Op.shape[1]} model values; nop is {self.nop}")
        if Op.shape[0] != self.nwin[0] * self.nwin[1] * dimsd[2]:
            raise ValueError(f"Op has {Op.shape[0]} data values; a window has {self.nwin[0]} x {self.nwin[1]} x "
                             f"{dimsd[2]}")
        t0, t1 = (_axis_tapers(nwins[a], self.nwin[a], self.nover[a], tapertype, lambda t: t[len(t) // 2])
                  for a in (0, 1))
        self._setup(Op, dims, dimsd, dimsd, nwins, self.nwin, (self.nwin[0] - self.nover[0],
                    self.nwin[1] - self.nover[1]), t0, t1, tapertype, name)


def _window_design(dimsd, nwin, nover, nop):
    """``(nwins, dims, mwins_inends, dwins_inends)`` of windows ``nwin`` overlapping by ``nover`` along the leading
    ``len(nwin)`` axes of ``dimsd``, each window's model ``nop``, window-major"""
    st = [_slidingsteps(int(dimsd[a]), int(nwin[a]), int(nover[a])) for a in range(len(nwin))]
    nwins = tuple(len(s) for s in st)
    dims = tuple(nw * int(n) for nw, n in zip(nwins, nop))
    m = [np.arange(nw) * int(n) for nw, n in zip(nwins, nop)]
    return (nwins, dims, tuple((mi, mi + int(n)) for mi, n in zip(m, nop)),
            tuple((si, si + int(n)) for si, n in zip(st, nwin)))


def sliding1d_design(dimd, nwin, nover, nop, verb=False):
    """pylops.signalprocessing.sliding1d_design: ``(nwins, dim, mwin_inends, dwin_inends)`` of a :class:`Sliding1D`
    on a signal of ``dimd`` samples with windows of ``nwin`` samples overlapping by ``nover`` and an inner operator of
    ``nop`` model values: ``dim = nwins * nop``.  Host only."""
    nwins, dims, m, d = _window_design((dimd,), (nwin,), (nover,), (nop,))
    if verb:
        print(f"{nwins[0]} windows of {nwin} samples, model {dims[0]}, data {dimd}")
    return nwins[0], dims[0], m[0], d[0]


def patch2d_design(dimsd, nwin, nover, nop, verb=False):
    """pylops.signalprocessing.patch2d_design: ``(nwins, dims, mwins_inends, dwins_inends)`` of a :class:`Patch2D`
    on data ``dimsd = (n, nt)`` with patches ``nwin = (nwin0, nwin1)`` overlapping by ``nover`` and an inner operator
    of model ``nop``: ``nwins = (nwins0, nwins1)``, ``dims = (nwins0 * nop[0], nwins1 * nop[1])``.  Host only."""
    out = _window_design(dimsd, nwin, nover, nop)
    if verb:
        print(f"{out[0][0]} x {out[0][1]} patches of {tuple(nwin)}, model {out[1]}, data {tuple(dimsd)}")
    return out


def patch3d_design(dimsd, nwin, nover, nop, verb=False):
    """pylops.signalprocessing.patch3d_design: as :func:`patch2d_design` on data ``dimsd = (ny, nx, nt)`` with three
    window axes: ``nwins = (nwins0, nwins1, nwins2)``, ``dims = (nwins0 * nop[0], nwins1 * nop[1], nwins2 * nop[2])``.
    Host only."""
    out = _window_design(dimsd, nwin, nover, nop)
    if verb:
        print(f"{' x '.join(map(str, out[0]))} patches of {tuple(nwin)}, model {out[1]}, data {tuple(dimsd)}")
    return out


def _patch_tapers(nwins, nwin, nover, tapertype):
    """the float64 per-axis tapers ``[nwins_a][nwin_a]`` of b2_patch's three window axes (an axis with no windows:
    None; all None for ``tapertype=None``), the one statement of pylops' taper rules as remembered:

    - one axis (Sliding1D): ``taper(nwin, nover)``, the first window's leading and the last window's trailing
      ``nover`` samples set to 1;
    - two axes (Patch2D): ``taper2d(nwin[1], nwin[0], nover)``, the outer product of the two axis tapers, with the
      edge patches' outer ``nover`` rows / columns replaced by the middle row / column;
    - three axes (Patch3D): ``taper3d(nwin[2], nwin[:2], nover[:2])``, tapered along y and x and constant along t,
      with the same edge rule on all three axes (a no-op along t).

    An edge replacement by the middle value is, per axis, ``t[:nover] = t[nwin // 2]`` for the first window and
    ``t[nwin - nover:] = t[nwin // 2]`` for the last (one window: the last only), so the product of the axis tables
    is pylops' full taper bit for bit."""
    if tapertype is None:
        return [None, None, None]
    mid = lambda t: t[len(t) // 2]                                   # noqa: E731
    if len(nwin) == 1:
        return [None, None, _axis_tapers(nwins[0], nwin[0], nover[0], tapertype, lambda t: 1.0)]
    taps = [_axis_tapers(nwins[a], nwin[a], nover[a], tapertype, mid) for a in range(2)]
    if len(nwin) == 2:
        return [None] + taps
    return taps + [_axis_tapers(nwins[2], nwin[2], nover[2], None, mid)]


class _Patch(_Windowed):
    """The shared part of :class:`Sliding1D` / :class:`Patch2D` / :class:`Patch3D`: a section ``(n0, n1, nt)`` (each
    sample ``n_inner`` values) holding ``nwins0 x nwins1 x nwins2`` windows of ``nwin0 x nwin1`` traces and ``nwin2``
    samples, window ``w = (i0 * nwins1 + i1) * nwins2 + i2`` (Patch2D: ``n0 = 1``; Sliding1D: ``n0 = n1 = 1``), and
    the float64 per-axis tapers of :func:`_patch_tapers`, uploaded once; the fused launch is b2_radon_patches, the
    overlap-add b2_patch.  Each window's taper is formed on the device from the axis tapers and rounded once to the
    data's real dtype."""

    def _setup(self, Op, dims, dimsd, section, nwins, nwin, nover, tapertype, scalings, name):
        if scalings is not None:
            raise NotImplementedError(f"{type(self).__name__}: scalings={scalings!r} is not supported (None only)")
        model = math.prod(nwins) * Op.shape[1]
        if math.prod(dims) != model:
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows. Run "
                             f"{type(self).__name__.lower()}_design to identify the correct number of windows for the "
                             f"current model size...")
        if Op.shape[0] != math.prod(nwin):
            raise ValueError(f"Op has {Op.shape[0]} data values; a window has {' x '.join(map(str, nwin))}")
        k = 3 - len(nwin)
        taps = _patch_tapers(nwins, nwin, nover, tapertype)
        super()._setup(Op, dims, dimsd, math.prod(nwins), tapertype, name)
        self._section = (1,) * k + tuple(section)
        self._nwins = (1,) * k + tuple(nwins)
        self._nwin = (1,) * k + tuple(nwin)
        self._steps = (1,) * k + tuple(w - o for w, o in zip(nwin, nover))
        self._taps = [None if t is None else torch.as_tensor(np.ascontiguousarray(t, dtype=np.float64)).to("cuda")
                      for t in taps]

    def _fuse(self, Op):
        """take the fused path when ``Op`` is a Radon whose traces and samples are a window's"""
        if isinstance(Op, _Radon) and tuple(Op._geom[:2]) + (Op._nt,) == self._nwin:
            self._fused = Op

    def _tap_ptrs(self):
        return [_lib.ptr(t) for t in self._taps]

    def _fused_launch(self, x, y, real, cplx, adjoint):
        (n0, n1, ns), (nw0, nw1, nw2), (s0, s1, s2) = self._section, self._nwins, self._steps
        R = self._fused
        nhy, nhx, npy, npx, hy, hx, py, px, kind, interp = R._geom
        _lib.check(_lib.lib.b2_radon_patches(_lib.ctx(), x.data_ptr(), y.data_ptr(), R._nt, cplx, n0, n1, ns, nhy,
                                             nhx, npy, npx, hy, hx, py, px, kind, interp, nw0, nw1, nw2, s0, s1, s2,
                                             *self._tap_ptrs(), adjoint, _lib.code(real), _lib.stream()),
                   "b2_radon_patches")

    def _fold(self, src, dst, real, cplx, adjoint):
        (n0, n1, nt), (nw0, nw1, nw2), (l0, l1, l2), (s0, s1, s2) = (self._section, self._nwins, self._nwin,
                                                                      self._steps)
        _lib.check(_lib.lib.b2_patch(_lib.ctx(), src.data_ptr(), dst.data_ptr(), n0, n1, nt, cplx, nw0, nw1, nw2, l0,
                                     l1, l2, s0, s1, s2, *self._tap_ptrs(), adjoint, _lib.code(real),
                                     _lib.stream()), "b2_patch")


def _ints(name, v, n):
    v = tuple(int(a) for a in (v if np.ndim(v) else (v,)))
    if len(v) != n:
        raise ValueError(f"{name} must hold {n} entries; got {v}")
    return v


class Sliding1D(_Patch):
    """Rank-local sliding windows along a 1-D signal, pylops.signalprocessing.Sliding1D (pylops 2.x as remembered:
    pylops is not installed here to check it) inside MPIBlockDiag.  Windows of ``nwin`` samples start every
    ``nwin - nover`` samples of the ``dimd`` data samples (samples past the last window are 0 in the forward and
    ignored in the adjoint).  ``Op`` maps a window's model of ``nop`` values to its ``nwin`` samples; the model is
    ``dim = nwins * nop``, window ``w``'s block contiguous (:func:`sliding1d_design` sizes it)::

        y = sum over w ascending of R_w^T (tap_w * Op x_w),     x_w = Op^H (tap_w * R_w d)

    with ``tap_w`` pylops' ``taper(nwin, nover, tapertype)`` (hanning, cosine, cosinesquare or None), the first
    window's leading and the last window's trailing ``nover`` samples set to 1 (one window: the trailing ones only),
    rounded to the data's real dtype.  ``Op`` is a kernel operator of this package, applied by its own launch per
    window, then one b2_patch launch (csrc/sliding.cu).  Dtype rules, ``out=`` and complex data are ``Op``'s.
    ``TypeError`` for any other ``Op`` (products and ``.H`` included); ``ValueError`` for ``nwin > dimd``, ``nover``
    outside ``[0, nwin)``, ``dim`` other than ``nwins * nop``, an ``Op`` whose data are not ``nwin`` values and a
    hanning ``nover`` above ``nwin / 2``."""

    def __init__(self, Op, dim, dimd, nwin, nover, tapertype="hanning", name="S"):
        self._check_op(Op)
        dim, dimd = _ints("dim", dim, 1), _ints("dimd", dimd, 1)
        self.nwin, self.nover = int(nwin), int(nover)
        nwins = len(_slidingsteps(dimd[0], self.nwin, self.nover))
        self._setup(Op, dim, dimd, (dimd[0],), (nwins,), (self.nwin,), (self.nover,), tapertype, None, name)


class Patch2D(_Patch):
    """Rank-local time-space patches of a section, pylops.signalprocessing.Patch2D (pylops 2.x as remembered: pylops
    is not installed here to check it) inside MPIBlockDiag: local Radon (slope) denoising and interpolation of curved
    events, with ``Op`` a :class:`Radon2D` applied to every patch.  The data are ``dimsd = (n, nt)``; patches of
    ``nwin = (nwin0, nwin1)`` (traces, samples) overlap by ``nover`` and form a grid, patch ``w = i0 * nwins1 + i1``
    starting at ``(i0 * (nwin0 - nover0), i1 * (nwin1 - nover1))`` (traces and samples past the last patch are 0 in
    the forward and ignored in the adjoint).  ``Op`` maps ``nop`` model values to a patch's ``(nwin0, nwin1)`` data;
    the model is ``dims = (nwins0 * nop[0], nwins1 * nop[1])`` stored window-major, as BlockDiag orders its blocks
    (:func:`patch2d_design` sizes it).  Each sample sums, over i0 ascending, the sum over i1 ascending of its patches'
    ``tap_w * Op x_w``; the tapers are pylops' ``taper2d(nwin1, nwin0, nover, tapertype)``, the outer product of the
    two axis tapers, with the edge patches' outer ``nover`` rows / columns replaced by the taper's middle row /
    column (one patch along an axis: the trailing ones only), rounded to the data's real dtype.

    ``Op`` is a kernel operator of this package; a :class:`Radon2D` whose ``(nh, nt)`` data are a patch's is applied to
    every patch in one b2_radon_patches launch (csrc/radon.cu), equal bit for bit to the per-patch route; any other runs
    its own launch per patch, then one b2_patch launch (csrc/sliding.cu).  Dtype rules, ``out=`` and complex data are
    ``Op``'s.  ``TypeError`` for any other ``Op`` (products and ``.H`` included); ``NotImplementedError`` for
    ``scalings`` other than None; ``ValueError`` for ``nwin > n``, ``nover`` outside ``[0, nwin)``, ``dims`` other than
    the above, an ``Op`` whose model / data are not ``nop`` / a patch and a hanning ``nover`` above ``nwin / 2``."""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P"):
        self._check_op(Op)
        dims, dimsd = _ints("dims", dims, 2), _ints("dimsd", dimsd, 2)
        self.nwin, self.nover, self.nop = _ints("nwin", nwin, 2), _ints("nover", nover, 2), _ints("nop", nop, 2)
        self.scalings = scalings
        nwins = tuple(len(_slidingsteps(dimsd[a], self.nwin[a], self.nover[a])) for a in (0, 1))
        if Op.shape[1] != math.prod(self.nop) or dims != tuple(w * n for w, n in zip(nwins, self.nop)):
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows and Op's "
                             f"model of {Op.shape[1]} values (nop={self.nop}). Run patch2d_design to identify the "
                             f"correct number of windows for the current model size...")
        self._setup(Op, dims, dimsd, dimsd, nwins, self.nwin, self.nover, tapertype, scalings, name)
        self._fuse(Op)


class Patch3D(_Patch):
    """Rank-local time-space patches of a volume, pylops.signalprocessing.Patch3D (pylops 2.x as remembered) inside
    MPIBlockDiag: local 3-D Radon processing with ``Op`` a :class:`Radon3D`.  As :class:`Patch2D` over data
    ``dimsd = (ny, nx, nt)`` with three window axes: patches ``nwin = (nwin0, nwin1, nwin2)`` overlapping by ``nover``,
    patch ``w = (i0 * nwins1 + i1) * nwins2 + i2``, model ``dims = (nwins0 * nop[0], nwins1 * nop[1], nwins2 * nop[2])``
    window-major (:func:`patch3d_design` sizes it), each sample summed over i0, of i1, of i2, all ascending.  The tapers
    are pylops' ``taper3d(nwin2, nwin[:2], nover[:2], tapertype)``: tapered along y and x, constant along t, with the
    edge rule on all three axes (a no-op along t).  A :class:`Radon3D` whose data are a patch's takes one
    b2_radon_patches launch.  Apply paths, dtypes and errors as in :class:`Patch2D`."""

    def __init__(self, Op, dims, dimsd, nwin, nover, nop, tapertype="hanning", scalings=None, name="P"):
        self._check_op(Op)
        dims, dimsd = _ints("dims", dims, 3), _ints("dimsd", dimsd, 3)
        self.nwin, self.nover, self.nop = _ints("nwin", nwin, 3), _ints("nover", nover, 3), _ints("nop", nop, 3)
        self.scalings = scalings
        nwins = tuple(len(_slidingsteps(dimsd[a], self.nwin[a], self.nover[a])) for a in (0, 1, 2))
        if Op.shape[1] != math.prod(self.nop) or dims != tuple(w * n for w, n in zip(nwins, self.nop)):
            raise ValueError(f"Model shape (dims={dims}) is not consistent with chosen number of windows and Op's "
                             f"model of {Op.shape[1]} values (nop={self.nop}). Run patch3d_design to identify the "
                             f"correct number of windows for the current model size...")
        self._setup(Op, dims, dimsd, dimsd, nwins, self.nwin, self.nover, tapertype, scalings, name)
        self._fuse(Op)


class FFT(LocalOperator):
    """Rank-local real FFT along ``axis`` of a ``dims`` block -- the role of third-party
    ``pylops.signalprocessing.FFT(dims, axis, real=True, ifftshift_before=..., norm="ortho")`` inside
    MPIMDC (waveeqprocessing/MDC.py:55-58).  cuFFT through ``torch.fft`` (library plumbing, not a
    hot-path kernel: the FFTs are rank-replicated pre/post-processing around MPIFredholm1).
    pylops is absent from this image: the scaling convention restated here (orthonormal transform, positive
    frequencies scaled by sqrt(2) so that the adjoint of the one-sided transform is exact) follows pylops 2.x;
    it is checked through the MPIMDC fixtures (reference chain over the same restatement in NumPy)."""

    def __init__(self, dims, axis: int = 0, real: bool = True, ifftshift_before: bool = False, dtype=np.float64):
        if not real:
            raise NotImplementedError("only the real (one-sided) transform used by MDC is provided")
        self.dims = tuple(int(d) for d in dims)
        self.axis = axis % len(self.dims)
        self.nfft = self.dims[self.axis]
        self.nfo = self.nfft // 2 + 1
        self.dimsd = self.dims[:self.axis] + (self.nfo,) + self.dims[self.axis + 1:]
        self.shape = (int(np.prod(self.dimsd)), int(np.prod(self.dims)))
        self.ifftshift_before = ifftshift_before
        self.rdtype = _lib.torch_dtype(dtype)
        self.cdtype = {torch.float32: torch.complex64, torch.float64: torch.complex128}[self.rdtype]
        self.dtype = _lib.numpy_dtype(self.cdtype)
        self._npos = (self.nfft - 1) // 2          # bins 1 .. npos are "doubled" positive frequencies

    def _sl(self, lo, hi):
        s = [slice(None)] * len(self.dims)
        s[self.axis] = slice(lo, hi)
        return tuple(s)

    def _scale_band(self, out: torch.Tensor, src: torch.Tensor, a: float):
        """out = src with the positive-frequency band (bins 1 .. npos along ``axis``) scaled by ``a`` -- through
        b2_lincomb (copy + in-band scale: at most three launches, no eager torch elementwise pass)"""
        one = _lib.cpair(1.0)
        code = _lib.code(src.dtype)
        ctx, st = _lib.ctx(), _lib.stream()
        if self.axis == 0 and self._npos > 0 and src.is_contiguous():
            inner = int(np.prod(self.dimsd[1:])) if len(self.dimsd) > 1 else 1
            so, ss = out.reshape(-1), src.reshape(-1)
            lo, hi = inner, (1 + self._npos) * inner
            for b, e, coef in ((0, lo, 1.0), (lo, hi, a), (hi, ss.numel(), 1.0)):
                if e > b and (coef != 1.0 or so.data_ptr() != ss.data_ptr()):
                    _lib.check(_lib.lib.b2_lincomb(ctx, so[b:].data_ptr(), _lib.cpair(coef), ss[b:].data_ptr(), None, None,
                                                   e - b, code, 0, st), "b2_lincomb")
            return out
        if out.data_ptr() != src.data_ptr():
            out.copy_(src)
        out[self._sl(1, 1 + self._npos)] *= a
        return out

    def _matvec(self, x: torch.Tensor) -> torch.Tensor:
        x = x.reshape(self.dims)
        x = x.real if x.is_complex() else x
        x = x.to(self.rdtype)
        if self.ifftshift_before:
            x = torch.fft.ifftshift(x, dim=self.axis)
        y = torch.fft.rfft(x, n=self.nfft, dim=self.axis, norm="ortho")
        return self._scale_band(y, y, float(np.sqrt(2.0))).reshape(-1)

    def _rmatvec(self, x: torch.Tensor) -> torch.Tensor:
        x = x.reshape(self.dimsd)
        if x.dtype != self.cdtype:
            x = x.to(self.cdtype)
        xs = self._scale_band(torch.empty_like(x, memory_format=torch.contiguous_format), x.contiguous(),
                              float(1.0 / np.sqrt(2.0)))
        y = torch.fft.irfft(xs, n=self.nfft, dim=self.axis, norm="ortho")
        if self.ifftshift_before:
            y = torch.fft.fftshift(y, dim=self.axis)
        return y.reshape(-1)


class Identity(LocalOperator):
    """``pylops.Identity(N, M)``: keep the first N of M samples (adjoint: zero-pad) -- the frequency
    truncation of MDC (MDC.py:61-64)."""

    def __init__(self, N: int, M: int = None, dtype=np.float64):
        M = N if M is None else M
        self.shape = (int(N), int(M))
        self.dtype = _lib.numpy_dtype(_lib.torch_dtype(dtype))

    @staticmethod
    def _pad(x: torch.Tensor, n: int) -> torch.Tensor:
        """zero-padded copy of flat ``x`` to ``n`` elements: b2_lincomb (copy) + b2_fill (tail)"""
        x = x.reshape(-1).contiguous()
        y = torch.empty(n, dtype=x.dtype, device=x.device)
        code, ctx, st = _lib.code(x.dtype), _lib.ctx(), _lib.stream()
        if x.numel():
            _lib.check(_lib.lib.b2_lincomb(ctx, y.data_ptr(), _lib.cpair(1.0), x.data_ptr(), None, None, x.numel(), code, 0, st),
                       "b2_lincomb")
        if n > x.numel():
            _lib.check(_lib.lib.b2_fill(ctx, y[x.numel():].data_ptr(), _lib.cpair(0.0), n - x.numel(), code, st), "b2_fill")
        return y

    def _matvec(self, x: torch.Tensor) -> torch.Tensor:
        N, M = self.shape
        return x[:N] if N <= M else self._pad(x, N)

    def _rmatvec(self, x: torch.Tensor) -> torch.Tensor:
        N, M = self.shape
        return x[:M] if M <= N else self._pad(x, M)
