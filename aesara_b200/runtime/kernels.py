"""Launch wrappers: IR-level operations -> C-ABI calls on DeviceArrays."""

from __future__ import annotations

import collections
import ctypes as C
import os

import numpy as np
import torch

from ..codegen.careduce import careduce_source
from ..codegen.elemwise import elemwise_source
from ..ir import DTYPE_CODE
from . import lib as _lib
from .device import DeviceArray, stream_handle


class ElemwiseKernel:
    """One fused ``Elemwise{Composite}`` module (compiled on first use)."""

    _by_key = {}

    def __init__(self, expr):
        self.expr = expr
        self.src, self.meta = elemwise_source(expr)
        self.n_in = self.meta["n_in"]
        self.n_out = self.meta["n_out"]
        self.out_dtypes = [np.dtype(d) for d in expr["out_dtypes"]]
        self.in_dtypes = [np.dtype(d) for d in expr["inputs"]]
        self._handle = None
        nops = self.n_in + self.n_out
        self._itemsizes = (C.c_int32 * nops)(*self.meta["itemsizes"])
        self._ptrs = (C.c_void_p * nops)()

    @classmethod
    def get(cls, expr):
        import json

        key = json.dumps(expr, sort_keys=True, default=str)
        k = cls._by_key.get(key)
        if k is None:
            k = cls._by_key[key] = cls(expr)
        return k

    def compile(self):
        """NVRTC-compile (disk cached); does not need a GPU."""
        return _lib.compile_cubin(self.src, "ew")

    def handle(self):
        if self._handle is None:
            self._handle = _lib.load_module(self.src, "ew")
        return self._handle

    def launch(self, shape, ins, outs):
        """ins/outs: DeviceArrays already broadcast-compatible with ``shape``
        (inputs may have size-1 dims where ``shape`` is larger)."""
        nd = len(shape)
        nops = self.n_in + self.n_out
        shp = (C.c_int64 * max(nd, 1))(*shape)
        strides = (C.c_int64 * max(nops * nd, 1))()
        k = 0
        for a in ins:
            self._ptrs[k] = a.ptr
            for d in range(nd):
                strides[k * nd + d] = 0 if a.shape[d] == 1 else a.strides[d]
            k += 1
        for a in outs:
            self._ptrs[k] = a.ptr
            for d in range(nd):
                strides[k * nd + d] = a.strides[d]
            k += 1
        lib = _lib.load()
        _lib.check(lib.ab_elemwise_launch(self.handle(), self.n_in, self.n_out, nd, shp,
                                          self._ptrs, strides, self._itemsizes,
                                          self.meta["vec"], self.meta["unroll"],
                                          stream_handle()))


def broadcast_shape(arrays, what="Elemwise"):
    """Run-time broadcast rule of ``elemwise_cgen.py:72-125``."""
    nd = arrays[0].ndim
    out = []
    for d in range(nd):
        n = 1
        for a in arrays:
            s = a.shape[d]
            if s != 1:
                if n != 1 and s != n:
                    raise ValueError(
                        f"Input dimension mismatch. (input[?].shape[{d}] = {s}, "
                        f"expected {n}) in {what}"
                    )
                n = s
        # a zero-size input makes the output zero-size
        if any(a.shape[d] == 0 for a in arrays):
            n = 0
        out.append(n)
    return tuple(out)


def elemwise_out_order(ins, shape):
    """Output layout rule of ``aesara/tensor/elemwise.py:912-925``: Fortran
    order iff every non-scalar input is F- but not C-contiguous."""
    big = [a for a in ins if a.size > 1 and a.ndim > 1]
    if big and all(a.is_f_contiguous() and not a.is_c_contiguous() for a in big) and all(
        a.shape == tuple(shape) for a in big
    ):
        return "F"
    return "C"


_IDENTITY = {}


def _identity_kernel(dtype):
    dt = np.dtype(dtype).name
    k = _IDENTITY.get(dt)
    if k is None:
        expr = {"inputs": [dt], "out_dtypes": [dt], "outputs": ["t0"], "name": f"copy_{dt}",
                "stmts": [{"op": "identity", "args": ["i0"], "dtype": dt, "in_dtypes": [dt]}]}
        k = _IDENTITY[dt] = ElemwiseKernel.get(expr)
    return k


def copy_into(dst: DeviceArray, src: DeviceArray):
    """dst[...] = src with NumPy broadcasting of src (strided copy kernel)."""
    if dst.size == 0:
        return
    if src.ndim < dst.ndim:
        src = src.view((1,) * (dst.ndim - src.ndim) + src.shape,
                       (0,) * (dst.ndim - src.ndim) + src.strides)
    if src.ndim != dst.ndim:
        raise ValueError("copy_into: source has more dimensions than destination")
    for d in range(dst.ndim):
        if src.shape[d] not in (1, dst.shape[d]):
            raise ValueError(f"could not broadcast input array from shape {src.shape} into shape {dst.shape}")
    if src.dtype != dst.dtype:
        k = _cast_kernel(src.dtype, dst.dtype)
    else:
        k = _identity_kernel(dst.dtype)
    k.launch(dst.shape, [src], [dst])


_CAST = {}


def _cast_kernel(src_dt, dst_dt):
    s, d = np.dtype(src_dt).name, np.dtype(dst_dt).name
    k = _CAST.get((s, d))
    if k is None:
        expr = {"inputs": [s], "out_dtypes": [d], "outputs": ["t0"], "name": f"cast_{s}_{d}",
                "stmts": [{"op": "cast", "args": ["i0"], "dtype": d, "in_dtypes": [s]}]}
        k = _CAST[(s, d)] = ElemwiseKernel.get(expr)
    return k


def contiguous_copy(a: DeviceArray, order="C") -> DeviceArray:
    out = DeviceArray.empty(a.shape, a.dtype, order=order)
    copy_into(out, a)
    return out


def cast_copy(a: DeviceArray, dtype) -> DeviceArray:
    """A C-contiguous copy of ``a`` in ``dtype`` (C conversion, like ``ndarray.astype``)."""
    out = DeviceArray.empty(a.shape, dtype)
    copy_into(out, a)
    return out


def add_into(dst: DeviceArray, src: DeviceArray):
    """dst[...] += src (IncSubtensor without set_instead_of_inc)."""
    dt = dst.dtype.name
    expr = {"inputs": [dt, src.dtype.name], "out_dtypes": [dt], "outputs": ["t0"],
            "name": f"inc_{dt}",
            "stmts": [{"op": "add", "args": ["i0", "i1"], "dtype": dt,
                       "in_dtypes": [dt, src.dtype.name]}]}
    if src.ndim < dst.ndim:
        src = src.view((1,) * (dst.ndim - src.ndim) + src.shape,
                       (0,) * (dst.ndim - src.ndim) + src.strides)
    ElemwiseKernel.get(expr).launch(dst.shape, [dst, src], [dst])


class CAReduceKernel:
    _by_key = {}

    def __init__(self, scalar_op, in_dtype, acc_dtype, out_dtype, pre_expr=None):
        self.src, self.meta = careduce_source(scalar_op, in_dtype, acc_dtype, out_dtype, pre_expr=pre_expr)
        self.out_dtype = np.dtype(out_dtype)
        self._handle = None

    @classmethod
    def get(cls, scalar_op, in_dtype, acc_dtype, out_dtype, pre_expr=None):
        import json

        key = (scalar_op, str(in_dtype), str(acc_dtype), str(out_dtype),
               json.dumps(pre_expr, sort_keys=True, default=str) if pre_expr is not None else None)
        k = cls._by_key.get(key)
        if k is None:
            k = cls._by_key[key] = cls(scalar_op, str(in_dtype), str(acc_dtype), str(out_dtype), pre_expr)
        return k

    def compile(self):
        return _lib.compile_cubin(self.src, "red")

    def handle(self):
        if self._handle is None:
            self._handle = _lib.load_module(self.src, "red")
        return self._handle

    def launch(self, x: DeviceArray, axis):
        nd = x.ndim
        mask = [1 if d in axis else 0 for d in range(nd)]
        out_shape = tuple(n for d, n in enumerate(x.shape) if not mask[d])
        out = DeviceArray.empty(out_shape, self.out_dtype)
        if out.size == 0:
            return out
        lib = _lib.load()
        shp = (C.c_int64 * max(nd, 1))(*x.shape)
        st = (C.c_int64 * max(nd, 1))(*x.strides)
        msk = (C.c_int32 * max(nd, 1))(*mask)
        ws_bytes = C.c_size_t()
        _lib.check(lib.ab_careduce_workspace_bytes(nd, shp, msk, self.meta["acc_itemsize"],
                                                   C.byref(ws_bytes)))
        ws = torch.empty(max(ws_bytes.value, 1), dtype=torch.uint8, device=x.owner.device)
        _lib.check(lib.ab_careduce_launch(self.handle(), nd, shp, st, msk, x.ptr, out.ptr,
                                          ws.data_ptr(), ws_bytes.value,
                                          self.meta["in_itemsize"], self.meta["acc_itemsize"],
                                          self.meta["out_itemsize"], stream_handle()))
        return out


def _blas_code(dtype):
    dt = np.dtype(dtype).name
    if dt not in ("float32", "float64"):
        raise TypeError(f"BLAS ops accept float32/float64 only, got {dt} (aesara/tensor/blas.py:613-629)")
    return DTYPE_CODE[dt]


def gemv(y: DeviceArray, alpha, A: DeviceArray, x: DeviceArray, beta):
    """In place: y <- beta*y + alpha*A@x."""
    lib = _lib.load()
    m, n = A.shape
    code = _blas_code(y.dtype)
    ws_bytes = C.c_size_t()
    _lib.check(lib.ab_gemv_workspace_bytes(code, m, n, A.strides[0], A.strides[1], C.byref(ws_bytes)))
    ws = torch.empty(max(ws_bytes.value, 1), dtype=torch.uint8, device=A.owner.device)
    _lib.check(lib.ab_gemv(code, m, n, float(alpha), A.ptr, A.strides[0], A.strides[1], x.ptr,
                           x.strides[0], float(beta), y.ptr, y.strides[0], ws.data_ptr(),
                           ws_bytes.value, stream_handle()))


def ger(A: DeviceArray, alpha, x: DeviceArray, y: DeviceArray):
    """In place: A <- A + alpha * outer(x, y)."""
    lib = _lib.load()
    m, n = A.shape
    _lib.check(lib.ab_ger(_blas_code(A.dtype), m, n, float(alpha), x.ptr, x.strides[0], y.ptr,
                          y.strides[0], A.ptr, A.strides[0], A.strides[1], stream_handle()))


class PackCache:
    """Tensor-core operand planes (bf16 / TF32 hi+lo) packed during one program
    evaluation.  Keyed by the source buffer's memory layout, so a matrix and its
    DimShuffle{1,0} view (X and X^T, h and h^T in an MLP backward pass) share one
    pack: the transposed use reads the same planes as an MN-major operand."""

    def __init__(self):
        self._e = {}
        self._unstored = {}

    def clear(self):
        self._e.clear()
        self._unstored.clear()

    def invalidate(self, owner):
        """Drop the packs of a buffer that a destructive (in-place) node just rewrote."""
        if self._e:
            dead = [k for k, e in self._e.items() if e[0]() is owner]
            for k in dead:
                del self._e[k]

    # a matrix that is read with the contraction along its ROWS and has at most this many
    # elements (weights) gets a transposed, K-major plane from a transposing pack; larger ones
    # are read as MN-major operands of their natural plane (the pack would cost more than the
    # tensor-pipe cycles it saves)
    TRANSPOSE_PACK_MAX = 64 * 1024 * 1024

    def never_stored(self, arr: DeviceArray):
        """``arr`` exists as bf16 plane(s) only (its float32 buffer was not written by the
        epilogue that produced it): packing from it would read garbage -- fail loudly."""
        # weak: a strong reference here would keep every evaluation's unwritten [M, N] float32
        # buffer alive (the caching allocator then has to cudaMalloc fresh ones each step)
        self._unstored[arr.ptr] = self._ref(arr.owner)

    def adopt(self, arr: DeviceArray, buf, pitch, transposed=False):
        """Register a bf16 plane written by a fused GEMM epilogue as the pack of ``arr``
        ([rows, k] float32, K-contiguous): the next product reads it without a pack pass.
        ``transposed``: the plane holds ``arr.T`` ([k, pitch] rows): the K-major operand of
        products that contract over the rows of ``arr``."""
        import weakref

        rows, k = arr.shape
        key = (arr.ptr, rows, k, arr.strides[0], 0, 2) + (("T",) if transposed else ())
        try:
            ref = weakref.ref(arr.owner)
        except TypeError:
            ref = (lambda o: (lambda: o))(arr.owner)
        self._e[key] = (ref, buf.data_ptr(), None, pitch, buf)

    @staticmethod
    def _ref(owner):
        import weakref

        try:
            return weakref.ref(owner)
        except TypeError:
            return (lambda o: (lambda: o))(owner)

    def _check_stored(self, arr):
        ref = self._unstored.get(arr.ptr)
        if ref is not None and ref() is arr.owner:
            raise RuntimeError("PackCache: asked to pack a matrix that was kept as a bf16 plane only "
                               "(the fused epilogue did not store its float32 values)")

    def operand(self, arr: DeviceArray, rows, k, s_r, s_k, precision):
        import weakref

        lib = _lib.load()
        # bf16 planes serve both orientations of a matrix (K-major / MN-major operand);
        # TF32 planes are always K-major, so a transposed use is a different pack
        share = precision == 2 and not os.environ.get("AB_GEMM_NO_MN")
        if s_k == 1 or k == 1:
            canon = (arr.ptr, rows, k, s_r, 0)
        elif s_r == 1 and share:
            canon = (arr.ptr, k, rows, s_k, 0)
        else:
            canon = (arr.ptr, rows, k, s_r, s_k)
        key = canon + (precision,)
        mn_use = not (s_k == 1 or k == 1) and s_r == 1 and share
        if mn_use:
            # contraction along the rows of the natural matrix: a transposed plane (written by
            # the epilogue that produced the matrix, or packed here for a small one) is K-major
            tkey = key + ("T",)
            ent = self._e.get(tkey)
            if ent is None and key not in self._e and rows * k <= self.TRANSPOSE_PACK_MAX \
                    and not os.environ.get("AB_GEMM_NO_TPACK"):
                self._check_stored(arr)
                nbytes = C.c_size_t()
                _lib.check(lib.ab_gemm_pack_kmajor_bytes(precision, rows, k, s_r, s_k, C.byref(nbytes)))
                buf = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=arr.owner.device)
                op = _lib.GemmOperand()
                _lib.check(lib.ab_gemm_pack_kmajor(precision, arr.ptr, rows, k, s_r, s_k, buf.data_ptr(),
                                                   nbytes.value, C.byref(op), stream_handle()))
                ent = self._e[tkey] = (self._ref(arr.owner), op.plane0, None, op.pitch, buf)
            if ent is not None and ent[0]() is arr.owner:
                return _lib.GemmOperand(ent[1], None, rows, k, ent[3], 0, precision)
        ent = self._e.get(key)
        if ent is not None and ent[0]() is arr.owner:
            _, p0, p1, pitch, _buf = ent
        else:
            self._check_stored(arr)
            nbytes = C.c_size_t()
            _lib.check(lib.ab_gemm_pack_bytes(precision, rows, k, s_r, s_k, C.byref(nbytes)))
            buf = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=arr.owner.device)
            op = _lib.GemmOperand()
            _lib.check(lib.ab_gemm_pack(precision, arr.ptr, rows, k, s_r, s_k, buf.data_ptr(),
                                        nbytes.value, C.byref(op), stream_handle()))
            p0, p1, pitch = op.plane0, op.plane1, op.pitch
            try:
                ref = weakref.ref(arr.owner)
            except TypeError:
                ref = (lambda o: (lambda: o))(arr.owner)
            self._e[key] = (ref, p0, p1, pitch, buf)
        mn = 0 if (s_k == 1 or k == 1) else (1 if (s_r == 1 and share) else 0)
        return _lib.GemmOperand(p0, p1, rows, k, pitch, mn, precision)


# tensor-core GEMM launches made through ``gemm``, keyed by (fused, precision, a_mn, b_mn): the
# operand layouts select the MMA loop (ahead-of-time kernels) or the entry point (fused modules),
# so tests can tell which of them ran.  CUDA-graph replays do not pass through here.
TC_LAUNCHES = collections.Counter()


def gemm(C_: DeviceArray, alpha, A: DeviceArray, B: DeviceArray, beta, precision=0, cache=None,
         cin: DeviceArray = None, epilogue=None):
    """C <- beta*Cin + alpha*A@B (Cin = C, i.e. in place, unless ``cin`` is given).
    ``epilogue`` (a ``gemmfuse.EpilogueRequest``) asks for the fused variant: C <- f(that,
    operands); it is marked ``applied`` only if the tensor-core path took it."""
    lib = _lib.load()
    m, k = A.shape
    k2, n = B.shape
    code = _blas_code(C_.dtype)
    if C_.dtype == np.float32 and lib.ab_gemm_tensorcore_eligible(m, n, k):
        cache = cache if cache is not None else PackCache()
        opa = cache.operand(A, m, k, A.strides[0], A.strides[1], precision)
        opb = cache.operand(B, n, k, B.strides[1], B.strides[0], precision)
        TC_LAUNCHES[(epilogue is not None, precision, opa.mn_major, opb.mn_major)] += 1
        cin_args = (None, 0, 0) if cin is None else (cin.ptr, cin.strides[0], cin.strides[1])
        if epilogue is not None:
            if cin is None:
                # in place (C_ holds z): value 0 may be kept as a bf16 plane only, with C left
                # unwritten, so beta*z is read through C_in
                cin_args = (C_.ptr, C_.strides[0], C_.strides[1])
            ep = _lib.GemmEpilogue()
            ep.module = epilogue.fusion.handle()
            ep.n_operands = len(epilogue.operands)
            for i, a in enumerate(epilogue.operands):
                ep.ptr[i] = a.ptr
                ep.rs[i] = 0 if a.shape[0] == 1 else a.strides[0]
                ep.cs[i] = 0 if a.shape[1] == 1 else a.strides[1]
            plan = epilogue.out_plan
            ep.n_outputs = len(plan)
            arrays, shadows, tshadows = [], [], []
            for i, (store, want_shadow, want_t) in enumerate(plan):
                # value 0 lives in C_; a value that is not stored still gets its (unwritten)
                # float32 buffer: it is what identifies the bf16 plane in the pack cache
                arr = C_ if i == 0 else DeviceArray.empty((m, n), "float32")
                arrays.append(arr)
                if i >= 1 and store:
                    ep.out_f32[i] = arr.ptr
                    ep.out_rs[i] = arr.strides[0]
                sh = None
                if want_shadow and arr.strides == (n, 1):
                    buf = torch.empty(m * n * 2, dtype=torch.uint8, device=A.owner.device)
                    ep.shadow_bf16[i] = buf.data_ptr()
                    ep.shadow_pitch[i] = n
                    sh = (buf, n)
                shadows.append(sh)
                tsh = None
                if want_t and arr.strides == (n, 1):
                    pitch_t = (m + 7) // 8 * 8
                    tbuf = torch.empty(n * pitch_t * 2, dtype=torch.uint8, device=A.owner.device)
                    ep.shadow_t_bf16 = tbuf.data_ptr()
                    ep.shadow_t_pitch = pitch_t
                    tsh = (tbuf, pitch_t)
                tshadows.append(tsh)
            if epilogue.colsum or epilogue.fullsum:
                rows, cols = C.c_int64(), C.c_int64()
                _lib.check(lib.ab_gemm_fused_layout(m, n, C.byref(rows), C.byref(cols)))
                if epilogue.colsum:
                    epilogue.colsum_ws = DeviceArray.empty((rows.value, n), "float64")
                    ep.colsum_ws = epilogue.colsum_ws.ptr
                if epilogue.fullsum:
                    epilogue.fullsum_ws = DeviceArray.empty((rows.value * cols.value,), "float64")
                    ep.fullsum_ws = epilogue.fullsum_ws.ptr
            c_ptr = C_.ptr if plan[0][0] else None
            _lib.check(lib.ab_gemm_packed_fused(precision, m, n, k, float(alpha), C.byref(opa), C.byref(opb),
                                                float(beta), *cin_args, c_ptr, C_.strides[0],
                                                C_.strides[1], C.byref(ep), stream_handle()))
            epilogue.applied = True
            epilogue.arrays, epilogue.shadows, epilogue.tshadows = arrays, shadows, tshadows
            return
        need = C.c_size_t()
        _lib.check(lib.ab_gemm_packed_workspace_bytes(precision, m, n, k, C.byref(need)))
        ws = torch.empty(need.value, dtype=torch.uint8, device=A.owner.device) if need.value else None
        _lib.check(lib.ab_gemm_packed(precision, m, n, k, float(alpha), C.byref(opa), C.byref(opb),
                                      float(beta), *cin_args, C_.ptr, C_.strides[0], C_.strides[1],
                                      ws.data_ptr() if ws is not None else None, need.value,
                                      stream_handle()))
        return
    if cin is not None:
        if float(beta) != 0.0:
            copy_into(C_, cin)
    ws_bytes = C.c_size_t()
    _lib.check(lib.ab_gemm_workspace_bytes(code, precision, m, n, k, A.strides[0], A.strides[1],
                                           B.strides[0], B.strides[1], C.byref(ws_bytes)))
    ws = torch.empty(max(ws_bytes.value, 1), dtype=torch.uint8, device=A.owner.device)
    _lib.check(lib.ab_gemm(code, precision, m, n, k, float(alpha), A.ptr, A.strides[0],
                           A.strides[1], B.ptr, B.strides[0], B.strides[1], float(beta), C_.ptr,
                           C_.strides[0], C_.strides[1], ws.data_ptr(), ws_bytes.value,
                           stream_handle()))


# -- dense linear algebra (csrc/ab_linalg.cu) ----------------------------------------------
class LinalgStatus:
    """The device status word of one linear-algebra node: reset when made, written by every
    factorisation and solve of the node, read once by :meth:`check` (one synchronisation)."""

    def __init__(self):
        self.word = DeviceArray.empty((1,), "uint64")
        _lib.check(_lib.load().ab_linalg_status_reset(self.word.ptr, stream_handle()))

    def check(self, nan_on_error=False):
        """Raise the reference's exception for what the kernels found: ``ValueError`` for a
        non-finite checked operand, ``numpy.linalg.LinAlgError`` for a matrix that is not
        positive definite or a zero diagonal (not raised when ``nan_on_error``: the factor is
        NaN already).  Inside a CUDA-graph capture it raises ``AbError`` before reading."""
        rc = _lib.load().ab_linalg_status_check(self.word.ptr, stream_handle())
        if rc == 0:
            return
        msg = _lib.load().ab_last_error().decode(errors="replace")
        if rc == 3:
            raise ValueError(msg)
        if rc == 7:
            if nan_on_error:
                return
            raise np.linalg.LinAlgError(msg)
        raise _lib.AbError(rc, msg)


def _workspace(nbytes, like: DeviceArray):
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=like.owner.device)


def cholesky(a: DeviceArray, lower, status: LinalgStatus, nan_on_error=False, check_finite=True) -> DeviceArray:
    """The lower or upper Cholesky factor of the symmetric matrix built from that triangle of
    ``a`` (float32 / float64, any strides), as a new C-contiguous matrix."""
    lib = _lib.load()
    n = a.shape[0]
    out = DeviceArray.empty((n, n), a.dtype)
    code = DTYPE_CODE[a.dtype.name]
    need = C.c_size_t()
    _lib.check(lib.ab_cholesky_workspace_bytes(code, n, C.byref(need)))
    ws = _workspace(need.value, a)
    _lib.check(lib.ab_cholesky(code, n, a.ptr, a.strides[0], a.strides[1], int(bool(lower)), int(bool(nan_on_error)),
                               int(bool(check_finite)), out.ptr, status.word.ptr, ws.data_ptr(), need.value,
                               stream_handle()))
    return out


def trsm(a: DeviceArray, b: DeviceArray, lower, trans, unit_diagonal, status: LinalgStatus, check_finite=True,
         check_singular=True, out: DeviceArray = None) -> DeviceArray:
    """op(a)^-1 b for triangular ``a`` (op = transpose when ``trans``), ``b`` a vector or a
    matrix of a's dtype with any strides; the result is C-contiguous (``out``, which may be
    ``b`` itself when ``b`` is C-contiguous, or a new array)."""
    lib = _lib.load()
    n = a.shape[0]
    nrhs = 1 if b.ndim == 1 else b.shape[1]
    if out is None:
        out = DeviceArray.empty(b.shape, a.dtype)
    code = DTYPE_CODE[a.dtype.name]
    need = C.c_size_t()
    _lib.check(lib.ab_trsm_workspace_bytes(code, n, nrhs, C.byref(need)))
    ws = _workspace(need.value, a)
    b_rs = b.strides[0] if b.shape[0] > 1 else nrhs
    b_cs = (b.strides[1] if b.shape[1] > 1 else 1) if b.ndim == 2 else 1
    _lib.check(lib.ab_trsm(code, n, nrhs, a.ptr, a.strides[0], a.strides[1], int(bool(lower)), int(bool(trans)),
                           int(bool(unit_diagonal)), b.ptr, b_rs, b_cs, out.ptr, int(bool(check_finite)),
                           int(bool(check_singular)), status.word.ptr, ws.data_ptr(), need.value, stream_handle()))
    return out
