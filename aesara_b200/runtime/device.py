"""Device-resident n-d arrays for the GPU runtime.

A :class:`DeviceArray` is (owner, pointer, dtype, shape, element strides) —
the device analogue of the NumPy arrays that live in the reference's storage
cells (``aesara/link/basic.py:39`` ``Container``).  Views (``DimShuffle``,
``Subtensor``, ``Reshape``) share the owner, exactly like the reference's
``view_map`` ops share NumPy bases.  PyTorch provides the allocator, the
streams and the host<->device copies (plumbing only — no torch op computes).
"""

from __future__ import annotations

import numpy as np
import torch

PINNED_MIN_BYTES = 1 << 16  # device->host copies at least this big use page-locked memory
SMALL_STAGE_BYTES = 1 << 20  # host->device copies up to this size are staged through page-locked memory
_TORCH_BYTES = torch.uint8


def current_device():
    return torch.cuda.current_device()


def stream_handle():
    """Raw ``cudaStream_t`` of torch's current stream (int)."""
    return torch.cuda.current_stream().cuda_stream


def c_strides(shape):
    st, acc = [], 1
    for n in reversed(shape):
        st.append(acc)
        acc *= max(int(n), 1)
    return tuple(reversed(st))


def f_strides(shape):
    st, acc = [], 1
    for n in shape:
        st.append(acc)
        acc *= max(int(n), 1)
    return tuple(st)


class DeviceArray:
    """A strided view of device memory.  Strides are in elements."""

    __slots__ = ("owner", "ptr", "dtype", "shape", "strides", "itemsize", "__weakref__")

    def __init__(self, owner, ptr, dtype, shape, strides):
        self.owner = owner  # torch uint8 tensor (or any object keeping memory alive)
        self.ptr = int(ptr)
        self.dtype = np.dtype(dtype)
        self.itemsize = self.dtype.itemsize
        self.shape = tuple(int(s) for s in shape)
        self.strides = tuple(int(s) for s in strides)

    # -- construction -------------------------------------------------------
    @staticmethod
    def empty(shape, dtype, order="C", device=None):
        dtype = np.dtype(dtype)
        shape = tuple(int(s) for s in shape)
        n = 1
        for s in shape:
            if s < 0:
                raise ValueError("negative dimensions are not allowed")
            n *= s
        dev = torch.device("cuda", current_device() if device is None else device)
        buf = torch.empty(max(n * dtype.itemsize, 1), dtype=_TORCH_BYTES, device=dev)
        st = c_strides(shape) if order == "C" else f_strides(shape)
        return DeviceArray(buf, buf.data_ptr(), dtype, shape, st)

    @staticmethod
    def from_numpy(a, device=None, pinned_ok=True):
        a = np.asarray(a)
        # (np.ascontiguousarray would promote 0-d arrays to 1-d)
        src = a if a.flags.c_contiguous else np.array(a, order="C")
        out = DeviceArray.empty(src.shape, src.dtype, device=device)
        if src.size:
            hb = torch.from_numpy(src.reshape(-1).view(np.uint8))
            if not hb.is_pinned() and hb.numel() <= SMALL_STAGE_BYTES:
                # A copy from pageable memory is synchronous: issued behind queued kernels it
                # blocks the host until they have run (a hidden device synchronisation per
                # staged scalar).  Small values go through a page-locked staging block of
                # torch's caching host allocator instead, which the allocator keeps alive until
                # the stream has consumed it.
                st = torch.empty(hb.numel(), dtype=_TORCH_BYTES, pin_memory=True)
                st.copy_(hb)
                hb = st
            out.owner[: hb.numel()].copy_(hb, non_blocking=hb.is_pinned())
        return out

    @staticmethod
    def upload(a, copy_stream, consumer_stream):
        """Host -> device for a function argument.  A page-locked source is copied on
        ``copy_stream`` and the returned event marks its arrival (the consumer waits on it
        at first use) together with the source buffer, which must stay alive until then;
        a pageable source is copied synchronously (second result ``None``)."""
        a = np.asarray(a)
        src = a if a.flags.c_contiguous else np.array(a, order="C")
        if not src.flags.writeable:
            src = src.copy()
        if not src.size:
            return DeviceArray.empty(src.shape, src.dtype), None
        hb = torch.from_numpy(src.reshape(-1).view(np.uint8))
        if not hb.is_pinned():
            out = DeviceArray.empty(src.shape, src.dtype)
            out.owner[: hb.numel()].copy_(hb)
            return out, None
        # The destination is allocated ON the copy stream: the caching allocator then orders its
        # reuse against earlier copy-stream work only, and the copy need not wait for whatever
        # the consumer stream still has queued (an upload of row block i+1 overlaps the
        # evaluation of row block i, shard.ChunkedHostExecutor).  record_stream keeps the block
        # from being recycled while the consumer stream uses it.
        with torch.cuda.stream(copy_stream):
            out = DeviceArray.empty(src.shape, src.dtype)
            out.owner[: hb.numel()].copy_(hb, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        out.owner.record_stream(consumer_stream)
        return out, (ev, hb)  # the caller keeps ``hb`` alive until the event has completed

    @staticmethod
    def download_all(values):
        """``to_numpy`` for a list of outputs with one synchronisation."""
        from .kernels import contiguous_copy

        res, waits = [], False
        for v in values:
            if not isinstance(v, DeviceArray):
                res.append(np.asarray(v))
                continue
            if v.nbytes < PINNED_MIN_BYTES:
                res.append(v.to_numpy())
                continue
            src = v if v.is_c_contiguous() else contiguous_copy(v)
            off = src.ptr - src.owner.data_ptr()
            if src.owner.dtype == _TORCH_BYTES:
                t = src.owner[off : off + src.nbytes]
            else:
                t = src.owner.contiguous().view(-1).view(_TORCH_BYTES)[off : off + src.nbytes]
            host = torch.empty(src.nbytes, dtype=_TORCH_BYTES, pin_memory=True)
            host.copy_(t, non_blocking=True)
            waits = True
            res.append(host.numpy().view(src.dtype).reshape(src.shape))
        if waits:
            torch.cuda.current_stream().synchronize()
        return res

    @staticmethod
    def from_torch(t):
        """Wrap a (dense) torch CUDA tensor without copying."""
        dt = {
            torch.float32: "float32", torch.float64: "float64", torch.int64: "int64",
            torch.int32: "int32", torch.int16: "int16", torch.int8: "int8",
            torch.uint8: "uint8", torch.bool: "bool",
        }[t.dtype]
        return DeviceArray(t, t.data_ptr(), dt, tuple(t.shape), tuple(t.stride()))

    # -- properties -----------------------------------------------------------
    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        n = 1
        for s in self.shape:
            n *= s
        return n

    @property
    def nbytes(self):
        return self.size * self.itemsize

    def is_c_contiguous(self):
        acc = 1
        for n, s in zip(reversed(self.shape), reversed(self.strides)):
            if n == 1:
                continue
            if s != acc:
                return False
            acc *= n
        return True

    def is_f_contiguous(self):
        acc = 1
        for n, s in zip(self.shape, self.strides):
            if n == 1:
                continue
            if s != acc:
                return False
            acc *= n
        return True

    # -- views ----------------------------------------------------------------
    def view(self, shape, strides, offset_elems=0):
        return DeviceArray(self.owner, self.ptr + offset_elems * self.itemsize, self.dtype,
                           shape, strides)

    def dimshuffle(self, new_order):
        """``aesara/tensor/elemwise.py:222-239``: transpose + insert/drop size-1 dims."""
        kept = [o for o in new_order if o != "x"]
        for d in range(self.ndim):
            if d not in kept and self.shape[d] != 1:
                raise ValueError("DimShuffle: cannot drop a non-broadcastable dimension")
        shape = [1 if o == "x" else self.shape[o] for o in new_order]
        strides = [0 if o == "x" else self.strides[o] for o in new_order]
        return self.view(shape, strides)

    def broadcast_to(self, shape):
        """NumPy ``broadcast_to`` as a stride-0 view (tensor/extra_ops.py:1613)."""
        shape = tuple(int(s) for s in shape)
        if len(shape) < self.ndim:
            raise ValueError("broadcast_to: input has more dimensions than the requested shape")
        lead = len(shape) - self.ndim
        strides = [0] * lead
        for n, s, want in zip(self.shape, self.strides, shape[lead:]):
            if n == want:
                strides.append(s)
            elif n == 1:
                strides.append(0)
            else:
                raise ValueError(f"broadcast_to: cannot broadcast {self.shape} to {shape}")
        return self.view(shape, strides)

    def diagonal(self, offset=0, axis1=0, axis2=1):
        """``ndarray.diagonal`` as a view: the two axes collapse into one (stride s1 + s2)
        that becomes the LAST axis, like NumPy."""
        nd = self.ndim
        axis1 %= nd
        axis2 %= nd
        if axis1 == axis2:
            raise ValueError("axis1 and axis2 cannot be the same")
        n1, n2 = self.shape[axis1], self.shape[axis2]
        s1, s2 = self.strides[axis1], self.strides[axis2]
        if offset >= 0:
            length, off = max(0, min(n1, n2 - offset)), offset * s2
        else:
            length, off = max(0, min(n1 + offset, n2)), -offset * s1
        keep = [d for d in range(nd) if d not in (axis1, axis2)]
        shape = [self.shape[d] for d in keep] + [length]
        strides = [self.strides[d] for d in keep] + [s1 + s2]
        return self.view(shape, strides, off if length > 0 else 0)

    def index(self, idx):
        """Basic NumPy indexing (ints and slices) -> view."""
        idx = tuple(idx) + (slice(None),) * (self.ndim - len(idx))
        if len(idx) > self.ndim:
            raise IndexError("too many indices for array")
        off, shape, strides = 0, [], []
        for d, (i, n, s) in enumerate(zip(idx, self.shape, self.strides)):
            if isinstance(i, slice):
                start, stop, step = i.indices(n)
                ln = len(range(start, stop, step))
                off += start * s if ln > 0 else 0
                shape.append(ln)
                strides.append(s * step)
            else:
                i = int(i)
                if i < -n or i >= n:
                    raise IndexError(f"index {i} is out of bounds for axis {d} with size {n}")
                if i < 0:
                    i += n
                off += i * s
        return self.view(shape, strides, off)

    def reshape_view(self, shape):
        """Reshape without copying; only valid for C-contiguous arrays."""
        shape = [int(s) for s in shape]
        if -1 in shape:
            known = 1
            for s in shape:
                if s != -1:
                    known *= s
            shape[shape.index(-1)] = self.size // max(known, 1)
        n = 1
        for s in shape:
            n *= s
        if n != self.size:
            raise ValueError(f"cannot reshape array of size {self.size} into shape {tuple(shape)}")
        if not self.is_c_contiguous():
            raise ValueError("reshape_view needs a C-contiguous array")
        return self.view(shape, c_strides(shape))

    # -- host transfer ----------------------------------------------------------
    def to_numpy(self):
        """Device -> host.  Large arrays land in a page-locked block from torch's caching
        host allocator (a fresh pageable array page-faults on every page it receives) and
        the returned ndarray owns that block
        through its base, so results are never recycled under the caller
        (``Out(borrow=False)`` semantics, compile/function/types.py:1067-1117)."""
        from .kernels import contiguous_copy

        src = self if self.is_c_contiguous() else contiguous_copy(self)
        if not src.size:
            return np.empty(src.shape, dtype=src.dtype)
        base_off = src.ptr - src.owner.data_ptr()
        if isinstance(src.owner, torch.Tensor) and src.owner.dtype == _TORCH_BYTES:
            t = src.owner[base_off : base_off + src.nbytes]
        else:  # a wrapped typed torch tensor
            t = src.owner.contiguous().view(-1).view(_TORCH_BYTES)[base_off : base_off + src.nbytes]
        if src.nbytes >= PINNED_MIN_BYTES:
            host = torch.empty(src.nbytes, dtype=_TORCH_BYTES, pin_memory=True)
            host.copy_(t, non_blocking=True)
            torch.cuda.current_stream(t.device).synchronize()
        else:
            host = t.cpu()
        return host.numpy().view(src.dtype).reshape(src.shape)

    def copy(self):
        """A C-contiguous device copy (the device analogue of ``ndarray.copy``)."""
        from .kernels import contiguous_copy

        return contiguous_copy(self)

    def __deepcopy__(self, memo):
        return self.copy()

    def __array__(self, dtype=None, copy=None):
        a = self.to_numpy()
        return a if dtype is None else a.astype(dtype)

    def item(self):
        return self.to_numpy().reshape(()).item() if self.size == 1 else self.to_numpy().item()

    def __repr__(self):
        return f"DeviceArray(shape={self.shape}, dtype={self.dtype.name}, strides={self.strides})"
