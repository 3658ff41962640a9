"""Device-resident shared variables (SURVEY.md §8f N4).

Reference: ``aesara/compile/sharedvalue.py:47-131`` (``SharedVariable``: a ``Container``
cell shared by every ``Function`` that uses the variable; ``get_value(borrow,
return_internal_type)``; ``set_value``) and ``aesara/tensor/sharedvar.py:22-85``
(``TensorSharedVariable`` / ``tensor_constructor``).

With a host-typed linker the value of a shared variable is a NumPy array: a B200 function
would upload the weights on every call and download every ``updates=`` result.
``B200SharedVariable`` keeps the ordinary ``TensorType`` (so every Op and rewrite applies
unchanged) but lets its storage cell hold a ``DeviceArray``:

* ``B200VM`` (``linker.py``) applies ``update_mapping`` itself (``need_update_inputs = False``,
  as the C VM does, ``link/vm.py:326-335``) and writes the *device* result straight into the
  cell of a ``B200SharedVariable`` — no download, and the next call consumes it without an
  upload;
* ``get_value()`` downloads (a NumPy array, as any caller of the reference expects);
  ``get_value(return_internal_type=True)`` hands out the ``DeviceArray`` (the documented
  purpose of that flag, ``sharedvalue.py:99-107``);
* ``set_value`` accepts a NumPy array (uploaded lazily by the next call) or a ``DeviceArray``.

Functions compiled with another linker see the NumPy view through ``Container.value``
only after ``sync_to_host()``; sharing one variable between a B200 function and a C-linker
function therefore needs that call (or ``aesara.shared`` for such variables).
"""

from __future__ import annotations

import copy
import weakref

import numpy as np

from .compat.bootstrap import load_aesara

load_aesara()

from aesara.tensor.sharedvar import TensorSharedVariable  # noqa: E402
from aesara.tensor.type import TensorType  # noqa: E402

_DEVICE_CELLS = {}  # id(storage list) -> weakref to the variable that owns it


def is_device_value(v):
    """A device array (duck-typed so the host logic is testable without a GPU)."""
    return not isinstance(v, np.ndarray) and hasattr(v, "to_numpy") and hasattr(v, "ptr")


def owns_cell(cell):
    """True if ``cell`` (a 1-element storage list) belongs to a live B200SharedVariable."""
    ref = _DEVICE_CELLS.get(id(cell))
    var = ref() if ref is not None else None
    return var is not None and var.container.storage is cell


class B200SharedVariable(TensorSharedVariable):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        cell = self.container.storage
        key = id(cell)
        _DEVICE_CELLS[key] = weakref.ref(self, lambda _r, k=key: _DEVICE_CELLS.pop(k, None))

    # -- value access -----------------------------------------------------------------
    def get_value(self, borrow=False, return_internal_type=False):
        v = self.container.storage[0]
        if is_device_value(v):
            if return_internal_type:
                return v if borrow else v.copy()
            return v.to_numpy()
        return super().get_value(borrow=borrow, return_internal_type=return_internal_type)

    def set_value(self, new_value, borrow=False):
        if is_device_value(new_value):
            if np.dtype(new_value.dtype).name != self.type.dtype or len(new_value.shape) != self.type.ndim:
                raise TypeError(
                    f"{self}: expected {self.type.dtype} with {self.type.ndim} dims, got "
                    f"{np.dtype(new_value.dtype).name} with {len(new_value.shape)}")
            self.container.storage[0] = new_value if borrow else new_value.copy()
            return
        super().set_value(new_value, borrow=borrow)

    def is_on_device(self):
        return is_device_value(self.container.storage[0])

    def sync_to_host(self):
        """Replace a device-resident value by its NumPy copy (for non-B200 functions)."""
        v = self.container.storage[0]
        if is_device_value(v):
            self.container.storage[0] = v.to_numpy()
        return self.container.storage[0]

    def zero(self, borrow=False):
        v = self.container.storage[0]
        if is_device_value(v):
            self.container.storage[0] = np.zeros(v.shape, dtype=v.dtype)
            return
        super().zero(borrow=borrow)

    def __deepcopy__(self, memo):
        self.sync_to_host()
        cls = type(self)
        new = cls(type=self.type, value=copy.deepcopy(self.container.storage[0], memo), strict=None,
                  name=self.name)
        memo[id(self)] = new
        return new


def shared(value, name=None, strict=False, allow_downcast=None, borrow=False, shape=None):
    """``aesara.shared`` for values that should live on the GPU between calls
    (same arguments as ``tensor_constructor``, ``tensor/sharedvar.py:48-85``)."""
    if is_device_value(value):
        dev = value
        value = np.empty((0,) * len(dev.shape), dtype=dev.dtype)  # placeholder for the type
    else:
        dev = None
        value = np.asarray(value)
    if shape is None:
        shape = (None,) * value.ndim
    var = B200SharedVariable(
        type=TensorType(value.dtype, shape=shape),
        value=np.array(value, copy=(not borrow)),
        strict=strict,
        allow_downcast=allow_downcast,
        name=name,
    )
    if dev is not None:
        var.set_value(dev, borrow=borrow)
    return var


# -- registration with ``aesara.shared`` (compile/sharedvalue.py:213 ``shared_constructor``) --
def _device_array_constructor(value, name=None, strict=False, allow_downcast=None, borrow=False,
                              shape=None, **kwargs):
    return shared(value, name=name, strict=strict, allow_downcast=allow_downcast, borrow=borrow,
                  shape=shape)


_NDARRAY_DEFAULT = None


def register_shared_constructor(ndarrays=False):
    """Teach ``aesara.shared`` about device values.

    Always: ``aesara.shared(DeviceArray)`` yields a :class:`B200SharedVariable` holding that
    array (the ``singledispatch`` registry of ``compile/sharedvalue.py:213-222``, the way
    ``tensor/sharedvar.py:48`` registers ``np.ndarray``).

    ``ndarrays=True``: NumPy arrays given to ``aesara.shared`` also become
    ``B200SharedVariable``s, so an unchanged user script keeps its parameters on the GPU
    between calls (their values move to the device at the first ``updates=`` of a B200
    function).  Opt-in, because a function compiled with another linker that shares such a
    variable needs ``sync_to_host()`` first.  ``ndarrays=False`` restores the default."""
    global _NDARRAY_DEFAULT
    from aesara.compile.sharedvalue import shared_constructor

    from .runtime.device import DeviceArray

    if shared_constructor.dispatch(DeviceArray) is not _device_array_constructor:
        shared_constructor.register(DeviceArray, _device_array_constructor)
    if _NDARRAY_DEFAULT is None:
        _NDARRAY_DEFAULT = shared_constructor.dispatch(np.ndarray)
    if ndarrays:
        shared_constructor.register(np.ndarray, _device_array_constructor)
    else:
        shared_constructor.register(np.ndarray, _NDARRAY_DEFAULT)
