"""aesara_b200 — a Hopper (H100, sm_90a) execution backend behind Aesara's Linker.

``import aesara_b200`` registers linker ``"b200"`` and mode ``"B200"`` with the
reference front-end when it is importable (``aesara_b200.linker``).  The device
runtime itself (``aesara_b200.runtime``, ``aesara_b200.ir``) has no Aesara
dependency: lowered programs run wherever ``libaesara_b200.so`` and an H100 are.
"""

__version__ = "0.1.0"

from .ir import Program  # noqa: F401


def frontend_available():
    from .compat import bootstrap

    return bootstrap.available()


def __getattr__(name):
    # lazy: importing the linker imports the (heavy) reference front-end
    if name in ("B200Linker", "B200VM", "mode", "register"):
        from . import linker

        return getattr(linker, name)
    if name in ("shared", "B200SharedVariable"):
        from . import sharedvar

        return getattr(sharedvar, name)
    if name == "check_function":
        from .debug import check_function

        return check_function
    if name == "ProgramExecutor":
        from .runtime.vm import ProgramExecutor

        return ProgramExecutor
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


def _auto_register():
    import os

    if os.environ.get("AESARA_B200_NO_AUTOREGISTER"):
        return
    try:
        if frontend_available():
            from . import linker  # noqa: F401
    except Exception:  # the front-end is optional at run time
        pass


_auto_register()
