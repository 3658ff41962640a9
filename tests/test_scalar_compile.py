"""CPU: every scalar op of the device table compiles at every input dtype the front end admits.

The generated body of a scalar op is a C++ expression over the ``ab_types.cuh`` typedefs, and
C++ overload resolution depends on the operand types (``floor`` of an ``int`` is ambiguous
between the float and double overloads).  A body that does not compile surfaces only when a
graph with that op at that dtype first runs.  Here each op of ``scalar_cuda.TABLE`` is lowered
the way the front end lowers it (``lower.lower_scalar_op``: output dtype from the reference's
own ``output_types``) at every combination of the 11 device dtypes that those rules accept, and
all bodies go through NVRTC with the runtime's options in one translation unit.  A body either
compiles or ``emit_body`` refuses it with ``UnsupportedScalar`` at code-generation time.
Needs no GPU.
"""
import itertools

import pytest

DTYPES = ["bool", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64",
          "float32", "float64"]


def _scalar_ops():
    """(name, scalar Op instance) for every class the lowering maps to a device table entry."""
    from aesara_b200.compat import bootstrap

    if not bootstrap.available():
        pytest.skip("reference front-end (oracle/_ref) not present")
    bootstrap.load_aesara()
    import aesara.scalar.basic as sb
    import aesara.scalar.math as sm

    from aesara_b200.lower import _SCALAR_OPS

    ops = {}
    for mod in (sb, sm):
        for name, v in sorted(vars(mod).items()):
            if isinstance(v, sb.ScalarOp) and type(v).__name__ in _SCALAR_OPS:
                ops.setdefault(f"{type(v).__name__}:{name}", v)
    # one instance per class is enough, except Cast (one per target) and InRange (open / closed)
    keep = {}
    for key, v in ops.items():
        cls = key.split(":")[0]
        if cls in ("Cast", "InRange") or cls not in {k.split(":")[0] for k in keep}:
            keep[key] = v
    return keep


def _bodies():
    from aesara_b200.codegen.scalar_cuda import UnsupportedScalar, emit_body
    from aesara_b200.lower import UnsupportedOp, lower_scalar_op

    bodies, refused, n_sig = [], [], 0
    for key, op in _scalar_ops().items():
        # variadic ops (add, mul, mean) at two operands
        for dts in itertools.product(DTYPES, repeat=op.nin if op.nin > 0 else 2):
            try:
                expr = lower_scalar_op(op, list(dts))
            except (TypeError, NotImplementedError, UnsupportedOp):
                continue  # the reference's output-type rules reject this combination
            if any(st["dtype"] not in DTYPES for st in expr["stmts"]):
                continue  # casts to float16 / complex: no device representation
            n_sig += 1
            name = f"b{len(bodies)}"
            try:
                bodies.append((name, f"{key}({', '.join(dts)})", emit_body(expr, fn_name=name)))
            except UnsupportedScalar as e:
                refused.append((key, dts, str(e)))
    return bodies, refused, n_sig


def test_every_table_op_compiles_at_every_admitted_dtype():
    from aesara_b200.codegen.elemwise import _read
    from aesara_b200.codegen.scalar_cuda import TABLE
    from aesara_b200.lower import _SCALAR_OPS
    from aesara_b200.runtime import lib

    bodies, refused, n_sig = _bodies()
    lowered = {_SCALAR_OPS[label.split(":")[0]] for _, label, _ in bodies}
    # every table entry was exercised
    missing = set(TABLE) - lowered
    assert not missing, f"no admitted dtype signature reached {sorted(missing)}"
    assert n_sig > 3000 and len(bodies) > 2500, (n_sig, len(bodies))
    # only the float-only ops refuse, and only for integer or bool outputs
    for key, dts, msg in refused:
        assert "output" in msg or "float" in msg, (key, dts, msg)
    head = _read("ab_types.cuh").replace("#pragma once", "")
    src = "\n".join([head] + [b for _, _, b in bodies])
    try:
        lib.compile_cubin(src, "scalar_table")
    except lib.AbError as e:
        # name the bodies NVRTC rejected (its log gives the line numbers of the unit)
        lines = src.splitlines()
        bad = set()
        for tok in str(e).split("("):
            num = tok.split(")")[0]
            if num.isdigit() and 0 < int(num) <= len(lines):
                for k in range(int(num) - 1, -1, -1):
                    if lines[k].startswith("__device__") and " b" in lines[k]:
                        bad.add(lines[k].split("void ")[1].split("(")[0])
                        break
        labels = [label for name, label, _ in bodies if name in bad]
        pytest.fail(f"NVRTC rejected {len(labels)} bodies: {labels[:20]}\n{str(e)[:2000]}")
