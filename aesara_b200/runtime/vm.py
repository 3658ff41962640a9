"""Program executor: the device-side analogue of the reference's VM.

What ``CLazyLinker_call`` does for the C-linker (``lazylinker_c.c:752-890``;
Python twin ``aesara/link/vm.py:338-421`` ``Loop``) — walk the nodes in order,
run each thunk, drop intermediates after their last use, report the failing
node — is done here over a lowered :class:`~aesara_b200.ir.Program`.  Tensor
work is launched asynchronously on the current CUDA stream through the C ABI;
int64 shape arithmetic (SURVEY.md a9) is evaluated on the host *before* the
launches that depend on it, without device synchronisation.

There is no CPU fallback for tensor work: a node kind without a device
implementation raises ``NotImplementedError`` at construction time.
"""

from __future__ import annotations

import copy
import os

import numpy as np
import torch

from ..ir import Node, Program
from . import host_eval
from . import kernels as K
from .device import DeviceArray

_EXEC = {}


def _op(name):
    def deco(fn):
        _EXEC[name] = fn
        return fn

    return deco


class NodeError(RuntimeError):
    """Raised with the position of the failing node (``vm.position_of_error``)."""

    def __init__(self, position, node, exc, inputs=None):
        super().__init__(f"{type(exc).__name__}: {exc}\nwhile running node {position}: {node.label or node.op}")
        self.position = position
        self.node = node
        self.original = exc
        # the values the failing node was given (what ``raise_with_op`` prints shapes and
        # strides of, aesara/link/utils.py:340-356); filled in by the executor
        self.inputs = inputs


def is_host(v):
    return not isinstance(v, DeviceArray)


def touched_bytes(v):
    """Bytes of device memory a kernel moves for this operand: broadcast (stride 0)
    dimensions are read once (SURVEY 8d: "distinct input bytes + output bytes")."""
    if not isinstance(v, DeviceArray):
        return 0
    n = v.itemsize
    for s, st in zip(v.shape, v.strides):
        if st != 0 or s == 0:
            n *= s
    return n


# Input positions whose *values* a node needs on the host (allocation shapes, indices, axes,
# BLAS scalars, loop counts): everything the reference computes with int64 shape arithmetic
# (SURVEY.md a9).  "all" = every input, ("from", k) = inputs k.. .
_HOST_SLOTS = {
    "AllocEmpty": "all", "MakeVector": "all", "ScalarOp": "all", "Tri": "all", "Eye": "all",
    "ARange": "all", "ScalarFromTensor": "all",
    "Alloc": ("from", 1), "BroadcastTo": ("from", 1), "Subtensor": ("from", 1),
    "IncSubtensor": ("from", 2), "Assert": ("from", 1),
    "Reshape": (1,), "Join": (0,), "Split": (1, 2), "Gemm": (1, 4), "Gemv": (1, 4), "Ger": (1,),
    "Dot22Scalar": (2,), "IfElse": (0,),
    # the Generator, the size and the dtype code of a random variable (the draws' key is taken
    # from the Generator on the host, lower.py)
    "RandomVariable": (0, 1, 2),
}
# node kinds through which "needed on the host" propagates from an output to the inputs (the
# value is *computed* from them); Shape/Shape_i read only metadata and stop the propagation
_HOST_TRANSPARENT = {"Elemwise", "CAReduce", "DimShuffle", "Subtensor", "TensorFromScalar",
                     "ScalarFromTensor", "Reshape", "MakeVector", "Join", "View", "DeepCopy",
                     "ScalarOp", "Assert", "Alloc", "BroadcastTo", "IfElse", "Split",
                     "AdvancedSubtensor1", "ARange", "MaxAndArgmax", "CumOp"}


def host_needed_vars(program):
    """Variables whose values some node needs on the host, closed backwards through the
    nodes that compute them.  A tensor *argument* of the function outside this set is data,
    whatever its size, and is uploaded; inside it (and small) it stays a host value so that
    shapes and indices never cost a device synchronisation."""
    need = set()
    for n in program.nodes:
        slots = _HOST_SLOTS.get(n.op)
        if n.op == "Scan":
            info = n.params["info"]
            n_outs = (len(info["mit_mot_in_slices"]) + len(info["mit_sot_in_slices"])
                      + len(info["sit_sot_in_slices"]))
            first_nit = 1 + info["n_seqs"] + n_outs + info["n_shared_outs"]
            slots = (0,) + tuple(range(first_nit, first_nit + info["n_nit_sot"]))
        if slots is None:
            continue
        if slots == "all":
            idx = range(len(n.inputs))
        elif slots[0] == "from":
            idx = range(slots[1], len(n.inputs))
        else:
            idx = [k for k in slots if k < len(n.inputs)]
        need.update(n.inputs[k] for k in idx)
    for n in reversed(program.nodes):
        if n.op in _HOST_TRANSPARENT and any(v in need for v in n.outputs):
            need.update(n.inputs)
    return need


class ProgramExecutor:
    def __init__(self, program: Program, precision: int = 0, host_outputs: bool = True,
                 time_nodes: bool = False):
        self.program = program
        self.precision = precision
        self.host_outputs = host_outputs
        self.time_nodes = time_nodes
        self.position_of_error = -1
        self._const_host = {}
        self._const_dev = {}
        self._staged = {}
        for vid, v in enumerate(program.vars):
            if v.const is not None:
                self._const_host[vid] = v.const if v.kind == "tensor" else v.const.dtype.type(v.const.item())
            elif v.const_other is not None:
                c = v.const_other
                self._const_host[vid] = None if "none" in c else slice(*c["slice"])
        missing = sorted({n.op for n in program.nodes if n.op not in _EXEC})
        if missing:
            raise NotImplementedError(
                "B200 runtime has no implementation for node kind(s): " + ", ".join(missing)
            )
        self._steps = [_EXEC[n.op] for n in program.nodes]
        # per-node private state (kernels, nested executors)
        self._state = [dict() for _ in program.nodes]
        # liveness: drop a value right after its last consumer (allow_gc semantics,
        # aesara/link/vm.py:666-683)
        last = {}
        for i, n in enumerate(program.nodes):
            for v in n.inputs:
                last[v] = i
        keep = set(program.outputs) | set(program.inputs)
        self._free_after = [[] for _ in program.nodes]
        for v, i in last.items():
            if v not in keep and v not in self._const_host:
                self._free_after[i].append(v)
        self.node_events = None
        self.trace = None  # debug: {node index: [host copies of its outputs]} (aesara_b200/debug.py)
        self._first_use = {}
        for i, n in enumerate(program.nodes):
            for v in n.inputs:
                self._first_use.setdefault(v, i)
        self._host_needed = host_needed_vars(program)
        self._subset_cache = {}
        self._copy_streams = {}
        self._inflight = []
        self.pack_cache = K.PackCache()
        # input positions each node rewrites in place (destroy_map): their cached GEMM
        # packs must be dropped after the node ran
        self._destroys = []
        for n in program.nodes:
            d = []
            if "destroy" in n.params:  # the Op's own destroy_map, emitted by lower.py
                d = sorted(int(v) for v in n.params["destroy"])
            elif n.op == "Elemwise":
                d = sorted(set(int(v) for v in n.params.get("inplace", {}).values()))
            elif n.op in ("Gemm", "Gemv", "Ger", "IncSubtensor", "AdvancedIncSubtensor1",
                          "AdvancedIncSubtensor") and n.params.get("inplace"):
                d = [0]
            elif n.op == "Scan":
                d = sorted({int(i) for v in n.params.get("destroy_map", {}).values() for i in v})
            self._destroys.append(d)
        # function inputs some node rewrites in place (directly or through a view of them):
        # their device copies are never shared between calls
        root = {}
        for n in program.nodes:
            if n.op in ("DimShuffle", "Subtensor", "Reshape", "View", "BroadcastTo", "ExtractDiag",
                        "Assert", "IfElse") and n.inputs:
                for o in n.outputs:
                    root[o] = root.get(n.inputs[0], n.inputs[0])
        self._destroyed_inputs = set()
        for n, d in zip(program.nodes, self._destroys):
            for pos in d:
                if pos < len(n.inputs):
                    v = n.inputs[pos]
                    self._destroyed_inputs.add(root.get(v, v))
            if d:  # an in-place result aliases the operand it overwrote
                for o in n.outputs:
                    v = n.inputs[d[0]]
                    root[o] = root.get(v, v)
        # row-region fusion (runtime/rowfuse.py): member nodes are skipped and the region runs
        # as one kernel at the position of its last node; operands of skipped nodes must
        # stay alive until then
        from .rowfuse import RowFusion

        from .gemmfuse import GemmEpilogueFusion

        self._fusions = RowFusion.detect(program, self._destroys)
        taken = {i for f in self._fusions for i in f.members}
        # GEMM-epilogue regions under the reduced-precision product policies only: the
        # fp32-faithful kernels spend three tensor-core passes per product, and the Elemwise /
        # CAReduce kernels of the unfused graph run at the HBM roof, so a region saves little
        # there.  AB_GEMM_FUSE_FP32=1 keeps them (tests).
        if self.precision == 0 and not os.environ.get("AB_GEMM_FUSE_FP32"):
            gemm_regions = []
        else:
            gemm_regions = GemmEpilogueFusion.detect(program, self._destroys, taken)
        for f in gemm_regions:
            f.exact_sums = self.precision == 0
            f.planes = self.precision == 2
        self._fusions += gemm_regions
        from .redfuse import ReducePreFusion

        taken = {i for f in self._fusions for i in f.members}
        self._fusions += ReducePreFusion.detect(program, self._destroys, taken)
        self._gemm_epilogue = None
        self._fusion_of = {}
        for f in self._fusions:
            for i in f.members:
                self._fusion_of[i] = f
                if i != f.last:
                    self._free_after[f.last].extend(self._free_after[i])
                    self._free_after[i] = []
        self.fused_regions_run = 0
        # output hook (shard.ShardedExecutor): called as hook(k, value) right after the node
        # (or region) that produces function output k has been launched, so that a collective
        # on a finished gradient overlaps the rest of the evaluation
        self.output_hook = None
        self._out_storage = None
        producer = {v: i for i, n in enumerate(program.nodes) for v in n.outputs}
        self._outputs_of_node = {}
        for k, v in enumerate(program.outputs):
            i = producer.get(v)
            if i is None:
                continue
            f = self._fusion_of.get(i)
            if f is not None:
                i = getattr(f, "anchor", f.last)
            self._outputs_of_node.setdefault(i, []).append((k, v))
        self.prepare()

    # ------------------------------------------------------------------
    def prepare(self):
        """Build (and NVRTC-compile, no GPU needed) the statically known kernels."""
        for i, n in enumerate(self.program.nodes):
            st = self._state[i]
            if n.op == "Elemwise":
                st["kernel"] = K.ElemwiseKernel.get(n.params["expr"])
                st["host_ok"] = host_eval.supports(n.params["expr"])
            elif n.op == "CAReduce":
                p = n.params
                st["kernel"] = K.CAReduceKernel.get(p["scalar_op"], p["in_dtype"],
                                                    p["acc_dtype"], p["out_dtype"])
            elif n.op == "Scan":
                from .scan import ScanRunner

                st["runner"] = ScanRunner(n, self)

    def compile_all(self):
        """Force JIT compilation of every module (used by build()/tests on CPU)."""
        n = 0
        for st in self._state:
            k = st.get("kernel")
            if k is not None:
                k.compile()
                n += 1
            r = st.get("runner")
            if r is not None:
                n += r.inner.compile_all()
        for f in self._fusions:
            n += f.compile_all()
        return n

    # ------------------------------------------------------------------
    def dev(self, v, key=None, dtype=None):
        """Device view of a value.  Host values are uploaded; uploads of
        unchanged values (constants, shape-derived scalars) are reused."""
        if isinstance(v, DeviceArray):
            return v
        a = np.asarray(v) if dtype is None else np.asarray(v, dtype=dtype)
        if key is None:
            return DeviceArray.from_numpy(a)
        ent = self._staged.get(key)
        sig = (a.dtype.str, a.shape, a.tobytes())
        if ent is not None and ent[0] == sig:
            return ent[1]
        d = DeviceArray.from_numpy(a)
        self._staged[key] = (sig, d)
        return d

    def const_dev(self, vid):
        d = self._const_dev.get(vid)
        if d is None:
            d = self._const_dev[vid] = DeviceArray.from_numpy(self._const_host[vid])
        return d

    # ------------------------------------------------------------------
    def needed_nodes(self, output_subset):
        """Which nodes must run so that the outputs at the given positions (plus every
        update output, ``aesara/link/vm.py:540-551``) are computed: their ancestors, with
        fused regions kept whole."""
        key = tuple(sorted(set(int(k) for k in output_subset) | {o for o, _ in self.program.updates}))
        hit = self._subset_cache.get(key)
        if hit is not None:
            return hit
        prog = self.program
        want = {prog.outputs[k] for k in key}
        needed = [False] * len(prog.nodes)
        changed = True
        while changed:
            changed = False
            for i in range(len(prog.nodes) - 1, -1, -1):
                n = prog.nodes[i]
                if not needed[i] and any(v in want for v in n.outputs):
                    needed[i] = changed = True
                if needed[i]:
                    before = len(want)
                    want.update(n.inputs)
                    changed = changed or len(want) != before
            for f in self._fusions:
                if any(needed[m] for m in f.members) and not all(needed[m] for m in f.members):
                    for m in f.members:
                        needed[m] = True
                    changed = True
        self._subset_cache[key] = (needed, key)
        return needed, key

    def __call__(self, *inputs, output_subset=None, out_storage=None):
        """``out_storage`` ({output position: DeviceArray}): where the caller would like those
        outputs to be written (a Scan step hands the rows of its output buffers,
        runtime/scan.py); honoured by the node that allocates the output when shape, dtype and
        layout agree — the caller checks identity and copies otherwise."""
        prog = self.program
        self._out_storage = None
        if out_storage:
            self._out_storage = {prog.outputs[k]: a for k, a in out_storage.items()}
        if len(inputs) != len(prog.inputs):
            raise TypeError(f"expected {len(prog.inputs)} inputs, got {len(inputs)}")
        needed = None
        if output_subset is not None:
            needed, computed_outputs = self.needed_nodes(output_subset)
        env = dict(self._const_host)
        self.pack_cache.clear()
        # host tensors are uploaded on a copy stream in order of first use, so that a
        # page-locked argument's transfer overlaps the nodes that do not need it yet
        pending = {}
        uploads = []
        for vid, val in zip(prog.inputs, inputs):
            var = prog.vars[vid]
            if isinstance(val, DeviceArray):
                if var.kind != "tensor":
                    raise TypeError("device arrays can only feed tensor inputs")
                if val.dtype.name != var.dtype or val.ndim != var.ndim:
                    raise TypeError(
                        f"input {var.name or vid}: expected {var.dtype} with {var.ndim} dims, "
                        f"got {val.dtype.name} with {val.ndim}"
                    )
            elif var.kind == "tensor":
                val = np.asarray(val)
                if val.dtype.name != var.dtype:
                    val = val.astype(var.dtype)
                if val.ndim != var.ndim:
                    raise TypeError(
                        f"input {var.name or vid}: wrong number of dimensions: expected "
                        f"{var.ndim}, got {val.ndim} with shape {val.shape}"
                    )
                # data goes to the device whatever its size; only values that drive shapes /
                # indices / BLAS scalars (host_needed_vars) stay host-side while they are small
                if vid not in self._host_needed or val.size > host_eval.MAX_HOST_ELEMS:
                    if val.size <= host_eval.MAX_HOST_ELEMS and vid not in self._destroyed_inputs:
                        # a handful of bytes: staged once per distinct value (a replayed CUDA
                        # graph holds no host copy, runtime/graph.py keys on these bytes)
                        env[vid] = self.dev(val, key=("arg", vid))
                    else:
                        uploads.append((self._first_use.get(vid, 0), vid, val))
                    continue
            elif var.kind == "scalar":
                val = np.dtype(var.dtype).type(val)
            env[vid] = val
        if uploads:
            uploads.sort(key=lambda u: u[0])
            cur = torch.cuda.current_stream()
            for ev, _ in self._inflight:  # sources of the previous call's uploads
                ev.synchronize()
            self._inflight = []
            for _, vid, val in uploads:
                env[vid], tok = DeviceArray.upload(val, self._copy_stream_for(cur), cur)
                if tok is not None:
                    pending[vid] = tok[0]
                    self._inflight.append(tok)
        events = [] if self.time_nodes else None
        nodes = prog.nodes
        for i, step in enumerate(self._steps):
            node = nodes[i]
            if needed is not None and not needed[i]:
                continue
            if pending:
                for v in node.inputs:
                    ev = pending.pop(v, None)
                    if ev is not None:
                        torch.cuda.current_stream().wait_event(ev)
            fusion = self._fusion_of.get(i)
            if fusion is not None:
                # a region runs once, at its anchor (its last node unless the region says
                # otherwise); the other member positions are skipped
                if i == getattr(fusion, "anchor", fusion.last):
                    if events is not None:
                        e0 = torch.cuda.Event(enable_timing=True)
                        e1 = torch.cuda.Event(enable_timing=True)
                        e0.record()
                    try:
                        done = fusion.run(self, env)
                    except Exception as exc:
                        self.position_of_error = i
                        raise NodeError(i, node, exc, [env.get(v) for v in node.inputs]) from exc
                    if not done:
                        self._run_nodes(fusion.members, env)
                    else:
                        self.fused_regions_run += 1
                    if events is not None:
                        e1.record()
                        inside = {v for m in fusion.members for v in nodes[m].outputs}
                        ext = {v for m in fusion.members for v in nodes[m].inputs if v not in inside}
                        nbytes = sum(touched_bytes(env.get(v)) for v in ext)
                        nbytes += sum(touched_bytes(env.get(v)) for v in inside)
                        events.append((i, e0, e1, nbytes))
                    if self.trace is not None:
                        # values a fused region does not materialise are simply absent
                        for m in fusion.members:
                            vals = [env.get(v) for v in nodes[m].outputs]
                            if all(v is not None for v in vals):
                                self.trace[m] = [v.to_numpy() if isinstance(v, DeviceArray) else np.array(v, copy=True)
                                                 for v in vals]
                    if self.output_hook is not None:
                        for k, v in self._outputs_of_node.get(i, ()):
                            self.output_hook(k, env[v])
                if i == fusion.last:
                    for v in self._free_after[i]:
                        env.pop(v, None)
                continue
            if events is not None:
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                e0.record()
            try:
                outs = step(self, i, node, [env[v] for v in node.inputs])
            except NodeError:
                raise
            except Exception as exc:
                self.position_of_error = i
                raise NodeError(i, node, exc, [env.get(v) for v in node.inputs]) from exc
            if len(node.outputs) == 1:
                env[node.outputs[0]] = outs
            else:
                for vid, o in zip(node.outputs, outs):
                    env[vid] = o
            if events is not None:
                e1.record()
                seen, nbytes = set(), 0
                for v in node.inputs:
                    a = env.get(v)
                    if isinstance(a, DeviceArray) and (a.ptr, a.shape, a.strides) not in seen:
                        seen.add((a.ptr, a.shape, a.strides))
                        nbytes += touched_bytes(a)
                nbytes += sum(touched_bytes(env.get(v)) for v in node.outputs)
                events.append((i, e0, e1, nbytes))
            for pos in self._destroys[i]:
                d = env.get(node.inputs[pos])
                if isinstance(d, DeviceArray):
                    self.pack_cache.invalidate(d.owner)
            if self.output_hook is not None:
                for k, v in self._outputs_of_node.get(i, ()):
                    self.output_hook(k, env[v])
            if self.trace is not None:
                vals = [env[v] for v in node.outputs]
                self.trace[i] = [v.to_numpy() if isinstance(v, DeviceArray)
                                 else (None if v is None or isinstance(v, slice)
                                       else copy.deepcopy(v) if isinstance(v, np.random.Generator)
                                       else np.array(v, copy=True))
                                 for v in vals]
            for v in self._free_after[i]:
                env.pop(v, None)
        self.node_events = events
        self.pack_cache.clear()
        for ev in pending.values():  # inputs no node consumed (returned as they are)
            torch.cuda.current_stream().wait_event(ev)
        if needed is None:
            outs = [env[v] for v in prog.outputs]
        else:  # outputs nobody asked for are not computed (None, as in the reference VM)
            outs = [env[v] if k in computed_outputs else None for k, v in enumerate(prog.outputs)]
        if self.host_outputs:
            got = DeviceArray.download_all([o for o in outs if o is not None])
            it = iter(got)
            outs = [None if o is None else next(it) for o in outs]
        return outs

    def _run_nodes(self, indices, env):
        """Plain execution of the given nodes (a fused region whose operands did not fit)."""
        nodes = self.program.nodes
        for i in indices:
            node = nodes[i]
            try:
                outs = self._steps[i](self, i, node, [env[v] for v in node.inputs])
            except NodeError:
                raise
            except Exception as exc:
                self.position_of_error = i
                raise NodeError(i, node, exc, [env.get(v) for v in node.inputs]) from exc
            if len(node.outputs) == 1:
                env[node.outputs[0]] = outs
            else:
                for vid, o in zip(node.outputs, outs):
                    env[vid] = o
            for pos in self._destroys[i]:
                d = env.get(node.inputs[pos])
                if isinstance(d, DeviceArray):
                    self.pack_cache.invalidate(d.owner)

    def _copy_stream_for(self, cur):
        st = self._copy_streams.get(cur.device)
        if st is None:
            st = self._copy_streams[cur.device] = torch.cuda.Stream(device=cur.device)
        return st

    def node_times_ms(self):
        """Per-node device time of the last call (needs ``time_nodes=True``)."""
        if not self.node_events:
            return []
        torch.cuda.synchronize()
        return [(i, self.program.nodes[i].op, e0.elapsed_time(e1)) for i, e0, e1, _ in self.node_events]

    def node_stats(self):
        """(node index, op, device ms, bytes of device memory the node's operands span) of the
        last call (needs ``time_nodes=True``); a fused region is reported at its last node."""
        if not self.node_events:
            return []
        torch.cuda.synchronize()
        return [(i, self.program.nodes[i].op, e0.elapsed_time(e1), nb) for i, e0, e1, nb in self.node_events]


# ---------------------------------------------------------------------------
# node implementations
# ---------------------------------------------------------------------------
def _as_dev_inputs(ex, i, node, args):
    out = []
    for k, (vid, a) in enumerate(zip(node.inputs, args)):
        if isinstance(a, DeviceArray):
            out.append(a)
        elif vid in ex._const_host:
            out.append(ex.const_dev(vid))
        else:
            out.append(ex.dev(a, key=(i, k), dtype=ex.program.vars[vid].dtype))
    return out


@_op("Elemwise")
def _elemwise(ex, i, node, args):
    st = ex._state[i]
    p = node.params
    n_out = len(node.outputs)
    if all(is_host(a) for a in args) and st["host_ok"]:
        hargs = [np.asarray(a) for a in args]
        shape = np.broadcast_shapes(*[a.shape for a in hargs]) if hargs else ()
        size = int(np.prod(shape)) if shape else 1
        if size <= host_eval.MAX_HOST_ELEMS:
            outs = host_eval.eval_expr(p["expr"], hargs)
            outs = [np.array(np.broadcast_to(o, shape)) for o in outs]
            return outs[0] if n_out == 1 else outs
    ins = _as_dev_inputs(ex, i, node, args)
    shape = K.broadcast_shape(ins, node.label or "Elemwise")
    kern = st["kernel"]
    outs = []
    inplace = p.get("inplace", {})
    order = None
    for k in range(n_out):
        ip = inplace.get(str(k))
        dt = kern.out_dtypes[k]
        if ip is not None and ins[ip].shape == shape and ins[ip].dtype == dt and not is_host(args[ip]):
            outs.append(ins[ip])
        else:
            if order is None:
                order = K.elemwise_out_order(ins, shape)
            want = ex._out_storage.get(node.outputs[k]) if ex._out_storage else None
            if (want is not None and want.shape == tuple(shape) and want.dtype == dt and order == "C"
                    and want.is_c_contiguous()):
                outs.append(want)  # the caller's buffer (a row of a Scan output ring)
            else:
                outs.append(DeviceArray.empty(shape, dt, order=order))
    if all(n != 0 for n in shape) or not shape:
        kern.launch(shape, ins, outs)
    return outs[0] if n_out == 1 else outs


@_op("ScalarOp")
def _scalarop(ex, i, node, args):
    expr = node.params["expr"]
    if not host_eval.supports(expr):
        raise NotImplementedError(f"host scalar expression {expr.get('name')} is not supported")
    vals = [a.to_numpy() if isinstance(a, DeviceArray) else a for a in args]
    outs = host_eval.eval_expr(expr, vals)
    outs = [o.dtype.type(o.item()) for o in outs]
    return outs[0] if len(node.outputs) == 1 else outs


@_op("DimShuffle")
def _dimshuffle(ex, i, node, args):
    (x,) = args
    order = node.params["new_order"]
    if isinstance(x, DeviceArray):
        return x.dimshuffle(order)
    x = np.asarray(x)
    kept = [o for o in order if o != "x"]
    drop = [d for d in range(x.ndim) if d not in kept]
    for d in drop:
        if x.shape[d] != 1:
            raise ValueError("DimShuffle: cannot drop a non-broadcastable dimension")
    y = x.transpose(kept + drop)
    return y.reshape([1 if o == "x" else x.shape[o] for o in order])


_NP_REDUCE = {"add": np.add, "mul": np.multiply, "maximum": np.maximum, "minimum": np.minimum,
              "and": np.bitwise_and, "or": np.bitwise_or, "xor": np.bitwise_xor}


@_op("CAReduce")
def _careduce(ex, i, node, args):
    (x,) = args
    p = node.params
    axis = tuple(p["axis"])
    if is_host(x) and p["scalar_op"] not in _NP_REDUCE:
        x = ex.dev(np.asarray(x))
    if is_host(x):  # shape arithmetic such as prod(shape)
        xa = np.asarray(x).astype(p["acc_dtype"])
        out = _NP_REDUCE[p["scalar_op"]].reduce(xa, axis=axis, dtype=p["acc_dtype"]) if axis else xa
        return np.asarray(out).astype(p["out_dtype"])
    if p["scalar_op"] in ("maximum", "minimum") and any(x.shape[a] == 0 for a in axis):
        raise ValueError("zero-size array to reduction operation with no identity")
    if not axis:
        out = DeviceArray.empty(x.shape, p["out_dtype"])
        K.copy_into(out, x)
        return out
    return ex._state[i]["kernel"].launch(x, axis)


# -- row ops -------------------------------------------------------------------------
def _as_c_contiguous(x):
    return x if x.is_c_contiguous() else K.contiguous_copy(x)


@_op("Softmax")
def _softmax(ex, i, node, args):
    import ctypes as C

    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    p = node.params
    ins = [_as_c_contiguous(a) for a in _as_dev_inputs(ex, i, node, args)]
    x = ins[-1] if p["mode"] == 2 else ins[0]  # SoftmaxGrad(dy, sm): shapes agree
    if p["mode"] == 2 and ins[0].shape != ins[1].shape:
        raise ValueError(f"SoftmaxGrad: shapes {ins[0].shape} and {ins[1].shape} differ")
    if x.dtype.name not in ("float32", "float64"):
        raise TypeError(f"Softmax on dtype {x.dtype.name}")
    axis = p["axis"]
    if axis is None:
        outer, r, inner = 1, x.size, 1
    else:
        axis = axis % x.ndim
        outer = int(np.prod(x.shape[:axis])) if axis else 1
        r = x.shape[axis]
        inner = int(np.prod(x.shape[axis + 1:])) if axis + 1 < x.ndim else 1
    out = DeviceArray.empty(x.shape, x.dtype)
    a0 = ins[0].ptr
    a1 = ins[1].ptr if p["mode"] == 2 else None
    _lib.check(_lib.load().ab_softmax(DTYPE_CODE[x.dtype.name], p["mode"], outer, r, inner, a0, a1,
                                      out.ptr, stream_handle()))
    return out


@_op("MaxAndArgmax")
def _maxandargmax(ex, i, node, args):
    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    (x,) = _as_dev_inputs(ex, i, node, args)
    axes = node.params["axes"]
    keep = [d for d in range(x.ndim) if d not in axes]
    # kept axes in front, reduced axes flattened at the back (math.py:175-184)
    xt = x.dimshuffle(keep + list(axes)) if keep + list(axes) != list(range(x.ndim)) else x
    xt = _as_c_contiguous(xt)
    kept_shape = tuple(x.shape[d] for d in keep)
    outer = int(np.prod(kept_shape)) if kept_shape else 1
    r = int(np.prod([x.shape[d] for d in axes])) if axes else 1
    only_arg = node.params.get("argmax_only", False)
    omax = None if only_arg else DeviceArray.empty(kept_shape, x.dtype)
    oidx = DeviceArray.empty(kept_shape, "int64")
    _lib.check(_lib.load().ab_max_and_argmax(DTYPE_CODE[x.dtype.name], outer, r, xt.ptr,
                                             None if omax is None else omax.ptr, oidx.ptr,
                                             stream_handle()))
    return oidx if only_arg else [omax, oidx]


# -- BLAS family -------------------------------------------------------------------
def _scalar_value(v):
    if isinstance(v, DeviceArray):
        return v.item()  # device-resident alpha/beta: one D2H read
    return np.asarray(v).item()


def _fresh_like(x, shape=None):
    return DeviceArray.empty(x.shape if shape is None else shape, x.dtype)


@_op("Dot22")
def _dot22(ex, i, node, args):
    x, y = _as_dev_inputs(ex, i, node, args)
    if x.shape[1] != y.shape[0]:
        raise ValueError(f"Shape mismatch: x has {x.shape[1]} cols (and {x.shape[0]} rows) but y has "
                         f"{y.shape[0]} rows (and {y.shape[1]} cols)")
    z = DeviceArray.empty((x.shape[0], y.shape[1]), x.dtype)
    K.gemm(z, 1.0, x, y, 0.0, ex.precision, cache=ex.pack_cache, epilogue=ex._gemm_epilogue)
    return z


@_op("Dot22Scalar")
def _dot22scalar(ex, i, node, args):
    x, y = _as_dev_inputs(ex, i, node, args[:2])
    a = _scalar_value(args[2])
    if x.shape[1] != y.shape[0]:
        raise ValueError("Shape mismatch in Dot22Scalar")
    z = DeviceArray.empty((x.shape[0], y.shape[1]), x.dtype)
    K.gemm(z, a, x, y, 0.0, ex.precision, cache=ex.pack_cache, epilogue=ex._gemm_epilogue)
    return z


@_op("Gemm")
def _gemm(ex, i, node, args):
    z, a, x, y, b = args
    z, x, y = _as_dev_inputs(ex, i, Node("Gemm", [node.inputs[0], node.inputs[2], node.inputs[3]], []), [z, x, y])
    a, b = _scalar_value(a), _scalar_value(b)
    if x.shape[1] != y.shape[0]:
        raise ValueError(f"Shape mismatch: x has {x.shape[1]} cols (and {x.shape[0]} rows) but y has "
                         f"{y.shape[0]} rows (and {y.shape[1]} cols)")
    m, n = x.shape[0], y.shape[1]
    if z.shape != (m, n):
        if z.shape[0] in (1, m) and z.shape[1] in (1, n):  # z broadcast (blas.py:995-999)
            zz = DeviceArray.empty((m, n), z.dtype)
            K.copy_into(zz, z)
            z = zz
        else:
            raise ValueError(f"Shape mismatch: z has shape {z.shape} but x.y has shape {(m, n)}")
    elif not node.params["inplace"] or is_host(args[0]):
        # Gemm{no_inplace}: out = b*z + a*x.y without first copying z (blas.py:1065-1093
        # copies z into the output and calls BLAS with beta): the epilogue reads z directly
        out = DeviceArray.empty((m, n), z.dtype)
        K.gemm(out, a, x, y, b, ex.precision, cache=ex.pack_cache, cin=z, epilogue=ex._gemm_epilogue)
        return out
    K.gemm(z, a, x, y, b, ex.precision, cache=ex.pack_cache, epilogue=ex._gemm_epilogue)
    return z


@_op("Gemv")
def _gemv(ex, i, node, args):
    y, alpha, A, x, beta = args
    y, A, x = _as_dev_inputs(ex, i, Node("Gemv", [node.inputs[0], node.inputs[2], node.inputs[3]], []), [y, A, x])
    alpha, beta = _scalar_value(alpha), _scalar_value(beta)
    if A.shape[0] != y.shape[0] or A.shape[1] != x.shape[0]:
        raise ValueError(
            "Incompatible shapes for gemv "
            f"(beta * y + alpha * dot(A, x)). y: {y.shape}, A: {A.shape}, x: {x.shape}"
        )
    if not node.params["inplace"] or is_host(args[0]):
        yy = DeviceArray.empty(y.shape, y.dtype)
        if beta != 0.0:
            K.copy_into(yy, y)
        y = yy
    K.gemv(y, alpha, A, x, beta)
    return y


@_op("Ger")
def _ger(ex, i, node, args):
    A, alpha, x, y = args
    A, x, y = _as_dev_inputs(ex, i, Node("Ger", [node.inputs[0], node.inputs[2], node.inputs[3]], []), [A, x, y])
    alpha = _scalar_value(alpha)
    if A.shape != (x.shape[0], y.shape[0]):
        raise ValueError("Shape mismatch in Ger: A %s, x %s, y %s" % (A.shape, x.shape, y.shape))
    if not node.params["inplace"] or is_host(args[0]):
        A = K.contiguous_copy(A)
    K.ger(A, alpha, x, y)
    return A


@_op("Dot")
def _dot(ex, i, node, args):
    x, y = _as_dev_inputs(ex, i, node, args)
    # operands of two dtypes (float32 h times a float64 dropout-scaled mask) are upcast to the
    # output dtype first, as np.dot does (tensor/math.py:1879); the products take one dtype
    dt = np.dtype(ex.program.vars[node.outputs[0]].dtype)
    if x.dtype != dt:
        x = K.cast_copy(x, dt)
    if y.dtype != dt:
        y = K.cast_copy(y, dt)
    if x.ndim == 1 and y.ndim == 1:
        if x.shape != y.shape:
            raise ValueError(f"shapes {x.shape} and {y.shape} not aligned")
        out = DeviceArray.empty((1,), x.dtype)
        K.gemv(out, 1.0, x.view((1, x.shape[0]), (0, x.strides[0])), y, 0.0)
        return out.view((), ())
    if x.ndim == 2 and y.ndim == 1:
        out = DeviceArray.empty((x.shape[0],), x.dtype)
        K.gemv(out, 1.0, x, y, 0.0)
        return out
    if x.ndim == 1 and y.ndim == 2:
        out = DeviceArray.empty((y.shape[1],), x.dtype)
        K.gemv(out, 1.0, y.dimshuffle([1, 0]), x, 0.0)
        return out
    if x.ndim == 2 and y.ndim == 2:
        z = DeviceArray.empty((x.shape[0], y.shape[1]), x.dtype)
        K.gemm(z, 1.0, x, y, 0.0, ex.precision, cache=ex.pack_cache, epilogue=ex._gemm_epilogue)
        return z
    raise NotImplementedError("Dot with ndim > 2")


# -- allocation / copies ---------------------------------------------------------------
def _int(v):
    if isinstance(v, DeviceArray):
        return int(v.item())
    return int(np.asarray(v).item())


@_op("AllocEmpty")
def _allocempty(ex, i, node, args):
    return DeviceArray.empty([_int(s) for s in args], node.params["dtype"])


@_op("Alloc")
def _alloc(ex, i, node, args):
    v, *shape = args
    shape = [_int(s) for s in shape]
    vid = node.inputs[0]
    var = ex.program.vars[node.outputs[0]]
    n = int(np.prod(shape)) if shape else 1
    if is_host(v) and n <= host_eval.MAX_HOST_ELEMS:
        return np.array(np.broadcast_to(np.asarray(v, dtype=var.dtype), shape))
    src = v if isinstance(v, DeviceArray) else (
        ex.const_dev(vid) if vid in ex._const_host else ex.dev(v, key=(i, 0), dtype=var.dtype))
    out = DeviceArray.empty(shape, var.dtype)
    K.copy_into(out, src)
    return out


@_op("BroadcastTo")
def _broadcast_to(ex, i, node, args):
    v, *shape = args
    shape = [_int(s) for s in shape]
    vid = node.inputs[0]
    var = ex.program.vars[node.outputs[0]]
    n = int(np.prod(shape)) if shape else 1
    if is_host(v) and n <= host_eval.MAX_HOST_ELEMS:
        return np.broadcast_to(np.asarray(v, dtype=var.dtype), shape)
    src = v if isinstance(v, DeviceArray) else (
        ex.const_dev(vid) if vid in ex._const_host else ex.dev(v, key=(i, 0), dtype=var.dtype))
    return src.broadcast_to(shape)


@_op("DeepCopy")
def _deepcopy(ex, i, node, args):
    (x,) = args
    if isinstance(x, DeviceArray):
        return K.contiguous_copy(x)
    return np.array(x, copy=True)


@_op("View")
def _view(ex, i, node, args):
    return args[0]


@_op("Reshape")
def _reshape(ex, i, node, args):
    x, shp = args
    shp = [int(s) for s in (shp.to_numpy() if isinstance(shp, DeviceArray) else np.asarray(shp)).reshape(-1)]
    if is_host(x):
        return np.reshape(x, shp)
    if not x.is_c_contiguous():
        x = K.contiguous_copy(x)
    return x.reshape_view(shp)


# -- host metadata ----------------------------------------------------------------------
@_op("Shape_i")
def _shape_i(ex, i, node, args):
    (x,) = args
    return np.asarray(np.shape(x)[node.params["i"]] if is_host(x) else x.shape[node.params["i"]],
                      dtype="int64")


@_op("Shape")
def _shape(ex, i, node, args):
    (x,) = args
    return np.asarray(np.shape(x) if is_host(x) else x.shape, dtype="int64")


@_op("ScalarFromTensor")
def _sft(ex, i, node, args):
    (x,) = args
    a = x.to_numpy() if isinstance(x, DeviceArray) else np.asarray(x)
    return a.dtype.type(a.item())


@_op("TensorFromScalar")
def _tfs(ex, i, node, args):
    return np.asarray(args[0])


@_op("MakeVector")
def _makevector(ex, i, node, args):
    vals = [a.item() if isinstance(a, DeviceArray) else np.asarray(a).item() for a in args]
    return np.asarray(vals, dtype=node.params["dtype"]).reshape(len(vals))


@_op("Assert")
def _assert(ex, i, node, args):
    val, *conds = args
    for c in conds:
        c = c.to_numpy() if isinstance(c, DeviceArray) else np.asarray(c)
        if not bool(np.all(c)):
            exc = {"ValueError": ValueError, "TypeError": TypeError}.get(node.params.get("exc"), AssertionError)
            raise exc(node.params["msg"])
    return val


# -- indexing -----------------------------------------------------------------------------
def _build_index(idx_list, runtime):
    it = iter(runtime)

    def elem(e):
        if e is None:
            return None
        if e == "in":
            return _int(next(it))
        return int(e)

    out = []
    for entry in idx_list:
        if "slice" in entry:
            out.append(slice(*[elem(e) for e in entry["slice"]]))
        else:
            out.append(elem(entry["index"]))
    return tuple(out)


@_op("Subtensor")
def _subtensor(ex, i, node, args):
    x, *rt = args
    idx = _build_index(node.params["idx_list"], rt)
    if is_host(x):
        return np.asarray(x)[idx]
    return x.index(idx)


@_op("IncSubtensor")
def _incsubtensor(ex, i, node, args):
    x, y, *rt = args
    p = node.params
    idx = _build_index(p["idx_list"], rt)
    if is_host(x) and is_host(y):
        x = np.array(x, copy=True)
        if p["set"]:
            x[idx] = y
        else:
            x[idx] += y
        return x
    vx = ex.program.vars[node.inputs[0]]
    xd = x if isinstance(x, DeviceArray) else ex.dev(x, dtype=vx.dtype)
    if not p["inplace"] or is_host(x):
        xd = K.contiguous_copy(xd)
    yd = y if isinstance(y, DeviceArray) else ex.dev(y, key=(i, 1), dtype=ex.program.vars[node.inputs[1]].dtype)
    view = xd.index(idx)
    if p["set"]:
        K.copy_into(view, yd)
    else:
        K.add_into(view, yd)
    return xd


def _rows_view(x):
    """x as [n_rows, inner] with a contiguous inner part (copy if needed)."""
    inner = 1
    for s in x.shape[1:]:
        inner *= s
    tail_contig = x.view(x.shape[1:], x.strides[1:]).is_c_contiguous() if x.ndim > 1 else True
    if not tail_contig:
        x = K.contiguous_copy(x)
    row_stride = x.strides[0] if x.shape[0] > 1 else max(inner, 1)
    return x, inner, row_stride


@_op("AdvancedSubtensor1")
def _advsub1(ex, i, node, args):
    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    x, idx = args
    if is_host(x) and is_host(idx):
        return np.take(np.asarray(x), np.asarray(idx), axis=0)
    x, idx = _as_dev_inputs(ex, i, node, [x, idx])
    if idx.ndim != 1:
        raise IndexError("AdvancedSubtensor1 needs a vector of indices")
    if idx.dtype.kind not in "iu":
        raise IndexError("index must be integers")
    x, inner, row_stride = _rows_view(x)
    out = DeviceArray.empty((idx.shape[0],) + x.shape[1:], x.dtype)
    try:
        _lib.check(_lib.load().ab_take_rows(x.itemsize, DTYPE_CODE[idx.dtype.name], x.ptr,
                                            row_stride, x.shape[0], inner, idx.ptr, idx.strides[0],
                                            idx.shape[0], out.ptr, 1, stream_handle()))
    except _lib.AbError as e:
        if e.code == 4:
            raise IndexError(str(e)) from None
        raise
    return out


def _ravel_indices(ex, i, node, x, idx_args):
    """k integer index vectors over the k leading dims of x -> (flat int64 row index on the
    device, x viewed as [prod(dims), *rest]) (``ab_ravel_index``)."""
    import ctypes as C

    from . import lib as _lib
    from .device import stream_handle

    k = len(idx_args)
    if k > x.ndim:
        raise IndexError(f"too many indices for array: array is {x.ndim}-dimensional, but {k} were indexed")
    idxs = []
    for a in idx_args:
        a = a if isinstance(a, DeviceArray) else ex.dev(np.atleast_1d(np.asarray(a)))
        if a.ndim == 0:
            a = a.reshape_view((1,))
        if a.ndim != 1 or a.dtype.kind not in "iu":
            raise IndexError("arrays used as indices must be integer vectors")
        if a.dtype != np.int64:
            a64 = DeviceArray.empty(a.shape, "int64")
            K.copy_into(a64, a)
            a = a64
        idxs.append(a)
    n = max(a.shape[0] for a in idxs)
    for a in idxs:
        if a.shape[0] not in (1, n):
            raise IndexError("shape mismatch: indexing arrays could not be broadcast together")
    dims = x.shape[:k]
    flat = DeviceArray.empty((n,), "int64")
    ptrs = (C.c_void_p * k)(*[a.ptr for a in idxs])
    strides = (C.c_int64 * k)(*[0 if a.shape[0] == 1 and n != 1 else a.strides[0] for a in idxs])
    cd = (C.c_int64 * k)(*dims)
    try:
        _lib.check(_lib.load().ab_ravel_index(k, ptrs, strides, cd, n, flat.ptr, 1, stream_handle()))
    except _lib.AbError as e:
        if e.code == 4:
            raise IndexError(str(e)) from None
        raise
    rows = 1
    for d in dims:
        rows *= d
    return flat, rows, n


@_op("AdvancedSubtensor")
def _advsub(ex, i, node, args):
    x, *idx = args
    if is_host(x) and all(is_host(a) for a in idx):
        return np.asarray(x)[tuple(np.asarray(a) for a in idx)]
    (x,) = _as_dev_inputs(ex, i, Node("AdvancedSubtensor", [node.inputs[0]], []), [x])
    k = len(idx)
    xc = _as_c_contiguous(x)
    flat, rows, n = _ravel_indices(ex, i, node, xc, idx)
    rest = xc.shape[k:]
    x2 = xc.reshape_view((rows,) + rest)
    out = _EXEC["AdvancedSubtensor1"](ex, i, Node("AdvancedSubtensor1", node.inputs[:2], node.outputs), [x2, flat])
    return out


@_op("AdvancedIncSubtensor")
def _advincsub(ex, i, node, args):
    p = node.params
    xa, ya, *idx = args
    x, y = _as_dev_inputs(ex, i, Node("AdvancedIncSubtensor", node.inputs[:2], []), [xa, ya])
    k = len(idx)
    if not p["inplace"] or is_host(xa) or not x.is_c_contiguous():
        x = K.contiguous_copy(x)
    flat, rows, n = _ravel_indices(ex, i, node, x, idx)
    rest = x.shape[k:]
    x2 = x.reshape_view((rows,) + rest)
    sub = Node("AdvancedIncSubtensor1", node.inputs[:3], node.outputs,
               {"inplace": True, "set": p["set"], "ignore_duplicates": p.get("ignore_duplicates", False)})
    _EXEC["AdvancedIncSubtensor1"](ex, i, sub, [x2, y, flat])
    return x


@_op("BatchedDot")
def _batched_dot(ex, i, node, args):
    x, y = _as_dev_inputs(ex, i, node, args)
    if x.shape[0] != y.shape[0]:
        raise TypeError(f"Inputs must have the same size in axis 0, but have sizes [{x.shape[0]}, {y.shape[0]}].")
    nb = x.shape[0]
    xm = x if x.ndim == 3 else x.view((nb, 1, x.shape[1]), (x.strides[0], 0, x.strides[1]))
    ym = y if y.ndim == 3 else y.view((nb, y.shape[1], 1), (y.strides[0], y.strides[1], 0))
    if xm.shape[2] != ym.shape[1]:
        raise ValueError(f"Shape mismatch: x has {xm.shape[2]} cols but y has {ym.shape[1]} rows")
    m, n = xm.shape[1], ym.shape[2]
    out = DeviceArray.empty((nb, m, n), x.dtype)
    for b in range(nb):  # one product per batch entry (tensor-core path when large enough)
        K.gemm(out.index((b,)), 1.0, xm.index((b,)), ym.index((b,)), 0.0, ex.precision, cache=ex.pack_cache)
    shape = (nb,) + ((m,) if x.ndim == 3 else ()) + ((n,) if y.ndim == 3 else ())
    return out.reshape_view(shape)


@_op("IfElse")
def _ifelse(ex, i, node, args):
    n = node.params["n_outs"]
    c = args[0]
    cond = bool(np.asarray(c.to_numpy() if isinstance(c, DeviceArray) else c).item())
    vals = args[1 : 1 + n] if cond else args[1 + n : 1 + 2 * n]
    return vals[0] if n == 1 else list(vals)


@_op("CumOp")
def _cumop(ex, i, node, args):
    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    (x,) = args
    p = node.params
    if is_host(x):
        xa = np.asarray(x)
        f = np.cumsum if p["mode"] == "add" else np.cumprod
        return f(xa, axis=p["axis"], dtype=xa.dtype)
    x = _as_c_contiguous(x)
    axis = p["axis"]
    if axis is None:
        shape, outer, L, inner = (x.size,), 1, x.size, 1
    else:
        axis %= x.ndim
        shape = x.shape
        outer = int(np.prod(shape[:axis], dtype=np.int64)) if axis else 1
        L = shape[axis]
        inner = int(np.prod(shape[axis + 1:], dtype=np.int64)) if axis + 1 < x.ndim else 1
    out = DeviceArray.empty(shape, x.dtype)
    if x.dtype == np.bool_:
        raise TypeError("CumOp on bool arrays is not implemented on the device")
    _lib.check(_lib.load().ab_cumulative(DTYPE_CODE[x.dtype.name], 1 if p["mode"] == "mul" else 0, x.ptr,
                                         out.ptr, outer, L, inner, stream_handle()))
    return out


@_op("ExtractDiag")
def _extract_diag(ex, i, node, args):
    (x,) = args
    p = node.params
    if is_host(x):
        return np.array(np.asarray(x).diagonal(p["offset"], p["axis1"], p["axis2"]), copy=True)
    d = x.diagonal(p["offset"], p["axis1"], p["axis2"])
    return d if p["view"] else K.contiguous_copy(d)


@_op("AllocDiag")
def _alloc_diag(ex, i, node, args):
    (v,) = args
    k = node.params["offset"]
    if is_host(v):
        return np.diag(np.asarray(v), k)
    n = v.shape[0] + abs(k)
    out = DeviceArray.empty((n, n), v.dtype)
    K.copy_into(out, ex.dev(np.zeros((1, 1), v.dtype), key=(i, "zero")))
    if v.shape[0]:
        K.copy_into(out.diagonal(k), v)
    return out


_TRI_EXPR = {}


@_op("Tri")
def _tri(ex, i, node, args):
    """``np.tri(N, M, k)``: out[r, c] = (c <= r + k), evaluated by one generated Elemwise
    kernel over a row-index column and a column-index row (both from ``ab_arange``)."""
    n, m, k = (int(np.asarray(a.to_numpy() if isinstance(a, DeviceArray) else a).item()) for a in args)
    dt = np.dtype(node.params["dtype"])
    if n * m <= host_eval.MAX_HOST_ELEMS:
        return np.tri(n, m, k, dtype=dt)
    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    rows = DeviceArray.empty((n,), "int64")
    cols = DeviceArray.empty((m,), "int64")
    lib = _lib.load()
    _lib.check(lib.ab_arange(DTYPE_CODE["int64"], 0.0, 1.0, k, 1, n, rows.ptr, stream_handle()))   # r + k
    _lib.check(lib.ab_arange(DTYPE_CODE["int64"], 0.0, 1.0, 0, 1, m, cols.ptr, stream_handle()))
    expr = _TRI_EXPR.get(dt.name)
    if expr is None:
        expr = _TRI_EXPR[dt.name] = {
            "inputs": ["int64", "int64"], "out_dtypes": [dt.name], "outputs": ["t1"], "name": f"tri_{dt.name}",
            "stmts": [{"op": "le", "args": ["i1", "i0"], "dtype": "bool", "in_dtypes": ["int64", "int64"]},
                      {"op": "cast", "args": ["t0"], "dtype": dt.name, "in_dtypes": ["bool"]}]}
    out = DeviceArray.empty((n, m), dt)
    r2 = rows.view((n, 1), (rows.strides[0], 0))
    c2 = cols.view((1, m), (0, cols.strides[0]))
    K.ElemwiseKernel.get(expr).launch((n, m), [r2, c2], [out])
    return out


@_op("Eye")
def _eye(ex, i, node, args):
    n, m, k = (int(np.asarray(a.to_numpy() if isinstance(a, DeviceArray) else a).item()) for a in args)
    dt = np.dtype(node.params["dtype"])
    if n * m <= host_eval.MAX_HOST_ELEMS:
        return np.eye(n, m, k, dtype=dt)
    out = DeviceArray.empty((n, m), dt)
    K.copy_into(out, ex.dev(np.zeros((1, 1), dt), key=(i, "zero")))
    diag = out.diagonal(k)
    if diag.size:
        K.copy_into(diag, ex.dev(np.ones((1,), dt), key=(i, "one")))
    return out


@_op("ARange")
def _arange(ex, i, node, args):
    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    vals = []
    for a in args:
        vals.append(np.asarray(a.to_numpy() if isinstance(a, DeviceArray) else a).item())
    start, stop, step = vals
    dt = np.dtype(node.params["dtype"])
    host = np.arange(start, stop, step, dtype=dt) if (abs(stop - start) / max(abs(step), 1e-300)) <= host_eval.MAX_HOST_ELEMS else None
    if host is not None:
        return host
    n = len(range(int(start), int(stop), int(step))) if dt.kind in "iu" else int(np.ceil((stop - start) / step))
    n = max(n, 0)
    out = DeviceArray.empty((n,), dt)
    _lib.check(_lib.load().ab_arange(DTYPE_CODE[dt.name], float(start), float(step), int(start), int(step),
                                     n, out.ptr, stream_handle()))
    return out


@_op("AdvancedIncSubtensor1")
def _advincsub1(ex, i, node, args):
    import ctypes as C

    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    p = node.params
    xa, ya, ia = args
    x, y, idx = _as_dev_inputs(ex, i, node, [xa, ya, ia])
    if idx.ndim != 1 or idx.dtype.kind not in "iu":
        raise IndexError("AdvancedIncSubtensor1 needs an integer vector of indices")
    if idx.dtype.name not in ("int32", "int64"):
        idx64 = DeviceArray.empty(idx.shape, "int64")
        K.copy_into(idx64, idx)
        idx = idx64
    if not p["inplace"] or is_host(xa) or not x.view(x.shape[1:], x.strides[1:]).is_c_contiguous():
        x = K.contiguous_copy(x)
    inner = 1
    for s in x.shape[1:]:
        inner *= s
    row_stride = x.strides[0] if x.shape[0] > 1 else max(inner, 1)
    # y broadcasts against x[idx] (shape [n_idx] + x.shape[1:])
    want = (idx.shape[0],) + x.shape[1:]
    if y.ndim < len(want):
        y = y.view((1,) * (len(want) - y.ndim) + y.shape, (0,) * (len(want) - y.ndim) + y.strides)
    for d, (ys, ws) in enumerate(zip(y.shape, want)):
        if ys not in (1, ws):
            raise ValueError(f"shape mismatch: value array of shape {y.shape} could not be broadcast "
                             f"to indexing result of shape {want}")
    if y.dtype != x.dtype:
        yy = DeviceArray.empty(y.shape, x.dtype)
        K.copy_into(yy, y)
        y = yy
    # flatten y's trailing dims into one strided "column" index when possible, else materialise
    yb = DeviceArray.empty(want, x.dtype)
    K.copy_into(yb, y)
    y_rs, y_cs = (inner, 1)
    # set: the last occurrence of a row wins (x[idx] = y); ignore_duplicates (from
    # AdvancedIncSubtensor): x[d] + y[last occurrence] (out[idx] += y); else np.add.at
    mode = 1 if p["set"] else (2 if p.get("ignore_duplicates") else 0)
    lib = _lib.load()
    ws_bytes = C.c_size_t()
    _lib.check(lib.ab_scatter_rows_workspace_bytes(mode, x.shape[0], C.byref(ws_bytes)))
    ws = DeviceArray.empty((ws_bytes.value,), "uint8") if ws_bytes.value else None
    try:
        _lib.check(lib.ab_scatter_rows(DTYPE_CODE[x.dtype.name], DTYPE_CODE[idx.dtype.name], mode,
                                       x.ptr, row_stride, x.shape[0], inner, idx.ptr, idx.strides[0],
                                       idx.shape[0], yb.ptr, y_rs, y_cs,
                                       ws.ptr if ws is not None else None, ws_bytes.value, 1,
                                       stream_handle()))
    except _lib.AbError as e:
        if e.code == 4:
            raise IndexError(str(e)) from None
        raise
    return x


@_op("Join")
def _join(ex, i, node, args):
    axis, *tensors = args
    axis = _int(axis)
    if all(is_host(t) for t in tensors):
        return np.concatenate([np.asarray(t) for t in tensors], axis=axis)
    ts = _as_dev_inputs(ex, i, Node("Join", list(node.inputs[1:]), []), tensors)
    nd = ts[0].ndim
    if axis < -nd or axis >= nd:
        raise IndexError(f"Join axis {axis} out of bounds [0, {nd})")
    axis %= nd
    shape = list(ts[0].shape)
    for t in ts[1:]:
        if t.ndim != nd or any(t.shape[d] != shape[d] for d in range(nd) if d != axis):
            raise ValueError("all the input array dimensions except for the concatenation axis must "
                             "match exactly")
    shape[axis] = sum(t.shape[axis] for t in ts)
    out = DeviceArray.empty(shape, ex.program.vars[node.outputs[0]].dtype)
    start = 0
    for t in ts:
        n = t.shape[axis]
        sl = [slice(None)] * nd
        sl[axis] = slice(start, start + n)
        if n:
            K.copy_into(out.index(tuple(sl)), t)
        start += n
    return out


@_op("Split")
def _split(ex, i, node, args):
    x, axis, splits = args
    axis = _int(axis)
    splits = [int(s) for s in (splits.to_numpy() if isinstance(splits, DeviceArray) else np.asarray(splits)).reshape(-1)]
    if len(splits) != node.params["len_splits"]:
        raise ValueError("Split: wrong number of split sizes")
    if is_host(x):
        x = np.asarray(x)
        if sum(splits) != x.shape[axis]:
            raise ValueError("Split: the split sizes do not sum to the input length along the axis")
        outs, start = [], 0
        for s in splits:
            sl = [slice(None)] * x.ndim
            sl[axis] = slice(start, start + s)
            outs.append(np.array(x[tuple(sl)]))
            start += s
        return outs[0] if len(outs) == 1 else outs
    axis %= x.ndim
    if sum(splits) != x.shape[axis] or any(s < 0 for s in splits):
        raise ValueError("Split: the split sizes do not sum to the input length along the axis")
    outs, start = [], 0
    for s in splits:
        sl = [slice(None)] * x.ndim
        sl[axis] = slice(start, start + s)
        outs.append(K.contiguous_copy(x.index(tuple(sl))))  # Split has no view_map: fresh buffers
        start += s
    return outs[0] if len(outs) == 1 else outs


@_op("Scan")
def _scan(ex, i, node, args):
    outs = ex._state[i]["runner"].run(args)
    return outs[0] if len(node.outputs) == 1 else outs


# -- random variables ---------------------------------------------------------------------
_RNG_DIST = {"uniform": 0, "normal": 1, "bernoulli": 2}


def _random_shape(size, pshapes):
    """``size`` if given (non-empty), else the broadcast parameter shape; the parameters must
    broadcast to it (NumPy's rule for ``Generator.uniform(..., size=...)``)."""
    size = tuple(int(s) for s in np.asarray(size).reshape(-1))
    shape = size if size else tuple(np.broadcast_shapes(*pshapes))
    try:
        full = tuple(np.broadcast_shapes(shape, *pshapes))
    except ValueError:
        full = None
    if full != shape:
        raise ValueError(f"shape mismatch: parameters of shapes {list(pshapes)} cannot be broadcast to size {shape}")
    return shape


def _check_host_param(dist, k, h):
    if dist == "normal" and k == 1 and np.any(h < 0):
        raise ValueError("scale < 0")
    if dist == "bernoulli" and not np.all((h >= 0) & (h <= 1)):
        raise ValueError("p < 0, p > 1 or p is NaN")


@_op("RandomVariable")
def _random_variable(ex, i, node, args):
    """RandomVariable (aesara/tensor/random/op.py:344 perform): the Generator is host state.
    It is drawn from in place when the Op is in place and copied first otherwise, exactly as
    the reference does, but it gives up one 64-bit key per call, which keys the device's
    Philox stream (csrc/ab_random.cu).  Parameters known on the host are checked there;
    device-resident ones by the kernel's error flag (one synchronisation)."""
    import ctypes as C

    from ..ir import DTYPE_CODE
    from . import lib as _lib
    from .device import stream_handle

    p = node.params
    dist = p["dist"]
    rng, size, _dtype, *params = args
    n_par = 1 if dist == "bernoulli" else 2
    params, pvids = params[-n_par:], node.inputs[-n_par:]
    pdt = np.dtype("float64" if dist == "bernoulli" else p["dtype"])
    if isinstance(size, DeviceArray):
        size = size.to_numpy()
    shape = _random_shape(size, [a.shape if isinstance(a, DeviceArray) else np.shape(a) for a in params])
    st = ex._state[i]
    views, check = [], 0
    for k, (vid, a) in enumerate(zip(pvids, params)):
        if isinstance(a, DeviceArray):
            if a.dtype != pdt:
                a = K.cast_copy(a, pdt)
            check = 1
        else:
            h = np.asarray(a).astype(pdt)  # the parameters take the output dtype first
            _check_host_param(dist, k, h)
            if vid in ex._const_host:
                d = st.get(("param", k))
                if d is None:
                    d = st[("param", k)] = DeviceArray.from_numpy(h)
                a = d
            else:
                a = ex.dev(h, key=(i, k))
        views.append(a.broadcast_to(shape))
    if not p["inplace"]:
        rng = copy.copy(rng)
    # one key per node and call: for full-range uint64 this is exactly one raw draw
    key = int(rng.integers(0, 2 ** 64, dtype=np.uint64))
    out = DeviceArray.empty(shape, p["dtype"])
    nd = len(shape)
    shp = (C.c_int64 * max(nd, 1))(*shape)
    ptrs = (C.c_void_p * n_par)(*[v.ptr for v in views])
    strides = (C.c_int64 * max(nd * n_par, 1))(*[s for v in views for s in v.strides])
    try:
        _lib.check(_lib.load().ab_random(_RNG_DIST[dist], DTYPE_CODE[p["dtype"]], key, nd, shp, n_par, ptrs,
                                         strides, out.ptr, check, stream_handle()))
    except _lib.AbError as e:
        if e.code == 3:
            raise ValueError(str(e)) from None
        raise
    return [rng, out]


# -- dense linear algebra ------------------------------------------------------------------
def _linalg_operands(ex, i, node, args):
    """The node's operands on the device in its output dtype (the reference computes in the
    dtype its make_node gives the output: float32 only when every operand is float32), with
    the shape checks of scipy.linalg."""
    dt = np.dtype(ex.program.vars[node.outputs[0]].dtype)
    out = []
    for x in _as_dev_inputs(ex, i, node, args):
        out.append(x if x.dtype == dt else K.cast_copy(x, dt))
    a = out[0]
    if a.ndim != 2 or a.shape[0] != a.shape[1]:
        raise ValueError(f"expected square matrix, got shape {a.shape}")
    if len(out) > 1 and out[1].shape[0] != a.shape[0]:
        raise ValueError(f"shapes of a {a.shape} and b {out[1].shape} are incompatible")
    return out


@_op("Cholesky")
def _cholesky(ex, i, node, args):
    """Cholesky (aesara/tensor/slinalg.py:64 perform): scipy.linalg.cholesky checks finiteness
    always; a matrix that is not positive definite raises LinAlgError, or gives an all-NaN
    factor under on_error="nan"."""
    (a,) = _linalg_operands(ex, i, node, args)
    nan = node.params["on_error"] == "nan"
    status = K.LinalgStatus()
    out = K.cholesky(a, node.params["lower"], status, nan_on_error=nan)
    status.check(nan_on_error=nan)
    return out


@_op("SolveTriangular")
def _solve_triangular(ex, i, node, args):
    """SolveTriangular (slinalg.py:301 perform, scipy.linalg.solve_triangular): trans 2 is 1
    for real data; a zero diagonal of a non-unit system raises LinAlgError."""
    a, b = _linalg_operands(ex, i, node, args)
    p = node.params
    status = K.LinalgStatus()
    x = K.trsm(a, b, p["lower"], p["trans"] != 0, p["unit_diagonal"], status, check_finite=p["check_finite"])
    if p["check_finite"] or not p["unit_diagonal"]:
        status.check()
    return x


def _cholesky_solves(a, b, status, check_finite):
    """x with L L^T x = b for the lower factor ``a``: two triangular solves, the second in place;
    like LAPACK potrs, the diagonal is not tested."""
    y = K.trsm(a, b, True, False, False, status, check_finite=check_finite, check_singular=False)
    return K.trsm(a, y, True, True, False, status, check_finite=False, check_singular=False, out=y)


@_op("CholeskySolve")
def _cholesky_solve(ex, i, node, args):
    """CholeskySolve (slinalg.py:158 perform, scipy.linalg.cho_solve): C holds the lower factor
    (lower) or the upper one, which is the lower factor of C^T."""
    c, b = _linalg_operands(ex, i, node, args)
    p = node.params
    status = K.LinalgStatus()
    x = _cholesky_solves(c if p["lower"] else c.dimshuffle([1, 0]), b, status, p["check_finite"])
    if p["check_finite"]:
        status.check()
    return x


@_op("Solve")
def _solve(ex, i, node, args):
    """Solve(assume_a="pos") (slinalg.py:388 perform, scipy.linalg.solve): the Cholesky factor
    of the symmetric matrix built from the named triangle, then two triangular solves."""
    a, b = _linalg_operands(ex, i, node, args)
    p = node.params
    status = K.LinalgStatus()
    # the upper triangle of a is the lower triangle of a^T
    factor = K.cholesky(a if p["lower"] else a.dimshuffle([1, 0]), True, status, check_finite=p["check_finite"])
    x = _cholesky_solves(factor, b, status, p["check_finite"])
    status.check()
    return x
