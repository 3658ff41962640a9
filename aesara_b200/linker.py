"""``B200Linker`` — the drop-in boundary (SURVEY.md §8b).

A subclass of ``aesara.link.basic.LocalLinker`` (``aesara/link/basic.py:240``):
``accept(fgraph, no_recycling, profile)`` then ``make_all(input_storage,
output_storage, storage_map) -> (fn, [Container in], [Container out], thunks,
order)``, the contract ``FunctionMaker`` drives (``compile/function/types.py:1586-1595,
1708``) and ``VMLinker.make_all`` implements for the C-linker
(``aesara/link/vm.py:1212-1324``).  Any graph compiles unchanged::

    import aesara_b200
    f = aesara.function([x, y], out, mode="B200")           # or mode=aesara_b200.mode()

The returned ``fn`` reproduces the VM semantics ``Function.__call__`` relies on
(``types.py:969-1048``): reads the input cells, writes the output cells, applies
the ``update_mapping`` output->input copies itself (``need_update_inputs = False``,
``vm.py:284-335``), exposes ``allow_gc``, ``storage_map``, ``nodes``, ``thunks`` and
``position_of_error`` so errors are re-raised through ``raise_with_op``.

Inputs may be NumPy arrays (uploaded each call, like any host-typed linker) or
``DeviceArray``s when ``Function.trust_input`` is set (SURVEY.md F7); outputs are
NumPy arrays by default, device arrays with ``device_outputs=True``.
"""

from __future__ import annotations

from copy import copy

import numpy as np

from .compat.bootstrap import load_aesara

load_aesara()

from aesara.compile.mode import Mode, predefined_linkers, predefined_modes, register_linker  # noqa: E402
from aesara.graph.rewriting.db import RewriteDatabaseQuery  # noqa: E402
from aesara.link.basic import Container, LocalLinker  # noqa: E402
from aesara.link.utils import map_storage  # noqa: E402

from .lower import lower_fgraph  # noqa: E402


class _NodeThunk:
    """Per-node placeholder kept for ``raise_with_op`` (``link/utils.py:270``)."""

    lazy = False

    def __init__(self, node, storage_map):
        self.inputs = [storage_map[v] for v in node.inputs]
        self.outputs = [storage_map[v] for v in node.outputs]


class B200VM:
    """The callable returned by :meth:`B200Linker.make_all` — what ``VM``/``CVM`` is to
    ``VMLinker`` (``aesara/link/vm.py:86-335, 1005-1174``)."""

    need_update_inputs = False

    def __init__(self, linker, fgraph, order, executor, input_storage, output_storage, storage_map):
        self.fgraph = fgraph
        self.nodes = order
        self.executor = executor
        self.input_storage = input_storage
        self.output_storage = output_storage
        self.storage_map = storage_map
        self.thunks = [_NodeThunk(n, storage_map) for n in order]
        self.allow_gc = linker.allow_gc
        self.position_of_error = -1
        self.call_counts = [0] * len(order)
        self.call_times = [0.0] * len(order)
        # cells the caller forbids us to recycle between calls are emptied first
        # (VMLinker.make_vm: pre_call_clear, vm.py:1017; Loop.__call__ vm.py:408-409)
        self.pre_call_clear = [storage_map[v] for v in (linker.no_recycling or []) if v in storage_map]
        upd = getattr(fgraph, "update_mapping", None) or {}
        self._updates = [(int(o), int(i)) for o, i in upd.items()]
        # FunctionMaker appends the update expressions after the user's outputs
        # (compile/function/types.py:1422-1432): those trailing outputs are never returned
        n_out = len(output_storage)
        self._updates_trail = sorted(o for o, _ in self._updates) == list(range(n_out - len(self._updates), n_out))
        self._host_out = not linker.device_outputs
        self.time_thunks = bool(getattr(linker, "profile", None))
        if self.time_thunks and hasattr(executor, "time_nodes"):
            executor.time_nodes = True
        self._replay = None
        if linker.cuda_graph and not self.time_thunks:
            # with shard="rows" the captured evaluation includes the NCCL all-reduces and the
            # side-stream fork/join of shard.ShardedExecutor (every rank captures and replays in
            # lock step: one cudaGraphLaunch per rank per evaluation)
            from .runtime.graph import GraphReplay

            self._replay = GraphReplay(executor)

    def __call__(self, output_subset=None):
        from .runtime.vm import NodeError
        from .sharedvar import is_device_value, owns_cell

        for cell in self.pre_call_clear:
            cell[0] = None
        args = [cell[0] for cell in self.input_storage]
        try:
            if output_subset is not None:
                # only the ancestors of the requested outputs (and of every update) run
                # (Stack.__call__, vm.py:536-563)
                outs = self.executor(*args, output_subset=output_subset)
            elif self._replay is not None and all(
                    is_device_value(a) or np.size(a) <= 64 for a in args):
                # device-resident arguments only: host arrays are uploaded by a copy stream,
                # which is not part of a captured evaluation
                outs = self._replay(*args)
            else:
                outs = self.executor(*args)
        except NodeError as e:
            self.position_of_error = e.position
            # raise_with_op reads shapes / strides / small values of the failing node's
            # inputs out of the thunk's cells (link/utils.py:340-356)
            if e.inputs is not None:
                for cell, val in zip(self.thunks[e.position].inputs, e.inputs):
                    if cell[0] is None:
                        cell[0] = val
            raise e.original from None
        finally:
            self._collect_times()
        dev_outs = list(outs)
        if self._host_out:
            # a trailing update output that feeds a device-resident shared variable is
            # never returned to the caller: do not download it
            keep_dev = set()
            if self._updates_trail:
                keep_dev = {o for o, i in self._updates if owns_cell(self.input_storage[i])}
            outs = [o if (k in keep_dev or not is_device_value(o)) else o.to_numpy()
                    for k, o in enumerate(outs)]
        for cell, val in zip(self.output_storage, outs):
            cell[0] = val
        for out_idx, in_idx in self._updates:  # UpdatingVM.perform_updates, vm.py:326-335
            cell = self.input_storage[in_idx]
            if owns_cell(cell):
                cell[0] = dev_outs[out_idx]       # stays on the device (sharedvar.py)
            else:
                v = outs[out_idx]
                cell[0] = v.to_numpy() if (self._host_out and is_device_value(v)) else v
        return outs

    # -- profiling (ProfileStats per-node times from CUDA events) ---------------------
    def _collect_times(self):
        if not self.time_thunks:
            return
        times = getattr(self.executor, "node_times_ms", None)
        if times is None:
            return
        for i, _op, ms in times():
            self.call_times[i] += ms * 1e-3
            self.call_counts[i] += 1

    def update_profile(self, profile):
        """``VM.update_profile`` (``link/vm.py:251-281``): per-Apply device time (CUDA events
        recorded around every node) and call counts."""
        for node, t, c in zip(self.nodes, self.call_times, self.call_counts):
            profile.apply_time.setdefault((self.fgraph, node), 0.0)
            profile.apply_time[(self.fgraph, node)] += t
            profile.apply_callcount.setdefault((self.fgraph, node), 0)
            profile.apply_callcount[(self.fgraph, node)] += c
            profile.apply_cimpl[node] = True  # native kernels, not Python `perform`
        for i in range(len(self.call_times)):
            self.call_times[i] = 0.0
            self.call_counts[i] = 0


class B200Linker(LocalLinker):
    """Link an optimised ``FunctionGraph`` to hand-written sm_90a kernels."""

    def __init__(self, allow_gc=True, precision="fp32", device_outputs=False, schedule=None,
                 cuda_graph=False, shard=None, shard_inputs=None, gather=False, host_chunks=0):
        super().__init__(allow_gc=allow_gc, scheduler=schedule)
        self.fgraph = None
        self.precision = precision
        self.device_outputs = device_outputs
        # shard="rows": each rank of the torch.distributed job gets its row block of the
        # sharded inputs (found by shardplan.infer_sharded_inputs, or named by shard_inputs =
        # {input position: axis}); how the outputs combine is derived from the graph
        # (shardplan.analyse, SURVEY 8e); a graph that is not a batch map raises ReplicasOnly
        if shard not in (None, "rows"):
            raise ValueError("shard must be None or 'rows'")
        self.shard = shard
        self.shard_inputs = shard_inputs
        self.gather = gather
        self.shard_plan = None
        # host_chunks=K: NumPy arguments of a batch-map graph are uploaded and evaluated in K
        # row blocks, the upload of one overlapping the evaluation of the previous
        # (shard.ChunkedHostExecutor); graphs that are not batch maps are evaluated whole
        self.host_chunks = int(host_chunks or 0)
        # replay each evaluation as ONE CUDA graph (runtime/graph.py) once the argument
        # addresses and shapes repeat: removes the per-node host cost, which is what the C
        # twin of the reference VM exists for (lazylinker_c.c).  Off by default because a
        # replayed evaluation returns the SAME output buffers every call (device outputs
        # must be consumed or copied before the next call).
        self.cuda_graph = cuda_graph
        self.no_recycling = []
        self.program = None

    def accept(self, fgraph, no_recycling=None, profile=None):
        if no_recycling is None:
            no_recycling = []
        if self.fgraph is not None and self.fgraph is not fgraph:
            # a linker instance is bound to one graph (pattern of link/basic.py:300-326)
            return type(self)(allow_gc=self.allow_gc, precision=self.precision,
                              device_outputs=self.device_outputs, cuda_graph=self.cuda_graph,
                              shard=self.shard, shard_inputs=self.shard_inputs,
                              gather=self.gather, host_chunks=self.host_chunks).accept(fgraph, no_recycling, profile)
        self.fgraph = fgraph
        self.no_recycling = no_recycling
        self.profile = profile
        return self

    def clone(self, allow_gc=None):
        new = copy(self)
        if allow_gc is not None:
            new._allow_gc = allow_gc
        return new

    def make_all(self, input_storage=None, output_storage=None, storage_map=None):
        from .runtime.vm import ProgramExecutor

        fgraph = self.fgraph
        order = self.schedule(fgraph)
        input_storage, output_storage, storage_map = map_storage(
            fgraph, order, input_storage, output_storage, storage_map
        )
        self.program = lower_fgraph(fgraph, order=order)
        prec = {"fp32": 0, "tf32": 1, "bf16": 2}.get(self.precision, self.precision)
        executor = ProgramExecutor(self.program, precision=prec, host_outputs=False)
        if self.shard == "rows":
            from . import shardplan
            from .shard import ShardedExecutor

            if self.shard_inputs is None:
                self.shard_plan = shardplan.infer_sharded_inputs(self.program)
            else:
                spec = [None] * len(self.program.inputs)
                for k, ax in dict(self.shard_inputs).items():
                    spec[int(k)] = int(ax)
                self.shard_plan = shardplan.analyse(self.program, spec)
            executor = ShardedExecutor(executor, self.shard_plan, gather=self.gather)
        elif self.host_chunks >= 2:
            from . import shardplan
            from .shard import ChunkedHostExecutor

            try:
                self.shard_plan = shardplan.infer_sharded_inputs(self.program)
                if all(a in (None, 0) for a in self.shard_plan.sharded_inputs):
                    executor = ChunkedHostExecutor(executor, self.shard_plan, self.host_chunks)
            except shardplan.ReplicasOnly:
                self.shard_plan = None  # not a batch map: evaluated whole
        fn = B200VM(self, fgraph, order, executor, input_storage, output_storage, storage_map)
        return (
            fn,
            [Container(i, s) for i, s in zip(fgraph.inputs, input_storage)],
            [Container(o, s, readonly=True) for o, s in zip(fgraph.outputs, output_storage)],
            fn.thunks,
            order,
        )


def mode(precision="fp32", device_outputs=False, optimizer=None, cuda_graph=False, shard=None,
         shard_inputs=None, gather=False, host_chunks=0):
    """An Aesara ``Mode`` using this backend with the ``fast_run`` rewrites the
    C-linker gets (SURVEY.md §7.1 step 1).  ``shard="rows"``: see :class:`B200Linker`."""
    if optimizer is None:
        optimizer = RewriteDatabaseQuery(include=["fast_run"])
    return Mode(B200Linker(precision=precision, device_outputs=device_outputs,
                           cuda_graph=cuda_graph, shard=shard, shard_inputs=shard_inputs,
                           gather=gather, host_chunks=host_chunks), optimizer)


def register():
    """``register_linker("b200")`` + ``register_mode("B200")`` (mode.py:54-58, 525-532)."""
    if "b200" not in predefined_linkers:
        register_linker("b200", B200Linker())
    if "B200" not in predefined_modes:
        predefined_modes["B200"] = mode()
    # get_target_language() (mode.py:535-555) raises for linker classes it does not know.
    # Rewrites that consult it (local_careduce_fusion, tensor/rewriting/elemwise.py:966) hold
    # their own reference (``from aesara.compile.mode import get_target_language``), so the
    # replacement is installed in every loaded module that has the original.  This backend
    # consumes the graphs the C-linker gets, so it answers like ``VMLinker`` with a compiler.
    import sys

    import aesara.compile.mode as _m

    _orig = _m.get_target_language
    if not getattr(_orig, "_b200", False):

        def get_target_language(mode=None):
            m = _m.get_default_mode() if mode is None else mode
            if isinstance(getattr(m, "linker", None), B200Linker):
                return ("c", "py")
            return _orig(mode)

        get_target_language._b200 = True
        for mod in list(sys.modules.values()):
            if mod is not None and getattr(mod, "__dict__", {}).get("get_target_language") is _orig:
                mod.get_target_language = get_target_language


register()
from .sharedvar import register_shared_constructor  # noqa: E402

register_shared_constructor()
