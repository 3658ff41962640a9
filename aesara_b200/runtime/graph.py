"""CUDA-graph replay of a whole program evaluation.

The reference amortises per-node overhead with a C re-implementation of the VM
loop (``CLazyLinker``, ``aesara/link/c/c_code/lazylinker_c.c:501-890``).  On a
GPU the equivalent cost is launch + Python dispatch per node; for small graphs
(README example: 6 nodes) and for ``Scan`` (hundreds of tiny steps) it
dominates.  ``GraphReplay`` captures every launch of one
``ProgramExecutor`` call — including the per-step launches of a ``Scan`` loop —
into a CUDA graph keyed on the input buffers' (pointer, shape, strides) and
replays it with a single ``cudaGraphLaunch``.

Capturable = no device→host read while evaluating (no ``ScalarFromTensor`` /
``Assert`` on device data, no ``as_while`` Scan) and no random variable: a replay would
reuse the key its capture drew from the Generator, so every replay would repeat the same
draws.  Such programs transparently fall back to eager execution.  Host-side shape arithmetic is evaluated at
capture time; a change of any input shape/pointer produces a new capture.
The returned output arrays are owned by the captured graph and are overwritten
by the next replay.
"""

from __future__ import annotations

import numpy as np
import torch

from .device import DeviceArray
from .vm import ProgramExecutor


class GraphReplay:
    def __init__(self, executor, max_graphs: int = 8):
        if executor.host_outputs:
            raise ValueError("GraphReplay needs an executor with host_outputs=False")
        self.ex = executor
        self.max_graphs = max_graphs
        self._graphs = {}
        # random variables draw a fresh key from their Generator on every call (runtime/vm.py)
        prog = getattr(executor, "program", None)
        self._uncapturable = prog is not None and any(n.op == "RandomVariable" for n in prog.nodes)
        self.replays = 0

    @staticmethod
    def _key(inputs):
        k = []
        for a in inputs:
            if isinstance(a, DeviceArray):
                k.append(("d", a.ptr, a.shape, a.strides, a.dtype.str))
            else:
                h = np.asarray(a)
                k.append(("h", h.dtype.str, h.shape, h.tobytes()))
        return tuple(k)

    def __call__(self, *inputs):
        if self._uncapturable:
            return self.ex(*inputs)
        key = self._key(inputs)
        ent = self._graphs.get(key)
        if ent is None:
            ent = self._capture(key, inputs)
            if ent is None:
                return self.ex(*inputs)
        graph, outs, _keep = ent
        graph.replay()
        self.replays += 1
        return outs

    def _capture(self, key, inputs):
        # eager warm-up: JIT/load modules, stage constants and host scalars
        self.ex(*inputs)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                outs = self.ex(*inputs)
        except Exception:
            # a node needed a host read (or another capture-illegal call): stay eager
            self._uncapturable = True
            torch.cuda.synchronize()
            return None
        if len(self._graphs) >= self.max_graphs:
            self._graphs.pop(next(iter(self._graphs)))
        ent = self._graphs[key] = (g, outs, list(inputs))
        return ent
