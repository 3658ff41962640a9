"""Scan inner graphs of the persistent cell kernel's family, built with the reference front end,
and their NumPy truths.

Every cell is written once, as a function ``fn(ops, gates, states) -> new states`` over an
``ops`` namespace, and evaluated three ways: symbolically (``aesara.scan`` step, float32
constants so that the matcher accepts them), on int64 arrays (the exact truth of the integer
cells) and on float64 arrays (the one-step truth of the transcendental cells).

``G`` gates are column blocks of ``pre = x_t + s_hs @ U``; ``S`` states, of which state ``hs``
multiplies ``U``.
"""
import functools
from collections import namedtuple

import numpy as np

F32 = np.float32
Cell = namedtuple("Cell", "name G S hs is_lstm exact fn")


def _g1s1(o, g, s):
    return [o.clip(g[0] + o.c(1))]


def _g3s1(o, g, s):
    return [o.clip(o.maximum(g[0], s[0]) + o.minimum(g[1], o.c(2)) - g[2])]


def _g2s3(o, g, s):
    a, b, c = s  # b multiplies U and enters the cell through the product only
    na = o.clip(g[0] - c)
    nb = o.clip(g[1] + a)
    return [na, nb, o.maximum(a, nb)]


def _g4s2_ch(o, g, s):
    c, h = s  # LSTM-shaped, states (c, h): h multiplies U
    nc = o.clip(o.minimum(g[1], c) + g[0] - o.maximum(g[3], o.c(0)))
    return [nc, o.clip(g[2] - nc)]


def _rnn_tanh(o, g, s):
    return [o.tanh(g[0])]


def _gated(o, g, s):
    z, r = o.sigmoid(g[0]), o.sigmoid(g[1])
    n = o.tanh(g[2] * r)
    return [(o.c(1) - z) * s[0] + z * n]


def _lstm_gates(o, g):
    return o.sigmoid(g[0]), o.sigmoid(g[1]), o.sigmoid(g[2]), o.tanh(g[3])  # i, f, o, g


def _lstm_hc(o, g, s):
    h, c = s
    i, f, og, gg = _lstm_gates(o, g)
    cn = f * c + i * gg
    return [og * o.tanh(cn), cn]


def _lstm_ch(o, g, s):
    c, h = s
    i, f, og, gg = _lstm_gates(o, g)
    cn = f * c + i * gg
    return [cn, og * o.tanh(cn)]


CELLS = {c.name: c for c in [
    # integer cells: add, minimum / maximum / clip and integer constants; states in [-8, 8]
    Cell("G1S1hs0", 1, 1, 0, False, True, _g1s1),
    Cell("G3S1hs0", 3, 1, 0, False, True, _g3s1),
    Cell("G2S3hs1", 2, 3, 1, False, True, _g2s3),
    Cell("G4S2hs1_ch", 4, 2, 1, False, True, _g4s2_ch),
    # transcendental cells
    Cell("rnn_tanh", 1, 1, 0, False, False, _rnn_tanh),
    Cell("gated", 3, 1, 0, False, False, _gated),
    Cell("lstm_hc", 4, 2, 0, True, False, _lstm_hc),
    Cell("lstm_ch", 4, 2, 1, False, False, _lstm_ch),
]}


class _SymOps:
    def __init__(self, at):
        self.at = at
        self.maximum, self.minimum = at.maximum, at.minimum
        self.sigmoid, self.tanh = at.sigmoid, at.tanh

    @staticmethod
    def c(v):
        return F32(v)

    def clip(self, v):
        return self.at.clip(v, F32(-8), F32(8))


class _IntOps:
    maximum, minimum = staticmethod(np.maximum), staticmethod(np.minimum)

    @staticmethod
    def c(v):
        return np.int64(v)

    @staticmethod
    def clip(v):
        return np.clip(v, -8, 8)


class _F64Ops:
    tanh = staticmethod(np.tanh)

    @staticmethod
    def c(v):
        return np.float64(v)

    @staticmethod
    def sigmoid(v):
        with np.errstate(over="ignore"):
            return 1.0 / (1.0 + np.exp(-v))


@functools.lru_cache(maxsize=None)
def program(name, variant="all"):
    """Lowered program of ``cell`` in a Scan over ``x`` [T, B, G*H] with initial states
    ``s0..`` [B, H] and ``U`` [H, G*H]; inputs ``(x, s0, .., U)``.  ``variant``:
      "all"       the full state sequences are the outputs (rings of length T, un-rotated);
      "last"      only ``s[-1]`` of every state (rings of length 2);
      "backwards" ``go_backwards=True``, full sequences;
      "wt"        the last input is ``W`` [G*H, H] and the Scan gets ``non_sequences=[W.T]``;
      "nsteps2"   ``n_steps = 2`` over a longer ``x``, full sequences."""
    from aesara_b200.graphs import _at, optimized_program

    aesara, at = _at()
    cell = CELLS[name]
    ops = _SymOps(at)
    x = at.ftensor3("x")
    s0 = [at.fmatrix(f"s{k}") for k in range(cell.S)]
    W = at.fmatrix("W")

    def step(x_t, *args):
        *s, U_ = args
        H = s[0].shape[1]
        pre = x_t + at.dot(s[cell.hs], U_)
        # (one gate is `pre` itself: a slice of it would be pushed into the operands of the dot)
        gates = [pre] if cell.G == 1 else [pre[:, k * H:(k + 1) * H] for k in range(cell.G)]
        out = cell.fn(ops, gates, list(s))
        return out if cell.S > 1 else out[0]

    seqs, _ = aesara.scan(step, sequences=[x], outputs_info=s0,
                          non_sequences=[W.T if variant == "wt" else W],
                          go_backwards=variant == "backwards",
                          n_steps=2 if variant == "nsteps2" else None)
    outs = list(seqs) if cell.S > 1 else [seqs]
    if variant == "last":
        outs = [o[-1] for o in outs]
    prog, _ = optimized_program([x] + s0 + [W], outs, name=f"scan_{name}_{variant}")
    return prog


def int_truth(name, x, s0, U):
    """Exact state sequences [T, B, H] of an integer cell (int64; the products in float64,
    exact for integers below 2**53)."""
    cell = CELLS[name]
    H = s0[0].shape[1]
    x = np.asarray(x).astype(np.int64)
    s = [np.asarray(a).astype(np.int64) for a in s0]
    Uf = np.asarray(U, np.float64)
    out = [[] for _ in s]
    for t in range(x.shape[0]):
        pre = x[t] + (s[cell.hs].astype(np.float64) @ Uf).astype(np.int64)
        s = cell.fn(_IntOps, [pre[:, g * H:(g + 1) * H] for g in range(cell.G)], s)
        for k, v in enumerate(s):
            out[k].append(v)
    return [np.stack(o) for o in out]


def f64_step(name, gates, states):
    """One step of a transcendental cell in float64."""
    return CELLS[name].fn(_F64Ops, gates, states)
