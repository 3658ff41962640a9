"""GPU: the persistent Scan cell kernel (csrc/ab_scan_cell_kernel.cuh) at every launch path.

The kernel computes ``pre = x_t + s_hs @ U`` as 64-row x (G*64)-column wgmma tiles (3xTF32), sums
K in 256-element segments (8 k-blocks of 32), and evaluates the cell on the tile.  Each case lands
on one named side of a switch, and its id says which: H and the segment split, tiles against the
132 SMs, the cell's gates / states / recurrent state (G, S, hs), the ring length of the state
buffers, and the operand layout.  Every case asserts the path it meant to reach (the ahead-of-time
LSTM or a generated cell), and the last test asserts that every path was reached.

Truth:
  * integer cells (add, minimum / maximum / clip, integer constants; x in [-3, 3], U in
    {-1, 0, 1}, states in [-8, 8]): every TF32 lo plane is zero and every product and partial
    sum is an integer below 2**24, so the kernel is exact and an int64 recurrence is the truth,
    compared state sequence by state sequence at any T;
  * transcendental cells: float64, one step at a time from the device's own previous states
    (the error does not compound), within the bound derived in ``_pre_bound`` / ``_Err``.
The graphs are built at test time with the reference front end (tests/_scan_cells.py).
"""
import collections
import os

import numpy as np
import pytest

from aesara_b200.compat import bootstrap
from tests import _scan_cells as SC

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not bootstrap.available(), reason="reference front-end (oracle/_ref) not present")]

U24 = 2.0 ** -24
REACHED = collections.defaultdict(set)
RATIOS = []


@pytest.fixture(scope="module")
def rt():
    import torch

    from aesara_b200.runtime import lib
    from aesara_b200.runtime.vm import ProgramExecutor

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return ProgramExecutor


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _runner(ex):
    return [st["runner"] for st in ex._state if "runner" in st][0]


def _split(H):
    """The K-segment split of the kernel: 8 k-blocks of 32 per segment."""
    nkb = -(-H // 32)
    return "1" if nkb <= 8 else f"{nkb // 8}x8+{nkb % 8}" if nkb % 8 else f"{nkb // 8}x8"


def _record(cell, kind, B, H):
    c = SC.CELLS[cell]
    REACHED["spec"].add((c.G, c.S, c.hs, kind))
    REACHED["split"].add(_split(H))
    if -(-B // 64) * (H // 64) > _sms():
        REACHED["tiles"].add(">sms")


def _expect_path(ex, kind, cell, B, H):
    r = _runner(ex)
    assert r.used_fast_path, f"{cell} B={B} H={H}: the persistent kernel did not run"
    assert r.fast_path_kind == kind, f"{cell} B={B} H={H}: ran the {r.fast_path_kind!r} cell, not {kind!r}"
    _record(cell, kind, B, H)


def _assert_exact(got, want, H, what, bitwise=False):
    """Equality (NaN == NaN; bit for bit with ``bitwise``); on a mismatch the first wrong
    (t, row, unit) and its 64 x 64 tile."""
    got = np.asarray(got, np.float32)
    want = np.asarray(want).astype(np.float32)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    if bitwise:
        bad = got.view(np.uint32) != want.view(np.uint32)
    else:
        bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if not bad.any():
        return
    idx = tuple(int(i) for i in np.argwhere(bad)[0])
    row, unit = idx[-2], idx[-1]
    raise AssertionError(
        f"{what}: {int(bad.sum())} of {bad.size} elements differ; first at (t, row, unit) = {idx} "
        f"in tile {(row // 64) * (H // 64) + unit // 64} (row block {row // 64}, unit block {unit // 64}): "
        f"got {got[idx]!r}, want {want[idx]!r}")


def _int_inputs(name, T, B, H, seed):
    c = SC.CELLS[name]
    rng = np.random.default_rng(seed)
    x = rng.integers(-3, 4, (T, B, c.G * H)).astype(np.float32)
    s0 = [rng.integers(-8, 9, (B, H)).astype(np.float32) for _ in range(c.S)]
    # about four non-zeros per column, spread over every K segment: pre stays mostly inside the
    # clip range, so a wrong term changes the state instead of being clipped away
    p = min(1.0, 4.0 / H)
    U = rng.choice(np.array([-1, 0, 1], np.float32), size=(H, c.G * H), p=[p / 2, 1 - p, p / 2])
    return x, s0, U


def _float_inputs(name, T, B, H, seed, saturate=0):
    """Random operands; the first ``saturate`` rows of x are +-1e4 at every step."""
    c = SC.CELLS[name]
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((T, B, c.G * H)).astype(np.float32)
    x[:, :saturate] = np.where(rng.random((T, saturate, c.G * H)) < 0.5, -1e4, 1e4)
    s0 = [(rng.standard_normal((B, H)) * 0.5).astype(np.float32) for _ in range(c.S)]
    U = (rng.standard_normal((H, c.G * H)) * 1.5 / np.sqrt(H)).astype(np.float32)
    return x, s0, U


def _dev(a):
    from aesara_b200.runtime.device import DeviceArray

    return DeviceArray.from_numpy(np.ascontiguousarray(a))


# ---------------------------------------------------------------------------------------------
# A. exact integer recurrences through the graph, every (G, S, hs) at every K split
# ---------------------------------------------------------------------------------------------
INT_CELLS = ["G1S1hs0", "G3S1hs0", "G2S3hs1", "G4S2hs1_ch"]
SHAPES = [  # id, H, B, T
    ("H64-seg1-B128-tiles2-T257", 64, 128, 257),
    ("H256-seg8-B200ragged-tiles16-T3", 256, 200, 3),
    ("H320-seg8+2-B200ragged-tiles20-T3", 320, 200, 3),
    ("H320-seg8+2-B2048-tiles160>sms-T2", 320, 2048, 2),
    ("H1088-seg4x8+2-B8<tile-tiles17-T3", 1088, 8, 3),
    ("H1088-seg4x8+2-B128-tiles34-T2", 1088, 128, 2),
]


@pytest.mark.parametrize("H,B,T", [s[1:] for s in SHAPES], ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize("cell", INT_CELLS)
def test_integer_cell_exact_state_sequences(rt, cell, H, B, T):
    x, s0, U = _int_inputs(cell, T, B, H, seed=H + B + T)
    ex = rt(SC.program(cell))
    got = ex(x, *s0, U)
    _expect_path(ex, "jit", cell, B, H)
    REACHED["ring"].add("T")
    for k, w in enumerate(SC.int_truth(cell, x, s0, U)):
        _assert_exact(got[k], w, H, f"{cell} state {k} (B={B}, H={H}, T={T})")


# ---------------------------------------------------------------------------------------------
# B. ring geometry and operand layouts through the C ABI (scan_cell.run_cell / run_lstm)
# ---------------------------------------------------------------------------------------------
def _direct(kind, spec, T, x, U, rings, pos):
    import torch

    from aesara_b200.runtime import scan_cell

    if kind == "lstm":
        scan_cell.run_lstm(T, x, U, rings[0], rings[1], pos[0], pos[1])
    else:
        scan_cell.run_cell(spec, T, x, U, rings, pos)
    torch.cuda.synchronize()


def _spec(rt, cell, B, H):
    spec = _runner(rt(SC.program(cell))).cell.match(B, H, SC.CELLS[cell].G)
    assert spec is not None and spec.is_lstm == SC.CELLS[cell].is_lstm
    return spec


def _ring(init, L, pos):
    """A state ring of L rows: the initial state at row (pos - 1) mod L, NaN everywhere else."""
    r = np.full((L,) + init.shape, np.nan, np.float32)
    r[(pos - 1) % L] = init
    return r


def _ring_want(init, seq, L, pos):
    r = _ring(init, L, pos)
    for t in range(len(seq)):
        r[(pos + t) % L] = seq[t]
    return r


def _sequences(kind, cell, spec, x, s0, U):
    """State sequences [T, B, H]: the integer truth, or (for the ahead-of-time LSTM, whose
    truth is not exact) the kernel itself on contiguous operands and rings of length T + 1."""
    if kind == "jit":
        return SC.int_truth(cell, x, s0, U)
    T = x.shape[0]
    rings = [_dev(_ring(s, T + 1, 1)) for s in s0]
    _direct(kind, spec, T, _dev(x), _dev(U), rings, [1] * len(s0))
    return [r.to_numpy()[1:] for r in rings]


def _ring_cases(T):
    cases = []
    for label, L in (("len1", 1), ("len2", 2), ("lenT", T), ("lenT+1", T + 1), ("len2T", 2 * T)):
        for p in sorted({0, 1 % L, L - 1}):
            cases.append((f"{label}-pos{p}", [L], [p]))
    return cases


RING_T = 5
DIRECT_KINDS = [("jit", "G2S3hs1"), ("lstm", "lstm_hc")]
_DIRECT_IDS = {"G2S3hs1": "jit-G2S3hs1", "lstm_hc": "lstm-G4S2hs0"}
RING_CASES = [(f"{_DIRECT_IDS[cell]}-{rid}", kind, cell, lens * SC.CELLS[cell].S, poss * SC.CELLS[cell].S)
              for kind, cell in DIRECT_KINDS for rid, lens, poss in _ring_cases(RING_T)]
# every state of the three-state cell on its own geometry
RING_CASES.append(("jit-G2S3hs1-mixed-len1,T+1,2-pos0,3,1", "jit", "G2S3hs1", [1, RING_T + 1, 2], [0, 3, 1]))


@pytest.mark.parametrize("kind,cell,lens,poss", [c[1:] for c in RING_CASES], ids=[c[0] for c in RING_CASES])
def test_ring_geometry(rt, kind, cell, lens, poss):
    """Rings of length 1 (the row read is the row written), 2, T, T + 1 and 2T at positions 0, 1
    and len - 1: the rows written hold the states of their steps, the rest keep their NaN bits."""
    c = SC.CELLS[cell]
    T, B, H = RING_T, 128, 64
    spec = _spec(rt, cell, B, H)
    x, s0, U = (_int_inputs if c.exact else _float_inputs)(cell, T, B, H, seed=sum(lens) + sum(poss))
    want = _sequences(kind, cell, spec, x, s0, U)
    rings = [_dev(_ring(s, L, p)) for s, L, p in zip(s0, lens, poss)]
    _direct(kind, spec, T, _dev(x), _dev(U), rings, poss)
    _record(cell, kind, B, H)
    for k, (r, L, p) in enumerate(zip(rings, lens, poss)):
        REACHED["ring"].add({1: "1", 2: "2", T: "T"}.get(L, str(L)))
        _assert_exact(r.to_numpy(), _ring_want(s0[k], want[k], L, p), H,
                      f"{kind} state {k}, ring of {L} at position {p}", bitwise=kind == "lstm")
        nan_rows = set(range(L)) - {(p - 1) % L} - {(p + t) % L for t in range(T)}
        for row in nan_rows:  # untouched rows keep their exact NaN bit pattern
            assert np.array_equal(r.to_numpy()[row].view(np.uint32),
                                  np.full((B, H), np.nan, np.float32).view(np.uint32)), (k, row)


LAYOUTS = ["x_reversed_negstep", "x_colslice_nanpad", "U_transposed", "U_colslice_nanpad"]


@pytest.mark.parametrize("kind,cell", DIRECT_KINDS, ids=[_DIRECT_IDS[c] for _, c in DIRECT_KINDS])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_operand_layouts(rt, kind, cell, layout):
    """x as a reversed view (negative step stride) and as a column slice of a wider buffer whose
    extra columns are NaN (a read past G*H poisons the states); U as a transposed view and as a
    slice of a wider NaN-padded matrix."""
    c = SC.CELLS[cell]
    T, B, H = 4, 200, 128
    GH = c.G * H
    spec = _spec(rt, cell, B, H)
    x, s0, U = (_int_inputs if c.exact else _float_inputs)(cell, T, B, H, seed=len(layout))
    xd, Ud, x_eff = _dev(x), _dev(U), x
    if layout == "x_reversed_negstep":
        xd = xd.index((slice(None, None, -1),))
        assert xd.strides[0] < 0
        x_eff = x[::-1]
    elif layout == "x_colslice_nanpad":
        wide = np.full((T, B, GH + 64), np.nan, np.float32)
        wide[..., :GH] = x
        xd = _dev(wide).index((slice(None), slice(None), slice(0, GH)))
        assert xd.strides[1] == GH + 64
    elif layout == "U_transposed":
        Ud = _dev(U.T).dimshuffle((1, 0))
        assert Ud.strides == (1, H)
    else:
        wide = np.full((H + 2, GH + 32), np.nan, np.float32)
        wide[1:H + 1, 16:16 + GH] = U
        Ud = _dev(wide).index((slice(1, H + 1), slice(16, 16 + GH)))
        assert Ud.strides == (GH + 32, 1)
    want = _sequences(kind, cell, spec, np.ascontiguousarray(x_eff), s0, U)
    rings = [_dev(_ring(s, T + 1, 1)) for s in s0]
    _direct(kind, spec, T, xd, Ud, rings, [1] * c.S)
    _record(cell, kind, B, H)
    REACHED["layout"].add(layout)
    for k, r in enumerate(rings):
        _assert_exact(r.to_numpy()[1:], want[k], H, f"{kind} {layout} state {k}", bitwise=kind == "lstm")


def test_misaligned_x_takes_the_general_loop(rt):
    """x 4 bytes off a 16-byte boundary: not eligible, refused by the C ABI before any launch,
    and the graph runs it on the general loop with the same answer."""
    from aesara_b200.runtime import lib, scan_cell
    from aesara_b200.runtime.device import DeviceArray, c_strides

    cell, T, B, H = "G2S3hs1", 4, 128, 128
    c = SC.CELLS[cell]
    x, s0, U = _int_inputs(cell, T, B, H, seed=4)
    flat = _dev(np.concatenate([np.zeros(1, np.float32), x.reshape(-1)]))
    xd = flat.view(x.shape, c_strides(x.shape), offset_elems=1)
    assert xd.ptr % 16 == 4
    rings = [_dev(_ring(s, T + 1, 1)) for s in s0]
    assert not scan_cell.eligible(xd, _dev(U), rings, T, c.G)
    with pytest.raises(lib.AbError):
        scan_cell.run_cell(_spec(rt, cell, B, H), T, xd, _dev(U), rings, [1] * c.S)
    ex = rt(SC.program(cell))
    got = ex(xd, *[_dev(s) for s in s0], _dev(U))
    assert not _runner(ex).used_fast_path
    REACHED["layout"].add("x_misaligned")
    for k, w in enumerate(SC.int_truth(cell, x, s0, U)):
        _assert_exact(got[k], w, H, f"misaligned x, state {k}")


# ---------------------------------------------------------------------------------------------
# C. float64 one-step truth of the transcendental cells
# ---------------------------------------------------------------------------------------------
def _pre_bound(xt, h, U):
    """float64 ``pre = x_t + h @ U`` and a bound on the kernel's error in it, per element.

    With p_k = h_k U_kj, S = sum |p_k| over a K range and A_m the partial sum of the p_k of a
    segment up to its k-step m (8 K per wgmma instruction, three instructions per k-step):
      * 3xTF32 products: hi = tf32(v) rounded to nearest, |v - hi| <= 2**-11 |v|, and
        lo = tf32(v - hi) leaves |v - hi - lo| <= 2**-22 |v|.  The kernel drops lo*lo and both
        lo roundings: |a b - (a_hi b_hi + a_hi b_lo + a_lo b_hi)| <= 3.01 * 2**-22 |a b|;
      * the tensor core's accumulate: the products are exact, aligned to the largest addend
        (accumulator included) and truncated, and the sum is normalised by truncation.  An
        instruction then loses less than one unit of 2**-23 of its largest addend per product
        and one of its result: at most 9 * 2**-23 (|A_{m-1}| + S_m) each, 27 per k-step;
      * the segments are folded into x_t in FP32 with round-to-nearest: u |running sum| each.
    The typical error of dropping one of the three wgmma terms is sqrt(K) |p| 2**-12, about
    three times the truncation term summed over a segment, and its largest over the elements
    of a step is several times that; a dropped K segment is larger still."""
    B, K = h.shape
    h64, U64 = h.astype(np.float64), U.astype(np.float64)
    ah, aU = np.abs(h64), np.abs(U64)
    run = xt.astype(np.float64).copy()
    E = np.zeros_like(run)
    for k0 in range(0, K, 256):
        k1 = min(k0 + 256, K)
        A = np.zeros_like(run)
        tc = np.zeros_like(run)
        S = np.zeros_like(run)
        for m0 in range(k0, k1, 8):
            Sm = ah[:, m0:m0 + 8] @ aU[m0:m0 + 8]
            tc += np.abs(A) + Sm
            S += Sm
            A += h64[:, m0:m0 + 8] @ U64[m0:m0 + 8]
        E += 3.01 * 2.0 ** -22 * S + 27 * 2.0 ** -23 * (1 + 2.0 ** -9) * tc
        run += A
        E += U24 * (np.abs(run) + E)
    return run, E


class _Err:
    """A float64 value with a bound on the device's error in it, through the cell's operations.
    Device operations: products and sums rounded to nearest (u = 2**-24 relative);
    expf and tanhf within 2 ulp (4u relative); sigmoid = 1 / (1 + expf(-v)) within 6u of its value
    (taken as 6u absolute, which also covers 1 - sigmoid(v) rewritten as sigmoid(-v)).  Input
    errors propagate with sigmoid' <= 1/4 and tanh' <= 1, products with |a| e_b + |b| e_a."""

    def __init__(self, v, e):
        self.v, self.e = v, e

    @staticmethod
    def c(v):
        return _Err(np.float64(v), 0.0)

    def _sum(self, o, sign):
        v = self.v + sign * o.v
        e = self.e + o.e
        return _Err(v, e + U24 * (np.abs(v) + e))

    def __add__(self, o):
        return self._sum(o, 1)

    def __sub__(self, o):
        return self._sum(o, -1)

    def __mul__(self, o):
        v = self.v * o.v
        e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
        return _Err(v, e + U24 * (np.abs(v) + e))

    @staticmethod
    def sigmoid(a):
        with np.errstate(over="ignore"):
            v = 1.0 / (1.0 + np.exp(-a.v))
        return _Err(v, 0.25 * a.e + 6 * U24)

    @staticmethod
    def tanh(a):
        v = np.tanh(a.v)
        return _Err(v, a.e + 4 * U24 * (np.abs(v) + a.e))


# the state that is exact (0, +-1 or an integer) in rows whose pre-activations saturate
_SAT_STATE = {"rnn_tanh": 0, "gated": 0, "lstm_hc": 1, "lstm_ch": 0}
F64_CASES = [("rnn_tanh", "jit"), ("gated", "jit"), ("lstm_hc", "lstm"), ("lstm_hc", "jit"), ("lstm_ch", "jit")]
F64_SHAPES = [("H64-seg1-B128-T9", 64, 128, 9), ("H320-seg8+2-B200-T3", 320, 200, 3),
              ("H1088-seg4x8+2-B8-T3", 1088, 8, 3)]


@pytest.mark.parametrize("H,B,T", [s[1:] for s in F64_SHAPES], ids=[s[0] for s in F64_SHAPES])
@pytest.mark.parametrize("cell,kind", F64_CASES, ids=[f"{c}-{k}" for c, k in F64_CASES])
def test_transcendental_cell_one_step_float64(rt, monkeypatch, cell, kind, H, B, T):
    c = SC.CELLS[cell]
    if kind == "jit" and c.is_lstm:
        monkeypatch.setenv("AB_SCAN_JIT", "1")
    sat = 2
    x, s0, U = _float_inputs(cell, T, B, H, seed=7 * H + B, saturate=sat)
    ex = rt(SC.program(cell))
    got = [np.asarray(g) for g in ex(x, *s0, U)]
    _expect_path(ex, kind, cell, B, H)
    worst = 0.0
    for t in range(T):
        prev = [s0[k] if t == 0 else got[k][t - 1] for k in range(c.S)]
        pre, E = _pre_bound(x[t], prev[c.hs], U)
        gates = [_Err(pre[:, g * H:(g + 1) * H], E[:, g * H:(g + 1) * H]) for g in range(c.G)]
        new = c.fn(_Err, gates, [_Err(p.astype(np.float64), 0.0) for p in prev])
        for k, want in enumerate(new):
            err = np.abs(got[k][t] - want.v)
            bound = want.e + 1e-37
            assert np.isfinite(got[k][t]).all(), f"{cell} state {k} step {t}: non-finite"
            ratio = err / bound
            worst = max(worst, float(ratio.max()))
            if (ratio > 1).any():
                i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
                raise AssertionError(
                    f"{cell} ({kind}) state {k} step {t}: {int((ratio > 1).sum())} elements beyond the bound; "
                    f"worst at (row, unit) = {i} in tile {(i[0] // 64) * (H // 64) + i[1] // 64}: "
                    f"got {got[k][t][i]!r}, float64 {want.v[i]!r}, bound {bound[i]:.3e}")
        k = _SAT_STATE[cell]
        _assert_exact(got[k][t][:sat], new[k].v[:sat], H, f"{cell} ({kind}) saturated rows, state {k}, step {t}")
    RATIOS.append((f"{cell}-{kind}-H{H}-B{B}", worst))


@pytest.mark.parametrize("H,B,T", [s[1:] for s in SHAPES], ids=[s[0] for s in SHAPES])
def test_lstm_ahead_of_time_equals_generated_bit_for_bit(rt, monkeypatch, H, B, T):
    x, s0, U = _float_inputs("lstm_hc", T, B, H, seed=H * 3 + B, saturate=1)
    ex = rt(SC.program("lstm_hc"))
    aot = ex(x, *s0, U)
    _expect_path(ex, "lstm", "lstm_hc", B, H)
    monkeypatch.setenv("AB_SCAN_JIT", "1")
    jit = ex(x, *s0, U)
    _expect_path(ex, "jit", "lstm_hc", B, H)
    for k, (a, j) in enumerate(zip(aot, jit)):
        _assert_exact(j, a, H, f"LSTM state {k}: generated vs ahead-of-time", bitwise=True)


# ---------------------------------------------------------------------------------------------
# D. front-end paths, eligibility, and state across calls
# ---------------------------------------------------------------------------------------------
def _general(rt, prog, ins):
    os.environ["AB_SCAN_NO_FAST"] = "1"
    try:
        ex = rt(prog)
        out = ex(*ins)
    finally:
        del os.environ["AB_SCAN_NO_FAST"]
    assert not _runner(ex).used_fast_path
    return out


GRAPH_VARIANTS = [("backwards", "G1S1hs0"), ("wt", "G1S1hs0"), ("last", "G2S3hs1"), ("all", "G2S3hs1"),
                  ("nsteps2", "G2S3hs1"), ("backwards", "G2S3hs1")]


@pytest.mark.parametrize("variant,cell", GRAPH_VARIANTS, ids=[f"{v}-{c}" for v, c in GRAPH_VARIANTS])
def test_front_end_graphs(rt, variant, cell):
    """go_backwards, non_sequences=[W.T], s[-1] only (rings of 2), the full sequences (rings of T,
    un-rotated after the kernel) and n_steps < len(x): fast path == integer truth == the oracle ==
    the general loop."""
    from oracle.program_np import run_program

    c = SC.CELLS[cell]
    T, B, H = 6, 200, 128
    x, s0, U = _int_inputs(cell, T, B, H, seed=len(variant))
    prog = SC.program(cell, variant)
    ins = [x] + s0 + [np.ascontiguousarray(U.T) if variant == "wt" else U]
    ex = rt(prog)
    got = ex(*ins)
    _expect_path(ex, "jit", cell, B, H)
    REACHED["graph"].add(variant)
    truth = SC.int_truth(cell, x[::-1] if variant == "backwards" else x[:2] if variant == "nsteps2" else x, s0, U)
    if variant == "last":
        truth = [w[-1] for w in truth]
        REACHED["ring"].add("2")
    oracle = run_program(prog, [np.array(a) for a in ins])
    general = _general(rt, prog, ins)
    assert len(got) == c.S
    for k in range(c.S):
        _assert_exact(got[k], truth[k], H, f"{variant} state {k} vs integer truth")
        _assert_exact(oracle[k], truth[k], H, f"{variant} state {k}: oracle vs integer truth")
        _assert_exact(general[k], got[k], H, f"{variant} state {k}: general loop vs fast path")


ELIGIBILITY = [("B128xH64-BH8192-fast", 128, 64, 4, True), ("B127xH64-BH8128-general", 127, 64, 4, False),
               ("B200xH96-Hnot64-general", 200, 96, 4, False), ("B200xH128-T1-general", 200, 128, 1, False)]


@pytest.mark.parametrize("B,H,T,fast", [e[1:] for e in ELIGIBILITY], ids=[e[0] for e in ELIGIBILITY])
def test_eligibility_edges(rt, B, H, T, fast):
    cell = "G3S1hs0"
    x, s0, U = _int_inputs(cell, T, B, H, seed=B + H + T)
    ex = rt(SC.program(cell))
    got = ex(x, *s0, U)
    if fast:
        _expect_path(ex, "jit", cell, B, H)
    else:
        assert not _runner(ex).used_fast_path, f"B={B} H={H} T={T} should run on the general loop"
    _assert_exact(got[0], SC.int_truth(cell, x, s0, U)[0], H, f"B={B} H={H} T={T}")


@pytest.mark.parametrize("kind,cell", [("jit", "G2S3hs1"), ("lstm", "lstm_hc")])
def test_row_isolation(rt, kind, cell):
    """A NaN in row r of x at step t0 stays in row r: every other row is bit-identical."""
    c = SC.CELLS[cell]
    T, B, H, r, t0 = 4, 200, 320, 137, 1
    x, s0, U = (_int_inputs if c.exact else _float_inputs)(cell, T, B, H, seed=13)
    ex = rt(SC.program(cell))
    clean = [np.asarray(g) for g in ex(x, *s0, U)]
    xn = x.copy()
    xn[t0, r, 5] = np.nan
    dirty = [np.asarray(g) for g in ex(xn, *s0, U)]
    _expect_path(ex, kind, cell, B, H)
    keep = np.arange(B) != r
    for k in range(c.S):
        _assert_exact(dirty[k][:, keep], clean[k][:, keep], H, f"state {k} outside row {r}", bitwise=True)
    assert np.isnan(dirty[c.hs][t0:, r]).any(), "the NaN never reached the recurrent state"


def test_repeat_and_graph_replay(rt):
    """The same call twice is bit-identical (the row counters restart at zero), and a CUDA-graph
    replay of a generated-cell graph, three times, equals the eager run bit for bit."""
    from aesara_b200.runtime.device import DeviceArray
    from aesara_b200.runtime.graph import GraphReplay

    cell, T, B, H = "gated", 7, 200, 320
    x, s0, U = _float_inputs(cell, T, B, H, seed=21)
    ex = rt(SC.program(cell), host_outputs=False)
    dins = [DeviceArray.from_numpy(a) for a in [x] + s0 + [U]]
    first = [o.to_numpy() for o in ex(*dins)]
    _expect_path(ex, "jit", cell, B, H)
    second = [o.to_numpy() for o in ex(*dins)]
    for a, b in zip(first, second):
        _assert_exact(b, a, H, "second call", bitwise=True)
    replay = GraphReplay(ex)
    for _ in range(3):
        outs = replay(*dins)
    assert replay.replays >= 2
    REACHED["graph"].add("replay")
    for a, b in zip(first, outs):
        _assert_exact(b.to_numpy(), a, H, "graph replay", bitwise=True)


def test_one_executor_at_two_shapes(rt):
    cell = "G2S3hs1"
    ex = rt(SC.program(cell))
    for T, B, H in ((3, 200, 128), (2, 128, 320), (3, 200, 128)):
        x, s0, U = _int_inputs(cell, T, B, H, seed=B * H)
        got = ex(x, *s0, U)
        _expect_path(ex, "jit", cell, B, H)
        for k, w in enumerate(SC.int_truth(cell, x, s0, U)):
            _assert_exact(got[k], w, H, f"B={B} H={H} state {k}")
    assert {(200, 128, 2), (128, 320, 2)} <= set(_runner(ex).cell._cache)


@pytest.mark.parametrize("kind,cell", [("jit", "G1S1hs0"), ("lstm", "lstm_hc")])
def test_launch_count_does_not_grow_with_T(rt, kind, cell):
    from aesara_b200.runtime import lib

    c = SC.CELLS[cell]
    B, H = 128, 128
    ex = rt(SC.program(cell))
    counts = []
    for T in (2, 257):
        x, s0, U = (_int_inputs if c.exact else _float_inputs)(cell, T, B, H, seed=T)
        before = lib.load().ab_launch_count()
        ex(x, *s0, U)
        counts.append(lib.load().ab_launch_count() - before)
        _expect_path(ex, kind, cell, B, H)
    assert counts[0] == counts[1], f"launches at T=2 and T=257: {counts}"


# ---------------------------------------------------------------------------------------------
# every switch was reached (runs last)
# ---------------------------------------------------------------------------------------------
def test_zz_every_launch_path_was_reached():
    want_specs = {(1, 1, 0, "jit"), (3, 1, 0, "jit"), (2, 3, 1, "jit"), (4, 2, 1, "jit"),
                  (4, 2, 0, "lstm"), (4, 2, 0, "jit")}
    assert want_specs <= REACHED["spec"], sorted(want_specs - REACHED["spec"])
    assert {"1", "1x8+2", "4x8+2"} <= REACHED["split"], REACHED["split"]
    assert ">sms" in REACHED["tiles"]
    assert {"1", "2", "T"} <= REACHED["ring"], REACHED["ring"]
    assert set(LAYOUTS) | {"x_misaligned"} <= REACHED["layout"], REACHED["layout"]
    assert {"backwards", "wt", "last", "all", "nsteps2", "replay"} <= REACHED["graph"], REACHED["graph"]
    for name, r in RATIOS:
        print(f"error / bound {name}: {r:.3g}")
    assert RATIOS and max(r for _, r in RATIOS) <= 1.0
