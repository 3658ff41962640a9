"""GPU: the executor-level fused regions at every generated variant.

GEMM-epilogue regions (runtime/gemmfuse.py, codegen/gemm_epilogue.py, the AB_EPILOGUE half of
csrc/ab_gemm_tc_kernel.cuh) and row regions (runtime/rowfuse.py, codegen/rowfuse.py) are
generated per graph.  Each case lands on one named side of a switch and its id names it: the
compile-time ``AB_EP_*`` switches of the module, the run-time path of every epilogue operand
(``[1,1]`` scalar, static ``[1,N]`` row, run-time row by shuffle, the read-ahead ``[M,N]``
operand, a second ``[M,N]`` operand by ``ld8``, the strided loop), the per-call plan of every value
(float32, natural bf16 plane, transposed plane, plane only), the product (Dot22, Dot22Scalar,
Gemm with and without ``inplace``), the precision policy, and for row regions the register
blocking J = ceil(D / 128), the grid and the external operand classes.  Every case asserts the
path it took; the last test asserts that every side was reached.

Truth (tests/_fused_regions.py): integer operands in [-4, 4] (weights in {-1, 0, 1}, a few per
column) and programs of exact ops, so every product under bf16, TF32 and 3xTF32, every bf16 plane
of a region value, every float32 value and every column sum / total is exact, and the outputs
must equal a float64 NumPy evaluation bit for bit.  Transcendental programs must be bit-identical
to the node-by-node Elemwise kernels and within the CUDA Math API ulp bounds of
test_gpu_elemwise.py against float64.

Known limit, pinned in ``test_colsum_float32_overflow``: the epilogue adds the column sums and
totals of each 32-row block as float pairs (3xTF32) or float32 trees (bf16, TF32) before the
float64 pass; a column whose partial sums overflow float32 gives a non-finite sum there where the
node-by-node float64 CAReduce is finite.
"""
import collections

import numpy as np
import pytest

from aesara_b200.compat import bootstrap
from tests import _fused_regions as FR

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not bootstrap.available(), reason="reference front-end (oracle/_ref) not present")]

REACHED = collections.defaultdict(set)
NOTES = []
DIMS = {"M": 129, "N": 136, "K": 520, "P": 128}
PRECISIONS = (0, 1, 2)


@pytest.fixture(scope="module")
def rt():
    import torch

    from aesara_b200.runtime import lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return lib


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------- GEMM regions
def _gemm_inputs(case, dims, seed):
    """X-like operands dense in [-4, 4]; the right operands of products ternary and sparse (about
    eight non-zeros per column), so that region values stay within bf16's exact integers."""
    vals = FR.int_inputs(case, dims, seed)
    rng = np.random.default_rng(seed + 1)
    for k in ("W", "W2", "W3", "W4", "Gt"):
        if k in vals:
            a = vals[k]
            p = min(1.0, 8.0 / (a.shape[1] if k == "Gt" else a.shape[0]))
            vals[k] = rng.choice(np.array([-1, 0, 1], np.float32), size=a.shape, p=[p / 2, 1 - p, p / 2])
    return vals


class _Run:
    pass


def _run_gemm(monkeypatch, name, precision, dims=None, vals=None, seed=0, calls=1, fuse=True):
    from aesara_b200.runtime import kernels as K
    from aesara_b200.runtime.vm import ProgramExecutor

    case = FR.GEMM[name]
    dims = dict(DIMS, **(dims or {}))
    if precision == 0:
        monkeypatch.setenv("AB_GEMM_FUSE_FP32", "1")
    if not fuse:
        monkeypatch.setenv("AB_NO_GEMM_FUSE", "1")
    reqs = []
    real = K.gemm

    def gemm(C_, alpha, A, B, beta, precision=0, cache=None, cin=None, epilogue=None):
        before = dict(K.TC_LAUNCHES)
        real(C_, alpha, A, B, beta, precision, cache=cache, cin=cin, epilogue=epilogue)
        if epilogue is not None:
            launched = [k for k, n in K.TC_LAUNCHES.items() if n != before.get(k, 0)]
            reqs.append({"plan": list(epilogue.out_plan), "applied": epilogue.applied, "launch": launched,
                         "ops": [(0 if a.shape[0] == 1 else a.strides[0], 0 if a.shape[1] == 1 else a.strides[1],
                                  a.shape) for a in epilogue.operands]})

    monkeypatch.setattr(K, "gemm", gemm)
    prog = FR.gemm_program(name)
    ex = ProgramExecutor(prog, precision=precision)
    if not fuse:
        monkeypatch.delenv("AB_NO_GEMM_FUSE")
    vals = vals if vals is not None else _gemm_inputs(case, dims, seed)
    ins = [vals[k] for k in case.inputs]
    r = _Run()
    r.outs = [ex(*ins) for _ in range(calls)]
    r.got = r.outs[-1]
    r.ex, r.prog, r.reqs, r.vals, r.case, r.dims = ex, prog, reqs, vals, case, dims
    fs = [f for f in ex._fusions if type(f).__name__ == "GemmEpilogueFusion"]
    r.f = fs[0] if fs else None
    r.defines = FR.defines(r.f.source()) if r.f is not None else {}
    return r


def _assert_exact(got, want, what):
    got = np.asarray(got)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    g = got.astype(np.float64)
    bad = ~((g == want) | (np.isnan(g) & np.isnan(want)))
    if bad.any():
        idx = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements differ; first at {idx}: "
                             f"got {got[idx]!r}, want {want[idx]!r}")


def _classify(r, k, rs, cs, shape):
    if rs == 0 and cs == 0:
        return "scalar"
    if rs == 0:
        return "row_static" if (r.defines["AB_EP_ROWMASK"] >> k) & 1 else (
            "row_pre" if k == r.defines["AB_EP_PRE_OP"] else "row_shuffle")
    if cs == 0:
        return "col"
    if cs != 1:
        return "strided"
    kind = "mn_pre" if k == r.defines["AB_EP_PRE_OP"] else "mn_ld8"
    return kind + ("_reversed" if rs < 0 else "")


def _expect_fused(r, precision, ops=None):
    """The region ran fused, with the ``#define``s the catalogue names; records every side."""
    case = r.case
    assert r.f is not None, f"{case.name}: no GEMM-epilogue region detected"
    assert not r.f.broken, f"{case.name}: the fused launch was refused"
    assert r.ex.fused_regions_run >= 1, f"{case.name}: the region did not run"
    assert r.reqs and all(q["applied"] for q in r.reqs), f"{case.name}: the fused kernel did not take the product"
    d = r.defines
    want = case.expect["defines"]
    if want is not None:
        want = dict(want)
        if precision != 2:
            want["AB_EP_TPLANE"] = -1
        for k, v in want.items():
            assert d[k] == v, f"{case.name} precision {precision}: {k} = {d[k]}, expected {v}"
    assert d["AB_EP_EXACT_SUMS"] == (precision == 0)
    for key in ("NOPS", "NOUT", "COLSUM", "FULLSUM", "CIN", "TPLANE", "EXACT_SUMS"):
        REACHED[key].add(d["AB_EP_" + key])
    REACHED["PRE_OP"].add(d["AB_EP_PRE_OP"] if d["AB_EP_PRE_OP"] <= 0 else ">0")
    REACHED["ROWMASK"].add(d["AB_EP_ROWMASK"] != 0)
    for q in r.reqs:
        for k, (rs, cs, shape) in enumerate(q["ops"]):
            REACHED["operand"].add(_classify(r, k, rs, cs, shape))
        for store, nat, tr in q["plan"]:
            if store or nat or tr:
                REACHED["plan"].add(("f32" if store else "plane_only") + ("+nat" if nat else "") + ("+T" if tr else ""))
        for key in q["launch"]:
            if key[0]:
                REACHED["layout"].add((key[1], key[2], key[3]))
    g = r.prog.nodes[r.f.g]
    REACHED["product"].add(g.op + ("{inplace}" if g.params.get("inplace") else ""))
    REACHED["precision"].add(precision)
    M, N = r.dims["M"], r.dims["N"]
    REACHED["M"].add(M)
    REACHED["N"].add(N)
    if -(-M // 128) * -(-N // 128) > _sms():
        REACHED["tiles"].add(">sms")


def _check_truth(r, what):
    want = FR.truth(r.case, r.vals)
    for k, (g, w) in enumerate(zip(r.got, want)):
        _assert_exact(g, w, f"{what} output {k}")


CASES = [n for n, c in FR.GEMM.items() if c.exact and n not in ("mn_misaligned", "gemm_z_misaligned")]


@pytest.mark.parametrize("precision", PRECISIONS, ids=lambda p: f"prec{p}")
@pytest.mark.parametrize("name", CASES)
def test_gemm_region_exact(rt, monkeypatch, name, precision):
    r = _run_gemm(monkeypatch, name, precision, calls=2)
    _expect_fused(r, precision)
    _check_truth(r, f"{name} precision {precision}")
    for k, (a, b) in enumerate(zip(*r.outs)):
        _assert_exact(a, b, f"{name}: second call, output {k}")
    left = r.case.expect["left_out"]
    cand = [i for i, n in enumerate(r.prog.nodes) if i > r.f.g and n.op in ("Elemwise", "CAReduce")]
    assert len(cand) - (len(r.f.members) - 1) >= left
    if left:
        REACHED["shrink"].add(name)
    if any(not s and (n or t) for q in r.reqs for s, n, t in q["plan"]):
        assert r.f.f32_skipped >= 1


@pytest.mark.parametrize("precision", (0, 2), ids=lambda p: f"prec{p}")
@pytest.mark.parametrize("M,N", [(64, 64), (97, 136), (129, 520), (4099, 64), (4099, 136), (4099, 520), (64, 520)],
                         ids=lambda v: str(v))
@pytest.mark.parametrize("name", ["ops4", "col_full_diff", "plane_t_colsum"])
def test_gemm_region_shapes(rt, monkeypatch, name, M, N, precision):
    """Ragged 32-row warps and 128-row / 128-column tiles, a K tail (520 = 8 x 64 + 8), more tiles
    than SMs (each persistent CTA reuses its staging buffer)."""
    r = _run_gemm(monkeypatch, name, precision, dims={"M": M, "N": N})
    _expect_fused(r, precision)
    _check_truth(r, f"{name} {M}x{N} precision {precision}")


@pytest.mark.parametrize("K", [32 * 64 + 8, 2048], ids=lambda k: f"K{k}")
def test_gemm_region_long_k(rt, monkeypatch, K):
    r = _run_gemm(monkeypatch, "col_full_same", 2, dims={"M": 97, "N": 136, "K": K})
    _expect_fused(r, 2)
    _check_truth(r, f"K={K}")


@pytest.mark.parametrize("xt,wt", [(0, 1), (0, 0), (1, 1), (1, 0)], ids=["aK_bK", "aK_bMN", "aMN_bK", "aMN_bMN"])
def test_gemm_region_bf16_layouts(rt, monkeypatch, xt, wt):
    """The four bf16 entry points (K-/MN-major A and B) on a region with both sums: X or its
    transposed view, W or its transposed view, packed without the transposing pack (a row-major W
    is the MN-major B operand)."""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    case = FR.GEMM["col_full_same"]
    vals = _gemm_inputs(case, DIMS, 3)
    from aesara_b200.runtime.device import DeviceArray

    # the same values through transposed device views
    dv = dict(vals)
    if xt:
        dv["X"] = DeviceArray.from_numpy(np.ascontiguousarray(vals["X"].T)).dimshuffle([1, 0])
    if wt:
        dv["W"] = DeviceArray.from_numpy(np.ascontiguousarray(vals["W"].T)).dimshuffle([1, 0])
    r = _run_gemm(monkeypatch, "col_full_same", 2, vals=dv)
    r.vals = vals
    _expect_fused(r, 2)
    _check_truth(r, f"layout {xt}{wt}")
    keys = [k for q in r.reqs for k in q["launch"] if k[0]]
    assert keys == [(True, 2, xt, 1 - wt)], f"fused launch layouts {keys}"


@pytest.mark.parametrize("precision", PRECISIONS, ids=lambda p: f"prec{p}")
def test_gemm_inplace_planes(rt, monkeypatch, precision):
    """Dot22 -> Gemm{inplace}(h, ..) -> Elemwise{inplace}, with h also read by h @ W4 first: the
    region writes t into h's memory.  Under every policy t @ W3 must read t, not a pack of h (a
    stale pack is certain under 3xTF32, whose hi/lo pack is always a copy), and under bf16 the
    plane-only t has no float32 copy, so beta * z is read through C_in, not a null C."""
    r = _run_gemm(monkeypatch, "gemm_inplace", precision, calls=2)
    _expect_fused(r, precision)
    g = r.prog.nodes[r.f.g]
    assert g.op == "Gemm" and g.params["inplace"]
    _check_truth(r, f"gemm_inplace precision {precision}")
    for k, (a, b) in enumerate(zip(*r.outs)):
        _assert_exact(a, b, f"gemm_inplace precision {precision}: second call, output {k}")
    if precision == 2:
        assert r.reqs[0]["plan"][0][0] is False, "t was expected as a bf16 plane only"
        REACHED["inplace"].add("plane_only")
    REACHED["inplace"].add(precision)


@pytest.mark.parametrize("name,dims", [("bias_static", {"N": 68}), ("mn_misaligned", {}),
                                       ("gemm_z_misaligned", {})], ids=["n68", "op_misaligned", "z_misaligned"])
def test_gemm_region_refused(rt, monkeypatch, name, dims):
    """A fused launch the kernel refuses (N % 8 != 0, an [M,N] operand or z 4 bytes off 16-byte
    alignment) marks the region broken, runs node by node, and stays correct on the next call."""
    r = _run_gemm(monkeypatch, name, 2, dims=dims, calls=2)
    assert r.f is not None and r.f.broken, f"{name}: the region was not refused"
    assert r.ex.fused_regions_run == 0
    _check_truth(r, name)
    for k, (a, b) in enumerate(zip(*r.outs)):
        _assert_exact(a, b, f"{name}: second call, output {k}")
    REACHED["refusal"].add(name + str(dims))


@pytest.mark.parametrize("precision", (0, 2), ids=lambda p: f"prec{p}")
@pytest.mark.parametrize("kind", ["nan_element", "inf_pair_column", "nan_row_of_a"])
def test_gemm_region_nonfinite(rt, monkeypatch, kind, precision):
    """A NaN in one operand element reaches exactly its element, its column sum and the total;
    +inf and -inf in one column give a NaN column sum; a NaN row of A stays in its row."""
    case = FR.GEMM["col_full_same"]
    vals = _gemm_inputs(case, DIMS, 5)
    i, j = 70, 77
    if kind == "nan_element":
        vals["Z"][i, j] = np.nan
    elif kind == "inf_pair_column":
        vals["Y"][[3, 100], j] = np.inf
        vals["Z"][3, j], vals["Z"][100, j] = 1, -1
    else:
        vals["X"][i, :] = np.nan
    r = _run_gemm(monkeypatch, "col_full_same", precision, vals=vals)
    _expect_fused(r, precision)
    _check_truth(r, kind)
    h, cs, tot = r.got
    if kind == "nan_row_of_a":
        assert np.isnan(h[i]).all() and not np.isnan(np.delete(h, i, axis=0)).any()
    else:
        assert np.isnan(cs[j]) and np.isfinite(np.delete(cs, j)).all() and np.isnan(tot)
    REACHED["nonfinite"].add(kind)


@pytest.mark.parametrize("precision", PRECISIONS, ids=lambda p: f"prec{p}")
def test_colsum_float32_overflow(rt, monkeypatch, precision):
    """A column whose float32 partial sums overflow while its float64 sum is finite: rows 0, 2
    hold +2**127 and rows 32, 34 hold -2**127 (they cancel in float64).  The epilogue's float pairs
    (3xTF32) and float32 trees (bf16, TF32) add rows 0 and 2 to +inf in the first 32-row block and
    rows 32 and 34 to -inf in the second, so the fused column sum is not finite, where the
    node-by-node float64 CAReduce is finite.  This is the documented limit of the float-pair sums;
    every other column stays exact.  The total stays finite but loses the addends the +-2**127
    partials absorb: measured on an H100 80GB HBM3 (700 W), at this seed and under every policy,
    -363 against the float64 -530; pinned."""
    case = FR.GEMM["col_full_same"]
    vals = _gemm_inputs(case, DIMS, 6)
    j = 9
    big = np.float32(2.0 ** 127)
    vals["Y"][[0, 2, 32, 34], j] = big
    vals["Z"][[0, 2, 32, 34], j] = [1, 1, -1, -1]
    r = _run_gemm(monkeypatch, "col_full_same", precision, vals=vals)
    _expect_fused(r, precision)
    want = FR.truth(case, vals)
    h, cs, tot = r.got
    _assert_exact(h, want[0], "values")
    assert np.isfinite(want[1][j]) and np.isfinite(want[2])
    assert not np.isfinite(cs[j]), f"column sum {cs[j]!r}: the float32 overflow did not show"
    assert float(want[2]) == -530.0 and float(tot) == -363.0, f"total {tot!r} (float64: {want[2]!r})"
    _assert_exact(np.delete(cs, j), np.delete(want[1], j), "other columns")
    NOTES.append(f"float32 overflow, precision {precision}: column sum {cs[j]!r}, total {tot!r} "
                 f"(float64: {want[1][j]!r}, {want[2]!r})")
    REACHED["nonfinite"].add("overflow")


def test_gemm_region_late_operand(rt, monkeypatch):
    """An operand computed by another node of the graph (a [1, 1] factor from X's shape)."""
    r = _run_gemm(monkeypatch, "late_operand", 2)
    _expect_fused(r, 2)
    _check_truth(r, "late_operand")
    REACHED["anchor"].add("late" if r.f.anchor > r.f.g else "at_gemm")


def _ulps32(got, ref):
    ref = np.asarray(ref, np.float64)
    e = np.maximum(np.frexp(np.abs(ref))[1] - 1, -126)
    return np.abs(got.astype(np.float64) - ref) / np.ldexp(1.0, e - 23)


@pytest.mark.parametrize("precision", PRECISIONS, ids=lambda p: f"prec{p}")
def test_gemm_region_transcendental(rt, monkeypatch, precision):
    """tanh, sigmoid * exp and softplus of the exact product h = acc / 16 + b: bit-identical to the
    node-by-node Elemwise kernels; against float64 within tanh 2 ulp, softplus 3.5 ulp and
    sigmoid * exp 3.5 + 2 + 0.5 (the product's rounding) = 6 ulp."""
    vals = _gemm_inputs(FR.GEMM["transc"], DIMS, 7)
    r = _run_gemm(monkeypatch, "transc", precision, vals=vals)
    _expect_fused(r, precision)
    ref = _run_gemm(monkeypatch, "transc", precision, vals=vals, fuse=False)
    assert ref.ex.fused_regions_run == 0 or ref.f is None
    want = FR.truth(r.case, vals)
    for k, (g, n, w, bound) in enumerate(zip(r.got, ref.got, want, (2.0, 6.0, 3.5))):
        assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(n).view(np.uint32)), \
            f"output {k}: fused != node by node"
        u = float(np.max(_ulps32(np.asarray(g), w)))
        assert u <= bound, f"output {k}: {u} ulp > {bound}"


# ---------------------------------------------------------------------------- row regions
ROW_D = [4, 124, 128, 132, 384, 388, 640, 700, 896, 1020, 1024]


def _row_inputs(case, N, D, seed):
    vals = FR.int_inputs(case, {"N": N, "D": D}, seed)
    rng = np.random.default_rng(seed + 2)
    vals["w"] = rng.integers(-2, 3, D).astype(np.float32)
    # about a tenth of the rows inside the clip range, the rest clipped at +-8
    vals["w"][rng.random(D) < 0.5] = 0
    if "s" in vals:
        vals["s"] = np.float32(3)
    if "m" in vals:
        vals["m"] = rng.random(N) < 0.5
    return vals


def _run_row(name, N, D, seed=0, vals=None, X=None):
    from aesara_b200.runtime.vm import ProgramExecutor

    case = FR.ROW[name]
    prog = FR.row_program(name)
    ex = ProgramExecutor(prog)
    vals = vals if vals is not None else _row_inputs(case, N, D, seed)
    ins = [vals[k] if k != "X" or X is None else X for k in case.inputs]
    got = ex(*ins)
    fs = [f for f in ex._fusions if type(f).__name__ == "RowFusion"]
    assert len(fs) == 1, f"{name}: {len(fs)} row regions"
    return got, ex, fs[0], vals, case


def _row_truth(case, vals):
    return FR.truth(case, vals)


def _row_record(f, ex, N, D):
    assert ex.fused_regions_run == 1, "the row region did not run fused"
    J = (D + 127) // 128
    assert any(k[0] == J and m["handle"] is not None for k, m in f._modules.items()), f"J={J} module not used"
    REACHED["J"].add(J)
    rows = 8
    REACHED["rowN"].add("0" if N == 0 else "<8" if N < rows else "8" if N == rows else
                        ">grid" if N > _sms() * 6 * rows else ">8")
    REACHED["sums"].add(len(f.sums))


@pytest.mark.parametrize("D", ROW_D, ids=lambda d: f"D{d}")
def test_row_region_every_j(rt, D):
    got, ex, f, vals, case = _run_row("sums2", 257, D, seed=D)
    _row_record(f, ex, 257, D)
    for k, (g, w) in enumerate(zip(got, _row_truth(case, vals))):
        _assert_exact(g, w, f"D={D} output {k}")


@pytest.mark.parametrize("N", [1, 7, 8, 9, 132 * 6 * 8 + 1, 20000], ids=lambda n: f"N{n}")
def test_row_region_rows(rt, N):
    got, ex, f, vals, case = _run_row("sums1", N, 132, seed=N)
    _row_record(f, ex, N, 132)
    for k, (g, w) in enumerate(zip(got, _row_truth(case, vals))):
        _assert_exact(g, w, f"N={N} output {k}")


@pytest.mark.parametrize("name", ["sums0", "sums1", "sums2", "strided", "int32", "bool", "scalar"])
def test_row_region_operands(rt, name):
    got, ex, f, vals, case = _run_row(name, 300, 388, seed=11)
    _row_record(f, ex, 300, 388)
    for k, (g, w) in enumerate(zip(got, _row_truth(case, vals))):
        _assert_exact(g, w, f"{name} output {k}")
    key = [k for k, m in f._modules.items() if m["handle"] is not None][0]
    for cls, by_ptr, v in zip(key[1], key[2], f.ext):
        dt = ex.program.vars[v].dtype
        REACHED["row_ext"].add(f"{cls}:{dt}" + (":ptr" if by_ptr else ":value" if cls == "scal" else ""))
    if name == "strided":
        REACHED["row_ext"].add("strided")


@pytest.mark.parametrize("kind", ["N0", "D1028", "D130", "misaligned", "row_stride"])
def test_row_region_fallback(rt, kind):
    """Operands the row kernel does not take run node by node, and stay exact."""
    from aesara_b200.runtime.device import DeviceArray

    N, D, X = 50, 132, None
    if kind == "N0":
        N = 0
    elif kind == "D1028":
        D = 1028
    elif kind == "D130":
        D = 130
    case = FR.ROW["sums1"]
    vals = _row_inputs(case, N, D, 13)
    if kind == "misaligned":  # 4 bytes off 16-byte alignment
        buf = DeviceArray.from_numpy(np.concatenate([np.zeros(1, np.float32), vals["X"].ravel()]))
        X = buf.view((N, D), (D, 1), offset_elems=1)
    elif kind == "row_stride":  # rows 134 floats apart
        wide = np.zeros((N, D + 2), np.float32)
        wide[:, :D] = vals["X"]
        X = DeviceArray.from_numpy(wide).index((slice(None), slice(0, D)))
    got, ex, f, _, _ = _run_row("sums1", N, D, vals=vals, X=X)
    if X is not None:
        assert X.ptr % 16 or X.strides[0] % 4, "the view was meant to be misaligned"
    assert ex.fused_regions_run == 0, f"{kind}: the row region was expected to fall back"
    for k, (g, w) in enumerate(zip(got, _row_truth(case, vals))):
        _assert_exact(g, w, f"{kind} output {k}")
    REACHED["row_fallback"].add(kind)


def test_row_region_sigmoid(rt):
    """r = sigmoid(z / 8) - y per row.  Each z is exact (an integer), so r carries sigmoid's own
    error (3.5 ulp of r's sigmoid term, at most 3.5 * 2**-24 absolute since sigmoid < 1) plus the
    subtraction's rounding (2**-24 |r|).  X.T @ r: the kernel adds N terms per column, each
    |x| <= 4, in float32 (fmaf per lane, then the shuffle tree and the float32 partials per CTA
    summed in float64): at most (N - 1) * 2**-24 * sum |x r| of rounding, plus sum |x| times the
    per-row error above.  The sums of r add float64 partials of float32-rounded r."""
    N, D = 1000, 256
    got, ex, f, vals, case = _run_row("sigmoid", N, D, seed=17)
    _row_record(f, ex, N, D)
    want = _row_truth(case, vals)
    X = vals["X"].astype(np.float64)
    z = X @ vals["w"].astype(np.float64)
    r = 1.0 / (1.0 + np.exp(-z * 0.125)) - vals["y"]
    row_err = 4.5 * 2.0 ** -24 * (1 + np.abs(r))
    bound_gw = (N - 1) * 2.0 ** -24 * (np.abs(X).T @ np.abs(r)) + np.abs(X).T @ row_err
    assert np.all(np.abs(got[0] - want[0]) <= bound_gw), float(np.max(np.abs(got[0] - want[0]) / bound_gw))
    assert abs(float(got[1]) - float(want[1])) <= float(np.sum(row_err)) + 2.0 ** -24 * abs(float(want[1]))


# ---------------------------------------------------------------------------- every side
def test_zz_every_side_reached():
    expect = {
        "NOPS": {0, 1, 2, 3, 4}, "NOUT": {1, 2, 3}, "COLSUM": {-1, 0, 1, 2}, "FULLSUM": {-1, 0, 1},
        "CIN": {0, 1}, "PRE_OP": {-1, 0, ">0"}, "TPLANE": {-1, 0}, "EXACT_SUMS": {0, 1},
        "ROWMASK": {False, True},
        "operand": {"scalar", "row_static", "row_pre", "row_shuffle", "col", "mn_pre", "mn_ld8", "strided",
                    "mn_pre_reversed", "mn_ld8_reversed"},
        "plan": {"f32", "f32+nat", "plane_only+nat", "plane_only+T", "plane_only+nat+T"},
        "product": {"Dot22", "Dot22Scalar", "Gemm", "Gemm{inplace}"},
        "layout": {(2, 0, 0), (2, 0, 1), (2, 1, 0), (2, 1, 1)},
        "precision": {0, 1, 2}, "M": {64, 97, 129, 4099}, "N": {64, 136, 520}, "tiles": {">sms"},
        "shrink": {"shrink_ops5", "shrink_nout4", "shrink_colsum2"},
        "inplace": {0, 1, 2, "plane_only"},
        "refusal": {"bias_static{'N': 68}", "mn_misaligned{}", "gemm_z_misaligned{}"},
        "nonfinite": {"nan_element", "inf_pair_column", "nan_row_of_a", "overflow"},
        "J": set(range(1, 9)), "rowN": {"<8", "8", ">8", ">grid"}, "sums": {0, 1, 2},
        "row_ext": {"row:float32", "row:int32", "row:bool", "scal:float32:ptr", "scal:float32:value", "strided"},
        "row_fallback": {"N0", "D1028", "D130", "misaligned", "row_stride"},
    }
    for line in NOTES:
        print(line)
    print({k: sorted(map(str, v)) for k, v in REACHED.items()})
    missing = {k: sorted(map(str, v - REACHED[k])) for k, v in expect.items() if v - REACHED[k]}
    assert not missing, f"sides never reached: {missing}"
