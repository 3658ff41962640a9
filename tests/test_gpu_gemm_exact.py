"""GPU: the wgmma GEMM gives the exact product on every operand layout, scheduling path and
fused-epilogue entry point.

Operands hold small integers (|x| <= 4, or <= 2 at full size), possibly scaled by a power of
two.  They are exact in bf16, TF32 and float32, and so is every product.  The generator checks
that K * max|a| * max|b| <= 2^22 (in units of the operands' scale), so every partial sum a kernel
can form is an integer below 2^22 and exact in float32 as well: truncation in the tensor core's
accumulator, the order and rounding of segment folds, the order in which split-K partials are
added and alpha / beta from {1, 0.5, -2, 0} with an integer C_in cannot change the result.  The
float64 product cast to float32 is the answer, and every element must equal it; a mismatch is
reported by count, position and 128 x 128 tile, so a misplaced tile, k-block, chunk or swizzle
shows up as a pattern.

Which MMA loop or fused entry point ran is read from ``kernels.TC_LAUNCHES``; the last test
asserts that every one of them was launched in the session.  Rounding, which integers cannot
see, is checked against a policy-aware float64 truth (operands rounded to bf16 first).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests._cases import fused_vs_plain, load_case, mlp_inputs, mlp_truth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUM_BOUND = 1 << 22
FLT_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def K():
    import torch

    from aesara_b200.runtime import kernels, lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return kernels


# ----------------------------------------------------------------------------- helpers
def ints(rng, shape, amax=4, scale=1.0):
    return (rng.integers(-amax, amax + 1, size=shape) * scale).astype(np.float32)


def check_bound(k, amax, bmax):
    """Every partial sum of a length-k dot product of such operands is exact in float32."""
    assert k * amax * bmax <= SUM_BOUND, f"K={k}: partial sums may exceed 2^22"


def truth(a, b, alpha=1.0, beta=0.0, cin=None):
    """alpha * a @ b + beta * cin in float64 (on the device), which must be a float32 value."""
    import torch

    ad = torch.as_tensor(a, device="cuda").double()
    bd = torch.as_tensor(b, device="cuda").double()
    w = alpha * (ad @ bd)
    if cin is not None and beta != 0.0:
        w += beta * torch.as_tensor(cin, device="cuda").double()
    w = w.cpu().numpy()
    fin = np.isfinite(w)
    assert np.array_equal(w[fin], w[fin].astype(np.float32).astype(np.float64)), "truth is not a float32 value"
    return w.astype(np.float32)


def assert_exact(got, want, what):
    """Every element equal (NaN where NaN is expected); on a mismatch: how many, where, which tiles."""
    got = np.asarray(got, np.float32)
    want = np.asarray(want, np.float32)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        r, c = np.nonzero(bad)
        first = [(int(i), int(j), float(got[i, j]), float(want[i, j])) for i, j in zip(r[:6], c[:6])]
        tiles = sorted({(int(i) // 128, int(j) // 128) for i, j in zip(r, c)})
        raise AssertionError(
            f"{what}: {bad.sum()} of {got.size} elements wrong; first (row, col, got, want): {first}; "
            f"{len(tiles)} tiles (row // 128, col // 128): {tiles[:12]}{' ...' if len(tiles) > 12 else ''}")


def operand(x, layout, role):
    """The logical operand x (A [m, k] or B [k, n]) as a DeviceArray in the given layout:
    'k' K contiguous, 'mn' M / N contiguous (a transposed view of the stored matrix),
    'kpad' / 'mnpad' the same as a slice of a wider buffer (row pitch > extent)."""
    from aesara_b200.runtime.device import DeviceArray

    k_axis = 1 if role == "a" else 0
    fast = k_axis if layout.startswith("k") else 1 - k_axis
    store = x if fast == 1 else x.T
    pad = (-store.shape[1]) % 8 + 8 if layout.endswith("pad") else 0
    buf = np.zeros((store.shape[0], store.shape[1] + pad), np.float32)
    buf[:, : store.shape[1]] = store
    d = DeviceArray.from_numpy(buf)
    if pad:
        d = d.index((slice(None), slice(0, store.shape[1])))
    return d if fast == 1 else d.dimshuffle([1, 0])


def mn_flag(layout, precision, no_tpack, elems):
    """mn_major of the packed operand: bf16 only; a small matrix gets a transposing pack unless
    AB_GEMM_NO_TPACK is set (runtime/kernels.py PackCache.operand)."""
    from aesara_b200.runtime.kernels import PackCache

    return int(precision == 2 and layout.startswith("mn") and (no_tpack or elems > PackCache.TRANSPOSE_PACK_MAX))


def launched(K, before):
    return {k for k, v in K.TC_LAUNCHES.items() if v > before.get(k, 0)}


def run_gemm(K, a, b, precision, la="k", lb="k", alpha=1.0, beta=0.0, c0=None, cin=None, c_order="C",
             cache=None):
    """C <- alpha * A @ B + beta * (cin or C) through kernels.gemm; returns (C as NumPy, launched keys).
    With a separate cin, C starts as NaN: the kernel must not read it."""
    from collections import Counter

    from aesara_b200.runtime.device import DeviceArray

    m, n = a.shape[0], b.shape[1]
    init = c0 if c0 is not None else np.full((m, n), np.nan if cin is not None else 0.0, np.float32)
    C = DeviceArray.from_numpy(init) if c_order == "C" else DeviceArray.from_numpy(init.T.copy()).dimshuffle([1, 0])
    A, B = operand(a, la, "a"), operand(b, lb, "b")
    before = Counter(K.TC_LAUNCHES)
    K.gemm(C, alpha, A, B, beta, precision=precision, cache=cache,
           cin=DeviceArray.from_numpy(cin) if cin is not None else None)
    return C.to_numpy(), launched(K, before), (A, B)


def exact_case(K, m, n, k, precision, la="k", lb="k", no_tpack=False, alpha=1.0, beta=0.0, separate_cin=False,
               c_order="C", seed=0, what=""):
    rng = np.random.default_rng(seed + m + 3 * n + 7 * k + precision)
    check_bound(k, 4, 4)
    a, b = ints(rng, (m, k)), ints(rng, (k, n))
    c = ints(rng, (m, n), 64) if beta != 0.0 else None
    got, keys, ops = run_gemm(K, a, b, precision, la, lb, alpha, beta,
                              c0=None if separate_cin else c, cin=c if separate_cin else None, c_order=c_order)
    what = what or f"{m}x{n}x{k} precision {precision} {la}/{lb}"
    assert_exact(got, truth(a, b, alpha, beta, c), what)
    if K._lib.load().ab_gemm_tensorcore_eligible(m, n, k):
        want_key = (False, precision, mn_flag(la, precision, no_tpack, m * k), mn_flag(lb, precision, no_tpack, k * n))
        assert keys == {want_key}, f"{what}: launched {keys}, expected {want_key}"
    else:
        assert not keys, f"{what}: a tensor-core kernel ran below ab_gemm_tensorcore_eligible"
    return got


LAYOUTS = [("k", "k"), ("k", "mn"), ("mn", "k"), ("mn", "mn")]
# 330 units (2-3 tiles per CTA, M / N / K ragged: K tail 40 bf16 / 8 tf32); 63 tile rows with
# group_m 8 (a last group of 7 rows, 315 units); 18 bf16 k-blocks (segments of 16 + 2); K < one k-block
SHAPES = [(4099, 1153, 1000), (7957, 640, 520), (640, 768, 1100), (1000, 520, 33)]


# ----------------------------------------------------------------------------- the AOT kernels
@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("la,lb", LAYOUTS)
@pytest.mark.parametrize("precision,no_tpack", [(0, False), (1, False), (2, False), (2, True)])
def test_exact_every_layout(K, monkeypatch, m, n, k, la, lb, precision, no_tpack):
    """Both operand majors (MN-major stays MN-major under AB_GEMM_NO_TPACK, bf16; the transposing
    pack otherwise) on multi-unit, ragged-group, two-segment and sub-k-block shapes."""
    if no_tpack:
        monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    exact_case(K, m, n, k, precision, la, lb, no_tpack)


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_exact_padded_operands_and_column_major_c(K, monkeypatch, precision):
    """Operands sliced from wider buffers (pitch > extent) and a column-major C with beta != 0.
    Under TF32 the K-major slice is read in place (plan_operand's direct operand)."""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    m, n, k = 4099, 1153, 1000
    rng = np.random.default_rng(17 + precision)
    a, b, c = ints(rng, (m, k)), ints(rng, (k, n)), ints(rng, (m, n), 64)
    cache = K.PackCache()
    for la, lb in (("kpad", "mnpad"), ("mnpad", "kpad")):
        got, keys, (A, B) = run_gemm(K, a, b, precision, la, lb, -2.0, 0.5, c0=c, c_order="F", cache=cache)
        assert_exact(got, truth(a, b, -2.0, 0.5, c), f"precision {precision} {la}/{lb}, column-major C")
        assert keys == {(False, precision, mn_flag(la, precision, True, 0), mn_flag(lb, precision, True, 0))}
        if precision == 1 and la == "kpad":
            ent = cache._e[(A.ptr, m, k, A.strides[0], 0, 1)]
            assert ent[1] == A.ptr, "the TF32 K-major slice was packed instead of read in place"


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("la,lb", [("k", "k"), ("mn", "mn")])
@pytest.mark.parametrize("splits,alpha,beta", [(2, 0.5, -2.0), (3, -2.0, 1.0), (7, 1.0, 0.5), (3, 0.0, -2.0)])
def test_exact_split_k(K, monkeypatch, precision, la, lb, splits, alpha, beta):
    """Forced split-K at (700, 900, 9000) with alpha, beta and a separate C_in: 7 ranges are 336
    units under the tf32 policies (bf16 rounds to whole segments: 5 ranges, 240 units), so each
    CTA gets units from different K ranges; C starts as NaN and must not be read."""
    import ctypes as C

    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    monkeypatch.setenv("AB_GEMM_SPLITK", str(splits))
    m, n, k = 700, 900, 9000
    need = C.c_size_t()
    K._lib.check(K._lib.load().ab_gemm_packed_workspace_bytes(precision, m, n, k, C.byref(need)))
    assert need.value > 0, "expected the split-K path"
    exact_case(K, m, n, k, precision, la, lb, True, alpha, beta, separate_cin=True)


@pytest.mark.parametrize("knob", [("AB_GEMM_STAGES", "2"), ("AB_GEMM_GROUP_M", "3")])
@pytest.mark.parametrize("m,n,k", [(4099, 1153, 1000), (7957, 640, 520)])
@pytest.mark.parametrize("precision,la,lb", [(0, "k", "k"), (1, "mn", "k"), (2, "k", "k"), (2, "mn", "mn"),
                                              (2, "k", "mn")])
def test_exact_ring_and_unit_order(K, monkeypatch, knob, m, n, k, precision, la, lb):
    """Two ring stages (the ring wraps every second k-block, across unit boundaries) and a
    group_m of 3, on multi-unit shapes."""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    monkeypatch.setenv(*knob)
    exact_case(K, m, n, k, precision, la, lb, True, 0.5, 1.0)


@pytest.mark.parametrize("m,n,k", [(2300, 520, 1100), (8191, 1024, 600)])
@pytest.mark.parametrize("precision,la,lb", [(0, "k", "k"), (0, "mn", "mn"), (2, "k", "k"), (2, "k", "mn"),
                                              (2, "mn", "mn")])
def test_exact_four_cta_cluster(K, monkeypatch, m, n, k, precision, la, lb):
    """CTA pairs, which replaced the 4-CTA cluster this test is named after.
    AB_GEMM_CLUSTER=2 (CTA pairs, under the 3xTF32 policy too) on a ragged M (the second CTA of
    the last pair partly or wholly out of range) and on a multi-unit shape (~256 pair tiles for
    ~66 resident pairs), with K- and MN-major B (per-chunk multicast): exact, and bit-identical to
    the single-CTA kernel (AB_GEMM_CLUSTER=1)."""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    monkeypatch.setenv("AB_GEMM_CLUSTER", "2")
    got = exact_case(K, m, n, k, precision, la, lb, True, 1.0, -2.0, what=f"pair {m}x{n}x{k} {la}/{lb}")
    monkeypatch.setenv("AB_GEMM_CLUSTER", "1")
    single = exact_case(K, m, n, k, precision, la, lb, True, 1.0, -2.0)
    np.testing.assert_array_equal(got, single)


@pytest.mark.parametrize("m,n,k", [(512, 768, 640), (4096, 1152, 640), (1024, 256, 200), (300, 520, 512)])
@pytest.mark.parametrize("la,lb", [("mn", "k"), ("k", "mn"), ("mn", "mn")])
def test_exact_mn_major_3d_tiles(K, monkeypatch, m, n, k, la, lb):
    """MN-major bf16 tiles, one 2-D copy per 128-byte chunk, at MN extents that are multiples of
    64 and at ragged ones (300, 520).  (Named after the 3-D single-copy variant, which is gone.)"""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    exact_case(K, m, n, k, 2, la, lb, True)


@pytest.mark.parametrize("m,n,k", [(100, 70, 200), (300, 64, 33)])
@pytest.mark.parametrize("precision", [0, 2])
def test_exact_below_tensor_core_size(K, m, n, k, precision):
    """Products below ab_gemm_tensorcore_eligible take the SIMT kernel: the same exact check."""
    assert not K._lib.load().ab_gemm_tensorcore_eligible(m, n, k)
    for la, lb in LAYOUTS:
        exact_case(K, m, n, k, precision, la, lb, False, -2.0, 0.5)


def test_exact_tf32_low_planes(K):
    """3xTF32 planes, exactly: x = s (1 + m 2^-12), s = +-1, m in {0, 1}, splits into hi = s and
    lo = s m 2^-12 under any TF32 rounding.  The kernel forms lo*hi + hi*lo + hi*hi and drops
    lo*lo, so C = A @ B - loA @ loB, exact for K <= 1024 (|C| <= 2^10 in steps of 2^-12).  Pins the
    pairing of the four planes and the map_a1 / map_b1 offsets."""
    rng = np.random.default_rng(12)
    for (m, n, k), (la, lb) in (((4099, 1153, 1000), ("k", "k")), ((4099, 1153, 1000), ("mn", "mn")),
                                ((1000, 520, 36), ("k", "mn"))):
        sa, sb = rng.choice([-1.0, 1.0], (m, k)), rng.choice([-1.0, 1.0], (k, n))
        la_, lb_ = sa * rng.integers(0, 2, (m, k)) * 2.0 ** -12, sb * rng.integers(0, 2, (k, n)) * 2.0 ** -12
        a, b = (sa + la_).astype(np.float32), (sb + lb_).astype(np.float32)
        want = a.astype(np.float64) @ b.astype(np.float64) - la_ @ lb_
        assert np.array_equal(want, want.astype(np.float32).astype(np.float64))
        got, keys, _ = run_gemm(K, a, b, 0, la, lb)
        assert keys == {(False, 0, 0, 0)}
        assert_exact(got, want.astype(np.float32), f"3xTF32 planes {m}x{n}x{k} {la}/{lb}")


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("m,n,k,splits", [(4099, 1153, 1000, None), (700, 900, 9000, "3")])
def test_nonfinite_values_stay_in_their_row_and_column(K, monkeypatch, precision, m, n, k, splits):
    """A NaN at A[i, k0] (i in the last, ragged tile row) and one at B[k1, j]: exactly row i and
    column j of C are NaN, every other element is the exact product (no leak across tiles, into
    the out-of-range fill or through split-K partials)."""
    if splits:
        monkeypatch.setenv("AB_GEMM_SPLITK", splits)
    rng = np.random.default_rng(99 + k)
    a, b, c = ints(rng, (m, k)), ints(rng, (k, n)), ints(rng, (m, n), 64)
    want = truth(a, b, 0.5, -2.0, c)
    i, j = m - 2, n // 2 + 3
    a[i, k // 3] = np.nan
    b[k - 5, j] = np.nan
    want[i, :] = np.nan
    want[:, j] = np.nan
    got, keys, _ = run_gemm(K, a, b, precision, "k", "k", 0.5, -2.0, cin=c)
    assert keys == {(False, precision, 0, 0)}
    assert_exact(got, want, f"NaN placement, precision {precision}, {m}x{n}x{k}")


@pytest.mark.parametrize("precision", [0, 1])
def test_large_finite_values_stay_finite(K, precision):
    """A[i, k0] = FLT_MAX with B[k0, :] in {0, +-2^-10}: sgemm gives a finite row.  cvt.rna.tf32
    rounds FLT_MAX up to +Inf, so a 3xTF32 split of hi = Inf, lo = -Inf would turn that row into
    NaN; the pack takes the truncated value for hi when the rounded one overflows."""
    rng = np.random.default_rng(5)
    m, n, k = 1000, 1153, 520
    a, b = ints(rng, (m, k)), ints(rng, (k, n))
    i, k0 = 777, 300
    b[k0, :] = rng.choice([0.0, 2.0 ** -10, -(2.0 ** -10)], n)
    a[i, k0] = FLT_MAX
    a[i + 1, k0] = -FLT_MAX
    for la in ("k", "mn"):
        got, keys, _ = run_gemm(K, a, b, precision, la, "k")
        assert keys == {(False, precision, 0, 0)}  # tf32 operands are always packed K-major
        want = a.astype(np.float64) @ b.astype(np.float64)
        assert np.isfinite(got).all(), f"{la}: {np.count_nonzero(~np.isfinite(got))} non-finite elements"
        rows = [i, i + 1]
        err = np.max(np.abs(got[rows] - want[rows])) / np.max(np.abs(want[rows]))
        assert err < (1e-5 if precision == 0 else 2e-3), f"{la}: rows with FLT_MAX, normwise error {err:.3g}"
        keep = np.ones(m, bool)
        keep[rows] = False
        assert_exact(got[keep], want[keep].astype(np.float32), f"{la}: the other rows")


# ----------------------------------------------------------------------------- full size
@pytest.mark.parametrize("case", ["fwd_k_k", "fwd_k_mn", "wgrad_k_k", "wgrad_mn_mn"])
def test_exact_full_size_bf16(K, monkeypatch, case):
    """The cfg3 product shapes under the bf16 policy: 65536 x 4096 x 4096 (X @ W1) with W1
    K-major (transposing pack) and MN-major (AB_GEMM_NO_TPACK); 4096 x 4096 x 65536 (X^T @ dpre)
    with K-major operands and, as in production, both MN-major (268M elements each, over the
    transposing-pack limit).  Values in [-2, 2]: |C| <= 2^18.  Truth: torch float64 on the device."""
    import torch
    from collections import Counter

    from aesara_b200.runtime.device import DeviceArray

    fwd = case.startswith("fwd")
    M, N, Kd = (65536, 4096, 4096) if fwd else (4096, 4096, 65536)
    check_bound(Kd, 2, 2)
    g = torch.Generator(device="cuda").manual_seed(len(case) + Kd)
    la, lb = case.split("_")[1:]
    if case == "fwd_k_mn":
        monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")

    def make(rows, cols, layout, role):
        # the logical [rows, cols] operand stored so that its K (or M / N) index is contiguous
        k_axis = 1 if role == "a" else 0
        fast = k_axis if layout == "k" else 1 - k_axis
        shape = (rows, cols) if fast == 1 else (cols, rows)
        t = torch.randint(-2, 3, shape, device="cuda", generator=g, dtype=torch.int8).float()
        return t if fast == 1 else t.T

    a, b = make(M, Kd, la, "a"), make(Kd, N, lb, "b")
    C = DeviceArray.empty((M, N), "float32")
    before = Counter(K.TC_LAUNCHES)
    K.gemm(C, 1.0, DeviceArray.from_torch(a), DeviceArray.from_torch(b), 0.0, precision=2)
    want_key = (False, 2, int(la == "mn"), int(lb == "mn"))
    assert launched(K, before) == {want_key}
    got = C.owner.view(torch.float32)[: M * N].view(M, N)
    want = (a.double() @ b.double()).float()
    if not torch.equal(got, want):
        assert_exact(got.cpu().numpy(), want.cpu().numpy(), f"full size {case}")


# ----------------------------------------------------------------------------- rounding
def policy_errors(ks=(4096, 65536)):
    """bf16 policy against a policy-aware truth: operands rounded to bf16 (RNE, as the pack does),
    then multiplied in float64.  What is left is the float32 accumulation.  1536 x 1408 is 132
    output tiles: one unit per CTA and no split-K."""
    import ctypes as C
    from collections import Counter

    import torch

    from aesara_b200.runtime import kernels, lib
    from aesara_b200.runtime.device import DeviceArray

    errs = {}
    for k in ks:
        m, n = 1536, 1408
        need = C.c_size_t()
        lib.check(lib.load().ab_gemm_packed_workspace_bytes(2, m, n, k, C.byref(need)))
        assert need.value == 0
        g = torch.Generator(device="cuda").manual_seed(k)
        a = torch.randn(m, k, device="cuda", generator=g)
        b = torch.randn(k, n, device="cuda", generator=g)
        out = DeviceArray.empty((m, n), "float32")
        before = Counter(kernels.TC_LAUNCHES)
        kernels.gemm(out, 1.0, DeviceArray.from_torch(a), DeviceArray.from_torch(b), 0.0, precision=2)
        # B is row-major: MN-major once it is over the transposing-pack limit (K = 65536)
        assert launched(kernels, before) == {(False, 2, 0, mn_flag("mn", 2, "AB_GEMM_NO_TPACK" in os.environ, k * n))}
        want = a.bfloat16().double() @ b.bfloat16().double()
        got = out.owner.view(torch.float32)[: m * n].view(m, n).double()
        errs[k] = float((got - want).abs().max() / want.abs().max())
        del a, b, want, got
    return errs


POLICY_BAR = 1e-5


def test_bf16_accuracy_against_policy_aware_truth(K):
    """Norm-wise error of the bf16 policy once the operands' own rounding is taken out, against a
    bar of 1e-5 (2000 times tighter than the 2e-2 bar against the float32 operands).  Measured on
    an H100 80GB HBM3 (700 W): 1.08e-6 at K = 4096 and 1.10e-6 at K = 65536 with the default fold
    every 16 k-blocks; without folding (AB_GEMM_SEG_KB=0) 5.5e-6 and 8.5e-5, which this bar fails
    at K = 65536 (test_segment_fold_lengths_in_a_child_process)."""
    errs = policy_errors()
    print("bf16 policy-aware normwise error:", errs)
    for k, e in errs.items():
        assert e < POLICY_BAR, f"K={k}: {e:.3g}"


def _seg_child():
    """Run in a child process with AB_GEMM_SEG_KB set (read once per process in gemm_run):
    exact products under the policies that fold segments, then the bf16 rounding measure."""
    import torch

    from aesara_b200.runtime import kernels, lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    os.environ["AB_GEMM_NO_TPACK"] = "1"
    for precision in (0, 2):
        for (m, n, k), (la, lb) in (((4099, 1153, 1000), ("k", "mn")), ((640, 768, 1100), ("mn", "mn")),
                                    ((700, 900, 9000), ("k", "k"))):
            exact_case(kernels, m, n, k, precision, la, lb, True, 0.5, -2.0)
    os.environ["AB_GEMM_SPLITK"] = "3"
    exact_case(kernels, 700, 900, 9000, 2, "mn", "k", True, 1.0, 0.5, separate_cin=True)
    exact_case(kernels, 700, 900, 9000, 0, "k", "k", True, 1.0, 0.5, separate_cin=True)
    del os.environ["AB_GEMM_SPLITK"], os.environ["AB_GEMM_NO_TPACK"]
    return policy_errors()


def test_segment_fold_lengths_in_a_child_process():
    """AB_GEMM_SEG_KB = 1, 3 (fold after every / every third k-block) and 0 (never fold): the
    integer products stay exact, and without folding the bf16 policy-aware error at K = 65536 is
    over POLICY_BAR and ten times the default's: test_bf16_accuracy_against_policy_aware_truth
    sees the fold."""
    results = {}
    for seg in ("1", "3", "0"):
        env = dict(os.environ, AB_GEMM_SEG_KB=seg,
                   PYTHONPATH=os.pathsep.join(p for p in (ROOT, os.environ.get("PYTHONPATH")) if p))
        code = "import json; from tests import test_gpu_gemm_exact as t; print('SEG ' + json.dumps(t._seg_child()))"
        args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
        r = subprocess.run(args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, f"AB_GEMM_SEG_KB={seg}: child failed\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
        line = [ln for ln in r.stdout.splitlines() if ln.startswith("SEG ")][-1]
        results[seg] = {int(k): v for k, v in json.loads(line[4:]).items()}
    print("bf16 policy-aware normwise error by AB_GEMM_SEG_KB:", results)
    default = policy_errors()
    print("default segments:", default)
    for seg in ("1", "3"):
        assert max(results[seg].values()) < POLICY_BAR
    assert results["0"][65536] > max(POLICY_BAR, 10 * default[65536]), \
        f"no fold: {results['0'][65536]:.3g}, default segments: {default[65536]:.3g}"


# ----------------------------------------------------------------------------- fused entry points
@pytest.fixture(scope="module")
def rt(K):
    from aesara_b200.runtime.vm import ProgramExecutor

    return ProgramExecutor


# entry point -> (precision, environment, X as a transposed view, W1 as a transposed view, key)
ENTRY_POINTS = {
    "ab_gemm_ep_f16": (2, {}, False, False, (True, 2, 0, 0)),
    "ab_gemm_ep_f16_km": (2, {"AB_GEMM_NO_TPACK": "1"}, False, False, (True, 2, 0, 1)),
    "ab_gemm_ep_f16_mm": (2, {"AB_GEMM_NO_TPACK": "1"}, True, False, (True, 2, 1, 1)),
    "ab_gemm_ep_f16_mk": (2, {"AB_GEMM_NO_TPACK": "1"}, True, True, (True, 2, 1, 0)),
    "ab_gemm_ep_tf32_1p": (1, {}, False, False, (True, 1, 0, 0)),
    "ab_gemm_ep_tf32": (0, {"AB_GEMM_FUSE_FP32": "1"}, False, False, (True, 0, 0, 0)),
}
POLICY_TOL = {0: 1e-5, 1: 2e-3, 2: 2e-2}


@pytest.mark.parametrize("entry", list(ENTRY_POINTS))
def test_mlp_fused_entry_point(rt, K, monkeypatch, entry):
    """cfg3 at (B, H) = (4099, 520): 165 units, ragged M and N (N % 8 == 0), a K tail in h @ W2.
    Each of the six NVRTC entry points is launched (checked on TC_LAUNCHES); the weight gradients
    are bit-identical to node-by-node execution under the same environment and all outputs are
    within the policy tolerance of a float64 truth."""
    from collections import Counter

    from aesara_b200.runtime.device import DeviceArray

    precision, env, x_t, w1_t, key = ENTRY_POINTS[entry]
    for name, v in env.items():
        monkeypatch.setenv(name, v)
    prog, _, _ = load_case("cfg3_mlp")
    rng = np.random.default_rng(4099)
    B, H = 4099, 520
    ins = mlp_inputs(rng, B, H)

    def dev(i, a):
        t = (i == 0 and x_t) or (i == 2 and w1_t)
        return DeviceArray.from_numpy(a.T.copy()).dimshuffle([1, 0]) if t else DeviceArray.from_numpy(a)

    dins = [dev(i, a) for i, a in enumerate(ins)]
    ex = rt(prog, precision=precision)
    before = Counter(K.TC_LAUNCHES)
    fused = ex(*dins)
    assert ex.fused_regions_run == 3 and not any(f.broken for f in ex._fusions)
    keys = launched(K, before)
    assert key in keys, f"{entry}: launched {keys}"
    with monkeypatch.context() as mp:
        mp.setenv("AB_NO_GEMM_FUSE", "1")
        mp.setenv("AB_NO_RED_FUSE", "1")
        plain = rt(prog, precision=precision)(*dins)
    fused_vs_plain(fused, plain, entry, exact_sums=precision == 0)
    want = mlp_truth(ins)
    for k, (g, t) in enumerate(zip(fused, want)):
        e = float(np.max(np.abs(np.asarray(g, np.float64) - t)) / max(np.max(np.abs(t)), 1e-300))
        assert e < POLICY_TOL[precision], f"{entry} output {k}: normwise error {e:.3g}"


# ----------------------------------------------------------------------------- coverage
def test_zz_every_layout_and_entry_point_was_launched(K):
    """Every AOT MMA loop (four bf16 layouts, both TF32 precisions) and every fused entry point
    ran at least once in this session.  This reads the process-wide counter, so it relies on the
    whole module having run before it in the same process (file order, no -k selection that drops
    the cases above, no pytest-xdist); launches made by other modules of the session count too.
    When nothing ran at all (this test alone) it skips."""
    got = K.TC_LAUNCHES
    if not got:
        pytest.skip("no tensor-core GEMM ran in this session")
    print("tensor-core launches (fused, precision, a_mn, b_mn):", dict(sorted(got.items())))
    want = [(False, 2, a, b) for a in (0, 1) for b in (0, 1)] + [(False, 1, 0, 0), (False, 0, 0, 0)]
    want += [v[4] for v in ENTRY_POINTS.values()]
    missing = [k for k in want if not got[k]]
    assert not missing, f"never launched: {missing}"
