"""GPU: the BLAS-family kernels called directly through the C ABI, over the
shape / stride / alpha-beta cases of tests/tensor/test_blas.py (TestGemm :118-422,
TestGemv :1545-1752, TestGer :1861-2083) — ragged tiles, K tails, transposed and
padded operands, all three GEMM precisions.  Truth is a float64 NumPy product;
fp32-faithful mode must stay within rtol 1e-5 norm-wise (the bar vs sgemm)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    import torch

    from aesara_b200.runtime import kernels, lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return kernels


def _dev(a):
    from aesara_b200.runtime.device import DeviceArray

    return DeviceArray.from_numpy(a)


def _normwise(got, want):
    return float(np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-30))


GEMM_SHAPES = [
    (128, 256, 64), (130, 70, 96), (64, 64, 32), (257, 513, 100), (1000, 300, 36),
    (4096, 512, 1024), (300, 2000, 129), (128, 256, 33),
]


@pytest.mark.parametrize("m,n,k", GEMM_SHAPES)
@pytest.mark.parametrize("layout", ["nn", "tn", "nt", "tt", "padded"])
def test_gemm_fp32_faithful(K, m, n, k, layout):
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    c0 = rng.standard_normal((m, n)).astype("float32")
    A, B = _dev(a), _dev(b)
    if layout[0] == "t":
        A = _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    if layout[1] == "t":
        B = _dev(np.ascontiguousarray(b.T)).dimshuffle([1, 0])
    if layout == "padded":
        ap = np.zeros((m, k + 3), "float32"); ap[:, :k] = a
        bp = np.zeros((k, n + 5), "float32"); bp[:, :n] = b
        A = _dev(ap).index((slice(None), slice(0, k)))
        B = _dev(bp).index((slice(None), slice(0, n)))
    C = _dev(c0)
    K.gemm(C, 0.8, A, B, 0.4, precision=0)
    want = 0.4 * c0.astype(np.float64) + 0.8 * (a.astype(np.float64) @ b.astype(np.float64))
    err = _normwise(C.to_numpy(), want)
    assert err < 1e-5, f"3xTF32 gemm normwise error {err}"


@pytest.mark.parametrize("precision", [0, 2])
@pytest.mark.parametrize("layout", ["nn", "tn", "nt", "tt"])
@pytest.mark.parametrize("m,n,k", [(1024, 256, 192), (1500, 520, 1000), (4096, 1024, 512), (2300, 256, 4160)])
def test_gemm_four_cta_cluster_multicast(K, m, n, k, layout, precision):
    """With AB_GEMM_CLUSTER4 set, M >= 1024 takes the 4-CTA cluster kernel (four CTAs stacked along
    M sharing the B tile: each loads a quarter and multicasts it to all four).  Its per-element
    arithmetic is the single-CTA kernel's, so the result must be BIT-IDENTICAL to the default path
    for every operand layout (K-major and MN-major B quarters), ragged cluster tiles (trailing CTAs
    partly or wholly out of range) and both the 3xTF32 and bf16 policies; and inside tolerance of a
    float64 product."""
    import os

    rng = np.random.default_rng(m + n + k)
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    c0 = rng.standard_normal((m, n)).astype("float32")
    A, B = _dev(a), _dev(b)
    if layout[0] == "t":
        A = _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    if layout[1] == "t":
        B = _dev(np.ascontiguousarray(b.T)).dimshuffle([1, 0])
    os.environ["AB_GEMM_CLUSTER4"] = "1"   # the variant is off by default (slower, see cluster_pairs)
    try:
        C4 = _dev(c0)
        K.gemm(C4, 0.8, A, B, 0.4, precision=precision)
    finally:
        del os.environ["AB_GEMM_CLUSTER4"]
    C2 = _dev(c0)
    K.gemm(C2, 0.8, A, B, 0.4, precision=precision)
    got = C4.to_numpy()
    np.testing.assert_array_equal(got, C2.to_numpy())
    want = 0.4 * c0.astype(np.float64) + 0.8 * (a.astype(np.float64) @ b.astype(np.float64))
    assert _normwise(got, want) < (1e-5 if precision == 0 else 2e-2)


@pytest.mark.parametrize("layout", ["tn", "nt", "tt"])
@pytest.mark.parametrize("m,n,k", [(512, 768, 640), (1024, 256, 200), (320, 576, 4160), (300, 520, 512)])
def test_gemm_mn_major_tiles_as_one_bulk_copy(K, m, n, k, layout):
    """With AB_GEMM_MN3D set, bf16 MN-major operands (a matrix used transposed) arrive through a
    3-D tensor map, one cp.async.bulk.tensor per tile, when the MN extent is a multiple of 64;
    bit-identical to the default one-copy-per-chunk path, ragged extents keep that path."""
    import os

    rng = np.random.default_rng(m + n + k)
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    A, B = _dev(a), _dev(b)
    if layout[0] == "t":
        A = _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    if layout[1] == "n":
        pass  # B [k, n] row-major is MN-major as it stands
    else:
        B = _dev(np.ascontiguousarray(b.T)).dimshuffle([1, 0])
    os.environ["AB_GEMM_MN3D"] = "1"   # off by default (measured slower for MN-major A operands)
    try:
        C3 = _dev(np.zeros((m, n), "float32"))
        K.gemm(C3, 1.0, A, B, 0.0, precision=2)
    finally:
        del os.environ["AB_GEMM_MN3D"]
    C2 = _dev(np.zeros((m, n), "float32"))
    K.gemm(C2, 1.0, A, B, 0.0, precision=2)
    got = C3.to_numpy()
    np.testing.assert_array_equal(got, C2.to_numpy())
    want = a.astype(np.float64) @ b.astype(np.float64)
    assert _normwise(got, want) < 2e-2


@pytest.mark.parametrize("m,n,k", [(256, 256, 4096), (512, 256, 16384), (256, 512, 65536)])
@pytest.mark.parametrize("layout", ["nn", "tn"])
def test_gemm_long_k_accuracy(K, m, n, k, layout):
    """fp32-faithful mode must stay as accurate as an fp32 sgemm however long K is.
    The tensor core's FP32 accumulate truncates, so an unsegmented 3xTF32 product drifts
    linearly with K (3.4e-5 at K = 4096 before the K loop was segmented); the bar here is
    the error of NumPy's own float32 product against the float64 truth."""
    rng = np.random.default_rng(k + m)
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    A = _dev(a) if layout == "nn" else _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    C = _dev(np.zeros((m, n), "float32"))
    K.gemm(C, 1.0, A, _dev(b), 0.0, precision=0)
    want = a.astype(np.float64) @ b.astype(np.float64)
    e_dev = _normwise(C.to_numpy(), want)
    e_cpu = _normwise(a @ b, want)
    assert e_dev <= max(4.0 * e_cpu, 2e-6), f"K={k}: device {e_dev:.3g} vs fp32 CPU {e_cpu:.3g}"


@pytest.mark.parametrize("precision,tol", [(0, 3e-6), (2, 2e-2)])
@pytest.mark.parametrize("m,n,k", [(512, 768, 8192), (300, 520, 16384), (128, 256, 12288)])
def test_gemm_split_k(K, m, n, k, precision, tol):
    """Few output tiles and a long K: the K loop is split over several CTAs (pairs) and the
    partial products are summed by a second kernel (alpha, beta and a separate C_in must
    still be applied exactly once)."""
    from aesara_b200.runtime import lib as _lib
    import ctypes as C

    need = C.c_size_t()
    _lib.check(_lib.load().ab_gemm_packed_workspace_bytes(precision, m, n, k, C.byref(need)))
    assert need.value > 0, "this shape is expected to take the split-K path"
    rng = np.random.default_rng(k + n)
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    c0 = rng.standard_normal((m, n)).astype("float32")
    out = _dev(np.zeros((m, n), "float32"))
    K.gemm(out, 0.5, _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0]), _dev(b), -1.5, precision=precision,
           cin=_dev(c0))
    want = -1.5 * c0.astype(np.float64) + 0.5 * (a.astype(np.float64) @ b.astype(np.float64))
    err = _normwise(out.to_numpy(), want)
    assert err < tol, f"split-K gemm normwise error {err}"


@pytest.mark.parametrize("precision,tol", [(1, 2e-3), (2, 2e-2)])
def test_gemm_reduced_precision_policies(K, precision, tol):
    """TF32 / BF16 compute policies: stated looser tolerances (SURVEY §8d cfg3)."""
    rng = np.random.default_rng(5)
    m, n, k = 512, 384, 256
    a = rng.standard_normal((m, k)).astype("float32")
    b = rng.standard_normal((k, n)).astype("float32")
    C = _dev(np.zeros((m, n), "float32"))
    K.gemm(C, 1.0, _dev(a), _dev(b), 0.0, precision=precision)
    err = _normwise(C.to_numpy(), a.astype(np.float64) @ b.astype(np.float64))
    assert err < tol


@pytest.mark.parametrize("precision,tol", [(0, 1e-5), (1, 2e-3), (2, 2e-2)])
def test_pack_cache_shares_one_pack_between_a_matrix_and_its_transpose(K, precision, tol):
    """X (K-major A) and X^T (MN-major A) multiply from the same packed planes; an
    in-place rewrite of X invalidates them."""
    rng = np.random.default_rng(8)
    B_, H = 640, 256
    x = rng.standard_normal((B_, H)).astype("float32")
    w = rng.standard_normal((H, 192)).astype("float32")
    d = rng.standard_normal((B_, 320)).astype("float32")
    X, W, D = _dev(x), _dev(w), _dev(d)
    cache = K.PackCache()
    out1 = _dev(np.zeros((B_, 192), "float32"))
    out2 = _dev(np.zeros((H, 320), "float32"))
    K.gemm(out1, 1.0, X, W, 0.0, precision, cache=cache)
    n_after_first = len(cache._e)
    K.gemm(out2, 1.0, X.dimshuffle([1, 0]), D, 0.0, precision, cache=cache)
    # bf16: only D was packed, X's planes were reused as an MN-major operand;
    # TF32 planes are K-major only, so X^T is a second (transposing) pack
    x_packs = 1 if precision == 2 else 2
    assert len(cache._e) == n_after_first + x_packs
    assert _normwise(out1.to_numpy(), x.astype(np.float64) @ w) < tol
    assert _normwise(out2.to_numpy(), x.T.astype(np.float64) @ d) < tol
    cache.invalidate(X.owner)
    assert len(cache._e) == n_after_first  # W and D stay, every pack of X is gone


def test_gemm_beta_zero_ignores_uninitialised_c(K):
    rng = np.random.default_rng(1)
    a = rng.standard_normal((256, 128)).astype("float32")
    b = rng.standard_normal((128, 256)).astype("float32")
    C = _dev(np.full((256, 256), np.nan, "float32"))
    K.gemm(C, 1.0, _dev(a), _dev(b), 0.0)
    assert np.isfinite(C.to_numpy()).all()


def test_gemm_strided_output(K):
    rng = np.random.default_rng(2)
    a = rng.standard_normal((200, 64)).astype("float32")
    b = rng.standard_normal((64, 150)).astype("float32")
    cbuf = np.zeros((150, 200), "float32")
    Ct = _dev(cbuf).dimshuffle([1, 0])  # column-major C
    K.gemm(Ct, 1.0, _dev(a), _dev(b), 0.0)
    assert _normwise(Ct.to_numpy(), a.astype(np.float64) @ b.astype(np.float64)) < 1e-5


@pytest.mark.parametrize("m,n,k", [(50, 60, 33), (300, 200, 150)])
def test_gemm_f64(K, m, n, k):
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    c0 = rng.standard_normal((m, n))
    C = _dev(c0)
    K.gemm(C, -1.5, _dev(a), _dev(np.ascontiguousarray(b.T)).dimshuffle([1, 0]), 2.0)
    np.testing.assert_allclose(C.to_numpy(), 2.0 * c0 - 1.5 * (a @ b), rtol=1e-12, atol=1e-11)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("m,n", [(1, 1), (7, 3), (300, 129), (129, 300), (4096, 512), (33, 10000)])
@pytest.mark.parametrize("trans", [False, True])
def test_gemv(K, dtype, m, n, trans):
    rng = np.random.default_rng(m + n)
    a = rng.standard_normal((m, n)).astype(dtype)
    x = rng.standard_normal(n).astype(dtype)
    y0 = rng.standard_normal(m).astype(dtype)
    A = _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0]) if trans else _dev(a)
    for alpha, beta in [(1.0, 0.0), (0.5, 2.0)]:
        y = _dev(np.full(m, np.nan, dtype) if beta == 0.0 else y0)
        K.gemv(y, alpha, A, _dev(x), beta)
        want = alpha * (a.astype(np.float64) @ x) + (beta * y0 if beta else 0)
        tol = 1e-5 if dtype == "float32" else 1e-12
        assert _normwise(y.to_numpy(), want) < tol


def test_gemv_strided_vectors(K):
    rng = np.random.default_rng(9)
    a = rng.standard_normal((64, 48)).astype("float32")
    xb = rng.standard_normal(96).astype("float32")
    yb = np.zeros(128, "float32")
    x = _dev(xb).index((slice(None, None, 2),))
    y = _dev(yb).index((slice(None, None, 2),))
    K.gemv(y, 1.0, _dev(a), x, 0.0)
    assert _normwise(y.to_numpy(), a.astype(np.float64) @ xb[::2]) < 1e-5


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_ger(K, dtype):
    rng = np.random.default_rng(4)
    a = rng.standard_normal((130, 77)).astype(dtype)
    x = rng.standard_normal(130).astype(dtype)
    y = rng.standard_normal(77).astype(dtype)
    A = _dev(a)
    K.ger(A, 0.7, _dev(x), _dev(y))
    np.testing.assert_allclose(A.to_numpy(), a + 0.7 * np.outer(x, y), rtol=1e-5 if dtype == "float32" else 1e-12, atol=1e-6 if dtype == "float32" else 1e-14)
    At = _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    K.ger(At, 0.7, _dev(x), _dev(y))
    np.testing.assert_allclose(At.to_numpy(), a + 0.7 * np.outer(x, y), rtol=1e-5 if dtype == "float32" else 1e-12, atol=1e-6 if dtype == "float32" else 1e-14)


def test_careduce_large_patterns(K):
    """Reduction geometries at sizes where the split / two-stage paths engage."""
    rng = np.random.default_rng(11)
    x = rng.standard_normal((3000, 1030)).astype("float32")
    X = _dev(x)
    k = K.CAReduceKernel.get("add", "float32", "float64", "float32")
    for axis in [(0,), (1,), (0, 1)]:
        got = k.launch(X, axis).to_numpy()
        want = x.astype(np.float64).sum(axis=axis).astype("float32")
        np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-4)
    xt = _dev(np.ascontiguousarray(x.T)).dimshuffle([1, 0])
    np.testing.assert_allclose(k.launch(xt, (0,)).to_numpy(), x.astype(np.float64).sum(0).astype("float32"),
                               rtol=1e-6, atol=1e-4)
    km = K.CAReduceKernel.get("maximum", "float32", "float32", "float32")
    np.testing.assert_array_equal(km.launch(X, (0,)).to_numpy(), x.max(0))
    np.testing.assert_array_equal(km.launch(X, (0, 1)).to_numpy(), x.max())
