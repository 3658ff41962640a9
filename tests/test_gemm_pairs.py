"""GPU: the bf16 products on CTA pairs (two CTAs stacked along M that share the B tile by TMA
multicast, AB_GEMM_CLUSTER=2, the default for bf16 products of at least two tile rows).

Each output element sees the same MMAs and K-segment folds in a pair as in a single CTA, so the
pair must give the single-CTA kernel's bits (AB_GEMM_CLUSTER=1), and on small-integer operands
the exact product.  Covered: every operand layout; an odd number of tile rows (the second CTA of
the last pair wholly below M); M = 256 k + 37 (partly below M); more pairs of tiles than
resident pairs; the grouped unit order of a ragged square grid; the full-size weight gradients.
"""
import numpy as np
import pytest

from tests.test_gpu_gemm_exact import assert_exact, check_bound, ints, run_gemm, truth


@pytest.fixture(scope="module")
def K():
    import torch

    from aesara_b200.runtime import kernels, lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return kernels


def pair_and_single(K, monkeypatch, a, b, la, lb, alpha=1.0, beta=0.0, c0=None):
    outs = []
    for ctas in ("2", "1"):
        monkeypatch.setenv("AB_GEMM_CLUSTER", ctas)
        got, keys, _ = run_gemm(K, a, b, 2, la, lb, alpha, beta, c0=c0)
        assert keys == {(False, 2, int(la == "mn"), int(lb == "mn"))}, keys
        outs.append(got)
    monkeypatch.delenv("AB_GEMM_CLUSTER")
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("la,lb", [("k", "k"), ("k", "mn"), ("mn", "k"), ("mn", "mn")])
@pytest.mark.parametrize("m,n,k", [
    (128 * 7, 520, 1100),            # 7 tile rows: the last pair's second CTA is wholly below M
    (256 * 3 + 128 + 37, 640, 520),  # the last pair's second CTA has 37 rows inside M
    (256 * 5 + 37, 1153, 1000),  # its first CTA 37, its second none; ragged N and K
    (8192 + 128, 4096, 200),         # 33 pair rows x 32 columns = 1056 pair tiles for 66 resident pairs
])
def test_pair_matches_single_cta_exactly(K, monkeypatch, la, lb, m, n, k):
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")  # MN-major operands stay MN-major
    check_bound(k, 4, 4)
    rng = np.random.default_rng(m + 3 * n + 7 * k)
    a, b = ints(rng, (m, k)), ints(rng, (k, n))
    c = ints(rng, (m, n), 64)
    pair, single = pair_and_single(K, monkeypatch, a, b, la, lb, 0.5, -2.0, c)
    assert_exact(pair, truth(a, b, 0.5, -2.0, c), f"pairs {m}x{n}x{k} {la}/{lb}")
    assert np.array_equal(pair.view(np.uint32), single.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("group", [None, "3"])
def test_pair_grouped_order_on_a_ragged_square_grid(K, monkeypatch, group):
    """1832 x 1832: 15 x 15 tiles = 8 pair rows (the last one half below M) x 15 columns; the
    default groups of 4 pair rows, and groups of 3 (a last group of 2)."""
    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    if group:
        monkeypatch.setenv("AB_GEMM_GROUP_M", group)
    m = n = 1832
    k = 1100
    check_bound(k, 4, 4)
    rng = np.random.default_rng(11)
    a, b = ints(rng, (m, k)), ints(rng, (k, n))
    pair, single = pair_and_single(K, monkeypatch, a, b, "mn", "k")
    assert_exact(pair, truth(a, b), f"pairs {m}x{n}x{k}, groups of {group or 4}")
    assert np.array_equal(pair.view(np.uint32), single.view(np.uint32))


@pytest.mark.gpu
def test_pairs_are_the_default_for_bf16_products(K, monkeypatch):
    """Without the knob a bf16 product of two or more tile rows runs on pairs: same bits as
    forced pairs, and the same as forced single CTAs."""
    monkeypatch.delenv("AB_GEMM_CLUSTER", raising=False)
    rng = np.random.default_rng(2)
    a, b = ints(rng, (1000, 600)), ints(rng, (600, 768))
    default, _, _ = run_gemm(K, a, b, 2)
    pair, single = pair_and_single(K, monkeypatch, a, b, "k", "k")
    assert np.array_equal(default.view(np.uint32), pair.view(np.uint32))
    assert np.array_equal(default.view(np.uint32), single.view(np.uint32))
    assert_exact(default, truth(a, b), "default 1000x768x600")


@pytest.mark.gpu
@pytest.mark.parametrize("la", ["k", "mn"])
def test_full_size_weight_gradient_pair_is_bit_identical_to_single(K, monkeypatch, la):
    """4096 x 4096 x 65536 bf16 on random operands, A K-major (dW2 = h.T @ dout) or MN-major
    (dW1 = X.T @ dpre), B K-major."""
    import torch

    from aesara_b200.runtime.device import DeviceArray

    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    H, B = 4096, 65536
    gen = torch.Generator(device="cuda").manual_seed(4)
    if la == "k":
        A = DeviceArray.from_torch(torch.randn(H, B, device="cuda", generator=gen))
    else:
        A = DeviceArray.from_torch(torch.randn(B, H, device="cuda", generator=gen)).dimshuffle((1, 0))
    Bm = DeviceArray.from_torch(torch.randn(H, B, device="cuda", generator=gen)).dimshuffle((1, 0))
    cache = K.PackCache()
    outs = []
    for ctas in ("2", "1"):
        monkeypatch.setenv("AB_GEMM_CLUSTER", ctas)
        C = DeviceArray.empty((H, H), "float32")
        K.gemm(C, 1.0, A, Bm, 0.0, precision=2, cache=cache)
        outs.append(C.to_numpy())
    assert np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), \
        f"{(outs[0] != outs[1]).sum()} elements differ between pairs and single CTAs"


def test_resident_pairs_query_checks_its_arguments():
    import ctypes

    from aesara_b200.runtime import lib

    n = ctypes.c_int(0)
    assert lib.load().ab_gemm_max_clusters(2, 0, ctypes.byref(n)) != 0
    assert lib.load().ab_gemm_max_clusters(2, 2, None) != 0
