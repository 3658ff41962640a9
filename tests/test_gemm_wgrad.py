"""GPU: the grouped unit order of square tile grids with more tiles than the persistent grid has
CTAs (the weight gradients of the cfg3 MLP, 32 x 32 tiles).

An exact integer product on such a grid, whose last tile group and edge tiles are ragged, and
a weight-gradient-shaped product that must be bit-identical in the grouped order and in the
plain row order it replaces (AB_GEMM_GROUP_M=1).
"""
import numpy as np
import pytest

from tests.test_gpu_gemm_exact import assert_exact, check_bound, ints, launched, operand, truth


@pytest.fixture(scope="module")
def K():
    import torch

    from aesara_b200.runtime import kernels, lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return kernels


@pytest.mark.gpu
@pytest.mark.parametrize("la,lb", [("k", "k"), ("mn", "k"), ("mn", "mn")])
def test_exact_square_grid_grouped_order(K, monkeypatch, la, lb):
    """1832 x 1832: 15 x 15 tiles (225 units for 132 CTAs), the last tile row and column 40
    wide; the grouped order takes groups of 8 tile rows, so the last group has 7.  K = 1100
    bf16 is 18 k-blocks: a full segment, a short one and a ragged tail."""
    from collections import Counter

    from aesara_b200.runtime.device import DeviceArray

    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")  # MN-major operands stay MN-major
    m = n = 1832
    k = 1100
    check_bound(k, 4, 4)
    rng = np.random.default_rng(5)
    a, b = ints(rng, (m, k)), ints(rng, (k, n))
    C = DeviceArray.from_numpy(np.zeros((m, n), np.float32))
    before = Counter(K.TC_LAUNCHES)
    K.gemm(C, 1.0, operand(a, la, "a"), operand(b, lb, "b"), 0.0, precision=2)
    assert launched(K, before) == {(False, 2, int(la == "mn"), int(lb == "mn"))}
    assert_exact(C.to_numpy(), truth(a, b), f"{m}x{n}x{k} bf16 {la}/{lb}, grouped order")


@pytest.mark.gpu
@pytest.mark.parametrize("la", ["k", "mn"])
def test_weight_gradient_grouped_order_is_bit_identical_to_row_order(K, monkeypatch, la):
    """4096 x 4096 x 65536 bf16 (dW2 = h.T @ dout reads both operands K-major, dW1 = X.T @ dpre
    reads X MN-major) on random operands: the grouped order and the row order
    (AB_GEMM_GROUP_M=1) give the same bits, since each output element sees the same MMAs and
    folds in the same order."""
    from collections import Counter

    import torch

    from aesara_b200.runtime.device import DeviceArray

    monkeypatch.setenv("AB_GEMM_NO_TPACK", "1")
    H, B = 4096, 65536
    gen = torch.Generator(device="cuda").manual_seed(3)
    if la == "k":
        A = DeviceArray.from_torch(torch.randn(H, B, device="cuda", generator=gen))
    else:
        A = DeviceArray.from_torch(torch.randn(B, H, device="cuda", generator=gen)).dimshuffle((1, 0))
    Bm = DeviceArray.from_torch(torch.randn(H, B, device="cuda", generator=gen)).dimshuffle((1, 0))
    cache = K.PackCache()
    outs = []
    for group in (None, "1"):
        if group:
            monkeypatch.setenv("AB_GEMM_GROUP_M", group)
        C = DeviceArray.empty((H, H), "float32")
        before = Counter(K.TC_LAUNCHES)
        K.gemm(C, 1.0, A, Bm, 0.0, precision=2, cache=cache)
        assert launched(K, before) == {(False, 2, int(la == "mn"), 0)}
        outs.append(C.to_numpy())
    assert np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), \
        f"{(outs[0] != outs[1]).sum()} elements differ between the grouped and the row order"
