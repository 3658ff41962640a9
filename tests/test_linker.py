"""CPU (needs the reference front-end): the drop-in boundary.

`aesara.function(..., mode=B200)` must go through B200Linker.accept/make_all and
give Function-level semantics identical to the reference VM (storage cells,
shared-variable updates, output order).  No GPU here, so the *device executor*
is replaced by the oracle interpreter for these tests only — what is under test
is the linker/VM glue and the lowering, not the kernels (tests/test_gpu_parity.py
covers those on the GPU)."""
import numpy as np
import pytest

from aesara_b200.compat import bootstrap

pytestmark = pytest.mark.skipif(not bootstrap.available(), reason="reference front-end not available")


@pytest.fixture()
def aes():
    aesara = bootstrap.load_aesara()
    import aesara_b200.linker as L

    return aesara, L


class _FakeDeviceArray:
    """Host-backed stand-in for runtime.device.DeviceArray (no GPU in this container):
    what the VM / shared-variable logic needs to know is only "this value is on the device"."""

    uploads = 0
    downloads = 0

    def __init__(self, a):
        self._a = np.array(a, copy=True)
        self.ptr = id(self._a)
        self.dtype, self.shape = self._a.dtype, self._a.shape

    def to_numpy(self):
        type(self).downloads += 1
        return self._a.copy()

    def copy(self):
        return _FakeDeviceArray(self._a)

    def __array__(self, dtype=None, copy=None):
        return self.to_numpy() if dtype is None else self.to_numpy().astype(dtype)


class _OracleExecutor:
    """Stand-in with the ProgramExecutor call signature (tests only)."""

    device_results = False  # return _FakeDeviceArray outputs (as the real executor does)

    def __init__(self, program, **kw):
        self.program = program
        self.trace = None
        self.time_nodes = False

    def __call__(self, *inputs, output_subset=None):
        from oracle.program_np import run_program

        host = []
        for i in inputs:
            if isinstance(i, _FakeDeviceArray):
                host.append(i._a.copy())
            else:
                if isinstance(i, np.ndarray) and i.size > 64:
                    _FakeDeviceArray.uploads += 1
                host.append(np.array(i) if isinstance(i, np.ndarray) else i)
        outs = run_program(self.program, host, trace=self.trace)
        if output_subset is not None:
            keep = set(output_subset) | {o for o, _ in self.program.updates}
            outs = [o if k in keep else None for k, o in enumerate(outs)]
        if self.device_results:
            outs = [_FakeDeviceArray(o) if isinstance(o, np.ndarray) and o.ndim > 0 else o for o in outs]
        return outs

    def node_times_ms(self):
        return [(i, n.op, 0.25) for i, n in enumerate(self.program.nodes)]


def test_mode_and_linker_are_registered(aes):
    aesara, L = aes
    from aesara.compile.mode import get_mode, predefined_linkers

    assert "b200" in predefined_linkers
    m = get_mode("B200")
    assert isinstance(m.linker, L.B200Linker)
    from aesara.compile.mode import get_target_language

    assert get_target_language(m) == ("c", "py")  # the graphs the C-linker gets
    # the rewrite that consults it holds its own reference to the function (ADVICE r1)
    import aesara.tensor.rewriting.elemwise as E

    assert E.get_target_language(m) == ("c", "py")


def _same_program(a, b, path="program"):
    assert [n.op for n in a.nodes] == [n.op for n in b.nodes], path
    for k, (x, y) in enumerate(zip(a.nodes, b.nodes)):
        assert x.params.get("expr", {}).get("name") == y.params.get("expr", {}).get("name"), f"{path} node {k}"
        if x.op == "Scan":
            assert x.params["info"] == y.params["info"]
            _same_program(x.params["inner"], y.params["inner"], f"{path} node {k} inner")


@pytest.mark.parametrize("cfg", ["cfg1_readme", "cfg2_fused", "cfg3_mlp", "cfg5_logreg", "cfg4_lstm"])
def test_linker_path_lowers_to_the_committed_fixture(aes, cfg):
    """What ``aesara.function(..., mode="B200")`` links — outer graph AND the inner graph of
    a Scan — is the program committed under tests/golden (which the GPU tests replay), and it
    does not depend on another linker having compiled the Scan first (ADVICE r1: the inner
    graph is rewritten by lower.optimized_inner_fgraph, never by a side effect of op.fn)."""
    aesara, L = aes
    from aesara_b200 import graphs as G
    from tests._cases import load_case

    build = {"cfg1_readme": G.cfg1_readme, "cfg2_fused": G.cfg2_fused_elemwise, "cfg3_mlp": G.cfg3_mlp,
             "cfg5_logreg": G.cfg5_logreg, "cfg4_lstm": G.cfg4_lstm_scan}[cfg]
    i, o = build()
    f = aesara.function(i, o, mode=L.mode(), on_unused_input="ignore")
    prog = f.maker.linker.program
    want, _, _ = load_case(cfg)
    _same_program(prog, want)
    if cfg == "cfg4_lstm":
        inner = [n for n in prog.nodes if n.op == "Scan"][0].params["inner"]
        assert [n.op for n in inner.nodes].count("Gemm") == 1      # Dot -> Gemm happened
        assert sum(n.op == "Elemwise" and len(n.params["expr"]["stmts"]) >= 3 for n in inner.nodes) == 2
        # and the C-linker compiling the same graph afterwards changes nothing
        prog_c, _ = G.optimized_program(*build(), name=cfg)
        _same_program(prog_c, want)


def test_function_semantics_through_the_linker(aes, monkeypatch):
    aesara, L = aes
    import aesara.tensor as at
    import aesara_b200.runtime.vm as vm

    monkeypatch.setattr(vm, "ProgramExecutor", _OracleExecutor)
    x = at.fvector("x")
    acc = aesara.shared(np.zeros(5, "float32"), name="acc")
    out = at.tanh(x) * 2 + acc
    f = aesara.function([x], [out, out.sum()], updates=[(acc, acc + x)], mode=L.mode())
    assert isinstance(f.vm, L.B200VM)
    g = aesara.function([x], [out, out.sum()], updates=[], mode="FAST_RUN")
    xv = np.arange(5, dtype="float32")
    r1 = f(xv)
    np.testing.assert_allclose(r1[0], np.tanh(xv) * 2, rtol=1e-6)
    np.testing.assert_allclose(acc.get_value(), xv)          # update applied by the VM
    r2 = f(xv)
    np.testing.assert_allclose(r2[0], np.tanh(xv) * 2 + xv, rtol=1e-6)
    np.testing.assert_allclose(acc.get_value(), 2 * xv)
    assert len(r2) == 2 and r2[1].shape == ()
    acc.set_value(np.zeros(5, "float32"))
    np.testing.assert_allclose(g(xv)[0], r1[0], rtol=1e-6)


def test_unsupported_op_is_a_hard_error(aes):
    """No CPU fallback for tensor work: an Op without a device implementation
    fails at link time, naming the Op."""
    aesara, L = aes
    import aesara.tensor as at

    x = at.fmatrix("x")
    with pytest.raises(NotImplementedError, match="no device implementation"):
        aesara.function([x], at.linalg.det(x), mode=L.mode())


def test_linker_copies_bind_to_one_graph(aes):
    aesara, L = aes
    import aesara.tensor as at
    from aesara.graph.fg import FunctionGraph

    x = at.fvector("x")
    fg1 = FunctionGraph([x], [x * 2], clone=True)
    fg2 = FunctionGraph([x], [x + 1], clone=True)
    lk = L.B200Linker()
    a = lk.accept(fg1)
    b = a.accept(fg2)
    assert a is lk and b is not lk and b.fgraph is fg2
    assert lk.clone(allow_gc=False).allow_gc is False


def test_device_resident_shared_variable_updates(aes, monkeypatch):
    """SURVEY 8f N4: weights in `aesara_b200.shared` stay on the device across calls —
    the update result is written into the cell without a download and the next call does
    not upload it; `get_value` still hands NumPy to the caller."""
    aesara, L = aes
    import aesara.tensor as at
    import aesara_b200.runtime.vm as vm
    from aesara_b200.sharedvar import B200SharedVariable, shared

    monkeypatch.setattr(vm, "ProgramExecutor", _OracleExecutor)
    monkeypatch.setattr(_OracleExecutor, "device_results", True)
    _FakeDeviceArray.uploads = _FakeDeviceArray.downloads = 0
    x = at.fvector("x")
    W = shared(np.full(100, 0.5, "float32"), name="W")
    assert isinstance(W, B200SharedVariable) and not W.is_on_device()
    loss = ((W * x) ** 2).sum()
    f = aesara.function([x], loss, updates=[(W, W - 0.1 * aesara.grad(loss, W))], mode=L.mode())
    xv = np.linspace(-1, 1, 100).astype("float32")
    ref_W = np.full(100, 0.5, "float32")
    for step in range(3):
        l = f(xv)
        want = float(((ref_W * xv) ** 2).sum())
        np.testing.assert_allclose(l, want, rtol=1e-5)
        ref_W = ref_W - 0.1 * (2 * ref_W * xv * xv)
        assert W.is_on_device()
    # one upload of W (first call) + x each call; W's update was never downloaded
    assert _FakeDeviceArray.uploads == 1 + 3
    assert _FakeDeviceArray.downloads == 0
    np.testing.assert_allclose(W.get_value(), ref_W, rtol=1e-5)
    assert _FakeDeviceArray.downloads == 1
    internal = W.get_value(borrow=True, return_internal_type=True)
    assert isinstance(internal, _FakeDeviceArray)
    W.set_value(np.zeros(100, "float32"))
    assert not W.is_on_device()
    np.testing.assert_allclose(f(xv), 0.0)
    W.set_value(_FakeDeviceArray(np.ones(100, "float32")))
    np.testing.assert_allclose(f(xv), float((xv ** 2).sum()), rtol=1e-5)
    with pytest.raises(TypeError):
        W.set_value(_FakeDeviceArray(np.ones((2, 2), "float32")))
    # an ordinary aesara.shared keeps host semantics (its update IS downloaded)
    acc = aesara.shared(np.zeros(100, "float32"), name="acc")
    g = aesara.function([x], [], updates=[(acc, acc + x)], mode=L.mode())
    g(xv)
    assert isinstance(acc.container.storage[0], np.ndarray)
    np.testing.assert_allclose(acc.get_value(), xv)


def test_profile_receives_per_node_times(aes, monkeypatch):
    """`aesara.function(..., profile=True)`: the VM feeds ProfileStats per-Apply times and
    call counts (link/vm.py:251-281) — on the device these come from CUDA events."""
    aesara, L = aes
    import aesara.tensor as at
    import aesara_b200.runtime.vm as vm

    monkeypatch.setattr(vm, "ProgramExecutor", _OracleExecutor)
    x = at.fvector("x")
    f = aesara.function([x], at.tanh(x).sum(), mode=L.mode(), profile=True)
    for _ in range(3):
        f(np.ones(7, "float32"))
    prof = f.profile
    assert prof.fct_callcount == 3
    assert len(prof.apply_time) == len(f.maker.fgraph.apply_nodes)
    assert all(abs(t - 3 * 0.25e-3) < 1e-9 for t in prof.apply_time.values())
    assert all(c == 3 for c in prof.apply_callcount.values())


def test_dual_run_checker(aes, monkeypatch):
    """DualLinker-style harness: every node of the B200 run is compared with the reference
    thunk of the same Apply; a corrupted node is located."""
    aesara, L = aes
    import aesara.tensor as at
    import aesara_b200.runtime.vm as vm
    from aesara_b200.debug import DualRunMismatch, check_function

    monkeypatch.setattr(vm, "ProgramExecutor", _OracleExecutor)
    X, w = at.fmatrix("X"), at.fvector("w")
    out = [at.tanh(X @ w).sum(), at.exp(X).max(axis=0)]
    vals = [np.random.default_rng(0).standard_normal((9, 5)).astype("float32"),
            np.random.default_rng(1).standard_normal(5).astype("float32")]
    report = check_function([X, w], out, vals)
    assert len(report) >= 3 and all(isinstance(r[2], float) for r in report)
    report_c = check_function([X, w], out, vals, reference_linker="c")
    assert len(report_c) == len(report)

    import oracle.program_np as O

    orig = O._H["CAReduce"]
    monkeypatch.setitem(O._H, "CAReduce", lambda node, args, prog: orig(node, args, prog) * 1.001)
    with pytest.raises(DualRunMismatch) as ei:
        check_function([X, w], out, vals)
    assert "CAReduce" in str(ei.value.node.op.__class__.__mro__) or "Sum" in str(ei.value.node) or "Max" in str(ei.value.node)


def test_output_subset_no_recycling_and_error_cells(aes, monkeypatch):
    """VM semantics ``Function.__call__`` relies on (compile/function/types.py:830, 969-1048):
    ``output_subset`` computes only what was asked for plus the updates (vm.py:536-563),
    ``no_recycling`` cells are emptied before each call (vm.py:1017), and on failure the
    failing node's input cells hold the values ``raise_with_op`` prints (link/utils.py:340)."""
    aesara, L = aes
    import aesara.tensor as at
    import aesara_b200.runtime.vm as vm
    from aesara_b200.runtime.vm import NodeError, ProgramExecutor

    x = at.fvector("x")
    cnt = aesara.shared(np.zeros((), "float32"), name="cnt")
    outs = [at.tanh(x), at.exp(x).sum(), x * 3]
    # needed-node analysis on the real executor (construction needs no GPU)
    f_real = aesara.function([x], outs, updates=[(cnt, cnt + x.sum())], mode=L.mode())
    ex = f_real.vm.executor
    assert isinstance(ex, ProgramExecutor)
    needed, computed = ex.needed_nodes([1])
    ops = [n.op for n, k in zip(ex.program.nodes, needed) if k]
    assert computed == (1, 3) and 0 < sum(needed) < len(needed)
    assert "CAReduce" in ops
    all_needed, _ = ex.needed_nodes([0, 1, 2])
    assert all(all_needed)

    monkeypatch.setattr(vm, "ProgramExecutor", _OracleExecutor)
    monkeypatch.setattr(_OracleExecutor, "device_results", False)
    f = aesara.function([x], outs, updates=[(cnt, cnt + x.sum())], mode=L.mode())
    xv = np.arange(4, dtype="float32")
    r = f(xv, output_subset=[2])
    assert len(r) == 1
    np.testing.assert_allclose(r[0], 3 * xv)
    np.testing.assert_allclose(cnt.get_value(), xv.sum())      # the update still ran
    full = f(xv)
    assert len(full) == 3
    np.testing.assert_allclose(cnt.get_value(), 2 * xv.sum())

    # no_recycling: FunctionMaker passes the outputs (types.py:1604-1611)
    assert f.vm.pre_call_clear, "no_recycling cells were not registered"
    for cell in f.vm.pre_call_clear:
        cell[0] = "stale"
    f(xv)
    # error: the failing node's input cells are populated for raise_with_op
    class Boom(_OracleExecutor):
        def __call__(self, *a, **k):
            raise NodeError(0, self.program.nodes[0], ValueError("boom"), ["VALUE"] * len(self.program.nodes[0].inputs))

    monkeypatch.setattr(vm, "ProgramExecutor", Boom)
    g = aesara.function([x], at.tanh(x), mode=L.mode())
    with pytest.raises(ValueError, match="boom") as ei:
        g(xv)
    assert "Apply node that caused the error" in str(ei.value)
    assert "Inputs shapes" in str(ei.value)
    assert g.vm.position_of_error == 0


def test_shared_constructor_registration(aes):
    """``aesara.shared`` itself yields device-resident parameters (SURVEY 8f N4 wording):
    always for device values, for NumPy values after the opt-in."""
    aesara, L = aes
    from aesara_b200.sharedvar import B200SharedVariable, register_shared_constructor

    class Dev(_FakeDeviceArray):
        pass

    from aesara.compile.sharedvalue import shared_constructor
    from aesara_b200.runtime.device import DeviceArray

    assert shared_constructor.dispatch(DeviceArray).__name__ == "_device_array_constructor"
    v = aesara.shared(np.zeros(3, "float32"))
    assert not isinstance(v, B200SharedVariable)
    register_shared_constructor(ndarrays=True)
    try:
        w = aesara.shared(np.ones((2, 3), "float32"), name="w")
        assert isinstance(w, B200SharedVariable) and w.type.dtype == "float32" and w.type.ndim == 2
        np.testing.assert_array_equal(w.get_value(), np.ones((2, 3), "float32"))
    finally:
        register_shared_constructor(ndarrays=False)
    assert not isinstance(aesara.shared(np.zeros(3, "float32")), B200SharedVariable)


def test_in_place_scatter_is_a_destroyer(aes):
    """ADVICE r1: AdvancedIncSubtensor1{inplace} rewrites its input buffer; the executor must
    know, or cached GEMM operand planes of that buffer go stale."""
    aesara, L = aes
    import aesara.tensor as at

    W = at.fmatrix("W")
    idx = at.lvector("idx")
    y = at.fmatrix("y")
    x = at.fmatrix("x")
    W2 = at.inc_subtensor((W * 1.0)[idx], y)
    out = x @ W2
    f = aesara.function([W, idx, y, x], out, mode=L.mode())
    ex = f.vm.executor
    scat = [i for i, n in enumerate(ex.program.nodes) if n.op == "AdvancedIncSubtensor1"]
    assert scat
    for i in scat:
        if ex.program.nodes[i].params["inplace"]:
            assert ex._destroys[i] == [0]
