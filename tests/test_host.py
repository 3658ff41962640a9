"""CPU: host-side logic — the C-ABI library loads and exports every symbol the
header declares, the JIT compiles without a GPU, fixtures load, host evaluator
agrees with the oracle."""
import os
import re

import numpy as np
import pytest

from tests._cases import case_names, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "aesara_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ab_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from aesara_b200.runtime import lib

    L = lib.load()
    syms = header_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(L, s), f"libaesara_b200.so does not export {s}"
        assert s in lib.SIGNATURES, f"{s} has no ctypes signature"
    assert L.ab_version().decode().startswith("aesara_b200")


def test_no_device_is_a_loud_error():
    import torch

    from aesara_b200.runtime import lib

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    rc = lib.load().ab_init(0)
    assert rc != 0
    assert b"no CUDA device" in lib.load().ab_last_error()


@pytest.mark.parametrize("name", ["cfg2_fused", "cfg3_mlp", "cfg5_logreg", "ew_int_arith"])
def test_kernels_compile_for_sm90a_without_gpu(name):
    from aesara_b200.runtime.vm import ProgramExecutor

    prog, _, _ = load_case(name)
    ex = ProgramExecutor(prog)
    assert ex.compile_all() >= 1


def test_generated_source_shape():
    from aesara_b200.codegen.elemwise import elemwise_source

    prog, _, _ = load_case("cfg2_fused")
    expr = prog.nodes[0].params["expr"]
    src, meta = elemwise_source(expr)
    assert meta["vec"] == 4 and meta["n_in"] == 3 and meta["n_out"] == 1
    assert "ab_softplus" in src and "tanhf" in src and "ab_ew_flat_vec" in src


def test_every_fixture_is_executable_by_the_runtime():
    """Every node kind appearing in the fixtures has a device implementation."""
    from aesara_b200.runtime import vm

    for name in case_names():
        prog, _, _ = load_case(name)
        missing = {n.op for n in prog.nodes if n.op not in vm._EXEC}
        assert not missing, f"{name}: {missing}"


def test_host_eval_matches_oracle_on_shape_arithmetic():
    from aesara_b200.runtime import host_eval
    from oracle.scalar_np import eval_expr

    prog, _, _ = load_case("cfg4_lstm")
    rng = np.random.default_rng(0)
    n = 0
    for node in prog.nodes:
        if node.op in ("Elemwise", "ScalarOp"):
            expr = node.params["expr"]
            if not host_eval.supports(expr) or any(d.startswith("float") for d in expr["inputs"]):
                continue
            args = [np.asarray(rng.integers(-5, 9), dtype=d) for d in expr["inputs"]]
            a = host_eval.eval_expr(expr, args)
            b = eval_expr(expr, args)
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
            n += 1
    assert n >= 5


def test_host_eval_matches_oracle_on_float_expressions():
    """Every scalar expression of every fixture that the host evaluator accepts gives the
    oracle's value on float (and mixed) operands too: host_eval is a third implementation of
    the scalar ops (after the generated CUDA bodies and the oracle) and is pinned here."""
    from aesara_b200.runtime import host_eval
    from oracle.scalar_np import eval_expr

    rng = np.random.default_rng(5)
    special = np.array([0.0, -0.0, 1.5, -2.5, 3.0, -3.0, 0.5, 7.25, -7.25, 2.0])
    n_expr = n_float = 0
    for name in case_names():
        prog, _, _ = load_case(name)
        progs = [prog] + [n.params["inner"] for n in prog.nodes if n.op == "Scan"]
        for pg in progs:
            for node in pg.nodes:
                if node.op not in ("Elemwise", "ScalarOp"):
                    continue
                expr = node.params["expr"]
                if not host_eval.supports(expr):
                    continue
                n_expr += 1
                is_float = any(d.startswith("float") for d in expr["inputs"])
                n_float += is_float
                for trial in range(4):
                    args = []
                    for d in expr["inputs"]:
                        dt = np.dtype(d)
                        if dt.kind == "f":
                            v = rng.choice(special) if trial % 2 else rng.standard_normal() * 3
                        elif dt.kind == "b":
                            v = rng.random() < 0.5
                        else:
                            v = rng.integers(0 if dt.kind == "u" else -5, 9)
                        args.append(np.asarray(v).astype(dt))
                    a = host_eval.eval_expr(expr, args)
                    b = eval_expr(expr, args)
                    for x, y in zip(a, b):
                        assert np.asarray(x).dtype == np.asarray(y).dtype, (name, expr.get("name"))
                        np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=f"{name}: {expr.get('name')}")
    assert n_expr >= 100 and n_float >= 30


def _scan_runner(name):
    from aesara_b200.runtime.vm import ProgramExecutor

    prog, _, _ = load_case(name)
    ex = ProgramExecutor(prog)
    idx = [i for i, n in enumerate(prog.nodes) if n.op == "Scan"][0]
    return ex._state[idx]["runner"]


def test_cell_matcher_accepts_the_cfg4_inner_graph_as_the_lstm_member():
    """The matcher traces the inner program with address-only stand-ins (no GPU needed)."""
    r = _scan_runner("cfg4_lstm")
    assert r.cell is not None
    for B, H in ((256, 128), (8192, 1024)):
        spec = r.cell.match(B, H, 4)
        assert spec is not None and spec.is_lstm and (spec.gates, spec.states, spec.hs) == (4, 2, 0)
    assert r.cell.match(256, 128, 3) is None      # U would not be [H, 4H]


def test_cell_matcher_family_and_rejections():
    import copy

    # no loop-invariant product: not the family
    assert _scan_runner("scan_cumsum_allsteps").cell is None
    assert _scan_runner("scan_two_taps_nitsot").cell is None
    # the same structure with another cell (tanh on the output gate replaced by sigmoid) is still
    # a member of the family, but no longer the ahead-of-time LSTM: it gets a generated cell
    r = _scan_runner("cfg4_lstm")
    inner = r.inner.program
    for n in inner.nodes:
        if n.op == "Elemwise" and "tanh" in [s["op"] for s in n.params["expr"]["stmts"]]:
            n.params = copy.deepcopy(n.params)
            for s in n.params["expr"]["stmts"]:
                if s["op"] == "tanh":
                    s["op"] = "sigmoid"
    spec = r.cell.match(256, 128, 4)
    assert spec is not None and not spec.is_lstm
    assert "ab_cell_body" in spec.source() and "AB_CELL_GATES 4" in spec.source()
    # tanh-RNN (1 gate, 1 state) and a gated unit (3 gates, 1 state), from the reference
    for name, gates, states in (("scan_rnn_tanh_cell", 1, 1), ("scan_gated_unit_cell", 3, 1)):
        r = _scan_runner(name)
        assert r.cell is not None, name
        spec = r.cell.match(256, 64, gates)
        assert spec is not None and not spec.is_lstm and (spec.gates, spec.states, spec.hs) == (gates, states, 0)


def test_generated_scan_cells_compile_for_sm90a():
    """NVRTC (no GPU): the persistent Scan kernel with cells generated from inner graphs."""
    for name, gates in (("scan_rnn_tanh_cell", 1), ("scan_gated_unit_cell", 3), ("cfg4_lstm", 4)):
        spec = _scan_runner(name).cell.match(256, 64, gates)
        assert spec is not None
        spec.compile()


_SCAN_CELL_GRAPHS = [(name, "all") for name in ("G1S1hs0", "G3S1hs0", "G2S3hs1", "G4S2hs1_ch", "rnn_tanh",
                                                 "gated", "lstm_hc", "lstm_ch")] + [
    (name, v) for name in ("G1S1hs0", "G2S3hs1") for v in ("last", "backwards", "wt", "nsteps2")]


@pytest.mark.parametrize("name,variant", _SCAN_CELL_GRAPHS, ids=[f"{n}-{v}" for n, v in _SCAN_CELL_GRAPHS])
def test_scan_cell_graphs_of_the_device_suite_match_and_compile(name, variant):
    """The Scan graphs of tests/test_gpu_scan_cell.py, built with the reference front end: the
    matcher finds the expected (gates, states, recurrent state, LSTM) at every shape the suite
    runs, and the generated cell compiles for sm_90a (NVRTC, no GPU)."""
    from aesara_b200.compat import bootstrap

    if not bootstrap.available():
        pytest.skip("reference front-end (oracle/_ref) not present")
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests import _scan_cells as SC

    c = SC.CELLS[name]
    ex = ProgramExecutor(SC.program(name, variant))
    r = [st["runner"] for st in ex._state if "runner" in st][0]
    assert r.cell is not None
    for B, H in ((128, 64), (200, 128), (2048, 320), (8, 1088)):
        spec = r.cell.match(B, H, c.G)
        assert spec is not None, (B, H)
        assert (spec.gates, spec.states, spec.hs, spec.is_lstm) == (c.G, c.S, c.hs, c.is_lstm)
    spec.compile()


# ---------------------------------------------------------------- executor-level regions
def test_fusion_regions_detected_on_the_committed_programs():
    """Region detection is host logic over the lowered program: cfg5 has one row region
    (Gemv -> 3 Elemwise -> 2 Sum + Gemv(X.T)), cfg3 three Gemm->Elemwise pairs and one
    Sqr->Sum; graphs whose GEMM result has several consumers are left alone."""
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests._cases import load_case

    prog, _, _ = load_case("cfg5_logreg")
    ex = ProgramExecutor(prog)
    (f,) = ex._fusions
    assert type(f).__name__ == "RowFusion"
    ops = [prog.nodes[i].op for i in f.members]
    assert ops.count("Gemv") == 2 and ops.count("CAReduce") == 2 and ops.count("Elemwise") == 3
    assert f.last == max(f.members) and f.alpha1 == 1.0 and f.alpha2 == 1.0
    assert all(not ex._free_after[i] for i in f.members if i != f.last)  # operands stay alive

    prog, _, _ = load_case("cfg3_mlp")
    # fp32-faithful default: no GEMM-epilogue regions (the hi/lo kernels have no registers for
    # them: slower than node by node), the loss's Sqr -> Sum still runs as one reduction
    assert sorted(type(f).__name__ for f in ProgramExecutor(prog)._fusions) == ["ReducePreFusion"]
    ex = ProgramExecutor(prog, precision=2)
    kinds = sorted(type(f).__name__ for f in ex._fusions)
    assert kinds == ["GemmEpilogueFusion"] * 3  # Sqr -> Sum now lives inside the second region
    regions = sorted((f for f in ex._fusions), key=lambda f: f.g)
    ops = [[prog.nodes[i].op for i in f.members] for f in regions]
    assert ops[0] == ["Dot22", "Elemwise"]                                   # tanh(X@W1 + b1)
    assert sorted(ops[1]) == ["CAReduce", "CAReduce", "Elemwise", "Elemwise", "Elemwise", "Gemm"]
    assert sorted(ops[2]) == ["CAReduce", "Dot22", "Elemwise"]               # dpre and its column sums
    r2, r3 = regions[1], regions[2]
    # diff is never stored; dout (stored and/or bf16 plane) carries the column sums, Sqr(diff) the total
    assert len(r2.out_vars) == 2 and r2.out_vars[1] is None and r2.colsum == 0 and r2.fullsum == 1
    assert r3.colsum == 0 and r3.fullsum == -1
    # the second region waits for the 1/n factor computed after the Gemm node and runs before
    # the first product that reads dout
    assert r2.g < r2.anchor < min(c for v in r2.out_vars if v is not None for c in r2._consumers[v])
    assert regions[0].anchor == regions[0].g  # nothing to wait for: runs at the GEMM position
    for f in regions:
        assert f.anchor in f.members and f.last == max(f.members)
    shadows = [f.shadow_consumer for f in regions]
    assert shadows == [True, True, True]  # h, dout and dpre feed later products

    import os
    os.environ["AB_GEMM_FUSE_SINGLE"] = "1"
    try:
        ex1 = ProgramExecutor(prog, precision=2)
    finally:
        del os.environ["AB_GEMM_FUSE_SINGLE"]
    kinds = sorted(type(f).__name__ for f in ex1._fusions)
    assert kinds == ["GemmEpilogueFusion"] * 3 + ["ReducePreFusion"]         # round-1 regions
    assert all(len(f.members) == 2 for f in ex1._fusions)

    for name in ("softmax_classifier", "blas_dot22_layouts", "cfg4_lstm", "cfg1_readme"):
        prog, _, _ = load_case(name)
        assert not [f for f in ProgramExecutor(prog)._fusions if type(f).__name__ == "RowFusion"]


def _fused_region_names(kind):
    from tests import _fused_regions as FR

    return list(FR.GEMM if kind == "gemm" else FR.ROW)


@pytest.mark.parametrize("name", _fused_region_names("gemm"))
def test_fused_region_catalogue_detects_and_compiles(name, monkeypatch):
    """The GEMM-epilogue graphs of tests/test_gpu_fused_regions.py, built with the reference front
    end: each is one region with the member ops and ``#define``s the catalogue names under every
    precision policy (a region with more than it takes keeps its largest legal prefix), and the
    generated module compiles for sm_90a (NVRTC, no GPU)."""
    from aesara_b200.compat import bootstrap

    if not bootstrap.available():
        pytest.skip("reference front-end (oracle/_ref) not present")
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests import _fused_regions as FR

    monkeypatch.setenv("AB_GEMM_FUSE_FP32", "1")
    case = FR.GEMM[name]
    prog = FR.gemm_program(name)
    for precision in (0, 1, 2):
        fs = [f for f in ProgramExecutor(prog, precision=precision)._fusions
              if type(f).__name__ == "GemmEpilogueFusion"]
        assert len(fs) == 1, f"{name} precision {precision}: {len(fs)} regions"
        f = fs[0]
        d = FR.defines(f.source())
        assert d["AB_EP_EXACT_SUMS"] == (precision == 0)
        if case.expect["defines"] is not None:
            want = dict(case.expect["defines"], **({} if precision == 2 else {"AB_EP_TPLANE": -1}))
            assert {k: d[k] for k in want} == want, f"precision {precision}"
            assert [prog.nodes[m].op for m in f.members] == case.expect["ops"]
        later = [i for i, n in enumerate(prog.nodes) if i > f.g and n.op in ("Elemwise", "CAReduce")]
        assert len(later) - (len(f.members) - 1) == case.expect["left_out"]
        assert f.compile_all() == 1


@pytest.mark.parametrize("name", _fused_region_names("row"))
def test_row_region_catalogue_detects_and_compiles(name):
    """The row-region graphs of the same suite: one region each (two Gemv, the per-row Elemwise
    and the Sums), and its module compiles for sm_90a at every register blocking J = 1..8."""
    from aesara_b200.compat import bootstrap

    if not bootstrap.available():
        pytest.skip("reference front-end (oracle/_ref) not present")
    from aesara_b200.runtime import lib
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests import _fused_regions as FR

    prog = FR.row_program(name)
    (f,) = [f for f in ProgramExecutor(prog)._fusions if type(f).__name__ == "RowFusion"]
    ops = [prog.nodes[i].op for i in f.members]
    assert ops.count("Gemv") == 2 and ops.count("CAReduce") == len(f.sums) and f.g2 is not None
    assert len(f.sums) == {"sums0": 0, "sums2": 2}.get(name, 1)
    classes = tuple("scal" if prog.vars[v].ndim == 0 or prog.vars[v].const is not None else "row" for v in f.ext)
    by_ptr = tuple(prog.vars[v].ndim == 0 and prog.vars[v].const is None for v in f.ext)
    for J in range(1, 9):
        lib.compile_cubin(f._module(J, classes, by_ptr)["src"], "rowfuse")


def test_fused_gemm_refuses_beta_without_c_in():
    """``ab_gemm_packed_fused`` with beta != 0 and neither C nor C_in (a value kept as a bf16
    plane only) is an invalid call, refused before anything is launched."""
    import ctypes as C

    from aesara_b200.runtime import lib

    L = lib.load()
    M, N, K = 256, 256, 256
    A = lib.GemmOperand(16, None, M, K, K, 0, 2)
    B = lib.GemmOperand(16, None, N, K, K, 0, 2)
    ep = lib.GemmEpilogue()
    ep.module = 16
    ep.n_operands = 0
    ep.n_outputs = 1
    rc = L.ab_gemm_packed_fused(2, M, N, K, 1.0, C.byref(A), C.byref(B), 1.0, None, 0, 0, None, N, 1,
                                C.byref(ep), None)
    assert rc == 3  # AB_ERR_INVALID
    assert "C_in" in L.ab_last_error().decode()


def test_fused_kernel_sources_compile_for_sm90a():
    """NVRTC (no GPU needed): the row-region kernel, the wgmma GEMM with a generated
    epilogue, and the reduction with a fused pre-map."""
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests._cases import load_case

    for name in ("cfg5_logreg", "cfg3_mlp", "careduce_big_1d"):
        prog, _, _ = load_case(name)
        ex = ProgramExecutor(prog, precision=2 if name == "cfg3_mlp" else 0)
        assert ex._fusions
        for f in ex._fusions:
            assert f.compile_all() == 1


def test_gemm_epilogue_sources_follow_the_precision_policy(monkeypatch):
    """The generated GEMM-epilogue module depends on the executor's product policy: float-pair
    (float64-equivalent) sums and no transposed plane under the fp32-faithful default, float32
    tree sums and the transposed bf16 plane of a value whose consumer contracts over its rows
    under the bf16 policy (AB_EP_NO_TPLANE switches it off); bias rows are recognised
    statically.  The bf16-policy kernels of the cfg3
    regions compile (NVRTC, no GPU) with at most a small stack frame (no spills in the chunk loop)."""
    import re
    import subprocess
    import tempfile

    from aesara_b200.runtime import lib
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests._cases import load_case

    prog, _, _ = load_case("cfg3_mlp")
    monkeypatch.setenv("AB_GEMM_FUSE_FP32", "1")  # regions are off by default under the fp32-faithful policy

    def defines(src):
        out = {}  # the generated block comes first; the kernel header repeats some as #ifndef defaults
        for m in re.finditer(r"^#define (AB_EP_\w+) \(?(-?\d+)\)?$", src, re.M):
            out.setdefault(m.group(1), m.group(2))
        return out

    for precision, exact, tplane in ((0, "1", "-1"), (1, "0", "-1"), (2, "0", "0")):
        regions = sorted((f for f in ProgramExecutor(prog, precision=precision)._fusions), key=lambda f: f.g)
        d = [defines(f.source()) for f in regions]
        assert [x["AB_EP_EXACT_SUMS"] for x in d] == [exact] * 3
        assert [x["AB_EP_TPLANE"] for x in d] == [tplane] * 3    # h, dout, dpre: each feeds a weight gradient
        assert [x["AB_EP_ROWMASK"] for x in d] == ["1", "1", "0"]  # b1, b2 are [1, N] rows; region 3 reads h
        assert [x["AB_EP_COLSUM"] for x in d] == ["-1", "0", "0"] and [x["AB_EP_FULLSUM"] for x in d] == ["-1", "1", "-1"]
    monkeypatch.setenv("AB_EP_NO_TPLANE", "1")
    d = [defines(f.source()) for f in ProgramExecutor(prog, precision=2)._fusions]
    assert {x["AB_EP_TPLANE"] for x in d} == {"-1"}
    monkeypatch.delenv("AB_EP_NO_TPLANE")
    # no spills in the kernels the default bench launches (cuobjdump -res-usage of the cached cubin)
    import shutil

    if shutil.which("cuobjdump") is None:
        return
    for f in ProgramExecutor(prog, precision=2)._fusions:
        cubin = lib.compile_cubin(f.source(), "gemm_ep")
        with tempfile.NamedTemporaryFile(suffix=".cubin") as tf:
            tf.write(cubin)
            tf.flush()
            out = subprocess.run(["cuobjdump", "-res-usage", tf.name], capture_output=True, text=True).stdout
        m = re.search(r"Function ab_gemm_ep_f16:\s*\n\s*REG:(\d+) STACK:(\d+)", out)
        assert m is not None, out[:400]
        assert int(m.group(2)) <= 128, f"stack frame of the fused bf16 kernel: {m.group(0)}"  # was 184-264 with spills in the chunk loop


def test_staging_swizzle_is_conflict_free():
    """The shared-memory chunk of the fused GEMM epilogue (st_off in
    csrc/ab_gemm_tc_kernel.cuh): 32 rows x 32 floats,
    16-byte group g of row r stored at group g ^ (r & 7).  Restated here: every access pattern the
    kernels use touches each of the 32 banks at most once per shared-memory wavefront (128-bit
    accesses are served a quarter warp = 8 lanes at a time, 32-bit accesses a whole warp)."""
    def word(r, g, w=0):  # 32-bit word index of element 4 g + w of row r
        return r * 32 + ((g ^ (r & 7)) << 2) + w

    def banks128(addrs):  # a quarter warp of 128-bit accesses: 8 lanes x 4 consecutive banks
        return sorted(b for a in addrs for b in range(a % 32, a % 32 + 4))

    for g in range(8):  # fused_eval / cell epilogue: lane = row writes (reads) its group g
        for q in range(4):
            assert banks128([word(r, g) for r in range(8 * q, 8 * q + 8)]) == list(range(32))
    for i in range(8):  # pass 1 / restage: lanes 8 k .. 8 k + 7 handle row 4 i + k, lane % 8 = group
        for k in range(4):
            assert banks128([word(4 * i + k, g) for g in range(8)]) == list(range(32))
    for r in range(32):  # pass 2: lane c reads column c of row r (one 32-bit word per lane)
        assert sorted(word(r, c >> 2, c & 3) % 32 for c in range(32)) == list(range(32))
    # and the map is a bijection on the 1024 words of the chunk
    assert sorted(word(r, g, w) for r in range(32) for g in range(8) for w in range(4)) == list(range(1024))


def test_kernel_cache_is_thread_safe_and_prunable(tmp_path, monkeypatch):
    """runtime/lib.py: several threads compiling the same (and different) sources into one cache
    directory end with one valid cubin per source (the probe / temporary files of concurrent
    callers used to collide and send one of them to ~/.cache); ``prune_cache`` drops what no
    build has touched since a given time and keeps what was used."""
    import time
    from concurrent.futures import ThreadPoolExecutor

    from aesara_b200.runtime import lib

    monkeypatch.setenv("AESARA_B200_CACHE", str(tmp_path))
    srcs = [f'extern "C" __global__ void k{i}(float* p) {{ p[threadIdx.x] = {i}.0f; }}' for i in range(3)]
    with ThreadPoolExecutor(6) as pool:
        blobs = list(pool.map(lambda s: lib.compile_cubin(s, "t"), srcs * 4))
    assert lib.cache_dir() == str(tmp_path)
    files = sorted(f for f in os.listdir(tmp_path) if f.endswith(".cubin"))
    assert len(files) == 3 and not [f for f in os.listdir(tmp_path) if ".tmp" in f or f.startswith(".w")]
    assert all(b[:4] == b"\x7fELF" for b in blobs) and len({bytes(b) for b in blobs}) == 3
    old = time.time() - 3600
    for f in files[:2]:
        os.utime(os.path.join(tmp_path, f), (old, old))
    lib.compile_cubin(srcs[0], "t")  # a cache hit marks the file as used
    cutoff = time.time() - 60
    dropped = lib.prune_cache(cutoff)
    left = [f for f in os.listdir(tmp_path) if f.endswith(".cubin")]
    assert dropped >= 1 and len(left) == 3 - dropped
    for s in srcs:  # whatever was dropped is simply compiled again
        assert lib.compile_cubin(s, "t")[:4] == b"\x7fELF"


def test_regions_can_be_switched_off(monkeypatch):
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests._cases import load_case

    prog, _, _ = load_case("cfg3_mlp")
    for var in ("AB_NO_GEMM_FUSE", "AB_NO_RED_FUSE", "AB_NO_ROWFUSE"):
        monkeypatch.setenv(var, "1")
    assert not ProgramExecutor(prog)._fusions


def test_host_eval_compares_with_the_device_c_conversions():
    """The device bodies compare and combine typed operands under C's usual arithmetic
    conversions (int32 with uint32 is uint32, int64 with uint64 is uint64, int64 with float32
    is float32); host_eval, which answers the same expressions for small host operands, and the
    oracle give the same values, so one program has one answer wherever it runs."""
    from aesara_b200.runtime import host_eval
    from oracle.scalar_np import eval_expr

    def one(op, dts, out, vals):
        expr = {"inputs": list(dts), "out_dtypes": [out], "outputs": ["t0"],
                "stmts": [{"op": op, "args": [f"i{k}" for k in range(len(dts))], "dtype": out,
                           "in_dtypes": list(dts)}]}
        args = [np.asarray(v, dtype=d) for v, d in zip(vals, dts)]
        assert host_eval.supports(expr)
        h = host_eval.eval_expr(expr, args)[0]
        o = eval_expr(expr, args)[0]
        np.testing.assert_array_equal(h, o)
        return h.item()

    assert one("lt", ["int32", "uint32"], "bool", [-1, 5]) is False
    assert one("gt", ["int64", "uint64"], "bool", [-1, 5]) is True
    assert one("eq", ["int64", "float32"], "bool", [2 ** 24 + 1, 2 ** 24]) is True
    assert one("lt", ["int16", "uint16"], "bool", [-1, 5]) is True  # both promote to int
    assert one("add", ["int32", "uint32"], "int64", [-1, 0]) == 2 ** 32 - 1
    assert one("or", ["int32", "uint32"], "int64", [-1, 0]) == 2 ** 32 - 1
    assert one("switch", ["bool", "int32", "uint32"], "int64", [True, -1, 5]) == 2 ** 32 - 1
    assert one("clip", ["int32", "uint32", "uint32"], "int64", [-1, 2, 9]) == 9
    assert one("true_divide", ["int64", "float32"], "float64", [2 ** 24 + 1, 1.0]) == 2.0 ** 24
