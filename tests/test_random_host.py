"""CPU: random variables on the device -- the NumPy restatement of the Philox stream, the
lowering of RandomStream graphs, the refusals, and the sm_90a build of csrc/ab_random.cu.
The device draws themselves are checked in tests/test_gpu_random.py."""
import os
import re
import subprocess

import numpy as np
import pytest

from aesara_b200.compat import bootstrap
from oracle.random_np import philox4x32_10, philox_words, random_raw, random_sample

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not bootstrap.available(), reason="reference front-end not available")


@pytest.mark.parametrize("ctr, key, want", [
    ([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    """The Random123 known-answer vectors of Philox4x32-10."""
    got = philox4x32_10(np.array(ctr, np.uint64), key)
    assert " ".join(f"{int(w):08x}" for w in got) == want


def test_stream_words_and_transforms():
    key = 0x0123456789ABCDEF
    w = philox_words(key, 0, 3)
    ref = philox4x32_10(np.array([[b, 0, 0, 0] for b in range(3)], np.uint64), (0x89ABCDEF, 0x01234567)).reshape(-1)
    np.testing.assert_array_equal(w, ref)
    # block b > 2**32 puts the high half in counter word 1
    hi = philox_words(key, 2 ** 32 + 5, 1)
    np.testing.assert_array_equal(hi, philox4x32_10(np.array([5, 1, 0, 0], np.uint64), (0x89ABCDEF, 0x01234567)))
    u = random_raw("uniform", "float32", key, 5)
    np.testing.assert_array_equal(u, (philox_words(key, 0, 2)[:5] >> np.uint64(8)).astype(np.float64) * 2.0 ** -24)
    u64 = random_raw("uniform", "float64", key, 3)
    ww = philox_words(key, 0, 2)
    np.testing.assert_array_equal(u64[1], float(((int(ww[3]) << 32) | int(ww[2])) >> 11) * 2.0 ** -53)
    # chunking does not change the stream
    import oracle.random_np as P

    old, P._CHUNK_BLOCKS = P._CHUNK_BLOCKS, 3
    try:
        for dist, dt in (("uniform", "float32"), ("normal", "float64"), ("bernoulli", "int64")):
            a = random_raw(dist, dt, key, 37)
            P._CHUNK_BLOCKS = old
            b = random_raw(dist, dt, key, 37)
            P._CHUNK_BLOCKS = 3
            np.testing.assert_array_equal(a, b)
    finally:
        P._CHUNK_BLOCKS = old
    # an odd trailing normal element is z0 of the last pair
    z = random_raw("normal", "float32", key, 5)
    np.testing.assert_array_equal(z, random_raw("normal", "float32", key, 6)[:5])
    assert np.all((u >= 0) & (u < 1)) and np.all(np.isfinite(z))


def test_sample_edges_and_errors():
    key = 99
    assert random_sample("uniform", "float32", key, (), [0.0, 1.0]).shape == ()
    assert random_sample("normal", "float64", key, (0, 3), [0.0, 1.0]).shape == (0, 3)
    b = random_sample("bernoulli", "int64", key, (1000,), [np.array(0.0)])
    assert b.dtype == np.int64 and not b.any()
    assert random_sample("bernoulli", "int64", key, (1000,), [1.0]).all()
    with pytest.raises(ValueError, match="scale < 0"):
        random_sample("normal", "float32", key, (3,), [0.0, np.array([1.0, -1.0, 1.0])])
    for bad in (-0.1, 1.5, np.nan):
        with pytest.raises(ValueError, match="p < 0"):
            random_sample("bernoulli", "int64", key, (3,), [bad])


# -- lowering ---------------------------------------------------------------------------
def _lower(outputs, updates=None, mode=None):
    aesara = bootstrap.load_aesara()
    from aesara.compile.mode import Mode
    from aesara.graph.rewriting.db import RewriteDatabaseQuery

    from aesara_b200.lower import lower_fgraph

    mode = mode or Mode(linker="py", optimizer=RewriteDatabaseQuery(include=["fast_run"]))
    f = aesara.function([], outputs, mode=mode, updates=updates)
    return lower_fgraph(f.maker.fgraph)


@needs_ref
def test_randomstream_graph_lowers_to_random_variable_nodes():
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.tensor.random.utils import RandomStream

    srng = RandomStream(seed=3)
    u = srng.uniform(-1.0, 2.0, size=(4, 5))
    z = srng.normal(0.0, 1.0, size=(7,), dtype="float64")
    m = srng.bernoulli(0.3, size=(2, 2))
    d = srng.binomial(1, 0.5, size=(3,))
    prog = _lower([u, z, m, d, at.sum(u)])
    rv = [n for n in prog.nodes if n.op == "RandomVariable"]
    got = sorted((n.params["dist"], n.params["dtype"]) for n in rv)
    assert got == sorted([("uniform", "float32" if u.dtype == "float32" else "float64"),
                          ("normal", "float64"), ("bernoulli", "int64"), ("bernoulli", "int64")])
    # fast_run's random_make_inplace: every draw mutates its own Generator
    assert all(n.params["inplace"] for n in rv)
    assert all(n.params.get("destroy") == [0] for n in rv)
    for n in rv:
        assert prog.vars[n.inputs[0]].kind == "other"      # the Generator
        assert prog.vars[n.outputs[0]].kind == "other"
    # the rng updates are the program's updates
    assert len(prog.updates) == 4


@needs_ref
def test_without_rewrites_the_draws_are_not_inplace():
    bootstrap.load_aesara()
    from aesara.compile.mode import Mode
    from aesara.tensor.random.utils import RandomStream

    srng = RandomStream(seed=3)
    u = srng.uniform(0.0, 1.0, size=(3,))
    prog = _lower([u], mode=Mode(linker="py", optimizer=None))
    (n,) = [n for n in prog.nodes if n.op == "RandomVariable"]
    assert n.params == {"dist": "uniform", "dtype": u.dtype, "inplace": False}


@needs_ref
def test_unsupported_distributions_and_randomstate_are_named():
    bootstrap.load_aesara()
    import aesara
    import aesara.tensor as at
    from aesara.tensor.random.utils import RandomStream

    from aesara_b200.lower import UnsupportedOp

    srng = RandomStream(seed=1)
    for draw, name in ((srng.gamma(2.0, 1.0, size=(3,)), "gamma"), (srng.poisson(3.0, size=(3,)), "poisson"),
                       (srng.binomial(5, 0.5, size=(3,)), "binomial")):
        with pytest.raises(UnsupportedOp, match=name):
            _lower([draw])
    rs = aesara.shared(np.random.RandomState(0))
    with pytest.raises(UnsupportedOp, match="normal.*RandomState"):
        _lower([at.random.normal(0, 1, size=(3,), rng=rs)])


@needs_ref
def test_shardplan_refuses_random_variables():
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.compile.mode import Mode
    from aesara.graph.rewriting.db import RewriteDatabaseQuery
    from aesara.tensor.random.utils import RandomStream

    from aesara_b200 import shardplan
    from aesara_b200.lower import lower_fgraph

    aesara = bootstrap.load_aesara()
    x = at.matrix("x")
    srng = RandomStream(seed=0)
    y = x * srng.bernoulli(0.5, size=x.shape)
    f = aesara.function([x], y, mode=Mode(linker="py", optimizer=RewriteDatabaseQuery(include=["fast_run"])))
    prog = lower_fgraph(f.maker.fgraph)
    with pytest.raises(shardplan.ReplicasOnly, match="random variable"):
        shardplan.analyse(prog, [0] + [None] * (len(prog.inputs) - 1))
    with pytest.raises(shardplan.ReplicasOnly):
        shardplan.infer_sharded_inputs(prog)


@needs_ref
def test_oracle_interpreter_draws_the_stream_and_advances_the_generator():
    """run_program evaluates RandomVariable nodes (oracle/random_np.py installs the handler): the
    key is one full-range uint64 of the Generator, drawn in place under fast_run."""
    bootstrap.load_aesara()
    import copy

    import aesara.tensor as at
    from aesara.tensor.random.utils import RandomStream

    from oracle.program_np import run_program

    srng = RandomStream(seed=5)
    u = srng.uniform(-1.0, 3.0, size=(3, 4))
    b = srng.bernoulli(0.25, size=(7,))
    prog = _lower([u, b, at.sum(u)])
    gens = [s[0].get_value() for s in srng.state_updates]
    start = [copy.deepcopy(g) for g in gens]
    outs = run_program(prog, gens)
    keys = [int(copy.deepcopy(g).integers(0, 2 ** 64, dtype=np.uint64)) for g in start]
    want = {"uniform": random_sample("uniform", u.dtype, keys[0], (3, 4), [-1.0, 3.0]),
            "bernoulli": random_sample("bernoulli", "int64", keys[1], (7,), [0.25])}
    np.testing.assert_array_equal(outs[0], want["uniform"])
    np.testing.assert_array_equal(outs[1], want["bernoulli"])
    for g, s0 in zip(gens, start):  # in place: the input Generators themselves advanced once
        s0.integers(0, 2 ** 64, dtype=np.uint64)
        assert g.bit_generator.state == s0.bit_generator.state


def test_random_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    src = os.path.join(ROOT, "aesara_b200", "csrc", "ab_random.cu")
    r = subprocess.run([nvcc, "-c", src, "-o", str(tmp_path / "r.o"), "-gencode", "arch=compute_90a,code=sm_90a",
                        "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    kernels = re.findall(r"Compiling entry function '(\w*random_kernel\w*)' for 'sm_90a'", r.stdout)
    assert len(kernels) == 10, r.stdout  # uniform / normal x f32 / f64, Bernoulli; scalar or strided parameters
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert spills and all(s == ("0", "0") for s in spills), r.stdout
    frames = re.findall(r"(\d+) bytes stack frame", r.stdout)
    assert all(f == "0" for f in frames), r.stdout
