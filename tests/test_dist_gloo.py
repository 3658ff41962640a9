"""CPU, world_size 2 over gloo: the host-side sharding logic (row blocks, packed
exchange layout, mean-of-shards weights) reproduces the unsharded result.  The
per-shard evaluation uses the oracle interpreter here; on the GPU the same
logic drives the device executor (bench.py --gpus N)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from aesara_b200.shard import ALLREDUCE_MIN_ELEMS, combine_weights, exchange_plan, pack_layout, row_block


def test_row_blocks_cover_and_balance():
    for n, w in [(10, 3), (7, 8), (1 << 20, 8), (0, 2)]:
        blocks = [row_block(n, w, r) for r in range(w)]
        assert blocks[0][0] == 0 and blocks[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(blocks, blocks[1:]))
        sizes = [b - a for a, b in blocks]
        assert max(sizes) - min(sizes) <= 1


def test_pack_layout_alignment():
    L = pack_layout([(), (5,), (3, 3)])
    assert L.offsets == [0, 4, 12] and L.total == 24


def test_exchange_plan_by_payload():
    assert exchange_plan(514, 8) == "allgather"                   # cfg5: (D+2) floats
    assert exchange_plan(2 * 4096 * 4096 + 2 * 4096 + 4, 8) == "allreduce"   # cfg3 gradients
    assert exchange_plan(ALLREDUCE_MIN_ELEMS, 2) == "allreduce"
    assert exchange_plan(1 << 30, 1) == "allgather"               # nothing to exchange


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n_rows, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle.program_np import run_program
    from tests._cases import load_case

    prog, _, _ = load_case("cfg5_logreg")
    rng = np.random.default_rng(7)
    X = rng.standard_normal((n_rows, 16)).astype("float32")
    y = (rng.random(n_rows) < 0.5).astype("float32")
    w = (rng.standard_normal(16) * 0.1).astype("float32")
    a, b = row_block(n_rows, world, rank)
    outs = run_program(prog, [X[a:b], y[a:b], w, np.float32(0.1)])
    L = pack_layout([np.shape(o) for o in outs])
    flat = torch.zeros(L.total, dtype=torch.float32)
    for o, off in zip(outs, L.offsets):
        o = np.asarray(o, "float32").reshape(-1)
        flat[off : off + o.size] = torch.from_numpy(o.copy())
    gathered = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    rows = [row_block(n_rows, world, r) for r in range(world)]
    wts = combine_weights("mean", [e - s for s, e in rows])
    comb = sum(wt * g for wt, g in zip(wts, gathered)).numpy()
    # the large-payload plan: weight the local buffer, one all_reduce (shard.exchange_plan)
    reduced = flat * wts[rank]
    dist.all_reduce(reduced, op=dist.ReduceOp.SUM)
    np.testing.assert_allclose(reduced.numpy(), comb, rtol=1e-6, atol=1e-7)
    if rank == 0:
        full = run_program(prog, [X, y, w, np.float32(0.1)])
        res = []
        for o, s, off in zip(full, L.shapes, L.offsets):
            n = int(np.prod(s)) if s else 1
            res.append((np.asarray(o, "float32").reshape(-1), comb[off : off + n]))
        q.put([(a.tolist(), b.tolist()) for a, b in res])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_sharded_logreg_matches_unsharded_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, 101, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=100)
    for p in procs:
        p.join(timeout=30)
        assert p.exitcode == 0
    for full, comb in res:
        np.testing.assert_allclose(comb, full, rtol=2e-5, atol=1e-6)


def _worker_plan(rank, world, port, case, n_rows, q):
    """The combination rule comes from the graph (shardplan), not from the caller."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from aesara_b200 import shardplan
    from oracle.program_np import run_program
    from tests._cases import load_case

    prog, _, _ = load_case(case)
    plan = shardplan.infer_sharded_inputs(prog)
    rng = np.random.default_rng(11)
    H = 24
    ins = [rng.standard_normal((n_rows, H)).astype("float32"), rng.standard_normal((n_rows, H)).astype("float32"),
           (rng.standard_normal((H, H)) / 5).astype("float32"), (rng.standard_normal(H) * 0.1).astype("float32"),
           (rng.standard_normal((H, H)) / 5).astype("float32"), (rng.standard_normal(H) * 0.1).astype("float32")]
    a, b = row_block(n_rows, world, rank)
    local = [x[a:b] if ax == 0 else x for x, ax in zip(ins, plan.sharded_inputs)]
    outs = run_program(prog, local)
    n_local = torch.tensor([float(b - a)], dtype=torch.float64)
    n_tot = n_local.clone()
    dist.all_reduce(n_tot)
    w = float(n_local / n_tot)
    combined = []
    for o, mode in zip(outs, plan.outputs):
        t = torch.from_numpy(np.array(o, dtype=np.float32).reshape(-1).copy())
        if mode[0] == "mean":
            t *= w
        assert mode[0] in ("mean", "sum")
        dist.all_reduce(t)
        combined.append(t.numpy())
    if rank == 0:
        full = run_program(prog, ins)
        q.put([(np.asarray(f, "float32").reshape(-1).tolist(), c.tolist()) for f, c in zip(full, combined)])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_sharded_mlp_combines_by_the_plan_gloo():
    """cfg3 over 2 ranks with UNEQUAL row blocks (33 rows): the analysis says `mean` for the loss
    and every gradient; weighting each rank by its share of the rows reproduces the unsharded
    evaluation."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_plan, args=(r, 2, port, "cfg3_mlp", 33, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = q.get(timeout=100)
    for p in procs:
        p.join(timeout=30)
        assert p.exitcode == 0
    for full, comb in res:
        np.testing.assert_allclose(comb, full, rtol=3e-5, atol=1e-6)
