"""The fused embedding-bag kernels (csrc/cuda/ops_embbag.cu) through ``ops.StoreEmbeddingBag`` on an H100: against
the float64 rule ``embedding_bag_reference``, bit for bit against themselves, against the torch route, in multi-hot
DeepFM, and on multi-rank stores (three logical ranks on one GPU, as in test_gpu_fused_multirank.py): rows owned by a
peer, local replicas and keys whose relocation is in flight."""
import functools
import threading
import time

import numpy as np
import pytest
import torch

from harness import run_cluster
from test_gpu_fused_multirank import _idiom, _load, _mover

gpu = pytest.mark.gpu
WORLD = 3
RTOL, ATOL = 2e-4, 2e-5


def _cuda_server(dim, num_keys, job):
    import adapm_b200 as ad

    s = ad.Server(2 * dim, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                  job=f"{job}_{np.random.randint(1 << 30)}", device=0)
    return s, ad.Worker(0, s)


def _table(num_keys, dim, g):
    t = torch.randn(num_keys, 2 * dim, generator=g) * 0.5
    t[:, dim:] = torch.rand(num_keys, dim, generator=g)
    t[: num_keys // 8, dim:] = 0.0              # accumulators at exactly 0: a key with G == 0 must stay finite
    return t


def _rows(kv, num_keys, dim):
    v = torch.empty(num_keys * 2 * dim, device=kv.server.device)
    kv.wait(kv.pull(torch.arange(num_keys, device=kv.server.device), v))
    return v.view(num_keys, 2 * dim).cpu()


HOT = 5


def _hard_bags(g, num_keys, nbags=3000, big=10_000):
    """empty bags, one bag of `big` keys, and key HOT at every other position (>= 10 000 occurrences over most bags)"""
    lens = torch.randint(0, 9, (nbags,), generator=g)
    lens[::97] = 0
    lens[17] = big
    nnz = int(lens.sum())
    keys = torch.randint(0, num_keys, (nnz,), generator=g)
    keys[::2] = HOT
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    assert int((keys == HOT).sum()) >= 10_000
    return keys, offsets


def _run(kv, bag, keys, offsets, w, grad):
    dev = kv.server.device
    out = bag(keys.to(dev), offsets.to(dev), w.to(dev) if w is not None else None)
    out.backward(grad.to(dev))
    torch.cuda.synchronize()
    return out.detach().cpu()


MODES = [("sum", False), ("mean", False), ("sum", True)]


@gpu
# float4 per lane (VPL) 1 to 4; dim 4 and 8 give 1 and 2 lanes per bag
@pytest.mark.parametrize("dim", [4, 20, 64, 128, 512, 8, 132, 256, 260, 384])
def test_forward_and_step_match_float64_rule(dim):
    from adapm_b200 import _C
    from adapm_b200.ops import StoreEmbeddingBag, embedding_bag_reference

    num_keys = 20_000
    server, kv = _cuda_server(dim, num_keys, f"bag{dim}")
    try:
        for mode, weighted in MODES:
            g = torch.Generator().manual_seed(dim + 3 * weighted + 5 * (mode == "mean"))
            table = _table(num_keys, dim, g)
            keys, offsets = _hard_bags(g, num_keys)
            w = torch.rand(keys.numel(), generator=g) * 2 - 0.5 if weighted else None
            grad = torch.randn(offsets.numel() - 1, dim, generator=g) * 1e-3
            _load(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, mode=mode, lr=0.05, grad_scale=7.0)
            n0 = _C.kernel_launches()
            out = _run(kv, bag, keys, offsets, w, grad)
            assert _C.kernel_launches() - n0 == 5        # forward 1 + backward 4 (the radix sort counted as one)
            ref_out, ref_table = embedding_bag_reference(table, keys, offsets, w, mode, grad, lr=0.05, grad_scale=7.0)
            what = f"dim {dim} {mode} weighted={weighted}"
            # fp32 sums in key order: a bag's error grows with its length; allow 1e-5 of the bag's sum of |w x|
            abs_sum, _ = embedding_bag_reference(table.abs(), keys, offsets, w.abs() if w is not None else None, mode)
            err = (out.double() - ref_out).abs()
            assert bool((err <= 1e-4 * ref_out.abs() + 1e-5 * abs_sum + 1e-6).all()), (what, float(err.max()))
            assert torch.all(out[offsets[1:] == offsets[:-1]] == 0), what
            rows = _rows(kv, num_keys, dim)
            assert torch.isfinite(rows).all(), what
            torch.testing.assert_close(rows.double(), ref_table, rtol=RTOL, atol=ATOL, msg=lambda m: f"{what}: {m}")
            s = bag.stats.tolist()
            assert s[3] == torch.unique(keys).numel() and s[2] == 0 and s[1] == 0, (what, s)
    finally:
        kv.finalize()
        server.shutdown()


@gpu
def test_launch_counts():
    from adapm_b200 import _C
    from adapm_b200.ops import StoreEmbeddingBag

    server, kv = _cuda_server(20, 1000, "baglaunch")
    try:
        bag = StoreEmbeddingBag(server, kv, 20)
        dev = server.device
        keys = torch.randint(0, 1000, (500,), device=dev)
        offsets = torch.arange(0, 501, 5, device=dev)
        torch.cuda.synchronize()
        n0 = _C.kernel_launches()
        out = bag(keys, offsets)
        assert _C.kernel_launches() - n0 == 1
        out.sum().backward()
        assert _C.kernel_launches() - n0 == 5
        torch.cuda.synchronize()
    finally:
        kv.finalize()
        server.shutdown()


def _deepfm_batch(g, B=8192, F=26, L=8, num_keys=1_000_000):
    lens = torch.randint(1, L + 1, (B * F,), generator=g)
    per = num_keys // F
    field = torch.repeat_interleave(torch.arange(B * F) % F, lens)
    u = torch.rand(int(lens.sum()), generator=g, dtype=torch.float64)
    keys = (per * u ** 3).long().clamp(max=per - 1) + field * per
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    return keys, offsets


@gpu
def test_two_runs_on_fresh_stores_are_bit_identical():
    from adapm_b200.ops import StoreEmbeddingBag

    dim, num_keys = 20, 1_000_000
    g = torch.Generator().manual_seed(11)
    keys, offsets = _deepfm_batch(g, num_keys=num_keys)
    w = torch.rand(keys.numel(), generator=g)
    grad = torch.randn(offsets.numel() - 1, dim, generator=g) * 1e-3
    table = _table(num_keys, dim, g)
    res = []
    for run in range(2):
        server, kv = _cuda_server(dim, num_keys, f"bagdet{run}")
        try:
            _load(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, lr=0.05, grad_scale=8192.0)
            out = _run(kv, bag, keys, offsets, w, grad)
            res.append((out, _rows(kv, num_keys, dim)))
        finally:
            kv.finalize()
            server.shutdown()
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
    assert not torch.equal(res[0][1], table)


@gpu
@pytest.mark.parametrize("mode", ["sum", "mean"])
def test_fused_route_matches_torch_route_at_deepfm_shape(mode):
    from adapm_b200.ops import StoreEmbeddingBag

    dim, num_keys = 20, 1_000_000
    g = torch.Generator().manual_seed(12)
    keys, offsets = _deepfm_batch(g, num_keys=num_keys)
    grad = torch.randn(offsets.numel() - 1, dim, generator=g) * 1e-4
    table = _table(num_keys, dim, g)
    res = {}
    for impl in ("fused", "torch"):
        server, kv = _cuda_server(dim, num_keys, f"bagroute{impl}")
        try:
            _load(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, mode=mode, lr=0.05, grad_scale=8192.0, impl=impl)
            out = _run(kv, bag, keys, offsets, None, grad)
            kv.waitall()
            res[impl] = (out, _rows(kv, num_keys, dim))
        finally:
            kv.finalize()
            server.shutdown()
    torch.testing.assert_close(res["fused"][0], res["torch"][0], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(res["fused"][1], res["torch"][1], rtol=1e-4, atol=1e-6)


def _deepfm_cfg(multi_hot):
    from adapm_b200.models.deepfm import DeepFMConfig

    return DeepFMConfig(num_features=26 * 2000, num_fields=26, embed_dim=16, hidden=(128, 128), batch_size=1024,
                        precision="fp32", lr_dense=3e-3, multi_hot=multi_hot)


@gpu
def test_multi_hot_of_length_one_matches_single_hot_deepfm():
    from adapm_b200.models.deepfm import DeepFM, synthetic_ctr_batch

    out = {}
    for mh in (0, 1):
        cfg = _deepfm_cfg(mh)
        server, kv = _cuda_server(cfg.emb_len, cfg.num_features, f"fm{mh}")
        try:
            model = DeepFM(server, kv, cfg)
            model.init_model()
            losses, first = [], None
            for s in range(5):
                ids, y = synthetic_ctr_batch(cfg, s)
                if mh:
                    off = torch.arange(ids.numel() + 1, dtype=torch.int64)
                    losses.append(model.step(ids.reshape(-1), y, offsets=off))
                else:
                    losses.append(model.step(ids, y))
                kv.advance_clock()
                if s == 0:
                    kv.waitall()
                    first = _rows(kv, cfg.num_features, cfg.emb_len)
            kv.waitall()
            torch.cuda.synchronize()
            out[mh] = (losses, _rows(kv, cfg.num_features, cfg.emb_len), model.rows_pushed, first)
        finally:
            kv.finalize()
            server.shutdown()
    np.testing.assert_allclose(out[1][0], out[0][0], rtol=1e-4)
    # after one step the rows differ by the order of the gradient sums only (amplified up to lr / sqrt(acc) = 50 x for
    # the fresh accumulators of 1e-6); later steps also see the MLPs drift apart (Adam amplifies the last-bit
    # differences of small gradients), still far below the per-step update of lr = 0.05
    torch.testing.assert_close(out[1][3], out[0][3], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(out[1][1], out[0][1], rtol=1e-3, atol=1e-4)
    assert out[1][2] == out[0][2]


@gpu
def test_multi_hot_deepfm_trains_on_gpu():
    from adapm_b200.models.deepfm import DeepFM, synthetic_multi_hot_batch

    cfg = _deepfm_cfg(8)
    server, kv = _cuda_server(cfg.emb_len, cfg.num_features, "fmtrain")
    try:
        model = DeepFM(server, kv, cfg)
        model.init_model()
        losses = []
        for s in range(40):
            ids, off, y = synthetic_multi_hot_batch(cfg, s % 8)
            losses.append(model.step(ids, y, offsets=off))
            kv.advance_clock()
        assert all(np.isfinite(losses)), losses
        assert np.mean(losses[-5:]) < np.mean(losses[:5]) - 0.02, losses
        assert model.bag.stats[3].item() == model.rows_pushed > 0
    finally:
        kv.finalize()
        server.shutdown()


# ---------------------------------------------------------------------------------------------- several ranks
DIM = 20


def _spread(rank, m, g):
    """m distinct keys for ``rank``, disjoint from the other ranks' keys, 3 in 4 homed on another rank"""
    j = torch.arange(m)
    home = torch.where(j % 4 == 0, torch.full_like(j, rank), (rank + 1 + (j // 4) % 2) % WORLD)
    return WORLD * (rank * m + j) + home


def _bag_batch(pool, g, nbags=96, L=6, w=False):
    lens = torch.randint(0, L + 1, (nbags,), generator=g)
    keys = pool[torch.randint(0, pool.numel(), (int(lens.sum()),), generator=g)]
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    weights = torch.rand(keys.numel(), generator=g) if w else None
    grad = torch.randn(nbags, DIM, generator=g) * 1e-2
    return keys, offsets, weights, grad


def _fused_step(server, kv, bag, b, stream):
    keys, offsets, w, grad = b
    dev = server.device
    with torch.cuda.stream(stream):
        out = bag(keys.to(dev), offsets.to(dev), w.to(dev) if w is not None else None)
        out.backward(grad.to(dev))
    stream.synchronize()
    return out.detach().cpu()


def _apply_rule(table, batches):
    from adapm_b200.ops import embedding_bag_reference

    outs = []
    for keys, offsets, w, grad in batches:
        out, table = embedding_bag_reference(table, keys, offsets, w, "sum", grad, lr=0.05, grad_scale=3.0)
        outs.append(out)
    return table, outs


def _peer_worker(kv, server, wid, table, batches):
    from adapm_b200.ops import StoreEmbeddingBag

    rank = server.my_rank()
    n = table.shape[0]
    if rank == 0:
        _load(kv, [(torch.arange(n), table)])
    kv.waitall(); kv.barrier()
    bag = StoreEmbeddingBag(server, kv, DIM, lr=0.05, grad_scale=3.0)
    out = _fused_step(server, kv, bag, batches[rank], torch.cuda.Stream(server.device))
    kv.barrier()
    rows = _rows(kv, n, DIM) if rank == 0 else None
    kv.barrier()
    kv.finalize()
    return {"out": out, "rows": rows, "stats": bag.stats.tolist()}


@gpu
def test_peer_rows_match_float64_rule():
    """three ranks, no intents, disjoint key sets (3 in 4 rows owned by a peer), all ranks at once"""
    m = 160
    n = WORLD * WORLD * m
    g = torch.Generator().manual_seed(21)
    table = _table(n, DIM, g)
    batches = [_bag_batch(_spread(r, m, g), g, w=r == 1) for r in range(WORLD)]
    res = run_cluster(functools.partial(_peer_worker, table=table, batches=batches), world=WORLD, workers=1,
                      mode="threads", value_lengths=2 * DIM, num_keys=n, dtype="float32", backend="cuda")
    ref_table, _ = _apply_rule(table, batches)
    torch.testing.assert_close(res[0][0]["rows"].double(), ref_table, rtol=RTOL, atol=ATOL)
    for r in range(WORLD):
        _, (ref_out,) = _apply_rule(table, [batches[r]])
        torch.testing.assert_close(res[r][0]["out"].double(), ref_out, rtol=RTOL, atol=ATOL)
        s = res[r][0]["stats"]
        keys = batches[r][0]
        assert s[3] == torch.unique(keys).numel() and s[1] > 0 and s[2] == 0, (r, s)


def _replica_worker(kv, server, wid, table, batches):
    from adapm_b200.ops import StoreEmbeddingBag

    rank = server.my_rank()
    n = table.shape[0]
    if rank == 0:
        _load(kv, [(torch.arange(n), table)])
    kv.waitall(); kv.barrier()
    mine = torch.unique(batches[rank][0])
    c = kv.current_clock()
    kv.intent(mine, c, c + 1_000_000)
    for _ in range(50):
        kv.advance_clock()
        _idiom(kv)
        missing = sum(not server.is_local(int(k)) for k in mine)
        if server.allreduce_sum([float(missing)])[0] == 0:
            break
    local = all(server.is_local(int(k)) for k in mine)
    bag = StoreEmbeddingBag(server, kv, DIM, lr=0.05, grad_scale=3.0)
    stream = torch.cuda.Stream(server.device)
    out = None
    for turn in range(WORLD):
        if turn == rank:
            out = _fused_step(server, kv, bag, batches[rank], stream)
        _idiom(kv)
    rows = _rows(kv, n, DIM)
    kv.barrier()
    kv.finalize()
    return {"out": out, "rows": rows, "stats": bag.stats.tolist(), "local": local}


@gpu
def test_replicas_match_float64_rule_in_turn_order():
    """replication_only, overlapping batches: after the intents every rank's rows are local; ranks 0, 1, 2 run one
    step each with a propagation round between them; every rank then reads the three steps applied in that order"""
    n = 600
    g = torch.Generator().manual_seed(22)
    table = _table(n, DIM, g)
    pool = torch.arange(n)
    batches = [_bag_batch(pool[torch.randperm(n, generator=g)[:200]], g) for _ in range(WORLD)]
    res = run_cluster(functools.partial(_replica_worker, table=table, batches=batches), world=WORLD, workers=1,
                      mode="threads", value_lengths=2 * DIM, num_keys=n, dtype="float32", backend="cuda",
                      options={"sys.techniques": "replication_only"})
    assert sum(r["counters"]["replica_setups"] for r in res.values()) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())
    ref_table, ref_outs = _apply_rule(table, batches)
    for r in range(WORLD):
        out = res[r][0]
        assert out["local"], f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"].double(), ref_table, rtol=RTOL, atol=ATOL, msg=lambda m: f"rank {r}: {m}")
        torch.testing.assert_close(out["out"].double(), ref_outs[r], rtol=RTOL, atol=ATOL)
        s = out["stats"]
        assert s[1] == 0 and s[2] == 0 and s[3] == torch.unique(batches[r][0]).numel(), (r, s)


INFLIGHT_STEPS = 32


def _inflight_worker(kv, server, wid, table, steps, done):
    from adapm_b200.ops import StoreEmbeddingBag

    rank = server.my_rank()
    n = table.shape[0]
    if rank == 0:
        _load(kv, [(torch.arange(n), table)])
    kv.waitall(); kv.barrier()
    out = {}
    if rank < 2:
        out["iters"] = _mover(kv, rank, torch.arange(n), done)
    else:
        bag = StoreEmbeddingBag(server, kv, DIM, lr=0.05, grad_scale=3.0)
        stream = torch.cuda.Stream(server.device)
        outs = []
        try:
            for b in steps:
                outs.append(_fused_step(server, kv, bag, b, stream))
                time.sleep(0.03)          # spread the steps over many sync rounds
        finally:
            done.set()
        out["outs"], out["stats"] = outs, bag.stats.tolist()
    kv.barrier()
    for _ in range(8):
        kv.advance_clock()
    _idiom(kv)
    if rank == 2:
        out["rows"] = _rows(kv, n, DIM)
    kv.barrier()
    kv.finalize()
    return out


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_steps_lose_no_update_while_keys_move(technique):
    """ranks 0 and 1 keep relocating all keys between them; rank 2 runs 32 forward + backward steps on those keys"""
    n = 448
    g = torch.Generator().manual_seed(23)
    table = _table(n, DIM, g)
    steps = [_bag_batch(torch.arange(n), g, nbags=64, w=i % 2 == 1) for i in range(INFLIGHT_STEPS)]
    done = threading.Event()
    res = run_cluster(functools.partial(_inflight_worker, table=table, steps=steps, done=done), world=WORLD, workers=1,
                      mode="threads", value_lengths=2 * DIM, num_keys=n, dtype="float32", backend="cuda",
                      options={"sys.techniques": technique})
    out = res[2][0]
    s = out["stats"]
    relocations = sum(r["counters"]["relocations"] for r in res.values())
    info = f"{technique}: stats {s}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values()), info
    assert s[3] == sum(torch.unique(b[0]).numel() for b in steps), info
    ref_table, ref_outs = _apply_rule(table, steps)
    torch.testing.assert_close(out["rows"].double(), ref_table, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}: {m}")
    for i, (o, r) in enumerate(zip(out["outs"], ref_outs)):
        torch.testing.assert_close(o.double(), r, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}, step {i}: {m}")
