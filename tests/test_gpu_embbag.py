"""The fused embedding-bag kernels (csrc/cuda/ops_embbag.cu) through ``ops.StoreEmbeddingBag`` on an H100: against
the float64 rule ``embedding_bag_reference``, bit for bit against themselves, against the torch route, in multi-hot
DeepFM, and on multi-rank stores (three logical ranks on one GPU, run by multirank.py): rows owned by a peer,
local replicas and keys whose relocation is in flight."""
import numpy as np
import pytest
import torch

from multirank import WORLD, Case, load_rows, on_peer_rows, on_replicas, one_rank_store, spread_keys, while_keys_move

gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5


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
    with one_rank_store(2 * dim, num_keys, "cuda", "float32") as (server, kv):
        for mode, weighted in MODES:
            g = torch.Generator().manual_seed(dim + 3 * weighted + 5 * (mode == "mean"))
            table = _table(num_keys, dim, g)
            keys, offsets = _hard_bags(g, num_keys)
            w = torch.rand(keys.numel(), generator=g) * 2 - 0.5 if weighted else None
            grad = torch.randn(offsets.numel() - 1, dim, generator=g) * 1e-3
            load_rows(kv, [(torch.arange(num_keys), table)])
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


@gpu
def test_launch_counts():
    from adapm_b200 import _C
    from adapm_b200.ops import StoreEmbeddingBag

    with one_rank_store(2 * 20, 1000, "cuda", "float32") as (server, kv):
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
        with one_rank_store(2 * dim, num_keys, "cuda", "float32") as (server, kv):
            load_rows(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, lr=0.05, grad_scale=8192.0)
            out = _run(kv, bag, keys, offsets, w, grad)
            res.append((out, _rows(kv, num_keys, dim)))
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
        with one_rank_store(2 * dim, num_keys, "cuda", "float32") as (server, kv):
            load_rows(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, mode=mode, lr=0.05, grad_scale=8192.0, impl=impl)
            out = _run(kv, bag, keys, offsets, None, grad)
            kv.waitall()
            res[impl] = (out, _rows(kv, num_keys, dim))
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
        with one_rank_store(2 * cfg.emb_len, cfg.num_features, "cuda", "float32") as (server, kv):
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
    with one_rank_store(2 * cfg.emb_len, cfg.num_features, "cuda", "float32") as (server, kv):
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


# ---------------------------------------------------------------------------------------------- several ranks
DIM = 20


def _bag_batch(pool, g, nbags=96, L=6, w=False):
    lens = torch.randint(0, L + 1, (nbags,), generator=g)
    keys = pool[torch.randint(0, pool.numel(), (int(lens.sum()),), generator=g)]
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    weights = torch.rand(keys.numel(), generator=g) if w else None
    grad = torch.randn(nbags, DIM, generator=g) * 1e-2
    return keys, offsets, weights, grad


def _apply_rule(table, batches):
    from adapm_b200.ops import embedding_bag_reference

    outs = []
    for keys, offsets, w, grad in batches:
        out, table = embedding_bag_reference(table, keys, offsets, w, "sum", grad, lr=0.05, grad_scale=3.0)
        outs.append(out)
    return table, outs


def _case(table):
    """one forward and backward per batch through a StoreEmbeddingBag of this rank; a step returns the forward output"""
    def open_bag(server, kv):
        from adapm_b200.ops import StoreEmbeddingBag

        bag = StoreEmbeddingBag(server, kv, DIM, lr=0.05, grad_scale=3.0)
        dev = server.device

        def step(b):
            keys, offsets, w, grad = b
            out = bag(keys.to(dev), offsets.to(dev), w.to(dev) if w is not None else None)
            out.backward(grad.to(dev))
            return out.detach().cpu()

        step.totals = lambda: (None, bag.stats.tolist())
        return step

    n = table.shape[0]
    return Case(2 * DIM, n, [(torch.arange(n), table)], lambda b: torch.unique(b[0]), open_bag)


@gpu
def test_peer_rows_match_float64_rule():
    """three ranks, no intents, disjoint key sets (3 in 4 rows owned by a peer), all ranks at once"""
    m = 160
    n = WORLD * WORLD * m
    g = torch.Generator().manual_seed(21)
    table = _table(n, DIM, g)
    batches = [_bag_batch(spread_keys(r, m, g), g, w=r == 1) for r in range(WORLD)]
    res = on_peer_rows(_case(table), batches, in_turns=False)
    ref_table, _ = _apply_rule(table, batches)
    torch.testing.assert_close(res[0]["rows"][0].double(), ref_table, rtol=RTOL, atol=ATOL)
    for r in range(WORLD):
        _, (ref_out,) = _apply_rule(table, [batches[r]])
        torch.testing.assert_close(res[r]["outs"][0].double(), ref_out, rtol=RTOL, atol=ATOL)
        s = res[r]["stats"]
        keys = batches[r][0]
        assert s[3] == torch.unique(keys).numel() and s[1] > 0 and s[2] == 0, (r, s)


@gpu
def test_replicas_match_float64_rule_in_turn_order():
    """replication_only, overlapping batches: after the intents every rank's rows are local; ranks 0, 1, 2 run one
    step each with a propagation round between them; every rank then reads the three steps applied in that order"""
    n = 600
    g = torch.Generator().manual_seed(22)
    table = _table(n, DIM, g)
    pool = torch.arange(n)
    batches = [_bag_batch(pool[torch.randperm(n, generator=g)[:200]], g) for _ in range(WORLD)]
    res = on_replicas(_case(table), batches)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    ref_table, ref_outs = _apply_rule(table, batches)
    for r in range(WORLD):
        out = res[r]
        assert out["local"], f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref_table, rtol=RTOL, atol=ATOL,
                                   msg=lambda m: f"rank {r}: {m}")
        torch.testing.assert_close(out["outs"][0].double(), ref_outs[r], rtol=RTOL, atol=ATOL)
        s = out["stats"]
        assert s[1] == 0 and s[2] == 0 and s[3] == torch.unique(batches[r][0]).numel(), (r, s)


INFLIGHT_STEPS = 32


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_steps_lose_no_update_while_keys_move(technique):
    """ranks 0 and 1 keep relocating all keys between them; rank 2 runs 32 forward + backward steps on those keys"""
    n = 448
    g = torch.Generator().manual_seed(23)
    table = _table(n, DIM, g)
    steps = [_bag_batch(torch.arange(n), g, nbags=64, w=i % 2 == 1) for i in range(INFLIGHT_STEPS)]
    res = while_keys_move(_case(table), steps, technique)
    out = res[2]
    s = out["stats"]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: stats {s}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res), info
    assert s[3] == sum(torch.unique(b[0]).numel() for b in steps), info
    ref_table, ref_outs = _apply_rule(table, steps)
    torch.testing.assert_close(out["rows"][0].double(), ref_table, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}: {m}")
    for i, (o, r) in enumerate(zip(out["outs"], ref_outs)):
        torch.testing.assert_close(o.double(), r, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}, step {i}: {m}")
