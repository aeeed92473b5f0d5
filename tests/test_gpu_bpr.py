"""Implicit-feedback matrix factorisation on the H100: the fused BPR step (``ops.mf_bpr_step``) against the float64 rule
``bpr_reference_step`` on one GPU and on three logical ranks of one GPU (peer rows, replicas, keys in flight),
``MatrixFactorization.recommend`` against ``topk_reference``, and the model's quality on planted data."""
import functools

import numpy as np
import pytest
import torch

from harness import WRAP, run_cluster, wrap_calls
from multirank import (WORLD, Case, Fused, on_peer_rows, on_replicas, one_rank_store, reads_while_keys_move,
                       rejected_on_ranks, while_keys_move)
from test_bpr_cpu import QUALITY_MIN_RATIO, train_quality

gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5
EPS, LAM = 0.05, 0.02


def _init_table(num_keys, r, g):
    t = torch.randn(num_keys, 2 * r, generator=g, dtype=torch.float64) * (1.0 / r ** 0.5)
    t[:, r:] = torch.rand(num_keys, r, generator=g, dtype=torch.float64) * 0.5 + 1e-3
    return t


def _batch(nu, ni, B, n, g, distinct=False, hot=False):
    """(user keys, positive item keys, negative item keys [B, n]); users are keys [0, nu), items [nu, nu + ni).
    distinct: no key twice in the step; hot: user 0 and item nu in each of the first 64 positives, a negative equal to its
    positive and a negative repeated within one positive"""
    if distinct:
        users = torch.randperm(nu, generator=g)[:B]
        it = nu + torch.randperm(ni, generator=g)[:B * (1 + n)]
        pos, neg = it[:B], it[B:].view(B, n)
    else:
        users = torch.randint(0, nu, (B,), generator=g)
        pos = nu + torch.randint(0, ni, (B,), generator=g)
        neg = nu + torch.randint(0, ni, (B, n), generator=g)
        if hot:
            users[:64:2] = 0
            pos[1:64:2] = nu
            neg[0, 0] = pos[0]
            if n > 1:
                neg[1, 1] = neg[1, 0]
    return users, pos, neg


def _rule(table, batches, r):
    from adapm_b200.ops import bpr_reference_step

    n = table.shape[0]
    with one_rank_store(2 * r, n, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        loss, pushes = 0.0, 0
        for b in batches:
            l, u = bpr_reference_step(kv, *b, r, EPS, LAM)
            loss += l; pushes += u
        rows = torch.empty(n * 2 * r, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * r), loss, pushes


def _fused(table, batches, r, deterministic):
    from adapm_b200 import _C
    from adapm_b200.ops import mf_bpr_step

    n = table.shape[0]
    with one_rank_store(2 * r, n, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.float().contiguous().view(-1)))
        dev = s.device
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        l0 = _C.kernel_launches()
        for b in batches:
            mf_bpr_step(s, *(t.to(dev).contiguous() for t in b), r, EPS, LAM, loss, stats, deterministic=deterministic)
        torch.cuda.synchronize()
        launches = _C.kernel_launches() - l0
        rows = torch.empty(n * 2 * r, dtype=torch.float32)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * r).double(), float(loss.item()), stats.tolist(), launches


RANKS = (4, 128, 132, 256, 260, 384, 512)       # VPL 1, 1, 2, 2, 3, 3, 4; 132 and 260 end in a partial float4 row


def _det_cases():
    return ([pytest.param(r, n, 64, id=f"{r}-{n}") for r in RANKS for n in (1, 12)]
            + [pytest.param(r, 256, 64, id=f"{r}-256") for r in (4, 260, 512)]
            + [pytest.param(128, 12, WRAP, id="128-12-wrap")])


@gpu
@pytest.mark.parametrize("rank,n,B", _det_cases())
def test_deterministic_step_matches_float64_rule(rank, n, B):
    """Repeated users, a hot item, a negative equal to its positive, a repeated negative; two steps."""
    B = wrap_calls(B, 4)
    nu, ni = max(40, B // 4), max(300, B)
    g = torch.Generator().manual_seed(rank * 7 + n)
    table = _init_table(nu + ni, rank, g)
    batches = [_batch(nu, ni, B, n, g, hot=True) for _ in range(2)]
    ref, ref_loss, ref_pushes = _rule(table, batches, rank)
    rows, loss, stats, launches = _fused(table, batches, rank, deterministic=True)
    assert launches == 3 * len(batches)                  # index, step, apply
    assert stats[3] == ref_pushes == len(batches) * B * (2 + n) and stats[2] == 0, (stats, ref_pushes)
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss), (loss, ref_loss)
    rows2, loss2, _, _ = _fused(table, batches, rank, deterministic=True)
    assert torch.equal(rows, rows2) and loss == loss2     # bit-identical runs


@gpu
@pytest.mark.parametrize("rank,n,B", [pytest.param(r, 12, 150, id=f"{r}") for r in RANKS]
                         + [pytest.param(4, 1, WRAP, id="4-1-wrap")])
def test_inplace_step_matches_rule_on_distinct_keys(rank, n, B):
    B = wrap_calls(B, 4)
    nu, ni = B, B * (1 + n)
    g = torch.Generator().manual_seed(rank * 11 + n)
    table = _init_table(nu + ni, rank, g)
    batches = [_batch(nu, ni, B, n, g, distinct=True) for _ in range(2)]
    ref, ref_loss, ref_pushes = _rule(table, batches, rank)
    rows, loss, stats, launches = _fused(table, batches, rank, deterministic=False)
    assert launches == len(batches)
    assert stats[3] == ref_pushes and stats[0] == len(batches) * B * (2 + n) and stats[2] == 0, stats
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss)


@gpu
def test_step_arguments_are_checked():
    from adapm_b200.ops import mf_bpr_step

    with one_rank_store(16, 64, "cuda", "float32") as (s, kv):
        dev = s.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        loss = torch.zeros(1, device=dev)
        for rank, neg in ((6, torch.zeros(2, 1)), (8, torch.zeros(2, 0)), (8, torch.zeros(2, 257)), (516, torch.zeros(2, 1)),
                          (8, torch.zeros(3, 1))):
            with pytest.raises(ValueError):
                mf_bpr_step(s, k, k + 1, neg.long().to(dev), rank, 0.1, 0.0, loss)
        with pytest.raises(TypeError):
            mf_bpr_step(s, k.int(), k + 1, torch.zeros(2, 1, dtype=torch.int64, device=dev), 8, 0.1, 0.0, loss)


@gpu
def test_deterministic_step_rejected_on_several_ranks():
    from adapm_b200.ops import mf_bpr_step

    def call(server):
        dev = server.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        mf_bpr_step(server, k, k + 1, torch.ones(2, 3, dtype=torch.int64, device=dev), 8, 0.1, 0.0,
                    torch.zeros(1, device=dev), deterministic=True)

    assert rejected_on_ranks(call)


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
def _case(table, r):
    from adapm_b200.ops import mf_bpr_step

    def step(server, b, loss, stats):
        dev = server.device
        mf_bpr_step(server, *(t.to(dev).contiguous() for t in b), r, EPS, LAM, loss, stats)

    n = table.shape[0]
    return Case(2 * r, n, [(torch.arange(n), table)], lambda b: torch.unique(torch.cat([t.reshape(-1) for t in b])),
                lambda server, kv: Fused(server, step))


@gpu
def test_step_on_peer_rows():
    """Key k is owned by rank k % 3, so two in three rows of every rank's step live on a peer; each rank runs one step
    in turn; the result is the three steps applied in rank order."""
    nu, ni, B, n, r = 600, 3000, 60, 12, 132
    g = torch.Generator().manual_seed(5)
    table = _init_table(nu + ni, r, g)
    batches = [_batch(nu, ni, B, n, g, distinct=True) for _ in range(WORLD)]
    res = on_peer_rows(_case(table, r), batches, in_turns=True)
    ref, ref_loss, ref_pushes = _rule(table, batches, r)
    assert sum(x["stats"][3] for x in res) == ref_pushes
    assert sum(x["stats"][1] for x in res) > 0       # peer rows were read
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(sum(x["loss"] for x in res), ref_loss, rtol=1e-4, atol=1e-3)


@gpu
def test_step_on_replicas():
    """``replication_only``: the three ranks' batches overlap (keys distinct within a rank); after every rank declared
    intent for its batch, all its rows are local, most of them replicas. Ranks 0, 1, 2 then run one step each with a
    propagation round between them; every rank must read the three steps applied in that order."""
    B, n, r = 40, 12, 128
    nu, ni = 2 * B, 2 * B * (1 + n)
    g = torch.Generator().manual_seed(21)
    table = _init_table(nu + ni, r, g)
    batches = [_batch(nu, ni, B, n, g, distinct=True) for _ in range(WORLD)]
    res = on_replicas(_case(table, r), batches)
    assert sum(x["counters"]["replica_setups"] for x in res) > 0
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    ref, _, _ = _rule(table, batches, r)
    for k in range(WORLD):
        out = res[k]
        assert out["local"] and out["replicas"] > 0, f"rank {k}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL,
                                   msg=lambda m: f"rows read on rank {k}: {m}")
        s = out["stats"]
        assert s[0] == B * (2 + n) and s[1] == 0 and s[2] == 0 and s[3] == B * (2 + n), (k, s)


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_step_loses_no_update_while_keys_move(technique):
    """Ranks 0 and 1 keep relocating every key (and, with ``all``, may replicate it); rank 2 runs 32 steps (keys
    distinct within a step)."""
    nu, ni, B, n, r = 64, 448, 16, 12, 64
    g = torch.Generator().manual_seed(9)
    table = _init_table(nu + ni, r, g)
    batches = [_batch(nu, ni, B, n, g, distinct=True) for _ in range(32)]
    res = while_keys_move(_case(table, r), batches, technique)
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(x["counters"]["protocol_errors"] == 0 for x in res), info
    ref, ref_loss, ref_pushes = _rule(table, batches, r)
    assert out["stats"][3] == ref_pushes == 32 * B * (2 + n), info
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(out["loss"], ref_loss, rtol=1e-4, atol=1e-3)


# ---------------------------------------------------------------------------------------------- recommend
def _rec_model(server, kv, W, H, data):
    from adapm_b200.models.mf import MatrixFactorization, MFConfig

    m, r = W.shape
    cfg = MFConfig(num_rows=m, num_cols=H.shape[0], rank=r, loss="bpr")
    return MatrixFactorization(server, kv, cfg, data)


def _rec_inputs(g, m=300, n=1000, r=64):
    """integer factors in [-8, 8]: every score is exact in fp32 (and in bf16 operands), and many tie"""
    from adapm_b200.models.mf import SparseMatrix

    W = torch.randint(-8, 9, (m, r), generator=g).float()
    H = torch.randint(-8, 9, (n, r), generator=g).float()
    H[10] = H[20]                                    # two equal items
    cnt = torch.randint(0, 30, (m,), generator=g)
    cnt[0] = n - 5                                   # a user with fewer than k unseen items
    ii = torch.repeat_interleave(torch.arange(m), cnt).numpy()
    jj = torch.cat([torch.randperm(n, generator=g)[:int(c)] for c in cnt]).numpy()
    data = SparseMatrix(ii, jj, np.ones(ii.shape[0], np.float32), m, n, 1, 0)
    return W, H, data


def _factor_rows(W, H, fck):
    """(keys, rows [m + n, 2 r]) of the factors, items from key ``fck`` on"""
    m, r = W.shape
    rows = torch.zeros(m + H.shape[0], 2 * r)
    rows[:m, :r], rows[m:, :r] = W, H
    return torch.cat([torch.arange(m), torch.arange(H.shape[0]) + fck]), rows


def _load_factors(kv, model, W, H, dev):
    keys, rows = _factor_rows(W, H, model.fck)
    kv.wait(kv.set(keys.to(dev), rows.view(-1).to(dev)))
    kv.waitall()


@gpu
@pytest.mark.parametrize("k", [1, 10, 64])
def test_recommend_matches_topk_reference(k):
    from adapm_b200.ops import topk_reference

    g = torch.Generator().manual_seed(k)
    W, H, data = _rec_inputs(g)
    m, n = W.shape[0], H.shape[0]
    with one_rank_store(2 * W.shape[1], m + n, "cuda", "float32") as (s, kv):
        model = _rec_model(s, kv, W, H, data)
        _load_factors(kv, model, W, H, s.device)
        users = np.arange(m)
        seen = data.seen(users)
        idx, vals = model.recommend(users, k, seen=seen)
        idx2, vals2 = model.recommend(users, k, seen=seen)
        plain_idx, plain_vals = model.recommend(users[:50], k)
    assert torch.equal(idx, idx2) and torch.equal(vals, vals2)
    excluded = torch.zeros(m, n, dtype=torch.bool)
    excluded[torch.repeat_interleave(torch.arange(m), seen[0][1:] - seen[0][:-1]), seen[1]] = True
    scores = (W.double() @ H.double().t()).float()
    rv, ri = topk_reference(scores, k, excluded)
    assert torch.equal(idx.cpu(), ri) and torch.equal(vals.cpu(), rv)
    pv, pi = topk_reference(scores[:50], k)
    assert torch.equal(plain_idx.cpu(), pi) and torch.equal(plain_vals.cpu(), pv)
    if k == 64:
        assert int((idx[0] == -1).sum()) == k - 5


@gpu
def test_recommend_bit_identical_while_keys_move():
    from adapm_b200.models.mf import MFConfig

    g = torch.Generator().manual_seed(31)
    W, H, data = _rec_inputs(g, m=201, n=3000)           # 201 users: the first item key is 201 on 1 and on 3 ranks
    users = np.arange(W.shape[0])
    seen = data.seen(users)
    with one_rank_store(2 * W.shape[1], W.shape[0] + H.shape[0], "cuda", "float32") as (s, kv):
        model = _rec_model(s, kv, W, H, data)
        _load_factors(kv, model, W, H, s.device)
        exp = tuple(t.cpu() for t in model.recommend(users, 10, seen=seen))

    # the data keeps the one-rank partitioning: all users are in rank 2's row block
    def read(server, kv, stats):
        model = _rec_model(server, kv, W, H, data)
        return lambda: {"top10": model.recommend(users, 10, seen=seen)}

    n = W.shape[0] + H.shape[0]
    fck = MFConfig(num_rows=W.shape[0], num_cols=H.shape[0], rank=W.shape[1]).first_col_key(WORLD)
    case = Case(2 * W.shape[1], n, [_factor_rows(W, H, fck)])
    res = reads_while_keys_move(case, read, {"top10": exp}, torch.arange(0, n, 4), "relocation_only")
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    info = f"{out['reps']} repetitions, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert not out["mism"], info


# ---------------------------------------------------------------------------------------------- quality and DSGD
@gpu
def test_fused_bpr_quality_on_planted_data():
    rec, ndcg, pop, rnd = train_quality("cuda", deterministic=True)
    print(f"fused BPR recall@10 {rec:.4f} ndcg@10 {ndcg:.4f}, popularity {pop:.4f}, random {rnd:.4f}")
    assert rec >= QUALITY_MIN_RATIO * pop, (rec, pop)


def _dsgd_worker(kv, server, wid, q):
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    rank, world = server.my_rank(), server.num_servers()
    data, test = SparseMatrix.synthetic_implicit(q["users"], q["items"], q["per_row"], q["rank_true"], world, rank,
                                                 seed=q["seed"])
    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"], algorithm="dsgd", eps=q["eps"],
                   lam=q["lam"], batch_nnz=1024, loss="bpr", num_negatives=q["negatives"], bold_driver=False)
    model = MatrixFactorization(server, kv, cfg, data)
    model.init_model()
    kv.barrier()
    model.run_epoch(0)                                # warm-up: the row and column intents take effect
    torch.cuda.synchronize()
    model.stats.zero_()
    losses = [model.run_epoch(e) for e in range(1, 4)]
    torch.cuda.synchronize()
    stats = model.stats.tolist()
    kv.wait_sync()
    kv.barrier()
    rec = model.evaluate_ranking(*test, k=10)
    kv.barrier()
    kv.finalize()
    return {"stats": stats, "losses": losses, "rec": rec}


@gpu
def test_dsgd_on_three_ranks_has_no_slow_rows_after_warm_up():
    from test_bpr_cpu import QUALITY

    q = dict(QUALITY, users=900, items=600)
    from adapm_b200.models.mf import MFConfig

    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"])
    res = run_cluster(functools.partial(_dsgd_worker, q=q), world=WORLD, workers=1, mode="threads",
                      value_lengths=cfg.row_len, num_keys=cfg.num_keys(WORLD), dtype="float32", backend="cuda")
    for k in range(WORLD):
        out = res[k][0]
        assert out["stats"][2] == 0 and out["stats"][3] > 0, (k, out["stats"])
        assert out["losses"][-1] < out["losses"][0], (k, out["losses"])
    rec = sum(res[k][0]["rec"][0] for k in range(WORLD)) / sum(res[k][0]["rec"][2] for k in range(WORLD))
    assert rec > 0.1, rec
    assert all(x["counters"]["protocol_errors"] == 0 for x in res.values())
