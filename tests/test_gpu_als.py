"""Alternating least squares on the H100: ``ops.als_solve`` and ``ops.als_gram`` against float64 (backward error of the
solve, element-wise error of the Gram matrix), bit-identical runs and target orders, other-side rows on peers, on
replicas and in flight on three logical ranks of one GPU, a full ALS epoch on three ranks, and the model's quality and
monotone objective on planted data."""
import functools

import pytest
import torch

from harness import run_cluster
from multirank import WORLD, Case, on_peer_rows, on_replicas, one_rank_store, while_keys_move
from test_als_cpu import ALS_QUALITY_MIN_RATIO, train_als_quality

gpu = pytest.mark.gpu
U = 2.0 ** -24
LAM = 0.1


def _problem(rank, counts, no, g, implicit):
    """targets are keys [0, nt), other-side rows keys [nt, nt + no); target t has counts[t] entries (repeats included);
    other-side factors of N(0, 1 / rank); returns (table fp32 [nt + no, 2 rank], targets, offsets, others, a, b).
    The targets' factors start at 0: the pushed difference is then the solution itself, so the row holds exactly what
    the kernel solved (from a non-zero start, w_old + (x - w_old) rounds at the scale of w_old)."""
    nt = len(counts)
    table = torch.randn(nt + no, 2 * rank, generator=g) / rank ** 0.5
    table[:nt, :rank] = 0.0
    table[:, rank:] = torch.rand(nt + no, rank, generator=g)
    offsets = torch.zeros(nt + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(counts, dtype=torch.int64), 0)
    nnz = int(offsets[-1])
    others = nt + torch.randint(0, no, (nnz,), generator=g)
    x = torch.randint(1, 5, (nnz,), generator=g).float()
    if implicit:
        a, b = 2.0 * x, 1.0 + 2.0 * x
    else:
        a, b = torch.ones(nnz), x - 2.5
    return table, torch.arange(nt), offsets, others, a, b


def _fused(table, rank, targets, offsets, others, a, b, implicit, order=None, gram_keys=None):
    """runs als_gram (implicit) and als_solve on a one-GPU store; returns (rows fp32, G or None, stats)"""
    from adapm_b200.ops import als_gram, als_solve

    n = table.shape[0]
    with one_rank_store(2 * rank, n, "cuda", "float32") as (s, kv):
        dev = s.device
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        G = als_gram(s, gram_keys.to(dev), rank) if implicit else None
        t, off, o, aa, bb = targets, offsets, others, a, b
        if order is not None:                  # the same targets in another order (each keeps its entries)
            cnt = offsets[1:] - offsets[:-1]
            idx = torch.cat([torch.arange(int(offsets[i]), int(offsets[i + 1])) for i in order.tolist()])
            t, o, aa, bb = targets[order], others[idx], a[idx], b[idx]
            off = torch.zeros_like(offsets)
            off[1:] = torch.cumsum(cnt[order], 0)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        als_solve(s, *(v.to(dev).contiguous() for v in (t, off, o, aa, bb)), rank, LAM, G, stats)
        torch.cuda.synchronize()
        rows = torch.empty(n * 2 * rank)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * rank), (G.cpu() if G is not None else None), stats.tolist()


def _normal_equations(table, rank, t, offsets, others, a, b, G):
    """A_64, r_64 of target t in float64 from the fp32 rows (and the fp32 G the kernel was given)"""
    e0, e1 = int(offsets[t]), int(offsets[t + 1])
    H = table[others[e0:e1], :rank].double()
    A = LAM * torch.eye(rank, dtype=torch.float64) + (H.t() * a[e0:e1].double()) @ H
    if G is not None:
        A += G.double()
    return A, (b[e0:e1].double().unsqueeze(1) * H).sum(0)


CASES = [pytest.param(r, imp, id=f"{r}-{'implicit' if imp else 'explicit'}") for r in (4, 64, 128) for imp in (False, True)]


@gpu
@pytest.mark.parametrize("rank,implicit", CASES)
def test_solve_matches_float64_rule(rank, implicit):
    """Entry counts 0, 1, rank - 1 and 5 003 (the chunk loop runs many times); normwise backward error of every target
    within 4 (rank + n_t) 2^-24, the AdaGrad half untouched, bit-identical runs and target orders."""
    g = torch.Generator().manual_seed(rank * 3 + implicit)
    counts = [5003, 0, 1, rank - 1, 0, 7, rank - 1, 1]
    no = 6000
    table, targets, offsets, others, a, b = _problem(rank, counts, no, g, implicit)
    gram_keys = torch.arange(len(counts), len(counts) + no)
    rows, G, stats = _fused(table, rank, targets, offsets, others, a, b, implicit, gram_keys=gram_keys)
    nt = len(counts)
    assert stats[3] == nt and stats[2] == 0 and stats[0] == int(offsets[-1]), stats
    worst = 0.0
    for t in range(nt):
        n_t = counts[t]
        if n_t == 0:                                   # r = 0: the row becomes exactly 0
            assert torch.equal(rows[t, :rank], torch.zeros(rank))
            continue
        A, r = _normal_equations(table, rank, t, offsets, others, a, b, G)
        x = rows[t, :rank].double()
        be = float(torch.linalg.norm(A @ x - r) / (torch.linalg.matrix_norm(A, 2) * torch.linalg.norm(x)
                                                   + torch.linalg.norm(r)))
        worst = max(worst, be / (4 * (rank + n_t) * U))
        assert be <= 4 * (rank + n_t) * U, (t, n_t, be)
    print(f"rank {rank} implicit {implicit}: max backward error / bound {worst:.4f}")
    torch.testing.assert_close(rows[:, rank:], table[:, rank:], rtol=0, atol=0)          # AdaGrad half untouched
    torch.testing.assert_close(rows[nt:], table[nt:], rtol=0, atol=0)                    # the other side untouched
    if implicit:
        H = table[nt:, :rank].double()
        G64 = H.t() @ H
        bound = 2 * no * U * (H.abs().t() @ H.abs())
        assert bool(((G.double() - G64).abs() <= bound).all())
        assert torch.equal(G, G.t())
    rows2, G2, _ = _fused(table, rank, targets, offsets, others, a, b, implicit, gram_keys=gram_keys)
    assert torch.equal(rows, rows2) and (G is None or torch.equal(G, G2))
    perm = torch.randperm(nt, generator=g)
    rows3, _, _ = _fused(table, rank, targets, offsets, others, a, b, implicit, order=perm, gram_keys=gram_keys)
    assert torch.equal(rows, rows3)


@gpu
def test_gram_is_bit_identical_and_matches_float64_over_many_partials():
    from adapm_b200.ops import als_gram

    rank, n = 36, 5000                                        # 5 partials of 1 024 keys, the last one partial
    g = torch.Generator().manual_seed(4)
    table = torch.randn(n, 2 * rank, generator=g)
    with one_rank_store(2 * rank, n, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        keys = torch.randperm(n, generator=g).to(s.device)
        G1, G2 = als_gram(s, keys, rank), als_gram(s, keys, rank)
    assert torch.equal(G1, G2)
    H = table[:, :rank].double()
    assert bool(((G1.cpu().double() - H.t() @ H).abs() <= 2 * n * U * (H.abs().t() @ H.abs())).all())


@gpu
def test_solve_arguments_are_checked():
    from adapm_b200.ops import als_solve

    with one_rank_store(16, 64, "cuda", "float32") as (s, kv):
        d = s.device
        t = torch.tensor([0, 1], device=d)
        off = torch.tensor([0, 1, 2], device=d)
        o = torch.tensor([10, 11], device=d)
        one = torch.ones(2, device=d)
        bad = [dict(rank=6), dict(rank=132), dict(lam=0.0), dict(a=-one), dict(t=torch.tensor([0, 0], device=d)),
               dict(off=torch.tensor([0, 2, 1], device=d)), dict(off=torch.tensor([1, 1, 2], device=d)),
               dict(gram=torch.zeros(4, 4, device=d))]
        for kw in bad:
            args = dict(t=t, off=off, o=o, a=one, b=one, rank=8, lam=0.1, gram=None) | kw
            with pytest.raises(ValueError):
                als_solve(s, args["t"], args["off"], args["o"], args["a"], args["b"], args["rank"], args["lam"],
                          args["gram"])
        with pytest.raises(TypeError):
            als_solve(s, t.int(), off, o, one, one, 8, 0.1)


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
def _reference(table, rank, targets, offsets, others, a, b, G):
    """the float64 rule on a CPU store holding the fp32 rows"""
    from adapm_b200.ops import als_reference_solve

    n = table.shape[0]
    with one_rank_store(2 * rank, n, "cpu", "float64") as (_, kv):
        kv.wait(kv.set(torch.arange(n), table.double().contiguous().view(-1)))
        als_reference_solve(kv, targets, offsets, others, a, b, rank, LAM, G)
        rows = torch.empty(n * 2 * rank, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * rank)


def _check_rows(rows, ref, rank, nt):
    """fp32 solve against the float64 rule: well-conditioned problems (lam and the entries keep A away from singular)"""
    torch.testing.assert_close(rows[:nt, :rank].double(), ref[:nt, :rank], rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(rows[nt:].double(), ref[nt:], rtol=0, atol=0)


def _multi_problem(seed, rank=64, nt=60, no=900):
    g = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, 200, (nt,), generator=g).tolist()
    counts[0] = 3000
    return _problem(rank, counts, no, g, implicit=False)


def _case(table, rank):
    """a batch is a problem (table, targets, offsets, others, a, b): one als_solve without Gram matrix"""
    def open_solver(server, kv):
        from adapm_b200.ops import als_solve

        dev = server.device
        stats = torch.zeros(4, dtype=torch.int64, device=dev)

        def step(prob):
            als_solve(server, *(v.to(dev).contiguous() for v in prob[1:]), rank, LAM, None, stats)

        step.totals = lambda: (None, stats.tolist())
        return step

    n = table.shape[0]
    return Case(2 * rank, n, [(torch.arange(n), table)], lambda prob: torch.unique(torch.cat([prob[1], prob[3]])),
                open_solver)


@gpu
def test_solve_reads_other_side_rows_on_peers():
    rank = 64
    prob = _multi_problem(5, rank)
    # only rank 1 solves; key k lives on rank k % 3: two thirds of the rows are peer rows
    res = on_peer_rows(_case(prob[0], rank), [None, prob, None], in_turns=True)
    stats = res[1]["stats"]
    nt = prob[1].numel()
    assert stats[1] > 0 and stats[0] + stats[1] + stats[2] == int(prob[2][-1]) and stats[3] == nt, stats
    _check_rows(res[0]["rows"][0], _reference(*prob[:1], rank, *prob[1:], None), rank, nt)


@gpu
def test_solve_on_replicated_rows():
    rank = 64
    prob = _multi_problem(7, rank)
    case = _case(prob[0], rank)
    # every rank wants every row, so most become replicas; only rank 2 solves
    res = on_replicas(case, [None, None, prob], intent_keys=case.keys_of(prob))
    assert sum(x["counters"]["replica_setups"] for x in res) > 0
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    out = res[2]
    assert out["local"] and out["replicas"] > 0
    s = out["stats"]
    assert s[0] == int(prob[2][-1]) and s[1] == 0 and s[2] == 0 and s[3] == prob[1].numel(), s
    ref = _reference(*prob[:1], rank, *prob[1:], None)
    for k in range(WORLD):
        _check_rows(res[k]["rows"][0], ref, rank, prob[1].numel())


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_solve_loses_no_update_while_keys_move(technique):
    """Ranks 0 and 1 keep relocating every key; rank 2 runs 12 half-steps that alternate the two sides, so every
    solve reads the rows the previous one wrote. The result is the 12 half-steps applied in order. About 60 entries per
    user and 50 per item at rank 16 keep every system well conditioned, so fp32 stays close to the float64 rule."""
    rank, nu, ni = 16, 60, 80
    g = torch.Generator().manual_seed(9)
    table = torch.randn(nu + ni, 2 * rank, generator=g) / rank ** 0.5
    table[:, rank:] = 0.0
    ii = torch.randint(0, nu, (4000,), generator=g)
    jj = torch.randint(0, ni, (4000,), generator=g)
    x = torch.randint(1, 5, (4000,), generator=g).float()

    def side(t_idx, o_idx, first_t, first_o, n_t):
        order = torch.argsort(t_idx, stable=True)
        cnt = torch.bincount(t_idx, minlength=n_t)
        off = torch.zeros(n_t + 1, dtype=torch.int64)
        off[1:] = torch.cumsum(cnt, 0)
        return (None, torch.arange(n_t) + first_t, off, o_idx[order] + first_o, torch.ones(4000), x[order])

    halves = [side(ii, jj, 0, nu, nu), side(jj, ii, nu, 0, ni)] * 6
    probs = [(table,) + h[1:] for h in halves]
    res = while_keys_move(_case(table, rank), probs, technique)
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(x["counters"]["protocol_errors"] == 0 for x in res), info
    assert out["stats"][3] == 6 * (nu + ni), info
    # the float64 rule, half-step by half-step, from the same start
    from adapm_b200.ops import als_reference_solve

    with one_rank_store(2 * rank, nu + ni, "cpu", "float64") as (_, kv):
        kv.wait(kv.set(torch.arange(nu + ni), table.double().contiguous().view(-1)))
        for h in halves:
            als_reference_solve(kv, *h[1:], rank, LAM)
        ref = torch.empty((nu + ni) * 2 * rank, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(nu + ni), ref))
    torch.testing.assert_close(out["rows"][0].double(), ref.view(nu + ni, 2 * rank), rtol=2e-3, atol=2e-4)


# ---------------------------------------------------------------------------------------------- the model
def _epoch_worker(kv, server, wid, q):
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    rank, world = server.my_rank(), server.num_servers()
    data, _ = SparseMatrix.synthetic_implicit(q["users"], q["items"], q["per_row"], q["rank_true"], world, rank,
                                              seed=q["seed"])
    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"], algorithm="als", loss="implicit",
                   lam=q["lam"], alpha=q["alpha"])
    model = MatrixFactorization(server, kv, cfg, data)
    model.init_model()
    kv.barrier()
    objs = [server.allreduce_sum([model.run_epoch(0)])[0]]    # warm-up: the row and column intents take effect
    torch.cuda.synchronize()
    model.stats.zero_()
    objs += [server.allreduce_sum([model.run_epoch(e)])[0] for e in (1, 2)]
    stats = model.stats.tolist()
    kv.wait_sync()
    kv.barrier()
    fck = cfg.first_col_key(world)
    lo, hi = data.row_block()
    clo, chi = data.col_block()
    mine = list(range(lo, hi)) + [k + fck for k in range(clo, chi)]
    owned = all(server.owner_of(k) == rank for k in mine)
    out = {"stats": stats, "objs": objs, "owned": owned}
    if rank == 0:
        W, H = model.pull_factors()
        out["W"], out["H"] = W.clone(), H.clone()
    kv.barrier()
    kv.finalize()
    return out


@gpu
def test_als_epoch_on_three_ranks_is_local_and_bit_identical():
    from adapm_b200.models.mf import MFConfig
    from test_als_cpu import ALS_QUALITY

    q = dict(ALS_QUALITY, users=900, items=600)
    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"])
    runs = []
    for _ in range(2):
        res = run_cluster(functools.partial(_epoch_worker, q=q), world=WORLD, workers=1, mode="threads",
                          value_lengths=cfg.row_len, num_keys=cfg.num_keys(WORLD), dtype="float32", backend="cuda")
        assert all(x["counters"]["protocol_errors"] == 0 for x in res.values())
        for k in range(WORLD):
            out = res[k][0]
            s = out["stats"]
            assert s[2] == 0 and s[3] > 0, (k, s)                       # no slow-path rows after warm-up
            assert out["owned"], k                                      # every target is owned here: local pushes
            assert out["objs"][2] <= out["objs"][1] * (1 + 1e-5) and out["objs"][1] <= out["objs"][0] * (1 + 1e-5)
        runs.append(res[0][0])
    assert torch.equal(runs[0]["W"], runs[1]["W"]) and torch.equal(runs[0]["H"], runs[1]["H"])


@gpu
def test_fused_als_quality_and_monotone_objective_on_planted_data():
    rec, ndcg, pop, objs = train_als_quality("cuda")
    print(f"fused ALS recall@10 {rec:.4f} ndcg@10 {ndcg:.4f}, popularity {pop:.4f}; objective per half-step {objs}")
    assert rec >= ALS_QUALITY_MIN_RATIO * pop, (rec, pop)
    assert all(b <= a * (1 + 1e-5) for a, b in zip(objs, objs[1:])), objs
