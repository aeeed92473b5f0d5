"""TransE on the H100: the fused step (``ops.kge_transe_step``) against the float64 rule ``transe_reference_step``, the
distance kernels (``ops.gather_dist_rank_count`` / ``gather_dist_topk``) against a float64 ``cdist`` oracle, both on
three logical ranks of one GPU (peer rows, replicas, keys in flight), and the model's quality on the FB15k-237 toy set."""
import os

import pytest
import torch

from harness import WRAP, wrap_calls
from multirank import (WORLD, Case, Fused, on_peer_rows, on_replicas, one_rank_store, reads_while_keys_move,
                       rejected_on_ranks, while_keys_move)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kge_fb15k237_toy")
gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5


def _init_table(num_keys, d, g):
    t = torch.randn(num_keys, 2 * d, generator=g, dtype=torch.float64) * 0.3
    t[:, d:] = torch.rand(num_keys, d, generator=g, dtype=torch.float64) * 0.5 + 1e-3
    return t


def _batch(ne, nr, B, nn, g, distinct=False, hot=False):
    """(subj, rel keys, obj, neg [B, nn]); distinct: no key twice in the step; hot: entity 0 is in each of the first
    64 triples"""
    if distinct:
        e = torch.randperm(ne, generator=g)[:B * (2 + nn)]
        subj, obj, neg = e[:B], e[B:2 * B], e[2 * B:].view(B, nn)
        rel = ne + torch.randperm(nr, generator=g)[:B]
    else:
        subj, obj = torch.randint(0, ne, (B,), generator=g), torch.randint(0, ne, (B,), generator=g)
        rel = ne + torch.randint(0, nr, (B,), generator=g)
        neg = torch.randint(0, ne, (B, nn), generator=g)
        if hot:
            subj[:64:2] = 0; obj[1:64:2] = 0
            neg[0, 0] = obj[0]                  # a negative equal to the positive's object
    return subj, rel, obj, neg


def _rule(table, batches, d, p, margin, eta, ge, gr):
    """batches applied one after another by the float64 rule on a float64 CPU store; returns (rows, loss, pushes)"""
    from adapm_b200.ops import transe_reference_step

    n = table.shape[0]
    with one_rank_store(2 * d, n, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        loss, pushes = 0.0, 0
        for b in batches:
            l, u = transe_reference_step(kv, *b, d, p, margin, eta, ge, gr)
            loss += l; pushes += u
        rows = torch.empty(n * 2 * d, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * d), loss, pushes


def _fused(table, batches, d, p, margin, eta, ge, gr, deterministic):
    """the same on a one-GPU store; returns (rows, loss, stats, kernel launches)"""
    from adapm_b200 import _C
    from adapm_b200.ops import kge_transe_step

    n = table.shape[0]
    with one_rank_store(2 * d, n, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.float().contiguous().view(-1)))
        dev = s.device
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        l0 = _C.kernel_launches()
        for b in batches:
            kge_transe_step(s, *(t.to(dev).contiguous() for t in b), d, p, margin, eta, ge, gr, loss, stats,
                            deterministic=deterministic)
        torch.cuda.synchronize()
        launches = _C.kernel_launches() - l0
        rows = torch.empty(n * 2 * d, dtype=torch.float32)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * d).double(), float(loss.item()), stats.tolist(), launches


def _cases(B, wrap_d, wrap_p):
    """d 4, 152, 260, 384 and 512 (4 float4 per lane: VPL 1 to 4) with B triples, crossed with p; and one (wrap_d,
    wrap_p) case whose triples wrap the kernel's resident grid"""
    return ([pytest.param(d, p, B, id=f"{d}-{p}") for p in (1, 2) for d in (4, 152, 260, 384, 512)]
            + [pytest.param(wrap_d, wrap_p, WRAP, id=f"{wrap_d}-{wrap_p}-wrap")])


@gpu
@pytest.mark.parametrize("d,p,B", _cases(64, 64, 1))
def test_deterministic_step_matches_float64_rule(d, p, B):
    """Repeated keys in every role, one entity in the first 64 triples, a negative equal to the positive; two steps."""
    B = wrap_calls(B, 4)
    ne, nr, nn = max(300, 2 * B), max(20, B // 16), 12
    g = torch.Generator().manual_seed(d * 7 + p)
    table = _init_table(ne + nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, hot=True) for _ in range(2)]
    args = (d, p, 1.0 if p == 1 else 0.02, 0.05, 0.01, 0.02)   # margins with active and inactive pairs
    ref, ref_loss, ref_pushes = _rule(table, batches, *args)
    rows, loss, stats, launches = _fused(table, batches, *args, deterministic=True)
    assert launches == 3 * len(batches)                  # index, step, apply
    assert stats[3] == ref_pushes and stats[2] == 0, (stats, ref_pushes)
    assert 3 * B * 2 < ref_pushes < B * 2 * (3 + nn)     # active and inactive pairs
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss), (loss, ref_loss)
    rows2, loss2, _, _ = _fused(table, batches, *args, deterministic=True)
    assert torch.equal(rows, rows2) and loss == loss2     # bit-identical runs


@gpu
@pytest.mark.parametrize("d,p,B", _cases(150, 64, 2))
def test_inplace_step_matches_rule_on_distinct_keys(d, p, B):
    B, nn = wrap_calls(B, 4), 12
    ne, nr = max(4000, B * (2 + nn)), max(200, B)
    g = torch.Generator().manual_seed(d * 11 + p)
    table = _init_table(ne + nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(2)]
    args = (d, p, 1.0, 0.05, 0.01, 0.02)
    ref, ref_loss, ref_pushes = _rule(table, batches, *args)
    rows, loss, stats, launches = _fused(table, batches, *args, deterministic=False)
    assert launches == len(batches)
    assert stats[3] == ref_pushes and stats[0] == len(batches) * B * (3 + nn), stats
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss)


@gpu
def test_deterministic_step_rejected_on_several_ranks():
    from adapm_b200.ops import kge_transe_step

    def call(server):
        dev = server.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        kge_transe_step(server, k, k + 10, k, torch.zeros(2, 4, dtype=torch.int64, device=dev), 8, 1, 1.0, 0.1, 0.0,
                        0.0, torch.zeros(1, device=dev), deterministic=True)

    assert rejected_on_ranks(call)


# ---------------------------------------------------------------------------------------------- distance kernels
def _dist_oracle(q, E, p, normalize):
    """float64 distances [M, N] of the rule (NaN rows stay NaN)"""
    E = E.double()
    if normalize:
        E = E / E.norm(dim=1, keepdim=True).clamp(min=1e-12)
    return torch.cdist(q.double(), E, p=float(p))


def _tol(D):
    """fp32 summation error bound of a distance (|D| * dim * 2^-23, generous)"""
    return 1e-5 * (1 + D.abs())


def _check_rank(raw, filt, D, true_col, excluded):
    dt = D.gather(1, true_col.view(-1, 1))
    for i in range(D.shape[0]):
        row, t = D[i], dt[i]
        close = (row - t).abs() <= _tol(t)
        strict = (row < t - _tol(t))
        strict[true_col[i]] = False; close[true_col[i]] = False
        lo, hi = int(strict.sum()), int((strict | close).sum())
        assert lo <= int(raw[i]) <= hi, (i, int(raw[i]), lo, hi)
        ex = excluded[i]
        lo_f, hi_f = int((strict & ~ex).sum()), int(((strict | close) & ~ex).sum())
        assert lo_f <= int(filt[i]) <= hi_f, (i, int(filt[i]), lo_f, hi_f)


def _check_topk(vals, idx, D, k, excluded):
    for i in range(D.shape[0]):
        ok = ~torch.isnan(D[i]) & ~excluded[i]
        cand = torch.nonzero(ok).view(-1)
        got = idx[i][idx[i] >= 0]
        assert got.numel() == min(k, cand.numel())
        assert not bool(excluded[i][got].any()) and not bool(torch.isnan(D[i][got]).any())
        torch.testing.assert_close(-vals[i][:got.numel()].double(), D[i][got], rtol=1e-5, atol=1e-5)
        if got.numel() < k:
            assert bool((idx[i][got.numel():] == -1).all()) and bool(torch.isinf(vals[i][got.numel():]).all())
        if cand.numel() > got.numel():       # the k-th selected is no farther than anything left out, up to fp32
            rest = torch.ones(D.shape[1], dtype=torch.bool); rest[got] = False
            rest &= ok
            worst = D[i][got].max()
            assert float(D[i][rest].min()) >= float(worst) - float(_tol(worst))
        d_got = -vals[i][:got.numel()]
        assert bool((d_got[1:] >= d_got[:-1]).all())                            # nearest first
        same = d_got[1:] == d_got[:-1]
        assert bool((got[1:][same] > got[:-1][same]).all())                     # ties to the smaller column


def _dist_inputs(M, N, d, g):
    rows = torch.randn(N + 3, d, generator=g)
    rows[5] = float("nan")                           # a NaN row: never counted, never selected
    rows[7] = rows[8]                                # two equal rows: a tie
    q = torch.randn(M, d, generator=g) * 0.5
    keys = torch.randperm(N + 3, generator=g)[:N]
    keys[:3] = torch.tensor([5, 7, 8])
    true_col = torch.randint(0, N, (M,), generator=g)
    true_col[0] = 1                                 # the true column is a tie partner
    counts = torch.randint(0, 8, (M,), generator=g)
    off = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)])
    cols = torch.cat([torch.sort(torch.randperm(N, generator=g)[:int(c)]).values for c in counts])
    excluded = torch.zeros(M, N, dtype=torch.bool)
    excluded[torch.repeat_interleave(torch.arange(M), counts), cols] = True
    return rows, q, keys, true_col, (off, cols), excluded


@gpu
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("p", [1, 2])
def test_distance_kernels_match_float64_cdist(p, normalize):
    from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk

    M, N, d = 70, 1000, 152                          # N is not a multiple of the 64-column tile
    g = torch.Generator().manual_seed(p * 2 + normalize)
    rows, q, keys, true_col, (off, cols), excluded = _dist_inputs(M, N, d, g)
    with one_rank_store(d, N + 3, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(N + 3), rows.contiguous().view(-1)))
        dev = s.device
        qd, kd, td, ex = q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev))
        stats = torch.zeros(3, dtype=torch.int64, device=dev)
        raw, filt = gather_dist_rank_count(s, qd, kd, d, p, normalize, td, ex, stats=stats)
        raw2, filt2 = gather_dist_rank_count(s, qd, kd, d, p, normalize, td, ex)
        assert torch.equal(raw, raw2) and torch.equal(filt, filt2)
        assert stats.tolist()[2] == 0
        D = _dist_oracle(q, rows[keys], p, normalize)
        _check_rank(raw.cpu(), filt.cpu(), D, true_col, excluded)
        for k in (1, 10, 64):
            vals, idx = gather_dist_topk(s, qd, kd, d, k, p, normalize, exclude=ex)
            vals2, idx2 = gather_dist_topk(s, qd, kd, d, k, p, normalize, exclude=ex)
            assert torch.equal(vals, vals2) and torch.equal(idx, idx2)
            _check_topk(vals.cpu(), idx.cpu(), D, k, excluded)
        qo = torch.empty(M * d + 1, device=dev)[1:].view(M, d)                     # a view 4 bytes off 16-byte alignment
        qo.copy_(qd)
        assert qo.is_contiguous() and qo.data_ptr() % 16
        assert all(torch.equal(a, b) for a, b in zip(gather_dist_rank_count(s, qo, kd, d, p, normalize, td, ex), (raw, filt)))
        assert all(torch.equal(a, b) for a, b in zip(gather_dist_topk(s, qo, kd, d, 10, p, normalize, exclude=ex),
                                                     gather_dist_topk(s, qd, kd, d, 10, p, normalize, exclude=ex)))
        vals, idx = gather_dist_topk(s, qd, kd[:20], d, 64, p, normalize)         # fewer columns than k: padding
        assert bool((idx[:, 19:] == -1).all()) and bool((vals[:, 19:] == float("-inf")).all())


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
def _case(table, d, p, ge, gr):
    """TransE steps at margin 1 and eta 0.05 with L2 weights ``ge``, ``gr``"""
    from adapm_b200.ops import kge_transe_step

    def step(server, b, loss, stats):
        dev = server.device
        kge_transe_step(server, *(t.to(dev).contiguous() for t in b), d, p, 1.0, 0.05, ge, gr, loss, stats)

    n = table.shape[0]
    return Case(2 * d, n, [(torch.arange(n), table)], lambda b: torch.unique(torch.cat([t.reshape(-1) for t in b])),
                lambda server, kv: Fused(server, step))


@gpu
def test_step_on_peer_rows():
    """Key k is owned by rank k % 3, so two in three rows of every rank's step live on a peer; each rank runs one step
    in turn; the result is the three steps applied in rank order."""
    ne, nr, B, nn, d, p = 3000, 90, 60, 12, 152, 1
    g = torch.Generator().manual_seed(5)
    table = _init_table(ne + nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(WORLD)]
    res = on_peer_rows(_case(table, d, p, 0.0, 0.0), batches, in_turns=True)
    ref, ref_loss, ref_pushes = _rule(table, batches, d, p, 1.0, 0.05, 0.0, 0.0)
    assert sum(r["stats"][3] for r in res) == ref_pushes
    assert sum(r["stats"][1] for r in res) > 0       # peer rows were read
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(sum(r["loss"] for r in res), ref_loss, rtol=1e-4, atol=1e-3)


@gpu
@pytest.mark.parametrize("p", [1, 2])
def test_step_on_replicas(p):
    """``replication_only``: the three ranks' batches overlap (keys distinct within a rank); after every rank declared
    intent for its batch, all its rows are local, most of them replicas (a push sets the replica's dirty byte). Ranks
    0, 1, 2 then run one step each with a propagation round between them; every rank must read the three steps applied
    in that order."""
    B, nn, d = 40, 12, 152
    ne, nr = 2 * B * (2 + nn), 2 * B
    g = torch.Generator().manual_seed(21 + p)
    table = _init_table(ne + nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(WORLD)]
    res = on_replicas(_case(table, d, p, 0.01, 0.02), batches)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    args = (d, p, 1.0, 0.05, 0.01, 0.02)
    ref, _, _ = _rule(table, batches, *args)
    for r in range(WORLD):
        out = res[r]
        assert out["local"] and out["replicas"] > 0, f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"rows read on rank {r}: {m}")
        _, before_loss, before_pushes = _rule(table, batches[:r], *args) if r else (None, 0.0, 0)
        _, upto_loss, upto_pushes = _rule(table, batches[:r + 1], *args)
        s = out["stats"]
        assert s[0] == B * (3 + nn) and s[1] == 0 and s[2] == 0 and s[3] == upto_pushes - before_pushes, (r, s)
        torch.testing.assert_close(out["loss"], upto_loss - before_loss, rtol=1e-4, atol=1e-3)


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_step_loses_no_update_while_keys_move(technique):
    """Ranks 0 and 1 keep relocating every key (and, with ``all``, may replicate it); rank 2 runs 32 steps (keys
    distinct within a step)."""
    ne, nr, B, nn, d, p = 448, 48, 16, 12, 64, 2
    g = torch.Generator().manual_seed(9)
    table = _init_table(ne + nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(32)]
    res = while_keys_move(_case(table, d, p, 0.0, 0.0), batches, technique)
    out = res[2]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(r["counters"]["protocol_errors"] == 0 for r in res), info
    ref, ref_loss, ref_pushes = _rule(table, batches, d, p, 1.0, 0.05, 0.0, 0.0)
    assert out["stats"][3] == ref_pushes, info
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(out["loss"], ref_loss, rtol=1e-4, atol=1e-3)


DK, DD, DM = 1 << 15, 152, 64


def _dist_all(server, q, keys, true_col, ex, stats=None):
    from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk

    out = {}
    for p, norm in ((1, True), (2, False)):
        out[f"rank{p}"] = gather_dist_rank_count(server, q, keys, DD, p, norm, true_col, ex, stats=stats)
        for k in (1, 10, 64):
            out[f"top{k}_{p}"] = gather_dist_topk(server, q, keys, DD, k, p, norm, exclude=ex, stats=stats)
    return out


def _dist_mr_inputs():
    g = torch.Generator().manual_seed(77)
    rows, q, keys, true_col, ex, _ = _dist_inputs(DM, DK - 3, DD, g)
    return rows, q, keys, true_col, ex


@gpu
def test_distance_kernels_bit_identical_while_keys_move():
    rows, q, keys, true_col, (off, cols) = _dist_mr_inputs()
    with one_rank_store(DD, DK, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(DK), rows.contiguous().view(-1)))
        dev = s.device
        exp = _dist_all(s, q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev)))
        exp = {k: tuple(t.cpu() for t in v) for k, v in exp.items()}

    def read(server, kv, stats):
        dev = server.device
        args = (q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev)))
        return lambda: _dist_all(server, *args, stats=stats)

    res = reads_while_keys_move(Case(DD, DK, [(torch.arange(DK), rows)]), read, exp, torch.arange(0, DK, 8),
                                "relocation_only")
    out = res[2]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{out['reps']} repetitions, stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert not out["mism"], f"{info}; mismatches: {sorted({k for _, k in out['mism']})}"
    assert out["stats"][2] == 0, info


# ---------------------------------------------------------------------------------------------- quality
@gpu
def test_fused_transe_quality_on_fb15k237_toy():
    """The fused step and the fused distance evaluation reach the CPU test's thresholds (published: MRR 0.60,
    Hits@10 84.86 %) with TransE L1, d = 152, eta 0.1, margin 3, neg_ratio 6, gamma 0, 12 epochs of 70 triples."""
    from adapm_b200.models.kge import KGE, KGEConfig, evaluate_fused, load_triples

    tr, va, te = (load_triples(os.path.join(GOLDEN, f"{n}.del")) for n in ("train", "valid", "test"))
    cfg = KGEConfig(num_entities=280, num_relations=112, embed_dim=152, algorithm="TransE", p_norm=1, margin=3.0,
                    eta=0.1, neg_ratio=6, gamma_entity=0.0, gamma_relation=0.0, batch_triples=70, deterministic=True)
    with one_rank_store(cfg.value_lengths(), cfg.num_keys, "cuda", "float32") as (server, kv):
        model = KGE(server, kv, cfg)
        model.init_model()
        for epoch in range(1, 13):
            perm = tr[torch.randperm(tr.shape[0], generator=torch.Generator().manual_seed(epoch * 977))]
            for s in range(0, perm.shape[0], cfg.batch_triples):
                model.step(perm[s:s + cfg.batch_triples])
                kv.advance_clock()
        torch.cuda.synchronize()
        known = torch.cat([tr, va, te])
        ev = evaluate_fused(model, te, known)
        full = model.evaluate(te, known)
        idx, vals = model.predict(te[:8, 0], te[:8, 1], "object", k=10, known=known)
    print("TransE toy test (GPU):", ev)
    assert ev["mrr"] >= 0.50 and ev["hits@10"] >= 0.80, ev
    assert abs(full["mrr"] - ev["mrr"]) < 1e-9
    assert idx.shape == (8, 10) and bool((vals[:, :-1] >= vals[:, 1:]).all())
