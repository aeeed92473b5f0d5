"""RotatE on the H100: the fused step (``ops.kge_rotate_step``) against the float64 rule ``rotate_reference_step``, the
complex-metric distance kernels (``ops.gather_dist_rank_count`` / ``gather_dist_topk`` with ``p="complex"``) against a
float64 oracle, both on three logical ranks of one GPU (peer rows, replicas, keys in flight), and the model's quality on
the FB15k-237 toy set."""
import numpy as np
import pytest
import torch

from harness import WRAP, wrap_calls
from multirank import (WORLD, Case, Fused, on_peer_rows, on_replicas, one_rank_store, reads_while_keys_move,
                       rejected_on_ranks, while_keys_move)
from test_gpu_transe import _check_rank, _check_topk, _dist_inputs

gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5


def _lens(ne, nr, d):
    return torch.tensor([2 * d] * ne + [d] * nr, dtype=torch.int64)


def _init_table(ne, nr, d, g):
    """flat float64 rows: entities [z | acc] (2 d), relations [phases | acc] (d)"""
    e = torch.randn(ne, 2 * d, generator=g, dtype=torch.float64) * 0.3
    e[:, d:] = torch.rand(ne, d, generator=g, dtype=torch.float64) * 0.5 + 1e-3
    r = (torch.rand(nr, d, generator=g, dtype=torch.float64) * 2 - 1) * np.pi
    r[:, d // 2:] = torch.rand(nr, d // 2, generator=g, dtype=torch.float64) * 0.5 + 1e-3
    return torch.cat([e.reshape(-1), r.reshape(-1)])


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
            neg[1, nn - 1] = subj[1]            # a negative equal to the positive's subject
    return subj, rel, obj, neg


def _rule(table, ne, nr, batches, d, gamma, alpha, eta, ge):
    """batches applied one after another by the float64 rule on a float64 CPU store; returns (rows, loss, pushes)"""
    from adapm_b200.ops import rotate_reference_step

    with one_rank_store(_lens(ne, nr, d), ne + nr, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(ne + nr), table.contiguous()))
        loss, pushes = 0.0, 0
        for b in batches:
            l, u = rotate_reference_step(kv, *b, d, gamma, alpha, eta, ge)
            loss += l; pushes += u
        rows = torch.empty(table.numel(), dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne + nr), rows))
        return rows, loss, pushes


def _fused(table, ne, nr, batches, d, gamma, alpha, eta, ge, deterministic):
    """the same on a one-GPU store; returns (rows, loss, stats, kernel launches)"""
    from adapm_b200 import _C
    from adapm_b200.ops import kge_rotate_step

    with one_rank_store(_lens(ne, nr, d), ne + nr, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(ne + nr), table.float().contiguous()))
        dev = s.device
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        l0 = _C.kernel_launches()
        for b in batches:
            kge_rotate_step(s, *(t.to(dev).contiguous() for t in b), d, gamma, alpha, eta, ge, loss, stats,
                            deterministic=deterministic)
        torch.cuda.synchronize()
        launches = _C.kernel_launches() - l0
        rows = torch.empty(table.numel(), dtype=torch.float32)
        kv.wait(kv.pull(torch.arange(ne + nr), rows))
        return rows.double(), float(loss.item()), stats.tolist(), launches


# (d, 2n): float4 per lane (VPL) 1, 2, 4, 3, 3; 2n = 2 is the fewest negatives the step takes
SHAPES = [(8, 12), (152, 256), (512, 64), (264, 2), (384, 64)]


def _cases(B):
    """SHAPES with B triples crossed with alpha, and one case whose triples wrap the kernel's resident grid"""
    return ([pytest.param(d, nn, a, B, id=f"{d}-{nn}-{a}") for a in (0.0, 1.0) for d, nn in SHAPES]
            + [pytest.param(8, 12, 1.0, WRAP, id="8-12-1.0-wrap")])


@gpu
@pytest.mark.parametrize("d,nn,alpha,B", _cases(64))
def test_deterministic_step_matches_float64_rule(d, nn, alpha, B):
    """Repeated keys in every role, one entity in the first 64 triples, negatives equal to the positive's rows; two
    steps."""
    B = wrap_calls(B, 4)
    ne, nr = max(300, 2 * B), max(20, B // 16)
    g = torch.Generator().manual_seed(d * 7 + nn + int(alpha))
    table = _init_table(ne, nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, hot=True) for _ in range(2)]
    args = (d, 0.3 * d, alpha, 0.05, 0.01)          # gamma near the typical distance
    ref, ref_loss, ref_pushes = _rule(table, ne, nr, batches, *args)
    rows, loss, stats, launches = _fused(table, ne, nr, batches, *args, deterministic=True)
    assert launches == 3 * len(batches)                  # index, step, apply
    assert stats[3] == ref_pushes == 2 * B * (3 + nn) and stats[2] == 0, (stats, ref_pushes)
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss), (loss, ref_loss)
    rows2, loss2, _, _ = _fused(table, ne, nr, batches, *args, deterministic=True)
    assert torch.equal(rows, rows2) and loss == loss2     # bit-identical runs


@gpu
@pytest.mark.parametrize("d,nn,alpha,B", _cases(60))
def test_inplace_step_matches_rule_on_distinct_keys(d, nn, alpha, B):
    B = wrap_calls(B, 4)
    nr, ne = max(200, B), B * (2 + nn) + 100
    g = torch.Generator().manual_seed(d * 11 + nn + int(alpha))
    table = _init_table(ne, nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(2)]
    args = (d, 0.3 * d, alpha, 0.05, 0.01)          # gamma near the typical distance
    ref, ref_loss, ref_pushes = _rule(table, ne, nr, batches, *args)
    rows, loss, stats, launches = _fused(table, ne, nr, batches, *args, deterministic=False)
    assert launches == len(batches)
    assert stats[3] == ref_pushes and stats[0] == len(batches) * B * (3 + nn), stats
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss)


@gpu
def test_deterministic_step_rejected_on_several_ranks():
    from adapm_b200.ops import kge_rotate_step

    def call(server):
        dev = server.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        kge_rotate_step(server, k, k + 10, k, torch.zeros(2, 4, dtype=torch.int64, device=dev), 8, 2.0, 1.0, 0.1, 0.0,
                        torch.zeros(1, device=dev), deterministic=True)

    assert rejected_on_ranks(call)


# ---------------------------------------------------------------------------------------------- distance kernels
def _dist_oracle(q, E):
    """float64 complex-metric distances [M, N] (NaN rows stay NaN)"""
    from adapm_b200.ops import complex_dist

    return complex_dist(q.double(), E.double())


@gpu
def test_complex_distance_kernels_match_float64_oracle():
    from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk

    M, N, d = 70, 1000, 152                          # N is not a multiple of the 64-column tile
    g = torch.Generator().manual_seed(31)
    rows, q, keys, true_col, (off, cols), excluded = _dist_inputs(M, N, d, g)
    with one_rank_store(_lens(N + 3, 0, d // 2), N + 3, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(N + 3), rows.contiguous().view(-1)))
        dev = s.device
        qd, kd, td, ex = q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev))
        stats = torch.zeros(3, dtype=torch.int64, device=dev)
        raw, filt = gather_dist_rank_count(s, qd, kd, d, "complex", False, td, ex, stats=stats)
        raw2, filt2 = gather_dist_rank_count(s, qd, kd, d, "complex", False, td, ex)
        assert torch.equal(raw, raw2) and torch.equal(filt, filt2)
        assert stats.tolist()[2] == 0
        D = _dist_oracle(q, rows[keys])
        _check_rank(raw.cpu(), filt.cpu(), D, true_col, excluded)
        for k in (1, 10, 64):
            vals, idx = gather_dist_topk(s, qd, kd, d, k, "complex", False, exclude=ex)
            vals2, idx2 = gather_dist_topk(s, qd, kd, d, k, "complex", False, exclude=ex)
            assert torch.equal(vals, vals2) and torch.equal(idx, idx2)
            _check_topk(vals.cpu(), idx.cpu(), D, k, excluded)
        qo = torch.empty(M * d + 1, device=dev)[1:].view(M, d)                     # a view 4 bytes off 16-byte alignment
        qo.copy_(qd)
        assert qo.is_contiguous() and qo.data_ptr() % 16
        assert all(torch.equal(a, b) for a, b in
                   zip(gather_dist_rank_count(s, qo, kd, d, "complex", False, td, ex), (raw, filt)))
        vals, idx = gather_dist_topk(s, qd, kd[:20], d, 64, "complex", False)     # fewer columns than k: padding
        assert bool((idx[:, 19:] == -1).all()) and bool((vals[:, 19:] == float("-inf")).all())
        assert not bool((idx[:, :19] == 0).any())                                   # column 0 is the NaN row


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
def _case(table, ne, nr, d, ge):
    """RotatE steps at gamma 6, alpha 1 and eta 0.05 with L2 weight ``ge``"""
    from adapm_b200.ops import kge_rotate_step

    def step(server, b, loss, stats):
        dev = server.device
        kge_rotate_step(server, *(t.to(dev).contiguous() for t in b), d, 6.0, 1.0, 0.05, ge, loss, stats)

    return Case(_lens(ne, nr, d), ne + nr, [(torch.arange(ne + nr), table)],
                lambda b: torch.unique(torch.cat([t.reshape(-1) for t in b])), lambda server, kv: Fused(server, step))


@gpu
def test_step_on_peer_rows():
    """Key k is owned by rank k % 3, so two in three rows of every rank's step live on a peer; each rank runs one step
    in turn; the result is the three steps applied in rank order."""
    ne, nr, B, nn, d = 3000, 90, 60, 12, 152
    g = torch.Generator().manual_seed(5)
    table = _init_table(ne, nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(WORLD)]
    res = on_peer_rows(_case(table, ne, nr, d, 0.0), batches, in_turns=True)
    ref, ref_loss, ref_pushes = _rule(table, ne, nr, batches, d, 6.0, 1.0, 0.05, 0.0)
    assert sum(r["stats"][3] for r in res) == ref_pushes
    assert sum(r["stats"][1] for r in res) > 0       # peer rows were read
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(sum(r["loss"] for r in res), ref_loss, rtol=1e-4, atol=1e-3)


@gpu
def test_step_on_replicas():
    """``replication_only``: the three ranks' batches overlap (keys distinct within a rank); after every rank declared
    intent for its batch, all its rows are local, most of them replicas. Ranks 0, 1, 2 then run one step each with a
    propagation round between them; every rank must read the three steps applied in that order."""
    B, nn, d = 40, 12, 152
    ne, nr = 2 * B * (2 + nn), 2 * B
    g = torch.Generator().manual_seed(23)
    table = _init_table(ne, nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(WORLD)]
    res = on_replicas(_case(table, ne, nr, d, 0.01), batches)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    args = (d, 6.0, 1.0, 0.05, 0.01)
    ref, _, _ = _rule(table, ne, nr, batches, *args)
    for r in range(WORLD):
        out = res[r]
        assert out["local"] and out["replicas"] > 0, f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"rows read on rank {r}: {m}")
        _, before_loss, before_pushes = _rule(table, ne, nr, batches[:r], *args) if r else (None, 0.0, 0)
        _, upto_loss, upto_pushes = _rule(table, ne, nr, batches[:r + 1], *args)
        s = out["stats"]
        assert s[0] == B * (3 + nn) and s[1] == 0 and s[2] == 0 and s[3] == upto_pushes - before_pushes, (r, s)
        torch.testing.assert_close(out["loss"], upto_loss - before_loss, rtol=1e-4, atol=1e-3)


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_step_loses_no_update_while_keys_move(technique):
    """Ranks 0 and 1 keep relocating every key (and, with ``all``, may replicate it); rank 2 runs 32 steps (keys
    distinct within a step)."""
    ne, nr, B, nn, d = 448, 48, 16, 12, 64
    g = torch.Generator().manual_seed(9)
    table = _init_table(ne, nr, d, g)
    batches = [_batch(ne, nr, B, nn, g, distinct=True) for _ in range(32)]
    res = while_keys_move(_case(table, ne, nr, d, 0.0), batches, technique)
    out = res[2]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(r["counters"]["protocol_errors"] == 0 for r in res), info
    ref, ref_loss, ref_pushes = _rule(table, ne, nr, batches, d, 6.0, 1.0, 0.05, 0.0)
    assert out["stats"][3] == ref_pushes, info
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(out["loss"], ref_loss, rtol=1e-4, atol=1e-3)


DK, DD, DM = 1 << 15, 152, 64


def _dist_all(server, q, keys, true_col, ex, stats=None):
    from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk

    out = {"rank": gather_dist_rank_count(server, q, keys, DD, "complex", False, true_col, ex, stats=stats)}
    for k in (1, 10, 64):
        out[f"top{k}"] = gather_dist_topk(server, q, keys, DD, k, "complex", False, exclude=ex, stats=stats)
    return out


def _dist_mr_inputs():
    g = torch.Generator().manual_seed(78)
    rows, q, keys, true_col, ex, _ = _dist_inputs(DM, DK - 3, DD, g)
    return rows, q, keys, true_col, ex


@gpu
def test_complex_distance_kernels_bit_identical_while_keys_move():
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
def test_fused_rotate_quality_on_fb15k237_toy():
    """The fused deterministic step and the fused complex-distance evaluation on the toy set, with the settings of the
    CPU test (test_rotate_cpu.GOLDEN_SETTINGS: d 152, gamma 9, alpha 0). Measured on an H100: filtered test MRR 0.562
    (object side 0.600, subject side 0.525), Hits@10 0.855; the thresholds are 0.05 below."""
    from test_rotate_cpu import _golden_rotate_cfg, train_golden

    ev, fused = train_golden("cuda", _golden_rotate_cfg(deterministic=True))
    print("RotatE toy test (GPU):", ev, fused)
    assert abs(ev["mrr"] - fused["mrr"]) < 1e-9
    assert fused["mrr"] >= GPU_MRR - 0.05 and fused["hits@10"] >= GPU_HITS10 - 0.05, fused


GPU_MRR, GPU_HITS10 = 0.562, 0.855
