"""The fused FFM step and forward (``ops.StoreFFM``, csrc/cuda/ops_ffm.cu) against ``ffm_reference_step`` /
``ffm_reference_forward`` (float64): at every backward instantiation, at the edges of the envelope and with a batch that
wraps the forward's grid; bit-identical runs; one push per distinct key; on three logical ranks of one GPU (peer rows,
replicas, keys in flight); quality on the planted data of the CPU test."""
import pytest
import torch

from multirank import WORLD, Case, on_peer_rows, on_replicas, one_rank_store, while_keys_move
from test_ffm_cpu import QUALITY_MIN_AUC_GAIN, QUALITY_MIN_LOGLOSS_GAIN, base_rate_logloss, train_ffm_quality

gpu = pytest.mark.gpu
ETA, LAM = 0.2, 1e-3
U = 2.0 ** -24


def _table(n, F, k, g):
    """libffm-like rows: w small, V ~ U[0, 1/sqrt(k)], accumulators in [1, 2)"""
    E = 4 + F * k
    t = torch.zeros(n, 2 * E, dtype=torch.float64)
    t[:, 0] = torch.randn(n, generator=g, dtype=torch.float64) * 0.1
    t[:, 4:E] = torch.rand(n, F * k, generator=g, dtype=torch.float64) / k ** 0.5
    t[:, E:] = 1.0 + torch.rand(n, E, generator=g, dtype=torch.float64)
    return t.float().double()


def _batch(F, per_field, B, g):
    """ids [B, F] skewed towards the small ids of each field (the hottest keys have runs over many tiles), labels"""
    local = (per_field * torch.rand(B, F, generator=g, dtype=torch.float64) ** 3).long().clamp_max(per_field - 1)
    ids = local + torch.arange(F) * per_field
    return ids, (torch.rand(B, generator=g) < 0.5).float()


def _rule(table, batches, k, r):
    """the batches applied in order by the float64 rule; returns (rows, losses, logits of the first batch)"""
    from adapm_b200.ops import ffm_reference_forward, ffm_reference_step

    n, L = table.shape
    with one_rank_store(L, n, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        logits = ffm_reference_forward(kv, batches[0][0], k, r)
        losses = [ffm_reference_step(kv, ids, y, k, ETA, LAM, r) for ids, y in batches]
        rows = torch.empty(n * L, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, L), losses, logits


def _fused(table, batches, F, k, r):
    """(rows, losses, logits of the first batch, stats) after the fused steps on a fresh one-GPU store"""
    from adapm_b200.ops import StoreFFM

    n, L = table.shape
    with one_rank_store(L, n, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.float().contiguous().view(-1)))
        kv.waitall()
        torch.cuda.synchronize()
        op = StoreFFM(s, F, k, ETA, LAM, r)
        dev = s.device
        logits = op.forward(batches[0][0].to(dev)).double().cpu()
        losses = [op.step(ids.to(dev), y.to(dev)) for ids, y in batches]
        torch.cuda.synchronize()
        rows = torch.empty(n * L)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, L).double(), [float(x) for x in losses], logits, op.stats.tolist()


def _tolerances(F, k, batches):
    """fp32 error bounds from the summation lengths, with gamma_n = n 2^-24: phi is a sum of L_phi = F + k F (F - 1) / 2
    terms, all >= 0 but the small w, so its error is at most 2 gamma_(L_phi) |phi|; a key's gradient adds L_G
    occurrences, each through its example's phi, so an update -eta G / sqrt(acc + G^2) (acc >= 1) is off by at most
    eta * 4 gamma_(L_phi + L_G) per step, and an accumulator acc + G^2 by that share of its size. Returns (update
    tolerance, relative accumulator tolerance, relative logit tolerance)."""
    L_phi = F + k * F * (F - 1) // 2
    L_G = max(int(torch.unique(ids, return_counts=True)[1].max()) for ids, _ in batches)
    gamma = 4 * (L_phi + L_G + 16) * U * len(batches)
    return ETA * gamma, gamma, 2 * L_phi * U


# (F, k, B, ids per field): each backward instantiation VPL = ceil((1 + F k / 4) / 32), the envelope's edges (F = 2,
# F = 64, k = 32, F k = 512) and a batch that wraps the forward's grid (F = 2: 16 CTAs per SM, 132 SMs)
CASES = [(2, 4, 5000, 40), (24, 4, 512, 60), (39, 4, 512, 60), (39, 8, 256, 60), (32, 12, 256, 60), (64, 8, 128, 30),
         (16, 32, 256, 40)]


@gpu
@pytest.mark.parametrize("F,k,B,per_field", CASES)
def test_step_and_forward_match_float64_rule(F, k, B, per_field):
    g = torch.Generator().manual_seed(F * 100 + k)
    r = 1.0 / F
    table = _table(F * per_field, F, k, g)
    batches = [_batch(F, per_field, B, g) for _ in range(2)]
    rows, losses, logits, stats = _fused(table, batches, F, k, r)
    ref, ref_losses, ref_logits = _rule(table, batches, k, r)
    tol_v, tol_a, rel_phi = _tolerances(F, k, batches)
    tol_phi = rel_phi * max(1.0, float(ref_logits.abs().max()))
    E = 4 + F * k
    hot = int(torch.unique(batches[0][0], return_counts=True)[1].max())
    print(f"F {F} k {k} B {B}: hottest key {hot} occurrences; tolerances {tol_phi:.2e} {tol_v:.2e} {tol_a:.2e}; "
          f"errors {float((logits - ref_logits).abs().max()):.2e} {float((rows[:, :E] - ref[:, :E]).abs().max()):.2e} "
          f"{float(((rows[:, E:] - ref[:, E:]) / ref[:, E:]).abs().max()):.2e}")
    if B > 1024:
        assert hot > 8 * 32                                  # the finish pass adds partials of many tiles
    torch.testing.assert_close(logits, ref_logits, rtol=0, atol=tol_phi)
    torch.testing.assert_close(rows[:, :E], ref[:, :E], rtol=0, atol=tol_v)
    torch.testing.assert_close(rows[:, E:], ref[:, E:], rtol=tol_a, atol=0)
    for x, y in zip(losses, ref_losses):
        assert abs(x - y) <= B * (tol_phi + 1e-6) + 2 * B * U * abs(y), (x, y)   # + gamma_B of the sum over examples
    distinct = sum(int(torch.unique(ids).numel()) for ids, _ in batches)
    assert stats[3] == distinct                              # one push per distinct key and step
    assert stats[0] == 3 * B * F + distinct and stats[1] == 0 and stats[2] == 0, stats


@gpu
def test_two_runs_are_bit_identical():
    F, k, B, per_field = 39, 4, 4096, 50
    g = torch.Generator().manual_seed(77)
    table = _table(F * per_field, F, k, g)
    batches = [_batch(F, per_field, B, g) for _ in range(3)]
    a = _fused(table, batches, F, k, 1.0 / F)
    b = _fused(table, batches, F, k, 1.0 / F)
    assert torch.equal(a[0], b[0]) and a[1] == b[1] and torch.equal(a[2], b[2])


@gpu
def test_step_arguments_are_checked():
    from adapm_b200.ops import StoreFFM

    F, k = 4, 4
    with one_rank_store(2 * (4 + F * k), 64, "cuda", "float32") as (s, kv):
        dev = s.device
        op = StoreFFM(s, F, k)
        ids, y = torch.zeros(8, F, dtype=torch.int64, device=dev), torch.zeros(8, device=dev)
        for a, b, err in ((ids.cpu(), y, TypeError), (ids.int(), y, TypeError), (ids, y.cpu(), TypeError),
                          (ids, y.double(), TypeError), (ids[:, :3], y, ValueError), (ids, y[:4], ValueError)):
            with pytest.raises(err):
                op.step(a, b)
        with pytest.raises(TypeError):
            op.forward(ids.float())
        for kw in (dict(k=8), dict(num_fields=3), dict(eta=-1.0), dict(lam=-1.0)):
            with pytest.raises(ValueError):
                StoreFFM(s, **(dict(num_fields=F, k=k) | kw))


@gpu
def test_quality_on_planted_data_passes_the_cpu_threshold():
    ll, auc = train_ffm_quality("cuda")
    ll_lin, auc_lin = train_ffm_quality("cuda", pair_scale=0.0)
    base = base_rate_logloss()
    print(f"GPU FFM logloss {ll:.4f} auc {auc:.4f}; linear auc {auc_lin:.4f}; base rate {base:.4f}")
    assert auc >= auc_lin + QUALITY_MIN_AUC_GAIN and ll <= base - QUALITY_MIN_LOGLOSS_GAIN


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
F3, K3, PF3 = 8, 8, 40


def _case(table):
    """one StoreFFM step per batch; a step returns its loss"""
    def open_ffm(server, kv):
        from adapm_b200.ops import StoreFFM

        op = StoreFFM(server, F3, K3, ETA, LAM, 1.0 / F3)
        dev = server.device

        def step(b):
            ids, y = b
            return float(op.step(ids.to(dev), y.to(dev)))

        step.totals = lambda: (None, op.stats.tolist())
        return step

    n = table.shape[0]
    return Case(table.shape[1], n, [(torch.arange(n), table)], lambda b: torch.unique(b[0]), open_ffm)


@gpu
def test_step_on_peer_rows():
    """key k is owned by rank k % 3: two in three rows of every step live on a peer; the ranks step in turn"""
    g = torch.Generator().manual_seed(5)
    table = _table(F3 * PF3, F3, K3, g)
    batches = [_batch(F3, PF3, 256, g) for _ in range(WORLD)]
    res = on_peer_rows(_case(table), batches, in_turns=True)
    ref, ref_losses, _ = _rule(table, batches, K3, 1.0 / F3)
    tol_v, tol_a, _ = _tolerances(F3, K3, batches)
    E = 4 + F3 * K3
    rows = res[0]["rows"][0].double()
    assert sum(x["stats"][3] for x in res) == sum(int(torch.unique(i).numel()) for i, _ in batches)
    assert sum(x["stats"][1] for x in res) > 0
    torch.testing.assert_close(rows[:, :E], ref[:, :E], rtol=0, atol=tol_v)
    torch.testing.assert_close(rows[:, E:], ref[:, E:], rtol=tol_a, atol=0)
    torch.testing.assert_close(sum(x["outs"][0] for x in res), sum(ref_losses), rtol=1e-4, atol=1e-3)


@gpu
def test_step_on_replicas():
    """``replication_only``: after the intents every rank's batch rows are local, most of them replicas; the ranks
    step in turn with a propagation round between them, and every rank reads the three steps applied in order"""
    g = torch.Generator().manual_seed(21)
    table = _table(F3 * PF3, F3, K3, g)
    batches = [_batch(F3, PF3, 128, g) for _ in range(WORLD)]
    res = on_replicas(_case(table), batches)
    assert sum(x["counters"]["replica_setups"] for x in res) > 0
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    ref, _, _ = _rule(table, batches, K3, 1.0 / F3)
    tol_v, tol_a, _ = _tolerances(F3, K3, batches)
    E = 4 + F3 * K3
    for k in range(WORLD):
        out = res[k]
        rows = out["rows"][0].double()
        assert out["local"] and out["replicas"] > 0, f"rank {k}: batch keys not local after the intents"
        torch.testing.assert_close(rows[:, :E], ref[:, :E], rtol=0, atol=tol_v)
        torch.testing.assert_close(rows[:, E:], ref[:, E:], rtol=tol_a, atol=0)
        assert out["stats"][1] == 0 and out["stats"][2] == 0, (k, out["stats"])


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_step_loses_no_update_while_keys_move(technique):
    """ranks 0 and 1 keep relocating every key (and, with ``all``, may replicate it); rank 2 runs 24 steps"""
    g = torch.Generator().manual_seed(9)
    table = _table(F3 * PF3, F3, K3, g)
    batches = [_batch(F3, PF3, 64, g) for _ in range(24)]
    res = while_keys_move(_case(table), batches, technique)
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(x["counters"]["protocol_errors"] == 0 for x in res), info
    ref, ref_losses, _ = _rule(table, batches, K3, 1.0 / F3)
    tol_v, tol_a, _ = _tolerances(F3, K3, batches)
    E = 4 + F3 * K3
    rows = out["rows"][0].double()
    assert out["stats"][3] == sum(int(torch.unique(i).numel()) for i, _ in batches), info
    torch.testing.assert_close(rows[:, :E], ref[:, :E], rtol=0, atol=tol_v)
    torch.testing.assert_close(rows[:, E:], ref[:, E:], rtol=tol_a, atol=0)
    torch.testing.assert_close(sum(out["outs"]), sum(ref_losses), rtol=1e-4, atol=1e-3)
