"""The fused kernels on stores with several ranks: rows owned by a peer, local replicas, keys whose relocation is in
flight, and the in-place word2vec step of one GPU.

Every fused op resolves each row to one of four outcomes (``dev::resolve_fast`` in ``pm_kernels.cuh``): a local owned
row, a local replica (the update also sets the dirty byte), a peer's owned row (the update bumps the owner's version) or
none, for a key in a transitional state, which takes the generic out-of-line path. On several GPUs these branches are
the hot path. The scenarios (three logical ranks on one GPU) are the runners of ``multirank.py``; ``Op`` is their case.

Training steps are compared with the float64 rule (``kge_reference_step``, ``mf_reference_step`` and
``sgns_reference_step`` below, applied through a float64 CPU store), gathers bit for bit with the same op on a
one-rank store loaded with the same rows.
"""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from harness import run_cluster
from multirank import (WORLD, Case, Fused, load_rows, make_local, on_peer_rows, on_replicas, one_rank_store, pull_rows,
                       reads_while_keys_move, spread_keys, while_keys_move)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5


# ---------------------------------------------------------------------------------------------- float64 references
def sgns_reference_step(kv, centers, contexts, negatives, d, alpha):
    """One word2vec SGNS step by the rule of the fused kernels, through Pull / Push on ``kv`` (rows ``[emb d | AdaGrad
    d]``): every pair-target reads the state at the start of the step, a negative equal to the pair's context is
    skipped, |f| > 6 saturates, updates of repeated keys add up. Returns the summed logistic loss."""
    B, neg = negatives.shape
    dt = kv.server.dtype
    tk = torch.cat([contexts.view(B, 1), negatives], 1)

    def pull(keys):
        v = torch.empty(keys.numel() * 2 * d, dtype=dt)
        kv.wait(kv.pull(keys.contiguous().view(-1), v))
        return v.view(*keys.shape, 2 * d)

    r0, r1 = pull(centers), pull(tk)
    e0, a0, e1, a1 = r0[:, :d], r0[:, d:], r1[..., :d], r1[..., d:]
    label = torch.zeros(B, neg + 1, dtype=dt)
    label[:, 0] = 1
    f = (e0.unsqueeze(1) * e1).sum(-1)
    g = label - torch.sigmoid(f)
    g = torch.where(f > 6, label - 1, g)
    g = torch.where(f < -6, label, g)
    valid = torch.ones(B, neg + 1, dtype=torch.bool)
    valid[:, 1:] = negatives != contexts.view(B, 1)
    g = g * valid
    g0 = (g.unsqueeze(-1) * e1).sum(1)
    g1 = g.unsqueeze(-1) * e0.unsqueeze(1)
    kv.wait(kv.push(centers.contiguous(), torch.cat([alpha * g0 / torch.sqrt(a0 + g0 * g0), g0 * g0], 1).contiguous().view(-1)))
    upd = torch.cat([alpha * g1 / torch.sqrt(a1 + g1 * g1), g1 * g1], -1)[valid]
    kv.wait(kv.push(tk[valid].contiguous(), upd.contiguous().view(-1)))
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    return float((torch.log1p(torch.exp(-z)) * valid).sum())


class Op:
    """One fused training op at one shape: store layout, batches of distinct keys, the fused call and its reference; with
    ``init`` set, a case of the ``multirank`` runners.

    ``kind``: ``sgns`` (d, neg, impl, B), ``complex`` / ``rescal`` (d = embed_dim, p_e, p_r, n calls) or ``mf`` (d = rank,
    n non-zeros). Entity keys (all keys for sgns / mf) are ``[0, ne)``, relation keys ``[ne, ne + nr)``."""

    def __init__(self, kind, d, neg=0, impl="auto", n=32, p_e=0.0, p_r=0.0, ne=0, nr=0, lr=None):
        self.kind, self.d, self.neg, self.impl, self.n, self.p_e, self.p_r = kind, d, neg, impl, n, p_e, p_r
        self.ne, self.nr = ne, nr
        self.init = None
        self.lr = lr if lr is not None else {"sgns": 0.05, "complex": 0.1, "rescal": 0.1, "mf": 0.05}[kind]

    def __repr__(self):
        return f"{self.kind}(d={self.d}, neg={self.neg}, impl={self.impl}, p={self.p_e}/{self.p_r})"

    def sized(self, ne, nr=0):
        """a copy of this op on a store with ``ne`` entity and ``nr`` relation keys"""
        return Op(self.kind, self.d, self.neg, self.impl, self.n, self.p_e, self.p_r, ne, nr, self.lr)

    # ---- layout
    @property
    def kge(self):
        return self.kind in ("complex", "rescal")

    @property
    def cfg(self):
        from adapm_b200.models.kge import KGEConfig

        return KGEConfig(num_entities=self.ne, num_relations=self.nr, embed_dim=self.d, neg_ratio=1, eta=self.lr,
                         algorithm="ComplEx" if self.kind == "complex" else "RESCAL", dropout_entity=self.p_e,
                         dropout_relation=self.p_r)

    @property
    def ent_len(self):
        return 2 * self.d

    @property
    def rel_len(self):
        return self.cfg.relation_len if self.kge else 2 * self.d

    @property
    def value_lengths(self):
        return self.cfg.value_lengths() if self.kge else 2 * self.d

    @property
    def num_keys(self):
        return self.cfg.num_keys if self.kge else self.ne

    def key_len(self, k):
        return self.rel_len if self.kge and self.ne <= k < self.ne + self.nr else self.ent_len

    def need(self):
        """(entity keys, relation keys) of one batch (all distinct)"""
        if self.kind == "sgns":
            return self.n * (self.neg + 2), 0
        if self.kge:
            return 2 * self.n, self.n
        return 2 * self.n, 0

    def init_rows(self, g):
        """[(keys, float32 rows)] for every key group: embeddings ~ 0.3 N(0, 1), AdaGrad accumulators in (1e-3, 1]"""
        groups = [(torch.arange(self.ne), self.ent_len)]
        if self.kge:
            groups.append((torch.arange(self.ne, self.ne + self.nr), self.rel_len))
        out = []
        for keys, ln in groups:
            h = ln // 2
            rows = torch.cat([torch.randn(keys.numel(), h, generator=g) * 0.3,
                              torch.rand(keys.numel(), h, generator=g) + 1e-3], 1)
            out.append((keys, rows))
        return out

    # ---- batches
    def batch(self, ents, rels, g, seed=0):
        n = self.n
        if self.kind == "sgns":
            return {"centers": ents[:n], "contexts": ents[n:2 * n], "negatives": ents[2 * n:].reshape(n, self.neg)}
        if self.kge:
            return {"S": ents[:n], "O": ents[n:2 * n], "R": rels[:n], "L": (torch.rand(n, generator=g) < 0.3).float(),
                    "seed": seed}
        return {"rk": ents[:n], "ck": ents[n:2 * n], "x": torch.randn(n, generator=g)}

    def keys_of(self, b):
        if self.kind == "sgns":
            return torch.cat([b["centers"], b["contexts"], b["negatives"].reshape(-1)])
        if self.kge:
            return torch.cat([b["S"], b["O"], b["R"]])
        return torch.cat([b["rk"], b["ck"]])

    def without_call(self, b, i):
        keep = torch.arange(self.n) != i
        out = {k: (v[keep] if torch.is_tensor(v) else v) for k, v in b.items()}
        if self.kge and (self.p_e > 0 or self.p_r > 0):
            out["mask_rows"] = keep
        return out

    def updates(self, b):
        """row updates of one batch of distinct keys (stats[3])"""
        return self.keys_of(b).numel()

    def slow_calls(self):
        """calls that take the generic path although all their rows are resolvable (stats[2])"""
        if self.kind == "complex" and self.d % 8:
            return self.n
        if self.kind == "mf" and self.d % 4:
            return self.n
        return 0

    # ---- the fused op and its rule
    def open(self, server, kv):
        return Fused(server, self.fused)

    def fused(self, server, b, loss, stats):
        from adapm_b200.ops import kge_complex_step, kge_rescal_step, mf_step, sgns_step

        dev = server.device
        if self.kind == "sgns":
            sgns_step(server, b["centers"].to(dev), b["contexts"].to(dev), b["negatives"].contiguous().to(dev), self.d,
                      self.lr, loss, stats, impl=self.impl)
        elif self.kge:
            fn = kge_complex_step if self.kind == "complex" else kge_rescal_step
            fn(server, b["S"].to(dev), b["R"].to(dev), b["O"].to(dev), b["L"].to(dev), self.d, self.lr,
               self.cfg.gamma_entity, self.cfg.gamma_relation, loss, stats, self.p_e, self.p_r, b["seed"])
        else:
            ones = torch.ones(self.n, dtype=torch.int32, device=dev)
            mf_step(server, b["rk"].to(dev), b["ck"].to(dev), b["x"].to(dev), ones, ones, self.d, self.lr, 0.02, loss,
                    stats)

    def reference(self, kv, b):
        if self.kind == "sgns":
            return sgns_reference_step(kv, b["centers"], b["contexts"], b["negatives"], self.d, self.lr)
        if self.kge:
            from adapm_b200.models.kge import kge_reference_step
            from adapm_b200.ops import kge_dropout_mask

            masks = None
            if self.p_e > 0 or self.p_r > 0:
                n, el, rl = self.n, self.ent_len // 2, self.rel_len // 2
                masks = (kge_dropout_mask(b["seed"], n, 0, el, self.p_e),
                         kge_dropout_mask(b["seed"], n, 1, rl, self.p_r, relation=True),
                         kge_dropout_mask(b["seed"], n, 2, el, self.p_e))
                if "mask_rows" in b:
                    masks = tuple(m[b["mask_rows"]] for m in masks)
            return kge_reference_step(kv, b["S"], b["R"], b["O"], b["L"], self.cfg, masks=masks)
        from adapm_b200.models.mf import mf_reference_step

        ones = torch.ones(b["rk"].numel(), dtype=torch.int32)
        return mf_reference_step(kv, b["rk"], b["ck"], b["x"], ones, ones, self.d, self.lr, 0.02)


def reference_run(op, init, steps, drop=None, stale=None):
    """Applies ``steps`` (batches) one after another by the float64 rule, from the rows ``init``. Returns (rows per key
    group, summed loss). Negative controls: ``drop = (step, call)`` leaves one call out; ``stale = (step, key)`` lets
    step ``step`` read row ``key`` as it was before step ``step - 1`` (the update of ``step - 1`` to that row itself is
    kept)."""
    with one_rank_store(op.value_lengths, op.num_keys, "cpu", "float64") as (_, kv):
        load_rows(kv, init)
        loss, snap = 0.0, None
        for i, b in enumerate(steps):
            if drop is not None and drop[0] == i:
                b = op.without_call(b, drop[1])
            if stale is not None and stale[0] == i + 1:
                snap = torch.empty(op.key_len(stale[1]), dtype=torch.float64)
                kv.wait(kv.pull(torch.tensor([stale[1]]), snap))
            if stale is not None and stale[0] == i:
                k = torch.tensor([stale[1]])
                cur = torch.empty_like(snap)
                kv.wait(kv.pull(k, cur))
                kv.wait(kv.set(k, snap.clone()))
                loss += op.reference(kv, b)
                new = torch.empty_like(snap)
                kv.wait(kv.pull(k, new))
                kv.wait(kv.set(k, cur + (new - snap)))
            else:
                loss += op.reference(kv, b)
        return pull_rows(kv, init, torch.float64), loss


def _assert_rows(got, ref, what):
    for i, (a, b) in enumerate(zip(got, ref)):
        torch.testing.assert_close(a.double(), b, rtol=RTOL, atol=ATOL, msg=lambda m: f"{what}, key group {i}: {m}")


# ---------------------------------------------------------------------------------------------- 1. peer rows
PEER_OPS = [Op("sgns", 64, 5, "tma", n=64), Op("sgns", 200, 30, "tma", n=64), Op("sgns", 300, 25, "tma", n=64),
            Op("sgns", 336, 3, "tma", n=64), Op("sgns", 128, 5, "ldg", n=64), Op("sgns", 512, 3, "ldg", n=64),
            Op("sgns", 64, 40, "auto", n=64),
            Op("complex", 512), Op("complex", 128), Op("complex", 20),
            Op("rescal", 32), Op("rescal", 12), Op("rescal", 32, p_e=0.25, p_r=0.3), Op("rescal", 12, p_e=0.3, p_r=0.2),
            Op("mf", 128), Op("mf", 64), Op("mf", 10)]


@gpu
@pytest.mark.parametrize("op", PEER_OPS, ids=repr)
def test_fused_steps_on_peer_rows_match_float64_rule(op):
    """Three ranks, no intents: each runs one step on its own keys (distinct, disjoint across ranks, 3 in 4 owned by a
    peer), all at once. The key sets are disjoint, so the order of the ranks does not matter and the rule is exact."""
    ne_need, nr_need = op.need()
    op = op.sized(WORLD * WORLD * ne_need, WORLD * WORLD * nr_need)
    g = torch.Generator().manual_seed(op.d * 7 + op.neg + int(100 * op.p_e))
    op.init = op.init_rows(g)
    batches = [op.batch(spread_keys(r, ne_need, g), op.ne + spread_keys(r, nr_need, g) if nr_need else None, g,
                        seed=0x5EED + r) for r in range(WORLD)]
    res = on_peer_rows(op, batches, in_turns=False)
    ref_rows, ref_loss = reference_run(op, op.init, batches)
    _assert_rows(res[0]["rows"], ref_rows, repr(op))
    for r in range(WORLD):
        out = res[r]
        b = batches[r]
        ref_l = reference_run(op, op.init, [b])[1]
        torch.testing.assert_close(out["loss"], ref_l, rtol=1e-3 if op.kind == "sgns" else 1e-4, atol=1e-3)
        s = out["stats"]
        assert 3 * out["remote"] >= 2 * op.updates(b), out["remote"]
        assert s[3] == op.updates(b) and s[2] == op.slow_calls(), (r, s, op.slow_calls())
        assert s[1] > 0 or op.slow_calls() == op.n, (r, s)     # (the generic path counts no rows)


# ---------------------------------------------------------------------------------------------- 2. replica rows
REPLICA_OPS = [Op("sgns", 300, 25, "tma", n=32), Op("complex", 128), Op("rescal", 32), Op("mf", 64)]


@gpu
@pytest.mark.parametrize("op", REPLICA_OPS, ids=repr)
def test_fused_steps_on_replicas_match_float64_rule(op):
    """``replication_only``, three ranks whose batches overlap (distinct within a rank): after every rank declared
    intent for its batch, all its rows are local (owned or replica). Ranks 0, 1, 2 then run one step each, with a
    propagation round between them; at the end every rank reads every key and must see the three steps applied in
    that order (read-your-writes, convergence)."""
    ne_need, nr_need = op.need()
    op = op.sized(2 * ne_need, 2 * nr_need)
    g = torch.Generator().manual_seed(op.d + 11)
    op.init = op.init_rows(g)
    batches = [op.batch(torch.randperm(op.ne, generator=g)[:ne_need],
                        op.ne + torch.randperm(op.nr, generator=g)[:nr_need] if nr_need else None, g, seed=0x7E + r)
               for r in range(WORLD)]
    res = on_replicas(op, batches)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    ref_rows, _ = reference_run(op, op.init, batches)
    for r in range(WORLD):
        out = res[r]
        assert out["local"], f"rank {r}: batch keys not local after the intents"
        _assert_rows(out["rows"], ref_rows, f"{op}, rows read on rank {r}")
        s = out["stats"]
        n_rows = op.updates(batches[r])
        assert s[0] == n_rows and s[1] == 0 and s[2] == op.slow_calls() and s[3] == n_rows, (r, s)
    # each rank's loss: its step on the state left by the ranks before it
    for r in range(WORLD):
        _, before = reference_run(op, op.init, batches[:r])
        _, upto = reference_run(op, op.init, batches[:r + 1])
        torch.testing.assert_close(res[r]["loss"], upto - before, rtol=1e-3 if op.kind == "sgns" else 1e-4, atol=1e-3)


# ---------------------------------------------------------------------------------------------- 3. keys in flight
INFLIGHT_STEPS = 32
INFLIGHT_OPS = {"sgns": lambda: Op("sgns", 64, 5, "tma", n=32, ne=448),
                "ldg": lambda: Op("sgns", 128, 5, "ldg", n=32, ne=448),
                "complex": lambda: Op("complex", 128, n=32, ne=96, nr=48),
                "rescal": lambda: Op("rescal", 32, n=32, ne=96, nr=48),
                "mf": lambda: Op("mf", 64, n=32, ne=128)}


def _inflight_steps(op, seed=3):
    """INFLIGHT_STEPS batches, keys distinct within each batch, drawn from all keys of the store"""
    g = torch.Generator().manual_seed(seed)
    init = op.init_rows(g)
    ne_need, nr_need = op.need()
    steps = [op.batch(torch.randperm(op.ne, generator=g)[:ne_need],
                      op.ne + torch.randperm(op.nr, generator=g)[:nr_need] if nr_need else None, g, seed=0xF1 + i)
             for i in range(INFLIGHT_STEPS)]
    return init, steps


def negative_controls(op, init, steps):
    """The rule with one call of a middle step dropped, and with one row read one step stale. Returns
    ``(reference, [(what, rows, loss)])``; each variant must be told apart from the reference at the tolerance of
    the comparison, or that comparison could not see a lost update or a stale read."""
    ref = reference_run(op, init, steps)
    mid = len(steps) // 2
    k_prev, k_cur = set(op.keys_of(steps[mid - 1]).tolist()), op.keys_of(steps[mid]).tolist()
    key = next(k for k in k_cur if k in k_prev)
    return ref, [("one call dropped", *reference_run(op, init, steps, drop=(mid, 0))),
                 ("one row read one step stale", *reference_run(op, init, steps, stale=(mid, key)))]


def _differs(rows, ref_rows):
    try:
        _assert_rows(rows, ref_rows, "")
        return False
    except AssertionError:
        return True


@pytest.mark.parametrize("name", sorted(INFLIGHT_OPS))
def test_inflight_reference_detects_lost_and_stale_updates(name):
    """Host-only: at the step sizes of the keys-in-flight tests, a dropped call and a stale read each move the rows by
    more than the comparison's tolerance."""
    op = INFLIGHT_OPS[name]()
    init, steps = _inflight_steps(op)
    (ref_rows, _), variants = negative_controls(op, init, steps)
    for what, rows, _ in variants:
        assert _differs(rows, ref_rows), f"{op}: {what} is within rtol={RTOL}, atol={ATOL} of the rule"


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
@pytest.mark.parametrize("name", sorted(INFLIGHT_OPS))
def test_fused_steps_lose_no_update_while_keys_move(name, technique):
    """Ranks 0 and 1 keep relocating all keys between them; rank 2 runs INFLIGHT_STEPS steps on those keys (one stream,
    keys distinct within a step). Whatever state a row is in when a step meets it (peer owner, relocation source,
    relocation target being filled), the result is rank 2's steps applied one after another."""
    op = INFLIGHT_OPS[name]()
    op.init, steps = _inflight_steps(op)
    res = while_keys_move(op, steps, technique)
    out = res[2]
    s = out["stats"]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{op} {technique}: stats {s} (remote rows {s[1]}, slow-path calls {s[2]}), relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res), info
    assert s[3] == sum(op.updates(b) for b in steps), info
    ref_rows, ref_loss = reference_run(op, op.init, steps)
    _assert_rows(out["rows"], ref_rows, info)
    torch.testing.assert_close(out["loss"], ref_loss, rtol=1e-3 if op.kind == "sgns" else 1e-4, atol=1e-3)


# ---- gathers of rows in flight: nobody writes the rows, so every result has one exact expectation
GATHER_KEYS, GATHER_DIM, GATHER_M = 1 << 16, 200, 64
GATHER_TOPK = (1, 10, 64)
GATHER_REPS = 16


def _gather_inputs():
    g = torch.Generator().manual_seed(99)
    rows = torch.randn(GATHER_KEYS, GATHER_DIM, generator=g)
    q = torch.randn(GATHER_M, GATHER_DIM, generator=g)
    keys = torch.randperm(GATHER_KEYS, generator=g)
    true_col = torch.randint(0, GATHER_KEYS, (GATHER_M,), generator=g)
    counts = torch.randint(0, 6, (GATHER_M,), generator=g)
    off = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)])
    cols = torch.cat([torch.sort(torch.randperm(GATHER_KEYS, generator=g)[:int(c)]).values for c in counts])
    scale = torch.rand(GATHER_KEYS, generator=g) + 0.5
    return rows, q, keys, true_col, (off, cols), scale


def _gather_all(server, q, keys, true_col, exclude, scale, stats=None):
    from adapm_b200.ops import gather_gemm, gather_gemm_rank_count, gather_gemm_topk

    scores = gather_gemm(server, q, keys, GATHER_DIM, stats=stats)
    true_score = scores.gather(1, true_col.view(-1, 1)).view(-1)
    out = {"scores": scores,
           "rank": gather_gemm_rank_count(server, q, keys, GATHER_DIM, true_score, true_col, stats=stats)}
    for k in GATHER_TOPK:
        out[f"top{k}"] = gather_gemm_topk(server, q, keys, GATHER_DIM, k, exclude=exclude, col_scale=scale, stats=stats)
    return out


def _one_rank_expectation():
    rows, q, keys, true_col, (off, cols), scale = _gather_inputs()
    with one_rank_store(GATHER_DIM, GATHER_KEYS, "cuda", "float32") as (s, w):
        w.wait(w.set(torch.arange(GATHER_KEYS), rows.view(-1)))
        dev = s.device
        exp = _gather_all(s, q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev)), scale.to(dev))
        torch.cuda.synchronize()
        return {k: (tuple(t.cpu() for t in v) if isinstance(v, tuple) else v.cpu()) for k, v in exp.items()}


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_gathers_of_rows_in_flight_are_exact(technique):
    """2^16 rows of 200 floats, 8192 of them relocating between ranks 0 and 1 all the time; rank 2 repeats gather_gemm,
    gather_gemm_rank_count and gather_gemm_topk (k = 1, 10, 64, with exclusions and column scales) over all keys. Each
    result equals, bit for bit, the same op on a one-rank store loaded with the same rows: a row read as zeros, or
    half-way through its transfer, shows as a wrong score."""
    exp = _one_rank_expectation()
    rows, q, keys, true_col, (off, cols), scale = _gather_inputs()

    def read(server, kv, stats):
        dev = server.device
        args = (q.to(dev), keys.to(dev), true_col.to(dev), (off.to(dev), cols.to(dev)), scale.to(dev))
        return lambda: _gather_all(server, *args, stats=stats)

    block = torch.arange(0, GATHER_KEYS, 8)       # 8192 keys move between ranks 0 and 1, spread over all tiles
    res = reads_while_keys_move(Case(GATHER_DIM, GATHER_KEYS, [(torch.arange(GATHER_KEYS), rows)]), read, exp, block,
                                technique, min_reps=GATHER_REPS, max_reps=50 * GATHER_REPS)
    out = res[2]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: {out['reps']} repetitions, stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res), info
    assert not out["mism"], f"{info}; mismatches (repetition, result): {out['mism']}"
    assert out["stats"][2] == 0, info


# ---------------------------------------------------------------------------------------------- 4. in-place TMA, world=1
def inplace_sgns_check(d, neg):
    """The distinct-key comparison of the one-GPU SGNS step (test_gpu_ops.py) for impl="tma", run in a process with
    ADAPM_SGNS_DETERMINISTIC=0: the in-place kernel sgns_step_tma_kernel<VPL, 128>, one launch."""
    from adapm_b200 import _C

    assert os.environ.get("ADAPM_SGNS_DETERMINISTIC") == "0"
    op = Op("sgns", d, neg, "tma", n=64)
    op.ne = 2 * (op.n * (neg + 2) + 10)
    g = torch.Generator().manual_seed(d * 1000 + neg)
    init = op.init_rows(g)
    b = op.batch(torch.randperm(op.ne, generator=g)[:op.need()[0]], None, g)
    b["negatives"][0, 0] = b["contexts"][0]          # a negative equal to the context is skipped
    with one_rank_store(2 * d, op.ne, "cuda", "float32") as (s, kv):
        load_rows(kv, init)
        dev = s.device
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        b_dev = {k: v.to(dev) for k, v in b.items()}
        torch.cuda.synchronize()
        n0 = _C.kernel_launches()
        from adapm_b200.ops import sgns_step

        sgns_step(s, b_dev["centers"], b_dev["contexts"], b_dev["negatives"].contiguous(), d, op.lr, loss, stats, impl="tma")
        launches = _C.kernel_launches() - n0
        torch.cuda.synchronize()
        got = pull_rows(kv, init)
    ref_rows, ref_loss = reference_run(op, init, [b])
    _assert_rows(got, ref_rows, f"in-place sgns d={d} neg={neg}")
    torch.testing.assert_close(float(loss.item()), ref_loss, rtol=1e-3, atol=1e-3)
    st = stats.tolist()
    assert launches == 1, launches
    assert st[1] == 0 and st[2] == 0 and st[3] == op.updates(b) - 1, st
    print(f"ok d={d} neg={neg} stats={st}")


@gpu
@pytest.mark.parametrize("d,neg", [(64, 5), (200, 30), (300, 25)])
def test_inplace_tma_sgns_step_matches_reference(d, neg):
    env = dict(os.environ, ADAPM_SGNS_DETERMINISTIC="0")
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            f"import test_gpu_fused_multirank as t; t.inplace_sgns_check({d}, {neg})")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and f"ok d={d}" in r.stdout, (r.stdout + r.stderr)[-4000:]


# ---------------------------------------------------------------------------------------------- 5. sampler
SAMPLER_KEYS = 300


def _local_sampler_worker(kv, server, wid, weights):
    from adapm_b200.ops import DeviceSampler

    rank = server.my_rank()
    kv.barrier()
    mine = torch.arange(rank * 60, rank * 60 + 120) % SAMPLER_KEYS     # overlapping sets: relocations and replicas
    make_local(kv, server, mine)
    local0 = torch.tensor([server.is_local(k) for k in range(SAMPLER_KEYS)])
    sampler = DeviceSampler(server, weights=weights)
    n = 1 << 21
    keys = sampler.sample(n, seed=1234 + rank, local_only=True)
    torch.cuda.synchronize()
    local1 = torch.tensor([server.is_local(k) for k in range(SAMPLER_KEYS)])
    hist = torch.bincount(keys.cpu(), minlength=SAMPLER_KEYS).double() / n
    out = {"local0": local0, "local1": local1, "hist": hist, "stats": sampler.stats.tolist(),
           "mine_local": bool(local0[mine].all())}
    kv.barrier()
    kv.finalize()
    return out


@gpu
def test_local_only_sampling_draws_local_keys_by_weight():
    """After intents made a known set local on every rank, DeviceSampler(local_only=True) draws only local keys, with
    the frequencies of the weights restricted to them (rejection sampling, no give-ups)."""
    g = torch.Generator().manual_seed(5)
    weights = torch.rand(SAMPLER_KEYS, generator=g, dtype=torch.float64) ** 3 + 0.01
    res = run_cluster(functools.partial(_local_sampler_worker, weights=weights), world=WORLD, workers=1, mode="threads",
                      value_lengths=4, num_keys=SAMPLER_KEYS, dtype="float32", backend="cuda")
    for r in range(WORLD):
        out = res[r][0]
        assert out["mine_local"], r
        assert torch.equal(out["local0"], out["local1"]), f"rank {r}: residency changed while sampling"
        st = out["stats"]
        assert st[0] > 0 and st[1] == 0, (r, st)
        local = out["local0"]
        assert 0 < int(local.sum()) < SAMPLER_KEYS, int(local.sum())
        assert float(out["hist"][~local].sum()) == 0.0, f"rank {r} drew non-local keys"
        p = weights * local
        p = p / p.sum()
        err = float((out["hist"] - p).abs().max())
        assert err < 3e-3, (r, err)


@gpu
def test_log_uniform_sampling_matches_its_distribution():
    from adapm_b200.ops import DeviceSampler

    n, first = 1000, 17
    with one_rank_store(4, first + n + 5, "cuda", "float32") as (s, _):
        sampler = DeviceSampler(s, distribution="log-uniform", num_keys=n, first_key=first)
        draws = 1 << 22
        keys = sampler.sample(draws, seed=42).cpu()
    assert int(keys.min()) == first and int(keys.max()) == first + n - 1, (int(keys.min()), int(keys.max()))
    hist = torch.bincount(keys - first, minlength=n).double() / draws
    j = torch.arange(n, dtype=torch.float64)
    p = torch.log((j + 2) / (j + 1)) / np.log(n + 1)
    err = float((hist - p).abs().max())
    assert err < 3e-3, err
