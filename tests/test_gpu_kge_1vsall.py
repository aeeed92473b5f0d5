"""KGE 1vsAll step on the H100 (csrc/cuda/ops_kge_1vsall.cu): every pushed row against the float64 rule with the bf16
operands emulated, at the shapes where the kernels change (entity counts around the 128-row tile, the split-K of the long
contractions, several query chunks, ComplEx and RESCAL dims), bit-identical runs, the three-rank scenarios of
tests/multirank.py, and the quality of ComplEx 1vsAll on the FB15k-237 toy set."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multirank import WORLD, Case, on_peer_rows, on_replicas, one_rank_store, while_keys_move  # noqa: E402

gpu = pytest.mark.gpu
ETA, GE, GR = 0.1, 0.01, 0.02


def _cfg(algo, ne, nr, d):
    from adapm_b200.models.kge import KGEConfig

    return KGEConfig(num_entities=ne, num_relations=nr, embed_dim=d, algorithm=algo, eta=ETA, gamma_entity=GE,
                     gamma_relation=GR)


def _tables(cfg, seed):
    """entity rows [ne, 2 d] and relation rows [nr, rel_len]: values of std 0.3, accumulators 1 (a mid-training state in
    which an update depends smoothly on its gradient)"""
    g = torch.Generator().manual_seed(seed)
    ne, nr, d, rl = cfg.num_entities, cfg.num_relations, cfg.embed_dim, cfg.relation_len
    scale = 0.3 if cfg.algorithm == "ComplEx" else 0.3 / np.sqrt(d) ** 0.5
    E = torch.cat([torch.randn(ne, d, generator=g) * scale, torch.ones(ne, d)], 1)
    R = torch.cat([torch.randn(nr, rl // 2, generator=g) * scale, torch.ones(nr, rl // 2)], 1)
    return E, R


def _triples(cfg, B, seed):
    g = torch.Generator().manual_seed(seed + 1)
    t = torch.stack([torch.randint(0, cfg.num_entities, (B,), generator=g),
                     torch.randint(0, cfg.num_relations, (B,), generator=g),
                     torch.randint(0, cfg.num_entities, (B,), generator=g)], 1)
    t[0, 2] = t[0, 0]                                   # s == o
    if B > 2:
        t[1] = t[0]                                     # a repeated triple
    return t


def _reference(cfg, E, R, batches):
    """the float64 rule with emulated bf16 operands, one batch after another, on a CPU store"""
    from adapm_b200 import ops

    with one_rank_store(cfg.value_lengths(), cfg.num_keys, "cpu", "float64") as (server, kv):
        ne, nr = cfg.num_entities, cfg.num_relations
        kv.wait(kv.set(torch.arange(ne), E.double().reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), R.double().reshape(-1)))
        loss = sum(ops.kge_1vsall_reference_step(kv, b, cfg, emulate_bf16=True) for b in batches)
        e = torch.empty(E.numel(), dtype=torch.float64)
        r = torch.empty(R.numel(), dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne), e))
        kv.wait(kv.pull(torch.arange(ne, ne + nr), r))
    return e.view_as(E), r.view_as(R), loss


def _check(cfg, old, got, want):
    """Rows [x + u | a + g^2] against the rule. With bf16 operands emulated, the GPU and the rule differ where an operand
    computed in fp32 (a query, an element of G) rounds to the other side of a bf16 boundary than its float64 value:
    such a flip moves one term of a gradient by 2^-8 of itself. Allowing four flips on the largest term, plus fp32
    accumulation, bounds |g_gpu - g_rule| by tol = 2^-6 max|g|; with a = 1, |du| <= eta tol and |d g^2| <= (2 max|g| +
    tol) tol."""
    d = old.shape[1] // 2
    g2 = want[:, d:] - old[:, d:]
    gmax = float(g2.max().sqrt())
    tol = 2.0 ** -6 * gmax
    du = (got[:, :d].double() - want[:, :d]).abs().max()
    dg = (got[:, d:].double() - want[:, d:]).abs().max()
    assert du <= ETA * tol, (float(du), ETA * tol)
    assert dg <= (2 * gmax + tol) * tol, (float(dg), (2 * gmax + tol) * tol)


def _run_gpu(cfg, E, R, batches, max_bytes=1 << 30):
    from adapm_b200 import ops

    with one_rank_store(cfg.value_lengths(), cfg.num_keys, "cuda", "float32") as (server, kv):
        ne, nr = cfg.num_entities, cfg.num_relations
        kv.wait(kv.set(torch.arange(ne), E.reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), R.reshape(-1)))
        loss = torch.zeros(1, device=server.device)
        for b in batches:
            b = b.to(server.device)
            ops.kge_1vsall_step(kv, b[:, 0].contiguous(), (b[:, 1] + ne).contiguous(), b[:, 2].contiguous(), ne,
                                cfg.algorithm, cfg.embed_dim, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, loss,
                                max_bytes=max_bytes)
        torch.cuda.synchronize()
        e = torch.empty(E.numel())
        r = torch.empty(R.numel())
        kv.wait(kv.pull(torch.arange(ne), e))
        kv.wait(kv.pull(torch.arange(ne, ne + nr), r))
    return e.view_as(E), r.view_as(R), float(loss.item())


SHAPES = [
    # algo, ne, nr, d, B, max_bytes: entity counts around the 128 tile
    ("ComplEx", 1, 3, 8, 5, 1 << 30),
    ("ComplEx", 127, 7, 8, 40, 1 << 30),
    ("ComplEx", 128, 7, 8, 40, 1 << 30),
    ("ComplEx", 129, 7, 8, 40, 1 << 30),
    ("ComplEx", 300, 11, 8, 40, 1 << 30),
    # long-K split of G E (N = 2000: 32 k-blocks over one output tile) and of G^T Q (1024 queries, 3 row tiles)
    ("ComplEx", 2000, 13, 64, 4, 1 << 30),
    ("ComplEx", 300, 11, 16, 512, 1 << 30),
    # several query chunks (128 queries each, the last one partial)
    ("ComplEx", 300, 11, 32, 200, 128 * (4 * 300 + 2 * 304 + 2 * 300)),
    # ComplEx dims, one not a multiple of 64 (nor of 8)
    ("ComplEx", 300, 11, 2, 64, 1 << 30),
    ("ComplEx", 300, 11, 100, 64, 1 << 30),
    ("ComplEx", 500, 11, 512, 300, 1 << 30),
    ("RESCAL", 300, 11, 8, 64, 1 << 30),
    ("RESCAL", 600, 11, 64, 300, 1 << 30),
]


@gpu
@pytest.mark.parametrize("algo,ne,nr,d,B,max_bytes", SHAPES)
def test_step_matches_float64_rule(algo, ne, nr, d, B, max_bytes):
    cfg = _cfg(algo, ne, nr, d)
    E, R = _tables(cfg, seed=ne + d + B)
    b = _triples(cfg, B, seed=ne * 7 + d)
    e, r, loss = _run_gpu(cfg, E, R, [b], max_bytes)
    we, wr, wloss = _reference(cfg, E, R, [b])
    assert abs(loss - wloss) <= 1e-4 * abs(wloss) + 1e-3, (loss, wloss)
    _check(cfg, E.double(), e, we)
    used = torch.zeros(nr, dtype=torch.bool)
    used[b[:, 1]] = True
    _check(cfg, R[used].double(), r[used], wr[used])
    assert torch.equal(r[~used], R[~used])


@gpu
@pytest.mark.parametrize("algo,d", [("ComplEx", 64), ("RESCAL", 16)])
def test_runs_are_bit_identical(algo, d):
    cfg = _cfg(algo, 2000, 5, d)
    E, R = _tables(cfg, seed=3)
    batches = [_triples(cfg, 96, seed=10 + i) for i in range(5)]
    first = _run_gpu(cfg, E, R, batches, max_bytes=128 * (8 * 2000 + 2 * 2000))   # two query chunks per step
    second = _run_gpu(cfg, E, R, batches, max_bytes=128 * (8 * 2000 + 2 * 2000))
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1]) and first[2] == second[2]
    assert not torch.equal(first[0], E)


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
class _Stepper:
    def __init__(self, server, kv, cfg):
        self.server, self.kv, self.cfg = server, kv, cfg
        self.loss = torch.zeros(1, device=server.device)

    def __call__(self, b):
        from adapm_b200 import ops

        cfg, ne = self.cfg, self.cfg.num_entities
        b = b.to(self.server.device)
        ops.kge_1vsall_step(self.kv, b[:, 0].contiguous(), (b[:, 1] + ne).contiguous(), b[:, 2].contiguous(), ne,
                            cfg.algorithm, cfg.embed_dim, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, self.loss)

    def totals(self):
        return float(self.loss.item()), [0, 0, 0, 0]


MR_CFG = ("ComplEx", 90, 6, 16)


def _mr_case():
    cfg = _cfg(*MR_CFG)
    E, R = _tables(cfg, seed=77)
    ne, nr = cfg.num_entities, cfg.num_relations
    init = [(torch.arange(ne), E), (torch.arange(ne, ne + nr), R)]
    keys_of = lambda b: torch.unique(torch.cat([torch.arange(ne), b[:, 1] + ne]))
    return cfg, E, R, Case(cfg.value_lengths(), cfg.num_keys, init, keys_of, lambda server, kv: _Stepper(server, kv, cfg))


def _check_rows(cfg, E, R, rows, batches):
    we, wr, _ = _reference(cfg, E, R, batches)
    _check(cfg, E.double(), rows[0].view_as(E), we)
    used = torch.zeros(cfg.num_relations, dtype=torch.bool)
    used[torch.cat([b[:, 1] for b in batches])] = True
    _check(cfg, R[used].double(), rows[1].view_as(R)[used], wr[used])


@gpu
def test_step_on_peer_rows():
    cfg, E, R, case = _mr_case()
    batches = [_triples(cfg, 24, seed=200 + k) for k in range(WORLD)]
    res = on_peer_rows(case, batches, in_turns=True)
    assert all(x["remote"] > 0 for x in res)
    _check_rows(cfg, E, R, res[0]["rows"], batches)


@gpu
def test_step_on_replicas():
    cfg, E, R, case = _mr_case()
    batches = [_triples(cfg, 24, seed=300 + k) for k in range(WORLD)]
    res = on_replicas(case, batches)
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    for k in range(WORLD):
        assert res[k]["local"] and res[k]["replicas"] > 0
        _check_rows(cfg, E, R, res[k]["rows"], batches)


@gpu
def test_step_loses_no_update_while_keys_move():
    cfg, E, R, case = _mr_case()
    batches = [_triples(cfg, 24, seed=400 + k) for k in range(8)]
    res = while_keys_move(case, batches, "relocation_only")
    assert sum(x["counters"]["relocations"] for x in res) > 0
    _check_rows(cfg, E, R, res[2]["rows"], batches)


# ---------------------------------------------------------------------------------------------- quality
@gpu
def test_complex_1vsall_quality_on_fb15k237_toy():
    """The settings of test_kge_1vsall_cpu.test_complex_1vsall_quality_on_fb15k237_toy on the CUDA backend: filtered test
    MRR 0.589 and Hits@10 0.888 measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit. The thresholds are 0.05
    below the measured values."""
    from test_kge_1vsall_cpu import train_toy

    ev = train_toy("cuda", "1vsAll")
    print("ComplEx 1vsAll toy test (H100):", ev)
    assert ev["mrr"] >= GPU_MRR - 0.05 and ev["hits@10"] >= GPU_HITS10 - 0.05, ev


GPU_MRR, GPU_HITS10 = 0.589, 0.888
