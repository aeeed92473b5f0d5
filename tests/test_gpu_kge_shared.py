"""KGE sampled-softmax step on the H100 (kge_shared_core in csrc/cuda/ops_kge_1vsall.cu): every pushed row against the
float64 rule with the bf16 operands emulated, at the shapes where the kernels change (batches around the 128-triple
chunk, negative counts around the list tile, ComplEx and RESCAL dims, tiny entity sets full of duplicates and masks,
large ones where every other row must stay bit-for-bit), bit-identical runs, the three-rank scenarios of
tests/multirank.py, and the quality of ComplEx sampled softmax on the FB15k-237 toy set."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multirank import WORLD, Case, on_peer_rows, on_replicas, one_rank_store, while_keys_move  # noqa: E402
from test_gpu_kge_1vsall import _cfg, _check, _tables  # noqa: E402

gpu = pytest.mark.gpu


def _batch(cfg, B, S, seed):
    g = torch.Generator().manual_seed(seed + 1)
    ne = cfg.num_entities
    t = torch.stack([torch.randint(0, ne, (B,), generator=g), torch.randint(0, cfg.num_relations, (B,), generator=g),
                     torch.randint(0, ne, (B,), generator=g)], 1)
    t[0, 2] = t[0, 0]                                   # s == o
    if B > 2:
        t[1] = t[0]                                     # a repeated triple
    neg = torch.randint(0, ne, (S,), generator=g)
    if S > 2:
        neg[0], neg[1] = t[0, 2], t[-1, 0]             # negatives equal to an answer and to a given entity
    return t, neg


def _reference(cfg, E, R, batches):
    """the float64 rule with emulated bf16 operands, one (triples, negatives) batch after another, on a CPU store"""
    from adapm_b200 import ops

    with one_rank_store(cfg.value_lengths(), cfg.num_keys, "cpu", "float64") as (server, kv):
        ne, nr = cfg.num_entities, cfg.num_relations
        kv.wait(kv.set(torch.arange(ne), E.double().reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), R.double().reshape(-1)))
        loss = sum(ops.kge_shared_reference_step(kv, t, n, cfg, emulate_bf16=True) for t, n in batches)
        e = torch.empty(E.numel(), dtype=torch.float64)
        r = torch.empty(R.numel(), dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne), e))
        kv.wait(kv.pull(torch.arange(ne, ne + nr), r))
    return e.view_as(E), r.view_as(R), loss


def _step(kv, cfg, t, neg, loss):
    from adapm_b200 import ops

    ne = cfg.num_entities
    t, neg = t.cuda(), neg.cuda()
    ops.kge_shared_step(kv, t[:, 0].contiguous(), (t[:, 1] + ne).contiguous(), t[:, 2].contiguous(), neg, ne,
                        cfg.algorithm, cfg.embed_dim, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, loss)


def _run_gpu(cfg, E, R, batches):
    with one_rank_store(cfg.value_lengths(), cfg.num_keys, "cuda", "float32") as (server, kv):
        ne, nr = cfg.num_entities, cfg.num_relations
        kv.wait(kv.set(torch.arange(ne), E.reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), R.reshape(-1)))
        loss = torch.zeros(1, device=server.device)
        for t, neg in batches:
            _step(kv, cfg, t, neg, loss)
        torch.cuda.synchronize()
        e = torch.empty(E.numel())
        r = torch.empty(R.numel())
        kv.wait(kv.pull(torch.arange(ne), e))
        kv.wait(kv.pull(torch.arange(ne, ne + nr), r))
    return e.view_as(E), r.view_as(R), float(loss.item())


SHAPES = [
    # algo, ne, nr, d, B, S
    # batches around the 128-triple chunk, on 5 entities: duplicates and masked columns everywhere
    ("ComplEx", 5, 3, 8, 1, 0),
    ("ComplEx", 5, 3, 8, 127, 1),
    ("ComplEx", 5, 3, 8, 128, 100),
    ("ComplEx", 5, 3, 8, 129, 128),
    ("ComplEx", 5, 3, 8, 300, 1000),
    # negative counts around the 128-column tile of the list (2 * 128 + S columns)
    ("ComplEx", 300, 11, 64, 300, 0),
    ("ComplEx", 300, 11, 64, 129, 1),
    ("ComplEx", 300, 11, 64, 128, 128),
    ("ComplEx", 300, 11, 64, 127, 1000),
    # ComplEx dims, one not a multiple of 64 (nor of 8)
    ("ComplEx", 300, 11, 2, 300, 100),
    ("ComplEx", 300, 11, 100, 129, 100),
    ("ComplEx", 500, 11, 512, 300, 1000),
    ("RESCAL", 5, 3, 8, 129, 100),
    ("RESCAL", 300, 11, 64, 300, 128),
    # a large entity set: every row outside the step's keys stays bit-for-bit
    ("ComplEx", 100_000, 11, 64, 300, 1000),
    ("RESCAL", 100_000, 11, 8, 129, 100),
]


@gpu
@pytest.mark.parametrize("algo,ne,nr,d,B,S", SHAPES)
def test_step_matches_float64_rule(algo, ne, nr, d, B, S):
    cfg = _cfg(algo, ne, nr, d)
    E, R = _tables(cfg, seed=ne + d + B + S)
    t, neg = _batch(cfg, B, S, seed=ne * 7 + d + S)
    e, r, loss = _run_gpu(cfg, E, R, [(t, neg)])
    we, wr, wloss = _reference(cfg, E, R, [(t, neg)])
    assert abs(loss - wloss) <= 1e-4 * abs(wloss) + 1e-3, (loss, wloss)
    touched = torch.zeros(ne, dtype=torch.bool)
    touched[torch.cat([t[:, 0], t[:, 2], neg])] = True
    _check(cfg, E[touched].double(), e[touched], we[touched])
    assert torch.equal(e[~touched], E[~touched])
    used = torch.zeros(nr, dtype=torch.bool)
    used[t[:, 1]] = True
    _check(cfg, R[used].double(), r[used], wr[used])
    assert torch.equal(r[~used], R[~used])


@gpu
@pytest.mark.parametrize("algo,d", [("ComplEx", 64), ("RESCAL", 16)])
def test_runs_are_bit_identical(algo, d):
    cfg = _cfg(algo, 2000, 5, d)
    E, R = _tables(cfg, seed=3)
    batches = [_batch(cfg, 300, 200, seed=10 + i) for i in range(5)]
    first = _run_gpu(cfg, E, R, batches)
    second = _run_gpu(cfg, E, R, batches)
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1]) and first[2] == second[2]
    assert not torch.equal(first[0], E)


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
MR_CFG = ("ComplEx", 90, 6, 16)
MR_NEG = torch.tensor([3, 17, 17, 40, 88, 5, 61])


class _Stepper:
    def __init__(self, server, kv, cfg):
        self.server, self.kv, self.cfg = server, kv, cfg
        self.loss = torch.zeros(1, device=server.device)

    def __call__(self, b):
        _step(self.kv, self.cfg, b, MR_NEG, self.loss)

    def totals(self):
        return float(self.loss.item()), [0, 0, 0, 0]


def _mr_case():
    cfg = _cfg(*MR_CFG)
    E, R = _tables(cfg, seed=77)
    ne, nr = cfg.num_entities, cfg.num_relations
    init = [(torch.arange(ne), E), (torch.arange(ne, ne + nr), R)]
    keys_of = lambda b: torch.unique(torch.cat([b[:, 0], b[:, 2], MR_NEG, b[:, 1] + ne]))
    return cfg, E, R, Case(cfg.value_lengths(), cfg.num_keys, init, keys_of, lambda server, kv: _Stepper(server, kv, cfg))


def _mr_batches(cfg, n, seed):
    return [_batch(cfg, 24, 0, seed=seed + k)[0] for k in range(n)]


def _check_rows(cfg, E, R, rows, batches):
    we, wr, _ = _reference(cfg, E, R, [(b, MR_NEG) for b in batches])
    _check(cfg, E.double(), rows[0].view_as(E), we)
    used = torch.zeros(cfg.num_relations, dtype=torch.bool)
    used[torch.cat([b[:, 1] for b in batches])] = True
    _check(cfg, R[used].double(), rows[1].view_as(R)[used], wr[used])


@gpu
def test_step_on_peer_rows():
    cfg, E, R, case = _mr_case()
    batches = _mr_batches(cfg, WORLD, 200)
    res = on_peer_rows(case, batches, in_turns=True)
    assert all(x["remote"] > 0 for x in res)
    _check_rows(cfg, E, R, res[0]["rows"], batches)


@gpu
def test_step_on_replicas():
    cfg, E, R, case = _mr_case()
    batches = _mr_batches(cfg, WORLD, 300)
    res = on_replicas(case, batches)
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    for k in range(WORLD):
        assert res[k]["local"] and res[k]["replicas"] > 0
        _check_rows(cfg, E, R, res[k]["rows"], batches)


@gpu
def test_step_loses_no_update_while_keys_move():
    cfg, E, R, case = _mr_case()
    batches = _mr_batches(cfg, 8, 400)
    res = while_keys_move(case, batches, "relocation_only")
    assert sum(x["counters"]["relocations"] for x in res) > 0
    _check_rows(cfg, E, R, res[2]["rows"], batches)


# ---------------------------------------------------------------------------------------------- quality
@gpu
def test_complex_sampled_softmax_quality_on_fb15k237_toy():
    """The settings of test_kge_shared_cpu.test_complex_sampled_softmax_quality_on_fb15k237_toy on the CUDA backend
    (negatives from the device sampler): filtered test MRR 0.568 and Hits@10 0.862 measured on an NVIDIA H100 80GB HBM3
    at a 700 W power limit (1vsAll: 0.589 / 0.888). The thresholds are 0.05 below the measured values."""
    from test_kge_shared_cpu import train_shared_toy

    ev = train_shared_toy("cuda")
    print("ComplEx sampled-softmax toy test (H100):", ev)
    assert ev["mrr"] >= GPU_MRR - 0.05 and ev["hits@10"] >= GPU_HITS10 - 0.05, ev


GPU_MRR, GPU_HITS10 = 0.568, 0.862
