"""KGE sampled-softmax training without a GPU: the float64 rule ``kge_shared_reference_step`` against the loss written
independently and differentiated by autograd, its agreement with the 1vsAll rule when one chunk's list holds every
entity once, the input checks of the op and the model, the spill-free build of the new kernels, the app on two CPU
ranks, and the filtered-ranking quality of ComplEx on the FB15k-237 toy set (tests/golden/kge_fb15k237_toy)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kge_fb15k237_toy")
CHUNK = 128


def _store(cfg, dtype="float64"):
    import adapm_b200 as ad

    s = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                  fabric="inproc", job=f"shared_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def autograd_rule(E, A, Rr, Ar, triples, negatives, cfg):
    """Sampled softmax written as one float64 loss and differentiated by autograd. Per chunk of 128 triples, every
    query is scored with the model's score function against each column of [subjects, objects, negatives]; the columns
    holding the answer, other than its own slot, are left out of the cross-entropy; L2 is 0.5 gamma |x|^2 per triple.
    Returns (new entity rows, new relation rows of the distinct relations in ascending order, cross-entropy)."""
    d = cfg.embed_dim
    s, r, o = triples[:, 0], triples[:, 1], triples[:, 2]
    uniq, inv = torch.unique(r, return_inverse=True)
    E = E.clone().requires_grad_()
    Rl = Rr[uniq].clone().requires_grad_()
    if cfg.algorithm == "ComplEx":
        h = d // 2

        def sc(a, rr, b):
            return (rr[:h] * (a[:h] * b[:h] + a[h:] * b[h:]) + rr[h:] * (a[:h] * b[h:] - a[h:] * b[:h])).sum()
    else:
        def sc(a, rr, b):
            return a @ rr.view(d, d) @ b
    ce = torch.zeros((), dtype=torch.float64)
    for c0 in range(0, s.numel(), CHUNK):
        idx = range(c0, min(s.numel(), c0 + CHUNK))
        cols = [int(s[i]) for i in idx] + [int(o[i]) for i in idx] + [int(x) for x in negatives]
        n = len(idx)
        for t, i in enumerate(idx):
            rel = Rl[inv[i]]
            for obj_query in (True, False):
                answer = int(o[i]) if obj_query else int(s[i])
                own = n + t if obj_query else t
                z = [sc(E[s[i]], rel, E[x]) if obj_query else sc(E[x], rel, E[o[i]])
                     for j, x in enumerate(cols) if j == own or x != answer]
                own_at = sum(1 for j, x in enumerate(cols[:own]) if x != answer)
                ce = ce + torch.logsumexp(torch.stack(z), 0) - z[own_at]
    l2 = 0.5 * cfg.gamma_entity * ((E[s] ** 2).sum() + (E[o] ** 2).sum()) + 0.5 * cfg.gamma_relation * (Rl[inv] ** 2).sum()
    ge, gr = torch.autograd.grad(ce + l2, [E, Rl])

    def upd(x, a, g):
        return torch.cat([x + torch.where(g == 0, torch.zeros_like(g), -cfg.eta * g / torch.sqrt(a + g * g)), a + g * g], 1)

    return upd(E.detach(), A, ge), upd(Rr[uniq], Ar[uniq], gr), float(ce.detach())


def _random_tables(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    ne, nr, d, rl = cfg.num_entities, cfg.num_relations, cfg.embed_dim, cfg.relation_len
    E, A = torch.randn(ne, d, generator=g, dtype=torch.float64), torch.rand(ne, d, generator=g, dtype=torch.float64)
    Rr = torch.randn(nr, rl // 2, generator=g, dtype=torch.float64)
    Ar = torch.rand(nr, rl // 2, generator=g, dtype=torch.float64)
    return E, A, Rr, Ar


def _run_reference(cfg, tables, triples, negatives, **kw):
    from adapm_b200 import ops

    E, A, Rr, Ar = tables
    ne, nr = cfg.num_entities, cfg.num_relations
    server, kv = _store(cfg)
    try:
        kv.wait(kv.set(torch.arange(ne), torch.cat([E, A], 1).reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), torch.cat([Rr, Ar], 1).reshape(-1)))
        loss = ops.kge_shared_reference_step(kv, triples, negatives, cfg, **kw)
        new_e = torch.empty(ne * cfg.entity_len, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne), new_e))
        new_r = torch.empty(nr * cfg.relation_len, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne, ne + nr), new_r))
    finally:
        kv.finalize()
        server.shutdown()
    return new_e.view(ne, -1), new_r.view(nr, -1), loss


def _cfg(algo, d, ne, nr, **kw):
    from adapm_b200.models.kge import KGEConfig

    return KGEConfig(num_entities=ne, num_relations=nr, embed_dim=d, algorithm=algo, eta=0.3, gamma_entity=0.05,
                     gamma_relation=0.02, **kw)


def _many(B, ne, nr, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.stack([torch.randint(0, ne, (B,), generator=g), torch.randint(0, nr, (B,), generator=g),
                     torch.randint(0, ne, (B,), generator=g)], 1)
    t[0, 2] = t[0, 0]                      # s == o
    t[1] = t[0]                            # a repeated triple
    return t


CASES = [
    # one chunk: duplicate subjects, objects and relations, s == o, repeated triples; negatives that repeat, that equal
    # a query's answer (2, 3) and a given entity (0, 4)
    ("ComplEx", 4, 9, 3, [[0, 1, 2], [0, 1, 3], [4, 0, 4], [2, 2, 0], [3, 1, 3], [0, 0, 2], [0, 1, 2]], [2, 7, 7, 0, 4, 3]),
    ("ComplEx", 6, 5, 2, [[1, 0, 1], [1, 0, 1], [2, 1, 4]], []),                     # S = 0
    ("RESCAL", 3, 9, 3, [[0, 1, 2], [0, 1, 3], [4, 0, 4], [2, 2, 0], [3, 1, 3], [0, 0, 2]], [8, 2, 2, 4]),
    ("RESCAL", 2, 1, 1, [[0, 0, 0]], [0]),
    # three chunks, the last one partial (300 triples over 7 entities: every list is full of duplicates)
    ("ComplEx", 4, 7, 3, 300, [1, 5, 5]),
    ("RESCAL", 2, 7, 2, 300, []),
]


@pytest.mark.parametrize("algo,d,ne,nr,trip,neg", CASES)
def test_reference_matches_autograd(algo, d, ne, nr, trip, neg):
    cfg = _cfg(algo, d, ne, nr)
    tables = _random_tables(cfg, 7)
    triples = _many(trip, ne, nr, seed=ne + d) if isinstance(trip, int) else torch.tensor(trip, dtype=torch.int64)
    negatives = torch.tensor(neg, dtype=torch.int64)
    new_e, new_r, loss = _run_reference(cfg, tables, triples, negatives)
    want_e, want_r, want_loss = autograd_rule(*tables, triples, negatives, cfg)
    uniq = torch.unique(triples[:, 1])
    assert abs(loss - want_loss) <= 1e-10 * max(1.0, abs(want_loss))
    torch.testing.assert_close(new_e, want_e, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(new_r[uniq], want_r, rtol=1e-10, atol=1e-12)
    E, A, Rr, Ar = tables
    untouched = torch.ones(nr, dtype=torch.bool)
    untouched[uniq] = False
    assert torch.equal(new_r[untouched], torch.cat([Rr, Ar], 1)[untouched])


def test_rows_outside_the_step_are_unchanged():
    """only the batch's entities, the negatives and the batch's relations move; a negative-only entity gets no L2 (its
    gradient is its candidate columns alone, so with every one of its columns masked it does not move)"""
    cfg = _cfg("ComplEx", 4, 30, 5)
    tables = _random_tables(cfg, 11)
    triples = torch.tensor([[0, 1, 2], [3, 1, 4], [5, 2, 5]])
    negatives = torch.tensor([9, 9, 20])
    new_e, new_r, _ = _run_reference(cfg, tables, triples, negatives)
    old_e = torch.cat(tables[:2], 1)
    touched = torch.zeros(30, dtype=torch.bool)
    touched[torch.tensor([0, 2, 3, 4, 5, 9, 20])] = True
    assert torch.equal(new_e[~touched], old_e[~touched])
    assert not (new_e[touched] == old_e[touched]).all(1).any()
    old_r = torch.cat(tables[2:], 1)
    assert torch.equal(new_r[torch.tensor([0, 3, 4])], old_r[torch.tensor([0, 3, 4])])


@pytest.mark.parametrize("algo,d", [("ComplEx", 6), ("RESCAL", 3)])
def test_one_list_of_every_entity_is_1vsall(algo, d):
    """one chunk whose list [subjects, objects, negatives] holds every entity exactly once masks nothing: the step is
    then the 1vsAll rule"""
    from adapm_b200 import ops

    ne, nr = 11, 3
    cfg = _cfg(algo, d, ne, nr)
    tables = _random_tables(cfg, 5)
    perm = torch.randperm(ne, generator=torch.Generator().manual_seed(1))
    triples = torch.stack([perm[:4], torch.tensor([0, 2, 0, 1]), perm[4:8]], 1)
    got_e, got_r, got_loss = _run_reference(cfg, tables, triples, perm[8:])
    E, A, Rr, Ar = tables
    server, kv = _store(cfg)
    try:
        kv.wait(kv.set(torch.arange(ne), torch.cat([E, A], 1).reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), torch.cat([Rr, Ar], 1).reshape(-1)))
        want_loss = ops.kge_1vsall_reference_step(kv, triples, cfg)
        want_e = torch.empty(ne * cfg.entity_len, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne), want_e))
        want_r = torch.empty(nr * cfg.relation_len, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne, ne + nr), want_r))
    finally:
        kv.finalize()
        server.shutdown()
    assert abs(got_loss - want_loss) <= 1e-12 * abs(want_loss)
    torch.testing.assert_close(got_e, want_e.view(ne, -1), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(got_r, want_r.view(nr, -1), rtol=1e-12, atol=1e-14)


def test_emulate_bf16_rounds_the_operands():
    """emulate_bf16 changes the result by about the bf16 rounding of the operands, and nothing else"""
    cfg = _cfg("ComplEx", 8, 20, 3)
    tables = _random_tables(cfg, 3)
    triples, negatives = torch.tensor([[0, 1, 5], [7, 2, 7]]), torch.tensor([3, 11, 5])
    e0, r0, l0 = _run_reference(cfg, tables, triples, negatives)
    e1, r1, l1 = _run_reference(cfg, tables, triples, negatives, emulate_bf16=True)
    assert l0 != l1 and abs(l0 - l1) < 0.05 * abs(l0)
    assert not torch.equal(e0, e1)
    assert (e0 - e1).abs().max() < 0.05 * (e0 - torch.cat(tables[:2], 1)).abs().max()


def test_input_checks():
    from adapm_b200 import ops
    from adapm_b200.models.kge import KGE, KGEConfig

    cfg = KGEConfig(num_entities=10, num_relations=2, embed_dim=4, algorithm="ComplEx")
    server, kv = _store(cfg, "float32")
    t = torch.zeros(3, dtype=torch.int64)
    loss = torch.zeros(1)
    args = (10, "ComplEx", 4, 0.1, 0.0, 0.0, loss)
    try:
        with pytest.raises(ValueError, match="ComplEx and RESCAL"):
            ops.kge_shared_step(kv, t, t + 10, t, t, 10, "TransE", 4, 0.1, 0.0, 0.0, loss)
        for bad in (0, 3, 1026, 2.5, True):
            with pytest.raises(ValueError, match="embed_dim"):
                ops.kge_shared_step(kv, t, t + 10, t, t, 10, "ComplEx", bad, 0.1, 0.0, 0.0, loss)
        with pytest.raises(ValueError, match="num_entities"):
            ops.kge_shared_step(kv, t, t + 10, t, t, 0, *args[1:])
        with pytest.raises(ValueError, match="CUDA int64"):
            ops.kge_shared_step(kv, t, t + 10, t, t, *args)          # CPU tensors
        with pytest.raises(ValueError, match="CUDA int64"):
            ops.kge_shared_step(kv, t.int(), t + 10, t, t, *args)
        with pytest.raises(ValueError, match="entity ids"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 0, 10]]), torch.tensor([1]), cfg)
        with pytest.raises(ValueError, match="entity ids"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 0, 1]]), torch.tensor([10]), cfg)
        with pytest.raises(ValueError, match="entity ids"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 0, 1]]), torch.tensor([-1]), cfg)
        with pytest.raises(ValueError, match="relation ids"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 2, 1]]), torch.tensor([1]), cfg)
        with pytest.raises(ValueError, match="even"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 0, 1]]), torch.tensor([1]),
                                          KGEConfig(num_entities=10, embed_dim=3))
        with pytest.raises(ValueError, match="ComplEx and RESCAL"):
            ops.kge_shared_reference_step(kv, torch.tensor([[0, 0, 1]]), torch.tensor([1]),
                                          KGEConfig(num_entities=10, embed_dim=4, algorithm="RotatE"))
        for kw in (dict(algorithm="TransE"), dict(algorithm="RotatE"), dict(dropout_entity=0.1),
                   dict(dropout_relation=0.1), dict(shared_negatives=-1), dict(shared_negatives=2.5)):
            with pytest.raises(ValueError):
                KGE(server, kv, KGEConfig(num_entities=10, num_relations=2, embed_dim=4,
                                          **{"train_type": "sampled_softmax", **kw}))
    finally:
        kv.finalize()
        server.shutdown()


def test_new_kernels_do_not_spill():
    """the sampled-softmax kernels and the batched GEMM, from the -Xptxas -v logs of the in-tree build"""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    names = ("gemm_batched_kernel", "gather_bf16_kernel", "kge_shared_lse_kernel", "kge_shared_grad_kernel",
             "kge_shared_entity_kernel")
    for name in names:
        assert name in k, sorted(k)
        assert k[name]["spill"] == 0, (name, k[name])


def test_kge_app_sampled_softmax_two_ranks():
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", "2", "--backend", "cpu", "-m", "adapm_b200.apps.kge",
                        "--", "--dataset", GOLDEN + "/", "--num_entities", "280", "--num_relations", "112", "--embed_dim",
                        "16", "--num_epochs", "2", "--algorithm", "RESCAL", "--train_type", "sampled_softmax",
                        "--shared_negatives", "32", "--eval_freq", "2", "--eval_truncate_va", "50", "--neg_ratio", "0"],
                       cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "[kge] epoch 2: cross-entropy loss" in out and "[kge] test: {" in out, out[-2000:]
    l1, l2 = (float(line.split("loss ")[1].split()[0]) for line in out.splitlines()
              if line.startswith("[kge] epoch") and "cross-entropy loss" in line)
    assert np.isfinite(l1) and l2 < l1, out[-2000:]


def train_shared_toy(backend, epochs=12, shared_negatives=64):
    """ComplEx at d 100, eta 0.1, 70-triple batches with sampled softmax on the toy set's training split, one rank; the
    filtered test metrics against train + valid + test."""
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, load_triples

    cfg = KGEConfig(num_entities=280, num_relations=112, algorithm="ComplEx", embed_dim=100, eta=0.1, batch_triples=70,
                    train_type="sampled_softmax", shared_negatives=shared_negatives)
    tr, va, te = (load_triples(os.path.join(GOLDEN, f"{n}.del")) for n in ("train", "valid", "test"))
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend=backend,
                       fabric="inproc", job=f"shared_toy_{np.random.randint(1 << 30)}",
                       **({"device": 0} if backend == "cuda" else {}))
    kv = ad.Worker(0, server)
    try:
        model = KGE(server, kv, cfg)
        model.init_model()
        for epoch in range(1, epochs + 1):
            perm = tr[torch.randperm(tr.shape[0], generator=torch.Generator().manual_seed(epoch * 977))]
            for s in range(0, perm.shape[0], cfg.batch_triples):
                model.step(perm[s:s + cfg.batch_triples])
                kv.advance_clock()
        return model.evaluate(te, torch.cat([tr, va, te]))
    finally:
        kv.finalize()
        server.shutdown()


def test_complex_sampled_softmax_quality_on_fb15k237_toy():
    """ComplEx sampled softmax, d 100, eta 0.1, 12 epochs of 70-triple batches, 64 shared negatives, CPU backend:
    filtered test MRR 0.592 and Hits@10 0.888 measured. At the same settings negative sampling (neg_ratio 6) reaches
    0.375 / 0.681 and 1vsAll 0.590 / 0.885. The thresholds are 0.05 below the measured values."""
    ev = train_shared_toy("cpu")
    print("ComplEx sampled-softmax toy test:", ev)
    assert ev["mrr"] >= CPU_MRR - 0.05 and ev["hits@10"] >= CPU_HITS10 - 0.05, ev


CPU_MRR, CPU_HITS10 = 0.592, 0.888
