"""KGE 1vsAll training without a GPU: the float64 rule ``kge_1vsall_reference_step`` against the cross-entropy loss written
independently and differentiated by autograd, the input checks of the op and the model, the app on two CPU ranks, and
the filtered-ranking quality of ComplEx 1vsAll on the FB15k-237 toy set (tests/golden/kge_fb15k237_toy)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kge_fb15k237_toy")


def _store(cfg, dtype="float64"):
    import adapm_b200 as ad

    s = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                  fabric="inproc", job=f"onevsall_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def autograd_rule(E, A, Rr, Ar, triples, cfg):
    """1vsAll written as one float64 loss (cross-entropy of both queries of every triple against all entities, plus the
    L2 terms as 0.5 gamma |x|^2 per triple) and differentiated by autograd; returns (new entity rows, new relation rows
    of the distinct relations in ascending order, cross-entropy)."""
    d = cfg.embed_dim
    s, r, o = triples[:, 0], triples[:, 1], triples[:, 2]
    uniq, inv = torch.unique(r, return_inverse=True)
    E = E.clone().requires_grad_()
    Rl = Rr[uniq].clone().requires_grad_()
    rel = Rl[inv]
    if cfg.algorithm == "ComplEx":
        h = d // 2
        sc = lambda a, rr, b: (rr[:, :h] * (a[:, :h] * b[:, :h] + a[:, h:] * b[:, h:])
                               + rr[:, h:] * (a[:, :h] * b[:, h:] - a[:, h:] * b[:, :h])).sum(-1)
    else:
        sc = lambda a, rr, b: torch.einsum("bi,bij,bj->b", a, rr.view(-1, d, d), b)
    B, N = s.numel(), E.shape[0]
    # score of (s, r, x) and (x, r, o) for every x, straight from the model's score function
    zo = torch.stack([sc(E[s], rel, E[x].expand(B, d)) for x in range(N)], 1)
    zs = torch.stack([sc(E[x].expand(B, d), rel, E[o]) for x in range(N)], 1)
    ce = torch.nn.functional.cross_entropy(zo, o, reduction="sum") + torch.nn.functional.cross_entropy(zs, s, reduction="sum")
    l2 = 0.5 * cfg.gamma_entity * ((E[s] ** 2).sum() + (E[o] ** 2).sum()) + 0.5 * cfg.gamma_relation * (rel ** 2).sum()
    ge, gr = torch.autograd.grad(ce + l2, [E, Rl])

    def upd(x, a, g):
        return torch.cat([x + torch.where(g == 0, torch.zeros_like(g), -cfg.eta * g / torch.sqrt(a + g * g)), a + g * g], 1)

    return upd(E.detach(), A, ge), upd(Rr[uniq], Ar[uniq], gr), float(ce.detach())


CASES = [
    # duplicate subjects, objects and relations, and s == o
    ("ComplEx", 4, 9, 3, [[0, 1, 2], [0, 1, 3], [4, 0, 4], [2, 2, 0], [3, 1, 3], [0, 0, 2]]),
    ("ComplEx", 6, 5, 2, [[1, 0, 1], [1, 0, 1], [2, 1, 4]]),
    ("RESCAL", 3, 9, 3, [[0, 1, 2], [0, 1, 3], [4, 0, 4], [2, 2, 0], [3, 1, 3], [0, 0, 2]]),
    ("RESCAL", 2, 1, 1, [[0, 0, 0]]),
]


@pytest.mark.parametrize("algo,d,ne,nr,trip", CASES)
def test_reference_matches_autograd(algo, d, ne, nr, trip):
    from adapm_b200 import ops
    from adapm_b200.models.kge import KGEConfig

    cfg = KGEConfig(num_entities=ne, num_relations=nr, embed_dim=d, algorithm=algo, eta=0.3, gamma_entity=0.05,
                    gamma_relation=0.02)
    g = torch.Generator().manual_seed(7)
    el, rl = cfg.entity_len, cfg.relation_len
    E, A = torch.randn(ne, d, generator=g, dtype=torch.float64), torch.rand(ne, d, generator=g, dtype=torch.float64)
    Rr = torch.randn(nr, rl // 2, generator=g, dtype=torch.float64)
    Ar = torch.rand(nr, rl // 2, generator=g, dtype=torch.float64)
    triples = torch.tensor(trip, dtype=torch.int64)
    server, kv = _store(cfg)
    try:
        kv.wait(kv.set(torch.arange(ne), torch.cat([E, A], 1).reshape(-1)))
        kv.wait(kv.set(torch.arange(ne, ne + nr), torch.cat([Rr, Ar], 1).reshape(-1)))
        loss = ops.kge_1vsall_reference_step(kv, triples, cfg)
        new_e = torch.empty(ne * el, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne), new_e))
        new_r = torch.empty(nr * rl, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(ne, ne + nr), new_r))
    finally:
        kv.finalize()
        server.shutdown()
    want_e, want_r, want_loss = autograd_rule(E, A, Rr, Ar, triples, cfg)
    uniq = torch.unique(triples[:, 1])
    assert abs(loss - want_loss) <= 1e-10 * max(1.0, abs(want_loss))
    torch.testing.assert_close(new_e.view(ne, el), want_e, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(new_r.view(nr, rl)[uniq], want_r, rtol=1e-10, atol=1e-12)
    untouched = torch.ones(nr, dtype=torch.bool)
    untouched[uniq] = False
    assert torch.equal(new_r.view(nr, rl)[untouched], torch.cat([Rr, Ar], 1)[untouched])


def test_emulate_bf16_rounds_the_operands():
    """emulate_bf16 changes the result by about the bf16 rounding of the operands, and nothing else"""
    from adapm_b200 import ops
    from adapm_b200.models.kge import KGEConfig

    cfg = KGEConfig(num_entities=20, num_relations=3, embed_dim=8, algorithm="ComplEx", eta=0.1)
    out = []
    for emulate in (False, True):
        server, kv = _store(cfg)
        try:
            g = torch.Generator().manual_seed(3)
            kv.wait(kv.set(torch.arange(cfg.num_keys - 2), torch.cat([torch.randn(23, 8, generator=g, dtype=torch.float64),
                                                                      torch.full((23, 8), 1e-6, dtype=torch.float64)], 1)
                           .reshape(-1)))
            loss = ops.kge_1vsall_reference_step(kv, torch.tensor([[0, 1, 5], [7, 2, 7]]), cfg, emulate_bf16=emulate)
            v = torch.empty(20 * 16, dtype=torch.float64)
            kv.wait(kv.pull(torch.arange(20), v))
            out.append((loss, v))
        finally:
            kv.finalize()
            server.shutdown()
    assert out[0][0] != out[1][0] and abs(out[0][0] - out[1][0]) < 0.05 * abs(out[0][0])
    assert not torch.equal(out[0][1], out[1][1])


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
            ops.kge_1vsall_step(kv, t, t + 10, t, 10, "TransE", 4, 0.1, 0.0, 0.0, loss)
        for bad in (0, 3, 1026, 2.5, True):
            with pytest.raises(ValueError, match="embed_dim"):
                ops.kge_1vsall_step(kv, t, t + 10, t, 10, "ComplEx", bad, 0.1, 0.0, 0.0, loss)
        with pytest.raises(ValueError, match="max_bytes"):
            ops.kge_1vsall_step(kv, t, t + 10, t, *args, max_bytes=128 * 80 - 1)
        with pytest.raises(ValueError, match="num_entities"):
            ops.kge_1vsall_step(kv, t, t + 10, t, 0, *args[1:])
        with pytest.raises(ValueError, match="CUDA int64"):
            ops.kge_1vsall_step(kv, t, t + 10, t, *args)          # CPU tensors
        with pytest.raises(ValueError, match="CUDA int64"):
            ops.kge_1vsall_step(kv, t.int(), t + 10, t, *args)
        with pytest.raises(ValueError, match="entity ids"):
            ops.kge_1vsall_reference_step(kv, torch.tensor([[0, 0, 10]]), cfg)
        with pytest.raises(ValueError, match="relation ids"):
            ops.kge_1vsall_reference_step(kv, torch.tensor([[0, 2, 1]]), cfg)
        with pytest.raises(ValueError, match="even"):
            ops.kge_1vsall_reference_step(kv, torch.tensor([[0, 0, 1]]), KGEConfig(num_entities=10, embed_dim=3))
        for kw in (dict(algorithm="TransE"), dict(algorithm="RotatE"), dict(dropout_entity=0.1),
                   dict(dropout_relation=0.1), dict(train_type="KvsAll")):
            with pytest.raises(ValueError):
                KGE(server, kv, KGEConfig(num_entities=10, num_relations=2, embed_dim=4,
                                          **{"train_type": "1vsAll", **kw}))
    finally:
        kv.finalize()
        server.shutdown()


def test_kge_app_1vsall_two_ranks():
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", "2", "--backend", "cpu", "-m", "adapm_b200.apps.kge",
                        "--", "--dataset", GOLDEN + "/", "--num_entities", "280", "--num_relations", "112", "--embed_dim",
                        "16", "--num_epochs", "2", "--algorithm", "RESCAL", "--train_type", "1vsAll", "--eval_freq", "2",
                        "--eval_truncate_va", "50", "--neg_ratio", "0"],
                       cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "[kge] epoch 2: cross-entropy loss" in out and "[kge] test: {" in out, out[-2000:]
    l1, l2 = (float(line.split("loss ")[1].split()[0]) for line in out.splitlines()
              if line.startswith("[kge] epoch") and "cross-entropy loss" in line)
    assert np.isfinite(l1) and l2 < l1, out[-2000:]


def train_toy(backend, train_type, epochs=12):
    """ComplEx at d 100, eta 0.1, 70-triple batches on the toy set's training split, one rank; the filtered test
    metrics against train + valid + test."""
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, load_triples

    cfg = KGEConfig(num_entities=280, num_relations=112, algorithm="ComplEx", embed_dim=100, eta=0.1, batch_triples=70,
                    train_type=train_type)
    tr, va, te = (load_triples(os.path.join(GOLDEN, f"{n}.del")) for n in ("train", "valid", "test"))
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend=backend,
                       fabric="inproc", job=f"onevsall_toy_{np.random.randint(1 << 30)}",
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


def test_complex_1vsall_quality_on_fb15k237_toy():
    """ComplEx 1vsAll, d 100, eta 0.1, 12 epochs of 70-triple batches, CPU backend: filtered test MRR 0.590 and Hits@10
    0.885 measured (model seed 134827). Negative sampling at the same d, epochs and eta (neg_ratio 6) reaches 0.375 /
    0.681. The thresholds are 0.05 below the measured values."""
    ev = train_toy("cpu", "1vsAll")
    print("ComplEx 1vsAll toy test:", ev)
    assert ev["mrr"] >= CPU_MRR - 0.05 and ev["hits@10"] >= CPU_HITS10 - 0.05, ev


CPU_MRR, CPU_HITS10 = 0.590, 0.885
