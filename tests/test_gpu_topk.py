"""Top-k retrieval on the tensor cores (ops_topk.cu): gemm_nt_topk and gather_gemm_topk against a stable
(score descending, column ascending) sort of the scores of gemm_nt_bf16 / gather_gemm, bit for bit; memory bound;
KGE.predict and Word2Vec.most_similar against dense references."""
import pytest
import torch

from harness import run_cluster

pytestmark = pytest.mark.gpu


def _csr(mask: torch.Tensor):
    """bool [M, N] -> (offsets int64 [M + 1], cols int64 [nnz]) with ascending columns per row."""
    off = torch.zeros(mask.shape[0] + 1, dtype=torch.int64, device=mask.device)
    off[1:] = torch.cumsum(mask.sum(1), 0)
    return off, mask.nonzero()[:, 1].contiguous()


def _assert_same(got, ref):
    (gv, gi), (rv, ri) = got, ref
    assert torch.equal(gi, ri), (gi[:4], ri[:4])
    assert torch.equal(gv, rv), (gv[:4], rv[:4])


@pytest.mark.parametrize("M,N,K", [(1, 7, 8), (333, 129, 200), (100, 1000, 72), (2048, 14951, 512), (4096, 65536, 304)])
def test_gemm_nt_topk_matches_sorted_gemm_bit_for_bit(M, N, K):
    from adapm_b200.ops import gemm_nt_bf16, gemm_nt_topk, topk_reference

    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 7 * K)
    q = torch.randn(M, K, device="cuda", generator=g)
    e = torch.randn(N, K, device="cuda", generator=g)
    scores = gemm_nt_bf16(q, e)
    cs = torch.rand(N, device="cuda", generator=g) + 0.5
    mask = torch.rand(M, N, device="cuda", generator=g) < 0.02
    mask[0, 3:] = True                                     # row 0: fewer than k eligible columns -> padding
    excl = _csr(mask)
    for k in (1, 10, 64):
        _assert_same(gemm_nt_topk(q, e, k), topk_reference(scores, k))
        _assert_same(gemm_nt_topk(q, e, k, col_scale=cs), topk_reference(scores * cs, k))
        got = gemm_nt_topk(q, e, k, exclude=excl, col_scale=cs)
        _assert_same(got, topk_reference(scores * cs, k, mask))
        if k > 3:
            assert (got[1][0, 3:] == -1).all() and got[0][0, 3:].isneginf().all()


def test_gemm_nt_topk_ties_nan_and_determinism():
    """duplicated rows of e give exactly equal scores: the smaller column comes first; NaN columns never appear"""
    from adapm_b200.ops import gemm_nt_bf16, gemm_nt_topk, topk_reference

    g = torch.Generator(device="cuda").manual_seed(11)
    M, N, K = 700, 5000, 128
    q = torch.randn(M, K, device="cuda", generator=g)
    e = torch.randn(N, K, device="cuda", generator=g)
    src = torch.randint(0, N, (400,), device="cuda", generator=g)
    dst = torch.randint(0, N, (400,), device="cuda", generator=g)
    e[dst] = e[src]
    v = torch.randn(K, device="cuda", generator=g)
    e[[17, 2500, 4000, 4999]] = v                             # ties that cross column tiles and slices
    e[123] = float("nan")
    scores = gemm_nt_bf16(q, e)
    for k in (1, 10, 64):
        got = gemm_nt_topk(q, e, k)
        _assert_same(got, topk_reference(scores, k))
        assert not (got[1] == 123).any()
        _assert_same(gemm_nt_topk(q, e, k), got)             # repeated calls are bit-identical
    top4 = gemm_nt_topk(v.view(1, -1), e, 4)[1][0].tolist()
    assert top4 == [17, 2500, 4000, 4999], top4


def _store(nk, row_len, rows, job):
    import adapm_b200 as ad

    server = ad.Server(row_len, num_keys=nk, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc", job=job,
                       device=0)
    kv = ad.Worker(0, server)
    for i in range(0, nk, 1 << 16):
        kv.set(torch.arange(i, min(nk, i + (1 << 16)), device=server.device), rows[i:i + (1 << 16)].reshape(-1))
    kv.waitall()
    return server, kv


def test_gather_gemm_topk_matches_sorted_gather_gemm():
    from adapm_b200.ops import gather_gemm, gather_gemm_topk, topk_reference

    nk, d = 20000, 200
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = torch.randn(nk, 2 * d, device="cuda", generator=g)
    rows[77] = rows[5]                                       # an exact tie
    server, kv = _store(nk, 2 * d, rows, "topkg")
    keys = torch.randperm(nk, device="cuda", generator=g)
    q = torch.randn(513, d, device="cuda", generator=g)
    scores = gather_gemm(server, q, keys, d)
    cs = torch.rand(nk, device="cuda", generator=g) + 0.5
    mask = torch.rand(513, nk, device="cuda", generator=g) < 0.01
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    for k in (1, 10, 64):
        got = gather_gemm_topk(server, q, keys, d, k, stats=stats)
        _assert_same(got, topk_reference(scores, k))
        _assert_same(gather_gemm_topk(server, q, keys, d, k), got)
        _assert_same(gather_gemm_topk(server, q, keys, d, k, exclude=_csr(mask), col_scale=cs),
                     topk_reference(scores * cs, k, mask))
    torch.cuda.synchronize()
    assert stats[0].item() >= 3 * nk and stats[1].item() == 0
    kv.finalize(); server.shutdown()


def test_gather_gemm_topk_memory_stays_small():
    """M = 4096 queries against 2^20 store rows of d = 300: a score matrix would take 16 GB."""
    from adapm_b200.ops import gather_gemm_topk

    nk, d = 1 << 20, 300
    g = torch.Generator(device="cuda").manual_seed(2)
    server, kv = _store(nk, 2 * d, torch.randn(nk, 2 * d, device="cuda", generator=g), "topkmem")
    keys = torch.arange(nk, device="cuda")
    q = torch.randn(4096, d, device="cuda", generator=g)
    gather_gemm_topk(server, q, keys, d, 10)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    vals, idx = gather_gemm_topk(server, q, keys, d, 10)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 64 << 20, extra
    assert (idx >= 0).all() and torch.isfinite(vals).all()
    kv.finalize(); server.shutdown()


def _near_tie_match(ids, ref_scores, k, tol):
    """ids [n, k] from a bf16 path vs fp32 scores [n, N] (ineligible columns at -inf): a returned column may differ from
    the fp32 top-k only where the fp32 scores are within tol of the k-th best"""
    kth = torch.sort(ref_scores, dim=1, descending=True).values[:, k - 1]
    got = ref_scores.gather(1, ids.clamp(min=0))
    assert (ids >= 0).all()
    assert (got >= kth.view(-1, 1) - tol.view(-1, 1)).all()
    better = ref_scores > (kth + tol).view(-1, 1)
    hit = torch.zeros_like(better)
    hit.scatter_(1, ids, True)
    assert not (better & ~hit).any()


def test_kge_predict_and_topk_hits_match_fused_eval():
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, complex_query, evaluate_fused, synthetic_triples
    from adapm_b200.ops import gather_gemm_topk

    cfg = KGEConfig(num_entities=900, num_relations=11, embed_dim=64, neg_ratio=2, batch_triples=512)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="kgetopk", device=0)
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    tr = synthetic_triples(cfg, 3000, seed=4)
    for s in range(0, tr.shape[0], cfg.batch_triples):
        model.step(tr[s:s + cfg.batch_triples])
    torch.cuda.synchronize()
    dev, d, ne = server.device, cfg.embed_dim, cfg.num_entities
    test = tr[:400].to(dev)
    ref = evaluate_fused(model, test, tr)
    E, _, R, _ = model.pull_embeddings(dev)
    all_ent = torch.arange(ne, device=dev)
    hits = {1: 0, 3: 0, 10: 0}
    for side in ("object", "subject"):
        given, true_e = (test[:, 0], test[:, 2]) if side == "object" else (test[:, 2], test[:, 0])
        q = complex_query(E[given], R[test[:, 1]], conj=(side == "subject"))
        off, cols = model._known_answers(given, test[:, 1], side, tr)
        rows = torch.repeat_interleave(torch.arange(test.shape[0], device=dev), off[1:] - off[:-1])
        other = torch.zeros(test.shape[0], ne, dtype=torch.bool, device=dev)
        other[rows, cols] = True
        other[torch.arange(test.shape[0], device=dev), true_e] = False       # rank the true answer among the rest
        _, idx = gather_gemm_topk(server, q, all_ent, d, 10, exclude=_csr(other))
        for k in hits:
            hits[k] += int((idx[:, :k] == true_e.view(-1, 1)).any(1).sum())
        # KGE.predict against the dense fp32 scores, all known answers filtered
        ids, vals = model.predict(given, test[:, 1], side=side, k=10, known=tr)
        known = other.clone()
        known[torch.arange(test.shape[0], device=dev), true_e] = True
        sc = (q @ E.t()).masked_fill(known, float("-inf"))
        tol = 1e-2 * (q.abs() @ E.abs().t()).amax(1)          # bf16 operands: about 2^-8 of sum |q_i e_i|
        _near_tie_match(ids, sc, 10, tol)
        assert not known.gather(1, ids).any()
        assert ((vals - sc.gather(1, ids)).abs() <= tol.view(-1, 1)).all()
    n = 2 * test.shape[0]
    for k, name in ((1, "hits@1"), (3, "hits@3"), (10, "hits@10")):
        assert abs(hits[k] / n - ref[name]) <= 1e-2, (k, hits[k] / n, ref)
    kv.finalize(); server.shutdown()


def test_word2vec_most_similar_matches_dense_cosine():
    import adapm_b200 as ad
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig, syn0_key, zipf_counts

    cfg = Word2VecConfig(vocab_size=30000, embed_dim=100, batch_pairs=1024)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="w2vtopk", device=0)
    kv = ad.Worker(0, server)
    model = Word2Vec(server, kv, cfg, zipf_counts(cfg.vocab_size))
    model.init_model()
    g = torch.Generator(device="cuda").manual_seed(3)
    V, d = cfg.vocab_size, cfg.embed_dim
    E = torch.randn(V, d, device="cuda", generator=g)
    E[101] = 3 * E[100]                                        # same direction as word 100
    kv.set(syn0_key(torch.arange(V, device="cuda")), torch.cat([E, torch.full_like(E, 1e-6)], 1).reshape(-1))
    kv.waitall()
    words = torch.cat([torch.tensor([100, 101], device="cuda"), torch.randint(0, V, (300,), device="cuda", generator=g)])
    norms = model.syn0_norms()
    torch.testing.assert_close(norms, 1 / E.norm(dim=1))
    for k in (1, 10, 64):
        ids, cos = model.most_similar(words, k=k, norms=norms)
        assert not (ids == words.view(-1, 1)).any()
        ref = (E[words] / E[words].norm(dim=1, keepdim=True)) @ (E / E.norm(dim=1, keepdim=True)).t()
        ref[torch.arange(words.numel()), words] = float("-inf")
        _near_tie_match(ids, ref, k, torch.full((words.numel(),), 2e-2, device="cuda"))
        torch.testing.assert_close(cos, ref.gather(1, ids), atol=2e-2, rtol=0)
        assert ids[0, 0].item() == 101 and ids[1, 0].item() == 100
    kv.finalize(); server.shutdown()


def _two_gpu_worker(kv, server, wid):
    import torch
    from adapm_b200.ops import gather_gemm_topk, gemm_nt_topk

    nk, d = 6000, 136
    g = torch.Generator().manual_seed(8)
    rows = torch.randn(nk, 2 * d, generator=g)
    if wid == 0:
        kv.set(torch.arange(nk), rows.clone().view(-1))
    kv.waitall(); kv.barrier()
    dev = server.device
    keys = torch.randperm(nk, generator=g).to(dev)
    q = torch.randn(300, d, generator=g).to(dev)
    stats = torch.zeros(2, dtype=torch.int64, device=dev)
    out = {}
    for k in (1, 10, 64):
        got = gather_gemm_topk(server, q, keys, d, k, stats=stats)
        ref = gemm_nt_topk(q, rows.to(dev)[keys][:, :d], k)      # one GPU, same bf16 operands and k-block order
        out[k] = bool(torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]))
    torch.cuda.synchronize()
    out["stats"] = stats.tolist()
    kv.barrier()
    kv.finalize()
    return out


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs at least 2 GPUs")
def test_gather_gemm_topk_two_gpus_matches_one_gpu():
    res = run_cluster(_two_gpu_worker, world=2, workers=1, mode="procs", value_lengths=2 * 136, num_keys=6000,
                      dtype="float32", backend="cuda")
    for r in res.values():
        out = r[0]
        assert out[1] and out[10] and out[64], out
        assert out["stats"][1] > 0, f"expected rows gathered from the peer GPU: {out['stats']}"
