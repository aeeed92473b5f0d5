"""Top-k retrieval on the CPU backend (KGE.predict, Word2Vec.most_similar) against brute-force float64 references,
and the argument checks of the top-k ops (which run before anything touches a device)."""
import uuid

import numpy as np
import pytest
import torch


def _server(value_lengths, num_keys):
    import adapm_b200 as ad

    server = ad.Server(value_lengths, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                       job=f"topk{uuid.uuid4().hex[:6]}")
    return server, ad.Worker(0, server)


def _brute_topk(scores: np.ndarray, k: int, excluded=None):
    """float64 reference: per row the k best eligible columns, score descending, ties to the smaller column."""
    out_i, out_v = [], []
    for i, row in enumerate(scores):
        cand = [(-row[j], j) for j in range(row.size) if not (excluded is not None and j in excluded[i])]
        cand.sort()
        cand = cand[:k]
        out_i.append([j for _, j in cand] + [-1] * (k - len(cand)))
        out_v.append([-s for s, _ in cand] + [-np.inf] * (k - len(cand)))
    return np.array(out_i, dtype=np.int64), np.array(out_v)


@pytest.mark.parametrize("algo", ["ComplEx", "RESCAL", "TransE", "RotatE"])
@pytest.mark.parametrize("side", ["object", "subject"])
def test_kge_predict_cpu_matches_float64_bruteforce(algo, side):
    """Embeddings with quarter-integer entries (TransE: entity rows with one entry of +-1 or +-2, so normalising is exact)
    make every score exact in float32, so ties are exact: duplicated entity rows must come out in ascending id order,
    and filtering must remove exactly the known answers. RotatE's scores round, so its rows are drawn at random and the
    order may differ only between scores within float32 rounding of each other."""
    from adapm_b200.models.kge import KGE, KGEConfig

    cfg = KGEConfig(num_entities=40, num_relations=3, embed_dim=8 if algo == "RotatE" else 4, algorithm=algo)
    server, kv = _server(cfg.value_lengths(), cfg.num_keys)
    model = KGE(server, kv, cfg)
    g = torch.Generator().manual_seed(5)
    d, ne, nr = cfg.embed_dim, cfg.num_entities, cfg.num_relations
    if algo == "TransE":
        E = torch.zeros(ne, d, dtype=torch.float64)
        E[torch.arange(ne), torch.randint(0, d, (ne,), generator=g)] = (
            torch.tensor([-2.0, -1.0, 1.0, 2.0], dtype=torch.float64)[torch.randint(0, 4, (ne,), generator=g)])
    elif algo == "RotatE":
        E = torch.randn(ne, d, generator=g, dtype=torch.float64).float().double()
    else:
        E = torch.randint(-3, 4, (ne, d), generator=g).double() / 4
    E[7] = E[3]; E[20] = E[3]; E[11] = E[30]               # exact ties
    if algo == "RotatE":
        R = ((torch.rand(nr, d // 2, generator=g, dtype=torch.float64) * 2 - 1) * np.pi).float().double()
    else:
        R = torch.randint(-2, 3, (nr, cfg.relation_len // 2), generator=g).double() / 4
    ent_rows = torch.cat([E, torch.full((ne, d), 1e-6, dtype=torch.float64)], 1).float()
    rel_rows = torch.cat([R, torch.full_like(R, 1e-6)], 1).float()
    kv.set(torch.arange(ne), ent_rows.reshape(-1))
    kv.set(torch.arange(ne, ne + nr), rel_rows.reshape(-1))
    kv.waitall()

    ents = torch.tensor([3, 0, 11, 25, 39])
    rels = torch.tensor([0, 1, 2, 1, 0])
    known = torch.tensor([[3, 0, 7], [3, 0, 20], [0, 1, 5], [11, 2, 30], [25, 1, 3], [39, 0, 39],
                          [7, 0, 3], [20, 0, 3], [5, 1, 0], [30, 2, 11], [3, 1, 25], [3, 0, 7]])
    for k, kn in ((5, None), (10, known), (64, known)):
        ids, vals = model.predict(ents, rels, side=side, k=k, known=kn)
        assert ids.shape == (5, k) and vals.shape == (5, k) and ids.dtype == torch.int64 and vals.dtype == torch.float32
        if algo == "ComplEx":
            h = d // 2
            a, r = E[ents], R[rels]
            are, aim, rre, rim = a[:, :h], a[:, h:], r[:, :h], r[:, h:]
            if side == "object":
                q = torch.cat([rre * are - rim * aim, rre * aim + rim * are], 1)
            else:
                q = torch.cat([rre * are + rim * aim, rre * aim - rim * are], 1)
            scores = q @ E.t()
        elif algo == "RESCAL":
            Rm = R[rels].view(-1, d, d)
            q = torch.einsum("bi,bij->bj", E[ents], Rm) if side == "object" else torch.einsum("bij,bj->bi", Rm, E[ents])
            scores = q @ E.t()
        elif algo == "TransE":                             # -|s^ + r - o^|_1, candidates o (object) or s (subject)
            En = E / E.norm(dim=1, keepdim=True)
            q = En[ents] + R[rels] if side == "object" else En[ents] - R[rels]
            scores = -(q.unsqueeze(1) - En.unsqueeze(0)).abs().sum(-1)
        else:                                              # -sum_i |s_i e^{i theta_i} - o_i|
            Z = torch.view_as_complex(E.view(ne, d // 2, 2).contiguous())
            rho = torch.exp(1j * R[rels]).unsqueeze(1)
            if side == "object":
                scores = -(Z[ents].unsqueeze(1) * rho - Z.unsqueeze(0)).abs().sum(-1)
            else:
                scores = -(Z.unsqueeze(0) * rho - Z[ents].unsqueeze(1)).abs().sum(-1)
        excl = None
        if kn is not None:
            excl = [set() for _ in range(5)]
            for s, r, o in kn.tolist():
                for i in range(5):
                    if side == "object" and (s, r) == (int(ents[i]), int(rels[i])):
                        excl[i].add(o)
                    if side == "subject" and (o, r) == (int(ents[i]), int(rels[i])):
                        excl[i].add(s)
        ref_i, ref_v = _brute_topk(scores.numpy(), k, excl)
        if algo == "RotatE":
            got_i, n_ok = ids.numpy(), min(k, ne)
            np.testing.assert_allclose(vals.double().numpy()[:, :n_ok], ref_v[:, :n_ok], rtol=1e-6, atol=1e-5)
            assert np.array_equal(np.isneginf(vals.numpy()), np.isneginf(ref_v))
            for i in range(5):
                for a, b, va in zip(got_i[i], ref_i[i], ref_v[i]):
                    if a != b:    # only a near-tie may swap
                        assert a >= 0 and abs(float(scores[i, a]) - va) < 1e-5, (i, a, b)
                for tied in ((3, 7, 20), (11, 30)):        # exact ties keep ascending ids
                    got = [j for j in got_i[i].tolist() if j in tied]
                    assert got == sorted(got), (i, got)
        else:
            assert np.array_equal(ids.numpy(), ref_i), (k, ids, ref_i)
            assert np.array_equal(vals.double().numpy(), ref_v), (k, vals, ref_v)
        if kn is not None:
            for i in range(5):
                assert not (set(ids[i].tolist()) & excl[i])
    kv.finalize(); server.shutdown()


def test_word2vec_most_similar_cpu_matches_float64_bruteforce():
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig, syn0_key, zipf_counts

    cfg = Word2VecConfig(vocab_size=50, embed_dim=8, negative=2, batch_pairs=32)
    server, kv = _server(cfg.row_len, cfg.num_keys)
    model = Word2Vec(server, kv, cfg, zipf_counts(cfg.vocab_size))
    g = torch.Generator().manual_seed(9)
    V, d = cfg.vocab_size, cfg.embed_dim
    E = torch.randint(-4, 5, (V, d), generator=g).float()
    E[9] = E[2]; E[33] = E[2]; E[40] = 2 * E[17]              # same direction: exact cosine ties
    E[5] = 0                                                  # a zero row never qualifies
    rows = torch.cat([E, torch.full((V, d), 1e-6)], 1)
    kv.set(syn0_key(torch.arange(V)), rows.reshape(-1))
    kv.waitall()
    words = torch.tensor([2, 17, 9, 44, 0])
    norms = model.syn0_norms()
    nz = E.norm(dim=1) > 0
    assert torch.isinf(norms[5]) and torch.allclose(norms[nz], 1 / E[nz].norm(dim=1))
    for k in (1, 10, 64):
        ids, cos = model.most_similar(words, k=k, norms=norms)
        assert ids.shape == (5, k) and cos.dtype == torch.float32
        E64 = E.double()
        cos64 = (E64[words] @ E64.t()) / (E64[words].norm(dim=1, keepdim=True) * E64.norm(dim=1).view(1, -1))
        excl = [{int(w)} | {5} for w in words]                  # the query itself; the zero row has NaN scores
        ref_i, ref_v = _brute_topk(cos64.numpy(), k, excl)
        got_i = ids.numpy()
        for i, w in enumerate(words.tolist()):
            assert w not in got_i[i] and 5 not in got_i[i]
            n_ok = min(k, V - 2)
            assert (got_i[i, n_ok:] == -1).all() and np.isneginf(cos[i, n_ok:].numpy()).all()
            np.testing.assert_allclose(cos[i, :n_ok].double().numpy(), ref_v[i, :n_ok], rtol=0, atol=1e-6)
            # identical ids except where float32 rounding may reorder near-equal scores
            for a, b, va in zip(got_i[i, :n_ok], ref_i[i, :n_ok], ref_v[i, :n_ok]):
                if a != b:
                    assert abs(cos64[i, a] - va) < 1e-6, (i, a, b)
        # exact ties (same direction) keep ascending ids
        if k >= 10:
            row = ids[0].tolist()
            assert row.index(9) < row.index(33)
    kv.finalize(); server.shutdown()


def test_topk_reference_order_padding_and_nan():
    from adapm_b200.ops import topk_reference

    s = torch.tensor([[1.0, 3.0, 3.0, float("nan"), -float("inf"), 2.0],
                      [0.5, 0.5, 0.5, 0.5, 0.5, 0.5]])
    ex = torch.zeros(2, 6, dtype=torch.bool)
    ex[0, 5] = True; ex[1, :4] = True
    v, i = topk_reference(s, 6, ex)
    assert i[0].tolist() == [1, 2, 0, 4, -1, -1]
    assert v[0].tolist()[:4] == [3.0, 3.0, 1.0, -float("inf")] and v[0, 4:].isneginf().all()
    assert i[1].tolist() == [4, 5, -1, -1, -1, -1]
    v, i = topk_reference(s, 8)
    assert i[0].tolist() == [1, 2, 5, 0, 4, -1, -1, -1]


def test_topk_ops_reject_bad_arguments():
    from adapm_b200.ops import gather_gemm_topk, gemm_nt_topk

    q, e = torch.zeros(4, 16), torch.zeros(10, 16)
    for k in (0, 65, -1, 2.5):
        with pytest.raises(ValueError):
            gemm_nt_topk(q, e, k)
    with pytest.raises(ValueError):
        gemm_nt_topk(q, torch.zeros(10, 8), 3)                      # K mismatch
    with pytest.raises(ValueError):
        gemm_nt_topk(q, e, 3, col_scale=torch.ones(9))              # one scale per column
    with pytest.raises(TypeError):
        gemm_nt_topk(q, e, 3, col_scale=torch.ones(10, dtype=torch.float64))
    cols = torch.tensor([1, 4, 2], dtype=torch.int64)
    for off in (torch.tensor([0, 1, 2, 3], dtype=torch.int64),        # M + 1 entries needed
                torch.tensor([0, 2, 1, 3, 3], dtype=torch.int64),     # not monotone
                torch.tensor([0, 1, 2, 2, 2], dtype=torch.int64),     # does not end at nnz
                torch.tensor([1, 1, 2, 3, 3], dtype=torch.int64)):    # does not start at 0
        with pytest.raises(ValueError):
            gemm_nt_topk(q, e, 3, exclude=(off, cols))
    with pytest.raises(TypeError):
        gemm_nt_topk(q, e, 3, exclude=(torch.tensor([0, 1, 2, 3, 3], dtype=torch.int32), cols))
    with pytest.raises(TypeError):                                    # a valid call on CPU tensors: not a CUDA tensor
        gemm_nt_topk(q, e, 3, exclude=(torch.tensor([0, 1, 2, 3, 3], dtype=torch.int64), cols))
    with pytest.raises(TypeError):
        gather_gemm_topk(None, q, torch.arange(10), 16, 3)           # keys must be a CUDA tensor
