"""Paragraph vectors without a GPU: the native document streams against the word streams, the float64 inference rule
against an independently written per-document loop, the key layout, input checks, the app through the launcher,
quality on planted topics with the CPU backend, and the inference kernels' build facts."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from multirank import one_rank_store
from test_build_budget import _kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Planted topics (see planted_corpus): 8 topics, chance 1/8 = 0.125 for both measures. The CPU runs measured an
# own-topic share of the 10 nearest training documents of 0.979 (PV-DBOW) and 0.930 (PV-DM), and a share of held-out
# documents whose nearest training document has their topic of 0.738 (PV-DBOW) and 1.000 (PV-DM). The thresholds are
# far above chance and leave room for other runs (the GPU test trains with dbow_words).
SHARE_MIN = 0.6
INFER_MIN = 0.6


# ---------------------------------------------------------------------------------------------- streams
def _line_corpus(path):
    """Lines with disjoint vocabularies: line j uses the words "j_a", "j_b", ... (each at least twice, so min_count 2
    keeps them). Line 3 is empty and line 6 holds only words seen once (filtered): neither is a sentence."""
    rng = np.random.default_rng(5)
    lines = []
    for j in range(11):
        if j == 3:
            lines.append("")
        elif j == 6:
            lines.append("once_x once_y once_z")
        else:
            n_w = int(rng.integers(2, 6))
            words = [f"{j}_{chr(97 + k)}" for k in range(n_w)]
            toks = words * 2 + list(rng.choice(words, int(rng.integers(0, 12))))
            rng.shuffle(toks)
            lines.append(" ".join(toks))
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return lines


def _drain(it, valid_attr):
    out = []
    for b in it:
        n = getattr(b, valid_attr)
        out.append((b[:, :n] if valid_attr == "valid_pairs" else b[:n]).clone())
        assert b.unique_keys.numel() == torch.unique(b[b >= 0]).numel()
        assert set(b.unique_keys.tolist()) == set(b[b >= 0].tolist())
    return out


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("subsample", [0.0, 0.2])
def test_doc_streams_are_the_word_streams_plus_document_keys(tmp_path, world, subsample):
    from adapm_b200.utils.text import NativeCorpus

    path = str(tmp_path / "docs.txt")
    _line_corpus(path)
    vocab = NativeCorpus.build(path, 2).vocabulary()
    V = len(vocab.words)
    line_of = {i: int(w.split("_")[0]) for i, w in enumerate(vocab.words) if "_" in w}
    W, B = 3, 7
    for rank in range(world):
        nc = NativeCorpus.from_vocabulary(vocab).encode(path, rank, world)
        assert nc.num_lines() == 11
        lines = nc.sentence_lines()
        assert lines.tolist() == [j for j in range(11) if j % world == rank and j not in (3, 6)]
        for epoch in (0, 1):
            seed = 9 + rank
            ref = torch.cat(_drain(nc.pair_batches(W, subsample, B, seed, epoch), "valid_pairs"), 1)
            with_words = torch.cat(_drain(nc.doc_pair_batches(W, subsample, B, seed, True, epoch), "valid_pairs"), 1)
            only_docs = torch.cat(_drain(nc.doc_pair_batches(W, subsample, B, seed, False, epoch), "valid_pairs"), 1)
            is_doc = with_words[0] >= 2 * V
            assert torch.equal(with_words[:, ~is_doc], ref)
            assert torch.equal(with_words[:, is_doc], only_docs)
            assert bool((only_docs[0] >= 2 * V).all()) and bool((only_docs[1] % 2 == 1).all())
            # every document key is 2 V + the line of its word
            words = (only_docs[1] - 1) // 2
            assert only_docs[0].tolist() == [2 * V + line_of[int(w)] for w in words]
            if subsample == 0.0:            # every position of every sentence is walked, in order
                sents = [s for s in nc.sentences() if s.size >= 2]
                assert words.tolist() == np.concatenate(sents).tolist()
            wref = torch.cat(_drain(nc.window_batches(W, subsample, B, seed, epoch), "valid_windows"))
            docw = torch.cat(_drain(nc.doc_window_batches(W, subsample, B, seed, epoch), "valid_windows"))
            assert docw.shape[1] == 2 + 2 * W
            assert torch.equal(torch.cat([docw[:, :1], docw[:, 2:]], 1), wref)
            assert docw[:, 1].tolist() == [2 * V + line_of[int(c - 1) // 2] for c in docw[:, 0]]


def test_doc_window_stream_rejects_a_window_over_15(tmp_path):
    from adapm_b200.utils.text import NativeCorpus

    path = str(tmp_path / "docs.txt")
    _line_corpus(path)
    nc = NativeCorpus.build(path, 2).encode(path)
    with pytest.raises(ValueError):
        next(nc.doc_window_batches(16, 0.0, 8, 1))


# ---------------------------------------------------------------------------------------------- the inference rule
M64 = (1 << 64) - 1


def _mix(x):
    x &= M64
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & M64
    return x ^ (x >> 33)


def _oracle(rows, words, t, tab, dm, d, neg, win, E, alpha, min_alpha, seed):
    """one document, one position at a time, in Python floats (float64); rows: key -> float64 [d]"""
    prob, alias, n, first, stride = tab
    base = _mix(_mix(seed) ^ (t & M64))
    v = np.array([np.float32((np.float32((_mix(base ^ ((1 << 63) | k)) >> 40) * 2.0 ** -24) - np.float32(0.5))
                             / np.float32(d)) for k in range(d)], dtype=np.float64)
    a = np.full(d, float(np.float32(1e-6)))
    total = 0.0
    L = len(words)
    for e in range(E):
        ae = alpha - e * (alpha - min_alpha) / max(1, E - 1)
        es = _mix(base ^ ((1 << 62) | e))
        for i in range(L):
            pos = 2 * words[i] + 1
            targets = [(pos, 1.0)]
            for j in range(neg):
                h = _mix(es ^ (((i * neg + j) * 0x9E3779B97F4A7C15) & M64))
                hi, lo = h >> 32, h & 0xFFFFFFFF
                b = (hi * n) >> 32
                u = np.float32(lo) * np.float32(2.0 ** -32)
                key = first + (b if u < prob[b] else int(alias[b])) * stride
                if key != pos:
                    targets.append((key, 0.0))
            hv = v.copy()
            if dm:
                r = win - _mix(_mix(es) ^ i) % win
                ctx = [j for j in range(max(0, i - r), min(L, i + r + 1)) if j != i]
                for j in ctx:
                    hv = hv + rows[2 * words[j]]
                hv = hv / (1 + len(ctx))
            neu = np.zeros(d)
            for key, label in targets:
                f = float(hv @ rows[key])
                g = label - 1 if f > 6 else (label if f < -6 else label - 1 / (1 + np.exp(-f)))
                z = min(6.0, max(-6.0, f if label else -f))
                total += np.log1p(np.exp(-z))
                neu += g * rows[key]
            v = v + ae * neu / np.sqrt(a + neu * neu)
            a = a + neu * neu
    return v, total


def _random_store(s, kv, V, d, seed, scale=0.6):
    """every word key gets a random row (scaled so that some scores saturate), accumulators 1"""
    g = torch.Generator().manual_seed(seed)
    rows = torch.ones(2 * V, 2 * d)
    rows[:, :d] = (torch.rand(2 * V, d, generator=g) - 0.5) * scale
    kv.begin_setup()
    kv.wait(kv.set(torch.arange(2 * V, dtype=torch.int64), rows.view(-1)))
    kv.end_setup()
    return {k: rows[k, :d].double().numpy() for k in range(2 * V)}


@pytest.mark.parametrize("dm", [0, 1])
@pytest.mark.parametrize("V", [3, 40])
def test_reference_matches_a_per_document_loop(dm, V):
    from adapm_b200.ops import DeviceSampler, doc2vec_infer_reference

    d, neg, win, E = 8, 4, 3, 3
    with one_rank_store(2 * d, 2 * V + 5, "cpu", "float32") as (s, kv):
        rows = _random_store(s, kv, V, d, 3 + V)
        counts = np.arange(V, 0, -1, dtype=np.float64) ** 1.5
        sp = DeviceSampler(s, weights=torch.from_numpy(counts ** 0.75), first_key=1, key_stride=2)
        rng = np.random.default_rng(V)
        docs = [rng.integers(0, V, n).tolist() for n in (0, 1, 2, 7, 7)]
        ids = [5, 17, 2 ** 40 + 3, 0, 1]
        off = np.concatenate([[0], np.cumsum([len(x) for x in docs])])
        tok = np.array(sum(docs, []), dtype=np.int64)
        kw = dict(dm=bool(dm), embed_dim=d, negative=neg, window=win, epochs=E, alpha=0.05, min_alpha=0.01, seed=77)
        got, loss = doc2vec_infer_reference(kv, torch.from_numpy(tok), torch.from_numpy(off.astype(np.int64)),
                                            torch.tensor(ids), sp, **kw)
        tab = (sp.prob.numpy(), sp.alias.numpy(), sp.n, sp.first_key, sp.key_stride)
        total = 0.0
        for m, doc in enumerate(docs):
            want, lw = _oracle(rows, doc, ids[m], tab, dm, d, neg, win, E, 0.05, 0.01, 77)
            np.testing.assert_allclose(got[m], want, rtol=1e-12, atol=1e-14)
            total += lw
        assert loss == pytest.approx(total, rel=1e-12)
        if V == 3:        # the tiny vocabulary makes draws equal to the positive: they must have been skipped
            n_eq = 0
            for m, doc in enumerate(docs):
                base = _mix(_mix(77) ^ ids[m])
                es = _mix(base ^ (1 << 62))
                for i, w in enumerate(doc):
                    for j in range(neg):
                        h = _mix(es ^ (((i * neg + j) * 0x9E3779B97F4A7C15) & M64))
                        b = ((h >> 32) * V) >> 32
                        u = np.float32(h & 0xFFFFFFFF) * np.float32(2.0 ** -32)
                        n_eq += (b if u < tab[0][b] else tab[1][b]) == w
            assert n_eq > 0


def test_reference_draws_are_the_sampler_replay():
    """the draws of one document's epoch are sample_keys_reference with the epoch seed"""
    from adapm_b200.ops import _mix64_int, sample_keys_reference

    prob = np.array([0.5, 1.0, 0.25], dtype=np.float32)
    alias = np.array([1, 1, 1], dtype=np.int32)
    t, e, seed, neg, i = 12, 2, 99, 5, 3
    es = _mix64_int(_mix64_int(_mix64_int(seed) ^ t) ^ ((1 << 62) | e))
    keys = sample_keys_reference((i + 1) * neg, es, prob=prob, alias=alias, first_key=1, key_stride=2)
    for j in range(neg):
        h = _mix(es ^ (((i * neg + j) * 0x9E3779B97F4A7C15) & M64))
        b = ((h >> 32) * 3) >> 32
        u = np.float32(h & 0xFFFFFFFF) * np.float32(2.0 ** -32)
        assert keys[i * neg + j] == 1 + 2 * (b if u < prob[b] else alias[b])


def test_initial_vectors_depend_on_id_and_seed_only():
    from adapm_b200.ops import doc2vec_initial_vectors

    a = doc2vec_initial_vectors(3, [4, 9, 4], 12)
    assert a.dtype == np.float32 and np.array_equal(a[0], a[2]) and not np.array_equal(a[0], a[1])
    assert np.abs(a).max() <= 0.5 / 12 and not np.array_equal(a, doc2vec_initial_vectors(4, [4, 9, 4], 12))


# ---------------------------------------------------------------------------------------------- layout
def _model(s, kv, path, **kw):
    from adapm_b200.models.doc2vec import Doc2Vec, Doc2VecConfig
    from adapm_b200.utils.text import NativeCorpus

    nc = NativeCorpus.build(path, kw.pop("min_count", 2)).encode(path, s.my_rank(), s.num_servers())
    cfg = Doc2VecConfig(**{**dict(embed_dim=8, window=2, negative=3, batch_pairs=16, batch_windows=8, epochs=2,
                                  subsample=0.0), **kw})
    return Doc2Vec(s, kv, cfg, nc)


def _rows(kv, keys, d):
    out = torch.empty(len(keys) * 2 * d)
    kv.wait(kv.pull(torch.as_tensor(keys, dtype=torch.int64), out))
    return out.view(len(keys), 2 * d)


@pytest.mark.parametrize("dm", [0, 1])
def test_layout_init_sampler_and_steps(tmp_path, dm):
    from adapm_b200.models.doc2vec import num_keys
    from adapm_b200.ops import sample_keys_reference

    path = str(tmp_path / "docs.txt")
    _line_corpus(path)
    from adapm_b200.utils.text import NativeCorpus

    V = len(NativeCorpus.build(path, 2).vocabulary().words)
    d = 8
    with one_rank_store(2 * d, num_keys(V, 11), "cpu", "float32") as (s, kv):
        m = _model(s, kv, path, dm=dm, dbow_words=1)
        m.init_model()
        docs = _rows(kv, list(range(2 * V, 2 * V + 11)), d)
        syn0 = _rows(kv, list(range(0, 2 * V, 2)), d)
        for r in (docs, syn0):
            assert bool((r[:, d:] == np.float32(1e-6)).all())
            assert float(r[:, :d].abs().max()) <= 0.5 / d and float(r[:, :d].abs().min()) > 0
        assert len(torch.unique(docs[:, :d], dim=0)) == 11
        draws = sample_keys_reference(1 << 16, 5, prob=m.sampler.prob, alias=m.sampler.alias, first_key=1, key_stride=2)
        assert draws.min() >= 1 and draws.max() < 2 * V and bool((draws % 2 == 1).all())
        before = _rows(kv, list(range(num_keys(V, 11))), d)
        b = next(iter(m.batches(0)))
        valid = b.valid_windows if dm else b.valid_pairs
        for _ in range(2):      # syn1 rows start at zero: the input rows move from the second step on
            m.w2v.step(b[:valid] if dm else b[:, :valid].contiguous())
        after = _rows(kv, list(range(num_keys(V, 11))), d)
        changed = set(torch.nonzero((after != before).any(1)).view(-1).tolist())
        touched = set(b[b >= 0].tolist())
        assert changed and changed <= touched | set(range(1, 2 * V, 2))   # and the negatives, syn1 keys
        assert {k for k in changed if k >= 2 * V} == {k for k in touched if k >= 2 * V}


# ---------------------------------------------------------------------------------------------- input checks
def test_invalid_configs_raise_value_error(tmp_path):
    from adapm_b200.models.doc2vec import num_keys

    path = str(tmp_path / "docs.txt")
    _line_corpus(path)
    with one_rank_store(16, num_keys(40, 11), "cpu", "float32") as (s, kv):
        for kw in (dict(hs=True), dict(negative=0), dict(dm=1, window=16), dict(epochs=0), dict(min_alpha=0.0),
                   dict(dm=2)):
            with pytest.raises(ValueError):
                _model(s, kv, path, **kw)
    with one_rank_store(16, 10, "cpu", "float32") as (s, kv):   # too few keys for the documents
        with pytest.raises(ValueError):
            _model(s, kv, path)


def test_inference_arguments_are_checked_before_anything_runs():
    from adapm_b200.ops import DeviceSampler, doc2vec_infer_reference

    with one_rank_store(16, 20, "cpu", "float32") as (s, kv):
        sp = DeviceSampler(s, weights=torch.ones(10), first_key=1, key_stride=2)
        tok, off, ids = torch.tensor([1, 2, 3]), torch.tensor([0, 1, 3]), torch.tensor([0, 1])
        good = dict(dm=True, embed_dim=8, negative=3, window=2, epochs=2, alpha=0.05, min_alpha=0.01, seed=1)
        doc2vec_infer_reference(kv, tok, off, ids, sp, **good)
        for bad in (dict(embed_dim=6), dict(embed_dim=340), dict(negative=0), dict(negative=32), dict(window=16),
                    dict(window=0), dict(epochs=0), dict(min_alpha=0.0), dict(min_alpha=0.1)):
            with pytest.raises(ValueError):
                doc2vec_infer_reference(kv, tok, off, ids, sp, **{**good, **bad})
        with pytest.raises(TypeError):
            doc2vec_infer_reference(kv, tok, off, ids, sp, **{**good, "embed_dim": 8.0})
        with pytest.raises(ValueError):                                      # word 3 is not one of 3 words
            doc2vec_infer_reference(kv, tok, off, ids, sp, num_words=3, **good)
        for args, exc in (((torch.tensor([1, 2, 10]), off, ids), ValueError),         # word id out of range
                          ((torch.tensor([1, 2, -1]), off, ids), ValueError),
                          ((tok, torch.tensor([0, 2, 1]), ids), ValueError),          # not monotone
                          ((tok, torch.tensor([0, 1, 2]), ids), ValueError),          # does not end at the tokens
                          ((tok, torch.tensor([0, 3]), ids), ValueError),             # M + 1 offsets
                          ((tok.int(), off, ids), TypeError),
                          ((tok, off, ids.float()), TypeError),
                          ((torch.zeros(10001, dtype=torch.int64), torch.tensor([0, 10001]), torch.tensor([0])),
                           ValueError)):                                               # over 10 000 words
            with pytest.raises(exc):
                doc2vec_infer_reference(kv, *args, sp, **good)


# ---------------------------------------------------------------------------------------------- quality
def planted_corpus(path, n_docs=400, n_held=80, K=8, seed=1):
    """K topics with 30 words each over 300 Zipf background words; a document of 40-80 words takes 60 % of them from
    its topic. Returns (topics of the training documents, held-out documents as word lists, their topics)."""
    rng = np.random.default_rng(seed)
    bg = np.arange(1, 301) ** -1.0
    bg /= bg.sum()

    def doc(k):
        n = int(rng.integers(40, 81))
        own = rng.random(n) < 0.6
        return [f"t{k}_{rng.integers(0, 30)}" if o else f"b{rng.choice(300, p=bg)}" for o in own]

    topics = rng.integers(0, K, n_docs)
    with open(path, "w") as f:
        f.writelines(" ".join(doc(k)) + "\n" for k in topics)
    held_topics = rng.integers(0, K, n_held)
    return topics, [doc(k) for k in held_topics], held_topics


def train_planted(backend, path, dm, **kw):
    """Returns (own-topic share of the 10 nearest training documents, share of held-out documents whose nearest
    training document has their topic, per-epoch (loss, items), the trained document vectors on the host)."""
    from adapm_b200.models.doc2vec import Doc2Vec, Doc2VecConfig, num_keys
    from adapm_b200.utils.text import NativeCorpus

    topics, held, held_topics = planted_corpus(path)
    nc = NativeCorpus.build(path, 1)
    cfg = Doc2VecConfig(**{**dict(dm=dm, embed_dim=32, window=4, negative=5, epochs=15, alpha=0.05, min_alpha=0.005,
                                  batch_pairs=2048, batch_windows=1024, subsample=0.0, infer_epochs=30,
                                  infer_alpha=0.05, infer_min_alpha=0.005, model_seed=11), **kw})
    V, D = len(nc.vocabulary().words), len(topics)
    with one_rank_store(cfg.row_len, num_keys(V, D), backend, "float32") as (s, kv):
        nc.encode(path, 0, 1)
        m = Doc2Vec(s, kv, cfg, nc)
        m.init_model()
        losses = m.train()
        idx, _ = m.most_similar_docs(np.arange(D), 10)
        vec = m.infer(held)
        near, _ = m.most_similar_docs(vec, 1)
        vecs = m.doc_vectors().cpu()
    idx, near = idx.cpu().numpy(), near.cpu().numpy()
    share = float(np.mean(topics[idx] == topics[:, None]))
    inferred = float(np.mean(topics[near[:, 0]] == held_topics))
    return share, inferred, losses, vecs


@pytest.mark.parametrize("dm", [0, 1])
def test_cpu_quality_on_planted_topics(tmp_path, dm):
    share, inferred, losses, _ = train_planted("cpu", str(tmp_path / "topics.txt"), dm)
    print(f"planted topics dm={dm}: own-topic share of the 10 nearest {share:.3f}, held-out nearest topic "
          f"{inferred:.3f} (chance 0.125), losses {[round(l / max(1, n), 4) for l, n in losses]}")
    assert losses[-1][0] / losses[-1][1] < losses[0][0] / losses[0][1]
    assert share >= SHARE_MIN and inferred >= INFER_MIN, (share, inferred)


# ---------------------------------------------------------------------------------------------- app
def _app(args, world=2):
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu",
                        "-m", "adapm_b200.apps.doc2vec", "--"] + args, cwd=ROOT, capture_output=True, text=True,
                       timeout=300)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("dm", [0, 1])
def test_app_runs_on_two_cpu_ranks_and_writes_vectors(tmp_path, dm):
    from adapm_b200.models.word2vec import read_word2vec_binary

    path = str(tmp_path / "docs.txt")
    _, held, _ = planted_corpus(path, n_docs=60, n_held=5)
    with open(tmp_path / "new.txt", "w") as f:
        f.writelines(" ".join(h) + "\n" for h in held)
    out, docs, inf = (str(tmp_path / n) for n in ("words.bin", "docs.bin", "inferred.bin"))
    rc, log = _app(["--input_file", path, "--output_file", out, "--doc_output_file", docs, "--infer_file",
                    str(tmp_path / "new.txt"), "--infer_output_file", inf, "--embed_dim", "16", "--window", "3",
                    "--negative", "3", "--min_count", "1", "--num_iterations", "2", "--batch_pairs", "512",
                    "--batch_windows", "256", "--dm", str(dm), "--dbow_words", "1", "--infer_epochs", "5"])
    assert rc == 0, log[-3000:]
    assert "[d2v] epoch 1 done" in log and "protocol errors 0" in log, log[-3000:]
    words, wv = read_word2vec_binary(out)
    names, dv = read_word2vec_binary(docs)
    inames, iv = read_word2vec_binary(inf)
    assert wv.shape[1] == dv.shape[1] == iv.shape[1] == 16
    assert names == [str(j) for j in range(60)] and inames == [str(j) for j in range(5)]
    assert np.isfinite(dv).all() and np.isfinite(iv).all()


@pytest.mark.parametrize("flags,message", [
    (["--dm", "1", "--window", "16"], "--window must be in [1, 15] with --dm 1"),
    (["--negative", "0"], "--negative must be at least 1"),
    (["--infer_file", "x.txt"], "--infer_file needs --infer_output_file"),
])
def test_app_rejects_invalid_flags(flags, message, tmp_path):
    path = str(tmp_path / "docs.txt")
    planted_corpus(path, n_docs=20, n_held=1)
    rc, log = _app(["--input_file", path, "--output_file", str(tmp_path / "v.bin"), "--num_iterations", "1"] + flags,
                   world=1)
    assert rc != 0 and message in log, log[-2000:]


# ---------------------------------------------------------------------------------------------- build facts
def test_inference_kernels_do_not_spill():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    for name in ("doc2vec_infer_kernel<false>", "doc2vec_infer_kernel<true>"):
        assert name in k, sorted(n for n in k if "doc2vec" in n)
        assert k[name]["spill"] == 0, (name, k[name])
