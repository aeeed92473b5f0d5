"""word2vec CBOW without a GPU: the fp32 Pull / Push step ``cbow_reference_step`` against an independent float64 NumPy
form of the rule, the window loaders (native ``NativeCorpus.window_batches`` and NumPy ``windows_from_sentences``),
the app on two CPU ranks, and a learning check on a planted-topic corpus."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = os.path.join(ROOT, "data", "lm", "small.txt")


def _server(row_len, num_keys, job, backend="cpu", dtype="float32"):
    import adapm_b200 as ad

    s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend=backend, fabric="inproc",
                  job=f"{job}_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def numpy_rule(table, centers, contexts, negatives, d, alpha):
    """The CBOW rule in float64 on a dense table [keys, 2 d] (a new table and the summed loss): every window reads the
    start-of-step table; h = mean of the context embeddings (repeats count), targets the centre (label 1) and the
    negatives (label 0, one equal to the centre skipped); one AdaGrad contribution per (window, target) and one per
    context occurrence, all added up."""
    t = np.asarray(table, dtype=np.float64)
    out = t.copy()
    loss = 0.0
    centers, contexts, negatives = np.asarray(centers), np.asarray(contexts), np.asarray(negatives)
    for w in range(centers.shape[0]):
        c = int(centers[w])
        ctx = [int(k) for k in contexts[w] if k >= 0]
        if c < 0 or not ctx:
            continue
        h = sum(t[k, :d] for k in ctx) / len(ctx)
        neu = np.zeros(d)
        for j, k in enumerate([c] + [int(x) for x in negatives[w]]):
            if j > 0 and k == c:
                continue
            label = 1.0 if j == 0 else 0.0
            f = float(h @ t[k, :d])
            g = label - 1 if f > 6 else (label if f < -6 else label - 1 / (1 + np.exp(-f)))
            z = min(max(f if label else -f, -6.0), 6.0)
            loss += np.log1p(np.exp(-z))
            neu += g * t[k, :d]
            gr = g * h
            out[k, :d] += alpha * gr / np.sqrt(t[k, d:] + gr * gr)
            out[k, d:] += gr * gr
        for k in ctx:
            out[k, :d] += alpha * neu / np.sqrt(t[k, d:] + neu * neu)
            out[k, d:] += neu * neu
    return out, loss


def torch_rule64(table, centers, contexts, negatives, d, alpha, chunk=1024):
    """numpy_rule vectorised in float64 torch (for the GPU tests' batch sizes): (new table, loss)"""
    t = table.double()
    out = t.clone()
    loss = 0.0
    for a in range(0, centers.numel(), chunk):
        c, x, n = centers[a:a + chunk], contexts[a:a + chunk], negatives[a:a + chunk]
        B, C = x.shape
        T = n.shape[1] + 1
        xm = (x >= 0) & (c >= 0).view(B, 1)
        cnt = xm.sum(1)
        act = (c >= 0) & (cnt > 0)
        xm &= act.view(B, 1)
        xk = x.clamp(min=0)
        h = (t[xk, :d] * xm.unsqueeze(-1)).sum(1) / cnt.clamp(min=1).view(B, 1)
        tk = torch.cat([c.view(B, 1), n], 1).clamp(min=0)
        tm = act.view(B, 1).repeat(1, T)
        tm[:, 1:] &= n != c.view(B, 1)
        et, at = t[tk, :d], t[tk, d:]
        label = torch.zeros(B, T, dtype=torch.float64)
        label[:, 0] = 1
        f = (h.unsqueeze(1) * et).sum(-1)
        g = torch.where(f > 6, label - 1, torch.where(f < -6, label, label - torch.sigmoid(f))) * tm
        neu = (g.unsqueeze(-1) * et).sum(1)
        gr = g.unsqueeze(-1) * h.unsqueeze(1)
        out.index_add_(0, tk[tm], torch.cat([alpha * gr / torch.sqrt(at + gr * gr), gr * gr], -1)[tm])
        gx = neu.unsqueeze(1).expand(B, C, d)
        ax = t[xk, d:]
        out.index_add_(0, xk[xm], torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)[xm])
        z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
        loss += float((torch.log1p(torch.exp(-z)) * tm).sum())
    return out, loss


def corner_batch(g, vocab, B, C, neg):
    """windows with every corner of the rule: padding rows (centre -1), windows without contexts, a context word repeated
    in one window, negatives equal to the centre, and words that are a context in one window and a target in another"""
    centers = 2 * torch.randint(0, vocab, (B,), generator=g) + 1
    lens = torch.randint(0, C + 1, (B,), generator=g)
    contexts = torch.full((B, C), -1, dtype=torch.int64)
    for w in range(B):
        n = int(lens[w])
        contexts[w, :n] = 2 * torch.randint(0, vocab, (n,), generator=g)
    negatives = 2 * torch.randint(0, vocab, (B, neg), generator=g) + 1
    centers[B - 3:] = -1                                  # padding rows (their contexts must not train either)
    contexts[B - 2, :2] = 2 * 3
    contexts[0, :] = -1                                   # a window without context
    contexts[1, :3] = torch.tensor([10, 10, 10])          # word 5 three times in one window
    negatives[2, :] = centers[2]                          # every negative equal to the centre
    negatives[3, 0] = centers[3]
    centers[4] = 2 * 7 + 1                                # word 7: target here ...
    contexts[5, 0] = 2 * 7                                # ... and context there
    return centers, contexts, negatives


def _table(g, vocab, d):
    t = torch.randn(2 * vocab, 2 * d, generator=g) * 0.4
    t[:, d:] = torch.rand(2 * vocab, d, generator=g) + 1e-3
    return t


def test_reference_step_matches_float64_rule():
    from adapm_b200.models.word2vec import cbow_reference_step

    vocab, d, alpha = 60, 12, 0.2
    g = torch.Generator().manual_seed(5)
    table = _table(g, vocab, d)
    server, kv = _server(2 * d, 2 * vocab, "cbowref")
    try:
        kv.wait(kv.set(torch.arange(2 * vocab), table.contiguous().view(-1)))
        ref = table.double().numpy()
        for step in range(3):
            c, x, n = corner_batch(g, vocab, 40, 8, 5)
            ref, ref_loss = numpy_rule(ref, c, x, n, d, alpha)
            loss = cbow_reference_step(kv, c, x, n, d, alpha)
            rows = torch.empty(2 * vocab * 2 * d)
            kv.wait(kv.pull(torch.arange(2 * vocab), rows))
            np.testing.assert_allclose(rows.view(2 * vocab, 2 * d).double().numpy(), ref, rtol=2e-5, atol=2e-6,
                                       err_msg=f"step {step}")
            assert loss == pytest.approx(ref_loss, rel=1e-5), step
    finally:
        kv.finalize()
        server.shutdown()


def test_vectorised_rule_matches_the_loop_form():
    g = torch.Generator().manual_seed(6)
    table = _table(g, 60, 8)
    c, x, n = corner_batch(g, 60, 50, 6, 4)
    a, la = numpy_rule(table, c, x, n, 8, 0.1)
    b, lb = torch_rule64(table, c, x, n, 8, 0.1, chunk=7)
    np.testing.assert_allclose(b.numpy(), a, rtol=1e-12, atol=1e-12)
    assert lb == pytest.approx(la, rel=1e-12)


# ---------------------------------------------------------------------------------------------- loaders
def _native(path=SMALL, min_count=1):
    from adapm_b200.utils.text import NativeCorpus

    return NativeCorpus.build(path, min_count).encode(path)


def _check_windows(batches, sentences, window, batch_windows):
    """every valid row is a centre with its neighbours inside a window shrink; padding rows are all -1. Returns the
    valid rows."""
    cols = 1 + 2 * window
    rows = []
    for b in batches:
        assert b.shape == (batch_windows, cols) and b.dtype == torch.int64
        v = b.valid_windows
        assert torch.all(b[v:] == -1)
        assert torch.all(b[:v, 0] >= 0) and torch.all(b[:v, 0] % 2 == 1)
        rows.append(b[:v])
    rows = torch.cat(rows)
    # walk the sentences in order: the centre words follow the (subsampled) corpus word by word
    i = 0
    for s in sentences:
        for pos in range(len(s)):
            r = rows[i]
            assert int(r[0]) == 2 * s[pos] + 1
            ctx = r[1:][r[1:] >= 0]
            assert torch.all(r[1 + ctx.numel():] == -1), "padding only after the contexts"
            n = ctx.numel()
            assert 1 <= n <= 2 * window
            # the contexts are s[lo:pos] + s[pos+1:hi] for a radius r in [1, window]
            ok = False
            for rad in range(1, window + 1):
                lo, hi = max(0, pos - rad), min(len(s), pos + rad + 1)
                exp = [2 * int(x) for x in list(s[lo:pos]) + list(s[pos + 1:hi])]
                if exp == ctx.tolist():
                    ok = True
                    break
            assert ok, (pos, ctx.tolist())
            i += 1
    assert i == rows.shape[0]
    return rows


def _expand(rows):
    ctx = rows[:, 1:]
    m = ctx >= 0
    return torch.stack([ctx[m], rows[:, :1].expand_as(ctx)[m]])


@pytest.mark.parametrize("window", [1, 5, 16])
def test_window_batches_cover_the_corpus_in_windows(window):
    nc = _native()
    sents = [s for s in nc.sentences() if len(s) >= 2]
    rows = _check_windows(list(nc.window_batches(window, 0.0, 777, seed=3, epoch=0)), sents, window, 777)
    assert rows.shape[0] == sum(len(s) for s in sents) == nc.num_tokens()


def test_window_batches_are_reproducible_and_match_pair_batches():
    nc = _native()
    for sub in (0.0, 1e-3):
        a = torch.cat([b[:b.valid_windows] for b in nc.window_batches(5, sub, 500, seed=11, epoch=1)])
        b = torch.cat([b[:b.valid_windows] for b in nc.window_batches(5, sub, 500, seed=11, epoch=1)])
        c = torch.cat([b[:b.valid_windows] for b in nc.window_batches(5, sub, 500, seed=11, epoch=2)])
        assert torch.equal(a, b)
        assert a.shape != c.shape or not torch.equal(a, c)
        pairs = torch.cat([p[:, :p.valid_pairs] for p in nc.pair_batches(5, sub, 1000, seed=11, epoch=1)], 1)
        assert torch.equal(_expand(a), pairs), sub
    # subsampling drops words: fewer windows than corpus words
    assert a.shape[0] < nc.num_tokens()


def test_window_batches_unique_keys_and_padding():
    nc = _native()
    bs = list(nc.window_batches(3, 0.0, 4096, seed=1))
    last = bs[-1]
    assert last.valid_windows < 4096 and torch.all(last[last.valid_windows:] == -1)
    for b in bs:
        k = b[b >= 0]
        assert torch.equal(torch.sort(b.unique_keys).values, torch.unique(k))
    with pytest.raises(ValueError):
        next(nc.window_batches(17, 0.0, 10, seed=1))


def test_numpy_windows_from_sentences():
    from adapm_b200.utils.text import pairs_from_sentences, windows_from_sentences

    g = np.random.default_rng(0)
    sents = [g.integers(0, 50, size=int(n)) for n in g.integers(2, 30, size=80)]
    bs = list(windows_from_sentences(iter(sents), 4, 64, np.random.default_rng(9)))
    rows = _check_windows(bs, sents, 4, 64)
    assert rows.shape[0] == sum(len(s) for s in sents)
    pairs = torch.cat(list(pairs_from_sentences(iter(sents), 4, 100, np.random.default_rng(9))), 1)
    assert torch.equal(_expand(rows), pairs)


def test_synthetic_windows_are_shrunk_windows():
    from adapm_b200.models.word2vec import SyntheticWindows, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=1000, window=5, batch_windows=300, cbow=True)
    b = SyntheticWindows(cfg, zipf_counts(1000), 0).batch(0)
    assert b.shape == (300, 11) and torch.all(b[:, 0] % 2 == 1)
    n = (b[:, 1:] >= 0).sum(1)
    assert torch.all(n % 2 == 0) and torch.all((n >= 2) & (n <= 10))
    assert torch.all(b[:, 1:][b[:, 1:] >= 0] % 2 == 0)


# ---------------------------------------------------------------------------------------------- model and app
def test_cbow_option_checks():
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig

    server, kv = _server(8, 200, "cbowchk")
    try:
        with pytest.raises(ValueError):
            Word2Vec(server, kv, Word2VecConfig(vocab_size=100, embed_dim=4, cbow=True, shared_negatives=32))
        m = Word2Vec(server, kv, Word2VecConfig(vocab_size=100, embed_dim=4, cbow=True))
        with pytest.raises(ValueError):
            m.run_steps([], 0, 0)
    finally:
        kv.finalize()
        server.shutdown()


def _launch(args, world=2):
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu"] + args, cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.parametrize("loader", ["native", "python"])
def test_app_cbow_two_ranks_with_checkpoint_roundtrip(tmp_path, loader):
    base = ["-m", "adapm_b200.apps.word2vec", "--", "--input_file", SMALL, "--embed_dim", "16", "--num_iterations", "1",
            "--min_count", "5", "--negative", "3", "--cbow", "1", "--batch_windows", "2048", "--loader", loader]
    ck = str(tmp_path / "vec")
    rc, out = _launch(base + ["--write_results", "1", "--output_file", ck])
    assert rc == 0 and os.path.exists(ck + ".epoch.0"), out[-2000:]
    assert "windows on rank 0" in out, out[-2000:]
    rc, out = _launch(base + ["--init_model", ck + ".epoch.0", "--data_words", "4000"])
    assert rc == 0 and "initialised" in out, out[-2000:]
    rc, out = _launch(base + ["--shared_negatives", "32"])
    assert rc != 0 and "ValueError" in out, out[-2000:]


# ---------------------------------------------------------------------------------------------- learning check
TOPICS, PER_TOPIC = 40, 25
# Mean share of each word's 10 nearest words (most_similar) that share its topic after 4 epochs; measured 1.00 on the
# CPU backend (fp32 Pull / Push) and 1.00 with the deterministic step on an H100, against 0.02 for random vectors.
TOPIC_PRECISION = 0.8


def planted_corpus(seed=0, n_sent=3000, length=12):
    """sentences of `length` words drawn uniformly from one of TOPICS topics of PER_TOPIC words (word ids 1.. : id 0 is
    the sentence delimiter of the vocabulary)"""
    g = np.random.default_rng(seed)
    topic = g.integers(0, TOPICS, n_sent)
    return [1 + t * PER_TOPIC + g.integers(0, PER_TOPIC, length) for t in topic]


def train_planted(backend, epochs=4, seed=0, d=32):
    """CBOW on the planted corpus; returns (per-epoch mean loss, topic precision, syn0 rows)"""
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig
    from adapm_b200.utils.text import windows_from_sentences

    V = 1 + TOPICS * PER_TOPIC
    cfg = Word2VecConfig(vocab_size=V, embed_dim=d, negative=5, window=4, starting_alpha=0.05, batch_windows=1024,
                         cbow=True, model_seed=seed + 1)
    kw = {"device": 0} if backend == "cuda" else {}
    import adapm_b200 as ad

    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend=backend,
                       fabric="inproc", job=f"planted_{np.random.randint(1 << 30)}", **kw)
    kv = ad.Worker(0, server)
    try:
        counts = np.ones(V)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        sents = planted_corpus(seed)
        losses = []
        for ep in range(epochs):
            tot, n = 0.0, 0
            for b in windows_from_sentences(iter(sents), cfg.window, cfg.batch_windows, np.random.default_rng([seed, ep])):
                if model.cuda:
                    model.loss.zero_()
                loss = model.step(b.pin_memory() if model.cuda else b)
                tot += float(loss.sum())
                n += b.valid_windows * (cfg.negative + 1)
                kv.advance_clock()
            losses.append(tot / n)
            model.set_alpha((ep + 1) / epochs)
        words = torch.arange(1, V)
        idx, _ = model.most_similar(words, k=10)
        idx = idx.cpu()
        same = ((idx - 1) // PER_TOPIC) == ((words.view(-1, 1) - 1) // PER_TOPIC)
        prec = float(same.double().mean())
        rows = torch.empty(V * 2 * d, device=server.device if model.cuda else "cpu")
        kv.wait(kv.pull(torch.arange(V, device=rows.device) * 2, rows, model.cuda))
        return losses, prec, rows.cpu()
    finally:
        kv.finalize()
        server.shutdown()


def test_cbow_learns_planted_topics_on_cpu():
    losses, prec, _ = train_planted("cpu")
    print(f"cpu planted topics: losses {losses}, topic precision {prec:.3f}")
    assert losses[-1] < losses[0]
    assert prec > TOPIC_PRECISION, prec
