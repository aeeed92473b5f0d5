"""word2vec hierarchical softmax without a GPU: the Huffman tree (against a transcription of word2vec.c's construction,
prefix-freeness, Kraft's equality and the Huffman cost), the fp32 Pull / Push step ``hs_reference_step`` against
independent float64 forms of the rule, the app on two CPU ranks, and a learning check on the planted-topic corpus."""
import heapq
import os

import numpy as np
import pytest
import torch

from test_cbow_cpu import PER_TOPIC, SMALL, TOPIC_PRECISION, TOPICS, _launch, _server, planted_corpus


# ---------------------------------------------------------------------------------------------- the tree
def w2v_c_tree(counts):
    """word2vec.c's CreateBinaryTree, transcribed: words sorted by count (descending, ties by id), the two-queue merge.
    Returns per word id (path of inner nodes root first, code bits root first)."""
    V = len(counts)
    order = sorted(range(V), key=lambda w: (-counts[w], w))
    count = [float(counts[w]) for w in order] + [1e300] * V
    binary, parent = [0] * (2 * V), [0] * (2 * V)
    pos1, pos2 = V - 1, V
    for a in range(V - 1):
        mins = []
        for _ in range(2):
            if pos1 >= 0 and count[pos1] < count[pos2]:
                mins.append(pos1); pos1 -= 1
            else:
                mins.append(pos2); pos2 += 1
        count[V + a] = count[mins[0]] + count[mins[1]]
        parent[mins[0]] = parent[mins[1]] = V + a
        binary[mins[1]] = 1
    out = [None] * V
    for p in range(V):
        code, point, b = [], [], p
        while True:
            code.append(binary[b]); point.append(b)
            b = parent[b]
            if b == 2 * V - 2:
                break
        n = len(code)
        path = [V - 2] + [point[n - i] - V for i in range(1, n)]        # vocab[a].point[n - b] = point[b] - V
        out[order[p]] = (path, code[::-1])
    return out


def _paths(tree):
    off, nodes, codes = tree.offsets.numpy(), tree.nodes.numpy(), tree.codes.numpy().view(np.uint32)
    return [(list(nodes[off[w]:off[w + 1]]), [int(codes[w] >> j) & 1 for j in range(off[w + 1] - off[w])])
            for w in range(len(codes))]


@pytest.mark.parametrize("V,seed", [(2, 0), (3, 1), (3, 2), (300, 3), (517, 4)])
def test_tree_matches_word2vec_c_construction(V, seed):
    from adapm_b200.utils.text import huffman_tree

    g = np.random.default_rng(seed)
    counts = g.integers(1, 8, V)            # many ties
    tree = huffman_tree(counts)
    assert _paths(tree) == w2v_c_tree(list(counts))
    assert tree.max_len == max(len(p) for p, _ in w2v_c_tree(list(counts)))
    assert tree.offsets.dtype == torch.int64 and tree.nodes.dtype == torch.int32 and tree.codes.dtype == torch.int32


@pytest.mark.parametrize("V,seed", [(2, 0), (50, 1), (1000, 2)])
def test_tree_is_prefix_free_kraft_and_optimal(V, seed):
    from adapm_b200.utils.text import huffman_tree

    g = np.random.default_rng(seed)
    counts = np.floor(1e4 / np.arange(1, V + 1) ** 1.1) + g.integers(1, 3, V)
    tree = huffman_tree(counts)
    paths = _paths(tree)
    words = ["".join(map(str, c)) for _, c in paths]
    assert len(set(words)) == V
    srt = sorted(words)
    assert not any(b.startswith(a) for a, b in zip(srt, srt[1:]))
    assert sum(2.0 ** -len(c) for c in words) == 1.0
    # the same code prefix walks the same inner nodes: a path is determined by its code bits
    node_of = {}
    for p, c in paths:
        for j in range(len(c)):
            assert node_of.setdefault("".join(map(str, c[:j])), p[j]) == p[j]
    assert sorted(set(n for p, _ in paths for n in p)) == list(range(V - 1))
    h = [float(c) for c in counts]
    heapq.heapify(h)
    cost = 0.0
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        cost += a + b
        heapq.heappush(h, a + b)
    assert sum(counts[w] * len(paths[w][1]) for w in range(V)) == pytest.approx(cost, rel=1e-12)


def test_shuffled_counts_give_the_same_tree_up_to_the_permutation():
    from adapm_b200.utils.text import huffman_tree

    g = np.random.default_rng(7)
    counts = g.permutation(np.arange(1, 401) ** 2).astype(np.float64)   # distinct counts
    perm = g.permutation(400)
    shuffled = np.empty_like(counts)
    shuffled[perm] = counts                                             # word w is word perm[w] after the shuffle
    a, b = _paths(huffman_tree(counts)), _paths(huffman_tree(shuffled))
    assert all(a[w] == b[perm[w]] for w in range(400))


def test_tree_input_checks():
    from adapm_b200.utils.text import huffman_tree

    for bad in ([], [3.0], [1, 0, 2], [1, -1, 2], [1.0, float("nan")]):
        with pytest.raises(ValueError):
            huffman_tree(bad)
    fib = [1, 1]
    while len(fib) < 40:
        fib.append(fib[-1] + fib[-2])
    with pytest.raises(ValueError, match="39"):
        huffman_tree(fib)
    assert huffman_tree(fib[:33]).max_len == 32


# ---------------------------------------------------------------------------------------------- the rule
def numpy_hs_rule(table, centers, contexts, tree, d, alpha):
    """The hierarchical-softmax rule in float64 on a dense table [keys, 2 d] (a new table and the summed loss): every
    item reads the start-of-step table; h = mean of the context embeddings; node j of the centre word's path has label
    1 - code bit j; |f| >= 6 skips the node's update and its neu1e term but counts its loss."""
    t = np.asarray(table, dtype=np.float64)
    out = t.copy()
    loss = 0.0
    paths = _paths(tree)
    for i in range(len(centers)):
        c = int(centers[i])
        ctx = [int(k) for k in contexts[i] if k >= 0]
        if c < 0 or not ctx:
            continue
        h = sum(t[k, :d] for k in ctx) / len(ctx)
        neu = np.zeros(d)
        nodes, code = paths[c // 2]
        for n, bit in zip(nodes, code):
            k = 2 * n + 1
            label = 1.0 - bit
            f = float(h @ t[k, :d])
            z = min(max(f if label else -f, -6.0), 6.0)
            loss += np.log1p(np.exp(-z))
            if abs(f) >= 6:
                continue
            g = label - 1 / (1 + np.exp(-f))
            neu += g * t[k, :d]
            gr = g * h
            out[k, :d] += alpha * gr / np.sqrt(t[k, d:] + gr * gr)
            out[k, d:] += gr * gr
        for k in ctx:
            out[k, :d] += alpha * neu / np.sqrt(t[k, d:] + neu * neu)
            out[k, d:] += neu * neu
    return out, loss


def skipgram_hs_loop(table, syn1_words, syn0_words, tree, d, alpha):
    """Skip-gram hierarchical softmax as word2vec.c writes it, in float64: for each pair, syn0[last_word] is trained on
    the path of the other word (code, point); pairs read the start-of-step table and their updates add up."""
    t = np.asarray(table, dtype=np.float64)
    out = t.copy()
    loss = 0.0
    paths = _paths(tree)
    for word, last_word in zip(syn1_words, syn0_words):
        l1 = 2 * int(last_word)
        neu1e = np.zeros(d)
        point, code = paths[int(word)]
        for dd in range(len(code)):
            l2 = 2 * point[dd] + 1
            f = float(t[l1, :d] @ t[l2, :d])
            loss += np.log1p(np.exp(-min(max(f if code[dd] == 0 else -f, -6.0), 6.0)))
            if f <= -6 or f >= 6:
                continue
            g = 1 - code[dd] - 1 / (1 + np.exp(-f))
            neu1e += g * t[l2, :d]
            gr = g * t[l1, :d]
            out[l2, :d] += alpha * gr / np.sqrt(t[l2, d:] + gr * gr)
            out[l2, d:] += gr * gr
        out[l1, :d] += alpha * neu1e / np.sqrt(t[l1, d:] + neu1e * neu1e)
        out[l1, d:] += neu1e * neu1e
    return out, loss


def torch_hs_rule64(table, centers, contexts, tree, d, alpha, chunk=1024):
    """numpy_hs_rule vectorised in float64 torch (for the GPU tests' batch sizes): (new table, loss, skipped nodes)"""
    t = table.double()
    out = t.clone()
    loss, skipped = 0.0, 0
    off, nodes, codes = tree.offsets.cpu(), tree.nodes.cpu().long(), tree.codes.cpu()
    L = tree.max_len
    j = torch.arange(L)
    for a in range(0, centers.numel(), chunk):
        c, x = centers[a:a + chunk], contexts[a:a + chunk]
        B, C = x.shape
        xm = (x >= 0) & (c >= 0).view(B, 1)
        cnt = xm.sum(1)
        act = (c >= 0) & (cnt > 0)
        xm &= act.view(B, 1)
        xk = x.clamp(min=0)
        h = (t[xk, :d] * xm.unsqueeze(-1)).sum(1) / cnt.clamp(min=1).view(B, 1)
        w = torch.where(act, c // 2, torch.zeros_like(c))
        tm = act.view(B, 1) & (j.view(1, L) < (off[w + 1] - off[w]).view(B, 1))
        tk = 2 * nodes[torch.where(tm, off[w].view(B, 1) + j, torch.zeros_like(off[w]).view(B, 1))] + 1
        label = (1 - ((codes[w].view(B, 1) >> j.to(torch.int32)) & 1)).double()
        et, at = t[tk, :d], t[tk, d:]
        f = (h.unsqueeze(1) * et).sum(-1)
        um = tm & (f.abs() < 6)
        skipped += int((tm & ~um).sum())
        g = (label - torch.sigmoid(f)) * um
        neu = (g.unsqueeze(-1) * et).sum(1)
        gr = g.unsqueeze(-1) * h.unsqueeze(1)
        out.index_add_(0, tk[um], torch.cat([alpha * gr / torch.sqrt(at + gr * gr), gr * gr], -1)[um])
        gx = neu.unsqueeze(1).expand(B, C, d)
        ax = t[xk, d:]
        out.index_add_(0, xk[xm], torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)[xm])
        z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
        loss += float((torch.log1p(torch.exp(-z)) * tm).sum())
    return out, loss, skipped


def hs_corner_batch(g, vocab, B, C):
    """items with every corner of the rule: padding rows (centre -1), items without contexts, a context word repeated
    in one item, and a word that is a context in one item, a centre in another and (as inner node) on paths"""
    centers = 2 * torch.randint(0, vocab, (B,), generator=g) + 1
    lens = torch.randint(0, C + 1, (B,), generator=g)
    contexts = torch.full((B, C), -1, dtype=torch.int64)
    for i in range(B):
        n = int(lens[i])
        contexts[i, :n] = 2 * torch.randint(0, vocab, (n,), generator=g)
    centers[B - 3:] = -1                                  # padding rows (their contexts must not train either)
    contexts[B - 2, :1] = 2 * 3
    contexts[0, :] = -1                                   # an item without context
    contexts[1, :3] = torch.tensor([10, 10, 10])          # word 5 three times in one item
    centers[4] = 2 * 7 + 1                                # word 7: centre here ...
    contexts[5, 0] = 2 * 7                                # ... and context there
    return centers, contexts


def hs_table(g, vocab, d, big_nodes=()):
    """random rows; the syn1 rows of the inner nodes in big_nodes are scaled up so that their |f| often passes 6"""
    t = torch.randn(2 * vocab, 2 * d, generator=g) * 0.4
    t[:, d:] = torch.rand(2 * vocab, d, generator=g) + 1e-3
    for n in big_nodes:
        t[2 * n + 1, :d] *= 25
    return t


def _counts(vocab, seed):
    return np.random.default_rng(seed).integers(1, 1000, vocab).astype(np.float64)


def test_reference_step_matches_float64_rule():
    from adapm_b200.models.word2vec import hs_reference_step
    from adapm_b200.utils.text import huffman_tree

    vocab, d, alpha = 60, 12, 0.2
    g = torch.Generator().manual_seed(5)
    tree = huffman_tree(_counts(vocab, 1))
    table = hs_table(g, vocab, d, big_nodes=(vocab - 2, 3))
    server, kv = _server(2 * d, 2 * vocab, "hsref")
    try:
        kv.wait(kv.set(torch.arange(2 * vocab), table.contiguous().view(-1)))
        ref = table.double().numpy()
        skipped = 0
        for step in range(3):
            c, x = hs_corner_batch(g, vocab, 40, 8)
            _, _, sk = torch_hs_rule64(torch.from_numpy(ref), c, x, tree, d, alpha)
            skipped += sk
            ref, ref_loss = numpy_hs_rule(ref, c, x, tree, d, alpha)
            loss = hs_reference_step(kv, c, x, tree, d, alpha)
            rows = torch.empty(2 * vocab * 2 * d)
            kv.wait(kv.pull(torch.arange(2 * vocab), rows))
            np.testing.assert_allclose(rows.view(2 * vocab, 2 * d).double().numpy(), ref, rtol=2e-5, atol=2e-6,
                                       err_msg=f"step {step}")
            assert loss == pytest.approx(ref_loss, rel=1e-5), step
        assert skipped > 0                                # the |f| >= 6 rule was exercised
    finally:
        kv.finalize()
        server.shutdown()


def test_vectorised_rule_matches_the_loop_form():
    from adapm_b200.utils.text import huffman_tree

    g = torch.Generator().manual_seed(6)
    tree = huffman_tree(_counts(60, 2))
    table = hs_table(g, 60, 8, big_nodes=(58,))
    c, x = hs_corner_batch(g, 60, 50, 6)
    a, la = numpy_hs_rule(table, c, x, tree, 8, 0.1)
    b, lb, sk = torch_hs_rule64(table, c, x, tree, 8, 0.1, chunk=7)
    assert sk > 0
    np.testing.assert_allclose(b.numpy(), a, rtol=1e-12, atol=1e-12)
    assert lb == pytest.approx(la, rel=1e-12)


def test_one_context_is_word2vec_c_skipgram():
    from adapm_b200.models.word2vec import hs_reference_step
    from adapm_b200.utils.text import huffman_tree

    vocab, d, alpha = 50, 8, 0.1
    g = torch.Generator().manual_seed(8)
    tree = huffman_tree(_counts(vocab, 3))
    table = hs_table(g, vocab, d, big_nodes=(vocab - 2,))
    syn1_words = torch.randint(0, vocab, (64,), generator=g)
    syn0_words = torch.randint(0, vocab, (64,), generator=g)
    server, kv = _server(2 * d, 2 * vocab, "hssg")
    try:
        kv.wait(kv.set(torch.arange(2 * vocab), table.contiguous().view(-1)))
        ref, ref_loss = skipgram_hs_loop(table, syn1_words, syn0_words, tree, d, alpha)
        loss = hs_reference_step(kv, 2 * syn1_words + 1, (2 * syn0_words).view(-1, 1), tree, d, alpha)
        rows = torch.empty(2 * vocab * 2 * d)
        kv.wait(kv.pull(torch.arange(2 * vocab), rows))
        np.testing.assert_allclose(rows.view(2 * vocab, 2 * d).double().numpy(), ref, rtol=2e-5, atol=2e-6)
        assert loss == pytest.approx(ref_loss, rel=1e-5)
    finally:
        kv.finalize()
        server.shutdown()


# ---------------------------------------------------------------------------------------------- model and app
def test_hs_option_checks():
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig

    server, kv = _server(8, 200, "hschk")
    try:
        with pytest.raises(ValueError, match="not supported"):
            Word2Vec(server, kv, Word2VecConfig(vocab_size=100, embed_dim=4, hs=True))      # negative = 25
        with pytest.raises(ValueError, match="not supported"):
            Word2Vec(server, kv, Word2VecConfig(vocab_size=100, embed_dim=4, hs=True, negative=0, shared_negatives=32))
        m = Word2Vec(server, kv, Word2VecConfig(vocab_size=100, embed_dim=4, hs=True, negative=0))
        with pytest.raises(ValueError):
            m.run_steps([], 0, 0)
    finally:
        kv.finalize()
        server.shutdown()


def test_intent_keys_are_the_batch_syn0_keys_and_its_path_nodes():
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig

    vocab = 300
    server, kv = _server(8, 2 * vocab, "hsint")
    try:
        m = Word2Vec(server, kv, Word2VecConfig(vocab_size=vocab, embed_dim=4, hs=True, negative=0),
                     _counts(vocab, 4))
        g = np.random.default_rng(0)
        for _ in range(3):
            b = torch.from_numpy(np.stack([2 * g.integers(0, vocab, 500), 2 * g.integers(0, vocab, 500) + 1]))
            keys = m.intent_keys_hs(b.reshape(-1)).numpy()
            paths = _paths(m.tree)
            want = set(b[0].tolist()) | {2 * n + 1 for w in b[1].tolist() for n in paths[w // 2][0]}
            syn1 = keys[keys % 2 == 1]
            assert len(set(syn1.tolist())) == len(syn1)
            assert set(keys.tolist()) == want
            assert m.loss_terms(b) == sum(len(paths[w // 2][0]) for w in b[1].tolist())
    finally:
        kv.finalize()
        server.shutdown()


@pytest.mark.parametrize("cbow", [0, 1])
def test_app_hs_two_ranks_with_checkpoint_roundtrip(tmp_path, cbow):
    base = ["-m", "adapm_b200.apps.word2vec", "--", "--input_file", SMALL, "--embed_dim", "16", "--num_iterations", "1",
            "--min_count", "5", "--negative", "0", "--hs", "1", "--cbow", str(cbow), "--batch_windows", "2048",
            "--batch_pairs", "4096"]
    ck = str(tmp_path / "vec")
    rc, out = _launch(base + ["--write_results", "1", "--output_file", ck])
    assert rc == 0 and os.path.exists(ck + ".epoch.0"), out[-2000:]
    assert ("windows" if cbow else "pairs") + " on rank 0" in out, out[-2000:]
    loss = float(out.split("last batch loss ")[1].split()[0])
    assert 0 < loss < np.log(2) + 0.05, out[-2000:]       # per path node, near log 2 from syn1 = 0
    rc, out = _launch(base + ["--init_model", ck + ".epoch.0", "--data_words", "4000"])
    assert rc == 0 and "initialised" in out, out[-2000:]


def test_app_hs_option_checks():
    base = ["-m", "adapm_b200.apps.word2vec", "--", "--synthetic_vocab", "100", "--embed_dim", "8", "--num_iterations",
            "1", "--hs", "1", "--synthetic_batches", "1", "--batch_pairs", "64"]
    rc, out = _launch(base + ["--negative", "5"], world=1)
    assert rc != 0 and "ValueError" in out and "not supported" in out, out[-2000:]
    rc, out = _launch(base + ["--negative", "0", "--shared_negatives", "32"], world=1)
    assert rc != 0 and "ValueError" in out, out[-2000:]


# ---------------------------------------------------------------------------------------------- learning check
def train_planted_hs(backend, cbow, epochs=4, seed=0, d=32):
    """hierarchical softmax on the planted corpus of test_cbow_cpu; returns (per-epoch loss per path node, topic
    precision, syn0 rows)"""
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig
    from adapm_b200.utils.text import pairs_from_sentences, windows_from_sentences
    import adapm_b200 as ad

    V = 1 + TOPICS * PER_TOPIC
    cfg = Word2VecConfig(vocab_size=V, embed_dim=d, negative=0, hs=True, window=4, starting_alpha=0.05,
                         batch_windows=1024, batch_pairs=4096, cbow=bool(cbow), model_seed=seed + 1)
    kw = {"device": 0} if backend == "cuda" else {}
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend=backend,
                       fabric="inproc", job=f"planted_hs_{np.random.randint(1 << 30)}", **kw)
    kv = ad.Worker(0, server)
    try:
        counts = np.ones(V)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        sents = planted_corpus(seed)
        losses = []
        for ep in range(epochs):
            tot, n = 0.0, 0
            rng = np.random.default_rng([seed, ep])
            if cbow:
                it = windows_from_sentences(iter(sents), cfg.window, cfg.batch_windows, rng)
            else:
                it = (b for b in pairs_from_sentences(iter(sents), cfg.window, cfg.batch_pairs, rng)
                      if b.shape[1] == cfg.batch_pairs)
            for b in it:
                if model.cuda:
                    model.loss.zero_()
                loss = model.step(b.pin_memory() if model.cuda else b)
                tot += float(loss.sum())
                n += model.loss_terms(b)
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


@pytest.mark.parametrize("cbow", [0, 1])
def test_hs_learns_planted_topics_on_cpu(cbow):
    losses, prec, _ = train_planted_hs("cpu", cbow)
    print(f"cpu hs (cbow={cbow}) planted topics: losses {losses}, topic precision {prec:.3f}")
    assert losses[-1] < losses[0]
    assert prec > TOPIC_PRECISION, prec
