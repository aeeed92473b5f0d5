"""GloVe without a GPU: the co-occurrence reference (``utils.text.cooccurrence_reference``) against a plain per-position
loop and across rank partitions, the float64 step rule (``ops.glove_reference_step``) against a hand computation,
quality on planted topics with the CPU backend, the app end to end through the launcher, and the register budget of
the fused GloVe kernels."""
import math
import os
import subprocess
import sys
from collections import defaultdict
from fractions import Fraction

import numpy as np
import pytest
import torch

from multirank import one_rank_store
from test_build_budget import _kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = os.path.join(ROOT, "data", "lm", "small.txt")
MODES = [(s, w) for s in (True, False) for w in (True, False)]

# Planted-topic quality: fraction of each topic word's 10 nearest neighbours (cosine of W + C) in its own topic. Chance
# is 24 / 519 = 0.046. The CPU run of train_planted reaches 0.995; the threshold leaves room for the fp32 GPU run.
QUALITY_MIN = 0.9


def _loop_counts(sentences, window, symmetric, weighted, rank=0, world=1):
    """X as {(a, b): Fraction}, one position pair at a time"""
    X = defaultdict(Fraction)
    for s in sentences:
        for p in range(len(s)):
            for k in range(1, window + 1):
                if p + k >= len(s):
                    break
                a, b = int(s[p]), int(s[p + k])
                w = Fraction(1, k) if weighted else Fraction(1)
                if a % world == rank:
                    X[(a, b)] += w
                if symmetric and b % world == rank:
                    X[(b, a)] += w
    return X


def _small_sentences():
    from adapm_b200.utils.text import NativeCorpus

    c = NativeCorpus.build(SMALL, 5)
    c.encode(SMALL, 0, 1)
    return c.sentences(), len(c.vocabulary().words)


HAND = [np.array([3]), np.array([1, 2]), np.array([4, 4, 5, 4, 4, 1, 0]), np.array([2, 2, 2])]


def _check_equal(ref, X):
    rows, cols, x = ref
    assert rows.dtype == np.int32 and cols.dtype == np.int32 and x.dtype == np.float32
    keys = list(zip(rows.tolist(), cols.tolist()))
    assert keys == sorted(X), "keys differ or are not sorted"
    want = np.array([float(X[k]) for k in keys], dtype=np.float32)
    assert np.array_equal(x, want)


@pytest.mark.parametrize("symmetric,weighted", MODES)
@pytest.mark.parametrize("window", [1, 3, 10])
def test_reference_counts_equal_a_plain_loop_on_hand_made_sentences(symmetric, weighted, window):
    """a one-word line, windows longer than the line, a word repeated inside one window"""
    from adapm_b200.utils.text import cooccurrence_reference

    _check_equal(cooccurrence_reference(HAND, 6, window, symmetric, weighted), _loop_counts(HAND, window, symmetric, weighted))


@pytest.mark.parametrize("symmetric,weighted", MODES)
def test_reference_counts_equal_a_plain_loop_on_the_small_corpus(symmetric, weighted):
    from adapm_b200.utils.text import cooccurrence_reference

    sents, V = _small_sentences()
    _check_equal(cooccurrence_reference(sents, V, 5, symmetric, weighted), _loop_counts(sents, 5, symmetric, weighted))


@pytest.mark.parametrize("symmetric", [True, False])
def test_rank_partitions_are_disjoint_and_make_the_whole_matrix(symmetric):
    from adapm_b200.utils.text import cooccurrence_reference

    sents, V = _small_sentences()
    full = cooccurrence_reference(sents, V, 8, symmetric, True)
    parts = [cooccurrence_reference(sents, V, 8, symmetric, True, r, 3) for r in range(3)]
    for r, p in enumerate(parts):
        assert np.all(p[0] % 3 == r)
    rows = np.concatenate([p[0] for p in parts]).astype(np.int64)
    cols = np.concatenate([p[1] for p in parts]).astype(np.int64)
    x = np.concatenate([p[2] for p in parts])
    order = np.argsort(rows * V + cols)
    assert np.array_equal(rows[order], full[0]) and np.array_equal(cols[order], full[1])
    assert np.array_equal(x[order], full[2])


def test_reference_rejects_a_window_above_16():
    from adapm_b200.utils.text import cooccurrence_reference

    with pytest.raises(ValueError):
        cooccurrence_reference(HAND, 6, 17)


# ---------------------------------------------------------------------------------------------- the step rule
def test_reference_step_equals_a_hand_computation():
    """three non-zeros: word 0 twice (a repeated key within the batch), one X >= x_max; rows read at the start"""
    from adapm_b200.ops import glove_reference_step

    d, D, eta, x_max, alpha = 4, 8, 0.1, 10.0, 0.75
    g = torch.Generator().manual_seed(3)
    table = torch.zeros(6, 2 * D, dtype=torch.float64)
    table[:, :d + 1] = torch.randn(6, d + 1, generator=g, dtype=torch.float64) * 0.3
    table[:, D:D + d + 1] = torch.rand(6, d + 1, generator=g, dtype=torch.float64) + 0.5
    words, ctxs = torch.tensor([0, 0, 2]), torch.tensor([1, 3, 5])
    x = torch.tensor([2.0, 25.0, 7.0])
    with one_rank_store(2 * D, 6, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(6), table.contiguous().view(-1)))
        loss, pushes = glove_reference_step(kv, words, ctxs, x, d, eta, x_max, alpha)
        got = torch.empty(6 * 2 * D, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(6), got))
    got = got.view(6, 2 * D)
    want = table.clone()
    want_loss = 0.0
    for wk, ck, X in zip(words.tolist(), ctxs.tolist(), x.double().tolist()):
        w, c = table[wk], table[ck]
        diff = float((w[:d] * c[:d]).sum()) + float(w[d]) + float(c[d]) - math.log(X)
        f = (X / x_max) ** alpha if X < x_max else 1.0
        want_loss += 0.5 * f * diff * diff
        for key, own, other in ((wk, w, c), (ck, c, w)):
            for e in range(d + 1):
                ge = f * diff * (float(other[e]) if e < d else 1.0)
                want[key, e] += -eta * ge / math.sqrt(float(own[D + e]) + ge * ge)
                want[key, D + e] += ge * ge
    assert pushes == 6
    assert abs(loss - want_loss) <= 1e-12 * max(1.0, want_loss)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-14)
    assert torch.all(got[:, d + 1:D] == 0) and torch.all(got[:, D + d + 1:] == 0)      # the padding stays 0


def test_reference_step_checks_its_shape():
    from adapm_b200.ops import glove_reference_step

    with pytest.raises(ValueError):
        glove_reference_step(None, torch.zeros(1, dtype=torch.int64), torch.ones(1, dtype=torch.int64), torch.ones(1), 6,
                             0.1, 10.0, 0.75)


# ---------------------------------------------------------------------------------------------- quality
def planted_corpus(path, seed=5, topics=20, per_topic=25, function_words=20, lines=1500, length=20):
    """Lines of ``length`` words: each line draws 80 % of its words from one topic (uniformly) and 20 % from Zipf-
    frequent function words shared by all topics. Returns the topic of each topic word (by word string)."""
    rng = np.random.default_rng(seed)
    fz = 1.0 / np.arange(1, function_words + 1)
    fz /= fz.sum()
    topic_of = {f"t{t}w{i}": t for t in range(topics) for i in range(per_topic)}
    with open(path, "w") as f:
        for _ in range(lines):
            t = rng.integers(topics)
            words = [f"t{t}w{rng.integers(per_topic)}" if rng.random() < 0.8 else f"fn{rng.choice(function_words, p=fz)}"
                     for _ in range(length)]
            f.write(" ".join(words) + "\n")
    return topic_of


def train_planted(tmp_path, backend, deterministic=False, epochs=15):
    """Trains on the planted corpus; returns the mean own-topic share of the topic words' 10 nearest neighbours."""
    from adapm_b200.models.glove import GloVe, GloVeConfig
    from adapm_b200.utils.text import NativeCorpus

    path = os.path.join(str(tmp_path), "planted.txt")
    topic_of = planted_corpus(path)
    corpus = NativeCorpus.build(path, 1)
    corpus.encode(path, 0, 1)
    words = corpus.vocabulary().words
    cfg = GloVeConfig(vocab_size=len(words), embed_dim=16, window=5, eta=0.05, x_max=10.0, batch_entries=4096,
                      deterministic=deterministic, model_seed=7)
    with one_rank_store(cfg.row_len, cfg.num_keys, backend, "float32") as (s, kv):
        model = GloVe(s, kv, cfg)
        model.init_model()
        model.build_cooccurrence(corpus)
        losses = [model.train_epoch(e) for e in range(epochs)]
        q = [i for i, w in enumerate(words) if w in topic_of]
        idx, _ = model.most_similar(q, 10)
    idx = idx.cpu().tolist()
    share = np.mean([np.mean([topic_of.get(words[j]) == topic_of[words[i]] for j in row]) for i, row in zip(q, idx)])
    return float(share), losses


def test_cpu_quality_on_planted_topics(tmp_path):
    share, losses = train_planted(tmp_path, "cpu")
    print(f"planted topics: own-topic share of the 10 nearest neighbours {share:.4f} (chance 0.046), losses "
          f"{losses[0]:.1f} -> {losses[-1]:.1f}")
    assert losses[-1] < losses[0]
    assert share >= QUALITY_MIN, share


# ---------------------------------------------------------------------------------------------- app
def _app(args, world=2, cwd=ROOT):
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu",
                        "-m", "adapm_b200.apps.glove", "--"] + args, cwd=cwd, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


def test_app_runs_on_two_cpu_ranks_and_writes_vectors(tmp_path):
    out = str(tmp_path / "vectors.txt")
    voc = str(tmp_path / "vocab.txt")
    rc, log = _app(["--input_file", SMALL, "--vector_size", "8", "--iter", "2", "--window_size", "4",
                    "--output_file", out, "--vocab_save", voc, "--batch_entries", "32768"])
    assert rc == 0, log[-3000:]
    assert "[glove] iter 2: cost" in log and "protocol errors 0" in log, log[-3000:]
    assert "non-zeros" in log
    vocab = [ln.rsplit(" ", 1)[0] for ln in open(voc)]
    lines = open(out).read().splitlines()
    assert len(lines) == len(vocab)
    for ln, w in zip(lines[:50], vocab):
        parts = ln.split(" ")
        assert parts[0] == w and len(parts) == 9
        assert all(math.isfinite(float(v)) for v in parts[1:])


@pytest.mark.parametrize("flags,message", [
    (["--window_size", "17"], "--window_size must be in"),
    (["--vector_size", "10"], "--vector_size must be a multiple of 4"),
    (["--deterministic", "1"], "--deterministic 1 needs a single GPU"),
])
def test_app_rejects_invalid_flags(flags, message, tmp_path):
    rc, log = _app(["--input_file", SMALL, "--iter", "1", "--output_file", str(tmp_path / "v.txt")] + flags)
    assert rc != 0 and message in log, log[-2000:]


# ---------------------------------------------------------------------------------------------- build facts
def test_glove_kernels_stay_within_their_register_budget():
    """launch bounds of 3 CTAs of 256 threads per SM allow 85 registers; every instantiation stays at or below 80
    without spills"""
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    names = [f"glove_step_kernel<{v}, {fx}>" for v in range(4) for fx in ("false", "true")]
    for name in names:
        assert name in k, sorted(n for n in k if "glove" in n)
        assert k[name]["regs"] <= 80 and k[name]["spill"] == 0, (name, k[name])
    for name, v in k.items():
        if name.startswith("cooc_"):
            assert v["spill"] == 0, (name, v)
