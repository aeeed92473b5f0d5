"""The deterministic one-GPU SGNS step applies a key with exactly one entry in the step (a "singleton") in its score
pass: that pass already holds everything the key's one update needs, and no other warp touches the row during the step.
Every other key is grouped and gathered as before. These tests build steps whose key counts mix the two kinds: target
singletons next to keys with exactly two entries, singleton centers whose targets are heavy keys, keys that are
singletons only because their other occurrence is a negative equal to the pair's context (which adds nothing), and a
step with no singletons at all. Rows and loss are checked against the float64 start-of-step rule; a Zipf run at the
benchmark's width is checked bit for bit against what the step computed before singletons were applied in the score
pass (tests/golden/sgns_det_singletons, made by running this file as a script).

    python tests/test_gpu_sgns_singletons.py OUT_DIR    # writes golden.json and rows.npy of the golden run"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_sgns_gather import _run_steps, cluster1  # noqa: E402,F401  (cluster1 is a fixture)

gpu = pytest.mark.gpu
DIMS = [16, 52, 300, 336]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgns_det_singletons")


def _entries_per_key(centers, contexts, negatives, n_keys):
    """Entries of each key that add something: centers, contexts, and negatives other than the pair's context."""
    valid = negatives != contexts.view(-1, 1)
    return torch.bincount(torch.cat([centers, contexts, negatives[valid]]), minlength=n_keys)


def _split(keys, neg):
    keys = keys.view(-1, neg + 2)
    return keys[:, 0].clone(), keys[:, 1].clone(), keys[:, 2:].contiguous()


def _shuffled_without_context_negatives(pool, neg, g):
    """A random order of the key pool cut into pairs, drawn again until no negative equals its pair's context (so every
    occurrence of a key adds to its row)."""
    while True:
        centers, contexts, negatives = _split(pool[torch.randperm(pool.numel(), generator=g)], neg)
        if not (negatives == contexts.view(-1, 1)).any():
            return centers, contexts, negatives


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_singletons_next_to_two_entry_keys(cluster1, d):  # noqa: F811
    """A third of the slots hold keys that occur once, the rest keys that occur exactly twice, so singletons and the
    smallest gathered keys sit side by side in the same pairs. A key that is a singleton in one step occurs twice in the
    next, and the other way round."""
    B, neg, n_keys = 512, 5, 3000
    n_single = B * (neg + 2) // 3
    n_double = (B * (neg + 2) - n_single) // 2
    g = torch.Generator().manual_seed(d + 1)
    batches = []
    for _ in range(3):
        perm = torch.randperm(n_keys, generator=g)
        pool = torch.cat([perm[:n_single], perm[n_single:n_single + n_double].repeat(2)])
        batch = _shuffled_without_context_negatives(pool, neg, g)
        cnt = _entries_per_key(*batch, n_keys)
        assert (cnt == 1).sum() == n_single and (cnt == 2).sum() == n_double
        batches.append(batch)
    _run_steps(cluster1, d, neg, n_keys, batches, seed=d + 2)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_singleton_centers_with_heavy_targets(cluster1, d):  # noqa: F811
    """Every center occurs once in the step; all targets come from 20 keys with about 300 entries each, which span
    several gather ranges. The centers' updates are applied in the score pass, the targets' ones gathered."""
    B, neg, words = 1024, 5, 20
    n_keys = words + 2 * B
    g = torch.Generator().manual_seed(2 * d + 3)
    batches = []
    for _ in range(2):
        centers = words + torch.randperm(2 * B, generator=g)[:B]
        tk = torch.randint(0, words, (B, neg + 1), generator=g)
        batch = (centers, tk[:, 0].clone(), tk[:, 1:].contiguous())
        cnt = _entries_per_key(*batch, n_keys)
        assert (cnt[centers] == 1).all() and (cnt[:words] > 64).all()
        batches.append(batch)
    _run_steps(cluster1, d, neg, n_keys, batches, seed=d + 4)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_singletons_whose_other_occurrence_adds_nothing(cluster1, d):  # noqa: F811
    """In every third pair one or two negatives equal the pair's context. Those negatives add nothing, so the context is
    the key's one entry and a singleton; the remaining keys occur once or twice."""
    B, neg, n_keys = 768, 5, 5000
    g = torch.Generator().manual_seed(3 * d + 5)
    batches = []
    for _ in range(2):
        perm = torch.randperm(n_keys, generator=g)
        n = B * (neg + 2)
        pool = torch.cat([perm[:n // 2], perm[n // 2:3 * n // 4].repeat(2)])
        centers, contexts, negatives = _shuffled_without_context_negatives(pool, neg, g)
        negatives[::3, 1] = contexts[::3]
        negatives[::6, 4] = contexts[::6]
        cnt = _entries_per_key(centers, contexts, negatives, n_keys)
        seen = torch.bincount(torch.cat([centers, contexts, negatives.view(-1)]), minlength=n_keys)
        assert ((cnt == 1) & (seen > 1)).any()
        batches.append((centers, contexts, negatives))
    _run_steps(cluster1, d, neg, n_keys, batches, seed=d + 6)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_a_step_without_singletons(cluster1, d):  # noqa: F811
    """48 keys with about 56 entries each, every one a center in some pairs and a target in others: no key is applied
    in the score pass."""
    B, neg, words = 384, 5, 48
    g = torch.Generator().manual_seed(4 * d + 7)
    k = torch.randint(0, words, (B, neg + 2), generator=g)
    batch = (k[:, 0].clone(), k[:, 1].clone(), k[:, 2:].contiguous())
    cnt = _entries_per_key(*batch, words)
    assert cnt.min() >= 2
    _run_steps(cluster1, d, neg, words, [batch], seed=d + 8)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_ranges_of_two_entry_keys(cluster1, d):  # noqa: F811
    """Every key of the step has exactly two entries, so each 64-entry gather range holds 32 keys that start in both
    halves of the warp's two-lane-round key lookup."""
    B, neg = 512, 5
    n_keys = B * (neg + 2) // 2
    g = torch.Generator().manual_seed(5 * d + 9)
    batch = _shuffled_without_context_negatives(torch.arange(n_keys).repeat(2), neg, g)
    assert (_entries_per_key(*batch, n_keys) == 2).all()
    _run_steps(cluster1, d, neg, n_keys, [batch], seed=d + 10)


def _golden_cfg():
    from adapm_b200.models.word2vec import Word2VecConfig

    return Word2VecConfig(vocab_size=20000, embed_dim=300, negative=25, batch_pairs=4096)


def _golden_run(server, worker):
    """Three 4096-pair Zipf steps at d = 300 and 25 negatives: the steps' losses, the SHA-256 of the whole table after
    them, and 256 sampled rows (for a look at where two runs differ)."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, zipf_counts

    cfg = _golden_cfg()
    counts = zipf_counts(cfg.vocab_size)
    model = Word2Vec(server, worker, cfg, counts)
    model.init_model()
    data = SyntheticPairs(cfg, counts, 0, seed=1)
    losses = []
    for s in range(3):
        model.loss.zero_()
        model.step(data.batch(s))
        losses.append(model.loss.item())
        worker.advance_clock()
    torch.cuda.synchronize()
    rows = torch.empty(cfg.num_keys, cfg.row_len)
    worker.pull(torch.arange(cfg.num_keys), rows)
    sha = hashlib.sha256(rows.numpy().tobytes()).hexdigest()
    keys = torch.randperm(cfg.num_keys, generator=torch.Generator().manual_seed(0))[:256].sort().values
    return {"losses": losses, "table_sha256": sha, "row_keys": keys.tolist()}, rows[keys].numpy()


@gpu
def test_zipf_steps_match_the_golden(cluster1):  # noqa: F811
    """The steps' losses and the whole table are bit-identical to what the step computed before singletons were
    applied in the score pass."""
    with open(os.path.join(GOLDEN, "golden.json")) as f:
        want = json.load(f)
    cfg = _golden_cfg()
    server, kv = cluster1(cfg.row_len, cfg.num_keys)
    got, rows = _golden_run(server, kv)
    want_rows = np.load(os.path.join(GOLDEN, "rows.npy"))
    assert got["row_keys"] == want["row_keys"]
    differ = np.flatnonzero((rows.view(np.uint32) != want_rows.view(np.uint32)).any(1))
    assert differ.size == 0, [want["row_keys"][i] for i in differ[:16]]
    assert got["losses"] == want["losses"]
    assert got["table_sha256"] == want["table_sha256"]


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import adapm_b200 as ad

    out = sys.argv[1]
    cfg = _golden_cfg()
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="sgns_golden", device=0)
    worker = ad.Worker(0, server)
    meta, rows = _golden_run(server, worker)
    worker.finalize()
    server.shutdown()
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "golden.json"), "w") as f:
        json.dump(meta, f, indent=1)
    np.save(os.path.join(out, "rows.npy"), rows)
    print(json.dumps({k: meta[k] for k in ("losses", "table_sha256")}))
