"""node2vec without a GPU: the CSR graph, the native edge-list reader, the numpy walk reference against node2vec's
analytic transition probabilities (chi-square), the pair reference against ``pairs_from_sentences``, input checks,
quality on a planted partition with the CPU backend, the app through the launcher, and the walk kernels' build facts."""
import math
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

from multirank import one_rank_store
from test_build_budget import _kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Planted partition, 20 communities of 50 nodes (chance 0.05 for the share). The CPU run of train_planted measured an
# own-community share of the 10 nearest neighbours of 1.000 and a held-out AUC of 0.948; the thresholds leave room for
# the fp32 GPU run.
SHARE_MIN = 0.9
AUC_MIN = 0.9


# ---------------------------------------------------------------------------------------------- graphs
def _triangle_path_hub():
    """a triangle 0-1-2, a path 2-3-4-5, a hub 6 joined to 0, 3, 5, 7, 8, 9 and a self-loop on 9"""
    e = [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4), (4, 5), (6, 0), (6, 3), (6, 5), (6, 7), (6, 8), (6, 9), (9, 9)]
    return [a for a, _ in e], [b for _, b in e]


def _directed_dangling():
    """directed, with nodes 4 and 5 lacking out-edges and a 2-cycle 0 <-> 1"""
    e = [(0, 1), (1, 0), (0, 2), (2, 3), (3, 0), (3, 1), (1, 3), (2, 4), (3, 5), (0, 3)]
    return [a for a, _ in e], [b for _, b in e]


def _weighted():
    e = [(0, 1, 1.0), (0, 2, 3.0), (1, 2, 0.5), (2, 3, 2.0), (3, 0, 1.5), (1, 3, 4.0), (3, 4, 0.25), (4, 0, 1.0)]
    return [a for a, _, _ in e], [b for _, b, _ in e], [w for _, _, w in e]


GRAPHS = {
    "triangle_path_hub": lambda: _triangle_path_hub() + (None, False),
    "directed_dangling": lambda: _directed_dangling() + (None, True),
    "weighted": lambda: _weighted() + (False,),
}


def _graph(name):
    from adapm_b200.utils.graph import Graph

    src, dst, w, directed = GRAPHS[name]()
    return Graph.from_edges(src, dst, w, directed)


def test_csr_merges_duplicates_stores_both_directions_and_quantises_weights():
    from adapm_b200.utils.graph import Graph

    g = Graph.from_edges([0, 1, 2, 2, 1], [1, 0, 2, 0, 0], [1.0, 2.0, 5.0, 4.0, 1.0], directed=False, num_nodes=4)
    # undirected: 0-1 given three times (weights 1 + 2 + 1 per direction), 2-0 once, a self-loop on 2 stored once
    assert g.offsets.tolist() == [0, 2, 3, 5, 5]
    assert g.neighbors.tolist() == [1, 2, 0, 0, 2]
    assert g.neighbors.dtype == torch.int32 and g.offsets.dtype == torch.int64
    full = 1 << 24
    assert g.cum_weights.tolist() == [full, full + full, full, round(4 / 5 * full), round(4 / 5 * full) + full]
    assert g.degrees().tolist() == [2, 1, 2, 0]


# ---------------------------------------------------------------------------------------------- walk statistics
def _alpha(g, t, x, p, q):
    if x == t:
        return 1.0 / p
    off, nb = g.offsets.numpy(), g.neighbors.numpy()
    return 1.0 if x in set(nb[off[t]:off[t + 1]].tolist()) else 1.0 / q


def _edge_weights(g, v):
    off = g.offsets.numpy()
    nb = g.neighbors.numpy()[off[v]:off[v + 1]].tolist()
    if not g.weighted:
        return nb, [1.0] * len(nb)
    cw = g.cum_weights.numpy()[off[v]:off[v + 1]]
    return nb, np.diff(np.concatenate([[0], cw])).astype(np.float64).tolist()


def _chi2_sf(x, k):
    """upper tail of the chi-square distribution (Wilson-Hilferty)"""
    z = ((x / k) ** (1 / 3) - (1 - 2 / (9 * k))) / math.sqrt(2 / (9 * k))
    return 0.5 * math.erfc(z / math.sqrt(2))


@pytest.mark.parametrize("name", list(GRAPHS))
@pytest.mark.parametrize("p,q", [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25), (0.5, 2.0)])
def test_reference_transitions_follow_node2vecs_probabilities(name, p, q):
    """second-order steps (t, v) -> x counted over many walks against P(x | t, v) ~ alpha(t, x) w(v, x); first steps
    against w(v, x) alone"""
    from adapm_b200.ops import random_walks_reference

    g = _graph(name)
    n = g.num_nodes
    reps = 3000
    w = random_walks_reference(g, np.repeat(np.arange(n), reps), np.tile(np.arange(reps), n), 6, p, q, seed=11, epoch=2)
    counts = defaultdict(lambda: defaultdict(int))
    for k in range(1, w.shape[1]):
        prev = w[:, k - 2] if k >= 2 else np.full(w.shape[0], -1)
        ok = w[:, k] >= 0
        assert np.all(w[~ok, k:] == -1)           # a walk stays ended
        for t, v, x in zip(prev[ok].tolist(), w[ok, k - 1].tolist(), w[ok, k].tolist()):
            counts[(t, v)][x] += 1
    chi, dof, contexts = 0.0, 0, 0
    for (t, v), obs in counts.items():
        nb, wt = _edge_weights(g, v)
        assert set(obs) <= set(nb), ((t, v), obs, nb)
        pr = np.array([wt[i] * (_alpha(g, t, x, p, q) if t >= 0 else 1.0) for i, x in enumerate(nb)])
        pr /= pr.sum()
        tot = sum(obs.values())
        exp = tot * pr
        if len(nb) < 2 or exp.min() < 5:
            continue
        o = np.array([obs.get(x, 0) for x in nb], dtype=np.float64)
        chi += float(((o - exp) ** 2 / exp).sum())
        dof += len(nb) - 1
        contexts += 1
    assert contexts >= 5, contexts
    pval = _chi2_sf(chi, dof)
    print(f"{name} p={p} q={q}: chi2 {chi:.1f} on {dof} dof over {contexts} contexts, p-value {pval:.3g}")
    assert pval > 1e-4, (chi, dof)


def test_walks_depend_on_the_walk_id_only():
    """a walk is the same whichever call, chunk or batch it comes from; other seeds, epochs or walk numbers differ"""
    from adapm_b200.ops import random_walks_reference

    g = _graph("triangle_path_hub")
    n = g.num_nodes
    starts, nums = np.repeat(np.arange(n), 4), np.tile(np.arange(4), n)
    full = random_walks_reference(g, starts, nums, 12, 0.5, 2.0, seed=5, epoch=1)
    perm = np.random.default_rng(0).permutation(starts.size)
    parts = [random_walks_reference(g, starts[perm[i:i + 7]], nums[perm[i:i + 7]], 12, 0.5, 2.0, seed=5, epoch=1)
             for i in range(0, starts.size, 7)]
    assert np.array_equal(np.concatenate(parts), full[perm])
    for kw in (dict(seed=6, epoch=1), dict(seed=5, epoch=2)):
        assert not np.array_equal(random_walks_reference(g, starts, nums, 12, 0.5, 2.0, **kw), full)
    assert not np.array_equal(full[::4], full[1::4])


# ---------------------------------------------------------------------------------------------- pairs
class _Shrinks:
    """an rng for pairs_from_sentences that returns given window shrinks in order"""

    def __init__(self, b):
        self.b = iter(b)

    def integers(self, lo, hi):
        v = next(self.b)
        assert lo <= v < hi
        return v


@pytest.mark.parametrize("window", [1, 3, 10])
def test_reference_pairs_follow_pairs_from_sentences(window):
    from adapm_b200.ops import _mix64_int, _mix64_np, random_walks_reference, walk_pairs_reference
    from adapm_b200.utils.text import pairs_from_sentences

    g = _graph("directed_dangling")
    walks = random_walks_reference(g, np.repeat(np.arange(g.num_nodes), 5), 0, 9, 2.0, 0.5, seed=3)
    walks[2] = -1                                       # a row without any node
    walks[3, 1:] = -1                                   # a lone start
    seed = 77
    got = walk_pairs_reference(walks, window, seed)
    shrinks = []
    sentences = []
    for r, row in enumerate(walks):
        L = int((row >= 0).sum())
        if L == 0:
            continue
        sentences.append(row[:L])
        for i in range(L):
            h = int(_mix64_np(np.array([_mix64_int(seed) ^ (r << 32 | i)], dtype=np.uint64))[0])
            shrinks.append(((h >> 32) * window) >> 32)
    want = list(pairs_from_sentences(sentences, window, 1 << 40, _Shrinks(shrinks)))
    want = want[0].numpy() if want else np.zeros((2, 0), dtype=np.int64)
    assert got.dtype == np.int64 and np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------- edge lists
def _numpy_parse(path):
    rows = [ln.split() for ln in open(path) if ln.strip() and not ln.strip().startswith("#")]
    src = np.array([int(r[0]) for r in rows], dtype=np.int64)
    dst = np.array([int(r[1]) for r in rows], dtype=np.int64)
    w = np.array([float(r[2]) for r in rows]) if rows and len(rows[0]) == 3 else None
    ids = np.unique(np.concatenate([src, dst]))
    return np.searchsorted(ids, src), np.searchsorted(ids, dst), w, ids


@pytest.mark.parametrize("weighted", [False, True])
def test_edge_list_reader_equals_a_numpy_parse(tmp_path, weighted):
    from adapm_b200.utils.graph import read_edge_list

    rng = np.random.default_rng(4)
    path = tmp_path / "g.txt"
    with open(path, "w") as f:
        f.write("# Directed graph (each unordered pair of nodes is saved once)\n# FromNodeId\tToNodeId\n\n")
        for i in range(500):
            a, b = rng.integers(0, 10 ** 9, 2)
            wt = f"\t{rng.random() * 10:.6g}" if weighted else ""
            f.write(f"{a}\t{b}{wt}\r\n" if i % 7 == 0 else f"  {a} {b}{wt}\n")
            if i % 50 == 0:
                f.write("   # a comment\n   \n")
        f.write(f"17 17{' 2.5' if weighted else ''}")                # a self-loop on the last line, no newline
    got = read_edge_list(str(path))
    want = _numpy_parse(path)
    for g, w in zip(got, want):
        if w is None:
            assert g is None
        else:
            assert g.dtype == w.dtype and np.array_equal(g, w)


@pytest.mark.parametrize("body,line", [
    ("1 2\n3 x\n", 2),
    ("1 2\n3\n", 2),
    ("1 2 1.0 7\n", 1),
    ("# c\n-1 2\n", 2),
    ("1 2 1.0\n2 3\n", 2),
    ("1 2\n2 3 0.5\n", 2),
    ("1 2 abc\n", 1),
    ("1.5 2\n", 1),
])
def test_edge_list_reader_rejects_malformed_lines_with_their_number(tmp_path, body, line):
    from adapm_b200.utils.graph import read_edge_list

    path = tmp_path / "bad.txt"
    path.write_text(body)
    with pytest.raises(ValueError, match=f"bad.txt:{line}:"):
        read_edge_list(str(path))


# ---------------------------------------------------------------------------------------------- input checks
def test_invalid_inputs_raise_value_error():
    from adapm_b200.ops import random_walks, random_walks_reference, walk_pairs_reference
    from adapm_b200.utils.graph import Graph

    g = _graph("triangle_path_hub")
    for kw in (dict(p=0.0), dict(q=-1.0), dict(p=float("nan")), dict(walk_length=1)):
        args = dict(walk_length=5, p=1.0, q=1.0)
        args.update(kw)
        with pytest.raises(ValueError):
            random_walks_reference(g, [0], 0, args["walk_length"], args["p"], args["q"])
    for s in ([-1], [g.num_nodes]):
        with pytest.raises(ValueError):
            random_walks_reference(g, s, 0, 5)
    with pytest.raises(ValueError):
        random_walks_reference(g, [0], -1, 5)
    with pytest.raises(ValueError):
        walk_pairs_reference(np.zeros((1, 3), dtype=np.int64), 0)
    with pytest.raises(ValueError, match="CUDA device"):
        random_walks(g, [0], 0, 5)
    for src, dst, w, n in (([-1], [0], None, None), ([0], [1], [0.0], None), ([0], [1], [float("inf")], None),
                           ([0], [1], [-2.0], None), ([0], [5], None, 3), ([0], [1], None, 1 << 31)):
        with pytest.raises(ValueError):
            Graph.from_edges(src, dst, w, num_nodes=n)


def test_model_rejects_invalid_configs():
    from adapm_b200.models.node2vec import Node2Vec, Node2VecConfig, num_keys

    g = _graph("triangle_path_hub")
    for kw in (dict(p=0.0), dict(walk_length=1), dict(window=0), dict(num_walks=0)):
        cfg = Node2VecConfig(dimensions=8, **kw)
        with one_rank_store(cfg.row_len, num_keys(g.num_nodes), "cpu", "float32") as (s, kv):
            with pytest.raises(ValueError):
                Node2Vec(s, kv, g, cfg)


# ---------------------------------------------------------------------------------------------- quality
def planted_split(seed=1):
    """20 communities of 50 nodes (p_in 0.3, p_out 0.001); 10 % of the edges held out, as many non-edges sampled"""
    from adapm_b200.models.node2vec import sample_non_edges, split_edges
    from adapm_b200.utils.graph import Graph, planted_partition

    s, d = planted_partition(20, 50, 0.3, 0.001, seed=seed)
    ts, td, _, held = split_edges(s, d, 0.1, False, seed + 4)
    neg = sample_non_edges(s, d, 1000, held.shape[1], False, seed + 5)
    return Graph.from_edges(ts, td, num_nodes=1000), held, neg


def planted_config(**kw):
    from adapm_b200.models.node2vec import Node2VecConfig

    base = dict(dimensions=32, walk_length=40, num_walks=5, window=5, negative=5, batch_pairs=4096, iter=2,
                walkers_per_chunk=1000, model_seed=3)
    base.update(kw)
    return Node2VecConfig(**base)


def train_planted(backend, **kw):
    """Returns (own-community share of the 10 nearest neighbours, held-out AUC, per-epoch losses)."""
    from adapm_b200.models.node2vec import Node2Vec, num_keys

    g, held, neg = planted_split()
    cfg = planted_config(**kw)
    with one_rank_store(cfg.row_len, num_keys(g.num_nodes), backend, "float32") as (s, kv):
        m = Node2Vec(s, kv, g, cfg)
        m.init_model()
        losses = [m.train_epoch(e) for e in range(cfg.iter)]
        auc = m.link_prediction_auc(held, neg)
        idx, _ = m.most_similar(np.arange(g.num_nodes), 10)
    idx = idx.cpu().numpy()
    share = float(np.mean(idx // 50 == (np.arange(g.num_nodes) // 50)[:, None]))
    return share, auc, losses


def test_cpu_quality_on_a_planted_partition():
    share, auc, losses = train_planted("cpu")
    print(f"planted partition: own-community share {share:.4f} (chance 0.05), held-out AUC {auc:.4f}, losses {losses}")
    assert losses[-1][0] / losses[-1][1] < losses[0][0] / losses[0][1]
    assert share >= SHARE_MIN and auc >= AUC_MIN, (share, auc)


def test_roc_auc_counts_ties_as_half():
    from adapm_b200.models.node2vec import roc_auc

    assert roc_auc([3.0, 2.0], [1.0, 0.0]) == 1.0
    assert roc_auc([1.0], [1.0]) == 0.5
    assert roc_auc([2.0, 0.0], [1.0, 1.0]) == 0.5


# ---------------------------------------------------------------------------------------------- app
def _write_planted(path):
    from adapm_b200.utils.graph import planted_partition

    s, d = planted_partition(10, 30, 0.3, 0.002, seed=2)
    with open(path, "w") as f:
        f.write("# planted partition, sparse ids\n")
        f.writelines(f"{7 * a + 100} {7 * b + 100}\n" for a, b in zip(s, d))


def _app(args, world=2):
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu",
                        "-m", "adapm_b200.apps.node2vec", "--"] + args, cwd=ROOT, capture_output=True, text=True,
                       timeout=300)
    return r.returncode, r.stdout + r.stderr


def test_app_runs_on_two_cpu_ranks_and_writes_vectors(tmp_path):
    inp, out = str(tmp_path / "g.edgelist"), str(tmp_path / "g.emb")
    _write_planted(inp)
    rc, log = _app(["--input", inp, "--output", out, "--dimensions", "16", "--walk-length", "20", "--num_walks", "4",
                    "--window-size", "5", "--iter", "2", "--holdout", "0.1", "--batch_pairs", "2048", "--p", "0.5",
                    "--q", "2"])
    assert rc == 0, log[-3000:]
    assert "[node2vec] epoch 2:" in log and "held-out AUC" in log and "protocol errors 0" in log, log[-3000:]
    lines = open(out).read().splitlines()
    assert lines[0] == "300 16"
    ids = sorted(int(ln.split(" ")[0]) for ln in lines[1:])
    assert ids == [7 * v + 100 for v in range(300)]
    assert all(len(ln.split(" ")) == 17 for ln in lines[1:])


@pytest.mark.parametrize("flags,message", [
    (["--p", "0"], "--p and --q must be positive"),
    (["--holdout", "1.5"], "--holdout must be in"),
    (["--weighted"], "--weighted needs a weight column"),
])
def test_app_rejects_invalid_flags(flags, message, tmp_path):
    inp = str(tmp_path / "g.edgelist")
    _write_planted(inp)
    rc, log = _app(["--input", inp, "--output", str(tmp_path / "v.emb"), "--iter", "1"] + flags, world=1)
    assert rc != 0 and message in log, log[-2000:]


# ---------------------------------------------------------------------------------------------- build facts
def test_walk_kernels_do_not_spill():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    names = [f"node2vec_walk_kernel<{w}, {s}>" for w in ("false", "true") for s in ("false", "true")]
    names += ["walk_pair_count_kernel", "walk_pair_write_kernel"]
    for name in names:
        assert name in k, sorted(n for n in k if "walk" in n)
        assert k[name]["spill"] == 0 and k[name]["regs"] <= 64, (name, k[name])
