"""node2vec on the H100: the device walks (all four kernel instantiations) and pairs bit for bit against the numpy
references, reproducible one-GPU training, quality on a planted partition, and three logical ranks of one GPU whose
walks together are the one-rank walks and whose training with intents is free of protocol errors."""
import numpy as np
import pytest
import torch

from harness import run_cluster
from test_node2vec_cpu import AUC_MIN, SHARE_MIN, _graph, planted_config, planted_split, train_planted

gpu = pytest.mark.gpu
WORLD = 3
PQ = [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25)]


def _rmat(weighted, directed, scale=12):
    """R-MAT: hubs with degrees in the hundreds; directed R-MAT leaves many nodes without out-edges"""
    from adapm_b200.utils.graph import Graph, rmat_edges

    s, d, w = rmat_edges(scale, 8, seed=9, weighted=weighted)
    return Graph.from_edges(s, d, w, directed, num_nodes=1 << scale)


CASES = {
    "triangle_path_hub": lambda: _graph("triangle_path_hub"),
    "directed_dangling": lambda: _graph("directed_dangling"),
    "weighted_small": lambda: _graph("weighted"),
    "rmat": lambda: _rmat(False, False),
    "rmat_weighted_directed": lambda: _rmat(True, True),
}


@gpu
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("p,q", PQ)
def test_device_walks_equal_the_reference_bit_for_bit(case, p, q):
    from adapm_b200.ops import random_walks, random_walks_reference

    g = CASES[case]()
    n = g.num_nodes
    reps = max(2, 4000 // n)
    starts, nums = np.repeat(np.arange(n), reps), np.tile(np.arange(reps), n)
    perm = np.random.default_rng(1).permutation(starts.size)
    starts, nums = starts[perm], nums[perm]
    want = random_walks_reference(g, starts, nums, 20, p, q, seed=123, epoch=4)
    gd = g.to("cuda")
    got = random_walks(gd, starts, nums, 20, p, q, seed=123, epoch=4).cpu().numpy()
    assert np.array_equal(got, want)
    # several chunks of a size that does not divide the starts, and starts given as a device tensor
    chunk = 777
    parts = [random_walks(gd, torch.from_numpy(starts[i:i + chunk]).cuda(), nums[i:i + chunk], 20, p, q, seed=123,
                          epoch=4) for i in range(0, starts.size, chunk)]
    assert np.array_equal(torch.cat(parts).cpu().numpy(), want)
    if case.startswith("directed"):
        assert (want == -1).any()


@gpu
@pytest.mark.parametrize("window", [1, 5, 10])
def test_device_pairs_equal_the_reference_bit_for_bit(window):
    from adapm_b200.ops import random_walks, walk_pairs, walk_pairs_reference

    g = _rmat(False, True).to("cuda")
    n = g.num_nodes
    walks = random_walks(g, np.arange(n), 0, 30, 0.5, 2.0, seed=5)
    got = walk_pairs(walks, window, seed=99)
    want = walk_pairs_reference(walks.cpu().numpy(), window, 99)
    assert got.shape[1] > 0 and np.array_equal(got.cpu().numpy(), want)


@gpu
def test_walk_op_arguments_are_checked():
    from adapm_b200.ops import random_walks, walk_pairs

    g = _graph("triangle_path_hub").to("cuda")
    for args in (([0], 0, 5, 0.0, 1.0), ([0], 0, 5, 1.0, -1.0), ([0], 0, 1, 1.0, 1.0), ([99], 0, 5, 1.0, 1.0)):
        with pytest.raises(ValueError):
            random_walks(g, *args)
    w = random_walks(g, [0, 1], 0, 5)
    with pytest.raises(ValueError):
        walk_pairs(w, 0)
    with pytest.raises(TypeError):
        walk_pairs(w.cpu(), 3)


@gpu
def test_two_one_gpu_trainings_write_identical_vectors(tmp_path):
    from adapm_b200.models.node2vec import Node2Vec, num_keys
    from multirank import one_rank_store

    g, _, _ = planted_split()
    cfg = planted_config(iter=1, p=0.5, q=2.0, walkers_per_chunk=700)
    files = []
    for run in range(2):
        with one_rank_store(cfg.row_len, num_keys(g.num_nodes), "cuda", "float32") as (s, kv):
            m = Node2Vec(s, kv, g, cfg)
            m.init_model()
            m.train_epoch(0)
            path = tmp_path / f"v{run}.emb"
            m.write_vectors(str(path))
        files.append(path.read_bytes())
    assert len(files[0]) > 1000 and files[0] == files[1]


@gpu
def test_cuda_quality_on_a_planted_partition():
    share, auc, losses = train_planted("cuda")
    print(f"planted partition on the GPU: own-community share {share:.4f}, held-out AUC {auc:.4f}, losses {losses}")
    assert share >= SHARE_MIN and auc >= AUC_MIN, (share, auc)


def _rank_worker(kv, server, wid, cfg):
    from adapm_b200.models.node2vec import Node2Vec
    from adapm_b200.ops import random_walks

    g, held, neg = planted_split()
    m = Node2Vec(server, kv, g, cfg)
    starts, nums = m.epoch_starts(0)
    walks = random_walks(m.graph, starts, nums, cfg.walk_length, cfg.p, cfg.q, cfg.model_seed, 0).cpu().numpy()
    m.init_model()
    kv.barrier()
    losses = [m.train_epoch(e) for e in range(cfg.iter)]
    torch.cuda.synchronize()
    kv.wait_sync()
    kv.barrier()
    auc = m.link_prediction_auc(held, neg) if server.my_rank() == 0 else None
    kv.barrier()
    kv.finalize()
    return {"starts": starts, "nums": nums, "walks": walks, "losses": losses, "auc": auc}


@gpu
def test_three_ranks_walk_like_one_and_train_with_intents():
    from adapm_b200.models.node2vec import num_keys
    from adapm_b200.ops import random_walks

    g, _, _ = planted_split()
    cfg = planted_config(p=0.5, q=2.0, walkers_per_chunk=400)
    res = run_cluster(lambda kv, s, wid: _rank_worker(kv, s, wid, cfg), world=WORLD, workers=1, mode="threads",
                      value_lengths=cfg.row_len, num_keys=num_keys(g.num_nodes), dtype="float32", backend="cuda")
    outs = [res[r][0] for r in range(WORLD)]
    starts = np.concatenate([o["starts"] for o in outs])
    nums = np.concatenate([o["nums"] for o in outs])
    walks = np.concatenate([o["walks"] for o in outs])
    assert np.array_equal(np.sort(starts), np.repeat(np.arange(g.num_nodes), cfg.num_walks))
    one = random_walks(g.to("cuda"), starts, nums, cfg.walk_length, cfg.p, cfg.q, cfg.model_seed, 0).cpu().numpy()
    assert np.array_equal(walks, one)
    for r, o in enumerate(outs):
        assert o["starts"].size and np.all(o["starts"] % WORLD == r)
        assert all(l[1] > 0 for l in o["losses"])
    auc = outs[0]["auc"]
    print(f"three ranks: held-out AUC {auc:.4f}")
    assert auc >= AUC_MIN, auc
    assert all(res[r]["counters"]["protocol_errors"] == 0 for r in range(WORLD))
