"""The gather pass of the deterministic one-GPU SGNS step finds all keys of a warp's 64-entry range at once and streams
their rows and the entries' vectors through shared-memory rings ahead of the math. These tests build steps whose key
counts put the range boundaries where that indexing can go wrong: 64 one-entry keys in one range, ranges that start
inside a key the previous range owns, light keys on either side of a key that spans many ranges, and keys with exactly
64 and 65 entries. Rows and loss are checked against the float64 start-of-step rule at row widths that use one, two
and three float4 per lane, up to d = 336, the widest row the deterministic step takes (wider rows do not fit its
score pass's ring and are trained in place)."""
import pytest
import torch

from test_gpu_sgns_gather import _run_steps, cluster1  # noqa: F401  (cluster1 is a fixture)

gpu = pytest.mark.gpu
DIMS = [16, 52, 300, 336]


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_ranges_of_distinct_one_entry_keys(cluster1, d):  # noqa: F811
    """Every key of the step has one entry, so each range holds 64 keys and its key lookup takes both lane rounds."""
    B, neg = 512, 5
    keys = torch.randperm(B * (neg + 2), generator=torch.Generator().manual_seed(d)).view(B, neg + 2)
    _run_steps(cluster1, d, neg, B * (neg + 2), [(keys[:, 0].clone(), keys[:, 1].clone(), keys[:, 2:].contiguous())],
               seed=d)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_ranges_that_start_inside_a_light_key(cluster1, d):  # noqa: F811
    """About 20 entries per key: most range boundaries fall inside a light key, which the range that holds its first
    entry applies; every key is a center in some pairs and a target in others."""
    B, neg, words = 1024, 5, 360
    g = torch.Generator().manual_seed(11 * d)
    batches = []
    for _ in range(2):
        k = torch.randint(0, words, (B, neg + 2), generator=g)
        batches.append((k[:, 0].clone(), k[:, 1].clone(), k[:, 2:].contiguous()))
    _run_steps(cluster1, d, neg, words, batches, seed=5 * d)


@gpu
@pytest.mark.parametrize("d", DIMS)
def test_light_keys_around_a_key_that_spans_ranges(cluster1, d):  # noqa: F811
    """Key 0 fills the first negative slot of every pair (1536 entries, 24 ranges) among light keys of about 8 entries.
    Key 1 is the context of exactly 64 pairs (the largest light key), key 2 of exactly 65 (the smallest heavy one);
    ten more pairs draw their context as a negative too, which adds nothing."""
    B, neg, words = 1536, 4, 1000
    g = torch.Generator().manual_seed(3 * d + 1)
    batches = []
    for _ in range(2):
        centers = torch.randint(3, words, (B,), generator=g)
        contexts = torch.randint(3, words, (B,), generator=g)
        contexts[:64] = 1
        contexts[64:129] = 2
        negatives = torch.randint(3, words, (B, neg), generator=g)
        negatives[:, 0] = 0
        negatives[200:210, 1] = contexts[200:210]
        perm = torch.randperm(B, generator=g)
        batches.append((centers[perm], contexts[perm], negatives[perm].contiguous()))
    _run_steps(cluster1, d, neg, words, batches, seed=7 * d)


@gpu
def test_zipf_steps_at_the_benchmark_width_repeat_bit_for_bit(cluster1):  # noqa: F811
    """16 384-pair Zipf steps at d = 300 and 25 negatives give the same rows and losses in two runs."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=100000, embed_dim=300, negative=25, batch_pairs=16384)
    counts = zipf_counts(cfg.vocab_size)
    runs = []
    for _ in range(2):
        server, kv = cluster1(cfg.row_len, cfg.num_keys)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        data = SyntheticPairs(cfg, counts, 0)
        losses = []
        for s in range(4):
            model.loss.zero_()
            model.step(data.batch(s))
            losses.append(model.loss.item())
        torch.cuda.synchronize()
        rows = torch.empty(cfg.num_keys, cfg.row_len)
        kv.pull(torch.arange(cfg.num_keys), rows)
        runs.append((losses, rows))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])


def test_gather_and_scatter_kernels_do_not_spill():
    """The gather kernels keep two 256-thread blocks per SM (at most 128 registers) without spilling; so does the
    scatter that writes the entry descriptors (ptxas, no GPU)."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    names = ["sgns_det_gather_kernel<%d>" % v for v in (1, 2, 3)] + ["sgns_det_group_kernel<true>"]
    for n in names:
        assert n in k, sorted(x for x in k if x.startswith("sgns_det_"))
        assert k[n]["regs"] <= 128 and k[n]["spill"] == 0, (n, k[n])
