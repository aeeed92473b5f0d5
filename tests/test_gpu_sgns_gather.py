"""The deterministic one-GPU SGNS step groups each step's contributions by key and lets one warp gather and apply each
row's update (a key with many contributions is split across several warps that add exact int64 partial sums). These
tests cover what that grouping has to get right: keys that are a center in some pairs and a target in others, a key with
far more contributions than one warp's range, partial vector lanes and 31 targets, and bit-for-bit repeatability."""
import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu


@pytest.fixture()
def cluster1():
    import adapm_b200 as ad

    made = []

    def make(row_len, num_keys, **kw):
        s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                      job=f"gather{len(made)}_{np.random.randint(1 << 30)}", device=0, **kw)
        w = ad.Worker(0, s)
        made.append((s, w))
        return s, w

    yield make
    for s, w in made:
        w.finalize()
        s.shutdown()


def _start_of_step_reference(ref, centers, contexts, negatives, d, alpha):
    """float64: every pair reads the rows at the start of the step, the step adds all pairs' updates."""
    B, neg = negatives.shape
    tk = torch.cat([contexts.view(B, 1), negatives], 1)
    e0, a0 = ref[centers, :d], ref[centers, d:]
    e1, a1 = ref[tk][:, :, :d], ref[tk][:, :, d:]
    label = torch.zeros(B, neg + 1, dtype=torch.float64)
    label[:, 0] = 1
    f = (e0.unsqueeze(1) * e1).sum(-1)
    gr = label - torch.sigmoid(f)
    gr = torch.where(f > 6, label - 1, gr)
    gr = torch.where(f < -6, label, gr)
    valid = torch.ones(B, neg + 1, dtype=torch.bool)
    valid[:, 1:] = negatives != contexts.view(B, 1)
    gr = gr * valid
    grad0 = (gr.unsqueeze(-1) * e1).sum(1)
    grad1 = gr.unsqueeze(-1) * e0.unsqueeze(1)
    new = ref.clone()
    new[:, :d].index_add_(0, centers, alpha * grad0 / torch.sqrt(a0 + grad0 ** 2))
    new[:, d:].index_add_(0, centers, grad0 ** 2)
    keep = valid.view(-1)
    new[:, :d].index_add_(0, tk.view(-1)[keep], (alpha * grad1 / torch.sqrt(a1 + grad1 ** 2)).view(-1, d)[keep])
    new[:, d:].index_add_(0, tk.view(-1)[keep], (grad1 ** 2).view(-1, d)[keep])
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    return new, (torch.log1p(torch.exp(-z)) * valid).sum()


def _run_steps(cluster1, d, neg, n_keys, batches, seed):
    from adapm_b200.ops import sgns_step

    server, kv = cluster1(2 * d, n_keys)
    dev = server.device
    g = torch.Generator().manual_seed(seed)
    rows = torch.empty(n_keys, 2 * d, dtype=torch.float64)
    rows[:, :d] = torch.randn(n_keys, d, generator=g, dtype=torch.float64) * 0.3
    rows[:, d:] = torch.rand(n_keys, d, generator=g, dtype=torch.float64) + 1e-3
    allk = torch.arange(n_keys)
    kv.set(allk, rows.float().clone().view(-1))
    ref = rows.float().double()
    alpha = 0.05
    for centers, contexts, negatives in batches:
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        sgns_step(server, centers.to(dev), contexts.to(dev), negatives.contiguous().to(dev), d, alpha, loss, stats,
                  impl="tma")
        torch.cuda.synchronize()
        ref, ref_loss = _start_of_step_reference(ref, centers, contexts, negatives, d, alpha)
        torch.testing.assert_close(loss.cpu()[0].double(), ref_loss, rtol=1e-4, atol=1e-3)
        got = torch.empty(n_keys * 2 * d)
        kv.pull(allk, got)
        got = got.view(n_keys, 2 * d).double()
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-5)
        ref = got      # the next step starts from the stored float32 state


@gpu
@pytest.mark.parametrize("d,neg", [(300, 25), (200, 30), (16, 30), (52, 7)])
def test_keys_that_are_centers_and_targets_in_one_step(cluster1, d, neg):
    """Centers and targets come from one small pool, so a row that one warp updates is another pair's center: the
    gather pass must use the center's start-of-step embedding, not the row it may already have updated."""
    B, words = 384, 48
    g = torch.Generator().manual_seed(7 * d + neg)
    batches = []
    for _ in range(3):
        centers = torch.randint(0, words, (B,), generator=g)
        tk = torch.randint(0, words, (B, neg + 1), generator=g)
        batches.append((centers, tk[:, 0].clone(), tk[:, 1:].contiguous()))
    _run_steps(cluster1, d, neg, words, batches, seed=d + neg)


@gpu
@pytest.mark.parametrize("d", [300, 16, 132, 256])
def test_one_key_with_more_entries_than_many_ranges(cluster1, d):
    """One negative in almost every slot of 512 pairs (about 12 800 contributions to one row, far more than one warp's
    range), another key as the context of every pair, and a few pairs whose context is that hot key."""
    B, neg, words = 512, 25, 200
    g = torch.Generator().manual_seed(d)
    batches = []
    for _ in range(2):
        centers = torch.randint(2, words, (B,), generator=g)
        contexts = torch.full((B,), 1, dtype=torch.int64)
        contexts[::37] = 0                      # negative == context: those slots add nothing
        negatives = torch.zeros(B, neg, dtype=torch.int64)
        negatives[:, -3:] = torch.randint(0, words, (B, 3), generator=g)
        batches.append((centers, contexts, negatives))
    _run_steps(cluster1, d, neg, words, batches, seed=3 * d)


@gpu
def test_zipf_steps_repeat_bit_for_bit(cluster1):
    """4096-pair Zipf steps (hot rows split across warps, centers that are also targets) give the same rows and losses
    in every run."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=20000, embed_dim=200, negative=30, batch_pairs=4096)
    counts = zipf_counts(cfg.vocab_size)
    runs = []
    for _ in range(2):
        server, kv = cluster1(cfg.row_len, cfg.num_keys)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        data = SyntheticPairs(cfg, counts, 0)
        losses = []
        for s in range(6):
            model.loss.zero_()
            model.step(data.batch(s))
            losses.append(model.loss.item())
        torch.cuda.synchronize()
        rows = torch.empty(cfg.num_keys, cfg.row_len)
        kv.pull(torch.arange(cfg.num_keys), rows)
        runs.append((losses, rows))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])


def test_deterministic_sgns_kernels_do_not_spill():
    """The score, grouping and gather kernels stay within their register bounds without spilling (ptxas, no GPU)."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    names = [n for n in k if n.startswith(("sgns_score_tma_kernel", "sgns_det_"))]
    assert {"sgns_score_tma_kernel<3>", "sgns_det_gather_kernel<3>", "sgns_det_finish_kernel"} <= set(names), names
    for n in names:
        assert k[n]["regs"] <= 128 and k[n]["spill"] == 0, (n, k[n])
