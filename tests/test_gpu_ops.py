"""Numerics of the hand-written sm_90a kernels against plain PyTorch fp32 references."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture()
def cluster1():
    import adapm_b200 as ad

    made = []

    def make(row_len, num_keys, **kw):
        s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                      job=f"ops{len(made)}_{np.random.randint(1 << 30)}", device=0, **kw)
        w = ad.Worker(0, s)
        made.append((s, w))
        return s, w

    yield make
    for s, w in made:
        w.finalize()
        s.shutdown()


def test_extension_is_native():
    from adapm_b200 import _C

    assert _C.cuda_available()
    assert _C.__file__.endswith(".so") and "adapm_b200" in _C.__file__


def test_pull_push_set_device_and_host_paths(cluster1):
    server, kv = cluster1(64, 1000)
    dev = server.device
    g = torch.Generator().manual_seed(0)
    keys = torch.randperm(1000, generator=g)[:300]
    vals = torch.randn(300, 64, generator=g)
    # host path set, device path pull
    kv.set(keys, vals.clone().view(-1))
    out = torch.empty(300 * 64, device=dev)
    kv.wait(kv.pull(keys.to(dev), out, True))
    torch.testing.assert_close(out.cpu().view(300, 64), vals)
    # device path push (with duplicate keys: additive), host path pull
    dk = torch.cat([keys[:100], keys[:100]]).to(dev)
    dv = torch.ones(200, 64, device=dev) * 0.5
    kv.wait(kv.push(dk, dv.view(-1), True))
    out2 = torch.empty(300 * 64)
    kv.pull(keys, out2)
    ref = vals.clone()
    ref[:100] += 1.0
    torch.testing.assert_close(out2.view(300, 64), ref)
    assert kv.pull_if_local(int(keys[0]), torch.empty(64))


def test_mixed_value_lengths(cluster1):
    lens = torch.full((50,), 8, dtype=torch.int64)
    lens[10] = 20
    lens[40] = 4
    server, kv = cluster1(lens, 50)
    keys = torch.tensor([3, 10, 40, 7])
    vals = torch.arange(8 + 20 + 4 + 8, dtype=torch.float32)
    kv.push(keys, vals)
    out = torch.zeros_like(vals)
    kv.pull(keys, out)
    torch.testing.assert_close(out, vals)
    assert kv.get_key_size(10) == 20 and kv.get_key_size(40) == 4
    # device path on a mixed-length store (per-key offsets computed on the device)
    dev = server.device
    dout = torch.zeros(vals.numel(), device=dev)
    kv.wait(kv.pull(keys.to(dev), dout, True))
    torch.testing.assert_close(dout.cpu(), vals)
    kv.wait(kv.push(keys.to(dev), torch.ones(vals.numel(), device=dev), True))
    kv.pull(keys, out)
    torch.testing.assert_close(out, vals + 1)


@pytest.mark.parametrize("d,neg,impl", [(300, 25, "tma"), (300, 25, "ldg"), (128, 5, "tma"), (128, 5, "ldg"),
                                        (64, 40, "auto"), (512, 3, "auto"), (200, 30, "tma"), (16, 2, "tma")])
def test_sgns_step_matches_pytorch_reference(cluster1, d, neg, impl):
    """Distinct keys per batch -> every row is touched by exactly one pair-target, so the batched kernel and the
    PyTorch fp32 formula must agree (AdaGrad with the pulled accumulator, |f|>6 saturation, negative==target skip)."""
    from adapm_b200.ops import sgns_step

    B = 64
    n_keys = 2 * (B * (neg + 2) + 10)
    server, kv = cluster1(2 * d, n_keys)
    dev = server.device
    g = torch.Generator().manual_seed(d * 1000 + neg)
    rows = torch.empty(n_keys, 2 * d)
    rows[:, :d] = torch.randn(n_keys, d, generator=g) * 0.3
    rows[:, d:] = torch.rand(n_keys, d, generator=g) + 1e-3
    allk = torch.arange(n_keys)
    kv.set(allk, rows.clone().view(-1))
    perm = torch.randperm(n_keys // 2, generator=g)
    centers = 2 * perm[:B]
    tw = perm[B:B + B * (neg + 1)].view(B, neg + 1)
    contexts = 2 * tw[:, 0] + 1
    negatives = 2 * tw[:, 1:] + 1
    negatives[0, 0] = contexts[0]  # exercises the "negative == positive target" skip
    alpha = 0.05
    loss = torch.zeros(1, device=dev)
    stats = torch.zeros(4, dtype=torch.int64, device=dev)
    sgns_step(server, centers.to(dev), contexts.to(dev), negatives.contiguous().to(dev), d, alpha, loss, stats, impl=impl)
    torch.cuda.synchronize()
    got = torch.empty(n_keys * 2 * d)
    kv.pull(allk, got)
    got = got.view(n_keys, 2 * d)

    # ---- reference
    ref = rows.clone()
    e0, a0 = rows[centers, :d], rows[centers, d:]
    tk = torch.cat([contexts.view(B, 1), negatives], 1)
    e1, a1 = rows[tk][:, :, :d], rows[tk][:, :, d:]
    label = torch.zeros(B, neg + 1); label[:, 0] = 1
    f = (e0.unsqueeze(1) * e1).sum(-1)
    gr = label - torch.sigmoid(f)
    gr = torch.where(f > 6, label - 1, gr)
    gr = torch.where(f < -6, label, gr)
    valid = torch.ones(B, neg + 1, dtype=torch.bool)
    valid[:, 1:] = negatives != contexts.view(B, 1)
    gr = gr * valid
    grad0 = (gr.unsqueeze(-1) * e1).sum(1)
    grad1 = gr.unsqueeze(-1) * e0.unsqueeze(1)
    ref[centers, :d] += alpha * grad0 / torch.sqrt(a0 + grad0 ** 2)
    ref[centers, d:] += grad0 ** 2
    upd_e = alpha * grad1 / torch.sqrt(a1 + grad1 ** 2)
    upd_a = grad1 ** 2
    for b in range(B):
        for t in range(neg + 1):
            if valid[b, t]:
                ref[tk[b, t], :d] += upd_e[b, t]
                ref[tk[b, t], d:] += upd_a[b, t]
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-5)
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    ref_loss = (torch.log1p(torch.exp(-z)) * valid).sum()
    torch.testing.assert_close(loss.cpu()[0], ref_loss, rtol=1e-3, atol=1e-3)
    s = stats.tolist()
    assert s[1] == 0 and s[2] == 0 and s[3] == int(valid.sum()) + B


@pytest.mark.parametrize("d,neg", [(300, 25), (128, 5), (64, 2)])
def test_sgns_steps_with_repeated_keys_match_start_of_step_reference(cluster1, d, neg):
    """Few distinct keys, so every row is updated by many pairs of a step, over several steps: on one GPU every pair
    reads the state at the start of the step and the step adds all pairs' updates, which the fp64 formula below
    computes exactly (an accumulator that is not cleared, or an update applied twice, shows up in the next step)."""
    from adapm_b200.ops import sgns_step

    B, words = 256, 40
    n_keys = 2 * words
    server, kv = cluster1(2 * d, n_keys)
    dev = server.device
    g = torch.Generator().manual_seed(d + neg)
    rows = torch.empty(n_keys, 2 * d, dtype=torch.float64)
    rows[:, :d] = torch.randn(n_keys, d, generator=g, dtype=torch.float64) * 0.3
    rows[:, d:] = torch.rand(n_keys, d, generator=g, dtype=torch.float64) + 1e-3
    allk = torch.arange(n_keys)
    kv.set(allk, rows.float().clone().view(-1))
    ref = rows.float().double()
    alpha = 0.05
    for step in range(3):
        centers = 2 * torch.randint(0, words, (B,), generator=g)
        tk = 2 * torch.randint(0, words, (B, neg + 1), generator=g) + 1
        contexts, negatives = tk[:, 0].clone(), tk[:, 1:].contiguous()
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        sgns_step(server, centers.to(dev), contexts.to(dev), negatives.to(dev), d, alpha, loss, stats, impl="tma")
        torch.cuda.synchronize()

        e0, a0 = ref[centers, :d], ref[centers, d:]
        e1, a1 = ref[tk][:, :, :d], ref[tk][:, :, d:]
        label = torch.zeros(B, neg + 1, dtype=torch.float64); label[:, 0] = 1
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
        new[:, :d].index_add_(0, tk.view(-1), (alpha * grad1 / torch.sqrt(a1 + grad1 ** 2)).view(-1, d))
        new[:, d:].index_add_(0, tk.view(-1), (grad1 ** 2).view(-1, d))
        ref = new
        z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
        ref_loss = (torch.log1p(torch.exp(-z)) * valid).sum()
        torch.testing.assert_close(loss.cpu()[0].double(), ref_loss, rtol=1e-4, atol=1e-3)

        got = torch.empty(n_keys * 2 * d)
        kv.pull(allk, got)
        got = got.view(n_keys, 2 * d).double()
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-5)
        ref = got      # the next step starts from the stored float32 state


def test_device_sampler_distribution(cluster1):
    from adapm_b200.ops import DeviceSampler

    server, kv = cluster1(8, 2000)
    w = torch.tensor([1.0, 2.0, 3.0, 4.0, 0.0, 10.0])
    s = DeviceSampler(server, weights=w, first_key=1, key_stride=2)
    out = s.sample(600_000, seed=123)
    torch.cuda.synchronize()
    assert int(out.min()) >= 1 and int(out.max()) <= 11 and bool(((out - 1) % 2 == 0).all())
    freq = torch.bincount((out - 1) // 2, minlength=6).double().cpu() / out.numel()
    torch.testing.assert_close(freq, (w / w.sum()).double(), atol=3e-3, rtol=0)
    u = DeviceSampler(server, distribution="uniform", first_key=100, num_keys=50)
    o2 = u.sample(100_000, seed=5)
    assert int(o2.min()) == 100 and int(o2.max()) == 149
    # different seeds give different streams, same seed is reproducible
    assert not torch.equal(s.sample(1000, seed=1), s.sample(1000, seed=2))
    assert torch.equal(s.sample(1000, seed=9), s.sample(1000, seed=9))


def test_word2vec_training_reduces_loss(cluster1):
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=5000, embed_dim=64, negative=5, batch_pairs=2048)
    server, kv = cluster1(cfg.row_len, cfg.num_keys)
    counts = zipf_counts(cfg.vocab_size)
    model = Word2Vec(server, kv, cfg, counts)
    model.init_model()
    data = SyntheticPairs(cfg, counts, 0)
    losses = []
    for s in range(30):
        model.loss.zero_()
        model.step(data.batch(s % 3))
        losses.append(model.loss.item())
    assert losses[-1] < 0.9 * losses[0]


def test_word2vec_steps_are_deterministic_on_one_gpu(cluster1):
    """Zipf batches touch hot rows from many pairs of the same step; on one GPU the step still computes the same rows
    and losses, bit for bit, in every run."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=5000, embed_dim=64, negative=5, batch_pairs=2048)
    counts = zipf_counts(cfg.vocab_size)
    runs = []
    for _ in range(2):
        server, kv = cluster1(cfg.row_len, cfg.num_keys)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        data = SyntheticPairs(cfg, counts, 0)
        losses = []
        for s in range(20):
            model.loss.zero_()
            model.step(data.batch(s))
            losses.append(model.loss.item())
        torch.cuda.synchronize()
        rows = torch.empty(cfg.num_keys, cfg.row_len)
        kv.pull(torch.arange(cfg.num_keys), rows)
        runs.append((losses, rows))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])


def test_native_step_driver_matches_python_loop(cluster1):
    """ops.SgnsLoop (C++ step driver: prefetched H2D, sampler, fused step, D2H of the loss, clock) does per step
    exactly what the Python loop over step() does: same seeds -> same negatives -> same losses and update counts."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=4000, embed_dim=64, negative=5, batch_pairs=1024)
    counts = zipf_counts(cfg.vocab_size)
    data = SyntheticPairs(cfg, counts, 0)
    n = 12
    batches = [data.batch(s).pin_memory() for s in range(n)]
    out = []
    for native in (False, True):
        server, kv = cluster1(cfg.row_len, cfg.num_keys)
        model = Word2Vec(server, kv, cfg, counts)
        model.init_model()
        loss_host = torch.zeros(n).pin_memory()
        if native:
            model.run_steps(batches, 0, n, resident=False, loss_host=loss_host)
            torch.cuda.synchronize()
            losses = loss_host.tolist()
        else:
            losses = []
            for s in range(n):
                model.loss.zero_()
                model.step(batches[s])
                losses.append(model.loss.item())
                kv.advance_clock()
        torch.cuda.synchronize()
        out.append((losses, model.stats.tolist()[3], kv.current_clock(), model.step_no))
        kv.finalize(); server.shutdown()
    (lp, up, cp, sp), (ln, un, cn, sn) = out
    assert up == un and cp == cn == n and sp == sn == n
    assert ln[-1] < ln[0]
    # same seeds -> same negatives; the first step starts from identical tables (only the float reduction order differs),
    # later steps inherit the Hogwild races inside a step (pairs of one batch update shared rows concurrently)
    assert abs(lp[0] - ln[0]) <= 1e-4 * abs(lp[0]) + 1e-2, (lp[0], ln[0])
    assert all(abs(a - b) <= 3e-2 * abs(a) for a, b in zip(lp, ln)), (lp, ln)
    # device-resident variant
    server, kv = cluster1(cfg.row_len, cfg.num_keys)
    model = Word2Vec(server, kv, cfg, counts)
    model.init_model()
    dev_batches = [b.to(server.device) for b in batches]
    model.run_steps(dev_batches, 2, 6, resident=True, intent_batches=batches)
    torch.cuda.synchronize()
    assert model.stats.tolist()[3] > 0 and kv.current_clock() == 6


@pytest.mark.parametrize("nh", [512, 128, 20])
def test_kge_complex_step_matches_pytorch_reference(cluster1, nh):
    """Distinct keys per call -> the fused kernel must equal the reference formula evaluated in PyTorch
    (nh=20 exercises the generic scalar path: 20/8 is not integral)."""
    from adapm_b200.models.kge import KGEConfig, kge_reference_step
    from adapm_b200.ops import kge_complex_step
    import adapm_b200 as ad

    n = 48
    cfg = KGEConfig(num_entities=2 * n + 5, num_relations=n + 3, embed_dim=nh, neg_ratio=1)
    server, kv = cluster1(cfg.value_lengths(), cfg.num_keys)
    dev = server.device
    g = torch.Generator().manual_seed(nh)
    ek = torch.arange(cfg.num_entities)
    rk = torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations)
    erows = torch.cat([torch.randn(cfg.num_entities, nh, generator=g) * 0.3, torch.rand(cfg.num_entities, nh, generator=g) + 1e-3], 1)
    rrows = torch.cat([torch.randn(cfg.num_relations, nh, generator=g) * 0.3, torch.rand(cfg.num_relations, nh, generator=g) + 1e-3], 1)
    kv.set(ek, erows.clone().view(-1)); kv.set(rk, rrows.clone().view(-1))
    perm = torch.randperm(cfg.num_entities, generator=g)
    S, O = perm[:n], perm[n:2 * n]
    R = torch.randperm(cfg.num_relations, generator=g)[:n] + cfg.num_entities
    L = (torch.arange(n) % 3 == 0).float()
    loss = torch.zeros(1, device=dev)
    stats = torch.zeros(4, dtype=torch.int64, device=dev)
    kge_complex_step(server, S.to(dev), R.to(dev), O.to(dev), L.to(dev), nh, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, loss, stats)
    torch.cuda.synchronize()
    got_e = torch.empty(cfg.num_entities * 2 * nh); kv.pull(ek, got_e)
    got_r = torch.empty(cfg.num_relations * 2 * nh); kv.pull(rk, got_r)

    # reference: the same calls through a CPU store with the PyTorch formula
    ref_server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                           fabric="inproc", job=f"kgeref{nh}")
    ref_kv = ad.Worker(0, ref_server)
    ref_kv.set(ek, erows.clone().view(-1)); ref_kv.set(rk, rrows.clone().view(-1))
    ref_loss = kge_reference_step(ref_kv, S, R, O, L, cfg)
    ref_e = torch.empty_like(got_e); ref_kv.pull(ek, ref_e)
    ref_r = torch.empty_like(got_r); ref_kv.pull(rk, ref_r)
    ref_kv.finalize(); ref_server.shutdown()
    torch.testing.assert_close(got_e, ref_e, rtol=3e-4, atol=3e-5)
    torch.testing.assert_close(got_r, ref_r, rtol=3e-4, atol=3e-5)
    torch.testing.assert_close(loss.cpu()[0], torch.tensor(ref_loss), rtol=1e-3, atol=1e-3)
    assert stats.tolist()[3] == 3 * n


@pytest.mark.parametrize("algo,d,p_e,p_r", [("RESCAL", 32, 0.0, 0.0), ("RESCAL", 64, 0.0, 0.0), ("RESCAL", 12, 0.0, 0.0),
                                            ("RESCAL", 32, 0.3, 0.2), ("ComplEx", 128, 0.25, 0.4), ("ComplEx", 20, 0.5, 0.0)])
def test_kge_rescal_and_dropout_match_pytorch_reference(cluster1, algo, d, p_e, p_r):
    """The fused RESCAL kernel (s^T R o, rank-1 relation gradient) and the in-kernel dropout of both KGE kernels
    against the reference formula in PyTorch; the dropout mask is a pure function of (seed, call, row, element) that
    ``ops.kge_dropout_mask`` reproduces on the host, so the comparison is exact up to fp32 rounding."""
    from adapm_b200.models.kge import KGEConfig, kge_reference_step
    from adapm_b200.ops import kge_complex_step, kge_rescal_step, kge_dropout_mask
    import adapm_b200 as ad

    n = 40
    cfg = KGEConfig(num_entities=2 * n + 5, num_relations=n + 3, embed_dim=d, neg_ratio=1, algorithm=algo,
                    dropout_entity=p_e, dropout_relation=p_r)
    server, kv = cluster1(cfg.value_lengths(), cfg.num_keys)
    dev = server.device
    g = torch.Generator().manual_seed(d + int(100 * p_e))
    el, rl = cfg.entity_len // 2, cfg.relation_len // 2
    ek = torch.arange(cfg.num_entities)
    rk = torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations)
    erows = torch.cat([torch.randn(cfg.num_entities, el, generator=g) * 0.3, torch.rand(cfg.num_entities, el, generator=g) + 1e-3], 1)
    rrows = torch.cat([torch.randn(cfg.num_relations, rl, generator=g) * 0.3, torch.rand(cfg.num_relations, rl, generator=g) + 1e-3], 1)
    kv.set(ek, erows.clone().view(-1)); kv.set(rk, rrows.clone().view(-1))
    perm = torch.randperm(cfg.num_entities, generator=g)
    S, O = perm[:n], perm[n:2 * n]
    R = torch.randperm(cfg.num_relations, generator=g)[:n] + cfg.num_entities
    L = (torch.arange(n) % 3 == 0).float()
    loss = torch.zeros(1, device=dev)
    stats = torch.zeros(4, dtype=torch.int64, device=dev)
    seed = 0x1234_5678_9ABC
    fused = kge_complex_step if algo == "ComplEx" else kge_rescal_step
    fused(server, S.to(dev), R.to(dev), O.to(dev), L.to(dev), d, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, loss, stats,
          p_e, p_r, seed)
    torch.cuda.synchronize()
    got_e = torch.empty(cfg.num_entities * 2 * el); kv.pull(ek, got_e)
    got_r = torch.empty(cfg.num_relations * 2 * rl); kv.pull(rk, got_r)

    masks = None
    if p_e > 0 or p_r > 0:
        masks = (kge_dropout_mask(seed, n, 0, el, p_e), kge_dropout_mask(seed, n, 1, rl, p_r, relation=True),
                 kge_dropout_mask(seed, n, 2, el, p_e))
        assert p_e == 0 or 0.0 < float((masks[0] == 0).float().mean()) < 1.0
    ref_server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                           fabric="inproc", job=f"kgeref{algo}{d}{int(100 * p_e)}")
    ref_kv = ad.Worker(0, ref_server)
    ref_kv.set(ek, erows.clone().view(-1)); ref_kv.set(rk, rrows.clone().view(-1))
    ref_loss = kge_reference_step(ref_kv, S, R, O, L, cfg, masks=masks)
    ref_e = torch.empty_like(got_e); ref_kv.pull(ek, ref_e)
    ref_r = torch.empty_like(got_r); ref_kv.pull(rk, ref_r)
    ref_kv.finalize(); ref_server.shutdown()
    torch.testing.assert_close(got_e, ref_e, rtol=5e-4, atol=5e-5)
    torch.testing.assert_close(got_r, ref_r, rtol=5e-4, atol=5e-5)
    torch.testing.assert_close(loss.cpu()[0], torch.tensor(ref_loss), rtol=1e-3, atol=1e-3)
    assert stats.tolist()[3] == 3 * n


@pytest.mark.parametrize("rank", [128, 64, 10])
def test_mf_step_matches_pytorch_reference(cluster1, rank):
    from adapm_b200.models.mf import mf_reference_step
    from adapm_b200.ops import mf_step
    import adapm_b200 as ad

    n, nk = 64, 300
    server, kv = cluster1(2 * rank, nk)
    dev = server.device
    g = torch.Generator().manual_seed(rank)
    keys = torch.arange(nk)
    rows = torch.cat([torch.randn(nk, rank, generator=g) * 0.3, torch.rand(nk, rank, generator=g)], 1)
    kv.set(keys, rows.clone().view(-1))
    perm = torch.randperm(nk, generator=g)
    rk, ck = perm[:n], perm[n:2 * n]
    x = torch.randn(n, generator=g)
    rn = torch.randint(1, 50, (n,), generator=g, dtype=torch.int32)
    cn = torch.randint(1, 50, (n,), generator=g, dtype=torch.int32)
    loss = torch.zeros(1, device=dev)
    stats = torch.zeros(4, dtype=torch.int64, device=dev)
    mf_step(server, rk.to(dev), ck.to(dev), x.to(dev), rn.to(dev), cn.to(dev), rank, 0.05, 0.02, loss, stats)
    torch.cuda.synchronize()
    got = torch.empty(nk * 2 * rank); kv.pull(keys, got)
    ref_server = ad.Server(2 * rank, num_keys=nk, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc", job=f"mfref{rank}")
    ref_kv = ad.Worker(0, ref_server)
    ref_kv.set(keys, rows.clone().view(-1))
    ref_loss = mf_reference_step(ref_kv, rk, ck, x, rn, cn, rank, 0.05, 0.02)
    ref = torch.empty_like(got); ref_kv.pull(keys, ref)
    ref_kv.finalize(); ref_server.shutdown()
    torch.testing.assert_close(got, ref, rtol=3e-4, atol=3e-5)
    torch.testing.assert_close(loss.cpu()[0], torch.tensor(ref_loss), rtol=1e-3, atol=1e-3)
    assert stats.tolist()[3] == 2 * n


@pytest.mark.parametrize("d,B,Nn", [(300, 256, 128), (128, 512, 256), (64, 64, 32)])
def test_sgns_shared_negatives_tensor_core_step(cluster1, d, B, Nn):
    """Shared-negative SGNS on the wgmma GEMMs (ops_sgns_shared.cu) against the fp32 PyTorch reference of the same
    op: the contractions run with bf16 operands (fp32 accumulation), so gradients agree to bf16 rounding; the AdaGrad
    accumulator update g^2 and the embedding update are compared on the rows after ONE step."""
    from adapm_b200.ops import SgnsSharedStep, sgns_shared_reference_step

    n_keys = 2 * (B + Nn + 16)
    server, kv = cluster1(2 * d, n_keys)
    dev = server.device
    g = torch.Generator().manual_seed(17 * d + B)
    rows = torch.empty(n_keys, 2 * d)
    rows[:, :d] = torch.randn(n_keys, d, generator=g) * 0.3
    rows[:, d:] = torch.rand(n_keys, d, generator=g) + 1e-2
    allk = torch.arange(n_keys)
    kv.set(allk, rows.clone().view(-1))
    words = torch.randperm(n_keys // 2, generator=g)
    centers = 2 * words[torch.randint(0, B // 2, (B,), generator=g)]            # duplicates among the centers
    contexts = 2 * words[torch.randint(0, words.numel(), (B,), generator=g)] + 1   # ... and contexts that are negatives too
    negatives = 2 * words[:Nn] + 1
    contexts[0] = negatives[3]      # a shared negative that is the positive target of pair 0: masked for that pair
    alpha = 0.05
    step = SgnsSharedStep(server, kv, B, Nn, d)
    loss = torch.zeros(1, device=dev)
    step(centers.to(dev), contexts.to(dev), negatives.to(dev), alpha, loss)
    torch.cuda.synchronize()
    got = torch.empty(n_keys * 2 * d)
    kv.pull(allk, got)
    got = got.view(n_keys, 2 * d)
    ref, ref_loss = sgns_shared_reference_step(rows, centers, contexts, negatives, d, alpha)
    emu, emu_loss = sgns_shared_reference_step(rows, centers, contexts, negatives, d, alpha, emulate_bf16=True)
    # untouched rows are bit-identical
    touched = torch.zeros(n_keys, dtype=torch.bool)
    touched[centers] = True; touched[contexts] = True; touched[negatives] = True
    assert torch.equal(got[~touched], rows[~touched])
    # tight: against the reference with the GEMM operands rounded to bf16 like the tensor-core path (differences left:
    # accumulation order, __expf); loose: against plain fp32 (bf16 rounding of the operands, a few per cent of the step)
    for half, name in ((slice(0, d), "embedding"), (slice(d, 2 * d), "adagrad")):
        scale = (ref[:, half] - rows[:, half]).abs().max().item()
        err_emu = (got[:, half] - emu[:, half]).abs().max().item()
        err_f32 = (got[:, half] - ref[:, half]).abs().max().item()
        assert err_emu <= 1.5e-2 * scale, (name, err_emu, scale)
        assert err_f32 <= 0.12 * scale, (name, err_f32, scale)
    assert abs(loss.item() - emu_loss.item()) <= 1e-3 * abs(emu_loss.item())
    assert abs(loss.item() - ref_loss.item()) <= 1e-2 * abs(ref_loss.item())
