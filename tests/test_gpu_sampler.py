"""The device key sampler (``sample_kernel``, ops_sampler.cu) draw for draw against ``ops.sample_keys_reference``.

Every draw is a pure function of ``(seed, draw, try, table, residency)``, so the keys are compared exactly, not by
histogram: a swapped hash half, a ``<=`` for ``<``, a lost stride or a wrong seed changes single keys. The tables the
kernel draws from are checked against their weights with the exact distribution of ``sampler_cases.table_errors``.
"""
import functools

import numpy as np
import pytest
import torch

from harness import run_cluster
from multirank import WORLD, make_local, one_rank_store
from sampler_cases import WEIGHT_SETS, table, table_errors, weights

pytestmark = pytest.mark.gpu

SEEDS = [7, 0xF00D_0000_0000_0000]        # the second has the high bit set; both tie u == prob[b] on the Zipf table


@pytest.fixture(scope="module")
def store():
    with one_rank_store(4, 64, "cuda", "float32") as (s, _):
        yield s


def _device_keys(sampler, n, seed, out=None, **kw):
    keys = sampler.sample(n, seed, out=out, **kw)
    torch.cuda.synchronize()
    return keys.cpu().numpy()


def _ties(prob, alias, n, seed):
    """draws whose ``u`` equals ``prob`` of their bucket and whose bucket aliases elsewhere: the draws that ``u <=
    prob`` would give the other key"""
    from adapm_b200.ops import _sampler_hash

    ties = 0
    for s in range(0, n, 1 << 22):
        h = _sampler_hash(seed, np.arange(s, min(n, s + (1 << 22)), dtype=np.uint64), 0)
        b = ((h >> np.uint64(32)) * np.uint64(prob.size) >> np.uint64(32)).astype(np.int64)
        u = (h & np.uint64(0xFFFFFFFF)).astype(np.uint32).astype(np.float32) * np.float32(2.0 ** -32)
        ties += int(((u == prob[b]) & (alias[b] != b)).sum())
    return ties


@pytest.mark.parametrize("seed", SEEDS, ids=["seed", "high-bit-seed"])
@pytest.mark.parametrize("name", WEIGHT_SETS)
def test_alias_draws_match_reference(store, name, seed):
    """The word2vec shape (Zipf^0.75 over 10^6 words, syn1 keys ``2 w + 1``) with 10^7 + 1 draws; the other sets with
    2^20 + 3 draws, at ``first_key, key_stride`` of 0, 1 and 5, 3. The table the sampler built is the builder's, and is
    checked against its weights."""
    from adapm_b200.ops import DeviceSampler, sample_keys_reference

    w = weights(name)
    first, stride = (1, 2) if name == "zipf-1m" else ((0, 1) if WEIGHT_SETS.index(name) % 2 else (5, 3))
    n = 10 ** 7 + 1 if name == "zipf-1m" else (1 << 20) + 3
    sampler = DeviceSampler(store, weights=torch.from_numpy(w), first_key=first, key_stride=stride)
    prob, alias = sampler.prob.cpu().numpy(), sampler.alias.cpu().numpy()
    want_p, want_a = table(w)
    assert np.array_equal(prob, want_p) and np.array_equal(alias, want_a)
    assert table_errors(w, prob, alias) == []
    got = _device_keys(sampler, n, seed)
    want = sample_keys_reference(n, seed, prob=prob, alias=alias, first_key=first, key_stride=stride)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (bad.size, bad[:5], got[bad[:5]], want[bad[:5]])
    if name == "zipf-1m":
        assert _ties(prob, alias, n, seed) > 0     # the draws include the edge u == prob[b]


@pytest.mark.parametrize("num_keys", [1, 50, (1 << 20) + 3, (1 << 31) - 1])
@pytest.mark.parametrize("seed", SEEDS, ids=["seed", "high-bit-seed"])
def test_uniform_draws_match_reference(store, num_keys, seed):
    from adapm_b200.ops import DeviceSampler, sample_keys_reference

    n = (1 << 20) + 5
    for first, stride in ((100, 3), (0, 1)):
        sampler = DeviceSampler(store, distribution="uniform", num_keys=num_keys, first_key=first, key_stride=stride)
        got = _device_keys(sampler, n, seed)
        want = sample_keys_reference(n, seed, distribution="uniform", num_keys=num_keys, first_key=first,
                                     key_stride=stride)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (first, stride, bad.size, bad[:5], got[bad[:5]], want[bad[:5]])


@pytest.mark.parametrize("n", [1, 31, 257, 10 ** 7 + 1])
def test_draw_counts_and_out_slices(store, n):
    """Draw counts that are not multiples of the block (256) or of the warp of the stats reduction (32), into a slice
    of a larger tensor: the elements around the slice stay as they were."""
    from adapm_b200.ops import DeviceSampler, sample_keys_reference

    w = weights("zeros")
    for sampler in (DeviceSampler(store, weights=torch.from_numpy(w), first_key=1, key_stride=2),
                    DeviceSampler(store, distribution="uniform", num_keys=1001, first_key=3)):
        big = torch.full((n + 40,), -7, dtype=torch.int64, device=store.device)
        out = _device_keys(sampler, n, SEEDS[1], out=big[17:17 + n])
        ref_kw = (dict(prob=sampler.prob.cpu().numpy(), alias=sampler.alias.cpu().numpy()) if sampler.kind == 0 else
                  dict(distribution="uniform", num_keys=sampler.n))
        want = sample_keys_reference(n, SEEDS[1], first_key=sampler.first_key, key_stride=sampler.key_stride, **ref_kw)
        assert np.array_equal(out, want)
        b = big.cpu()
        assert np.array_equal(b[17:17 + n].numpy(), want)
        assert bool((b[:17] == -7).all()) and bool((b[17 + n:] == -7).all())


LOG_WINDOW = 1e-12


@pytest.mark.parametrize("num_keys", [1000, 10 ** 5, 10 ** 6])
def test_log_uniform_draws_match_float64_rule(store, num_keys):
    """``floor(exp(u ln(n + 1))) - 1`` with ``u = hi 2^-32``: the device takes ``exp`` in double, so its keys equal the
    float64 replay except where the float64 value of ``exp(u ln(n + 1))`` lies within ``LOG_WINDOW`` (relative) of an
    integer, where the two ``exp`` may round to different sides. The mismatch rate is printed."""
    from adapm_b200.ops import DeviceSampler, _sampler_hash, sample_keys_reference

    n, first, stride = 1 << 22, 17, 2
    sampler = DeviceSampler(store, distribution="log-uniform", num_keys=num_keys, first_key=first, key_stride=stride)
    got = _device_keys(sampler, n, SEEDS[0])
    want = sample_keys_reference(n, SEEDS[0], distribution="log-uniform", num_keys=num_keys, first_key=first,
                                 key_stride=stride)
    hi = _sampler_hash(SEEDS[0], np.arange(n, dtype=np.uint64), 0) >> np.uint64(32)
    x = np.exp(hi.astype(np.float64) * 2.0 ** -32 * np.log(num_keys + 1))
    near = np.abs(x - np.rint(x)) <= LOG_WINDOW * x
    bad = got != want
    print(f"log-uniform n={num_keys}: {int(bad.sum())} of {n} draws differ from the float64 rule "
          f"(rate {bad.mean():.3g}), {int(near.sum())} within {LOG_WINDOW:g} of an integer")
    assert not (bad & ~near).any(), np.flatnonzero(bad & ~near)[:10]
    assert int(got.min()) >= first and int(got.max()) <= first + (num_keys - 1) * stride
    assert bool(((got - first) % stride == 0).all())


# ---------------------------------------------------------------------------------------------- local-only rejection
WORDS = 150          # sampled keys 2 w + 1 of a store of 2 WORDS keys, as word2vec's syn1 keys


def _local_replay_worker(kv, server, wid, weights):
    from adapm_b200.ops import DeviceSampler

    rank = server.my_rank()
    kv.barrier()
    mine = (2 * (torch.arange(rank * 30, rank * 30 + 60) % WORDS) + 1)      # overlapping sets: replicas and moves
    make_local(kv, server, mine)
    keys_all = range(2 * WORDS)
    local0 = np.array([server.is_local(k) for k in keys_all])
    out = {"local0": local0, "runs": []}
    syn1_local = local0[1::2]
    zero_local = weights * ~syn1_local         # its resident keys weigh nothing: every draw gives up
    for w, tries in ((weights, 64), (weights, 1), (weights, 2), (zero_local, 64), (zero_local, 3)):
        sampler = DeviceSampler(server, weights=torch.from_numpy(w), first_key=1, key_stride=2)
        n = (1 << 18) + 3 if tries > 3 else (1 << 16) + 1
        seed = 1000 * rank + tries
        sampler.stats.zero_()
        keys = sampler.sample(n, seed, local_only=True, max_tries=tries)
        torch.cuda.synchronize()
        out["runs"].append(dict(w=w, tries=tries, n=n, seed=seed, keys=keys.cpu().numpy(),
                                stats=sampler.stats.tolist(), prob=sampler.prob.cpu().numpy(),
                                alias=sampler.alias.cpu().numpy()))
    out["local1"] = np.array([server.is_local(k) for k in keys_all])
    out["mine_local"] = bool(local0[mine.numpy()].all())
    kv.barrier()
    kv.finalize()
    return out


def test_local_only_draws_replay_on_three_ranks():
    """After intents made a known set of keys local on every rank, ``local_only`` draws equal the replay of the
    rejection loop with the residency read from ``server.is_local``: the keys, the draws made (``stats[0]``) and the
    give-ups (``stats[1]``). At ``max_tries`` 1 and 2 draws give up and keep their last, non-resident key; on a table
    whose resident keys weigh nothing, every draw gives up after ``max_tries`` draws."""
    from adapm_b200.ops import sample_keys_reference

    g = np.random.default_rng(5)
    w = g.random(WORDS) ** 3 + 0.01
    res = run_cluster(functools.partial(_local_replay_worker, weights=w), world=WORLD, workers=1, mode="threads",
                      value_lengths=4, num_keys=2 * WORDS, dtype="float32", backend="cuda")
    for r in range(WORLD):
        out = res[r][0]
        assert out["mine_local"], r
        assert np.array_equal(out["local0"], out["local1"]), f"rank {r}: residency changed while sampling"
        resident = out["local0"]
        assert 0 < int(resident[1::2].sum()) < WORDS, int(resident[1::2].sum())
        for run in out["runs"]:
            keys, checks, misses = sample_keys_reference(run["n"], run["seed"], prob=run["prob"], alias=run["alias"],
                                                         first_key=1, key_stride=2, resident=resident,
                                                         max_tries=run["tries"])
            tag = (r, run["tries"], float(run["w"].sum()))
            bad = np.flatnonzero(run["keys"] != keys)
            assert bad.size == 0, (tag, bad.size, bad[:5])
            assert run["stats"] == [checks, misses], (tag, run["stats"], checks, misses)
            if run["w"] is not w:                               # zero-weight resident set
                assert misses == run["n"] and checks == run["n"] * run["tries"], tag
            elif run["tries"] <= 2:
                assert misses > 0, tag
            else:
                assert misses == 0, tag


# ---------------------------------------------------------------------------------------------- native SGNS loop
def test_native_sgns_loop_negatives_follow_the_seed_rule():
    """``_C.SgnsLoop`` draws the negatives of step ``s`` at seed ``(model_seed 1000003 + rank 7919 + s) mod 2^48``, as
    ``Word2Vec.sample_negatives`` does. Two steps through the loop (the second as a separate call that starts at
    batch 2) against ``ops.sgns_step`` on a second store with the negatives of ``sample_keys_reference`` at that seed:
    the one-GPU step is deterministic, so rows and losses agree bit for bit only if the negatives do."""
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts
    from adapm_b200.ops import sample_keys_reference, sgns_step

    cfg = Word2VecConfig(vocab_size=4000, embed_dim=64, negative=5, batch_pairs=1024, model_seed=(1 << 31) + 12345)
    counts = zipf_counts(cfg.vocab_size)
    data = SyntheticPairs(cfg, counts, 0)
    batches = [data.batch(s).pin_memory() for s in range(3)]
    B, neg = cfg.batch_pairs, cfg.negative
    with one_rank_store(cfg.row_len, cfg.num_keys, "cuda", "float32") as (sa, kva), \
            one_rank_store(cfg.row_len, cfg.num_keys, "cuda", "float32") as (sb, kvb):
        loop = Word2Vec(sa, kva, cfg, counts)
        loop.init_model()
        loss_host = torch.zeros(3).pin_memory()
        loop.run_steps(batches, 0, 1, loss_host=loss_host)
        loop.run_steps(batches, 2, 1, loss_host=loss_host)
        torch.cuda.synchronize()
        py = Word2Vec(sb, kvb, cfg, counts)
        py.init_model()
        losses = []
        for step, b in ((0, batches[0]), (1, batches[2])):
            seed = (cfg.model_seed * 1000003 + 0 * 7919 + step) & 0xFFFFFFFFFFFF
            negs = sample_keys_reference(B * neg, seed, prob=py.sampler.prob, alias=py.sampler.alias, first_key=1,
                                         key_stride=2)
            py.step_no = step
            assert np.array_equal(py.sample_negatives().cpu().numpy(), negs), step     # the Python path's rule
            kd = b.to(sb.device)
            loss = torch.zeros(1, device=sb.device)
            sgns_step(sb, kd[0], kd[1], torch.from_numpy(negs).to(sb.device).view(B, neg), cfg.embed_dim, py.alpha, loss)
            losses.append(float(loss.item()))
        torch.cuda.synchronize()
        rows_a, rows_b = torch.empty(cfg.num_keys * cfg.row_len), torch.empty(cfg.num_keys * cfg.row_len)
        kva.pull(torch.arange(cfg.num_keys), rows_a)
        kvb.pull(torch.arange(cfg.num_keys), rows_b)
    assert [loss_host[0].item(), loss_host[2].item()] == losses
    assert torch.equal(rows_a, rows_b)
