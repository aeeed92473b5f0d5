"""GloVe on the H100: the device co-occurrence counter (``ops.glove_cooccurrence``) bit for bit against the numpy
reference, the fused step (``ops.glove_step``) against the float64 rule ``glove_reference_step`` on one GPU and on three
logical ranks of one GPU (peer rows, replicas, keys in flight), determinism of the step and of the app,
``GloVe.most_similar`` against ``topk_reference``, and quality on planted topics."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from harness import WRAP, wrap_calls
from multirank import WORLD, Case, Fused, on_peer_rows, on_replicas, one_rank_store, rejected_on_ranks, while_keys_move
from test_glove_cpu import QUALITY_MIN, SMALL, _small_sentences, train_planted

gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5
ETA, X_MAX, ALPHA = 0.05, 10.0, 0.75
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- co-occurrence
def _zipf_sentences(n_tokens, V, seed=11):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, V + 1)
    p /= p.sum()
    tok = rng.choice(V, size=n_tokens, p=p).astype(np.int32)
    lens = rng.integers(1, 40, size=n_tokens // 10)
    off = np.concatenate([[0], np.cumsum(lens)])
    off = off[off < n_tokens]
    off = np.concatenate([off, [n_tokens]]).astype(np.int64)
    return tok, off


def _device(tok, off, V, window, sym, dw, rank=0, world=1, **kw):
    from adapm_b200.ops import glove_cooccurrence

    info = {}
    r, c, x = glove_cooccurrence(torch.from_numpy(tok).cuda(), torch.from_numpy(off).cuda(), V, window, sym, dw, rank,
                                 world, info=info, **kw)
    return (r.cpu().numpy(), c.cpu().numpy(), x.cpu().numpy()), info


def _same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g, w)


MODES = [(s, w) for s in (True, False) for w in (True, False)]


@gpu
@pytest.mark.parametrize("sym,dw", MODES)
@pytest.mark.parametrize("window", [1, 5, 15, 16])
def test_device_counts_match_the_reference_on_the_small_corpus(window, sym, dw):
    from adapm_b200.utils.text import cooccurrence_reference

    sents, V = _small_sentences()
    tok = np.concatenate(sents).astype(np.int32)
    off = np.concatenate([[0], np.cumsum([s.size for s in sents])]).astype(np.int64)
    got, info = _device(tok, off, V, window, sym, dw)
    _same(got, cooccurrence_reference(sents, V, window, sym, dw))
    assert info["chunks"] == 1


@gpu
@pytest.mark.parametrize("sym,dw", MODES)
@pytest.mark.parametrize("window", [1, 5, 15, 16])
def test_device_counts_match_the_reference_on_a_zipf_corpus(window, sym, dw):
    from adapm_b200.utils.text import cooccurrence_reference

    tok, off = _zipf_sentences(1_000_000, 30_000)
    want = cooccurrence_reference([tok[off[i]:off[i + 1]] for i in range(off.size - 1)], 30_000, window, sym, dw)
    got, _ = _device(tok, off, 30_000, window, sym, dw)
    _same(got, want)
    if window == 15 and sym and dw:
        # a budget that forces many chunks and merges gives the same result
        small, info = _device(tok, off, 30_000, window, sym, dw, max_bytes=400 << 20)
        assert info["chunks"] >= 4, info
        _same(small, want)


@gpu
def test_each_rank_of_three_counts_its_rows():
    from adapm_b200.utils.text import cooccurrence_reference

    tok, off = _zipf_sentences(300_000, 5_000, seed=3)
    sents = [tok[off[i]:off[i + 1]] for i in range(off.size - 1)]
    for r in range(3):
        got, _ = _device(tok, off, 5_000, 10, True, True, r, 3)
        assert np.all(got[0] % 3 == r)
        _same(got, cooccurrence_reference(sents, 5_000, 10, True, True, r, 3))


@gpu
def test_cooccurrence_arguments_are_checked():
    from adapm_b200.ops import glove_cooccurrence

    t = torch.zeros(4, dtype=torch.int32, device="cuda")
    o = torch.tensor([0, 4], dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        glove_cooccurrence(t, o, 10, 17)
    with pytest.raises(ValueError):
        glove_cooccurrence(t, torch.tensor([0, 3], dtype=torch.int64, device="cuda"), 10, 5)
    with pytest.raises(TypeError):
        glove_cooccurrence(t.long(), o, 10, 5)
    with pytest.raises(RuntimeError):
        glove_cooccurrence(t, o, 10, 5, max_bytes=1 << 20)


# ---------------------------------------------------------------------------------------------- the step
def _init_table(V, d, g):
    D = d + 4
    t = torch.zeros(2 * V, 2 * D, dtype=torch.float64)
    t[:, :d + 1] = torch.randn(2 * V, d + 1, generator=g, dtype=torch.float64) * (0.5 / d ** 0.5)
    t[:, D:D + d + 1] = torch.rand(2 * V, d + 1, generator=g, dtype=torch.float64) + 0.5
    return t


def _batch(V, B, g, distinct=False, hot=False):
    """(word keys 2 i, context keys 2 j + 1, X); hot: word 0 in every other of the first 64 non-zeros, context 1 in the
    others, and X >= x_max for some"""
    if distinct:
        i, j = torch.randperm(V, generator=g)[:B], torch.randperm(V, generator=g)[:B]
    else:
        i, j = torch.randint(0, V, (B,), generator=g), torch.randint(0, V, (B,), generator=g)
        if hot:
            i[:64:2] = 0
            j[1:64:2] = 0
    x = torch.rand(B, generator=g) * 2 * X_MAX + 0.05
    return 2 * i, 2 * j + 1, x.float()


def _rule(table, batches, d):
    from adapm_b200.ops import glove_reference_step

    n = table.shape[0]
    with one_rank_store(2 * (d + 4), n, "cpu", "float64") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        loss, pushes = 0.0, 0
        for b in batches:
            l, u = glove_reference_step(kv, *b, d, ETA, X_MAX, ALPHA)
            loss += l; pushes += u
        rows = torch.empty(n * 2 * (d + 4), dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, -1), loss, pushes


def _fused(table, batches, d, deterministic):
    from adapm_b200 import _C
    from adapm_b200.ops import glove_step

    n = table.shape[0]
    with one_rank_store(2 * (d + 4), n, "cuda", "float32") as (s, kv):
        kv.wait(kv.set(torch.arange(n), table.float().contiguous().view(-1)))
        dev = s.device
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        l0 = _C.kernel_launches()
        for b in batches:
            glove_step(s, *(t.to(dev).contiguous() for t in b), d, ETA, X_MAX, ALPHA, loss, stats,
                       deterministic=deterministic)
        torch.cuda.synchronize()
        launches = _C.kernel_launches() - l0
        rows = torch.empty(n * 2 * (d + 4), dtype=torch.float32)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, -1).double(), float(loss.item()), stats.tolist(), launches


# D = d + 4 float4 per row: VPL 1 up to d = 124, 2 up to 252, 3 up to 380; larger d take the generic path
DIMS = (4, 124, 128, 252, 256, 300, 380, 384, 508)


@gpu
@pytest.mark.parametrize("d,B", [pytest.param(d, 300, id=str(d)) for d in DIMS] + [pytest.param(124, WRAP, id="124-wrap")])
def test_deterministic_step_matches_float64_rule(d, B):
    """hot repeated words and contexts, X on both sides of x_max; two steps; bit-identical reruns"""
    B = wrap_calls(B, 3)
    V = max(400, B // 2)
    g = torch.Generator().manual_seed(d * 7 + 1)
    table = _init_table(V, d, g)
    batches = [_batch(V, B, g, hot=True) for _ in range(2)]
    ref, ref_loss, ref_pushes = _rule(table, batches, d)
    rows, loss, stats, launches = _fused(table, batches, d, deterministic=True)
    assert launches == 3 * len(batches)                  # index, step, apply
    assert stats[3] == ref_pushes == len(batches) * 2 * B, (stats, ref_pushes)
    assert stats[2] == (len(batches) * B if d > 380 else 0), stats
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss), (loss, ref_loss)
    rows2, loss2, _, _ = _fused(table, batches, d, deterministic=True)
    assert torch.equal(rows, rows2) and loss == loss2


@gpu
@pytest.mark.parametrize("d,B", [pytest.param(d, 150, id=str(d)) for d in DIMS] + [pytest.param(4, WRAP, id="4-wrap")])
def test_inplace_step_matches_rule_on_distinct_keys(d, B):
    B = wrap_calls(B, 3)
    V = 2 * B
    g = torch.Generator().manual_seed(d * 11 + 2)
    table = _init_table(V, d, g)
    batches = [_batch(V, B, g, distinct=True) for _ in range(2)]
    ref, ref_loss, ref_pushes = _rule(table, batches, d)
    rows, loss, stats, launches = _fused(table, batches, d, deterministic=False)
    assert launches == len(batches)
    generic = d > 380                                    # every non-zero takes the generic path (one slow count each)
    assert stats[3] == ref_pushes and stats[0] == (0 if generic else len(batches) * 2 * B), stats
    assert stats[2] == (len(batches) * B if generic else 0), stats
    torch.testing.assert_close(rows, ref, rtol=RTOL, atol=ATOL)
    assert abs(loss - ref_loss) <= 1e-4 * max(1.0, ref_loss)


@gpu
def test_step_arguments_are_checked():
    from adapm_b200.ops import glove_step

    with one_rank_store(16, 64, "cuda", "float32") as (s, kv):
        dev = s.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        x = torch.ones(2, device=dev)
        loss = torch.zeros(1, device=dev)
        for d in (6, 0, 512):
            with pytest.raises(ValueError):
                glove_step(s, k, k + 1, x, d, 0.1, 10.0, 0.75, loss)
        with pytest.raises(ValueError):
            glove_step(s, k, k + 1, torch.ones(3, device=dev), 4, 0.1, 10.0, 0.75, loss)
        with pytest.raises(TypeError):
            glove_step(s, k.int(), k + 1, x, 4, 0.1, 10.0, 0.75, loss)


@gpu
def test_deterministic_step_rejected_on_several_ranks():
    from adapm_b200.ops import glove_step

    def call(server):
        dev = server.device
        k = torch.zeros(2, dtype=torch.int64, device=dev)
        glove_step(server, k, k + 1, torch.ones(2, device=dev), 4, 0.1, 10.0, 0.75, torch.zeros(1, device=dev),
                   deterministic=True)

    assert rejected_on_ranks(call)


# ---------------------------------------------------------------------------------------------- three ranks, one GPU
def _case(table, d):
    from adapm_b200.ops import glove_step

    def step(server, b, loss, stats):
        dev = server.device
        glove_step(server, *(t.to(dev).contiguous() for t in b), d, ETA, X_MAX, ALPHA, loss, stats)

    n = table.shape[0]
    return Case(2 * (d + 4), n, [(torch.arange(n), table)], lambda b: torch.unique(torch.cat([b[0], b[1]])),
                lambda server, kv: Fused(server, step))


@gpu
def test_step_on_peer_rows():
    V, B, d = 1500, 200, 128
    g = torch.Generator().manual_seed(5)
    table = _init_table(V, d, g)
    batches = [_batch(V, B, g, distinct=True) for _ in range(WORLD)]
    res = on_peer_rows(_case(table, d), batches, in_turns=True)
    ref, ref_loss, ref_pushes = _rule(table, batches, d)
    assert sum(x["stats"][3] for x in res) == ref_pushes
    assert sum(x["stats"][1] for x in res) > 0
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(sum(x["loss"] for x in res), ref_loss, rtol=1e-4, atol=1e-3)


@gpu
def test_step_on_replicas():
    B, d = 60, 300
    V = 2 * B
    g = torch.Generator().manual_seed(21)
    table = _init_table(V, d, g)
    batches = [_batch(V, B, g, distinct=True) for _ in range(WORLD)]
    res = on_replicas(_case(table, d), batches)
    assert sum(x["counters"]["replica_setups"] for x in res) > 0
    assert all(x["counters"]["protocol_errors"] == 0 for x in res)
    ref, _, _ = _rule(table, batches, d)
    for k in range(WORLD):
        out = res[k]
        assert out["local"] and out["replicas"] > 0, f"rank {k}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
        s = out["stats"]
        assert s[0] == 2 * B and s[1] == 0 and s[2] == 0 and s[3] == 2 * B, (k, s)


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_step_loses_no_update_while_keys_move(technique):
    V, B, d = 256, 32, 64
    g = torch.Generator().manual_seed(9)
    table = _init_table(V, d, g)
    batches = [_batch(V, B, g, distinct=True) for _ in range(32)]
    res = while_keys_move(_case(table, d), batches, technique)
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    info = f"{technique}: stats {out['stats']}, relocations {relocations}"
    print(info)
    assert relocations > 0 and all(x["counters"]["protocol_errors"] == 0 for x in res), info
    ref, ref_loss, ref_pushes = _rule(table, batches, d)
    assert out["stats"][3] == ref_pushes == 32 * 2 * B, info
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(out["loss"], ref_loss, rtol=1e-4, atol=1e-3)


# ---------------------------------------------------------------------------------------------- model and app
@gpu
def test_most_similar_matches_topk_reference(tmp_path):
    from adapm_b200.models.glove import GloVe, GloVeConfig
    from adapm_b200.ops import exclusion_mask, gemm_nt_bf16, topk_reference
    from adapm_b200.utils.text import NativeCorpus

    corpus = NativeCorpus.build(SMALL, 5)
    corpus.encode(SMALL, 0, 1)
    V = len(corpus.vocabulary().words)
    cfg = GloVeConfig(vocab_size=V, embed_dim=32, window=5, batch_entries=8192, deterministic=True)
    with one_rank_store(cfg.row_len, cfg.num_keys, "cuda", "float32") as (s, kv):
        model = GloVe(s, kv, cfg)
        model.init_model()
        model.build_cooccurrence(corpus)
        for e in range(3):
            model.train_epoch(e)
        q = torch.arange(1, 200)
        idx, vals = model.most_similar(q, 10)
        E = model.vectors()
    inv = 1.0 / E.norm(dim=1)
    qq = E[q.cuda()] * inv[q.cuda()].view(-1, 1)
    scores = gemm_nt_bf16(qq, E) * inv.view(1, -1)
    excl = exclusion_mask((torch.arange(q.numel() + 1, device="cuda"), q.cuda()), V)
    rv, ri = topk_reference(scores, 10, excl)
    assert torch.equal(idx, ri) and torch.equal(vals, rv)
    assert not bool((idx == q.cuda().view(-1, 1)).any())


@gpu
def test_gpu_quality_on_planted_topics(tmp_path):
    share, losses = train_planted(tmp_path, "cuda", deterministic=True)
    print(f"planted topics on the GPU: own-topic share {share:.4f}, losses {losses[0]:.1f} -> {losses[-1]:.1f}")
    assert losses[-1] < losses[0]
    assert share >= QUALITY_MIN, share


@gpu
def test_app_writes_identical_vectors_twice_in_deterministic_mode(tmp_path):
    outs = []
    for run in range(2):
        out = str(tmp_path / f"v{run}.txt")
        r = subprocess.run([sys.executable, "-m", "adapm_b200.apps.glove", "--input_file", SMALL, "--vector_size", "32",
                            "--iter", "5", "--backend", "cuda", "--deterministic", "1", "--output_file", out], cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        assert "[glove] iter 5: cost" in r.stdout
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] and len(outs[0]) > 0
