"""The fused CBOW step (csrc/cuda/ops_cbow.cu) through ``ops.cbow_step`` on an H100: the deterministic one-GPU step
against the float64 rule over consecutive steps (with a hot word that takes the heavy-key path of the gather) and bit
for bit against itself, the in-place kernel on one GPU, the in-place kernel on multi-rank stores (three logical ranks on
one GPU, run by multirank.py: peer rows, replicas, keys in flight), training end to end, and the build
budget of the kernels."""
import glob
import os
import re
import subprocess
import sys

import pytest
import torch

from multirank import (WORLD, Case, Fused, load_rows, on_peer_rows, on_replicas, one_rank_store, rejected_on_ranks,
                       while_keys_move)
from test_cbow_cpu import TOPIC_PRECISION, corner_batch, torch_rule64, train_planted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5
# (the hot word moves by up to ALPHA per context occurrence, 10 000 times per step; at 0.05 its neu1e^2 terms summed over
# three steps leave the deterministic step's fixed-point AdaGrad range of 2^27 per element and step, see ops_cbow.cu)
ALPHA = 0.01


def _table(g, n_keys, d):
    t = torch.randn(n_keys, 2 * d, generator=g) * (0.5 / d ** 0.5)
    t[:, d:] = torch.rand(n_keys, d, generator=g) * 0.1 + 1e-3
    return t


def _rows(kv, n, d):
    v = torch.empty(n * 2 * d, device=kv.server.device)
    kv.wait(kv.pull(torch.arange(n, device=kv.server.device), v, True))
    return v.view(n, 2 * d).cpu()


def _step(server, b, d, loss, stats, deterministic=None):
    dev = server.device
    from adapm_b200.ops import cbow_step

    c, x, n = (t.to(dev).contiguous() for t in b)
    cbow_step(server, c, x, n, d, ALPHA, loss, stats, deterministic=deterministic)


def _updates(b):
    """pushes of the rule: per active window its non-skipped targets and its context occurrences"""
    c, x, n = b
    xm = (x >= 0) & (c >= 0).view(-1, 1)
    act = (c >= 0) & (xm.sum(1) > 0)
    tm = torch.cat([torch.ones_like(c, dtype=torch.bool).view(-1, 1), n != c.view(-1, 1)], 1) & act.view(-1, 1)
    return int(tm.sum() + (xm & act.view(-1, 1)).sum())


HOT = 3


def _hot_batch(g, vocab, B, C, neg, step):
    """corner cases plus word HOT as a context in >= 10 000 windows and the centre of some"""
    c, x, n = corner_batch(g, vocab, B, C, neg)
    hot = torch.arange(B) % 6 != 5
    x[hot, C - 1] = 2 * HOT
    x[10:20, C - 1] = -1
    c[7 + step::97] = 2 * HOT + 1
    assert int((x == 2 * HOT).any(1).sum()) >= 10_000
    return c, x, n


# float4 per lane (VPL) 1 up to d 128, 2 up to 256, 3 up to 336
SHAPES = [(4, 5), (64, 1), (100, 25), (128, 31), (300, 25), (336, 5), (300, 1), (300, 5), (300, 31), (132, 5),
          (200, 25), (256, 31)]


@gpu
@pytest.mark.parametrize("d,neg", SHAPES)
def test_deterministic_step_matches_float64_rule(d, neg):
    from adapm_b200 import _C

    vocab = 3000
    g = torch.Generator().manual_seed(d * 100 + neg)
    table = _table(g, 2 * vocab, d)
    with one_rank_store(2 * d, 2 * vocab, "cuda", "float32") as (server, kv):
        load_rows(kv, [(torch.arange(2 * vocab), table)])
        kv.waitall()
        dev = server.device
        ref = table.double()
        for step in range(3):
            b = _hot_batch(g, vocab, 12_500, 10, neg, step)
            loss = torch.zeros(1, device=dev)
            stats = torch.zeros(4, dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            n0 = _C.kernel_launches()
            _step(server, b, d, loss, stats)
            torch.cuda.synchronize()
            assert _C.kernel_launches() - n0 == 8
            ref, ref_loss = torch_rule64(ref, *b, d, ALPHA)
            rows = _rows(kv, 2 * vocab, d)
            what = f"d {d} neg {neg} step {step}"
            assert torch.isfinite(rows).all(), what
            torch.testing.assert_close(rows.double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"{what}: {m}")
            assert float(loss) == pytest.approx(ref_loss, rel=1e-4), what
            s = stats.tolist()
            assert s[3] == _updates(b) and s[2] == 0 and s[1] == 0, (what, s)


def _bits_run(d, neg, steps):
    with one_rank_store(2 * d, 2 * 3000, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(1)
        load_rows(kv, [(torch.arange(6000), _table(g, 6000, d))])
        kv.waitall()
        loss = torch.zeros(1, device=server.device)
        for b in steps:
            _step(server, b, d, loss, None)
        torch.cuda.synchronize()
        return _rows(kv, 6000, d), loss.cpu()


@gpu
def test_two_runs_on_fresh_stores_are_bit_identical():
    g = torch.Generator().manual_seed(2)
    steps = [_hot_batch(g, 3000, 12_500, 10, 25, s) for s in range(3)]
    r1, l1 = _bits_run(300, 25, steps)
    r2, l2 = _bits_run(300, 25, steps)
    assert torch.equal(r1, r2) and torch.equal(l1, l2)


@gpu
def test_launch_counts():
    from adapm_b200 import _C

    with one_rank_store(2 * 64, 2000, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(3)
        load_rows(kv, [(torch.arange(2000), _table(g, 2000, 64))])
        b = corner_batch(g, 1000, 300, 8, 5)
        loss = torch.zeros(1, device=server.device)
        torch.cuda.synchronize()
        n0 = _C.kernel_launches()
        _step(server, b, 64, loss, None)
        assert _C.kernel_launches() - n0 == 8          # index, score, count, scan (2), scatter, gather, finish
        _step(server, b, 64, loss, None, deterministic=False)
        assert _C.kernel_launches() - n0 == 9          # the in-place kernel
        torch.cuda.synchronize()


def _distinct_batch(g, words, B, C, neg, pad=True):
    """B windows whose keys are all distinct within the step, drawn from `words` (at least B * (C + 1 + neg) words)"""
    p = words[torch.randperm(words.numel(), generator=g)]
    x = 2 * p[:B * C].view(B, C)
    t = 2 * p[B * C:B * (C + 1 + neg)].view(B, 1 + neg) + 1
    if pad:
        x[torch.rand(B, C, generator=g) < 0.3] = -1
        x[:, 0] = 2 * p[:B * C].view(B, C)[:, 0]
    return t[:, 0].contiguous(), x, t[:, 1:].contiguous()


@gpu
@pytest.mark.parametrize("d,neg", [(64, 5), (300, 25), (336, 30), (4, 1), (132, 5), (256, 30)])
def test_inplace_kernel_on_one_gpu_matches_rule(d, neg):
    from adapm_b200 import _C

    vocab = 4000
    with one_rank_store(2 * d, 2 * vocab, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(d + neg)
        table = _table(g, 2 * vocab, d)
        load_rows(kv, [(torch.arange(2 * vocab), table)])
        kv.waitall()
        ref = table.double()
        dev = server.device
        for step in range(3):
            b = _distinct_batch(g, torch.arange(vocab), 90, 10, neg)
            loss = torch.zeros(1, device=dev)
            stats = torch.zeros(4, dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            n0 = _C.kernel_launches()
            _step(server, b, d, loss, stats, deterministic=False)
            torch.cuda.synchronize()
            assert _C.kernel_launches() - n0 == 1
            ref, ref_loss = torch_rule64(ref, *b, d, ALPHA)
            torch.testing.assert_close(_rows(kv, 2 * vocab, d).double(), ref, rtol=RTOL, atol=ATOL)
            assert float(loss) == pytest.approx(ref_loss, rel=1e-4)
            s = stats.tolist()
            assert s[3] == _updates(b) and s[2] == 0, s


@gpu
def test_deterministic_true_is_rejected_on_several_ranks():
    from adapm_b200.ops import cbow_step

    def call(server):
        dev = server.device
        z = torch.zeros(4, dtype=torch.int64, device=dev)
        cbow_step(server, z, z.view(4, 1), z.view(4, 1), 8, 0.1, torch.zeros(1, device=dev), deterministic=True)

    assert rejected_on_ranks(call, value_lengths=16, num_keys=100)


# ---------------------------------------------------------------------------------------------- several ranks
DIM, NEG, CTX = 64, 5, 6


def _ranks_words(rank, m):
    return torch.arange(rank * m, (rank + 1) * m)


def _apply(table, batches):
    loss = []
    for b in batches:
        table, l = torch_rule64(table, *b, DIM, ALPHA)
        loss.append(l)
    return table, loss


def _keys_of(b):
    c, x, n = b
    k = torch.cat([c, x.reshape(-1), n.reshape(-1)])
    return torch.unique(k[k >= 0])


def _case(table):
    n = table.shape[0]
    return Case(2 * DIM, n, [(torch.arange(n), table)], _keys_of,
                lambda server, kv: Fused(server, lambda s, b, loss, stats: _step(s, b, DIM, loss, stats)))


@gpu
def test_peer_rows_match_float64_rule():
    """three ranks, no intents, disjoint words per rank (2 in 3 keys owned by a peer), all ranks at once"""
    m = 600
    g = torch.Generator().manual_seed(21)
    table = _table(g, 2 * WORLD * m, DIM)
    batches = [_distinct_batch(g, _ranks_words(r, m), 48, CTX, NEG) for r in range(WORLD)]
    res = on_peer_rows(_case(table), batches, in_turns=False)
    ref, _ = _apply(table.double(), batches)
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)
    for r in range(WORLD):
        out = res[r]
        _, (ref_l,) = _apply(table.double(), [batches[r]])
        assert out["loss"] == pytest.approx(ref_l, rel=1e-4)
        s = out["stats"]
        assert s[3] == _updates(batches[r]) and s[1] > 0 and s[2] == 0, (r, s)


@gpu
def test_replicas_match_float64_rule_in_turn_order():
    """replication_only, overlapping words across ranks (distinct within a rank): ranks 0, 1, 2 run one step each with
    a propagation round between them; every rank then reads the three steps applied in that order"""
    vocab = 900
    g = torch.Generator().manual_seed(22)
    table = _table(g, 2 * vocab, DIM)
    batches = [_distinct_batch(g, torch.arange(vocab), 40, CTX, NEG) for _ in range(WORLD)]
    res = on_replicas(_case(table), batches)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    ref, losses = _apply(table.double(), batches)
    for r in range(WORLD):
        out = res[r]
        assert out["local"], f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"rank {r}: {m}")
        assert out["loss"] == pytest.approx(losses[r], rel=1e-4)
        s = out["stats"]
        assert s[1] == 0 and s[2] == 0 and s[3] == _updates(batches[r]), (r, s)


INFLIGHT_STEPS = 32


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_steps_lose_no_update_while_keys_move(technique):
    """ranks 0 and 1 keep relocating all keys between them; rank 2 runs 32 steps on those keys (distinct within a step)"""
    vocab = 224
    g = torch.Generator().manual_seed(23)
    table = _table(g, 2 * vocab, DIM)
    steps = [_distinct_batch(g, torch.arange(vocab), 16, CTX, NEG) for _ in range(INFLIGHT_STEPS)]
    res = while_keys_move(_case(table), steps, technique)
    out = res[2]
    s = out["stats"]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: stats {s}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res), info
    assert s[3] == sum(_updates(b) for b in steps), info
    ref, losses = _apply(table.double(), steps)
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}: {m}")
    assert out["loss"] == pytest.approx(sum(losses), rel=1e-3), info


# ---------------------------------------------------------------------------------------------- end to end
@gpu
def test_cbow_learns_planted_topics_on_gpu_bit_identically():
    losses, prec, rows = train_planted("cuda")
    print(f"gpu planted topics: losses {losses}, topic precision {prec:.3f}")
    assert losses[-1] < losses[0]
    assert prec > TOPIC_PRECISION, prec
    _, _, rows2 = train_planted("cuda")
    assert torch.equal(rows, rows2)


@gpu
def test_app_cbow_on_cuda(tmp_path):
    ck = str(tmp_path / "vec")
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", "1", "--backend", "cuda", "-m",
                        "adapm_b200.apps.word2vec", "--", "--input_file", os.path.join(ROOT, "data", "lm", "small.txt"),
                        "--embed_dim", "64", "--num_iterations", "2", "--min_count", "5", "--negative", "5", "--cbow",
                        "1", "--batch_windows", "4096", "--write_results", "1", "--output_file", ck],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and os.path.exists(ck + ".epoch.1"), out[-3000:]
    assert "windows on rank 0" in out, out[-3000:]


# ---------------------------------------------------------------------------------------------- build budget
def test_cbow_kernels_stay_within_their_register_budget():
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    for v in (1, 2, 3):
        step = k[f"cbow_step_kernel<{v}>"]
        assert step["regs"] <= 104 and step["spill"] == 0, (v, step)
        score = k[f"cbow_score_kernel<{v}>"]
        assert score["regs"] <= 128 and score["spill"] == 0, (v, score)


def test_cbow_inplace_kernel_uses_the_tma_ring():
    import shutil

    so = glob.glob(os.path.join(ROOT, "adapm_b200", "_C*.so"))
    if not so or shutil.which("cuobjdump") is None:
        pytest.skip("no built extension or no cuobjdump")
    sass = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True).stdout
    ops, cur = set(), False
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = "cbow_step_kernel" in m.group(1)
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if m and cur:
            ops.add(m.group(1))
    assert any(o.startswith("UBLKCP") for o in ops) and any(o.startswith("UBLKRED") for o in ops), sorted(ops)
