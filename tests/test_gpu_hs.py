"""word2vec hierarchical softmax on the GPU (ops.hs_step): the deterministic step against the float64 rule at every VPL,
with trees whose longest path is 1, a middle length, 31 and 32 nodes, bit-identical runs, launch counts, the in-place
kernel on one GPU and on multi-rank stores (peer rows, replicas, keys in flight), training end to end, and the build
budget of the new kernels."""
import glob
import os
import re
import subprocess
import sys

import pytest
import torch

from multirank import WORLD, Case, Fused, load_rows, on_peer_rows, on_replicas, one_rank_store, while_keys_move
from test_cbow_cpu import TOPIC_PRECISION
from test_hs_cpu import torch_hs_rule64, train_planted_hs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
RTOL, ATOL = 2e-4, 2e-5
ALPHA = 0.01


def _tree(kind):
    """kind: 'l1' (2 words, every path 1 node), 'mid' (3000 Zipf words), 'l31' / 'l32' (Fibonacci counts)"""
    from adapm_b200.models.word2vec import zipf_counts
    from adapm_b200.utils.text import huffman_tree

    if kind == "l1":
        return huffman_tree([3, 5])
    if kind == "mid":
        return huffman_tree(zipf_counts(3000, 1.1, total=1e6))
    fib = [1, 1]
    while len(fib) < (33 if kind == "l32" else 32):
        fib.append(fib[-1] + fib[-2])
    return huffman_tree(fib)


def _table(g, n_keys, d, tree=None):
    """random rows. With a tree, node V-3 (a child of the root, on about half the paths) is the constant row 6 and the
    syn0 rows have mean 1/d per element, so that its f = 6 sum(h) straddles 6 and many items skip it; a sum of terms of
    one sign keeps f well-conditioned near the threshold, where fp32 and float64 must agree on skipping"""
    t = torch.randn(n_keys, 2 * d, generator=g) * (0.5 / d ** 0.5)
    t[:, d:] = torch.rand(n_keys, d, generator=g) * 0.1 + 1e-3
    if tree is not None and tree.num_words >= 3:
        t[0::2, :d] += 1.0 / d
        t[2 * (tree.num_words - 3) + 1, :d] = 6.0
    return t


def _rows(kv, n, d):
    v = torch.empty(n * 2 * d, device=kv.server.device)
    kv.wait(kv.pull(torch.arange(n, device=kv.server.device), v, True))
    return v.view(n, 2 * d).cpu()


def _step(server, b, tree, d, loss, stats, deterministic=None):
    from adapm_b200.ops import hs_step

    c, x = (t.to(server.device).contiguous() for t in b)
    hs_step(server, c, x, tree, d, ALPHA, loss, stats, deterministic=deterministic)


def _updates(b, tree, skipped):
    """pushes of the rule: per active item its path nodes that were not skipped and its context occurrences"""
    c, x = b
    xm = (x >= 0) & (c >= 0).view(-1, 1)
    act = (c >= 0) & (xm.sum(1) > 0)
    w = c[act] // 2
    off = tree.offsets.cpu()
    return int((off[w + 1] - off[w]).sum()) - skipped + int(xm[act].sum())


def _batch(g, vocab, tree, B, C):
    """items over `vocab` context words and the tree's words: padding rows, items without contexts, repeated contexts"""
    V = tree.num_words
    c = 2 * torch.randint(0, V, (B,), generator=g) + 1
    lens = torch.randint(0, C + 1, (B,), generator=g)
    x = torch.where(torch.arange(C).view(1, C) < lens.view(B, 1), 2 * torch.randint(0, vocab, (B, C), generator=g), -1)
    x[:, 0] = 2 * torch.randint(0, vocab, (B,), generator=g)
    c[B - 3:] = -1                                        # padding rows
    x[0, :] = -1                                          # an item without context
    if C >= 3:
        x[1, :3] = 10                                     # word 5 three times in one item
    return c, x


# (d, C, tree): every VPL (float4 per lane: 1 up to d 128, 2 up to 256, 3 up to 336), C 1 and 10, every tree
SHAPES = [(4, 1, "mid"), (64, 10, "l1"), (100, 10, "mid"), (128, 1, "l31"), (132, 10, "l32"), (256, 10, "mid"),
          (300, 1, "mid"), (300, 10, "l32"), (336, 10, "l31"), (336, 1, "l1")]


@gpu
@pytest.mark.parametrize("d,C,kind", SHAPES)
def test_deterministic_step_matches_float64_rule(d, C, kind):
    from adapm_b200 import _C

    vocab = 3000
    g = torch.Generator().manual_seed(d * 100 + C)
    tree = _tree(kind)
    table = _table(g, 2 * vocab, d, tree)
    with one_rank_store(2 * d, 2 * vocab, "cuda", "float32") as (server, kv):
        load_rows(kv, [(torch.arange(2 * vocab), table)])
        kv.waitall()
        dev = server.device
        tdev = tree.to(dev)
        ref = table.double()
        for step in range(3):
            b = _batch(g, vocab, tree, 12_500, C)       # the root's 12 497 entries take the gather's heavy-key path
            loss = torch.zeros(1, device=dev)
            stats = torch.zeros(4, dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            n0 = _C.kernel_launches()
            _step(server, b, tdev, d, loss, stats)
            torch.cuda.synchronize()
            assert _C.kernel_launches() - n0 == 8
            ref, ref_loss, skipped = torch_hs_rule64(ref, *b, tree, d, ALPHA)
            rows = _rows(kv, 2 * vocab, d)
            what = f"d {d} C {C} tree {kind} step {step}"
            assert torch.isfinite(rows).all(), what
            torch.testing.assert_close(rows.double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"{what}: {m}")
            assert float(loss) == pytest.approx(ref_loss, rel=1e-4), what
            s = stats.tolist()
            assert s[3] == _updates(b, tree, skipped) and s[2] == 0 and s[1] == 0, (what, s)
            if kind != "l1":
                assert skipped > 0, what


def _bits_run(d, steps, tree):
    with one_rank_store(2 * d, 2 * 3000, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(1)
        load_rows(kv, [(torch.arange(6000), _table(g, 6000, d, tree))])
        kv.waitall()
        loss = torch.zeros(1, device=server.device)
        tdev = tree.to(server.device)
        for b in steps:
            _step(server, b, tdev, d, loss, None)
        torch.cuda.synchronize()
        return _rows(kv, 6000, d), loss.cpu()


@gpu
def test_two_runs_on_fresh_stores_are_bit_identical():
    g = torch.Generator().manual_seed(2)
    tree = _tree("mid")
    steps = [_batch(g, 3000, tree, 12_500, 10) for _ in range(3)]
    r1, l1 = _bits_run(300, steps, tree)
    r2, l2 = _bits_run(300, steps, tree)
    assert torch.equal(r1, r2) and torch.equal(l1, l2)


@gpu
def test_launch_counts():
    from adapm_b200 import _C

    with one_rank_store(2 * 64, 2000, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(3)
        load_rows(kv, [(torch.arange(2000), _table(g, 2000, 64))])
        b = _batch(g, 1000, _tree("l31"), 300, 8)
        tdev = _tree("l31").to(server.device)
        loss = torch.zeros(1, device=server.device)
        torch.cuda.synchronize()
        n0 = _C.kernel_launches()
        _step(server, b, tdev, 64, loss, None)
        assert _C.kernel_launches() - n0 == 8          # index, score, count, scan (2), scatter, gather, finish
        _step(server, b, tdev, 64, loss, None, deterministic=False)
        assert _C.kernel_launches() - n0 == 9          # the in-place kernel
        torch.cuda.synchronize()


@gpu
def test_argument_checks():
    from adapm_b200.ops import hs_step

    with one_rank_store(2 * 64, 2000, "cuda", "float32") as (server, kv):
        dev = server.device
        tree = _tree("mid").to(dev)
        c = torch.ones(4, dtype=torch.int64, device=dev)
        x = torch.zeros(4, 1, dtype=torch.int64, device=dev)
        loss = torch.zeros(1, device=dev)
        with pytest.raises(ValueError):
            hs_step(server, c, x, tree, 62, 0.1, loss)
        with pytest.raises(ValueError):
            hs_step(server, c, x, tree, 340, 0.1, loss)
        with pytest.raises(ValueError):
            hs_step(server, c, torch.zeros(4, 33, dtype=torch.int64, device=dev), tree, 64, 0.1, loss)
        with pytest.raises(ValueError):
            hs_step(server, c, x, type(tree)(tree.offsets, tree.nodes, tree.codes, 33), 64, 0.1, loss)
        with pytest.raises(TypeError):
            hs_step(server, c, x, _tree("mid"), 64, 0.1, loss)           # the tree on the host


def _single_items(g, words, tree, n, C):
    """n one-item steps (the root is on every path: keys are distinct within a step only with one item per step);
    contexts distinct, some padded"""
    out = []
    for _ in range(n):
        p = words[torch.randperm(words.numel(), generator=g)[:C]]
        x = (2 * p).view(1, C)
        x[0, 1:][torch.rand(C - 1, generator=g) < 0.3] = -1
        c = 2 * torch.randint(0, tree.num_words, (1,), generator=g) + 1
        out.append((c, x))
    return out


@gpu
@pytest.mark.parametrize("d,C,kind", [(64, 10, "mid"), (300, 1, "l32"), (336, 10, "l31"), (4, 10, "mid"),
                                      (132, 1, "l1"), (256, 10, "mid")])
def test_inplace_kernel_on_one_gpu_matches_rule(d, C, kind):
    from adapm_b200 import _C

    vocab = 4000
    with one_rank_store(2 * d, 2 * vocab, "cuda", "float32") as (server, kv):
        g = torch.Generator().manual_seed(d + C)
        tree = _tree(kind)
        table = _table(g, 2 * vocab, d, tree)
        load_rows(kv, [(torch.arange(2 * vocab), table)])
        kv.waitall()
        ref, ref_loss, n_upd = table.double(), 0.0, 0
        dev = server.device
        tdev = tree.to(dev)
        loss = torch.zeros(1, device=dev)
        stats = torch.zeros(4, dtype=torch.int64, device=dev)
        for b in _single_items(g, torch.arange(vocab), tree, 24, C):
            torch.cuda.synchronize()
            n0 = _C.kernel_launches()
            _step(server, b, tdev, d, loss, stats, deterministic=False)
            torch.cuda.synchronize()
            assert _C.kernel_launches() - n0 == 1
            ref, l, sk = torch_hs_rule64(ref, *b, tree, d, ALPHA)
            ref_loss += l
            n_upd += _updates(b, tree, sk)
        torch.testing.assert_close(_rows(kv, 2 * vocab, d).double(), ref, rtol=RTOL, atol=ATOL)
        assert float(loss) == pytest.approx(ref_loss, rel=1e-4)
        s = stats.tolist()
        assert s[3] == n_upd and s[2] == 0, s


# ---------------------------------------------------------------------------------------------- several ranks
DIM, CTX = 64, 6


def _apply(table, steps, tree):
    loss = 0.0
    for b in steps:
        table, l, _ = torch_hs_rule64(table, *b, tree, DIM, ALPHA)
        loss += l
    return table, loss


def _rank_steps(g, tree, n_words, n):
    return [_single_items(g, torch.arange(n_words), tree, n, CTX) for _ in range(WORLD)]


def _keys_of(steps, tree):
    off, nodes = tree.offsets, tree.nodes.long()
    ks = []
    for c, x in steps:
        ks.append(x[x >= 0])
        for w in (c[c >= 0] // 2).tolist():
            ks.append(2 * nodes[off[w]:off[w + 1]] + 1)
    return torch.unique(torch.cat(ks))


def _case(table, tree):
    """a batch is a list of steps, run one after another"""
    def open_steps(server, kv):
        tdev = tree.to(server.device)

        def run(server, steps, loss, stats):
            for b in steps:
                _step(server, b, tdev, DIM, loss, stats)

        return Fused(server, run)

    n = table.shape[0]
    return Case(2 * DIM, n, [(torch.arange(n), table)], lambda steps: _keys_of(steps, tree), open_steps)


@gpu
def test_peer_rows_match_float64_rule():
    """three ranks, no intents (2 in 3 keys owned by a peer), the ranks' steps in turn"""
    vocab = 900
    g = torch.Generator().manual_seed(21)
    tree = _tree("mid")
    table = _table(g, 2 * max(vocab, tree.num_words), DIM, tree)
    steps = _rank_steps(g, tree, vocab, 12)
    res = on_peer_rows(_case(table, tree), steps, in_turns=True)
    ref = table.double()
    for r in range(WORLD):
        before = ref
        ref, ref_l = _apply(ref, steps[r], tree)
        out = res[r]
        assert out["loss"] == pytest.approx(ref_l, rel=1e-4)
        n_upd = 0
        for b in steps[r]:
            before, _, sk = torch_hs_rule64(before, *b, tree, DIM, ALPHA)
            n_upd += _updates(b, tree, sk)
        s = out["stats"]
        assert s[3] == n_upd and s[1] > 0 and s[2] == 0, (r, s)
    torch.testing.assert_close(res[0]["rows"][0].double(), ref, rtol=RTOL, atol=ATOL)


@gpu
def test_replicas_match_float64_rule_in_turn_order():
    """replication_only, overlapping keys across ranks: ranks 0, 1, 2 run their steps in turn with a propagation round
    between them; every rank then reads the steps applied in that order"""
    vocab = 900
    g = torch.Generator().manual_seed(22)
    tree = _tree("mid")
    table = _table(g, 2 * max(vocab, tree.num_words), DIM, tree)
    steps = _rank_steps(g, tree, vocab, 8)
    res = on_replicas(_case(table, tree), steps)
    assert sum(r["counters"]["replica_setups"] for r in res) > 0
    assert all(r["counters"]["protocol_errors"] == 0 for r in res)
    ref = table.double()
    losses = []
    for r in range(WORLD):
        ref, l = _apply(ref, steps[r], tree)
        losses.append(l)
    for r in range(WORLD):
        out = res[r]
        assert out["local"], f"rank {r}: batch keys not local after the intents"
        torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"rank {r}: {m}")
        assert out["loss"] == pytest.approx(losses[r], rel=1e-4)
        assert out["stats"][1] == 0 and out["stats"][2] == 0, (r, out["stats"])


INFLIGHT_STEPS = 32


@gpu
@pytest.mark.parametrize("technique", ["relocation_only", "all"])
def test_steps_lose_no_update_while_keys_move(technique):
    """ranks 0 and 1 keep relocating all keys between them; rank 2 runs 32 one-item steps on those keys"""
    vocab = 224
    g = torch.Generator().manual_seed(23)
    tree = _tree("l31")
    table = _table(g, 2 * vocab, DIM, tree)
    steps = _single_items(g, torch.arange(vocab), tree, INFLIGHT_STEPS, CTX)
    res = while_keys_move(_case(table, tree), [[b] for b in steps], technique)
    out = res[2]
    s = out["stats"]
    relocations = sum(r["counters"]["relocations"] for r in res)
    info = f"{technique}: stats {s}, relocations {relocations}"
    print(info)
    assert relocations > 0, info
    assert all(r["counters"]["protocol_errors"] == 0 for r in res), info
    ref, n_upd, ref_loss = table.double(), 0, 0.0
    for b in steps:
        ref, l, sk = torch_hs_rule64(ref, *b, tree, DIM, ALPHA)
        n_upd += _updates(b, tree, sk)
        ref_loss += l
    assert s[3] == n_upd, info
    torch.testing.assert_close(out["rows"][0].double(), ref, rtol=RTOL, atol=ATOL, msg=lambda m: f"{info}: {m}")
    assert out["loss"] == pytest.approx(ref_loss, rel=1e-3), info


# ---------------------------------------------------------------------------------------------- end to end
@gpu
@pytest.mark.parametrize("cbow", [0, 1])
def test_hs_learns_planted_topics_on_gpu_bit_identically(cbow):
    losses, prec, rows = train_planted_hs("cuda", cbow)
    print(f"gpu hs (cbow={cbow}) planted topics: losses {losses}, topic precision {prec:.3f}")
    assert losses[-1] < losses[0]
    assert prec > TOPIC_PRECISION, prec
    _, _, rows2 = train_planted_hs("cuda", cbow)
    assert torch.equal(rows, rows2)


@gpu
@pytest.mark.parametrize("cbow", [0, 1])
def test_app_hs_on_cuda(tmp_path, cbow):
    ck = str(tmp_path / "vec")
    r = subprocess.run([sys.executable, "-m", "adapm_b200.launch", "-s", "1", "--backend", "cuda", "-m",
                        "adapm_b200.apps.word2vec", "--", "--input_file", os.path.join(ROOT, "data", "lm", "small.txt"),
                        "--embed_dim", "64", "--num_iterations", "2", "--min_count", "5", "--negative", "0", "--hs", "1",
                        "--cbow", str(cbow), "--batch_windows", "4096", "--batch_pairs", "8192", "--write_results", "1",
                        "--output_file", ck],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and os.path.exists(ck + ".epoch.1"), out[-3000:]
    assert ("windows" if cbow else "pairs") + " on rank 0" in out, out[-3000:]


# ---------------------------------------------------------------------------------------------- build budget
def test_hs_kernels_stay_within_their_register_budget():
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    for v in (1, 2, 3):
        step = k[f"hs_step_kernel<{v}>"]
        assert step["regs"] <= 104 and step["spill"] == 0, (v, step)
        score = k[f"hs_score_kernel<{v}>"]
        assert score["regs"] <= 128 and score["spill"] == 0, (v, score)


def test_hs_inplace_kernel_uses_the_tma_ring():
    import shutil

    so = glob.glob(os.path.join(ROOT, "adapm_b200", "_C*.so"))
    if not so or shutil.which("cuobjdump") is None:
        pytest.skip("no built extension or no cuobjdump")
    sass = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True).stdout
    ops, cur = set(), False
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = "hs_step_kernel" in m.group(1)
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if m and cur:
            ops.add(m.group(1))
    assert any(o.startswith("UBLKCP") for o in ops) and any(o.startswith("UBLKRED") for o in ops), sorted(ops)
