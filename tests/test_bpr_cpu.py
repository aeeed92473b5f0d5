"""Implicit-feedback matrix factorisation without a GPU: the BPR rule (``ops.bpr_reference_step``) against a hand-written
float64 formula and against autograd, recommendation and Recall / NDCG against brute force, the app end to end, quality
on planted data, and the build facts of the fused BPR kernel (no spills, a dispatch table that covers every
instantiation)."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_build_budget import _kernels
from test_gpu_dispatch import _param_sets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "data")


def _store(row_len, num_keys, dtype="float64"):
    import adapm_b200 as ad

    s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                  job=f"bpr_cpu_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def _table(n, r, g, acc=(0.05, 0.5)):
    t = torch.randn(n, 2 * r, generator=g, dtype=torch.float64) * 0.5
    t[:, r:] = torch.rand(n, r, generator=g, dtype=torch.float64) * (acc[1] - acc[0]) + acc[0]
    return t


def _run_rule(table, users, pos, neg, r, eps, lam):
    from adapm_b200.ops import bpr_reference_step

    n = table.shape[0]
    s, kv = _store(2 * r, n)
    try:
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        loss, pushes = bpr_reference_step(kv, users, pos, neg, r, eps, lam)
        rows = torch.empty(n * 2 * r, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, 2 * r), loss, pushes
    finally:
        kv.finalize()
        s.shutdown()


def _hand_rule(table, users, pos, neg, r, eps, lam):
    """the rule written out positive by positive, negative by negative (start-of-step reads, summed pushes)"""
    out = table.clone()
    loss = 0.0
    for b in range(users.numel()):
        u, i = int(users[b]), int(pos[b])
        w, h = table[u, :r], table[i, :r]
        C, S = 0.0, torch.zeros(r, dtype=torch.float64)
        for j in neg[b].tolist():
            hj = table[j, :r]
            x = float(w @ h - w @ hj)
            loss += math.log1p(math.exp(-x))
            c = 1.0 / (1.0 + math.exp(x))
            C += c
            S += c * hj
            g = c * w + lam * hj
            out[j, :r] += -eps * g / torch.sqrt(table[j, r:] + g * g)
            out[j, r:] += g * g
        for key, g in ((u, S - C * h + lam * w), (i, -C * w + lam * h)):
            out[key, :r] += -eps * g / torch.sqrt(table[key, r:] + g * g)
            out[key, r:] += g * g
    return out, loss


@pytest.mark.parametrize("r,n", [(4, 1), (6, 3), (16, 5)])
def test_reference_step_matches_hand_written_rule(r, n):
    """repeated users, a negative equal to its positive, a negative repeated within one positive"""
    g = torch.Generator().manual_seed(r * 10 + n)
    nu, ni = 5, 9
    table = _table(nu + ni, r, g)
    B = 7
    users = torch.tensor([0, 1, 0, 2, 3, 0, 4])
    pos = nu + torch.randint(0, ni, (B,), generator=g)
    neg = nu + torch.randint(0, ni, (B, n), generator=g)
    neg[1, 0] = pos[1]                          # a negative equal to its positive: x = 0, the two h_i terms cancel
    if n > 1:
        neg[2, 1] = neg[2, 0]                   # a negative repeated within one positive
    rows, loss, pushes = _run_rule(table, users, pos, neg, r, 0.05, 0.02)
    want, want_loss = _hand_rule(table, users, pos, neg, r, 0.05, 0.02)
    assert pushes == B * (2 + n)
    torch.testing.assert_close(rows, want, rtol=1e-12, atol=1e-12)
    assert abs(loss - want_loss) <= 1e-12 * max(1.0, want_loss)


def test_negative_equal_to_positive_cancels_on_the_item():
    """with every negative equal to the positive, x = 0 and c = 1/2 per negative: the item gets g_i = -3/2 w + lam h and
    three pushes of g_j = w / 2 + lam h, whose w terms sum to zero"""
    r, lam = 8, 0.1
    g = torch.Generator().manual_seed(3)
    table = _table(2, r, g)
    users, pos = torch.tensor([0]), torch.tensor([1])
    neg = torch.tensor([[1, 1, 1]])
    rows, loss, pushes = _run_rule(table, users, pos, neg, r, 0.05, lam)
    assert pushes == 5 and abs(loss - 3 * math.log(2.0)) < 1e-12
    w, h, ah = table[0, :r], table[1, :r], table[1, r:]
    gi, gj = -1.5 * w + lam * h, 0.5 * w + lam * h
    dv = sum(-0.05 * gg / torch.sqrt(ah + gg * gg) for gg in (gi, gj, gj, gj))
    torch.testing.assert_close(rows[1, :r], h + dv, rtol=1e-12, atol=1e-12)


def test_rule_gradient_matches_autograd():
    """distinct keys, so each row gets one push: g = -dv sqrt(acc + g^2) / eps with g^2 the accumulator's increase,
    against autograd of sum softplus(-x_j) + lam / 2 |row|^2 per push"""
    r, n, B, eps, lam = 12, 4, 6, 0.07, 0.03
    g = torch.Generator().manual_seed(11)
    nk = B * (2 + n)
    table = _table(nk, r, g)
    keys = torch.randperm(nk, generator=g)
    users, pos, neg = keys[:B], keys[B:2 * B], keys[2 * B:].view(B, n)
    rows, loss, _ = _run_rule(table, users, pos, neg, r, eps, lam)
    dv, da = rows[:, :r] - table[:, :r], rows[:, r:] - table[:, r:]
    g_rule = -dv * torch.sqrt(table[:, r:] + da) / eps
    torch.testing.assert_close(g_rule.abs(), da.sqrt(), rtol=1e-9, atol=1e-12)
    leaf = table[:, :r].clone().requires_grad_(True)
    W, H, Hn = leaf[users], leaf[pos], leaf[neg]
    x = (W * H).sum(-1, keepdim=True) - torch.einsum("br,bnr->bn", W, Hn)
    total = torch.nn.functional.softplus(-x).sum() + lam / 2 * (leaf ** 2).sum()
    total.backward()
    torch.testing.assert_close(g_rule, leaf.grad, rtol=1e-9, atol=1e-12)
    assert abs(loss - float(torch.nn.functional.softplus(-x.detach()).sum())) < 1e-9


# ---------------------------------------------------------------------------------------------- ranking
def _model(W, H, data, algorithm="dsgd", rank=None):
    """a MatrixFactorization on a float32 CPU store with factors W [m, r], H [n, r]"""
    import adapm_b200 as ad
    from adapm_b200.models.mf import MatrixFactorization, MFConfig

    m, r = W.shape
    n = H.shape[0]
    cfg = MFConfig(num_rows=m, num_cols=n, rank=r, algorithm=algorithm, loss="bpr")
    s, kv = _store(2 * r, cfg.num_keys(1), dtype="float32")
    model = MatrixFactorization(s, kv, cfg, data)
    rows = torch.zeros(m + n, 2 * r)
    rows[:m, :r], rows[m:, :r] = torch.as_tensor(W), torch.as_tensor(H)
    kv.wait(kv.set(torch.cat([torch.arange(m), torch.arange(n) + model.fck]), rows.view(-1)))
    return model, s, kv


def _brute_topk(W, H, seen_rows, k):
    """per user: items by score descending, ties to the smaller id, seen items left out, (-1, -inf) padding"""
    out_i, out_v = [], []
    for u in range(W.shape[0]):
        sc = (W[u].astype(np.float64) @ H.T.astype(np.float64))
        cand = sorted((-sc[j], j) for j in range(H.shape[0]) if j not in seen_rows[u])[:k]
        ids = [j for _, j in cand] + [-1] * (k - len(cand))
        vals = [-v for v, _ in cand] + [-math.inf] * (k - len(cand))
        out_i.append(ids); out_v.append(vals)
    return np.array(out_i), np.array(out_v)


def _ranking_data(g):
    """8 users x 12 items, integer factors (many equal scores), user 5 has seen 8 items so k = 10 pads its list"""
    from adapm_b200.models.mf import SparseMatrix

    m, n, r = 8, 12, 4
    W = np.asarray(torch.randint(-2, 3, (m, r), generator=g), dtype=np.float32)
    H = np.asarray(torch.randint(-2, 3, (n, r), generator=g), dtype=np.float32)
    H[3] = H[7]                                          # two equal items: equal scores for every user
    ii, jj = [], []
    for u in range(m):
        cnt = 8 if u == 5 else int(torch.randint(1, 5, (1,), generator=g))
        items = torch.randperm(n, generator=g)[:cnt].tolist()
        ii += [u] * cnt; jj += items
    ii, jj = np.array(ii), np.array(jj)
    ii, jj = np.concatenate([ii, ii[:3]]), np.concatenate([jj, jj[:3]])      # duplicate interactions
    data = SparseMatrix(ii, jj, np.ones(ii.shape[0], np.float32), m, n, 1, 0)
    return W, H, data


def test_seen_is_a_sorted_csr_of_the_training_items():
    from adapm_b200.models.mf import SparseMatrix

    W, H, data = _ranking_data(torch.Generator().manual_seed(1))
    off, items = data.seen([5, 0, 5])
    assert off.dtype == torch.int64 and items.dtype == torch.int64 and off[0] == 0 and off[-1] == items.numel()
    for q, u in enumerate([5, 0, 5]):
        want = sorted(set(data.j[data.i == u].tolist()))
        assert items[off[q]:off[q + 1]].tolist() == want
    two = SparseMatrix(data.i, data.j, data.x, 8, 12, 2, 1)         # rank 1 of 2 holds rows 4..7
    two.seen([4, 7])
    with pytest.raises(ValueError):
        two.seen([3])


@pytest.mark.parametrize("k", [1, 3, 10])
def test_recommend_matches_brute_force(k):
    g = torch.Generator().manual_seed(k)
    W, H, data = _ranking_data(g)
    model, s, kv = _model(W, H, data)
    try:
        users = np.arange(8)
        seen = data.seen(users)
        idx, vals = model.recommend(users, k, seen=seen)
        seen_rows = [set(seen[1][seen[0][u]:seen[0][u + 1]].tolist()) for u in users]
        bi, bv = _brute_topk(W, H, seen_rows, k)
        assert idx.dtype == torch.int64 and vals.dtype == torch.float32 and idx.shape == (8, k)
        np.testing.assert_array_equal(idx.numpy(), bi)
        np.testing.assert_array_equal(vals.numpy(), bv.astype(np.float32))
        idx2, _ = model.recommend(users, k)                            # no exclusion
        bi2, _ = _brute_topk(W, H, [set()] * 8, k)
        np.testing.assert_array_equal(idx2.numpy(), bi2)
        if k == 10:
            assert (idx[5] == -1).sum() == 6                           # 12 items, 8 seen: 4 left
    finally:
        kv.finalize()
        s.shutdown()


def test_evaluate_ranking_matches_brute_force():
    g = torch.Generator().manual_seed(7)
    W, H, data = _ranking_data(g)
    k = 3
    # held-out items: user 0 has two (one of them also a training item), user 1 only training items (empty T_u: skipped),
    # user 5 more than k, users 2, 3 one each; users 4, 6, 7 none
    tr = {u: set(data.j[data.i == u].tolist()) for u in range(8)}
    unseen = {u: [j for j in range(12) if j not in tr[u]] for u in range(8)}
    test = [(0, unseen[0][0]), (0, sorted(tr[0])[0]), (1, sorted(tr[1])[0]), (2, unseen[2][3]), (3, unseen[3][0]),
            (5, unseen[5][0]), (5, unseen[5][1]), (5, unseen[5][2]), (5, unseen[5][3]), (2, unseen[2][3])]
    ti, tj = np.array([a for a, _ in test]), np.array([b for _, b in test])
    model, s, kv = _model(W, H, data)
    try:
        rec, ndcg, users = model.evaluate_ranking(ti, tj, k)
    finally:
        kv.finalize()
        s.shutdown()
    bi, _ = _brute_topk(W, H, [tr[u] for u in range(8)], k)
    want_r, want_n, want_u = 0.0, 0.0, 0
    for u in range(8):
        T = {b for a, b in test if a == u} - tr[u]
        if not T:
            continue
        want_u += 1
        L = bi[u].tolist()
        want_r += len(set(L) & T) / min(k, len(T))
        dcg = sum(1 / math.log2(p + 2) for p, it in enumerate(L) if it in T)
        want_n += dcg / sum(1 / math.log2(p + 2) for p in range(min(k, len(T))))
    assert users == want_u == 4
    assert abs(rec - want_r) < 1e-12 and abs(ndcg - want_n) < 1e-12


# ---------------------------------------------------------------------------------------------- the app
def _launch(args, world):
    if world == 1:
        cmd = [sys.executable, "-m", "adapm_b200.apps.mf", "--backend", "cpu"] + args
    else:
        cmd = [sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu", "-m", "adapm_b200.apps.mf",
               "--"] + args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


BPR_LINE = r"\[mf\] epoch {}: local BPR loss ([\d.e+]+), eps [\d.e-]+, test recall@10 ([\d.]+), ndcg@10 ([\d.]+)"


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("algorithm", ["dsgd", "plain"])
def test_app_trains_bpr_and_reports_recall(algorithm, world):
    args = ["--loss", "bpr", "--synthetic_nnz", "40000", "--num_rows", "1000", "--num_cols", "400", "--rank", "16",
            "--epochs", "4", "--eps", "0.1", "--lambda", "0.01", "--num_negatives", "2", "--batch_nnz", "2048",
            "--algorithm", algorithm]
    rc, out = _launch(args, world)
    assert rc == 0, out[-3000:]
    first, last = re.search(BPR_LINE.format(0), out), re.search(BPR_LINE.format(3), out)
    assert first and last, out[-3000:]
    assert float(last.group(1)) < float(first.group(1)), out[-3000:]            # falling loss
    assert float(last.group(2)) > float(first.group(2)), out[-3000:]            # rising recall
    assert "protocol errors 0" in out, out[-1500:]


def test_app_bpr_on_a_coordinate_file_with_a_test_file():
    rc, out = _launch(["--dataset", os.path.join(D, "mf", "train.mmc"), "--rank", "4", "--epochs", "2", "--loss", "bpr",
                       "--eval_k", "3"], 2)
    assert rc == 0, out[-3000:]
    assert re.search(r"\[mf\] epoch 1: local BPR loss [\d.e+]+, eps [\d.e-]+, test recall@3 [\d.]+, ndcg@3 [\d.]+", out), \
        out[-3000:]


def test_squared_loss_runs_print_what_they_printed():
    """the squared-loss app ignores the BPR flags: the same run with and without them prints the same epochs"""
    base = ["--dataset", os.path.join(D, "mf", "train.mmc"), "--rank", "2", "--epochs", "3"]
    rc, out = _launch(base, 1)
    rc2, out2 = _launch(base + ["--loss", "squared", "--num_negatives", "4", "--eval_k", "5"], 1)
    assert rc == 0 and rc2 == 0, (out + out2)[-3000:]
    lines = [re.sub(r" \([\d.]+s\)", "", ln) for ln in out.splitlines() if ln.startswith("[mf] epoch")]
    lines2 = [re.sub(r" \([\d.]+s\)", "", ln) for ln in out2.splitlines() if ln.startswith("[mf] epoch")]
    assert len(lines) == 3 and lines == lines2
    assert all(re.fullmatch(r"\[mf\] epoch \d: local squared error [\d.e+-]+, eps [\d.e-]+, test rmse [\d.]+", ln)
               for ln in lines), lines


# ---------------------------------------------------------------------------------------------- quality
# Planted data and schedule shared with the GPU quality test (tests/test_gpu_bpr.py)
QUALITY = dict(users=1500, items=600, per_row=40, rank_true=8, seed=3, rank=32, eps=0.1, lam=0.01, negatives=4,
               epochs=8, batch=4096)
# Measured on the CPU backend: popularity Recall@10 0.115 (random 0.017); BPR after 8 epochs Recall@10 0.245, NDCG@10
# 0.271 (2.1x popularity). The threshold leaves room for other draws of the negatives (the GPU samples its own).
QUALITY_MIN_RATIO = 1.8


def popularity_recall(data, test, k):
    """Recall@k of ranking every user's unseen items by their training count (ties to the smaller id)"""
    from adapm_b200.ops import topk_reference

    ti, tj = test
    pairs = np.unique(ti.astype(np.int64) * data.num_cols + tj)
    pairs = pairs[~np.isin(pairs, np.unique(data.i.astype(np.int64) * data.num_cols + data.j))]
    ti, tj = pairs // data.num_cols, pairs % data.num_cols
    users, start = np.unique(ti, return_index=True)
    end = np.append(start[1:], ti.shape[0])
    off, cols = data.seen(users)
    ex = torch.zeros(users.shape[0], data.num_cols, dtype=torch.bool)
    ex[torch.repeat_interleave(torch.arange(users.shape[0]), off[1:] - off[:-1]), cols] = True
    pop = torch.from_numpy(data.col_nnz_all.astype(np.float32)).expand(users.shape[0], -1).clone()
    _, idx = topk_reference(pop, k, ex)
    return float(np.mean([np.isin(idx[r].numpy(), tj[start[r]:end[r]]).sum() / min(k, end[r] - start[r])
                          for r in range(users.shape[0])]))


def train_quality(backend, deterministic=False):
    """BPR on the planted data of QUALITY; returns (recall@10, ndcg@10, popularity recall@10, random recall@10)"""
    import adapm_b200 as ad
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    q = QUALITY
    data, test = SparseMatrix.synthetic_implicit(q["users"], q["items"], q["per_row"], q["rank_true"], 1, 0, seed=q["seed"])
    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"], algorithm="dsgd", eps=q["eps"], lam=q["lam"],
                   batch_nnz=q["batch"], loss="bpr", num_negatives=q["negatives"], bold_driver=False,
                   deterministic=deterministic)
    s = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend=backend,
                  fabric="inproc", job=f"bpr_q_{np.random.randint(1 << 30)}", **({"device": 0} if backend == "cuda" else {}))
    kv = ad.Worker(0, s)
    try:
        model = MatrixFactorization(s, kv, cfg, data)
        model.init_model()
        for e in range(q["epochs"]):
            model.run_epoch(e)
        rec, ndcg, users = model.evaluate_ranking(*test, k=10)
    finally:
        kv.finalize()
        s.shutdown()
    return rec / users, ndcg / users, popularity_recall(data, test, 10), 10 / q["items"]


def test_bpr_beats_popularity_on_planted_data():
    rec, ndcg, pop, rnd = train_quality("cpu")
    print(f"BPR recall@10 {rec:.4f} ndcg@10 {ndcg:.4f}, popularity {pop:.4f}, random {rnd:.4f}")
    assert pop > 3 * rnd                       # the popularity signal is real
    assert rec >= QUALITY_MIN_RATIO * pop, (rec, pop)


# ---------------------------------------------------------------------------------------------- build
# One row per instantiation of the fused BPR step: (kernel, rank that selects it, the numeric GPU test that runs it).
# The deterministic rows' ranks are cases of the deterministic rule test, the in-place rows' of the in-place test.
BPR_GPU = "test_gpu_bpr.py::"
BPR_DISPATCH = [
    *[(f"mf_bpr_step_kernel<{v}, true>", {"rank": r}, BPR_GPU + "test_deterministic_step_matches_float64_rule")
      for v, r in ((1, 128), (2, 132), (3, 260), (4, 512))],
    *[(f"mf_bpr_step_kernel<{v}, false>", {"rank": r}, BPR_GPU + "test_inplace_step_matches_rule_on_distinct_keys")
      for v, r in ((1, 4), (2, 256), (3, 384), (4, 512))],
]


def _bpr_kernels():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    return {name: v for name, v in k.items() if name.startswith("mf_bpr_step_kernel<")}


def test_bpr_kernels_do_not_spill():
    k = _bpr_kernels()
    assert len(k) == 8, sorted(k)
    for name, v in k.items():
        assert v["spill"] == 0, (name, v)


def test_bpr_dispatch_table_names_every_instantiation():
    built = set(_bpr_kernels())
    rows = [r[0] for r in BPR_DISPATCH]
    assert len(rows) == len(set(rows))
    assert set(rows) == built, (sorted(built - set(rows)), sorted(set(rows) - built))


def test_bpr_dispatch_shapes_are_cases_of_their_tests():
    import importlib

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    for kernel, shape, test in BPR_DISPATCH:
        mod, fn = test.split("::")
        sets = _param_sets(getattr(importlib.import_module(mod[:-3]), fn))
        assert any(all(s.get(a) == b for a, b in shape.items()) for s in sets), (kernel, shape, test)
        vpl = int(kernel.split("<")[1].split(",")[0])
        assert (shape["rank"] // 4 + 31) // 32 == vpl, (kernel, shape)
