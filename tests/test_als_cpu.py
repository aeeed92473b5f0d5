"""Alternating least squares without a GPU: the float64 rule (``ops.als_reference_solve``) against ``numpy.linalg.solve``
and against the gradient of the dense Hu-Koren-Volinsky objective, the monotone objective of the model, argument
checks, the app end to end, quality on planted data, and the build facts of the ALS kernels (no spills, a dispatch
table that covers every instantiation)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_bpr_cpu import QUALITY, popularity_recall
from test_build_budget import _kernels
from test_gpu_dispatch import _param_sets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "data")


def _store(row_len, num_keys, dtype="float64"):
    import adapm_b200 as ad

    s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                  job=f"als_cpu_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def _run(table, *args, **kw):
    from adapm_b200.ops import als_reference_solve

    n, L = table.shape
    s, kv = _store(L, n)
    try:
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        solved = als_reference_solve(kv, *args, **kw)
        rows = torch.empty(n * L, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, L), solved
    finally:
        kv.finalize()
        s.shutdown()


@pytest.mark.parametrize("implicit", [False, True])
def test_reference_solve_matches_numpy_on_hand_built_systems(implicit):
    """targets 0..3 (target 1 without entries, target 2 with a duplicate entry), other rows 4..9"""
    r, lam = 4, 0.3
    g = torch.Generator().manual_seed(2)
    table = torch.randn(10, 2 * r, generator=g, dtype=torch.float64)
    targets = torch.tensor([2, 0, 1, 3])
    ents = {2: [(5, 2.0), (5, 2.0), (7, 1.0)], 0: [(4, 1.0), (9, 3.0)], 1: [], 3: [(8, 0.5), (6, 4.0), (4, 1.0)]}
    offsets = torch.tensor([0, 3, 5, 5, 8])
    others = torch.tensor([o for t in targets.tolist() for o, _ in ents[t]])
    x = torch.tensor([v for t in targets.tolist() for _, v in ents[t]], dtype=torch.float64)
    alpha = 1.5
    a, b = (alpha * x, 1 + alpha * x) if implicit else (torch.ones_like(x), x)
    H = table[:, :r].numpy()
    G = H[4:].T @ H[4:] if implicit else np.zeros((r, r))
    rows, solved = _run(table, targets, offsets, others, a.float(), b.float(), r, lam,
                        torch.from_numpy(G) if implicit else None)
    assert solved == 4
    for t in targets.tolist():
        A, rhs = G + lam * np.eye(r), np.zeros(r)
        for o, v in ents[t]:                    # a duplicate entry counts twice
            c = alpha * v if implicit else 1.0
            A += c * np.outer(H[o], H[o])
            rhs += (1 + alpha * v if implicit else v) * H[o]
        np.testing.assert_allclose(rows[t, :r].numpy(), np.linalg.solve(A, rhs), rtol=1e-10, atol=1e-12)
        np.testing.assert_array_equal(rows[t, r:].numpy(), table[t, r:].numpy())          # AdaGrad half untouched
    np.testing.assert_array_equal(rows[1, :r].numpy(), np.zeros(r))                       # no entries: r = 0 -> 0
    np.testing.assert_array_equal(rows[4:].numpy(), table[4:].numpy())


def test_implicit_half_step_zeroes_the_gradient_of_the_dense_objective():
    """m x n toy problem in float64: after solving every user, d/dW of sum_{u,i} c_ui (p_ui - w_u.h_i)^2 + lam |W|^2
    vanishes (autograd over the full matrix; c = 1 + alpha x and p = 1 on entries, c = 1 and p = 0 elsewhere)"""
    m, n, r, lam, alpha = 7, 9, 4, 0.2, 3.0
    g = torch.Generator().manual_seed(5)
    table = torch.randn(m + n, 2 * r, generator=g, dtype=torch.float64)
    X = (torch.rand(m, n, generator=g) < 0.3).double() * torch.randint(1, 4, (m, n), generator=g)
    X[3] = 0.0                                  # a user without entries
    ui, ii = X.nonzero(as_tuple=True)
    x = X[ui, ii]
    offsets = torch.zeros(m + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.bincount(ui, minlength=m), 0)
    H = table[m:, :r]
    rows, _ = _run(table, torch.arange(m), offsets, ii + m, (alpha * x).float(), (1 + alpha * x).float(), r, lam,
                   H.t() @ H)
    W = rows[:m, :r].clone().requires_grad_(True)
    C, P = 1 + alpha * X, (X > 0).double()
    loss = (C * (P - W @ H.t()) ** 2).sum() + lam * (W ** 2).sum()
    loss.backward()
    assert float(W.grad.abs().max()) < 1e-10, W.grad


# Planted data of the BPR quality test (tests/test_bpr_cpu.py), trained by implicit ALS
ALS_QUALITY = dict(QUALITY, lam=5.0, alpha=4.0, epochs=4)
# Measured on the CPU backend (float64): implicit ALS after 4 epochs Recall@10 0.258, NDCG@10 0.292 against 0.115 for
# popularity (2.25x; BPR reaches 0.245). The threshold leaves room for fp32 on the GPU.
ALS_QUALITY_MIN_RATIO = 2.0


def train_als_quality(backend, dtype="float32"):
    """implicit ALS on ALS_QUALITY's planted data; returns (recall@10, ndcg@10, popularity recall@10, the objective
    after every half-step)"""
    import adapm_b200 as ad
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    q = ALS_QUALITY
    data, test = SparseMatrix.synthetic_implicit(q["users"], q["items"], q["per_row"], q["rank_true"], 1, 0, seed=q["seed"])
    cfg = MFConfig(num_rows=q["users"], num_cols=q["items"], rank=q["rank"], algorithm="als", loss="implicit",
                   lam=q["lam"], alpha=q["alpha"])
    s = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend=backend,
                  fabric="inproc", job=f"als_q_{np.random.randint(1 << 30)}", dtype=dtype,
                  **({"device": 0} if backend == "cuda" else {}))
    kv = ad.Worker(0, s)
    try:
        model = MatrixFactorization(s, kv, cfg, data)
        model.init_model()
        objs = [model.als_objective()]
        for _ in range(q["epochs"]):
            for side in ("rows", "cols"):
                model.als_half_step(side)
                objs.append(model.als_objective())
        rec, ndcg, users = model.evaluate_ranking(*test, k=10)
    finally:
        kv.finalize()
        s.shutdown()
    return rec / users, ndcg / users, popularity_recall(data, test, 10), objs


def test_implicit_als_beats_popularity_and_never_increases_its_objective():
    rec, ndcg, pop, objs = train_als_quality("cpu", dtype="float64")
    print(f"ALS recall@10 {rec:.4f} ndcg@10 {ndcg:.4f}, popularity {pop:.4f}; objective {objs}")
    assert rec >= ALS_QUALITY_MIN_RATIO * pop, (rec, pop)
    assert all(b <= a * (1 + 1e-12) for a, b in zip(objs, objs[1:])), objs


def test_explicit_objective_never_increases_over_six_half_steps():
    import adapm_b200 as ad
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    data = SparseMatrix.synthetic(300, 120, 6000, 6, 1, 0, seed=4)
    cfg = MFConfig(num_rows=300, num_cols=120, rank=8, algorithm="als", lam=0.5)
    s, kv = _store(cfg.row_len, cfg.num_keys(1))
    try:
        model = MatrixFactorization(s, kv, cfg, data)
        model.init_model()
        objs = [model.als_objective()]
        for side in ("rows", "cols") * 3:
            model.als_half_step(side)
            objs.append(model.als_objective())
    finally:
        kv.finalize()
        s.shutdown()
    assert all(b <= a * (1 + 1e-12) for a, b in zip(objs, objs[1:])), objs
    assert objs[-1] < 0.5 * objs[0], objs


def test_arguments_are_checked():
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix
    from adapm_b200.ops import als_reference_solve

    s, kv = _store(16, 64)
    try:
        t, off, o, one = torch.tensor([0, 1]), torch.tensor([0, 1, 2]), torch.tensor([10, 11]), torch.ones(2)
        bad = [dict(rank=6), dict(rank=132), dict(rank=0), dict(lam=0.0), dict(lam=-1.0), dict(a=-one),
               dict(t=torch.tensor([0, 0])), dict(off=torch.tensor([0, 2, 1])), dict(off=torch.tensor([1, 1, 2])),
               dict(off=torch.tensor([0, 1, 3])), dict(gram=torch.zeros(4, 4)), dict(b=torch.ones(3))]
        for kw in bad:
            args = dict(t=t, off=off, o=o, a=one, b=one, rank=8, lam=0.1, gram=None) | kw
            with pytest.raises(ValueError):
                als_reference_solve(kv, args["t"], args["off"], args["o"], args["a"], args["b"], args["rank"],
                                    args["lam"], args["gram"])
        data = SparseMatrix(np.array([0]), np.array([0]), np.ones(1, np.float32), 4, 4, 1, 0)
        for cfg in (MFConfig(num_rows=4, num_cols=4, rank=4, algorithm="als", loss="bpr"),
                    MFConfig(num_rows=4, num_cols=4, rank=4, algorithm="dsgd", loss="implicit"),
                    MFConfig(num_rows=4, num_cols=4, rank=4, algorithm="als", lam=0.0)):
            with pytest.raises(ValueError):
                MatrixFactorization(s, kv, cfg, data)
    finally:
        kv.finalize()
        s.shutdown()


def test_csr_blocks_hold_every_row_longest_first():
    from adapm_b200.models.mf import SparseMatrix

    i = np.array([0, 5, 5, 2, 5, 2, 7, 1])
    j = np.array([3, 1, 1, 0, 2, 3, 0, 2])
    data = SparseMatrix(i, j, np.arange(8, dtype=np.float32), 8, 4, 2, 1)     # rank 1 of 2: rows 4..7, columns 2..3
    t, off, o, x = data.als_csr("rows")
    assert t.tolist() == [5, 7, 4, 6] and off.tolist() == [0, 3, 4, 4, 4]
    assert o.tolist() == [1, 1, 2, 0] and x.tolist() == [1, 2, 4, 6]
    t, off, o, x = data.als_csr("cols")
    assert t.tolist() == [2, 3] and off.tolist() == [0, 2, 4]                # equal counts: the smaller column first
    assert o.tolist() == [5, 1, 0, 2] and x.tolist() == [4, 7, 0, 5]        # every rank's entries of the block


# ---------------------------------------------------------------------------------------------- the app
def _launch(args, world):
    if world == 1:
        cmd = [sys.executable, "-m", "adapm_b200.apps.mf", "--backend", "cpu"] + args
    else:
        cmd = [sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu", "-m", "adapm_b200.apps.mf",
               "--"] + args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


OBJ = r"\[mf\] epoch {}: objective ([\d.e+]+)"


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("loss", ["squared", "implicit"])
def test_app_trains_als(loss, world):
    args = ["--algorithm", "als", "--loss", loss, "--synthetic_nnz", "40000", "--num_rows", "1000", "--num_cols", "400",
            "--rank", "16", "--epochs", "3", "--lambda", "1.0", "--alpha", "2"]
    rc, out = _launch(args, world)
    assert rc == 0, out[-3000:]
    objs = [float(re.search(OBJ.format(e), out).group(1)) for e in range(3)]
    assert objs[2] <= objs[1] <= objs[0], (objs, out[-3000:])
    if loss == "implicit":
        m = re.search(OBJ.format(2) + r", test recall@10 ([\d.]+), ndcg@10 ([\d.]+)", out)
        assert m and float(m.group(2)) > 0.1, out[-3000:]
    assert "protocol errors 0" in out, out[-1500:]


def test_app_als_on_a_coordinate_file_with_a_test_file():
    path = os.path.join(D, "mf", "train.mmc")
    rc, out = _launch(["--dataset", path, "--rank", "4", "--epochs", "2", "--algorithm", "als"], 2)
    assert rc == 0, out[-3000:]
    assert re.search(OBJ.format(1) + r", test rmse [\d.]+", out), out[-3000:]
    # its values are centred ratings: implicit feedback needs interaction strengths >= 0
    rc, out = _launch(["--dataset", path, "--rank", "4", "--epochs", "1", "--algorithm", "als", "--loss", "implicit"], 1)
    assert rc != 0 and "needs entry values >= 0" in out, out[-3000:]


def test_app_rejects_als_with_bpr_and_implicit_without_als():
    for args in (["--algorithm", "als", "--loss", "bpr"], ["--loss", "implicit"]):
        rc, out = _launch(args + ["--num_rows", "10", "--num_cols", "10", "--epochs", "1"], 1)
        assert rc != 0 and "error" in out, out[-2000:]


# ---------------------------------------------------------------------------------------------- build
# One row per instantiation of the ALS kernels: (kernel, shape that selects it, the numeric GPU test that runs it). The
# padded rank KP is 32 up to rank 32, 64 up to 64 and 128 above.
ALS_GPU = "test_gpu_als.py::test_solve_matches_float64_rule"
ALS_DISPATCH = [
    *[(f"als_solve_kernel<{kp}>", {"rank": r}, ALS_GPU) for kp, r in ((32, 4), (64, 64), (128, 128))],
    *[(f"als_gram_kernel<{kp}>", {"rank": r, "implicit": True}, ALS_GPU) for kp, r in ((32, 4), (64, 64), (128, 128))],
    ("als_gram_reduce_kernel", {"rank": 4, "implicit": True}, ALS_GPU),
]


def _als_kernels():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    return {name: v for name, v in k.items() if name.startswith("als_")}


def test_als_kernels_do_not_spill():
    k = _als_kernels()
    assert len(k) == 7, sorted(k)
    for name, v in k.items():
        assert v["spill"] == 0, (name, v)


def test_als_dispatch_table_names_every_instantiation():
    built = set(_als_kernels())
    rows = [r[0] for r in ALS_DISPATCH]
    assert len(rows) == len(set(rows))
    assert set(rows) == built, (sorted(built - set(rows)), sorted(set(rows) - built))


def test_als_dispatch_shapes_are_cases_of_their_tests():
    import importlib

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    for kernel, shape, test in ALS_DISPATCH:
        mod, fn = test.split("::")
        sets = _param_sets(getattr(importlib.import_module(mod[:-3]), fn))
        assert any(all(s.get(a) == b for a, b in shape.items()) for s in sets), (kernel, shape, test)
        if "<" in kernel:
            kp = int(kernel.split("<")[1].rstrip(">"))
            assert kp == (32 if shape["rank"] <= 32 else 64 if shape["rank"] <= 64 else 128), (kernel, shape)
