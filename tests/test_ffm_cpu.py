"""Field-aware factorisation machines without a GPU: the float64 rule (``ops.ffm_reference_step``) against a
hand-written loop over pairs and against autograd, argument checks, held-out logloss and AUC against brute force, the
app end to end, quality on planted data, and the build facts of the FFM kernels (no spills, a dispatch table that
covers every instantiation)."""
import itertools
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


def _store(row_len, num_keys, dtype="float64"):
    import adapm_b200 as ad

    s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                  job=f"ffm_cpu_{np.random.randint(1 << 30)}", dtype=dtype)
    return s, ad.Worker(0, s)


def _table(n, F, k, g):
    """rows [w, 0, 0, 0 | V | AdaGrad]: w and V random, positive accumulators"""
    E = 4 + F * k
    t = torch.zeros(n, 2 * E, dtype=torch.float64)
    t[:, 0] = torch.randn(n, generator=g, dtype=torch.float64) * 0.1
    t[:, 4:E] = torch.randn(n, F * k, generator=g, dtype=torch.float64) * 0.5
    t[:, E:] = torch.rand(n, E, generator=g, dtype=torch.float64) + 0.5
    return t


def _step(table, ids, labels, k, eta, lam, r):
    from adapm_b200.ops import ffm_reference_step

    n, L = table.shape
    s, kv = _store(L, n)
    try:
        kv.wait(kv.set(torch.arange(n), table.contiguous().view(-1)))
        loss = ffm_reference_step(kv, ids, labels, k, eta, lam, r)
        rows = torch.empty(n * L, dtype=torch.float64)
        kv.wait(kv.pull(torch.arange(n), rows))
        return rows.view(n, L), loss
    finally:
        kv.finalize()
        s.shutdown()


# keys 0..9; key 3 is in examples 0, 1 and 2 (fields 0 and 2), key 7 in fields 1 and 3 of example 1
IDS = torch.tensor([[3, 5, 1, 8], [3, 7, 2, 7], [0, 9, 3, 6]])
LABELS = torch.tensor([1.0, 0.0, 1.0])


def _loop_rule(t, ids, y, k, eta, lam, r):
    """the rule, written out with Python loops over examples, pairs and occurrences (float64)"""
    B, F = ids.shape
    E = 4 + F * k
    V = lambda key, f: t[key, 4 + f * k:4 + (f + 1) * k]
    G, loss = {}, 0.0
    kap = []
    for b in range(B):
        x = ids[b].tolist()
        phi = sum(float(t[x[f], 0]) for f in range(F))
        for f1 in range(F):
            for f2 in range(f1 + 1, F):
                phi += r * float(V(x[f1], f2) @ V(x[f2], f1))
        loss += float(np.logaddexp(0.0, phi)) - float(y[b]) * phi
        kap.append(1.0 / (1.0 + np.exp(-phi)) - float(y[b]))
    for b in range(B):                           # occurrences in position order b * F + f
        x = ids[b].tolist()
        for f in range(F):
            g = G.setdefault(x[f], torch.zeros(E, dtype=torch.float64))
            g[0] += kap[b] + lam * t[x[f], 0]
            for f2 in range(F):
                if f2 != f:
                    g[4 + f2 * k:4 + (f2 + 1) * k] += kap[b] * r * V(x[f2], f) + lam * V(x[f], f2)
    new = t.clone()
    for key, g in G.items():
        acc = t[key, E:]
        new[key, :E] += torch.where(g != 0, -eta * g / torch.sqrt(acc + g * g), torch.zeros_like(g))
        new[key, E:] += g * g
    return new, loss


@pytest.mark.parametrize("r", [1.0, 0.25])
def test_reference_step_matches_a_loop_over_pairs(r):
    k, eta, lam = 4, 0.2, 0.01
    table = _table(10, 4, k, torch.Generator().manual_seed(3))
    rows, loss = _step(table, IDS, LABELS, k, eta, lam, r)
    want, want_loss = _loop_rule(table, IDS, LABELS, k, eta, lam, r)
    np.testing.assert_allclose(rows.numpy(), want.numpy(), rtol=1e-12, atol=1e-14)
    assert loss == pytest.approx(want_loss, rel=1e-12)
    np.testing.assert_array_equal(rows[4].numpy(), table[4].numpy())          # keys not in the batch: untouched


def test_reference_gradient_is_autograd_of_the_batch_loss():
    """the pushed G of every key is d/d(row) of sum_b loss_b + lam/2 |row|^2 per occurrence's terms: recovered from
    the push (G^2 in the accumulator, the sign from the value update) and compared with autograd on phi"""
    F, k, eta, lam, r = 4, 4, 0.2, 0.01, 0.5
    E = 4 + F * k
    table = _table(10, F, k, torch.Generator().manual_seed(4))
    rows, _ = _step(table, IDS, LABELS, k, eta, lam, r)
    G = torch.sqrt(rows[:, E:] - table[:, E:]) * -torch.sign(rows[:, :E] - table[:, :E])
    T = table[:, :E].clone().requires_grad_(True)
    x = T[IDS]                                                            # [B, F, E]
    Vb = x[:, :, 4:].reshape(3, F, F, k)
    phi = x[:, :, 0].sum(1) + r * torch.triu(torch.einsum("bijd,bjid->bij", Vb, Vb), 1).sum((1, 2))
    loss = (torch.nn.functional.softplus(phi) - LABELS.double() * phi).sum()
    # lam term per occurrence (b, f): lam/2 |w|^2 + lam/2 sum_{f2 != f} |V_f2|^2
    own = torch.ones(F, F, dtype=torch.float64) - torch.eye(F, dtype=torch.float64)
    reg = 0.5 * lam * ((x[:, :, 0] ** 2).sum() + ((Vb ** 2).sum(-1) * own).sum())
    (grad,) = torch.autograd.grad(loss + reg, T)
    np.testing.assert_allclose(G.numpy(), grad.numpy(), rtol=1e-7, atol=1e-7)


def test_own_field_block_and_padding_receive_exactly_zero():
    F, k = 3, 4
    E = 4 + F * k
    ids = torch.tensor([[0, 3, 6], [1, 4, 7], [0, 5, 6]])                  # field f holds keys 3f .. 3f + 2 only
    table = _table(9, F, k, torch.Generator().manual_seed(5))
    rows, _ = _step(table, ids, torch.tensor([1.0, 0.0, 0.0]), k, 0.2, 0.01, 1.0)
    for key in range(9):
        f = key // 3
        own = slice(4 + f * k, 4 + (f + 1) * k)
        for sl in (slice(1, 4), own, slice(E + 1, E + 4), slice(E + own.start, E + own.stop)):
            np.testing.assert_array_equal(rows[key, sl].numpy(), table[key, sl].numpy())
        if key in ids:
            assert not torch.equal(rows[key, 4:E], table[key, 4:E])


def test_arguments_are_checked():
    from adapm_b200.ops import StoreFFM, ffm_reference_forward, ffm_reference_step

    F, k = 4, 4
    s, kv = _store(2 * (4 + F * k), 16)
    try:
        ids, y = torch.zeros(2, F, dtype=torch.int64), torch.zeros(2)
        bad_type = [dict(ids=ids.int()), dict(ids=ids.view(-1)), dict(y=y.double())]
        bad_value = [dict(ids=torch.zeros(2, 3, dtype=torch.int64)), dict(k=8), dict(k=6), dict(eta=-0.1),
                     dict(lam=-1e-3), dict(y=torch.zeros(3))]
        for kw, err in [(b, TypeError) for b in bad_type] + [(b, ValueError) for b in bad_value]:
            a = dict(ids=ids, y=y, k=k, eta=0.2, lam=0.0) | kw
            with pytest.raises(err):
                ffm_reference_step(kv, a["ids"], a["y"], a["k"], a["eta"], a["lam"])
        with pytest.raises(TypeError):
            ffm_reference_forward(kv, ids.float(), k)
        with pytest.raises(ValueError):                      # the fused op runs on CUDA servers only
            StoreFFM(s, F, k)
    finally:
        kv.finalize()
        s.shutdown()
    for F, k in ((1, 4), (65, 4), (4, 0), (4, 36), (4, 2), (40, 16)):      # outside the envelope
        s, kv = _store(2 * (4 + F * k), 16)
        try:
            with pytest.raises(ValueError):
                ffm_reference_step(kv, torch.zeros(1, F, dtype=torch.int64), torch.zeros(1), k, 0.2, 0.0)
        finally:
            kv.finalize()
            s.shutdown()


def test_logloss_and_auc_match_brute_force():
    from adapm_b200.models.ffm import logloss_auc

    g = np.random.default_rng(7)
    p = np.round(g.random(300), 2)                       # many ties
    y = (g.random(300) < p).astype(np.float64)
    ll, auc = logloss_auc(p, y)
    assert ll == pytest.approx(-np.mean(y * np.log(p.clip(1e-15)) + (1 - y) * np.log((1 - p).clip(1e-15))), rel=1e-12)
    pos, neg = p[y == 1], p[y == 0]
    pairs = [(a > b) + 0.5 * (a == b) for a, b in itertools.product(pos, neg)]
    assert auc == pytest.approx(np.mean(pairs), rel=1e-12)


def test_evaluate_matches_brute_force_on_the_reference_forward():
    from adapm_b200.models.ffm import FFM, FFMConfig, logloss_auc, synthetic_ffm_batch
    from adapm_b200.ops import ffm_reference_forward

    cfg = FFMConfig(num_features=4 * 50, num_fields=4, k=4, batch_size=64)
    s, kv = _store(cfg.row_len, cfg.num_features)
    try:
        m = FFM(s, kv, cfg)
        m.init_model()
        batches = [synthetic_ffm_batch(cfg, b, held_out=True) for b in range(3)]
        ll, auc = m.evaluate(batches)
        phi = torch.cat([ffm_reference_forward(kv, i, cfg.k, 1 / cfg.num_fields) for i, _ in batches]).numpy()
    finally:
        kv.finalize()
        s.shutdown()
    p = 1 / (1 + np.exp(-phi))
    y = torch.cat([b[1] for b in batches]).numpy()
    assert (ll, auc) == pytest.approx(logloss_auc(p, y), rel=1e-12)
    pairs = [(a > b) + 0.5 * (a == b) for a, b in itertools.product(p[y == 1], p[y == 0])]
    assert auc == pytest.approx(np.mean(pairs), rel=1e-12)


# ---------------------------------------------------------------------------------------------- quality
# Planted data: 8 fields of 60 ids, k 4, 600 steps of 256 examples, 8 held-out batches. Measured on the CPU backend
# (float64): FFM logloss 0.594 AUC 0.753; the linear model (pair_scale 0) AUC 0.518; the base rate logloss 0.693.
QUALITY = dict(num_features=8 * 60, num_fields=8, k=4, batch_size=256, steps=600, test_batches=8)
QUALITY_MIN_AUC_GAIN = 0.15          # over the linear model
QUALITY_MIN_LOGLOSS_GAIN = 0.05      # under the base-rate logloss


def train_ffm_quality(backend, pair_scale=None, dtype="float32"):
    """(logloss, AUC) on QUALITY's held-out batches after training"""
    import adapm_b200 as ad
    from adapm_b200.models.ffm import FFM, FFMConfig, synthetic_ffm_batch

    q = QUALITY
    cfg = FFMConfig(num_features=q["num_features"], num_fields=q["num_fields"], k=q["k"], batch_size=q["batch_size"])
    s = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend=backend,
                  fabric="inproc", job=f"ffm_q_{np.random.randint(1 << 30)}", dtype=dtype,
                  **({"device": 0} if backend == "cuda" else {}))
    kv = ad.Worker(0, s)
    try:
        m = FFM(s, kv, cfg, pair_scale=pair_scale)
        m.init_model()
        for st in range(q["steps"]):
            m.step(*synthetic_ffm_batch(cfg, st))
        return m.evaluate(synthetic_ffm_batch(cfg, b, held_out=True) for b in range(q["test_batches"]))
    finally:
        kv.finalize()
        s.shutdown()


def base_rate_logloss():
    from adapm_b200.models.ffm import FFMConfig, logloss_auc, synthetic_ffm_batch

    q = QUALITY
    cfg = FFMConfig(num_features=q["num_features"], num_fields=q["num_fields"], k=q["k"], batch_size=q["batch_size"])
    y = np.concatenate([synthetic_ffm_batch(cfg, b, held_out=True)[1].numpy() for b in range(q["test_batches"])])
    return logloss_auc(np.full(y.size, y.mean()), y)[0]


def test_ffm_beats_the_linear_model_and_the_base_rate_on_planted_data():
    ll, auc = train_ffm_quality("cpu", dtype="float64")
    ll_lin, auc_lin = train_ffm_quality("cpu", pair_scale=0.0, dtype="float64")
    base = base_rate_logloss()
    print(f"FFM logloss {ll:.4f} auc {auc:.4f}; linear logloss {ll_lin:.4f} auc {auc_lin:.4f}; base rate {base:.4f}")
    assert auc >= auc_lin + QUALITY_MIN_AUC_GAIN, (auc, auc_lin)
    assert ll <= base - QUALITY_MIN_LOGLOSS_GAIN, (ll, base)


# ---------------------------------------------------------------------------------------------- the app
def _launch(args, world):
    if world == 1:
        cmd = [sys.executable, "-m", "adapm_b200.apps.ctr", "--backend", "cpu"] + args
    else:
        cmd = [sys.executable, "-m", "adapm_b200.launch", "-s", str(world), "--backend", "cpu", "-m",
               "adapm_b200.apps.ctr", "--"] + args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


SMALL = ["--num_features", "2000", "--num_fields", "8", "--embed_dim", "4", "--batch_size", "128", "--steps", "10"]


@pytest.mark.parametrize("world", [1, 2])
def test_app_trains_ffm_and_prints_the_held_out_line(world):
    rc, out = _launch(["--model", "ffm", "--eta", "0.1", "--lam", "1e-4"] + SMALL, world)
    assert rc == 0, out[-3000:]
    assert len(re.findall(r"\[ctr\] step \d+: loss [\d.]+ \(\d+ examples/s/rank\)", out)) == 5, out[-3000:]
    m = re.search(r"\[ctr\] test logloss ([\d.]+) auc ([\d.]+)", out)
    assert m and 0 < float(m.group(1)) < 1 and 0 <= float(m.group(2)) <= 1, out[-3000:]
    assert "protocol errors 0" in out, out[-1500:]


def test_app_deepfm_output_has_no_ffm_line_and_ffm_refuses_multi_hot():
    rc, out = _launch(SMALL, 1)
    assert rc == 0, out[-3000:]
    assert len(re.findall(r"\[ctr\] step \d+: loss [\d.]+ \(\d+ examples/s/rank\)", out)) == 5, out[-3000:]
    assert "test logloss" not in out
    rc, out = _launch(["--model", "ffm", "--multi_hot", "2"] + SMALL, 1)
    assert rc != 0 and "--multi_hot is not supported with --model ffm" in out, out[-2000:]


# ---------------------------------------------------------------------------------------------- build
# One row per instantiation of the FFM kernels: (kernel, shape that selects it, the numeric GPU test that runs it). The
# backward's float4 per lane is VPL = ceil((1 + F k / 4) / 32).
FFM_GPU = "test_gpu_ffm.py::test_step_and_forward_match_float64_rule"
FFM_VPL_SHAPE = {1: (24, 4), 2: (39, 4), 3: (39, 8), 4: (32, 12), 5: (64, 8)}
FFM_DISPATCH = [
    ("ffm_fwd_kernel", {"F": 2, "k": 4}, FFM_GPU),
    ("ffm_loss_sum_kernel", {"F": 2, "k": 4}, FFM_GPU),
    *[(f"{name}<{v}>", {"F": F, "k": k}, FFM_GPU)
      for name in ("ffm_grad_tile_kernel", "ffm_grad_finish_kernel") for v, (F, k) in FFM_VPL_SHAPE.items()],
]


def _ffm_kernels():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    return {name: v for name, v in k.items() if name.startswith("ffm_")}


def test_ffm_kernels_do_not_spill():
    k = _ffm_kernels()
    assert len(k) == 12, sorted(k)
    for name, v in k.items():
        assert v["spill"] == 0, (name, v)


def test_ffm_dispatch_table_names_every_instantiation():
    built = set(_ffm_kernels())
    rows = [r[0] for r in FFM_DISPATCH]
    assert len(rows) == len(set(rows))
    assert set(rows) == built, (sorted(built - set(rows)), sorted(set(rows) - built))


def test_ffm_dispatch_shapes_are_cases_of_their_tests():
    import importlib

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    for kernel, shape, test in FFM_DISPATCH:
        mod, fn = test.split("::")
        sets = _param_sets(getattr(importlib.import_module(mod[:-3]), fn))
        assert any(all(s.get(a) == b for a, b in shape.items()) for s in sets), (kernel, shape, test)
        if "<" in kernel:
            vpl = int(kernel.split("<")[1].rstrip(">"))
            assert vpl == (1 + shape["F"] * shape["k"] // 4 + 31) // 32, (kernel, shape)
