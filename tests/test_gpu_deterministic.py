"""Deterministic one-GPU KGE (ComplEx, RESCAL) and MF steps (``deterministic=True``): every call of a step reads the
state at the start of the step, the updates are summed in fixed point and applied once per row, so that repeated keys
follow the documented start-of-step rule and two runs from the same inputs agree bit for bit."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


@pytest.fixture()
def cluster1():
    import adapm_b200 as ad

    made = []

    def make(row_len, num_keys, **kw):
        s = ad.Server(row_len, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                      job=f"det{len(made)}_{np.random.randint(1 << 30)}", device=0, **kw)
        w = ad.Worker(0, s)
        made.append((s, w))
        return s, w

    yield make
    for s, w in made:
        w.finalize()
        s.shutdown()


def _cpu_f64(value_lengths, num_keys, job):
    import adapm_b200 as ad

    s = ad.Server(value_lengths, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                  job=f"{job}_{np.random.randint(1 << 30)}", dtype="float64")
    return s, ad.Worker(0, s)


def _pull(kv, keys, n_vals, dtype=torch.float32):
    out = torch.empty(n_vals, dtype=dtype)
    kv.wait(kv.pull(keys, out))
    return out


# ---------------------------------------------------------------------------------------------- start-of-step numerics
@gpu
@pytest.mark.parametrize("algo,d,p_e,p_r", [("ComplEx", 512, 0.0, 0.0), ("ComplEx", 128, 0.25, 0.4),
                                            ("ComplEx", 20, 0.0, 0.0), ("RESCAL", 32, 0.0, 0.0),
                                            ("RESCAL", 12, 0.0, 0.0), ("RESCAL", 32, 0.3, 0.2),
                                            ("RESCAL", 12, 0.2, 0.3)])
def test_kge_steps_with_repeated_keys_match_start_of_step_reference(cluster1, algo, d, p_e, p_r):
    """12 entities and 3 relations over 256 calls: every row is updated by many calls of each step. Over 3 steps the
    deterministic kernels equal the reference rule (all calls read the start-of-step state) evaluated on a float64 CPU
    store loaded with the GPU's state (an accumulator that is not cleared, or a row applied twice, shows in step 2)."""
    from adapm_b200.models.kge import KGEConfig, kge_reference_step
    from adapm_b200.ops import kge_complex_step, kge_dropout_mask, kge_rescal_step

    n = 256
    cfg = KGEConfig(num_entities=12, num_relations=3, embed_dim=d, neg_ratio=1, algorithm=algo, eta=0.05,
                    dropout_entity=p_e, dropout_relation=p_r)
    server, kv = cluster1(cfg.value_lengths(), cfg.num_keys)
    dev = server.device
    g = torch.Generator().manual_seed(d + int(100 * p_e) + (1000 if algo == "RESCAL" else 0))
    el, rl = cfg.entity_len // 2, cfg.relation_len // 2
    ek = torch.arange(cfg.num_entities)
    rk = torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations)
    erows = torch.cat([torch.randn(cfg.num_entities, el, generator=g) * 0.3, torch.rand(cfg.num_entities, el, generator=g) + 1e-3], 1)
    rrows = torch.cat([torch.randn(cfg.num_relations, rl, generator=g) * 0.3, torch.rand(cfg.num_relations, rl, generator=g) + 1e-3], 1)
    kv.set(ek, erows.clone().view(-1)); kv.set(rk, rrows.clone().view(-1))
    ref_server, ref_kv = _cpu_f64(cfg.value_lengths(), cfg.num_keys, f"detkge{algo}{d}")
    fused = kge_complex_step if algo == "ComplEx" else kge_rescal_step
    try:
        for step in range(3):
            torch.cuda.synchronize()
            e0 = _pull(kv, ek, cfg.num_entities * 2 * el)
            r0 = _pull(kv, rk, cfg.num_relations * 2 * rl)
            ref_kv.wait(ref_kv.set(ek, e0.double())); ref_kv.wait(ref_kv.set(rk, r0.double()))
            S = torch.randint(0, cfg.num_entities, (n,), generator=g)
            O = torch.randint(0, cfg.num_entities, (n,), generator=g)
            R = torch.randint(0, cfg.num_relations, (n,), generator=g) + cfg.num_entities
            L = (torch.rand(n, generator=g) < 0.3).float()
            seed = 0x5EED_0000 + 17 * step
            loss = torch.zeros(1, device=dev)
            stats = torch.zeros(4, dtype=torch.int64, device=dev)
            fused(server, S.to(dev), R.to(dev), O.to(dev), L.to(dev), d, cfg.eta, cfg.gamma_entity, cfg.gamma_relation,
                  loss, stats, p_e, p_r, seed, deterministic=True)
            torch.cuda.synchronize()
            masks = None
            if p_e > 0 or p_r > 0:
                masks = (kge_dropout_mask(seed, n, 0, el, p_e), kge_dropout_mask(seed, n, 1, rl, p_r, relation=True),
                         kge_dropout_mask(seed, n, 2, el, p_e))
            ref_loss = kge_reference_step(ref_kv, S, R, O, L, cfg, masks=masks)
            got_e = _pull(kv, ek, cfg.num_entities * 2 * el).double()
            got_r = _pull(kv, rk, cfg.num_relations * 2 * rl).double()
            ref_e = _pull(ref_kv, ek, cfg.num_entities * 2 * el, torch.float64)
            ref_r = _pull(ref_kv, rk, cfg.num_relations * 2 * rl, torch.float64)
            torch.testing.assert_close(got_e, ref_e, rtol=2e-4, atol=2e-5)
            torch.testing.assert_close(got_r, ref_r, rtol=2e-4, atol=2e-5)
            torch.testing.assert_close(loss.cpu()[0].double(), torch.tensor(ref_loss, dtype=torch.float64), rtol=1e-4, atol=0)
            s = stats.tolist()
            assert s[1] == 0 and s[2] == (n if algo == "ComplEx" and d % 8 else 0) and s[3] == 3 * n, s
    finally:
        ref_kv.finalize(); ref_server.shutdown()


@gpu
@pytest.mark.parametrize("rank", [128, 64, 10])
def test_mf_steps_with_repeated_keys_match_start_of_step_reference(cluster1, rank):
    """20 rows and 8 columns over 512 non-zeros, 3 steps, against mf_reference_step on a float64 CPU store loaded with
    the GPU's state at the start of every step (rank 10 runs the generic scalar path)."""
    from adapm_b200.models.mf import mf_reference_step
    from adapm_b200.ops import mf_step

    n, nr, nc = 512, 20, 8
    nk = nr + nc
    server, kv = cluster1(2 * rank, nk)
    dev = server.device
    g = torch.Generator().manual_seed(rank)
    keys = torch.arange(nk)
    rows = torch.cat([torch.randn(nk, rank, generator=g) * 0.3, torch.rand(nk, rank, generator=g)], 1)
    kv.set(keys, rows.clone().view(-1))
    ref_server, ref_kv = _cpu_f64(2 * rank, nk, f"detmf{rank}")
    try:
        for step in range(3):
            torch.cuda.synchronize()
            ref_kv.wait(ref_kv.set(keys, _pull(kv, keys, nk * 2 * rank).double()))
            rk = torch.randint(0, nr, (n,), generator=g)
            ck = torch.randint(0, nc, (n,), generator=g) + nr
            x = torch.randn(n, generator=g)
            rn = torch.bincount(rk, minlength=nr)[rk].to(torch.int32)
            cn = torch.bincount(ck - nr, minlength=nc)[ck - nr].to(torch.int32)
            loss = torch.zeros(1, device=dev)
            stats = torch.zeros(4, dtype=torch.int64, device=dev)
            mf_step(server, rk.to(dev), ck.to(dev), x.to(dev), rn.to(dev), cn.to(dev), rank, 0.05, 0.02, loss, stats,
                    deterministic=True)
            torch.cuda.synchronize()
            ref_loss = mf_reference_step(ref_kv, rk, ck, x, rn, cn, rank, 0.05, 0.02)
            got = _pull(kv, keys, nk * 2 * rank).double()
            ref = _pull(ref_kv, keys, nk * 2 * rank, torch.float64)
            torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-5)
            torch.testing.assert_close(loss.cpu()[0].double(), torch.tensor(ref_loss, dtype=torch.float64), rtol=1e-4, atol=0)
            s = stats.tolist()
            assert s[1] == 0 and s[2] == (n if rank % 4 else 0) and s[3] == 2 * n, s
    finally:
        ref_kv.finalize(); ref_server.shutdown()


# ---------------------------------------------------------------------------------------------- bit-identical runs
@gpu
@pytest.mark.parametrize("algo,d", [("ComplEx", 128), ("RESCAL", 32)])
def test_kge_training_is_bit_identical_across_runs(cluster1, algo, d):
    """Zipf triples put many calls of every step on the hot entities and relations; two runs of 10 steps from the same
    seeds give the same losses and rows, bit for bit."""
    from adapm_b200.models.kge import KGE, KGEConfig, synthetic_triples

    cfg = KGEConfig(num_entities=2000, num_relations=60, embed_dim=d, algorithm=algo, batch_triples=512,
                    deterministic=True)
    tr = synthetic_triples(cfg, 10 * cfg.batch_triples, seed=0)
    runs = []
    for _ in range(2):
        server, kv = cluster1(cfg.value_lengths(), cfg.num_keys)
        model = KGE(server, kv, cfg)
        model.init_model()
        losses = []
        for s in range(10):
            model.loss.zero_()
            model.step(tr[s * cfg.batch_triples:(s + 1) * cfg.batch_triples])
            losses.append(model.loss.item())
        torch.cuda.synchronize()
        ent = _pull(kv, torch.arange(cfg.num_entities), cfg.num_entities * cfg.entity_len)
        rel = _pull(kv, torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations),
                    cfg.num_relations * cfg.relation_len)
        runs.append((losses, ent, rel))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])


@gpu
def test_mf_epochs_are_bit_identical_across_runs(cluster1):
    from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix

    cfg = MFConfig(num_rows=400, num_cols=150, rank=32, algorithm="plain", batch_nnz=4096, deterministic=True)
    data = SparseMatrix.synthetic(cfg.num_rows, cfg.num_cols, 30000, 8, 1, 0, seed=0)
    runs = []
    for _ in range(2):
        server, kv = cluster1(cfg.row_len, cfg.num_keys(1))
        model = MatrixFactorization(server, kv, cfg, data)
        model.init_model()
        losses = [model.run_epoch(e) for e in range(2)]
        torch.cuda.synchronize()
        runs.append((losses, _pull(kv, torch.arange(cfg.num_keys(1)), cfg.num_keys(1) * cfg.row_len)))
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])


# ---------------------------------------------------------------------------------------------- default, multi-rank
@gpu
def test_default_steps_are_one_in_place_launch(cluster1):
    """Without ``deterministic`` every op is one kernel launch, as before; deterministic steps are three (index, step,
    apply)."""
    from adapm_b200 import _C
    from adapm_b200.models.kge import KGEConfig
    from adapm_b200.ops import kge_complex_step, kge_rescal_step, mf_step

    n = 64
    for algo, d in (("ComplEx", 64), ("RESCAL", 16)):
        cfg = KGEConfig(num_entities=50, num_relations=5, embed_dim=d, algorithm=algo)
        server, kv = cluster1(cfg.value_lengths(), cfg.num_keys)
        dev = server.device
        S = torch.randint(0, 50, (n,), device=dev)
        O = torch.randint(0, 50, (n,), device=dev)
        R = torch.randint(50, 55, (n,), device=dev)
        L = torch.zeros(n, device=dev)
        loss = torch.zeros(1, device=dev)
        fused = kge_complex_step if algo == "ComplEx" else kge_rescal_step
        for det, want in ((None, 1), (True, 3)):
            kw = {} if det is None else {"deterministic": det}
            l0 = _C.kernel_launches()
            fused(server, S, R, O, L, d, 0.1, 1e-3, 1e-3, loss, **kw)
            assert _C.kernel_launches() - l0 == want, (algo, det)
    server, kv = cluster1(2 * 16, 40)
    dev = server.device
    rk = torch.randint(0, 20, (n,), device=dev)
    ck = torch.randint(20, 40, (n,), device=dev)
    ones = torch.ones(n, dtype=torch.int32, device=dev)
    loss = torch.zeros(1, device=dev)
    for det, want in ((None, 1), (True, 3)):
        kw = {} if det is None else {"deterministic": det}
        l0 = _C.kernel_launches()
        mf_step(server, rk, ck, torch.randn(n, device=dev), ones, ones, 16, 0.05, 0.02, loss, **kw)
        assert _C.kernel_launches() - l0 == want, det
    torch.cuda.synchronize()


def _reject_on_two_ranks(kv, server, wid):
    from adapm_b200.ops import kge_complex_step, mf_step

    dev = server.device
    k = torch.zeros(4, dtype=torch.int64, device=dev)
    f = torch.zeros(4, device=dev)
    loss = torch.zeros(1, device=dev)
    out = []
    try:
        kge_complex_step(server, k, k, k, f, 4, 0.1, 0.0, 0.0, loss, deterministic=True)
    except ValueError as e:
        out.append(str(e))
    try:
        mf_step(server, k, k, f, k.int(), k.int(), 2, 0.1, 0.0, loss, deterministic=True)
    except ValueError as e:
        out.append(str(e))
    kv.barrier()
    return out


@gpu
def test_deterministic_steps_are_rejected_on_several_ranks():
    from harness import run_cluster

    res = run_cluster(_reject_on_two_ranks, world=2, workers=1, mode="threads", value_lengths=4, num_keys=16,
                      dtype="float32", backend="cuda")
    for rank in (0, 1):
        msgs = res[rank][0]
        assert len(msgs) == 2 and all("single-GPU" in m for m in msgs), msgs


# ---------------------------------------------------------------------------------------------- apps
def _app(args):
    r = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, capture_output=True, text=True, timeout=600)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    return out


def _losses(out, tag):
    return [re.sub(r"\s*\([\d.]+s\)\s*$", "", ln) for ln in out.splitlines() if ln.startswith(f"[{tag}] epoch")]


@gpu
def test_apps_with_deterministic_flag_repeat_bit_for_bit(tmp_path):
    kge_out, mf_out = [], []
    for i in range(2):
        emb = tmp_path / f"kge{i}"
        out = _app(["adapm_b200.apps.kge", "--dataset", os.path.join(ROOT, "data", "kge"), "--embed_dim", "16",
                    "--num_epochs", "2", "--deterministic", "1", "--backend", "cuda", "--write_embeddings", str(emb)])
        kge_out.append((_losses(out, "kge"), {f: (emb / f).read_bytes() for f in sorted(os.listdir(emb))}))
        fac = tmp_path / f"mf{i}"
        fac.mkdir()
        out = _app(["adapm_b200.apps.mf", "--dataset", os.path.join(ROOT, "data", "mf", "train.mmc"), "--epochs", "3",
                    "--deterministic", "1", "--backend", "cuda", "--export_prefix", str(fac) + "/"])
        mf_out.append((_losses(out, "mf"), {f: (fac / f).read_bytes() for f in sorted(os.listdir(fac))}))
    for a, b in (kge_out, mf_out):
        assert a[0] and a[0] == b[0], (a[0], b[0])
        assert a[1] and a[1] == b[1]
    assert len(kge_out[0][0]) == 2 and "export.epoch.2.entities.bin" in kge_out[0][1]
    assert len(mf_out[0][0]) == 3 and "W.mma" in mf_out[0][1]


def test_apps_reject_deterministic_on_several_ranks():
    env = dict(os.environ, WORLD_SIZE="2")
    for app in ("adapm_b200.apps.kge", "adapm_b200.apps.mf"):
        r = subprocess.run([sys.executable, "-m", app, "--deterministic", "1"], cwd=ROOT, env=env, capture_output=True,
                           text=True, timeout=120)
        assert r.returncode != 0 and "--deterministic 1 needs a single GPU" in r.stderr, r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- register budget
def test_deterministic_kernels_do_not_spill():
    """The vectorised deterministic kernels stay within their launch bounds without spilling (ptxas, no GPU)."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    for name, regs in (("kge_step_fx_kernel<1>", 128), ("kge_step_fx_kernel<2>", 128),
                       ("mf_step_fx_kernel<1>", 80), ("mf_step_fx_kernel<2>", 80)):
        assert name in k, sorted(k)
        assert k[name]["regs"] <= regs and k[name]["spill"] == 0, (name, k[name])
