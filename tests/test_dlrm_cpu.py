"""DLRM without a GPU: the torch route of ``ops.dlrm_interaction`` against the float64 rule, its limits, DLRM on CPU
servers with 1 and 2 ranks (single- and multi-hot) and on planted data, the Criteo reader, the app, and the register
budget of the interaction kernels."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from harness import run_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(B, F, E, seed=0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, E, generator=g, dtype=dtype), torch.randn(B, F, E, generator=g, dtype=dtype),
            torch.randn(B, (E + F * (F + 1) // 2 + 7) // 8 * 8, generator=g, dtype=dtype))


# (B, F, E): F 1 / 26 / 63, E 4 / 128 / 512, B 1; E + F (F + 1) / 2 is a multiple of 8 (no pad) at (F 7, E 4) and
# (F 15, E 16), and needs padding elsewhere
TORCH_SHAPES = [(5, 1, 4), (7, 26, 128), (3, 63, 512), (1, 26, 128), (4, 3, 8), (2, 63, 4), (6, 7, 4), (3, 15, 16),
                (1, 1, 512)]


@pytest.mark.parametrize("B,F,E", TORCH_SHAPES)
def test_torch_route_matches_float64_rule(B, F, E):
    from adapm_b200.ops import dlrm_interaction, dlrm_interaction_reference, dlrm_interaction_width

    z, e, g = _inputs(B, F, E, seed=B * 1000 + F * 10 + E)
    W = dlrm_interaction_width(F, E)
    R_ref, dz_ref, de_ref = dlrm_interaction_reference(z, e, g)
    z.requires_grad_(True)
    e.requires_grad_(True)
    R = dlrm_interaction(z, e)
    assert R.shape == (B, W) and R.dtype == torch.float32
    R.backward(g)
    tol = dict(rtol=1e-4, atol=1e-4 * E ** 0.5)
    torch.testing.assert_close(R.double(), R_ref, **tol)
    assert torch.all(R[:, E + F * (F + 1) // 2:] == 0)
    torch.testing.assert_close(z.grad.double(), dz_ref, **tol)
    torch.testing.assert_close(e.grad.double(), de_ref, **tol)


def test_width_padding():
    from adapm_b200.ops import dlrm_interaction_width

    assert dlrm_interaction_width(26, 128) == 480          # 128 + 351 = 479, padded
    assert dlrm_interaction_width(3, 8) == 16              # 8 + 6 = 14, padded
    assert dlrm_interaction_width(1, 4) == 8
    assert dlrm_interaction_width(7, 4) == 32              # 4 + 28, no padding


def test_pair_order_by_hand():
    """F 2: T = [z; e0; e1], pairs (1, 0), (2, 0), (2, 1) as in torch.tril_indices(3, 3, -1)."""
    from adapm_b200.ops import dlrm_interaction, dlrm_interaction_reference

    z = torch.tensor([[1.0, 0, 0, 0]])
    e = torch.tensor([[[2.0, 1, 0, 0], [3.0, 0, 5, 0]]])
    expect = [1, 0, 0, 0, 2, 3, 6, 0]                      # <e0, z> = 2, <e1, z> = 3, <e1, e0> = 6, one pad column
    assert dlrm_interaction(z, e).tolist() == [expect]
    assert dlrm_interaction_reference(z, e)[0].tolist() == [expect]
    i, j = torch.tril_indices(3, 3, offset=-1)
    assert list(zip(i.tolist(), j.tolist())) == [(1, 0), (2, 0), (2, 1)]
    # backward by hand: dR = one-hot on pair (2, 1) -> de1 += e0, de0 += e1, dz = dR[:, :E]
    dR = torch.tensor([[0.5, 0, 0, 0, 0, 0, 1, 7]])
    _, dz, de = dlrm_interaction_reference(z, e, dR)
    assert dz.tolist() == [[0.5, 0, 0, 0]]
    assert de.tolist() == [[[3.0, 0, 5, 0], [2.0, 1, 0, 0]]]


@pytest.mark.parametrize("B,F,E,msg", [
    (2, 0, 8, "1 <= F and F + 1 <= 64"),
    (2, 64, 8, "1 <= F and F + 1 <= 64"),
    (2, 4, 6, "E a multiple of 4 in [4, 512]"),
    (2, 4, 0, "E a multiple of 4 in [4, 512]"),
    (2, 4, 516, "E a multiple of 4 in [4, 512]"),
])
def test_limits_are_refused(B, F, E, msg):
    from adapm_b200.ops import dlrm_interaction

    for impl in ("auto", "torch", "fused"):
        with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace("[", r"\[").replace("+", r"\+")):
            dlrm_interaction(torch.zeros(B, E), torch.zeros(B, F, E), impl=impl)


def test_size_limit_and_argument_checks():
    from adapm_b200.ops import dlrm_interaction

    W = 480                                                # F 26, E 128
    B = (1 << 31) // W + 1
    z = torch.zeros(B, 128).expand(B, 128)                 # no memory: the check runs before anything is read
    e = torch.zeros(1, 26, 128).expand(B, 26, 128)
    with pytest.raises(ValueError, match=r"B \* W < 2\^31"):
        dlrm_interaction(z, e)
    with pytest.raises(TypeError, match="float32"):
        dlrm_interaction(torch.zeros(2, 8, dtype=torch.float64), torch.zeros(2, 3, 8))
    with pytest.raises(ValueError, match=r"e must be \[B, F, E\]"):
        dlrm_interaction(torch.zeros(2, 8), torch.zeros(3, 3, 8))
    with pytest.raises(ValueError, match="z must be"):
        dlrm_interaction(torch.zeros(2, 3, 8), torch.zeros(2, 3, 8))
    with pytest.raises(ValueError, match="impl"):
        dlrm_interaction(torch.zeros(2, 8), torch.zeros(2, 3, 8), impl="bmm")
    with pytest.raises(ValueError, match="CUDA"):
        dlrm_interaction(torch.zeros(2, 8), torch.zeros(2, 3, 8), impl="fused")


# ------------------------------------------------------------------------------------------------ the model
def _small_cfg(**kw):
    from adapm_b200.models.dlrm import DLRMConfig

    base = dict(num_features=8 * 250, num_fields=8, num_dense=13, embed_dim=16, bottom=(32,), top=(64, 32),
                lr_sparse=0.1, lr_dense=3e-3, batch_size=256, precision="fp32")
    base.update(kw)
    return DLRMConfig(**base)


def _train_worker(kv, server, wid, cfg, steps, cycle):
    from adapm_b200.models.dlrm import DLRM, synthetic_dlrm_batch

    model = DLRM(server, kv, cfg)
    model.init_model()
    losses = []
    for s in range(steps):
        dense, ids, *off, y = synthetic_dlrm_batch(cfg, s % cycle, server.my_rank())
        model.signal_intent(ids, kv.current_clock() + 1)
        losses.append(model.step(dense, ids, y, offsets=off[0] if off else None))
        kv.advance_clock()
    kv.barrier()
    kv.finalize()
    return {"losses": losses, "rows_pushed": model.rows_pushed}


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("multi_hot", [0, 4])
def test_dlrm_lowers_the_loss(world, multi_hot):
    cfg = _small_cfg(multi_hot=multi_hot, pooling="mean" if world == 2 else "sum")
    res = run_cluster(lambda kv, server, wid: _train_worker(kv, server, wid, cfg, 24, 4), world=world, workers=1,
                      mode="threads", value_lengths=cfg.row_len, num_keys=cfg.num_features)
    for r in range(world):
        l = res[r][0]["losses"]
        assert all(np.isfinite(l)), l
        assert np.mean(l[-4:]) < np.mean(l[:4]) - 0.01, l
        assert res[r][0]["rows_pushed"] > 0


# held-out AUC after 600 steps of the planted-data config below on a CPU server: 0.7952 (the planted dense term
# alone: 0.6575 on the same batches)
PLANTED_AUC_MIN = 0.75
PLANTED_TEST_BATCHES = 8


def planted_run(server, kv, steps=600):
    """Trains DLRM on planted data; returns (held-out AUC of the model, AUC of the planted dense term alone)."""
    from adapm_b200.models.dlrm import DLRM, planted_dense_term, synthetic_dlrm_batch
    from adapm_b200.models.ffm import logloss_auc

    cfg = planted_cfg()
    model = DLRM(server, kv, cfg)
    model.init_model()
    for s in range(steps):
        dense, ids, y = synthetic_dlrm_batch(cfg, s, 0)
        model.step(dense, ids, y)
        kv.advance_clock()
    test = [synthetic_dlrm_batch(cfg, b, 0, held_out=True) for b in range(PLANTED_TEST_BATCHES)]
    _, auc = model.evaluate(test)
    dense_only = np.concatenate([planted_dense_term(cfg, d) for d, _, _ in test])
    _, auc_dense = logloss_auc(1 / (1 + np.exp(-dense_only)), torch.cat([y for _, _, y in test]).numpy())
    return auc, auc_dense


def planted_cfg():
    return _small_cfg(num_features=8 * 100, batch_size=512, lr_sparse=0.05)


def test_planted_data_auc_beats_the_dense_term():
    import adapm_b200 as ad

    cfg = planted_cfg()
    server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend="cpu",
                       fabric="inproc", job=f"dlrm_planted_{np.random.randint(1 << 30)}")
    kv = ad.Worker(0, server)
    try:
        auc, auc_dense = planted_run(server, kv)
    finally:
        kv.finalize()
        server.shutdown()
    assert auc > PLANTED_AUC_MIN, (auc, auc_dense)
    assert auc > auc_dense + 0.05, (auc, auc_dense)


def test_synthetic_batches():
    from adapm_b200.models.dlrm import planted_dense_term, synthetic_dlrm_batch

    cfg = _small_cfg(batch_size=64)
    dense, ids, y = synthetic_dlrm_batch(cfg, 3)
    assert dense.shape == (64, 13) and dense.dtype == torch.float32 and bool((dense >= 0).all())
    assert ids.shape == (64, 8) and ids.dtype == torch.int64 and y.shape == (64,)
    assert torch.all(ids // 250 == torch.arange(8))
    d2, i2, y2 = synthetic_dlrm_batch(cfg, 3)
    assert torch.equal(dense, d2) and torch.equal(ids, i2) and torch.equal(y, y2)
    dh, ih, _ = synthetic_dlrm_batch(cfg, 3, held_out=True)
    assert not torch.equal(ih, ids) and not torch.equal(dh, dense)
    assert planted_dense_term(cfg, dense).shape == (64,)
    cfg = _small_cfg(batch_size=64, multi_hot=5)
    dense, ids, off, y = synthetic_dlrm_batch(cfg, 3)
    lens = off[1:] - off[:-1]
    assert off.numel() == 64 * 8 + 1 and int(off[-1]) == ids.numel()
    assert int(lens.min()) >= 1 and int(lens.max()) <= 5
    assert torch.all(ids // 250 == torch.repeat_interleave(torch.arange(64 * 8) % 8, lens))


def test_deepfm_dense_net_is_unchanged():
    """DenseNet takes its widths for DLRM; DeepFM's default still builds F * k -> hidden -> 1 from model_seed."""
    from adapm_b200.models.deepfm import DeepFMConfig, DenseNet

    cfg = DeepFMConfig(num_fields=4, embed_dim=8, hidden=(16, 16), model_seed=7)
    net = DenseNet(cfg, use_tensor_cores=False)
    g = torch.Generator().manual_seed(7)
    dims = [32, 16, 16, 1]
    for i, w in enumerate(net.w):
        assert torch.equal(w.data, torch.randn(dims[i + 1], dims[i], generator=g) * (2.0 / dims[i]) ** 0.5)
    assert net(torch.randn(5, 32)).shape == (5,)


# ------------------------------------------------------------------------------------------------ Criteo reader
def _line(label, dense, cats):
    return "\t".join([str(label)] + [str(v) for v in dense] + list(cats)) + "\n"


def test_criteo_reader(tmp_path):
    from adapm_b200.utils.criteo import criteo_batches

    per_field = 100
    rows = []
    for n in range(5):
        dense = [n, "", -3, 7] + [1] * 9
        cats = [f"{(n * 977 + f * 13) & 0xffffffff:08x}" for f in range(26)]
        cats[2] = ""                                       # missing categorical value
        rows.append(_line(n % 2, dense, cats))
    p = tmp_path / "day.tsv"
    p.write_text("".join(rows))
    batches = list(criteo_batches(str(p), 2, 26 * per_field))
    assert [b[0].shape[0] for b in batches] == [2, 2, 1]   # short last batch
    dense = torch.cat([b[0] for b in batches])
    ids = torch.cat([b[1] for b in batches])
    y = torch.cat([b[2] for b in batches])
    assert y.tolist() == [0, 1, 0, 1, 0]
    assert torch.allclose(dense[:, 0], torch.log1p(torch.arange(5.0)))
    assert torch.all(dense[:, 1] == 0) and torch.all(dense[:, 2] == 0)      # empty and negative
    assert torch.allclose(dense[:, 3], torch.full((5,), float(np.log1p(7))))
    lo = torch.arange(26) * per_field
    assert torch.all((ids >= lo) & (ids < lo + per_field))
    assert torch.all(ids[:, 2] == 2 * per_field)                            # the reserved key of a missing value
    for n in range(5):
        for f in (0, 5, 25):
            assert int(ids[n, f]) == f * per_field + 1 + ((n * 977 + f * 13) % (per_field - 1))


@pytest.mark.parametrize("bad,msg", [
    ("1\t2\t3\n", "expected 40"),
    (_line(2, [1] * 13, ["0"] * 26), "label must be 0 or 1"),
    (_line(1, ["x"] + [1] * 12, ["0"] * 26), "integer feature"),
    (_line(1, [1] * 13, ["zz"] + ["0"] * 25), "not hexadecimal"),
])
def test_criteo_reader_rejects_malformed_lines(tmp_path, bad, msg):
    from adapm_b200.utils.criteo import criteo_batches

    good = _line(0, [1] * 13, ["0a"] * 26)
    p = tmp_path / "bad.tsv"
    p.write_text(good + good + bad + good)
    with pytest.raises(ValueError, match=f":3: .*{msg}"):
        list(criteo_batches(str(p), 8, 26 * 10))


# ------------------------------------------------------------------------------------------------ the app
def _app(*args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "adapm_b200.apps.ctr", "--backend", "cpu", "--model", "dlrm", *args],
                          cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)


def test_ctr_app_dlrm_synthetic():
    r = _app("--num_features", "5000", "--num_fields", "6", "--embed_dim", "8", "--steps", "5", "--batch_size", "128",
             "--bottom", "16", "--top", "32,16", "--precision", "fp32", "--multi_hot", "3", "--test_batches", "2")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[ctr] step 5: loss" in r.stdout and "examples/s/rank" in r.stdout, r.stdout[-2000:]
    assert "[ctr] test logloss" in r.stdout and " auc " in r.stdout, r.stdout[-2000:]


def test_ctr_app_dlrm_criteo_files(tmp_path):
    rng = np.random.default_rng(0)
    rows = [_line(int(rng.integers(2)), [int(v) if v >= 0 else "" for v in rng.integers(-2, 50, 13)],
                  [f"{int(v):08x}" if v % 5 else "" for v in rng.integers(0, 1 << 32, 26)]) for _ in range(300)]
    (tmp_path / "train.tsv").write_text("".join(rows[:200]))
    (tmp_path / "test.tsv").write_text("".join(rows[200:]))
    r = _app("--num_features", "2600", "--embed_dim", "8", "--steps", "4", "--batch_size", "50", "--bottom", "16",
             "--top", "16", "--data", str(tmp_path / "train.tsv"), "--test_data", str(tmp_path / "test.tsv"))
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[ctr] step 4: loss" in r.stdout, r.stdout[-2000:]
    assert "[ctr] test logloss" in r.stdout, r.stdout[-2000:]


def test_ctr_app_dlrm_refuses_fp8_block_tables():
    r = _app("--table_precision", "fp8_block", "--steps", "1")
    assert r.returncode != 0 and "fp8_block is not supported with --model dlrm" in r.stderr, r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ register budget
def test_interaction_kernels_do_not_spill():
    """`-Xptxas -v` of the in-tree build: both kernels of ops_dlrm.cu (one instantiation each) keep their state in
    registers."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    mine = {n: v for n, v in k.items() if n.startswith("dlrm_")}
    assert set(mine) == {"dlrm_interaction_fwd_kernel", "dlrm_interaction_bwd_kernel"}, sorted(mine)
    for n, v in mine.items():
        assert v["spill"] == 0, (n, v)
