"""StoreEmbeddingBag on CPU servers (pull + F.embedding_bag + push, the torch route) against the float64 rule
``embedding_bag_reference``, its argument checks, and multi-hot DeepFM on 1 and 2 ranks."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from harness import run_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _server(dim, num_keys, job):
    import adapm_b200 as ad

    s = ad.Server(2 * dim, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cpu", fabric="inproc",
                  job=f"{job}_{np.random.randint(1 << 30)}")
    return s, ad.Worker(0, s)


def _table(num_keys, dim, g):
    t = torch.randn(num_keys, 2 * dim, generator=g)
    t[:, dim:] = torch.rand(num_keys, dim, generator=g)        # AdaGrad accumulators >= 0
    t[: num_keys // 8, dim:] = 0.0                              # some at exactly 0 (G == 0 must give 0, not NaN)
    return t


def _bags(g, num_keys):
    """bags with an empty bag at the start, in the middle and at the end, a key repeated inside a bag and one repeated
    across bags"""
    lens = [0, 3, 1, 0, 5, 2, 7, 0, 4, 1, 0]
    keys = torch.randint(0, num_keys, (sum(lens),), generator=g)
    keys[1:3] = keys[0]            # repeated inside bag 1
    keys[10] = keys[0]             # and in bag 5 and 6
    keys[14] = keys[0]
    offsets = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int64)
    return keys, offsets


CASES = [(mode, weighted, dim) for dim in (4, 20, 64) for mode, weighted in (("sum", False), ("mean", False), ("sum", True))]


@pytest.mark.parametrize("mode,weighted,dim", CASES)
def test_cpu_route_matches_float64_rule(mode, weighted, dim):
    num_keys = 64
    g = torch.Generator().manual_seed(dim * 3 + weighted + (mode == "mean") * 7)
    table = _table(num_keys, dim, g)
    keys, offsets = _bags(g, num_keys)
    w = torch.rand(keys.numel(), generator=g) * 2 - 0.5 if weighted else None
    from adapm_b200.ops import StoreEmbeddingBag, embedding_bag_reference

    server, kv = _server(dim, num_keys, "bag")
    try:
        kv.wait(kv.set(torch.arange(num_keys), table.contiguous().view(-1)))
        bag = StoreEmbeddingBag(server, kv, dim, mode=mode, lr=0.1, grad_scale=3.0)
        assert bag.impl == "torch"
        out = bag(keys, offsets, w)
        grad = torch.randn(out.shape, generator=g)
        grad[2] = 0.0                                           # keys only in bag 2 get G == 0
        ref_out, ref_table = embedding_bag_reference(table, keys, offsets, w, mode, grad, lr=0.1, grad_scale=3.0)
        torch.testing.assert_close(out.double(), ref_out, rtol=1e-5, atol=1e-6)
        assert torch.all(out[offsets[1:] == offsets[:-1]] == 0)     # empty bags
        (out * grad).sum().backward()
        kv.waitall()
        rows = torch.empty(num_keys * 2 * dim)
        kv.wait(kv.pull(torch.arange(num_keys), rows))
        rows = rows.view(num_keys, 2 * dim)
        assert torch.isfinite(rows).all()
        torch.testing.assert_close(rows.double(), ref_table, rtol=1e-5, atol=1e-6)
        assert bag.take_rows_updated() == torch.unique(keys).numel()
    finally:
        kv.finalize()
        server.shutdown()


def test_reference_update_rule_by_hand():
    """G = scale * sum of c_i * grad_out[bag(i)]; row += [-lr G / sqrt(acc + G^2) | G^2]"""
    from adapm_b200.ops import embedding_bag_reference

    table = torch.tensor([[1.0, 2.0, 4.0, 0.0], [3.0, 5.0, 1.0, 1.0]])
    keys = torch.tensor([0, 1, 0])
    offsets = torch.tensor([0, 2, 3])
    out, new = embedding_bag_reference(table, keys, offsets, mode="mean", grad_out=torch.tensor([[2.0, 0.0], [1.0, 0.0]]),
                                       lr=0.5, grad_scale=2.0)
    torch.testing.assert_close(out, torch.tensor([[2.0, 3.5], [1.0, 2.0]], dtype=torch.float64))
    G0 = 2.0 * (2.0 / 2 + 1.0)         # key 0: bag 0 (mean over 2) and bag 1
    G1 = 2.0 * (2.0 / 2)
    exp = torch.tensor([[1.0 - 0.5 * G0 / (4.0 + G0 ** 2) ** 0.5, 2.0, 4.0 + G0 ** 2, 0.0],
                        [3.0 - 0.5 * G1 / (1.0 + G1 ** 2) ** 0.5, 5.0, 1.0 + G1 ** 2, 1.0]], dtype=torch.float64)
    torch.testing.assert_close(new, exp)


def test_argument_checks_raise():
    from adapm_b200.ops import StoreEmbeddingBag

    server, kv = _server(8, 32, "bagargs")
    try:
        for dim in (0, 2, 6, 516, 1024):
            with pytest.raises(ValueError):
                StoreEmbeddingBag(server, kv, dim)
        with pytest.raises(ValueError):                         # row_len != 2 * dim
            StoreEmbeddingBag(server, kv, 4)
        with pytest.raises(ValueError):
            StoreEmbeddingBag(server, kv, 8, mode="max")
        with pytest.raises(ValueError):
            StoreEmbeddingBag(server, kv, 8, impl="fused")      # CPU server
        bag = StoreEmbeddingBag(server, kv, 8)
        mean = StoreEmbeddingBag(server, kv, 8, mode="mean")
        keys, offsets = torch.tensor([1, 2, 3]), torch.tensor([0, 1, 3])
        with pytest.raises(TypeError):
            bag(keys.to(torch.int32), offsets)
        with pytest.raises(TypeError):
            bag(keys, offsets.to(torch.float32))
        with pytest.raises(TypeError):
            bag(keys.view(1, 3), offsets)
        with pytest.raises(ValueError):
            bag(keys, torch.zeros(0, dtype=torch.int64))        # offsets needs nbags + 1 entries
        for bad in ([0, 1, 4], [1, 1, 3], [0, 2, 1, 3]):
            with pytest.raises(ValueError):
                bag(keys, torch.tensor(bad))
        with pytest.raises(ValueError):
            mean(keys, offsets, torch.ones(3))                  # weights need mode='sum'
        with pytest.raises(TypeError):
            bag(keys, offsets, torch.ones(3, dtype=torch.float64))
        with pytest.raises(ValueError):
            bag(keys, offsets, torch.ones(4))
        with pytest.raises(ValueError):                         # nnz >= 2^31 (a view: nothing is allocated)
            bag(torch.zeros(1, dtype=torch.int64).expand(1 << 31), offsets)
        if torch.cuda.is_available():
            with pytest.raises(TypeError):
                bag(keys.cuda(), offsets)
    finally:
        kv.finalize()
        server.shutdown()


def _multi_hot_worker(kv, server, wid, cfg, steps):
    from adapm_b200.models.deepfm import DeepFM, synthetic_multi_hot_batch

    model = DeepFM(server, kv, cfg)
    model.init_model()
    losses = []
    for s in range(steps):
        ids, off, y = synthetic_multi_hot_batch(cfg, s % 4, server.my_rank())
        model.signal_intent(ids, kv.current_clock() + 1)
        losses.append(model.step(ids, y, offsets=off))
        kv.advance_clock()
    kv.barrier()
    kv.finalize()
    return {"losses": losses, "rows_pushed": model.rows_pushed}


@pytest.mark.parametrize("world", [1, 2])
def test_multi_hot_deepfm_lowers_the_loss(world):
    from adapm_b200.models.deepfm import DeepFMConfig

    cfg = DeepFMConfig(num_features=2000, num_fields=6, embed_dim=8, hidden=(32, 32), batch_size=256, precision="fp32",
                       lr_sparse=0.05, lr_dense=3e-3, multi_hot=4, pooling="mean" if world == 2 else "sum")
    res = run_cluster(lambda kv, server, wid: _multi_hot_worker(kv, server, wid, cfg, 24), world=world, workers=1,
                      mode="threads", value_lengths=cfg.row_len, num_keys=cfg.num_features)
    for r in range(world):
        l = res[r][0]["losses"]
        assert all(np.isfinite(l)), l
        assert np.mean(l[-4:]) < np.mean(l[:4]) - 0.01, l
        assert res[r][0]["rows_pushed"] > 0


def test_synthetic_multi_hot_batch_shape():
    from adapm_b200.models.deepfm import DeepFMConfig, synthetic_multi_hot_batch

    cfg = DeepFMConfig(num_features=26 * 1000, batch_size=64, multi_hot=8)
    ids, off, y = synthetic_multi_hot_batch(cfg, 3)
    lens = off[1:] - off[:-1]
    assert off.numel() == 64 * 26 + 1 and int(off[-1]) == ids.numel()
    assert int(lens.min()) >= 1 and int(lens.max()) <= 8
    field = torch.repeat_interleave(torch.arange(64 * 26) % 26, lens)
    assert torch.all(ids // 1000 == field)
    ids2, off2, y2 = synthetic_multi_hot_batch(cfg, 3)
    assert torch.equal(ids, ids2) and torch.equal(off, off2) and torch.equal(y, y2)


def test_ctr_app_multi_hot_prints_steps():
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "adapm_b200.apps.ctr", "--backend", "cpu", "--multi_hot", "3", "--steps", "3",
                        "--batch_size", "128", "--num_features", "5000", "--embed_dim", "8"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[ctr] step 3: loss" in r.stdout, r.stdout[-2000:]


def test_embedding_bag_kernels_do_not_spill():
    """`-Xptxas -v` of the in-tree build: every kernel of ops_embbag.cu keeps its state in registers."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    mine = {n: v for n, v in k.items() if n.startswith("embbag_")}
    assert {"embbag_prep_kernel", "embbag_fwd_kernel<1>", "embbag_fwd_kernel<4>", "embbag_grad_tile_kernel<1>",
            "embbag_grad_tile_kernel<4>", "embbag_grad_finish_kernel<1>", "embbag_grad_finish_kernel<4>"} <= set(mine), sorted(mine)
    for n, v in mine.items():
        assert v["spill"] == 0, (n, v)
