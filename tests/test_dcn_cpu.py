"""DLRM-DCNv2 without a GPU: the torch route of ``ops.dcn_cross`` against the float64 rule, its limits, DLRM with the
cross network on planted data, the app, and the register budget and Hopper instructions of the cross kernels."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dcn_inputs(B, F, E, r, L, seed=0):
    """z, e, V, W, b, grad_out at the scale of a trained layer: V and W Xavier-normal, b small"""
    g = torch.Generator().manual_seed(seed)
    N = (F + 1) * E
    std = (2.0 / (N + r)) ** 0.5
    return (torch.randn(B, E, generator=g), torch.randn(B, F, E, generator=g),
            torch.randn(L, r, N, generator=g) * std, torch.randn(L, N, r, generator=g) * std,
            torch.randn(L, N, generator=g) * 0.1, torch.randn(B, N, generator=g))


# (B, F, E, r, L): L 1 and 3, r below and above N, B 1, N not a multiple of 8
TORCH_SHAPES = [(5, 3, 4, 8, 1), (7, 3, 4, 40, 3), (1, 26, 8, 64, 3), (9, 7, 16, 512, 1), (4, 2, 3, 5, 2),
                (3, 1, 8, 16, 3)]


@pytest.mark.parametrize("B,F,E,r,L", TORCH_SHAPES)
def test_torch_route_matches_float64_rule(B, F, E, r, L):
    from adapm_b200.ops import dcn_cross, dcn_cross_reference

    z, e, V, W, b, g = dcn_inputs(B, F, E, r, L, seed=B * 100 + F * 10 + r + L)
    ref = dcn_cross_reference(z, e, V, W, b, g)
    leaves = [t.clone().requires_grad_(True) for t in (z, e, V, W, b)]
    x = dcn_cross(*leaves)
    assert x.shape == (B, (F + 1) * E) and x.dtype == torch.float32
    x.backward(g)
    tol = dict(rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(x.double(), ref[0], **tol)
    for leaf, want in zip(leaves, ref[1:]):
        assert leaf.grad.shape == want.shape
        torch.testing.assert_close(leaf.grad.double(), want, **tol)


def test_reference_without_rounding_is_the_plain_rule():
    """bf16_operands rounds only operands: on values exact in bf16 with exact products the two agree."""
    from adapm_b200.ops import dcn_cross_reference

    z = torch.tensor([[1.0, 2.0]])
    e = torch.tensor([[[0.5, -1.0]]])
    V = torch.tensor([[[1.0, 0.0, 0.0, 1.0]]])                       # h = x_1 + x_4
    W = torch.tensor([[[1.0], [0.0], [2.0], [0.0]]])
    b = torch.tensor([[0.0, 1.0, 0.0, 0.0]])
    x, *_ = dcn_cross_reference(z, e, V, W, b)
    # x0 = [1, 2, .5, -1], h = 0, u = [0, 1, 0, 0], x1 = x0 * u + x0
    assert x.tolist() == [[1.0, 4.0, 0.5, -1.0]]
    assert dcn_cross_reference(z, e, V, W, b, bf16_operands=True)[0].tolist() == x.tolist()


def _args(B=4, F=3, E=8, r=16, L=2):
    z, e, V, W, b, _ = dcn_inputs(B, F, E, r, L)
    return [z, e, V, W, b]


def _refused(exc, msg, args, impls=("auto", "torch", "fused")):
    from adapm_b200.ops import dcn_cross

    for impl in impls:
        with pytest.raises(exc, match=msg):
            dcn_cross(*args, impl=impl)


def test_shapes_and_types_are_refused():
    a = _args()
    _refused(TypeError, "float32", [a[0].double()] + a[1:])
    _refused(TypeError, "W must be a float32", a[:3] + [a[3].half()] + a[4:])
    _refused(ValueError, "z must be", [a[0][None]] + a[1:])
    _refused(ValueError, r"e must be \[B, F, E\]", [a[0], a[1][:3]] + a[2:])
    _refused(ValueError, r"V must be \[L, r, N\]", a[:2] + [a[2][:, :, :-1]] + a[3:])
    _refused(ValueError, r"W must be \[L, N, r\]", a[:3] + [a[3][:, :, :-1]] + a[4:])
    _refused(ValueError, r"b must be \[L, N\]", a[:4] + [a[4][:1]])
    _refused(ValueError, "impl", a, impls=("bmm",))


def test_limits_are_refused():
    _refused(ValueError, r"1 <= L <= 8", _args(L=9))
    z, e, V, W, b = _args(L=1)
    _refused(ValueError, r"1 <= L <= 8", [z, e, V[:0], W[:0], b[:0]])
    B, N = (1 << 31) // 32 + 1, 32                     # F 3, E 8: no memory, the check runs before anything is read
    z = torch.zeros(1, 8).expand(B, 8)
    e = torch.zeros(1, 3, 8).expand(B, 3, 8)
    _refused(ValueError, r"B \* N < 2\^31", [z, e, V, W, b])
    # the fused route only: its 16-byte TMA rows, its rank range and CUDA tensors
    _refused(ValueError, "multiples of 8", _args(E=3, r=8), impls=("fused",))      # N = 12
    _refused(ValueError, "multiples of 8", _args(r=12), impls=("fused",))
    _refused(ValueError, r"8 <= r <= 1024", _args(r=1032), impls=("fused",))
    _refused(ValueError, "CUDA", _args(), impls=("fused",))
    from adapm_b200.ops import dcn_cross

    for a in (_args(E=3, r=8), _args(r=12), _args(r=1032), _args(r=4)):   # the torch route takes any N and r
        assert dcn_cross(*a, impl="torch").shape == (4, 4 * a[0].shape[1])


# ------------------------------------------------------------------------------------------------ the model
def test_dot_model_is_unchanged():
    """interaction='dot' builds the same bottom and top parameters from a seed as before, and no cross network."""
    from adapm_b200.models.deepfm import DenseNet
    from adapm_b200.models.dlrm import DLRMConfig

    cfg = DLRMConfig(num_fields=4, embed_dim=8, num_dense=5, bottom=(16,), top=(32, 16), precision="fp32")
    dot = _model(cfg)
    assert dot.cross is None
    assert torch.equal(dot.top.w[0], DenseNet(cfg, False, dims=[cfg.interaction_width, 32, 16, 1],
                                              seed=cfg.model_seed + 1).w[0])
    dcn = _model(DLRMConfig(**{**cfg.__dict__, "interaction": "dcn", "cross_rank": 8, "cross_layers": 2}))
    for a, b in zip(dot.bottom.parameters(), dcn.bottom.parameters()):
        assert torch.equal(a, b)
    assert dcn.top.w[0].shape == (32, 40) and dcn.cross.V.shape == (2, 8, 40) and dcn.cross.W.shape == (2, 40, 8)
    assert torch.all(dcn.cross.b == 0)
    g = torch.Generator().manual_seed(cfg.model_seed + 2)
    assert torch.equal(dcn.cross.V.data, torch.randn(2, 8, 40, generator=g) * (2.0 / 48) ** 0.5)
    n_opt = sum(p.numel() for grp in dcn.opt.param_groups for p in grp["params"])
    assert n_opt == sum(p.numel() for m in (dcn.bottom, dcn.top, dcn.cross) for p in m.parameters())


def _model(cfg):
    from adapm_b200.models.dlrm import DLRM

    class _Server:             # what the constructor reads of a server: no rows are pulled
        backend, device, _uniform_len = "cpu", torch.device("cpu"), cfg.row_len

    return DLRM(_Server(), None, cfg)


# held-out AUC after 600 steps of the planted-data config of test_dlrm_cpu.py with a 3-layer rank-64 cross network
# (N 144) on a CPU server: 0.7323 (the planted dense term alone: 0.6575 on the same batches)
PLANTED_AUC_MIN = 0.72
PLANTED_TEST_BATCHES = 8


def planted_dcn_cfg():
    from test_dlrm_cpu import planted_cfg

    return planted_cfg().__class__(**{**planted_cfg().__dict__, "interaction": "dcn", "cross_layers": 3,
                                      "cross_rank": 64})


def planted_dcn_run(server, kv, steps=600):
    """Trains DLRM-DCNv2 on planted data; returns (held-out AUC, AUC of the planted dense term alone)."""
    from adapm_b200.models.dlrm import DLRM, planted_dense_term, synthetic_dlrm_batch
    from adapm_b200.models.ffm import logloss_auc

    cfg = planted_dcn_cfg()
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


def test_planted_data_auc_beats_the_dense_term():
    import adapm_b200 as ad

    cfg = planted_dcn_cfg()
    server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend="cpu",
                       fabric="inproc", job=f"dcn_planted_{np.random.randint(1 << 30)}")
    kv = ad.Worker(0, server)
    try:
        auc, auc_dense = planted_dcn_run(server, kv)
    finally:
        kv.finalize()
        server.shutdown()
    print(f"planted held-out AUC {auc:.4f}, planted dense term alone {auc_dense:.4f}")
    assert auc > PLANTED_AUC_MIN, (auc, auc_dense)
    assert auc > auc_dense + 0.05, (auc, auc_dense)


# ------------------------------------------------------------------------------------------------ the app
def _app(*args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "adapm_b200.apps.ctr", "--backend", "cpu", *args],
                          cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)


def test_ctr_app_dlrm_dcn():
    r = _app("--model", "dlrm", "--interaction", "dcn", "--cross_layers", "2", "--cross_rank", "16",
             "--num_features", "5000", "--num_fields", "6", "--embed_dim", "8", "--steps", "5", "--batch_size", "128",
             "--bottom", "16", "--top", "32,16", "--precision", "fp32", "--multi_hot", "3", "--test_batches", "2")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[ctr] step 5: loss" in r.stdout and "[ctr] test logloss" in r.stdout, r.stdout[-2000:]


@pytest.mark.parametrize("model", ["deepfm", "ffm"])
def test_ctr_app_refuses_dcn_without_dlrm(model):
    r = _app("--model", model, "--interaction", "dcn", "--steps", "1")
    assert r.returncode != 0 and "--interaction dcn needs --model dlrm" in r.stderr, r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ the build
def test_cross_kernels_do_not_spill():
    """`-Xptxas -v` of the in-tree build: every kernel of ops_dcn.cu keeps its state in registers."""
    from test_build_budget import _kernels

    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    mine = {n: v for n, v in k.items() if n.startswith("dcn_")}
    assert {"dcn_stage_kernel", "dcn_bwd_elem_kernel", "dcn_sum_kernel"} <= set(mine), sorted(mine)
    assert sum(n.startswith("dcn_gemm_kernel<") for n in mine) == 4, sorted(mine)
    for n, v in mine.items():
        assert v["spill"] == 0, (n, v)


def test_cross_gemms_run_on_the_tensor_cores():
    """SASS of the in-tree extension: each of the four GEMM epilogue instantiations is a wgmma (HGMMA) kernel fed by
    TMA (UTMALDG)."""
    import glob
    import shutil

    so = glob.glob(os.path.join(ROOT, "adapm_b200", "_C*.so"))
    if not so or shutil.which("cuobjdump") is None:
        pytest.skip("no built extension or no cuobjdump")
    sass = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True).stdout
    per, cur = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            per[cur] = set()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur:
            per[cur].add(m.group(1))
    gemms = [k for k in per if "dcn_gemm_kernel" in k]
    assert len(gemms) == 4, sorted(per)
    for k in gemms:
        assert {"HGMMA", "UTMALDG", "SYNCS"} <= per[k], (k, sorted(per[k]))
