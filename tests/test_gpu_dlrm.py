"""The fused DLRM interaction kernels (csrc/cuda/ops_dlrm.cu) on an H100: against the float64 rule at the limits,
bit for bit against themselves, in a multi-hot DLRM step against the torch route, in the profiler trace of a step,
and DLRM on planted data."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from multirank import one_rank_store

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(B, F, E, seed):
    g = torch.Generator().manual_seed(seed)
    W = (E + F * (F + 1) // 2 + 7) // 8 * 8
    return (torch.randn(B, E, generator=g), torch.randn(B, F, E, generator=g), torch.randn(B, W, generator=g))


def _fused(z, e, g):
    from adapm_b200.ops import dlrm_interaction

    z = z.cuda().requires_grad_(True)
    e = e.cuda().requires_grad_(True)
    R = dlrm_interaction(z, e, impl="fused")
    R.backward(g.cuda())
    torch.cuda.synchronize()
    return R.detach().cpu(), z.grad.cpu(), e.grad.cpu()


# (B, F, E): the MLPerf shape, F 63 (16 row blocks, 136 tiles), E 512 and E 4, F 1, B 1, a small-E shape, and B not a
# multiple of anything (one CTA per example, 128 threads: 8-lane tiles and 4-row blocks are the tiles)
SHAPES = [(257, 26, 128), (33, 63, 512), (100, 63, 4), (65, 1, 4), (1, 26, 128), (1001, 8, 16), (7, 5, 512),
          (3, 26, 132)]


@gpu
@pytest.mark.parametrize("B,F,E", SHAPES)
def test_fused_matches_float64_rule(B, F, E):
    from adapm_b200.ops import dlrm_interaction_reference

    z, e, g = _inputs(B, F, E, seed=B + F * 7 + E * 131)
    R, dz, de = _fused(z, e, g)
    R_ref, dz_ref, de_ref = dlrm_interaction_reference(z, e, g)
    # fp32 sums of E (forward) and F + 1 (backward) unit-variance products
    torch.testing.assert_close(R.double(), R_ref, rtol=1e-5, atol=2e-6 * E ** 0.5 * 4)
    P = F * (F + 1) // 2
    assert torch.all(R[:, E + P:] == 0) and torch.equal(R[:, :E], z)
    tol = dict(rtol=1e-5, atol=2e-6 * (F + 1) ** 0.5 * E ** 0.5 * 4)
    torch.testing.assert_close(dz.double(), dz_ref, **tol)
    torch.testing.assert_close(de.double(), de_ref, **tol)


@gpu
def test_fused_is_bit_identical_across_runs():
    z, e, g = _inputs(3000, 26, 128, seed=5)
    a = _fused(z, e, g)
    b = _fused(z, e, g)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _dlrm_steps(impl, steps=4):
    from adapm_b200.models.dlrm import DLRM, DLRMConfig, synthetic_dlrm_batch

    cfg = DLRMConfig(num_features=26 * 500, embed_dim=64, bottom=(64,), top=(128, 64), batch_size=512, multi_hot=4,
                     precision="fp32", lr_sparse=0.05)
    with one_rank_store(cfg.row_len, cfg.num_features, "cuda", "float32") as (server, kv):
        model = DLRM(server, kv, cfg, impl=impl)
        model.init_model()
        losses, touched = [], []
        for s in range(steps):
            dense, ids, off, y = synthetic_dlrm_batch(cfg, s, 0)
            losses.append(model.step(dense, ids, y, offsets=off))
            touched.append(ids)
        keys = torch.unique(torch.cat(touched)).cuda()
        rows = torch.empty(keys.numel() * cfg.row_len, device="cuda")
        kv.wait(kv.pull(keys, rows))
        return losses, rows.view(keys.numel(), -1).cpu()


@gpu
def test_multi_hot_step_matches_torch_route():
    lf, rf = _dlrm_steps("fused")
    lt, rt = _dlrm_steps("torch")
    np.testing.assert_allclose(lf, lt, rtol=1e-4)
    torch.testing.assert_close(rf, rt, rtol=1e-3, atol=1e-5)


_CHILD = r"""
import json, torch
from torch.profiler import ProfilerActivity, profile
from multirank import one_rank_store
from test_build_budget import kernel_name
from adapm_b200.ops import StoreEmbeddingBag, dlrm_interaction

store = one_rank_store(2 * 128, 26 * 1000, "cuda", "float32")
server, kv = store.__enter__()
bag = StoreEmbeddingBag(server, kv, 128)
B = 256
keys = torch.randint(0, 26 * 1000, (B * 26,), device="cuda")
off = torch.arange(B * 26 + 1, device="cuda")
z = torch.randn(B, 128, device="cuda", requires_grad=True)
w = torch.randn(B, 480, device="cuda")

def step():
    R = dlrm_interaction(z, bag(keys, off).view(B, 26, 128))
    (R * w).sum().backward()

step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
print("KERNELS " + json.dumps([kernel_name(e.name) for e in ev]))
store.__exit__(None, None, None)
"""


@gpu
def test_profiler_trace_has_the_two_kernels_between_the_bags():
    """In a fresh process (the CUDA activity records of torch.profiler can stop arriving in a long session)."""
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    dl = [i for i, n in enumerate(names) if n.startswith("dlrm_")]
    assert [names[i] for i in dl] == ["dlrm_interaction_fwd_kernel", "dlrm_interaction_bwd_kernel"], names
    fwd_bag = [i for i, n in enumerate(names) if n.startswith("embbag_fwd_kernel")]
    bwd_bag = [i for i, n in enumerate(names) if n.startswith("embbag_prep_kernel")]
    assert fwd_bag and bwd_bag and max(fwd_bag) < dl[0] < dl[1] < min(bwd_bag), names
    assert not any("bmm" in n.lower() or "gemm" in n.lower() for n in names), names


@gpu
def test_planted_data_auc_on_the_h100():
    from test_dlrm_cpu import PLANTED_AUC_MIN, planted_cfg, planted_run

    cfg = planted_cfg()
    with one_rank_store(cfg.row_len, cfg.num_features, "cuda", "float32") as (server, kv):
        auc, auc_dense = planted_run(server, kv)
    print(f"planted held-out AUC {auc:.4f}, planted dense term alone {auc_dense:.4f}")
    assert auc > PLANTED_AUC_MIN, (auc, auc_dense)
    assert auc > auc_dense + 0.05, (auc, auc_dense)
