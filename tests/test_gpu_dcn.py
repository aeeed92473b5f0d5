"""The fused DCN-v2 cross network (csrc/cuda/ops_dcn.cu) on an H100: against the float64 rule with and without bf16
operands where the tiles change, bit for bit against itself, in the profiler trace of a forward and backward, in
multi-hot DLRM-DCNv2 steps against the torch route, and on planted data."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from multirank import one_rank_store
from test_dcn_cpu import dcn_inputs

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fused(z, e, V, W, b, g):
    from adapm_b200.ops import dcn_cross

    leaves = [t.cuda().requires_grad_(True) for t in (z, e, V, W, b)]
    x = dcn_cross(*leaves, impl="fused")
    x.backward(g.cuda())
    torch.cuda.synchronize()
    return [x.detach().cpu()] + [t.grad.cpu() for t in leaves]


def _errs(a, ref):
    """|a - ref| elementwise, relative to the largest |ref|"""
    return (a.double() - ref).abs() / ref.abs().max().clamp(min=1e-30)


# (B, F, E, r, L): B 1 / 127 / 129 / 3000 (row tiles of 128, transposed pitch 8), N 128 / 136 / 3456 (column tiles
# and k-blocks of 64), r 8 / 64 / 200 / 512, L 1 and 3
SHAPES = [(1, 7, 16, 8, 1), (127, 16, 8, 64, 3), (129, 16, 8, 200, 1), (3000, 7, 16, 64, 3), (129, 26, 128, 512, 3),
          (3000, 26, 128, 512, 1), (127, 7, 16, 512, 3), (1, 26, 128, 200, 3)]
NAMES = ["x_L", "dz", "de", "dV", "dW", "db"]


@gpu
@pytest.mark.parametrize("B,F,E,r,L", SHAPES)
def test_fused_matches_float64_rule(B, F, E, r, L):
    from adapm_b200.ops import dcn_cross_reference

    args = dcn_inputs(B, F, E, r, L, seed=B + F * 7 + r * 131 + L)
    got = _fused(*args)
    emu = dcn_cross_reference(*args, bf16_operands=True)
    plain = dcn_cross_reference(*args)
    for name, a, want, exact in zip(NAMES, got, emu, plain):
        assert a.shape == want.shape, name
        # the same roundings as the fused route: what is left is fp32 accumulation (below 1e-6 at the small shapes),
        # except where an fp32 sum and its float64 counterpart round to neighbouring bf16 values (one unit in 2^8 of an
        # operand) and the flip travels through the later layers; at N 3456 and L 3 (H100 80GB HBM3) that reaches
        # 2.5e-3 of the largest value, in under 0.4 % of the elements
        err = _errs(a, want)
        big = float((err > 1e-3).double().mean())
        print(f"{name}: max {float(err.max()):.2e}, share above 1e-3 {big:.1e}, "
              f"against the plain rule {float(_errs(a, exact).max()):.2e}")
        assert float(err.max()) < 5e-3 and big < 1e-2, (name, float(err.max()), big)
        # against the plain rule: bf16 operands (8 significant bits) through L layers; at most 6.2e-3 measured
        assert float(_errs(a, exact).max()) < 2e-2, (name, float(_errs(a, exact).max()))


@gpu
@pytest.mark.parametrize("B,F,E,r,L", [(3000, 26, 128, 512, 3), (8192, 7, 16, 64, 2)])
def test_fused_is_bit_identical_across_runs(B, F, E, r, L):
    """the second shape has one weight-gradient tile and K = B = 8192 long: its k-blocks are split, and the partial
    tiles added in split order"""
    args = dcn_inputs(B, F, E, r, L, seed=11)
    a = _fused(*args)
    b = _fused(*args)
    for name, x, y in zip(NAMES, a, b):
        assert torch.equal(x, y), name


_CHILD = r"""
import json, torch
from torch.profiler import ProfilerActivity, profile
from test_build_budget import kernel_name
from test_dcn_cpu import dcn_inputs
from adapm_b200.ops import dcn_cross

z, e, V, W, b, g = [t.cuda() for t in dcn_inputs(256, 26, 128, 512, 3, seed=3)]
leaves = [t.requires_grad_(True) for t in (z, e, V, W, b)]

def step():
    for t in leaves:
        t.grad = None
    x = dcn_cross(*leaves, impl="fused")
    torch.cuda.synchronize()
    x.backward(g)

step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
print("KERNELS " + json.dumps([kernel_name(e.name) for e in ev]))
"""


@gpu
def test_profiler_trace_has_only_the_ops_kernels():
    """In a fresh process (the CUDA activity records of torch.profiler can stop arriving in a long session). Forward:
    the stage kernel, then h and cross GEMMs per layer; backward: per layer the elementwise pass, the db sum and four
    GEMMs; nothing else between the first and the last of them in either direction."""
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    stage = names.index("dcn_stage_kernel")
    fwd = names[stage:stage + 7]
    assert fwd == ["dcn_stage_kernel"] + ["dcn_gemm_kernel<0>", "dcn_gemm_kernel<1>"] * 3, names
    first = names.index("dcn_bwd_elem_kernel")
    last = max(i for i, n in enumerate(names) if n.startswith("dcn_"))
    bwd = names[first:last + 1]
    assert all(n.startswith("dcn_") for n in bwd), names
    per_layer = ["dcn_bwd_elem_kernel", "dcn_sum_kernel", "dcn_gemm_kernel<0>", "dcn_gemm_kernel<2>",
                 "dcn_gemm_kernel<3>", "dcn_gemm_kernel<3>"]
    assert bwd == per_layer * 3, names
    assert not any("gemm" in n.lower() and not n.startswith("dcn_") for n in names), names
    assert not any(n.lower().startswith(("cutlass", "sm90_", "ampere_", "cublas")) for n in names), names


def _dcn_steps(impl, steps=4):
    from adapm_b200.models.dlrm import DLRM, DLRMConfig, synthetic_dlrm_batch

    cfg = DLRMConfig(num_features=26 * 500, embed_dim=64, bottom=(64,), top=(128, 64), batch_size=512, multi_hot=4,
                     precision="fp32", lr_sparse=0.05, interaction="dcn", cross_layers=3, cross_rank=64)
    with one_rank_store(cfg.row_len, cfg.num_features, "cuda", "float32") as (server, kv):
        model = DLRM(server, kv, cfg, impl=impl)
        model.init_model()
        everything = torch.arange(cfg.num_features, device="cuda")

        def rows():
            out = torch.empty(cfg.num_features * cfg.row_len, device="cuda")
            kv.wait(kv.pull(everything, out))
            return out.view(cfg.num_features, -1).cpu()

        before = rows()
        losses = []
        for s in range(steps):
            dense, ids, off, y = synthetic_dlrm_batch(cfg, s, 0)
            losses.append(model.step(dense, ids, y, offsets=off))
        return losses, torch.nonzero((rows() != before).any(1)).view(-1)


@gpu
def test_multi_hot_dcn_steps_match_torch_route():
    """the same rows are updated (AdaGrad's first step moves a row by lr * sign(g), so the values themselves differ
    wherever a gradient element is near zero), and the losses agree to bf16 accuracy"""
    lf, kf = _dcn_steps("fused")
    lt, kt = _dcn_steps("torch")
    assert kf.numel() > 0 and torch.equal(kf, kt)
    np.testing.assert_allclose(lf, lt, rtol=1e-2)                 # bf16 cross GEMMs against fp32


@gpu
def test_planted_data_auc_on_the_h100():
    from test_dcn_cpu import PLANTED_AUC_MIN, planted_dcn_cfg, planted_dcn_run

    cfg = planted_dcn_cfg()
    with one_rank_store(cfg.row_len, cfg.num_features, "cuda", "float32") as (server, kv):
        auc, auc_dense = planted_dcn_run(server, kv)
    print(f"planted held-out AUC {auc:.4f}, planted dense term alone {auc_dense:.4f}")
    assert auc > PLANTED_AUC_MIN, (auc, auc_dense)
    assert auc > auc_dense + 0.05, (auc, auc_dense)
