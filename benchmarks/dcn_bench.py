"""DLRM-DCNv2 on one GPU: the fused low-rank cross network (ops_dcn.cu) against the torch route, and full DLRM-DCNv2
steps.

    fused     ``ops.dcn_cross(impl="fused")``: bf16 wgmma GEMMs with the elementwise work in their epilogues
    torch     ``impl="torch"``: the fp32 rule with matmul on cuBLAS, TF32 off
    autocast  ``impl="torch"`` under ``torch.autocast(dtype=torch.bfloat16)``: bf16 cuBLAS GEMMs, the elementwise work
              in separate PyTorch kernels (a comparison arm of this benchmark only, not a route of the library)

Cross-network rows (forward + backward, z, e, V, W and b leaves that require grad, x.backward(dx)): B 8192 and 65536
with F 26, E 128, r 512, L 3 (MLPerf DLRM-DCNv2, N 3456), and B 8192 with F 7, E 16, r 64, L 3 (N 128). The arms
alternate, so that all see the same clocks and neighbours. From shapes: flops = 12 B N r L (two GEMMs forward and
four backward per layer, 2 B N r each); elementwise bytes = 24 B N L, the lower bound of a layer that keeps its fp32
residual stream in memory (forward: read x_0 and x_l, write x_{l+1}; backward: read G and x_0, write dx_l; 4 bytes
each). Each row gives both bounds at the H100 SXM data sheet's 989 TFLOP/s (dense bf16) and 3.35 TB/s: data-sheet
figures, not measurements; ``bound`` names the larger.

``--kernels``: per-kernel device times of the fused route at the MLPerf shape, B 8192, from torch.profiler (a run of
its own, after the timed rows).

Step rows: one full DLRM-DCNv2 step (bottom MLP 512-256, the cross network, top MLP 1024-1024-512-256, bf16 tensor-core
MLPs, Adam, the fused embedding bags with their AdaGrad push) at the MLPerf shape, 10^7 keys, B 8192, single-hot and
multi-hot (bags of 1..8), the fused and torch cross routes alternating step for step on one store.

Every row: median of ``--iters`` (default 20) after ``--warmup``, timed with CUDA events and a synchronize. Every JSON
line carries the device name and power limit of the card, read in the same run."""
import argparse
import contextlib
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.ops import dcn_cross  # noqa: E402
from benchmarks.app_bench import device_info  # noqa: E402
from benchmarks.dlrm_bench import timed_ms  # noqa: E402

HBM_DATASHEET_BPS = 3.35e12
BF16_DATASHEET_FLOPS = 989e12
ARMS = ("fused", "torch", "autocast")


def cross_inputs(B, F, E, r, L):
    g = torch.Generator(device="cuda").manual_seed(B + F + E + r + L)
    N = (F + 1) * E
    std = (2.0 / (N + r)) ** 0.5

    def rn(*shape, scale=1.0):
        return (torch.randn(*shape, device="cuda", generator=g) * scale).requires_grad_(True)

    leaves = [rn(B, E), rn(B, F, E), rn(L, r, N, scale=std), rn(L, N, r, scale=std), rn(L, N, scale=0.1)]
    return leaves, torch.randn(B, N, device="cuda", generator=g)


def run_arm(arm, leaves, dx):
    for t in leaves:
        t.grad = None
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if arm == "autocast" else contextlib.nullcontext()
    with ctx:
        x = dcn_cross(*leaves, impl="fused" if arm == "fused" else "torch")
    x.backward(dx)


def bench_cross(B, F, E, r, L, iters, warmup, info):
    leaves, dx = cross_inputs(B, F, E, r, L)
    N = (F + 1) * E
    ts = {a: [] for a in ARMS}
    for _ in range(warmup):
        for a in ARMS:
            run_arm(a, leaves, dx)
    torch.cuda.synchronize()
    for _ in range(iters):
        for a in ARMS:
            ts[a].append(timed_ms(lambda: run_arm(a, leaves, dx)))
    flops, nbytes = 12 * B * N * r * L, 24 * B * N * L
    t_flops, t_bytes = flops / BF16_DATASHEET_FLOPS * 1e3, nbytes / HBM_DATASHEET_BPS * 1e3
    out = {}
    for a, t in ts.items():
        ms = sorted(t)[len(t) // 2]
        out[a] = ms
        print(json.dumps({"bench": "dcn_cross", "impl": a, "B": B, "F": F, "E": E, "N": N, "r": r, "L": L,
                          "ms": round(ms, 4), "TFLOPs": round(flops / ms / 1e9, 1),
                          "elementwise_bytes": nbytes, "share_of_3.35TBps": round(t_bytes / ms, 3),
                          "share_of_989TFLOPs": round(t_flops / ms, 3),
                          "bound": "bytes" if t_bytes > t_flops else "flops", **info}), flush=True)
    return out


def kernel_times(B, F, E, r, L, info, reps=5):
    """per-kernel device time (ms per forward + backward) of the fused route"""
    from torch.profiler import ProfilerActivity, profile

    leaves, dx = cross_inputs(B, F, E, r, L)
    run_arm("fused", leaves, dx)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            run_arm("fused", leaves, dx)
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.replace("(anonymous namespace)::", "").replace("adapm::cudaops::", "")
        name = name.replace("void ", "").split("(")[0]
        us = ev.time_range.end - ev.time_range.start
        c, t = tot.get(name, (0, 0.0))
        tot[name] = (c + 1, t + us)
    for name, (c, us) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        print(json.dumps({"bench": "dcn_kernels", "B": B, "F": F, "E": E, "r": r, "L": L, "kernel": name,
                          "launches_per_call": c / reps, "ms_per_call": round(us / reps / 1e3, 4), **info}), flush=True)


def bench_steps(multi_hot, iters, warmup, info, num_features=10_000_000, B=8192):
    from adapm_b200.models.dlrm import DLRM, DLRMConfig, synthetic_dlrm_batch

    cfg = DLRMConfig(num_features=num_features, batch_size=B, multi_hot=multi_hot, interaction="dcn")
    server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"dcn_bench_{os.getpid()}_{multi_hot}", device=0)
    kv = ad.Worker(0, server)
    models = {impl: DLRM(server, kv, cfg, impl=impl) for impl in ("fused", "torch")}
    models["fused"].init_model()
    batches = []
    for s in range(4):
        dense, ids, *off, y = synthetic_dlrm_batch(cfg, s, 0)
        batches.append((dense.cuda(), ids.cuda(), off[0].cuda() if off else None, y.cuda()))
    ts = {impl: [] for impl in models}
    for i in range(warmup + iters):
        for impl, m in models.items():
            dense, ids, off, y = batches[i % len(batches)]
            t = timed_ms(lambda: m.step(dense, ids, y, offsets=off, return_tensor=True))
            if i >= warmup:
                ts[impl].append(t)
    for impl, t in ts.items():
        ms = sorted(t)[len(t) // 2]
        print(json.dumps({"bench": "dcn_step", "impl": impl, "multi_hot": multi_hot, "B": B, "num_keys": num_features,
                          "L": cfg.cross_layers, "r": cfg.cross_rank, "ms": round(ms, 3),
                          "examples_per_s": round(B / ms * 1e3), **info}), flush=True)
    kv.finalize()
    server.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no_steps", action="store_true", help="cross-network rows only")
    ap.add_argument("--kernels", action="store_true", help="also the per-kernel times of the fused route")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dcn_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = device_info()
    for B, F, E, r, L in ((8192, 26, 128, 512, 3), (65536, 26, 128, 512, 3), (8192, 7, 16, 64, 3)):
        bench_cross(B, F, E, r, L, args.iters, args.warmup, info)
        torch.cuda.empty_cache()
    if args.kernels:
        kernel_times(8192, 26, 128, 512, 3, info)
    if not args.no_steps:
        for multi_hot in (0, 8):
            bench_steps(multi_hot, args.iters, args.warmup, info)


if __name__ == "__main__":
    main()
