"""DLRM on one GPU: the fused dot interaction (ops_dlrm.cu) against the torch route, and full DLRM steps.

    fused   ``ops.dlrm_interaction(impl="fused")``: one kernel forward, one backward
    torch   ``impl="torch"``: cat, bmm, the tril gather and cat; autograd's scatter, bmm and split backward

Interaction rows (forward + backward, z and e leaves that require grad, R.backward(dR)):
    B 8192 / 65536, F 26, E 128 (MLPerf), and B 8192, F 8, E 16 (small E).
Bytes are the lower bound from shapes: forward reads z and e and writes R; backward reads dR, z and e and writes dz and
de. TB/s is those bytes over the measured time; the share is of the H100 SXM data sheet's 3.35 TB/s, a data-sheet
figure, not a measurement.

Step rows: one full DLRM step (bottom MLP 512-256, top 1024-1024-512-256, bf16 tensor-core MLPs, Adam, the fused
embedding bags with their AdaGrad push) at the MLPerf shape, 10^7 keys, B 8192, single-hot and multi-hot (bags of
1..8), the two interaction routes alternating step for step on one store.

Every row: median of ``--iters`` (default 20) after ``--warmup``, timed with CUDA events and a synchronize. Every JSON
line carries the device name and power limit of the card, read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.ops import dlrm_interaction, dlrm_interaction_width  # noqa: E402
from benchmarks.app_bench import device_info  # noqa: E402

HBM_DATASHEET_BPS = 3.35e12


def timed_ms(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def interaction_bytes(B: int, F: int, E: int):
    W = dlrm_interaction_width(F, E)
    te = B * (F + 1) * E * 4                 # z and e
    return te + B * W * 4, B * W * 4 + 2 * te   # forward: read T, write R; backward: read dR and T, write dz and de


def bench_interaction(B, F, E, iters, warmup, info):
    g = torch.Generator(device="cuda").manual_seed(B + F + E)
    z = torch.randn(B, E, device="cuda", generator=g).requires_grad_(True)
    e = torch.randn(B, F, E, device="cuda", generator=g).requires_grad_(True)
    dR = torch.randn(B, dlrm_interaction_width(F, E), device="cuda", generator=g)

    def run(impl):
        z.grad = e.grad = None
        dlrm_interaction(z, e, impl=impl).backward(dR)

    ts = {"fused": [], "torch": []}
    for _ in range(warmup):
        run("fused"); run("torch")
    torch.cuda.synchronize()
    for _ in range(iters):                   # alternating, so both routes see the same clocks and neighbours
        for impl in ts:
            ts[impl].append(timed_ms(lambda: run(impl)))
    fb, bb = interaction_bytes(B, F, E)
    for impl, t in ts.items():
        ms = sorted(t)[len(t) // 2]
        print(json.dumps({"bench": "dlrm_interaction", "impl": impl, "B": B, "F": F, "E": E, "ms": round(ms, 4),
                          "bytes": fb + bb, "TBps": round((fb + bb) / ms / 1e9, 3),
                          "share_of_3.35TBps": round((fb + bb) / ms / 1e9 / 3.35, 3), **info}), flush=True)
    return {impl: sorted(t)[len(t) // 2] for impl, t in ts.items()}


def bench_steps(multi_hot, iters, warmup, info, num_features=10_000_000, B=8192):
    from adapm_b200.models.dlrm import DLRM, DLRMConfig, synthetic_dlrm_batch

    cfg = DLRMConfig(num_features=num_features, batch_size=B, multi_hot=multi_hot)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"dlrm_bench_{os.getpid()}_{multi_hot}", device=0)
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
        print(json.dumps({"bench": "dlrm_step", "impl": impl, "multi_hot": multi_hot, "B": B, "num_keys": num_features,
                          "ms": round(ms, 3), "examples_per_s": round(B / ms * 1e3), **info}), flush=True)
    kv.finalize()
    server.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no_steps", action="store_true", help="interaction rows only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dlrm_bench.py needs a CUDA device")
    info = device_info()
    for B, F, E in ((8192, 26, 128), (65536, 26, 128), (8192, 8, 16)):
        bench_interaction(B, F, E, args.iters, args.warmup, info)
    if not args.no_steps:
        for multi_hot in (0, 8):
            bench_steps(multi_hot, args.iters, args.warmup, info)


if __name__ == "__main__":
    main()
