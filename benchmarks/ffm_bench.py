"""Field-aware factorisation machines on the parameter store, one GPU: the fused FFM step against the PyTorch route.

    fused  ``ops.StoreFFM.step``: forward with the partner blocks on chip, radix sort, per-tile sums, finish (one push
           per distinct key); csrc/cuda/ops_ffm.cu
    torch  the fp32 PyTorch route on the same CUDA store: distinct keys -> pull -> index gather into [B, F, F, k] ->
           autograd of the batch loss (with the same per-occurrence L2 term) -> AdaGrad -> push

Shapes: B 8 192 examples of F = 39 fields (Criteo) with k = 4 and 8, and F = 24 with k = 4, over 10^7 keys, ids skewed
within each field as ``models.ffm.synthetic_ffm_batch`` draws them. Reported: device-timed ms per step, examples/s, and
the least-HBM-traffic share: every distinct row of the step read once and written once (2 * 2E * 4 bytes), at the H100
SXM data-sheet figure of 3.35 TB/s, over the measured step time.

Every number is the median of ``--iters`` (>= 20) CUDA-event-timed steps after ``--warmup`` steps, the two routes
alternating in one process on the same seeded batches. Each JSON line carries the card's name and power limit, read by
``nvidia-smi`` in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.ffm import FFM, FFMConfig, synthetic_ffm_batch  # noqa: E402

SHAPES = {"criteo_k4": (39, 4), "criteo_k8": (39, 8), "f24_k4": (24, 4)}
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
NUM_KEYS = 10_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power)}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(arms: dict, iters: int, warmup: int) -> dict:
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in arms}
    for _ in range(iters):
        for k, fn in arms.items():
            ts[k].append(timed(fn))
    return {k: float(np.median(v)) for k, v in ts.items()}


def torch_step(kv, cfg: FFMConfig, ids, y):
    """the FFM rule in fp32 PyTorch on the store: pull the distinct rows, gather, autograd, AdaGrad, push"""
    B, F, k, E = ids.shape[0], cfg.num_fields, cfg.k, cfg.row_values
    r, lam, eta = cfg.pair_scale, cfg.lam, cfg.eta
    uniq, inv = torch.unique(ids.view(-1), return_inverse=True)
    rows = torch.empty(uniq.numel() * 2 * E, device=ids.device)
    kv.wait(kv.pull(uniq, rows, True))
    rows = rows.view(-1, 2 * E)
    with torch.enable_grad():
        val = rows[:, :E].detach().clone().requires_grad_(True)
        x = val[inv].view(B, F, E)
        w, V = x[:, :, 0], x[:, :, 4:].reshape(B, F, F, k)              # V[b, f1, f2] = V[x_bf1][f2]
        P = (V * V.transpose(1, 2)).sum(-1)
        phi = w.sum(1) + r * torch.triu(P, 1).sum((1, 2))
        loss = (torch.nn.functional.softplus(phi) - y * phi).sum()
        own = 1.0 - torch.eye(F, device=ids.device)
        reg = 0.5 * lam * ((w * w).sum() + ((V * V).sum(-1) * own).sum())
        (G,) = torch.autograd.grad(loss + reg, val)
    acc = rows[:, E:]
    upd = torch.where(G != 0, -eta * G / torch.sqrt(acc + G * G), torch.zeros_like(G))
    kv.push(uniq, torch.cat([upd, G * G], 1).contiguous().view(-1), True)
    return loss.detach()


def run_shape(info, name, F, k, B, iters, warmup):
    cfg = FFMConfig(num_features=NUM_KEYS, num_fields=F, k=k, batch_size=B)
    server = ad.Server(cfg.row_len, num_keys=NUM_KEYS, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"ffm_bench{os.getpid()}_{name}", device=0)
    kv = ad.Worker(0, server)
    try:
        model = FFM(server, kv, cfg)
        model.init_model()
        dev = server.device
        batches = [tuple(t.to(dev) for t in synthetic_ffm_batch(cfg, s)) for s in range(4)]
        torch.cuda.synchronize()
        distinct = float(np.mean([torch.unique(ids).numel() for ids, _ in batches]))
        it = {"fused": 0, "torch": 0}

        def fused():
            ids, y = batches[it["fused"] % len(batches)]
            it["fused"] += 1
            model.op.step(ids, y)

        def torch_route():
            ids, y = batches[it["torch"] % len(batches)]
            it["torch"] += 1
            torch_step(kv, cfg, ids, y)

        ms = alternate({"fused": fused, "torch": torch_route}, iters, warmup)
        least_s = distinct * 2 * cfg.row_len * 4 / HBM_BYTES_PER_S
        for route, t in ms.items():
            row = {**info, "bench": "ffm_step", "shape": name, "route": route, "B": B, "F": F, "k": k,
                   "num_keys": NUM_KEYS, "distinct_rows": distinct, "ms_per_step": t, "examples_per_s": B / t * 1e3,
                   "least_hbm_traffic_share": least_s / (t * 1e-3),
                   "least_hbm_traffic_basis": "distinct rows read + written once at 3.35 TB/s (H100 SXM data sheet)"}
            print(json.dumps(row), flush=True)
        print(json.dumps({**info, "bench": "ffm_step", "shape": name, "speedup_fused_over_torch": ms["torch"] / ms["fused"]}),
              flush=True)
    finally:
        kv.finalize()
        server.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be >= 20")
    if not torch.cuda.is_available():
        sys.exit("ffm_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    for name in args.shapes.split(","):
        F, k = SHAPES[name]
        run_shape(info, name, F, k, args.batch, args.iters, args.warmup)
    return 0


if __name__ == "__main__":
    sys.exit(main())
