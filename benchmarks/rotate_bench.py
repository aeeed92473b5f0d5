"""RotatE on the parameter store, one GPU: the fused step and the complex-metric evaluation kernels.

    step   ``ops.kge_rotate_step`` in place (one launch) against the deterministic variant (index, step, apply), at the
           FB15k shape (14 951 entities, 1 345 relations), 8 192 triples per step, d = 256 and 512, 2n = 12 and 256
           negatives per triple, alpha 1. Reported: device-timed ms per step, triples/s and pushes/s (read from
           stats[3]), and the least HBM traffic of the step: every distinct row the step touches read once and written
           once (entity rows 2 d floats, relation rows d floats), over the kernel time as a share of the H100 SXM's
           3.35 TB/s. The kernel itself reads every negative row twice and pushes every (triple, row) pair separately,
           so repeated rows are served from L2.
    eval   ``ops.gather_dist_rank_count`` and ``ops.gather_dist_topk`` (k = 10) with ``p="complex"`` against the PyTorch
           route (pull the candidate rows, ``ops.complex_dist`` in fp32, then count or ``topk``), 2 048 queries against
           all entities, d = 256.

Every number is the median of ``--iters`` (>= 20) CUDA-event-timed runs after ``--warmup`` runs, with the variants
alternating in one process. Each JSON line carries the card's name, power limit and maximum SM clock, read by
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
from adapm_b200.models.kge import KGEConfig  # noqa: E402
from adapm_b200.ops import complex_dist, gather_dist_rank_count, gather_dist_topk, kge_rotate_step  # noqa: E402

NE, NR = 14951, 1345
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power), "max_sm_mhz": float(clock)}


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


def store(d: int):
    cfg = KGEConfig(num_entities=NE, num_relations=NR, embed_dim=d, algorithm="RotatE")
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"rotate_bench{os.getpid()}_{d}", device=0)
    kv = ad.Worker(0, server)
    g = torch.Generator().manual_seed(d)
    ent = torch.randn(NE, 2 * d, generator=g) * 0.1
    ent[:, d:] = 1e-6
    rel = (torch.rand(NR, d, generator=g) * 2 - 1) * np.pi
    rel[:, d // 2:] = 1e-6
    kv.wait(kv.set(torch.arange(NE + NR), torch.cat([ent.view(-1), rel.view(-1)])))
    return server, kv


def least_bytes(b, d):
    """every distinct row of the step read once and written once"""
    s, r, o, n = b
    ents = torch.unique(torch.cat([s, o, n.reshape(-1)])).numel()
    rels = torch.unique(r).numel()
    return 2 * 4 * (ents * 2 * d + rels * d)


def step_rows(info, d, B, nn, iters, warmup):
    server, kv = store(d)
    dev = server.device
    g = torch.Generator().manual_seed(7)
    batches = []
    for _ in range(4):
        s, o = torch.randint(0, NE, (B,), generator=g), torch.randint(0, NE, (B,), generator=g)
        r = NE + torch.randint(0, NR, (B,), generator=g)
        n = torch.randint(0, NE, (B, nn), generator=g)
        batches.append(tuple(t.to(dev).contiguous() for t in (s, r, o, n)))
    hbm = float(np.mean([least_bytes(b, d) for b in batches]))
    loss = torch.zeros(1, device=dev)
    stats = {k: torch.zeros(4, dtype=torch.int64, device=dev) for k in ("in_place", "deterministic")}
    calls = {"in_place": 0, "deterministic": 0}
    gamma = 0.05 * d     # about the distance of two random rows at this init

    def arm(name):
        def fn():
            b = batches[calls[name] % len(batches)]
            calls[name] += 1
            kge_rotate_step(server, *b, d, gamma, 1.0, 0.1, 0.0, loss, stats[name], deterministic=name == "deterministic")
        return fn

    ms = alternate({k: arm(k) for k in calls}, iters, warmup)
    for name, t in ms.items():
        pushes = int(stats[name][3]) / calls[name]
        print(json.dumps({**info, "bench": "rotate_step", "variant": name, "d": d, "triples": B, "negatives": nn,
                          "ms": round(t, 4), "triples_per_s": round(B / t * 1e3), "pushes_per_s": round(pushes / t * 1e3),
                          "pushes_per_triple": round(pushes / B, 2), "least_hbm_mb": round(hbm / 1e6, 1),
                          "least_hbm_fraction": round(hbm / HBM_BYTES_PER_S / (t * 1e-3), 3)}), flush=True)
    kv.finalize()
    server.shutdown()


def eval_rows(info, d, M, iters, warmup):
    server, kv = store(d)
    dev = server.device
    g = torch.Generator().manual_seed(11)
    q = (torch.randn(M, d, generator=g) * 0.1).to(dev)
    keys = torch.arange(NE, dtype=torch.int64, device=dev)
    true_col = torch.randint(0, NE, (M,), generator=g).to(dev)

    def torch_rows():
        buf = torch.empty(NE * 2 * d, device=dev)
        kv.wait(kv.pull(keys, buf, True))
        return buf.view(NE, 2 * d)[:, :d]

    def torch_rank():
        D = complex_dist(q, torch_rows())
        dt = D.gather(1, true_col.view(-1, 1))
        return (D < dt).sum(1)

    def torch_topk():
        return torch.topk(-complex_dist(q, torch_rows()), 10, dim=1)

    arms = {"rank_fused": lambda: gather_dist_rank_count(server, q, keys, d, "complex", False, true_col),
            "rank_torch": torch_rank,
            "topk_fused": lambda: gather_dist_topk(server, q, keys, d, 10, "complex", False),
            "topk_torch": torch_topk}
    ms = alternate(arms, iters, warmup)
    for name, t in ms.items():
        print(json.dumps({**info, "bench": "rotate_eval", "variant": name, "d": d, "queries": M, "candidates": NE,
                          "ms": round(t, 4)}), flush=True)
    kv.finalize()
    server.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--triples", type=int, default=8192)
    ap.add_argument("--queries", type=int, default=2048)
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")
    if not torch.cuda.is_available():
        sys.exit("rotate_bench needs a CUDA device")
    info = card()
    for d in (256, 512):
        for nn in (12, 256):
            step_rows(info, d, args.triples, nn, args.iters, args.warmup)
    eval_rows(info, 256, args.queries, args.iters, args.warmup)


if __name__ == "__main__":
    main()
