"""TransE on the parameter store, one GPU: the fused step and the distance evaluation kernels.

    step   ``ops.kge_transe_step`` in place (one launch) against the deterministic variant (index, step, apply), at the
           FB15k shape (14 951 entities, 1 345 relations), d = 152 and 512, neg_ratio 6, 8 192 triples per step, L1.
           Reported: device-timed ms per step, triples/s and pushes/s (pushes = 3 per triple + one per active pair,
           read from stats[3]).
    eval   ``ops.gather_dist_rank_count`` and ``ops.gather_dist_topk`` (k = 10) against the PyTorch route (pull the
           candidate rows, normalise, ``torch.cdist``, then count or ``topk``), 2 048 queries against all entities,
           d = 152, L1 with normalised candidates. The operations bound counts 2 fp32 add-class operations per (query,
           candidate, element) at 128 lanes x SMs x the card's maximum SM clock; the fraction is that bound over the
           kernel time.

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
from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk, kge_transe_step  # noqa: E402

NE, NR = 14951, 1345


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
    cfg = KGEConfig(num_entities=NE, num_relations=NR, embed_dim=d, algorithm="TransE")
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"transe_bench{os.getpid()}_{d}", device=0)
    kv = ad.Worker(0, server)
    g = torch.Generator().manual_seed(d)
    keys = torch.arange(NE + NR)
    rows = torch.randn(keys.numel(), 2 * d, generator=g) * 0.1
    rows[:, d:] = 1e-6
    kv.wait(kv.set(keys, rows.view(-1)))
    return server, kv


def step_rows(info, d, B, neg_ratio, iters, warmup):
    server, kv = store(d)
    dev = server.device
    g = torch.Generator().manual_seed(7)
    batches = []
    for _ in range(4):
        s, o = torch.randint(0, NE, (B,), generator=g), torch.randint(0, NE, (B,), generator=g)
        r = NE + torch.randint(0, NR, (B,), generator=g)
        n = torch.randint(0, NE, (B, 2 * neg_ratio), generator=g)
        batches.append(tuple(t.to(dev).contiguous() for t in (s, r, o, n)))
    loss = torch.zeros(1, device=dev)
    stats = {k: torch.zeros(4, dtype=torch.int64, device=dev) for k in ("in_place", "deterministic")}
    calls = {"in_place": 0, "deterministic": 0}

    def arm(name):
        def fn():
            b = batches[calls[name] % len(batches)]
            calls[name] += 1
            kge_transe_step(server, *b, d, 1, 3.0, 0.1, 0.0, 0.0, loss, stats[name], deterministic=name == "deterministic")
        return fn

    ms = alternate({k: arm(k) for k in calls}, iters, warmup)
    for name, t in ms.items():
        pushes = int(stats[name][3]) / calls[name]
        print(json.dumps({**info, "bench": "transe_step", "variant": name, "d": d, "triples": B, "neg_ratio": neg_ratio,
                          "ms": round(t, 4), "triples_per_s": round(B / t * 1e3), "pushes_per_s": round(pushes / t * 1e3),
                          "pushes_per_triple": round(pushes / B, 2)}), flush=True)
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
        e = buf.view(NE, 2 * d)[:, :d]
        return e / e.norm(dim=1, keepdim=True).clamp(min=1e-12)

    def torch_rank():
        D = torch.cdist(q, torch_rows(), p=1.0)
        dt = D.gather(1, true_col.view(-1, 1))
        return (D < dt).sum(1)

    def torch_topk():
        return torch.topk(-torch.cdist(q, torch_rows(), p=1.0), 10, dim=1)

    arms = {"rank_fused": lambda: gather_dist_rank_count(server, q, keys, d, 1, True, true_col),
            "rank_torch": torch_rank,
            "topk_fused": lambda: gather_dist_topk(server, q, keys, d, 10, 1, True),
            "topk_torch": torch_topk}
    ms = alternate(arms, iters, warmup)
    props = torch.cuda.get_device_properties(0)
    bound_ms = 2.0 * M * NE * d / (128 * props.multi_processor_count * info["max_sm_mhz"] * 1e6) * 1e3
    for name, t in ms.items():
        row = {**info, "bench": "transe_eval", "variant": name, "d": d, "queries": M, "candidates": NE, "ms": round(t, 4)}
        if name.endswith("fused"):
            row.update(ops_bound_ms=round(bound_ms, 4), ops_bound_fraction=round(bound_ms / t, 3))
        print(json.dumps(row), flush=True)
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
        sys.exit("transe_bench needs a CUDA device")
    info = card()
    for d in (152, 512):
        step_rows(info, d, args.triples, 6, args.iters, args.warmup)
    eval_rows(info, 152, args.queries, args.iters, args.warmup)


if __name__ == "__main__":
    main()
