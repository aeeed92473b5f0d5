"""Implicit-feedback matrix factorisation on the parameter store, one GPU: the fused BPR step and recommendation.

    step       ``ops.mf_bpr_step`` in place (one launch) and deterministic (index, step, apply) at the MovieLens-20M shape
               (138 493 users, 26 744 items) and a large shape (10^7 users, 10^6 items), rank 128, 65 536 positives per
               step, n = 1, 8 and 64 uniform negatives. Reported: device-timed ms per step, positives/s and the achieved
               bytes/s against the H100 SXM's 3.35 TB/s, with (2 + n) rows read and (2 + n) rows reduced per positive,
               2 * rank * 4 bytes each. ``ops.mf_step`` (squared loss, two rows per non-zero) runs as an anchor on as many
               non-zeros as touch the same number of rows.
    recommend  ``MatrixFactorization.recommend`` (pull the users' rows, then ``ops.gather_gemm_topk`` over the item keys
               with the seen items excluded) for 2 048 users with about 150 seen items each, top 10, against both
               catalogues, next to the PyTorch route (pull every item row, ``torch.mm``, mask the seen items, ``topk``).

Every number is the median of ``--iters`` (>= 20) CUDA-event-timed runs after ``--warmup`` runs, with the variants
alternating in one process. Each JSON line carries the card's name and power limit, read by ``nvidia-smi`` in the same
run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix  # noqa: E402
from adapm_b200.ops import mf_bpr_step, mf_step  # noqa: E402

SHAPES = {"ml20m": (138493, 26744), "large": (10_000_000, 1_000_000)}
HBM_BYTES_PER_S = 3.35e12
RANK = 128


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


def store(users: int, items: int):
    """a one-GPU store with the MF key layout, factors ~ N(0, 0.1^2) and zero accumulators, filled on the device"""
    cfg = MFConfig(num_rows=users, num_cols=items, rank=RANK)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"bpr_bench{os.getpid()}_{users}", device=0)
    kv = ad.Worker(0, server)
    dev = server.device
    g = torch.Generator(device=dev).manual_seed(users)
    chunk = 1 << 20
    for s in range(0, cfg.num_keys(1), chunk):
        k = torch.arange(s, min(cfg.num_keys(1), s + chunk), dtype=torch.int64, device=dev)
        rows = torch.zeros(k.numel(), 2 * RANK, device=dev)
        rows[:, :RANK] = torch.randn(k.numel(), RANK, generator=g, device=dev) * 0.1
        kv.wait(kv.set(k, rows.view(-1)))
    kv.waitall()
    torch.cuda.synchronize()
    return cfg, server, kv


def step_rows(info, name, cfg, server, B, iters, warmup):
    dev = server.device
    fck = cfg.first_col_key(1)
    g = torch.Generator(device=dev).manual_seed(7)
    loss = torch.zeros(1, device=dev)
    row_bytes = 2 * RANK * 4
    for n in (1, 8, 64):
        batches = []
        for _ in range(4):
            u = torch.randint(0, cfg.num_rows, (B,), generator=g, device=dev)
            i = fck + torch.randint(0, cfg.num_cols, (B,), generator=g, device=dev)
            j = fck + torch.randint(0, cfg.num_cols, (B, n), generator=g, device=dev)
            batches.append((u, i, j))
        nnz = B * (2 + n) // 2                      # squared-loss anchor: the same number of rows, two per non-zero
        anchor = (torch.randint(0, cfg.num_rows, (nnz,), generator=g, device=dev),
                  fck + torch.randint(0, cfg.num_cols, (nnz,), generator=g, device=dev),
                  torch.randn(nnz, generator=g, device=dev), torch.ones(nnz, dtype=torch.int32, device=dev),
                  torch.ones(nnz, dtype=torch.int32, device=dev))
        calls = {"in_place": 0, "deterministic": 0}

        def arm(v):
            def fn():
                b = batches[calls[v] % len(batches)]
                calls[v] += 1
                mf_bpr_step(server, *b, RANK, 0.05, 0.01, loss, deterministic=v == "deterministic")
            return fn

        arms = {v: arm(v) for v in calls}
        arms["mf_step_anchor"] = lambda: mf_step(server, *anchor, RANK, 0.01, 0.05, loss)
        ms = alternate(arms, iters, warmup)
        moved = 2 * B * (2 + n) * row_bytes             # (2 + n) rows read and (2 + n) rows reduced per positive
        for v, t in ms.items():
            row = {**info, "bench": "bpr_step", "shape": name, "users": cfg.num_rows, "items": cfg.num_cols,
                   "rank": RANK, "negatives": n, "variant": v, "ms": round(t, 4)}
            if v == "mf_step_anchor":
                row.update(nnz=nnz, nnz_per_s=round(nnz / t * 1e3))
            else:
                bps = moved / (t * 1e-3)
                row.update(positives=B, positives_per_s=round(B / t * 1e3), bytes_per_s=round(bps),
                           hbm_fraction=round(bps / HBM_BYTES_PER_S, 3))
            print(json.dumps(row), flush=True)


def recommend_rows(info, name, cfg, server, kv, M, iters, warmup):
    dev = server.device
    rng = np.random.default_rng(3)
    users = rng.choice(cfg.num_rows, M, replace=False)
    per = rng.integers(100, 201, M)                   # about 150 seen items per user
    ii = np.repeat(users, per)
    jj = np.concatenate([rng.choice(cfg.num_cols, p, replace=False) for p in per])
    data = SparseMatrix(ii, jj, np.ones(ii.shape[0], np.float32), cfg.num_rows, cfg.num_cols, 1, 0)
    model = MatrixFactorization(server, kv, cfg, data)
    seen = data.seen(users)
    seen_dev = (seen[0].to(dev), seen[1].to(dev))
    ukeys = torch.from_numpy(users).to(dev)
    ikeys = torch.arange(cfg.num_cols, dtype=torch.int64, device=dev) + cfg.first_col_key(1)
    mask_rows = torch.repeat_interleave(torch.arange(M, device=dev), seen_dev[0][1:] - seen_dev[0][:-1])

    def torch_route():
        q = torch.empty(M * 2 * RANK, device=dev)
        kv.wait(kv.pull(ukeys, q, True))
        e = torch.empty(cfg.num_cols * 2 * RANK, device=dev)
        kv.wait(kv.pull(ikeys, e, True))
        s = q.view(M, 2 * RANK)[:, :RANK] @ e.view(-1, 2 * RANK)[:, :RANK].t()
        s[mask_rows, seen_dev[1]] = float("-inf")
        return torch.topk(s, 10, dim=1)

    ms = alternate({"fused": lambda: model.recommend(users, 10, seen=seen_dev), "torch": torch_route}, iters, warmup)
    for v, t in ms.items():
        print(json.dumps({**info, "bench": "bpr_recommend", "shape": name, "users": M, "items": cfg.num_cols,
                          "rank": RANK, "k": 10, "seen_per_user": round(float(per.mean()), 1), "variant": v,
                          "ms": round(t, 4)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--positives", type=int, default=65536)
    ap.add_argument("--queries", type=int, default=2048)
    ap.add_argument("--shapes", default="ml20m,large")
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")
    if not torch.cuda.is_available():
        sys.exit("bpr_bench needs a CUDA device")
    info = card()
    for name in args.shapes.split(","):
        users, items = SHAPES[name]
        cfg, server, kv = store(users, items)
        step_rows(info, name, cfg, server, args.positives, args.iters, args.warmup)
        recommend_rows(info, name, cfg, server, kv, args.queries, args.iters, args.warmup)
        kv.finalize()
        server.shutdown()


if __name__ == "__main__":
    main()
