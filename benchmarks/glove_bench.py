"""GloVe on the parameter store, one GPU: the co-occurrence count and the fused step.

    cooc   ``ops.glove_cooccurrence`` on a seeded Zipf corpus (``--vocab`` words, ``--tokens`` tokens in lines of 10 to
           30 words, symmetric, distance-weighted) at windows 10 and 15, against a PyTorch route with the same memory
           budget (per token chunk: packed keys, ``torch.unique(return_inverse=True)`` + ``index_add_`` of the int64
           numerators, then the same with the running result). Reported: device-synchronised seconds per count,
           tokens/s and the non-zeros.
    step   ``ops.glove_step`` in place (one launch) and deterministic (index, step, apply), and the PyTorch route (pull
           the step's rows, the rule in fp32 PyTorch, push the updates), at V = 400 000 and 1 000 000, d = 300, 2^18
           non-zeros per step with Zipf-distributed words and contexts. Reported: ms per step and the least-traffic
           share: each distinct row of the step read and written once, at the H100 SXM's 3.35 TB/s, over the step time.

Every number is the median of ``--runs`` timed runs after a warm-up, with the variants alternating in one process. Each
JSON line carries the card's name and power limit, read by ``nvidia-smi`` in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.ops import glove_cooccurrence, glove_step  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power)}


def synced(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def alternate(arms: dict, runs: int, warmup: int) -> dict:
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    ts = {k: [] for k in arms}
    for _ in range(runs):
        for k, fn in arms.items():
            ts[k].append(synced(fn))
    return {k: float(np.median(v)) for k, v in ts.items()}


def zipf(n, V, gen):
    p = 1.0 / torch.arange(1, V + 1, dtype=torch.float64, device="cuda")
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    for i in range(0, n, 1 << 24):              # torch.multinomial draws at most 2^24 samples per call
        m = min(1 << 24, n - i)
        out[i:i + m] = torch.multinomial(p.float(), m, replacement=True, generator=gen)
    return out


def corpus(V, n_tokens, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tok = zipf(n_tokens, V, gen).int()
    lens = torch.randint(10, 31, (n_tokens // 10 + 1,), generator=gen, device="cuda")
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(lens, 0)])
    off = torch.cat([off[off < n_tokens], torch.tensor([n_tokens], device="cuda")])
    return tok, off


def torch_cooc(tok, off, V, window, lw, max_bytes):
    """the PyTorch route: packed keys, unique + index_add_ per chunk, merged into the running result the same way"""
    n = tok.numel()
    sid = torch.repeat_interleave(torch.arange(off.numel() - 1, device="cuda"), off[1:] - off[:-1])
    per_tok = 2 * window * 8 * 16               # keys, numerators, their concatenation, unique's sort and inverse
    T = max(1, int(max_bytes // per_tok))
    keys = torch.zeros(0, dtype=torch.int64, device="cuda")
    sums = torch.zeros(0, dtype=torch.int64, device="cuda")
    t64 = tok.long()
    for t0 in range(0, n, T):
        t1 = min(n, t0 + T + window)
        ck, cn = [keys], [sums]
        for k in range(1, window + 1):
            lo, hi = t0, min(t0 + T, t1 - k)
            if hi <= lo:
                continue
            same = sid[lo:hi] == sid[lo + k:hi + k]
            a, b = t64[lo:hi][same], t64[lo + k:hi + k][same]
            ck += [a * V + b, b * V + a]
            cn += [torch.full((2 * a.numel(),), lw // k, dtype=torch.int64, device="cuda")]
        allk = torch.cat(ck)
        alln = torch.cat([sums] + cn[1:])
        keys, inv = torch.unique(allk, return_inverse=True)
        sums = torch.zeros(keys.numel(), dtype=torch.int64, device="cuda").index_add_(0, inv, alln)
    return keys, (sums.double() / lw).float()


def bench_cooc(args, info):
    tok, off = corpus(args.vocab, args.tokens, 1)
    for window in (10, 15):
        lw = int(np.lcm.reduce(np.arange(1, window + 1)))
        out = {}

        def ours():
            out["nnz"] = glove_cooccurrence(tok, off, args.vocab, window, True, True, max_bytes=args.max_bytes)[0].numel()

        def plain():
            out["nnz_torch"] = torch_cooc(tok, off, args.vocab, window, lw, args.max_bytes)[0].numel()
            torch.cuda.empty_cache()         # the device count allocates outside PyTorch's caching allocator

        arms = {"device": ours, "pytorch": plain} if not args.skip_torch else {"device": ours}
        t = alternate(arms, args.runs, 1)
        for k, s in t.items():
            print(json.dumps({"bench": "glove_cooc", "arm": k, "window": window, "tokens": args.tokens,
                              "vocab": args.vocab, "seconds": round(s, 4), "tokens_per_s": round(args.tokens / s),
                              "nnz": out["nnz"], "max_bytes": args.max_bytes, **info}), flush=True)
        if "nnz_torch" in out:
            assert out["nnz_torch"] == out["nnz"], (out["nnz_torch"], out["nnz"])


def bench_step(args, info):
    d, D, B = 300, 304, 1 << 18
    for V in (400_000, 1_000_000):
        ad.setup(2 * V, 1)
        s = ad.Server(2 * D, num_keys=2 * V, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                      job=f"glove_bench_{V}", device=0)
        kv = ad.Worker(0, s)
        gen = torch.Generator(device="cuda").manual_seed(V)
        for i in range(0, 2 * V, 1 << 18):
            k = torch.arange(i, min(2 * V, i + (1 << 18)), device="cuda")
            rows = torch.zeros(k.numel(), 2 * D, device="cuda")
            rows[:, :d + 1] = (torch.rand(k.numel(), d + 1, generator=gen, device="cuda") - 0.5) / d
            rows[:, D:D + d + 1] = 1.0
            kv.wait(kv.set(k, rows.view(-1)))
        kv.waitall()
        steps = []
        for _ in range(4):
            wk, ck = 2 * zipf(B, V, gen), 2 * zipf(B, V, gen) + 1
            x = 1.0 + torch.rand(B, generator=gen, device="cuda") * 50
            steps.append((wk, ck, x))
        distinct = float(np.mean([torch.unique(torch.cat([w, c])).numel() for w, c, _ in steps]))
        loss = torch.zeros(1, device="cuda")
        it = {"n": 0}

        def nxt():
            it["n"] += 1
            return steps[it["n"] % len(steps)]

        def fused(det):
            return lambda: glove_step(s, *nxt(), d, 0.05, 100.0, 0.75, loss, deterministic=det)

        def plain():
            wk, ck, x = nxt()
            keys = torch.cat([wk, ck])
            r = torch.empty(2 * B * 2 * D, device="cuda")
            kv.wait(kv.pull(keys, r, True))
            r = r.view(2 * B, 2 * D)
            W, C = r[:B], r[B:]
            diff = (W[:, :d] * C[:, :d]).sum(1) + W[:, d] + C[:, d] - torch.log(x)
            f = torch.where(x < 100.0, (x / 100.0) ** 0.75, torch.ones_like(x))
            fd = (f * diff).unsqueeze(1)
            g = torch.zeros(2 * B, D, device="cuda")
            g[:B, :d], g[B:, :d] = fd * C[:, :d], fd * W[:, :d]
            g[:B, d], g[B:, d] = fd[:, 0], fd[:, 0]
            ue = torch.where(g != 0, -0.05 * g * torch.rsqrt(r[:, D:] + g * g), torch.zeros_like(g))
            kv.wait(kv.push(keys, torch.cat([ue, g * g], 1).contiguous().view(-1), True))

        t = alternate({"inplace": fused(False), "deterministic": fused(True), "pytorch": plain}, args.runs, 3)
        least = distinct * 2 * D * 4 * 2 / HBM_BYTES_PER_S
        for k, sec in t.items():
            print(json.dumps({"bench": "glove_step", "arm": k, "vocab": V, "d": d, "nnz_per_step": B,
                              "distinct_rows": distinct, "ms": round(sec * 1e3, 4),
                              "least_traffic_share": round(least / sec, 4), **info}), flush=True)
        kv.finalize()
        s.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--tokens", type=int, default=100_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--max_bytes", type=int, default=32 << 30)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--skip_torch", action="store_true", help="time only the device count")
    ap.add_argument("--only", choices=["cooc", "step"], default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("glove_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    if args.only in (None, "cooc"):
        bench_cooc(args, info)
    if args.only in (None, "step"):
        bench_step(args, info)


if __name__ == "__main__":
    main()
