"""word2vec CBOW on the parameter store, one GPU: ``ops.cbow_step`` deterministic (index, score, group, gather,
finish) and in place (one kernel), against skip-gram on the same windows and against a pull + PyTorch + push route.

Shape: 1M words (2M keys), d 300, 25 negatives, window 5, 8 192 windows per step drawn like the loader's
(``SyntheticWindows``: Zipf words, windows shrunk by b uniform in [0, 5)). Reported per variant: device-timed ms per
step, corpus words per second (one window per corpus word), updates per second (pushes, read from stats[3]) and the
least-HBM-traffic share: every distinct row of the step read once and written once (2 x 2400 bytes) at 3.35 TB/s, over
the step time. Skip-gram runs ``ops.sgns_step`` (deterministic on one GPU) on the same windows expanded into
(context, centre) pairs: the same corpus words.

Every number is the median of ``--iters`` (>= 20) CUDA-event-timed steps after ``--warmup`` steps, the variants
alternating in one process; the JSON line carries the card's name, power limit and maximum SM clock, read by
``nvidia-smi`` in the same run.

    python benchmarks/cbow_bench.py [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.word2vec import SyntheticWindows, Word2VecConfig, zipf_counts  # noqa: E402
from adapm_b200.ops import DeviceSampler, cbow_step, sgns_step  # noqa: E402

HBM_BPS = 3.35e12


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


def torch_route(kv, c, x, n, d, alpha):
    """pull the step's rows, the CBOW rule in fp32 PyTorch on the GPU, push the updates"""
    B, C = x.shape
    keys = torch.cat([x.reshape(-1), c, n.reshape(-1)])
    keys = keys[keys >= 0]
    uk, inv = torch.unique(keys, return_inverse=True)
    rows = torch.empty(uk.numel() * 2 * d, device=c.device)
    kv.wait(kv.pull(uk, rows, True))
    rows = rows.view(-1, 2 * d)
    pos = torch.full((B * C,), -1, dtype=torch.int64, device=c.device)
    xm = x.reshape(-1) >= 0
    pos[xm] = inv[:int(xm.sum())]
    pos = pos.view(B, C)
    tk = torch.cat([c.view(B, 1), n], 1)
    tpos = torch.searchsorted(uk, tk)
    m = (pos >= 0).unsqueeze(-1)
    h = (rows[pos.clamp(min=0), :d] * m).sum(1) / m.sum(1).clamp(min=1)
    et, at = rows[tpos, :d], rows[tpos, d:]
    label = torch.zeros(B, tk.shape[1], device=c.device)
    label[:, 0] = 1
    valid = torch.ones_like(label, dtype=torch.bool)
    valid[:, 1:] = n != c.view(B, 1)
    f = (h.unsqueeze(1) * et).sum(-1)
    g = torch.where(f > 6, label - 1, torch.where(f < -6, label, label - torch.sigmoid(f))) * valid
    neu = (g.unsqueeze(-1) * et).sum(1)
    gt = g.unsqueeze(-1) * h.unsqueeze(1)
    ut = torch.cat([alpha * gt / torch.sqrt(at + gt * gt), gt * gt], -1)[valid]
    gx = neu.unsqueeze(1).expand(B, C, d)[pos >= 0]
    ax = rows[pos[pos >= 0], d:]
    ux = torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)
    kv.wait(kv.push(torch.cat([tk[valid], x[pos >= 0]]), torch.cat([ut, ux]).contiguous().view(-1), True))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--negative", type=int, default=25)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--batch_windows", type=int, default=8192)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cbow_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    cfg = Word2VecConfig(vocab_size=args.vocab, embed_dim=args.dim, negative=args.negative, window=args.window,
                         batch_windows=args.batch_windows, cbow=True)
    d = cfg.embed_dim
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"cbow_bench{os.getpid()}", device=0)
    kv = ad.Worker(0, server)
    dev = server.device
    counts = zipf_counts(cfg.vocab_size)
    for a in range(0, cfg.num_keys, 1 << 20):
        k = torch.arange(a, min(cfg.num_keys, a + (1 << 20)), device=dev)
        rows = torch.rand(k.numel(), 2 * d, device=dev) * (1.0 / d) - 0.5 / d
        rows[:, d:] = 1e-3
        kv.wait(kv.set(k, rows.view(-1), True))
    kv.waitall()
    sampler = DeviceSampler(server, weights=torch.from_numpy(np.power(counts, 0.75)), first_key=1, key_stride=2)
    data = SyntheticWindows(cfg, counts, 0)
    n_batches = 8
    batches = []
    for s in range(n_batches):
        w = data.batch(s).to(dev)
        c, x = w[:, 0].contiguous(), w[:, 1:].contiguous()
        n = sampler.sample(c.numel() * cfg.negative, seed=s).view(c.numel(), cfg.negative)
        m = x >= 0
        pairs = (x[m].contiguous(), c.view(-1, 1).expand_as(x)[m].contiguous())
        pn = sampler.sample(pairs[0].numel() * cfg.negative, seed=1000 + s).view(-1, cfg.negative)
        keys = torch.cat([x[m], c, n.reshape(-1)])
        batches.append({"c": c, "x": x, "n": n, "pairs": pairs, "pn": pn, "rows": int(torch.unique(keys).numel()),
                        "pair_rows": int(torch.unique(torch.cat([pairs[0], pairs[1], pn.reshape(-1)])).numel())})
    loss = torch.zeros(1, device=dev)
    stats = {k: torch.zeros(4, dtype=torch.int64, device=dev) for k in ("det", "inplace", "sgns")}
    state = {"i": 0}

    def arm(name):
        def run():
            b = batches[state["i"] % n_batches]
            if name == "det":
                cbow_step(server, b["c"], b["x"], b["n"], d, 0.001, loss, stats["det"])
            elif name == "inplace":
                cbow_step(server, b["c"], b["x"], b["n"], d, 0.001, loss, stats["inplace"], deterministic=False)
            elif name == "sgns":
                sgns_step(server, b["pairs"][0], b["pairs"][1], b["pn"], d, 0.001, loss, stats["sgns"])
            else:
                torch_route(kv, b["c"], b["x"], b["n"], d, 0.001)
        return run

    arms = {k: arm(k) for k in ("det", "inplace", "sgns", "torch")}
    for _ in range(args.warmup):
        for fn in arms.values():
            fn()
        state["i"] += 1
    torch.cuda.synchronize()
    for s in stats.values():
        s.zero_()
    ts = {k: [] for k in arms}
    used = []
    for _ in range(args.iters):
        used.append(batches[state["i"] % n_batches])
        for k, fn in arms.items():
            ts[k].append(timed(fn))
        state["i"] += 1
    ms = {k: float(np.median(v)) for k, v in ts.items()}
    words = args.batch_windows                      # one window per corpus word (the synthetic batches are full)
    rows = float(np.mean([b["rows"] for b in used]))
    pair_rows = float(np.mean([b["pair_rows"] for b in used]))
    row_bytes = 2 * d * 4
    out = {"bench": "cbow", **info, "vocab": args.vocab, "dim": d, "negative": args.negative, "window": args.window,
           "batch_windows": words, "pairs_per_step": float(np.mean([b["pairs"][0].numel() for b in used])),
           "iters": args.iters}
    for k in ("det", "inplace", "sgns"):
        t = ms[k] / 1e3
        upd = stats[k][3].item() / args.iters
        r = pair_rows if k == "sgns" else rows
        out[k] = {"ms_per_step": round(ms[k], 4), "words_per_s": round(words / t), "updates_per_s": round(upd / t),
                  "least_hbm_share": round(2 * r * row_bytes / HBM_BPS / t, 4)}
    out["torch"] = {"ms_per_step": round(ms["torch"], 4), "words_per_s": round(words / (ms["torch"] / 1e3))}
    print(json.dumps(out), flush=True)
    kv.finalize()
    server.shutdown()


if __name__ == "__main__":
    main()
