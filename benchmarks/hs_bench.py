"""word2vec hierarchical softmax on the parameter store, one GPU: ``ops.hs_step`` deterministic (index, score, group,
gather, finish) and in place (one kernel), against negative sampling on the same batches and against a pull + PyTorch +
push route of the hierarchical-softmax rule.

Shape: 1M Zipf words (2M keys), d 300; skip-gram at 32 768 pairs per step (``SyntheticPairs``) and CBOW at 8 192
windows of radius 5 per step (``SyntheticWindows``). Negative sampling runs ``ops.sgns_step`` (skip-gram) or
``ops.cbow_step`` (CBOW) with 25 negatives; on one GPU both are deterministic, as is ``hs_step`` by default. Reported per
arm: device-timed ms per step, the distinct output (syn1) rows and all distinct rows the step touches, and the
least-HBM-traffic share: every distinct row read once and written once (2 x 2400 bytes) at 3.35 TB/s, over the step
time. The step is bounded by memory bandwidth (a few flops per row byte), so that share is its share of peak.

Every number is the median of ``--iters`` (>= 20) CUDA-event-timed steps after ``--warmup`` steps, the arms alternating
on the same batches in one process; the JSON lines carry the card's name, power limit and maximum SM clock, read by
``nvidia-smi`` in the same run. Two host-side times are reported too (CPU, not GPU, numbers): building the 1M-word
Huffman tree, and expanding one skip-gram batch's syn1 words into the path-node keys that ``Word2Vec.signal_intent``
hands to Intent.

    python benchmarks/hs_bench.py [--iters 20] [--warmup 5]
"""
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
from adapm_b200.models.word2vec import (SyntheticPairs, SyntheticWindows, Word2Vec, Word2VecConfig,  # noqa: E402
                                        zipf_counts)
from adapm_b200.ops import DeviceSampler, cbow_step, hs_step, sgns_step  # noqa: E402
from adapm_b200.utils.text import huffman_tree  # noqa: E402

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


def path_keys(tree, c):
    """[B, max_len] syn1 keys of the path nodes of the items' centres (-1 past a path's end or for c < 0)"""
    L = tree.max_len
    w = torch.where(c >= 0, c // 2, torch.zeros_like(c))
    j = torch.arange(L, device=c.device)
    m = (c >= 0).view(-1, 1) & (j.view(1, L) < (tree.offsets[w + 1] - tree.offsets[w]).view(-1, 1))
    idx = torch.where(m, tree.offsets[w].view(-1, 1) + j, torch.zeros_like(m, dtype=torch.int64))
    return torch.where(m, 2 * tree.nodes[idx].long() + 1, -1), w


def torch_route(kv, tree, c, x, d, alpha):
    """pull the step's rows, the hierarchical-softmax rule in fp32 PyTorch on the GPU, push the updates"""
    B, C = x.shape
    tk, w = path_keys(tree, c)
    L = tk.shape[1]
    keys = torch.cat([x.reshape(-1), tk.reshape(-1)])
    keys = keys[keys >= 0]
    uk = torch.unique(keys)
    rows = torch.empty(uk.numel() * 2 * d, device=c.device)
    kv.wait(kv.pull(uk, rows, True))
    rows = rows.view(-1, 2 * d)
    xm, tm = x >= 0, tk >= 0
    pos = torch.searchsorted(uk, x.clamp(min=0))
    tpos = torch.searchsorted(uk, tk.clamp(min=0))
    h = (rows[pos, :d] * xm.unsqueeze(-1)).sum(1) / xm.sum(1, keepdim=True).clamp(min=1)
    et, at = rows[tpos, :d], rows[tpos, d:]
    label = (1 - ((tree.codes[w].view(B, 1) >> torch.arange(L, device=c.device, dtype=torch.int32)) & 1)).float()
    f = (h.unsqueeze(1) * et).sum(-1)
    um = tm & (f.abs() < 6)
    g = (label - torch.sigmoid(f)) * um
    neu = (g.unsqueeze(-1) * et).sum(1)
    gt = g.unsqueeze(-1) * h.unsqueeze(1)
    ut = torch.cat([alpha * gt / torch.sqrt(at + gt * gt), gt * gt], -1)[um]
    gx = neu.unsqueeze(1).expand(B, C, d)[xm]
    ax = rows[pos[xm], d:]
    ux = torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)
    kv.wait(kv.push(torch.cat([tk[um], x[xm]]), torch.cat([ut, ux]).contiguous().view(-1), True))


def host_times(counts, cfg):
    """host ms: the Huffman tree of the vocabulary; expanding one skip-gram batch into its intent keys (median of 20)"""
    t = time.perf_counter()
    huffman_tree(counts)
    tree_ms = (time.perf_counter() - t) * 1e3
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                       fabric="inproc", job=f"hs_bench_host{os.getpid()}")
    kv = ad.Worker(0, server)
    hcfg = Word2VecConfig(vocab_size=cfg.vocab_size, embed_dim=4, negative=0, hs=True, batch_pairs=cfg.batch_pairs)
    model = Word2Vec(server, kv, hcfg, counts)
    data = SyntheticPairs(hcfg, counts, 0)
    ts = []
    for s in range(20):
        b = data.batch(s)
        t = time.perf_counter()
        model.intent_keys_hs(b.reshape(-1))
        ts.append((time.perf_counter() - t) * 1e3)
    kv.finalize()
    server.shutdown()
    return {"tree_build_host_ms": round(tree_ms, 1), "intent_keys_host_ms": round(float(np.median(ts)), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--negative", type=int, default=25)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--batch_pairs", type=int, default=32768)
    ap.add_argument("--batch_windows", type=int, default=8192)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("hs_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    info = card()
    cfg = Word2VecConfig(vocab_size=args.vocab, embed_dim=args.dim, negative=args.negative, window=args.window,
                         batch_pairs=args.batch_pairs, batch_windows=args.batch_windows)
    d = cfg.embed_dim
    counts = zipf_counts(cfg.vocab_size)
    host = host_times(counts, cfg)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"hs_bench{os.getpid()}", device=0)
    kv = ad.Worker(0, server)
    dev = server.device
    for a in range(0, cfg.num_keys, 1 << 20):
        k = torch.arange(a, min(cfg.num_keys, a + (1 << 20)), device=dev)
        rows = torch.rand(k.numel(), 2 * d, device=dev) * (1.0 / d) - 0.5 / d
        rows[:, d:] = 1e-3
        kv.wait(kv.set(k, rows.view(-1), True))
    kv.waitall()
    tree = huffman_tree(counts).to(dev)
    sampler = DeviceSampler(server, weights=torch.from_numpy(np.power(counts, 0.75)), first_key=1, key_stride=2)
    n_batches = 8
    loss = torch.zeros(1, device=dev)
    for mode in ("skipgram", "cbow"):
        batches = []
        for s in range(n_batches):
            if mode == "cbow":
                wb = SyntheticWindows(cfg, counts, 0).batch(s).to(dev)
                c, x = wb[:, 0].contiguous(), wb[:, 1:].contiguous()
            else:
                pb = SyntheticPairs(cfg, counts, 0).batch(s).to(dev)
                c, x = pb[1].contiguous(), pb[0].contiguous().view(-1, 1)   # the syn1 word's path, one context
            n = sampler.sample(c.numel() * cfg.negative, seed=s).view(c.numel(), cfg.negative)
            tk, _ = path_keys(tree, c)
            hs_out = torch.unique(tk[tk >= 0])
            ns_out = torch.unique(torch.cat([c, n.reshape(-1)]))
            xs = torch.unique(x[x >= 0])
            batches.append({"c": c, "x": x, "n": n,
                            "rows": {"hs": hs_out.numel() + xs.numel(), "ns": ns_out.numel() + xs.numel()},
                            "out_rows": {"hs": hs_out.numel(), "ns": ns_out.numel()}})
        stats = {k: torch.zeros(4, dtype=torch.int64, device=dev) for k in ("hs_det", "hs_inplace", "ns")}
        state = {"i": 0}

        def arm(name):
            def run():
                b = batches[state["i"] % n_batches]
                if name == "hs_det":
                    hs_step(server, b["c"], b["x"], tree, d, 0.001, loss, stats[name])
                elif name == "hs_inplace":
                    hs_step(server, b["c"], b["x"], tree, d, 0.001, loss, stats[name], deterministic=False)
                elif name == "ns" and mode == "cbow":
                    cbow_step(server, b["c"], b["x"], b["n"], d, 0.001, loss, stats[name])
                elif name == "ns":
                    sgns_step(server, b["x"].view(-1), b["c"], b["n"], d, 0.001, loss, stats[name])
                else:
                    torch_route(kv, tree, b["c"], b["x"], d, 0.001)
            return run

        arms = {k: arm(k) for k in ("hs_det", "hs_inplace", "ns", "torch")}
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
        row_bytes = 2 * d * 4
        items = args.batch_windows if mode == "cbow" else args.batch_pairs
        out = {"bench": "hs", "mode": mode, **info, **host, "vocab": args.vocab, "dim": d, "items_per_step": items,
               "max_len": tree.max_len, "negative": args.negative, "iters": args.iters,
               "bound": "HBM bandwidth"}
        for k in ("hs_det", "hs_inplace", "ns", "torch"):
            t = float(np.median(ts[k])) / 1e3
            kind = "ns" if k == "ns" else "hs"
            r = float(np.mean([b["rows"][kind] for b in used]))
            o = float(np.mean([b["out_rows"][kind] for b in used]))
            e = {"ms_per_step": round(t * 1e3, 4), "output_rows": round(o), "rows": round(r),
                 "least_hbm_share": round(2 * r * row_bytes / HBM_BPS / t, 4)}
            if k in stats:
                e["updates_per_s"] = round(stats[k][3].item() / args.iters / t)
            out[k] = e
        print(json.dumps(out), flush=True)
    kv.finalize()
    server.shutdown()


if __name__ == "__main__":
    main()
