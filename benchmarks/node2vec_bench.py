"""node2vec on one GPU: walk generation, pair expansion, and their share of an epoch next to the skip-gram step.

The graph is R-MAT (``--scale`` 20, ``--edge-factor`` 16: 2^20 nodes and about 3.1 * 10^7 stored edges, both directions, with
power-law degrees and hubs), unweighted and with uniform (0, 1] weights. Measured:

    walks     ``ops.random_walks`` of one walk of 80 nodes from every node, for (p, q) = (1, 1) (the first-order kernel),
              (0.25, 4) and (4, 0.25). Reported: walk steps per second (steps actually taken; a walk from a node without
              edges takes none).
    torch     the same walks by a vectorised PyTorch implementation of the same rejection rule (``torch_walks``: per
              step, every pending walk draws a candidate and accepts it against alpha / alpha_max, with PyTorch's RNG).
    pairs     ``ops.walk_pairs`` of the unweighted (1, 1) walks at window 10, including its one host synchronisation.
              Reported: pairs per second.
    epoch     one chunk of ``--chunk`` walks as the model runs it: walks + pairs, then ``ops.sgns_step`` (d 128, 5
              negatives drawn by the device sampler) over the pairs in slices of 32768. Reported: the share of the
              chunk's time spent on walks and pairs.

Every number is the median of ``--runs`` (20) device-synchronised runs after a warm-up; the PyTorch walks, which take
seconds each at second order, are the median of ``--torch-runs`` (3). The JSON line carries the card's name
and power limit, read by ``nvidia-smi`` in the same run."""
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
from adapm_b200.ops import DeviceSampler, random_walks, sgns_step, walk_pairs, walk_thresholds  # noqa: E402
from adapm_b200.utils.graph import Graph, rmat_edges  # noqa: E402

PQ = [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power)}


def median_time(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def torch_walks(g, starts, L, p, q, gen):
    """node2vec walks in vectorised PyTorch with the kernels' rule (first-order draw, then acceptance against
    alpha / alpha_max), drawing with PyTorch's RNG"""
    off, nbr = g.offsets, g.neighbors.long()
    n = g.num_nodes
    deg = off[1:] - off[:-1]
    edge_key = torch.repeat_interleave(torch.arange(n, device=off.device), deg) * n + nbr
    if g.weighted:
        total = torch.zeros(n + 1, dtype=torch.int64, device=off.device)
        last = (off[1:] - 1).clamp(min=0)
        total[1:] = torch.cumsum(torch.where(deg > 0, g.cum_weights[last], 0), 0)
        glob = g.cum_weights + torch.repeat_interleave(total[:-1], deg)
    (t_ret, t_in, t_out), second = walk_thresholds(p, q)
    out = torch.full((starts.numel(), L), -1, dtype=torch.int64, device=off.device)
    out[:, 0] = starts
    v, t = starts.clone(), torch.full_like(starts, -1)
    alive = torch.arange(starts.numel(), device=off.device)
    for k in range(1, L):
        alive = alive[deg[v[alive]] > 0]
        if alive.numel() == 0:
            break
        x_new = torch.empty_like(alive)
        pend = torch.arange(alive.numel(), device=off.device)
        while pend.numel():
            w = alive[pend]
            vv = v[w]
            u = torch.rand(w.numel(), generator=gen, device=off.device, dtype=torch.float64)
            if g.weighted:
                tot = g.cum_weights[off[vv + 1] - 1]
                e = torch.searchsorted(glob, total[vv] + (u * tot).long(), right=True)
            else:
                e = off[vv] + (u * deg[vv]).long()
            x = nbr[e]
            if second and k >= 2:
                tt = t[w]
                key = tt * n + x
                pos = torch.searchsorted(edge_key, key).clamp(max=edge_key.numel() - 1)
                thr = torch.where(x == tt, t_ret, torch.where(edge_key[pos] == key, t_in, t_out))
                acc = torch.randint(0, 1 << 24, (w.numel(),), generator=gen, device=off.device) < thr
            else:
                acc = torch.ones_like(pend, dtype=torch.bool)
            x_new[pend[acc]] = x[acc]
            pend = pend[~acc]
        out[alive, k] = x_new
        t[alive] = v[alive]
        v[alive] = x_new
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edge-factor", type=int, default=16)
    ap.add_argument("--walk-length", type=int, default=80)
    ap.add_argument("--window", type=int, default=10)
    ap.add_argument("--chunk", type=int, default=65536, help="walks of the epoch-share chunk")
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--torch-runs", type=int, default=3, help="runs of the PyTorch walks, seconds each at second order")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    L, R, W = args.walk_length, args.runs, args.warmup
    res = {"bench": "node2vec", **card(), "scale": args.scale, "edge_factor": args.edge_factor, "walk_length": L,
           "runs": R, "walks": {}, "torch_walks": {}}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for weighted in (False, True):
        t0 = time.time()
        s, d, w = rmat_edges(args.scale, args.edge_factor, seed=1, weighted=weighted)
        g = Graph.from_edges(s, d, w, directed=False, num_nodes=1 << args.scale).to("cuda")
        del s, d, w
        res["nodes"], res["stored_edges"] = g.num_nodes, g.num_edges
        print(f"graph weighted={weighted}: {g.num_nodes} nodes, {g.num_edges} stored edges ({time.time() - t0:.1f}s "
              "on the host)", flush=True)
        starts = torch.arange(g.num_nodes, dtype=torch.int64)
        starts_dev = starts.cuda()
        for p, q in PQ:
            name = f"{'weighted' if weighted else 'unweighted'} p={p:g} q={q:g}"
            walks = random_walks(g, starts, 0, L, p, q, seed=7)
            steps = int((walks >= 0).sum()) - g.num_nodes
            t = median_time(lambda: random_walks(g, starts, 0, L, p, q, seed=7), R, W)
            tt = median_time(lambda: torch_walks(g, starts_dev, L, p, q, gen), args.torch_runs, 1)
            res["walks"][name] = {"steps": steps, "s": t, "steps_per_s": steps / t}
            res["torch_walks"][name] = {"s": tt, "steps_per_s": steps / tt, "device_speedup": tt / t}
            print(f"{name}: {steps / t / 1e6:.1f} M steps/s ({t * 1e3:.2f} ms), PyTorch {steps / tt / 1e6:.2f} M "
                  f"steps/s ({tt * 1e3:.1f} ms)", flush=True)
            if not weighted and p == 1.0:
                pairs = walk_pairs(walks, args.window, seed=3)
                tp = median_time(lambda: walk_pairs(walks, args.window, seed=3), R, W)
                res["pairs"] = {"pairs": int(pairs.shape[1]), "s": tp, "pairs_per_s": pairs.shape[1] / tp}
                print(f"pairs: {pairs.shape[1] / tp / 1e6:.1f} M pairs/s ({tp * 1e3:.2f} ms)", flush=True)
                del pairs
            del walks
        if not weighted:
            res["epoch"] = epoch_share(g, args, R, W)
        del g
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


def epoch_share(g, args, R, W):
    """walks + pairs of one chunk against sgns_step over its pairs (d 128, 5 negatives), for (1, 1) and (0.25, 4)"""
    d, neg, B = 128, 5, 32768
    n = g.num_nodes
    ad.setup(2 * n, 1)
    server = ad.Server(2 * d, num_keys=2 * n, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                       job=f"n2v_{os.getpid()}", device=0)
    kv = ad.Worker(0, server)
    try:
        for i in range(0, 2 * n, 1 << 18):
            k = torch.arange(i, min(2 * n, i + (1 << 18)), device="cuda")
            rows = torch.full((k.numel(), 2 * d), 1e-6, device="cuda")
            rows[:, :d] = (torch.rand(k.numel(), d, device="cuda") - 0.5) / d
            kv.wait(kv.set(k, rows.view(-1)))
        kv.waitall()
        deg = g.degrees().double().cpu()
        sampler = DeviceSampler(server, weights=deg.pow(0.75), first_key=1, key_stride=2)
        negs = torch.empty(B * neg, dtype=torch.int64, device="cuda")
        loss = torch.zeros(1, device="cuda")
        starts = torch.from_numpy(np.random.default_rng(2).permutation(n)[:args.chunk])
        out = {}
        for p, q in PQ[:2]:
            pairs = walk_pairs(random_walks(g, starts, 0, args.walk_length, p, q, seed=7), args.window, seed=3)
            P = pairs.shape[1] // B * B

            def gen():
                walk_pairs(random_walks(g, starts, 0, args.walk_length, p, q, seed=7), args.window, seed=3)

            def train():
                for i, b in enumerate(range(0, P, B)):
                    sampler.sample(B * neg, i, out=negs)
                    sgns_step(server, pairs[0, b:b + B], pairs[1, b:b + B], negs, d, 0.025, loss)

            tg, ts = median_time(gen, R, W), median_time(train, R, W)
            ts_all = ts * pairs.shape[1] / max(P, 1)
            key = f"p={p:g} q={q:g}"
            out[key] = {"walks": int(starts.numel()), "pairs": int(pairs.shape[1]), "walks_pairs_s": tg,
                        "sgns_s": ts_all, "walks_pairs_share": tg / (tg + ts_all)}
            print(f"epoch chunk {key}: walks + pairs {tg * 1e3:.2f} ms, sgns_step {ts_all * 1e3:.2f} ms over "
                  f"{pairs.shape[1]} pairs: walks + pairs take {100 * tg / (tg + ts_all):.1f} %", flush=True)
        return out
    finally:
        kv.finalize()
        server.shutdown()


if __name__ == "__main__":
    main()
