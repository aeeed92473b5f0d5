"""Alternating least squares on the parameter store, one GPU: ``ops.als_solve`` and ``ops.als_gram`` (implicit loss).

Seeded data with heavy-tailed entry counts on both sides (users and items drawn from power laws, repeats kept as
entries): the MovieLens-20M shape (138 493 users x 26 744 items, 20 M entries, longest item about 67 000 entries) and
10^6 users x 10^5 items with 5 * 10^7 entries, at ranks 64 and 128. Reported per shape and rank:
  - ms per user half-step, per item half-step and per Gram matrix (median of ``--iters`` CUDA-event-timed runs);
  - the achieved FP32 rate against the H100 SXM's 67 TFLOP/s, counting ``sum_t (2 n_t k^2 + k^3 / 3 + 4 k^2)``;
  - the longest single target solved alone (one CTA): how long a CTA holds the sync round's grace period at most;
  - the same half-step by pull + PyTorch (count-bucketed padded ``bmm``, batched ``cholesky`` / ``cholesky_solve``,
    push), median of 3;
  - one BPR epoch over the same entries (``ops.mf_bpr_step``, 65 536 positives and one negative each, in place), for
    scale.
Each JSON line carries the card's name and power limit, read by ``nvidia-smi`` in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.mf import MFConfig  # noqa: E402
from adapm_b200.ops import als_gram, als_solve, mf_bpr_step  # noqa: E402

SHAPES = {"ml20m": (138493, 26744, 20_000_000, 67_000, 9_000), "large": (1_000_000, 100_000, 50_000_000, 300_000, 20_000)}
FP32_FLOPS = 67e12
LAM, ALPHA = 0.1, 1.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power)}


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def power_law(n, draws, top, g, dev):
    """draws indices of [0, n) with p_i ~ (i + 1)^-s, s chosen so that index 0 gets about `top` draws; the indices
    are shuffled so that popularity is not ordered by id"""
    lo, hi = 0.0, 2.0
    i = torch.arange(1, n + 1, dtype=torch.float64)
    for _ in range(50):
        s = (lo + hi) / 2
        p = i ** -s
        if float(p[0] / p.sum()) * draws < top:
            lo = s
        else:
            hi = s
    cdf = torch.cumsum(i ** -s, 0)
    cdf = (cdf / cdf[-1]).to(dev)
    idx = torch.searchsorted(cdf, torch.rand(draws, generator=g, device=dev, dtype=torch.float64))
    return torch.randperm(n, generator=g, device=dev)[idx.clamp_(max=n - 1)]


def side(t_idx, o_keys, n_t, first_t):
    """CSR of one side, longest target first: (targets, offsets, others, a, b) with x = 1 (implicit)"""
    cnt = torch.bincount(t_idx, minlength=n_t)
    order_t = torch.argsort(-cnt, stable=True)
    pos = torch.empty_like(order_t)
    pos[order_t] = torch.arange(n_t, device=t_idx.device)
    order = torch.argsort(pos[t_idx], stable=True)
    off = torch.zeros(n_t + 1, dtype=torch.int64, device=t_idx.device)
    off[1:] = torch.cumsum(cnt[order_t], 0)
    nnz = t_idx.numel()
    a = torch.full((nnz,), ALPHA, device=t_idx.device)
    return order_t + first_t, off, o_keys[order].contiguous(), a, a + 1.0


def raw_solve(server, sd, k, G):
    """``als_solve`` without the wrapper's argument checks (they synchronise with the host): the kernel alone"""
    t, off, o, a, b = sd
    ad._C.als_solve(server._impl.backend_handle(), torch.cuda.current_stream().cuda_stream, t.data_ptr(), off.data_ptr(),
                    o.data_ptr(), a.data_ptr(), b.data_ptr(), t.numel(), k, LAM, G.data_ptr(), 0)


def flops(off, k):
    n = (off[1:] - off[:-1]).double()
    return float((2 * n * k * k + k ** 3 / 3 + 4 * k * k).sum())


def torch_half_step(kv, server, t, off, o, a, b, k, G, other_keys, budget=1 << 27):
    """the same half-step by pull + PyTorch: every other-side row pulled once, targets bucketed by entry count (powers
    of two), padded bmm, batched Cholesky, push of [w_new - w_old | 0]"""
    dev = server.device
    H = torch.empty(other_keys.numel() * 2 * k, device=dev)
    kv.wait(kv.pull(other_keys, H, True))
    H = H.view(-1, 2 * k)[:, :k]
    o = o - other_keys[0]
    W = torch.empty(t.numel() * 2 * k, device=dev)
    kv.wait(kv.pull(t, W, True))
    W = W.view(-1, 2 * k)[:, :k]
    cnt = off[1:] - off[:-1]
    bucket = torch.ceil(torch.log2(cnt.clamp(min=1).double())).long()
    upd = torch.zeros(t.numel(), 2 * k, device=dev)
    base = G + LAM * torch.eye(k, device=dev)
    for bk in torch.unique(bucket).tolist():
        sel = (bucket == bk).nonzero().squeeze(1)
        L = 1 << bk
        step = max(1, budget // (L * k))
        for s in range(0, sel.numel(), step):
            ts = sel[s:s + step]
            j = torch.arange(L, device=dev)
            idx = off[ts, None] + j
            m = j < cnt[ts, None]
            idx = torch.where(m, idx, 0)
            Hp = H[o[idx]] * m[..., None]
            A = base + torch.bmm(Hp.transpose(1, 2) * a[idx][:, None, :] * m[:, None, :], Hp)
            r = torch.bmm((b[idx] * m)[:, None, :], Hp).squeeze(1)
            x = torch.cholesky_solve(r[..., None], torch.linalg.cholesky(A)).squeeze(-1)
            upd[ts, :k] = x - W[ts]
    kv.wait(kv.push(t, upd.view(-1), True))


def run(name, k, iters, warmup, info):
    users, items, nnz, top_item, top_user = SHAPES[name]
    cfg = MFConfig(num_rows=users, num_cols=items, rank=k)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"als_bench{os.getpid()}_{name}_{k}", device=0)
    kv = ad.Worker(0, server)
    dev = server.device
    g = torch.Generator(device=dev).manual_seed(users + k)
    fck = cfg.first_col_key(1)
    for s in range(0, cfg.num_keys(1), 1 << 20):
        keys = torch.arange(s, min(cfg.num_keys(1), s + (1 << 20)), device=dev)
        rows = torch.zeros(keys.numel(), 2 * k, device=dev)
        rows[:, :k] = torch.rand(keys.numel(), k, generator=g, device=dev) / k ** 0.5
        kv.wait(kv.set(keys, rows.view(-1)))
    kv.waitall()
    ui = power_law(users, nnz, top_user, g, dev)
    ij = power_law(items, nnz, top_item, g, dev)
    user_side = side(ui, ij + fck, users, 0)
    item_side = side(ij, ui, items, fck)
    user_keys = torch.arange(users, device=dev)
    item_keys = torch.arange(items, device=dev) + fck
    torch.cuda.synchronize()
    als_solve(server, *user_side, k, LAM, als_gram(server, item_keys, k))     # the checked op once per side
    als_solve(server, *item_side, k, LAM, als_gram(server, user_keys, k))
    G_items = als_gram(server, item_keys, k)
    G_users = als_gram(server, user_keys, k)
    out = dict(info, shape=name, users=users, items=items, nnz=nnz, rank=k,
               longest_user=int((user_side[1][1] - user_side[1][0]).item()),
               longest_item=int((item_side[1][1] - item_side[1][0]).item()))
    ms = {
        "gram_items_ms": median_ms(lambda: als_gram(server, item_keys, k), iters, warmup),
        "gram_users_ms": median_ms(lambda: als_gram(server, user_keys, k), iters, warmup),
        "user_half_step_ms": median_ms(lambda: raw_solve(server, user_side, k, G_items), iters, warmup),
        "item_half_step_ms": median_ms(lambda: raw_solve(server, item_side, k, G_users), iters, warmup),
    }
    out.update(ms)
    for s, key, other in ((user_side, "user", item_keys), (item_side, "item", user_keys)):
        f = flops(s[1], k)
        out[f"{key}_tflops"] = f / (ms[f"{key}_half_step_ms"] * 1e-3) / 1e12
        out[f"{key}_share_of_67tflops"] = out[f"{key}_tflops"] * 1e12 / FP32_FLOPS
        t, off, o, a, b = s
        n0 = int(off[1])
        one = (t[:1].contiguous(), off[:2].contiguous(), o[:n0].contiguous(), a[:n0].contiguous(), b[:n0].contiguous())
        G = G_items if key == "user" else G_users
        out[f"longest_{key}_alone_ms"] = median_ms(lambda: raw_solve(server, one, k, G), iters, warmup)
        out[f"{key}_half_step_pytorch_ms"] = median_ms(lambda: torch_half_step(kv, server, *s, k, G, other), 3, 1)
    # BPR epoch over the same entries, for scale
    loss = torch.zeros(1, device=dev)
    B = 65536
    perm = torch.randperm(nnz, generator=g, device=dev)
    uk, ik = ui[perm].contiguous(), (ij[perm] + fck).contiguous()
    negs = (torch.randint(0, items, (nnz, 1), generator=g, device=dev) + fck).contiguous()

    def bpr_epoch():
        for s0 in range(0, nnz, B):
            mf_bpr_step(server, uk[s0:s0 + B], ik[s0:s0 + B], negs[s0:s0 + B], k, 0.01, 0.01, loss)

    out["bpr_epoch_ms"] = median_ms(bpr_epoch, 3, 1)
    print(json.dumps(out), flush=True)
    kv.finalize()
    server.shutdown()
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="ml20m,large")
    ap.add_argument("--ranks", default="64,128")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("als_bench needs a CUDA device")
    info = card()
    for name in args.shapes.split(","):
        for k in (int(r) for r in args.ranks.split(",")):
            run(name, k, args.iters, args.warmup, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
