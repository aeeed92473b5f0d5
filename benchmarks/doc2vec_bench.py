"""Paragraph-vector benchmark on one GPU: inference (``ops.doc2vec_infer``) against the same rule in PyTorch, and the
PV-DBOW / PV-DM training steps for context.

    python benchmarks/doc2vec_bench.py [--docs 65536] [--vocab 1000000] [--reps 20] [--torch_reps 5]

Inference: ``--docs`` documents of 100-300 Zipf words over a ``--vocab`` vocabulary, negative 5, 20 epochs, PV-DBOW and
PV-DM (window 5), d 100 and 300. The kernel arm is one ``doc2vec_infer`` call (one launch per epoch), timed with CUDA
events; the PyTorch arm runs the same rule in float32, vectorised over documents and sequential over positions, on rows
pulled once into a dense table (the pull is not timed; each epoch's draws are hashed on the device inside the arm).
The arms alternate within the run; each time is the median after one warm-up call. Row bytes are the rows the rule
reads (``1 + valid negatives`` targets per position, and for PV-DM its context rows), counted from the same hashes,
times ``4 d``, over the kernel time, against the
H100 SXM data sheet's 3.35 TB/s. Training: the fused skip-gram and CBOW steps at 32 768 pairs / 8 192 windows, d 300,
negative 5, with document keys in the batches. The card's name and power limit are printed with the results.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the name from torch still identifies the card
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def zipf_docs(n_docs, vocab, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(100, 301, n_docs)
    p = np.arange(1, vocab + 1, dtype=np.float64) ** -1.0
    cdf = np.cumsum(p / p.sum())
    tok = np.minimum(np.searchsorted(cdf, rng.random(int(lens.sum()))), vocab - 1).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return torch.from_numpy(tok), torch.from_numpy(off)


def _s64(x):
    return x - (1 << 64) if x >= 1 << 63 else x


def mix64_t(x):
    """hash.cuh's mix64 on int64 CUDA tensors (wrapping multiplies, logical shifts)"""
    x = x ^ ((x >> 33) & 0x7FFFFFFF)
    x = x * _s64(0xff51afd7ed558ccd)
    x = x ^ ((x >> 33) & 0x7FFFFFFF)
    x = x * _s64(0xc4ceb9fe1a85ec53)
    return x ^ ((x >> 33) & 0x7FFFFFFF)


def epoch_draws(base, e, Lmax, kw, sp):
    """the rule's [M, Lmax, neg] negatives and [M, Lmax] PV-DM radii of epoch e, on the device (alias tables only)"""
    dev = base.device
    neg, win = kw["negative"], kw["window"]
    es = mix64_t(base ^ ((1 << 62) | e))
    pos = torch.arange(Lmax, device=dev, dtype=torch.int64)
    n = pos[:, None] * neg + torch.arange(neg, device=dev)[None, :]
    h = mix64_t(es[:, None, None] ^ (n[None] * _s64(0x9E3779B97F4A7C15)))
    hi, lo = (h >> 32) & 0xFFFFFFFF, h & 0xFFFFFFFF
    i = (hi * sp.n) >> 32
    u = lo.to(torch.float32) * 2.0 ** -32
    draws = sp.first_key + torch.where(u < sp.prob[i], i, sp.alias[i].long()) * sp.key_stride
    hs = mix64_t(mix64_t(es)[:, None] ^ pos[None, :])
    r = win - torch.remainder(torch.remainder((hs >> 1) & 0x7FFFFFFFFFFFFFFF, win) * 2 + (hs & 1), win)  # unsigned mod
    return draws, r


def doc_base(kw, ids):
    from adapm_b200.ops import _doc2vec_base

    return torch.from_numpy(_doc2vec_base(kw["seed"], ids.numpy()).view(np.int64)).cuda()


def rows_read(tok, off, ids, sp, kw):
    """rows the rule reads over the call: valid targets per position, plus PV-DM's contexts"""
    dev = sp.prob.device
    lens = (off[1:] - off[:-1]).to(dev)
    Lmax = int(lens.max())
    offd, tokd = off.to(dev), tok.to(dev)
    pos = torch.arange(Lmax, device=dev)
    has = pos[None, :] < lens[:, None]
    words = torch.where(has, tokd[torch.clamp(offd[:-1, None] + pos[None, :], max=tok.numel() - 1)], 0)
    base = doc_base(kw, ids)
    total = 0
    for e in range(kw["epochs"]):
        draws, r = epoch_draws(base, e, Lmax, kw, sp)
        total += int((has[:, :, None] & (draws != 2 * words[:, :, None] + 1)).sum()) + int(has.sum())
        if kw["dm"]:
            C = torch.minimum(lens[:, None], pos[None, :] + r + 1) - torch.clamp(pos[None, :] - r, min=0) - 1
            total += int((C * has).sum())
    return total


def torch_rule(E_dense, tok, off, ids, sp, kw):
    """the rule in float32 PyTorch over a dense table of the rows (keys index it), vectorised over documents"""
    from adapm_b200.ops import doc2vec_initial_vectors

    dev = E_dense.device
    d, neg, win = kw["embed_dim"], kw["negative"], kw["window"]
    lens = (off[1:] - off[:-1]).to(dev)
    M, Lmax = lens.numel(), int(lens.max())
    v = torch.from_numpy(doc2vec_initial_vectors(kw["seed"], ids.numpy(), d)).to(dev)
    a = torch.full((M, d), 1e-6, device=dev)
    pos = torch.arange(Lmax, device=dev)
    has = pos[None, :] < lens[:, None]
    offd = off.to(dev)
    words = torch.where(has, tok.to(dev)[torch.clamp(offd[:-1, None] + pos[None, :], max=tok.numel() - 1)], 0)
    label = torch.zeros(1, 1 + neg, device=dev)
    label[0, 0] = 1
    loss = torch.zeros((), device=dev)
    base = doc_base(kw, ids)
    for e, ae in enumerate(kw["alphas"]):
        draws, radius = epoch_draws(base, e, Lmax, kw, sp)
        for i in range(Lmax):
            act = torch.nonzero(has[:, i]).view(-1)
            pk = 2 * words[act, i] + 1
            dr = draws[act, i]
            tk = torch.cat([pk[:, None], dr], 1)
            valid = torch.ones_like(tk, dtype=torch.bool)
            valid[:, 1:] = dr != pk[:, None]
            T = E_dense[tk]
            h = v[act]
            if kw["dm"]:
                r = radius[act, i]
                acc_h = h.clone()
                cnt = torch.ones(act.numel(), device=dev)
                for delta in range(-win, win + 1):
                    j = i + delta
                    if delta == 0 or j < 0 or j >= Lmax:
                        continue
                    m = (abs(delta) <= r) & has[act, j]
                    acc_h += torch.where(m[:, None], E_dense[2 * words[act, j]], 0.0)
                    cnt += m
                h = acc_h / cnt[:, None]
            f = torch.einsum("ad,atd->at", h, T)
            g = torch.where(f > 6, label - 1, torch.where(f < -6, label, label - torch.sigmoid(f))) * valid
            z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
            loss += (torch.log1p(torch.exp(-z)) * valid).sum()
            neu = torch.einsum("at,atd->ad", g, T)
            v[act] += ae * neu / torch.sqrt(a[act] + neu * neu)
            a[act] += neu * neu
    return v, loss


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def bench_inference(args, d, dm, results):
    import adapm_b200 as ad
    from adapm_b200.ops import DeviceSampler, _doc2vec_alphas, doc2vec_infer

    Vw, dev = args.vocab, torch.device("cuda", 0)
    kw = dict(dm=dm, embed_dim=d, negative=5, window=5, epochs=20, alpha=0.025, min_alpha=0.0001, seed=7)
    s = ad.Server(2 * d, num_keys=2 * Vw, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                  job=f"d2vb{d}{int(dm)}", device=0)
    kv = ad.Worker(0, s)
    g = torch.Generator(device="cuda").manual_seed(d)
    kv.begin_setup()
    for i in range(0, 2 * Vw, 1 << 18):
        k = torch.arange(i, min(2 * Vw, i + (1 << 18)), device=dev)
        rows = torch.ones(k.numel(), 2 * d, device=dev)
        rows[:, :d] = (torch.rand(k.numel(), d, generator=g, device=dev) - 0.5) * (2.0 / d ** 0.5)
        kv.wait(kv.set(k, rows.view(-1), True))
    kv.end_setup()
    counts = np.arange(1, Vw + 1, dtype=np.float64) ** -1.0 * 1e9
    sp = DeviceSampler(s, weights=torch.from_numpy(counts ** 0.75), first_key=1, key_stride=2)
    tok, off = zipf_docs(args.docs, Vw, 11)
    ids = torch.arange(args.docs, dtype=torch.int64)
    positions = int(tok.numel()) * kw["epochs"]
    n_rows = rows_read(tok, off, ids, sp, kw)
    tok_d, off_d, ids_d = tok.to(dev), off.to(dev), ids.to(dev)
    # the PyTorch arm: every row the documents can read, pulled once into a dense table indexed by key
    E_dense = torch.empty(2 * Vw, 2 * d, device=dev)
    kv.wait(kv.pull(torch.arange(2 * Vw, device=dev), E_dense.view(-1), True))
    E_dense = E_dense[:, :d].contiguous()
    kw_t = dict(kw, alphas=_doc2vec_alphas(kw["epochs"], kw["alpha"], kw["min_alpha"]))
    run_k = lambda: doc2vec_infer(s, tok_d, off_d, ids_d, sp, **kw)          # noqa: E731
    run_t = lambda: torch_rule(E_dense, tok, off, ids, sp, kw_t)              # noqa: E731
    vk, vt = run_k(), run_t()[0]
    err = float((vk - vt).abs().max())
    tk, tt = [], []
    for r in range(args.reps):
        tk.append(timed(run_k))
        if r < args.torch_reps:
            tt.append(timed(run_t))
    mk, mt = float(np.median(tk)), float(np.median(tt))
    res = dict(arm="inference", dm=int(dm), d=d, docs=args.docs, positions=positions, kernel_s=mk,
               kernel_range_s=[min(tk), max(tk)], kernel_reps=len(tk), torch_s=mt, torch_range_s=[min(tt), max(tt)],
               torch_reps=len(tt), docs_per_s=args.docs / mk, positions_per_s=positions / mk, speedup=mt / mk,
               rows_read=n_rows, row_bytes_per_s=n_rows * 4 * d / mk, share_of_hbm=n_rows * 4 * d / mk / HBM_BPS,
               max_abs_diff_vs_torch=err)
    print(json.dumps(res), flush=True)
    results.append(res)
    del E_dense
    kv.finalize()
    s.shutdown()


def bench_training(args, dm, results):
    import adapm_b200 as ad
    from adapm_b200.models.word2vec import Word2Vec, Word2VecConfig, zipf_counts

    V, d, D = 100000, 300, 100000
    cfg = Word2VecConfig(vocab_size=V, embed_dim=d, negative=5, window=5, batch_pairs=32768, batch_windows=8192,
                         cbow=bool(dm))
    s = ad.Server(2 * d, num_keys=2 * V + D, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                  job=f"d2vt{int(dm)}", device=0)
    kv = ad.Worker(0, s)
    m = Word2Vec(s, kv, cfg, zipf_counts(V))
    m.init_model()
    rng = np.random.default_rng(3)
    p = zipf_counts(V)
    cdf = np.cumsum(p / p.sum())
    dev = s.device

    def batch():
        if dm:
            w = np.minimum(np.searchsorted(cdf, rng.random((8192, 10))), V - 1)
            out = np.concatenate([2 * w[:, :1] + 1, 2 * V + rng.integers(0, D, (8192, 1)), 2 * w[:, 1:]], 1)
        else:
            w = np.minimum(np.searchsorted(cdf, rng.random(32768)), V - 1)
            out = np.stack([2 * V + rng.integers(0, D, 32768), 2 * w + 1])
        return torch.from_numpy(out.astype(np.int64)).to(dev)

    bs = [batch() for _ in range(4)]
    for b in bs:
        m.step_resident(b)
    ts = [timed(lambda: m.step_resident(bs[i % 4])) for i in range(args.reps)]
    res = dict(arm="training", dm=int(dm), d=d, step_s=float(np.median(ts)), range_s=[min(ts), max(ts)],
               items_per_step=8192 if dm else 32768)
    print(json.dumps(res), flush=True)
    results.append(res)
    kv.finalize()
    s.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--docs", type=int, default=65536)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--dims", default="100,300")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--torch_reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("doc2vec_bench needs a CUDA device")
    torch.cuda.set_device(0)
    print(f"card: {card()}", flush=True)
    results = []
    for d in (int(x) for x in args.dims.split(",")):
        for dm in (False, True):
            bench_inference(args, d, dm, results)
    for dm in (False, True):
        bench_training(args, dm, results)
    print(f"card: {card()}", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
