"""Fused top-k retrieval (ops_topk.cu) against the plain-PyTorch route, one GPU.

(a) word2vec nearest neighbours: a store of 2^20 keys with rows of 600 floats (d = 300 embedding + AdaGrad half),
    M in {1, 256, 4096} queries, k = 10, cosine (column scale 1/||e||), the query word excluded.
    fused   ``gather_gemm_topk`` straight from the store
    torch   pull all rows to a dense fp32 buffer, slice the embeddings to a bf16 matrix once, then per chunk of
            queries (scores <= 2 GB) ``q @ E.T`` (bf16) * scale, the query column set to -inf, ``torch.topk``;
            timed with the pull ("torch_with_pull_ms") and without it ("torch_ms")
(b) KGE link prediction at FB15k scale: 2048 queries x 14 951 entities x d = 512, k = 10, filtered (32 known answers
    per query).
    fused   ``gemm_nt_topk`` with the known answers as exclusions
    torch   ``gemm_nt_bf16`` (scores to HBM), scatter -inf at the known answers, ``torch.topk``

Times are CUDA events around each call, median of ``--iters`` (default 20) runs after 3 warm-up runs. Every JSON line
carries the device name and power limit of the card."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.ops import gather_gemm_topk, gemm_nt_bf16, gemm_nt_topk  # noqa: E402
from benchmarks.app_bench import device_info  # noqa: E402


def timed(fn, iters: int, warmup: int = 3) -> float:
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def word2vec_nn(info: dict, iters: int) -> None:
    nk, d, k = 1 << 20, 300, 10
    dev = torch.device("cuda:0")
    server = ad.Server(2 * d, num_keys=nk, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                       job=f"topkbench{os.getpid()}", device=0)
    kv = ad.Worker(0, server)
    g = torch.Generator(device=dev).manual_seed(1)
    for i in range(0, nk, 1 << 16):
        rows = torch.randn(1 << 16, 2 * d, device=dev, generator=g)
        kv.set(torch.arange(i, i + (1 << 16), device=dev), rows.view(-1))
    kv.waitall()
    keys = torch.arange(nk, device=dev)
    dense = torch.empty(nk * 2 * d, dtype=torch.float32, device=dev)

    def pull_dense():
        kv.wait(kv.pull(keys, dense, True))
        return dense.view(nk, 2 * d)[:, :d].to(torch.bfloat16)

    E = pull_dense()
    scale = 1.0 / E.float().norm(dim=1)
    chunk = max(1, (2 << 30) // (4 * nk))              # fp32 scores of one chunk <= 2 GB

    def torch_route(E, q, words):
        vals, idx = [], []
        qb = q.to(torch.bfloat16)
        for c in range(0, q.shape[0], chunk):
            s = (qb[c:c + chunk] @ E.t()).float() * scale
            s.scatter_(1, words[c:c + chunk].view(-1, 1), float("-inf"))
            v, i = torch.topk(s, k, dim=1)
            vals.append(v); idx.append(i)
        return torch.cat(vals), torch.cat(idx)

    for M in (1, 256, 4096):
        words = torch.randint(0, nk, (M,), device=dev, generator=g)
        q = E[words].float() * scale[words].view(-1, 1)
        excl = (torch.arange(M + 1, dtype=torch.int64, device=dev), words.contiguous())
        fused = lambda: gather_gemm_topk(server, q, keys, d, k, exclude=excl, col_scale=scale)  # noqa: E731
        t_fused = timed(fused, iters)
        t_torch = timed(lambda: torch_route(E, q, words), iters)
        t_pull = timed(lambda: torch_route(pull_dense(), q, words), iters)
        fi = fused()[1]
        ti = torch_route(E, q, words)[1]
        agree = float((fi == ti).float().mean())
        print(json.dumps({"bench": "word2vec_nearest_neighbours", "keys": nk, "d": d, "M": M, "k": k,
                          "fused_ms": round(t_fused, 4), "torch_ms": round(t_torch, 4),
                          "torch_with_pull_ms": round(t_pull, 4), "speedup_vs_torch": round(t_torch / t_fused, 3),
                          "speedup_vs_torch_with_pull": round(t_pull / t_fused, 3),
                          "same_index_fraction": round(agree, 4), **info}), flush=True)
    del dense, E
    kv.finalize(); server.shutdown()


def kge_link_prediction(info: dict, iters: int) -> None:
    M, N, K, k, n_known = 2048, 14951, 512, 10, 32
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(2)
    q = torch.randn(M, K, device=dev, generator=g)
    e = torch.randn(N, K, device=dev, generator=g)
    cols = torch.sort(torch.randint(0, N, (M, n_known), device=dev, generator=g), dim=1).values
    mask = torch.zeros(M, N, dtype=torch.bool, device=dev)
    mask.scatter_(1, cols, True)
    off = torch.zeros(M + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(mask.sum(1), 0)
    excl = (off, mask.nonzero()[:, 1].contiguous())
    q16, e16 = q.to(torch.bfloat16), e.to(torch.bfloat16)

    def torch_route():
        s = gemm_nt_bf16(q16, e16)
        s.masked_fill_(mask, float("-inf"))
        return torch.topk(s, k, dim=1)

    fused = lambda: gemm_nt_topk(q16, e16, k, exclude=excl)  # noqa: E731
    t_fused = timed(fused, iters)
    t_torch = timed(torch_route, iters)
    same = float((fused()[1] == torch_route().indices).float().mean())
    print(json.dumps({"bench": "kge_link_prediction_filtered", "M": M, "N": N, "d": K, "k": k,
                      "known_per_query": n_known, "fused_ms": round(t_fused, 4), "torch_ms": round(t_torch, 4),
                      "speedup_vs_torch": round(t_torch / t_fused, 3), "same_index_fraction": round(same, 4),
                      **info}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", choices=("word2vec", "kge"), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("topk_bench needs a CUDA device")
    torch.cuda.set_device(0)
    info = device_info()
    if args.only in (None, "kge"):
        kge_link_prediction(info, max(20, args.iters))
    if args.only in (None, "word2vec"):
        word2vec_nn(info, max(20, args.iters))


if __name__ == "__main__":
    main()
