"""Multi-hot embedding bags on the parameter store (ops_embbag.cu) against the torch route, one GPU.

    fused   ``StoreEmbeddingBag(impl="fused")``: one pooled-gather kernel that reads the rows through the directory; the
            backward sorts (key, position), sums each key's gradient in position order and pushes one AdaGrad update
            per distinct key (four launches)
    torch   ``StoreEmbeddingBag(impl="torch")`` on the same CUDA store: ``torch.unique`` -> ``worker.pull`` ->
            ``F.embedding_bag`` -> autograd -> AdaGrad -> ``worker.push`` (the CPU-server path, run on CUDA tensors)

Shapes (bag lengths uniform in [1, L], ids skewed within each field as in the CTR app):
    deepfm     B = 8192, F = 26, L = 8, E = 20, 10^8 keys
    dlrm       B = 2048, F = 26, L = 32, E = 128, 10^7 keys
    single     B = 8192, F = 26, L = 1, E = 20, 10^8 keys
and one full multi-hot DeepFM step (the deepfm shape, MLP 400x3, bf16 tensor-core MLP).

Each row: median of ``--iters`` (default 20) runs after ``--warmup`` runs, CUDA events around the work and a
synchronize; the two routes alternate on the same seeded batches in one process. ``fwd`` is the forward alone,
``step`` forward + backward (the update lands in the store). Bytes/s of the forward are computed from its lower bound
nnz * E * 4 read + nbags * E * 4 written and compared with the H100 SXM data-sheet HBM3 rate (3.35 TB/s), which is a
data-sheet figure, not a measurement. Every JSON line carries the device name and power limit of the card."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.ops import StoreEmbeddingBag  # noqa: E402
from benchmarks.app_bench import device_info  # noqa: E402

HBM_DATASHEET_BPS = 3.35e12


def median_ms(fn, iters: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def batch(seed: int, B: int, F: int, L: int, num_keys: int, dev):
    rng = np.random.default_rng([seed, B, F, L])
    lens = rng.integers(1, L + 1, size=B * F)
    bag = np.repeat(np.arange(B * F, dtype=np.int64), lens)
    per = num_keys // F
    local = np.minimum((per * rng.random(bag.size) ** 3).astype(np.int64), per - 1)
    keys = torch.from_numpy(local + (bag % F) * per).to(dev)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).to(dev)
    return keys, offsets


def store(E: int, num_keys: int, job: str):
    server = ad.Server(2 * E, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                       job=f"{job}{os.getpid()}", device=0)
    return server, ad.Worker(0, server)


def bags_row(info, name, server, kv, E, B, F, L, num_keys, iters, warmup, nb=4):
    dev = server.device
    batches = [batch(s, B, F, L, num_keys, dev) for s in range(nb)]
    touched = torch.unique(torch.cat([k for k, _ in batches]))
    g = torch.Generator(device=dev).manual_seed(1)
    for i in range(0, touched.numel(), 1 << 18):
        kk = touched[i:i + (1 << 18)]
        rows = torch.randn(kk.numel(), 2 * E, device=dev, generator=g) * 0.01
        rows[:, E:] = 1e-6
        kv.set(kk, rows.view(-1))
    kv.waitall()
    grads = [torch.randn(o.numel() - 1, E, device=dev, generator=g) * 1e-4 for _, o in batches]
    arms = {impl: StoreEmbeddingBag(server, kv, E, lr=0.05, grad_scale=float(B), impl=impl) for impl in ("fused", "torch")}
    it = {"fused": 0, "torch": 0}

    def fwd(impl):
        i = it[impl] % nb
        it[impl] += 1
        with torch.no_grad():
            arms[impl](*batches[i])

    def step(impl):
        i = it[impl] % nb
        it[impl] += 1
        arms[impl](*batches[i]).backward(grads[i])

    res = {"fused": {"fwd": [], "step": []}, "torch": {"fwd": [], "step": []}}
    for _ in range(warmup):
        for impl in arms:
            fwd(impl); step(impl)
    kv.waitall()
    for _ in range(iters):                  # alternate the routes, one run each per round
        for impl in arms:
            res[impl]["fwd"].append(median_ms(lambda: fwd(impl), 1, 0))
            res[impl]["step"].append(median_ms(lambda: step(impl), 1, 0))
            kv.waitall()
    nnz = float(np.mean([k.numel() for k, _ in batches]))
    nbags = B * F
    fwd_bytes = nnz * E * 4 + nbags * E * 4
    out = {"shape": name, "B": B, "F": F, "L": L, "E": E, "keys": num_keys, "nnz_mean": int(nnz),
           "distinct_keys_mean": int(np.mean([torch.unique(k).numel() for k, _ in batches])),
           "fwd_bytes_lower_bound": int(fwd_bytes), **info}
    for impl in arms:
        f = float(np.median(res[impl]["fwd"])); s = float(np.median(res[impl]["step"]))
        out[f"{impl}_fwd_ms"] = round(f, 4)
        out[f"{impl}_step_ms"] = round(s, 4)
        out[f"{impl}_fwd_GBps"] = round(fwd_bytes / (f * 1e-3) / 1e9, 1)
        out[f"{impl}_fwd_share_of_hbm_datasheet"] = round(fwd_bytes / (f * 1e-3) / HBM_DATASHEET_BPS, 3)
    out["step_speedup_fused_over_torch"] = round(out["torch_step_ms"] / out["fused_step_ms"], 2)
    print(json.dumps(out), flush=True)


def deepfm_step_row(info, iters, warmup, num_keys):
    from adapm_b200.models.deepfm import DeepFM, DeepFMConfig, synthetic_multi_hot_batch

    cfg = DeepFMConfig(num_features=num_keys, multi_hot=8)
    server, kv = store(cfg.emb_len, cfg.num_features, "embbagfm")
    try:
        model = DeepFM(server, kv, cfg)
        model.init_model()
        bs = [tuple(t.pin_memory() for t in synthetic_multi_hot_batch(cfg, s)) for s in range(4)]
        it = [0]

        def one():
            ids, off, y = bs[it[0] % len(bs)]
            it[0] += 1
            model.step(ids, y, offsets=off, return_tensor=True)

        ms = median_ms(one, iters, warmup)
        print(json.dumps({"shape": "deepfm full multi-hot step", "B": cfg.batch_size, "F": cfg.num_fields, "L": 8,
                          "E": cfg.emb_len, "keys": num_keys, "mlp": list(cfg.hidden), "precision": cfg.precision,
                          "fused_step_ms": round(ms, 3), "examples_per_s": round(cfg.batch_size / (ms * 1e-3)), **info}),
              flush=True)
    finally:
        kv.finalize()
        server.shutdown()


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="", help="comma list of deepfm,single,dlrm,step (default: all)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("embbag_bench needs a CUDA device", file=sys.stderr)
        return 2
    torch.cuda.set_device(0)
    info = device_info()
    only = set(args.only.split(",")) if args.only else {"deepfm", "single", "dlrm", "step"}
    if only & {"deepfm", "single"}:
        server, kv = store(20, 100_000_000, "embbag20")
        try:
            if "deepfm" in only:
                bags_row(info, "deepfm", server, kv, 20, 8192, 26, 8, 100_000_000, args.iters, args.warmup)
            if "single" in only:
                bags_row(info, "single-hot", server, kv, 20, 8192, 26, 1, 100_000_000, args.iters, args.warmup)
        finally:
            kv.finalize()
            server.shutdown()
    if "dlrm" in only:
        server, kv = store(128, 10_000_000, "embbag128")
        try:
            bags_row(info, "dlrm", server, kv, 128, 2048, 26, 32, 10_000_000, args.iters, args.warmup)
        finally:
            kv.finalize()
            server.shutdown()
    if "step" in only:
        deepfm_step_row(info, args.iters, args.warmup, 100_000_000)
    return 0


if __name__ == "__main__":
    sys.exit(main())
