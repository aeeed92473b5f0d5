"""Where the time of the deterministic one-GPU word2vec step goes: per-pass device time at the bench.py shape (1M
vocabulary, d = 300, 25 negatives, 32768 pairs per step), each pass's algorithmic HBM bytes computed from the step's
key counts, and the achieved rate as a fraction of the H100 SXM data-sheet 3.35 TB/s.

    python benchmarks/sgns_det_passes.py [--steps 200] [--dim 300] [--negative 25]

Per-kernel device times come from torch.profiler (CUDA activity records) over --steps steps after a warm-up; the step
time is taken with CUDA events around the same steps without the profiler. Kernels are grouped into passes by name, so
the script also reports the passes of the earlier accumulator-based step (index, step, apply). Prints one JSON line with
the device name and power limit."""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts  # noqa: E402

HBM_GBS = 3350.0   # H100 SXM data sheet

# kernel name fragment -> pass (first match wins)
PASSES = [("sgns_det_index_kernel", "index"), ("fx_index_kernel", "index"),
          ("sgns_score_tma_kernel", "score"), ("sgns_step_tma_fx_kernel", "step"),
          ("sgns_det_group_kernel", "group"), ("DeviceScan", "group"),
          ("sgns_det_gather_kernel", "gather"), ("sgns_det_finish_kernel", "finish"),
          ("fx_apply_kernel", "apply"), ("sample_kernel", "sampler")]


def device_info() -> dict:
    info = {"device": torch.cuda.get_device_name(0), "power_limit": "not measured"}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
            info = {"device": name, "power_limit": power}
    except (OSError, subprocess.SubprocessError):
        pass
    return info


def key_counts(batch, negs, B, neg):
    centers, contexts = batch[0], batch[1]
    negs = negs.view(B, neg)
    valid = negs != contexts.view(B, 1)
    targets = torch.cat([contexts, negs[valid]])
    allk = torch.cat([centers, targets])
    keys, n = torch.unique(allk, return_counts=True)
    single = keys[n == 1]
    return {"pairs": B, "entries": int(B + targets.numel()), "centers": int(torch.unique(centers).numel()),
            "targets": int(torch.unique(targets).numel()), "keys": int(keys.numel()),
            # keys with one entry in the step, which the score pass applies; those of them that are centers
            "singletons": int(single.numel()), "singleton_centers": int(torch.isin(centers, single).sum())}


def pass_bytes(kc, d, neg):
    """Least HBM traffic of each pass (bytes), from the step's key counts: each distinct row is read once (written once
    where the pass updates it), per-pair and per-entry buffers once each way."""
    P, E, C, U = kc["pairs"], kc["entries"], kc["centers"], kc["keys"]
    S, SC = kc.get("singletons", 0), kc.get("singleton_centers", 0)
    half, row, key = 4 * d, 8 * d, 8
    slots = P * (neg + 2)
    return {
        # gather-based step
        "index": slots * key + U * (key + 4),
        "score": U * half + S * (half + row) + (P - SC) * half + C * half + slots * 4,   # rows' embedding halves;
                                                                            # one-entry rows: AdaGrad half read, row
                                                                            # written; g0, snapshot, gs
        "group": 2 * slots * key + 2 * E * 8 + E * 12 + 3 * U * 4,          # keys twice; descriptors + kid, gs + pcid
                                                                            # read for them; counts and scan
        "gather": 2 * (U - S) * row + (P - SC) * half + C * half + (E - S) * 8,   # the other rows read + written; g0,
                                                                                  # snapshot; descriptors
        "finish": U * 12,
        # accumulator-based step
        "step": U * row + P * half + 2 * U * 2 * row,                       # rows; 8-byte accumulators read + written
        "apply": 2 * U * 2 * row + 2 * U * row,                             # accumulators read + cleared; rows read + written
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--negative", type=int, default=25)
    ap.add_argument("--batch-pairs", type=int, default=32768)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sgns_det_passes.py needs a CUDA device")
    cfg = Word2VecConfig(vocab_size=args.vocab, embed_dim=args.dim, negative=args.negative, batch_pairs=args.batch_pairs)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", device=0)
    worker = ad.Worker(0, server)
    counts = zipf_counts(cfg.vocab_size, cfg.zipf_exponent)
    model = Word2Vec(server, worker, cfg, counts)
    model.init_model()
    data = SyntheticPairs(cfg, counts, 0, seed=1)
    K, W = args.steps, args.warmup
    batches = [data.batch(s).to("cuda") for s in range(W + 2 * K)]

    def run(first, n):
        for s in range(first, first + n):
            model.loss.zero_()
            model.step_resident(batches[s])
            worker.advance_clock()

    run(0, W)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run(W, K)
    b.record()
    torch.cuda.synchronize()
    step_ms = a.elapsed_time(b) / K

    kc = key_counts(batches[W + K - 1].view(2, -1), model._neg, cfg.batch_pairs, cfg.negative)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(W + K, K)
        torch.cuda.synchronize()
    per = defaultdict(float)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = next((p for frag, p in PASSES if frag in e.name), None)
        if name is not None:
            per[name] += e.time_range.elapsed_us() / 1e3 / K          # us -> ms per step
    nbytes = pass_bytes(kc, cfg.embed_dim, cfg.negative)
    passes = {}
    for p, ms in per.items():
        entry = {"ms": round(ms, 4)}
        if p in nbytes and ms > 0:
            gbs = nbytes[p] / (ms * 1e-3) / 1e9
            entry.update(gb=round(nbytes[p] / 1e9, 4), gbs=round(gbs, 1), fraction_of_hbm=round(gbs / HBM_GBS, 3))
        passes[p] = entry
    print(json.dumps({"bench": "sgns_det_passes", **device_info(), "ms_per_step": round(step_ms, 4),
                      "key_counts": kc, "passes": passes,
                      "note": "per-pass times from torch.profiler over %d steps; bytes = least HBM traffic of the pass "
                              "from the step's key counts; fraction of the 3.35 TB/s H100 SXM data-sheet rate" % K}))
    worker.finalize()
    server.shutdown()


if __name__ == "__main__":
    main()
