"""Device-timed updates/s of the fused KGE (ComplEx, FB15k scale, d=512; RESCAL, d=64) and MF (d=128) steps on one GPU
(BASELINE.md configs 3 and 4), in place and deterministic (``deterministic=True``: start-of-step reads, fixed-point sums,
one apply pass), with the achieved fraction of the HBM data-sheet bandwidth for the in-place steps.

Both modes run in the same process on the same batches; the timed rounds alternate between them, and each mode's
figure is the median over its rounds. Every line carries the device name and power limit (a read-only
``nvidia-smi --query-gpu`` query)."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.kge import KGE, KGEConfig, synthetic_triples  # noqa: E402
from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix  # noqa: E402

MODES = ("in_place", "deterministic")


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


def ab_time(step, rounds: int, k: int) -> dict:
    """step(i, deterministic) enqueues step i; rounds x (k steps in place, k steps deterministic), alternating.
    Returns the median ms per step of each mode."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {m: [] for m in MODES}
    i = 0
    for r in range(rounds):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):
            torch.cuda.synchronize()
            a.record()
            for _ in range(k):
                step(i, m == "deterministic")
                i += 1
            b.record(); torch.cuda.synchronize()
            ms[m].append(a.elapsed_time(b) / k)
    return {m: float(np.median(v)) for m, v in ms.items()}


def report(bench: str, config: str, ms: dict, updates: int, dev: dict, row_bytes: int = 0, **extra) -> None:
    out = {"bench": bench, "config": config, **dev}
    for m in MODES:
        out[f"ms_per_step_{m}"] = ms[m]
        out[f"updates_per_s_{m}"] = updates / ms[m] * 1e3
    out["deterministic_over_in_place"] = ms["deterministic"] / ms["in_place"]
    if row_bytes:
        gbs = updates / ms["in_place"] * 1e3 * 2 * row_bytes / 1e9
        out["algorithmic_gbs_in_place"] = gbs
        out["frac_of_datasheet_hbm_in_place"] = gbs / 3350.0     # H100 SXM data sheet (HBM3)
    out.update(extra)
    print(json.dumps(out), flush=True)


def bench_kge(cfg: KGEConfig, job: str, rounds: int, k: int, dev: dict, config: str, note: str) -> None:
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=job, device=0)
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    tr = synthetic_triples(cfg, cfg.batch_triples * 16, seed=1)
    batches = [tr[i * cfg.batch_triples:(i + 1) * cfg.batch_triples].pin_memory() for i in range(16)]

    def step(i, det):
        model.cfg.deterministic = det
        model.step(batches[i % 16])

    for i in range(4):   # warm-up of both modes (allocates the deterministic scratch)
        step(i, i % 2 == 1)
    ms = ab_time(step, rounds, k)
    upd = cfg.batch_triples * cfg.updates_per_triple
    report(f"kge_{cfg.algorithm.lower()}_step", config, ms, upd, dev, cfg.entity_len * 4 if cfg.algorithm == "ComplEx" else 0,
           calls_per_step=cfg.batch_triples * (1 + 2 * cfg.neg_ratio), note=note)
    kv.finalize(); server.shutdown()


def main():
    dev = device_info()
    # ---------------- KGE ComplEx, FB15k scale
    bench_kge(KGEConfig(embed_dim=512, batch_triples=8192), "benchkge", 6, 10, dev,
              "FB15k scale (14951 ent, 1345 rel), d=512, neg_ratio=6",
              "67 MB model: rows are L2/HBM resident, traffic is mostly L2 hits")
    # ---------------- KGE RESCAL, d=64: relation rows are 64 x 64 matrices, ~106 k calls per step on <= 1345 relations
    bench_kge(KGEConfig(embed_dim=64, algorithm="RESCAL", batch_triples=8192), "benchrescal", 4, 3, dev,
              "FB15k scale (14951 ent, 1345 rel), RESCAL d=64, neg_ratio=6",
              "relation rows 32 KB; every call adds a full relation-matrix update")

    # ---------------- MF, d=128
    cfg = MFConfig(num_rows=2_000_000, num_cols=200_000, rank=128, algorithm="plain", batch_nnz=1 << 18)
    data = SparseMatrix.synthetic(cfg.num_rows, cfg.num_cols, (1 << 18) * 8, 8, 1, 0, seed=3)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="benchmf", device=0)
    kv = ad.Worker(0, server)
    model = MatrixFactorization(server, kv, cfg, data)
    model.init_model()
    from adapm_b200.ops import mf_step

    d = server.device
    n = cfg.batch_nnz
    packs = []
    for s in range(8):
        sl = slice(s * n, (s + 1) * n)
        packs.append((torch.from_numpy(data.i[sl]).to(d), (torch.from_numpy(data.j[sl]) + model.fck).to(d),
                      torch.from_numpy(data.x[sl]).to(d), torch.from_numpy(data.row_nnz_all[data.i[sl]]).to(d),
                      torch.from_numpy(data.col_nnz_all[data.j[sl]]).to(d)))

    def step(i, det):
        mf_step(server, *packs[i % 8], cfg.rank, 0.01, 0.05, model.loss, model.stats, deterministic=det)

    for i in range(4):
        step(i, i % 2 == 1)
    ms = ab_time(step, 6, 10)
    report("mf_step", "2M x 200k, rank 128 (2.25 GB of factors), uniform non-zeros", ms, 2 * n, dev, cfg.row_len * 4)
    kv.finalize(); server.shutdown()


if __name__ == "__main__":
    main()
