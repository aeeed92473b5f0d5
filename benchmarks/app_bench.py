"""Device-timed updates/s of the fused KGE (ComplEx, FB15k scale, d=512) and MF (d=128) steps on one GPU
(BASELINE.md configs 3 and 4), with the achieved fraction of the measured HBM copy bandwidth."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200.models.kge import KGE, KGEConfig, synthetic_triples  # noqa: E402
from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix  # noqa: E402


def main():
    datasheet_hbm_gbs = 3350.0     # H100 SXM data sheet (HBM3)
    # ---------------- KGE ComplEx, FB15k scale
    cfg = KGEConfig(embed_dim=512, batch_triples=8192)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="benchkge", device=0)
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    tr = synthetic_triples(cfg, cfg.batch_triples * 16, seed=1)
    batches = [tr[i * cfg.batch_triples:(i + 1) * cfg.batch_triples].pin_memory() for i in range(16)]
    for i in range(5):
        model.step(batches[i])
    torch.cuda.synchronize()
    K = 50
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(K):
        model.step(batches[i % 16])
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / K
    upd = cfg.batch_triples * cfg.updates_per_triple
    row_bytes = cfg.entity_len * 4
    print(json.dumps({"bench": "kge_complex_step", "config": "FB15k scale (14951 ent, 1345 rel), d=512, neg_ratio=6",
                      "ms_per_step": ms, "updates_per_s": upd / ms * 1e3,
                      "algorithmic_gbs": upd / ms * 1e3 * 2 * row_bytes / 1e9,
                      "note": "67 MB model: rows are L2/HBM resident, traffic is mostly L2 hits"}), flush=True)
    kv.finalize(); server.shutdown()

    # ---------------- MF, d=128
    cfg = MFConfig(num_rows=2_000_000, num_cols=200_000, rank=128, algorithm="plain", batch_nnz=1 << 18)
    data = SparseMatrix.synthetic(cfg.num_rows, cfg.num_cols, (1 << 18) * 8, 8, 1, 0, seed=3)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys(1), num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="benchmf", device=0)
    kv = ad.Worker(0, server)
    model = MatrixFactorization(server, kv, cfg, data)
    model.init_model()
    from adapm_b200.ops import mf_step

    dev = server.device
    n = cfg.batch_nnz
    packs = []
    for s in range(8):
        sl = slice(s * n, (s + 1) * n)
        packs.append((torch.from_numpy(data.i[sl]).to(dev), (torch.from_numpy(data.j[sl]) + model.fck).to(dev),
                      torch.from_numpy(data.x[sl]).to(dev), torch.from_numpy(data.row_nnz_all[data.i[sl]]).to(dev),
                      torch.from_numpy(data.col_nnz_all[data.j[sl]]).to(dev)))
    for p in packs[:3]:
        mf_step(server, *p, cfg.rank, 0.01, 0.05, model.loss, model.stats)
    torch.cuda.synchronize()
    a.record()
    for i in range(K):
        mf_step(server, *packs[i % 8], cfg.rank, 0.01, 0.05, model.loss, model.stats)
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / K
    upd = 2 * n
    gbs = upd / ms * 1e3 * 2 * cfg.row_len * 4 / 1e9
    print(json.dumps({"bench": "mf_step", "config": "2M x 200k, rank 128 (2.25 GB of factors), uniform non-zeros",
                      "ms_per_step": ms, "updates_per_s": upd / ms * 1e3, "algorithmic_gbs": gbs,
                      "frac_of_datasheet_hbm": gbs / datasheet_hbm_gbs}), flush=True)
    kv.finalize(); server.shutdown()


if __name__ == "__main__":
    main()
