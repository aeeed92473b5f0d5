"""Matrix-factorisation application (reference apps/matrix_factorization.cc), same flag names.

    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.mf -- --dataset train.mmc --rank 10 --algorithm dsgd --epochs 10
    python -m adapm_b200.apps.mf --synthetic_nnz 2000000 --num_rows 100000 --num_cols 20000 --rank 128
    python -m adapm_b200.apps.mf --loss bpr --num_negatives 4 --synthetic_nnz 2000000 --num_rows 50000 --rank 64

``--loss bpr``: implicit feedback (every entry is an interaction, its value is ignored), BPR against sampled negative
items; each epoch reports the BPR loss and, with a test set, Recall@K and NDCG@K of top-K lists without seen items.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np
import torch

import adapm_b200 as ad
from adapm_b200.apps._common import (add_ablation_options, add_system_options, enforce_full_replication, id_permutation,
                                      strip_dashes, system_options)
from adapm_b200.models.mf import MatrixFactorization, MFConfig, SparseMatrix
from adapm_b200.utils.mmio import read_matrix_market_coo


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--dataset", default=None, help="MatrixMarket coordinate file")
    ap.add_argument("--synthetic_nnz", type=int, default=0)
    ap.add_argument("--num_rows", type=int, default=10000)
    ap.add_argument("--num_cols", type=int, default=2000)
    ap.add_argument("--rank", "-r", type=int, default=10)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--num_threads", "-t", type=int, default=1)
    ap.add_argument("--algorithm", default="dsgd", choices=["dsgd", "columnwise", "plain"])
    ap.add_argument("--eps", type=float, default=0.01)
    ap.add_argument("--lambda", dest="lam", type=float, default=0.05)
    ap.add_argument("--signal_intent_cols", type=int, default=1000)
    ap.add_argument("--batch_nnz", type=int, default=1 << 18)
    ap.add_argument("--bold_driver", type=int, default=1)
    ap.add_argument("--export_prefix", default="")
    ap.add_argument("--model_seed", type=int, default=134827)
    ap.add_argument("--increase_step_factor", type=float, default=1.05, help="bold driver: factor after a successful epoch")
    ap.add_argument("--decrease_step_factor", type=float, default=0.5, help="bold driver: factor after an unsuccessful epoch")
    ap.add_argument("--signal_intent_rows", type=int, default=1, help="localise this rank's row parameters (default on)")
    ap.add_argument("--wor_blocks", type=int, default=1, help="WOR schedule for the DSGD blocks")
    ap.add_argument("--wor_points", type=int, default=1, help="WOR schedule for the data points")
    ap.add_argument("--compute_loss", type=int, default=1, help="report the training (and test, when <dataset> has a test file) loss")
    ap.add_argument("--init_parameters", type=int, default=2,
                    help="0: no init, 1: read W.mma / H.mma next to the dataset, 2: draw random factors")
    ap.add_argument("--early_stop", type=int, default=0, help="stop an epoch after N data points (debugging)")
    ap.add_argument("--max_runtime", type=float, default=float("inf"), help="stop after this many seconds")
    ap.add_argument("--prevent_full_model_pull", type=int, default=0,
                    help="accepted for parity: losses are accumulated inside the step, the model is never pulled in full")
    ap.add_argument("--write_generated_factors", default="", help="path prefix to write the initial factors to")
    ap.add_argument("--deterministic", type=int, default=0, choices=[0, 1],
                    help="one GPU: every non-zero of a batch reads the start-of-batch state, bit-identical runs")
    ap.add_argument("--loss", default="squared", choices=["squared", "bpr"],
                    help="squared: explicit ratings; bpr: implicit feedback (every entry is an interaction, values ignored)")
    ap.add_argument("--num_negatives", type=int, default=1, help="bpr: sampled negative items per interaction")
    ap.add_argument("--eval_k", type=int, default=10, help="bpr: length of the recommendation lists for recall / ndcg")
    add_ablation_options(ap)
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    world = int(__import__("os").environ.get("WORLD_SIZE", "1"))
    if args.deterministic and world > 1:
        ap.error("--deterministic 1 needs a single GPU (WORLD_SIZE=1): on several GPUs rows move between ranks during a step")
    rank = int(__import__("os").environ.get("RANK", "0"))
    bpr = args.loss == "bpr"
    if bpr and args.num_negatives < 1:
        ap.error("--num_negatives must be >= 1")
    test = None
    if args.dataset:
        i, j, x, m, n = read_matrix_market_coo(args.dataset)
        if args.enforce_random_keys:      # row / column ids are labels: relabel them randomly (same on every rank)
            fr, fc = id_permutation(m, args.model_seed, True), id_permutation(n, args.model_seed + 1, True)
            i, j = fr[i], fc[j]
        data = SparseMatrix(i, j, x, m, n, world, rank)
        tpath = args.dataset.replace("train", "test")
        if args.compute_loss and tpath != args.dataset and os.path.exists(tpath):
            ti, tj, tx, _, _ = read_matrix_market_coo(tpath)
            if args.enforce_random_keys:
                ti, tj = fr[ti], fc[tj]
            # bpr: every rank ranks the items of its own row block, so it keeps the whole test set
            test = (ti, tj) if bpr else (ti[rank::world], tj[rank::world], tx[rank::world])
    elif bpr:
        m, n = args.num_rows, args.num_cols
        data, test = SparseMatrix.synthetic_implicit(m, n, max(1, (args.synthetic_nnz or 200000) // m), 8, world, rank,
                                                     seed=args.model_seed)
        if not args.compute_loss:
            test = None
    else:
        m, n = args.num_rows, args.num_cols
        data = SparseMatrix.synthetic(m, n, args.synthetic_nnz or 200000, 8, world, rank, seed=args.model_seed)
    cfg = MFConfig(num_rows=m, num_cols=n, rank=args.rank, algorithm=args.algorithm, eps=args.eps, lam=args.lam,
                   batch_nnz=args.batch_nnz, signal_intent_cols=args.signal_intent_cols, bold_driver=bool(args.bold_driver),
                   model_seed=args.model_seed, eps_inc=args.increase_step_factor, eps_dec=args.decrease_step_factor,
                   signal_intent_rows=bool(args.signal_intent_rows), wor_blocks=bool(args.wor_blocks),
                   wor_points=bool(args.wor_points), early_stop=args.early_stop, deterministic=bool(args.deterministic),
                   loss=args.loss, num_negatives=args.num_negatives,
                   sampling_scheme=getattr(args, "sampling.scheme") or "local")
    ad.setup(cfg.num_keys(world), 1)   # one worker per rank: the per-thread loops of the reference are batched kernels here
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args),
                       dtype={"float": "float32", "double": "float64"}[args.value_type])
    kv = ad.Worker(0, server)
    model = MatrixFactorization(server, kv, cfg, data)
    if args.init_parameters == 2:
        model.init_model()
    elif args.init_parameters == 1:
        d = os.path.dirname(args.dataset or ".")
        model.init_model()                 # row intents etc.; the factors are overwritten from the files
        model.load_factors(os.path.join(d, "W.mma"), os.path.join(d, "H.mma"))
    if args.write_generated_factors:
        model.write_factors(args.write_generated_factors)
    if args.enforce_full_replication:
        enforce_full_replication(kv, cfg.num_keys(world))
    kv.barrier()
    prev, t0 = None, time.time()
    for epoch in range(args.epochs):
        loss = model.run_epoch(epoch)
        kv.barrier()
        model.bold_driver(loss, prev)
        prev = loss
        if args.compute_loss and bpr:
            msg = f"[mf] epoch {epoch}: local BPR loss {loss:.6g}, eps {model.eps:.4g}"
            if test is not None:
                kv.wait_sync()
                tr = server.allreduce_sum([float(v) for v in model.evaluate_ranking(*test, k=args.eval_k)])
                users = max(1.0, float(tr[2]))
                msg += f", test recall@{args.eval_k} {tr[0] / users:.4f}, ndcg@{args.eval_k} {tr[1] / users:.4f}"
            if server.my_rank() == 0:
                print(msg + f" ({time.time() - t0:.1f}s)", flush=True)
        elif args.compute_loss:
            msg = f"[mf] epoch {epoch}: local squared error {loss:.6g}, eps {model.eps:.4g}"
            if test is not None:
                kv.wait_sync()
                tl = server.allreduce_sum([model.evaluate(*test), float(len(test[2]))])
                msg += f", test rmse {float((tl[0] / max(1.0, float(tl[1]))) ** 0.5):.4f}"
            if server.my_rank() == 0:
                print(msg + f" ({time.time() - t0:.1f}s)", flush=True)
        if time.time() - t0 > args.max_runtime:
            break
    if args.export_prefix:
        model.write_factors(args.export_prefix)
    kv.barrier()
    kv.finalize()
    if server.my_rank() == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
