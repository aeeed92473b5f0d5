"""CTR application (BASELINE config #5) on the bindings-style API: DeepFM, a field-aware factorisation machine
(``--model ffm``, libffm's model: one latent vector per field in every feature's row; ``--embed_dim`` is its k), or
DLRM (``--model dlrm``: bottom MLP over the dense features, dot interaction, top MLP; synthetic planted data, or
Criteo TSV files with ``--data`` / ``--test_data``), or DLRM-DCNv2 (``--model dlrm --interaction dcn``: a low-rank
cross network of ``--cross_layers`` layers of rank ``--cross_rank`` instead of the dot interaction).

    python -m adapm_b200.launch -s 8 --backend cuda -m adapm_b200.apps.ctr -- --num_features 100000000
    python -m adapm_b200.apps.ctr --backend cpu --num_features 20000 --steps 30 --batch_size 512
    python -m adapm_b200.apps.ctr --backend cpu --num_features 20000 --steps 30 --batch_size 512 --multi_hot 3
    python -m adapm_b200.apps.ctr --backend cpu --model ffm --num_features 20000 --num_fields 8 --embed_dim 4 --steps 30
    python -m adapm_b200.apps.ctr --backend cpu --model dlrm --num_features 20000 --steps 30 --batch_size 512
    python -m adapm_b200.apps.ctr --backend cpu --model dlrm --interaction dcn --cross_rank 64 --steps 30 --batch_size 512
"""
from __future__ import annotations

import argparse
import itertools
import sys
import time

import torch

import adapm_b200 as ad
from adapm_b200.apps._common import add_system_options, strip_dashes, system_options
from adapm_b200.models.deepfm import DeepFM, DeepFMConfig, synthetic_ctr_batch, synthetic_multi_hot_batch
from adapm_b200.models.ffm import FFM, FFMConfig, synthetic_ffm_batch


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default="deepfm", choices=["deepfm", "ffm", "dlrm"])
    ap.add_argument("--num_features", type=int, default=1_000_000)
    ap.add_argument("--num_fields", type=int, default=26)
    ap.add_argument("--embed_dim", type=int, default=16, help="DeepFM: embedding size; FFM: k, latent values per field")
    ap.add_argument("--batch_size", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--read_ahead", type=int, default=4)
    ap.add_argument("--precision", default="bf16", choices=["fp32", "bf16", "fp8"], help="DeepFM only: the dense GEMMs")
    ap.add_argument("--table_precision", default="fp32", choices=["fp32", "fp8_block"],
                    help="DeepFM only. fp8_block: train on the values a block-scaled e4m3 embedding table would deliver "
                         "(fp32 master rows)")
    ap.add_argument("--multi_hot", type=int, default=0,
                    help="> 0: every field holds a bag of 1..L ids, pooled into one embedding (fused kernels on CUDA)")
    ap.add_argument("--pooling", default="sum", choices=["sum", "mean"], help="pooling of multi-hot bags")
    ap.add_argument("--eta", type=float, default=0.2, help="FFM, DLRM: AdaGrad step size (DLRM: of the embedding rows)")
    ap.add_argument("--lam", type=float, default=2e-5, help="FFM: L2 regularisation")
    ap.add_argument("--test_batches", type=int, default=4, help="FFM, DLRM: held-out batches evaluated after training")
    ap.add_argument("--num_dense", type=int, default=13, help="DLRM: dense features (13 in Criteo data)")
    ap.add_argument("--bottom", default="512,256", help="DLRM: hidden widths of the bottom MLP (num_dense -> ... -> E)")
    ap.add_argument("--top", default="1024,1024,512,256", help="DLRM: hidden widths of the top MLP (W -> ... -> 1)")
    ap.add_argument("--data", default=None, help="DLRM: Criteo TSV training data (default: synthetic planted data)")
    ap.add_argument("--test_data", default=None, help="DLRM: Criteo TSV held-out data (needed with --data)")
    ap.add_argument("--interaction", default="dot", choices=["dot", "dcn"],
                    help="DLRM: dot interaction, or dcn (DLRM-DCNv2's low-rank cross network)")
    ap.add_argument("--cross_layers", type=int, default=3, help="DLRM with --interaction dcn: cross layers")
    ap.add_argument("--cross_rank", type=int, default=512, help="DLRM with --interaction dcn: rank of each layer")
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    if args.interaction != "dot" and args.model != "dlrm":
        ap.error(f"--interaction {args.interaction} needs --model dlrm")
    if args.model == "ffm":
        if args.multi_hot > 0:
            ap.error("--multi_hot is not supported with --model ffm (one id per field)")
        return run_ffm(args)
    if args.model == "dlrm":
        if args.table_precision != "fp32":
            ap.error("--table_precision fp8_block is not supported with --model dlrm")
        if args.data and not args.test_data:
            ap.error("--data needs --test_data")
        try:
            widths = [tuple(int(w) for w in getattr(args, n).split(",") if w) for n in ("bottom", "top")]
        except ValueError:
            ap.error("--bottom and --top take comma-separated integers")
        return run_dlrm(args, *widths)
    cfg = DeepFMConfig(num_features=args.num_features, num_fields=args.num_fields, embed_dim=args.embed_dim,
                       batch_size=args.batch_size, read_ahead=args.read_ahead, precision=args.precision,
                       table_precision=args.table_precision, multi_hot=args.multi_hot, pooling=args.pooling)
    ad.setup(cfg.num_features, 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    model = DeepFM(server, kv, cfg)
    model.init_model()
    rank = server.my_rank()
    # look-ahead: while step s runs, the distinct feature ids of step s + read_ahead are signalled (parallel/schedules.py)
    from ..parallel.schedules import LookaheadIntents

    batches = {}

    def batch(b):
        if b not in batches:
            batches[b] = synthetic_multi_hot_batch(cfg, b, rank) if cfg.multi_hot else synthetic_ctr_batch(cfg, b, rank)
        return batches[b]

    look = LookaheadIntents(kv, args.steps + cfg.read_ahead, cfg.read_ahead, lambda b: batch(b)[0]) if server.num_servers() > 1 else None
    if look:
        look.prime()
    t0, losses = time.time(), []
    for s in range(args.steps):
        if look:
            look.signal(s)
        if cfg.multi_hot:
            ids, off, y = batch(s)
            batches.pop(s - 1, None)
            losses.append(model.step(ids, y, offsets=off))
        else:
            ids, y = batch(s)
            batches.pop(s - 1, None)
            losses.append(model.step(ids, y))
        kv.advance_clock()
        if rank == 0 and (s + 1) % max(1, args.steps // 5) == 0:
            print(f"[ctr] step {s + 1}: loss {sum(losses[-10:]) / len(losses[-10:]):.4f} "
                  f"({(s + 1) * cfg.batch_size / (time.time() - t0):.0f} examples/s/rank)", flush=True)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


def run_ffm(args) -> int:
    cfg = FFMConfig(num_features=args.num_features, num_fields=args.num_fields, k=args.embed_dim, eta=args.eta,
                    lam=args.lam, batch_size=args.batch_size, read_ahead=args.read_ahead)
    ad.setup(cfg.num_features, 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    model = FFM(server, kv, cfg)
    model.init_model()
    rank = server.my_rank()
    from ..parallel.schedules import LookaheadIntents

    batches = {}

    def batch(b):
        if b not in batches:
            batches[b] = synthetic_ffm_batch(cfg, b, rank)
        return batches[b]

    look = LookaheadIntents(kv, args.steps + cfg.read_ahead, cfg.read_ahead, lambda b: batch(b)[0]) if server.num_servers() > 1 else None
    if look:
        look.prime()
    t0, losses = time.time(), []
    for s in range(args.steps):
        if look:
            look.signal(s)
        ids, y = batch(s)
        batches.pop(s - 1, None)
        losses.append(model.step(ids, y))
        kv.advance_clock()
        if rank == 0 and (s + 1) % max(1, args.steps // 5) == 0:
            print(f"[ctr] step {s + 1}: loss {sum(losses[-10:]) / len(losses[-10:]):.4f} "
                  f"({(s + 1) * cfg.batch_size / (time.time() - t0):.0f} examples/s/rank)", flush=True)
    kv.barrier()
    ll, auc = model.evaluate(synthetic_ffm_batch(cfg, b, rank, held_out=True) for b in range(args.test_batches))
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(f"[ctr] test logloss {ll:.4f} auc {auc:.4f}", flush=True)
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


def run_dlrm(args, bottom=(512, 256), top=(1024, 1024, 512, 256)) -> int:
    from adapm_b200.models.dlrm import DLRM, DLRMConfig, synthetic_dlrm_batch
    from adapm_b200.utils.criteo import CRITEO_DENSE, CRITEO_FIELDS, criteo_batches

    num_fields, num_dense = args.num_fields, args.num_dense
    if args.data:
        num_fields, num_dense = CRITEO_FIELDS, CRITEO_DENSE
    cfg = DLRMConfig(num_features=args.num_features, num_fields=num_fields, num_dense=num_dense,
                     embed_dim=args.embed_dim, bottom=bottom, top=top, lr_sparse=args.eta, batch_size=args.batch_size,
                     read_ahead=args.read_ahead, precision=args.precision, multi_hot=0 if args.data else args.multi_hot,
                     pooling=args.pooling, interaction=args.interaction, cross_layers=args.cross_layers,
                     cross_rank=args.cross_rank)
    ad.setup(cfg.num_features, 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    model = DLRM(server, kv, cfg)
    model.init_model()
    rank, world = server.my_rank(), server.num_servers()
    from ..parallel.schedules import LookaheadIntents

    # a data file is read once, in order; rank r trains on its batches r, r + world, ...
    train = (itertools.islice(criteo_batches(args.data, cfg.batch_size, cfg.num_features), rank, None, world)
             if args.data else None)
    batches, pending = {}, [0]          # pending[0]: the index of the next batch read from the data file

    def batch(b):
        """batch b, None past the end of the data file"""
        if train is None:
            if b not in batches:
                batches[b] = synthetic_dlrm_batch(cfg, b, rank)
            return batches[b]
        while pending[0] <= b:
            nxt = next(train, None)
            if nxt is None:
                return None
            batches[pending[0]] = nxt
            pending[0] += 1
        return batches.get(b)

    def keys_of(b):
        x = batch(b)
        return x[1] if x is not None else torch.zeros(0, dtype=torch.int64)

    look = LookaheadIntents(kv, args.steps + cfg.read_ahead, cfg.read_ahead, keys_of) if world > 1 else None
    if look:
        look.prime()
    t0, losses = time.time(), []
    for s in range(args.steps):
        if look:
            look.signal(s)
        x = batch(s)
        if x is None:
            break
        batches.pop(s - 1, None)
        dense, ids, *off, y = x
        losses.append(model.step(dense, ids, y, offsets=off[0] if off else None))
        kv.advance_clock()
        if rank == 0 and (s + 1) % max(1, args.steps // 5) == 0:
            print(f"[ctr] step {s + 1}: loss {sum(losses[-10:]) / len(losses[-10:]):.4f} "
                  f"({(s + 1) * cfg.batch_size / (time.time() - t0):.0f} examples/s/rank)", flush=True)
    kv.barrier()
    if args.test_data:
        test = itertools.islice(criteo_batches(args.test_data, cfg.batch_size, cfg.num_features), args.test_batches)
    else:
        test = (synthetic_dlrm_batch(cfg, b, rank, held_out=True) for b in range(args.test_batches))
    ll, auc = model.evaluate(test)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(f"[ctr] test logloss {ll:.4f} auc {auc:.4f}", flush=True)
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
