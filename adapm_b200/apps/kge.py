"""Knowledge-graph-embedding application (reference apps/knowledge_graph_embeddings.cc), same flag names.

    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.kge -- --dataset apps/data/kge/ --num_entities 280 \\
        --num_relations 112 --embed_dim 100 --num_epochs 12 --algorithm ComplEx --eval_freq 4
    python -m adapm_b200.apps.kge --synthetic 100000 --embed_dim 128           (FB15k-shaped synthetic triples)
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

import adapm_b200 as ad
from adapm_b200.apps._common import (add_ablation_options, add_system_options, enforce_full_replication, id_permutation,
                                      strip_dashes, system_options, wants_sync_push)
from adapm_b200.models.kge import KGE, KGEConfig, evaluate_fused, load_triples, synthetic_triples
from adapm_b200.utils.allreduce import ps_allreduce


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--dataset", default=None, help="directory with train.del / valid.del / test.del (s r o per line)")
    ap.add_argument("--synthetic", type=int, default=0, help="number of synthetic training triples")
    ap.add_argument("--algorithm", default="ComplEx", choices=["ComplEx", "RESCAL", "TransE", "RotatE"])
    ap.add_argument("--train_type", default="negative_sampling", choices=["negative_sampling", "1vsAll", "sampled_softmax"],
                    help="negative_sampling: BCE over neg_ratio corrupted subjects and objects per triple; 1vsAll "
                         "(ComplEx, RESCAL): softmax cross-entropy of every query against all entities (neg_ratio unused); "
                         "sampled_softmax (ComplEx, RESCAL): softmax cross-entropy against the chunk's subjects and objects "
                         "and --shared_negatives entities shared by the batch (neg_ratio unused)")
    ap.add_argument("--shared_negatives", type=int, default=1024,
                    help="sampled_softmax: entities sampled per step, shared by the whole batch")
    ap.add_argument("--transe_norm", type=int, default=1, choices=[1, 2], help="TransE: L1 or L2 distance")
    ap.add_argument("--margin", type=float, default=1.0,
                    help="TransE: margin of the ranking loss; RotatE: gamma of the sigmoid loss")
    ap.add_argument("--adversarial_temperature", type=float, default=1.0,
                    help="RotatE: temperature alpha of the self-adversarial negative weights (0: uniform weights)")
    ap.add_argument("--embed_dim", type=int, default=10)
    ap.add_argument("--num_threads", "-t", type=int, default=1)
    ap.add_argument("--num_epochs", type=int, default=10)
    ap.add_argument("--eta", type=float, default=0.1)
    ap.add_argument("--gamma_entity", type=float, default=1e-3)
    ap.add_argument("--gamma_relation", type=float, default=1e-3)
    ap.add_argument("--dropout_entity", type=float, default=0.0)
    ap.add_argument("--dropout_relation", type=float, default=0.0)
    ap.add_argument("--neg_ratio", type=int, default=6)
    ap.add_argument("--eval_freq", type=int, default=-1)
    ap.add_argument("--num_entities", type=int, default=14951)
    ap.add_argument("--num_relations", type=int, default=1345)
    ap.add_argument("--signal_intent_ahead", type=int, default=4, help="batches of look-ahead")
    ap.add_argument("--signal_initial_relations_intent", type=int, default=0)
    ap.add_argument("--batch_triples", type=int, default=0,
                    help="triples per step; 0 = auto: min(4096, max(32, num_entities / 4)) (all triples of a step read the "
                         "state at the start of the step, so a step must stay small relative to the number of entities)")
    ap.add_argument("--model_path", default="")
    ap.add_argument("--write_end_checkpoint", type=int, default=0)
    ap.add_argument("--write_every", type=int, default=1)
    ap.add_argument("--eval_truncate_tr", type=int, default=2048)
    ap.add_argument("--model_seed", type=int, default=134827)
    ap.add_argument("--max_runtime", type=float, default=float("inf"))
    ap.add_argument("--write_embeddings", default="", help="directory to checkpoint the model to after each epoch "
                                                           "(the reference's spelling of --model_path)")
    ap.add_argument("--init_parameters", default="", help="'none', 'uniform{a/b}' or 'normal{mean/std}' (default normal{0/0.1})")
    ap.add_argument("--eval_initial", type=int, default=0, help="run an evaluation before the first epoch")
    ap.add_argument("--eval_truncate_va", type=int, default=0, help="truncate the validation set in evaluations (0: all)")
    ap.add_argument("--max_N", type=int, default=-1, help="artificial maximum of training triples per worker (fast tests)")
    ap.add_argument("--read_partitioned_dataset", type=int, default=0,
                    help="read train.partitioned.<servers>x<threads>.del: block b of the file is trained by worker b")
    ap.add_argument("--deterministic", type=int, default=0, choices=[0, 1],
                    help="one GPU: every call of a batch reads the start-of-batch state, bit-identical runs")
    add_ablation_options(ap)
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    if args.deterministic and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        ap.error("--deterministic 1 needs a single GPU (WORLD_SIZE=1): on several GPUs rows move between ranks during a step")

    if args.batch_triples <= 0:
        args.batch_triples = min(4096, max(32, args.num_entities // 4))
    cfg = KGEConfig(num_entities=args.num_entities, num_relations=args.num_relations, embed_dim=args.embed_dim,
                    algorithm=args.algorithm, neg_ratio=args.neg_ratio, eta=args.eta, gamma_entity=args.gamma_entity,
                    gamma_relation=args.gamma_relation, dropout_entity=args.dropout_entity,
                    dropout_relation=args.dropout_relation, batch_triples=args.batch_triples,
                    read_ahead=args.signal_intent_ahead, sampling_scheme=getattr(args, "sampling.scheme") or "local",
                    signal_initial_relations_intent=bool(args.signal_initial_relations_intent), model_seed=args.model_seed,
                    deterministic=bool(args.deterministic), p_norm=args.transe_norm, margin=args.margin,
                    adversarial_temperature=args.adversarial_temperature, train_type=args.train_type,
                    shared_negatives=args.shared_negatives)
    if args.write_embeddings and not args.model_path:
        os.makedirs(args.write_embeddings, exist_ok=True)
        args.model_path = os.path.join(args.write_embeddings, "")
    world_env = int(os.environ.get("WORLD_SIZE", "1"))
    if args.dataset:
        tr_name = "train.del"
        if args.read_partitioned_dataset:
            tr_name = f"train.partitioned.{world_env}x{args.num_threads}.del"
        tr = load_triples(os.path.join(args.dataset, tr_name))
        va = load_triples(os.path.join(args.dataset, "valid.del"))
        te = load_triples(os.path.join(args.dataset, "test.del"))
    else:
        n = args.synthetic or 100000
        allt = synthetic_triples(cfg, n + 2000, seed=args.model_seed)
        tr, va, te = allt[:n], allt[n:n + 1000], allt[n + 1000:]
    if args.enforce_random_keys:
        # entity / relation ids are labels: relabel them with a random permutation (keys = ids), the same on every rank
        fe = torch.from_numpy(id_permutation(cfg.num_entities, args.model_seed, True))
        fr = torch.from_numpy(id_permutation(cfg.num_relations, args.model_seed + 1, True))
        tr, va, te = (torch.stack([fe[t[:, 0]], fr[t[:, 1]], fe[t[:, 2]]], 1) for t in (tr, va, te))
    if args.eval_truncate_va:
        va = va[: args.eval_truncate_va]
    ad.setup(cfg.num_keys, 1)   # one worker per rank: the per-thread loops of the reference are batched kernels here
    server = ad.Server(cfg.value_lengths(), backend=args.backend, options=system_options(args),
                       dtype={"float": "float32", "double": "float64"}[args.value_type])
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model(init=args.init_parameters)
    rank, world = server.my_rank(), server.num_servers()
    if args.read_partitioned_dataset:
        n_blk = world * args.num_threads        # the file holds the blocks one after the other, equal sizes
        per = (tr.shape[0] + n_blk - 1) // n_blk
        mine = tr[rank * args.num_threads * per:(rank + 1) * args.num_threads * per]
    else:
        mine = tr[rank::world]                  # data parallelism: each worker trains on its partition
    if args.max_N >= 0:
        mine = mine[: args.max_N]
    if args.enforce_full_replication:
        enforce_full_replication(kv, cfg.num_keys)
    sync_push = wants_sync_push(args)
    known = torch.cat([tr, va, te])
    t0 = time.time()
    if args.eval_initial:
        ev = model.evaluate_distributed(va, known)      # collective: every rank ranks its share (kge.cc:555-709)
        if rank == 0:
            print(f"[kge] initial valid: {ev}", flush=True)
    for epoch in range(1, args.num_epochs + 1):
        perm = mine[torch.randperm(mine.shape[0], generator=torch.Generator().manual_seed(epoch * 977 + rank))]
        starts = list(range(0, perm.shape[0], cfg.batch_triples))
        if model.cuda:
            model.loss.zero_()
        bce = 0.0
        for j, f in enumerate(starts[:cfg.read_ahead]):       # prime the look-ahead window of this epoch
            model.signal_intent(perm[f:f + cfg.batch_triples], kv.current_clock() + j)
        for bi, s in enumerate(starts):
            if bi + cfg.read_ahead < len(starts):
                f = starts[bi + cfg.read_ahead]
                model.signal_intent(perm[f:f + cfg.batch_triples], kv.current_clock() + cfg.read_ahead)
            out = model.step(perm[s:s + cfg.batch_triples])
            if not model.cuda:
                bce += float(out)
            elif sync_push:
                torch.cuda.current_stream().synchronize()
            kv.advance_clock()
        if model.cuda:
            bce = float(model.loss.item())
        kv.barrier()
        total = ps_allreduce(kv, cfg.loss_key, torch.tensor([bce, 0.0]))     # loss all-reduce through the PS
        if rank == 0:
            kind = {"TransE": "margin", "RotatE": "self-adversarial"}.get(cfg.algorithm, "bce")
            kind = "cross-entropy" if cfg.train_type in ("1vsAll", "sampled_softmax") else kind
            print(f"[kge] epoch {epoch}: {kind} loss {float(total[0]):.4f} ({time.time() - t0:.1f}s)", flush=True)
        if args.eval_freq > 0 and epoch % args.eval_freq == 0:
            ev = model.evaluate_distributed(va, known)
            trn = model.evaluate_distributed(tr, known, truncate=args.eval_truncate_tr) if args.eval_truncate_tr else None
            if rank == 0:
                print(f"[kge] epoch {epoch} valid: {ev}" + (f" train: {trn}" if trn else ""), flush=True)
        if args.model_path and epoch % args.write_every == 0:
            model.save(args.model_path, epoch, write_checkpoint=bool(args.write_end_checkpoint) and epoch == args.num_epochs)
        if time.time() - t0 > args.max_runtime:
            break
    if rank == 0:
        if model.cuda and cfg.algorithm in ("ComplEx", "TransE", "RotatE") and cfg.embed_dim % 4 == 0:
            # fused gather + wgmma GEMM (ComplEx) or distance kernel (TransE, RotatE) + rank count: entity rows are read from
            # every GPU's HBM in-kernel
            print(f"[kge] test (fused gather-GEMM eval): {evaluate_fused(model, te, known)}", flush=True)
    ev = model.evaluate_distributed(te, known)
    if rank == 0:
        print(f"[kge] test: {ev}", flush=True)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
