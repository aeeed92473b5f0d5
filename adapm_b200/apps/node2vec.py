"""node2vec / DeepWalk application (Grover and Leskovec, 2016): the flag names of the node2vec reference implementation,
with dashes or underscores.

    python -m adapm_b200.apps.node2vec --input graph.edgelist --output graph.emb --dimensions 128 --p 0.25 --q 4
    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.node2vec -- --input graph.edgelist --holdout 0.1

The input is a SNAP-style edge list (``src dst [weight]`` per line, ``#`` comments); ids may be sparse. Every rank
reads it and builds the same graph; each rank walks from its own nodes and trains the shared skip-gram model. The
vectors are written in word2vec's text format with the file's node ids. With ``--holdout FRACTION`` a seeded share of
the edges (both directions of an undirected edge) is left out of training, and the held-out link-prediction AUC
against as many sampled non-edges is printed after each epoch.
"""
from __future__ import annotations

import argparse
import sys
import time

import numpy as np

import adapm_b200 as ad
from adapm_b200.apps._common import (add_ablation_options, add_system_options, enforce_full_replication, strip_dashes,
                                      system_options)
from adapm_b200.models.node2vec import Node2Vec, Node2VecConfig, num_keys, sample_non_edges, split_edges
from adapm_b200.utils.graph import Graph, read_edge_list


def _flag(ap, name, **kw):
    ap.add_argument("--" + name, "--" + name.replace("-", "_"), dest=name.replace("-", "_"), **kw)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    _flag(ap, "input", required=True, help="edge list: 'src dst [weight]' per line")
    _flag(ap, "output", default="graph.emb", help="where the vectors go (word2vec text format)")
    _flag(ap, "dimensions", type=int, default=128)
    _flag(ap, "walk-length", type=int, default=80, help="nodes per walk, the start included")
    _flag(ap, "num-walks", type=int, default=10, help="walks from every node per epoch")
    _flag(ap, "window-size", type=int, default=10)
    _flag(ap, "iter", type=int, default=1, help="epochs")
    _flag(ap, "p", type=float, default=1.0, help="return parameter")
    _flag(ap, "q", type=float, default=1.0, help="in-out parameter")
    ap.add_argument("--weighted", dest="weighted", action="store_true", help="use the third column as edge weights")
    ap.add_argument("--unweighted", dest="weighted", action="store_false")
    ap.add_argument("--directed", dest="directed", action="store_true")
    ap.add_argument("--undirected", dest="directed", action="store_false")
    ap.set_defaults(weighted=False, directed=False)
    _flag(ap, "workers", type=int, default=1, help="accepted for compatibility: the ranks come from the launcher")
    _flag(ap, "negative", type=int, default=5)
    _flag(ap, "alpha", type=float, default=0.025, help="starting learning rate")
    _flag(ap, "batch-pairs", type=int, default=32768, help="skip-gram pairs per step")
    _flag(ap, "walkers-per-chunk", type=int, default=4096, help="walks generated at a time")
    _flag(ap, "holdout", type=float, default=0.0, help="share of the edges held out for link prediction")
    _flag(ap, "model-seed", type=int, default=134827)
    add_ablation_options(ap)
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    if not 0.0 <= args.holdout < 1.0:
        ap.error(f"--holdout must be in [0, 1), got {args.holdout}")
    if args.p <= 0 or args.q <= 0:
        ap.error(f"--p and --q must be positive, got {args.p}, {args.q}")

    src, dst, weight, ids = read_edge_list(args.input)
    if args.weighted and weight is None:
        ap.error("--weighted needs a weight column in the edge list")
    held = non_edges = None
    if args.holdout > 0:
        src, dst, kept, held = split_edges(src, dst, args.holdout, args.directed, args.model_seed)
        weight = weight[kept] if weight is not None else None
        non_edges = sample_non_edges(np.concatenate([src, held[0]]), np.concatenate([dst, held[1]]), ids.size,
                                     held.shape[1], args.directed, args.model_seed + 1)
    graph = Graph.from_edges(src, dst, weight if args.weighted else None, args.directed, num_nodes=ids.size)
    graph.node_ids = ids
    cfg = Node2VecConfig(dimensions=args.dimensions, walk_length=args.walk_length, num_walks=args.num_walks,
                         window=args.window_size, p=args.p, q=args.q, negative=args.negative,
                         batch_pairs=args.batch_pairs, iter=args.iter, alpha=args.alpha,
                         walkers_per_chunk=args.walkers_per_chunk, model_seed=args.model_seed)
    ad.setup(num_keys(graph.num_nodes), 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    rank = server.my_rank()
    model = Node2Vec(server, kv, graph, cfg)
    model.init_model()
    if rank == 0:
        print(f"[node2vec] {graph.num_nodes} nodes, {graph.num_edges} stored edges"
              f"{f', {held.shape[1]} held out' if held is not None else ''}, world {server.num_servers()}", flush=True)
    if args.enforce_full_replication:
        enforce_full_replication(kv, num_keys(graph.num_nodes))
    kv.barrier()
    for epoch in range(args.iter):
        t0 = time.time()
        loss, pairs = server.allreduce_sum(list(model.train_epoch(epoch)))
        kv.barrier()
        line = f"[node2vec] epoch {epoch + 1}: loss {loss / max(1.0, pairs * (cfg.negative + 1)):.6f}, {int(pairs)} pairs"
        if held is not None:
            kv.wait_sync()
            if rank == 0:
                line += f", held-out AUC {model.link_prediction_auc(held, non_edges):.4f}"
            kv.barrier()
        if rank == 0:
            print(f"{line} ({time.time() - t0:.2f}s)", flush=True)
    model.write_vectors(args.output)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
