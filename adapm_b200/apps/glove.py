"""GloVe application (Pennington et al., 2014): flag names follow glove.c's tools, with underscores.

    python -m adapm_b200.apps.glove --input_file corpus.txt --vector_size 100 --window_size 15 --iter 25
    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.glove -- --input_file corpus.txt --vector_size 48

Every rank builds (or loads) the vocabulary, encodes the whole corpus and counts the co-occurrence rows of its own
words (word w belongs to rank w % world); it then trains on them with the fused GloVe step. The vectors are written in
GloVe's text format (``word v1 ... vd``), ``W + C`` with ``--model 2`` and ``W`` with ``--model 1``.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import adapm_b200 as ad
from adapm_b200.apps._common import (add_ablation_options, add_system_options, enforce_full_replication, strip_dashes,
                                      system_options)
from adapm_b200.models.glove import GloVe, GloVeConfig
from adapm_b200.utils.text import NativeCorpus, Vocabulary


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--input_file", required=True, help="text corpus, one sentence per line")
    ap.add_argument("--vocab_save", default=None, help="write the vocabulary (word count per line) here")
    ap.add_argument("--vocab_retrieve", default=None, help="read the vocabulary from here instead of building it")
    ap.add_argument("--min_count", type=int, default=5)
    ap.add_argument("--window_size", type=int, default=15, help="context words on each side, at most 16")
    ap.add_argument("--symmetric", type=int, default=1, choices=[0, 1], help="1: count left and right context")
    ap.add_argument("--distance_weighting", type=int, default=1, choices=[0, 1],
                    help="1: a pair k words apart adds 1 / k; 0: it adds 1")
    ap.add_argument("--vector_size", type=int, default=100, help="a multiple of 4 in [4, 508]")
    ap.add_argument("--iter", type=int, default=25)
    ap.add_argument("--eta", type=float, default=0.05)
    ap.add_argument("--x_max", type=float, default=100.0)
    ap.add_argument("--alpha", type=float, default=0.75)
    ap.add_argument("--batch_entries", type=int, default=1 << 16, help="co-occurrence non-zeros per step")
    ap.add_argument("--read_ahead", type=int, default=2, help="batches of look-ahead for intent signalling")
    ap.add_argument("--model", type=int, default=2, choices=[1, 2], help="2: write W + C; 1: write W")
    ap.add_argument("--output_file", default="vectors.txt")
    ap.add_argument("--write_results", type=int, default=1, choices=[0, 1])
    ap.add_argument("--deterministic", type=int, default=0, choices=[0, 1],
                    help="one GPU: every non-zero of a batch reads the start-of-batch state, bit-identical runs")
    ap.add_argument("--model_seed", type=int, default=134827)
    ap.add_argument("--max_bytes", type=int, default=0,
                    help="device-memory budget of the co-occurrence count in bytes (0: the default, 8 GiB)")
    add_ablation_options(ap)
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if not 1 <= args.window_size <= 16:
        ap.error(f"--window_size must be in [1, 16], got {args.window_size}")
    if args.vector_size % 4 or not 4 <= args.vector_size <= 508:
        ap.error(f"--vector_size must be a multiple of 4 in [4, 508], got {args.vector_size}")
    if args.deterministic and world > 1:
        ap.error("--deterministic 1 needs a single GPU (WORLD_SIZE=1): on several GPUs rows move between ranks during a step")

    if args.vocab_retrieve:
        corpus = NativeCorpus.from_vocabulary(Vocabulary.load(args.vocab_retrieve))
    else:
        corpus = NativeCorpus.build(args.input_file, args.min_count)
    vocab = corpus.vocabulary()
    corpus.encode(args.input_file, 0, 1)                  # every rank counts its rows from the whole corpus
    cfg = GloVeConfig(vocab_size=len(vocab.words), embed_dim=args.vector_size, window=args.window_size,
                      symmetric=bool(args.symmetric), distance_weighting=bool(args.distance_weighting), eta=args.eta,
                      x_max=args.x_max, alpha=args.alpha, batch_entries=args.batch_entries, read_ahead=args.read_ahead,
                      deterministic=bool(args.deterministic), model_seed=args.model_seed, max_bytes=args.max_bytes or None)
    ad.setup(cfg.num_keys, 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    rank = server.my_rank()
    if args.vocab_save and rank == 0:
        vocab.save(args.vocab_save)
    model = GloVe(server, kv, cfg)
    model.init_model()
    t0 = time.time()
    nnz = model.build_cooccurrence(corpus)
    print(f"[glove] rank {rank}: {corpus.num_tokens()} tokens, vocabulary {cfg.vocab_size}, {nnz} non-zeros "
          f"(co-occurrence {time.time() - t0:.2f}s)", flush=True)
    if args.enforce_full_replication:
        enforce_full_replication(kv, cfg.num_keys)
    kv.barrier()
    total_nnz = server.allreduce_sum([float(nnz)])[0]
    for epoch in range(args.iter):
        t1 = time.time()
        loss = server.allreduce_sum([model.train_epoch(epoch)])[0]
        kv.barrier()
        if rank == 0:
            print(f"[glove] iter {epoch + 1}: cost {loss / max(1.0, total_nnz):.6f} ({time.time() - t1:.2f}s)", flush=True)
    if args.write_results:
        model.write_vectors(args.output_file, vocab.words, model=args.model)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
