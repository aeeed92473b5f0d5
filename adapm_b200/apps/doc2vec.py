"""Paragraph-vector (doc2vec) application: word2vec's flag names plus ``--dm``, ``--dbow_words`` and inference flags.

    python -m adapm_b200.apps.doc2vec --input_file docs.txt --doc_output_file docs.bin --dm 0 --dbow_words 1
    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.doc2vec -- --input_file docs.txt --infer_file new.txt \\
        --infer_output_file new.bin

Every line of the input file is one document; document ``j`` is line ``j`` (0-based), and rank ``r`` trains the lines
``r, r + world, ...``. Word vectors go to ``--output_file`` and document vectors to ``--doc_output_file``, both in
word2vec's binary format (documents named by their line index). With ``--infer_file`` rank 0 infers a vector for every
line of that file against the trained word rows and writes them to ``--infer_output_file`` (named by line index).
"""
from __future__ import annotations

import argparse
import sys
import time

import adapm_b200 as ad
from adapm_b200.apps._common import add_system_options, strip_dashes, system_options
from adapm_b200.models.doc2vec import Doc2Vec, Doc2VecConfig, num_keys, write_vectors_binary
from adapm_b200.utils.text import NativeCorpus


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--input_file", "-f", required=True, help="one document per line")
    ap.add_argument("--output_file", "-o", default="vectors.bin", help="word vectors (binary word2vec format)")
    ap.add_argument("--doc_output_file", default="docvectors.bin", help="document vectors, named by line index")
    ap.add_argument("--num_iterations", "-i", type=int, default=10)
    ap.add_argument("--window", "-w", type=int, default=5)
    ap.add_argument("--embed_dim", "-v", type=int, default=100)
    ap.add_argument("--negative", type=int, default=5)
    ap.add_argument("--min_count", type=int, default=5)
    ap.add_argument("--starting_alpha", type=float, default=0.025)
    ap.add_argument("--min_alpha", type=float, default=0.0001)
    ap.add_argument("--subsample", type=float, default=1e-3)
    ap.add_argument("--read_sentences_ahead", type=int, default=4, help="batches of look-ahead for intent signalling")
    ap.add_argument("--signal_intent", type=int, default=1)
    ap.add_argument("--model_seed", type=int, default=134827)
    ap.add_argument("--batch_pairs", type=int, default=32768, help="PV-DBOW: pairs per step")
    ap.add_argument("--batch_windows", type=int, default=8192, help="PV-DM: windows per step")
    ap.add_argument("--dm", type=int, default=0, choices=[0, 1],
                    help="1 = PV-DM (the mean of the document and context rows); 0 = PV-DBOW")
    ap.add_argument("--dbow_words", type=int, default=0, choices=[0, 1],
                    help="PV-DBOW: also train skip-gram word pairs in the same batches")
    ap.add_argument("--infer_file", default=None, help="documents to infer vectors for, one per line")
    ap.add_argument("--infer_output_file", default=None)
    ap.add_argument("--infer_epochs", type=int, default=20)
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))
    if args.negative < 1:
        ap.error(f"--negative must be at least 1, got {args.negative}")
    if args.dm and not 1 <= args.window <= 15:
        ap.error(f"--window must be in [1, 15] with --dm 1, got {args.window}")
    if args.infer_file and not args.infer_output_file:
        ap.error("--infer_file needs --infer_output_file")
    if args.num_iterations < 1 or args.infer_epochs < 1:
        ap.error("--num_iterations and --infer_epochs must be at least 1")

    corpus = NativeCorpus.build(args.input_file, args.min_count)
    vocab = corpus.vocabulary()
    cfg = Doc2VecConfig(dm=args.dm, dbow_words=args.dbow_words, embed_dim=args.embed_dim, window=args.window,
                        negative=args.negative, alpha=args.starting_alpha, min_alpha=args.min_alpha,
                        epochs=args.num_iterations, batch_pairs=args.batch_pairs, batch_windows=args.batch_windows,
                        subsample=args.subsample, model_seed=args.model_seed, read_ahead=args.read_sentences_ahead,
                        signal_intent=bool(args.signal_intent), infer_epochs=args.infer_epochs,
                        infer_alpha=args.starting_alpha, infer_min_alpha=args.min_alpha)
    with open(args.input_file, "rb") as f:        # the documents, counted as the native encoder counts lines
        n_docs = sum(1 for _ in f)
    ad.setup(num_keys(len(vocab.words), n_docs), 1)
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    rank, world = server.my_rank(), server.num_servers()
    corpus.encode(args.input_file, rank, world)
    model = Doc2Vec(server, kv, cfg, corpus)
    model.init_model()
    if rank == 0:
        print(f"[d2v] {len(vocab.words)} words, {model.num_docs} documents, {'PV-DM' if cfg.dm else 'PV-DBOW'}, "
              f"world {world}", flush=True)
    kv.barrier()
    t0 = time.time()
    for epoch in range(cfg.epochs):
        loss, items = server.allreduce_sum(list(model.train_epoch(epoch)))
        kv.barrier()
        if rank == 0:
            unit = "windows" if cfg.dm else "pairs"
            print(f"[d2v] epoch {epoch} done: loss {loss / max(1.0, items * (cfg.negative + 1)):.6f}, {int(items)} "
                  f"{unit}, {time.time() - t0:.1f}s", flush=True)
    model.write_checkpoint(args.output_file, args.doc_output_file, vocab.words)
    if args.infer_file:
        kv.wait_sync()
        if rank == 0:
            with open(args.infer_file, errors="ignore") as f:
                docs = [line.split() for line in f]
            vecs = model.infer(docs).cpu().numpy()
            write_vectors_binary(args.infer_output_file, [str(j) for j in range(len(docs))], vecs)
            print(f"[d2v] inferred {len(docs)} documents ({cfg.infer_epochs} epochs each)", flush=True)
    kv.barrier()
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
