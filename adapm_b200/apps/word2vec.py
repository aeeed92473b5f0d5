"""word2vec application (reference apps/word2vec.cc), flags keep the reference's names.

    python -m adapm_b200.launch -s 2 -m adapm_b200.apps.word2vec -- --input_file corpus.txt --embed_dim 100 ...
    python -m adapm_b200.apps.word2vec --synthetic_vocab 100000 --num_iterations 1     (synthetic Zipf corpus)
"""
from __future__ import annotations

import argparse
import sys
import time

import numpy as np
import torch

import adapm_b200 as ad
from adapm_b200.apps._common import (add_ablation_options, add_system_options, enforce_full_replication, id_permutation,
                                      strip_dashes, system_options, wants_sync_push)
from adapm_b200.models.word2vec import (SyntheticPairs, SyntheticWindows, Word2Vec, Word2VecConfig, load_checkpoint,
                                        syn0_key, syn1_key, zipf_counts)
from adapm_b200.utils.text import (NativeCorpus, Vocabulary, pairs_from_sentences, read_sentences,
                                   windows_from_sentences)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--num_threads", "-t", type=int, default=1)
    ap.add_argument("--num_iterations", "-i", type=int, default=15)
    ap.add_argument("--input_file", "-f", default=None)
    ap.add_argument("--output_file", "-o", default="vectors.bin")
    ap.add_argument("--vocab_save", default=None)
    ap.add_argument("--vocab_retrieve", default=None)
    ap.add_argument("--window", "-w", type=int, default=5)
    ap.add_argument("--embed_dim", "-v", type=int, default=200)
    ap.add_argument("--negative", type=int, default=25)
    ap.add_argument("--shared_negatives", type=int, default=0,
                    help="> 0 = one set of this many negatives per batch (cuda: contractions on the tensor cores, a multiple "
                         "of 32, batch_pairs too; cpu: the same rule through Pull / Push); 0 = the reference's private negatives")
    ap.add_argument("--min_count", type=int, default=5)
    ap.add_argument("--neg_power", type=float, default=0.75)
    ap.add_argument("--starting_alpha", type=float, default=0.025)
    ap.add_argument("--subsample", type=float, default=1e-4)
    ap.add_argument("--read_sentences_ahead", type=int, default=4, help="batches of look-ahead for intent signalling")
    ap.add_argument("--signal_intent", type=int, default=1)
    ap.add_argument("--write_results", type=int, default=0)
    ap.add_argument("--binary", type=int, default=1)
    ap.add_argument("--model_seed", type=int, default=134827)
    ap.add_argument("--max_runtime", type=float, default=float("inf"))
    ap.add_argument("--batch_pairs", type=int, default=32768)
    ap.add_argument("--cbow", type=int, default=0, choices=[0, 1],
                    help="1 = continuous bag of words (word2vec.c's -cbow 1): one window per corpus word, the mean of the "
                         "context rows scored against the centre and the negatives; 0 = skip-gram (window <= 16 for CBOW)")
    ap.add_argument("--batch_windows", type=int, default=8192, help="CBOW: windows per step")
    ap.add_argument("--hs", type=int, default=0, choices=[0, 1],
                    help="1 = hierarchical softmax (word2vec.c's -hs 1): each item is scored against the inner nodes on "
                         "the Huffman path of its word instead of negatives; needs --negative 0")
    ap.add_argument("--synthetic_vocab", type=int, default=0, help="train on a synthetic Zipf corpus of this vocabulary size")
    ap.add_argument("--synthetic_batches", type=int, default=50)
    ap.add_argument("--init_model", default="random",
                    help="'random' (syn0 ~ U(-.5,.5)/d, syn1 = 0), 'none', or the path of a checkpoint written with "
                         "--write_results (its .syn1 companion is used when present)")
    ap.add_argument("--data_words", type=int, default=0, help="stop an epoch after this many training pairs per rank (0: all)")
    ap.add_argument("--clustered_input", type=int, default=0,
                    help="accepted for parity: the loader always gives rank r the lines r, r + world, ...")
    ap.add_argument("--debug_mode", "-d", type=int, default=0)
    ap.add_argument("--num_keys", "-k", type=int, default=0, help="accepted for parity (derived from the vocabulary: 2 * |V|)")
    add_ablation_options(ap)
    ap.add_argument("--loader", default="native", choices=["native", "python"],
                    help="native: C++ vocabulary / encoder / background pair generator (csrc/adapm/corpus.cc); "
                         "python: the numpy reference implementation (utils/text.py)")
    add_system_options(ap)
    args = ap.parse_args(strip_dashes(argv if argv is not None else sys.argv[1:]))

    if args.cbow and args.shared_negatives > 0:
        raise ValueError("--shared_negatives is a skip-gram option: it cannot be combined with --cbow 1")
    if args.hs and (args.negative > 0 or args.shared_negatives > 0):
        raise ValueError("--hs 1 with negative sampling is not supported: run hierarchical softmax with --negative 0 "
                         "and without --shared_negatives")
    rng = np.random.default_rng(args.model_seed)
    words = None
    native = None
    if args.input_file:
        if args.vocab_retrieve:
            vocab = Vocabulary.load(args.vocab_retrieve)
            if args.loader == "native":
                native = NativeCorpus.from_vocabulary(vocab)
        elif args.loader == "native":
            native = NativeCorpus.build(args.input_file, args.min_count)
            vocab = native.vocabulary()
        else:
            vocab = Vocabulary.build(args.input_file, args.min_count)
        if args.vocab_save:
            vocab.save(args.vocab_save)
        if args.enforce_random_keys:
            # word ids are labels: shuffling the vocabulary order assigns the keys 2*id / 2*id+1 randomly
            fw = id_permutation(len(vocab.words), args.model_seed, True)
            sw, sc = [None] * len(fw), np.empty_like(vocab.counts)
            for i, j in enumerate(fw):
                sw[j], sc[j] = vocab.words[i], vocab.counts[i]
            vocab = Vocabulary(sw, sc)
            if native is not None:
                native = NativeCorpus.from_vocabulary(vocab)
        counts, words = vocab.counts.astype(np.float64), vocab.words
        V = len(words)
    else:
        V = args.synthetic_vocab or 100000
        counts = zipf_counts(V)
    cfg = Word2VecConfig(vocab_size=V, embed_dim=args.embed_dim, negative=args.negative, window=args.window,
                         starting_alpha=args.starting_alpha, neg_power=args.neg_power, batch_pairs=args.batch_pairs,
                         read_ahead=args.read_sentences_ahead, signal_intent=bool(args.signal_intent),
                         sampling_scheme=getattr(args, "sampling.scheme") or "local", model_seed=args.model_seed,
                         shared_negatives=args.shared_negatives, cbow=bool(args.cbow), batch_windows=args.batch_windows,
                         hs=bool(args.hs))
    ad.setup(cfg.num_keys, 1)   # one worker per rank: the per-thread loops of the reference are batched kernels here
    server = ad.Server(cfg.row_len, backend=args.backend, options=system_options(args))
    kv = ad.Worker(0, server)
    model = Word2Vec(server, kv, cfg, counts)
    if args.init_model == "random":
        model.init_model()
    elif args.init_model != "none":
        model.init_model()                                  # words that are not in the checkpoint start randomly
        n = load_checkpoint(model, args.init_model, words)
        if server.my_rank() == 0:
            print(f"[w2v] initialised {n} of {V} words from {args.init_model}", flush=True)
    if args.enforce_full_replication:
        enforce_full_replication(kv, cfg.num_keys)
    sync_push = wants_sync_push(args)
    rank, world = server.my_rank(), server.num_servers()

    if args.input_file and native is not None:
        native.encode(args.input_file, rank, world)      # this rank's share of the lines, as word ids

    def batches(epoch):
        if cfg.cbow:
            if args.input_file and native is not None:
                yield from native.window_batches(args.window, args.subsample, cfg.batch_windows, args.model_seed + rank,
                                                 epoch, pin=model.cuda)
            elif args.input_file:
                sents = read_sentences(args.input_file, vocab, rank, world, args.subsample, rng)
                yield from windows_from_sentences(sents, args.window, cfg.batch_windows, rng)
            else:
                data = SyntheticWindows(cfg, counts, rank, seed=epoch + 1)
                for s in range(args.synthetic_batches):
                    yield data.batch(s)
            return
        if args.input_file and native is not None:
            yield from native.pair_batches(args.window, args.subsample, cfg.batch_pairs, args.model_seed + rank, epoch,
                                           pin=model.cuda)
        elif args.input_file:
            sents = read_sentences(args.input_file, vocab, rank, world, args.subsample, rng)
            yield from pairs_from_sentences(sents, args.window, cfg.batch_pairs, rng)
        else:
            data = SyntheticPairs(cfg, counts, rank, seed=epoch + 1)
            for s in range(args.synthetic_batches):
                yield data.batch(s)

    t0 = time.time()
    total_pairs, est_total = 0, None
    for epoch in range(args.num_iterations):
        it = batches(epoch)
        window = []
        epoch_pairs = 0
        for b in it:
            window.append(b)
            if len(window) <= cfg.read_ahead:
                model.signal_intent(b, kv.current_clock() + len(window) - 1)
                continue
            model.signal_intent(b, kv.current_clock() + cfg.read_ahead)
            cur = window.pop(0)
            if model.cuda:
                model.loss.zero_()
            last = _full(cur, cfg, model.cuda)
            loss = model.step(last)
            if sync_push and model.cuda:
                torch.cuda.current_stream().synchronize()
            kv.advance_clock()
            total_pairs += _items(cur, cfg)
            epoch_pairs += _items(cur, cfg)
            if time.time() - t0 > args.max_runtime or (args.data_words and epoch_pairs >= args.data_words):
                break
        for cur in window:
            if model.cuda:
                model.loss.zero_()
            last = _full(cur, cfg, model.cuda)
            loss = model.step(last)
            kv.advance_clock()
            total_pairs += _items(cur, cfg)
        model.set_alpha((epoch + 1) / args.num_iterations)
        kv.barrier()
        if rank == 0:
            unit, per_step = ("windows", cfg.batch_windows) if cfg.cbow else ("pairs", cfg.batch_pairs)
            # (hierarchical softmax: per path node of the last batch's items)
            terms = model.loss_terms(last) if cfg.hs else per_step * (cfg.negative + 1)
            print(f"[w2v] epoch {epoch} done: {total_pairs} {unit} on rank 0, {time.time() - t0:.1f}s, "
                  f"last batch loss {float(loss) / max(1, terms):.4f}", flush=True)
        if args.write_results:
            model.write_checkpoint(f"{args.output_file}.epoch.{epoch}", words)
    kv.finalize()
    if rank == 0:
        print(server.stats(), flush=True)
    server.shutdown()
    return 0


def _items(b: torch.Tensor, cfg) -> int:
    """real pairs / windows of a batch"""
    if cfg.cbow:
        return getattr(b, "valid_windows", b.shape[0])
    return getattr(b, "valid_pairs", b.shape[1])


def _full(b: torch.Tensor, cfg, cuda: bool) -> torch.Tensor:
    """the batch at the fixed size of the fused kernel (window batches are padded by their loaders)"""
    if cfg.cbow or not cuda or b.shape[1] == cfg.batch_pairs:
        return b
    return _pad(b, cfg.batch_pairs)


def _pad(b: torch.Tensor, n: int) -> torch.Tensor:
    """pad a short final batch by repeating pairs (the fused kernel works on fixed-size batches)."""
    reps = (n + b.shape[1] - 1) // b.shape[1]
    return b.repeat(1, reps)[:, :n].contiguous()


if __name__ == "__main__":
    sys.exit(main())
