"""Corpus handling for word2vec (reference apps/word2vec.cc:147-364: vocabulary building, sorting by
count, min_count pruning, frequent-word subsampling, per-worker file partitioning)."""
from __future__ import annotations

from collections import Counter
from dataclasses import dataclass
from typing import Iterator, List

import numpy as np
import torch


class Vocabulary:
    def __init__(self, words: List[str], counts: np.ndarray):
        self.words, self.counts = words, counts
        self.index = {w: i for i, w in enumerate(words)}

    @staticmethod
    def build(path: str, min_count: int = 5) -> "Vocabulary":
        c = Counter()
        with open(path, "r", errors="ignore") as f:
            for line in f:
                c.update(line.split())
        items = sorted(((w, n) for w, n in c.items() if n >= min_count), key=lambda t: -t[1])
        # like word2vec.c, index 0 is the sentence delimiter token
        words = ["</s>"] + [w for w, _ in items]
        counts = np.array([max(1, sum(1 for _ in open(path, errors="ignore")))] + [n for _, n in items], dtype=np.int64)
        return Vocabulary(words, counts)

    def save(self, path: str) -> None:
        with open(path, "w") as f:
            for w, n in zip(self.words, self.counts):
                f.write(f"{w} {int(n)}\n")

    @staticmethod
    def load(path: str) -> "Vocabulary":
        words, counts = [], []
        with open(path) as f:
            for line in f:
                w, n = line.rsplit(" ", 1)
                words.append(w); counts.append(int(n))
        return Vocabulary(words, np.array(counts, dtype=np.int64))


@dataclass
class HuffmanTree:
    """Huffman coding of a vocabulary for hierarchical softmax (:func:`huffman_tree`), as a CSR: word ``w``'s path is
    the inner nodes ``nodes[offsets[w]:offsets[w + 1]]`` (int32, root first; node ``n`` is the syn1 row
    ``2 n + 1``), and bit ``j`` of ``codes[w]`` (int32 holding the uint32 bit pattern) is its code bit at depth ``j``.
    ``max_len`` is the longest path."""
    offsets: torch.Tensor
    nodes: torch.Tensor
    codes: torch.Tensor
    max_len: int

    @property
    def num_words(self) -> int:
        return self.codes.numel()

    def to(self, device) -> "HuffmanTree":
        return HuffmanTree(self.offsets.to(device), self.nodes.to(device), self.codes.to(device), self.max_len)


def huffman_tree(counts) -> HuffmanTree:
    """Builds the Huffman tree of word2vec.c's ``CreateBinaryTree`` over ``counts`` (one positive count per word id, in
    any order), so that paths and codes match word2vec.c and gensim: words ordered by count (descending, ties by word
    id), the two-queue O(V) merge, inner nodes numbered ``0 .. V-2`` in creation order (the root is ``V-2``), code bit 1
    for the second-smallest child of each merge. Native (C++); raises ``ValueError`` for fewer than 2 words, a count
    that is not > 0, or a tree deeper than 32 levels."""
    from .. import _C

    c = np.asarray(counts, dtype=np.float64)
    if c.ndim != 1:
        raise ValueError(f"counts must be one-dimensional, got shape {c.shape}")
    off, nodes, codes, max_len = _C.huffman_tree(np.ascontiguousarray(c))
    return HuffmanTree(torch.from_numpy(off), torch.from_numpy(nodes), torch.from_numpy(codes.view(np.int32)),
                       int(max_len))


def read_sentences(path: str, vocab: Vocabulary, rank: int, world: int, subsample: float, rng) -> Iterator[np.ndarray]:
    """This rank's share of the corpus (line i belongs to rank i % world), as arrays of word ids with
    frequent-word subsampling (word2vec.c rule)."""
    total = float(vocab.counts.sum())
    with open(path, "r", errors="ignore") as f:
        for li, line in enumerate(f):
            if li % world != rank:
                continue
            ids = np.array([vocab.index[w] for w in line.split() if w in vocab.index], dtype=np.int64)
            if subsample > 0 and ids.size:
                fr = vocab.counts[ids] / total
                keep = (np.sqrt(fr / subsample) + 1) * subsample / fr
                ids = ids[rng.random(ids.size) < keep]
            if ids.size > 1:
                yield ids


def pairs_from_sentences(sentences: Iterator[np.ndarray], window: int, batch_pairs: int, rng) -> Iterator[torch.Tensor]:
    """(center, context) key batches [2, B]: for every position a random window shrink b in [0, window)
    like the reference (word2vec.cc:672-690); centers are syn0 keys of the context word, targets syn1 keys."""
    buf_c, buf_t, n = [], [], 0
    for s in sentences:
        L = s.size
        for pos in range(L):
            b = int(rng.integers(0, window))
            lo, hi = max(0, pos - (window - b)), min(L, pos + (window - b) + 1)
            ctx = np.concatenate([s[lo:pos], s[pos + 1:hi]])
            if ctx.size == 0:
                continue
            buf_c.append(2 * ctx)                                   # syn0 key of the context word
            buf_t.append(np.full(ctx.size, 2 * s[pos] + 1))         # syn1 key of the centre word
            n += ctx.size
            if n >= batch_pairs:
                c, t = np.concatenate(buf_c), np.concatenate(buf_t)
                yield torch.from_numpy(np.stack([c[:batch_pairs], t[:batch_pairs]]))
                buf_c, buf_t = [c[batch_pairs:]], [t[batch_pairs:]]
                n = buf_c[0].size
    if n:
        yield torch.from_numpy(np.stack([np.concatenate(buf_c), np.concatenate(buf_t)]))


def windows_from_sentences(sentences: Iterator[np.ndarray], window: int, batch_windows: int, rng) -> Iterator[torch.Tensor]:
    """CBOW window batches [batch_windows, 1 + 2 * window]: column 0 the syn1 key of the centre word, then the syn0 keys
    of its context words in sentence order, padded with -1. The window shrink is drawn like :func:`pairs_from_sentences`
    (same rng calls), so expanding the windows into (context, centre) pairs gives its pairs. A short last batch is padded
    with windows whose centre is -1; ``valid_windows`` of each batch tells how many are real."""
    if not 1 <= window <= 16:
        raise ValueError(f"window must be in [1, 16], got {window}")
    cols = 1 + 2 * window
    cur = np.full((batch_windows, cols), -1, dtype=np.int64)
    n = 0
    for s in sentences:
        L = s.size
        for pos in range(L):
            b = int(rng.integers(0, window))
            lo, hi = max(0, pos - (window - b)), min(L, pos + (window - b) + 1)
            ctx = np.concatenate([s[lo:pos], s[pos + 1:hi]])
            if ctx.size == 0:
                continue
            cur[n] = -1
            cur[n, 0] = 2 * s[pos] + 1                               # syn1 key of the centre word
            cur[n, 1:1 + ctx.size] = 2 * ctx                         # syn0 keys of the context words
            n += 1
            if n == batch_windows:
                t = torch.from_numpy(cur.copy())
                t.valid_windows = n
                yield t
                n = 0
    if n:
        cur[n:] = -1
        t = torch.from_numpy(cur.copy())
        t.valid_windows = n
        yield t


def cooccurrence_reference(sentences, vocab_size: int, window: int, symmetric: bool = True,
                           distance_weighting: bool = True, rank: int = 0, world: int = 1):
    """GloVe's co-occurrence matrix in numpy (the rule of ``ops.glove_cooccurrence``, its tests' oracle and the CPU
    backend's counter). ``sentences``: arrays of word ids in ``[0, vocab_size)``; windows never cross a sentence. For
    every pair of positions where word ``a`` comes ``k <= window`` positions before word ``b``, ``X[a][b] += 1 / k`` (1
    without ``distance_weighting``), with ``symmetric`` also ``X[b][a]``; only rows ``a % world == rank`` are kept.
    Numerators over ``lcm(1..window)`` are summed as int64 by packed key ``a * V + b`` and divided once (float64, then
    rounded to float32). Returns ``(rows int32, cols int32, x float32)`` sorted by ``(row, col)``."""
    if not 1 <= int(window) <= 16:
        raise ValueError(f"window must be in [1, 16], got {window}")
    V, window = int(vocab_size), int(window)
    lw = int(np.lcm.reduce(np.arange(1, window + 1))) if distance_weighting else 1
    sents = [np.asarray(s, dtype=np.int64) for s in sentences if len(s)]
    if not sents:
        e = np.zeros(0, np.int32)
        return e, e.copy(), np.zeros(0, np.float32)
    tok = np.concatenate(sents)
    sid = np.repeat(np.arange(len(sents)), [s.size for s in sents])
    keys, nums = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for k in range(1, min(window, tok.size - 1) + 1):
        same = sid[k:] == sid[:-k]
        a, b = tok[:-k][same], tok[k:][same]
        num = lw // k if distance_weighting else 1
        for r, c in ((a, b), (b, a)) if symmetric else ((a, b),):
            m = r % world == rank
            keys.append(r[m] * V + c[m])
            nums.append(np.full(int(m.sum()), num, dtype=np.int64))
    keys, nums = np.concatenate(keys), np.concatenate(nums)
    uniq, inv = np.unique(keys, return_inverse=True)
    sums = np.zeros(uniq.size, dtype=np.int64)
    if keys.size:
        order = np.argsort(inv, kind="stable")
        sums = np.add.reduceat(nums[order], np.searchsorted(inv[order], np.arange(uniq.size)))
    return (uniq // V).astype(np.int32), (uniq % V).astype(np.int32), (sums / lw).astype(np.float32)


# ------------------------------------------------------------------------------------------ native loader
class NativeCorpus:
    """C++ corpus (csrc/adapm/corpus.{h,cc}): same vocabulary rules as :class:`Vocabulary` (count-descending, ties by
    first occurrence, ``</s>`` = word 0), plus the encoded sentences of this rank and background generators of
    skip-gram pairs and CBOW windows."""

    def __init__(self, impl):
        self._impl = impl

    @staticmethod
    def build(path: str, min_count: int = 5) -> "NativeCorpus":
        from .. import _C

        return NativeCorpus(_C.Corpus.build(path, int(min_count)))

    @staticmethod
    def from_vocabulary(vocab: Vocabulary) -> "NativeCorpus":
        from .. import _C

        return NativeCorpus(_C.Corpus.from_vocab(list(vocab.words), [int(c) for c in vocab.counts]))

    def vocabulary(self) -> Vocabulary:
        return Vocabulary(list(self._impl.words()), np.array(self._impl.counts(), dtype=np.int64))

    def encode(self, path: str, rank: int = 0, world: int = 1) -> "NativeCorpus":
        self._impl.encode(path, int(rank), int(world))
        return self

    def num_tokens(self) -> int:
        return self._impl.num_tokens()

    def num_sentences(self) -> int:
        return self._impl.num_sentences()

    def sentences(self) -> List[np.ndarray]:
        """The encoded sentences (copies; for tests and small corpora)."""
        import ctypes

        n, ns = self.num_tokens(), self.num_sentences()
        tok = np.ctypeslib.as_array((ctypes.c_int32 * max(n, 1)).from_address(self._impl.tokens_ptr()))[:n].copy()
        off = np.ctypeslib.as_array((ctypes.c_int64 * (ns + 1)).from_address(self._impl.sentence_offsets_ptr())).copy()
        return [tok[off[i]:off[i + 1]] for i in range(ns)]

    def arrays(self):
        """The encoded sentences as ``(tokens int32 [n_tokens], offsets int64 [n_sentences + 1])`` numpy copies: sentence
        ``s`` is ``tokens[offsets[s]:offsets[s + 1]]`` (the input of ``ops.glove_cooccurrence``)."""
        import ctypes

        n, ns = self.num_tokens(), self.num_sentences()
        tok = np.ctypeslib.as_array((ctypes.c_int32 * max(n, 1)).from_address(self._impl.tokens_ptr()))[:n].copy()
        off = np.ctypeslib.as_array((ctypes.c_int64 * (ns + 1)).from_address(self._impl.sentence_offsets_ptr())).copy()
        return tok, off

    def sentence_lines(self) -> np.ndarray:
        """The 0-based file line of every encoded sentence (int64 numpy copy): lines without an in-vocabulary word are
        not sentences, so sentence ``s`` is line ``sentence_lines()[s]``, the document ``s`` of paragraph vectors."""
        import ctypes

        ns = self.num_sentences()
        return np.ctypeslib.as_array((ctypes.c_int64 * max(ns, 1)).from_address(self._impl.sentence_lines_ptr()))[:ns].copy()

    def num_lines(self) -> int:
        """Lines of the encoded file, every rank's: the number of documents."""
        return self._impl.num_lines()

    def pair_batches(self, window: int, subsample: float, batch_pairs: int, seed: int, epoch: int = 0,
                     pin: bool = False, queue_depth: int = 8) -> Iterator[torch.Tensor]:
        """[2, batch_pairs] key batches of one epoch, generated by a background C++ thread. A short final batch is
        padded by repeating its pairs; ``valid_pairs`` of the yielded tensor tells how many are real."""
        from .. import _C

        ps = _C.PairStream(self._impl, int(window), float(subsample), int(batch_pairs), int(seed), int(queue_depth))
        ps.start_epoch(int(epoch))
        while True:
            t = torch.empty(2, batch_pairs, dtype=torch.int64)
            if pin:
                t = t.pin_memory()
            u = torch.empty(2 * batch_pairs, dtype=torch.int64)
            valid, n_u = ps.next_with_unique(t.data_ptr(), u.data_ptr())
            if valid == 0:
                return
            t.valid_pairs = int(valid)
            t.unique_keys = u[:n_u]          # what to call Intent() with (deduplicated on the loader thread)
            yield t

    def window_batches(self, window: int, subsample: float, batch_windows: int, seed: int, epoch: int = 0,
                       pin: bool = False, queue_depth: int = 8) -> Iterator[torch.Tensor]:
        """CBOW window batches [batch_windows, 1 + 2 * window] of one epoch (layout of :func:`windows_from_sentences`),
        generated by a background C++ thread with the rng draws of :meth:`pair_batches`: for the same seed and epoch,
        expanding the windows into (context, centre) pairs gives its pairs. ``window <= 16``. A short final batch is
        padded with windows whose centre is -1; ``valid_windows`` tells how many are real, ``unique_keys`` holds the
        batch's distinct keys (for Intent)."""
        from .. import _C

        if not 1 <= window <= _C.window_stream_max_window:
            raise ValueError(f"window must be in [1, {_C.window_stream_max_window}], got {window}")
        ws = _C.WindowStream(self._impl, int(window), float(subsample), int(batch_windows), int(seed), int(queue_depth))
        ws.start_epoch(int(epoch))
        cols = ws.columns()
        while True:
            t = torch.empty(batch_windows, cols, dtype=torch.int64)
            if pin:
                t = t.pin_memory()
            u = torch.empty(batch_windows * cols, dtype=torch.int64)
            valid, n_u = ws.next_with_unique(t.data_ptr(), u.data_ptr())
            if valid == 0:
                return
            t.valid_windows = int(valid)
            t.unique_keys = u[:n_u]
            yield t

    def doc_pair_batches(self, window: int, subsample: float, batch_pairs: int, seed: int, dbow_words: bool,
                         epoch: int = 0, pin: bool = False, queue_depth: int = 8) -> Iterator[torch.Tensor]:
        """PV-DBOW key batches [2, batch_pairs] of one epoch (doc2vec), from a background C++ thread with the draws of
        :meth:`pair_batches`. Every walked position gives the pair ``(2 V + line, 2 w + 1)`` of its document's key and its
        word, followed with ``dbow_words`` by the position's skip-gram pairs as :meth:`pair_batches` emits them. A short
        final batch is padded by repeating its pairs; ``valid_pairs`` and ``unique_keys`` as for :meth:`pair_batches`."""
        from .. import _C

        ps = _C.DocPairStream(self._impl, int(window), float(subsample), int(batch_pairs), int(seed), bool(dbow_words),
                              int(queue_depth))
        ps.start_epoch(int(epoch))
        while True:
            t = torch.empty(2, batch_pairs, dtype=torch.int64)
            if pin:
                t = t.pin_memory()
            u = torch.empty(2 * batch_pairs, dtype=torch.int64)
            valid, n_u = ps.next_with_unique(t.data_ptr(), u.data_ptr())
            if valid == 0:
                return
            t.valid_pairs = int(valid)
            t.unique_keys = u[:n_u]
            yield t

    def doc_window_batches(self, window: int, subsample: float, batch_windows: int, seed: int, epoch: int = 0,
                           pin: bool = False, queue_depth: int = 8) -> Iterator[torch.Tensor]:
        """PV-DM window batches [batch_windows, 2 + 2 * window] of one epoch (doc2vec): the centre's syn1 key, the
        document's key ``2 V + line``, then the contexts as :meth:`window_batches` lays them out, with its draws.
        ``window <= 15``. Padding, ``valid_windows`` and ``unique_keys`` as for :meth:`window_batches`."""
        from .. import _C

        if not 1 <= window <= _C.doc_window_stream_max_window:
            raise ValueError(f"window must be in [1, {_C.doc_window_stream_max_window}], got {window}")
        ws = _C.DocWindowStream(self._impl, int(window), float(subsample), int(batch_windows), int(seed),
                                int(queue_depth))
        ws.start_epoch(int(epoch))
        cols = ws.columns()
        while True:
            t = torch.empty(batch_windows, cols, dtype=torch.int64)
            if pin:
                t = t.pin_memory()
            u = torch.empty(batch_windows * cols, dtype=torch.int64)
            valid, n_u = ws.next_with_unique(t.data_ptr(), u.data_ptr())
            if valid == 0:
                return
            t.valid_windows = int(valid)
            t.unique_keys = u[:n_u]
            yield t
