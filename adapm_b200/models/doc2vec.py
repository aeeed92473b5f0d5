"""Paragraph vectors (Le and Mikolov, 2014; gensim's Doc2Vec) on the parameter store: PV-DBOW and PV-DM with negative
sampling, trained on the fused word2vec steps, and inference of vectors for new documents on the device.

Keys extend word2vec's: word ``w`` keeps ``syn0 = 2 w`` and ``syn1 = 2 w + 1``, and document ``j`` (line ``j`` of the
corpus file, 0-based) is key ``doc_key(j) = 2 V + j``, a row ``[embedding | AdaGrad]`` like the others. Document rows
start like syn0 rows, ``U(-0.5, 0.5) / d`` with accumulators 1e-6. Negatives are drawn over the syn1 word keys only
(weights ``count^0.75``), so a document key is never a negative.

- PV-DBOW (``dm=0``) is skip-gram whose input row is the document's: the native ``DocPairStream`` emits ``(doc key,
  syn1 word)`` for every walked position, and with ``dbow_words`` the position's skip-gram word pairs after it. The
  batches run through ``ops.sgns_step``.
- PV-DM (``dm=1``, mean) is CBOW with the document's row as one more context: ``DocWindowStream`` windows ``[centre
  syn1, doc key, contexts]`` run through ``ops.cbow_step``, so ``1 + 2 window <= 32`` contexts and ``window <= 15``.

Both are the unchanged steps of an owned :class:`Word2Vec`, deterministic on one GPU as they are; the CPU backend runs
the same batches through ``sgns_reference_step`` / ``cbow_reference_step``. The learning rate falls linearly from
``alpha`` to ``min_alpha`` over the epochs. Inference (``ops.doc2vec_infer``; ``ops.doc2vec_infer_reference`` on the
CPU backend) trains one new vector per document against the frozen word rows.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .word2vec import Word2Vec, Word2VecConfig


@dataclass
class Doc2VecConfig:
    dm: int = 0                      # 0 = PV-DBOW, 1 = PV-DM (mean of the document and context rows)
    dbow_words: int = 0              # PV-DBOW: also train skip-gram word pairs in the same batches
    embed_dim: int = 100
    window: int = 5
    negative: int = 5
    alpha: float = 0.025
    min_alpha: float = 0.0001
    epochs: int = 10
    batch_pairs: int = 32768         # PV-DBOW pairs per step
    batch_windows: int = 8192        # PV-DM windows per step
    subsample: float = 1e-3
    model_seed: int = 134827
    read_ahead: int = 4              # batches of look-ahead for intent signalling
    signal_intent: bool = True
    hs: bool = False                 # hierarchical softmax: not supported for documents
    infer_epochs: int = 20
    infer_alpha: float = 0.025
    infer_min_alpha: float = 0.0001

    @property
    def row_len(self) -> int:
        return 2 * self.embed_dim


def num_keys(vocab_size: int, num_docs: int) -> int:
    return 2 * int(vocab_size) + int(num_docs)


class Doc2Vec:
    """``corpus``: a :class:`adapm_b200.utils.text.NativeCorpus` encoded for this rank (``encode(path, rank, world)``);
    its file's lines are the documents. The store needs ``num_keys(V, corpus.num_lines())`` keys of ``row_len``."""

    def __init__(self, server, worker, cfg: Doc2VecConfig, corpus, counts: Optional[np.ndarray] = None):
        if cfg.hs:
            raise ValueError("hierarchical softmax is not supported for paragraph vectors: use negative sampling")
        if cfg.negative < 1:
            raise ValueError(f"negative must be at least 1, got {cfg.negative}")
        if cfg.dm not in (0, 1) or cfg.dbow_words not in (0, 1):
            raise ValueError("dm and dbow_words must be 0 or 1")
        if cfg.dm and not 1 <= cfg.window <= 15:
            raise ValueError(f"PV-DM needs window in [1, 15] (the document and 2 window contexts <= 32), got {cfg.window}")
        if cfg.window < 1 or cfg.epochs < 1 or cfg.infer_epochs < 1:
            raise ValueError("window, epochs and infer_epochs must be at least 1")
        if not (0 < cfg.min_alpha <= cfg.alpha and 0 < cfg.infer_min_alpha <= cfg.infer_alpha):
            raise ValueError("need 0 < min_alpha <= alpha and 0 < infer_min_alpha <= infer_alpha")
        self.server, self.worker, self.cfg, self.corpus = server, worker, cfg, corpus
        self.vocab_size = int(corpus._impl.vocab_size())
        self.num_docs = corpus.num_lines()
        if server.num_keys() < num_keys(self.vocab_size, self.num_docs):
            raise ValueError(f"the store has {server.num_keys()} keys, paragraph vectors need "
                             f"{num_keys(self.vocab_size, self.num_docs)} (2 V + documents)")
        if counts is None:
            counts = np.asarray(corpus._impl.counts(), dtype=np.float64)
        self.w2v = Word2Vec(server, worker, Word2VecConfig(
            vocab_size=self.vocab_size, embed_dim=cfg.embed_dim, negative=cfg.negative, window=cfg.window,
            starting_alpha=cfg.alpha, batch_pairs=cfg.batch_pairs, read_ahead=cfg.read_ahead,
            signal_intent=cfg.signal_intent, model_seed=cfg.model_seed, cbow=bool(cfg.dm),
            batch_windows=cfg.batch_windows), counts)
        self.cuda = self.w2v.cuda
        self.dev = server.device
        if not self.cuda:               # the draw tables of inference, as the device sampler builds them
            from ..ops import DeviceSampler

            self.sampler = DeviceSampler(server, weights=torch.from_numpy(np.power(counts, 0.75)), first_key=1,
                                         key_stride=2)
        else:
            self.sampler = self.w2v.sampler

    def doc_key(self, j):
        return 2 * self.vocab_size + j

    # ------------------------------------------------------------------ model init
    def init_model(self, chunk: int = 1 << 16) -> None:
        """Word rows as word2vec initialises them, then each rank sets the document keys it is home for."""
        self.w2v.init_model()
        cfg, world, rank, d = self.cfg, self.server.num_servers(), self.server.my_rank(), self.cfg.embed_dim
        gen = torch.Generator(device=self.dev.type).manual_seed(cfg.model_seed * 7919 + 1 + rank)
        first = self.doc_key(0)
        keys_all = torch.arange(first + (rank - first) % world, first + self.num_docs, world, dtype=torch.int64)
        self.worker.begin_setup()
        for i in range(0, keys_all.numel(), chunk):
            k = keys_all[i:i + chunk].to(self.dev)
            rows = torch.empty(k.numel(), 2 * d, dtype=torch.float32, device=self.dev)
            rows[:, d:] = 1e-6
            rows[:, :d] = (torch.rand(k.numel(), d, generator=gen, device=self.dev, dtype=torch.float32) - 0.5) / d
            self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    # ------------------------------------------------------------------ training
    def epoch_alpha(self, epoch: int) -> float:
        cfg = self.cfg
        return cfg.alpha - epoch * (cfg.alpha - cfg.min_alpha) / max(1, cfg.epochs - 1)

    def batches(self, epoch: int):
        cfg, seed = self.cfg, self.cfg.model_seed + self.server.my_rank()
        if cfg.dm:
            return self.corpus.doc_window_batches(cfg.window, cfg.subsample, cfg.batch_windows, seed, epoch, pin=self.cuda)
        return self.corpus.doc_pair_batches(cfg.window, cfg.subsample, cfg.batch_pairs, seed, bool(cfg.dbow_words),
                                            epoch, pin=self.cuda)

    def train_epoch(self, epoch: int):
        """One epoch of this rank's documents, one clock per step; the intents of a batch are signalled ``read_ahead``
        steps ahead with its distinct keys (its document keys included). Returns ``(summed loss, items)``: items are
        pairs (PV-DBOW) or windows (PV-DM), and the loss sums ``negative + 1`` terms per item."""
        cfg, kv, w2v = self.cfg, self.worker, self.w2v
        w2v.alpha = self.epoch_alpha(epoch)
        if self.cuda:
            w2v.loss.zero_()
        loss, items = 0.0, 0
        ahead = []

        def run(b):
            nonlocal loss, items
            valid = getattr(b, "valid_windows", None) if cfg.dm else getattr(b, "valid_pairs", None)
            if self.cuda:
                w2v.step_resident(b.to(self.dev, non_blocking=True))
            else:
                loss += float(w2v.step(b[:valid] if cfg.dm else b[:, :valid].contiguous()))
            kv.advance_clock()
            items += int(valid)

        for b in self.batches(epoch):
            ahead.append(b)
            w2v.signal_intent(b, kv.current_clock() + len(ahead) - 1)
            if len(ahead) > cfg.read_ahead:
                run(ahead.pop(0))
        for b in ahead:
            run(b)
        if self.cuda:
            loss = float(w2v.loss.item())
        return loss, items

    def train(self, epochs: Optional[int] = None):
        return [self.train_epoch(e) for e in range(self.cfg.epochs if epochs is None else epochs)]

    # ------------------------------------------------------------------ inference
    def encode(self, docs):
        """(tokens int64, offsets int64) of ``docs``: sequences of word ids, or of words (unknown ones are dropped)."""
        ids = []
        for doc in docs:
            if isinstance(doc, str):
                doc = doc.split()
            w = [self.corpus._impl.lookup(t) if isinstance(t, str) else int(t) for t in doc]
            ids.append(np.asarray([x for x in w if x >= 0], dtype=np.int64))
        lens = np.array([x.size for x in ids], dtype=np.int64)
        offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        tokens = np.concatenate(ids) if ids else np.zeros(0, dtype=np.int64)
        return torch.from_numpy(tokens.astype(np.int64)), torch.from_numpy(offsets)

    def infer(self, docs, doc_ids=None, seed: Optional[int] = None, loss: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Vectors (float32 ``[len(docs), d]``, on the server's device) for documents that need not be in the training
        data: each is trained ``infer_epochs`` times over its words against the frozen word rows, from ``infer_alpha``
        down to ``infer_min_alpha`` (``ops.doc2vec_infer``). ``docs``: strings, lists of words or lists of word ids.
        ``doc_ids`` (default ``0 .. n-1``) and ``seed`` (default ``model_seed``) pick each document's starting vector
        and draws, so a document's vector does not depend on the other documents of the call."""
        from ..ops import doc2vec_infer, doc2vec_infer_reference

        cfg = self.cfg
        tokens, offsets = self.encode(docs)
        ids = torch.arange(offsets.numel() - 1, dtype=torch.int64) if doc_ids is None else \
            torch.as_tensor(np.asarray(doc_ids), dtype=torch.int64).reshape(-1)
        kw = dict(dm=bool(cfg.dm), embed_dim=cfg.embed_dim, negative=cfg.negative, window=cfg.window,
                  epochs=cfg.infer_epochs, alpha=cfg.infer_alpha, min_alpha=cfg.infer_min_alpha,
                  seed=cfg.model_seed if seed is None else int(seed), num_words=self.vocab_size)
        if self.cuda:
            return doc2vec_infer(self.server, tokens, offsets, ids, self.sampler, loss=loss, **kw)
        v, total = doc2vec_infer_reference(self.worker, tokens, offsets, ids, self.sampler, **kw)
        if loss is not None:
            loss += total
        return torch.from_numpy(v.astype(np.float32))

    # ------------------------------------------------------------------ retrieval
    def doc_vectors(self, docs=None, chunk: int = 1 << 16) -> torch.Tensor:
        """The trained vectors of documents ``docs`` (default: all), float32 ``[n, d]`` on the server's device."""
        d, kv = self.cfg.embed_dim, self.worker
        j = torch.arange(self.num_docs, dtype=torch.int64) if docs is None else \
            torch.as_tensor(np.asarray(docs), dtype=torch.int64).reshape(-1)
        if j.numel() and (int(j.min()) < 0 or int(j.max()) >= self.num_docs):
            raise ValueError(f"document ids must be in [0, {self.num_docs})")
        out = torch.empty(j.numel(), d, dtype=torch.float32, device=self.dev)
        for i in range(0, j.numel(), chunk):
            k = self.doc_key(j[i:i + chunk]).to(self.dev)
            rows = torch.empty(k.numel() * 2 * d, dtype=torch.float32, device=self.dev)
            kv.wait(kv.pull(k, rows, self.cuda))
            out[i:i + k.numel()] = rows.view(-1, 2 * d)[:, :d]
        return out

    def most_similar_docs(self, queries, k: int = 10, norms: Optional[torch.Tensor] = None):
        """The ``k`` trained documents nearest to each query by cosine similarity. ``queries``: document ids (a
        document never returns itself) or a float ``[n, d]`` tensor of vectors (e.g. from :meth:`infer`). Returns
        ``(document ids int64 [n, k], cosine float32 [n, k])``, best first, ties to the smaller id, ``(-1, -inf)``
        padding. CUDA: ``ops.gather_gemm_topk`` over the document keys with the inverse norms as the column scale (bf16
        operands, fp32 accumulation), without pulling the model; CPU: ``ops.topk_reference``. ``norms``: the inverse
        norms of every document row (computed here when omitted)."""
        d, D = self.cfg.embed_dim, self.num_docs
        is_vec = isinstance(queries, torch.Tensor) and queries.is_floating_point()
        if norms is None:
            norms = 1.0 / self.doc_vectors().norm(dim=1)
        if is_vec:
            if queries.dim() != 2 or queries.shape[1] != d:
                raise ValueError(f"query vectors must be [n, {d}]")
            q = queries.to(self.dev, torch.float32)
            q = q / q.norm(dim=1, keepdim=True)
            n = q.shape[0]
        else:
            j = torch.as_tensor(np.asarray(queries), dtype=torch.int64).reshape(-1)
            n = j.numel()
            q = self.doc_vectors(j) * norms[j.to(self.dev)].view(-1, 1)
        if self.cuda:
            from ..ops import gather_gemm_topk

            excl = None if is_vec else (torch.arange(n + 1, dtype=torch.int64, device=self.dev), j.to(self.dev))
            vals, idx = gather_gemm_topk(self.server, q.contiguous(),
                                         self.doc_key(torch.arange(D, dtype=torch.int64, device=self.dev)), d, k,
                                         exclude=excl, col_scale=norms.contiguous())
            return idx, vals
        from ..ops import _check_topk, topk_reference

        _check_topk(n, D, k, None, None)
        scores = (q @ self.doc_vectors().t()) * norms.view(1, -1)
        excluded = None
        if not is_vec:
            excluded = torch.zeros(n, D, dtype=torch.bool)
            excluded[torch.arange(n), j] = True
        vals, idx = topk_reference(scores, int(k), excluded)
        return idx, vals

    # ------------------------------------------------------------------ output
    def write_checkpoint(self, path: str, doc_path: Optional[str] = None, words=None) -> None:
        """Word vectors in word2vec's binary format (``Word2Vec.write_checkpoint``) and, with ``doc_path``, the document
        vectors in the same format, each named by its line index. Rank 0 writes."""
        self.w2v.write_checkpoint(path, words)
        if doc_path is not None and self.server.my_rank() == 0:
            write_vectors_binary(doc_path, [str(j) for j in range(self.num_docs)], self.doc_vectors().cpu().numpy())


def write_vectors_binary(path: str, names, vecs: np.ndarray) -> None:
    """word2vec's binary format: ``"<n> <d>\\n"``, then per vector its name, a space, d float32 and a newline."""
    vecs = np.ascontiguousarray(vecs, dtype=np.float32)
    with open(path, "wb") as f:
        f.write(f"{vecs.shape[0]} {vecs.shape[1]}\n".encode())
        for name, v in zip(names, vecs):
            f.write(name.encode() + b" " + v.tobytes() + b"\n")
