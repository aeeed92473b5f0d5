"""GloVe word embeddings (Pennington et al., 2014) on the parameter store.

Two tables of word vectors with a bias each, keyed like word2vec: word ``w``'s vector is key ``2 w``, its context vector
key ``2 w + 1``. A row is ``[vector (d) | bias, 0, 0, 0 | AdaGrad (d + 4)]``. Each rank counts the co-occurrence rows
of its own words (``w % world == rank``) from the whole corpus (``ops.glove_cooccurrence`` on CUDA, the numpy
reference on CPU) and trains on them with the fused weighted least-squares step (``ops.glove_step``; the float64 rule
``ops.glove_reference_step`` on CPU). A rank's word rows are private to it; the context rows are shared by every rank,
and each batch's keys are announced ``read_ahead`` batches early with intents, so the store relocates or replicates
them ahead of the step.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from ..parallel.schedules import LookaheadIntents


@dataclass
class GloVeConfig:
    vocab_size: int
    embed_dim: int = 100
    window: int = 15
    symmetric: bool = True
    distance_weighting: bool = True
    eta: float = 0.05
    x_max: float = 100.0
    alpha: float = 0.75
    batch_entries: int = 1 << 16
    read_ahead: int = 2
    signal_intent: bool = True
    deterministic: bool = False
    model_seed: int = 134827
    max_bytes: Optional[int] = None       # device-memory budget of the co-occurrence count (None: the op's default)

    @property
    def row_len(self) -> int:
        return 2 * (self.embed_dim + 4)

    @property
    def num_keys(self) -> int:
        return 2 * self.vocab_size


def word_key(w):
    return 2 * w


def context_key(w):
    return 2 * w + 1


class GloVe:
    def __init__(self, server, worker, cfg: GloVeConfig):
        from ..ops import _check_glove_dim

        _check_glove_dim(cfg.embed_dim)
        if not 1 <= cfg.window <= 16:
            raise ValueError(f"window must be in [1, 16], got {cfg.window}")
        if cfg.deterministic and server.num_servers() > 1:
            raise ValueError("deterministic=True needs a single-GPU server")
        self.server, self.worker, self.cfg = server, worker, cfg
        self.cuda = server.backend == "cuda"
        self.dev = server.device if self.cuda else torch.device("cpu")
        self.rows = self.cols = self.x = None
        if self.cuda:
            self.loss = torch.zeros(1, dtype=torch.float32, device=self.dev)
            self.stats = torch.zeros(4, dtype=torch.int64, device=self.dev)

    @property
    def nnz(self) -> int:
        return 0 if self.x is None else int(self.x.numel())

    # ------------------------------------------------------------------ model init
    def init_model(self, chunk: int = 1 << 16) -> None:
        """Each rank sets the keys it is home for: vectors and biases ``(U[0,1) - 0.5) / d``, AdaGrad accumulators 1.0
        (glove.c's initial ``gradsq``), padding 0."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        d, D = cfg.embed_dim, cfg.embed_dim + 4
        gen = torch.Generator(device=self.dev).manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        keys_all = torch.arange(rank, cfg.num_keys, world, dtype=torch.int64)
        for i in range(0, keys_all.numel(), chunk):
            k = keys_all[i:i + chunk].to(self.dev)
            rows = torch.zeros(k.numel(), 2 * D, dtype=torch.float32, device=self.dev)
            rows[:, :d + 1] = (torch.rand(k.numel(), d + 1, generator=gen, device=self.dev) - 0.5) / d
            rows[:, D:D + d + 1] = 1.0
            self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    # ------------------------------------------------------------------ co-occurrence
    def build_cooccurrence(self, corpus) -> int:
        """Counts this rank's co-occurrence rows from ``corpus`` (a ``NativeCorpus`` that encoded the whole file:
        ``encode(path, 0, 1)``). Returns the number of non-zeros."""
        cfg, rank, world = self.cfg, self.server.my_rank(), self.server.num_servers()
        if self.cuda:
            from ..ops import GLOVE_COOC_MAX_BYTES, glove_cooccurrence

            tok, off = corpus.arrays()
            with torch.cuda.device(self.dev):
                r, c, x = glove_cooccurrence(torch.from_numpy(tok).to(self.dev), torch.from_numpy(off).to(self.dev),
                                             cfg.vocab_size, cfg.window, cfg.symmetric, cfg.distance_weighting, rank,
                                             world, cfg.max_bytes or GLOVE_COOC_MAX_BYTES)
        else:
            from ..utils.text import cooccurrence_reference

            r, c, x = (torch.from_numpy(a) for a in cooccurrence_reference(
                corpus.sentences(), cfg.vocab_size, cfg.window, cfg.symmetric, cfg.distance_weighting, rank, world))
        self.rows, self.cols, self.x = r.long(), c.long(), x
        return self.nnz

    def set_cooccurrence(self, rows: torch.Tensor, cols: torch.Tensor, x: torch.Tensor) -> None:
        """Train on the given non-zeros instead of counting them."""
        self.rows, self.cols = rows.long().to(self.dev), cols.long().to(self.dev)
        self.x = x.float().to(self.dev)

    # ------------------------------------------------------------------ training
    def train_epoch(self, epoch: int) -> float:
        """One pass over this rank's non-zeros in an order drawn from ``(model_seed, epoch)``, in batches of
        ``batch_entries``; one clock per batch. Returns this rank's summed loss ``sum f diff^2 / 2``."""
        cfg, kv = self.cfg, self.worker
        n = self.nnz
        gen = torch.Generator(device=self.dev).manual_seed(cfg.model_seed * 1000003 + epoch)
        perm = torch.randperm(n, generator=gen, device=self.dev)
        wk, ck, xs = word_key(self.rows[perm]), context_key(self.cols[perm]), self.x[perm].contiguous()
        B = cfg.batch_entries
        nb = (n + B - 1) // B
        intents = None
        if cfg.signal_intent and self.server.num_servers() > 1:
            intents = LookaheadIntents(kv, nb, cfg.read_ahead,
                                       lambda b: torch.cat([wk[b * B:(b + 1) * B], ck[b * B:(b + 1) * B]]))
            intents.prime()
        total = 0.0
        if self.cuda:
            from ..ops import glove_step

            self.loss.zero_()
        else:
            from ..ops import glove_reference_step
        for b in range(nb):
            if intents is not None:
                intents.signal(b)
            s = slice(b * B, (b + 1) * B)
            if self.cuda:
                glove_step(self.server, wk[s], ck[s], xs[s], cfg.embed_dim, cfg.eta, cfg.x_max, cfg.alpha, self.loss,
                           self.stats, deterministic=cfg.deterministic)
            else:
                total += glove_reference_step(kv, wk[s], ck[s], xs[s], cfg.embed_dim, cfg.eta, cfg.x_max, cfg.alpha)[0]
            kv.advance_clock()
        return float(self.loss.item()) if self.cuda else total

    # ------------------------------------------------------------------ vectors
    def vectors(self, model: int = 2, chunk: int = 1 << 15) -> torch.Tensor:
        """The dense word vectors float32 [vocab, d] on the server's device, pulled in chunks: ``W + C`` (``model=2``,
        glove.c's ``-model 2``) or ``W`` (``model=1``)."""
        cfg, d, D = self.cfg, self.cfg.embed_dim, self.cfg.embed_dim + 4
        V, kv = cfg.vocab_size, self.worker
        out = torch.empty(V, d, dtype=torch.float32, device=self.dev)
        for i in range(0, V, chunk):
            w = torch.arange(i, min(V, i + chunk), dtype=torch.int64, device=self.dev)
            rows = torch.empty(w.numel() * 2 * D, dtype=torch.float32, device=self.dev)
            kv.wait(kv.pull(word_key(w), rows, self.cuda))
            out[i:i + w.numel()] = rows.view(-1, 2 * D)[:, :d]
            if model == 2:
                kv.wait(kv.pull(context_key(w), rows, self.cuda))
                out[i:i + w.numel()] += rows.view(-1, 2 * D)[:, :d]
        return out

    def most_similar(self, words, k: int = 10, vectors: Optional[torch.Tensor] = None):
        """The ``k`` nearest words of each word in ``words`` by cosine similarity of ``W + C`` (:meth:`vectors`); the
        query word itself is never returned. Returns ``(word ids int64 [n, k], cosine float32 [n, k])``, best first;
        equal scores go to the smaller word id; ``(-1, -inf)`` pads a row when fewer than ``k`` words qualify. ``1 <= k
        <= 64``. CUDA backend: ``ops.gemm_nt_topk`` (bf16 operands, fp32 accumulation) on the normalised queries with
        ``1 / ||e_j||`` as the column scale; CPU backend: fp32 PyTorch with the same order (``ops.topk_reference``)."""
        from ..ops import _check_topk, gemm_nt_topk, topk_reference

        E = self.vectors() if vectors is None else vectors
        V = E.shape[0]
        w = torch.as_tensor(words, dtype=torch.int64).reshape(-1).to(E.device)
        n = w.numel()
        inv = 1.0 / E.norm(dim=1)
        q = (E[w] * inv[w].view(-1, 1)).contiguous()
        if self.cuda:
            excl = (torch.arange(n + 1, dtype=torch.int64, device=E.device), w.contiguous())
            vals, idx = gemm_nt_topk(q, E, k, exclude=excl, col_scale=inv.contiguous())
            return idx, vals
        _check_topk(n, V, k, None, None)
        excluded = torch.zeros(n, V, dtype=torch.bool)
        excluded[torch.arange(n), w] = True
        vals, idx = topk_reference((q @ E.t()) * inv.view(1, -1), int(k), excluded)
        return idx, vals

    def write_vectors(self, path: str, words=None, model: int = 2, chunk: int = 1 << 15) -> None:
        """GloVe's text format, one ``word v1 ... vd`` line per word (``W + C`` or, with ``model=1``, ``W``), written by
        rank 0."""
        self.worker.wait_sync()
        if self.server.my_rank() != 0:
            return
        E = self.vectors(model).cpu().numpy()
        with open(path, "w") as f:
            for i in range(0, E.shape[0], chunk):
                for j, row in enumerate(E[i:i + chunk]):
                    word = words[i + j] if words is not None else f"w{i + j}"
                    f.write(word + " " + " ".join(f"{v:.6f}" for v in row) + "\n")
