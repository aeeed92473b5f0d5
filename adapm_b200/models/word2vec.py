"""word2vec skip-gram (SGNS) or continuous bag of words (CBOW) with negative sampling + AdaGrad on the parameter manager.

Behavioural parity with the reference application ``apps/word2vec.cc``:

* keys: ``syn0[w] = 2w``, ``syn1[w] = 2w + 1`` (word2vec.cc:83-105); row = ``[embedding | AdaGrad]``
  of ``2 * embed_dim`` floats (word2vec.cc:1101);
* per (center, context) pair: 1 positive + ``negative`` negative targets, sigmoid saturating at
  ``|f| > 6``, worker-side AdaGrad using the pulled accumulator (word2vec.cc:420-429,682-745);
* negatives ~ unigram^0.75 (word2vec.cc:125-144) through ``PrepareSample/PullSample`` semantics
  (``sampling.scheme``: ``local`` rejects non-resident keys, ``naive``/``preloc`` use the drawn keys);
* intent: the keys of a future batch are signalled ``read_ahead`` clocks ahead (word2vec.cc:563-606),
  one clock per batch instead of one per sentence;
* init: syn0 ~ U(-0.5, 0.5)/d, syn1 = 0, accumulators 1e-6 (word2vec.cc:805-831);
* checkpoint: ``"<vocab> <dim>\\n"`` then per word ``"<word> "`` + ``dim`` raw float32 + ``"\\n"``
  (word2vec.cc:367-416).

GPU-first differences: the per-pair loop of the reference is one batched kernel
(``ops.sgns_step``) that fuses pull, scoring, AdaGrad and push over local HBM / NVLink peers.

CBOW (``cbow=True``, word2vec.c's ``-cbow 1``, which the reference does not implement) trains one window per corpus word:
the mean ``h`` of the context rows is scored against the centre's syn1 row and the negatives, each target gets
``g_t h`` and every context occurrence the unscaled ``neu1e = sum_t g_t t`` (word2vec.c), each through worker-side
AdaGrad (``cbow_reference_step``; ``ops.cbow_step`` on the GPU). Batches are windows ``[B, 1 + 2 window]`` (centre syn1
key, context syn0 keys, -1 padding) from ``NativeCorpus.window_batches`` or ``windows_from_sentences``.

Hierarchical softmax (``hs=True``, word2vec.c's ``-hs 1``, with ``negative=0``) replaces the negatives by the inner nodes
on the Huffman path of the syn1-side word (``utils.text.huffman_tree`` over the model's counts, word2vec.c's tree):
node ``n`` is the row ``syn1_key(n)``, its label is ``1 - code bit``, and a node with ``|f| >= 6`` is skipped
(``hs_reference_step``; ``ops.hs_step`` on the GPU). Skip-gram trains ``syn0[context]`` on the centre word's path
(word2vec.c's pairing: the pair batch's syn1 word supplies the path, its syn0 word is the one context); CBOW trains the
window's mean on the centre's path. No negatives are drawn.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import LOCAL


@dataclass
class Word2VecConfig:
    vocab_size: int = 1_000_000
    embed_dim: int = 300
    negative: int = 25
    window: int = 5
    starting_alpha: float = 0.025
    neg_power: float = 0.75
    batch_pairs: int = 32768
    read_ahead: int = 4              # batches of look-ahead for intent signalling
    sampling_scheme: str = "local"   # local | naive | preloc
    signal_intent: bool = True
    model_seed: int = 134827
    zipf_exponent: float = 1.0       # synthetic corpus skew
    max_inflight: int = 3            # steps the host may run ahead of the GPU (bounds the sync grace period)
    intent_prepass: bool = False     # experimental: device-side Intent for keys that are already local (ops.IntentPrepass)
    shared_negatives: int = 0        # > 0: ONE set of this many negatives per batch, contractions on the tensor cores
                                     # (ops.SgnsSharedStep); 0: `negative` private negatives per pair (the reference)
    cbow: bool = False               # continuous bag of words (word2vec.c -cbow 1) instead of skip-gram
    batch_windows: int = 8192        # CBOW: windows per step
    hs: bool = False                 # hierarchical softmax (word2vec.c -hs 1) instead of negative sampling (negative = 0)

    @property
    def row_len(self) -> int:
        return 2 * self.embed_dim

    @property
    def num_keys(self) -> int:
        return 2 * self.vocab_size

    @property
    def window_columns(self) -> int:
        # CBOW batch columns: the centre, then up to 2 * window contexts
        return 1 + 2 * self.window

    @property
    def updates_per_pair(self) -> int:
        # 1 (syn0) + (negative + 1) (syn1) additive row updates, BASELINE.md section 3
        return 1 + (self.negative + 1)


def syn0_key(w):
    return 2 * w


def syn1_key(w):
    return 2 * w + 1


def zipf_counts(vocab_size: int, exponent: float = 1.0, total: float = 1e9) -> np.ndarray:
    """Word frequencies of a synthetic corpus with the named vocabulary size (rank-frequency Zipf)."""
    r = np.arange(1, vocab_size + 1, dtype=np.float64)
    p = r ** (-exponent)
    p /= p.sum()
    return np.maximum(1.0, p * total)


class SyntheticPairs:
    """Synthetic (center, context) pair stream: both words ~ Zipf(vocab). Deterministic per
    (seed, rank, step); batches are produced in pinned host memory like a real data loader."""

    def __init__(self, cfg: Word2VecConfig, counts: np.ndarray, rank: int, seed: int = 1, pin: bool = False):
        self.cfg, self.rank, self.seed = cfg, rank, seed
        p = counts / counts.sum()
        self.cdf = np.cumsum(p)
        self.cdf[-1] = 1.0
        self.pin = pin

    def batch(self, step: int):
        rng = np.random.default_rng([self.seed, self.rank, step])
        B = self.cfg.batch_pairs
        u = rng.random(2 * B)
        w = np.searchsorted(self.cdf, u, side="right").astype(np.int64)
        np.clip(w, 0, self.cfg.vocab_size - 1, out=w)
        t = torch.from_numpy(np.stack([syn0_key(w[:B]), syn1_key(w[B:])]))  # [2, B] keys
        if self.pin:
            t = t.pin_memory()
        return t


class SyntheticWindows:
    """Synthetic CBOW window batches [batch_windows, 1 + 2 window] drawn like the loader's: a stream of Zipf words read
    as one long sentence, and for each of ``batch_windows`` consecutive positions a window shrunk by b uniform in
    [0, window). Deterministic per (seed, rank, step)."""

    def __init__(self, cfg: Word2VecConfig, counts: np.ndarray, rank: int, seed: int = 1, pin: bool = False):
        self.cfg, self.rank, self.seed = cfg, rank, seed
        p = counts / counts.sum()
        self.cdf = np.cumsum(p)
        self.cdf[-1] = 1.0
        self.pin = pin

    def batch(self, step: int):
        rng = np.random.default_rng([self.seed, self.rank, step, 1])
        B, W = self.cfg.batch_windows, self.cfg.window
        w = np.searchsorted(self.cdf, rng.random(B + 2 * W), side="right").astype(np.int64)
        np.clip(w, 0, self.cfg.vocab_size - 1, out=w)
        r = W - rng.integers(0, W, B)                                   # shrunk radius per window
        off = np.concatenate([np.arange(-W, 0), np.arange(1, W + 1)])  # context offsets in sentence order
        pos = np.arange(W, W + B)
        ctx = syn0_key(w[pos[:, None] + off[None, :]])
        keep = np.abs(off)[None, :] <= r[:, None]
        out = np.full((B, 1 + 2 * W), -1, dtype=np.int64)
        out[:, 0] = syn1_key(w[pos])
        order = np.argsort(~keep, axis=1, kind="stable")                # kept contexts first, in sentence order
        out[:, 1:] = np.where(np.take_along_axis(keep, order, 1), np.take_along_axis(ctx, order, 1), -1)
        t = torch.from_numpy(out)
        if self.pin:
            t = t.pin_memory()
        return t


class Word2Vec:
    def __init__(self, server, worker, cfg: Word2VecConfig, counts: Optional[np.ndarray] = None):
        self.server, self.worker, self.cfg = server, worker, cfg
        self.counts = counts if counts is not None else zipf_counts(cfg.vocab_size, cfg.zipf_exponent)
        assert len(self.counts) == cfg.vocab_size
        if cfg.cbow and cfg.shared_negatives > 0:
            raise ValueError("shared_negatives is a skip-gram option: CBOW draws its own negatives per window")
        if cfg.hs and (cfg.negative > 0 or cfg.shared_negatives > 0):
            raise ValueError("hierarchical softmax together with negative sampling is not supported: set negative=0 "
                             "and shared_negatives=0 with hs=True")
        self.cuda = server.backend == "cuda"
        self.alpha = cfg.starting_alpha
        self.step_no = 0
        weights = np.power(self.counts, cfg.neg_power)
        self.tree = None
        if cfg.hs:
            from ..utils.text import huffman_tree

            host = huffman_tree(self.counts)
            self._tree_host = (host.offsets.numpy(), host.nodes.numpy())
            self._seen = np.zeros(cfg.vocab_size, dtype=np.int32)   # intent_keys_hs's marker array (words, nodes)
            self.tree = host.to(server.device) if self.cuda else host
        if self.cuda:
            from ..ops import DeviceSampler

            # negatives are syn1 keys: first key 1, stride 2
            self.sampler = DeviceSampler(server, weights=torch.from_numpy(weights), first_key=1, key_stride=2)
            dev = server.device
            self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
            self.stats = torch.zeros(4, dtype=torch.int64, device=dev)
            # a step's key batch: [2, batch_pairs] pairs, or CBOW windows [batch_windows, 1 + 2 window]
            shape = (cfg.batch_windows, cfg.window_columns) if cfg.cbow else (2, cfg.batch_pairs)
            n_items = cfg.batch_windows if cfg.cbow else cfg.batch_pairs
            self._neg = torch.empty(n_items * cfg.negative, dtype=torch.int64, device=dev)
            self._keys_dev = [torch.empty(*shape, dtype=torch.int64, device=dev)
                              for _ in range(max(1, cfg.max_inflight) + 1)]
            self._events = [None] * len(self._keys_dev)
            # data-loader side: the NEXT batch is copied host->device on a copy stream while the current step runs
            self._copy_stream = torch.cuda.Stream(device=dev)
            self._pf_bufs = [torch.empty(*shape, dtype=torch.int64, device=dev)
                             for _ in range(max(1, cfg.max_inflight) + 2)]
            self._pf_no = 0
            self._pf = None
            self._prepass = None
            import os as _os

            if (cfg.intent_prepass or _os.environ.get("ADAPM_INTENT_PREPASS")) and server.num_servers() > 1:
                from ..ops import IntentPrepass

                self._prepass = IntentPrepass(server, worker, max_keys=2 * cfg.batch_pairs)
        else:
            w = torch.from_numpy(weights)
            self._neg_cdf = torch.cumsum(w / w.sum(), 0)
            self._gen = torch.Generator().manual_seed(cfg.model_seed + 17 * server.my_rank())

    # ------------------------------------------------------------------ model init
    def init_model(self, chunk: int = 1 << 16) -> None:
        """Each rank initialises the keys it is home for (set, not push, so re-runs are idempotent)."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        d = cfg.embed_dim
        dev = self.server.device
        gen = torch.Generator(device=dev.type if dev.type == "cuda" else "cpu").manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        keys_all = torch.arange(rank, cfg.num_keys, world, dtype=torch.int64)
        for i in range(0, keys_all.numel(), chunk):
            k = keys_all[i:i + chunk].to(dev)
            rows = torch.empty(k.numel(), 2 * d, dtype=torch.float32, device=dev)
            rows[:, d:] = 1e-6
            emb = (torch.rand(k.numel(), d, generator=gen, device=dev, dtype=torch.float32) - 0.5) / d
            is_syn0 = (k % 2 == 0).view(-1, 1)
            rows[:, :d] = torch.where(is_syn0, emb, torch.zeros_like(emb))
            self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    # ------------------------------------------------------------------ intent
    def signal_intent(self, keys_host: torch.Tensor, clock: int) -> None:
        """keys_host: [2, B] (syn0 keys, syn1 keys) or CBOW windows [B, 1 + 2 window] of a future batch (CPU tensor)."""
        if not self.cfg.signal_intent or self.server.num_servers() == 1:
            return
        # batches of the native loader carry their distinct keys (deduplicated on the loader thread)
        keys = getattr(keys_host, "unique_keys", None)
        if keys is None:
            keys = keys_host.reshape(-1)
            if self.cfg.cbow:
                keys = keys[keys >= 0]                 # window padding
        if self.cfg.hs:
            keys = self.intent_keys_hs(keys)
        if self.cuda and self._prepass is not None:
            self._prepass.harvest()                    # left-overs of earlier batches -> host path
            self._prepass.submit(keys, clock, clock + 1)
            return
        self.worker.intent(keys, clock, clock + 1)

    def intent_keys_hs(self, keys: torch.Tensor) -> torch.Tensor:
        """Hierarchical softmax: the rows a batch with these keys touches, i.e. its syn0 keys and the syn1 keys of the
        inner nodes on the paths of its syn1 words, each once. Paths share their top levels, so the nodes are
        deduplicated with a marker array (the position that last wrote each node) rather than by sorting."""
        k = keys.numpy() if isinstance(keys, torch.Tensor) else np.asarray(keys)
        off, nodes = self._tree_host
        seen = self._seen

        def once(v):                      # each value of v once: the position that wrote it last keeps it
            pos = np.arange(v.size)
            seen[v] = pos
            return v[seen[v] == pos]

        words = once(k[(k & 1) == 1] >> 1)
        start, lens = off[words], off[words + 1] - off[words]
        n = int(lens.sum())
        idx = np.repeat(start - np.cumsum(lens) + lens, lens) + np.arange(n)   # positions of every path entry
        path = once(nodes[idx])
        return torch.from_numpy(np.concatenate([k[(k & 1) == 0], 2 * path.astype(np.int64) + 1]))

    def loss_terms(self, keys_host: torch.Tensor) -> int:
        """Terms of a batch's summed loss: hierarchical softmax, the path nodes of its items; else ``negative + 1`` per
        item."""
        cfg = self.cfg
        centres = keys_host[:, 0] if cfg.cbow else keys_host[1]
        if not cfg.hs:
            return int(centres.numel()) * (cfg.negative + 1)
        off = self._tree_host[0]
        w = centres[centres >= 0].numpy() >> 1
        return int((off[w + 1] - off[w]).sum())

    # ------------------------------------------------------------------ one training step
    def step(self, keys_host: torch.Tensor) -> torch.Tensor:
        """Runs one batch. ``keys_host``: [2, B] int64 CPU tensor (pinned for the e2e path); CBOW: windows
        [batch_windows, 1 + 2 window] (column 0 the centre's syn1 key, then context syn0 keys, -1 = padding).
        Returns the device tensor that accumulates the summed loss (read it with ``.item()``/copy)."""
        cfg = self.cfg
        if self.cuda:
            slot = self.step_no % len(self._keys_dev)
            if self._events[slot] is not None:
                self._events[slot].synchronize()   # bounded run-ahead: at most max_inflight steps queued
            if self._pf is not None and self._pf[0] is keys_host:
                kd = self._pf_bufs[self._pf[1]]                      # H2D of this step's inputs was prefetched
                torch.cuda.current_stream().wait_event(self._pf[2])
                self._pf = None
            else:
                kd = self._keys_dev[slot]
                kd.copy_(keys_host, non_blocking=True)               # H2D of this step's inputs
            if not cfg.hs:
                self.sample_negatives()
            self._device_step(*self._operands(kd))
            ev = self._events[slot] or torch.cuda.Event()
            ev.record()
            self._events[slot] = ev
            self.step_no += 1
            return self.loss
        return self._step_cpu(keys_host)

    def _operands(self, kd: torch.Tensor):
        if self.cfg.cbow:                 # (centres, contexts) of the windows, contiguous for the kernel
            return kd[:, 0].contiguous(), kd[:, 1:].contiguous()
        return kd[0], kd[1]

    def prefetch(self, keys_host: torch.Tensor) -> None:
        """Start the host->device copy of a future step's key batch (pinned memory) on the copy stream; the
        next ``step(keys_host)`` with the same tensor uses the prefetched copy."""
        if not self.cuda:
            return
        b = self._pf_no % len(self._pf_bufs)
        self._pf_no += 1
        with torch.cuda.stream(self._copy_stream):
            self._pf_bufs[b].copy_(keys_host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        self._pf = (keys_host, b, ev)

    def sample_negatives(self) -> torch.Tensor:
        """PrepareSample/PullSample on the device: draws batch_pairs*negative (CBOW: batch_windows*negative) syn1 keys; the ``local``
        scheme rejects keys that are not resident in this GPU's HBM."""
        cfg = self.cfg
        local_only = cfg.sampling_scheme == "local" and self.server.num_servers() > 1
        seed = (cfg.model_seed * 1000003 + self.server.my_rank() * 7919 + self.step_no) & 0xFFFFFFFFFFFF
        return self.sampler.sample(self._neg.numel(), seed, local_only=local_only, out=self._neg)

    def _device_step(self, centers: torch.Tensor, contexts: torch.Tensor) -> None:
        from ..ops import SgnsSharedStep, sgns_step

        cfg = self.cfg
        if cfg.hs:
            from ..ops import hs_step

            if cfg.cbow:
                hs_step(self.server, centers, contexts, self.tree, cfg.embed_dim, self.alpha, self.loss, self.stats)
            else:                         # the pair's syn1 word supplies the path, its syn0 word is the one context
                hs_step(self.server, contexts, centers.view(-1, 1), self.tree, cfg.embed_dim, self.alpha, self.loss,
                        self.stats)
        elif cfg.cbow:
            from ..ops import cbow_step

            cbow_step(self.server, centers, contexts, self._neg.view(centers.numel(), cfg.negative), cfg.embed_dim,
                      self.alpha, self.loss, self.stats)
        elif cfg.shared_negatives > 0:
            if getattr(self, "_shared", None) is None:
                self._shared = SgnsSharedStep(self.server, self.worker, cfg.batch_pairs, cfg.shared_negatives, cfg.embed_dim)
            self._shared(centers, contexts, self._neg[:cfg.shared_negatives], self.alpha, self.loss)
        else:
            sgns_step(self.server, centers, contexts, self._neg, cfg.embed_dim, self.alpha, self.loss, self.stats)

    def step_resident(self, keys_dev: torch.Tensor) -> torch.Tensor:
        """Same as step() for a key batch that already lives on the device."""
        slot = self.step_no % len(self._events)
        if self._events[slot] is not None:
            self._events[slot].synchronize()
        if not self.cfg.hs:
            self.sample_negatives()
        self._device_step(*self._operands(keys_dev))
        ev = self._events[slot] or torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        self.step_no += 1
        return self.loss

    # ------------------------------------------------------------------ native step driver
    def run_steps(self, batches, first: int, n: int, resident: bool = False, loss_host: Optional[torch.Tensor] = None,
                  intent_batches=None) -> None:
        """Runs steps ``first .. first+n-1`` from C++ (``ops.SgnsLoop``: Intent for batch ``s + read_ahead``, bounded
        run-ahead, prefetched H2D of the step's keys, sampler + fused SGNS kernel, D2H of the loss into
        ``loss_host[s]``, clock tick) - the same work per step as ``signal_intent`` + ``step`` + ``advance_clock`` in a
        Python loop, without Python in it. ``batches``: sequence of [2, B] int64 key batches - pinned host tensors, or
        device tensors with ``resident=True`` (entries of steps that are not run may be None); the keys for Intent come
        from ``intent_batches`` (default: ``batches``): host tensors that may carry ``unique_keys`` (their distinct keys)."""
        from .. import _C

        cfg = self.cfg
        if cfg.cbow or cfg.hs:
            raise ValueError("run_steps drives negative-sampling skip-gram steps only: run CBOW and hierarchical-softmax "
                             "steps with step()")
        assert self.cuda, "run_steps needs the cuda backend"
        if getattr(self, "_loop", None) is None:
            local_only = cfg.sampling_scheme == "local" and self.server.num_servers() > 1
            sp = self.sampler
            self._loop = _C.SgnsLoop(self.worker._impl.handle(), self.server._impl.backend_handle(), cfg.batch_pairs,
                                     cfg.negative, cfg.embed_dim, cfg.read_ahead, max(1, cfg.max_inflight),
                                     self.server.my_rank(), bool(cfg.signal_intent and self.server.num_servers() > 1),
                                     local_only, cfg.model_seed, sp.kind, sp.prob.data_ptr(), sp.alias.data_ptr(), sp.n,
                                     sp.first_key, sp.key_stride, sp.stats.data_ptr())
            self._loop_cache = {}
        ib = intent_batches if intent_batches is not None else batches
        key = (id(batches), id(ib), resident)
        tabs = self._loop_cache.get(key)
        if tabs is None or tabs[3] != len(batches):
            ptrs = [b.data_ptr() if b is not None else 0 for b in batches]
            ik, ic, keep = [], [], []
            for b in ib:
                u = getattr(b, "unique_keys", None)
                if u is None:
                    u = b.view(-1) if not b.is_cuda else b.view(-1).cpu()
                    keep.append(u)
                ik.append(u.data_ptr()); ic.append(u.numel())
            tabs = (ptrs, ik, ic, len(batches), keep, batches, ib)   # (the tensors are kept alive with the table)
            self._loop_cache[key] = tabs
        self._loop.run(torch.cuda.current_stream().cuda_stream, int(first), int(n), bool(resident), tabs[0], tabs[1], tabs[2],
                       self.loss.data_ptr(), loss_host.data_ptr() if loss_host is not None else 0, self.stats.data_ptr(),
                       self.step_no, float(self.alpha))
        self.step_no += int(n)

    # reference-semantics step through the public Pull/Push API (CPU backend; also the numerics oracle)
    def _step_cpu(self, keys_host: torch.Tensor) -> torch.Tensor:
        cfg, kv, d = self.cfg, self.worker, self.cfg.embed_dim
        if cfg.hs:
            if cfg.cbow:
                loss = hs_reference_step(kv, keys_host[:, 0], keys_host[:, 1:], self.tree, d, self.alpha)
            else:
                loss = hs_reference_step(kv, keys_host[1], keys_host[0].view(-1, 1), self.tree, d, self.alpha)
            self.step_no += 1
            return torch.tensor([loss], dtype=torch.float32)
        if cfg.cbow:
            B = keys_host.shape[0]
            u = torch.rand(B * cfg.negative, generator=self._gen, dtype=torch.float64)
            negw = torch.searchsorted(self._neg_cdf, u).clamp_(max=cfg.vocab_size - 1)
            loss = cbow_reference_step(kv, keys_host[:, 0], keys_host[:, 1:], syn1_key(negw).view(B, cfg.negative), d,
                                       self.alpha)
            self.step_no += 1
            return torch.tensor([loss], dtype=torch.float32)
        centers, contexts = keys_host[0], keys_host[1]
        B = centers.numel()
        if cfg.shared_negatives > 0:      # one set of negatives for the batch (the GEMM formulation), through Pull / Push
            u = torch.rand(cfg.shared_negatives, generator=self._gen, dtype=torch.float64)
            negs = syn1_key(torch.searchsorted(self._neg_cdf, u).clamp_(max=cfg.vocab_size - 1))
            loss = sgns_shared_pull_push_step(kv, centers, contexts, negs, d, self.alpha)
            self.step_no += 1
            return torch.tensor([loss], dtype=torch.float32)
        u = torch.rand(B * cfg.negative, generator=self._gen, dtype=torch.float64)
        negw = torch.searchsorted(self._neg_cdf, u).clamp_(max=cfg.vocab_size - 1)
        negs = syn1_key(negw).view(B, cfg.negative)
        loss = sgns_reference_step(kv, centers, contexts, negs, d, self.alpha)
        self.step_no += 1
        return torch.tensor([loss], dtype=torch.float32)

    def set_alpha(self, progress: float) -> None:
        """Linear decay like the reference (word2vec.cc:551-559)."""
        self.alpha = max(self.cfg.starting_alpha * (1.0 - progress), self.cfg.starting_alpha * 1e-4)

    # ------------------------------------------------------------------ nearest neighbours
    def syn0_norms(self, chunk: int = 1 << 16) -> torch.Tensor:
        """``1 / ||syn0[w]||`` for every word (float32 [vocab], on the server's device; ``inf`` for a zero row), read
        with a chunked Pull. Pass it to :meth:`most_similar` to reuse it across calls."""
        cfg, d, kv = self.cfg, self.cfg.embed_dim, self.worker
        dev = self.server.device if self.cuda else torch.device("cpu")
        out = torch.empty(cfg.vocab_size, dtype=torch.float32, device=dev)
        for i in range(0, cfg.vocab_size, chunk):
            w = torch.arange(i, min(cfg.vocab_size, i + chunk), dtype=torch.int64, device=dev)
            rows = torch.empty(w.numel() * 2 * d, dtype=torch.float32, device=dev)
            kv.wait(kv.pull(syn0_key(w), rows, self.cuda))
            out[i:i + w.numel()] = 1.0 / rows.view(-1, 2 * d)[:, :d].norm(dim=1)
        return out

    def most_similar(self, words, k: int = 10, norms: Optional[torch.Tensor] = None):
        """The ``k`` nearest words of each word in ``words`` by cosine similarity of the syn0 embeddings; the query
        word itself is never returned. Returns ``(word ids int64 [n, k], cosine float32 [n, k])``, best first; equal
        scores go to the smaller word id; ``(-1, -inf)`` pads a row when fewer than ``k`` words qualify (zero rows
        give NaN scores and never qualify). ``norms``: the output of :meth:`syn0_norms` (computed here when omitted).
        ``1 <= k <= 64``.

        CUDA backend: the query rows are pulled and normalised, and ``ops.gather_gemm_topk`` scores them against all
        syn0 rows of the store (bf16 operands, fp32 accumulation, times ``norms`` as the column scale) without
        pulling the model. CPU backend: fp32 PyTorch with the same order (``ops.topk_reference``)."""
        cfg, d, kv = self.cfg, self.cfg.embed_dim, self.worker
        V = cfg.vocab_size
        w = torch.as_tensor(words, dtype=torch.int64).reshape(-1)
        n = w.numel()
        dev = self.server.device if self.cuda else torch.device("cpu")
        w = w.to(dev)
        if norms is None:
            norms = self.syn0_norms()
        rows = torch.empty(n * 2 * d, dtype=torch.float32, device=dev)
        kv.wait(kv.pull(syn0_key(w), rows, self.cuda))
        q = rows.view(n, 2 * d)[:, :d] * norms[w].view(-1, 1)
        if self.cuda:
            from ..ops import gather_gemm_topk

            excl = (torch.arange(n + 1, dtype=torch.int64, device=dev), w.contiguous())
            vals, idx = gather_gemm_topk(self.server, q, syn0_key(torch.arange(V, dtype=torch.int64, device=dev)), d, k,
                                         exclude=excl, col_scale=norms)
            return idx, vals
        from ..ops import _check_topk, topk_reference

        _check_topk(n, V, k, None, None)
        E = torch.empty(V * 2 * d, dtype=torch.float32)
        kv.wait(kv.pull(syn0_key(torch.arange(V, dtype=torch.int64)), E))
        scores = (q @ E.view(V, 2 * d)[:, :d].t()) * norms.view(1, -1)
        excluded = torch.zeros(n, V, dtype=torch.bool)
        excluded[torch.arange(n), w] = True
        vals, idx = topk_reference(scores, int(k), excluded)
        return idx, vals

    # ------------------------------------------------------------------ checkpoint
    def write_checkpoint(self, path: str, words=None, write_syn1: bool = False, chunk: int = 1 << 15) -> None:
        """Binary word2vec format of the reference (word2vec.cc:367-416); rank 0 pulls the model."""
        cfg, d = self.cfg, self.cfg.embed_dim
        self.worker.wait_sync()
        if self.server.my_rank() != 0:
            return

        def dump(fn, key_fn):
            with open(fn, "wb") as f:
                f.write(f"{cfg.vocab_size} {d}\n".encode())
                for i in range(0, cfg.vocab_size, chunk):
                    w = torch.arange(i, min(cfg.vocab_size, i + chunk), dtype=torch.int64)
                    vals = torch.empty(w.numel() * 2 * d, dtype=torch.float32)
                    self.worker.wait(self.worker.pull(key_fn(w), vals))
                    emb = vals.view(-1, 2 * d)[:, :d].contiguous().numpy()
                    for j in range(w.numel()):
                        word = words[i + j] if words is not None else f"w{i + j}"
                        f.write(word.encode() + b" ")
                        f.write(emb[j].tobytes())
                        f.write(b"\n")

        dump(path, syn0_key)
        if write_syn1:
            dump(path + ".syn1", syn1_key)


def sgns_shared_pull_push_step(kv, centers, contexts, negatives, d: int, alpha: float) -> float:
    """Shared-negative SGNS step through the public Pull / Push API (any backend): the same rule as the tensor-core
    variant (``ops.SgnsSharedStep``), computed with ``ops.sgns_shared_reference_step`` on the pulled rows."""
    from ..ops import sgns_shared_reference_step

    keys = torch.cat([centers.view(-1), contexts.view(-1), negatives.view(-1)])
    uk, inv = torch.unique(keys, return_inverse=True)
    rows = torch.empty(uk.numel() * 2 * d, dtype=torch.float32)
    kv.wait(kv.pull(uk, rows))
    rows = rows.view(-1, 2 * d)
    B, Nn = centers.numel(), negatives.numel()
    new, loss = sgns_shared_reference_step(rows, inv[:B], inv[B:2 * B], inv[2 * B:], d, alpha)
    kv.wait(kv.push(uk, (new - rows).contiguous().view(-1)))
    return float(loss)


def read_word2vec_binary(path: str):
    """Parses the binary word2vec format written by write_checkpoint: returns (words, float32 [V, d])."""
    with open(path, "rb") as f:
        buf = f.read()
    nl = buf.index(b"\n")
    V, d = (int(t) for t in buf[:nl].split())
    pos = nl + 1
    words, vecs = [], np.empty((V, d), dtype=np.float32)
    for i in range(V):
        sp = buf.index(b" ", pos)
        words.append(buf[pos:sp].decode(errors="replace"))
        vecs[i] = np.frombuffer(buf, dtype=np.float32, count=d, offset=sp + 1)
        pos = sp + 1 + 4 * d + 1      # vector + trailing newline
    return words, vecs


def load_checkpoint(model: "Word2Vec", path: str, words=None, chunk: int = 1 << 15) -> int:
    """``init_model=<path>`` of the reference (word2vec.cc:832-900): syn0 from ``path``, syn1 from ``path.syn1`` when it
    exists; AdaGrad accumulators restart at 1e-6. Words are matched by name when ``words`` (this job's vocabulary) is
    given, by position otherwise. Collective (every rank sets the keys it is home for). Returns #words loaded."""
    cfg, d = model.cfg, model.cfg.embed_dim
    world, rank = model.server.num_servers(), model.server.my_rank()
    loaded = 0
    model.worker.begin_setup()
    for fn, key_fn in ((path, syn0_key), (path + ".syn1", syn1_key)):
        try:
            fw, vecs = read_word2vec_binary(fn)
        except FileNotFoundError:
            if fn == path:
                raise
            continue
        assert vecs.shape[1] == d, f"{fn}: dimension {vecs.shape[1]} != embed_dim {d}"
        if words is not None:
            index = {w: i for i, w in enumerate(words)}
            ids = np.array([index.get(w, -1) for w in fw], dtype=np.int64)
        else:
            ids = np.arange(len(fw), dtype=np.int64)
        ok = (ids >= 0) & (ids < cfg.vocab_size)
        ids, vecs = ids[ok], vecs[ok]
        keys = key_fn(torch.from_numpy(ids))
        mine = (keys % world) == rank
        keys, rows_e = keys[mine], torch.from_numpy(vecs)[mine]
        for a in range(0, keys.numel(), chunk):
            rows = torch.full((min(chunk, keys.numel() - a), 2 * d), 1e-6, dtype=torch.float32)
            rows[:, :d] = rows_e[a:a + chunk]
            model.worker.wait(model.worker.set(keys[a:a + chunk], rows.view(-1)))
        if fn == path:
            loaded = int(ok.sum())
    model.worker.waitall()
    model.worker.end_setup()
    return loaded


def sgns_reference_step(kv, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor, d: int,
                        alpha: float) -> float:
    """Plain PyTorch fp32 SGNS step through Pull/Push with the reference's exact update rule.
    All pairs read the state at the start of the step (the batched-kernel semantics)."""
    B = centers.numel()
    neg = negatives.shape[1]
    tk = torch.cat([contexts.view(B, 1), negatives], 1)            # [B, 1+neg] target keys
    r0 = torch.empty(B * 2 * d, dtype=torch.float32)
    kv.wait(kv.pull(centers, r0))
    r1 = torch.empty(B * (1 + neg) * 2 * d, dtype=torch.float32)
    kv.wait(kv.pull(tk.reshape(-1), r1))
    r0 = r0.view(B, 2 * d)
    r1 = r1.view(B, 1 + neg, 2 * d)
    e0, a0 = r0[:, :d], r0[:, d:]
    e1, a1 = r1[:, :, :d], r1[:, :, d:]
    label = torch.zeros(B, 1 + neg)
    label[:, 0] = 1
    f = (e0.unsqueeze(1) * e1).sum(-1)
    sig = torch.sigmoid(f)
    g = label - sig
    g = torch.where(f > 6, label - 1, g)
    g = torch.where(f < -6, label, g)
    valid = torch.ones(B, 1 + neg, dtype=torch.bool)
    valid[:, 1:] = negatives != contexts.view(B, 1)                 # negatives equal to the target are skipped
    g = g * valid
    grad0 = (g.unsqueeze(-1) * e1).sum(1)
    grad1 = g.unsqueeze(-1) * e0.unsqueeze(1)
    u1a = grad1 * grad1
    u1e = alpha * grad1 / torch.sqrt(a1 + u1a)
    u0a = grad0 * grad0
    u0e = alpha * grad0 / torch.sqrt(a0 + u0a)
    sel = valid.reshape(-1)
    kv.wait(kv.push(tk.reshape(-1)[sel], torch.cat([u1e, u1a], -1).view(-1, 2 * d)[sel].contiguous().view(-1)))
    kv.wait(kv.push(centers, torch.cat([u0e, u0a], -1).contiguous().view(-1)))
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    return float((torch.log1p(torch.exp(-z)) * valid).sum())


def cbow_reference_step(kv, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor, d: int,
                        alpha: float) -> float:
    """Plain PyTorch fp32 CBOW step through Pull/Push, the rule of ``ops.cbow_step``. ``centers``: [B] syn1 keys (< 0:
    the window does nothing), ``contexts``: [B, C] syn0 keys (-1 = padding), ``negatives``: [B, neg] syn1 keys. All
    windows read the state at the start of the step: ``h`` = mean of the C context embeddings (a repeated word counts
    every time), targets the centre (label 1) and the negatives (label 0; one equal to the centre is skipped),
    ``g = label - sigmoid(h . t)`` saturated at |f| > 6, one AdaGrad push of ``g h`` per (window, target) and one of
    ``neu1e = sum_t g t`` (not divided by C, as word2vec.c) per context occurrence; updates of repeated keys add up.
    Returns the summed logistic loss."""
    centers, contexts, negatives = centers.reshape(-1), contexts.reshape(centers.numel(), -1), negatives
    B, C = contexts.shape
    neg = negatives.shape[1]
    xm = (contexts >= 0) & (centers >= 0).view(B, 1)
    n_ctx = xm.sum(1)
    active = (centers >= 0) & (n_ctx > 0)
    xm &= active.view(B, 1)
    tk = torch.cat([centers.view(B, 1), negatives], 1)              # [B, 1 + neg] target keys
    tm = active.view(B, 1).repeat(1, 1 + neg)
    tm[:, 1:] &= negatives != centers.view(B, 1)
    xkeys, tkeys = contexts[xm], tk[tm]
    rows = torch.empty((xkeys.numel() + tkeys.numel()) * 2 * d, dtype=torch.float32)
    kv.wait(kv.pull(torch.cat([xkeys, tkeys]), rows))
    rows = rows.view(-1, 2 * d)
    rx, rt = rows[:xkeys.numel()], rows[xkeys.numel():]
    ex = torch.zeros(B, C, d)
    ex[xm] = rx[:, :d]
    h = ex.sum(1) / n_ctx.clamp(min=1).view(B, 1).to(torch.float32)
    et, at = torch.zeros(B, 1 + neg, d), torch.ones(B, 1 + neg, d)
    et[tm], at[tm] = rt[:, :d], rt[:, d:]
    label = torch.zeros(B, 1 + neg)
    label[:, 0] = 1
    f = (h.unsqueeze(1) * et).sum(-1)
    g = label - torch.sigmoid(f)
    g = torch.where(f > 6, label - 1, g)
    g = torch.where(f < -6, label, g)
    g = g * tm
    neu1e = (g.unsqueeze(-1) * et).sum(1)                           # [B, d]
    gt = g.unsqueeze(-1) * h.unsqueeze(1)
    ut = torch.cat([alpha * gt / torch.sqrt(at + gt * gt), gt * gt], -1)[tm]
    gx = neu1e.unsqueeze(1).expand(B, C, d)[xm]
    ax = rx[:, d:]
    ux = torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)
    kv.wait(kv.push(torch.cat([tkeys, xkeys]), torch.cat([ut, ux]).contiguous().view(-1)))
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    return float((torch.log1p(torch.exp(-z)) * tm).sum())


def hs_reference_step(kv, centers: torch.Tensor, contexts: torch.Tensor, tree, d: int, alpha: float) -> float:
    """Plain PyTorch fp32 hierarchical-softmax step through Pull/Push, the rule of ``ops.hs_step``. ``centers``: [B]
    syn1 keys ``2 w + 1`` (< 0: the item does nothing), ``contexts``: [B, C] syn0 keys (-1 = padding; C = 1 for
    skip-gram), ``tree``: a :class:`adapm_b200.utils.text.HuffmanTree`. All items read the state at the start of the
    step: ``h`` = mean of the C context embeddings (a repeated word counts every time); node j of word w's path
    (row ``2 node + 1``) has label ``1 - bit j of codes[w]`` and score ``f_j = h . node``; a node with ``|f_j| >= 6``
    gets no update and adds nothing to ``neu1e`` (word2vec.c), else ``g_j = label - sigmoid(f_j)``, one AdaGrad push of
    ``g_j h`` per (item, node) and one of ``neu1e = sum_j g_j node_j`` per context occurrence; updates of repeated keys
    add up. An item without a context does nothing. Returns the summed logistic loss over every path node, skipped or
    not."""
    centers = centers.reshape(-1)
    B = centers.numel()
    contexts = contexts.reshape(B, -1)
    C = contexts.shape[1]
    off, nodes, codes = tree.offsets.cpu(), tree.nodes.cpu(), tree.codes.cpu()
    L = int(tree.max_len)
    xm = (contexts >= 0) & (centers >= 0).view(B, 1)
    n_ctx = xm.sum(1)
    active = (centers >= 0) & (n_ctx > 0)
    xm &= active.view(B, 1)
    w = torch.where(active, centers // 2, torch.zeros_like(centers))
    start, lens = off[w], off[w + 1] - off[w]
    j = torch.arange(L)
    tm = active.view(B, 1) & (j.view(1, L) < lens.view(B, 1))          # [B, L] path nodes
    node = nodes[torch.where(tm, start.view(B, 1) + j.view(1, L), torch.zeros_like(tm, dtype=torch.int64))].long()
    label = (1 - ((codes[w].view(B, 1) >> j.view(1, L).to(torch.int32)) & 1)).to(torch.float32)
    xkeys, tkeys = contexts[xm], (2 * node + 1)[tm]
    rows = torch.empty((xkeys.numel() + tkeys.numel()) * 2 * d, dtype=torch.float32)
    kv.wait(kv.pull(torch.cat([xkeys, tkeys]), rows))
    rows = rows.view(-1, 2 * d)
    rx, rt = rows[:xkeys.numel()], rows[xkeys.numel():]
    ex = torch.zeros(B, C, d)
    ex[xm] = rx[:, :d]
    h = ex.sum(1) / n_ctx.clamp(min=1).view(B, 1).to(torch.float32)
    et, at = torch.zeros(B, L, d), torch.ones(B, L, d)
    et[tm], at[tm] = rt[:, :d], rt[:, d:]
    f = (h.unsqueeze(1) * et).sum(-1)
    um = tm & (f.abs() < 6)                                           # nodes that get an update
    g = (label - torch.sigmoid(f)) * um
    neu1e = (g.unsqueeze(-1) * et).sum(1)
    gt = g.unsqueeze(-1) * h.unsqueeze(1)
    ut = torch.cat([alpha * gt / torch.sqrt(at + gt * gt), gt * gt], -1)[um]
    gx = neu1e.unsqueeze(1).expand(B, C, d)[xm]
    ax = rx[:, d:]
    ux = torch.cat([alpha * gx / torch.sqrt(ax + gx * gx), gx * gx], -1)
    kv.wait(kv.push(torch.cat([(2 * node + 1)[um], xkeys]), torch.cat([ut, ux]).contiguous().view(-1)))
    z = torch.where(label > 0.5, f, -f).clamp(-6, 6)
    return float((torch.log1p(torch.exp(-z)) * tm).sum())
