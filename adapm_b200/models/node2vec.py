"""node2vec (Grover and Leskovec, 2016) and DeepWalk (``p = q = 1``) graph embeddings on the parameter store.

A node is a word of skip-gram word2vec: node ``v``'s vector is key ``2 v`` (syn0), its context vector key ``2 v + 1``
(syn1), and training is an unchanged negative-sampling skip-gram :class:`Word2Vec` whose vocabulary is the node set.
Negatives are drawn by ``deg^0.75``, so isolated nodes are never drawn. The "corpus" is random walks, generated on the
device next to the step (``ops.random_walks``, ``ops.walk_pairs``) instead of on the host.

An epoch, on each rank: the walks start at this rank's nodes (``v % world == rank``), ``num_walks`` times each, in an
order shuffled by ``(model_seed, epoch)``. They are generated in chunks of ``walkers_per_chunk`` walks; each chunk's
walks become skip-gram pairs, and the pairs run through ``Word2Vec.step_resident`` in slices of ``batch_pairs``, the
remainder carried into the next chunk (the last one of an epoch is padded by repeating its pairs). The learning rate
decays linearly over the run's walks, as word2vec's does over its words. Reading a chunk's pair count is the only
host round trip of a chunk (the steps keep Word2Vec's bounded run-ahead, ``max_inflight``); on several ranks the
distinct keys of the next chunk are signalled then as one intent over the clocks its steps will span, so the store
relocates or replicates them while the current chunk trains.

The CPU backend generates the same walks and pairs with the numpy references and trains with Word2Vec's CPU step.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .word2vec import Word2Vec, Word2VecConfig, syn0_key


@dataclass
class Node2VecConfig:
    dimensions: int = 128
    walk_length: int = 80
    num_walks: int = 10
    window: int = 10
    p: float = 1.0
    q: float = 1.0
    negative: int = 5
    batch_pairs: int = 32768
    iter: int = 1
    alpha: float = 0.025
    walkers_per_chunk: int = 4096
    model_seed: int = 134827
    signal_intent: bool = True

    @property
    def row_len(self) -> int:
        return 2 * self.dimensions


def num_keys(num_nodes: int) -> int:
    return 2 * int(num_nodes)


class Node2Vec:
    def __init__(self, server, worker, graph, cfg: Node2VecConfig):
        from ..ops import _check_walk_length, _check_window, walk_thresholds

        _check_walk_length(cfg.walk_length)
        _check_window(cfg.window)
        walk_thresholds(cfg.p, cfg.q)
        if cfg.num_walks < 1 or cfg.walkers_per_chunk < 1 or cfg.batch_pairs < 1:
            raise ValueError("num_walks, walkers_per_chunk and batch_pairs must be positive")
        self.server, self.worker, self.cfg = server, worker, cfg
        self.cuda = server.backend == "cuda"
        self.dev = server.device if self.cuda else torch.device("cpu")
        self.graph = graph.to(self.dev)
        n = graph.num_nodes
        deg = graph.degrees().cpu().numpy().astype(np.float64)
        if not deg.any():
            raise ValueError("the graph has no edges")
        self.w2v = Word2Vec(server, worker, Word2VecConfig(vocab_size=n, embed_dim=cfg.dimensions, negative=cfg.negative,
                                                           window=cfg.window, starting_alpha=cfg.alpha,
                                                           batch_pairs=cfg.batch_pairs, model_seed=cfg.model_seed),
                            counts=deg)
        world, rank = server.num_servers(), server.my_rank()
        self.my_nodes = np.arange(rank, n, world, dtype=np.int64)
        self.intents = cfg.signal_intent and world > 1
        if self.cuda and self.intents:
            self._mark = torch.empty(n + 1, dtype=torch.uint8, device=self.dev)
            self._mark_host = torch.empty(n + 1, dtype=torch.uint8).pin_memory()

    @property
    def num_nodes(self) -> int:
        return self.graph.num_nodes

    def init_model(self) -> None:
        self.w2v.init_model()

    # ------------------------------------------------------------------ walks
    def epoch_starts(self, epoch: int):
        """This rank's walks of an epoch as ``(starts, walk numbers)`` int64 numpy arrays: walk number ``r`` of every
        node of the rank, ``r = 0 .. num_walks - 1``, the nodes of each round in an order drawn from ``(model_seed,
        epoch, r)``."""
        cfg = self.cfg
        starts = [np.random.default_rng([cfg.model_seed, epoch, r]).permutation(self.my_nodes)
                  for r in range(cfg.num_walks)]
        return np.concatenate(starts), np.repeat(np.arange(cfg.num_walks, dtype=np.int64), self.my_nodes.size)

    def _chunk(self, epoch: int, c: int, starts, walk_nos):
        """the pairs [2, P] of chunk c, and its distinct nodes (numpy) when intents are signalled"""
        from ..ops import random_walks, random_walks_reference, walk_pairs, walk_pairs_reference

        cfg, C, n = self.cfg, self.cfg.walkers_per_chunk, self.num_nodes
        s, wn = starts[c * C:(c + 1) * C], walk_nos[c * C:(c + 1) * C]
        pseed = ((cfg.model_seed * 1000003 + epoch) * 1000003 + self.server.my_rank()) * 1000003 + c
        if not self.cuda:
            walks = random_walks_reference(self.graph, s, wn, cfg.walk_length, cfg.p, cfg.q, cfg.model_seed, epoch)
            nodes = np.unique(walks[walks >= 0]) if self.intents else None
            return torch.from_numpy(walk_pairs_reference(walks, cfg.window, pseed)), nodes
        walks = random_walks(self.graph, s, wn, cfg.walk_length, cfg.p, cfg.q, cfg.model_seed, epoch)
        if self.intents:            # the nodes are marked on the device and copied back under walk_pairs' one sync
            self._mark.zero_()
            self._mark.index_fill_(0, torch.where(walks < 0, n, walks).view(-1), 1)
            self._mark_host.copy_(self._mark, non_blocking=True)
        pairs = walk_pairs(walks, cfg.window, pseed)
        nodes = np.flatnonzero(self._mark_host[:n].numpy()) if self.intents else None
        return pairs, nodes

    def _signal(self, nodes, start: int, n_steps: int) -> None:
        k = torch.from_numpy(nodes.astype(np.int64))
        self.worker.intent(torch.cat([syn0_key(k), syn0_key(k) + 1]), start, start + n_steps + 1)

    # ------------------------------------------------------------------ training
    def train_epoch(self, epoch: int):
        """One epoch of this rank's walks; one clock per step. Returns ``(summed loss, pairs trained)`` of this rank."""
        cfg, kv, w2v = self.cfg, self.worker, self.w2v
        B, C = cfg.batch_pairs, cfg.walkers_per_chunk
        starts, walk_nos = self.epoch_starts(epoch)
        total_walks = max(1, starts.size * cfg.iter)
        n_chunks = (starts.size + C - 1) // C
        carry = torch.empty(2, 0, dtype=torch.int64, device=self.dev)
        loss, pairs_done = 0.0, 0
        if self.cuda:
            w2v.loss.zero_()
        nxt = self._chunk(epoch, 0, starts, walk_nos) if n_chunks else None
        if nxt is not None and self.intents:
            self._signal(nxt[1], kv.current_clock(), (nxt[0].shape[1] + B - 1) // B)
        for c in range(n_chunks):
            pairs = torch.cat([carry, nxt[0]], 1) if carry.shape[1] else nxt[0]
            n_full = pairs.shape[1] // B
            last = c + 1 == n_chunks
            if not last:
                nxt = self._chunk(epoch, c + 1, starts, walk_nos)
                if self.intents:
                    rest = pairs.shape[1] - n_full * B
                    self._signal(nxt[1], kv.current_clock() + n_full, (rest + nxt[0].shape[1] + B - 1) // B)
            batches = [pairs[:, b * B:(b + 1) * B] for b in range(n_full)]
            carry = pairs[:, n_full * B:]
            if last and carry.shape[1]:          # the epoch's last pairs, padded by repeating them
                idx = torch.arange(B, device=self.dev) % carry.shape[1]
                batches.append(carry[:, idx])
                carry = carry[:, :0]
            done = c * C
            chunk_walks = min(C, starts.size - done)
            for b, keys in enumerate(batches):
                w2v.set_alpha((epoch * starts.size + done + chunk_walks * (b + 1) / len(batches)) / total_walks)
                if self.cuda:
                    w2v.step_resident(keys)
                else:
                    loss += float(w2v.step(keys.contiguous()))
                kv.advance_clock()
                pairs_done += B
        if self.cuda:
            loss = float(w2v.loss.item())
        return loss, pairs_done

    # ------------------------------------------------------------------ evaluation and output
    def vectors(self, chunk: int = 1 << 16) -> torch.Tensor:
        """The node vectors (syn0) float32 [num_nodes, dimensions], on the server's device."""
        d, n, kv = self.cfg.dimensions, self.num_nodes, self.worker
        out = torch.empty(n, d, dtype=torch.float32, device=self.dev)
        for i in range(0, n, chunk):
            v = torch.arange(i, min(n, i + chunk), dtype=torch.int64, device=self.dev)
            rows = torch.empty(v.numel() * 2 * d, dtype=torch.float32, device=self.dev)
            kv.wait(kv.pull(syn0_key(v), rows, self.cuda))
            out[i:i + v.numel()] = rows.view(-1, 2 * d)[:, :d]
        return out

    def link_prediction_auc(self, pos_edges, neg_edges, vectors: Optional[torch.Tensor] = None) -> float:
        """ROC AUC of telling the edges ``pos_edges`` from the non-edges ``neg_edges`` (each ``[2, k]`` node ids) by the
        dot product of their node vectors; ties count one half."""
        E = (self.vectors() if vectors is None else vectors).double()

        def scores(e):
            e = torch.as_tensor(np.asarray(e), dtype=torch.int64).reshape(2, -1).to(E.device)
            return (E[e[0]] * E[e[1]]).sum(1).cpu().numpy()

        return roc_auc(scores(pos_edges), scores(neg_edges))

    def most_similar(self, nodes, k: int = 10):
        """The ``k`` nearest nodes of each node by cosine similarity of the node vectors (``Word2Vec.most_similar``:
        the store's top-k on CUDA); the node itself is never returned. Returns ``(node ids [n, k], cosine [n, k])``."""
        return self.w2v.most_similar(nodes, k)

    def write_vectors(self, path: str, chunk: int = 1 << 15) -> None:
        """word2vec's text format, written by rank 0: a ``num_nodes dimensions`` line, then ``id v1 ... vd`` per node,
        with the ids of the input file when the graph has them."""
        self.worker.wait_sync()
        if self.server.my_rank() != 0:
            return
        E = self.vectors().cpu().numpy()
        ids = self.graph.node_ids if self.graph.node_ids is not None else np.arange(self.num_nodes)
        with open(path, "w") as f:
            f.write(f"{E.shape[0]} {E.shape[1]}\n")
            for i in range(0, E.shape[0], chunk):
                f.writelines(f"{int(ids[i + j])} " + " ".join(f"{x:.6f}" for x in row) + "\n"
                             for j, row in enumerate(E[i:i + chunk]))


def roc_auc(pos: np.ndarray, neg: np.ndarray) -> float:
    """Mann-Whitney estimate of the ROC AUC of scores ``pos`` over ``neg``, ties counting one half."""
    pos, neg = np.asarray(pos, dtype=np.float64), np.asarray(neg, dtype=np.float64)
    if pos.size == 0 or neg.size == 0:
        raise ValueError("roc_auc needs at least one positive and one negative score")
    _, inv, cnt = np.unique(np.concatenate([pos, neg]), return_inverse=True, return_counts=True)
    rank = (np.cumsum(cnt) - (cnt - 1) / 2.0)[inv.reshape(-1)]               # 1-based, ties averaged
    return float((rank[:pos.size].sum() - pos.size * (pos.size + 1) / 2.0) / (pos.size * neg.size))


def split_edges(src, dst, fraction: float, directed: bool, seed: int):
    """Holds out a seeded ``fraction`` of the distinct edges (undirected: of the pairs ``u < v``, so both directions
    leave together; self-loops always stay). Returns ``(train_src, train_dst, train_index, held [2, k])``:
    ``train_index`` selects the kept input lines (for their weights)."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    if not 0.0 <= fraction < 1.0:
        raise ValueError(f"the held-out fraction must be in [0, 1), got {fraction}")
    a, b = (src, dst) if directed else (np.minimum(src, dst), np.maximum(src, dst))
    n = int(max(src.max(), dst.max())) + 1 if src.size else 1
    uniq, inv = np.unique(a * n + b, return_inverse=True)
    cand = np.flatnonzero(uniq // n != uniq % n)
    rng = np.random.default_rng(seed)
    held = np.zeros(uniq.size, dtype=bool)
    held[rng.choice(cand, int(round(fraction * cand.size)), replace=False)] = True
    keep = ~held[inv.reshape(-1)]
    h = uniq[held]
    return src[keep], dst[keep], np.flatnonzero(keep), np.stack([h // n, h % n])


def sample_non_edges(src, dst, num_nodes: int, count: int, directed: bool, seed: int) -> np.ndarray:
    """``count`` distinct seeded node pairs ``[2, count]`` that are not edges of ``(src, dst)`` (either direction when
    undirected) and not self-loops."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    n = int(num_nodes)
    a, b = (src, dst) if directed else (np.minimum(src, dst), np.maximum(src, dst))
    edges = np.unique(a * n + b)
    rng = np.random.default_rng(seed)
    got = np.zeros(0, dtype=np.int64)
    while got.size < count:
        u, v = rng.integers(0, n, 2 * count), rng.integers(0, n, 2 * count)
        if not directed:
            u, v = np.minimum(u, v), np.maximum(u, v)
        k = u * n + v
        k = k[(u != v) & ~np.isin(k, edges)]
        got = np.concatenate([got, k[~np.isin(k, got)]])
        _, first = np.unique(got, return_index=True)
        got = got[np.sort(first)]
    got = got[:count]
    return np.stack([got // n, got % n])
