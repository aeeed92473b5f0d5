"""Graphs for the walk-based embeddings (node2vec, DeepWalk): a CSR on the host or a device, the native SNAP edge-list
reader, and seeded synthetic generators (planted partition, R-MAT)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

WEIGHT_BITS = 24          # a node's largest edge weight is quantised to 2^24
MAX_NODES = (1 << 31) - 1


@dataclass
class Graph:
    """A CSR graph: node ``v``'s out-neighbours are ``neighbors[offsets[v]:offsets[v + 1]]`` (int64 offsets, int32
    neighbours sorted within each node). A weighted graph also has ``cum_weights`` (int64) there: the inclusive prefix
    sums of the node's quantised edge weights. ``node_ids`` (int64 numpy, optional): the id of each node in the input
    file."""
    offsets: torch.Tensor
    neighbors: torch.Tensor
    cum_weights: Optional[torch.Tensor]
    directed: bool
    node_ids: Optional[np.ndarray] = None

    @property
    def num_nodes(self) -> int:
        return self.offsets.numel() - 1

    @property
    def num_edges(self) -> int:
        """stored edges: an undirected edge counts in both directions, a self-loop once"""
        return self.neighbors.numel()

    @property
    def weighted(self) -> bool:
        return self.cum_weights is not None

    @property
    def device(self) -> torch.device:
        return self.offsets.device

    def degrees(self) -> torch.Tensor:
        return self.offsets[1:] - self.offsets[:-1]

    def to(self, device) -> "Graph":
        return Graph(self.offsets.to(device), self.neighbors.to(device),
                     None if self.cum_weights is None else self.cum_weights.to(device), self.directed, self.node_ids)

    @staticmethod
    def from_edges(src, dst, weight=None, directed: bool = False, num_nodes: Optional[int] = None) -> "Graph":
        """Builds the CSR of the edges ``src[i] -> dst[i]`` (array-likes of non-negative integer ids). Undirected input
        stores both directions (a self-loop once); duplicate edges are merged, their weights added. With ``weight``,
        each positive finite weight becomes ``max(1, rint(w / max_w(node) * 2^24))`` against the largest weight of its
        source node, so draws compare integers. ``num_nodes`` defaults to the largest id + 1. ``ValueError`` on a
        negative id, an id >= ``num_nodes``, a non-positive or non-finite weight, or more than 2^31 - 1 nodes."""
        src = np.asarray(src).reshape(-1)
        dst = np.asarray(dst).reshape(-1)
        if src.shape != dst.shape:
            raise ValueError(f"src and dst differ in length: {src.size} and {dst.size}")
        for name, a in (("src", src), ("dst", dst)):
            if a.size and not np.issubdtype(a.dtype, np.integer):
                raise ValueError(f"{name} must hold integer node ids, got dtype {a.dtype}")
        src, dst = src.astype(np.int64), dst.astype(np.int64)
        if src.size and min(int(src.min()), int(dst.min())) < 0:
            raise ValueError("node ids must be non-negative")
        top = int(max(src.max(), dst.max())) + 1 if src.size else 0
        n = top if num_nodes is None else int(num_nodes)
        if n > MAX_NODES:
            raise ValueError(f"a graph has at most 2^31 - 1 nodes, got {n}")
        if top > n:
            raise ValueError(f"node id {top - 1} is not below num_nodes = {n}")
        w = None
        if weight is not None:
            w = np.asarray(weight, dtype=np.float64).reshape(-1)
            if w.shape != src.shape:
                raise ValueError(f"weight has {w.size} entries for {src.size} edges")
            if not np.all(np.isfinite(w)) or not np.all(w > 0):
                raise ValueError("edge weights must be positive and finite")
        if not directed:
            loop = src == dst
            src, dst = np.concatenate([src, dst[~loop]]), np.concatenate([dst, src[~loop]])
            if w is not None:
                w = np.concatenate([w, w[~loop]])
        uniq, inv = np.unique(src * n + dst, return_inverse=True)      # sorted by (source, neighbour), merged
        s, d = uniq // max(n, 1), uniq % max(n, 1)
        offsets = np.concatenate([[0], np.cumsum(np.bincount(s, minlength=n))]).astype(np.int64)
        cum = None
        if w is not None:
            ws = np.bincount(inv.reshape(-1), weights=w, minlength=uniq.size)
            wmax = np.zeros(n, dtype=np.float64)
            np.maximum.at(wmax, s, ws)
            q = np.maximum(1, np.rint(ws / wmax[s] * float(1 << WEIGHT_BITS))).astype(np.int64)
            total = np.concatenate([[0], np.cumsum(q)])
            cum = torch.from_numpy(total[1:] - np.repeat(total[offsets[:-1]], np.diff(offsets)))
        return Graph(torch.from_numpy(offsets), torch.from_numpy(d.astype(np.int32)), cum, bool(directed))


def read_edge_list(path: str):
    """Reads a SNAP-style edge list (``src dst [weight]`` per line, ``#`` comments) with the native parser. Ids are
    relabelled ``0 .. n-1`` in ascending order of the file's ids. Returns ``(src int64, dst int64, weight float64 or
    None, ids int64)``, numpy arrays; ``ids[label]`` is the file's id. A malformed line raises ``ValueError`` naming its
    line number."""
    from .. import AdapmError, _C

    try:
        return _C.read_edge_list(str(path))
    except AdapmError as e:
        raise ValueError(str(e)) from None


def planted_partition(communities: int, size: int, p_in: float, p_out: float, seed: int = 0):
    """Undirected edges of a planted-partition (stochastic block) graph: ``communities`` groups of ``size`` nodes, node
    ``v`` in group ``v // size``; each pair inside a group is an edge with probability ``p_in``, each pair across groups
    with ``p_out``. Returns ``(src, dst)`` int64 numpy arrays with ``src < dst``."""
    rng = np.random.default_rng(seed)
    n = communities * size
    iu, ju = np.triu_indices(n, 1)
    same = iu // size == ju // size
    keep = rng.random(iu.size) < np.where(same, p_in, p_out)
    return iu[keep].astype(np.int64), ju[keep].astype(np.int64)


def rmat_edges(scale: int, edge_factor: int, a: float = 0.57, b: float = 0.19, c: float = 0.19, seed: int = 0,
               weighted: bool = False):
    """R-MAT edges (Chakrabarti et al., 2004; the Graph500 parameters by default): ``edge_factor * 2^scale`` directed
    edges over ``2^scale`` nodes, each placed by ``scale`` recursive quadrant draws, which gives power-law degrees and
    hubs. Node ids are permuted at random so the hubs are spread over the id range. Returns ``(src, dst, weight)``
    int64 / float64 numpy arrays; ``weight`` is uniform in (0, 1] when ``weighted``, else None."""
    rng = np.random.default_rng(seed)
    m = edge_factor << scale
    src = np.zeros(m, dtype=np.int64)
    dst = np.zeros(m, dtype=np.int64)
    for bit in range(scale):
        u = rng.random(m)
        right = (u >= a) & (u < a + b) | (u >= a + b + c)
        down = u >= a + b
        src |= down.astype(np.int64) << bit
        dst |= right.astype(np.int64) << bit
    perm = rng.permutation(1 << scale).astype(np.int64)
    w = 1.0 - rng.random(m) if weighted else None
    return perm[src], perm[dst], w
