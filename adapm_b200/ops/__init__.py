"""Torch-facing wrappers of the hand-written sm_90a kernels (csrc/cuda/ops_*.cu).

All ops take CUDA tensors, run on the current CUDA stream and operate directly on the
parameter store of a ``Server`` with ``backend='cuda'`` (local HBM and NVLink-mapped peers).
They fail loudly when the native extension or a CUDA device is missing - there is no eager
fallback on a GPU box.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from .. import _C


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _i64(t: torch.Tensor, name: str) -> torch.Tensor:
    if not (t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous CUDA int64 tensor")
    return t


def sgns_step(server, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor, embed_dim: int,
              alpha: float, loss: torch.Tensor, stats: Optional[torch.Tensor] = None, impl: str = "auto") -> None:
    """Fused word2vec SGNS step (pull + score + AdaGrad + push) on ``server``'s store.

    ``centers``/``contexts``: [B] syn0 / syn1 keys; ``negatives``: [B, neg] syn1 keys;
    ``loss``: float32[1] accumulated (+=) with the summed logistic loss;
    ``stats``: optional int64[4] accumulated with (local rows, remote rows, slow-path rows, updates).
    ``impl``: ``tma`` (rows prefetched by the TMA engine into a shared-memory ring), ``ldg`` (register
    variant) or ``auto`` (tma when the shape fits, else ldg).

    On one GPU the tma step is deterministic: every pair reads the rows at the start of the step and two runs from
    the same inputs give bit-identical rows and loss. It takes ``embed_dim <= 336`` (a multiple of 4) and
    ``neg <= 30``. Outside that window ``auto`` runs the in-place register kernel, whose runs are not reproducible
    when keys repeat, and ``tma`` raises ``AdapmError``.
    """
    _i64(centers, "centers"); _i64(contexts, "contexts"); _i64(negatives, "negatives")
    B = centers.numel()
    neg = negatives.numel() // max(B, 1)
    if contexts.numel() != B or negatives.numel() != B * neg:
        raise ValueError("contexts must have B entries and negatives B*neg entries")
    if not (loss.is_cuda and loss.dtype == torch.float32):
        raise TypeError("loss must be a CUDA float32 tensor")
    _C.sgns_step(server._impl.backend_handle(), _stream(centers), centers.data_ptr(), contexts.data_ptr(),
                 negatives.data_ptr(), B, neg, int(embed_dim), float(alpha), loss.data_ptr(),
                 stats.data_ptr() if stats is not None else 0, {"auto": 0, "ldg": 1, "tma": 2}[impl])


CBOW_MAX_DIM = 336
CBOW_MAX_TARGETS = 32
CBOW_MAX_CONTEXTS = 32


def cbow_step(server, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor, embed_dim: int,
              alpha: float, loss: torch.Tensor, stats: Optional[torch.Tensor] = None,
              deterministic: Optional[bool] = None) -> None:
    """Fused word2vec CBOW step (csrc/cuda/ops_cbow.cu) on ``server``'s store: one window per ``centers[i]`` (syn1 key;
    < 0: the window does nothing) with the syn0 keys ``contexts[i]`` ([B, C], -1 = padding) and the syn1 keys
    ``negatives[i]`` ([B, neg]). The rule is :func:`adapm_b200.models.word2vec.cbow_reference_step`'s: ``h`` = mean of
    the context embeddings, one AdaGrad push per (window, target) of ``g_t h`` and one per context occurrence of
    ``neu1e = sum_t g_t t``; a negative equal to the centre is skipped. ``loss``: float32[1], accumulated (+=);
    ``stats``: optional int64[4] accumulated with (local rows, remote rows, slow-path rows, updates).
    ``4 <= embed_dim <= 336`` and a multiple of 4, ``1 + neg <= 32``, ``C <= 32``.

    ``deterministic``: ``None`` picks the deterministic step on a single-GPU server (start-of-step reads, updates
    grouped by key and summed in fixed point: bit-identical runs, 8 launches) and the in-place kernel (one launch,
    Hogwild between windows) on several GPUs; ``False`` forces the in-place kernel; ``True`` on several GPUs raises
    ``ValueError``."""
    _i64(centers, "centers"); _i64(contexts, "contexts"); _i64(negatives, "negatives"); _f32(loss, "loss")
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not (
            4 <= int(embed_dim) <= CBOW_MAX_DIM and int(embed_dim) % 4 == 0):
        raise ValueError(f"embed_dim must be a multiple of 4 in [4, {CBOW_MAX_DIM}], got {embed_dim}")
    B = centers.numel()
    if contexts.dim() != 2 or contexts.shape[0] != B or not 1 <= contexts.shape[1] <= CBOW_MAX_CONTEXTS:
        raise ValueError(f"contexts must be [B, C] with 1 <= C <= {CBOW_MAX_CONTEXTS}, got {tuple(contexts.shape)}")
    if negatives.dim() != 2 or negatives.shape[0] != B or negatives.shape[1] + 1 > CBOW_MAX_TARGETS:
        raise ValueError(f"negatives must be [B, neg] with 1 + neg <= {CBOW_MAX_TARGETS}, got {tuple(negatives.shape)}")
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, server.num_servers() == 1 if deterministic is None else deterministic)
    _C.cbow_step(server._impl.backend_handle(), _stream(centers), centers.data_ptr(), contexts.data_ptr(),
                 negatives.data_ptr(), B, int(contexts.shape[1]), int(negatives.shape[1]), int(embed_dim), float(alpha),
                 loss.data_ptr(), stats.data_ptr() if stats is not None else 0, det)


def hs_step(server, centers: torch.Tensor, contexts: torch.Tensor, tree, embed_dim: int, alpha: float,
            loss: torch.Tensor, stats: Optional[torch.Tensor] = None, deterministic: Optional[bool] = None) -> None:
    """Fused word2vec hierarchical-softmax step (csrc/cuda/ops_cbow.cu, the CBOW body with Huffman-path targets) on
    ``server``'s store. Item ``i`` has the syn1 key ``centers[i] = 2 w + 1`` (< 0: the item does nothing) and the syn0
    keys ``contexts[i]`` ([B, C], -1 = padding; skip-gram passes C = 1). Its targets are the inner nodes on word
    ``w``'s path in ``tree`` (a :class:`adapm_b200.utils.text.HuffmanTree` on the device; node ``n`` is the row
    ``2 n + 1``), labelled ``1 - code bit``. The rule is
    :func:`adapm_b200.models.word2vec.hs_reference_step`'s: ``h`` = mean of the context embeddings, a node with
    ``|h . node| >= 6`` is skipped (but counted in the loss), one AdaGrad push per (item, node) of ``g h`` and one per
    context occurrence of ``neu1e = sum_j g_j node_j``. ``loss``: float32[1], accumulated (+=); ``stats``: optional
    int64[4] accumulated with (local rows, remote rows, slow-path rows, updates). ``4 <= embed_dim <= 336`` and a
    multiple of 4, ``C <= 32``, ``tree.max_len <= 32``. Centres must be syn1 keys of words in the tree.

    ``deterministic`` as for :func:`cbow_step`: ``None`` picks the deterministic step (8 launches, bit-identical runs)
    on a single-GPU server and the in-place kernel (one launch) on several GPUs; ``True`` on several GPUs raises."""
    _i64(centers, "centers"); _i64(contexts, "contexts"); _f32(loss, "loss")
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not (
            4 <= int(embed_dim) <= CBOW_MAX_DIM and int(embed_dim) % 4 == 0):
        raise ValueError(f"embed_dim must be a multiple of 4 in [4, {CBOW_MAX_DIM}], got {embed_dim}")
    B = centers.numel()
    if contexts.dim() != 2 or contexts.shape[0] != B or not 1 <= contexts.shape[1] <= CBOW_MAX_CONTEXTS:
        raise ValueError(f"contexts must be [B, C] with 1 <= C <= {CBOW_MAX_CONTEXTS}, got {tuple(contexts.shape)}")
    if not 1 <= int(tree.max_len) <= CBOW_MAX_TARGETS:
        raise ValueError(f"the tree's paths must be 1 to {CBOW_MAX_TARGETS} nodes long, got max_len {tree.max_len}")
    V = tree.codes.numel()
    for t, name, dt, n in ((tree.offsets, "tree.offsets", torch.int64, V + 1), (tree.nodes, "tree.nodes", torch.int32, None),
                           (tree.codes, "tree.codes", torch.int32, V)):
        if not (t.device == centers.device and t.dtype == dt and t.is_contiguous() and (n is None or t.numel() == n)):
            raise TypeError(f"{name} must be a contiguous {dt} tensor on {centers.device}"
                            + (f" with {n} entries" if n is not None else ""))
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, server.num_servers() == 1 if deterministic is None else deterministic)
    _C.hs_step(server._impl.backend_handle(), _stream(centers), centers.data_ptr(), contexts.data_ptr(), B,
               int(contexts.shape[1]), tree.offsets.data_ptr(), tree.nodes.data_ptr(), tree.codes.data_ptr(), V,
               int(tree.max_len), int(embed_dim), float(alpha), loss.data_ptr(),
               stats.data_ptr() if stats is not None else 0, det)


class SgnsSharedStep:
    """word2vec SGNS with one set of negatives shared by all pairs of a batch, on the tensor cores
    (csrc/cuda/ops_sgns_shared.cu; SURVEY K7's GEMM formulation, an option next to the reference-faithful fused step).

    Per step: ONE Pull of the rows ``[centers | contexts | shared negatives]`` through the store (any protocol state,
    local HBM or NVLink), three wgmma GEMMs (scores, center gradient, negative gradient; bf16 operands, fp32
    accumulation) with three elementwise kernels around them, ONE Push of the additive ``[embedding | AdaGrad]`` updates.
    ``B`` pairs x ``Nn`` negatives = B * Nn sample pairs for 2 B + Nn rows of traffic.
    """

    def __init__(self, server, worker, batch_pairs: int, shared_negatives: int, embed_dim: int):
        if batch_pairs % 32 or shared_negatives % 32:
            raise ValueError("batch_pairs and shared_negatives must be multiples of 32")
        self.server, self.worker = server, worker
        self.B, self.Nn, self.d = int(batch_pairs), int(shared_negatives), int(embed_dim)
        dev = server.device
        rows = 2 * self.B + self.Nn
        self.keys = torch.empty(rows, dtype=torch.int64, device=dev)
        self.R = torch.empty(rows * 2 * self.d, dtype=torch.float32, device=dev)
        self.U = torch.empty(rows * 2 * self.d, dtype=torch.float32, device=dev)
        self.ws = torch.empty(_C.sgns_shared_workspace_bytes(self.B, self.Nn, self.d), dtype=torch.uint8, device=dev)
        self._push_ts = None

    def __call__(self, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor, alpha: float,
                 loss: torch.Tensor) -> None:
        """``centers`` / ``contexts``: [B] syn0 / syn1 keys, ``negatives``: [Nn] syn1 keys (CUDA int64);
        ``loss``: CUDA float32[1], accumulated (+=) with the summed logistic loss of the B * (1 + Nn) sample pairs."""
        B, Nn = self.B, self.Nn
        if centers.numel() != B or contexts.numel() != B or negatives.numel() != Nn:
            raise ValueError(f"expected {B} centers / contexts and {Nn} shared negatives")
        if not (loss.is_cuda and loss.dtype == torch.float32):
            raise TypeError("loss must be a CUDA float32 tensor")
        if self._push_ts is not None:      # the previous step's Push: done long ago (same stream), retire its ticket
            self.worker.wait(self._push_ts)
        k = self.keys
        k[:B].copy_(centers.view(-1)); k[B:2 * B].copy_(contexts.view(-1)); k[2 * B:].copy_(negatives.view(-1))
        self.worker.wait(self.worker.pull(k, self.R, True))
        _C.sgns_shared_core(_stream(k), self.R.data_ptr(), k[B:2 * B].data_ptr(), k[2 * B:].data_ptr(), B, Nn, self.d,
                            float(alpha), self.ws.data_ptr(), self.U.data_ptr(), loss.data_ptr())
        self._push_ts = self.worker.push(k, self.U, True)


def sgns_shared_reference_step(table: torch.Tensor, centers: torch.Tensor, contexts: torch.Tensor, negatives: torch.Tensor,
                               d: int, alpha: float, emulate_bf16: bool = False):
    """Plain fp32 PyTorch reference of :class:`SgnsSharedStep` on a dense ``[keys, 2 d]`` table (tests): returns
    ``(new_table, loss)``. Same rule as the kernels: all gradients from the values before the step, AdaGrad accumulator
    read before the update, duplicates add up. ``emulate_bf16`` rounds the operands of the three contractions to bf16
    like the tensor-core path does (fp32 accumulation, everything else fp32)."""
    t = table.to(torch.float32)
    e0, a0 = t[centers, :d], t[centers, d:]
    ec, ac = t[contexts, :d], t[contexts, d:]
    en, an = t[negatives, :d], t[negatives, d:]

    def grad(f, label):
        g = label - torch.sigmoid(f)
        g = torch.where(f > 6, torch.full_like(f, label - 1.0), g)
        return torch.where(f < -6, torch.full_like(f, label), g)

    def rnd(x):
        return x.to(torch.bfloat16).to(torch.float32) if emulate_bf16 else x

    fp = (e0 * ec).sum(-1)
    gp = grad(fp, 1.0)
    e0m, enm = rnd(e0), rnd(en)
    S = e0m @ enm.t()
    mask = contexts.view(-1, 1) != negatives.view(1, -1)
    G = grad(S, 0.0) * mask
    loss = torch.log1p(torch.exp(-fp.clamp(-6, 6))).sum() + (torch.log1p(torch.exp(S.clamp(-6, 6))) * mask).sum()
    Gm = rnd(G)
    g0 = Gm @ enm + gp.unsqueeze(1) * ec
    gc = gp.unsqueeze(1) * e0
    gn = Gm.t() @ e0m
    out = t.clone()
    for keys, g, a in ((centers, g0, a0), (contexts, gc, ac), (negatives, gn, an)):
        ua = g * g
        out.index_add_(0, keys, torch.cat([alpha * g * torch.rsqrt(a + ua), ua], 1))
    return out, loss


class DeviceSampler:
    """Key sampler on the GPU: alias table (any weights, e.g. unigram^0.75), uniform or log-uniform.

    ``local_only=True`` implements the reference's *local* sampling scheme (sampling.h:361-446):
    draws are rejected until the key is resident in this GPU's HBM (owned or usable replica).

    Draw ``i`` of a call is a pure function of ``(seed, i)`` and the table; :func:`sample_keys_reference` replays it bit
    for bit and :func:`alias_draw_probabilities` gives the exact distribution a table draws. ``ValueError`` on weights
    that are negative, NaN or infinite, none or all zero, or more than 2^31 - 1 of them, and on ``num_keys`` outside
    ``[1, 2^32)``.
    """

    def __init__(self, server, *, weights: Optional[torch.Tensor] = None, distribution: str = "alias",
                 first_key: int = 0, key_stride: int = 1, num_keys: Optional[int] = None):
        self.server = server
        self.first_key, self.key_stride = int(first_key), int(key_stride)
        dev = server.device
        if weights is not None:
            w = torch.as_tensor(weights, dtype=torch.float64)
            n = w.numel()
            if n > (1 << 31) - 1:                    # before the weights are copied: the int32 alias cannot index them
                raise ValueError(f"{n} weights, at most 2^31 - 1 fit the alias table")
            w = w.contiguous().cpu()
            prob = torch.empty(n, dtype=torch.float32)
            alias = torch.empty(n, dtype=torch.int32)
            try:
                _C.build_alias_table(w.data_ptr(), n, prob.data_ptr(), alias.data_ptr())
            except _C.AdapmError as e:
                raise ValueError(str(e)) from None
            self.kind, self.n = 0, n
            self.prob, self.alias = prob.to(dev), alias.to(dev)
        else:
            if num_keys is None:
                raise ValueError("num_keys is required for uniform / log-uniform sampling")
            if distribution not in ("uniform", "log-uniform"):
                raise ValueError(f"distribution must be 'uniform' or 'log-uniform' without weights, got {distribution!r}")
            if not 1 <= int(num_keys) < 1 << 32:     # the bucket is (hi * num_keys) >> 32 in 64 bits
                raise ValueError(f"num_keys must be in [1, 2^32), got {num_keys}")
            self.kind = _SAMPLER_KINDS[distribution]
            self.n = int(num_keys)
            self.prob = torch.zeros(1, dtype=torch.float32, device=dev)
            self.alias = torch.zeros(1, dtype=torch.int32, device=dev)
        self.stats = torch.zeros(2, dtype=torch.int64, device=dev)  # (residency checks, give-ups)

    def sample(self, n: int, seed: int, local_only: bool = False, out: Optional[torch.Tensor] = None,
               max_tries: int = 64) -> torch.Tensor:
        if out is None:
            out = torch.empty(n, dtype=torch.int64, device=self.server.device)
        _i64(out, "out")
        _C.sample_keys(self.server._impl.backend_handle(), _stream(out), self.kind, self.prob.data_ptr(),
                       self.alias.data_ptr(), self.n, self.first_key, self.key_stride, out.data_ptr(), out.numel(),
                       int(seed) & 0xFFFFFFFFFFFFFFFF, bool(local_only), int(max_tries), self.stats.data_ptr())
        return out


def track_current_stream(server) -> None:
    """Tell the sync engine that kernels touching the store run on the current CUDA stream."""
    _C.track_stream(server._impl.backend_handle(), torch.cuda.current_stream().cuda_stream)


def _f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous CUDA float32 tensor")
    return t


def _check_deterministic(server, deterministic: bool) -> bool:
    if deterministic and server.num_servers() > 1:
        raise ValueError("deterministic=True needs a single-GPU server: on several GPUs rows move between ranks "
                         "during the step")
    return bool(deterministic)


def kge_complex_step(server, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, labels: torch.Tensor,
                     embed_dim: int, eta: float, gamma_entity: float, gamma_relation: float, loss: torch.Tensor,
                     stats: Optional[torch.Tensor] = None, dropout_entity: float = 0.0, dropout_relation: float = 0.0,
                     seed: int = 0, deterministic: bool = False) -> None:
    """Fused ComplEx training calls: for every i, one Model::train(s[i], r[i], o[i], label[i]) of the
    reference (pull 3 rows, optional dropout on the pulled copies, score, BCE gradient, L2 on positives, AdaGrad,
    push 3 rows). The dropout mask is ``kge_dropout_mask(seed, ...)``.

    ``deterministic=True`` (single-GPU servers only, else ``ValueError``): every call reads the state at the start of
    the step, the updates are summed in fixed point and applied once per row after the step, so that the same inputs
    give bit-identical rows and loss in every run (three kernel launches instead of one). The default adds the updates
    in place."""
    _i64(subj, "subj"); _i64(rel, "rel"); _i64(obj, "obj"); _f32(labels, "labels"); _f32(loss, "loss")
    n = subj.numel()
    if not (rel.numel() == n and obj.numel() == n and labels.numel() == n):
        raise ValueError("subj, rel, obj and labels must have the same length")
    det = _check_deterministic(server, deterministic)
    _C.kge_complex_step(server._impl.backend_handle(), _stream(subj), subj.data_ptr(), rel.data_ptr(), obj.data_ptr(),
                        labels.data_ptr(), n, int(embed_dim), float(eta), float(gamma_entity), float(gamma_relation),
                        loss.data_ptr(), stats.data_ptr() if stats is not None else 0, float(dropout_entity),
                        float(dropout_relation), int(seed) & 0xFFFFFFFFFFFFFFFF, det)


def kge_rescal_step(server, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, labels: torch.Tensor,
                    embed_dim: int, eta: float, gamma_entity: float, gamma_relation: float, loss: torch.Tensor,
                    stats: Optional[torch.Tensor] = None, dropout_entity: float = 0.0, dropout_relation: float = 0.0,
                    seed: int = 0, deterministic: bool = False) -> None:
    """Fused RESCAL training calls (score s^T R o, rank-1 relation gradient; relation rows are 2*d*d floats).
    ``deterministic``: as for :func:`kge_complex_step`."""
    _i64(subj, "subj"); _i64(rel, "rel"); _i64(obj, "obj"); _f32(labels, "labels"); _f32(loss, "loss")
    n = subj.numel()
    if not (rel.numel() == n and obj.numel() == n and labels.numel() == n):
        raise ValueError("subj, rel, obj and labels must have the same length")
    det = _check_deterministic(server, deterministic)
    _C.kge_rescal_step(server._impl.backend_handle(), _stream(subj), subj.data_ptr(), rel.data_ptr(), obj.data_ptr(),
                       labels.data_ptr(), n, int(embed_dim), float(eta), float(gamma_entity), float(gamma_relation),
                       loss.data_ptr(), stats.data_ptr() if stats is not None else 0, float(dropout_entity),
                       float(dropout_relation), int(seed) & 0xFFFFFFFFFFFFFFFF, det)


KGE_1VSALL_MAX_DIM = 1024
_KGE_1VSALL_MODELS = {"ComplEx": 0, "RESCAL": 1}


def _kge_1vsall_chunk(num_entities: int, queries: int, max_bytes: int) -> int:
    """Query rows per chunk: a multiple of 128 (the GEMM's row tile) whose fp32 scores and bf16 G and G^T fit
    ``max_bytes``; at most the batch's queries rounded up to 128."""
    n, npad = int(num_entities), (int(num_entities) + 7) // 8 * 8
    chunk = int(max_bytes) // (4 * n + 2 * npad + 2 * n) // 128 * 128
    if chunk < 128:
        raise ValueError(f"max_bytes={max_bytes} is too small for one tile of 128 queries against {n} entities "
                         f"(needs {128 * (4 * n + 2 * npad + 2 * n)} bytes)")
    return min(chunk, (int(queries) + 127) // 128 * 128)


def _check_kge_1vsall_shape(algorithm: str, embed_dim: int, kind: str = "1vsAll") -> None:
    if algorithm not in _KGE_1VSALL_MODELS:
        raise ValueError(f"{kind} training is defined for ComplEx and RESCAL, got {algorithm!r}")
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not 1 <= int(embed_dim) <= KGE_1VSALL_MAX_DIM:
        raise ValueError(f"embed_dim must be an integer in [1, {KGE_1VSALL_MAX_DIM}], got {embed_dim}")
    if algorithm == "ComplEx" and int(embed_dim) % 2:
        raise ValueError(f"ComplEx needs an even embed_dim (real half + imaginary half), got {embed_dim}")


def kge_1vsall_step(kv, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, num_entities: int, algorithm: str,
                    embed_dim: int, eta: float, gamma_entity: float, gamma_relation: float, loss: torch.Tensor,
                    max_bytes: int = 1 << 30) -> None:
    """1vsAll training step of ComplEx or RESCAL (csrc/cuda/ops_kge_1vsall.cu) on the store of the worker ``kv``.

    Each triple ``(subj[i], rel[i], obj[i])`` (entity keys in ``[0, num_entities)``, relation keys after them; CUDA int64)
    gives the queries ``(s, r, ?)`` and ``(?, r, o)`` with the query vectors of ``KGE._query``. Each is scored against
    every entity, ``z = <q, e_x>``, with the loss ``logsumexp(z) - z_answer``; ``loss`` (CUDA float32[1]) is accumulated
    (+=) with the sum over the ``2 B`` queries. The gradients, all from the rows at the start of the step, are
    ``softmax - onehot`` through the scores to every entity (``G^T Q``) and to the queries (``G E``), carried back to the
    given entity and the relation; L2 (``gamma_entity`` on s and o, ``gamma_relation`` on r) is added once per triple.
    Every entity row and every distinct relation row then gets one AdaGrad update ``[-eta g / sqrt(a + g^2) | g^2]``.

    One Pull of all entity rows and the batch's relation rows and one Push of their updates go through ``kv``, so the
    step works in every protocol state (local, replica, peer, in flight). The three contractions use bf16 operands and
    fp32 accumulation on the tensor cores; ``kge_1vsall_reference_step(..., emulate_bf16=True)`` is the same rule in
    float64. No floating-point atomics: on one GPU two runs with the same arguments give bit-identical rows and loss.

    ``embed_dim`` is any integer up to ``KGE_1VSALL_MAX_DIM`` (1024), even for ComplEx; the op pads it to a multiple of 8
    for the GEMMs. Queries are processed in chunks of a multiple of 128 so that the ``[chunk, N]`` fp32 scores and bf16
    G and G^T stay within ``max_bytes``. ``ValueError`` on another algorithm, a bad ``embed_dim``, ``max_bytes`` too
    small for one chunk of 128 queries, tensors of the wrong device, dtype or length, row lengths that do not match the
    model, or keys out of range."""
    _check_kge_1vsall_shape(algorithm, embed_dim)
    d, N = int(embed_dim), int(num_entities)
    server = kv.server
    if not 1 <= N < server.num_keys():
        raise ValueError(f"num_entities must be in [1, {server.num_keys()}), got {num_entities}")
    B = subj.numel()
    chunk = _kge_1vsall_chunk(N, 2 * B, max_bytes)
    for t, name in ((subj, "subj"), (rel, "rel"), (obj, "obj")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous CUDA int64 tensor")
    if not (rel.numel() == B and obj.numel() == B and B > 0):
        raise ValueError("subj, rel and obj must have the same, non-zero length")
    if not (isinstance(loss, torch.Tensor) and loss.is_cuda and loss.dtype == torch.float32 and loss.numel() >= 1):
        raise ValueError("loss must be a CUDA float32 tensor")
    if server.backend != "cuda" or server.dtype != torch.float32:
        raise ValueError("kge_1vsall_step needs a float32 CUDA store (kge_1vsall_reference_step is the other route)")
    lo_e, hi_e, lo_r, hi_r = torch.stack([torch.minimum(subj.min(), obj.min()), torch.maximum(subj.max(), obj.max()),
                                          rel.min(), rel.max()]).tolist()
    if lo_e < 0 or hi_e >= N:
        raise ValueError(f"entity keys must be in [0, {N}), got [{lo_e}, {hi_e}]")
    if lo_r < N or hi_r >= server.num_keys():
        raise ValueError(f"relation keys must be in [{N}, {server.num_keys()}), got [{lo_r}, {hi_r}]")
    rl = 2 * d * (d if algorithm == "RESCAL" else 1)
    uniq, inv = torch.unique(rel, return_inverse=True)
    lens = server._lens_t[uniq.cpu()] if server._uniform_len is None else torch.full((1,), server._uniform_len)
    if server.get_len(0) != 2 * d or N > 1 and server.get_len(N - 1) != 2 * d or bool((lens != rl).any()):
        raise ValueError(f"{algorithm} at embed_dim {d} needs entity rows of {2 * d} and relation rows of {rl} values")
    dev = subj.device
    nrel = uniq.numel()
    rel_pos = torch.argsort(inv, stable=True).to(torch.int32)
    rel_off = torch.zeros(nrel + 1, dtype=torch.int64, device=dev)
    rel_off[1:] = torch.cumsum(torch.bincount(inv, minlength=nrel), 0)
    ents = torch.stack([subj, obj], 1).view(-1)          # position 2 i: subject of triple i, 2 i + 1: its object
    ent_pos = torch.argsort(ents, stable=True).to(torch.int32)
    ent_off = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    ent_off[1:] = torch.cumsum(torch.bincount(ents, minlength=N), 0)
    keys = torch.cat([torch.arange(N, dtype=torch.int64, device=dev), uniq])
    R = torch.empty(N * 2 * d + nrel * rl, dtype=torch.float32, device=dev)
    kv.wait(kv.pull(keys, R, True))
    U = torch.empty_like(R)
    ws = torch.empty(_C.kge_1vsall_workspace_bytes(N, B, d, chunk), dtype=torch.uint8, device=dev)
    inv32 = inv.to(torch.int32)
    _C.kge_1vsall_core(_stream(subj), _KGE_1VSALL_MODELS[algorithm], R.data_ptr(), subj.data_ptr(), obj.data_ptr(),
                       inv32.data_ptr(), ent_off.data_ptr(), ent_pos.data_ptr(), rel_off.data_ptr(), rel_pos.data_ptr(),
                       N, nrel, B, d, chunk, float(eta), float(gamma_entity), float(gamma_relation), ws.data_ptr(),
                       U.data_ptr(), loss.data_ptr())
    kv.wait(kv.push(keys, U, True))


def kge_1vsall_reference_step(kv, triples: torch.Tensor, cfg, emulate_bf16: bool = False) -> float:
    """The rule of :func:`kge_1vsall_step` in float64 through Pull / Push on either backend: the CPU route of the model
    (and of float64 stores) and the test oracle. ``triples``: [B, 3] (subject, relation id, object); ``cfg``: a
    ``KGEConfig`` (``algorithm`` ComplEx or RESCAL, ``num_entities``, ``embed_dim``, ``eta``, ``gamma_entity``,
    ``gamma_relation``). ``emulate_bf16`` rounds the operands of the three contractions (queries, entities, G) to bf16
    as the tensor-core path does. Returns the summed loss of the ``2 B`` queries."""
    _check_kge_1vsall_shape(cfg.algorithm, cfg.embed_dim)
    d, N = cfg.embed_dim, cfg.num_entities
    dt = kv.server.dtype
    tr = torch.as_tensor(triples, dtype=torch.int64).view(-1, 3).cpu()
    s, r, o = tr[:, 0], tr[:, 1], tr[:, 2]
    if tr.numel() == 0 or int(torch.minimum(s, o).min()) < 0 or int(torch.maximum(s, o).max()) >= N:
        raise ValueError(f"triples must be non-empty with entity ids in [0, {N})")
    if int(r.min()) < 0 or int(r.max()) >= cfg.num_relations:
        raise ValueError(f"relation ids must be in [0, {cfg.num_relations})")
    uniq, inv = torch.unique(r, return_inverse=True)
    el, rl = 2 * d, cfg.relation_len

    def pull(keys, ln):
        v = torch.empty(keys.numel() * ln, dtype=dt)
        kv.wait(kv.pull(keys.contiguous(), v))
        return v.view(-1, ln).double()

    ent, rr = pull(torch.arange(N), el), pull(uniq + N, rl)
    E, A, Rr, Ar = ent[:, :d], ent[:, d:], rr[:, :rl // 2], rr[:, rl // 2:]
    rel = Rr[inv]
    Es, Eo = E[s], E[o]

    def rnd(x):
        return x.to(torch.bfloat16).double() if emulate_bf16 else x

    Q = _kge_queries(cfg, Es, Eo, rel)
    ans = torch.cat([o, s])
    rows = torch.arange(ans.numel())
    Qm, Em = rnd(Q), rnd(E)
    Z = Qm @ Em.t()
    lse = torch.logsumexp(Z, 1)
    loss = float((lse - Z[rows, ans]).sum())
    G = torch.exp(Z - lse.unsqueeze(1))
    G[rows, ans] -= 1
    Gm = rnd(G)
    dQ, C = Gm @ Em, Gm.t() @ Qm
    ds, do, dr = _kge_query_grads(cfg, Es, Eo, rel, dQ)
    gE = C.clone()
    gE.index_add_(0, s, ds + cfg.gamma_entity * Es)
    gE.index_add_(0, o, do + cfg.gamma_entity * Eo)
    gR = torch.zeros_like(Rr).index_add_(0, inv, dr + cfg.gamma_relation * rel)
    kv.wait(kv.push(torch.arange(N), _kge_adagrad_rows(cfg, gE, A, dt)))
    kv.wait(kv.push((uniq + N).contiguous(), _kge_adagrad_rows(cfg, gR, Ar, dt)))
    return loss


def _kge_queries(cfg, Es, Eo, rel):
    """[object queries; subject queries] of ``KGE._query`` for the triples with subject rows Es, object rows Eo and
    relation rows rel (float64)"""
    from ..models.kge import complex_query

    if cfg.algorithm == "ComplEx":
        return torch.cat([complex_query(Es, rel, conj=False), complex_query(Eo, rel, conj=True)])
    Rm = rel.view(-1, cfg.embed_dim, cfg.embed_dim)
    return torch.cat([torch.einsum("bi,bij->bj", Es, Rm), torch.einsum("bij,bj->bi", Rm, Eo)])


def _kge_query_grads(cfg, Es, Eo, rel, dQ):
    """The gradients (subject, object, relation) of the triples, given dQ = the loss's gradient w.r.t. the queries of
    :func:`_kge_queries`, without L2"""
    d, B = cfg.embed_dim, Es.shape[0]
    dqo, dqs = dQ[:B], dQ[B:]
    if cfg.algorithm == "ComplEx":
        h = d // 2
        rre, rim, a, b, a2, b2 = rel[:, :h], rel[:, h:], dqo[:, :h], dqo[:, h:], dqs[:, :h], dqs[:, h:]
        sre, sim, ore, oim = Es[:, :h], Es[:, h:], Eo[:, :h], Eo[:, h:]
        ds = torch.cat([rre * a + rim * b, rre * b - rim * a], 1)
        do = torch.cat([rre * a2 - rim * b2, rim * a2 + rre * b2], 1)
        dr = torch.cat([sre * a + sim * b + ore * a2 + oim * b2, sre * b - sim * a + oim * a2 - ore * b2], 1)
        return ds, do, dr
    Rm = rel.view(-1, d, d)
    ds = torch.einsum("bij,bj->bi", Rm, dqo)
    do = torch.einsum("bi,bij->bj", dqs, Rm)
    dr = (torch.einsum("bi,bj->bij", Es, dqo) + torch.einsum("bi,bj->bij", dqs, Eo)).reshape(B, -1)
    return ds, do, dr


def _kge_adagrad_rows(cfg, g, a, dt):
    """the flat additive updates [-eta g / sqrt(a + g^2) | g^2] of rows with gradients g and accumulators a"""
    u = torch.where(g == 0, torch.zeros_like(g), -cfg.eta * g / torch.sqrt(a + g * g))
    return torch.cat([u, g * g], 1).to(dt).contiguous().view(-1)


KGE_SHARED_CHUNK = 128


def _kge_row_lengths_ok(server, keys: torch.Tensor, length: int) -> bool:
    lens = server._lens_t[keys.cpu()] if server._uniform_len is None else torch.full((1,), server._uniform_len)
    return not bool((lens != length).any())


def kge_shared_step(kv, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, negatives: torch.Tensor,
                    num_entities: int, algorithm: str, embed_dim: int, eta: float, gamma_entity: float,
                    gamma_relation: float, loss: torch.Tensor, max_bytes: int = 1 << 30) -> None:
    """Sampled-softmax training step of ComplEx or RESCAL with shared negatives (csrc/cuda/ops_kge_1vsall.cu) on the
    store of the worker ``kv``.

    The triples ``(subj[i], rel[i], obj[i])`` (entity keys in ``[0, num_entities)``, relation keys after them; CUDA
    int64) are cut into chunks of ``KGE_SHARED_CHUNK`` (128) consecutive triples. Chunk k has one candidate list
    ``[its subjects] ++ [its objects] ++ negatives`` (``negatives``: the S >= 0 entity keys shared by the whole batch;
    they may repeat). Each triple's object query ``(s, r, ?)`` and subject query ``(?, r, o)`` (the query vectors of
    ``KGE._query``) is scored against every column of its chunk's list, ``z_j = <q, e_j>``. The positive column is the
    answer's own slot in the chunk's object (or subject) block; every other column holding the answer is masked. The
    loss of a query is ``logsumexp(z over unmasked columns) - z_pos``; ``loss`` (CUDA float32[1]) is accumulated (+=)
    with the sum over the ``2 B`` queries. The gradients, all from the rows at the start of the step, are
    ``G = softmax - onehot`` (0 at masked columns) through the scores to the list's entities (``G^T Q``) and to the
    queries (``G E``), carried back to the given entity and the relation as in :func:`kge_1vsall_step`; L2
    (``gamma_entity`` on s and o, ``gamma_relation`` on r) is added once per triple, never to an entity that is only a
    negative. Every distinct entity and relation of the step gets one AdaGrad update ``[-eta g / sqrt(a + g^2) | g^2]``
    of the sum of all its occurrences; no other row changes. The cost is linear in B and S, whatever the entity count.

    One Pull of the step's distinct entity and relation keys and one Push of their updates go through ``kv``, so the
    step works in every protocol state (local, replica, peer, in flight). The three contractions run per chunk on the
    tensor cores (bf16 operands, fp32 accumulation); ``kge_shared_reference_step(..., emulate_bf16=True)`` is the same
    rule in float64. No floating-point atomics: on one GPU two runs with the same arguments give bit-identical rows and
    loss. ``embed_dim`` is any integer up to ``KGE_1VSALL_MAX_DIM`` (1024), even for ComplEx. ``ValueError`` on another
    algorithm, a bad ``embed_dim``, tensors of the wrong device, dtype, contiguity or length, keys out of range, row
    lengths that do not match the model, a store that is not float32 on CUDA, or a workspace larger than
    ``max_bytes``."""
    _check_kge_1vsall_shape(algorithm, embed_dim, "sampled-softmax")
    d, N = int(embed_dim), int(num_entities)
    server = kv.server
    if not 1 <= N < server.num_keys():
        raise ValueError(f"num_entities must be in [1, {server.num_keys()}), got {num_entities}")
    for t, name in ((subj, "subj"), (rel, "rel"), (obj, "obj"), (negatives, "negatives")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int64 and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous CUDA int64 tensor")
    B, S = subj.numel(), negatives.numel()
    if not (rel.numel() == B and obj.numel() == B and B > 0 and negatives.dim() == 1):
        raise ValueError("subj, rel and obj must have the same, non-zero length, and negatives must be one-dimensional")
    if not (isinstance(loss, torch.Tensor) and loss.is_cuda and loss.dtype == torch.float32 and loss.numel() >= 1):
        raise ValueError("loss must be a CUDA float32 tensor")
    if server.backend != "cuda" or server.dtype != torch.float32:
        raise ValueError("kge_shared_step needs a float32 CUDA store (kge_shared_reference_step is the other route)")
    ws_bytes = _C.kge_shared_workspace_bytes(B, S, d)
    if ws_bytes > int(max_bytes):
        raise ValueError(f"max_bytes={max_bytes} is too small: B={B}, S={S}, d={d} need a workspace of {ws_bytes} bytes")
    ents_all = torch.cat([subj, obj, negatives])
    lo_e, hi_e, lo_r, hi_r = torch.stack([ents_all.min(), ents_all.max(), rel.min(), rel.max()]).tolist()
    if lo_e < 0 or hi_e >= N:
        raise ValueError(f"entity keys must be in [0, {N}), got [{lo_e}, {hi_e}]")
    if lo_r < N or hi_r >= server.num_keys():
        raise ValueError(f"relation keys must be in [{N}, {server.num_keys()}), got [{lo_r}, {hi_r}]")
    rl = 2 * d * (d if algorithm == "RESCAL" else 1)
    ents, einv = torch.unique(ents_all, return_inverse=True)
    uniq, inv = torch.unique(rel, return_inverse=True)
    if not (_kge_row_lengths_ok(server, ents, 2 * d) and _kge_row_lengths_ok(server, uniq, rl)):
        raise ValueError(f"{algorithm} at embed_dim {d} needs entity rows of {2 * d} and relation rows of {rl} values")
    dev = subj.device
    ch = KGE_SHARED_CHUNK
    nch = (B + ch - 1) // ch
    Bp, Lr = nch * ch, (2 * ch + S + 7) // 8 * 8
    ls, lo, ln = einv[:B], einv[B:2 * B], einv[2 * B:]
    # the padded batch: padding triples point at row 0 and are masked (their list slots hold -1)
    pad = torch.full((Bp - B,), -1, dtype=torch.int64, device=dev)
    cand = torch.full((nch, Lr), -1, dtype=torch.int64, device=dev)
    cand[:, :ch] = torch.cat([ls, pad]).view(nch, ch)
    cand[:, ch:2 * ch] = torch.cat([lo, pad]).view(nch, ch)
    cand[:, 2 * ch:2 * ch + S] = ln
    s_p, o_p = torch.cat([ls, pad + 1]), torch.cat([lo, pad + 1])
    rel_p = torch.cat([inv, pad + 1]).to(torch.int32)
    base = torch.arange(Bp, dtype=torch.int64, device=dev).view(nch, ch)
    qorder = torch.cat([base, base + Bp], 1).view(-1)
    # occurrences: list columns in (chunk, column) order, then the given entities (2 i: subject, 2 i + 1: object)
    occ = torch.cat([cand.view(-1), torch.stack([ls, lo], 1).view(-1)])
    Ne = ents.numel()
    occ = torch.where(occ < 0, Ne, occ)
    ent_pos = torch.argsort(occ, stable=True).to(torch.int32)
    ent_off = torch.zeros(Ne + 1, dtype=torch.int64, device=dev)
    ent_off[1:] = torch.cumsum(torch.bincount(occ, minlength=Ne + 1)[:Ne], 0)
    nrel = uniq.numel()
    rel_pos = torch.argsort(inv, stable=True).to(torch.int32)
    rel_off = torch.zeros(nrel + 1, dtype=torch.int64, device=dev)
    rel_off[1:] = torch.cumsum(torch.bincount(inv, minlength=nrel), 0)
    keys = torch.cat([ents, uniq])
    R = torch.empty(Ne * 2 * d + nrel * rl, dtype=torch.float32, device=dev)
    kv.wait(kv.pull(keys, R, True))
    U = torch.empty_like(R)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _C.kge_shared_core(_stream(subj), _KGE_1VSALL_MODELS[algorithm], R.data_ptr(), s_p.data_ptr(), o_p.data_ptr(),
                       rel_p.data_ptr(), cand.data_ptr(), qorder.data_ptr(), ent_off.data_ptr(), ent_pos.data_ptr(),
                       rel_off.data_ptr(), rel_pos.data_ptr(), Ne, nrel, B, S, d, float(eta), float(gamma_entity),
                       float(gamma_relation), ws.data_ptr(), U.data_ptr(), loss.data_ptr())
    kv.wait(kv.push(keys, U, True))


def kge_shared_reference_step(kv, triples: torch.Tensor, negatives: torch.Tensor, cfg, emulate_bf16: bool = False) -> float:
    """The rule of :func:`kge_shared_step` in float64 through Pull / Push on either backend: the CPU route of the model
    (and of float64 stores) and the test oracle. ``triples``: [B, 3] (subject, relation id, object); ``negatives``: the
    S >= 0 shared entity ids; ``cfg``: a ``KGEConfig`` (``algorithm`` ComplEx or RESCAL, ``num_entities``,
    ``embed_dim``, ``eta``, ``gamma_entity``, ``gamma_relation``). ``emulate_bf16`` rounds the operands of the three
    contractions (queries, list entities, G) to bf16 as the tensor-core path does. Returns the summed loss of the ``2 B``
    queries."""
    _check_kge_1vsall_shape(cfg.algorithm, cfg.embed_dim, "sampled-softmax")
    N = cfg.num_entities
    dt = kv.server.dtype
    tr = torch.as_tensor(triples, dtype=torch.int64).view(-1, 3).cpu()
    neg = torch.as_tensor(negatives, dtype=torch.int64).view(-1).cpu()
    s, r, o = tr[:, 0], tr[:, 1], tr[:, 2]
    ents_all = torch.cat([s, o, neg])
    if tr.numel() == 0 or int(ents_all.min()) < 0 or int(ents_all.max()) >= N:
        raise ValueError(f"triples must be non-empty with entity ids (and negatives) in [0, {N})")
    if int(r.min()) < 0 or int(r.max()) >= cfg.num_relations:
        raise ValueError(f"relation ids must be in [0, {cfg.num_relations})")
    B = s.numel()
    ents, einv = torch.unique(ents_all, return_inverse=True)
    ls, lo, ln = einv[:B], einv[B:2 * B], einv[2 * B:]
    uniq, inv = torch.unique(r, return_inverse=True)
    rl = cfg.relation_len

    def pull(keys, width):
        v = torch.empty(keys.numel() * width, dtype=dt)
        kv.wait(kv.pull(keys.contiguous(), v))
        return v.view(-1, width).double()

    ent, rr = pull(ents, 2 * cfg.embed_dim), pull(uniq + N, rl)
    E, A, Rr, Ar = ent[:, :cfg.embed_dim], ent[:, cfg.embed_dim:], rr[:, :rl // 2], rr[:, rl // 2:]
    rel = Rr[inv]
    Es, Eo = E[ls], E[lo]

    def rnd(x):
        return x.to(torch.bfloat16).double() if emulate_bf16 else x

    Q = _kge_queries(cfg, Es, Eo, rel)
    Qm, Em = rnd(Q), rnd(E)
    dQ = torch.zeros_like(Q)
    gE = torch.zeros_like(E)
    loss = 0.0
    for c0 in range(0, B, KGE_SHARED_CHUNK):
        idx = torch.arange(c0, min(B, c0 + KGE_SHARED_CHUNK))
        n = idx.numel()
        lst = torch.cat([ls[idx], lo[idx], ln])                  # the chunk's list: subjects, objects, negatives
        qi = torch.cat([idx, idx + B])                           # its object queries, then its subject queries
        ans = torch.cat([lo[idx], ls[idx]])
        pos = torch.cat([n + torch.arange(n), torch.arange(n)])
        rows = torch.arange(2 * n)
        live = lst.view(1, -1) != ans.view(-1, 1)
        live[rows, pos] = True
        Ek = Em[lst]
        Z = (Qm[qi] @ Ek.t()).masked_fill(~live, float("-inf"))
        lse = torch.logsumexp(Z, 1)
        loss += float((lse - Z[rows, pos]).sum())
        G = torch.exp(Z - lse.unsqueeze(1))
        G[rows, pos] -= 1
        Gm = rnd(G)
        dQ[qi] = Gm @ Ek
        gE.index_add_(0, lst, Gm.t() @ Qm[qi])
    ds, do, dr = _kge_query_grads(cfg, Es, Eo, rel, dQ)
    gE.index_add_(0, ls, ds + cfg.gamma_entity * Es)
    gE.index_add_(0, lo, do + cfg.gamma_entity * Eo)
    gR = torch.zeros_like(Rr).index_add_(0, inv, dr + cfg.gamma_relation * rel)
    kv.wait(kv.push(ents, _kge_adagrad_rows(cfg, gE, A, dt)))
    kv.wait(kv.push((uniq + N).contiguous(), _kge_adagrad_rows(cfg, gR, Ar, dt)))
    return loss


TRANSE_MAX_DIM = 512
TRANSE_MAX_NEG = 64
_NORM_EPS = 1e-12


def _check_transe_shape(embed_dim: int, p: int) -> None:
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not (
            4 <= int(embed_dim) <= TRANSE_MAX_DIM and int(embed_dim) % 4 == 0):
        raise ValueError(f"embed_dim must be a multiple of 4 in [4, {TRANSE_MAX_DIM}], got {embed_dim}")
    if p not in (1, 2) or isinstance(p, bool):
        raise ValueError(f"p must be 1 or 2, got {p}")


def kge_transe_step(server, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, neg: torch.Tensor, embed_dim: int,
                    p: int, margin: float, eta: float, gamma_entity: float, gamma_relation: float, loss: torch.Tensor,
                    stats: Optional[torch.Tensor] = None, deterministic: bool = False) -> None:
    """Fused TransE training step (csrc/cuda/ops_transe.cu) on ``server``'s store: one warp per positive triple
    ``(subj[i], rel[i], obj[i])`` (store keys) with the entity keys ``neg[i]`` ([B, 2n]; the first n replace the object,
    the last n the subject). Rows are ``[embedding (embed_dim) | AdaGrad (embed_dim)]``; entity rows are normalised on
    read (``e / max(|e|_2, 1e-12)``), the store rows are never rescaled. The rule is :func:`transe_reference_step`'s:
    margin-ranking loss ``sum_j max(0, margin + D_pos - D_neg_j)`` with ``D = |s^ + r - o^|_p``, one AdaGrad push per
    row of the positive and one per negative of an active pair. ``loss``: float32[1], accumulated (+=); ``stats``:
    optional int64[4] accumulated with (local rows, peer rows, slow-path rows, pushes issued).

    ``deterministic=True`` (single-GPU servers only): start-of-step reads, fixed-point sums, bit-identical runs (three
    launches instead of one); the AdaGrad increment of one push is clamped to 2^24 there (see ops_transe.cu)."""
    _i64(subj, "subj"); _i64(rel, "rel"); _i64(obj, "obj"); _i64(neg, "neg"); _f32(loss, "loss")
    _check_transe_shape(embed_dim, p)
    B = subj.numel()
    if not (rel.numel() == B and obj.numel() == B):
        raise ValueError("subj, rel and obj must have the same length")
    if neg.dim() != 2 or neg.shape[0] != B or neg.shape[1] % 2 or neg.shape[1] > TRANSE_MAX_NEG:
        raise ValueError(f"neg must be [B, 2n] with 2n <= {TRANSE_MAX_NEG}, got {tuple(neg.shape)}")
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, deterministic)
    _C.kge_transe_step(server._impl.backend_handle(), _stream(subj), subj.data_ptr(), rel.data_ptr(), obj.data_ptr(),
                       neg.data_ptr(), B, int(neg.shape[1]), int(embed_dim), int(p), float(margin), float(eta),
                       float(gamma_entity), float(gamma_relation), loss.data_ptr(),
                       stats.data_ptr() if stats is not None else 0, det)


def transe_reference_step(kv, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, neg: torch.Tensor, embed_dim: int,
                          p: int, margin: float, eta: float, gamma_entity: float, gamma_relation: float):
    """The TransE rule of :func:`kge_transe_step` in float64 through Pull / Push (CPU servers, float64 rows, and the
    oracle of the tests). Every row is read at the start of the step. Returns ``(loss, pushes)``.

    Per positive triple with x = s^ + r - o^, D = |x|_p and u = dD/dx (sign(x) for p = 1, x / |x| for p = 2, 0 at 0):
    a negative pair j is active when ``margin + D_pos - D_neg_j > 0``. The gradients of an active pair: object
    corrupted - s^ and r get ``u - u_j``, o^ ``-u``, the negative's o'^ ``+u_j``; subject corrupted - s^ ``u``, r
    ``u - u_j``, o^ ``u_j - u``, s'^ ``-u_j``. Through the normalisation ``g_e = (g_e^ - e^ (e^ . g_e^)) / max(|e|, 1e-12)``;
    L2 adds ``gamma_entity * s``, ``gamma_relation * r``, ``gamma_entity * o`` on the raw rows. Pushes
    ``[-eta g / sqrt(acc + g^2) | g^2]`` (0 where g == 0) with the pulled accumulator: s, r and o once per triple with their
    summed gradients, every negative of an active pair once."""
    _check_transe_shape(embed_dim, p)
    d = int(embed_dim)
    subj, rel, obj = (t.reshape(-1).cpu() for t in (subj, rel, obj))
    neg = neg.cpu()
    B, nn = neg.shape
    n = nn // 2
    f64 = torch.float64

    def pull(keys):
        v = torch.empty(keys.numel() * 2 * d, dtype=kv.server.dtype)
        if keys.numel():
            kv.wait(kv.pull(keys.contiguous(), v))
        v = v.view(-1, 2 * d).to(f64)
        return v[:, :d], v[:, d:]

    def nrm(e):
        inv = 1.0 / e.norm(dim=-1, keepdim=True).clamp(min=_NORM_EPS)
        return e * inv, inv

    def dist(x):
        return x.abs().sum(-1) if p == 1 else x.norm(dim=-1)

    def ddx(x, D):
        if p == 1:
            return torch.sign(x)
        return torch.where(D.unsqueeze(-1) > 0, x / D.clamp(min=1e-300).unsqueeze(-1), torch.zeros_like(x))

    def back(g_hat, e_hat, inv):
        return (g_hat - e_hat * (e_hat * g_hat).sum(-1, keepdim=True)) * inv

    Es, As = pull(subj)
    Er, Ar = pull(rel)
    Eo, Ao = pull(obj)
    En, An = pull(neg.reshape(-1))
    En, An = En.view(B, nn, d), An.view(B, nn, d)
    sh, inv_s = nrm(Es)
    oh, inv_o = nrm(Eo)
    nh, inv_n = nrm(En)
    x = sh + Er - oh
    Dp = dist(x)
    xn = torch.cat([(sh + Er).unsqueeze(1) - nh[:, :n], nh[:, n:] + (Er - oh).unsqueeze(1)], 1)
    Dn = dist(xn)
    term = margin + Dp.unsqueeze(1) - Dn
    act = term > 0
    loss = float(term.clamp(min=0).sum())
    u = ddx(x, Dp)
    un = ddx(xn, Dn) * act.unsqueeze(-1)
    k = act.sum(1, keepdim=True).to(f64)
    Uo, Us = un[:, :n].sum(1), un[:, n:].sum(1)
    gs = back(k * u - Uo, sh, inv_s) + gamma_entity * Es
    gr = k * u - Uo - Us + gamma_relation * Er
    go = back(Us - k * u, oh, inv_o) + gamma_entity * Eo
    gn = back(torch.cat([un[:, :n], -un[:, n:]], 1), nh, inv_n)

    def upd(g, a):
        ue = torch.where(g != 0, -eta * g / torch.sqrt(a + g * g), torch.zeros_like(g))
        return torch.cat([ue, g * g], -1).to(kv.server.dtype).contiguous().view(-1)

    kv.wait(kv.push(subj.contiguous(), upd(gs, As)))
    kv.wait(kv.push(rel.contiguous(), upd(gr, Ar)))
    kv.wait(kv.push(obj.contiguous(), upd(go, Ao)))
    sel = act.reshape(-1)
    if bool(sel.any()):
        kv.wait(kv.push(neg.reshape(-1)[sel].contiguous(), upd(gn.reshape(-1, d)[sel], An.reshape(-1, d)[sel])))
    return loss, 3 * B + int(sel.sum())


ROTATE_MAX_DIM = 512
ROTATE_MAX_NEG = 256


def _check_rotate_shape(embed_dim: int) -> None:
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not (
            8 <= int(embed_dim) <= ROTATE_MAX_DIM and int(embed_dim) % 8 == 0):
        raise ValueError(f"embed_dim must be a multiple of 8 in [8, {ROTATE_MAX_DIM}], got {embed_dim}")


def _check_rotate_neg(neg: torch.Tensor, B: int) -> None:
    if neg.dim() != 2 or neg.shape[0] != B or neg.shape[1] % 2 or not 2 <= neg.shape[1] <= ROTATE_MAX_NEG:
        raise ValueError(f"neg must be [B, 2n] with 2 <= 2n <= {ROTATE_MAX_NEG}, got {tuple(neg.shape)}")


def kge_rotate_step(server, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, neg: torch.Tensor, embed_dim: int,
                    margin: float, adversarial_temperature: float, eta: float, gamma_entity: float, loss: torch.Tensor,
                    stats: Optional[torch.Tensor] = None, deterministic: bool = False) -> None:
    """Fused RotatE training step (csrc/cuda/ops_rotate.cu) on ``server``'s store: one warp per positive triple
    ``(subj[i], rel[i], obj[i])`` (store keys) with the entity keys ``neg[i]`` ([B, 2n], 2 <= 2n <= 256; the first n
    replace the object, the last n the subject). Entity rows are ``[z (embed_dim) | AdaGrad (embed_dim)]`` with ``z``
    interleaved ``(re_0, im_0, re_1, im_1, ...)``; relation rows are ``[phases (embed_dim / 2) | AdaGrad (embed_dim / 2)]``
    in radians; ``embed_dim % 8 == 0``, ``8 <= embed_dim <= 512``. The rule is :func:`rotate_reference_step`'s: distance
    ``D = sum_i |(s o rho - o)_i|``, loss ``softplus(D+ - margin) + 1/2 sum_side sum_j w_j softplus(margin - D_j)`` with
    the self-adversarial weights ``w = softmax(adversarial_temperature (margin - D))`` per side, one AdaGrad push per row
    of the positive and one per negative. ``loss``: float32[1], accumulated (+=); ``stats``: optional int64[4]
    accumulated with (local rows, peer rows, slow-path rows, pushes issued = (3 + 2n) per triple).

    ``deterministic=True`` (single-GPU servers only): start-of-step reads, fixed-point sums, bit-identical runs (three
    launches instead of one)."""
    _i64(subj, "subj"); _i64(rel, "rel"); _i64(obj, "obj"); _i64(neg, "neg"); _f32(loss, "loss")
    _check_rotate_shape(embed_dim)
    B = subj.numel()
    if not (rel.numel() == B and obj.numel() == B):
        raise ValueError("subj, rel and obj must have the same length")
    _check_rotate_neg(neg, B)
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, deterministic)
    _C.kge_rotate_step(server._impl.backend_handle(), _stream(subj), subj.data_ptr(), rel.data_ptr(), obj.data_ptr(),
                       neg.data_ptr(), B, int(neg.shape[1]), int(embed_dim), float(margin),
                       float(adversarial_temperature), float(eta), float(gamma_entity), loss.data_ptr(),
                       stats.data_ptr() if stats is not None else 0, det)


def _as_complex(e: torch.Tensor) -> torch.Tensor:
    """interleaved (re, im) rows [..., d] -> complex [..., d / 2]"""
    return torch.view_as_complex(e.reshape(*e.shape[:-1], -1, 2).contiguous())


def _as_interleaved(z: torch.Tensor) -> torch.Tensor:
    return torch.view_as_real(z).reshape(*z.shape[:-1], -1)


def rotate_reference_step(kv, subj: torch.Tensor, rel: torch.Tensor, obj: torch.Tensor, neg: torch.Tensor, embed_dim: int,
                          margin: float, adversarial_temperature: float, eta: float, gamma_entity: float):
    """The RotatE rule of :func:`kge_rotate_step` in float64 through Pull / Push (CPU servers, float64 rows, and the
    oracle of the tests). Every row is read at the start of the step. Returns ``(loss, pushes)``.

    Per positive triple, with rho = e^{i theta}, x = a o rho - b, D(x) = sum_i |x_i| and u = x / |x| (0 where |x_i| = 0):
    the positive x = s o rho - o, object-side negatives x_j = s o rho - o'_j, subject-side x_j = s'_j o rho - o;
    ``w_j = softmax_j(adversarial_temperature (margin - D_j))`` over the n negatives of a side (no gradient); loss
    ``softplus(D+ - margin) + 1/2 sum_side sum_j w_j softplus(margin - D_j)``. ``dD/da = conj(rho) o u``, ``dD/db = -u``,
    ``dD/dtheta_i = -Im(conj(u_i) a_i rho_i)``, scaled by ``sigmoid(D+ - margin)`` for the positive and
    ``-1/2 w_j sigmoid(margin - D_j)`` for negative j. L2 adds ``gamma_entity * s`` and ``gamma_entity * o`` to the raw
    entity rows; phases get none. Pushes ``[-eta g / sqrt(acc + g^2) | g^2]`` (0 where g == 0) with the pulled
    accumulator: s, r and o once per triple, every negative once."""
    _check_rotate_shape(embed_dim)
    d = int(embed_dim)
    m = d // 2
    subj, rel, obj = (t.reshape(-1).cpu() for t in (subj, rel, obj))
    neg = neg.cpu()
    B = subj.numel()
    _check_rotate_neg(neg, B)
    nn = neg.shape[1]
    h = nn // 2
    f64 = torch.float64
    alpha = float(adversarial_temperature)

    def pull(keys, ln):
        v = torch.empty(keys.numel() * 2 * ln, dtype=kv.server.dtype)
        if keys.numel():
            kv.wait(kv.pull(keys.contiguous(), v))
        v = v.view(-1, 2 * ln).to(f64)
        return v[:, :ln], v[:, ln:]

    def dist(x):
        return x.abs().sum(-1)

    def unit(x):
        a = x.abs()
        return torch.where(a > 0, x / torch.where(a > 0, a, torch.ones_like(a)), torch.zeros_like(x))

    def dtheta(u, p):
        return -(u.conj() * p).imag

    def softplus(x):
        return torch.logaddexp(x, torch.zeros_like(x))

    Es, As = pull(subj, d)
    Th, Ar = pull(rel, m)
    Eo, Ao = pull(obj, d)
    En, An = pull(neg.reshape(-1), d)
    s, o, n = _as_complex(Es), _as_complex(Eo), _as_complex(En).view(B, nn, m)
    rho = torch.complex(torch.cos(Th), torch.sin(Th))
    sr = s * rho
    nsr = n[:, h:] * rho.unsqueeze(1)
    x = sr - o
    xo = sr.unsqueeze(1) - n[:, :h]
    xs = nsr - o.unsqueeze(1)
    Dp = dist(x)
    Dn = torch.cat([dist(xo), dist(xs)], 1)
    z = alpha * (margin - Dn)
    w = torch.cat([torch.softmax(z[:, :h], 1), torch.softmax(z[:, h:], 1)], 1)
    loss = float(softplus(Dp - margin).sum() + 0.5 * (w * softplus(margin - Dn)).sum())
    cp = torch.sigmoid(Dp - margin).unsqueeze(1)
    cn = (-0.5 * w * torch.sigmoid(margin - Dn)).unsqueeze(2)
    u, uo, us = unit(x), unit(xo), unit(xs)
    rc = rho.conj()
    gs = (cp * u + (cn[:, :h] * uo).sum(1)) * rc
    go = -cp * u - (cn[:, h:] * us).sum(1)
    gt = cp * dtheta(u, sr) + (cn[:, :h] * dtheta(uo, sr.unsqueeze(1))).sum(1) + (cn[:, h:] * dtheta(us, nsr)).sum(1)
    gn = torch.cat([-cn[:, :h] * uo, cn[:, h:] * rc.unsqueeze(1) * us], 1)

    def upd(g, a):
        ue = torch.where(g != 0, -eta * g / torch.sqrt(a + g * g), torch.zeros_like(g))
        return torch.cat([ue, g * g], -1).to(kv.server.dtype).contiguous().view(-1)

    kv.wait(kv.push(subj.contiguous(), upd(_as_interleaved(gs) + gamma_entity * Es, As)))
    kv.wait(kv.push(rel.contiguous(), upd(gt, Ar)))
    kv.wait(kv.push(obj.contiguous(), upd(_as_interleaved(go) + gamma_entity * Eo, Ao)))
    kv.wait(kv.push(neg.reshape(-1).contiguous(), upd(_as_interleaved(gn).reshape(-1, d), An)))
    return loss, B * (3 + nn)


DIST_COMPLEX = 3          # the kernels' code of p = "complex"


def _dist_p(p, normalize) -> int:
    """validated metric code: 1, 2, or DIST_COMPLEX for p = "complex" (which never normalises)"""
    if isinstance(p, str):
        if p != "complex":
            raise ValueError(f"p must be 1, 2 or 'complex', got {p!r}")
        if normalize:
            raise ValueError("normalize=True is not defined for p='complex' (RotatE scores raw entity rows)")
        return DIST_COMPLEX
    if p not in (1, 2) or isinstance(p, bool):
        raise ValueError(f"p must be 1, 2 or 'complex', got {p}")
    return int(p)


def complex_dist(q: torch.Tensor, e: torch.Tensor, chunk_elems: int = 1 << 24) -> torch.Tensor:
    """``D[i, j] = sum_k |q_i,k - e_j,k|`` over the complex values of interleaved (re, im) rows ``q`` [M, dim] and ``e``
    [N, dim], in the dtype of the inputs, computed in column chunks of about ``chunk_elems`` elements."""
    M, dim = q.shape
    N = e.shape[0]
    qc = q.reshape(M, 1, dim // 2, 2)
    out = torch.empty(M, N, dtype=q.dtype, device=q.device)
    step = max(1, chunk_elems // max(1, M * dim))
    for j in range(0, N, step):
        diff = qc - e[j:j + step].reshape(1, -1, dim // 2, 2)
        out[:, j:j + step] = torch.linalg.vector_norm(diff, dim=-1).sum(-1)
    return out


def _dist_operands(server, q, keys, dim, p, normalize, exclude, stats, M):
    p = _dist_p(p, normalize)
    _i64(keys, "keys")
    _check_transe_shape(dim, 1)
    if q.dim() != 2 or q.shape[1] != int(dim):
        raise ValueError(f"q must be a matrix [M, dim = {dim}]")
    if not (q.is_cuda and q.device == keys.device):
        raise TypeError("q must be a CUDA tensor on the device of keys")
    _f32(q, "q")
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 2):
        raise TypeError("stats must be a CUDA int64 tensor with 2 entries")
    _check_topk(M, keys.numel(), 1, exclude, None)
    _, eo, ec = _topk_operands(q.device, exclude, None)
    if q.data_ptr() % 16:              # the kernels read q in 16-byte vectors: a view at an odd offset is copied
        q = q.clone()
    return q, eo, ec, p


def _dist_slices(server, M, N):
    return _C.dist_num_slices(server._impl.backend_handle(), M, N, _TOPK_GRACE_TILES if server.num_servers() > 1 else 0)


def gather_dist_rank_count(server, q: torch.Tensor, keys: torch.Tensor, dim: int, p: int, normalize: bool,
                           true_col: torch.Tensor, exclude=None, stats: Optional[torch.Tensor] = None):
    """Rank counts by distance against parameter-store rows (csrc/cuda/ops_dist.cu): with ``D(i, j) = |q_i - e_j|_p``
    (fp32 on the CUDA cores, ``e_j`` = the first ``dim`` values of store row ``keys[j]``, divided by
    ``max(|e_j|_2, 1e-12)`` when ``normalize``), returns int64 ``(raw, filtered)`` [M] with
    ``raw[i] = #{j != true_col[i] : D(i, j) < D(i, true_col[i])}`` and ``filtered`` the same without the columns of the
    CSR ``exclude = (offsets int64 [M + 1], cols int64 [nnz])`` (ascending per row, as for :func:`gather_gemm_topk`).
    The true distance comes from the kernel's own distance function, bit-identical to the column's. ``stats``: as for
    :func:`gather_gemm`; on several ranks the call waits and raises ``RuntimeError`` if a row could not be resolved.

    ``p="complex"`` (RotatE): ``D(i, j) = sum_k |(q_i - e_j)_k|`` over the complex values of interleaved (re, im) rows,
    each modulus and sum explicitly rounded in a fixed order; ``normalize`` must be False (else ``ValueError``)."""
    M = q.shape[0] if q.dim() == 2 else 0
    q, eo, ec, p = _dist_operands(server, q, keys, dim, p, normalize, exclude, stats, M)
    _i64(true_col, "true_col")
    if true_col.numel() != M:
        raise ValueError(f"true_col must have M = {M} entries")
    N = keys.numel()
    raw = torch.zeros(M, dtype=torch.int64, device=q.device)
    filt = torch.zeros(M, dtype=torch.int64, device=q.device)
    if M == 0:
        return raw, filt
    if N == 0 or bool(((true_col < 0) | (true_col >= N)).any()):
        raise ValueError("true_col entries must be column indices in [0, N)")
    dtrue = torch.empty(M, dtype=torch.float32, device=q.device)
    own = _gather_stats(server, stats, q.device)
    _C.gather_dist_rank_count(server._impl.backend_handle(), _stream(q), q.data_ptr(), keys.data_ptr(), M, N, int(dim),
                              int(p), bool(normalize), _dist_slices(server, M, N), true_col.data_ptr(), eo, ec,
                              dtrue.data_ptr(), raw.data_ptr(), filt.data_ptr(), own.data_ptr() if own is not None else 0)
    _gathered("gather_dist_rank_count", own, stats)
    return raw, filt


def gather_dist_topk(server, q: torch.Tensor, keys: torch.Tensor, dim: int, k: int, p: int, normalize: bool,
                     exclude=None, stats: Optional[torch.Tensor] = None):
    """The ``k`` columns of smallest distance per query (the distances of :func:`gather_dist_rank_count`): returns
    ``(values = -D fp32 [M, k], indices int64 [M, k])`` with :func:`gather_gemm_topk`'s conventions - smallest distance
    first, ties to the smaller column, NaN never selected, ``(-inf, -1)`` padding, ``1 <= k <= 64``, exclusions as a
    CSR; indices are positions into ``keys``. Per-slice lists are merged by the top-k merge kernel. ``p``: 1, 2 or
    ``"complex"``, as for :func:`gather_dist_rank_count`."""
    M = q.shape[0] if q.dim() == 2 else 0
    if isinstance(k, bool) or int(k) != k or not 1 <= int(k) <= TOPK_MAX_K:
        raise ValueError(f"k must be an integer in [1, {TOPK_MAX_K}], got {k}")
    q, eo, ec, p = _dist_operands(server, q, keys, dim, p, normalize, exclude, stats, M)
    k, N = int(k), keys.numel()
    if M == 0 or N == 0:
        return _topk_empty(M, k, q.device)
    S = _dist_slices(server, M, N)
    part_v, part_c, vals, idx = _topk_outputs(M, S, k, q.device)
    own = _gather_stats(server, stats, q.device)
    _C.gather_dist_topk(server._impl.backend_handle(), _stream(q), q.data_ptr(), keys.data_ptr(), M, N, int(dim), int(p),
                        bool(normalize), k, S, eo, ec, part_v.data_ptr(), part_c.data_ptr(), vals.data_ptr(),
                        idx.data_ptr(), own.data_ptr() if own is not None else 0)
    _gathered("gather_dist_topk", own, stats)
    return vals, idx


def dist_rank_reference(q: torch.Tensor, e: torch.Tensor, p: int, true_col: torch.Tensor, excluded=None):
    """PyTorch ``cdist`` ranking with the rule of :func:`gather_dist_rank_count` on dense candidates ``e`` [N, dim]
    (already normalised if wanted): ``(raw, filtered)`` int64 [M]; ``excluded``: bool [M, N] or None. ``p="complex"``
    uses :func:`complex_dist` (chunked; there is no ``cdist`` form of it)."""
    D = complex_dist(q, e) if isinstance(p, str) and p == "complex" else torch.cdist(q, e, p=float(p))
    dt = D.gather(1, true_col.view(-1, 1))
    better = D < dt
    better.scatter_(1, true_col.view(-1, 1), False)
    raw = better.sum(1)
    filt = (better & ~excluded).sum(1) if excluded is not None else raw.clone()
    return raw, filt


def _mix32(x: torch.Tensor) -> torch.Tensor:
    m = 0xFFFFFFFF
    x = x & m
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & m
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & m
    x = x ^ (x >> 16)
    return x


def kge_dropout_mask(seed: int, n_calls: int, which: int, n_elems: int, p: float, relation: bool = False) -> torch.Tensor:
    """The [n_calls, n_elems] scale mask (0 or 1/(1-p)) that the fused KGE kernels apply to the pulled copy of row
    ``which`` (0 subject, 1 relation, 2 object) of every training call - bit-exact mirror of the device function
    (csrc/cuda/ops_kge.cu: Dropout::keep), for the numerics tests."""
    if p <= 0:
        return torch.ones(n_calls, n_elems)
    seed &= 0xFFFFFFFFFFFFFFFF
    s32 = (((seed ^ (seed >> 32)) & 0xFFFFFFFF) * 2654435761 + (0x22 if relation else 0x11)) & 0xFFFFFFFF
    call = torch.arange(n_calls, dtype=torch.int64).view(-1, 1)
    elem = torch.arange(n_elems, dtype=torch.int64).view(1, -1)
    u = _mix32(_mix32((s32 + call * 3 + which) & 0xFFFFFFFF) ^ ((elem * 0x9E3779B9) & 0xFFFFFFFF))
    keep = ((u >> 8).to(torch.float32) * (1.0 / 16777216.0)) >= torch.tensor(p, dtype=torch.float32)
    return keep.to(torch.float32) * (1.0 / (1.0 - torch.tensor(p, dtype=torch.float32)))


def mf_step(server, row_keys: torch.Tensor, col_keys: torch.Tensor, x: torch.Tensor, row_nnz: torch.Tensor,
            col_nnz: torch.Tensor, rank: int, eps: float, lam: float, loss: torch.Tensor,
            stats: Optional[torch.Tensor] = None, deterministic: bool = False) -> None:
    """Fused matrix-factorisation SGD/AdaGrad step over a batch of non-zeros (reference apps/mf/update.h).
    ``deterministic``: as for :func:`kge_complex_step` (single-GPU servers only; the summed squared error is reduced in
    a fixed order)."""
    _i64(row_keys, "row_keys"); _i64(col_keys, "col_keys"); _f32(x, "x"); _f32(loss, "loss")
    for t, nm in ((row_nnz, "row_nnz"), (col_nnz, "col_nnz")):
        if not (t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()):
            raise TypeError(f"{nm} must be a contiguous CUDA int32 tensor")
    n = row_keys.numel()
    det = _check_deterministic(server, deterministic)
    _C.mf_step(server._impl.backend_handle(), _stream(x), row_keys.data_ptr(), col_keys.data_ptr(), x.data_ptr(),
               row_nnz.data_ptr(), col_nnz.data_ptr(), n, int(rank), float(eps), float(lam), loss.data_ptr(),
               stats.data_ptr() if stats is not None else 0, det)


BPR_MAX_RANK = 512
BPR_MAX_NEG = 256


def _check_bpr_shape(rank: int, neg: torch.Tensor, B: int) -> None:
    if isinstance(rank, bool) or int(rank) != rank or not (4 <= int(rank) <= BPR_MAX_RANK and int(rank) % 4 == 0):
        raise ValueError(f"rank must be a multiple of 4 in [4, {BPR_MAX_RANK}], got {rank}")
    if neg.dim() != 2 or neg.shape[0] != B or not 1 <= neg.shape[1] <= BPR_MAX_NEG:
        raise ValueError(f"neg must be [B = {B}, n] with 1 <= n <= {BPR_MAX_NEG}, got {tuple(neg.shape)}")


def mf_bpr_step(server, users: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor, rank: int, eps: float, lam: float,
                loss: torch.Tensor, stats: Optional[torch.Tensor] = None, deterministic: bool = False) -> None:
    """Fused BPR step of implicit-feedback matrix factorisation (csrc/cuda/ops_bpr.cu) on ``server``'s store: one warp
    per positive ``(users[b], pos[b])`` (store keys of a user row and an item row) with the item keys ``neg[b]``
    (int64 [B, n], 1 <= n <= 256, used as given: repeats and a negative equal to the positive included). Rows are the
    squared-loss layout ``[factors (rank) | AdaGrad (rank)]``, ``rank`` a multiple of 4 in [4, 512]. The rule is
    :func:`bpr_reference_step`'s: loss ``sum_j softplus(-x_j)`` with ``x_j = <w_u, h_i> - <w_u, h_j>``, one AdaGrad push
    per user, positive item and negative occurrence (``2 + n`` per positive). ``loss``: float32[1], accumulated (+=);
    ``stats``: optional int64[4] accumulated with (local rows, peer rows, slow-path rows, pushes issued).

    ``deterministic=True`` (single-GPU servers only): start-of-step reads, fixed-point sums, bit-identical runs (three
    launches instead of one); the AdaGrad increment of one push is clamped to 2^24 there (see ops_bpr.cu)."""
    _i64(users, "users"); _i64(pos, "pos"); _i64(neg, "neg"); _f32(loss, "loss")
    B = users.numel()
    if pos.numel() != B:
        raise ValueError("users and pos must have the same length")
    _check_bpr_shape(rank, neg, B)
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, deterministic)
    _C.mf_bpr_step(server._impl.backend_handle(), _stream(users), users.data_ptr(), pos.data_ptr(), neg.data_ptr(), B,
                   int(neg.shape[1]), int(rank), float(eps), float(lam), loss.data_ptr(),
                   stats.data_ptr() if stats is not None else 0, det)


def bpr_reference_step(kv, users: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor, rank: int, eps: float, lam: float):
    """The BPR rule of :func:`mf_bpr_step` in float64 through Pull / Push (CPU servers, float64 rows, and the oracle of
    the tests). Every row is read at the start of the step. Returns ``(loss, pushes)``.

    Per positive (u, i) with negatives j: ``x_j = <w_u, h_i> - <w_u, h_j>``, ``c_j = sigmoid(-x_j)``, ``C = sum_j c_j``,
    ``S = sum_j c_j h_j``; gradients ``g_u = S - C h_i + lam w_u``, ``g_i = -C w_u + lam h_i``, ``g_j = c_j w_u +
    lam h_j``; pushes ``[-eps g / sqrt(acc + g^2) | g^2]`` (0 where g == 0) with the pulled accumulator: u and i once per
    positive, every negative once per occurrence. The loss is ``sum softplus(-x_j)`` (no L2 term)."""
    users, pos = users.reshape(-1).cpu(), pos.reshape(-1).cpu()
    neg = neg.cpu()
    B = users.numel()
    if neg.dim() != 2 or neg.shape[0] != B or neg.shape[1] < 1:
        raise ValueError(f"neg must be [B = {B}, n] with n >= 1, got {tuple(neg.shape)}")
    n, r = neg.shape[1], int(rank)
    f64 = torch.float64

    def pull(keys):
        v = torch.empty(keys.numel() * 2 * r, dtype=kv.server.dtype)
        if keys.numel():
            kv.wait(kv.pull(keys.contiguous(), v))
        v = v.view(-1, 2 * r).to(f64)
        return v[:, :r], v[:, r:]

    W, Aw = pull(users)
    H, Ah = pull(pos)
    Hn, An = pull(neg.reshape(-1))
    Hn = Hn.view(B, n, r)
    x = (W * H).sum(-1, keepdim=True) - torch.einsum("br,bnr->bn", W, Hn)
    loss = float(torch.nn.functional.softplus(-x).sum())
    c = torch.sigmoid(-x)
    C = c.sum(1, keepdim=True)
    gu = torch.einsum("bn,bnr->br", c, Hn) - C * H + lam * W
    gi = -C * W + lam * H
    gn = c.unsqueeze(-1) * W.unsqueeze(1) + lam * Hn

    def upd(g, a):
        ue = torch.where(g != 0, -eps * g / torch.sqrt(a + g * g), torch.zeros_like(g))
        return torch.cat([ue, g * g], -1).to(kv.server.dtype).contiguous().view(-1)

    if B:
        kv.wait(kv.push(users.contiguous(), upd(gu, Aw)))
        kv.wait(kv.push(pos.contiguous(), upd(gi, Ah)))
        kv.wait(kv.push(neg.reshape(-1).contiguous(), upd(gn.reshape(-1, r), An)))
    return loss, B * (2 + n)


GLOVE_MAX_DIM = 508
GLOVE_MAX_WINDOW = 16
# default device-memory budget of glove_cooccurrence: leaves most of an 80 GB card to the training tables
GLOVE_COOC_MAX_BYTES = 8 << 30


def glove_cooccurrence(tokens: torch.Tensor, offsets: torch.Tensor, vocab_size: int, window: int,
                       symmetric: bool = True, distance_weighting: bool = True, rank: int = 0, world: int = 1,
                       max_bytes: int = GLOVE_COOC_MAX_BYTES, info: Optional[dict] = None):
    """GloVe's co-occurrence matrix (glove.c's ``cooccur.c``) of an encoded corpus, counted on the device
    (csrc/cuda/ops_cooc.cu). ``tokens``: int32 word ids in ``[0, vocab_size)``; ``offsets``: int64 ``[n_sentences + 1]``,
    sentence ``s`` is ``tokens[offsets[s]:offsets[s + 1]]`` (both contiguous CUDA tensors, e.g. from
    ``NativeCorpus.arrays()``). For every pair of positions of one sentence where word ``a`` comes ``k <= window``
    positions before word ``b``, ``X[a][b] += 1 / k`` (``1`` with ``distance_weighting=False``), and with ``symmetric``
    also ``X[b][a]``. Windows never cross a sentence. ``1 <= window <= 16``.

    Only rows ``a`` with ``a % world == rank`` are kept: ranks that each count the whole corpus get disjoint partitions
    that together make the full matrix. The sums are exact (integer numerators over ``lcm(1..window)`` in 64 bits,
    divided once and rounded to float32), so the result is bit-identical to :func:`utils.text.cooccurrence_reference`
    and independent of ``max_bytes``, which bounds the device memory of the call (the corpus is processed in token
    chunks whose sorted counts are merged; the working set is allocated with ``cudaMalloc``, outside PyTorch's caching
    allocator); a budget too small for the result raises ``RuntimeError``.

    Returns ``(rows int32, cols int32, x float32)`` on the device of ``tokens``, sorted by ``(row, col)``. ``info``: a
    dict that receives ``chunks`` (token chunks processed) and ``denominator`` (``lcm(1..window)`` or 1)."""
    if not (tokens.is_cuda and tokens.dtype == torch.int32 and tokens.is_contiguous() and tokens.dim() == 1):
        raise TypeError("tokens must be a contiguous 1-D CUDA int32 tensor")
    if not (offsets.is_cuda and offsets.dtype == torch.int64 and offsets.is_contiguous() and offsets.dim() == 1
            and offsets.device == tokens.device):
        raise TypeError("offsets must be a contiguous 1-D CUDA int64 tensor on the device of tokens")
    if offsets.numel() < 1 or int(offsets[0]) != 0 or int(offsets[-1]) != tokens.numel():
        raise ValueError("offsets must start at 0 and end at the number of tokens")
    if isinstance(window, bool) or int(window) != window or not 1 <= int(window) <= GLOVE_MAX_WINDOW:
        raise ValueError(f"window must be an integer in [1, {GLOVE_MAX_WINDOW}], got {window}")
    if not 1 <= int(world) or not 0 <= int(rank) < int(world):
        raise ValueError(f"rank must be in [0, world), got rank {rank}, world {world}")
    if int(vocab_size) < 1 or int(max_bytes) < 1:
        raise ValueError("vocab_size and max_bytes must be positive")
    dev = tokens.device
    with torch.cuda.device(dev):
        c = _C.Cooccurrence(_stream(tokens), tokens.data_ptr(), tokens.numel(), offsets.data_ptr(), offsets.numel() - 1,
                            int(vocab_size), int(window), bool(symmetric), bool(distance_weighting), int(rank),
                            int(world), int(max_bytes))
        n = c.run()
        rows = torch.empty(n, dtype=torch.int32, device=dev)
        cols = torch.empty(n, dtype=torch.int32, device=dev)
        x = torch.empty(n, dtype=torch.float32, device=dev)
        c.write(rows.data_ptr(), cols.data_ptr(), x.data_ptr())
        if info is not None:
            info["chunks"], info["denominator"] = c.chunks(), c.denominator()
        torch.cuda.current_stream(dev).synchronize()
        del c
    return rows, cols, x


def _check_glove_dim(embed_dim: int) -> None:
    if isinstance(embed_dim, bool) or int(embed_dim) != embed_dim or not (
            4 <= int(embed_dim) <= GLOVE_MAX_DIM and int(embed_dim) % 4 == 0):
        raise ValueError(f"embed_dim must be a multiple of 4 in [4, {GLOVE_MAX_DIM}], got {embed_dim}")


def _check_glove_rates(x_max: float, alpha: float) -> None:
    if not float(x_max) > 0 or not float(alpha) >= 0:
        raise ValueError(f"x_max must be > 0 and alpha >= 0, got x_max {x_max}, alpha {alpha}")


def glove_step(server, words: torch.Tensor, ctxs: torch.Tensor, x: torch.Tensor, embed_dim: int, eta: float,
               x_max: float, alpha: float, loss: torch.Tensor, stats: Optional[torch.Tensor] = None,
               deterministic: bool = False) -> None:
    """Fused GloVe step (csrc/cuda/ops_glove.cu) on ``server``'s store: one warp per non-zero ``(words[b], ctxs[b],
    x[b])``, where ``words`` holds the keys of word rows (``2 i``), ``ctxs`` those of context rows (``2 j + 1``) and
    ``x > 0`` the co-occurrence values. Rows are ``[vector (d) | bias, 0, 0, 0 | AdaGrad (d + 4)]``, ``d = embed_dim``
    a multiple of 4 in [4, 508]. The rule is :func:`glove_reference_step`'s: ``diff = <w, c> + b + b~ - ln X``, weight
    ``f = min(1, (X / x_max)^alpha)``, loss ``f diff^2 / 2``, one AdaGrad push per row and non-zero (``2`` per
    non-zero). ``loss``: float32[1], accumulated (+=); ``stats``: optional int64[4] accumulated with (local rows, peer
    rows, slow-path rows, pushes issued).

    The AdaGrad form is the project's (as for KGE and BPR): ``-eta g / sqrt(acc + g^2)`` with the accumulator as read,
    which bounds every update by ``eta``. glove.c instead divides by the old accumulator and clips gradients at 100;
    with the accumulators initialised to 1 (as ``GloVe.init_model`` does, glove.c's initial ``gradsq``) early steps
    behave alike.

    ``deterministic=True`` (single-GPU servers only): start-of-step reads, fixed-point sums, bit-identical runs (three
    launches instead of one); the AdaGrad increment of one push is clamped to 2^24 there (see ops_glove.cu)."""
    _i64(words, "words"); _i64(ctxs, "ctxs"); _f32(x, "x"); _f32(loss, "loss")
    B = words.numel()
    if ctxs.numel() != B or x.numel() != B:
        raise ValueError("words, ctxs and x must have the same length")
    _check_glove_dim(embed_dim)
    _check_glove_rates(x_max, alpha)
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    det = _check_deterministic(server, deterministic)
    _C.glove_step(server._impl.backend_handle(), _stream(words), words.data_ptr(), ctxs.data_ptr(), x.data_ptr(), B,
                  int(embed_dim), float(eta), float(x_max), float(alpha), loss.data_ptr(),
                  stats.data_ptr() if stats is not None else 0, det)


def glove_reference_step(kv, words: torch.Tensor, ctxs: torch.Tensor, x: torch.Tensor, embed_dim: int, eta: float,
                         x_max: float, alpha: float):
    """The GloVe rule of :func:`glove_step` in float64 through Pull / Push (CPU servers, float64 rows, and the oracle of
    the tests). Every row is read at the start of the step. Returns ``(loss, pushes)``.

    Per non-zero with word row ``(w, b)`` and context row ``(c, b~)``: ``diff = <w, c> + b + b~ - ln X``, ``f =
    (X / x_max)^alpha`` if ``X < x_max`` else 1, loss ``f diff^2 / 2``; gradients ``g_w = f diff c``, ``g_c = f diff
    w``, ``g_b = g_b~ = f diff``; pushes ``[-eta g / sqrt(acc + g^2) | g^2]`` (0 where g == 0, so the padding stays 0)
    with the pulled accumulator, each row once per non-zero."""
    _check_glove_dim(embed_dim)
    _check_glove_rates(x_max, alpha)
    words, ctxs = words.reshape(-1).cpu(), ctxs.reshape(-1).cpu()
    x = x.reshape(-1).cpu().to(torch.float64)
    B, d = words.numel(), int(embed_dim)
    if ctxs.numel() != B or x.numel() != B:
        raise ValueError("words, ctxs and x must have the same length")
    D = d + 4
    f64 = torch.float64

    def pull(keys):
        v = torch.empty(keys.numel() * 2 * D, dtype=kv.server.dtype)
        if keys.numel():
            kv.wait(kv.pull(keys.contiguous(), v))
        v = v.view(-1, 2 * D).to(f64)
        return v[:, :D], v[:, D:]

    W, Aw = pull(words)
    C, Ac = pull(ctxs)
    diff = (W[:, :d] * C[:, :d]).sum(-1) + W[:, d] + C[:, d] - torch.log(x)
    f = torch.where(x < x_max, (x / x_max) ** alpha, torch.ones_like(x))
    loss = float((0.5 * f * diff * diff).sum())
    fd = (f * diff).unsqueeze(-1)
    gw, gc = torch.zeros(B, D, dtype=f64), torch.zeros(B, D, dtype=f64)
    gw[:, :d], gc[:, :d] = fd * C[:, :d], fd * W[:, :d]
    gw[:, d], gc[:, d] = fd[:, 0], fd[:, 0]

    def upd(g, a):
        ue = torch.where(g != 0, -eta * g / torch.sqrt(a + g * g), torch.zeros_like(g))
        return torch.cat([ue, g * g], -1).to(kv.server.dtype).contiguous().view(-1)

    if B:
        kv.wait(kv.push(words.contiguous(), upd(gw, Aw)))
        kv.wait(kv.push(ctxs.contiguous(), upd(gc, Ac)))
    return loss, 2 * B


ALS_MAX_RANK = 128


def _check_als_rank(rank: int) -> None:
    if isinstance(rank, bool) or int(rank) != rank or not (4 <= int(rank) <= ALS_MAX_RANK and int(rank) % 4 == 0):
        raise ValueError(f"rank must be a multiple of 4 in [4, {ALS_MAX_RANK}], got {rank}")


def _check_als_args(targets, offsets, others, a, b, rank, lam, gram) -> None:
    _check_als_rank(rank)
    if not lam > 0:
        raise ValueError(f"lam must be > 0, got {lam}")
    n, nnz = targets.numel(), others.numel()
    if offsets.numel() != n + 1 or a.numel() != nnz or b.numel() != nnz:
        raise ValueError(f"offsets must have len(targets) + 1 = {n + 1} entries and a, b len(others) = {nnz}, got "
                         f"{offsets.numel()}, {a.numel()}, {b.numel()}")
    if int(offsets[0]) != 0 or int(offsets[-1]) != nnz or bool((offsets[1:] < offsets[:-1]).any()):
        raise ValueError("offsets must be monotone from 0 to len(others)")
    if nnz and not bool((a >= 0).all()):
        raise ValueError("a must be >= 0")
    if torch.unique(targets).numel() != n:
        raise ValueError("targets must be distinct")
    if gram is not None and not (gram.dtype == torch.float32 and tuple(gram.shape) == (rank, rank)):
        raise ValueError(f"gram must be float32 [{rank}, {rank}] or None, got {gram.dtype} {tuple(gram.shape)}")


def als_solve(server, targets: torch.Tensor, offsets: torch.Tensor, others: torch.Tensor, a: torch.Tensor,
              b: torch.Tensor, rank: int, lam: float, gram: Optional[torch.Tensor] = None,
              stats: Optional[torch.Tensor] = None) -> None:
    """One alternating-least-squares solve per target row (csrc/cuda/ops_als.cu) on ``server``'s store: target
    ``targets[t]`` (distinct store keys) has the entries ``others[offsets[t] .. offsets[t + 1])`` (store keys of the other
    side, repeats count as often as they occur) with weights ``a`` (>= 0) and ``b`` (float32). Rows are ``[factors
    (rank) | AdaGrad (rank)]``, ``rank`` a multiple of 4 in [4, 128]. The rule is :func:`als_reference_solve`'s:
    ``A = gram + lam I + sum_e a_e h_e h_e^T``, ``r = sum_e b_e h_e``, ``w <- A^{-1} r`` pushed as ``[w_new - w_old | 0]``
    (the AdaGrad half is untouched); a target without entries becomes ``0``. One CTA per target in the given order (pass
    the longest first); the result does not depend on the order and is bit-identical from run to run. Factorised by
    Cholesky in fp32: a pivot <= 0 leaves the target unchanged and uncounted. ``gram``: float32 [rank, rank] or None;
    ``stats``: optional int64[4] accumulated with (other rows local, other rows from peers, slow-path rows, rows solved).
    Every half-step must only read rows it does not write: targets and others are keys of different sides."""
    _i64(targets, "targets"); _i64(offsets, "offsets"); _i64(others, "others"); _f32(a, "a"); _f32(b, "b")
    if gram is not None:
        _f32(gram, "gram")
    _check_als_args(targets, offsets, others, a, b, rank, lam, gram)
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 4):
        raise TypeError("stats must be a CUDA int64 tensor with 4 entries")
    _C.als_solve(server._impl.backend_handle(), _stream(targets), targets.data_ptr(), offsets.data_ptr(),
                 others.data_ptr(), a.data_ptr(), b.data_ptr(), targets.numel(), int(rank), float(lam),
                 gram.data_ptr() if gram is not None else 0, stats.data_ptr() if stats is not None else 0)


def als_gram(server, keys: torch.Tensor, rank: int) -> torch.Tensor:
    """``G = sum_k h_k h_k^T`` (float32 [rank, rank]) over the factor halves of the store rows ``keys`` (CUDA int64), read
    wherever they live. Each 1 024 keys form a partial in fp32 (fixed order) and the partials are added in index order,
    so G is bit-identical from call to call and on every rank of a multi-rank store."""
    _i64(keys, "keys")
    _check_als_rank(rank)
    G = torch.empty(int(rank), int(rank), dtype=torch.float32, device=keys.device)
    _C.als_gram(server._impl.backend_handle(), _stream(keys), keys.data_ptr(), keys.numel(), int(rank), G.data_ptr())
    return G


def als_gram_reference(kv, keys: torch.Tensor, rank: int, chunk: int = 1 << 16) -> torch.Tensor:
    """:func:`als_gram` in float64 through Pull (CPU servers and the tests)."""
    keys = keys.reshape(-1).cpu()
    r = int(rank)
    G = torch.zeros(r, r, dtype=torch.float64)
    for s in range(0, keys.numel(), chunk):
        k = keys[s:s + chunk].contiguous()
        v = torch.empty(k.numel() * 2 * r, dtype=kv.server.dtype)
        kv.wait(kv.pull(k, v))
        H = v.view(-1, 2 * r)[:, :r].to(torch.float64)
        G += H.t() @ H
    return G


def als_reference_solve(kv, targets: torch.Tensor, offsets: torch.Tensor, others: torch.Tensor, a: torch.Tensor,
                        b: torch.Tensor, rank: int, lam: float, gram: Optional[torch.Tensor] = None,
                        chunk: int = 8192) -> int:
    """The rule of :func:`als_solve` in float64 through Pull / Push (CPU servers, float64 rows, and the oracle of the
    tests): per target ``A = gram + lam I + sum_e a_e h_e h_e^T``, ``r = sum_e b_e h_e``, ``w <- A^{-1} r`` by Cholesky,
    pushed as ``[w_new - w_old | 0]``; a target whose A is not positive definite is left unchanged. Every row is read
    before any is written. Returns the number of targets solved."""
    targets, offsets, others = targets.reshape(-1).cpu(), offsets.reshape(-1).cpu(), others.reshape(-1).cpu()
    a, b = a.reshape(-1).cpu().to(torch.float64), b.reshape(-1).cpu().to(torch.float64)
    if gram is not None:
        gram = gram.cpu()
    _check_als_args(targets, offsets, others, a, b, rank, lam, gram if gram is None else gram.float())
    n, r, f64 = targets.numel(), int(rank), torch.float64
    if n == 0:
        return 0

    def pull(keys):
        v = torch.empty(keys.numel() * 2 * r, dtype=kv.server.dtype)
        if keys.numel():
            kv.wait(kv.pull(keys.contiguous(), v))
        return v.view(-1, 2 * r)[:, :r].to(f64)

    W, H = pull(targets), pull(others)
    A = torch.zeros(n, r, r, dtype=f64)
    if gram is not None:
        A += gram.to(f64)
    A += lam * torch.eye(r, dtype=f64)
    owner = torch.repeat_interleave(torch.arange(n), offsets[1:] - offsets[:-1])
    rhs = torch.zeros(n, r, dtype=f64)
    rhs.index_add_(0, owner, b.unsqueeze(1) * H)
    for s in range(0, H.shape[0], chunk):
        h = H[s:s + chunk]
        A.index_add_(0, owner[s:s + chunk], a[s:s + chunk, None, None] * h.unsqueeze(2) * h.unsqueeze(1))
    L, info = torch.linalg.cholesky_ex(A)
    ok = info == 0
    x = torch.cholesky_solve(rhs[ok].unsqueeze(2), L[ok]).squeeze(2)
    upd = torch.zeros(int(ok.sum()), 2 * r, dtype=f64)
    upd[:, :r] = x - W[ok]
    if upd.shape[0]:
        kv.wait(kv.push(targets[ok].contiguous(), upd.to(kv.server.dtype).contiguous().view(-1)))
    return int(ok.sum())


def _bf16_k8(t: torch.Tensor) -> torch.Tensor:
    """contiguous bf16 copy whose K (last dim) is padded to a multiple of 8 (16-byte TMA row pitch)."""
    t = t.to(torch.bfloat16)
    k = t.shape[1]
    if k % 8:
        t = torch.nn.functional.pad(t, (0, 8 - k % 8))
    return t.contiguous()


def gemm_nt_bf16(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """C[M,N] fp32 = a[M,K] x b[N,K]^T on the Hopper tensor cores (hand-written wgmma/TMA kernel,
    bf16 operands, fp32 accumulation)."""
    if not (a.is_cuda and b.is_cuda and a.dim() == 2 and b.dim() == 2 and a.shape[1] == b.shape[1]):
        raise ValueError("gemm_nt_bf16 expects CUDA matrices a[M,K], b[N,K]")
    a16, b16 = _bf16_k8(a), _bf16_k8(b)
    M, N, K = a16.shape[0], b16.shape[0], a16.shape[1]
    c = torch.empty(M, N, dtype=torch.float32, device=a.device)
    _C.gemm_nt_bf16(_stream(a16), a16.data_ptr(), b16.data_ptr(), M, N, K, c.data_ptr(), N)
    return c


def gemm_nt_fp8(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """C = a @ b^T with e4m3 operands on the fp8 tensor-core path (wgmma e4m3), per-tensor scales
    chosen from the absolute maxima, fp32 accumulation; the scale product is applied in the epilogue."""
    if not (a.is_cuda and b.is_cuda and a.shape[1] == b.shape[1]):
        raise ValueError("gemm_nt_fp8 expects CUDA matrices a[M,K], b[N,K]")
    k = a.shape[1]
    if k % 16:
        pad = 16 - k % 16
        a = torch.nn.functional.pad(a, (0, pad)); b = torch.nn.functional.pad(b, (0, pad))
    sa = a.detach().abs().amax().clamp(min=1e-12) / 448.0
    sb = b.detach().abs().amax().clamp(min=1e-12) / 448.0
    a8 = (a / sa).to(torch.float8_e4m3fn).contiguous()
    b8 = (b / sb).to(torch.float8_e4m3fn).contiguous()
    M, N, K = a8.shape[0], b8.shape[0], a8.shape[1]
    c = torch.empty(M, N, dtype=torch.float32, device=a.device)
    _C.gemm_nt_e4m3(_stream(a8), a8.data_ptr(), b8.data_ptr(), M, N, K, c.data_ptr(), N, float(sa * sb))
    return c


def gemm_nt_rank_count(q: torch.Tensor, e: torch.Tensor, true_score: torch.Tensor, true_col: torch.Tensor) -> torch.Tensor:
    """counts[i] = #{j != true_col[i] : <q[i], e[j]> > true_score[i]} without materialising the score matrix
    (rank-count epilogue of the wgmma GEMM)."""
    q16, e16 = _bf16_k8(q), _bf16_k8(e)
    M, N, K = q16.shape[0], e16.shape[0], q16.shape[1]
    ts = true_score.to(torch.float32).contiguous()
    tc = true_col.to(torch.int32).contiguous()
    out = torch.zeros(M, dtype=torch.int32, device=q.device)
    _C.gemm_nt_bf16_rank_count(_stream(q16), q16.data_ptr(), e16.data_ptr(), M, N, K, ts.data_ptr(), tc.data_ptr(),
                               out.data_ptr())
    return out


def _gather_stats(server, stats: Optional[torch.Tensor], dev):
    """The stats buffer of a gather launch. On several ranks a private int64[3] - (local rows, peer rows, rows that could
    not be resolved and were staged as zeros) - that :func:`_gathered` checks after the launch."""
    if server.num_servers() == 1:      # every row is a local owned row
        return stats
    return torch.zeros(3, dtype=torch.int64, device=dev)


def _gathered(op: str, own: Optional[torch.Tensor], stats: Optional[torch.Tensor]) -> None:
    if own is None or own is stats:
        return
    if stats is not None:
        n = min(stats.numel(), 3)
        stats[:n] += own[:n]
    bad = int(own[2])                  # (waits for the launch)
    if bad:
        raise RuntimeError(f"{op}: {bad} store rows could not be resolved and were read as zeros")


def gather_gemm(server, q: torch.Tensor, keys: torch.Tensor, k: int, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """scores[M, N] = q[M, k] @ E^T where row n of E is the first ``k`` values of store row ``keys[n]`` - the rows
    are gathered inside the GEMM kernel from the local slab, local replicas or peer GPUs over NVLink (fused
    gather + wgmma GEMM); the gathered matrix never exists in HBM. ``stats``: optional int64 tensor accumulated with
    (rows gathered locally, rows gathered from peers[, rows that could not be resolved]). On several ranks the call
    waits for the kernel and raises ``RuntimeError`` if a row could not be resolved."""
    _i64(keys, "keys")
    q16 = _bf16_k8(q)
    M, N = q16.shape[0], keys.numel()
    c = torch.empty(M, N, dtype=torch.float32, device=q.device)
    own = _gather_stats(server, stats, q.device)
    _C.gather_gemm(server._impl.backend_handle(), _stream(q16), q16.data_ptr(), keys.data_ptr(), M, N, int(k), q16.shape[1],
                   c.data_ptr(), N, own.data_ptr() if own is not None else 0)
    _gathered("gather_gemm", own, stats)
    return c


def gather_gemm_rank_count(server, q: torch.Tensor, keys: torch.Tensor, k: int, true_score: torch.Tensor,
                           true_col: torch.Tensor, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """counts[i] = #{n != true_col[i] : <q[i], row(keys[n])[:k]> > true_score[i]}: fused gather + GEMM + ranking
    epilogue - neither the gathered rows nor the [M, N] scores are materialised. ``stats``: as for
    :func:`gather_gemm`."""
    _i64(keys, "keys")
    q16 = _bf16_k8(q)
    M, N = q16.shape[0], keys.numel()
    out = torch.zeros(M, dtype=torch.int32, device=q.device)
    ts = true_score.to(torch.float32).contiguous()
    tc = true_col.to(torch.int32).contiguous()
    own = _gather_stats(server, stats, q.device)
    _C.gather_gemm_rank_count(server._impl.backend_handle(), _stream(q16), q16.data_ptr(), keys.data_ptr(), M, N, int(k),
                              q16.shape[1], ts.data_ptr(), tc.data_ptr(), out.data_ptr(),
                              own.data_ptr() if own is not None else 0)
    _gathered("gather_gemm_rank_count", own, stats)
    return out


TOPK_MAX_K = 64
# gather_gemm_topk on several GPUs: each CTA stays registered in the sync round's grace epoch for all its tiles, so the
# slice count is chosen to keep a CTA at no more than this many 128-column tiles
_TOPK_GRACE_TILES = 64


def _check_topk(M: int, N: int, k: int, exclude, col_scale):
    """Validates the top-k arguments (shapes, dtypes and the exclusion CSR) before anything touches the device."""
    if isinstance(k, bool) or int(k) != k or not 1 <= int(k) <= TOPK_MAX_K:
        raise ValueError(f"k must be an integer in [1, {TOPK_MAX_K}], got {k}")
    if col_scale is not None:
        if col_scale.dtype != torch.float32:
            raise TypeError("col_scale must be float32")
        if col_scale.dim() != 1 or col_scale.numel() != N:
            raise ValueError(f"col_scale must have one entry per column ({N}), got shape {tuple(col_scale.shape)}")
    if exclude is not None:
        if not (isinstance(exclude, (tuple, list)) and len(exclude) == 2):
            raise ValueError("exclude must be a CSR pair (offsets int64 [M + 1], cols int64 [nnz])")
        off, cols = exclude
        if off.dtype != torch.int64 or cols.dtype != torch.int64:
            raise TypeError("exclude offsets and cols must be int64")
        if off.dim() != 1 or off.numel() != M + 1 or cols.dim() != 1:
            raise ValueError(f"exclude offsets must have M + 1 = {M + 1} entries and cols must be 1-D")
        if int(off[0]) != 0 or int(off[-1]) != cols.numel() or bool((off[1:] < off[:-1]).any()):
            raise ValueError("exclude offsets must start at 0, be monotone and end at nnz")


def _topk_operands(dev, exclude, col_scale):
    for t, nm in ((col_scale, "col_scale"),) + (((exclude[0], "exclude offsets"), (exclude[1], "exclude cols"))
                                                 if exclude is not None else ()):
        if t is not None and not (t.is_cuda and t.device == dev and t.is_contiguous()):
            raise TypeError(f"{nm} must be a contiguous CUDA tensor on {dev}")
    return (col_scale.data_ptr() if col_scale is not None else 0,
            exclude[0].data_ptr() if exclude is not None else 0,
            exclude[1].data_ptr() if exclude is not None else 0)


def _topk_outputs(M: int, S: int, k: int, dev):
    part_v = torch.empty(M * S * k, dtype=torch.float32, device=dev)
    part_c = torch.empty(M * S * k, dtype=torch.int32, device=dev)
    vals = torch.empty(M, k, dtype=torch.float32, device=dev)
    idx = torch.empty(M, k, dtype=torch.int64, device=dev)
    return part_v, part_c, vals, idx


def _topk_empty(M: int, k: int, dev):
    return (torch.full((M, k), float("-inf"), dtype=torch.float32, device=dev),
            torch.full((M, k), -1, dtype=torch.int64, device=dev))


def gemm_nt_topk(q: torch.Tensor, e: torch.Tensor, k: int, exclude=None, col_scale: Optional[torch.Tensor] = None):
    """Per row i of ``q`` the ``k`` best columns j of ``score(i, j) = <q_i, e_j>``, without an [M, N] score matrix.

    Returns ``(values fp32 [M, k], indices int64 [M, k])``. Scores are the fp32 wgmma accumulation of the bf16-rounded
    operands (bit-identical to ``gemm_nt_bf16(q, e)`` wherever that GEMM does not split K), multiplied once by
    ``col_scale[j]`` when ``col_scale`` (float32 [N]) is given. Order: score descending, ties to the smaller column;
    the result does not depend on how the work is split, and repeated calls are bit-identical.
    ``exclude = (offsets int64 [M + 1], cols int64 [nnz])``: columns ``cols[offsets[i]:offsets[i + 1]]`` (sorted
    ascending within each row) never appear in row i. NaN scores are never selected; a row with fewer than ``k``
    eligible columns is padded with ``(-inf, -1)``. ``1 <= k <= 64``. Extra device memory is O(M * S * k) for S column
    slices (S is chosen from the SM count)."""
    if not (q.dim() == 2 and e.dim() == 2 and q.shape[1] == e.shape[1]):
        raise ValueError("gemm_nt_topk expects matrices q[M, K], e[N, K]")
    M, N = q.shape[0], e.shape[0]
    _check_topk(M, N, k, exclude, col_scale)
    if not (q.is_cuda and e.is_cuda and q.device == e.device):
        raise TypeError("gemm_nt_topk expects CUDA tensors on one device")
    k = int(k)
    if M == 0 or N == 0:
        return _topk_empty(M, k, q.device)
    cs, eo, ec = _topk_operands(q.device, exclude, col_scale)
    q16, e16 = _bf16_k8(q), _bf16_k8(e)
    S = _C.topk_num_slices(M, N, 0)
    part_v, part_c, vals, idx = _topk_outputs(M, S, k, q.device)
    _C.gemm_nt_topk(_stream(q16), q16.data_ptr(), e16.data_ptr(), M, N, q16.shape[1], k, S, cs, eo, ec, part_v.data_ptr(),
                    part_c.data_ptr(), vals.data_ptr(), idx.data_ptr())
    return vals, idx


def gather_gemm_topk(server, q: torch.Tensor, keys: torch.Tensor, dim: int, k: int, exclude=None,
                     col_scale: Optional[torch.Tensor] = None, stats: Optional[torch.Tensor] = None):
    """:func:`gemm_nt_topk` against parameter-store rows: column n is the first ``dim`` values of store row
    ``keys[n]``, gathered inside the kernel from local HBM, local replicas or peer GPUs over NVLink (as
    :func:`gather_gemm`, whose scores it reproduces bit for bit). ``indices`` are positions into ``keys``. ``stats``:
    optional int64[2] accumulated with (rows gathered locally, rows gathered from peers), and with the rows that could
    not be resolved in a third entry if it has one; on several ranks the call waits for the kernels and raises
    ``RuntimeError`` if a row could not be resolved.

    On several GPUs every CTA of the kernel counts in the grace period of the sync rounds for all of its column tiles
    (at most 64), so a long retrieval delays the relocations of a concurrent sync round."""
    _i64(keys, "keys")
    if q.dim() != 2 or q.shape[1] != int(dim):
        raise ValueError(f"q must be a matrix [M, dim = {dim}]")
    M, N = q.shape[0], keys.numel()
    _check_topk(M, N, k, exclude, col_scale)
    if not (q.is_cuda and q.device == keys.device):
        raise TypeError("q must be a CUDA tensor on the device of keys")
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.numel() >= 2):
        raise TypeError("stats must be a CUDA int64 tensor with 2 entries")
    k = int(k)
    if M == 0 or N == 0:
        return _topk_empty(M, k, q.device)
    cs, eo, ec = _topk_operands(q.device, exclude, col_scale)
    q16 = _bf16_k8(q)
    S = _C.topk_num_slices(M, N, _TOPK_GRACE_TILES if server.num_servers() > 1 else 0)
    part_v, part_c, vals, idx = _topk_outputs(M, S, k, q.device)
    own = _gather_stats(server, stats, q.device)
    _C.gather_gemm_topk(server._impl.backend_handle(), _stream(q16), q16.data_ptr(), keys.data_ptr(), M, N, int(dim),
                        q16.shape[1], k, S, cs, eo, ec, part_v.data_ptr(), part_c.data_ptr(), vals.data_ptr(),
                        idx.data_ptr(), own.data_ptr() if own is not None else 0)
    _gathered("gather_gemm_topk", own, stats)
    return vals, idx


def topk_reference(scores: torch.Tensor, k: int, excluded: Optional[torch.Tensor] = None):
    """Plain PyTorch top-k with the rule of the top-k kernels (tests, CPU backends): per row the ``k`` best columns of
    ``scores`` [M, N], score descending, ties to the smaller column, ``excluded`` (bool [M, N]) and NaN columns never
    selected, ``(-inf, -1)`` padding. Returns ``(values [M, k], indices int64 [M, k])`` in the dtype of ``scores``."""
    M, N = scores.shape
    ok = ~torch.isnan(scores)
    if excluded is not None:
        ok &= ~excluded
    s = torch.where(ok, scores, torch.full_like(scores, float("-inf")))
    order = torch.sort(s, dim=1, descending=True, stable=True).indices          # ties keep the column order
    order = order.gather(1, torch.sort(ok.gather(1, order).to(torch.int8), dim=1, descending=True, stable=True).indices)
    kk = min(int(k), N)
    idx = order[:, :kk]
    vals = scores.gather(1, idx)
    valid = ok.gather(1, idx)
    vals = torch.where(valid, vals, torch.full_like(vals, float("-inf")))
    idx = torch.where(valid, idx, torch.full_like(idx, -1))
    if kk < k:
        vals = torch.cat([vals, vals.new_full((M, k - kk), float("-inf"))], 1)
        idx = torch.cat([idx, idx.new_full((M, k - kk), -1)], 1)
    return vals, idx


def exclusion_mask(exclude, n_cols: int) -> torch.Tensor:
    """The dense form of an exclusion CSR ``exclude = (offsets int64 [M + 1], cols int64 [nnz])``, as the top-k and
    rank-count ops take it: bool [M, n_cols], True at ``[i, cols[offsets[i]:offsets[i + 1]]]``. For
    :func:`topk_reference` and :func:`dist_rank_reference`."""
    off, cols = exclude
    mask = torch.zeros(off.numel() - 1, n_cols, dtype=torch.bool, device=off.device)
    mask[torch.repeat_interleave(torch.arange(off.numel() - 1, device=off.device), off[1:] - off[:-1]), cols] = True
    return mask


EMBEDDING_BAG_MAX_DIM = 512
_NNZ_LIMIT = 1 << 31


class _EmbeddingBagFn(torch.autograd.Function):
    """Autograd node of :class:`StoreEmbeddingBag`: the forward pools rows of the store, the backward pushes the
    AdaGrad updates into the store (it returns no gradient: the rows are not tensors of the graph)."""

    @staticmethod
    def forward(ctx, anchor, bag, keys, offsets, weights):
        ctx.bag = bag
        out, ctx.state = bag._forward(keys, offsets, weights)
        return out

    @staticmethod
    def backward(ctx, grad):
        ctx.bag._backward(ctx.state, grad)
        ctx.state = None
        return None, None, None, None, None


class StoreEmbeddingBag:
    """Multi-hot embedding bags over the rows of a parameter store: ``torch.nn.functional.embedding_bag`` with
    ``include_last_offset=True`` whose table is the store, trained by worker-side AdaGrad.

    Rows are ``[embedding (dim) | AdaGrad accumulator (dim)]`` (the server's value length must be ``2 * dim``).
    ``bag(keys, offsets, per_sample_weights=None)`` returns ``out [nbags, dim]`` with
    ``out[b] = sum_{i in [offsets[b], offsets[b + 1])} w_i * row(keys[i])[:dim]`` (``w_i`` = 1 without weights), divided
    by the bag length for ``mode="mean"``; an empty bag gives zeros. ``keys`` int64 ``[nnz]``, ``offsets`` int64
    ``[nbags + 1]`` (starts at 0, ends at nnz), ``per_sample_weights`` float32 ``[nnz]`` (``sum`` only, as in torch).
    Weights are data: they get no gradient.

    The result takes part in autograd: ``loss.backward()`` updates the rows in the store. For every distinct key ``k``
    ``G = grad_scale * sum_{occurrences i of k} w_i (/ len of i's bag with mean) * grad_out[bag of i]`` and the row
    gets ``[-lr * G / sqrt(acc + G^2) | G^2]`` added (``acc`` read when the update runs; 0 where ``G == 0``). Autograd
    runs a backward only if some input requires grad: the op passes :attr:`anchor`, an empty tensor that requires grad,
    so that the backward runs even when nothing else before the bag does.

    ``impl``: ``fused`` (CUDA servers; csrc/cuda/ops_embbag.cu) - the forward is one kernel that reads the rows through
    the directory (local HBM, replicas, peers over NVLink), the backward four launches (key/position prep, radix sort,
    per-tile sums, finish) that push one update per distinct key. Each bag and each key's gradient is summed in fp32
    in a fixed order, so on one GPU the same inputs give bit-identical outputs and rows. ``torch``: distinct keys ->
    ``worker.pull`` -> ``F.embedding_bag`` over the pulled rows -> autograd -> AdaGrad -> ``worker.push``; the path of
    CPU servers (``auto`` picks ``fused`` on CUDA servers, ``torch`` on CPU servers).

    ``stats`` (fused): int64[4] accumulated with (rows read or updated locally, on peers, through the slow path of keys
    in a transitional state, rows updated). Calls on one object must not overlap (one CUDA stream): the backward's
    scratch is owned by the object and grows on demand."""

    def __init__(self, server, worker, dim: int, mode: str = "sum", lr: float = 0.05, grad_scale: float = 1.0,
                 impl: str = "auto"):
        if isinstance(dim, bool) or int(dim) != dim or not (4 <= int(dim) <= EMBEDDING_BAG_MAX_DIM and int(dim) % 4 == 0):
            raise ValueError(f"dim must be a multiple of 4 in [4, {EMBEDDING_BAG_MAX_DIM}], got {dim}")
        if mode not in ("sum", "mean"):
            raise ValueError(f"mode must be 'sum' or 'mean', got {mode!r}")
        if impl not in ("auto", "fused", "torch"):
            raise ValueError(f"impl must be 'auto', 'fused' or 'torch', got {impl!r}")
        self.dim = int(dim)
        row_len = getattr(server, "_uniform_len", None)
        if row_len != 2 * self.dim:
            raise ValueError(f"rows must be [embedding (dim) | AdaGrad (dim)]: the server's value length is {row_len}, "
                             f"expected 2 * dim = {2 * self.dim}")
        if impl == "auto":
            impl = "fused" if server.backend == "cuda" else "torch"
        if impl == "fused" and server.backend != "cuda":
            raise ValueError("impl='fused' needs a server with backend='cuda'")
        self.server, self.worker, self.mode, self.impl = server, worker, mode, impl
        self.lr, self.grad_scale = float(lr), float(grad_scale)
        self.device = server.device
        self.anchor = torch.zeros(0, device=self.device, requires_grad=True)
        self._stats = torch.zeros(5, dtype=torch.int64, device=self.device) if impl == "fused" else None
        self._ws = None
        self._rows_updated = 0          # torch route
        self._rows_taken = 0

    @property
    def stats(self) -> Optional[torch.Tensor]:
        return self._stats[:4] if self._stats is not None else None

    def take_rows_updated(self) -> int:
        """Rows updated since the previous call (one per distinct key and backward)."""
        total = int(self._stats[3]) if self._stats is not None else self._rows_updated
        n, self._rows_taken = total - self._rows_taken, total
        return n

    def __call__(self, keys: torch.Tensor, offsets: torch.Tensor,
                 per_sample_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        keys, offsets, per_sample_weights = self._check(keys, offsets, per_sample_weights)
        return _EmbeddingBagFn.apply(self.anchor, self, keys, offsets, per_sample_weights)

    def _check(self, keys, offsets, weights):
        dev = self.device
        for t, nm in ((keys, "keys"), (offsets, "offsets")):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.int64 or t.dim() != 1:
                raise TypeError(f"{nm} must be a 1-D int64 tensor")
            if t.device != dev:
                raise TypeError(f"{nm} must be on the store's device {dev}, got {t.device}")
        nnz = keys.numel()
        if nnz >= _NNZ_LIMIT:
            raise ValueError(f"at most 2^31 - 1 keys per call, got {nnz}")
        if offsets.numel() < 1:
            raise ValueError("offsets must have nbags + 1 entries (include_last_offset form)")
        if weights is not None:
            if self.mode != "sum":
                raise ValueError("per_sample_weights are only supported with mode='sum'")
            if not isinstance(weights, torch.Tensor) or weights.dtype != torch.float32:
                raise TypeError("per_sample_weights must be a float32 tensor")
            if weights.device != dev:
                raise TypeError(f"per_sample_weights must be on the store's device {dev}, got {weights.device}")
            if weights.shape != keys.shape:
                raise ValueError(f"per_sample_weights must have one entry per key ({nnz}), got {tuple(weights.shape)}")
            weights = weights.contiguous()
        bad = (offsets[0] != 0) | (offsets[-1] != nnz)
        if offsets.numel() > 1:
            bad = bad | (offsets[1:] < offsets[:-1]).any()
        if bool(bad):
            raise ValueError(f"offsets must start at 0, be non-decreasing and end at nnz = {nnz}")
        return keys.contiguous(), offsets.contiguous(), weights

    # ---- fused route (CUDA servers)
    def _check_resolved(self, op):
        if self.server.num_servers() > 1 and int(self._stats[4]):   # (waits for the kernel)
            raise RuntimeError(f"StoreEmbeddingBag {op}: {int(self._stats[4])} store rows could not be resolved")

    def _forward(self, keys, offsets, weights):
        if self.impl == "torch":
            return self._forward_torch(keys, offsets, weights)
        nbags = offsets.numel() - 1
        out = torch.empty(nbags, self.dim, dtype=torch.float32, device=self.device)
        _C.embedding_bag_forward(self.server._impl.backend_handle(), _stream(keys), keys.data_ptr(), offsets.data_ptr(),
                                 weights.data_ptr() if weights is not None else 0, keys.numel(), nbags, self.dim,
                                 self.mode == "mean", out.data_ptr(), self._stats.data_ptr())
        self._check_resolved("forward")
        return out, (keys, offsets, weights)

    def _backward(self, state, grad):
        if self.impl == "torch":
            return self._backward_torch(state, grad)
        keys, offsets, weights = state
        nnz, nbags = keys.numel(), offsets.numel() - 1
        g = grad.to(torch.float32).contiguous()
        need = _C.embedding_bag_workspace_bytes(nnz, self.dim)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        _C.embedding_bag_backward(self.server._impl.backend_handle(), _stream(g), keys.data_ptr(), offsets.data_ptr(),
                                  weights.data_ptr() if weights is not None else 0, nnz, nbags, self.dim,
                                  self.mode == "mean", g.data_ptr(), self.lr, self.grad_scale, self._ws.data_ptr(),
                                  self._ws.numel(), self._stats.data_ptr())
        self._check_resolved("backward")

    # ---- torch route (CPU servers; the comparison arm of benchmarks/embbag_bench.py on CUDA servers)
    def _forward_torch(self, keys, offsets, weights):
        kv, d = self.worker, self.dim
        uniq, inv = torch.unique(keys, return_inverse=True)
        rows = torch.empty(uniq.numel() * 2 * d, dtype=self.server.dtype, device=self.device)
        kv.wait(kv.pull(uniq, rows, True))
        rows = rows.view(-1, 2 * d)
        with torch.enable_grad():
            emb = rows[:, :d].detach().clone().requires_grad_(True)
            out = torch.nn.functional.embedding_bag(inv, emb, offsets, mode=self.mode, per_sample_weights=weights,
                                                    include_last_offset=True)
        return out.detach(), (uniq, emb, rows[:, d:], out)

    def _backward_torch(self, state, grad):
        uniq, emb, acc, out = state
        (g,) = torch.autograd.grad(out, emb, grad.to(out.dtype))
        g = g * self.grad_scale
        upd = torch.where(g != 0, -self.lr * g / torch.sqrt(acc + g * g), torch.zeros_like(g))
        self.worker.push(uniq, torch.cat([upd, g * g], 1).contiguous().view(-1), True)
        self._rows_updated += int(uniq.numel())


def embedding_bag_reference(table: torch.Tensor, keys: torch.Tensor, offsets: torch.Tensor,
                            per_sample_weights: Optional[torch.Tensor] = None, mode: str = "sum",
                            grad_out: Optional[torch.Tensor] = None, lr: float = 0.05, grad_scale: float = 1.0):
    """The rule of :class:`StoreEmbeddingBag` in float64 on a dense table ``[num_keys, 2 * dim]`` (tests). Returns
    ``(out [nbags, dim], new_table)``; ``new_table`` is the table after the update for ``grad_out`` ``[nbags, dim]``
    (None without ``grad_out``)."""
    t = table.detach().to(torch.float64).cpu()
    d = t.shape[1] // 2
    keys, offsets = keys.cpu(), offsets.cpu()
    nb = offsets.numel() - 1
    lens = offsets[1:] - offsets[:-1]
    bag = torch.repeat_interleave(torch.arange(nb), lens)
    c = per_sample_weights.detach().cpu().double() if per_sample_weights is not None else torch.ones(keys.numel(),
                                                                                                    dtype=torch.float64)
    if mode == "mean":
        c = c / lens[bag].double()
    out = torch.zeros(nb, d, dtype=torch.float64).index_add_(0, bag, c[:, None] * t[keys, :d])
    if grad_out is None:
        return out, None
    uniq, inv = torch.unique(keys, return_inverse=True)
    G = torch.zeros(uniq.numel(), d, dtype=torch.float64).index_add_(
        0, inv, c[:, None] * grad_out.detach().cpu().double()[bag]) * grad_scale
    acc = t[uniq, d:]
    upd = torch.where(G != 0, -lr * G / torch.sqrt(acc + G * G), torch.zeros_like(G))
    new = t.clone()
    new[uniq, :d] += upd
    new[uniq, d:] += G * G
    return out, new


DLRM_MAX_ROWS = 64          # F + 1 (the bottom-MLP output and the F fields)


def dlrm_interaction_width(F: int, E: int) -> int:
    """W, the width of :func:`dlrm_interaction`'s output: E + F (F + 1) / 2 rounded up to a multiple of 8."""
    return (E + F * (F + 1) // 2 + 7) // 8 * 8


def _check_dlrm_args(z, e):
    for t, nm in ((z, "z"), (e, "e")):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
            raise TypeError(f"{nm} must be a float32 tensor")
    if z.dim() != 2 or e.dim() != 3:
        raise ValueError(f"z must be [B, E] and e [B, F, E], got {tuple(z.shape)} and {tuple(e.shape)}")
    if e.device != z.device:
        raise TypeError(f"z and e must be on one device, got {z.device} and {e.device}")
    B, E = z.shape
    F = e.shape[1]
    if e.shape[0] != B or e.shape[2] != E:
        raise ValueError(f"e must be [B, F, E] = [{B}, F, {E}], got {tuple(e.shape)}")
    if not 1 <= F <= DLRM_MAX_ROWS - 1:
        raise ValueError(f"dlrm_interaction needs 1 <= F and F + 1 <= {DLRM_MAX_ROWS}, got F = {F}")
    if E % 4 or not 4 <= E <= EMBEDDING_BAG_MAX_DIM:
        raise ValueError(f"dlrm_interaction needs E a multiple of 4 in [4, {EMBEDDING_BAG_MAX_DIM}], got E = {E}")
    W = dlrm_interaction_width(F, E)
    if B * W >= 1 << 31:
        raise ValueError(f"dlrm_interaction needs B * W < 2^31, got B = {B}, W = {W}")
    return B, F, E, W


def _dlrm_pairs(F: int, device):
    return torch.tril_indices(F + 1, F + 1, offset=-1, device=device)


def _dlrm_interaction_torch(z, e):
    B, F, E, W = z.shape[0], e.shape[1], z.shape[1], dlrm_interaction_width(e.shape[1], z.shape[1])
    T = torch.cat([z[:, None], e], 1)
    Z = torch.bmm(T, T.transpose(1, 2))
    i, j = _dlrm_pairs(F, z.device)
    pad = z.new_zeros(B, W - E - i.numel())
    return torch.cat([z, Z[:, i, j], pad], 1)


class _DlrmInteractionFn(torch.autograd.Function):
    """The fused route of :func:`dlrm_interaction`: one kernel each way (csrc/cuda/ops_dlrm.cu)."""

    @staticmethod
    def forward(ctx, z, e):
        B, F, E, W = _check_dlrm_args(z, e)
        z, e = _dlrm_aligned(z), _dlrm_aligned(e)
        R = torch.empty(B, W, dtype=torch.float32, device=z.device)
        _C.dlrm_interaction_forward(_stream(z), z.data_ptr(), e.data_ptr(), B, F, E, W, R.data_ptr())
        ctx.save_for_backward(z, e)
        return R

    @staticmethod
    def backward(ctx, dR):
        z, e = ctx.saved_tensors
        B, F, E = e.shape
        dR = _dlrm_aligned(dR.to(torch.float32))
        dz, de = torch.empty_like(z), torch.empty_like(e)
        _C.dlrm_interaction_backward(_stream(dR), dR.data_ptr(), z.data_ptr(), e.data_ptr(), B, F, E,
                                     dR.shape[1], dz.data_ptr(), de.data_ptr())
        return dz, de


def _dlrm_aligned(t: torch.Tensor) -> torch.Tensor:
    """contiguous, with a 16-byte aligned start (the kernels read and write float4)"""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def dlrm_interaction(z: torch.Tensor, e: torch.Tensor, impl: str = "auto") -> torch.Tensor:
    """DLRM's dot interaction (Naumov et al., 2019): ``R [B, W]`` from the bottom-MLP output ``z`` float32 ``[B, E]``
    and the pooled field embeddings ``e`` float32 ``[B, F, E]`` (as :class:`StoreEmbeddingBag` returns them, viewed
    ``[B, F, E]``). With ``T = [z; e_0; ..; e_{F-1}]`` (``F + 1`` rows), ``R[:, :E] = z``, ``R[:, E + p]`` is the dot
    product ``<T_i, T_j>`` of the p-th pair ``j < i`` in the order of ``torch.tril_indices(F + 1, F + 1, -1)``, and the
    ``W - E - F (F + 1) / 2`` pad columns (:func:`dlrm_interaction_width`) are 0; their gradients are ignored.

    Autograd reaches both ``z`` and ``e``. ``impl``: ``fused`` (CUDA tensors) - one kernel forward and one backward,
    fp32 sums in a fixed order, bit-identical reruns; ``torch`` - ``cat``, ``bmm``, the ``tril`` gather and ``cat``
    (CPU tensors, and the comparison arm of benchmarks/dlrm_bench.py); ``auto`` picks ``fused`` for CUDA tensors.
    Limits: ``1 <= F``, ``F + 1 <= 64``, ``E`` a multiple of 4 in [4, 512], ``B * W < 2^31``."""
    if impl not in ("auto", "fused", "torch"):
        raise ValueError(f"impl must be 'auto', 'fused' or 'torch', got {impl!r}")
    _check_dlrm_args(z, e)
    if impl == "auto":
        impl = "fused" if z.is_cuda else "torch"
    if impl == "torch":
        return _dlrm_interaction_torch(z, e)
    if not z.is_cuda:
        raise ValueError("impl='fused' needs CUDA tensors")
    return _DlrmInteractionFn.apply(z, e)


def dlrm_interaction_reference(z: torch.Tensor, e: torch.Tensor, grad_out: Optional[torch.Tensor] = None):
    """The rule of :func:`dlrm_interaction` in float64 on the CPU (tests): ``(R, dz, de)``; ``dz`` and ``de`` are the
    gradients for ``grad_out`` ``[B, W]`` (None without it)."""
    z64, e64 = z.detach().cpu().double(), e.detach().cpu().double()
    B, E = z64.shape
    F = e64.shape[1]
    W = dlrm_interaction_width(F, E)
    T = torch.cat([z64[:, None], e64], 1)                        # [B, N, E]
    i, j = _dlrm_pairs(F, "cpu")
    R = torch.zeros(B, W, dtype=torch.float64)
    R[:, :E] = z64
    R[:, E:E + i.numel()] = (T[:, i] * T[:, j]).sum(-1)
    if grad_out is None:
        return R, None, None
    g = grad_out.detach().cpu().double()
    dZ = torch.zeros(B, F + 1, F + 1, dtype=torch.float64)
    dZ[:, i, j] = g[:, E:E + i.numel()]
    dZ = dZ + dZ.transpose(1, 2)
    dT = torch.bmm(dZ, T)
    return R, g[:, :E] + dT[:, 0], dT[:, 1:]


DCN_MAX_LAYERS = 8
DCN_MIN_RANK = 8
DCN_MAX_RANK = 1024


def _check_dcn_args(z, e, V, W, b, fused: bool):
    """(B, E, N, r, L) of dcn_cross's arguments; ValueError / TypeError before anything is launched"""
    for t, nm in ((z, "z"), (e, "e"), (V, "V"), (W, "W"), (b, "b")):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
            raise TypeError(f"{nm} must be a float32 tensor")
        if t.device != z.device:
            raise TypeError(f"dcn_cross needs all tensors on one device, got {nm} on {t.device} and z on {z.device}")
    if z.dim() != 2 or e.dim() != 3:
        raise ValueError(f"z must be [B, E] and e [B, F, E], got {tuple(z.shape)} and {tuple(e.shape)}")
    B, E = z.shape
    F = e.shape[1]
    if e.shape[0] != B or e.shape[2] != E or F < 1 or E < 1:
        raise ValueError(f"e must be [B, F, E] = [{B}, F >= 1, {E}], got {tuple(e.shape)}")
    N = (F + 1) * E
    if V.dim() != 3 or V.shape[2] != N:
        raise ValueError(f"V must be [L, r, N] with N = (F + 1) E = {N}, got {tuple(V.shape)}")
    L, r = V.shape[0], V.shape[1]
    if tuple(W.shape) != (L, N, r):
        raise ValueError(f"W must be [L, N, r] = [{L}, {N}, {r}], got {tuple(W.shape)}")
    if tuple(b.shape) != (L, N):
        raise ValueError(f"b must be [L, N] = [{L}, {N}], got {tuple(b.shape)}")
    if not 1 <= L <= DCN_MAX_LAYERS:
        raise ValueError(f"dcn_cross needs 1 <= L <= {DCN_MAX_LAYERS}, got L = {L}")
    if B * N >= 1 << 31:
        raise ValueError(f"dcn_cross needs B * N < 2^31, got B = {B}, N = {N}")
    if fused:
        if B < 1:
            raise ValueError("impl='fused' needs B >= 1")
        if N % 8 or r % 8:
            raise ValueError(f"impl='fused' needs N and r multiples of 8 (16-byte TMA rows), got N = {N}, r = {r}")
        if not DCN_MIN_RANK <= r <= DCN_MAX_RANK:
            raise ValueError(f"impl='fused' needs {DCN_MIN_RANK} <= r <= {DCN_MAX_RANK}, got r = {r}")
        if not z.is_cuda:
            raise ValueError("impl='fused' needs CUDA tensors")
    return B, E, N, r, L


def _dcn_cross_torch(z, e, V, W, b):
    x0 = torch.cat([z, e.reshape(z.shape[0], -1)], 1)
    x = x0
    for l in range(V.shape[0]):
        x = x0 * (torch.matmul(torch.matmul(x, V[l].t()), W[l].t()) + b[l]) + x
    return x


def _dcn_fused_forward(z, e, V16, W16, b, train: bool):
    """x_L, and with ``train`` the bf16 tensors the backward reads: (x_l^T, h_l^T, u_l)"""
    B, E = z.shape
    L, r, N = V16.shape
    P = (B + 7) // 8 * 8
    dev = z.device
    bf = dict(dtype=torch.bfloat16, device=dev)
    x = torch.empty(B, N, dtype=torch.float32, device=dev)
    xb, hb = torch.empty(B, N, **bf), torch.empty(B, r, **bf)
    saved = (torch.empty(L, N, P, **bf), torch.empty(L, r, P, **bf), torch.empty(L, B, N, **bf)) if train else None
    xt, ht, ub = (t.data_ptr() for t in saved) if train else (0, 0, 0)
    _C.dcn_forward(_stream(z), z.data_ptr(), e.data_ptr(), B, E, N, r, L, V16.data_ptr(), W16.data_ptr(), b.data_ptr(),
                   xb.data_ptr(), hb.data_ptr(), x.data_ptr(), xt, ht, ub)
    return x, saved


class _DcnCrossFn(torch.autograd.Function):
    """The fused route of :func:`dcn_cross` (csrc/cuda/ops_dcn.cu): 1 + 2 L launches forward, and per layer an
    elementwise pass, the db sum and four GEMMs backward."""

    @staticmethod
    def forward(ctx, z, e, V, W, b):
        z, e, b = z.contiguous(), e.contiguous(), b.contiguous()
        x, saved = _dcn_fused_forward(z, e, V.to(torch.bfloat16).contiguous(), W.to(torch.bfloat16).contiguous(), b,
                                      train=True)
        ctx.save_for_backward(z, e, V, W, *saved)
        return x

    @staticmethod
    def backward(ctx, gx):
        z, e, V, W, xt, ht, ub = ctx.saved_tensors
        B, E = z.shape
        L, r, N = V.shape
        P = (B + 7) // 8 * 8
        dev = z.device
        Vt = V.transpose(1, 2).to(torch.bfloat16).contiguous()
        Wt = W.transpose(1, 2).to(torch.bfloat16).contiguous()
        gx = gx.to(torch.float32).contiguous()
        bf = dict(dtype=torch.bfloat16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        G, dx0 = torch.empty(B, N, **f32), torch.empty(B, N, **f32)
        Pb, Pt, dh, dht = torch.empty(B, N, **bf), torch.empty(N, P, **bf), torch.empty(B, r, **bf), torch.empty(r, P, **bf)
        ws = torch.empty(_C.dcn_workspace_floats(B, N, r), **f32)
        dz, de = torch.empty_like(z), torch.empty_like(e)
        dV, dW, db = torch.empty(L, r, N, **f32), torch.empty(L, N, r, **f32), torch.empty(L, N, **f32)
        _C.dcn_backward(_stream(gx), z.data_ptr(), e.data_ptr(), B, E, N, r, L, Vt.data_ptr(), Wt.data_ptr(),
                        xt.data_ptr(), ht.data_ptr(), ub.data_ptr(), gx.data_ptr(), G.data_ptr(), dx0.data_ptr(),
                        Pb.data_ptr(), Pt.data_ptr(), dh.data_ptr(), dht.data_ptr(), ws.data_ptr(), dz.data_ptr(),
                        de.data_ptr(), dV.data_ptr(), dW.data_ptr(), db.data_ptr())
        return dz, de, dV, dW, db


def dcn_cross(z: torch.Tensor, e: torch.Tensor, V: torch.Tensor, W: torch.Tensor, b: torch.Tensor,
              impl: str = "auto") -> torch.Tensor:
    """DCN-v2's low-rank cross network (Wang et al., 2021; torchrec's ``LowRankCrossNet``) on DLRM's features:
    ``x_L float32 [B, N]`` from ``x_0 = [z | e_0 | .. | e_{F-1}]`` (``N = (F + 1) E``) by the L layers
    ``x_{l+1} = x_0 * (W_l (V_l x_l) + b_l) + x_l``.

    ``z`` float32 ``[B, E]`` (the bottom-MLP output), ``e`` float32 ``[B, F, E]`` (the pooled fields, as for
    :func:`dlrm_interaction`), ``V [L, r, N]``, ``W [L, N, r]``, ``b [L, N]`` float32. Autograd reaches all five.
    ``impl``: ``fused`` (CUDA tensors) - the kernels of csrc/cuda/ops_dcn.cu, GEMMs on the tensor cores with bf16
    operands and fp32 accumulation, the residual stream in fp32, bit-identical reruns; ``torch`` - the fp32 rule with
    ``matmul`` (CPU tensors, and the comparison arm of benchmarks/dcn_bench.py); ``auto`` picks ``fused`` for CUDA
    tensors. Limits: ``1 <= L <= 8``, ``B * N < 2^31``; on ``fused`` also ``B >= 1``, ``N`` and ``r`` multiples of 8,
    ``8 <= r <= 1024``."""
    if impl not in ("auto", "fused", "torch"):
        raise ValueError(f"impl must be 'auto', 'fused' or 'torch', got {impl!r}")
    if impl == "auto":
        impl = "fused" if isinstance(z, torch.Tensor) and z.is_cuda else "torch"
    _check_dcn_args(z, e, V, W, b, fused=impl == "fused")
    if impl == "torch":
        return _dcn_cross_torch(z, e, V, W, b)
    if torch.is_grad_enabled() and any(t.requires_grad for t in (z, e, V, W, b)):
        return _DcnCrossFn.apply(z, e, V, W, b)
    return _dcn_fused_forward(z.contiguous(), e.contiguous(), V.to(torch.bfloat16).contiguous(),
                              W.to(torch.bfloat16).contiguous(), b.contiguous(), train=False)[0]


def dcn_cross_reference(z: torch.Tensor, e: torch.Tensor, V: torch.Tensor, W: torch.Tensor, b: torch.Tensor,
                        grad_out: Optional[torch.Tensor] = None, bf16_operands: bool = False):
    """The rule of :func:`dcn_cross` in float64 on the CPU (tests): ``(x_L, dz, de, dV, dW, db)``, the gradients for
    ``grad_out [B, N]`` (None without it). With ``bf16_operands`` the values are rounded to bf16 where the fused route
    rounds them: the GEMM operands x_l, h_l, V, W (forward) and P = G * x_0, dh, V, W (backward), and the saved u_l that
    the backward multiplies G by; sums stay float64."""
    def rb(t):
        return t.to(torch.bfloat16).double() if bf16_operands else t

    z64, e64 = z.detach().cpu().double(), e.detach().cpu().double()
    V64, W64, b64 = V.detach().cpu().double(), W.detach().cpu().double(), b.detach().cpu().double()
    B, E = z64.shape
    x0 = torch.cat([z64, e64.reshape(B, -1)], 1)
    x, xs, hs, us = x0, [], [], []
    for l in range(V64.shape[0]):
        xs.append(rb(x))
        hs.append(rb(xs[-1] @ rb(V64[l]).t()))
        u = hs[-1] @ rb(W64[l]).t() + b64[l]
        us.append(rb(u))
        x = x0 * u + x
    if grad_out is None:
        return x, None, None, None, None, None
    G = grad_out.detach().cpu().double()
    dx0 = torch.zeros_like(x0)
    dV, dW, db = torch.zeros_like(V64), torch.zeros_like(W64), torch.zeros_like(b64)
    for l in reversed(range(V64.shape[0])):
        P = G * x0
        dx0 += G * us[l]
        db[l] = P.sum(0)
        Pb = rb(P)
        dh = rb(Pb @ rb(W64[l]))
        dW[l] = Pb.t() @ hs[l]
        dV[l] = dh.t() @ xs[l]
        G = G + dh @ rb(V64[l])
    dx0 += G
    return x, dx0[:, :E], dx0[:, E:].reshape(e64.shape), dV, dW, db


FFM_MAX_FIELDS = 64
FFM_MAX_K = 32
FFM_MAX_FK = 512


def ffm_row_values(num_fields: int, k: int) -> int:
    """E, the values of an FFM row before its AdaGrad half: ``[w, 0, 0, 0 | V_0 | ... | V_{F-1}]``."""
    return 4 + int(num_fields) * int(k)


def _check_ffm_shape(num_fields, k, row_len) -> None:
    for v, nm in ((num_fields, "num_fields"), (k, "k")):
        if isinstance(v, bool) or int(v) != v:
            raise ValueError(f"{nm} must be an integer, got {v!r}")
    F, k = int(num_fields), int(k)
    if not 2 <= F <= FFM_MAX_FIELDS:
        raise ValueError(f"num_fields must be in [2, {FFM_MAX_FIELDS}], got {F}")
    if not (4 <= k <= FFM_MAX_K and k % 4 == 0):
        raise ValueError(f"k must be a multiple of 4 in [4, {FFM_MAX_K}], got {k}")
    if F * k > FFM_MAX_FK:
        raise ValueError(f"num_fields * k must be <= {FFM_MAX_FK}, got {F * k}")
    E = ffm_row_values(F, k)
    if row_len != 2 * E:
        raise ValueError(f"rows must be [w, 0, 0, 0 | V (num_fields * k) | AdaGrad]: the server's value length is "
                         f"{row_len}, expected 2 * (4 + num_fields * k) = {2 * E}")


def _check_ffm_rates(eta, lam) -> None:
    for v, nm in ((eta, "eta"), (lam, "lam")):
        if not float(v) >= 0.0:
            raise ValueError(f"{nm} must be >= 0, got {v}")


def _check_ffm_ids(ids, num_fields, device) -> int:
    if not isinstance(ids, torch.Tensor) or ids.dtype != torch.int64 or ids.dim() != 2:
        raise TypeError("ids must be a 2-D int64 tensor [B, num_fields]")
    if device is not None and ids.device != device:
        raise TypeError(f"ids must be on the store's device {device}, got {ids.device}")
    if ids.shape[1] != num_fields:
        raise ValueError(f"ids must have one column per field ({num_fields}), got {ids.shape[1]}")
    if ids.numel() >= _NNZ_LIMIT:
        raise ValueError(f"batch * num_fields must be < 2^31, got {ids.numel()}")
    return ids.shape[0]


def _check_ffm_labels(labels, B, device) -> None:
    if not isinstance(labels, torch.Tensor) or labels.dtype != torch.float32:
        raise TypeError("labels must be a float32 tensor")
    if device is not None and labels.device != device:
        raise TypeError(f"labels must be on the store's device {device}, got {labels.device}")
    if labels.dim() != 1 or labels.numel() != B:
        raise ValueError(f"labels must be [B = {B}], got {tuple(labels.shape)}")


class StoreFFM:
    """Field-aware factorisation machine (FFM, as in libffm) over the rows of a parameter store, trained by fused
    sm_90a kernels (csrc/cuda/ops_ffm.cu) on a CUDA server.

    A key's row is ``[w, 0, 0, 0 | V_0 | ... | V_{F-1} | AdaGrad of all E values]``, ``V_f`` its k-vector for field f
    and ``E = 4 + F k`` (the server's value length must be ``2 E``). ``ids`` int64 ``[B, F]``: the field of
    ``ids[b, f]`` is f. With ``r = pair_scale`` (``1 / F`` is libffm's instance normalisation of one-hot data)

    * ``phi_b = sum_f w[x_bf] + r sum_{f1<f2} <V[x_bf1][f2], V[x_bf2][f1]>``, ``kappa_b = sigmoid(phi_b) - y_b``, loss
      ``softplus(phi_b) - y_b phi_b``, all from the rows at the start of the step;
    * per distinct key, summed over its occurrences ``(b, f)`` in position order ``b F + f``: ``G_w = sum kappa_b +
      lam w`` and, for every field ``f2 != f``, ``G_(V, f2) = sum kappa_b r V[x_b,f2][f] + lam V_f2``;
    * one push per distinct key ``[-eta G / sqrt(acc + G^2) | G^2]`` (0 where ``G == 0``, so the own-field block and the
      padding never change), ``acc`` from the start of the step.

    ``step(ids, labels)`` returns the summed loss as a device tensor; ``forward(ids)`` the logits ``phi`` [B]. Both
    are sums in fp32 in a fixed order: on one GPU two runs from the same rows give bit-identical rows and loss.
    :func:`ffm_reference_step` is the same rule in float64 through Pull / Push.

    ``stats``: int64[4] accumulated with (rows read or updated locally, on peers, through the slow path of keys in a
    transitional state, rows updated: one per distinct key and step). On several ranks a step or forward that could
    not resolve a row raises ``RuntimeError``. Calls on one object must not overlap (one CUDA stream): the step's
    scratch is owned by the object and grows on demand."""

    def __init__(self, server, num_fields: int, k: int, eta: float = 0.2, lam: float = 2e-5, pair_scale: float = 1.0):
        if server.backend != "cuda":
            raise ValueError("StoreFFM needs a server with backend='cuda' (ffm_reference_step is the CPU route)")
        if getattr(server, "dtype", torch.float32) != torch.float32:
            raise ValueError("StoreFFM needs float32 rows")
        _check_ffm_shape(num_fields, k, getattr(server, "_uniform_len", None))
        _check_ffm_rates(eta, lam)
        self.server, self.num_fields, self.k = server, int(num_fields), int(k)
        self.eta, self.lam, self.pair_scale = float(eta), float(lam), float(pair_scale)
        self.device = server.device
        self._stats = torch.zeros(5, dtype=torch.int64, device=self.device)
        self._ws = None

    @property
    def stats(self) -> torch.Tensor:
        return self._stats[:4]

    def _check_resolved(self, op):
        if self.server.num_servers() > 1 and int(self._stats[4]):   # (waits for the kernel)
            raise RuntimeError(f"StoreFFM {op}: {int(self._stats[4])} store rows could not be resolved")

    def step(self, ids: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """One training step on ``ids`` [B, F] and ``labels`` float32 [B] in [0, 1]; returns the summed loss (float32
        [1] on the device)."""
        B = _check_ffm_ids(ids, self.num_fields, self.device)
        _check_ffm_labels(labels, B, self.device)
        _check_ffm_rates(self.eta, self.lam)
        ids, labels = ids.contiguous(), labels.contiguous()
        need = _C.ffm_workspace_bytes(B, self.num_fields, self.k)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        loss = torch.empty(1, dtype=torch.float32, device=self.device)
        _C.ffm_step(self.server._impl.backend_handle(), _stream(ids), ids.data_ptr(), labels.data_ptr(), B,
                    self.num_fields, self.k, self.pair_scale, self.eta, self.lam, self._ws.data_ptr(), self._ws.numel(),
                    loss.data_ptr(), self._stats.data_ptr())
        self._check_resolved("step")
        return loss

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        """The logits ``phi`` (float32 [B]) of ``ids`` [B, F]; the rows are not changed."""
        B = _check_ffm_ids(ids, self.num_fields, self.device)
        ids = ids.contiguous()
        out = torch.empty(B, dtype=torch.float32, device=self.device)
        _C.ffm_forward(self.server._impl.backend_handle(), _stream(ids), ids.data_ptr(), B, self.num_fields, self.k,
                       self.pair_scale, out.data_ptr(), self._stats.data_ptr())
        self._check_resolved("forward")
        return out


def _ffm_pull(kv, ids: torch.Tensor, k: int, pair_scale: float):
    """(distinct keys, their rows in float64 [U, 2E], position -> distinct key, phi [B], V [B, F, F, k])"""
    B, F = ids.shape
    E = ffm_row_values(F, k)
    uniq, inv = torch.unique(ids.reshape(-1), return_inverse=True)
    v = torch.empty(uniq.numel() * 2 * E, dtype=kv.server.dtype)
    if uniq.numel():
        kv.wait(kv.pull(uniq.contiguous(), v))
    rows = v.view(-1, 2 * E).to(torch.float64)
    x = rows[inv].view(B, F, 2 * E)
    V = x[:, :, 4:E].reshape(B, F, F, k)                  # V[b, f1, f2] = V[x_bf1][f2]
    P = torch.einsum("bijd,bjid->bij", V, V)              # <V[x_bi][j], V[x_bj][i]>
    phi = x[:, :, 0].sum(1) + pair_scale * torch.triu(P, diagonal=1).sum((1, 2))
    return uniq, rows, inv, phi, V


def _ffm_ids_cpu(ids):
    if not isinstance(ids, torch.Tensor) or ids.dim() != 2:
        raise TypeError("ids must be a 2-D int64 tensor [B, num_fields]")
    ids = ids.cpu()
    _check_ffm_ids(ids, ids.shape[1], None)
    return ids


def ffm_reference_forward(kv, ids: torch.Tensor, k: int, pair_scale: float = 1.0) -> torch.Tensor:
    """The logits of :class:`StoreFFM` in float64 (CPU tensor [B]) from rows read through Pull."""
    ids = _ffm_ids_cpu(ids)
    _check_ffm_shape(ids.shape[1], k, getattr(kv.server, "_uniform_len", None))
    return _ffm_pull(kv, ids, int(k), float(pair_scale))[3]


def ffm_reference_step(kv, ids: torch.Tensor, labels: torch.Tensor, k: int, eta: float, lam: float,
                       pair_scale: float = 1.0) -> float:
    """The rule of :class:`StoreFFM` in float64 through Pull / Push (CPU servers, and the oracle of the tests): every
    row is read at the start of the step, each distinct key gets one push. Returns the summed loss."""
    ids = _ffm_ids_cpu(ids)
    B, F = ids.shape
    _check_ffm_labels(labels.cpu(), B, None)
    _check_ffm_shape(F, k, getattr(kv.server, "_uniform_len", None))
    _check_ffm_rates(eta, lam)
    k, r = int(k), float(pair_scale)
    E = ffm_row_values(F, k)
    y = labels.cpu().to(torch.float64)
    uniq, rows, inv, phi, V = _ffm_pull(kv, ids, k, r)
    loss = float((torch.nn.functional.softplus(phi) - y * phi).sum())
    if B == 0:
        return loss
    kappa = (torch.sigmoid(phi) - y).view(B, 1, 1, 1)
    w = rows[inv, 0].view(B, F)
    c = torch.zeros(B, F, E, dtype=torch.float64)
    c[:, :, 0] = kappa.view(B, 1) + lam * w
    cv = kappa * r * V.transpose(1, 2) + lam * V          # [b, f, f2]: kappa r V[x_b,f2][f] + lam V[x_bf][f2]
    cv[:, torch.arange(F), torch.arange(F)] = 0.0          # no term for f2 == f
    c[:, :, 4:] = cv.reshape(B, F, F * k)
    G = torch.zeros(uniq.numel(), E, dtype=torch.float64).index_add_(0, inv, c.view(B * F, E))
    acc = rows[:, E:]
    upd = torch.where(G != 0, -eta * G / torch.sqrt(acc + G * G), torch.zeros_like(G))
    kv.wait(kv.push(uniq.contiguous(), torch.cat([upd, G * G], 1).to(kv.server.dtype).contiguous().view(-1)))
    return loss


class IntentPrepass:
    """Device-side pre-pass for ``Worker.intent`` (experimental; ``csrc/cuda/ops_intent.cu``).

    ``submit(keys, start, end)`` extends the intent end clock of every key that already has a usable local slot with an
    ``atomicMax`` on the device and collects the remaining keys; ``harvest()`` hands the collected keys of finished
    submissions to ``worker.intent`` (the host path: placeholder allocation + request to the owner). In steady state a
    few per cent of the keys take the host path, which takes the per-key work off the sync thread.
    """

    def __init__(self, server, worker, max_keys: int, depth: int = 4):
        self.server, self.worker = server, worker
        dev = server.device
        self.max_keys = int(max_keys)
        self._slots = []
        for _ in range(depth):
            self._slots.append({
                "keys": torch.empty(self.max_keys, dtype=torch.int64, device=dev),
                "out": torch.empty(self.max_keys, dtype=torch.int64, device=dev),
                "cnt": torch.zeros(1, dtype=torch.int32, device=dev),
                "h_out": torch.empty(self.max_keys, dtype=torch.int64).pin_memory(),
                "h_cnt": torch.zeros(1, dtype=torch.int32).pin_memory(),
                "ev": torch.cuda.Event(), "busy": False, "start": 0, "end": 0,
            })
        self._next = 0
        self.keys_total = 0
        self.keys_to_host = 0

    def submit(self, keys: torch.Tensor, start: int, end: int = 0) -> None:
        """keys: 1-D int64 (CPU or CUDA). One submission per call; blocks only if ``depth`` submissions are in flight."""
        end = int(end) if end else int(start) + 1
        s = self._slots[self._next % len(self._slots)]
        self._next += 1
        if s["busy"]:
            self._finish(s, block=True)
        n = keys.numel()
        if n > self.max_keys:
            raise ValueError(f"IntentPrepass: {n} keys > max_keys {self.max_keys}")
        kd = s["keys"][:n]
        kd.copy_(keys.view(-1), non_blocking=True)
        s["cnt"].zero_()
        _C.intent_prepass(self.server._impl.backend_handle(), _stream(kd), kd.data_ptr(), n, end, self.worker._impl.id(),
                          s["out"].data_ptr(), s["cnt"].data_ptr())
        s["h_cnt"].copy_(s["cnt"], non_blocking=True)
        s["h_out"][:n].copy_(s["out"][:n], non_blocking=True)
        s["ev"].record()
        s.update(busy=True, start=int(start), end=end, n=n)
        self.keys_total += n

    def _finish(self, s, block: bool) -> bool:
        if not s["busy"]:
            return True
        if not block and not s["ev"].query():
            return False
        s["ev"].synchronize()
        cnt = int(s["h_cnt"][0])
        if cnt:
            self.worker.intent(s["h_out"][:cnt].clone(), s["start"], s["end"])
        self.keys_to_host += cnt
        s["busy"] = False
        return True

    def harvest(self, block: bool = False) -> None:
        """Hands the left-over keys of completed submissions to the host path (all submissions when ``block``)."""
        for s in self._slots:
            self._finish(s, block)


# ---------------------------------------------------------------------------------------------- node2vec walks
_U64 = (1 << 64) - 1
_M1, _M2 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53)


def _mix64_np(x: np.ndarray) -> np.ndarray:
    """``mix64`` of csrc/cuda/hash.cuh on a uint64 array (integer arrays wrap on overflow)"""
    s = np.uint64(33)
    x = x ^ (x >> s)
    x = x * _M1
    x = x ^ (x >> s)
    x = x * _M2
    return x ^ (x >> s)


def _mix64_int(x: int) -> int:
    return int(_mix64_np(np.array([int(x) & _U64], dtype=np.uint64))[0])


def _umulhi_np(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """the high 64 bits of a * b for uint64 arrays (``__umul64hi``)"""
    m, s = np.uint64(0xFFFFFFFF), np.uint64(32)
    al, ah, bl, bh = a & m, a >> s, b & m, b >> s
    ll, hl, lh = al * bl, ah * bl, al * bh
    cross = (ll >> s) + (hl & m) + lh
    return ah * bh + (hl >> s) + (cross >> s)


def walk_thresholds(p: float, q: float):
    """The 24-bit acceptance thresholds of node2vec's rejection rule, ``max(1, round(alpha / alpha_max * 2^24))`` for
    alpha = 1 / p (return to the previous node), 1 (a neighbour of the previous node) and 1 / q (outward), and whether
    the walk is second order (not ``p == q == 1``)."""
    p, q = float(p), float(q)
    if not (math.isfinite(p) and math.isfinite(q) and p > 0 and q > 0):
        raise ValueError(f"p and q must be positive and finite, got p {p}, q {q}")
    a = (1.0 / p, 1.0, 1.0 / q)
    top = max(a)
    thr = tuple(max(1, int(round(x / top * (1 << 24)))) for x in a)
    return thr, not (p == 1.0 and q == 1.0)


def _check_walk_length(walk_length) -> int:
    if isinstance(walk_length, bool) or int(walk_length) != walk_length or int(walk_length) < 2:
        raise ValueError(f"walk_length must be an integer >= 2, got {walk_length}")
    return int(walk_length)


def _check_window(window) -> int:
    if isinstance(window, bool) or int(window) != window or int(window) < 1:
        raise ValueError(f"window must be an integer >= 1, got {window}")
    return int(window)


def _walk_starts(graph, starts, walk_numbers):
    """(starts, walk numbers) as int64 numpy arrays of one shape, checked against the graph"""
    s = (starts.cpu().numpy() if isinstance(starts, torch.Tensor) else np.asarray(starts)).reshape(-1)
    if s.size and not np.issubdtype(s.dtype, np.integer):
        raise ValueError(f"starts must be integer node ids, got dtype {s.dtype}")
    s = s.astype(np.int64)
    if isinstance(walk_numbers, torch.Tensor):
        walk_numbers = walk_numbers.cpu().numpy()
    wn = np.broadcast_to(np.asarray(walk_numbers, dtype=np.int64).reshape(-1) if np.ndim(walk_numbers) else
                         np.int64(walk_numbers), s.shape).astype(np.int64)
    if s.size and (int(s.min()) < 0 or int(s.max()) >= graph.num_nodes):
        raise ValueError(f"start ids must be in [0, {graph.num_nodes})")
    if wn.size and int(wn.min()) < 0:
        raise ValueError("walk numbers must be non-negative")
    return s, wn


def random_walks(graph, starts, walk_numbers, walk_length: int, p: float = 1.0, q: float = 1.0, seed: int = 0,
                 epoch: int = 0) -> torch.Tensor:
    """node2vec walks on the device (csrc/cuda/ops_walk.cu): walk ``w`` starts at ``starts[w]`` and is the
    ``walk_numbers[w]``-th walk from it (an int applies to every walk). Returns int64 ``[n, walk_length]`` on the graph's
    device; position 0 is the start, and the positions after a node without out-edges are -1. First order (DeepWalk)
    when ``p == q == 1``, else node2vec's second-order walk by rejection sampling; weighted graphs draw by their quantised
    weights. Every draw is a counter hash of ``(seed, epoch, start, walk number, step, trial)``, so a walk does not
    depend on which call, chunk or rank makes it, and :func:`random_walks_reference` gives the same walks bit for bit.

    ``starts`` and ``walk_numbers`` are checked on the host: pass CPU tensors or arrays to keep the call free of device
    synchronisation. ``ValueError`` on ``p, q <= 0``, ``walk_length < 2``, start ids out of range, or a graph that is
    not on a CUDA device."""
    if not graph.offsets.is_cuda:
        raise ValueError("random_walks needs a graph on a CUDA device (Graph.to('cuda')); use random_walks_reference "
                         "on the CPU")
    L = _check_walk_length(walk_length)
    (t_ret, t_in, t_out), second = walk_thresholds(p, q)
    s, wn = _walk_starts(graph, starts, walk_numbers)
    dev = graph.device
    out = torch.empty(s.size, L, dtype=torch.int64, device=dev)
    if s.size == 0:
        return out
    sd = torch.from_numpy(s).to(dev, non_blocking=True)
    wd = torch.from_numpy(np.ascontiguousarray(wn)).to(dev, non_blocking=True)
    with torch.cuda.device(dev):
        _C.node2vec_walks(_stream(out), graph.offsets.data_ptr(), graph.neighbors.data_ptr(),
                          graph.cum_weights.data_ptr() if graph.weighted else 0, sd.data_ptr(), wd.data_ptr(), s.size,
                          L, int(seed) & _U64, int(epoch) & _U64, t_ret, t_in, t_out, second, out.data_ptr())
    return out


def walk_pairs(walks: torch.Tensor, window: int, seed: int = 0) -> torch.Tensor:
    """Skip-gram pairs of walks ``[n, L]`` (int64 CUDA, -1 padding after a walk's end) in the layout ``sgns_step``
    takes: int64 ``[2, n_pairs]``, row 0 the syn0 keys ``2 walk[j]``, row 1 the syn1 keys ``2 walk[i] + 1``. Position
    ``i`` of walk row ``r`` draws a window shrink ``b`` in ``[0, window)`` by a counter hash of ``(seed, r, i)`` and pairs
    with every position ``j != i`` of its walk within ``window - b``: walk-major, then ``i``, then ascending ``j``, the
    order of ``utils.text.pairs_from_sentences``. Count kernel, cub scan, write kernel; reading the pair count is the
    call's one host synchronisation. :func:`walk_pairs_reference` is the same rule in numpy."""
    if not (walks.is_cuda and walks.dtype == torch.int64 and walks.dim() == 2 and walks.is_contiguous()):
        raise TypeError("walks must be a contiguous 2-D CUDA int64 tensor")
    W = _check_window(window)
    n, L = walks.shape
    dev = walks.device
    if n * L == 0:
        return torch.empty(2, 0, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        counts = torch.empty(n * L, dtype=torch.int64, device=dev)
        ends = torch.empty(n * L, dtype=torch.int64, device=dev)
        temp = torch.empty(max(1, _C.walk_pair_scan_bytes(n * L)), dtype=torch.uint8, device=dev)
        s = int(seed) & _U64
        _C.walk_pair_ends(_stream(walks), walks.data_ptr(), n, L, W, s, counts.data_ptr(), ends.data_ptr(),
                          temp.data_ptr(), temp.numel())
        P = int(ends[-1])
        out = torch.empty(2, P, dtype=torch.int64, device=dev)
        _C.walk_pairs_write(_stream(walks), walks.data_ptr(), n, L, W, s, ends.data_ptr(), P, out.data_ptr())
    return out


def random_walks_reference(graph, starts, walk_numbers, walk_length: int, p: float = 1.0, q: float = 1.0,
                           seed: int = 0, epoch: int = 0) -> np.ndarray:
    """The walks of :func:`random_walks` in numpy (int64 ``[n, walk_length]``), with the same integer rule; the CPU
    backend's walk generator and the device kernels' oracle. The graph may be on any device."""
    L = _check_walk_length(walk_length)
    (t_ret, t_in, t_out), second = walk_thresholds(p, q)
    s, wn = _walk_starts(graph, starts, walk_numbers)
    off = graph.offsets.cpu().numpy()
    nbr = graph.neighbors.cpu().numpy().astype(np.int64)
    n = graph.num_nodes
    deg = np.diff(off)
    src = np.repeat(np.arange(n, dtype=np.int64), deg)
    edge_key = src * n + nbr                                            # sorted: the CSR is sorted by (node, neighbour)
    if graph.weighted:
        cw = graph.cum_weights.cpu().numpy()
        total = np.zeros(n + 1, dtype=np.int64)
        last = off[1:] - 1
        total[1:] = np.cumsum(np.where(deg > 0, cw[np.maximum(last, 0)], 0))
        glob = (cw + np.repeat(total[:-1], deg)).astype(np.uint64)      # strictly increasing over all edges
    s0 = _mix64_int(_mix64_int(seed) ^ (int(epoch) & _U64))
    out = np.full((s.size, L), -1, dtype=np.int64)
    out[:, 0] = s
    base = _mix64_np(_mix64_np(np.uint64(s0) ^ s.astype(np.uint64)) ^ wn.astype(np.uint64))
    v, t = s.copy(), np.full(s.size, -1, dtype=np.int64)
    alive = np.arange(s.size)
    for k in range(1, L):
        alive = alive[deg[v[alive]] > 0]
        if alive.size == 0:
            break
        x_new = np.empty(alive.size, dtype=np.int64)
        pend = np.arange(alive.size)
        j = 0
        while pend.size:
            w = alive[pend]
            h = _mix64_np(base[w] ^ np.uint64((k << 32) | j))
            vv = v[w]
            if graph.weighted:
                r = _umulhi_np(h, cw[off[vv + 1] - 1].astype(np.uint64))
                e = np.searchsorted(glob, total[vv].astype(np.uint64) + r, side="right")
            else:
                e = off[vv] + ((h >> np.uint64(32)) * deg[vv].astype(np.uint64) >> np.uint64(32)).astype(np.int64)
            x = nbr[e]
            acc = np.ones(pend.size, dtype=bool)
            if second and k >= 2:
                u = (_mix64_np(h) >> np.uint64(40)).astype(np.int64)
                tt = t[w]
                key = tt * n + x
                pos = np.minimum(np.searchsorted(edge_key, key), max(edge_key.size - 1, 0))
                inn = (edge_key[pos] == key) if edge_key.size else np.zeros(pend.size, dtype=bool)
                thr = np.where(x == tt, t_ret, np.where(inn, t_in, t_out))
                acc = u < thr
            x_new[pend[acc]] = x[acc]
            pend = pend[~acc]
            j += 1
        out[alive, k] = x_new
        t[alive] = v[alive]
        v[alive] = x_new
    return out


def walk_pairs_reference(walks, window: int, seed: int = 0) -> np.ndarray:
    """The pairs of :func:`walk_pairs` in numpy: int64 ``[2, n_pairs]``."""
    W = _check_window(window)
    w = walks.cpu().numpy() if isinstance(walks, torch.Tensor) else np.asarray(walks, dtype=np.int64)
    n, L = w.shape
    r = np.arange(n, dtype=np.uint64).reshape(n, 1)
    i = np.arange(L, dtype=np.uint64).reshape(1, L)
    h = _mix64_np(np.uint64(_mix64_int(seed)) ^ ((r << np.uint64(32)) | i))
    rad = W - ((h >> np.uint64(32)) * np.uint64(W) >> np.uint64(32)).astype(np.int64)     # [n, L]
    delta = np.concatenate([np.arange(-W, 0), np.arange(1, W + 1)])                       # ascending j = i + delta
    jj = np.arange(L).reshape(1, L, 1) + delta.reshape(1, 1, -1)
    inside = (jj >= 0) & (jj < L)
    ctx = w[np.arange(n).reshape(n, 1, 1), np.clip(jj, 0, L - 1)]                           # [n, L, 2 W]
    keep = inside & (np.abs(delta).reshape(1, 1, -1) <= rad[:, :, None]) & (w[:, :, None] >= 0) & (ctx >= 0)
    centre = np.broadcast_to(w[:, :, None], keep.shape)
    return np.stack([2 * ctx[keep], 2 * centre[keep] + 1]).astype(np.int64)


# ---------------------------------------------------------------------------------------------- device key sampler
_SAMPLER_KINDS = {"alias": 0, "uniform": 1, "log-uniform": 2}


def _sampler_hash(seed: int, i: np.ndarray, t: int) -> np.ndarray:
    """the 64-bit hash of try ``t`` of draws ``i`` (uint64 array): ``mix64(seed ^ (i * C1 + t * C2))``"""
    ti = np.uint64((int(t) * 0xD1B54A32D192ED03) & _U64)
    return _mix64_np(np.uint64(int(seed) & _U64) ^ (i * np.uint64(0x9E3779B97F4A7C15) + ti))


def _sampler_draw(kind: int, h: np.ndarray, prob, alias, n_table: int, first: int, stride: int) -> np.ndarray:
    hi, lo = h >> np.uint64(32), (h & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    if kind == 2:
        x = np.exp(hi.astype(np.float64) * 2.0 ** -32 * math.log(n_table + 1))
        j = np.clip(np.floor(x).astype(np.int64) - 1, 0, n_table - 1)
    else:
        j = ((hi * np.uint64(n_table)) >> np.uint64(32)).astype(np.int64)
        if kind == 0:
            u = lo.astype(np.float32) * np.float32(2.0 ** -32)     # the device's round-to-nearest cast, exact scaling
            j = np.where(u < prob[j], j, alias[j].astype(np.int64))
    return first + j * stride


def sample_keys_reference(n: int, seed: int, *, distribution: str = "alias", prob=None, alias=None,
                          num_keys: Optional[int] = None, first_key: int = 0, key_stride: int = 1, resident=None,
                          max_tries: int = 64, chunk: int = 1 << 22):
    """The ``n`` keys of :meth:`DeviceSampler.sample` (csrc/cuda/ops_sampler.cu) in numpy, bit for bit; the device
    kernel's oracle. Draw ``i``, try ``t`` hashes ``h = mix64(seed ^ (i * 0x9E3779B97F4A7C15 + t * 0xD1B54A32D192ED03))``
    and splits it into ``hi = h >> 32`` and ``lo = h mod 2^32``:

    - ``alias`` (``prob`` float32 and ``alias`` int32 of the table): bucket ``b = (hi * n) >> 32``, ``u = float32(lo) *
      2^-32`` (round to nearest, as the device casts), index ``b if u < prob[b] else alias[b]``;
    - ``uniform`` over ``num_keys``: index ``(hi * num_keys) >> 32``;
    - ``log-uniform`` over ``num_keys``: index ``floor(exp(hi * 2^-32 * ln(num_keys + 1))) - 1`` in float64, clamped
      to ``[0, num_keys)``. The device takes ``exp`` in double too, so the two agree except where the value lies within
      a few ulps of an integer.

    The key is ``first_key + index * key_stride``. With ``resident`` (a bool array over keys: the residency the
    ``local_only`` kernel probes), a draw that is not resident is redrawn with ``t + 1`` until one is or ``max_tries``
    draws were made (then the last draw is kept: a give-up); returns ``(keys, checks, misses)``, the draws made and the
    give-ups, as the kernel counts them into ``stats``. Otherwise returns the keys (int64 numpy array)."""
    kind = _SAMPLER_KINDS[distribution]
    if kind == 0:
        prob = np.asarray(prob.cpu() if isinstance(prob, torch.Tensor) else prob, dtype=np.float32)
        alias = np.asarray(alias.cpu() if isinstance(alias, torch.Tensor) else alias, dtype=np.int64)
        n_table = prob.size
    else:
        n_table = int(num_keys)
    if isinstance(resident, torch.Tensor):
        resident = resident.cpu().numpy()
    keys = np.empty(int(n), dtype=np.int64)
    checks = misses = 0
    tries = max(1, int(max_tries))
    for s in range(0, int(n), chunk):
        idx = np.arange(s, min(int(n), s + chunk), dtype=np.uint64)
        k = _sampler_draw(kind, _sampler_hash(seed, idx, 0), prob, alias, n_table, first_key, key_stride)
        if resident is not None:
            checks += idx.size
            pend = np.flatnonzero(~resident[k])
            for t in range(1, tries):
                if pend.size == 0:
                    break
                k[pend] = _sampler_draw(kind, _sampler_hash(seed, idx[pend], t), prob, alias, n_table, first_key,
                                        key_stride)
                checks += pend.size
                pend = pend[~resident[k[pend]]]
            misses += pend.size
        keys[s:s + idx.size] = k
    return keys if resident is None else (keys, checks, misses)


def alias_draw_probabilities(prob, alias) -> np.ndarray:
    """The probability (float64 ``[n]``) with which the device draws each index from the alias table ``(prob, alias)``
    under the rule of :func:`sample_keys_reference`. Bucket ``i`` takes ``c_i = ceil((i+1) 2^32 / n) - ceil(i 2^32 / n)``
    of the ``hi`` values; of those, the ``L_i`` values of ``lo`` with ``float32(lo) 2^-32 < prob[i]`` (a binary search
    over ``lo``: the cast is monotone) draw ``i`` and the rest draw ``alias[i]``. ``P_j = sum c_i L_i / 2^64`` over
    the buckets that draw ``j``, summed in integers, so the only rounding is the final one to float64. Compare it with
    ``w / sum(w)``: it is the distribution of table and draw rule together, without sampling noise."""
    prob = np.asarray(prob.cpu() if isinstance(prob, torch.Tensor) else prob, dtype=np.float32)
    alias = np.asarray(alias.cpu() if isinstance(alias, torch.Tensor) else alias, dtype=np.int64)
    n = prob.size
    i = np.arange(n + 1, dtype=np.uint64)
    c = np.diff(((i << np.uint64(32)) + np.uint64(n - 1)) // np.uint64(n)).astype(np.int64)
    lo, hi = np.zeros(n, dtype=np.int64), np.full(n, 1 << 32, dtype=np.int64)   # L_i in [lo, hi]
    while True:
        active = lo < hi
        if not active.any():
            break
        mid = (lo + hi) >> 1
        at_or_above = mid.astype(np.float32) * np.float32(2.0 ** -32) >= prob
        hi = np.where(active & at_or_above, mid, hi)
        lo = np.where(active & ~at_or_above, mid + 1, lo)
    A, B = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)   # P = (A 2^16 + B) / 2^64; A, B <= 2^48
    for to, cnt in ((np.arange(n), lo), (alias, (1 << 32) - lo)):
        np.add.at(A, to, c * (cnt >> 16))
        np.add.at(B, to, c * (cnt & 0xFFFF))
    return A * 2.0 ** -48 + B * 2.0 ** -64


# ---------------------------------------------------------------------------------------------- doc2vec inference
DOC2VEC_MAX_DIM = 336
DOC2VEC_MAX_TARGETS = 32
DOC2VEC_MAX_WINDOW = 15
DOC2VEC_MAX_WORDS = 10000


def _int_arg(x, name: str) -> int:
    if isinstance(x, bool) or not isinstance(x, (int, np.integer)):
        raise TypeError(f"{name} must be an integer, got {type(x).__name__}")
    return int(x)


def _check_doc2vec_args(dm, embed_dim, negative, window, epochs, alpha, min_alpha):
    """Validates the scalar arguments of :func:`doc2vec_infer` (``ValueError`` / ``TypeError``)."""
    d, neg, win, E = (_int_arg(embed_dim, "embed_dim"), _int_arg(negative, "negative"), _int_arg(window, "window"),
                      _int_arg(epochs, "epochs"))
    if not (4 <= d <= DOC2VEC_MAX_DIM and d % 4 == 0):
        raise ValueError(f"embed_dim must be a multiple of 4 in [4, {DOC2VEC_MAX_DIM}], got {d}")
    if not 1 <= neg <= DOC2VEC_MAX_TARGETS - 1:
        raise ValueError(f"negative must be in [1, {DOC2VEC_MAX_TARGETS - 1}], got {neg}")
    if dm and not 1 <= win <= DOC2VEC_MAX_WINDOW:
        raise ValueError(f"PV-DM needs window in [1, {DOC2VEC_MAX_WINDOW}], got {win}")
    if E < 1:
        raise ValueError(f"epochs must be at least 1, got {E}")
    a, ma = float(alpha), float(min_alpha)
    if not (math.isfinite(a) and math.isfinite(ma) and 0.0 < ma <= a):
        raise ValueError(f"need 0 < min_alpha <= alpha, got alpha {alpha}, min_alpha {min_alpha}")
    return bool(dm), d, neg, win, E, a, ma


def _check_doc2vec_docs(tokens: torch.Tensor, offsets: torch.Tensor, doc_ids: torch.Tensor, num_words: int):
    """Checks the CSR documents on the host; returns (tokens, offsets, doc_ids) as int64 CPU tensors."""
    for t, name in ((tokens, "tokens"), (offsets, "offsets"), (doc_ids, "doc_ids")):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int64 or t.dim() != 1:
            raise TypeError(f"{name} must be a 1-D int64 tensor")
    tok, off, ids = tokens.cpu(), offsets.cpu(), doc_ids.cpu()
    M = ids.numel()
    if off.numel() != M + 1:
        raise ValueError(f"offsets must have M + 1 = {M + 1} entries for {M} doc_ids, got {off.numel()}")
    lens = off[1:] - off[:-1]
    if int(off[0]) != 0 or int(off[-1]) != tok.numel() or bool((lens < 0).any()):
        raise ValueError("offsets must start at 0, be monotone and end at the number of tokens")
    if M and int(lens.max()) > DOC2VEC_MAX_WORDS:
        raise ValueError(f"a document has {int(lens.max())} words, at most {DOC2VEC_MAX_WORDS} are allowed")
    if tok.numel() and (int(tok.min()) < 0 or int(tok.max()) >= num_words):
        raise ValueError(f"word ids must be in [0, {num_words})")
    return tok, off, ids


def _doc2vec_alphas(E: int, alpha: float, min_alpha: float):
    return [alpha - e * (alpha - min_alpha) / max(1, E - 1) for e in range(E)]


def doc2vec_infer(server, tokens: torch.Tensor, offsets: torch.Tensor, doc_ids: torch.Tensor, sampler, *, dm: bool,
                  embed_dim: int, negative: int, window: int, epochs: int, alpha: float, min_alpha: float, seed: int,
                  loss: Optional[torch.Tensor] = None, num_words: Optional[int] = None) -> torch.Tensor:
    """Paragraph-vector inference on the device (csrc/cuda/ops_doc2vec.cu): one new vector per document, trained against
    the store's frozen rows (word ``w``'s syn0 row is key ``2 w``, its syn1 row key ``2 w + 1``). Document ``m`` is the
    word ids ``tokens[offsets[m]:offsets[m + 1]]`` (int64 CSR, ``offsets`` [M + 1]) with the id ``doc_ids[m]``;
    ``sampler`` is the :class:`DeviceSampler` of the model's negatives. Returns float32 ``[M, embed_dim]``.

    The rule (the kernel file's header; :func:`doc2vec_infer_reference` in float64): the vector starts at
    ``(u - 0.5) / d`` from a counter hash of ``(seed, doc_ids[m], k)`` with AdaGrad state 1e-6; epoch ``e`` uses
    ``alpha_e = alpha - e (alpha - min_alpha) / max(1, epochs - 1)`` and visits the positions in order, scoring the
    word's syn1 row (label 1) and ``negative`` sampler draws (label 0; one equal to the word is skipped) against
    ``h = v`` (PV-DBOW, ``dm=False``) or the mean of ``v`` and the syn0 rows of a window shrunk by a hash draw (PV-DM),
    then ``v += alpha_e neu1e / sqrt(a + neu1e^2)``, ``a += neu1e^2``. Store rows are only read; a document's vector does
    not depend on the other documents of the call. ``loss``: CUDA float32 [1], accumulated (+=) with the summed
    logistic loss. Limits (checked before any launch, ``ValueError``): ``embed_dim`` a multiple of 4 in [4, 336],
    ``1 <= negative <= 31``, PV-DM ``1 <= window <= 15``, ``epochs >= 1``, ``0 < min_alpha <= alpha``, at most 10 000
    words per document, word ids outside ``[0, num_words)`` (default: every id whose rows are in the store);
    ``TypeError`` for tensors of the wrong dtype or shape.
    The documents are checked on the host, so device tensors cost a copy. One launch per epoch."""
    dm, d, neg, win, E, a, ma = _check_doc2vec_args(dm, embed_dim, negative, window, epochs, alpha, min_alpha)
    if not isinstance(sampler, DeviceSampler):
        raise TypeError("sampler must be a DeviceSampler")
    if loss is not None and not (loss.is_cuda and loss.dtype == torch.float32 and loss.numel() >= 1):
        raise TypeError("loss must be a CUDA float32 tensor")
    tok, off, ids = _check_doc2vec_docs(tokens, offsets, doc_ids,
                                        server.num_keys() // 2 if num_words is None else int(num_words))
    dev = server.device
    M = ids.numel()
    state = torch.empty(M, 2 * d, dtype=torch.float32, device=dev)
    if M == 0:
        return state[:, :d]
    tok_d = tok.to(dev) if tok.numel() else torch.zeros(1, dtype=torch.int64, device=dev)
    off_d, ids_d = off.to(dev), ids.to(dev)
    own = _gather_stats(server, None, dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for e, ae in enumerate(_doc2vec_alphas(E, a, ma)):
        _C.doc2vec_infer_epoch(server._impl.backend_handle(), stream, tok_d.data_ptr(), off_d.data_ptr(),
                               ids_d.data_ptr(), M, dm, d, neg, win, e, float(ae), int(seed) & _U64, sampler.kind,
                               sampler.prob.data_ptr(), sampler.alias.data_ptr(), sampler.n, sampler.first_key,
                               sampler.key_stride, state.data_ptr(), loss.data_ptr() if loss is not None else 0,
                               own.data_ptr() if own is not None else 0)
    _gathered("doc2vec_infer", own, None)
    return state[:, :d]


def _doc2vec_base(seed: int, doc_ids: np.ndarray) -> np.ndarray:
    return _mix64_np(np.uint64(_mix64_int(seed)) ^ doc_ids.astype(np.uint64))


def doc2vec_initial_vectors(seed: int, doc_ids, d: int) -> np.ndarray:
    """The documents' starting vectors of :func:`doc2vec_infer`, float32 ``[M, d]``: ``(u - 0.5) / d`` with
    ``u = (mix64(base ^ (2^63 | k)) >> 40) 2^-24`` and ``base = mix64(mix64(seed) ^ doc_id)``, in float32 as the
    kernel computes it."""
    ids = np.asarray(doc_ids, dtype=np.int64).reshape(-1)
    base = _doc2vec_base(seed, ids)
    k = np.arange(d, dtype=np.uint64) | np.uint64(1 << 63)
    u = (_mix64_np(base[:, None] ^ k[None, :]) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    return (u - np.float32(0.5)) / np.float32(d)


def doc2vec_infer_reference(kv, tokens, offsets, doc_ids, sampler, *, dm: bool, embed_dim: int, negative: int,
                            window: int, epochs: int, alpha: float, min_alpha: float, seed: int,
                            num_words: Optional[int] = None) -> tuple:
    """The rule of :func:`doc2vec_infer` in float64 through Pull (any backend): the initial vectors and PV-DM shrinks
    replayed in numpy, the negatives with the sampler's draw rule (:func:`sample_keys_reference`'s, seeded per document
    and epoch). ``sampler``: a :class:`DeviceSampler`, or a dict with its ``kind``, ``prob``, ``alias``, ``n``,
    ``first_key`` and ``key_stride``. Vectorised over documents, sequential over positions. Returns ``(vectors float64
    [M, d] numpy, summed loss)``."""
    dm, d, neg, win, E, a, ma = _check_doc2vec_args(dm, embed_dim, negative, window, epochs, alpha, min_alpha)
    sp = sampler if isinstance(sampler, dict) else {k: getattr(sampler, k) for k in
                                                    ("kind", "prob", "alias", "n", "first_key", "key_stride")}
    prob = np.asarray(sp["prob"].cpu() if isinstance(sp["prob"], torch.Tensor) else sp["prob"], dtype=np.float32)
    alias = np.asarray(sp["alias"].cpu() if isinstance(sp["alias"], torch.Tensor) else sp["alias"], dtype=np.int64)
    tok, off, ids = (torch.as_tensor(np.asarray(x), dtype=torch.int64) if not isinstance(x, torch.Tensor) else x
                     for x in (tokens, offsets, doc_ids))
    tok, off, ids = _check_doc2vec_docs(tok, off, ids,
                                        kv.server.num_keys() // 2 if num_words is None else int(num_words))
    tok, off, ids = tok.numpy(), off.numpy(), ids.numpy()
    M = ids.size
    lens = np.diff(off)
    v = doc2vec_initial_vectors(seed, ids, d).astype(np.float64)
    acc = np.full((M, d), 1e-6, dtype=np.float32).astype(np.float64)
    total = 0.0
    if M == 0 or tok.size == 0:
        return v, total
    have_k = np.zeros(0, dtype=np.int64)
    have_r = np.zeros((0, d))

    def fetch(keys):
        """the first d values of the store rows of keys (any shape), pulled once per distinct key"""
        nonlocal have_k, have_r
        miss = np.setdiff1d(keys, have_k)
        if miss.size:
            buf = torch.empty(miss.size * 2 * d, dtype=torch.float32)
            kv.wait(kv.pull(torch.from_numpy(miss), buf))
            have_k = np.concatenate([have_k, miss])
            have_r = np.concatenate([have_r, buf.view(miss.size, 2 * d)[:, :d].double().numpy()])
            order = np.argsort(have_k)
            have_k, have_r = have_k[order], have_r[order]
        return have_r[np.searchsorted(have_k, keys)]

    base = _doc2vec_base(seed, ids)
    kind, n_table, first, stride = int(sp["kind"]), int(sp["n"]), int(sp["first_key"]), int(sp["key_stride"])
    Lmax = int(lens.max())
    for e, ae in enumerate(_doc2vec_alphas(E, a, ma)):
        es = _mix64_np(base ^ np.uint64((1 << 62) | e))
        ss = _mix64_np(es)
        for i in range(Lmax):
            act = np.flatnonzero(lens > i)                                   # documents that have position i
            pos_key = 2 * tok[off[act] + i] + 1
            n = (np.uint64(i * neg) + np.arange(neg, dtype=np.uint64))[None, :]
            h = _mix64_np(es[act, None] ^ (n * np.uint64(0x9E3779B97F4A7C15)))
            draws = _sampler_draw(kind, h, prob, alias, n_table, first, stride)        # [A, neg]
            tkeys = np.concatenate([pos_key[:, None], draws], 1)
            valid = np.ones(tkeys.shape, dtype=bool)
            valid[:, 1:] = draws != pos_key[:, None]
            T = fetch(tkeys)                                                 # [A, 1 + neg, d]
            hv = v[act].copy()
            if dm:
                r = win - (_mix64_np(ss[act] ^ np.uint64(i)) % np.uint64(win)).astype(np.int64)
                for delta in range(-win, win + 1):                           # ascending context positions
                    j = i + delta
                    m = (delta != 0) & (np.abs(delta) <= r) & (j >= 0) & (j < lens[act])
                    if m.any():
                        hv[m] += fetch(2 * tok[off[act[m]] + j])
                C = np.minimum(lens[act], i + r + 1) - np.maximum(0, i - r) - 1
                hv /= (1 + C)[:, None]
            f = np.einsum("ad,atd->at", hv, T)
            label = np.zeros(f.shape)
            label[:, 0] = 1
            g = np.where(f > 6, label - 1, np.where(f < -6, label, label - 1 / (1 + np.exp(-f)))) * valid
            z = np.clip(np.where(label > 0.5, f, -f), -6, 6)
            total += float((np.log1p(np.exp(-z)) * valid).sum())
            neu = np.einsum("at,atd->ad", g, T)
            v[act] += ae * neu / np.sqrt(acc[act] + neu * neu)
            acc[act] += neu * neu
    return v, total
