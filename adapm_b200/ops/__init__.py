"""Torch-facing wrappers of the hand-written sm_90a kernels (csrc/cuda/ops_*.cu).

All ops take CUDA tensors, run on the current CUDA stream and operate directly on the
parameter store of a ``Server`` with ``backend='cuda'`` (local HBM and NVLink-mapped peers).
They fail loudly when the native extension or a CUDA device is missing - there is no eager
fallback on a GPU box.
"""
from __future__ import annotations

from typing import Optional

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
    variant) or ``auto`` (tma when the shape fits, else ldg; ``ADAPM_SGNS_IMPL`` overrides).
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
    """

    def __init__(self, server, *, weights: Optional[torch.Tensor] = None, distribution: str = "alias",
                 first_key: int = 0, key_stride: int = 1, num_keys: Optional[int] = None):
        self.server = server
        self.first_key, self.key_stride = int(first_key), int(key_stride)
        dev = server.device
        if weights is not None:
            w = torch.as_tensor(weights, dtype=torch.float64).contiguous().cpu()
            n = w.numel()
            prob = torch.empty(n, dtype=torch.float32)
            alias = torch.empty(n, dtype=torch.int32)
            _C.build_alias_table(w.data_ptr(), n, prob.data_ptr(), alias.data_ptr())
            self.kind, self.n = 0, n
            self.prob, self.alias = prob.to(dev), alias.to(dev)
        else:
            if num_keys is None:
                raise ValueError("num_keys is required for uniform / log-uniform sampling")
            self.kind = {"uniform": 1, "log-uniform": 2}[distribution]
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


def gather_gemm(server, q: torch.Tensor, keys: torch.Tensor, k: int, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """scores[M, N] = q[M, k] @ E^T where row n of E is the first ``k`` values of store row ``keys[n]`` - the rows
    are gathered inside the GEMM kernel from the local slab, local replicas or peer GPUs over NVLink (fused
    gather + wgmma GEMM); the gathered matrix never exists in HBM."""
    _i64(keys, "keys")
    q16 = _bf16_k8(q)
    M, N = q16.shape[0], keys.numel()
    c = torch.empty(M, N, dtype=torch.float32, device=q.device)
    _C.gather_gemm(server._impl.backend_handle(), _stream(q16), q16.data_ptr(), keys.data_ptr(), M, N, int(k), q16.shape[1],
                   c.data_ptr(), N, stats.data_ptr() if stats is not None else 0)
    return c


def gather_gemm_rank_count(server, q: torch.Tensor, keys: torch.Tensor, k: int, true_score: torch.Tensor,
                           true_col: torch.Tensor, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """counts[i] = #{n != true_col[i] : <q[i], row(keys[n])[:k]> > true_score[i]}: fused gather + GEMM + ranking
    epilogue - neither the gathered rows nor the [M, N] scores are materialised."""
    _i64(keys, "keys")
    q16 = _bf16_k8(q)
    M, N = q16.shape[0], keys.numel()
    out = torch.zeros(M, dtype=torch.int32, device=q.device)
    ts = true_score.to(torch.float32).contiguous()
    tc = true_col.to(torch.int32).contiguous()
    _C.gather_gemm_rank_count(server._impl.backend_handle(), _stream(q16), q16.data_ptr(), keys.data_ptr(), M, N, int(k),
                              q16.shape[1], ts.data_ptr(), tc.data_ptr(), out.data_ptr(),
                              stats.data_ptr() if stats is not None else 0)
    return out


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
