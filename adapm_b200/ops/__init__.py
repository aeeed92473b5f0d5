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
        need = _C.embedding_bag_workspace_bytes(nnz, nbags, self.dim)
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
