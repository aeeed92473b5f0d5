"""CTR prediction with DLRM (Naumov et al., 2019) on the parameter manager, and DLRM-DCNv2, MLPerf's recommendation
model since 2023.

* the sparse part - one row per feature id, ``[embedding (E) | AdaGrad (E)]`` - lives in the parameter manager; every
  (example, field) is a bag of ids pooled by ``ops.StoreEmbeddingBag`` (one id per bag for single-hot data), whose
  backward pushes one AdaGrad update per distinct id;
* the dense features go through the bottom MLP (num_dense -> bottom... -> E, ReLU on every layer);
* ``interaction="dot"``: ``ops.dlrm_interaction`` forms ``[z | <T_i, T_j> for j < i]`` from ``T = [z; e_1 .. e_F]``
  (one fused kernel each way on a CUDA server); ``interaction="dcn"``: ``ops.dcn_cross``, the low-rank cross network
  of DCN-v2 (Wang et al., 2021) over ``x_0 = [z | e_1 .. e_F]`` (bf16 tensor-core GEMMs with fused elementwise work on
  a CUDA server, fp32 on the torch route); the top MLP (W or N -> top... -> 1) gives the logit, BCE-with-logits the loss;
* the MLPs are replicated, trained by Adam; their gradients are all-reduced with ``torch.distributed`` when available,
  as in DeepFM. On a CUDA server their linear layers run on the hand-written wgmma GEMM (``precision``).
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
from torch import nn

from .deepfm import DenseNet
from .ffm import PLANT_DIM, PLANT_TYPES, logloss_auc


@dataclass
class DLRMConfig:
    num_features: int = 10_000_000      # total feature ids = PM keys, split evenly over the fields
    num_fields: int = 26
    num_dense: int = 13
    embed_dim: int = 128
    bottom: tuple = (512, 256)          # num_dense -> bottom... -> embed_dim
    top: tuple = (1024, 1024, 512, 256)  # W -> top... -> 1
    lr_sparse: float = 0.05             # AdaGrad step size of the embedding rows
    lr_dense: float = 1e-3              # Adam on the MLPs
    batch_size: int = 8192
    read_ahead: int = 4
    precision: str = "bf16"             # bf16 | fp8 | fp32 (dense GEMMs)
    multi_hot: int = 0                  # > 0: up to this many ids per field (synthetic_dlrm_batch); 0: one id per field
    pooling: str = "sum"                # sum | mean (multi-hot fields)
    model_seed: int = 1
    interaction: str = "dot"            # dot | dcn (DLRM-DCNv2: low-rank cross network)
    cross_layers: int = 3               # dcn: layers L
    cross_rank: int = 512               # dcn: rank r of V_l [r, N] and W_l [N, r]

    @property
    def row_len(self) -> int:           # [embedding | AdaGrad]
        return 2 * self.embed_dim

    @property
    def interaction_width(self) -> int:
        from ..ops import dlrm_interaction_width

        return dlrm_interaction_width(self.num_fields, self.embed_dim)

    @property
    def cross_width(self) -> int:       # N = (F + 1) E, the width of the cross network
        return (self.num_fields + 1) * self.embed_dim


class CrossNet(nn.Module):
    """The parameters of DCN-v2's low-rank cross network (``ops.dcn_cross``): ``V [L, r, N]`` and ``W [L, N, r]``
    Xavier-normal from ``seed``, ``b [L, N]`` zero."""

    def __init__(self, N: int, rank: int, layers: int, seed: int):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        std = (2.0 / (N + rank)) ** 0.5
        self.V = nn.Parameter(torch.randn(layers, rank, N, generator=g) * std)
        self.W = nn.Parameter(torch.randn(layers, N, rank, generator=g) * std)
        self.b = nn.Parameter(torch.zeros(layers, N))

    def forward(self, z, e, impl: str = "auto"):
        from ..ops import dcn_cross

        return dcn_cross(z, e, self.V, self.W, self.b, impl=impl)


class DLRM:
    def __init__(self, server, worker, cfg: DLRMConfig, impl: str = "auto"):
        """``impl`` selects the route of ``ops.dlrm_interaction`` or ``ops.dcn_cross`` (``auto``: the fused kernels on a
        CUDA server)."""
        from ..ops import StoreEmbeddingBag, dlrm_interaction_width

        if cfg.precision not in ("bf16", "fp8", "fp32"):
            raise ValueError(f"precision must be bf16, fp8 or fp32, got {cfg.precision!r}")
        if cfg.num_dense < 1:
            raise ValueError(f"num_dense must be >= 1, got {cfg.num_dense}")
        if cfg.interaction not in ("dot", "dcn"):
            raise ValueError(f"interaction must be dot or dcn, got {cfg.interaction!r}")
        self.server, self.worker, self.cfg, self.impl = server, worker, cfg, impl
        self.dev = server.device
        tc = server.backend == "cuda"
        E, W = cfg.embed_dim, dlrm_interaction_width(cfg.num_fields, cfg.embed_dim)
        self.bottom = DenseNet(cfg, tc, dims=[cfg.num_dense, *cfg.bottom, E], relu_last=True,
                               seed=cfg.model_seed).to(self.dev)
        self.cross = None
        if cfg.interaction == "dcn":
            W = cfg.cross_width
            self.cross = CrossNet(W, cfg.cross_rank, cfg.cross_layers, cfg.model_seed + 2).to(self.dev)
        self.top = DenseNet(cfg, tc, dims=[W, *cfg.top, 1], seed=cfg.model_seed + 1).to(self.dev)
        self.opt = torch.optim.Adam(self._dense_parameters(), lr=cfg.lr_dense)
        self.bag = StoreEmbeddingBag(server, worker, E, mode=cfg.pooling, lr=cfg.lr_sparse)
        self.step_no = 0
        self.rows_pushed = 0      # (key, row) updates applied so far (distinct feature rows per batch)

    def _dense_parameters(self):
        return [*self.bottom.parameters(), *self.top.parameters(), *(self.cross.parameters() if self.cross else ())]

    def init_model(self, chunk: int = 1 << 18) -> None:
        """Embeddings uniform in +-sqrt(1 / rows per field), accumulators 0; every rank initialises the keys it is home
        for."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        E = cfg.embed_dim
        bound = (1.0 / (cfg.num_features // cfg.num_fields)) ** 0.5
        gen = torch.Generator(device=self.dev.type).manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        keys = torch.arange(rank, cfg.num_features, world, dtype=torch.int64)
        for i in range(0, keys.numel(), chunk):
            kk = keys[i:i + chunk].to(self.dev)
            rows = torch.zeros(kk.numel(), cfg.row_len, device=self.dev)
            rows[:, :E] = (torch.rand(kk.numel(), E, generator=gen, device=self.dev) * 2 - 1) * bound
            self.worker.set(kk, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    def signal_intent(self, feat_ids: torch.Tensor, clock: int) -> None:
        if self.server.num_servers() > 1:
            self.worker.intent(feat_ids.reshape(-1), clock, clock + 1)

    def _bags(self, ids, offsets):
        """keys [nnz] and offsets [B * F + 1] on the device: single-hot ids [B, F] become bags of length 1"""
        F = self.cfg.num_fields
        if offsets is None:
            if ids.dim() != 2 or ids.shape[1] != F:
                raise ValueError(f"single-hot ids must be [B, {F}], got {tuple(ids.shape)}")
            keys = ids.to(self.dev, non_blocking=True).reshape(-1).contiguous()
            off = torch.arange(keys.numel() + 1, dtype=torch.int64, device=self.dev)
        else:
            keys = ids.to(self.dev, non_blocking=True).reshape(-1).contiguous()
            off = offsets.to(self.dev, non_blocking=True).reshape(-1).contiguous()
            if (off.numel() - 1) % F:
                raise ValueError(f"offsets must delimit B * {F} bags")
        return keys, off, (off.numel() - 1) // F

    def _logits(self, dense, ids, offsets):
        from ..ops import dlrm_interaction

        cfg = self.cfg
        keys, off, B = self._bags(ids, offsets)
        if dense.shape != (B, cfg.num_dense):
            raise ValueError(f"dense must be [{B}, {cfg.num_dense}], got {tuple(dense.shape)}")
        z = self.bottom(dense.to(self.dev, non_blocking=True).float())
        e = self.bag(keys, off).view(B, cfg.num_fields, cfg.embed_dim)
        if self.cross is not None:
            return self.top(self.cross(z, e, impl=self.impl)), B
        return self.top(dlrm_interaction(z, e, impl=self.impl)), B

    def step(self, dense: torch.Tensor, ids: torch.Tensor, labels: torch.Tensor,
             offsets: Optional[torch.Tensor] = None, return_tensor: bool = False):
        """dense float32 [B, num_dense]; ids int64 [B, F] (single-hot), or the flat [nnz] ids of all bags with
        ``offsets`` int64 [B * F + 1] (bag ``b * F + f`` holds field f of example b); labels float [B]. Returns the
        batch loss (a float, or the device tensor with ``return_tensor``)."""
        self.bag.grad_scale = float(ids.shape[0] if offsets is None else (offsets.numel() - 1) // self.cfg.num_fields)
        logit, B = self._logits(dense, ids, offsets)
        y = labels.to(self.dev, non_blocking=True).float()
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logit, y)
        self.opt.zero_grad(set_to_none=True)
        loss.backward()
        if torch.distributed.is_available() and torch.distributed.is_initialized() and self.server.num_servers() > 1:
            for p in self._dense_parameters():
                torch.distributed.all_reduce(p.grad)
                p.grad /= self.server.num_servers()
        self.opt.step()
        self.step_no += 1
        self.rows_pushed += self.bag.take_rows_updated()
        return loss.detach() if return_tensor else float(loss.detach())

    def predict(self, dense: torch.Tensor, ids: torch.Tensor, offsets: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Click probabilities [B] on the store's device (no update)."""
        with torch.no_grad():
            return torch.sigmoid(self._logits(dense, ids, offsets)[0])

    def evaluate(self, batches) -> tuple[float, float]:
        """(logloss, AUC) over ``batches`` of (dense, ids, labels) or (dense, ids, offsets, labels)."""
        ps, ys = [], []
        for b in batches:
            dense, ids, *off, y = b
            ps.append(self.predict(dense, ids, off[0] if off else None).double().cpu())
            ys.append(y.double().cpu())
        return logloss_auc(torch.cat(ps).numpy(), torch.cat(ys).numpy())


# ------------------------------------------------------------------------------------------------ planted data
DENSE_SCALE = 1.0       # weights of the two parts of the planted logit (each part has about unit variance)
PAIR_SCALE = 2.0


@functools.lru_cache(maxsize=4)
def _planted_dense(num_dense: int, seed: int):
    """(mean, std, weights) of the planted dense term: the log-count features are standardised by the mean and std of
    a fixed sample of their distribution; the weights are N(0, 1) / sqrt(num_dense)."""
    rng = np.random.default_rng([seed, 0xde15e])
    x = _log_counts(rng, 1 << 16, num_dense)
    return x.mean(0), x.std(0), rng.standard_normal(num_dense) / np.sqrt(num_dense)


def _log_counts(rng, B: int, num_dense: int) -> np.ndarray:
    """log(1 + count) of log-normal integer counts, like Criteo's dense features after the usual transform"""
    return np.log1p(np.floor(np.exp(rng.normal(1.0, 1.5, size=(B, num_dense))))).astype(np.float32)


def planted_dense_term(cfg: DLRMConfig, dense) -> np.ndarray:
    """The dense part of the planted logit of :func:`synthetic_dlrm_batch` for its dense features [B, num_dense]
    (before DENSE_SCALE). The dense features are drawn independently of the ids, so no model of the dense features
    alone ranks the labels better than this term."""
    mu, sd, a = _planted_dense(cfg.num_dense, cfg.model_seed)
    x = dense.numpy() if isinstance(dense, torch.Tensor) else np.asarray(dense)
    return ((x.astype(np.float64) - mu) / sd) @ a


@functools.lru_cache(maxsize=4)
def _planted_pairs(num_fields: int, num_features: int, seed: int) -> np.ndarray:
    """U [F, types, d]: the planted vector of feature type t (local id mod PLANT_TYPES) in field f. U[f] has zero mean
    under the distribution of f's types, so that no field carries the pair signal linearly."""
    F, M, d = num_fields, PLANT_TYPES, PLANT_DIM
    rng = np.random.default_rng([seed, 0xd1a])
    U = rng.standard_normal((F, M, d))
    per_field = num_features // F
    ids = np.arange(per_field)
    p_id = ((ids + 1) / per_field) ** (1 / 3) - (ids / per_field) ** (1 / 3)   # P(local id) under the u^3 skew
    p_type = np.bincount(ids % M, weights=p_id, minlength=M)
    return U - np.einsum("m,fmd->fd", p_type, U)[:, None]


def synthetic_dlrm_batch(cfg: DLRMConfig, step: int, rank: int = 0, held_out: bool = False):
    """Criteo-shaped batch: ``(dense float32 [B, num_dense], ids int64 [B, F], labels float32 [B])``, or with
    ``cfg.multi_hot`` ``(dense, ids int64 [nnz], offsets int64 [B * F + 1], labels)`` with bag lengths uniform in
    ``[1, multi_hot]``. Ids are skewed within each field's range as in ``deepfm.synthetic_ctr_batch``; the dense
    features are log-counts drawn independently of them. Labels are drawn from sigmoid of a planted logit
    ``DENSE_SCALE * planted_dense_term + PAIR_SCALE * sum_{f < g} <u_f, u_g> / sqrt(F (F - 1) / 2 * d)``, where
    ``u_f`` is the planted vector (:func:`_planted_pairs`) of field f's type (the mean over a multi-hot bag).
    ``held_out`` batches use their own seeds."""
    rng = np.random.default_rng([cfg.model_seed, rank, step, 1 if held_out else 0, cfg.multi_hot, 0xd1e])
    B, F = cfg.batch_size, cfg.num_fields
    per_field = cfg.num_features // F
    dense = _log_counts(rng, B, cfg.num_dense)
    U = _planted_pairs(F, cfg.num_features, cfg.model_seed)
    lens = rng.integers(1, cfg.multi_hot + 1, size=B * F) if cfg.multi_hot else np.ones(B * F, dtype=np.int64)
    bag = np.repeat(np.arange(B * F, dtype=np.int64), lens)
    u = rng.random(bag.size)
    local = np.minimum((per_field * u ** 3).astype(np.int64), per_field - 1)   # skewed towards small ids
    ids = local + (bag % F) * per_field
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    vec = np.add.reduceat(U[bag % F, local % PLANT_TYPES] / lens[bag][:, None], starts).reshape(B, F, PLANT_DIM)
    s = vec.sum(1)
    pair = 0.5 * ((s * s).sum(1) - (vec * vec).sum((1, 2))) / np.sqrt(max(1, F * (F - 1) // 2) * PLANT_DIM)
    logit = DENSE_SCALE * planted_dense_term(cfg, dense) + PAIR_SCALE * pair
    labels = (rng.random(B) < 1 / (1 + np.exp(-logit))).astype(np.float32)
    dense_t, ids_t, y = torch.from_numpy(dense), torch.from_numpy(ids), torch.from_numpy(labels)
    if cfg.multi_hot:
        offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        return dense_t, ids_t, torch.from_numpy(offsets), y
    return dense_t, ids_t.view(B, F), y
