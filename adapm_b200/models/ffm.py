"""CTR prediction with a field-aware factorisation machine (FFM, as in libffm) on the parameter manager.

Every feature id is one key whose row holds one latent k-vector per field, ``[w, 0, 0, 0 | V_0 .. V_{F-1} | AdaGrad]``
(``ops.StoreFFM``). The model is all sparse: a step is the fused FFM step on a CUDA server (csrc/cuda/ops_ffm.cu) and
``ops.ffm_reference_step`` (the same rule in float64 through Pull / Push) on a CPU server.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import torch


@dataclass
class FFMConfig:
    num_features: int = 1_000_000       # total feature ids = PM keys, split evenly over the fields
    num_fields: int = 39
    k: int = 4                          # latent values per field
    eta: float = 0.2
    lam: float = 2e-5
    normalize: bool = True              # libffm's instance normalisation of one-hot data: pair_scale = 1 / num_fields
    batch_size: int = 8192
    read_ahead: int = 4
    model_seed: int = 1

    @property
    def row_values(self) -> int:        # [w, 0, 0, 0 | V_0 .. V_{F-1}]
        return 4 + self.num_fields * self.k

    @property
    def row_len(self) -> int:           # values | AdaGrad
        return 2 * self.row_values

    @property
    def pair_scale(self) -> float:
        return 1.0 / self.num_fields if self.normalize else 1.0


class FFM:
    def __init__(self, server, worker, cfg: FFMConfig, pair_scale: float | None = None):
        """``pair_scale`` overrides ``cfg.pair_scale`` (0: the linear model ``sum_f w``, a baseline)."""
        from ..ops import _check_ffm_rates, _check_ffm_shape

        _check_ffm_shape(cfg.num_fields, cfg.k, getattr(server, "_uniform_len", None))
        _check_ffm_rates(cfg.eta, cfg.lam)
        self.server, self.worker, self.cfg = server, worker, cfg
        self.pair_scale = cfg.pair_scale if pair_scale is None else float(pair_scale)
        self.dev = server.device
        self.op = None
        if server.backend == "cuda":
            from ..ops import StoreFFM

            self.op = StoreFFM(server, cfg.num_fields, cfg.k, cfg.eta, cfg.lam, self.pair_scale)
        self.step_no = 0

    def init_model(self, chunk: int = 1 << 18) -> None:
        """libffm's initialisation: ``V ~ U[0, 1 / sqrt(k)]``, ``w = 0``, accumulators 1; every rank initialises the
        keys it is home for."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        E = cfg.row_values
        gen = torch.Generator(device=self.dev.type).manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        keys = torch.arange(rank, cfg.num_features, world, dtype=torch.int64)
        for i in range(0, keys.numel(), chunk):
            kk = keys[i:i + chunk].to(self.dev)
            rows = torch.zeros(kk.numel(), cfg.row_len, device=self.dev, dtype=self.server.dtype)
            rows[:, 4:E] = torch.rand(kk.numel(), E - 4, generator=gen, device=self.dev,
                                      dtype=self.server.dtype) / cfg.k ** 0.5
            rows[:, E:] = 1.0
            self.worker.set(kk, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    def signal_intent(self, feat_ids: torch.Tensor, clock: int) -> None:
        if self.server.num_servers() > 1:
            self.worker.intent(feat_ids.reshape(-1), clock, clock + 1)

    def step(self, feat_ids: torch.Tensor, labels: torch.Tensor, return_tensor: bool = False):
        """feat_ids [B, F] int64 (global feature ids), labels [B] float in [0, 1]. Returns the mean loss of the batch (a
        float, or a device tensor with ``return_tensor`` on a CUDA server - no host synchronisation then)."""
        B = feat_ids.shape[0]
        self.step_no += 1
        if self.op is not None:
            ids = feat_ids.to(self.dev, non_blocking=True).contiguous()
            y = labels.to(self.dev, non_blocking=True).float().contiguous()
            loss = self.op.step(ids, y)[0] / max(B, 1)
            return loss if return_tensor else float(loss)
        from ..ops import ffm_reference_step

        cfg = self.cfg
        loss = ffm_reference_step(self.worker, feat_ids, labels.float(), cfg.k, cfg.eta, cfg.lam, self.pair_scale)
        return loss / max(B, 1)

    def predict(self, feat_ids: torch.Tensor) -> torch.Tensor:
        """Click probabilities sigmoid(phi) [B] (float32 on the store's device, float64 on the CPU)."""
        if self.op is not None:
            return torch.sigmoid(self.op.forward(feat_ids.to(self.dev).contiguous()))
        from ..ops import ffm_reference_forward

        return torch.sigmoid(ffm_reference_forward(self.worker, feat_ids, self.cfg.k, self.pair_scale))

    def evaluate(self, batches) -> tuple[float, float]:
        """(logloss, AUC) of the model over ``batches`` of (feat_ids, labels); the AUC counts ties as half."""
        ps, ys = [], []
        for ids, y in batches:
            ps.append(self.predict(ids).double().cpu())
            ys.append(y.double().cpu())
        return logloss_auc(torch.cat(ps).numpy(), torch.cat(ys).numpy())


def logloss_auc(p: np.ndarray, y: np.ndarray) -> tuple[float, float]:
    """Mean log loss of probabilities ``p`` (clipped to [1e-15, 1 - 1e-15]) against labels ``y`` in {0, 1}, and the
    AUC: the share of (positive, negative) pairs whose positive scores higher, ties counted as half (NaN without
    both classes). The AUC is computed from the mean ranks of tied scores."""
    p = np.asarray(p, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    q = np.clip(p, 1e-15, 1 - 1e-15)
    ll = float(-(y * np.log(q) + (1 - y) * np.log(1 - q)).mean()) if p.size else float("nan")
    pos = y > 0.5
    n_pos, n_neg = int(pos.sum()), int((~pos).sum())
    if n_pos == 0 or n_neg == 0:
        return ll, float("nan")
    _, inv, cnt = np.unique(p, return_inverse=True, return_counts=True)
    first = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    mean_rank = first + (cnt + 1) / 2.0                  # 1-based ranks, ties share their mean rank
    r = mean_rank[inv]
    auc = (r[pos].sum() - n_pos * (n_pos + 1) / 2.0) / (n_pos * n_neg)
    return ll, float(auc)


PLANT_TYPES = 16        # planted latent vectors per (field, partner field): a feature's type is its local id mod 16
PLANT_DIM = 4


@functools.lru_cache(maxsize=4)
def _planted(num_fields: int, num_features: int, seed: int) -> np.ndarray:
    """The planted field-aware model T [F, types, F, d]: feature type t of field f meets partner field f2 with T[f, t,
    f2]. For every field f and partner f2, T[f, :, f2] has zero mean under the distribution of f's types, so that a
    feature's mean contribution over its partners is 0: the signal is in the field interactions, which a linear model
    cannot see."""
    F, M, d = num_fields, PLANT_TYPES, PLANT_DIM
    rng = np.random.default_rng([seed, 0x5eed])
    T = rng.standard_normal((F, M, F, d))
    per_field = num_features // F
    ids = np.arange(per_field)
    p_id = ((ids + 1) / per_field) ** (1 / 3) - (ids / per_field) ** (1 / 3)   # P(local id) under the u^3 skew
    p_type = np.bincount(ids % M, weights=p_id, minlength=M)
    T -= np.einsum("m,fmgd->fgd", p_type, T)[:, None]
    return T


def synthetic_ffm_batch(cfg: FFMConfig, step: int, rank: int = 0, held_out: bool = False):
    """CTR batch of one id per field: ``(ids int64 [B, F], labels float32 [B])``. Ids are skewed within each field's
    range as in ``deepfm.synthetic_ctr_batch``; labels are drawn from sigmoid of a planted, zero-mean, field-aware
    pair score (:func:`_planted`), scaled to unit variance. ``held_out`` batches use their own seeds."""
    rng = np.random.default_rng([cfg.model_seed, rank, step, 1 if held_out else 0, 0xff])
    B, F = cfg.batch_size, cfg.num_fields
    per_field = cfg.num_features // F
    u = rng.random((B, F))
    local = np.minimum((per_field * u ** 3).astype(np.int64), per_field - 1)   # skewed towards small ids
    ids = local + np.arange(F, dtype=np.int64) * per_field
    T = _planted(F, cfg.num_features, cfg.model_seed)
    t = local % PLANT_TYPES
    score = np.zeros(B)
    for f1 in range(F - 1):                  # sum_{f1<f2} <T[f1, t_f1, f2], T[f2, t_f2, f1]>
        a = T[f1, t[:, f1], f1 + 1:]                                         # [B, F - f1 - 1, d]
        b = T[np.arange(f1 + 1, F)[None, :], t[:, f1 + 1:], f1]              # [B, F - f1 - 1, d]
        score += (a * b).sum((1, 2))
    score /= np.sqrt(F * (F - 1) / 2 * PLANT_DIM)
    labels = (rng.random(B) < 1 / (1 + np.exp(-3 * score))).astype(np.float32)
    return torch.from_numpy(ids), torch.from_numpy(labels)
