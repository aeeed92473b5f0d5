"""CTR prediction with DeepFM on the parameter manager (BASELINE config #5).

The reference repository has no CTR model (README.md:23 points to a separate repo); this model is written
against the bindings-style API (``Worker.pull / push / intent / advance_clock``), like a user of the
reference's PyTorch bindings would:

* the sparse part - one row per feature id, ``[w(1) | v(k) | AdaGrad(1+k)]`` - lives in the parameter
  manager (up to 100M keys, sharded over the GPUs' HBM, relocated/replicated by intent);
* per batch: ``intent`` for a future batch, ``pull`` the rows of the batch's feature ids (device path:
  fused gather kernel, NVLink loads for remote rows), DeepFM forward/backward in PyTorch, worker-side
  AdaGrad, ``push`` the additive updates (device path: REDs into the owners' rows);
* the dense MLP is replicated; its gradients are all-reduced with ``torch.distributed`` when available.
  On a CUDA server the MLP's linear layers can run on the hand-written wgmma GEMM
  (``ops.gemm_nt_bf16``; ``precision='fp8'`` uses the e4m3 tensor-core path with per-tensor scales).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
import torch.nn as nn


@dataclass
class DeepFMConfig:
    num_features: int = 100_000_000     # total feature ids = PM keys
    num_fields: int = 26
    embed_dim: int = 16
    hidden: tuple = (400, 400, 400)
    lr_sparse: float = 0.05
    lr_dense: float = 1e-3
    batch_size: int = 8192
    read_ahead: int = 4
    precision: str = "bf16"             # bf16 | fp8 | fp32 (dense GEMMs)
    table_precision: str = "fp32"       # fp32 | fp8_block: the model sees the embedding values a block-scaled e4m3 table
                                        # (UE8M0 scale per 32 values, utils/blockscale.py) would deliver; the parameter
                                        # manager keeps fp32 master rows (deltas and AdaGrad accumulate in fp32)
    model_seed: int = 1

    @property
    def emb_len(self) -> int:           # [w | v] padded to a multiple of 4 floats (16-byte vector row accesses)
        return (1 + self.embed_dim + 3) // 4 * 4

    @property
    def row_len(self) -> int:           # [w | v | pad | acc_w | acc_v | pad]
        return 2 * self.emb_len


class TensorCoreLinear(torch.autograd.Function):
    """y = x @ W^T on the hand-written wgmma GEMM (bf16 or fp8 operands, fp32 accumulate)."""

    @staticmethod
    def forward(ctx, x, w, precision):
        from ..ops import gemm_nt_bf16, gemm_nt_fp8

        ctx.save_for_backward(x, w)
        ctx.precision = precision
        return gemm_nt_fp8(x, w) if precision == "fp8" else gemm_nt_bf16(x, w)

    @staticmethod
    def backward(ctx, gy):
        from ..ops import gemm_nt_bf16

        x, w = ctx.saved_tensors
        gx = gemm_nt_bf16(gy, w.t().contiguous())                   # [B,out] x [in,out]^T
        gw = gemm_nt_bf16(gy.t().contiguous(), x.t().contiguous())  # [out,B] x [in,B]^T
        return gx, gw, None


class DenseNet(nn.Module):
    def __init__(self, cfg: DeepFMConfig, use_tensor_cores: bool):
        super().__init__()
        dims = [cfg.num_fields * cfg.embed_dim] + list(cfg.hidden) + [1]
        g = torch.Generator().manual_seed(cfg.model_seed)
        self.w = nn.ParameterList([nn.Parameter(torch.randn(dims[i + 1], dims[i], generator=g) * (2.0 / dims[i]) ** 0.5)
                                   for i in range(len(dims) - 1)])
        self.b = nn.ParameterList([nn.Parameter(torch.zeros(dims[i + 1])) for i in range(len(dims) - 1)])
        self.tc, self.precision = use_tensor_cores, cfg.precision

    def forward(self, x):
        for i, (w, b) in enumerate(zip(self.w, self.b)):
            last = i == len(self.w) - 1
            if self.tc and not last and self.precision != "fp32":
                x = TensorCoreLinear.apply(x, w, self.precision) + b
            else:
                x = x @ w.t() + b
            if not last:
                x = torch.relu(x)
        return x.view(-1)


class DeepFM:
    def __init__(self, server, worker, cfg: DeepFMConfig):
        self.server, self.worker, self.cfg = server, worker, cfg
        self.cuda = server.backend == "cuda"
        self.dev = server.device
        self.net = DenseNet(cfg, use_tensor_cores=self.cuda).to(self.dev)
        self.opt = torch.optim.Adam(self.net.parameters(), lr=cfg.lr_dense)
        self.step_no = 0
        self.rows_pushed = 0      # (key,row) updates applied so far (distinct feature rows per batch)

    def init_model(self, chunk: int = 1 << 18) -> None:
        """v ~ N(0, 0.01), w = 0, accumulators 1e-6; every rank initialises the keys it is home for."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        k = cfg.embed_dim
        gen = torch.Generator(device=self.dev.type).manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        keys = torch.arange(rank, cfg.num_features, world, dtype=torch.int64)
        for i in range(0, keys.numel(), chunk):
            kk = keys[i:i + chunk].to(self.dev)
            rows = torch.zeros(kk.numel(), cfg.row_len, device=self.dev)
            rows[:, 1:1 + k] = torch.randn(kk.numel(), k, generator=gen, device=self.dev) * 0.01
            rows[:, cfg.emb_len:] = 1e-6
            self.worker.set(kk, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()

    def signal_intent(self, feat_ids: torch.Tensor, clock: int) -> None:
        if self.server.num_servers() > 1:
            self.worker.intent(feat_ids.reshape(-1), clock, clock + 1)

    def step(self, feat_ids: torch.Tensor, labels: torch.Tensor, return_tensor: bool = False):
        """feat_ids [B, F] int64 (global feature ids), labels [B] float (CPU / pinned / device tensors). Returns the
        batch loss (a float, or the device tensor with ``return_tensor`` - no host synchronisation then)."""
        cfg, kv = self.cfg, self.worker
        B, F, k = feat_ids.shape[0], cfg.num_fields, cfg.embed_dim
        ids = feat_ids.to(self.dev, non_blocking=True).reshape(-1).contiguous()
        y = labels.to(self.dev, non_blocking=True).float()
        uniq, inv = torch.unique(ids, return_inverse=True)
        rows = torch.empty(uniq.numel() * cfg.row_len, dtype=torch.float32, device=self.dev)
        kv.wait(kv.pull(uniq, rows, True))
        rows = rows.view(-1, cfg.row_len)
        el = cfg.emb_len
        emb = rows[:, :el].detach().clone().requires_grad_(True)      # [U, el]  (w | v | pad)
        acc = rows[:, el:]
        if cfg.table_precision == "fp8_block":
            from ..utils.blockscale import FakeQuantSTE

            e = FakeQuantSTE.apply(emb)[inv].view(B, F, el)           # straight-through: gradients reach the fp32 masters
        else:
            e = emb[inv].view(B, F, el)
        w1, v = e[:, :, 0], e[:, :, 1:1 + k]
        fm = w1.sum(1) + 0.5 * ((v.sum(1) ** 2) - (v ** 2).sum(1)).sum(1)
        logit = fm + self.net(v.reshape(B, F * k))
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logit, y)
        self.opt.zero_grad(set_to_none=True)
        loss.backward()
        if torch.distributed.is_available() and torch.distributed.is_initialized() and self.server.num_servers() > 1:
            for p in self.net.parameters():
                torch.distributed.all_reduce(p.grad)
                p.grad /= self.server.num_servers()
        self.opt.step()
        g = emb.grad * B                                             # sum over examples, like per-example SGD
        upd = torch.cat([-cfg.lr_sparse * g / torch.sqrt(acc + g * g), g * g], 1).contiguous()
        kv.push(uniq, upd.view(-1), True)
        self.step_no += 1
        self.rows_pushed += int(uniq.numel())
        return loss.detach() if return_tensor else float(loss.detach())


def synthetic_ctr_batch(cfg: DeepFMConfig, step: int, rank: int = 0):
    """Criteo-shaped synthetic batch: one id per field, ids Zipf-skewed within each field's range; the label
    depends on a hidden linear model so that training has signal."""
    rng = np.random.default_rng([cfg.model_seed, rank, step])
    per_field = cfg.num_features // cfg.num_fields
    u = rng.random((cfg.batch_size, cfg.num_fields))
    local = np.minimum((per_field * u ** 3).astype(np.int64), per_field - 1)   # skewed towards small ids
    ids = local + np.arange(cfg.num_fields, dtype=np.int64) * per_field
    score = (((local % 7) - 3) * (1.0 / cfg.num_fields)).sum(1)
    labels = (rng.random(cfg.batch_size) < 1 / (1 + np.exp(-3 * score))).astype(np.float32)
    return torch.from_numpy(ids), torch.from_numpy(labels)
