"""Matrix factorisation (DSGD / columnwise / plain SGD + AdaGrad, bold driver) on the parameter manager.

Behavioural parity with the reference application ``apps/matrix_factorization.cc`` + ``apps/mf/*.h``:

* keys: row factors ``0..m-1``, column factors from ``first_col_key`` (rows rounded up to the number of
  workers) (mf.cc:89-94,693); row = ``[factors(rank) | AdaGrad(rank)]`` (mf.cc:697);
* update rule UpdateNsqlL2Adagrad (apps/mf/update.h:32-70), 2 updates per non-zero;
* schedules: **dsgd** (W x W blocks, one sub-epoch per block column with a barrier and a per-block column
  intent, mf.cc:409-458, WOR block schedule apps/mf/data.h:182-210), **columnwise** (look-ahead intent on the
  next columns, mf.cc:459-522) and **plain** SGD (point look-ahead, mf.cc:523-579); row intents for the whole
  run (mf.cc:369-372);
* bold driver step-size control (mf.cc:593-605); loss = sum (x - w.h)^2 + lambda (|W|^2 + |H|^2)
  (apps/mf/loss.h:49-78); factors read/written as MatrixMarket array text ``W.mma / H.mma``
  (apps/mf/io.h:265-352).

The per-non-zero loop of the reference is one fused kernel over a batch of non-zeros (``ops.mf_step``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import CLOCK_MAX


@dataclass
class MFConfig:
    num_rows: int = 10_000_000
    num_cols: int = 1_000_000
    rank: int = 128
    algorithm: str = "dsgd"          # dsgd | columnwise | plain
    eps: float = 0.01                # initial step size
    lam: float = 0.05
    batch_nnz: int = 1 << 18
    signal_intent_cols: int = 1000   # columns of look-ahead (columnwise) / 0 = no column intent
    read_ahead: int = 4
    bold_driver: bool = True
    eps_inc: float = 1.05
    eps_dec: float = 0.5
    model_seed: int = 134827
    signal_intent_rows: bool = True  # localise this rank's row block for the whole run (mf.cc:640)
    wor_blocks: bool = True          # WOR schedule for the DSGD blocks (else the fixed rotation (rank + sub-epoch) % W)
    wor_points: bool = True          # WOR schedule for the data points within a block / epoch (else file order)
    early_stop: int = 0              # stop an epoch after N data points (debugging)
    deterministic: bool = False      # one GPU: start-of-step reads, bit-identical runs (ops.mf_step); the CPU backend
                                     # accepts it and already follows the start-of-step rule

    def first_col_key(self, num_workers: int) -> int:
        return ((self.num_rows + num_workers - 1) // num_workers) * num_workers

    def num_keys(self, num_workers: int) -> int:
        return self.first_col_key(num_workers) + self.num_cols

    @property
    def row_len(self) -> int:
        return 2 * self.rank


class SparseMatrix:
    """COO non-zeros of this rank's row block, grouped by column block (the DSGD stratification)."""

    def __init__(self, i: np.ndarray, j: np.ndarray, x: np.ndarray, num_rows: int, num_cols: int, world: int, rank: int):
        self.num_rows, self.num_cols, self.world, self.rank = num_rows, num_cols, world, rank
        self.row_nnz_all = np.bincount(i, minlength=num_rows).astype(np.int32)
        self.col_nnz_all = np.bincount(j, minlength=num_cols).astype(np.int32)
        self.rows_per_block = (num_rows + world - 1) // world
        self.cols_per_block = (num_cols + world - 1) // world
        mine = (i // self.rows_per_block) == rank                       # row partitioning (apps/mf/io.h:163-175)
        self.i, self.j, self.x = i[mine], j[mine], x[mine].astype(np.float32)
        blk = self.j // self.cols_per_block
        order = np.argsort(blk, kind="stable")
        self.i, self.j, self.x, blk = self.i[order], self.j[order], self.x[order], blk[order]
        self.block_start = np.searchsorted(blk, np.arange(world))
        self.block_end = np.searchsorted(blk, np.arange(world), side="right")

    @staticmethod
    def synthetic(num_rows: int, num_cols: int, nnz: int, rank_true: int, world: int, rank: int, seed: int = 0):
        rng = np.random.default_rng(seed)
        i = rng.integers(0, num_rows, nnz)
        j = rng.integers(0, num_cols, nnz)
        w = np.random.default_rng(seed + 1).standard_normal((min(num_rows, 4096), rank_true)).astype(np.float32)
        h = np.random.default_rng(seed + 2).standard_normal((min(num_cols, 4096), rank_true)).astype(np.float32)
        x = (w[i % w.shape[0]] * h[j % h.shape[0]]).sum(1) / np.sqrt(rank_true) + 0.01 * rng.standard_normal(nnz)
        return SparseMatrix(i, j, x.astype(np.float32), num_rows, num_cols, world, rank)

    def block(self, b: int):
        s, e = self.block_start[b], self.block_end[b]
        return self.i[s:e], self.j[s:e], self.x[s:e]


from ..parallel.schedules import column_intent_plan, wor_block_schedule  # noqa: E402,F401  (re-exported: tests, docs)


class MatrixFactorization:
    def __init__(self, server, worker, cfg: MFConfig, data: SparseMatrix):
        self.server, self.worker, self.cfg, self.data = server, worker, cfg, data
        # the fused kernel is float32; float64 rows (the reference's ValT = double) train through Pull / Push with the same
        # update rule (mf_reference_step) on either backend
        self.cuda = server.backend == "cuda" and server.dtype == torch.float32
        self.dtype = server.dtype
        self.world = server.num_servers()
        self.fck = cfg.first_col_key(self.world)
        self.eps = cfg.eps
        self.step_no = 0
        dev = server.device
        if self.cuda:
            self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
            self.stats = torch.zeros(4, dtype=torch.int64, device=dev)

    def row_key(self, i):
        return i

    def col_key(self, j):
        return j + self.fck

    def init_model(self, chunk: int = 1 << 16) -> None:
        cfg, world, rank = self.cfg, self.world, self.server.my_rank()
        gen = torch.Generator().manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        nk = cfg.num_keys(world)
        keys = torch.arange(rank, nk, world, dtype=torch.int64)
        keys = keys[(keys < cfg.num_rows) | (keys >= self.fck)]
        for s in range(0, keys.numel(), chunk):
            k = keys[s:s + chunk]
            rows = torch.empty(k.numel(), 2 * cfg.rank, dtype=self.dtype)
            rows[:, :cfg.rank] = (torch.rand(k.numel(), cfg.rank, generator=gen) / np.sqrt(cfg.rank)).to(self.dtype)
            rows[:, cfg.rank:] = 0.0
            if self.cuda:
                self.worker.set(k.to(self.server.device), rows.to(self.server.device).view(-1))
            else:
                self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()
        if world > 1 and cfg.signal_intent_rows:  # row intents for the whole run (mf.cc:369-372)
            lo = rank * self.data.rows_per_block
            hi = min(cfg.num_rows, lo + self.data.rows_per_block)
            self.worker.intent(torch.arange(lo, hi), 0, CLOCK_MAX)

    # one batch of non-zeros (numpy views of this rank's data)
    def step(self, i: np.ndarray, j: np.ndarray, x: np.ndarray) -> torch.Tensor:
        cfg = self.cfg
        rn = self.data.row_nnz_all[i]
        cn = self.data.col_nnz_all[j]
        if self.cuda:
            from ..ops import mf_step

            dev = self.server.device
            rk = torch.from_numpy(np.ascontiguousarray(i)).to(dev, non_blocking=True)
            ck = (torch.from_numpy(np.ascontiguousarray(j)) + self.fck).to(dev, non_blocking=True)
            mf_step(self.server, rk, ck, torch.from_numpy(np.ascontiguousarray(x)).to(dev, non_blocking=True),
                    torch.from_numpy(rn).to(dev, non_blocking=True), torch.from_numpy(cn).to(dev, non_blocking=True),
                    cfg.rank, self.eps, cfg.lam, self.loss, self.stats, deterministic=cfg.deterministic)
            self.step_no += 1
            return self.loss
        loss = mf_reference_step(self.worker, torch.from_numpy(i.astype(np.int64)),
                                 torch.from_numpy(j.astype(np.int64)) + self.fck, torch.from_numpy(x),
                                 torch.from_numpy(rn), torch.from_numpy(cn), cfg.rank, self.eps, cfg.lam)
        self.step_no += 1
        return torch.tensor([loss], dtype=torch.float32)

    def run_epoch(self, epoch: int) -> float:
        """One epoch with the configured schedule. Returns this rank's summed squared error."""
        cfg, kv, data, W = self.cfg, self.worker, self.data, self.world
        total = 0.0
        if self.cuda:
            self.loss.zero_()
        if cfg.algorithm == "dsgd":
            sched = (wor_block_schedule(W, epoch, cfg.model_seed) if cfg.wor_blocks
                     else np.array([[(r + se) % W for r in range(W)] for se in range(W)]))
            for se in range(W):
                b = int(sched[se, self.server.my_rank()])
                if cfg.signal_intent_cols != 0 and W > 1:
                    lo = b * data.cols_per_block
                    hi = min(cfg.num_cols, lo + data.cols_per_block)
                    kv.intent(torch.arange(lo, hi) + self.fck, kv.current_clock())
                    kv.wait_sync()
                i, j, x = data.block(b)
                perm = (np.random.default_rng(epoch * 131 + se).permutation(i.shape[0]) if cfg.wor_points
                        else np.arange(i.shape[0]))                                      # WOR point schedule
                if cfg.early_stop:
                    perm = perm[: cfg.early_stop]
                for s in range(0, perm.shape[0], cfg.batch_nnz):
                    p = perm[s:s + cfg.batch_nnz]
                    out = self.step(i[p], j[p], x[p])
                    if not self.cuda:
                        total += float(out)
                kv.advance_clock()
                kv.barrier()
        else:
            n = data.i.shape[0]
            if cfg.algorithm == "columnwise":
                order = np.argsort(data.j, kind="stable")
            else:
                order = np.random.default_rng(epoch).permutation(n) if cfg.wor_points else np.arange(n)
            if cfg.early_stop:
                order = order[: cfg.early_stop]
                n = order.shape[0]
            starts = list(range(0, n, cfg.batch_nnz))
            col_plan = None
            if cfg.algorithm == "columnwise" and W > 1:
                # Ranged intents like the reference's column-wise schedule (mf.cc:477-482: one Intent per column for the
                # clocks during which the column's data points are processed): the points are sorted by column, so a
                # column occupies a contiguous run of batches [first, last]; it is signalled ONCE, read_ahead batches before
                # its first one, for last - first + 1 clocks - not again in every batch it spans.
                col_plan = column_intent_plan(data.j[order], cfg.batch_nnz)
            for bi, s in enumerate(starts):
                fut = bi + cfg.read_ahead
                if W > 1 and fut < len(starts):
                    if col_plan is not None:
                        cols, dur, ptr = col_plan
                        lo, hi = int(ptr[fut]), int(ptr[fut + 1])
                        if hi > lo:
                            start = kv.current_clock() + cfg.read_ahead
                            for dd in np.unique(dur[lo:hi]):               # (almost always a single duration: 1 batch)
                                sel = cols[lo:hi][dur[lo:hi] == dd]
                                kv.intent(torch.from_numpy(sel.astype(np.int64)) + self.fck, start, start + int(dd))
                    else:
                        p = order[starts[fut]:starts[fut] + cfg.batch_nnz]
                        kv.intent(torch.from_numpy(np.unique(data.j[p])) + self.fck, kv.current_clock() + cfg.read_ahead)
                p = order[s:s + cfg.batch_nnz]
                out = self.step(data.i[p], data.j[p], data.x[p])
                if not self.cuda:
                    total += float(out)
                kv.advance_clock()
        if self.cuda:
            total = float(self.loss.item())
        return total

    def load_factors(self, w_path: str, h_path: str, chunk: int = 1 << 16) -> None:
        """``init_parameters=1``: initial factors from MatrixMarket array files W (rows x rank) and H (rank x cols);
        AdaGrad accumulators start at zero. Collective: every rank sets the keys it is home for."""
        from ..utils.mmio import read_matrix_market_array

        cfg, world, rank = self.cfg, self.world, self.server.my_rank()
        Wm = torch.from_numpy(read_matrix_market_array(w_path)).to(self.dtype)
        Hm = torch.from_numpy(read_matrix_market_array(h_path)).to(self.dtype).t().contiguous()
        assert Wm.shape == (cfg.num_rows, cfg.rank) and Hm.shape == (cfg.num_cols, cfg.rank), (Wm.shape, Hm.shape)
        self.worker.begin_setup()
        for first, M in ((0, Wm), (self.fck, Hm)):
            keys = torch.arange(M.shape[0], dtype=torch.int64) + first
            sel = (keys % world) == rank
            keys, vals = keys[sel], M[sel]
            for s in range(0, keys.numel(), chunk):
                rows = torch.zeros(min(chunk, keys.numel() - s), 2 * cfg.rank, dtype=self.dtype)
                rows[:, :cfg.rank] = vals[s:s + chunk]
                self.worker.wait(self.worker.set(keys[s:s + chunk], rows.view(-1)))
        self.worker.waitall()
        self.worker.end_setup()

    def evaluate(self, i: np.ndarray, j: np.ndarray, x: np.ndarray) -> float:
        """Summed squared error of the current factors on arbitrary entries (test set), through Pull."""
        cfg, kv = self.cfg, self.worker
        total = 0.0
        for s in range(0, len(x), 1 << 16):
            ri = torch.from_numpy(np.ascontiguousarray(i[s:s + (1 << 16)])).long()
            cj = torch.from_numpy(np.ascontiguousarray(j[s:s + (1 << 16)])).long()
            wv = torch.empty(ri.numel() * 2 * cfg.rank, dtype=self.dtype)
            kv.wait(kv.pull(self.row_key(ri), wv))
            hv = torch.empty(cj.numel() * 2 * cfg.rank, dtype=self.dtype)
            kv.wait(kv.pull(self.col_key(cj), hv))
            pred = (wv.view(-1, 2 * cfg.rank)[:, :cfg.rank] * hv.view(-1, 2 * cfg.rank)[:, :cfg.rank]).sum(1)
            total += float(((torch.from_numpy(np.ascontiguousarray(x[s:s + (1 << 16)])).to(self.dtype) - pred) ** 2).sum())
        return total

    def bold_driver(self, loss: float, prev_loss: Optional[float]) -> None:
        if not self.cfg.bold_driver or prev_loss is None:
            return
        self.eps *= self.cfg.eps_inc if loss < prev_loss else self.cfg.eps_dec

    def pull_factors(self):
        cfg, kv = self.cfg, self.worker
        wv = torch.empty(cfg.num_rows * 2 * cfg.rank, dtype=self.dtype)
        kv.wait(kv.pull(torch.arange(cfg.num_rows), wv))
        hv = torch.empty(cfg.num_cols * 2 * cfg.rank, dtype=self.dtype)
        kv.wait(kv.pull(torch.arange(cfg.num_cols) + self.fck, hv))
        return wv.view(-1, 2 * cfg.rank)[:, :cfg.rank], hv.view(-1, 2 * cfg.rank)[:, :cfg.rank]

    def write_factors(self, prefix: str) -> None:
        """MatrixMarket array text W.mma / H.mma (apps/mf/io.h:265-352)."""
        self.worker.wait_sync()
        if self.server.my_rank() != 0:
            return
        Wm, Hm = self.pull_factors()
        for name, M in (("W", Wm), ("H", Hm.t())):
            with open(f"{prefix}{name}.mma", "w") as f:
                f.write("%%MatrixMarket matrix array real general\n")
                f.write(f"{M.shape[0]} {M.shape[1]}\n")
                np.savetxt(f, M.t().contiguous().numpy().reshape(-1), fmt="%.9g")  # column-major


def mf_reference_step(kv, rk, ck, x, rn, cn, rank: int, eps: float, lam: float) -> float:
    n = rk.numel()
    dt = kv.server.dtype          # float32, or float64 like the reference's ValT
    wv = torch.empty(n * 2 * rank, dtype=dt)
    hv = torch.empty(n * 2 * rank, dtype=dt)
    kv.wait(kv.pull(rk.contiguous(), wv))
    kv.wait(kv.pull(ck.contiguous(), hv))
    wv, hv = wv.view(n, 2 * rank), hv.view(n, 2 * rank)
    w, aw, h, ah = wv[:, :rank], wv[:, rank:], hv[:, :rank], hv[:, rank:]
    e = x.to(dt) - (w * h).sum(1)
    f1 = (-2 * e).view(-1, 1)
    f2 = 2 * lam
    gw = -(f1 * h + f2 * w / rn.clamp(min=1).view(-1, 1))
    gh = -(f1 * w + f2 * h / cn.clamp(min=1).view(-1, 1))
    uw = torch.cat([eps * gw / torch.sqrt(aw + gw * gw + 1e-6), gw * gw], 1)
    uh = torch.cat([eps * gh / torch.sqrt(ah + gh * gh + 1e-6), gh * gh], 1)
    kv.wait(kv.push(rk.contiguous(), uw.contiguous().view(-1)))
    kv.wait(kv.push(ck.contiguous(), uh.contiguous().view(-1)))
    return float((e * e).sum())
