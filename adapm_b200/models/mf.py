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

Implicit feedback (``MFConfig.loss = "bpr"``, an addition of this implementation): every entry is an interaction, trained
with the BPR pairwise loss against sampled negative items in one fused kernel (``ops.mf_bpr_step``) on the same rows and
schedules; ``recommend`` ranks the items of a user with the seen ones left out, ``evaluate_ranking`` gives Recall@k and
NDCG@k.

Alternating least squares (``MFConfig.algorithm = "als"``, also an addition): each half-step solves every row of one
side exactly for the other side held fixed, one fused gather + Cholesky kernel per row (``ops.als_solve``). With
``loss = "squared"`` it minimises the objective above; with ``loss = "implicit"`` the Hu-Koren-Volinsky objective
``sum_{u,i} c_ui (p_ui - w_u.h_i)^2 + lambda (|W|^2 + |H|^2)`` over all pairs (``c = 1 + alpha x`` and ``p = 1`` on the
entries, ``c = 1`` and ``p = 0`` elsewhere) through the Gram matrix of the other side (``ops.als_gram``).
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
    algorithm: str = "dsgd"          # dsgd | columnwise | plain | als
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
    loss: str = "squared"            # squared (explicit ratings) | bpr (implicit feedback: every entry is an interaction)
                                     # | implicit (als only: the Hu-Koren-Volinsky weighted loss over all pairs)
    num_negatives: int = 1           # bpr: sampled negative items per positive
    sampling_scheme: str = "local"   # bpr on several ranks outside dsgd: "local" draws only resident items
    alpha: float = 1.0               # implicit: confidence c = 1 + alpha x of an entry with value x

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
        cb = (j // self.cols_per_block) == rank                          # this rank's column block (als)
        self._col_entries = (i[cb], j[cb], x[cb].astype(np.float32))
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

    @staticmethod
    def synthetic_implicit(num_rows: int, num_cols: int, per_row: int, rank_true: int, world: int, rank: int,
                           seed: int = 0, holdout: float = 0.2):
        """Implicit feedback with planted structure: user u draws ``per_row`` distinct items with probability
        proportional to ``exp(<p_u, q_i> / tau + b_i)``, p and q standard normal of dimension ``rank_true`` and
        ``b_i = -0.7 log(1 + pi(i))`` a heavy-tailed popularity over a random item order pi. A ``holdout`` fraction of
        each user's items (at least one when holdout > 0) goes to the test set. Returns ``(train SparseMatrix, (test_i,
        test_j))``; the test set holds every user's items, on every rank."""
        per_row = int(min(per_row, num_cols))
        rng = np.random.default_rng(seed)
        tau = 0.5 * np.sqrt(rank_true)
        P = rng.standard_normal((num_rows, rank_true))
        Q = rng.standard_normal((num_cols, rank_true))
        b = -0.7 * np.log1p(rng.permutation(num_cols).astype(np.float64))
        n_test = 0 if holdout <= 0 else max(1, int(round(per_row * holdout)))
        n_test = min(n_test, per_row - 1)
        tr_i, tr_j, te_i, te_j = [], [], [], []
        for s in range(0, num_rows, 1024):
            logits = P[s:s + 1024] @ Q.T / tau + b
            gumbel = -np.log(-np.log(rng.random(logits.shape)))
            items = np.argpartition(-(logits + gumbel), per_row - 1, axis=1)[:, :per_row]   # a random draw order
            items = np.take_along_axis(items, rng.random(items.shape).argsort(1), 1)
            users = np.repeat(np.arange(s, s + items.shape[0]), per_row).reshape(items.shape)
            tr_i.append(users[:, n_test:].ravel()); tr_j.append(items[:, n_test:].ravel())
            te_i.append(users[:, :n_test].ravel()); te_j.append(items[:, :n_test].ravel())
        i, j = np.concatenate(tr_i), np.concatenate(tr_j)
        train = SparseMatrix(i, j, np.ones(i.shape[0], np.float32), num_rows, num_cols, world, rank)
        return train, (np.concatenate(te_i), np.concatenate(te_j))

    def block(self, b: int):
        s, e = self.block_start[b], self.block_end[b]
        return self.i[s:e], self.j[s:e], self.x[s:e]

    def row_block(self):
        """[lo, hi): the rows of this rank's block"""
        lo = self.rank * self.rows_per_block
        return lo, min(self.num_rows, lo + self.rows_per_block)

    def col_block(self):
        """[lo, hi): the columns of this rank's block"""
        lo = self.rank * self.cols_per_block
        return lo, min(self.num_cols, lo + self.cols_per_block)

    def als_csr(self, side: str):
        """The entries of this rank's row block by row (``side = "rows"``) or of its column block by column
        (``"cols"``), every row / column of the block included, ordered by descending entry count (ties to the smaller
        index; entries in file order): ``(targets, offsets [n + 1], others, x)``, numpy, with row and column indices."""
        if side == "rows":
            lo, hi = self.row_block()
            t, o, x = self.i.astype(np.int64), self.j.astype(np.int64), self.x
        else:
            lo, hi = self.col_block()
            t, o, x = (self._col_entries[1].astype(np.int64), self._col_entries[0].astype(np.int64),
                       self._col_entries[2])
        cnt = np.bincount(t - lo, minlength=hi - lo)
        targets = np.argsort(-cnt, kind="stable")
        rank_of = np.empty_like(targets)
        rank_of[targets] = np.arange(targets.shape[0])
        order = np.argsort(rank_of[t - lo], kind="stable")
        offsets = np.zeros(targets.shape[0] + 1, dtype=np.int64)
        np.cumsum(cnt[targets], out=offsets[1:])
        return targets + lo, offsets, o[order], x[order]

    def seen(self, rows):
        """Training items of ``rows`` (all in this rank's row block, else ``ValueError``) as a CSR ``(offsets int64
        [n + 1], items int64)`` with each row's items distinct and ascending: the ``exclude`` of a recommendation."""
        rows = np.asarray(rows, dtype=np.int64).reshape(-1)
        lo, hi = self.row_block()
        if rows.size and (rows.min() < lo or rows.max() >= hi):
            raise ValueError(f"rows must lie in this rank's row block [{lo}, {hi})")
        if not hasattr(self, "_seen"):
            pairs = np.unique((self.i.astype(np.int64) - lo) * self.num_cols + self.j)
            start = np.searchsorted(pairs, np.arange(hi - lo + 1, dtype=np.int64) * self.num_cols)
            self._seen = (start, pairs % self.num_cols)
        start, items = self._seen
        a, e = start[rows - lo], start[rows - lo + 1]
        off = np.zeros(rows.size + 1, dtype=np.int64)
        np.cumsum(e - a, out=off[1:])
        idx = np.repeat(a - off[:-1], e - a) + np.arange(off[-1])
        return torch.from_numpy(off), torch.from_numpy(items[idx].astype(np.int64))


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
        if cfg.loss not in ("squared", "bpr", "implicit"):
            raise ValueError(f"loss must be 'squared', 'bpr' or 'implicit', got {cfg.loss!r}")
        if cfg.algorithm == "als" and cfg.loss == "bpr":
            raise ValueError("algorithm 'als' takes loss 'squared' or 'implicit', not 'bpr'")
        if cfg.loss == "implicit" and cfg.algorithm != "als":
            raise ValueError(f"loss 'implicit' needs algorithm 'als', got {cfg.algorithm!r}")
        if cfg.algorithm == "als" and not (cfg.lam > 0 and cfg.alpha >= 0):
            raise ValueError(f"als needs lam > 0 and alpha >= 0, got lam {cfg.lam}, alpha {cfg.alpha}")
        if cfg.loss == "implicit" and ((data.x < 0).any() or (data._col_entries[2] < 0).any()):
            raise ValueError("loss 'implicit' needs entry values >= 0 (interaction strengths)")
        if cfg.loss == "bpr" and cfg.num_negatives < 1:
            raise ValueError(f"num_negatives must be >= 1, got {cfg.num_negatives}")
        self._neg_range = (0, cfg.num_cols)          # bpr: the items negatives are drawn from (set per sub-epoch)
        self._samplers = {}
        self._gen = torch.Generator().manual_seed(cfg.model_seed * 3 + server.my_rank())
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
        if world > 1 and cfg.algorithm == "als":      # the column block is written by this rank in every item half-step
            lo, hi = self.data.col_block()
            self.worker.intent(torch.arange(lo, hi) + self.fck, 0, CLOCK_MAX)

    # one batch of non-zeros (numpy views of this rank's data)
    def step(self, i: np.ndarray, j: np.ndarray, x: np.ndarray) -> torch.Tensor:
        cfg = self.cfg
        if cfg.loss == "bpr":
            return self.bpr_step(i, j)
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

    def bpr_step(self, i: np.ndarray, j: np.ndarray) -> torch.Tensor:
        """One batch of positives (user i[b], item j[b]) with ``num_negatives`` items each, drawn uniformly from the
        current negative range: the sub-epoch's column block under dsgd, all items otherwise (on several ranks with the
        ``local`` scheme only items resident on this GPU)."""
        cfg = self.cfg
        lo, num = self._neg_range
        B, n = i.shape[0], cfg.num_negatives
        if self.cuda:
            from ..ops import DeviceSampler, mf_bpr_step

            dev = self.server.device
            smp = self._samplers.get((lo, num))
            if smp is None:
                smp = self._samplers[(lo, num)] = DeviceSampler(self.server, distribution="uniform",
                                                                first_key=self.fck + lo, num_keys=num)
            local_only = cfg.algorithm != "dsgd" and cfg.sampling_scheme == "local" and self.world > 1
            seed = (cfg.model_seed * 7 + self.server.my_rank() * 7919 + self.step_no) & 0xFFFFFFFFFFFF
            neg = smp.sample(B * n, seed, local_only=local_only).view(B, n)
            uk = torch.from_numpy(np.ascontiguousarray(i, dtype=np.int64)).to(dev, non_blocking=True)
            ik = (torch.from_numpy(np.ascontiguousarray(j, dtype=np.int64)) + self.fck).to(dev, non_blocking=True)
            mf_bpr_step(self.server, uk, ik, neg, cfg.rank, self.eps, cfg.lam, self.loss, self.stats,
                        deterministic=cfg.deterministic)
            self.step_no += 1
            return self.loss
        from ..ops import bpr_reference_step

        neg = torch.randint(lo, lo + num, (B, n), generator=self._gen) + self.fck
        loss, _ = bpr_reference_step(self.worker, torch.from_numpy(i.astype(np.int64)),
                                     torch.from_numpy(j.astype(np.int64)) + self.fck, neg, cfg.rank, self.eps, cfg.lam)
        self.step_no += 1
        return torch.tensor([loss], dtype=torch.float32)

    def run_epoch(self, epoch: int) -> float:
        """One epoch with the configured schedule. Returns this rank's summed squared error."""
        cfg, kv, data, W = self.cfg, self.worker, self.data, self.world
        if cfg.algorithm == "als":
            return self.als_epoch()
        total = 0.0
        if self.cuda:
            self.loss.zero_()
        if cfg.algorithm == "dsgd":
            sched = (wor_block_schedule(W, epoch, cfg.model_seed) if cfg.wor_blocks
                     else np.array([[(r + se) % W for r in range(W)] for se in range(W)]))
            for se in range(W):
                b = int(sched[se, self.server.my_rank()])
                blo = b * data.cols_per_block
                self._neg_range = (blo, max(0, min(cfg.num_cols, blo + data.cols_per_block) - blo))
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
            self._neg_range = (0, cfg.num_cols)
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

    # ------------------------------------------------------------------------------------------ alternating least squares
    def _als_block(self, side: str):
        """(target keys, offsets, other keys, a, b) of this rank's row (``"rows"``) or column (``"cols"``) block, longest
        target first; built once, on the device on CUDA"""
        cache = self.__dict__.setdefault("_als_blocks", {})
        if side not in cache:
            cfg = self.cfg
            t, off, o, x = self.data.als_csr(side)
            if side == "rows":
                t, o = t, o + self.fck
            else:
                t, o = t + self.fck, o
            x = x.astype(np.float64)
            if cfg.loss == "implicit":
                a, b = cfg.alpha * x, 1.0 + cfg.alpha * x
            else:
                a, b = np.ones_like(x), x
            blk = [torch.from_numpy(np.ascontiguousarray(v)) for v in (t, off, o)]
            blk += [torch.from_numpy(a.astype(np.float32)), torch.from_numpy(b.astype(np.float32))]
            if self.cuda:
                blk = [v.to(self.server.device) for v in blk]
            cache[side] = blk
        return cache[side]

    def _other_keys(self, side: str) -> torch.Tensor:
        """all keys of the side that the targets of ``side`` read (items for the row block, users for the column block)"""
        cfg = self.cfg
        keys = (torch.arange(cfg.num_cols, dtype=torch.int64) + self.fck if side == "rows"
                else torch.arange(cfg.num_rows, dtype=torch.int64))
        return keys.to(self.server.device) if self.cuda else keys

    def als_half_step(self, side: str) -> None:
        """Solve every row of this rank's row block (``side = "rows"``) or column block (``"cols"``) for the other side
        held fixed; collective (ends with a barrier)."""
        cfg, kv = self.cfg, self.worker
        t, off, o, a, b = self._als_block(side)
        implicit = cfg.loss == "implicit"
        if self.cuda:
            from ..ops import als_gram, als_solve

            gram = als_gram(self.server, self._other_keys(side), cfg.rank) if implicit else None
            als_solve(self.server, t, off, o, a, b, cfg.rank, cfg.lam, gram, self.stats)
            torch.cuda.current_stream(self.server.device).synchronize()
        else:
            from ..ops import als_gram_reference, als_reference_solve

            gram = als_gram_reference(kv, self._other_keys(side), cfg.rank) if implicit else None
            als_reference_solve(kv, t, off, o, a, b, cfg.rank, cfg.lam, gram)
        self.step_no += 1
        kv.advance_clock()
        kv.barrier()

    def als_epoch(self) -> float:
        """One ALS epoch: the row block, then the column block. Returns this rank's share of ``als_objective``."""
        self.als_half_step("rows")
        self.als_half_step("cols")
        return self.als_objective()

    def als_objective(self, chunk: int = 1 << 16) -> float:
        """This rank's share of the ALS objective, in float64 from pulled rows; the shares of all ranks sum to it
        (``server.allreduce_sum``). Squared: ``sum_e (x_e - w.h)^2`` over this rank's entries; implicit: ``sum_e [c_e
        (1 - w.h)^2 - (w.h)^2]`` over them (``c_e = 1 + alpha x_e``) plus ``sum_u w_u^T G w_u`` over this rank's users,
        G the Gram matrix of all items; both plus ``lambda (|W_block|^2 + |H_block|^2)`` of this rank's row and column
        blocks. Entries that occur twice count twice, as in the solve."""
        cfg, kv, data, r = self.cfg, self.worker, self.data, self.cfg.rank
        f64 = torch.float64

        def pull(keys):
            keys = torch.as_tensor(keys, dtype=torch.int64)
            v = torch.empty(keys.numel() * 2 * r, dtype=self.dtype,
                            device=self.server.device if self.cuda else "cpu")
            if keys.numel():
                if self.cuda:
                    kv.wait(kv.pull(keys.to(self.server.device), v, True))
                    torch.cuda.current_stream(self.server.device).synchronize()
                else:
                    kv.wait(kv.pull(keys, v))
            return v.view(-1, 2 * r)[:, :r].to(f64).cpu()

        total = 0.0
        for s in range(0, data.i.shape[0], chunk):
            w = pull(data.i[s:s + chunk].astype(np.int64))
            h = pull(data.j[s:s + chunk].astype(np.int64) + self.fck)
            pred = (w * h).sum(1)
            x = torch.from_numpy(data.x[s:s + chunk].astype(np.float64))
            if cfg.loss == "implicit":
                total += float(((1.0 + cfg.alpha * x) * (1.0 - pred) ** 2 - pred ** 2).sum())
            else:
                total += float(((x - pred) ** 2).sum())
        G = None
        if cfg.loss == "implicit":
            G = torch.zeros(r, r, dtype=f64)
            for s in range(0, cfg.num_cols, chunk):
                h = pull(np.arange(s, min(cfg.num_cols, s + chunk)) + self.fck)
                G += h.t() @ h
        for lo, hi, first, gram in ((*data.row_block(), 0, G), (*data.col_block(), self.fck, None)):
            for s in range(lo, hi, chunk):
                w = pull(np.arange(s, min(hi, s + chunk)) + first)
                total += cfg.lam * float((w * w).sum())
                if gram is not None:
                    total += float(((w @ gram) * w).sum())
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

    def recommend(self, rows, k: int = 10, seen=None):
        """The ``k`` items of highest score ``<w_u, h_i>`` for each user in ``rows``. Returns ``(item ids int64 [n, k],
        scores float32 [n, k])``, best first; equal scores go to the smaller item id. ``seen``: a CSR ``(offsets int64
        [n + 1], items int64)`` with each row's items ascending (e.g. ``data.seen(rows)``); those items are left out. A
        row with fewer than ``k`` items left is padded with ``(-1, -inf)``. ``1 <= k <= 64``.

        CUDA backend (float32 rows): only the users' rows are pulled; the scores against all items are computed from
        bf16-rounded operands in the fused gather + top-k kernel (``ops.gather_gemm_topk``), which reads the item rows
        wherever they live; this needs ``rank % 4 == 0`` (``ValueError`` otherwise). CPU route: fp32 PyTorch over the
        pulled item factors with the same order (``ops.topk_reference``)."""
        from ..ops import _check_topk, exclusion_mask, gather_gemm_topk, topk_reference

        cfg, kv = self.cfg, self.worker
        users = torch.as_tensor(np.asarray(rows), dtype=torch.int64).reshape(-1)
        n, N = users.numel(), cfg.num_cols
        if seen is not None:
            seen = (torch.as_tensor(seen[0], dtype=torch.int64), torch.as_tensor(seen[1], dtype=torch.int64))
        _check_topk(n, N, k, seen, None)
        if self.cuda:
            if cfg.rank % 4:
                raise ValueError(f"recommend on the GPU needs rank % 4 == 0, got rank {cfg.rank}")
            dev = self.server.device
            buf = torch.empty(n * 2 * cfg.rank, dtype=torch.float32, device=dev)
            if n:
                kv.wait(kv.pull(self.row_key(users).to(dev), buf, True))
            if not hasattr(self, "_item_keys"):
                self._item_keys = torch.arange(N, dtype=torch.int64, device=dev) + self.fck
            excl = (seen[0].to(dev), seen[1].to(dev)) if seen is not None else None
            vals, idx = gather_gemm_topk(self.server, buf.view(n, 2 * cfg.rank)[:, :cfg.rank], self._item_keys,
                                         cfg.rank, k, exclude=excl)
            return idx, vals
        wv = torch.empty(n * 2 * cfg.rank, dtype=self.dtype)
        if n:
            kv.wait(kv.pull(self.row_key(users), wv))
        hv = torch.empty(N * 2 * cfg.rank, dtype=self.dtype)
        kv.wait(kv.pull(torch.arange(N, dtype=torch.int64) + self.fck, hv))
        q = wv.view(n, 2 * cfg.rank)[:, :cfg.rank].float()
        E = hv.view(N, 2 * cfg.rank)[:, :cfg.rank].float()
        excluded = exclusion_mask(seen, N) if seen is not None else None
        vals, idx = topk_reference(q @ E.t(), int(k), excluded)
        return idx, vals

    def evaluate_ranking(self, test_i: np.ndarray, test_j: np.ndarray, k: int = 10, batch: int = 2048):
        """Recall@k and NDCG@k of the top-k lists of this rank's users with held-out items (the test pairs of users in
        this rank's row block; the rest are ignored). T_u: the held-out items of u that are not training items; L_u: u's
        top-k list with the training items left out. ``Recall@k = |L_u & T_u| / min(k, |T_u|)``, ``NDCG@k = sum over
        positions r of L_u with an item in T_u of 1 / log2(r + 2)``, divided by the same sum over ``r < min(k, |T_u|)``.
        Users with empty T_u are skipped. Returns ``(sum of recall, sum of ndcg, users)``: sums over ranks give the
        means (``server.allreduce_sum``)."""
        data = self.data
        lo, hi = data.row_block()
        ti, tj = np.asarray(test_i, dtype=np.int64), np.asarray(test_j, dtype=np.int64)
        mine = (ti >= lo) & (ti < hi)
        ti, tj = ti[mine], tj[mine]
        pairs = np.unique(ti * data.num_cols + tj)
        trained = np.unique((data.i.astype(np.int64)) * data.num_cols + data.j)
        pairs = pairs[~np.isin(pairs, trained, assume_unique=True)]
        ti, tj = pairs // data.num_cols, pairs % data.num_cols
        users, start = np.unique(ti, return_index=True)
        end = np.append(start[1:], ti.shape[0])
        disc = 1.0 / np.log2(np.arange(k) + 2.0)
        idcg = np.cumsum(disc)
        rec_sum, ndcg_sum = 0.0, 0.0
        for s in range(0, users.shape[0], batch):
            u = users[s:s + batch]
            idx, _ = self.recommend(u, k, seen=data.seen(u))
            idx = idx.cpu().numpy()
            for r in range(u.shape[0]):
                T = tj[start[s + r]:end[s + r]]
                hit = np.isin(idx[r], T)
                m = min(k, T.shape[0])
                rec_sum += hit.sum() / m
                ndcg_sum += float((disc * hit).sum()) / idcg[m - 1]
        return rec_sum, ndcg_sum, int(users.shape[0])

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
