"""Knowledge-graph embeddings (ComplEx, RESCAL) on the parameter manager.

Behavioural parity with the reference application ``apps/knowledge_graph_embeddings.cc``:

* keys: entities ``0..ne-1``, relations ``ne..ne+nr-1``, ``loss_key``, ``eval_key`` (len 20)
  (kge.cc:121-127,1296-1306); per-key value lengths (RESCAL relations are ``2*d*d``) (kge.cc:1243-1254);
* per training triple: one positive call and ``neg_ratio`` x {corrupted object, corrupted subject} negative
  calls, each pulling/pushing (s, r, o): ``3 * (1 + 2*neg_ratio)`` updates per triple (kge.cc:1107-1119);
* BCE gradient, L2 only on positives, AdaGrad with the pulled accumulator and init 1e-6
  (kge.cc:437-531,415-435,309); negatives uniform over entities through PrepareSample/PullSample
  (kge.cc:131-137,1063-1086);
* intent: ``Intent({s,r,o}, futureClock)`` ``signal_intent_ahead`` clocks ahead; optional long-term relation
  intent ``[0, CLOCK_MAX)`` (kge.cc:1022-1032); one clock per batch instead of per triple;
* filtered ranking evaluation (MRR, Hits@k) (kge.cc:555-774) - on the GPU one 1-vs-all score GEMM per side
  with the rank counted in the epilogue;
* checkpoints: ``export.epoch.N.{entities,relations}.bin`` (row-major float32 embeddings) and
  ``checkpoint.epoch.N.{entities,relations}[.adagrad].bin`` (raw float64) (kge.cc:327-401; the reference's
  byte-offset bug for the adagrad half is not replicated).

On the GPU the train calls of a batch run as ONE fused kernel - ``ops.kge_complex_step`` or, for RESCAL (relation
rows are d x d matrices), ``ops.kge_rescal_step`` - including dropout on the pulled copies (mask from a counter-based
hash, reproducible by ``ops.kge_dropout_mask``). The evaluation ranks subject, relation and object of every test
triple (kge.cc:716-774) and aggregates the reference's 19 metrics over the ranks through ``eval_key``
(kge.cc:592-709). The CPU backend runs the same calls through the public Pull/Push API with PyTorch math
(``kge_reference_step``, also the numerics oracle of the GPU tests).

``KGEConfig.deterministic`` selects the deterministic one-GPU variant of the fused kernels (start-of-step reads,
fixed-point sums, bit-identical runs); the CPU backend accepts it and already follows the start-of-step rule.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .. import CLOCK_MAX


@dataclass
class KGEConfig:
    num_entities: int = 14951
    num_relations: int = 1345
    embed_dim: int = 512            # ComplEx: real half + imaginary half
    algorithm: str = "ComplEx"      # ComplEx | RESCAL
    neg_ratio: int = 6
    eta: float = 0.1
    gamma_entity: float = 1e-3
    gamma_relation: float = 1e-3
    dropout_entity: float = 0.0      # training-time dropout on embeddings (kge.cc:405-413,478-484)
    dropout_relation: float = 0.0
    batch_triples: int = 4096
    read_ahead: int = 4
    sampling_scheme: str = "local"
    signal_intent: bool = True
    signal_initial_relations_intent: bool = False
    init_std: float = 0.1
    model_seed: int = 134827
    deterministic: bool = False      # one GPU: start-of-step reads, bit-identical runs (ops.kge_complex_step)

    @property
    def entity_len(self) -> int:
        return 2 * self.embed_dim

    @property
    def relation_len(self) -> int:
        return 2 * self.embed_dim * (self.embed_dim if self.algorithm == "RESCAL" else 1)

    @property
    def loss_key(self) -> int:
        return self.num_entities + self.num_relations

    @property
    def eval_key(self) -> int:
        return self.num_entities + self.num_relations + 1

    @property
    def num_keys(self) -> int:
        return self.num_entities + self.num_relations + 2

    def value_lengths(self) -> torch.Tensor:
        l = torch.empty(self.num_keys, dtype=torch.int64)
        l[: self.num_entities] = self.entity_len
        l[self.num_entities: self.num_entities + self.num_relations] = self.relation_len
        l[self.loss_key] = 2
        l[self.eval_key] = 20
        return l

    @property
    def updates_per_triple(self) -> int:
        return 3 * (1 + 2 * self.neg_ratio)


def synthetic_triples(cfg: KGEConfig, n: int, seed: int = 0) -> torch.Tensor:
    """FB15k-shaped synthetic triples: Zipf-skewed entities/relations, [n, 3] int64 (s, r, o)."""
    rng = np.random.default_rng(seed)

    def zipf(size, k):
        p = 1.0 / np.arange(1, k + 1) ** 0.8
        p /= p.sum()
        return rng.choice(k, size=size, p=p)

    perm_e = rng.permutation(cfg.num_entities)
    s = perm_e[zipf(n, cfg.num_entities)]
    r = zipf(n, cfg.num_relations)
    # learnable structure: 80% of the objects are a fixed function of (s, r), the rest is noise
    o_fn = perm_e[(s * 7 + r * 13 + 1) % cfg.num_entities]
    o = np.where(rng.random(n) < 0.8, o_fn, perm_e[zipf(n, cfg.num_entities)])
    return torch.from_numpy(np.stack([s, r, o], 1).astype(np.int64))


def load_triples(path: str) -> torch.Tensor:
    """TSV ``s r o`` per line (apps/data/kge/*.del)."""
    from .. import _C

    return torch.from_numpy(_C.read_triples(path))   # native parser (csrc/adapm/io.cc)


class KGE:
    def __init__(self, server, worker, cfg: KGEConfig):
        self.server, self.worker, self.cfg = server, worker, cfg
        # the fused kernels are float32; float64 rows (the reference's ValT = double, kge.cc:33) train through the
        # Pull / Push API with the same update rule (kge_reference_step) on either backend
        self.cuda = server.backend == "cuda" and server.dtype == torch.float32
        self.dtype = server.dtype
        self.step_no = 0
        dev = server.device
        self._gen = torch.Generator().manual_seed(cfg.model_seed + 31 * server.my_rank())
        if self.cuda:
            from ..ops import DeviceSampler

            self.sampler = DeviceSampler(server, distribution="uniform", first_key=0, num_keys=cfg.num_entities)
            self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
            self.stats = torch.zeros(4, dtype=torch.int64, device=dev)

    # ------------------------------------------------------------------ keys
    def entity_key(self, e):
        return e

    def relation_key(self, r):
        return r + self.cfg.num_entities

    # ------------------------------------------------------------------ init
    def init_model(self, chunk: int = 8192, init: str = "") -> None:
        """``init``: the reference's ``init_parameters`` syntax - ``normal{mean/std}`` (default ``normal{0/init_std}``),
        ``uniform{a/b}`` or ``none``; AdaGrad accumulators start at 1e-6."""
        cfg, world, rank = self.cfg, self.server.num_servers(), self.server.my_rank()
        kind, p1, p2 = "normal", 0.0, cfg.init_std
        if init:
            import re

            mt = re.fullmatch(r"(none|normal|uniform)(?:\{([-+.\deE]+)/([-+.\deE]+)\})?", init.strip())
            if not mt:
                raise ValueError(f"init_parameters: cannot parse '{init}' (none | uniform{{a/b}} | normal{{mean/std}})")
            kind = mt.group(1)
            if mt.group(2) is not None:
                p1, p2 = float(mt.group(2)), float(mt.group(3))
            elif kind == "uniform":
                p1, p2 = -cfg.init_std, cfg.init_std
        if kind == "none":
            if cfg.signal_initial_relations_intent and world > 1:
                self.worker.intent(torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations), 0, CLOCK_MAX)
            return
        gen = torch.Generator().manual_seed(cfg.model_seed + rank)
        self.worker.begin_setup()
        for first, count, ln in ((0, cfg.num_entities, cfg.entity_len),
                                 (cfg.num_entities, cfg.num_relations, cfg.relation_len)):
            keys = torch.arange(first + ((rank - first) % world), first + count, world, dtype=torch.int64)
            per = max(1, min(chunk, (64 << 20) // (4 * ln)))
            for i in range(0, keys.numel(), per):
                k = keys[i:i + per]
                rows = torch.empty(k.numel(), ln, dtype=self.dtype)
                if kind == "normal":
                    rows[:, : ln // 2] = (torch.randn(k.numel(), ln // 2, generator=gen) * p2 + p1).to(self.dtype)
                else:
                    rows[:, : ln // 2] = (torch.rand(k.numel(), ln // 2, generator=gen) * (p2 - p1) + p1).to(self.dtype)
                rows[:, ln // 2:] = 1e-6
                self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()
        if cfg.signal_initial_relations_intent and world > 1:
            self.worker.intent(torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations), 0, CLOCK_MAX)

    # ------------------------------------------------------------------ intent
    def signal_intent(self, triples: torch.Tensor, clock: int) -> None:
        if not self.cfg.signal_intent or self.server.num_servers() == 1:
            return
        keys = torch.cat([triples[:, 0], triples[:, 2], triples[:, 1] + self.cfg.num_entities])
        self.worker.intent(keys, clock, clock + 1)

    # ------------------------------------------------------------------ training calls of one batch
    def _expand(self, triples: torch.Tensor, neg_ent: torch.Tensor):
        """triples [B,3], neg_ent [B, 2*neg_ratio] entity ids -> flat (s, r, o, label) call lists in the
        reference's order: positive, then per j: (s, r, o'), (s', r, o)."""
        B, nr = triples.shape[0], self.cfg.neg_ratio
        s, r, o = triples[:, 0:1], triples[:, 1:2], triples[:, 2:3]
        C = 1 + 2 * nr
        S = s.expand(B, C).clone()
        O = o.expand(B, C).clone()
        S[:, 2::2] = neg_ent[:, nr:]          # corrupted subjects at odd positions 2,4,..
        O[:, 1::2] = neg_ent[:, :nr]          # corrupted objects at positions 1,3,..
        R = (r + self.cfg.num_entities).expand(B, C)
        L = torch.zeros(B, C, dtype=torch.float32, device=triples.device)
        L[:, 0] = 1
        return S.reshape(-1), R.reshape(-1).contiguous(), O.reshape(-1), L.reshape(-1)

    def step(self, triples_host: torch.Tensor) -> torch.Tensor:
        """One batch of positive triples ([B,3] int64 CPU tensor, pinned for the e2e path)."""
        cfg = self.cfg
        B = triples_host.shape[0]
        if self.cuda:
            from ..ops import kge_complex_step, kge_rescal_step

            tr = triples_host.to(self.server.device, non_blocking=True)
            local_only = cfg.sampling_scheme == "local" and self.server.num_servers() > 1
            seed = (cfg.model_seed * 7 + self.server.my_rank() * 7919 + self.step_no) & 0xFFFFFFFFFFFF
            neg = self.sampler.sample(B * 2 * cfg.neg_ratio, seed, local_only=local_only).view(B, 2 * cfg.neg_ratio)
            S, R, O, L = self._expand(tr, neg)
            fused = kge_complex_step if cfg.algorithm == "ComplEx" else kge_rescal_step
            fused(self.server, S, R, O, L, cfg.embed_dim, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, self.loss,
                  self.stats, cfg.dropout_entity, cfg.dropout_relation, seed, deterministic=cfg.deterministic)
            self.step_no += 1
            return self.loss
        neg = torch.randint(0, cfg.num_entities, (B, 2 * cfg.neg_ratio), generator=self._gen)
        S, R, O, L = self._expand(triples_host, neg)
        loss = kge_reference_step(self.worker, S, R, O, L, cfg)
        self.step_no += 1
        return torch.tensor([loss], dtype=torch.float32)

    # ------------------------------------------------------------------ full-model pull (eval / checkpoints)
    def pull_embeddings(self, device=None):
        """Returns (E [ne, d], Eg [ne, d], R [nr, rel_dim], Rg) by pulling the whole model through the API."""
        cfg, kv = self.cfg, self.worker
        ek = torch.arange(cfg.num_entities)
        ev = torch.empty(cfg.num_entities * cfg.entity_len, dtype=self.dtype)
        kv.wait(kv.pull(ek, ev))
        rk = torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations)
        rv = torch.empty(cfg.num_relations * cfg.relation_len, dtype=self.dtype)
        kv.wait(kv.pull(rk, rv))
        ev = ev.view(cfg.num_entities, cfg.entity_len)
        rv = rv.view(cfg.num_relations, cfg.relation_len)
        d, rd = cfg.embed_dim, cfg.relation_len // 2
        out = (ev[:, :d].contiguous(), ev[:, d:].contiguous(), rv[:, :rd].contiguous(), rv[:, rd:].contiguous())
        return tuple(t.to(device) for t in out) if device is not None else out

    def save(self, path_prefix: str, epoch: int, write_checkpoint: bool = False) -> None:
        self.worker.wait_sync()
        if self.server.my_rank() != 0:
            return
        E, Eg, R, Rg = self.pull_embeddings()
        E.numpy().astype(np.float32).tofile(f"{path_prefix}export.epoch.{epoch}.entities.bin")
        R.numpy().astype(np.float32).tofile(f"{path_prefix}export.epoch.{epoch}.relations.bin")
        if write_checkpoint:
            E.numpy().astype(np.float64).tofile(f"{path_prefix}checkpoint.epoch.{epoch}.entities.bin")
            R.numpy().astype(np.float64).tofile(f"{path_prefix}checkpoint.epoch.{epoch}.relations.bin")
            Eg.numpy().astype(np.float64).tofile(f"{path_prefix}checkpoint.epoch.{epoch}.entities.adagrad.bin")
            Rg.numpy().astype(np.float64).tofile(f"{path_prefix}checkpoint.epoch.{epoch}.relations.adagrad.bin")

    # ------------------------------------------------------------------ evaluation
    EVAL_METRICS = ("mrr_s", "mrr_r", "mrr_o", "mrr_s_raw", "mrr_o_raw", "mr_s", "mr_r", "mr_o", "mr_s_raw", "mr_o_raw",
                    "hits01_s", "hits01_r", "hits01_o", "hits03_s", "hits03_r", "hits03_o", "hits10_s", "hits10_r",
                    "hits10_o")   # slots 0..18 of the eval_key row (reference kge.cc:94-112)

    def rank_triples(self, triples: torch.Tensor, known: torch.Tensor, batch: int = 2048, use_tensor_cores: bool = True):
        """Ranks of the true subject / relation / object of every triple among all candidates (reference
        ``rank()``, kge.cc:716-774): subject and object ranks raw and filtered (other known-true answers do not count),
        the relation rank unfiltered like in the reference. Returns a dict of int64 tensors
        ``rank_s, rank_r, rank_o, rank_s_raw, rank_o_raw``. ``known``: all true triples (train+valid+test)."""
        cfg = self.cfg
        dev = self.server.device if self.cuda else torch.device("cpu")
        E, _, R, _ = self.pull_embeddings(dev)
        triples = triples.to(dev)
        known = torch.unique(known.to(dev), dim=0)   # duplicates must not be filtered twice
        d = cfg.embed_dim
        tc = self.cuda and use_tensor_cores
        if tc:
            from ..ops import gemm_nt_rank_count

            bf = lambda x: x.to(torch.bfloat16).float()   # score with the operands the tensor cores see
        else:
            bf = lambda x: x
        E_s, R_s = bf(E), bf(R)
        sr_key = known[:, 0] * cfg.num_relations + known[:, 1]
        or_key = known[:, 2] * cfg.num_relations + known[:, 1]
        order = torch.argsort(sr_key)
        sr_sorted, sr_ent = sr_key[order], known[order, 2]
        order = torch.argsort(or_key)
        or_sorted, or_ent = or_key[order], known[order, 0]
        out = {k: [] for k in ("rank_s", "rank_r", "rank_o", "rank_s_raw", "rank_o_raw")}

        def count_better(q, cand, true_score, true_idx):
            if tc:   # wgmma GEMM with the rank-count epilogue: the [B, candidates] scores never reach HBM
                return gemm_nt_rank_count(q, cand, true_score, true_idx).long() + 1
            scores = q @ cand.t()
            scores.scatter_(1, true_idx.view(-1, 1), float("-inf"))
            return (scores > true_score.view(-1, 1)).sum(1) + 1

        for i in range(0, triples.shape[0], batch):
            t = triples[i:i + batch]
            Es, Eo, Rr = E[t[:, 0]], E[t[:, 2]], R[t[:, 1]]
            for side in (0, 1):  # 0: predict object, 1: predict subject
                if cfg.algorithm == "ComplEx":
                    q = complex_query(Es if side == 0 else Eo, Rr, conj=(side == 1))
                else:
                    Rm = Rr.view(-1, d, d)
                    q = torch.einsum("bi,bij->bj", Es, Rm) if side == 0 else torch.einsum("bij,bj->bi", Rm, Eo)
                q = bf(q)
                true_e = t[:, 2] if side == 0 else t[:, 0]
                true_score = (q * E_s[true_e]).sum(1)
                raw = count_better(q, E_s, true_score, true_e)
                # filtering: other known answers of the same query do not count
                qkey = (t[:, 0] if side == 0 else t[:, 2]) * cfg.num_relations + t[:, 1]
                kks, kes = (sr_sorted, sr_ent) if side == 0 else (or_sorted, or_ent)
                lo = torch.searchsorted(kks, qkey)
                hi = torch.searchsorted(kks, qkey, right=True)
                cnt = hi - lo
                rows = torch.repeat_interleave(torch.arange(t.shape[0], device=dev), cnt)
                offs = torch.arange(rows.numel(), device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
                ents = kes[lo[rows] + offs]
                ks = (q[rows] * E_s[ents]).sum(1)
                better = (ks > true_score[rows]) & (ents != true_e[rows])
                filt = raw - torch.zeros_like(raw).index_add_(0, rows, better.to(raw.dtype))
                out["rank_o_raw" if side == 0 else "rank_s_raw"].append(raw)
                out["rank_o" if side == 0 else "rank_s"].append(filt)
            # relation side: score(s, r', o) = <q_r, R[r']> for all relations r'
            if cfg.algorithm == "ComplEx":
                h = d // 2
                sre, sim, ore, oim = Es[:, :h], Es[:, h:], Eo[:, :h], Eo[:, h:]
                qr = torch.cat([sre * ore + sim * oim, sre * oim - sim * ore], 1)
            else:
                qr = torch.einsum("bi,bj->bij", Es, Eo).reshape(t.shape[0], d * d)
            qr = bf(qr)
            true_score = (qr * R_s[t[:, 1]]).sum(1)
            out["rank_r"].append(count_better(qr, R_s, true_score, t[:, 1]))
        return {k: torch.cat(v) if v else torch.zeros(0, dtype=torch.int64, device=dev) for k, v in out.items()}

    @staticmethod
    def _metric_sums(ranks: dict) -> torch.Tensor:
        """The 19 partial sums of the reference (EVAL_METRICS order) as a float64 vector."""
        f = {k: v.double() for k, v in ranks.items()}
        s, r, o, sr, orr = f["rank_s"], f["rank_r"], f["rank_o"], f["rank_s_raw"], f["rank_o_raw"]
        vals = [(1 / s).sum(), (1 / r).sum(), (1 / o).sum(), (1 / sr).sum(), (1 / orr).sum(),
                s.sum(), r.sum(), o.sum(), sr.sum(), orr.sum()]
        for k in (1, 3, 10):
            vals += [(s <= k).double().sum(), (r <= k).double().sum(), (o <= k).double().sum()]
        return torch.stack([v.cpu() for v in vals])

    def evaluate(self, triples: torch.Tensor, known: torch.Tensor, batch: int = 2048, use_tensor_cores: bool = True):
        """Filtered ranking evaluation of ``triples`` on THIS rank. Returns the reference's 19 metrics plus the usual
        entity-side summary (``mrr`` / ``hits@k`` = mean over subject and object side)."""
        ranks = self.rank_triples(triples, known, batch, use_tensor_cores)
        return self._finish_metrics(self._metric_sums(ranks), triples.shape[0])

    def _finish_metrics(self, sums: torch.Tensor, n: int) -> dict:
        m = {k: float(v) / max(1, n) for k, v in zip(self.EVAL_METRICS, sums.tolist())}
        m["mrr"] = 0.5 * (m["mrr_s"] + m["mrr_o"])
        m["mrr_raw"] = 0.5 * (m["mrr_s_raw"] + m["mrr_o_raw"])
        for k, name in ((1, "hits01"), (3, "hits03"), (10, "hits10")):
            m[f"hits@{k}"] = 0.5 * (m[f"{name}_s"] + m[f"{name}_o"])
        m["n"] = int(n)
        return m

    def evaluate_distributed(self, triples: torch.Tensor, known: torch.Tensor, truncate: int = 0, batch: int = 2048,
                             use_tensor_cores: bool = True) -> dict:
        """The reference's distributed evaluation (kge.cc:555-709): every rank ranks its share of the test triples, the
        partial sums of the 19 metrics are aggregated through the ``eval_key`` row of the parameter manager (reset,
        barrier, push, barrier, pull) and rank 0 returns the normalised metrics (other ranks return {}). Collective:
        one call per rank, with the same ``triples`` everywhere."""
        cfg, kv = self.cfg, self.worker
        world, rank = self.server.num_servers(), self.server.my_rank()
        N = triples.shape[0] if truncate <= 0 else min(triples.shape[0], truncate)
        per = -(-N // world)
        mine = triples[rank * per: min(N, (rank + 1) * per)]
        ek = torch.tensor([cfg.eval_key], dtype=torch.int64)
        row = torch.zeros(20, dtype=self.server.dtype)
        if rank == 0:   # reset the aggregation row (it may hold the sums of the previous evaluation)
            kv.wait(kv.pull(ek, row))
            kv.wait(kv.push(ek, -row))
        kv.wait_sync() if world > 1 else None
        kv.barrier()
        part = torch.zeros(20, dtype=self.server.dtype)
        if mine.shape[0]:
            part[:19] = self._metric_sums(self.rank_triples(mine, known, batch, use_tensor_cores)).to(part.dtype)
        kv.wait(kv.push(ek, part))
        kv.wait_sync() if world > 1 else None
        kv.barrier()
        if rank != 0:
            kv.barrier()
            return {}
        kv.wait(kv.pull(ek, row))
        kv.barrier()
        return self._finish_metrics(row[:19].double(), N)


def complex_query(a: torch.Tensor, r: torch.Tensor, conj: bool) -> torch.Tensor:
    """Query vector q such that score(s, r, e) = <q, E[e]> for all e (object side), or the subject-side
    equivalent (conj=True): scores against all candidate subjects."""
    h = a.shape[1] // 2
    are, aim, rre, rim = a[:, :h], a[:, h:], r[:, :h], r[:, h:]
    if not conj:   # object side: q = [r_re s_re - r_im s_im | r_re s_im + r_im s_re]
        return torch.cat([rre * are - rim * aim, rre * aim + rim * are], 1)
    # subject side: d score / d s = [r_re o_re + r_im o_im | r_re o_im - r_im o_re]
    return torch.cat([rre * are + rim * aim, rre * aim - rim * are], 1)


def score_all(q: torch.Tensor, E: torch.Tensor, server=None) -> torch.Tensor:
    """1-vs-all scores [B, ne] = q @ E^T. With a CUDA server the hand-written wgmma GEMM is used
    (bf16 operands, fp32 accumulation in registers); otherwise a plain fp32 matmul."""
    if server is not None:
        from ..ops import gemm_nt_bf16

        if gemm_nt_bf16 is not None:
            return gemm_nt_bf16(q, E)
    return q @ E.t()


def kge_reference_step(kv, S, R, O, L, cfg: KGEConfig, masks=None) -> float:
    """Plain PyTorch fp32 training calls through Pull/Push with the reference's update rule
    (all calls of the batch read the state at the start of the step). ``masks`` = (subject, relation, object)
    dropout scale masks [n, len] (``ops.kge_dropout_mask``) instead of fresh random ones."""
    d = cfg.embed_dim
    n = S.numel()
    dt = kv.server.dtype      # float32, or float64 like the reference's ValT
    L = L.to(dt)

    def pull(keys, ln):
        v = torch.empty(n * ln, dtype=dt)
        kv.wait(kv.pull(keys.contiguous(), v))
        return v.view(n, ln)

    rs, ro = pull(S, cfg.entity_len), pull(O, cfg.entity_len)
    rr = pull(R, cfg.relation_len)
    Es, As, Eo, Ao = rs[:, :d], rs[:, d:], ro[:, :d], ro[:, d:]
    rd = cfg.relation_len // 2
    Er, Ar = rr[:, :rd], rr[:, rd:]
    if masks is not None:
        Es, Er, Eo = Es * masks[0], Er * masks[1], Eo * masks[2]
    elif cfg.dropout_entity > 0:      # Bernoulli mask + 1/(1-p) scaling, applied to the pulled copies only
        p = cfg.dropout_entity
        Es = Es * (torch.rand_like(Es) >= p) / (1 - p)
        Eo = Eo * (torch.rand_like(Eo) >= p) / (1 - p)
    if masks is None and cfg.dropout_relation > 0:
        p = cfg.dropout_relation
        Er = Er * (torch.rand_like(Er) >= p) / (1 - p)
    if cfg.algorithm == "ComplEx":
        h = d // 2
        sre, sim, rre, rim, ore, oim = Es[:, :h], Es[:, h:], Er[:, :h], Er[:, h:], Eo[:, :h], Eo[:, h:]
        sc = (rre * sre * ore + rre * sim * oim + rim * sre * oim - rim * sim * ore).sum(1)
        ds = torch.cat([rre * ore + rim * oim, rre * oim - rim * ore], 1)
        dr = torch.cat([sre * ore + sim * oim, sre * oim - sim * ore], 1)
        do = torch.cat([rre * sre - rim * sim, rre * sim + rim * sre], 1)
    else:  # RESCAL: s^T R o
        Rm = Er.view(n, d, d)
        sc = torch.einsum("bi,bij,bj->b", Es, Rm, Eo)
        ds = torch.einsum("bij,bj->bi", Rm, Eo)
        do = torch.einsum("bi,bij->bj", Es, Rm)
        dr = torch.einsum("bi,bj->bij", Es, Eo).reshape(n, d * d)
    dl = (torch.sigmoid(sc) - L).view(-1, 1)
    pos = (L > 0.5).view(-1, 1).to(dt)
    gs = dl * ds + pos * cfg.gamma_entity * Es
    gr = dl * dr + pos * cfg.gamma_relation * Er
    go = dl * do + pos * cfg.gamma_entity * Eo

    def upd(g, a):
        return torch.cat([-cfg.eta * g / torch.sqrt(a + g * g), g * g], 1).contiguous().view(-1)

    kv.wait(kv.push(S.contiguous(), upd(gs, As)))
    kv.wait(kv.push(R.contiguous(), upd(gr, Ar)))
    kv.wait(kv.push(O.contiguous(), upd(go, Ao)))
    y = torch.where(L > 0.5, sc, -sc).clamp(-30, 30)
    return float(torch.log1p(torch.exp(-y)).sum())


def evaluate_fused(model: "KGE", triples: torch.Tensor, known: torch.Tensor, batch: int = 2048) -> dict:
    """Filtered ranking without ever pulling the model: per batch only the rows of the queries, of the true
    answers and of the known answers are pulled (device Pull); the 1-vs-all scoring against ALL entities runs in
    the fused gather + wgmma GEMM + rank-count kernel (``ops.gather_gemm_rank_count``), which reads the entity
    rows from whichever GPU's HBM holds them. Works on any number of GPUs; every rank may evaluate its own share
    of the test triples concurrently."""
    from ..ops import gather_gemm_rank_count

    cfg, kv, dev = model.cfg, model.worker, model.server.device
    d, ne = cfg.embed_dim, cfg.num_entities
    triples = triples.to(dev)
    known = torch.unique(known.to(dev), dim=0)
    all_ent = torch.arange(ne, dtype=torch.int64, device=dev)
    sr_key = known[:, 0] * cfg.num_relations + known[:, 1]
    or_key = known[:, 2] * cfg.num_relations + known[:, 1]
    order = torch.argsort(sr_key); sr_sorted, sr_ent = sr_key[order], known[order, 2]
    order = torch.argsort(or_key); or_sorted, or_ent = or_key[order], known[order, 0]
    stats = torch.zeros(2, dtype=torch.int64, device=dev)

    def pull_emb(keys):
        keys = keys.contiguous()
        buf = torch.empty(keys.numel() * cfg.entity_len, dtype=torch.float32, device=dev)
        kv.wait(kv.pull(keys, buf, True))
        return buf.view(-1, cfg.entity_len)[:, :d]

    ranks_f, ranks_r = [], []
    for i in range(0, triples.shape[0], batch):
        t = triples[i:i + batch]
        Es, Eo = pull_emb(t[:, 0]), pull_emb(t[:, 2])
        Rr = pull_emb(t[:, 1] + ne)
        for side in (0, 1):
            q = complex_query(Es if side == 0 else Eo, Rr, conj=(side == 1)).to(torch.bfloat16).float()
            true_e = t[:, 2] if side == 0 else t[:, 0]
            Et = (Eo if side == 0 else Es).to(torch.bfloat16).float()
            true_score = (q * Et).sum(1)
            raw = gather_gemm_rank_count(model.server, q, all_ent, d, true_score, true_e, stats).long() + 1
            qkey = (t[:, 0] if side == 0 else t[:, 2]) * cfg.num_relations + t[:, 1]
            kks, kes = (sr_sorted, sr_ent) if side == 0 else (or_sorted, or_ent)
            lo = torch.searchsorted(kks, qkey)
            hi = torch.searchsorted(kks, qkey, right=True)
            cnt = hi - lo
            rows = torch.repeat_interleave(torch.arange(t.shape[0], device=dev), cnt)
            offs = torch.arange(rows.numel(), device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
            ents = kes[lo[rows] + offs]
            Ek = pull_emb(ents).to(torch.bfloat16).float() if ents.numel() else torch.empty(0, d, device=dev)
            better = ((q[rows] * Ek).sum(1) > true_score[rows]) & (ents != true_e[rows])
            filt = raw - torch.zeros_like(raw).index_add_(0, rows, better.to(raw.dtype))
            ranks_r.append(raw)
            ranks_f.append(filt)
    rf = torch.cat(ranks_f).double()
    rr = torch.cat(ranks_r).double()
    s = stats.tolist()
    return {"mrr": float((1 / rf).mean()), "mrr_raw": float((1 / rr).mean()),
            "hits@1": float((rf <= 1).double().mean()), "hits@3": float((rf <= 3).double().mean()),
            "hits@10": float((rf <= 10).double().mean()), "n": int(rf.numel() // 2),
            "gathered_rows_local": s[0], "gathered_rows_remote": s[1]}
