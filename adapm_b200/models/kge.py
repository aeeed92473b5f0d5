"""Knowledge-graph embeddings (ComplEx, RESCAL, TransE, RotatE) on the parameter manager.

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

TransE (``algorithm="TransE"``, L1 or L2 by ``p_norm``) is the translational model of the reference's toy-data README:
entity rows are normalised on read, a positive triple and its ``2 * neg_ratio`` negatives form margin-ranking pairs
(``margin``), and one fused kernel per batch (``ops.kge_transe_step``) streams the negatives; the CPU route and the
numerics oracle is ``ops.transe_reference_step``. Evaluation and prediction rank by distance: ``ops.gather_dist_rank_count``
and ``ops.gather_dist_topk`` on the GPU, ``torch.cdist`` on the CPU.

RotatE (``algorithm="RotatE"``) rotates the subject by the relation in the complex plane: entity rows hold ``embed_dim / 2``
complex values interleaved ``(re, im)``, relation rows ``embed_dim / 2`` phases in radians (``relation_len =
embed_dim``), and ``D = sum_i |s_i e^{i theta_i} - o_i|``. A positive triple and its ``2 * neg_ratio`` negatives train with
the sigmoid loss and self-adversarial negative weights (``margin`` is gamma, ``adversarial_temperature`` alpha) in one
fused kernel per batch (``ops.kge_rotate_step``); the CPU route and the numerics oracle is ``ops.rotate_reference_step``.
Subject and object ranks and predictions use the complex metric of ``ops.gather_dist_rank_count`` /
``ops.gather_dist_topk`` with ``p="complex"`` (``ops.complex_dist`` on the CPU); the relation side is computed in PyTorch.
``gamma_relation`` is not used by RotatE (phases get no L2).

``KGEConfig.train_type = "1vsAll"`` (ComplEx and RESCAL) trains LibKGE's 1vsAll type instead of negative sampling: each
query ``(s, r, ?)`` and ``(?, r, o)`` of a batch is scored against every entity with a softmax cross-entropy loss, and every
entity row gets one AdaGrad update per step (``ops.kge_1vsall_step`` on the tensor cores, deterministic on one GPU;
``ops.kge_1vsall_reference_step`` on the CPU backend and for float64 stores). ``neg_ratio`` is not used. Since every step
reads every entity, several ranks signal one intent for all entity keys over ``[0, CLOCK_MAX)`` at initialisation.

``KGEConfig.train_type = "sampled_softmax"`` (ComplEx and RESCAL) keeps that cross-entropy at any entity count: each step
draws ``shared_negatives`` entities (the negative sampler's seed and ``local_only`` rule), and each chunk of 128 triples
scores its queries against one list of its subjects, its objects and those shared negatives; other copies of a query's
answer in the list are masked. The step touches only the batch's entities, the negatives and the batch's relations
(``ops.kge_shared_step``: three per-chunk tensor-core contractions, cost linear in the batch and ``shared_negatives``,
deterministic on one GPU; ``ops.kge_shared_reference_step`` on the CPU backend and for float64 stores). Intents are
per batch, as for negative sampling. ``neg_ratio`` is not used.

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
    algorithm: str = "ComplEx"      # ComplEx | RESCAL | TransE | RotatE
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
    p_norm: int = 1                  # TransE only: L1 or L2 distance
    margin: float = 1.0              # TransE: margin of the ranking loss; RotatE: gamma of the sigmoid loss
    adversarial_temperature: float = 1.0   # RotatE only: alpha of the self-adversarial negative weights (0: uniform)
    train_type: str = "negative_sampling"  # or "1vsAll" (ComplEx, RESCAL): cross-entropy over every entity,
    #                                          or "sampled_softmax" (ComplEx, RESCAL): over shared sampled negatives
    shared_negatives: int = 1024     # sampled_softmax: entities drawn per step, shared by the whole batch
    max_bytes: int = 1 << 30         # 1vsAll: device memory for one chunk of scores and G (ops.kge_1vsall_step);
    #                                  sampled_softmax: the limit of the step's workspace (ops.kge_shared_step)

    @property
    def entity_len(self) -> int:
        return 2 * self.embed_dim

    @property
    def relation_len(self) -> int:
        if self.algorithm == "RotatE":   # [phases (d / 2) | AdaGrad (d / 2)]
            return self.embed_dim
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
        """ComplEx / RESCAL; a TransE triple pushes 3 rows plus one per active negative pair (count them instead), a
        RotatE triple 3 + 2 * neg_ratio rows."""
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
        if cfg.train_type not in ("negative_sampling", "1vsAll", "sampled_softmax"):
            raise ValueError("train_type must be 'negative_sampling', '1vsAll' or 'sampled_softmax', "
                             f"got {cfg.train_type!r}")
        if cfg.train_type != "negative_sampling":
            if cfg.algorithm not in ("ComplEx", "RESCAL"):
                raise ValueError(f"{cfg.train_type} training is defined for ComplEx and RESCAL, not {cfg.algorithm}")
            if cfg.dropout_entity > 0 or cfg.dropout_relation > 0:
                raise ValueError(f"dropout is not defined for {cfg.train_type} training")
        if cfg.train_type == "sampled_softmax" and (isinstance(cfg.shared_negatives, bool)
                                                    or int(cfg.shared_negatives) != cfg.shared_negatives
                                                    or cfg.shared_negatives < 0):
            raise ValueError(f"shared_negatives must be a non-negative integer, got {cfg.shared_negatives!r}")
        if cfg.algorithm == "RotatE":
            from ..ops import _check_rotate_shape

            _check_rotate_shape(cfg.embed_dim)
        # the fused kernels are float32; float64 rows (the reference's ValT = double, kge.cc:33) train through the
        # Pull / Push API with the same update rule (kge_reference_step) on either backend
        self.cuda = server.backend == "cuda" and server.dtype == torch.float32
        self.dtype = server.dtype
        self.step_no = 0
        self.pushes = 0                 # TransE / RotatE on the CPU route: rows pushed so far
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
        ``uniform{a/b}`` or ``none``; AdaGrad accumulators start at 1e-6. RotatE: the entity rows follow ``init``, the
        relation phases are drawn uniform in [-pi, pi) (``none`` skips both)."""
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
            self._long_term_intents()
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
                if cfg.algorithm == "RotatE" and first == cfg.num_entities:
                    rows[:, : ln // 2] = ((torch.rand(k.numel(), ln // 2, generator=gen, dtype=torch.float64) * 2 - 1)
                                          * np.pi).to(self.dtype)
                elif kind == "normal":
                    rows[:, : ln // 2] = (torch.randn(k.numel(), ln // 2, generator=gen) * p2 + p1).to(self.dtype)
                else:
                    rows[:, : ln // 2] = (torch.rand(k.numel(), ln // 2, generator=gen) * (p2 - p1) + p1).to(self.dtype)
                rows[:, ln // 2:] = 1e-6
                self.worker.set(k, rows.view(-1))
        self.worker.waitall()
        self.worker.end_setup()
        self._long_term_intents()

    def _long_term_intents(self) -> None:
        """The intents over ``[0, CLOCK_MAX)`` on several ranks: the relations on request, and every entity under 1vsAll,
        whose steps read all of them."""
        cfg = self.cfg
        if self.server.num_servers() == 1:
            return
        if cfg.signal_initial_relations_intent:
            self.worker.intent(torch.arange(cfg.num_entities, cfg.num_entities + cfg.num_relations), 0, CLOCK_MAX)
        if cfg.train_type == "1vsAll":
            self.worker.intent(torch.arange(cfg.num_entities), 0, CLOCK_MAX)

    # ------------------------------------------------------------------ intent
    def signal_intent(self, triples: torch.Tensor, clock: int) -> None:
        if not self.cfg.signal_intent or self.server.num_servers() == 1:
            return
        rels = triples[:, 1] + self.cfg.num_entities
        # under 1vsAll the entities are covered by the long-term intent of init_model
        keys = rels if self.cfg.train_type == "1vsAll" else torch.cat([triples[:, 0], triples[:, 2], rels])
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

    def _negatives(self, B: int):
        """The step's seed and its ``[B, 2 * neg_ratio]`` uniform negative entities, in the layout of ``_expand``
        (corrupted objects first)."""
        seed, neg = self._draw(B * 2 * self.cfg.neg_ratio)
        return seed, neg.view(B, 2 * self.cfg.neg_ratio)

    def _draw(self, n: int):
        """The step's seed and ``n`` uniform entities: the device sampler on CUDA (local keys only under the local scheme
        on several ranks), else the rank's generator."""
        cfg = self.cfg
        seed = (cfg.model_seed * 7 + self.server.my_rank() * 7919 + self.step_no) & 0xFFFFFFFFFFFF
        if self.cuda:
            local_only = cfg.sampling_scheme == "local" and self.server.num_servers() > 1
            return seed, self.sampler.sample(n, seed, local_only=local_only)
        return seed, torch.randint(0, cfg.num_entities, (n,), generator=self._gen)

    def step(self, triples_host: torch.Tensor) -> torch.Tensor:
        """One batch of positive triples ([B,3] int64 CPU tensor, pinned for the e2e path): one fused launch on CUDA,
        else the float64-capable reference rule through Pull/Push. ComplEx and RESCAL train the calls of ``_expand`` with
        dropout; TransE and RotatE train each positive against its ``2 * neg_ratio`` negatives and have no dropout."""
        from .. import ops

        cfg, ne = self.cfg, self.cfg.num_entities
        if cfg.algorithm in ("TransE", "RotatE") and (cfg.dropout_entity > 0 or cfg.dropout_relation > 0):
            raise ValueError(f"dropout is not defined for {cfg.algorithm}")
        tr = triples_host.to(self.server.device, non_blocking=True) if self.cuda else triples_host
        if cfg.train_type == "1vsAll":
            if self.cuda:
                ops.kge_1vsall_step(self.worker, tr[:, 0].contiguous(), (tr[:, 1] + ne).contiguous(),
                                    tr[:, 2].contiguous(), ne, cfg.algorithm, cfg.embed_dim, cfg.eta, cfg.gamma_entity,
                                    cfg.gamma_relation, self.loss, cfg.max_bytes)
            else:
                loss = ops.kge_1vsall_reference_step(self.worker, triples_host, cfg)
            self.step_no += 1
            return self.loss if self.cuda else torch.tensor([loss], dtype=torch.float32)
        if cfg.train_type == "sampled_softmax":
            _, neg = self._draw(int(cfg.shared_negatives))
            if self.cuda:
                ops.kge_shared_step(self.worker, tr[:, 0].contiguous(), (tr[:, 1] + ne).contiguous(),
                                    tr[:, 2].contiguous(), neg, ne, cfg.algorithm, cfg.embed_dim, cfg.eta,
                                    cfg.gamma_entity, cfg.gamma_relation, self.loss, cfg.max_bytes)
            else:
                loss = ops.kge_shared_reference_step(self.worker, triples_host, neg, cfg)
            self.step_no += 1
            return self.loss if self.cuda else torch.tensor([loss], dtype=torch.float32)
        seed, neg = self._negatives(tr.shape[0])
        if cfg.algorithm in ("ComplEx", "RESCAL"):
            S, R, O, L = self._expand(tr, neg)
            if self.cuda:
                fused = ops.kge_complex_step if cfg.algorithm == "ComplEx" else ops.kge_rescal_step
                fused(self.server, S, R, O, L, cfg.embed_dim, cfg.eta, cfg.gamma_entity, cfg.gamma_relation, self.loss,
                      self.stats, cfg.dropout_entity, cfg.dropout_relation, seed, deterministic=cfg.deterministic)
            else:
                loss = kge_reference_step(self.worker, S, R, O, L, cfg)
        else:
            if cfg.algorithm == "TransE":
                fused, reference = ops.kge_transe_step, ops.transe_reference_step
                args = (cfg.embed_dim, cfg.p_norm, cfg.margin, cfg.eta, cfg.gamma_entity, cfg.gamma_relation)
            else:
                fused, reference = ops.kge_rotate_step, ops.rotate_reference_step
                args = (cfg.embed_dim, cfg.margin, cfg.adversarial_temperature, cfg.eta, cfg.gamma_entity)
            s, r, o = tr[:, 0].contiguous(), (tr[:, 1] + ne).contiguous(), tr[:, 2].contiguous()
            if self.cuda:
                fused(self.server, s, r, o, neg, *args, self.loss, self.stats, deterministic=cfg.deterministic)
            else:
                loss, pushes = reference(self.worker, s, r, o, neg, *args)
                self.pushes += pushes
        self.step_no += 1
        return self.loss if self.cuda else torch.tensor([loss], dtype=torch.float32)

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
        """``export.epoch.N.{entities,relations}.bin`` (float32 embedding halves) and, with ``write_checkpoint``, the
        float64 ``checkpoint.epoch.N.*`` files with the AdaGrad halves. RotatE: entity rows are interleaved
        ``(re_0, im_0, re_1, im_1, ...)`` and relation exports hold the ``embed_dim / 2`` phases in radians."""
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

    def _metric(self):
        """How entity candidates are compared: ``"dot"`` (ComplEx, RESCAL; a higher score is better), else the
        ``(p, normalize)`` of ``ops.gather_dist_*`` / ``ops.dist_rank_reference`` (a smaller distance is better): TransE's
        ``p_norm`` against normalised entity rows, RotatE's ``"complex"`` distance against raw rows."""
        if self.cfg.algorithm in ("ComplEx", "RESCAL"):
            return "dot"
        return (self.cfg.p_norm, True) if self.cfg.algorithm == "TransE" else ("complex", False)

    def _pull_rows(self, keys: torch.Tensor, ln: int) -> torch.Tensor:
        """Device pull of the store rows of ``keys`` (row length ``ln``): their embedding halves, a [n, ln / 2] view."""
        buf = torch.empty(keys.numel() * ln, dtype=torch.float32, device=self.server.device)
        self.worker.wait(self.worker.pull(keys.contiguous(), buf, True))
        return buf.view(-1, ln)[:, : ln // 2]

    def rank_triples(self, triples: torch.Tensor, known: torch.Tensor, batch: int = 2048, use_tensor_cores: bool = True):
        """Ranks of the true subject / relation / object of every triple among all candidates (reference
        ``rank()``, kge.cc:716-774): subject and object ranks raw and filtered (other known-true answers do not count),
        the relation rank unfiltered like in the reference. Returns a dict of int64 tensors
        ``rank_s, rank_r, rank_o, rank_s_raw, rank_o_raw``. ``known``: all true triples (train+valid+test).

        A candidate counts when it is strictly better than the true answer (``_metric``). CUDA: the dot metric scores
        the whole pulled model with ``ops.gemm_nt_rank_count`` (or an fp32 matmul without ``use_tensor_cores``), the
        distance metrics pull only each batch's entity rows and ``ops.gather_dist_rank_count`` reads the candidates from
        the store. CPU: ``pull_embeddings()``, with ``ops.dist_rank_reference`` for the distance metrics. RotatE's
        relation side depends on the candidate's phases and is computed by ``_rotate_relation_ranks``."""
        from .. import ops

        cfg, d, ne, nr = self.cfg, self.cfg.embed_dim, self.cfg.num_entities, self.cfg.num_relations
        metric = self._metric()
        dev = self.server.device if self.cuda else torch.device("cpu")
        triples = triples.to(dev)
        answers = {side: self._answer_keys(known, side, dev) for side in ("object", "subject")}
        # Compute dtypes. CUDA ranks in fp32; on the tensor cores from bf16-rounded operands, so the true score is the
        # one the wgmma kernel sees. The CPU scores the dot metric in the store's dtype (float64 rows rank in float64,
        # like the reference's ValT = double) and the distance metrics always in float64, where a sum of |differences|
        # over d terms loses the least to rounding.
        tc = metric == "dot" and self.cuda and use_tensor_cores
        bf = (lambda x: x.to(torch.bfloat16).float()) if tc else (lambda x: x)
        normalize = metric != "dot" and metric[1]   # entity candidates only; relation candidates are raw rows
        if self.cuda and metric != "dot":
            R = self._pull_rows(torch.arange(ne, ne + nr, dtype=torch.int64, device=dev), cfg.relation_len)
            ent_rows = lambda keys: self._pull_rows(keys, cfg.entity_len)
            cand_e = torch.arange(ne, dtype=torch.int64, device=dev)
            cand_r = torch.arange(ne, ne + nr, dtype=torch.int64, device=dev)
        else:
            E, _, R, _ = self.pull_embeddings(dev)
            if metric != "dot":
                E, R = E.double(), R.double()
            ent_rows = lambda keys: E[keys]
            cand_e = normalize_rows(E) if normalize else bf(E)
            cand_r = bf(R)

        def count(q, cand, true, excl=None, norm=False):
            """(raw, filtered) counts of the candidates other than ``true`` that are strictly better; filtered leaves out
            the columns of the CSR ``excl``."""
            if metric != "dot":
                if self.cuda:
                    return ops.gather_dist_rank_count(self.server, q, cand, d, metric[0], norm, true.contiguous(), excl)
                return ops.dist_rank_reference(q, cand, metric[0], true,
                                               ops.exclusion_mask(excl, cand.shape[0]) if excl is not None else None)
            q = bf(q)
            true_score = (q * cand[true]).sum(1)
            if tc:   # wgmma GEMM with the rank-count epilogue: the [B, candidates] scores never reach HBM
                raw = ops.gemm_nt_rank_count(q, cand, true_score, true).long()
            else:
                scores = q @ cand.t()
                scores.scatter_(1, true.view(-1, 1), float("-inf"))
                raw = (scores > true_score.view(-1, 1)).sum(1)
            return raw, (_filter_dot(raw, q, true_score, true, excl, lambda cols: cand[cols]) if excl is not None else raw)

        out = {k: [] for k in ("rank_s", "rank_r", "rank_o", "rank_s_raw", "rank_o_raw")}
        for i in range(0, triples.shape[0], batch):
            t = triples[i:i + batch]
            Es, Eo, Rr = ent_rows(t[:, 0]), ent_rows(t[:, 2]), R[t[:, 1]]
            for side, given, true in (("object", t[:, 0], t[:, 2]), ("subject", t[:, 2], t[:, 0])):
                q = self._query(Es if side == "object" else Eo, Rr, side)
                excl = self._known_answers(given, t[:, 1], side, known, answers[side])
                raw, filt = count(q, cand_e, true, excl, normalize)
                out[f"rank_{side[0]}_raw"].append(raw + 1)
                out[f"rank_{side[0]}"].append(filt + 1)
            if cfg.algorithm == "RotatE":
                out["rank_r"].append(_rotate_relation_ranks(Es, Eo, R, t[:, 1]) + 1)
            else:
                out["rank_r"].append(count(self._relation_query(Es, Eo), cand_r, t[:, 1])[0] + 1)
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

    # ------------------------------------------------------------------ queries and link prediction
    def _query(self, ent_rows: torch.Tensor, rel_rows: torch.Tensor, side: str) -> torch.Tensor:
        """The entity-side query of ``rank_triples`` and ``predict``, compared with the candidates by ``_metric``:
        ComplEx and RESCAL score ``<q, E[candidate]>``; TransE ``q = s^ + r`` (objects) or ``o^ - r`` (subjects) against
        normalised entities; RotatE ``q = s o rho`` or ``o o conj(rho)`` against raw entities (exact, ``|rho_i| = 1``)."""
        cfg = self.cfg
        if cfg.algorithm == "ComplEx":
            return complex_query(ent_rows, rel_rows, conj=(side == "subject"))
        if cfg.algorithm == "TransE":
            e = normalize_rows(ent_rows)
            return (e + rel_rows if side == "object" else e - rel_rows).contiguous()
        if cfg.algorithm == "RotatE":
            return rotate_query(ent_rows, rel_rows, side == "subject")
        Rm = rel_rows.reshape(-1, cfg.embed_dim, cfg.embed_dim)
        if side == "object":
            return torch.einsum("bi,bij->bj", ent_rows, Rm)
        return torch.einsum("bij,bj->bi", Rm, ent_rows)

    def _relation_query(self, Es: torch.Tensor, Eo: torch.Tensor) -> torch.Tensor:
        """The relation-side query of ``rank_triples`` (not RotatE): ComplEx and RESCAL score ``<q, R[candidate]>``,
        TransE ``q = o^ - s^`` at the distance of ``_metric`` from the raw relation rows."""
        cfg = self.cfg
        if cfg.algorithm == "ComplEx":
            h = cfg.embed_dim // 2
            sre, sim, ore, oim = Es[:, :h], Es[:, h:], Eo[:, :h], Eo[:, h:]
            return torch.cat([sre * ore + sim * oim, sre * oim - sim * ore], 1)
        if cfg.algorithm == "TransE":
            return (normalize_rows(Eo) - normalize_rows(Es)).contiguous()
        return torch.einsum("bi,bj->bij", Es, Eo).reshape(Es.shape[0], cfg.embed_dim * cfg.embed_dim)

    def _answer_keys(self, known: torch.Tensor, side: str, dev) -> torch.Tensor:
        """The known triples as sorted, distinct keys ``(given * nr + relation) * ne + answer`` for ``side``'s queries:
        the known answers of one query are one run of them."""
        ne, nr = self.cfg.num_entities, self.cfg.num_relations
        known = torch.as_tensor(known, dtype=torch.int64).to(dev).view(-1, 3)
        given, ans = (known[:, 0], known[:, 2]) if side == "object" else (known[:, 2], known[:, 0])
        return torch.unique((given * nr + known[:, 1]) * ne + ans)

    def _known_answers(self, ents: torch.Tensor, rels: torch.Tensor, side: str, known: torch.Tensor, keys=None):
        """CSR ``(offsets [n + 1], cols)`` of the known answers of each query, ascending per row, each answer once.
        ``keys``: ``_answer_keys(known, side)`` when the caller has built them already."""
        ne, nr = self.cfg.num_entities, self.cfg.num_relations
        dev = ents.device
        comp = self._answer_keys(known, side, dev) if keys is None else keys
        qkey = (ents * nr + rels) * ne
        lo = torch.searchsorted(comp, qkey)
        cnt = torch.searchsorted(comp, qkey + ne) - lo
        offsets = torch.zeros(ents.numel() + 1, dtype=torch.int64, device=dev)
        offsets[1:] = torch.cumsum(cnt, 0)
        rows = torch.repeat_interleave(torch.arange(ents.numel(), device=dev), cnt)
        pos = torch.arange(rows.numel(), device=dev) - offsets[:-1][rows] + lo[rows]
        return offsets, comp[pos] % ne

    def predict(self, entities, relations, side: str = "object", k: int = 10, known=None):
        """The ``k`` most likely completions of each query: objects of ``(entities[i], relations[i], ?)`` for
        ``side="object"``, subjects of ``(?, relations[i], entities[i])`` for ``side="subject"``.

        Returns ``(entity ids int64 [n, k], scores float32 [n, k])``, best first; equal scores go to the smaller entity
        id. ``known``: triples [m, 3] (e.g. train + valid + test); every known answer of a query is left out (the
        filtered setting). A query with fewer than ``k`` candidates left is padded with ``(-1, -inf)``.
        ``1 <= k <= 64``. The query and the metric are the ones of ``rank_triples``; for TransE and RotatE the score is
        ``-distance``.

        CUDA backend (float32 rows): only the rows of the queries are pulled, and a fused gather + top-k kernel reads the
        entity rows wherever they live, on any number of GPUs: ``ops.gather_gemm_topk`` scores bf16-rounded operands for
        ComplEx and RESCAL, ``ops.gather_dist_topk`` computes fp32 distances for TransE and RotatE. CPU backend: fp32
        PyTorch over ``pull_embeddings()`` with the same order (``ops.topk_reference``)."""
        from .. import ops

        if side not in ("object", "subject"):
            raise ValueError(f"side must be 'object' or 'subject', got {side!r}")
        cfg = self.cfg
        d, ne = cfg.embed_dim, cfg.num_entities
        ents = torch.as_tensor(entities, dtype=torch.int64).reshape(-1)
        rels = torch.as_tensor(relations, dtype=torch.int64).reshape(-1)
        if ents.numel() != rels.numel():
            raise ValueError("entities and relations must have the same length")
        metric = self._metric()
        if self.cuda:
            dev = self.server.device
            ents, rels = ents.to(dev), rels.to(dev)
            q = self._query(self._pull_rows(ents, cfg.entity_len), self._pull_rows(rels + ne, cfg.relation_len), side)
            excl = self._known_answers(ents, rels, side, known) if known is not None else None
            keys = torch.arange(ne, dtype=torch.int64, device=dev)
            if metric == "dot":
                vals, idx = ops.gather_gemm_topk(self.server, q, keys, d, k, exclude=excl)
            else:
                vals, idx = ops.gather_dist_topk(self.server, q, keys, d, k, *metric, exclude=excl)
            return idx, vals
        ops._check_topk(ents.numel(), ne, k, None, None)
        E, _, R, _ = self.pull_embeddings()
        E, R = E.float(), R.float()   # fp32 scores, the dtype the CUDA route returns, whatever the store's dtype
        q = self._query(E[ents], R[rels], side)
        excluded = ops.exclusion_mask(self._known_answers(ents, rels, side, known), ne) if known is not None else None
        if metric == "dot":
            scores = q @ E.t()
        elif metric[0] == "complex":
            scores = -ops.complex_dist(q, E)
        else:
            scores = -torch.cdist(q, normalize_rows(E), p=float(metric[0]))
        vals, idx = ops.topk_reference(scores, int(k), excluded)
        return idx, vals


def rotate_query(e: torch.Tensor, theta: torch.Tensor, conj: bool) -> torch.Tensor:
    """RotatE query rows, interleaved (re, im): ``e o rho`` (object side) or ``e o conj(rho)`` (subject side, conj=True)
    with ``rho = e^{i theta}``; the distance to a candidate is ``ops.complex_dist(query, candidate)``."""
    n, d = e.shape
    z = e.reshape(n, d // 2, 2)
    re, im = z[..., 0], z[..., 1]
    c, s = torch.cos(theta), torch.sin(theta)
    if conj:
        s = -s
    return torch.stack([re * c - im * s, re * s + im * c], -1).reshape(n, d).contiguous()


def _rotate_relation_ranks(Es: torch.Tensor, Eo: torch.Tensor, R: torch.Tensor, true_rel: torch.Tensor,
                           chunk_elems: int = 1 << 24) -> torch.Tensor:
    """RotatE relation-side raw ranks - 1: ``#{r' != r : D(s, r', o) < D(s, r, o)}`` with ``D = sum_i |s_i rho'_i - o_i|``
    over every relation's phases ``R`` [nr, d / 2], in the dtype and on the device of the inputs, in relation chunks.
    The true relation's distance is read from the same matrix, so it cannot disagree with its column by rounding."""
    B, d = Es.shape
    nr, m = R.shape
    s, o = Es.reshape(B, 1, m, 2), Eo.reshape(B, 1, m, 2)
    D = torch.empty(B, nr, dtype=Es.dtype, device=Es.device)
    step = max(1, chunk_elems // max(1, B * d))
    for j in range(0, nr, step):
        c, sn = torch.cos(R[j:j + step]).unsqueeze(0), torch.sin(R[j:j + step]).unsqueeze(0)
        xr = s[..., 0] * c - s[..., 1] * sn - o[..., 0]
        xi = s[..., 0] * sn + s[..., 1] * c - o[..., 1]
        D[:, j:j + step] = torch.sqrt(xr * xr + xi * xi).sum(-1)
    dt = D.gather(1, true_rel.view(-1, 1))
    better = D < dt
    better.scatter_(1, true_rel.view(-1, 1), False)
    return better.sum(1)


def normalize_rows(e: torch.Tensor) -> torch.Tensor:
    """e / max(|e|_2, 1e-12) per row: the entity rows TransE scores with."""
    return e / e.norm(dim=-1, keepdim=True).clamp(min=1e-12)


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


def _filter_dot(raw: torch.Tensor, q: torch.Tensor, true_score: torch.Tensor, true: torch.Tensor, excl, answer_rows):
    """Filtered dot-metric counts: ``raw`` minus, per query, its known answers (CSR ``excl``) other than the true one that
    score strictly higher. ``answer_rows(cols)``: the candidate rows of the answers, as the raw count scored them."""
    off, cols = excl
    rows = torch.repeat_interleave(torch.arange(q.shape[0], device=q.device), off[1:] - off[:-1])
    better = ((q[rows] * answer_rows(cols)).sum(1) > true_score[rows]) & (cols != true[rows])
    return raw - torch.zeros_like(raw).index_add_(0, rows, better.to(raw.dtype))


def _ranking_summary(rf: torch.Tensor, rr: torch.Tensor) -> dict:
    """MRR and Hits@k of the filtered entity ranks ``rf`` and the raw MRR of ``rr`` (subject and object sides)."""
    rf, rr = rf.double(), rr.double()
    return {"mrr": float((1 / rf).mean()), "mrr_raw": float((1 / rr).mean()),
            "hits@1": float((rf <= 1).double().mean()), "hits@3": float((rf <= 3).double().mean()),
            "hits@10": float((rf <= 10).double().mean()), "n": int(rf.numel() // 2)}


def evaluate_fused(model: "KGE", triples: torch.Tensor, known: torch.Tensor, batch: int = 2048) -> dict:
    """Filtered ranking without ever pulling the model: per batch only the rows of the queries, of the true
    answers and of the known answers are pulled (device Pull); the 1-vs-all scoring against ALL entities runs in
    the fused gather + wgmma GEMM + rank-count kernel (``ops.gather_gemm_rank_count``), which reads the entity
    rows from whichever GPU's HBM holds them. Works on any number of GPUs; every rank may evaluate its own share
    of the test triples concurrently."""
    from ..ops import gather_gemm_rank_count

    if model.cfg.algorithm in ("TransE", "RotatE"):   # distance ranks from the store rows (ops.gather_dist_rank_count)
        ranks = model.rank_triples(triples, known, batch)
        return _ranking_summary(torch.cat([ranks["rank_o"], ranks["rank_s"]]),
                                torch.cat([ranks["rank_o_raw"], ranks["rank_s_raw"]]))
    cfg, dev = model.cfg, model.server.device
    d, ne, ln = cfg.embed_dim, cfg.num_entities, cfg.entity_len
    triples = triples.to(dev)
    answers = {side: model._answer_keys(known, side, dev) for side in ("object", "subject")}
    all_ent = torch.arange(ne, dtype=torch.int64, device=dev)
    stats = torch.zeros(2, dtype=torch.int64, device=dev)
    bf = lambda x: x.to(torch.bfloat16).float()   # the operands the tensor cores see

    def answer_rows(cols):
        return bf(model._pull_rows(cols, ln)) if cols.numel() else torch.empty(0, d, device=dev)

    ranks_f, ranks_r = [], []
    for i in range(0, triples.shape[0], batch):
        t = triples[i:i + batch]
        Es, Eo, Rr = model._pull_rows(t[:, 0], ln), model._pull_rows(t[:, 2], ln), model._pull_rows(t[:, 1] + ne, ln)
        for side, given, true in (("object", t[:, 0], t[:, 2]), ("subject", t[:, 2], t[:, 0])):
            q = bf(complex_query(Es if side == "object" else Eo, Rr, conj=(side == "subject")))
            true_score = (q * bf(Eo if side == "object" else Es)).sum(1)
            raw = gather_gemm_rank_count(model.server, q, all_ent, d, true_score, true, stats).long() + 1
            excl = model._known_answers(given, t[:, 1], side, known, answers[side])
            ranks_r.append(raw)
            ranks_f.append(_filter_dot(raw, q, true_score, true, excl, answer_rows))
    s = stats.tolist()
    return {**_ranking_summary(torch.cat(ranks_f), torch.cat(ranks_r)),
            "gathered_rows_local": s[0], "gathered_rows_remote": s[1]}
