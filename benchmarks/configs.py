"""BASELINE configs #3 (KGE ComplEx, FB15k scale, d = 512), #4 (matrix factorisation 10M x 1M, rank 128) and #5
(CTR DeepFM on a 100M-key table) behind ``bench.py --config kge|mf|ctr``. Same contract as the word2vec headline:
W warm-up steps (after P untimed placement steps for N > 1), then two timed loops of K steps each - ``e2e`` through the
public API with the step's inputs copied from pinned host memory and the loss read back every step, and ``value``
with device-resident inputs - CUDA events on the launching stream, barrier + synchronize on both sides, max over ranks.
"""
from __future__ import annotations

import json
import os
import time

import numpy as np
import torch
import torch.distributed as dist


class Ctx:
    def __init__(self, args, rank, world, local_rank, sampler_cls):
        self.args, self.rank, self.world, self.lr = args, rank, world, local_rank
        self.dev = torch.device("cuda", local_rank)
        self.sampler_cls = sampler_cls

    def barrier(self):
        if self.world > 1:
            dist.barrier(device_ids=[self.lr])
        torch.cuda.synchronize()

    def max_ms(self, *ms):
        t = torch.tensor(list(ms), dtype=torch.float64, device=self.dev)
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.tolist()


def _pm_counters(server):
    keep = ("relocations", "replica_setups", "refreshes", "protocol_errors")
    return {k: v for k, v in server.counters().items() if k in keep}


def timed_loops(ctx: Ctx, step_e2e, step_resident, K: int, W: int, P: int):
    """step_*(s) run step number s. Returns dict(e2e_ms, dev_ms, launches_e2e, launches_dev, clocks, host_ms)."""
    from adapm_b200 import _C

    stream = torch.cuda.current_stream()
    for s in range(P + W):
        step_e2e(s)
    ctx.barrier()
    sampler = ctx.sampler_cls(ctx.lr)
    if ctx.rank == 0 and not os.environ.get("ADAPM_BENCH_NO_SMI"):
        sampler.start()
    l0 = _C.kernel_launches()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ctx.barrier()
    ev[0].record(stream)
    t0 = time.perf_counter()
    for s in range(P + W, P + W + K):
        step_e2e(s)
    host_ms = (time.perf_counter() - t0) * 1e3 / K
    ev[1].record(stream)
    ctx.barrier()
    l1 = _C.kernel_launches()
    for s in range(P + W + K, P + W + K + 3):
        step_resident(s)
    ctx.barrier()
    l2 = _C.kernel_launches()
    ctx.barrier()
    ev[2].record(stream)
    for s in range(P + W + K + 3, P + W + 2 * K + 3):
        step_resident(s)
    ev[3].record(stream)
    ctx.barrier()
    l3 = _C.kernel_launches()
    clocks = sampler.stop() if ctx.rank == 0 else None
    e2e_ms, dev_ms = ctx.max_ms(ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3]))
    return {"e2e_ms": e2e_ms, "dev_ms": dev_ms, "launches_e2e": int(l1 - l0), "launches_dev": int(l3 - l2),
            "clocks": clocks, "host_ms": host_ms}


def _line(ctx, metric, model, cfgd, updates_per_step, t, K, W, h2d, d2h, extra):
    value = updates_per_step * K / (t["dev_ms"] * 1e-3)
    e2e = updates_per_step * K / (t["e2e_ms"] * 1e-3)
    out = {"metric": metric, "value": value, "unit": "updates/s", "n_gpus": ctx.world, "steps": K, "warmup": W,
           "ms_per_step": t["dev_ms"] / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
           "dtype": "fp32", "data": "synthetic", "impl": "native",
           "config": dict({"model": model, "parallelism": f"pm{ctx.world} (key-sharded store, intent-driven relocation/replication)",
                           "l2": "every step has its own random batch; tables larger than L2 except KGE (67 MB model, "
                                 "L2-resident by nature of the config)"}, **cfgd),
           "e2e": {"value": e2e, "unit": "updates/s", "ms_per_step": t["e2e_ms"] / K, "h2d_bytes_per_step": h2d,
                   "d2h_bytes_per_step": d2h},
           "gpu_launches": t["launches_dev"], "gpu_launches_e2e": t["launches_e2e"], "clocks": t["clocks"],
           "host_loop_ms_per_step": t["host_ms"]}
    out.update(extra)
    return out


# ---------------------------------------------------------------------------------------------------------- KGE
def run_kge(ctx: Ctx):
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, synthetic_triples

    a = ctx.args
    K, W = a.steps, a.warmup
    RA = 8
    P = a.placement_steps if a.placement_steps >= 0 else (3 * RA if ctx.world > 1 else 0)
    cfg = KGEConfig(embed_dim=512, batch_triples=8192, read_ahead=RA)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=ctx.rank, world=ctx.world,
                       backend="cuda", fabric="shm" if ctx.world > 1 else "inproc", device=ctx.lr, job=ad.default_job() + "k")
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    total = P + W + 2 * K + 3
    nb = min(total + RA + 2, 512)
    tr = synthetic_triples(cfg, cfg.batch_triples * nb, seed=100 + ctx.rank)
    batches = [tr[i * cfg.batch_triples:(i + 1) * cfg.batch_triples].pin_memory() for i in range(nb)]
    dev_batches = {}
    loss_host = torch.zeros(1).pin_memory()
    evq = []

    def bounded():
        e = torch.cuda.Event(); e.record(); evq.append(e)
        if len(evq) > 3:
            evq.pop(0).synchronize()

    def step_e2e(s):
        model.signal_intent(batches[(s + RA) % nb], kv.current_clock() + RA)
        model.loss.zero_()
        model.step(batches[s % nb])                       # H2D of the triples inside
        loss_host.copy_(model.loss, non_blocking=True)    # D2H of the step's loss
        kv.advance_clock()
        bounded()

    def step_res(s):
        model.signal_intent(batches[(s + RA) % nb], kv.current_clock() + RA)
        model.loss.zero_()
        b = dev_batches.get(s % nb)
        if b is None:
            b = dev_batches[s % nb] = batches[s % nb].to(ctx.dev)
        model.step(b)
        kv.advance_clock()
        bounded()

    for s in range(P + W + K, total):
        dev_batches[s % nb] = batches[s % nb].to(ctx.dev)
    for s in range(RA):
        model.signal_intent(batches[s], kv.current_clock() + s)
    t = timed_loops(ctx, step_e2e, step_res, K, W, P)
    st = model.stats.tolist()
    out = None
    if ctx.rank == 0:
        upd = ctx.world * cfg.batch_triples * cfg.updates_per_triple
        out = _line(ctx, "KGE ComplEx updates/sec (device-timed, max over ranks)",
                    "ComplEx, FB15k scale (14 951 entities, 1 345 relations), d=512 (rows 4 KB fp32 [emb|AdaGrad])",
                    {"batch_triples_per_gpu": cfg.batch_triples, "neg_ratio": cfg.neg_ratio, "global_batch": ctx.world * cfg.batch_triples,
                     "updates_per_triple": cfg.updates_per_triple, "intent_read_ahead": RA, "placement_steps": P},
                    upd, t, K, W, cfg.batch_triples * 3 * 8, 4,
                    {"locality": {"rows_local": st[0], "rows_remote": st[1], "rows_slow_path": st[2]},
                     "pm": _pm_counters(server)})
    kv.finalize(); server.shutdown()
    return out


# ---------------------------------------------------------------------------------------------------------- MF
def run_mf(ctx: Ctx):
    import adapm_b200 as ad
    from adapm_b200.models.mf import MFConfig
    from adapm_b200.ops import mf_step

    a = ctx.args
    K, W = a.steps, a.warmup
    world, rank, dev = ctx.world, ctx.rank, ctx.dev
    cfg = MFConfig(num_rows=10_000_000, num_cols=1_000_000, rank=128, algorithm="dsgd", batch_nnz=1 << 18)
    n = cfg.batch_nnz
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys(world), num_threads=1, rank=rank, world=world, backend="cuda",
                       fabric="shm" if world > 1 else "inproc", device=ctx.lr, job=ad.default_job() + "m")
    kv = ad.Worker(0, server)
    fck = cfg.first_col_key(world)
    rpb = (cfg.num_rows + world - 1) // world
    cpb = (cfg.num_cols + world - 1) // world
    kv.begin_setup()
    keys = torch.arange(rank, cfg.num_keys(world), world, dtype=torch.int64)
    keys = keys[(keys < cfg.num_rows) | (keys >= fck)]
    gen = torch.Generator(device=dev).manual_seed(rank)
    for s in range(0, keys.numel(), 1 << 18):
        k = keys[s:s + (1 << 18)].to(dev)
        rows = torch.zeros(k.numel(), cfg.row_len, device=dev)
        rows[:, :cfg.rank] = torch.rand(k.numel(), cfg.rank, generator=gen, device=dev) / cfg.rank ** 0.5
        kv.set(k, rows.view(-1))
    kv.waitall(); kv.end_setup()
    if world > 1:   # row block of this rank for the whole run (reference matrix_factorization.cc:369-372)
        kv.intent(torch.arange(rank * rpb, min(cfg.num_rows, (rank + 1) * rpb)), 0, ad.CLOCK_MAX)
    loss = torch.zeros(1, device=dev); stats = torch.zeros(4, dtype=torch.int64, device=dev)
    rng = np.random.default_rng(5 + rank)
    steps_per_block = 16          # a DSGD sub-epoch = 16 steps on one column block, then the blocks rotate
    P = 0
    total = W + 2 * K + 3
    loss_host = torch.zeros(1).pin_memory()
    cache = {}

    def host_batch(s):
        if s not in cache:
            se = s // steps_per_block
            b = (rank + se) % world
            i = torch.from_numpy(rng.integers(rank * rpb, min(cfg.num_rows, (rank + 1) * rpb), n))
            j = torch.from_numpy(rng.integers(b * cpb, min(cfg.num_cols, (b + 1) * cpb), n)) + fck
            x = torch.randn(n)
            cache[s] = tuple(t.pin_memory() for t in (i, j, x))
        return cache[s]

    rn = torch.full((n,), 20, dtype=torch.int32, device=dev)
    cn = torch.full((n,), 200, dtype=torch.int32, device=dev)
    for s in range(total + 1):
        host_batch(s)
    dev_cache = {s: tuple(t.to(dev) for t in host_batch(s)) for s in range(W + K, total)}

    def subepoch_boundary(s):
        if world > 1 and s % steps_per_block == 0:
            se = s // steps_per_block
            b = (rank + se) % world                 # DSGD stratum: no two ranks share a column block
            kv.intent(torch.arange(b * cpb, min(cfg.num_cols, (b + 1) * cpb)) + fck, kv.current_clock())
            kv.wait_sync()
            kv.barrier()

    def step_e2e(s):
        subepoch_boundary(s)
        i, j, x = (t.to(dev, non_blocking=True) for t in host_batch(s))     # H2D of the step's non-zeros
        loss.zero_()
        mf_step(server, i, j, x, rn, cn, cfg.rank, 0.01, 0.05, loss, stats)
        loss_host.copy_(loss, non_blocking=True)
        if (s + 1) % steps_per_block == 0:
            kv.advance_clock()

    def step_res(s):
        subepoch_boundary(s)
        i, j, x = dev_cache[s]
        loss.zero_()
        mf_step(server, i, j, x, rn, cn, cfg.rank, 0.01, 0.05, loss, stats)
        if (s + 1) % steps_per_block == 0:
            kv.advance_clock()

    t = timed_loops(ctx, step_e2e, step_res, K, W, P)
    st = stats.tolist()
    out = None
    if rank == 0:
        out = _line(ctx, "matrix factorisation updates/sec (device-timed, max over ranks)",
                    "MF 10M x 1M, rank 128 (rows 1 KB fp32 [factor|AdaGrad]), SGD + AdaGrad",
                    {"batch_nnz_per_gpu": n, "global_batch": world * n, "schedule": "DSGD block rotation every 16 steps "
                     "(intent for the next column block + WaitSync + barrier INSIDE the timed loops)" if world > 1 else "plain SGD",
                     "placement_steps": P},
                    world * 2 * n, t, K, W, n * 20, 4,
                    {"locality": {"rows_local": st[0], "rows_remote": st[1], "rows_slow_path": st[2]},
                     "pm": _pm_counters(server)})
    kv.finalize(); server.shutdown()
    return out


# ---------------------------------------------------------------------------------------------------------- CTR
def run_ctr(ctx: Ctx):
    import adapm_b200 as ad
    from adapm_b200.models.deepfm import DeepFM, DeepFMConfig, synthetic_ctr_batch

    a = ctx.args
    K, W = a.steps, a.warmup
    RA = 4
    P = a.placement_steps if a.placement_steps >= 0 else (3 * RA if ctx.world > 1 else 0)
    cfg = DeepFMConfig(num_features=int(os.environ.get("ADAPM_CTR_KEYS", 100_000_000)), read_ahead=RA, precision="fp8")
    server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=ctx.rank, world=ctx.world, backend="cuda",
                       fabric="shm" if ctx.world > 1 else "inproc", device=ctx.lr, job=ad.default_job() + "c",
                       options={"pool_factor": 1.5})
    kv = ad.Worker(0, server)
    model = DeepFM(server, kv, cfg)
    model.init_model()
    total = P + W + 2 * K + 3
    nb = total + RA + 2
    batches = [tuple(t.pin_memory() for t in synthetic_ctr_batch(cfg, s, ctx.rank)) for s in range(nb)]
    dev_b = {s: tuple(t.to(ctx.dev) for t in batches[s]) for s in range(P + W + K, total)}
    loss_host = torch.zeros(1).pin_memory()

    def step_e2e(s):
        model.signal_intent(batches[s + RA][0], kv.current_clock() + RA)
        l = model.step(*batches[s], return_tensor=True)     # H2D of ids + labels inside
        loss_host.copy_(l.detach().view(1), non_blocking=True)
        kv.advance_clock()

    def step_res(s):
        model.signal_intent(batches[s + RA][0], kv.current_clock() + RA)
        model.step(*dev_b[s], return_tensor=True)
        kv.advance_clock()

    for s in range(RA):
        model.signal_intent(batches[s][0], kv.current_clock() + s)
    t = timed_loops(ctx, step_e2e, step_res, K, W, P)
    out = None
    if ctx.rank == 0:
        # update = one (key,row) additive update applied at the owner: the distinct feature rows of a batch
        upd_step = ctx.world * float(model.rows_pushed) / max(1, model.step_no)
        out = _line(ctx, "CTR DeepFM sparse updates/sec (device-timed, max over ranks)",
                    f"DeepFM, {cfg.num_features} feature keys x {cfg.row_len} fp32 (emb 16 + AdaGrad), 26 fields, MLP 400x3 "
                    f"(dense GEMMs: wgmma {cfg.precision})",
                    {"batch_examples_per_gpu": cfg.batch_size, "global_batch": ctx.world * cfg.batch_size, "intent_read_ahead": RA,
                     "placement_steps": P, "examples_per_s": ctx.world * cfg.batch_size * K / (t["dev_ms"] * 1e-3),
                     "updates_per_step": "distinct feature rows of the batch (mean over the run)"},
                    upd_step, t, K, W, cfg.batch_size * (26 * 8 + 4), 4,
                    {"pm": _pm_counters(server)})
    kv.finalize(); server.shutdown()
    return out


RUNNERS = {"kge": run_kge, "mf": run_mf, "ctr": run_ctr}


def run(name, args, rank, world, local_rank, sampler_cls):
    out = RUNNERS[name](Ctx(args, rank, world, local_rank, sampler_cls))
    if rank == 0 and out is not None:
        print(json.dumps(out))
    return 0
