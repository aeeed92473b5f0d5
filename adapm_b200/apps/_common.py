"""Shared command-line plumbing of the applications: the reference's system options
(``sys.*``, ``sampling.*``; coloc_kv_server.h:205-222, sync_manager.h:805-814, sampling.h:166-170)
are accepted with their original names and forwarded to the server."""
from __future__ import annotations

import argparse
import threading

SYS_FLAGS = ["sys.zmq_threads", "sys.techniques", "sys.time_intent_actions", "sys.location_caches", "sys.channels",
             "sys.trace.keys", "sys.stats.out", "sys.sync.max_per_sec", "sys.sync.pause", "sys.sync.threshold",
             "sys.timing.initial_estimate", "sys.timing.autotune", "sys.timing.smoothing_factor",
             "sys.timing.buffer_quantile", "sampling.scheme", "sampling.pool_size", "sampling.reuse",
             "sampling.batch_size", "sampling.with_replacement",
             # additions of this implementation
             "sys.sync.sweep_period", "sys.sync.idle_period", "sys.sync.min_clocks", "sys.sync.min_clocks_wait_ms",
             "sys.stats.locality", "pool_factor", "pool_bytes", "wait_timeout_s"]


def add_system_options(ap: argparse.ArgumentParser) -> None:
    g = ap.add_argument_group("system options (same names as the reference)")
    for f in SYS_FLAGS:
        g.add_argument("--" + f, dest=f, default=None)
    g.add_argument("--backend", default=None, choices=["cpu", "cuda"])
    g.add_argument("--value_type", default="float", choices=["float", "double"],
                   help="type of the parameter values: float (fused sm_90a kernels) or double (the reference's ValT for kge "
                        "and mf; trains through Pull / Push with the same update rule on either backend)")


def add_ablation_options(ap: argparse.ArgumentParser) -> None:
    """Flags every reference application has for ablation experiments (word2vec.cc:1032-1044, mf.cc:645-650,
    kge.cc): random key assignment, full replication, synchronous pushes."""
    g = ap.add_argument_group("ablation options (same names as the reference)")
    g.add_argument("--enforce_random_keys", type=int, default=0, help="assign keys to ids randomly instead of in id order")
    g.add_argument("--enforce_full_replication", type=int, default=0,
                   help="signal intent for every key for the whole run (every rank replicates the whole model)")
    g.add_argument("--sync_push", type=int, default=0,
                   help="wait for each push (the fused GPU steps are stream-ordered; this adds a host wait per step)")
    g.add_argument("--async_push", type=int, default=None, help="inverse of --sync_push (kge spelling)")


def wants_sync_push(args) -> bool:
    if getattr(args, "async_push", None) is not None:
        return not bool(args.async_push)
    return bool(getattr(args, "sync_push", 0))


def id_permutation(n: int, seed: int, enabled: bool):
    """forwards[id] = shuffled id (identity when disabled), as a numpy int64 array (reference: `forwards`/`backwards`)."""
    import numpy as np

    if not enabled:
        return np.arange(n, dtype=np.int64)
    return np.random.default_rng(seed).permutation(n).astype(np.int64)


def enforce_full_replication(kv, num_keys: int) -> None:
    """Replicate all keys on all nodes throughout training (reference word2vec.cc:1003-1010)."""
    import torch

    import adapm_b200 as ad

    kv.intent(torch.arange(num_keys, dtype=torch.int64), 0, ad.CLOCK_MAX)
    kv.wait_sync()
    kv.barrier()
    kv.wait_sync()


def system_options(args) -> dict:
    return {f: getattr(args, f) for f in SYS_FLAGS if getattr(args, f, None) is not None}


def strip_dashes(argv):
    return [a for a in argv if a != "--"]


def run_workers(num_threads: int, fn) -> list:
    """fn(customer_id) in num_threads threads (the reference spawns worker threads per node)."""
    out, errs = [None] * num_threads, []

    def w(c):
        try:
            out[c] = fn(c)
        except BaseException as e:  # noqa
            errs.append(e)

    ths = [threading.Thread(target=w, args=(c,)) for c in range(num_threads)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    if errs:
        raise errs[0]
    return out
