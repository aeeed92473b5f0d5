"""Multi-rank scenarios for the fused-op tests: rows owned by a peer, local replicas, keys whose relocation is in flight.

All of this runs on ONE device: ``run_cluster(mode="threads")`` runs ``WORLD`` logical ranks in this process, with the
inproc fabric and peer pointers into the same HBM. The initial owner of key ``k`` is ``k % WORLD``, so remote keys are
chosen on purpose. Every rank runs its op on a CUDA stream of its own, so that one rank's kernels do not queue behind
another rank's on the legacy default stream (which synchronises with every other blocking stream of the device).

A runner takes a *case*, which describes one op on one store:

- ``value_lengths``, ``num_keys``: the store;
- ``init``: ``[(keys, rows)]``, the rows rank 0 loads (and the rows every read returns, in the same groups);
- ``keys_of(batch)``: the store keys a batch touches (intents, counts of remote keys);
- ``open(server, kv)``: this rank's stepper. ``step(batch)`` runs one batch on the current stream and may return a
  per-step output; ``step.totals()`` returns ``(loss or None, stats)``.

The runners own the streams, the synchronisation, the pacing and the turn order. Each returns a list with one dict per
rank: what the rank reported, plus its server's ``counters``.
"""
import contextlib
import threading
import time
from dataclasses import dataclass
from typing import Any, Callable, Optional

import numpy as np
import torch

from harness import run_cluster

WORLD = 3
MOVER_MIN_ITERS = 60
PACE_S = 0.03               # pause after each step while keys move: the steps spread over many sync rounds
READ_MIN_S = 3.0            # read-only ops repeat over at least this many seconds of relocation rounds


@dataclass
class Case:
    value_lengths: Any
    num_keys: int
    init: list
    keys_of: Optional[Callable] = None
    open: Optional[Callable] = None


class Fused:
    """The stepper of an op that adds into a device loss [1] and stats [4]: ``fn(server, batch, loss, stats)``."""

    def __init__(self, server, fn):
        self.server, self.fn = server, fn
        self.loss = torch.zeros(1, device=server.device)
        self.stats = torch.zeros(4, dtype=torch.int64, device=server.device)

    def __call__(self, batch):
        self.fn(self.server, batch, self.loss, self.stats)

    def totals(self):
        return float(self.loss.item()), self.stats.tolist()


@contextlib.contextmanager
def one_rank_store(value_lengths, num_keys, backend, dtype):
    """(server, worker) of a fresh one-rank store (device 0 for ``cuda``), finalized and shut down on exit"""
    import adapm_b200 as ad

    s = ad.Server(value_lengths, num_keys=num_keys, num_threads=1, rank=0, world=1, backend=backend, fabric="inproc",
                  job=f"one_{np.random.randint(1 << 30)}", dtype=dtype, **({"device": 0} if backend == "cuda" else {}))
    kv = ad.Worker(0, s)
    try:
        yield s, kv
    finally:
        kv.finalize()
        s.shutdown()


def settle(kv):
    """every request answered and two sync rounds on every rank: updates have reached owners and replicas"""
    kv.waitall(); kv.wait_sync(); kv.barrier(); kv.wait_sync(); kv.barrier()


def load_rows(kv, groups):
    for keys, rows in groups:
        kv.wait(kv.set(keys, rows.to(kv.server.dtype).contiguous().view(-1)))


def pull_rows(kv, groups, dtype=torch.float32):
    """the rows of ``groups``' keys, one tensor of each group's shape"""
    out = []
    for keys, rows in groups:
        v = torch.empty(rows.numel(), dtype=dtype)
        kv.wait(kv.pull(keys, v))
        out.append(v.view(rows.shape))
    return out


def spread_keys(rank, m, g):
    """m distinct keys for ``rank``, disjoint from the other ranks' keys, 3 in 4 of them homed on another rank (the
    initial owner of key k is k % world): keys < world * world * m."""
    j = torch.arange(m)
    home = torch.where(j % 4 == 0, torch.full_like(j, rank), (rank + 1 + (j // 4) % 2) % WORLD)
    keys = WORLD * (rank * m + j) + home
    return keys[torch.randperm(m, generator=g)]


def make_local(kv, server, keys):
    """Declares this rank's intent for ``keys`` and runs sync rounds until every rank's keys are local (at most 50)."""
    c = kv.current_clock()
    kv.intent(keys, c, c + 1_000_000)
    for _ in range(50):
        kv.advance_clock()
        settle(kv)
        missing = sum(not server.is_local(int(k)) for k in keys)
        if server.allreduce_sum([float(missing)])[0] == 0:
            break


def mover(kv, rank, block, done, max_iters=3000):
    """Ranks 0 and 1 pass ``block`` back and forth with intents (read-only: they never write a row) until ``done``."""
    probe = block[:4]
    buf = torch.zeros(kv.server.total_len(probe), dtype=kv.server.dtype)
    it = 0
    while (it < MOVER_MIN_ITERS or not done.is_set()) and it < max_iters:
        if it % 2 == rank:
            kv.intent(block, kv.current_clock(), kv.current_clock() + 3)
            if it % 16 < 2:
                kv.wait_sync()
        for _ in range(3):
            kv.advance_clock()
        kv.wait(kv.pull(probe, buf))
        it += 1
    return it


# ---------------------------------------------------------------------------------------------- the runners
def _cluster(worker, case, technique=None, world=WORLD):
    res = run_cluster(worker, world=world, workers=1, mode="threads", value_lengths=case.value_lengths,
                      num_keys=case.num_keys, dtype="float32", backend="cuda",
                      options={"sys.techniques": technique} if technique else None)
    return [dict(res[r][0], counters=res[r]["counters"]) for r in range(world)]


def _loaded(kv, server, case):
    if server.my_rank() == 0:
        load_rows(kv, case.init)
    kv.waitall(); kv.barrier()


def _steps(step, batches, stream, pause=0.0):
    """each batch on ``stream``, waited for; returns the per-step outputs"""
    outs = []
    for b in batches:
        with torch.cuda.stream(stream):
            outs.append(step(b))
        stream.synchronize()
        if pause:
            time.sleep(pause)
    return outs


def on_peer_rows(case, batches, in_turns):
    """No intents: rank r runs ``batches[r]`` (None: nothing) on the rows where rank 0 loaded them. ``in_turns=False``:
    all ranks at once, then a barrier; ``True``: ranks 0, 1, 2 one after another with a settle after each. Rank 0 then
    reads the rows. Per rank: ``loss``, ``stats``, ``outs``, ``remote`` (keys of its batch owned by another rank) and,
    on rank 0, ``rows``."""
    def worker(kv, server, wid):
        rank, b = server.my_rank(), batches[server.my_rank()]
        _loaded(kv, server, case)
        out = {"remote": 0 if b is None else sum(server.owner_of(int(k)) != rank for k in case.keys_of(b)), "outs": []}
        step = case.open(server, kv)
        stream = torch.cuda.Stream(server.device)
        for turn in range(WORLD) if in_turns else [rank]:        # (all at once: each rank's only turn is its own)
            if turn == rank and b is not None:
                out["outs"] = _steps(step, [b], stream)
            if in_turns:
                settle(kv)
            else:
                kv.barrier()
        out["loss"], out["stats"] = step.totals()
        if rank == 0:
            out["rows"] = pull_rows(kv, case.init)
        kv.barrier()
        kv.finalize()
        return out

    return _cluster(worker, case)


def on_replicas(case, batches, intent_keys=None):
    """``replication_only``: every rank declares intent for the keys of its batch (or for ``intent_keys``) and waits
    until all of them are local; it reports ``local`` and ``replicas`` (those keys owned by another rank). Ranks 0, 1, 2
    then run their batches (None: nothing) one after another with a settle after each, and every rank reads the rows.
    Per rank: ``local``, ``replicas``, ``loss``, ``stats``, ``outs``, ``rows``."""
    def worker(kv, server, wid):
        rank, b = server.my_rank(), batches[server.my_rank()]
        _loaded(kv, server, case)
        mine = case.keys_of(b) if intent_keys is None else intent_keys
        make_local(kv, server, mine)
        out = {"local": all(server.is_local(int(k)) for k in mine),
               "replicas": sum(server.owner_of(int(k)) != rank for k in mine), "outs": []}
        step = case.open(server, kv)
        stream = torch.cuda.Stream(server.device)
        for turn in range(WORLD):
            if turn == rank and b is not None:
                out["outs"] = _steps(step, [b], stream)
            settle(kv)
        out["loss"], out["stats"] = step.totals()
        out["rows"] = pull_rows(kv, case.init)
        kv.barrier()
        kv.finalize()
        return out

    return _cluster(worker, case, "replication_only")


def while_keys_move(case, steps, technique):
    """Ranks 0 and 1 keep relocating every key of ``case.init`` between them (``mover``); rank 2 runs ``steps`` one after
    another, each followed by a pause of ``PACE_S``. After eight clock advances and a settle, rank 2 reads the rows.
    Rank 2 reports ``loss``, ``stats``, ``outs`` and ``rows``."""
    done = threading.Event()

    def worker(kv, server, wid):
        rank = server.my_rank()
        _loaded(kv, server, case)
        out = {}
        if rank < 2:
            out["iters"] = mover(kv, rank, torch.cat([k for k, _ in case.init]), done)
        else:
            try:
                step = case.open(server, kv)
                out["outs"] = _steps(step, steps, torch.cuda.Stream(server.device), PACE_S)
            finally:
                done.set()
            out["loss"], out["stats"] = step.totals()
        kv.barrier()
        for _ in range(8):
            kv.advance_clock()
        settle(kv)
        if rank == 2:
            out["rows"] = pull_rows(kv, case.init)
        kv.barrier()
        kv.finalize()
        return out

    return _cluster(worker, case, technique)


def _same(got, want):
    if isinstance(want, tuple):
        return all(torch.equal(a.cpu(), b) for a, b in zip(got, want))
    return torch.equal(got.cpu(), want)


def reads_while_keys_move(case, read, expected, block, technique, min_reps=8, max_reps=200):
    """Ranks 0 and 1 keep relocating ``block`` between them; nobody writes a row, so every result has one exact
    expectation. ``read(server, kv, stats)`` returns a function that runs the read-only op once and returns
    ``{name: tensor or tuple of tensors}``; rank 2 repeats it at least ``min_reps`` times over at least ``READ_MIN_S``
    (at most ``max_reps`` times) and records ``(repetition, name)`` for every result that differs from ``expected``
    (the same names, on the host). Uses ``case``'s store and ``init`` only. Rank 2 reports ``mism``, ``reps`` and
    ``stats``."""
    done = threading.Event()

    def worker(kv, server, wid):
        rank = server.my_rank()
        _loaded(kv, server, case)
        out = {}
        if rank < 2:
            out["iters"] = mover(kv, rank, block, done)
        else:
            stream = torch.cuda.Stream(server.device)
            stats = torch.zeros(4, dtype=torch.int64, device=server.device)
            mism, reps = [], 0
            try:
                with torch.cuda.stream(stream):
                    once = read(server, kv, stats)
                    t0 = time.time()
                    while (reps < min_reps or time.time() - t0 < READ_MIN_S) and reps < max_reps:
                        mism += [(reps, k) for k, v in once().items() if not _same(v, expected[k])]
                        reps += 1
                stream.synchronize()
            finally:
                done.set()
            out.update(mism=mism, reps=reps, stats=stats.tolist())
        kv.barrier()
        settle(kv)
        kv.finalize()
        return out

    return _cluster(worker, case, technique)


def rejected_on_ranks(*calls, world=2, value_lengths=16, num_keys=64, match=""):
    """Whether every ``call(server)`` raises ``ValueError`` (with ``match`` in its message) on every rank of a
    ``world``-rank store."""
    def worker(kv, server, wid):
        raised = []
        for call in calls:
            try:
                call(server)
                raised.append(False)
            except ValueError as e:
                raised.append(match in str(e))
        kv.barrier()
        kv.finalize()
        return {"raised": all(raised)}

    res = _cluster(worker, Case(value_lengths, num_keys, []), world=world)
    return all(r["raised"] for r in res)
