"""Test harness: run a small parameter-manager cluster on one host.

``mode="threads"``: ranks are threads of this process (inproc fabric).
``mode="procs"``:   ranks are spawned processes (shm fabric) - the torchrun model.

This mirrors how the reference tests run (scheduler + N server processes on loopback,
tests/run_tests.sh:19-53), minus the scheduler, and the assertions of its five test
programs are ported in test_contract_*.py.
"""
from __future__ import annotations

import itertools
import multiprocessing as mp
import os
import threading
import traceback
import uuid

import torch

_job_counter = itertools.count()


def _rank_main(rank, world, workers, fn, server_kwargs, job, fabric, out, setup_fn):
    import adapm_b200 as ad

    errors = []
    results = {}
    try:
        value_lengths = server_kwargs.pop("value_lengths")
        if server_kwargs.get("backend") == "cuda" and fabric == "shm":
            import torch as _t

            server_kwargs["device"] = rank % _t.cuda.device_count()
        server = ad.Server(value_lengths, rank=rank, world=world, num_threads=workers, job=job, fabric=fabric,
                           **server_kwargs)
        if setup_fn is not None:
            setup_fn(server)

        def wmain(cid):
            try:
                w = ad.Worker(cid, server)
                r = fn(w, server, rank * workers + cid)
                results[cid] = r
            except BaseException:  # noqa
                errors.append(traceback.format_exc())

        ths = [threading.Thread(target=wmain, args=(c,)) for c in range(workers)]
        [t.start() for t in ths]
        [t.join() for t in ths]
        results["counters"] = server.counters()
        if not errors:
            server.shutdown()
    except BaseException:  # noqa
        errors.append(traceback.format_exc())
    out.put((rank, results, errors)) if hasattr(out, "put") else out.append((rank, results, errors))


def run_cluster(fn, world, workers, mode="threads", setup_fn=None, timeout=300, **server_kwargs):
    """Runs fn(worker, server, worker_id) on world*workers workers; returns {rank: {cid: result}}."""
    job = f"t{os.getpid()}_{next(_job_counter)}_{uuid.uuid4().hex[:6]}"
    server_kwargs.setdefault("backend", "cpu")
    opts = dict(server_kwargs.pop("options", {}) or {})
    opts.setdefault("wait_timeout_s", 60)
    server_kwargs["options"] = opts
    if mode == "threads":
        out = []
        ths = [threading.Thread(target=_rank_main, args=(r, world, workers, fn, dict(server_kwargs), job, "inproc", out, setup_fn))
               for r in range(world)]
        [t.start() for t in ths]
        [t.join(timeout) for t in ths]
        assert not any(t.is_alive() for t in ths), "cluster timed out"
        res = out
    else:
        # CUDA contexts do not survive fork(): GPU ranks are spawned, one device per rank
        ctx = mp.get_context("spawn" if server_kwargs.get("backend") == "cuda" else "fork")
        q = ctx.Queue()
        ps = [ctx.Process(target=_rank_main, args=(r, world, workers, fn, dict(server_kwargs), job, "shm", q, setup_fn))
              for r in range(world)]
        [p.start() for p in ps]
        res = []
        try:
            for _ in range(world):
                res.append(q.get(timeout=timeout))
        finally:
            for p in ps:
                p.join(10)
                if p.is_alive():
                    p.kill()
    errs = [e for (_, _, es) in res for e in es]
    assert not errs, "\n".join(errs)
    return {rank: results for (rank, results, _) in res}


# The fused training steps launch min(ceil(n / 8), num_sms * cap) blocks of 8 warps and loop over the n calls with a
# grid stride (cap: 16 for MF, 8 for ComplEx, 4 for RESCAL, TransE and RotatE). A test that passes n = WRAP runs
# wrap_calls(WRAP, cap) calls: 2.5 passes of the resident grid, so every warp runs a second call and some a third.
WRAP = "wrap"


def wrap_calls(n, cap):
    if n != WRAP:
        return n
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 5 * sms * cap * 8 // 2
