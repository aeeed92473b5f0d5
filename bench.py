#!/usr/bin/env python
"""Headline benchmark: word2vec SGNS updates/s on the intent-driven parameter manager.

    python bench.py --gpus N --steps K --warmup W [--impl native|reference|nccl] [--config word2vec]

Metric (BASELINE.json / BASELINE.md section 3): *updates/s*, an update = one (key,row) additive
update applied at the key's current owner; word2vec SGNS applies ``1 + (negative + 1)`` updates per
(center, context) pair. Config #2 of BASELINE.json: 1M-word vocabulary, d = 300, fp32 rows
``[embedding | AdaGrad]`` (2 400 B), negative = 25 (reference default, apps/word2vec.cc:1037),
Intent look-ahead + local PullSample. Synthetic Zipf corpus, random-init weights.

Two numbers are measured back to back after W warm-up steps, both with CUDA events on the
launching stream bracketed by barrier + synchronize, max over ranks:

* ``value``     device-resident inputs, K steps of {sampler kernel, fused SGNS kernel};
* ``e2e.value`` the public-API loop a user writes: every step copies that step's key batch from
                pinned host memory (H2D), signals intent for a future batch, advances the clock,
                runs the step and copies the loss back to pinned host memory (D2H).

For N > 1 launch with torchrun (one rank per GPU); weak scaling (fixed pairs per GPU per step).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="native", choices=["native", "reference", "nccl"])
    ap.add_argument("--config", default="word2vec", choices=["word2vec", "kge", "mf", "ctr"],
                    help="word2vec = BASELINE config #2 (the headline); kge / mf / ctr = configs #3 / #4 / #5 (benchmarks/configs.py)")
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--negative", type=int, default=25)
    ap.add_argument("--batch-pairs", type=int, default=32768)
    ap.add_argument("--read-ahead", type=int, default=32, help="intent look-ahead in steps (the reference reads 1000 sentences ahead)")
    ap.add_argument("--placement-steps", type=int, default=-1,
                    help="untimed training steps before the W warm-up steps that let the adaptive placement reach its steady "
                         "state (N > 1 only; default: 8 x read-ahead, 0 for N = 1)")
    ap.add_argument("--max-inflight", type=int, default=3, help="steps the host may run ahead of the GPU")
    ap.add_argument("--sampling", default="local", choices=["local", "naive"])
    ap.add_argument("--techniques", default="all")
    ap.add_argument("--no-intent", action="store_true")
    ap.add_argument("--sync-per-sec", type=float, default=1000)
    ap.add_argument("--loop", default="native", choices=["native", "python"],
                    help="who issues the steps of the timed loops: the C++ step driver (ops.SgnsLoop, GIL released) or a Python "
                         "loop over the same public calls")
    ap.add_argument("--profile", action="store_true", help="also report per-kernel device times")
    ap.add_argument("--intent-prepass", action="store_true",
                    help="experimental: device-side Intent for keys that are already local (ops.IntentPrepass)")
    ap.add_argument("--opt", action="append", default=[], metavar="KEY=VALUE",
                    help="extra server option (e.g. --opt sys.sync.idle_period=1); repeatable")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed as DIR/<name>.npy: its loss and "
                         "the rows of a fixed, seeded sample of keys (rank 0; word2vec only). On one GPU the same "
                         "arguments give the same inputs and the same outputs in every run")
    return ap.parse_args()


class ClockSampler:
    """Samples SM clocks / throttle reasons with nvidia-smi DURING the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx, self.p = gpu_index, None

    def start(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                       "-lms", "20", "-i", str(self.idx)], stdout=subprocess.PIPE,
                                      stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.p = None

    def stop(self):
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.p.terminate()
        try:
            out = self.p.communicate(timeout=5)[0]
        except Exception:
            out = ""
        sm, mx, reasons = [], [], set()
        for line in out.strip().splitlines():
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def reference_arm(args):
    # The reference (alexrenz/AdaPM) is a CPU-only C++14 project that needs libzmq, protobuf-lite,
    # Boost and Eigen headers; none is present in this offline image and pip cannot install it
    # (no setup.py at the root; bindings/setup.py fails compiling against missing zmq.h). See DESIGN.md.
    if int(os.environ.get("RANK", "0")) == 0:      # one line per job, also when launched with torchrun
        print(json.dumps({"impl": "reference", "unavailable":
                          "alexrenz/AdaPM needs libzmq+protoc/protobuf+Boost+Eigen (absent offline); it has no GPU path at all"}))
    return 0


def dump_outputs(out_dir, model, worker, last_batch, cfg, rank):
    """What the last timed step computed, as a caller of the step sees it: the step's summed logistic loss and the
    [embedding | AdaGrad] rows of 2048 keys of that step's batch plus 2048 keys of the whole table (fixed seed)."""
    import numpy as np
    import torch

    loss = float(model.loss.item())
    g = torch.Generator().manual_seed(0)
    batch_keys = torch.unique(last_batch.view(-1).cpu())
    keys = torch.cat([batch_keys[torch.randperm(batch_keys.numel(), generator=g)[:2048]],
                      torch.randint(0, cfg.num_keys, (2048,), generator=g)])
    keys = torch.unique(keys)
    rows = torch.empty(keys.numel(), cfg.row_len, dtype=torch.float32)
    worker.pull(keys, rows)
    if rank != 0:
        return
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.array([loss], dtype=np.float64))
    np.save(os.path.join(out_dir, "row_keys.npy"), keys.numpy().astype(np.float64))
    np.save(os.path.join(out_dir, "rows.npy"), rows.numpy())


def main():
    args = parse_args()
    if args.dump_outputs and (args.impl != "native" or args.config != "word2vec"):
        sys.exit("--dump-outputs is implemented for the native word2vec run")
    if args.impl == "reference":
        return reference_arm(args)

    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            sys.exit("bench.py --gpus N with N>1 must be launched with torch.distributed.run (one rank per GPU)")
        args.gpus = world
    if not torch.cuda.is_available():
        sys.exit("bench.py needs a CUDA device")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_DEBUG", "WARN")   # keep stdout to the one JSON line (NCCL prints its version banner there)
        dist.init_process_group("nccl", device_id=dev)

    def barrier():
        if world > 1:
            dist.barrier(device_ids=[local_rank])
        torch.cuda.synchronize()

    if args.impl == "nccl":
        from adapm_b200.parallel.nccl_baseline import run_nccl_word2vec

        return run_nccl_word2vec(args, rank, world, local_rank)
    if args.config != "word2vec":
        from benchmarks.configs import run as run_config

        rc = run_config(args.config, args, rank, world, local_rank, ClockSampler)
        if world > 1:
            dist.destroy_process_group()
        return rc

    import adapm_b200 as ad
    from adapm_b200 import _C
    from adapm_b200.models.word2vec import SyntheticPairs, Word2Vec, Word2VecConfig, zipf_counts

    cfg = Word2VecConfig(vocab_size=args.vocab, embed_dim=args.dim, negative=args.negative,
                         batch_pairs=args.batch_pairs, read_ahead=args.read_ahead, sampling_scheme=args.sampling,
                         signal_intent=not args.no_intent, max_inflight=args.max_inflight,
                         intent_prepass=args.intent_prepass)
    server = ad.Server(cfg.row_len, num_keys=cfg.num_keys, num_threads=1, rank=rank, world=world, backend="cuda",
                       fabric="shm" if world > 1 else "inproc", device=local_rank,
                       options=dict({"sys.techniques": args.techniques, "sys.sync.max_per_sec": args.sync_per_sec},
                                    **dict(kv.split("=", 1) for kv in args.opt)))
    worker = ad.Worker(0, server)
    counts = zipf_counts(cfg.vocab_size, cfg.zipf_exponent)
    model = Word2Vec(server, worker, cfg, counts)
    model.init_model()
    data = SyntheticPairs(cfg, counts, rank, seed=1)

    K, W, RA = args.steps, args.warmup, cfg.read_ahead
    # Steady state: a parameter manager adapts its placement to the access pattern, so the first steps of a job run on
    # a cold placement (every non-home row has to be requested once). P untimed training steps - same loop, same API -
    # precede the W warm-up steps; nothing is pre-localised outside the loop and timing starts more than RA steps after
    # the first intent, i.e. every timed step works on rows whose intent was signalled RA steps earlier INSIDE the loop.
    P = args.placement_steps if args.placement_steps >= 0 else (8 * RA if world > 1 else 0)
    n_prof = 640 if args.profile else 0
    total_steps = P + W + K + 3 + K + n_prof   # placement + warm-up + e2e loop + device-resident loop (+ profiling)
    # data loader: batches are read ahead into pinned host memory (the reference reads sentences ahead too). Every step
    # has its own batch (no ring that would re-use localised rows) up to 2048 batches = 1 GB of pinned keys.
    n_batches = min(total_steps + RA + 2, 2048)
    ring = [data.batch(s).pin_memory() for s in range(n_batches)]
    for b_ in ring:
        # like the native loader (utils.text.NativeCorpus.pair_batches): every batch carries its distinct keys, which is
        # what Intent() is called with - deduplication belongs to the loader thread, not to the training loop
        b_.unique_keys = torch.unique(b_)

    class _Batches:
        def __len__(self):
            return total_steps + RA + 2

        def __getitem__(self, i):
            if isinstance(i, slice):
                return [ring[j % len(ring)] for j in range(*i.indices(len(self)))]
            return ring[i % len(ring)]

    batches = _Batches()
    loss_host = torch.zeros(total_steps + 1, dtype=torch.float32).pin_memory()
    stream = torch.cuda.current_stream()

    # device-resident inputs of the second timed loop: exactly the batches of its steps (+ profiling windows)
    dev_first = P + W + K
    dev_ring = {s: batches[s].to(dev) for s in range(dev_first, min(total_steps, dev_first + 3 + K + n_prof))}
    from adapm_b200.ops import sgns_step

    def dev_batch(s):
        t = dev_ring.get(s)
        return t if t is not None else batches[s].to(dev)

    def train_step(s, resident):
        """One training step through the public API. resident=False: this step's key batch is copied
        from pinned host memory (H2D) and the loss is copied back (D2H); resident=True: the batch is
        already on the device and the loss stays there. Everything else is identical."""
        if s + RA < len(batches):
            model.signal_intent(batches[s + RA], worker.current_clock() + RA)
        model.loss.zero_()
        if resident:
            model.step_resident(dev_batch(s))
        else:
            model.step(batches[s])                                       # (prefetched) H2D copy + sampler + fused step
            loss_host[s:s + 1].copy_(model.loss, non_blocking=True)      # D2H read of the step result
            model.prefetch(batches[s + 1])                               # H2D of the next step's keys (copy stream)
        worker.advance_clock()

    native = args.loop == "native"
    host_list = [batches[i] for i in range(len(batches))]
    dev_list = [dev_ring.get(i) for i in range(len(batches))]

    def run_range(first, n, resident):
        """Steps first .. first+n-1: one call into the C++ step driver, or the Python loop over the same public calls."""
        if native:
            model.run_steps(dev_list if resident else host_list, first, n, resident=resident,
                            loss_host=None if resident else loss_host, intent_batches=host_list)
        else:
            for s_ in range(first, first + n):
                train_step(s_, resident)

    # ---------------- placement steps + warm-up: the same loop as the timed one
    for s in range(min(RA, len(batches))):
        model.signal_intent(batches[s], worker.current_clock() + s)     # the first RA steps have no earlier step to signal them
    run_range(0, P + W, False)
    barrier()
    counters0 = server.counters()
    stats0 = model.stats.tolist()

    sampler = ClockSampler(local_rank)
    if rank == 0 and not os.environ.get("ADAPM_BENCH_NO_SMI"):
        sampler.start()

    # ---------------- e2e timed region
    launches0 = _C.kernel_launches()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    ev0.record(stream)
    t_host0 = time.perf_counter()
    run_range(P + W, K, False)
    host_ms = (time.perf_counter() - t_host0) * 1e3 / K
    ev1.record(stream)
    barrier()
    e2e_ms = ev0.elapsed_time(ev1)
    launches_e2e = _C.kernel_launches() - launches0

    # ---------------- device-resident timed region (same loop, inputs already on the device)
    run_range(P + W + K, 3, True)
    barrier()
    launches1 = _C.kernel_launches()
    ev2, ev3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    ev2.record(stream)
    run_range(P + W + K + 3, K, True)
    ev3.record(stream)
    barrier()
    dev_ms = ev2.elapsed_time(ev3)
    launches_dev = _C.kernel_launches() - launches1
    counters1 = server.counters()
    stats1 = model.stats.tolist()
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, model, worker, batches[P + W + 2 * K + 2], cfg, rank)
    if rank == 0 and sampler.p is None:
        clocks = {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["clock sampling disabled (ADAPM_BENCH_NO_SMI)"]}

    # ---------------- optional: per-kernel device times (outside the timed regions)
    prof = None
    if args.profile:
        # diagnostic: the device-resident loop once more, now without the nvidia-smi clock sampler running
        PB = P + W + 2 * K
        base = PB + 3
        ev4, ev5 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        ev4.record(stream)
        for s in range(base, base + 100):
            train_step(s, True)
        ev5.record(stream)
        barrier()
        second_pass_ms = ev4.elapsed_time(ev5) / 100
        evs = []
        for s in range(PB + 103, PB + 143):
            a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            if s + RA < len(batches):
                model.signal_intent(batches[s + RA], worker.current_clock() + RA)
            kb = dev_batch(s)
            a.record(stream)
            model.sample_negatives()
            b.record(stream)
            sgns_step(server, kb[0], kb[1], model._neg, cfg.embed_dim, model.alpha, model.loss, model.stats)
            c.record(stream)
            worker.advance_clock()
            evs.append((a, b, c))
            if len(evs) % 2 == 0:
                c.synchronize()
        torch.cuda.synchronize()
        prof = {"sampler_ms": statistics.mean(a.elapsed_time(b) for a, b, c in evs),
                "sgns_ms": statistics.mean(b.elapsed_time(c) for a, b, c in evs),
                "sgns_ms_max": max(b.elapsed_time(c) for a, b, c in evs)}
        # host-side breakdown of the e2e loop (where does the Python thread spend its time?)
        sec = {"intent": 0.0, "wait_gpu": 0.0, "launch": 0.0, "d2h": 0.0, "prefetch": 0.0, "clock": 0.0}
        NP = 100
        pc = time.perf_counter
        for s in range(PB + 143, PB + 143 + NP):
            t0 = pc()
            if s + RA < len(batches):
                model.signal_intent(batches[s + RA], worker.current_clock() + RA)
            t1 = pc()
            ev = model._events[model.step_no % len(model._keys_dev)]
            if ev is not None:
                ev.synchronize()
            t2 = pc()
            model.loss.zero_()
            model.step(batches[s])
            t3 = pc()
            loss_host[s:s + 1].copy_(model.loss, non_blocking=True)
            t4 = pc()
            model.prefetch(batches[s + 1])
            t5 = pc()
            worker.advance_clock()
            t6 = pc()
            for k_, v_ in zip(sec, (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t5 - t4, t6 - t5)):
                sec[k_] += v_ * 1e3 / NP
        torch.cuda.synchronize()
        prof["host_ms"] = {k_: round(v_, 4) for k_, v_ in sec.items()}
        prof["cpus"] = len(os.sched_getaffinity(0))
        prof["resident_ms_without_clock_sampler"] = second_pass_ms
        # per-step device time distribution (steady contention or periodic stalls?) and the same loop with
        # intent signalling switched off (how much of the step time is relocation/replication churn?)
        tracing = bool(os.environ.get("ADAPM_SYNC_TRACE"))

        def per_step(first, n, intent):
            st0 = model.stats.tolist()
            marks = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
            barrier()
            marks[0].record(stream)
            for i, s in enumerate(range(first, first + n)):
                if intent and s + RA < len(batches):
                    model.signal_intent(batches[s + RA], worker.current_clock() + RA)
                model.loss.zero_()
                if tracing:
                    server._impl.trace_mark("step_begin", stream.cuda_stream)
                model.step_resident(dev_batch(s))
                if tracing:
                    server._impl.trace_mark("step_end", stream.cuda_stream)
                worker.advance_clock()
                marks[i + 1].record(stream)
            barrier()
            ts = sorted(marks[i].elapsed_time(marks[i + 1]) for i in range(n))
            st1 = model.stats.tolist()
            rows = [b_ - a_ for a_, b_ in zip(st0, st1)][:3]
            return {"mean": round(sum(ts) / n, 4), "p10": round(ts[n // 10], 4), "p50": round(ts[n // 2], 4),
                    "p90": round(ts[9 * n // 10], 4), "max": round(ts[-1], 4),
                    "rows_local_remote_slow": rows}
        first = PB + 243
        prof["steps_with_intent"] = per_step(first, 192, True)
        if tracing:   # kernel timeline of the round kernels and the steps, one file per rank
            os.makedirs("gpurun_out", exist_ok=True)
            server._impl.dump_trace(f"gpurun_out/kernel_trace.rank{rank}.tsv")
        prof["steps_without_intent"] = per_step(first + 192, 192, False)

    # max over ranks
    t = torch.tensor([e2e_ms, dev_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_ms, dev_ms = t.tolist()
    stats = model.stats.tolist()
    counters = server.counters()

    updates_per_step = world * cfg.batch_pairs * cfg.updates_per_pair
    value = updates_per_step * K / (dev_ms * 1e-3)
    e2e_value = updates_per_step * K / (e2e_ms * 1e-3)
    h2d = cfg.batch_pairs * 2 * 8
    if rank == 0:
        here = os.path.dirname(os.path.abspath(__file__))
        row_bytes = cfg.row_len * 4
        bytes_per_update = 2 * row_bytes  # read row + reduce row
        try:
            peaks = json.load(open(os.path.join(here, "MEASURED_PEAKS.json")))
            hbm = peaks["hbm_gbs"]
            denom = "measured"
        except Exception:
            hbm, denom = 3350.0, "H100 SXM data sheet"
        # same-box anchor: the NCCL-only arm (bench.py --impl nccl, stock PyTorch ops + all_to_all), measured on this pool
        # and recorded in baseline/nccl_arm.json by N (BASELINE.md section 6); the reference itself cannot be built
        vs_baseline, anchor = None, None
        try:
            arm = json.load(open(os.path.join(here, "baseline", "nccl_arm.json")))
            anchor = arm["updates_per_s"].get(str(world))
            if anchor:
                vs_baseline = value / anchor
        except Exception:
            pass
        # traffic of rank 0 inside the two timed loops (+ 3 steps between them), per step
        n_steps_win = 2 * K + 3
        dstat = [b_ - a_ for a_, b_ in zip(stats0, stats1)]
        dcnt = {k: counters1[k] - counters0[k] for k in counters1 if isinstance(counters1[k], int) and k in counters0}
        nv_step = (2 * dstat[1] * row_bytes                                             # fused step: remote row load + reduction
                   + (dcnt.get("refreshes", 0) + dcnt.get("relocations", 0)) * row_bytes  # round: owner row reads
                   + dcnt.get("deltas_shipped", 0) * row_bytes) / n_steps_win            # round: replica deltas (reductions)
        link_gbs = 450.0   # NVLink 4 data-sheet rate, one direction, per H100 SXM (not a measured copy rate)
        nv_time_ms = nv_step / (link_gbs * 1e9) * 1e3
        hbm_time_ms = cfg.batch_pairs * cfg.updates_per_pair * bytes_per_update / (hbm * 1e9) * 1e3
        out = {
            "metric": "word2vec SGNS updates/sec (device-timed, max over ranks)",
            "value": value, "unit": "updates/s", "n_gpus": world, "steps": K, "warmup": W,
            "ms_per_step": dev_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": vs_baseline,
            "dtype": "fp32", "data": "synthetic", "impl": "native",
            "config": {"model": "word2vec SGNS 1M-vocab d=300 (rows = [embedding|AdaGrad], 2400 B fp32)",
                       "vocab": cfg.vocab_size, "embed_dim": cfg.embed_dim, "negative": cfg.negative,
                       "global_batch": world * cfg.batch_pairs, "batch_pairs_per_gpu": cfg.batch_pairs,
                       "seq_len": None, "updates_per_pair": cfg.updates_per_pair,
                       "parallelism": f"pm{world} (key-sharded store, intent-driven relocation/replication)",
                       "sampling": cfg.sampling_scheme, "intent_read_ahead": RA,
                       "step_loop": "C++ step driver (ops.SgnsLoop, GIL released)" if native else "Python loop",
                       "placement_steps": P,
                       "placement_note": "P untimed training steps (same loop) run before the W warm-up steps so that the "
                                         "adaptive placement is in steady state; nothing is localised outside the loop",
                       "intent_keys": "distinct keys of the batch, prepared by the loader (outside the step loop)",
                       "l2": f"inputs larger than L2: 4.8 GB table; every step has its own random batch "
                             f"({len(ring)} distinct batches, {'no wrap' if len(ring) >= total_steps + RA + 2 else 'wraps'})",
                       "vs_baseline_anchor": ("bench.py --impl nccl on the same pool: %.4g updates/s at N=%d "
                                              "(baseline/nccl_arm.json)" % (anchor, world)) if anchor else None,
                       "note": "reference dtype is float32 (apps/word2vec.cc:40); rows stay fp32 for exact additive updates"},
            "e2e": {"value": e2e_value, "unit": "updates/s", "ms_per_step": e2e_ms / K,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4},
            "gpu_launches": int(launches_dev), "gpu_launches_e2e": int(launches_e2e),
            "clocks": clocks,
            "roofline": {"hbm_bytes_per_update": bytes_per_update,
                         "achieved_hbm_gbs_per_gpu": value / world * bytes_per_update / 1e9,
                         "fraction_of_hbm_peak": value / world * bytes_per_update / 1e9 / hbm, "peak": denom,
                         "nvlink_bytes_per_step_per_gpu": nv_step, "nvlink_gbs_per_gpu": nv_step / (dev_ms / K * 1e-3) / 1e9,
                         "nvlink_fraction_of_link": nv_step / (dev_ms / K * 1e-3) / 1e9 / link_gbs,
                         "roofline_ms_per_step": max(nv_time_ms, hbm_time_ms),
                         "fraction_of_roofline": max(nv_time_ms, hbm_time_ms) / (dev_ms / K),
                         "note": "roofline = slower of (algorithmic HBM bytes / measured copy bandwidth) and (bytes that "
                                 "crossed NVLink / 450 GB/s data-sheet rate); rank 0's counters over both timed loops"},
            "locality": {"rows_local": dstat[0], "rows_remote": dstat[1], "rows_slow_path": dstat[2]},
            "pm": {k: dcnt.get(k, 0) for k in ("relocations", "replica_setups", "replica_drops", "refreshes",
                                                "deltas_shipped", "sync_rounds", "protocol_errors")},
            "profile": prof, "host_loop_ms_per_step": host_ms,
            "host_loop_note": ("wall time of the e2e loop per step as seen by the calling thread. With --loop native it is "
                               "NOT host work: the C++ step driver blocks on its bounded run-ahead (max_inflight steps), "
                               "so it tracks the GPU step time; no Python runs inside the loop"
                               if args.loop == "native" else "Python loop: host work + waits of the bounded run-ahead"),
            "sync_report": server._impl.sync_report() if world > 1 else None,
            "loss_last": float(loss_host[P + W + K - 1]) / max(1, cfg.batch_pairs * (cfg.negative + 1)),
        }
        print(json.dumps(out))
    worker.finalize()
    server.shutdown()
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
