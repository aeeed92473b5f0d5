"""The CPU contract tests re-run on the CUDA backend: several logical ranks share one GPU
(inproc fabric), so the full relocation/replication protocol runs through the sm_90a kernels
with peer pointers that happen to live on the same device."""
import pytest

from harness import run_cluster
import test_contract_dynamic as dyn
import test_contract_locality as loc
import test_contract_many_keys as mk

pytestmark = pytest.mark.gpu


def _errs(res):
    return [e for r in res.values() for k, v in r.items() if k != "counters" for e in v]


def test_locality_api_cuda():
    res = run_cluster(loc._worker, world=3, workers=loc.NUM_LOCAL, mode="threads", value_lengths=1, num_keys=12,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))


@pytest.mark.parametrize("technique", ["all", "replication_only", "relocation_only"])
def test_dynamic_allocation_cuda(technique):
    world, workers = 3, 2
    res = run_cluster(dyn._dyn_worker, world=world, workers=workers, mode="threads", value_lengths=2, num_keys=20,
                      dtype="float32", backend="cuda", options={"sys.techniques": technique})
    total = world * workers * dyn.RUNS
    assert res[0][0] == [total, 2 * total], f"lost or duplicated updates: {res[0][0]}"
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())
    moved = sum(r["counters"]["relocations"] + r["counters"]["replica_setups"] for r in res.values())
    assert moved > 0


@pytest.mark.parametrize("technique", ["all", "replication_only", "relocation_only"])
def test_many_key_operations_cuda(technique):
    res = run_cluster(mk._worker, world=4, workers=2, mode="threads", value_lengths=mk.VPK, num_keys=mk.NUM_KEYS,
                      dtype="float32", backend="cuda", options={"sys.techniques": technique})
    errs = _errs(res)
    if technique == "relocation_only":
        errs = [e for e in errs if "were not local" not in e]
    assert not errs, "\n".join(errs)
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


def test_set_operation_cuda():
    res = run_cluster(dyn._set_worker, world=4, workers=2, mode="threads", value_lengths=2, num_keys=20,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))


def test_set_under_relocation_cuda():
    """Set on keys that two other ranks keep relocating: the kernel reports keys in flight and the worker repeats them
    after a round (the device-side grace period would otherwise wait for a kernel that waits for the round)."""
    res = run_cluster(dyn._set_under_relocation_worker, world=3, workers=1, mode="threads", value_lengths=2,
                      num_keys=dyn.SET_KEYS + 8, dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


def test_host_sequenced_round_cuda(monkeypatch):
    """ADAPM_HOST_ROUND=1 keeps the host-sequenced round (control-plane barriers, event-based grace) working."""
    monkeypatch.setenv("ADAPM_HOST_ROUND", "1")
    res = run_cluster(mk._worker, world=3, workers=2, mode="threads", value_lengths=mk.VPK, num_keys=mk.NUM_KEYS,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))


def test_many_distinct_value_lengths_cuda():
    """More distinct value lengths than size classes: keys of different lengths share a slab class (per-key length table)."""
    import torch

    nk = 150
    lens = torch.tensor([(k * 7) % 97 + 1 for k in range(nk)], dtype=torch.int64)
    res = run_cluster(loc._many_lengths_worker, world=3, workers=2, mode="threads", value_lengths=lens, num_keys=nk,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


@pytest.mark.parametrize("dtype", ["int64", "float64"])
def test_exact_value_types_cuda(dtype):
    """The reference's contract tests use `long` values so that sums are exact (tests/test_many_key_operations.cc:11) and
    its applications `double`: both run on the CUDA backend through the generic Pull/Push/Set kernels and the sync
    round (element-wise protocol path; the fused application kernels are float32)."""
    res = run_cluster(mk._worker, world=3, workers=2, mode="threads", value_lengths=mk.VPK, num_keys=mk.NUM_KEYS,
                      dtype=dtype, backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())
    world, workers = 3, 2
    res = run_cluster(dyn._dyn_worker, world=world, workers=workers, mode="threads", value_lengths=2, num_keys=20,
                      dtype=dtype, backend="cuda")
    total = world * workers * dyn.RUNS
    assert res[0][0] == [total, 2 * total], f"lost or duplicated updates: {res[0][0]}"


PP_KEYS = 96


def _prepass_worker(kv, server, wid):
    """Device-side Intent pre-pass (ops_intent.cu): keys with a usable local slot only get their end clock extended on the
    device, the others come back in a compacted list and go through Worker.intent."""
    import torch

    from adapm_b200.ops import IntentPrepass

    rank, world = server.my_rank(), server.num_servers()
    errors = []
    keys = torch.arange(PP_KEYS, dtype=torch.int64)
    kv.wait(kv.push(keys, torch.ones(PP_KEYS * 2, dtype=server.dtype)))
    kv.barrier()
    pp = IntentPrepass(server, kv, max_keys=PP_KEYS + 2)
    local0 = sum(1 for k in range(PP_KEYS) if server.is_local(k))
    # 1) first submission: exactly the keys that are not local yet go to the host path
    pp.submit(keys.to(server.device), kv.current_clock(), kv.current_clock() + 1000)
    pp.harvest(block=True)
    if pp.keys_to_host != PP_KEYS - local0:
        errors.append(f"rank {rank}: {pp.keys_to_host} keys went to the host, {PP_KEYS - local0} are not local")
    kv.wait_sync(); kv.barrier()
    kv.wait_sync(); kv.barrier()
    # 2) every key is local now (replica or relocated): the second submission stays on the device
    before = pp.keys_to_host
    pp.submit(keys.to(server.device), kv.current_clock(), kv.current_clock() + 2000)
    pp.harvest(block=True)
    if pp.keys_to_host != before:
        errors.append(f"rank {rank}: {pp.keys_to_host - before} keys of an all-local batch went to the host path")
    # 3) the extension is honoured: far beyond the first intent's end the keys are still local
    for _ in range(1500):
        kv.advance_clock()
    kv.wait_sync(); kv.barrier()
    kv.wait_sync(); kv.barrier()
    out = torch.zeros(PP_KEYS * 2, dtype=server.dtype)
    kv.wait(kv.pull(keys, out))
    if not torch.equal(out, torch.full_like(out, float(world))):
        errors.append(f"rank {rank}: pulled {out[:6].tolist()}, expected {float(world)}")
    if not kv.pull_if_local(3, torch.zeros(2, dtype=server.dtype)):
        errors.append(f"rank {rank}: key 3 is not local at clock {kv.current_clock()} although the pre-pass extended its intent")
    # 4) an out-of-range key is handed to the host path, which raises like Worker.intent does
    try:
        pp.submit(torch.tensor([1, PP_KEYS + 100], dtype=torch.int64), kv.current_clock(), kv.current_clock() + 1)
        pp.harvest(block=True)
        errors.append("out-of-range key was accepted")
    except Exception:  # noqa
        pass
    kv.barrier()
    kv.finalize()
    return errors


def test_intent_prepass_cuda():
    res = run_cluster(_prepass_worker, world=3, workers=1, mode="threads", value_lengths=2, num_keys=PP_KEYS + 8,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


def test_random_programs_are_exact_cuda():
    """The hypothesis property test of the protocol (tests/test_protocol_property.py: random Intent / device pre-pass /
    Push / Pull / clock / WaitSync programs on 3 ranks stay exact and give read-your-writes) on the CUDA backend with
    int64 rows; derandomized so that every box runs the same programs."""
    import functools

    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st

    import test_protocol_property as prop

    @settings(max_examples=8, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True, database=None)
    @given(programs=st.lists(prop.program, min_size=3, max_size=3),
           technique=st.sampled_from(["all", "replication_only", "relocation_only"]),
           idle_period=st.integers(1, 5), sweep_period=st.integers(0, 4))
    def check(programs, technique, idle_period, sweep_period):
        res = run_cluster(functools.partial(prop._run, programs=programs), world=3, workers=1, mode="threads",
                          value_lengths=prop.VPK, num_keys=prop.NUM_KEYS, dtype="int64", backend="cuda",
                          options={"sys.techniques": technique, "sys.sync.idle_period": idle_period,
                                   "sys.sync.sweep_period": sweep_period})
        total = [0] * prop.NUM_KEYS
        for r in res.values():
            errs, final, mine = r[0]
            assert not errs, errs
            total = [a + b for a, b in zip(total, mine)]
        for r in res.values():
            assert r[0][1] == total, (r[0][1], total)
            assert r["counters"]["protocol_errors"] == 0

    check()
