"""Multi-GPU contract tests: one process per GPU (shm control block + CUDA-IPC peer-mapped heaps),
i.e. the production topology. Needs >= 2 visible GPUs; skipped on a single-GPU machine."""
import pytest
import torch

from harness import run_cluster
import test_contract_dynamic as dyn
import test_contract_locality as loc
import test_contract_many_keys as mk

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                                 reason="needs at least 2 GPUs")]


def _errs(res):
    return [e for r in res.values() for k, v in r.items() if k != "counters" for e in v]


def _world(n):
    return min(n, torch.cuda.device_count())


def test_locality_api_multi_gpu():
    if torch.cuda.device_count() < 3:
        pytest.skip("the locality contract is written for exactly 3 nodes")
    res = run_cluster(loc._worker, world=3, workers=loc.NUM_LOCAL, mode="procs", value_lengths=1, num_keys=12,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))


def test_dynamic_allocation_multi_gpu():
    world, workers = _world(4), 2
    res = run_cluster(dyn._dyn_worker, world=world, workers=workers, mode="procs", value_lengths=2, num_keys=20,
                      dtype="float32", backend="cuda")
    total = world * workers * dyn.RUNS
    assert res[0][0] == [total, 2 * total], f"lost or duplicated updates: {res[0][0]}"
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


def test_many_key_operations_multi_gpu():
    res = run_cluster(mk._worker, world=_world(4), workers=2, mode="procs", value_lengths=mk.VPK, num_keys=mk.NUM_KEYS,
                      dtype="float32", backend="cuda")
    assert not _errs(res), "\n".join(_errs(res))
    assert all(r["counters"]["protocol_errors"] == 0 for r in res.values())


def _sgns_remote_worker(kv, server, wid):
    """Each rank runs the fused SGNS step on its own disjoint key set without any intent: about half of the rows
    are owned by the peer GPU, so the row loads (TMA / LDG over NVLink) and the 16-byte reductions into peer HBM are
    exercised; rank 0 then checks every row against the PyTorch fp32 formula."""
    import torch
    from adapm_b200.ops import sgns_step

    d, neg, B = 128, 5, 64
    world, rank = server.num_servers(), server.my_rank()
    per_rank = 2 * (B * (neg + 2) + 10)
    n_keys = per_rank * world
    g = torch.Generator().manual_seed(1234)
    rows = torch.empty(n_keys, 2 * d)
    rows[:, :d] = torch.randn(n_keys, d, generator=g) * 0.3
    rows[:, d:] = torch.rand(n_keys, d, generator=g) + 1e-3
    allk = torch.arange(n_keys)
    if wid == 0:
        kv.set(allk, rows.clone().view(-1))
    kv.waitall(); kv.barrier()
    dev = server.device
    calls = []
    for r in range(world):   # every rank derives all ranks' batches (needed for the reference on rank 0)
        gr = torch.Generator().manual_seed(77 + r)
        perm = torch.randperm(per_rank // 2, generator=gr) + r * (per_rank // 2)
        centers = 2 * perm[:B]
        tw = perm[B:B + B * (neg + 1)].view(B, neg + 1)
        calls.append((centers, 2 * tw[:, 0] + 1, 2 * tw[:, 1:] + 1))
    centers, contexts, negatives = calls[rank]
    loss = torch.zeros(1, device=dev)
    stats = torch.zeros(4, dtype=torch.int64, device=dev)
    for impl in ("tma", "ldg"):
        sgns_step(server, centers.to(dev), contexts.to(dev), negatives.contiguous().to(dev), d, 0.05, loss, stats, impl=impl)
    torch.cuda.synchronize()
    kv.barrier()
    out = {"stats": stats.tolist()}
    if wid == 0:
        got = torch.empty(n_keys * 2 * d)
        kv.pull(allk, got)
        ref = rows.clone()
        for _ in range(2):          # two steps (tma, ldg), applied sequentially by every rank on disjoint keys
            snap = ref.clone()
            for (c, ctx, ng) in calls:
                e0, a0 = snap[c, :d], snap[c, d:]
                tk = torch.cat([ctx.view(B, 1), ng], 1)
                e1, a1 = snap[tk][:, :, :d], snap[tk][:, :, d:]
                label = torch.zeros(B, neg + 1); label[:, 0] = 1
                f = (e0.unsqueeze(1) * e1).sum(-1)
                gs = label - torch.sigmoid(f)
                gs = torch.where(f > 6, label - 1, gs); gs = torch.where(f < -6, label, gs)
                grad0 = (gs.unsqueeze(-1) * e1).sum(1)
                grad1 = gs.unsqueeze(-1) * e0.unsqueeze(1)
                ref[c, :d] += 0.05 * grad0 / torch.sqrt(a0 + grad0 ** 2); ref[c, d:] += grad0 ** 2
                ue = 0.05 * grad1 / torch.sqrt(a1 + grad1 ** 2)
                ref.index_put_((tk.reshape(-1),), torch.cat([ue, grad1 ** 2], -1).view(-1, 2 * d), accumulate=True)
        out["max_err"] = float((got.view(n_keys, 2 * d) - ref).abs().max())
    kv.barrier()
    kv.finalize()
    return out


def test_sgns_step_over_nvlink_matches_reference():
    world = 2
    d, neg, B = 128, 5, 64
    per_rank = 2 * (B * (neg + 2) + 10)
    res = run_cluster(_sgns_remote_worker, world=world, workers=1, mode="procs", value_lengths=2 * d,
                      num_keys=per_rank * world, dtype="float32", backend="cuda")
    assert res[0][0]["max_err"] < 5e-4, res[0][0]
    for r in res.values():
        st = r[0]["stats"]
        assert st[1] > 0 and st[2] == 0, f"expected remote rows and no slow path: {st}"
