"""KGE 1vsAll training step on the parameter store, one GPU, FB15k shape (14 951 entities, 1 345 relations).

Arms, alternating in one process, median of ``--runs`` device-synchronised steps after ``--warmup``:
    1vsall   ``ops.kge_1vsall_step``: one Pull of every entity row and the batch's relation rows, the three bf16 wgmma
             contractions with the kernels around them, one Push
    torch    the same rule through PyTorch on the same rows: the same Pull, fp32 matmul, ``log_softmax``, autograd, the
             AdaGrad update in PyTorch, the same Push
    negsamp  the negative-sampling step of the model at the same B (``kge_complex_step`` / ``kge_rescal_step``,
             neg_ratio 6, deterministic), i.e. the other training type, not the same computation

Cases: ComplEx at d 512 and RESCAL at d 64, B = 1024 and 4096 triples (2 B queries). Reported per case: ms per step,
the achieved TFLOP/s of the three contractions (3 * 2 * 2B * N * d_padded over the step time: a whole-step rate, not a
kernel's), and the bytes of the N-row Pull and Push. Each JSON line carries the card's name and power limit, read by
``nvidia-smi`` in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import adapm_b200 as ad  # noqa: E402
from adapm_b200 import ops  # noqa: E402
from adapm_b200.models.kge import KGEConfig, complex_query  # noqa: E402

NE, NR = 14951, 1345


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit_w": float(power)}


def synced(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def alternate(arms: dict, runs: int, warmup: int) -> dict:
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    ts = {k: [] for k in arms}
    for _ in range(runs):
        for k, fn in arms.items():
            ts[k].append(synced(fn))
    return {k: float(np.median(v)) for k, v in ts.items()}


def torch_step(kv, cfg, s, r, o):
    """the 1vsAll rule in fp32 PyTorch between the same Pull and Push"""
    d, N = cfg.embed_dim, cfg.num_entities
    rl = cfg.relation_len
    uniq, inv = torch.unique(r, return_inverse=True)
    keys = torch.cat([torch.arange(N, device=s.device), uniq + N])
    R = torch.empty(N * 2 * d + uniq.numel() * rl, device=s.device)
    kv.wait(kv.pull(keys, R, True))
    ent, rr = R[:N * 2 * d].view(N, 2 * d), R[N * 2 * d:].view(-1, rl)
    E = ent[:, :d].clone().requires_grad_()
    Rl = rr[:, :rl // 2].clone().requires_grad_()
    rel = Rl[inv]
    if cfg.algorithm == "ComplEx":
        Q = torch.cat([complex_query(E[s], rel, False), complex_query(E[o], rel, True)])
    else:
        Rm = rel.view(-1, d, d)
        Q = torch.cat([torch.einsum("bi,bij->bj", E[s], Rm), torch.einsum("bij,bj->bi", Rm, E[o])])
    ans = torch.cat([o, s])
    loss = -torch.log_softmax(Q @ E.t(), 1).gather(1, ans.view(-1, 1)).sum()
    loss = loss + 0.5 * cfg.gamma_entity * ((E[s] ** 2).sum() + (E[o] ** 2).sum()) + 0.5 * cfg.gamma_relation * (rel ** 2).sum()
    ge, gr = torch.autograd.grad(loss, [E, Rl])

    def upd(g, a):
        return torch.cat([-cfg.eta * g / torch.sqrt(a + g * g), g * g], 1)

    U = torch.cat([upd(ge, ent[:, d:]).view(-1), upd(gr, rr[:, rl // 2:]).view(-1)])
    kv.wait(kv.push(keys, U, True))


def bench_case(algo, d, B, args, info):
    cfg = KGEConfig(num_entities=NE, num_relations=NR, embed_dim=d, algorithm=algo, eta=0.1)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"kge1vsall_bench_{np.random.randint(1 << 30)}", dtype="float32", device=0)
    kv = ad.Worker(0, server)
    try:
        g = torch.Generator().manual_seed(1)
        for first, n, ln in ((0, NE, cfg.entity_len), (NE, NR, cfg.relation_len)):
            rows = torch.cat([torch.randn(n, ln // 2, generator=g) * 0.1, torch.full((n, ln // 2), 1e-6)], 1)
            kv.wait(kv.set(torch.arange(first, first + n), rows.reshape(-1)))
        dev = server.device
        gd = torch.Generator(device=dev).manual_seed(2)
        s = torch.randint(0, NE, (B,), device=dev, generator=gd)
        r = torch.randint(0, NR, (B,), device=dev, generator=gd)
        o = torch.randint(0, NE, (B,), device=dev, generator=gd)
        loss = torch.zeros(1, device=dev)
        nrat = 6
        C = 1 + 2 * nrat
        S = s.view(-1, 1).expand(B, C).clone()
        O = o.view(-1, 1).expand(B, C).clone()
        S[:, 2::2] = torch.randint(0, NE, (B, nrat), device=dev, generator=gd)
        O[:, 1::2] = torch.randint(0, NE, (B, nrat), device=dev, generator=gd)
        Rk = (r + NE).view(-1, 1).expand(B, C).reshape(-1).contiguous()
        L = torch.zeros(B, C, device=dev)
        L[:, 0] = 1
        S, O, L = S.reshape(-1), O.reshape(-1), L.reshape(-1)
        neg = ops.kge_complex_step if algo == "ComplEx" else ops.kge_rescal_step
        arms = {
            "1vsall": lambda: ops.kge_1vsall_step(kv, s, r + NE, o, NE, algo, d, 0.1, 1e-3, 1e-3, loss),
            "torch": lambda: torch_step(kv, cfg, s, r, o),
            "negsamp": lambda: neg(server, S, Rk, O, L, d, 0.1, 1e-3, 1e-3, loss, None, deterministic=True),
        }
        t = alternate(arms, args.runs, args.warmup)
        dpad = (d + 7) // 8 * 8
        flops = 3 * 2 * 2 * B * NE * dpad
        nrel = int(torch.unique(r).numel())
        moved = (NE * cfg.entity_len + nrel * cfg.relation_len) * 4
        for k, v in t.items():
            rec = {"bench": "kge_1vsall", "arm": k, "algorithm": algo, "d": d, "B": B, "ms_per_step": round(v * 1e3, 3),
                   "pull_bytes": moved, "push_bytes": moved, **info}
            if k != "negsamp":
                rec["contraction_tflops"] = round(flops / v / 1e12, 1)
            print(json.dumps(rec), flush=True)
    finally:
        kv.finalize()
        server.shutdown()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kge_1vsall_bench needs a CUDA device")
    info = card()
    for algo, d in (("ComplEx", 512), ("RESCAL", 64)):
        for B in (1024, 4096):
            bench_case(algo, d, B, args, info)


if __name__ == "__main__":
    main()
