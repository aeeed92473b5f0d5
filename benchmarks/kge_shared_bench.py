"""KGE sampled-softmax training step on the parameter store, one GPU, against 1vsAll and negative sampling.

Arms, alternating in one process, median of ``--runs`` device-synchronised steps after ``--warmup``:
    shared_S  ``ops.kge_shared_step`` with S = 256, 1024, 4096 shared negatives: one Pull of the batch's entities, the
              negatives and the batch's relations, the three per-chunk bf16 wgmma contractions with the kernels around
              them, one Push
    1vsall    ``ops.kge_1vsall_step``: every entity row in and out (skipped where its workspace does not fit the
              free device memory with its Pull and Push buffers)
    negsamp   the negative-sampling step of the model (``kge_complex_step`` / ``kge_rescal_step``, neg_ratio 6,
              deterministic), i.e. another training type, not the same computation
    torch_S   the sampled-softmax rule through PyTorch between the same Pull and Push as shared_S (fp32 matmul, masked
              ``logsumexp``, autograd, the AdaGrad update in PyTorch), at S = 1024

Cases: ComplEx at d 512 and RESCAL at d 64, B = 4096 triples, N = 14 951 (FB15k) and 10^6 entities: the shared step's
cost should not depend on N, 1vsAll's grows with it. Reported per arm: ms per step; for the shared and 1vsAll arms the
contractions' TFLOP/s over the whole step (3 * 2 * 2B * L * d_padded, L = 2 * 128 + S for the shared step and N for
1vsAll: a whole-step rate, not a kernel's); the distinct rows and bytes pulled and pushed. Each JSON line carries the
card's name and power limit, read by ``nvidia-smi`` in the same run."""
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

NR, B = 1345, 4096
SHARED = (256, 1024, 4096)


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


def torch_step(kv, cfg, s, r, o, neg):
    """the sampled-softmax rule in fp32 PyTorch between the same Pull and Push as the shared step"""
    d, N, rl, ch = cfg.embed_dim, cfg.num_entities, cfg.relation_len, ops.KGE_SHARED_CHUNK
    ents, einv = torch.unique(torch.cat([s, o, neg]), return_inverse=True)
    uniq, inv = torch.unique(r, return_inverse=True)
    keys = torch.cat([ents, uniq + N])
    ne = ents.numel()
    R = torch.empty(ne * 2 * d + uniq.numel() * rl, device=s.device)
    kv.wait(kv.pull(keys, R, True))
    ent, rr = R[:ne * 2 * d].view(ne, 2 * d), R[ne * 2 * d:].view(-1, rl)
    E = ent[:, :d].clone().requires_grad_()
    Rl = rr[:, :rl // 2].clone().requires_grad_()
    rel = Rl[inv]
    n = s.numel()
    ls, lo, ln = einv[:n], einv[n:2 * n], einv[2 * n:]
    if cfg.algorithm == "ComplEx":
        Qo, Qs = complex_query(E[ls], rel, False), complex_query(E[lo], rel, True)
    else:
        Rm = rel.view(-1, d, d)
        Qo, Qs = torch.einsum("bi,bij->bj", E[ls], Rm), torch.einsum("bij,bj->bi", Rm, E[lo])
    nch = n // ch                                          # B is a multiple of the chunk
    lst = torch.cat([ls.view(nch, ch), lo.view(nch, ch), ln.view(1, -1).expand(nch, -1)], 1)     # [nch, L]
    Q = torch.cat([Qo.view(nch, ch, d), Qs.view(nch, ch, d)], 1)                                  # [nch, 2 ch, d]
    ans = torch.cat([lo.view(nch, ch), ls.view(nch, ch)], 1)
    pos = torch.cat([torch.arange(ch, 2 * ch), torch.arange(ch)]).to(s.device).expand(nch, -1)
    Z = torch.bmm(Q, E[lst].transpose(1, 2))
    live = lst.unsqueeze(1) != ans.unsqueeze(2)
    live.scatter_(2, pos.unsqueeze(2), True)
    Z = Z.masked_fill(~live, float("-inf"))
    loss = (torch.logsumexp(Z, 2) - Z.gather(2, pos.unsqueeze(2)).squeeze(2)).sum()
    loss = loss + 0.5 * cfg.gamma_entity * ((E[ls] ** 2).sum() + (E[lo] ** 2).sum()) + 0.5 * cfg.gamma_relation * (rel ** 2).sum()
    ge, gr = torch.autograd.grad(loss, [E, Rl])

    def upd(g, a):
        return torch.cat([-cfg.eta * g / torch.sqrt(a + g * g), g * g], 1)

    U = torch.cat([upd(ge, ent[:, d:]).view(-1), upd(gr, rr[:, rl // 2:]).view(-1)])
    kv.wait(kv.push(keys, U, True))


def bench_case(algo, d, NE, args, info):
    cfg = KGEConfig(num_entities=NE, num_relations=NR, embed_dim=d, algorithm=algo, eta=0.1, gamma_entity=1e-3,
                    gamma_relation=1e-3)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job=f"kgeshared_bench_{np.random.randint(1 << 30)}", dtype="float32", device=0)
    kv = ad.Worker(0, server)
    try:
        g = torch.Generator().manual_seed(1)
        for first, n, ln in ((0, NE, cfg.entity_len), (NE, NR, cfg.relation_len)):
            for c in range(0, n, 1 << 17):
                m = min(1 << 17, n - c)
                rows = torch.cat([torch.randn(m, ln // 2, generator=g) * 0.1, torch.full((m, ln // 2), 1e-6)], 1)
                kv.wait(kv.set(torch.arange(first + c, first + c + m), rows.reshape(-1)))
        dev = server.device
        gd = torch.Generator(device=dev).manual_seed(2)
        s = torch.randint(0, NE, (B,), device=dev, generator=gd)
        r = torch.randint(0, NR, (B,), device=dev, generator=gd)
        o = torch.randint(0, NE, (B,), device=dev, generator=gd)
        negs = {S: torch.randint(0, NE, (S,), device=dev, generator=gd) for S in SHARED}
        loss = torch.zeros(1, device=dev)
        nrat = 6
        C = 1 + 2 * nrat
        Sx = s.view(-1, 1).expand(B, C).clone()
        Ox = o.view(-1, 1).expand(B, C).clone()
        Sx[:, 2::2] = torch.randint(0, NE, (B, nrat), device=dev, generator=gd)
        Ox[:, 1::2] = torch.randint(0, NE, (B, nrat), device=dev, generator=gd)
        Rk = (r + NE).view(-1, 1).expand(B, C).reshape(-1).contiguous()
        L = torch.zeros(B, C, device=dev)
        L[:, 0] = 1
        Sx, Ox, L = Sx.reshape(-1), Ox.reshape(-1), L.reshape(-1)
        neg_step = ops.kge_complex_step if algo == "ComplEx" else ops.kge_rescal_step
        arms = {f"shared_{S}": (lambda S=S: ops.kge_shared_step(kv, s, r + NE, o, negs[S], NE, algo, d, 0.1, 1e-3,
                                                                 1e-3, loss)) for S in SHARED}
        rl = cfg.relation_len
        nrel = int(torch.unique(r).numel())
        full_bytes = (NE * cfg.entity_len + nrel * rl) * 4
        free = torch.cuda.mem_get_info(dev)[0]
        if _workspace_1vsall(NE, d) + 2 * full_bytes <= 0.8 * free:
            arms["1vsall"] = lambda: ops.kge_1vsall_step(kv, s, r + NE, o, NE, algo, d, 0.1, 1e-3, 1e-3, loss)
        else:
            print(json.dumps({"bench": "kge_shared", "arm": "1vsall", "algorithm": algo, "d": d, "N": NE, "B": B,
                              "skipped": "1vsAll does not fit: its workspace and Pull / Push buffers exceed 80 % of "
                                         "the free device memory",
                              **info}), flush=True)
        arms["negsamp"] = lambda: neg_step(server, Sx, Rk, Ox, L, d, 0.1, 1e-3, 1e-3, loss, None, deterministic=True)
        arms["torch_1024"] = lambda: torch_step(kv, cfg, s, r, o, negs[1024])
        t = alternate(arms, args.runs, args.warmup)
        dpad = (d + 7) // 8 * 8
        for k, v in t.items():
            rec = {"bench": "kge_shared", "arm": k, "algorithm": algo, "d": d, "N": NE, "B": B,
                   "ms_per_step": round(v * 1e3, 3), **info}
            if k.startswith(("shared", "torch")):
                S = int(k.split("_")[1])
                ents = int(torch.unique(torch.cat([s, o, negs[S]])).numel())
                rec["rows_moved"] = ents + nrel
                rec["pull_bytes"] = rec["push_bytes"] = (ents * cfg.entity_len + nrel * rl) * 4
                rec["contraction_tflops"] = round(3 * 2 * 2 * B * (2 * 128 + S) * dpad / v / 1e12, 1)
            elif k == "1vsall":
                rec["rows_moved"] = NE + nrel
                rec["pull_bytes"] = rec["push_bytes"] = full_bytes
                rec["contraction_tflops"] = round(3 * 2 * 2 * B * NE * dpad / v / 1e12, 1)
            print(json.dumps(rec), flush=True)
    finally:
        kv.finalize()
        server.shutdown()


def _workspace_1vsall(NE, d):
    from adapm_b200 import _C

    return _C.kge_1vsall_workspace_bytes(NE, B, d, ops._kge_1vsall_chunk(NE, 2 * B, 1 << 30))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kge_shared_bench needs a CUDA device")
    info = card()
    for algo, d in (("ComplEx", 512), ("RESCAL", 64)):
        for NE in (14951, 1_000_000):
            bench_case(algo, d, NE, args, info)


if __name__ == "__main__":
    main()
