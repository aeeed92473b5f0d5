"""``KGE.rank_triples`` on the CPU backend against its definition, by a float64 loop over all candidates: a rank is 1 + the
number of candidates other than the true one that are strictly better, and the filtered subject and object ranks leave
out the known answers of the query. The rows are chosen so the model's arithmetic is exact (ComplEx, RESCAL and TransE)
or every comparison is clear by far more than rounding (RotatE), so ranks must agree exactly, ties included."""
import itertools
import uuid

import numpy as np
import pytest
import torch

NE, NR = 30, 4


def _model(algo, p, dtype):
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig

    d = 8 if algo == "RotatE" else 4
    cfg = KGEConfig(num_entities=NE, num_relations=NR, embed_dim=d, algorithm=algo, p_norm=p)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cpu",
                       fabric="inproc", job=f"rank{uuid.uuid4().hex[:6]}", dtype=dtype)
    kv = ad.Worker(0, server)
    return cfg, server, kv, KGE(server, kv, cfg)


def _rows(cfg, g):
    """Entity rows E [ne, d] and relation rows R [nr, relation_len / 2] in float64, exactly representable in float32."""
    d, rd = cfg.embed_dim, cfg.relation_len // 2
    if cfg.algorithm == "RotatE":
        E = torch.randn(NE, d, generator=g, dtype=torch.float64).float().double()
        R = ((torch.rand(NR, rd, generator=g, dtype=torch.float64) * 2 - 1) * np.pi).float().double()
    elif cfg.algorithm == "TransE":   # one entry of +-1 or +-2: the normalised row is a signed unit vector, exactly
        E = torch.zeros(NE, d, dtype=torch.float64)
        E[torch.arange(NE), torch.randint(0, d, (NE,), generator=g)] = (
            torch.tensor([-2.0, -1.0, 1.0, 2.0], dtype=torch.float64)[torch.randint(0, 4, (NE,), generator=g)])
        R = torch.randint(-3, 4, (NR, rd), generator=g).double() / 4
    else:                             # quarter integers: every score is exact in float32
        E = torch.randint(-3, 4, (NE, d), generator=g).double() / 4
        R = torch.randint(-2, 3, (NR, rd), generator=g).double() / 4
    E[7] = E[3]; E[20] = E[3]; E[11] = E[25]        # duplicated rows: exact ties, never strictly better
    R[2] = R[0]
    return E, R


def _distance(cfg, E, R, s, r, o):
    """How bad the triple (s, r, o) is, in float64: smaller is better."""
    d = cfg.embed_dim
    es, er, eo = E[s], R[r], E[o]
    if cfg.algorithm == "ComplEx":
        h = d // 2
        sre, sim, rre, rim, ore, oim = es[:h], es[h:], er[:h], er[h:], eo[:h], eo[h:]
        return -float((rre * sre * ore + rre * sim * oim + rim * sre * oim - rim * sim * ore).sum())
    if cfg.algorithm == "RESCAL":
        return -float(es @ er.view(d, d) @ eo)
    if cfg.algorithm == "TransE":
        x = es / es.norm() + er - eo / eo.norm()
        return float(x.abs().sum()) if cfg.p_norm == 1 else float(x.norm())
    zs, zo = torch.view_as_complex(es.view(-1, 2).contiguous()), torch.view_as_complex(eo.view(-1, 2).contiguous())
    return float((zs * torch.exp(1j * er) - zo).abs().sum())


def _brute_ranks(cfg, E, R, triples, known):
    K = {tuple(t) for t in known.tolist()}
    out = {k: [] for k in ("rank_s", "rank_r", "rank_o", "rank_s_raw", "rank_o_raw")}
    for s, r, o in triples.tolist():
        true = _distance(cfg, E, R, s, r, o)
        cands = {
            "o": [(c, _distance(cfg, E, R, s, r, c), (s, r, c) in K) for c in range(NE) if c != o],
            "s": [(c, _distance(cfg, E, R, c, r, o), (c, r, o) in K) for c in range(NE) if c != s],
            "r": [(c, _distance(cfg, E, R, s, c, o), False) for c in range(NR) if c != r],
        }
        if cfg.algorithm == "RotatE":   # the brute force is unambiguous: only exact duplicates come near a true distance
            rows = {"o": E, "s": E, "r": R}
            true_id = {"o": o, "s": s, "r": r}
            for side, cs in cands.items():
                for c, dist, _ in cs:
                    assert abs(dist - true) > 1e-9 or torch.equal(rows[side][c], rows[side][true_id[side]]), (side, c)
        for side, cs in cands.items():
            better = [kn for _, dist, kn in cs if dist < true]
            if side == "r":
                out["rank_r"].append(1 + len(better))
            else:
                out[f"rank_{side}_raw"].append(1 + len(better))
                out[f"rank_{side}"].append(1 + sum(not kn for kn in better))
    return {k: torch.tensor(v, dtype=torch.int64) for k, v in out.items()}


@pytest.mark.parametrize("algo,p,dtype", [("ComplEx", 1, "float32"), ("ComplEx", 1, "float64"), ("RESCAL", 1, "float32"),
                                          ("TransE", 1, "float32"), ("TransE", 2, "float64"), ("RotatE", 1, "float32")])
def test_rank_triples_cpu_matches_definition(algo, p, dtype):
    cfg, server, kv, model = _model(algo, p, dtype)
    g = torch.Generator().manual_seed(11)
    E, R = _rows(cfg, g)
    kv.set(torch.arange(NE), torch.cat([E, torch.full_like(E, 1e-6)], 1).reshape(-1).to(server.dtype))
    kv.set(torch.arange(NE, NE + NR), torch.cat([R, torch.full_like(R, 1e-6)], 1).reshape(-1).to(server.dtype))
    kv.waitall()

    triples = torch.stack([torch.randint(0, NE, (40,), generator=g), torch.randint(0, NR, (40,), generator=g),
                           torch.randint(0, NE, (40,), generator=g)], 1)
    triples[0] = torch.tensor([3, 0, 25]); triples[1] = torch.tensor([7, 2, 11]); triples[2] = triples[3]
    extra = torch.stack([torch.randint(0, NE, (120,), generator=g), torch.randint(0, NR, (120,), generator=g),
                         torch.randint(0, NE, (120,), generator=g)], 1)
    # known answers that share a query with a test triple, some of them duplicated: each is filtered once
    near = torch.tensor([[s, r, c] for (s, r, _), c in itertools.product(triples[:6].tolist(), (7, 20, 11))]
                        + [[c, r, o] for (_, r, o), c in itertools.product(triples[:6].tolist(), (3, 25))])
    known = torch.cat([triples, extra, near, near[::2], triples[:5]])

    got = model.rank_triples(triples, known, batch=16)
    want = _brute_ranks(cfg, E, R, triples, known)
    assert set(got) == set(want)
    for k in want:
        assert got[k].dtype == torch.int64 and torch.equal(got[k], want[k]), (k, got[k], want[k])
    assert (want["rank_s"] < want["rank_s_raw"]).any() and (want["rank_o"] < want["rank_o_raw"]).any()
    kv.finalize(); server.shutdown()
