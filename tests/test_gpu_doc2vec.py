"""Paragraph vectors on the H100: ``ops.doc2vec_infer`` against its float64 rule, bit-for-bit reproducibility, read-only
store rows, the three-rank scenarios, and reproducible training with planted-topic quality."""
import numpy as np
import pytest
import torch

from multirank import WORLD, Case, on_peer_rows, on_replicas, one_rank_store, reads_while_keys_move
from test_doc2vec_cpu import INFER_MIN, SHARE_MIN, train_planted

gpu = pytest.mark.gpu
V = 2000


def _rows(d, seed, scale=0.6):
    g = torch.Generator().manual_seed(seed)
    t = torch.ones(2 * V, 2 * d)
    t[:, :d] = (torch.rand(2 * V, d, generator=g) - 0.5) * scale
    return t


def _load(kv, table):
    kv.begin_setup()
    kv.wait(kv.set(torch.arange(table.shape[0], dtype=torch.int64), table.contiguous().view(-1)))
    kv.end_setup()


def _sampler(server):
    from adapm_b200.ops import DeviceSampler

    w = np.arange(1, V + 1, dtype=np.float64) ** -0.75
    return DeviceSampler(server, weights=torch.from_numpy(w), first_key=1, key_stride=2)


def _docs(lengths, seed):
    rng = np.random.default_rng(seed)
    docs = [rng.integers(0, V, int(n)) for n in lengths]
    off = np.concatenate([[0], np.cumsum([len(x) for x in docs])]).astype(np.int64)
    tok = np.concatenate(docs).astype(np.int64) if docs else np.zeros(0, np.int64)
    return torch.from_numpy(tok), torch.from_numpy(off)


def _tolerance(kw, L):
    """float32 against float64: each of the E * L sequential updates moves an entry by at most alpha, and its float32
    rounding (d-term dots, the sigmoid, the AdaGrad quotient) is a relative error of at most about (d + 8) 2^-24; the
    bound below allows 4x that, summed over every update."""
    return kw["alpha"] * kw["epochs"] * max(L, 1) * (kw["embed_dim"] + 8) * 2.0 ** -22 + 1e-6


CASES = [  # (dm, d, negative, window, epochs, lengths)
    (0, 4, 1, 1, 1, [0, 1, 2, 7]),
    (1, 4, 5, 1, 2, [0, 1, 2, 7]),
    (1, 32, 5, 3, 3, [1, 2, 7, 7, 30]),
    (0, 100, 25, 5, 2, [7, 40, 2, 1]),
    (1, 128, 31, 15, 5, [0, 7, 50, 2]),
    (1, 300, 5, 7, 2, [1, 2, 7, 64]),
    (0, 336, 31, 2, 4, [2, 7, 33]),
    (1, 100, 5, 5, 1, [500, 10000]),
    (0, 100, 5, 5, 1, [500, 10000]),
    (1, 32, 5, 9, 2, list(np.random.default_rng(3).integers(0, 40, 3000))),
    (0, 100, 5, 5, 3, list(np.random.default_rng(4).integers(0, 40, 3000))),
]


@gpu
@pytest.mark.parametrize("dm,d,neg,win,E,lengths", CASES)
def test_inference_matches_the_float64_rule(dm, d, neg, win, E, lengths):
    from adapm_b200.ops import doc2vec_infer, doc2vec_infer_reference

    kw = dict(dm=bool(dm), embed_dim=d, negative=neg, window=win, epochs=E, alpha=0.05, min_alpha=0.005, seed=91)
    tok, off = _docs(lengths, d + neg)
    ids = torch.arange(len(lengths), dtype=torch.int64) * 7 + 3
    with one_rank_store(2 * d, 2 * V, "cuda", "float32") as (s, kv):
        _load(kv, _rows(d, d))
        sp = _sampler(s)
        loss = torch.zeros(1, device=s.device)
        got = doc2vec_infer(s, tok, off, ids, sp, loss=loss, **kw).cpu().double().numpy()
        want, want_loss = doc2vec_infer_reference(kv, tok, off, ids, sp, **kw)
    lens = np.diff(off.numpy())
    for m in range(len(lengths)):
        err = np.abs(got[m] - want[m]).max()
        assert err <= _tolerance(kw, lens[m]), (m, lens[m], err, _tolerance(kw, lens[m]))
    assert float(loss) == pytest.approx(want_loss, rel=1e-3)


@gpu
@pytest.mark.parametrize("dm", [0, 1])
def test_inference_is_bit_for_bit_reproducible_and_read_only(dm):
    from adapm_b200.ops import doc2vec_infer, doc2vec_initial_vectors

    d = 100
    kw = dict(dm=bool(dm), embed_dim=d, negative=5, window=5, epochs=3, alpha=0.025, min_alpha=0.001, seed=5)
    lengths = [0] + list(np.random.default_rng(8).integers(0, 60, 499))
    tok, off = _docs(lengths, 2)
    ids = torch.arange(len(lengths), dtype=torch.int64) + 1000
    table = _rows(d, 12)
    with one_rank_store(2 * d, 2 * V, "cuda", "float32") as (s, kv):
        _load(kv, table)
        sp = _sampler(s)
        a = doc2vec_infer(s, tok, off, ids, sp, **kw).cpu()
        b = doc2vec_infer(s, tok, off, ids, sp, **kw).cpu()
        assert torch.equal(a, b)
        assert torch.equal(a[0], torch.from_numpy(doc2vec_initial_vectors(5, [1000], d)[0]))
        perm = torch.randperm(len(lengths), generator=torch.Generator().manual_seed(1))
        lens = off[1:] - off[:-1]
        ptok = torch.cat([tok[off[j]:off[j + 1]] for j in perm.tolist()])
        poff = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens[perm], 0)])
        c = doc2vec_infer(s, ptok, poff, ids[perm], sp, **kw).cpu()
        assert torch.equal(c, a[perm])
        for j in (0, 7, 123, 499):
            alone = doc2vec_infer(s, tok[off[j]:off[j + 1]], torch.tensor([0, int(lens[j])]), ids[j:j + 1], sp, **kw)
            assert torch.equal(alone.cpu()[0], a[j])
        after = torch.empty(table.numel())
        kv.wait(kv.pull(torch.arange(2 * V, dtype=torch.int64), after))
        assert torch.equal(after.view_as(table), table)


# ---------------------------------------------------------------------------------------------- three ranks
KW = dict(dm=True, embed_dim=64, negative=5, window=4, epochs=2, alpha=0.05, min_alpha=0.005, seed=3)


class _Infer:
    def __init__(self, server):
        self.server, self.sp = server, _sampler(server)

    def __call__(self, batch):
        from adapm_b200.ops import doc2vec_infer

        return doc2vec_infer(self.server, *batch, self.sp, **KW).cpu()

    def totals(self):
        return None, [0, 0, 0, 0]


def _three_rank_inputs():
    d = KW["embed_dim"]
    table = _rows(d, 40)
    batches = []
    for r in range(WORLD):
        tok, off = _docs(list(np.random.default_rng(50 + r).integers(0, 30, 40)), 60 + r)
        batches.append((tok, off, torch.arange(40, dtype=torch.int64) + 100 * r))
    with one_rank_store(2 * d, 2 * V, "cuda", "float32") as (s, kv):
        _load(kv, table)
        step = _Infer(s)
        want = [step(b) for b in batches]
    case = Case(2 * d, 2 * V, [(torch.arange(2 * V), table)],
                lambda b: torch.unique(torch.cat([2 * b[0], 2 * b[0] + 1, torch.arange(1, 2 * V, 2)])),
                lambda server, kv: _Infer(server))
    return table, batches, want, case


@gpu
def test_inference_on_peer_rows_and_replicas_equals_one_rank():
    table, batches, want, case = _three_rank_inputs()
    for res in (on_peer_rows(case, batches, in_turns=False), on_replicas(case, batches)):
        for r in range(WORLD):
            assert torch.equal(res[r]["outs"][0], want[r]), r
        assert torch.equal(res[0]["rows"][0], table)
        assert all(x["counters"]["protocol_errors"] == 0 for x in res)


@gpu
def test_inference_while_keys_move_equals_one_rank():
    table, batches, want, case = _three_rank_inputs()

    def read(server, kv, stats):
        step = _Infer(server)
        return lambda: {"v": step(batches[2])}

    res = reads_while_keys_move(case, read, {"v": want[2]}, torch.arange(0, 2 * V, 3), "relocation_only")
    out = res[2]
    relocations = sum(x["counters"]["relocations"] for x in res)
    assert relocations > 0 and out["reps"] >= 8, (relocations, out["reps"])
    assert not out["mism"], out["mism"][:5]


# ---------------------------------------------------------------------------------------------- training
@gpu
@pytest.mark.parametrize("dm", [0, 1])
def test_training_is_reproducible_with_planted_topic_quality(tmp_path, dm):
    share, inferred, losses, vecs = train_planted("cuda", str(tmp_path / "topics.txt"), dm, dbow_words=1)
    print(f"H100 planted topics dm={dm}: own-topic share of the 10 nearest {share:.3f}, held-out nearest topic "
          f"{inferred:.3f} (chance 0.125)")
    assert share >= SHARE_MIN and inferred >= INFER_MIN, (share, inferred)
    again = train_planted("cuda", str(tmp_path / "topics2.txt"), dm, dbow_words=1)
    assert torch.equal(vecs, again[3]) and losses == again[2]
