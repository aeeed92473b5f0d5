"""The grouped AdaGrad push that gives one update per distinct key (csrc/cuda/grouped_push.cuh: radix sort, tile pass,
finish pass) is shared by the embedding-bag backward and the FFM step. These tests pin what both ops compute, bit for
bit, against tests/golden/grouped_push, made by running this file as a script: the bag outputs, the rows after the
step, the FFM losses and the statistics of one GPU, for every float4-per-lane (VPL) instantiation of both ops. The
other tests check these ops against float64 within a tolerance and against themselves run to run; these catch a
change that moves a result by one ulp.

    python tests/test_gpu_grouped_push.py OUT_DIR    # writes golden.json"""
import hashlib
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_ffm_cpu import FFM_VPL_SHAPE  # noqa: E402
from multirank import load_rows, one_rank_store  # noqa: E402
from test_gpu_embbag import MODES, _hard_bags, _rows, _run  # noqa: E402
from test_gpu_embbag import _table as _bag_table  # noqa: E402
from test_gpu_ffm import _batch, _fused  # noqa: E402
from test_gpu_ffm import _table as _ffm_table  # noqa: E402

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grouped_push", "golden.json")
BAG_DIMS = [20, 132, 260, 512]          # VPL 1 to 4
BAG_CASES = [f"{d}-{mode}{'-weighted' if w else ''}" for d in BAG_DIMS for mode, w in MODES]
FFM_CASES = [f"{v}-F{F}-k{k}" for v, (F, k) in FFM_VPL_SHAPE.items()]


def _sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def _bag_run(dim):
    """One forward and backward per mode on `_hard_bags` inputs (empty bags, one bag of 10 000 keys, one key at every
    other position, so its run spans hundreds of tiles): {case: SHA-256 of the output and of the table, stats}"""
    from adapm_b200.ops import StoreEmbeddingBag

    num_keys = 20_000
    out = {}
    with one_rank_store(2 * dim, num_keys, "cuda", "float32") as (server, kv):
        for mode, weighted in MODES:
            g = torch.Generator().manual_seed(dim + 3 * weighted + 5 * (mode == "mean"))
            table = _bag_table(num_keys, dim, g)
            keys, offsets = _hard_bags(g, num_keys)
            w = torch.rand(keys.numel(), generator=g) * 2 - 0.5 if weighted else None
            grad = torch.randn(offsets.numel() - 1, dim, generator=g) * 1e-3
            load_rows(kv, [(torch.arange(num_keys), table)])
            kv.waitall()
            bag = StoreEmbeddingBag(server, kv, dim, mode=mode, lr=0.05, grad_scale=7.0)
            pooled = _run(kv, bag, keys, offsets, w, grad)
            out[f"{dim}-{mode}{'-weighted' if weighted else ''}"] = {
                "out_sha256": _sha(pooled), "rows_sha256": _sha(_rows(kv, num_keys, dim)), "stats": bag.stats.tolist()}
    return out


def _ffm_run(v):
    """Two steps of 512 examples skewed towards each field's small ids (the hottest keys' runs cross many tiles):
    SHA-256 of the table after them, the steps' losses and the stats"""
    F, k = FFM_VPL_SHAPE[v]
    g = torch.Generator().manual_seed(1000 * v + F * 10 + k)
    per_field = 60
    table = _ffm_table(F * per_field, F, k, g)
    batches = [_batch(F, per_field, 512, g) for _ in range(2)]
    rows, losses, _, stats = _fused(table, batches, F, k, 1.0 / F)
    return {"rows_sha256": _sha(rows.float()), "losses": losses, "stats": stats}


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@gpu
@pytest.mark.parametrize("dim", BAG_DIMS)
def test_embedding_bag_matches_the_golden(dim):
    want = _golden()["bag"]
    got = _bag_run(dim)
    for case, v in got.items():
        assert v == want[case], case


@gpu
@pytest.mark.parametrize("vpl", sorted(FFM_VPL_SHAPE))
def test_ffm_step_matches_the_golden(vpl):
    want = _golden()["ffm"][FFM_CASES[vpl - 1]]
    assert _ffm_run(vpl) == want


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = sys.argv[1]
    golden = {"bag": {}, "ffm": {}}
    for d in BAG_DIMS:
        golden["bag"].update(_bag_run(d))
    for v in sorted(FFM_VPL_SHAPE):
        golden["ffm"][FFM_CASES[v - 1]] = _ffm_run(v)
    assert sorted(golden["bag"]) == sorted(BAG_CASES)
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "golden.json"), "w") as f:
        json.dump(golden, f, indent=1)
    print(json.dumps(golden))
