"""Which compiled instantiation of each fused training step runs at which shape, and which numeric test runs that shape.

Every fused step picks a template instantiation from the shape it is given (float4 per lane, p, the deterministic or
in-place mode, the generic scalar path). Each instantiation is separate machine code with its own tail guards, so a bug
in one does not show in the others. ``DISPATCH`` names, for every instantiation of the step families in the built
extension, a shape that selects it and the test that checks that shape against its float64 rule:
- the table is complete: every instantiation in the in-tree build (ptxas logs, no GPU) is a row;
- the rows' shapes are in the parametrize lists of the tests they name (no GPU);
- on the GPU, each row's shape launches its instantiation and no other of its family (``torch.profiler``).
It also checks that a shape just past each step's size limit is refused with ``AdapmError``, and the window of the
deterministic one-GPU SGNS step."""
import importlib
from collections import namedtuple

import numpy as np
import pytest
import torch

from test_build_budget import _kernels, kernel_name

gpu = pytest.mark.gpu

FAMILIES = ("sgns_step_kernel", "sgns_step_tma_kernel", "sgns_score_tma_kernel", "sgns_det_gather_kernel",
            "cbow_step_kernel", "cbow_score_kernel", "kge_step_kernel", "kge_step_fx_kernel", "kge_rescal_kernel",
            "kge_rescal_fx_kernel", "mf_step_kernel", "mf_step_fx_kernel", "transe_step_kernel", "rotate_step_kernel",
            "embbag_fwd_kernel", "embbag_grad_tile_kernel", "embbag_grad_finish_kernel")

# kernel: the instantiation; op: the runner below that launches it at `shape` (None: it runs only on several ranks or
# with ADAPM_SGNS_DETERMINISTIC=0, in the test named); shape: parameters of `test` (file::function) that select it
Row = namedtuple("Row", "kernel op shape test")
OPS = "test_gpu_ops.py::"
DET = "test_gpu_deterministic.py::"
SGNS = OPS + "test_sgns_step_matches_pytorch_reference"
SGNS_DET = OPS + "test_sgns_steps_with_repeated_keys_match_start_of_step_reference"
SGNS_GATHER = "test_gpu_sgns_gather.py::test_one_key_with_more_entries_than_many_ranges"
PEER = "test_gpu_fused_multirank.py::test_fused_steps_on_peer_rows_match_float64_rule"
TMA_INPLACE = "test_gpu_fused_multirank.py::test_inplace_tma_sgns_step_matches_reference"
CBOW_DET = "test_gpu_cbow.py::test_deterministic_step_matches_float64_rule"
CBOW = "test_gpu_cbow.py::test_inplace_kernel_on_one_gpu_matches_rule"
COMPLEX = OPS + "test_kge_complex_step_matches_pytorch_reference"
KGE_DET = DET + "test_kge_steps_with_repeated_keys_match_start_of_step_reference"
RESCAL = OPS + "test_kge_rescal_and_dropout_match_pytorch_reference"
MF = OPS + "test_mf_step_matches_pytorch_reference"
MF_DET = DET + "test_mf_steps_with_repeated_keys_match_start_of_step_reference"
TRANSE = "test_gpu_transe.py::test_{}_matches_{}"
ROTATE = "test_gpu_rotate.py::test_{}_matches_{}"
EMBBAG = "test_gpu_embbag.py::test_forward_and_step_match_float64_rule"
FX_TEST = {True: ("deterministic_step", "float64_rule"), False: ("inplace_step", "rule_on_distinct_keys")}
VPL_D = {1: 4, 2: 152, 3: 260, 4: 512}                                      # TransE d per float4 per lane
ROTATE_SHAPE = {1: (8, 12), 2: (152, 256), 3: (264, 2), 4: (512, 64)}        # RotatE (d, 2n)
TMA_OPS = {1: "sgns(d=64, neg=5, impl=tma, p=0.0/0.0)", 2: "sgns(d=200, neg=30, impl=tma, p=0.0/0.0)",
           3: "sgns(d=300, neg=25, impl=tma, p=0.0/0.0)"}
TMA_D = {1: (64, 5), 2: (200, 30), 3: (300, 25)}

DISPATCH = [
    Row("sgns_step_kernel<1>", "sgns", {"d": 64, "neg": 40, "impl": "auto"}, SGNS),
    Row("sgns_step_kernel<2>", "sgns", {"d": 132, "neg": 5, "impl": "ldg"}, SGNS),
    Row("sgns_step_kernel<3>", "sgns", {"d": 300, "neg": 25, "impl": "ldg"}, SGNS),
    Row("sgns_step_kernel<4>", "sgns", {"d": 512, "neg": 3, "impl": "auto"}, SGNS),
    Row("sgns_score_tma_kernel<1>", "sgns", {"d": 64, "neg": 2}, SGNS_DET),
    Row("sgns_score_tma_kernel<2>", "sgns", {"d": 132, "neg": 5}, SGNS_DET),
    Row("sgns_score_tma_kernel<3>", "sgns", {"d": 336, "neg": 30}, SGNS_DET),
    Row("sgns_det_gather_kernel<1>", "sgns", {"d": 16}, SGNS_GATHER),
    Row("sgns_det_gather_kernel<2>", "sgns", {"d": 132}, SGNS_GATHER),
    Row("sgns_det_gather_kernel<3>", "sgns", {"d": 300}, SGNS_GATHER),
    *[Row(f"sgns_step_tma_kernel<{v}, 104>", None, {"op": TMA_OPS[v]}, PEER) for v in (1, 2, 3)],
    *[Row(f"sgns_step_tma_kernel<{v}, 128>", None, {"d": TMA_D[v][0], "neg": TMA_D[v][1]}, TMA_INPLACE)
      for v in (1, 2, 3)],
    Row("cbow_score_kernel<1>", "cbow_fx", {"d": 128, "neg": 31}, CBOW_DET),
    Row("cbow_score_kernel<2>", "cbow_fx", {"d": 200, "neg": 25}, CBOW_DET),
    Row("cbow_score_kernel<3>", "cbow_fx", {"d": 300, "neg": 25}, CBOW_DET),
    Row("cbow_step_kernel<1>", "cbow", {"d": 64, "neg": 5}, CBOW),
    Row("cbow_step_kernel<2>", "cbow", {"d": 132, "neg": 5}, CBOW),
    Row("cbow_step_kernel<3>", "cbow", {"d": 300, "neg": 25}, CBOW),
    Row("kge_step_kernel<0>", "complex", {"nh": 18}, COMPLEX),
    Row("kge_step_kernel<1>", "complex", {"nh": 128}, COMPLEX),
    Row("kge_step_kernel<2>", "complex", {"nh": 264}, COMPLEX),
    Row("kge_step_fx_kernel<0>", "complex_fx", {"algo": "ComplEx", "d": 1064}, KGE_DET),
    Row("kge_step_fx_kernel<1>", "complex_fx", {"algo": "ComplEx", "d": 128}, KGE_DET),
    Row("kge_step_fx_kernel<2>", "complex_fx", {"algo": "ComplEx", "d": 264}, KGE_DET),
    Row("kge_rescal_kernel", "rescal", {"algo": "RESCAL", "d": 20}, RESCAL),
    Row("kge_rescal_fx_kernel", "rescal_fx", {"algo": "RESCAL", "d": 20}, KGE_DET),
    Row("mf_step_kernel<0>", "mf", {"rank": 260}, MF),
    Row("mf_step_kernel<1>", "mf", {"rank": 64}, MF),
    Row("mf_step_kernel<2>", "mf", {"rank": 132}, MF),
    Row("mf_step_fx_kernel<0>", "mf_fx", {"rank": 768}, MF_DET),
    Row("mf_step_fx_kernel<1>", "mf_fx", {"rank": 128}, MF_DET),
    Row("mf_step_fx_kernel<2>", "mf_fx", {"rank": 256}, MF_DET),
    *[Row(f"transe_step_kernel<{v}, {p}, {str(fx).lower()}>", "transe_fx" if fx else "transe",
          {"d": VPL_D[v], "p": p}, TRANSE.format(*FX_TEST[fx]))
      for v in (1, 2, 3, 4) for p in (1, 2) for fx in (False, True)],
    *[Row(f"rotate_step_kernel<{v}, {str(fx).lower()}>", "rotate_fx" if fx else "rotate",
          {"d": ROTATE_SHAPE[v][0], "nn": ROTATE_SHAPE[v][1]}, ROTATE.format(*FX_TEST[fx]))
      for v in (1, 2, 3, 4) for fx in (False, True)],
    *[Row(f"{k}<{v}>", "embbag", {"dim": dim}, EMBBAG)
      for k in ("embbag_fwd_kernel", "embbag_grad_tile_kernel", "embbag_grad_finish_kernel")
      for v, dim in ((1, 8), (2, 132), (3, 384), (4, 512))],
]


def family(kernel):
    return kernel.split("<")[0]


# ---------------------------------------------------------------------------------------------- no GPU
def test_dispatch_table_names_every_step_instantiation():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    built = {name for name in k if family(name) in FAMILIES}
    rows = [r.kernel for r in DISPATCH]
    assert len(rows) == len(set(rows)), "an instantiation has two rows"
    assert not built - set(rows), f"built but in no row of DISPATCH: {sorted(built - set(rows))}"
    assert not set(rows) - built, f"rows of DISPATCH that are not built: {sorted(set(rows) - built)}"


def _param_sets(fn):
    """the parameter sets of a test function: the product of its parametrize marks, as {argname: value}"""
    sets = [{}]
    for m in getattr(fn, "pytestmark", []):
        if m.name != "parametrize":
            continue
        names = m.args[0]
        names = [n.strip() for n in names.split(",")] if isinstance(names, str) else list(names)
        cases = []
        for v in m.args[1]:
            if type(v).__name__ == "ParameterSet":          # pytest.param(...)
                v = v.values
            elif len(names) == 1:
                v = (v,)
            cases.append(dict(zip(names, v)))
        sets = [{**a, **b} for a in sets for b in cases]
    return sets


def _matches(params, shape):
    return all(k in params and (params[k] == v or repr(params[k]) == v) for k, v in shape.items())


@pytest.mark.parametrize("row", DISPATCH, ids=lambda r: r.kernel)
def test_row_shape_is_a_case_of_its_numeric_test(row):
    module, fn = row.test.split("::")
    sets = _param_sets(getattr(importlib.import_module(module[:-3]), fn))
    assert any(_matches(p, row.shape) for p in sets), f"{row.test} has no case {row.shape}"


# ---------------------------------------------------------------------------------------------- runners (GPU)
def _server(value_lengths, num_keys):
    import adapm_b200 as ad

    s = ad.Server(value_lengths, num_keys=num_keys, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc",
                  job=f"dispatch_{np.random.randint(1 << 30)}", device=0)
    return s, ad.Worker(0, s)


def _fill(kv, keys, row_len, g):
    """rows [values | positive AdaGrad accumulators] of length row_len"""
    h = row_len // 2
    rows = torch.cat([torch.randn(keys.numel(), h, generator=g) * 0.3, torch.rand(keys.numel(), h, generator=g) + 1e-3], 1)
    kv.wait(kv.set(keys, rows.contiguous().view(-1)))


def _run(value_lengths, num_keys, fill, step):
    """a fresh one-GPU store, `fill(kv, g)`, then `step(server, kv, dev, g)` once"""
    s, kv = _server(value_lengths, num_keys)
    try:
        g = torch.Generator().manual_seed(1)
        fill(kv, g)
        kv.waitall()
        torch.cuda.synchronize()
        step(s, kv, s.device, g)
        torch.cuda.synchronize()
    finally:
        kv.finalize()
        s.shutdown()


def _uniform(row_len, num_keys, step):
    _run(row_len, num_keys, lambda kv, g: _fill(kv, torch.arange(num_keys), row_len, g), step)


def _loss(dev):
    return torch.zeros(1, device=dev), torch.zeros(4, dtype=torch.int64, device=dev)


def run_sgns(shape, impl=None):
    """256 pairs over 40 words: every key has several entries (the deterministic step's gather pass has work)"""
    from adapm_b200.ops import sgns_step

    d, neg, words = shape["d"], shape.get("neg", 25), 40

    def step(s, kv, dev, g):
        centers = 2 * torch.randint(0, words, (256,), generator=g)
        tk = 2 * torch.randint(0, words, (256, neg + 1), generator=g) + 1
        sgns_step(s, centers.to(dev), tk[:, 0].contiguous().to(dev), tk[:, 1:].contiguous().to(dev), d, 0.05,
                  *_loss(dev), impl=impl or shape.get("impl", "tma"))

    _uniform(2 * d, 2 * words, step)


def run_cbow(shape, det):
    from adapm_b200.ops import cbow_step

    d, neg, words = shape["d"], shape["neg"], 100

    def step(s, kv, dev, g):
        c = 2 * torch.randint(0, words, (256,), generator=g) + 1
        x = 2 * torch.randint(0, words, (256, 4), generator=g)
        n = 2 * torch.randint(0, words, (256, neg), generator=g) + 1
        cbow_step(s, c.to(dev), x.to(dev), n.to(dev), d, 0.01, *_loss(dev), deterministic=det)

    _uniform(2 * d, 2 * words, step)


def _triples(ne, nr, nn, g, B=64):
    return (torch.randint(0, ne, (B,), generator=g), ne + torch.randint(0, nr, (B,), generator=g),
            torch.randint(0, ne, (B,), generator=g), torch.randint(0, ne, (B, nn), generator=g))


def run_transe(shape, det):
    from adapm_b200.ops import kge_transe_step

    d, p, ne, nr = shape["d"], shape["p"], 300, 20

    def step(s, kv, dev, g):
        kge_transe_step(s, *(t.to(dev) for t in _triples(ne, nr, 12, g)), d, p, 1.0, 0.05, 0.01, 0.02, *_loss(dev),
                        deterministic=det)

    _uniform(2 * d, ne + nr, step)


def run_rotate(shape, det):
    from adapm_b200.ops import kge_rotate_step

    d, nn, ne, nr = shape["d"], shape["nn"], 600, 20

    def fill(kv, g):
        _fill(kv, torch.arange(ne), 2 * d, g)
        _fill(kv, torch.arange(ne, ne + nr), d, g)

    def step(s, kv, dev, g):
        kge_rotate_step(s, *(t.to(dev) for t in _triples(ne, nr, nn, g)), d, 0.3 * d, 1.0, 0.05, 0.01, *_loss(dev),
                        deterministic=det)

    _run(torch.tensor([2 * d] * ne + [d] * nr, dtype=torch.int64), ne + nr, fill, step)


def run_kge(algo, d, det):
    from adapm_b200.models.kge import KGEConfig
    from adapm_b200.ops import kge_complex_step, kge_rescal_step

    cfg = KGEConfig(num_entities=50, num_relations=5, embed_dim=d, algorithm=algo)

    def fill(kv, g):
        _fill(kv, torch.arange(50), cfg.entity_len, g)
        _fill(kv, torch.arange(50, 55), cfg.relation_len, g)

    def step(s, kv, dev, g):
        S, R, O, _ = _triples(50, 5, 1, g)
        fused = kge_complex_step if algo == "ComplEx" else kge_rescal_step
        fused(s, S.to(dev), R.to(dev), O.to(dev), (torch.rand(64, generator=g) < 0.3).float().to(dev), d, 0.1, 1e-3,
              1e-3, *_loss(dev), deterministic=det)

    _run(cfg.value_lengths(), cfg.num_keys, fill, step)


def run_mf(shape, det):
    from adapm_b200.ops import mf_step

    rank = shape["rank"]

    def step(s, kv, dev, g):
        ones = torch.ones(64, dtype=torch.int32, device=dev)
        mf_step(s, torch.randint(0, 20, (64,), generator=g).to(dev), torch.randint(20, 40, (64,), generator=g).to(dev),
                torch.randn(64, generator=g).to(dev), ones, ones, rank, 0.05, 0.02, *_loss(dev), deterministic=det)

    _uniform(2 * rank, 40, step)


def run_embbag(shape):
    from adapm_b200.ops import StoreEmbeddingBag

    dim = shape["dim"]

    def step(s, kv, dev, g):
        bag = StoreEmbeddingBag(s, kv, dim)
        out = bag(torch.randint(0, 1000, (500,), generator=g).to(dev), torch.arange(0, 501, 5, device=dev))
        out.sum().backward()

    _uniform(2 * dim, 1000, step)


RUN = {
    "sgns": run_sgns,
    "cbow": lambda s: run_cbow(s, False), "cbow_fx": lambda s: run_cbow(s, True),
    "transe": lambda s: run_transe(s, False), "transe_fx": lambda s: run_transe(s, True),
    "rotate": lambda s: run_rotate(s, False), "rotate_fx": lambda s: run_rotate(s, True),
    "complex": lambda s: run_kge("ComplEx", s["nh"], False), "complex_fx": lambda s: run_kge("ComplEx", s["d"], True),
    "rescal": lambda s: run_kge("RESCAL", s["d"], False), "rescal_fx": lambda s: run_kge("RESCAL", s["d"], True),
    "mf": lambda s: run_mf(s, False), "mf_fx": lambda s: run_mf(s, True),
    "embbag": run_embbag,
}


def launched(fn):
    """the kernels (kernel_name) that `fn()` launches, recorded by torch.profiler; a plain torch op runs first and must
    show up, so that a profiler that records nothing cannot pass"""
    from torch.profiler import ProfilerActivity, profile

    x = torch.ones(1 << 16, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        x.mul_(2.0)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any("elementwise" in n for n in names), f"the profiler recorded no kernel of a torch op: {sorted(names)}"
    return {kernel_name(n) for n in names}


# ---------------------------------------------------------------------------------------------- GPU
@gpu
@pytest.mark.parametrize("row", [r for r in DISPATCH if r.op], ids=lambda r: r.kernel)
def test_row_shape_launches_its_instantiation(row):
    names = launched(lambda: RUN[row.op](row.shape))
    same = sorted(n for n in names if family(n) == family(row.kernel))
    assert same == [row.kernel], f"{row.op} at {row.shape} launched {same}, expected only {row.kernel}"


def _det_sgns_rows(d, neg):
    """two deterministic steps from the same inputs: the rows after each, bit for bit"""
    from adapm_b200.ops import sgns_step

    out = []
    for _ in range(2):
        s, kv = _server(2 * d, 80)
        try:
            g = torch.Generator().manual_seed(d + neg)
            _fill(kv, torch.arange(80), 2 * d, g)
            kv.waitall()
            dev = s.device
            loss = torch.zeros(1, device=dev)
            for _ in range(2):
                centers = 2 * torch.randint(0, 40, (512,), generator=g)
                tk = 2 * torch.randint(0, 40, (512, neg + 1), generator=g) + 1
                sgns_step(s, centers.to(dev), tk[:, 0].contiguous().to(dev), tk[:, 1:].contiguous().to(dev), d, 0.05,
                          loss, impl="tma")
            torch.cuda.synchronize()
            rows = torch.empty(80 * 2 * d)
            kv.wait(kv.pull(torch.arange(80), rows))
            out.append((rows, loss.cpu()))
        finally:
            kv.finalize()
            s.shutdown()
    return out


@gpu
@pytest.mark.parametrize("d,neg", [(336, 30), (332, 30)])
def test_widest_deterministic_sgns_shapes_run_the_deterministic_step(d, neg):
    names = launched(lambda: run_sgns({"d": d, "neg": neg}, impl="auto"))
    assert {"sgns_score_tma_kernel<3>", "sgns_det_gather_kernel<3>"} <= names, sorted(names)
    assert not any(family(n) in ("sgns_step_kernel", "sgns_step_tma_kernel") for n in names), sorted(names)
    (r1, l1), (r2, l2) = _det_sgns_rows(d, neg)
    assert torch.equal(r1, r2) and torch.equal(l1, l2)


@gpu
@pytest.mark.parametrize("d,neg,kernel", [(340, 5, "sgns_step_kernel<3>"), (64, 31, "sgns_step_kernel<1>")])
def test_sgns_outside_the_deterministic_window(d, neg, kernel):
    """auto runs the in-place register kernel; an explicit tma request is refused, not silently downgraded"""
    from adapm_b200 import _C

    names = launched(lambda: run_sgns({"d": d, "neg": neg}, impl="auto"))
    assert sorted(n for n in names if family(n).startswith("sgns_")) == [kernel], sorted(names)
    with pytest.raises(_C.AdapmError, match="impl=\"tma\" takes"):
        run_sgns({"d": d, "neg": neg}, impl="tma")


def _refused(value_lengths, num_keys, call, match):
    from adapm_b200 import _C

    s, kv = _server(value_lengths, num_keys)
    try:
        dev = s.device
        k = torch.zeros(8, dtype=torch.int64, device=dev)
        f = torch.zeros(2048, device=dev)           # labels, x, the loss and the bags' output
        with pytest.raises(_C.AdapmError, match=match):
            call(s, k, f, s._impl.backend_handle(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    finally:
        kv.finalize()
        s.shutdown()


@gpu
def test_sizes_past_each_limit_are_refused():
    """one step past the largest size of each step: MF rank 772 and ComplEx nh 1072 (their staging buffers), RESCAL
    D 132, TransE and embedding bags d 516, RotatE d 520, CBOW d 340. The host code refuses them before any launch
    (the Python wrappers of TransE, RotatE, CBOW and the bags check first, so these go to the extension directly)."""
    from adapm_b200 import _C
    from adapm_b200.models.kge import KGEConfig
    from adapm_b200.ops import kge_complex_step, kge_rescal_step, mf_step

    _refused(2 * 772, 16, lambda s, k, f, h, st: mf_step(s, k, k + 1, f[:8], k.int() + 1, k.int() + 1, 772, 0.05, 0.0,
                                                         f[8:9]), "rank too large")
    for algo, d, match in (("ComplEx", 1072, "too large for the staging buffer"), ("RESCAL", 132, r"\[4, 128\]")):
        cfg = KGEConfig(num_entities=8, num_relations=2, embed_dim=d, algorithm=algo)
        fused = kge_complex_step if algo == "ComplEx" else kge_rescal_step
        _refused(cfg.value_lengths(), cfg.num_keys,
                 lambda s, k, f, h, st: fused(s, k, k + 8, k + 1, f[:8], d, 0.1, 0.0, 0.0, f[8:9]),
                 match)
    _refused(2 * 516, 16, lambda s, k, f, h, st: _C.kge_transe_step(
        h, st, k.data_ptr(), k.data_ptr(), k.data_ptr(), k.data_ptr(), 4, 2, 516, 1, 1.0, 0.1, 0.0, 0.0, f.data_ptr(), 0,
        False), r"\[4, 512\]")
    _refused(2 * 520, 16, lambda s, k, f, h, st: _C.kge_rotate_step(
        h, st, k.data_ptr(), k.data_ptr(), k.data_ptr(), k.data_ptr(), 4, 2, 520, 2.0, 1.0, 0.1, 0.0, f.data_ptr(), 0,
        False), r"\[8, 512\]")
    _refused(2 * 340, 16, lambda s, k, f, h, st: _C.cbow_step(
        h, st, k.data_ptr(), k.data_ptr(), k.data_ptr(), 4, 1, 1, 340, 0.01, f.data_ptr(), 0, True), r"\[4, 336\]")
    _refused(2 * 516, 16, lambda s, k, f, h, st: _C.embedding_bag_forward(
        h, st, k.data_ptr(), k.data_ptr(), 0, 4, 2, 516, False, f.data_ptr(), 0),
        r"\[4, 512\]")
