"""The ranking and retrieval kernels against float64, at the shapes where their tiles, rings and slices change.

Filtered ranks, link prediction and nearest neighbours come out of hand-written kernels whose mistakes do not crash: a
wrong tail tile or a miscounted tie shifts a reported metric. The cases here use operands on which the kernels' fp32
arithmetic is exact whatever its order, so each result is compared for equality with a float64 reference:
- GEMM and gather: integers in [-8, 8] are exact in bf16, and with K <= 1024 every partial sum is an integer below 2^24;
- fp8: integers of at most 15 are exact in e4m3; one operand stays in [-4, 4] so that the sums stay below 2^13 (the
  fp8 tensor cores add products to the accumulator at reduced precision);
- L1 and L2: integer rows, or under ``normalize`` rows whose norm is a power of two (the scaled rows stay dyadic), so
  the sums are exact and ``__fsqrt_rn`` rounds as a float32 square root does;
- the complex metric: slot k of every row is a multiple of one Pythagorean direction (3 + 4i, 5 + 12i, ...), so
  every modulus is an integer.
Integer scores tie often, so the tie rules (``>`` for ranks, the smaller column first for top-k) are checked at every
shape. One case with random fp8 operands and ``alpha != 1`` checks the scale against a derived error bound.

``RETRIEVAL`` mirrors ``test_gpu_dispatch.DISPATCH``: one row per built instantiation of the retrieval families, with a
shape that selects it and the numeric test that checks that shape. Without a GPU: the table is complete against the
ptxas logs, every row's shape is a case of its test, and every ring-fed row runs more k-blocks than the ring has
stages, so the producer's second pass over the ring (the flipped parity) is checked. On the GPU, each row's shape
launches its instantiation (``torch.profiler``, in a fresh process)."""
import json
import math
import os
import re
from collections import namedtuple
from contextlib import contextmanager

import pytest
import torch

from test_build_budget import ROOT, _kernels
from test_gpu_dispatch import _matches, _param_sets, _server, family, launched

gpu = pytest.mark.gpu

FAMILIES = ("gemm_nt_wgmma_kernel", "gather_gemm_kernel", "gemm_nt_topk_kernel", "gather_gemm_topk_kernel",
            "topk_merge_kernel", "dist_true_kernel", "dist_rank_kernel", "dist_topk_kernel", "cdist_true_kernel",
            "cdist_rank_kernel", "cdist_topk_kernel")
TOPK_KS = (1, 63, 64)

# M in {1, 128, 129, 300}, N in {1, 127, 128, 129, 3000}; K = 4 runs with a row pitch of 8, 384 is exactly six k-blocks
GATHER_SHAPES = [(1, 1, 4), (128, 127, 64), (129, 128, 72), (300, 129, 384), (1, 3000, 388), (129, 3000, 448),
                 (300, 3000, 1024), (128, 1, 1024), (300, 3000, 384)]
DENSE_SHAPES = [(1, 1, 8), (129, 127, 8), (128, 129, 384), (129, 3000, 392), (300, 3000, 1024), (1, 3000, 1024)]
# 768 and 896: six and seven k-blocks; K >= 4096 with at most 66 output tiles splits K over several CTAs
E4M3_SHAPES = [(128, 128, 768), (129, 300, 896), (200, 300, 4096), (1, 129, 8192)]
# M in {1, 64, 65, 300}, N in {1, 63, 64, 65, 5000}; dim 32 is exactly one chunk, 512 the largest
DIST_SHAPES = [(1, 1, 4), (64, 63, 8), (65, 64, 32), (300, 65, 36), (1, 5000, 152), (65, 5000, 512), (300, 5000, 8),
               (64, 5000, 32)]
METRICS = [(1, False), (1, True), (2, False), (2, True), ("complex", False)]
DIST_CASES = [(p, nz, M, N, dim) for p, nz in METRICS for M, N, dim in DIST_SHAPES if p != "complex" or dim % 8 == 0]
# 528 M tiles of 64 queries: one column slice (each CTA runs all 4 column tiles); M = 1 above gives one slice per tile
DIST_CASES += [(p, nz, 33792, 200, 8) for p, nz in METRICS]

# kernel: the instantiation; op: the runner below that launches it; shape: parameters of `test` that select it;
# ring: bytes per element of a kernel fed by the shared-memory ring (its shape must wrap the ring), else None
Row = namedtuple("Row", "kernel op shape test ring")
MOD = "test_gpu_retrieval.py::"
GATHER = MOD + "test_gather_ops_are_exact_on_integer_rows"
DENSE = MOD + "test_dense_gemm_rank_count_and_topk_are_exact"
E4M3 = MOD + "test_gemm_e4m3_is_exact_on_integers"
DIST = MOD + "test_distance_rank_count_and_topk_are_exact"
BIG = {"M": 300, "N": 3000, "K": 1024}
DIST_OF = {1: ("dist_true_kernel<1>", "dist_rank_kernel<1>", "dist_topk_kernel<1>"),
           2: ("dist_true_kernel<2>", "dist_rank_kernel<2>", "dist_topk_kernel<2>"),
           "complex": ("cdist_true_kernel", "cdist_rank_kernel", "cdist_topk_kernel")}

RETRIEVAL = [
    Row("gemm_nt_wgmma_kernel<0, 0>", "gemm", BIG, DENSE, 2),
    Row("gemm_nt_wgmma_kernel<1, 0>", "gemm_rank", BIG, DENSE, 2),
    Row("gemm_nt_wgmma_kernel<0, 1>", "gemm_e4m3", {"M": 129, "N": 300, "K": 896}, E4M3, 1),
    Row("gemm_nt_topk_kernel", "gemm_topk", BIG, DENSE, 2),
    Row("topk_merge_kernel", "gemm_topk", BIG, DENSE, None),
    Row("gather_gemm_kernel<0>", "gather", BIG, GATHER, 2),
    Row("gather_gemm_kernel<1>", "gather_rank", BIG, GATHER, 2),
    Row("gather_gemm_topk_kernel", "gather_topk", BIG, GATHER, 2),
    *[Row(kern, op, {"p": p, "normalize": p != "complex", "M": 65, "N": 5000, "dim": 512}, DIST, None)
      for p in (1, 2, "complex") for kern, op in zip(DIST_OF[p], ("dist_rank", "dist_rank", "dist_topk"))],
]


# ---------------------------------------------------------------------------------------------- no GPU
def test_retrieval_table_names_every_instantiation():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    built = {name for name in k if family(name) in FAMILIES}
    rows = [r.kernel for r in RETRIEVAL]
    assert len(rows) == len(set(rows)), "an instantiation has two rows"
    assert not built - set(rows), f"built but in no row of RETRIEVAL: {sorted(built - set(rows))}"
    assert not set(rows) - built, f"rows of RETRIEVAL that are not built: {sorted(set(rows) - built)}"


@pytest.mark.parametrize("row", RETRIEVAL, ids=lambda r: r.kernel)
def test_retrieval_row_shape_is_a_case_of_its_numeric_test(row):
    _, fn = row.test.split("::")
    sets = _param_sets(globals()[fn])
    assert any(_matches(p, row.shape) for p in sets), f"{row.test} has no case {row.shape}"


def test_ring_fed_rows_wrap_the_ring():
    """the producer's second pass over the ring (its empty-barrier parity flips) runs only past STAGES k-blocks of 128
    bytes; STAGES is read from the header, so a deeper ring makes this fail until the shapes follow"""
    src = open(os.path.join(ROOT, "adapm_b200", "csrc", "cuda", "wgmma_utils.cuh")).read()
    stages = int(re.search(r"constexpr int STAGES = (\d+);", src).group(1))
    ring = [r for r in RETRIEVAL if r.ring]
    assert {family(r.kernel) for r in ring} == {"gemm_nt_wgmma_kernel", "gather_gemm_kernel", "gemm_nt_topk_kernel",
                                                "gather_gemm_topk_kernel"}
    for r in ring:
        assert math.ceil(r.shape["K"] * r.ring / 128) > stages, (r.kernel, r.shape, stages)


# ---------------------------------------------------------------------------------------------- operands
def _ints(g, *shape, lim=8):
    return torch.randint(-lim, lim + 1, shape, generator=g).float()


def _stream():
    return torch.cuda.current_stream().cuda_stream


@contextmanager
def _store(blocks):
    """a one-GPU store whose keys hold the rows of `blocks` (float [n_b, L_b] each, in key order): rows of several lengths"""
    lengths = torch.cat([torch.full((b.shape[0],), b.shape[1], dtype=torch.int64) for b in blocks])
    s, kv = _server(lengths, lengths.numel())
    try:
        k0 = 0
        for b in blocks:
            kv.wait(kv.set(torch.arange(k0, k0 + b.shape[0]), b.contiguous().view(-1)))
            k0 += b.shape[0]
        kv.waitall()
        torch.cuda.synchronize()
        yield s
    finally:
        kv.finalize()
        s.shutdown()


def _exclusions(M, N, g):
    """up to 5 excluded columns per row: (CSR offsets, cols) and the bool mask [M, N]"""
    counts = torch.randint(0, min(N, 5) + 1, (M,), generator=g)
    cols = torch.cat([torch.sort(torch.randperm(N, generator=g)[:int(c)]).values for c in counts])
    off = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)])
    mask = torch.zeros(M, N, dtype=torch.bool)
    mask[torch.repeat_interleave(torch.arange(M), counts), cols] = True
    return (off, cols), mask


def _true_cols(M, N, g):
    """random true columns, with column 0 and the last column (in the partial last tile) among them"""
    t = torch.randint(0, N, (M,), generator=g)
    t[0] = 0
    t[M // 2] = N - 1
    return t


def _true_scores(S, tcol, g):
    """t_i = S[i, tcol[i]] for most rows; one row in three gets t_i - 1, so that its true column beats t_i and only the
    rule `col != true_col` keeps it out of the count"""
    ts = S.gather(1, tcol.view(-1, 1).to(S.device)).squeeze(1)
    lower = (torch.arange(S.shape[0]) % 3 == 1).to(S.device)
    return torch.where(lower, ts - 1, ts)


def _rank_ref(S, tcol, ts):
    better = S > ts.view(-1, 1)
    better.scatter_(1, tcol.view(-1, 1).to(S.device), False)
    return better.sum(1)


def _same(got, ref):
    (gv, gi), (rv, ri) = got, ref
    assert torch.equal(gi, ri), (gi[:2], ri[:2])
    assert torch.equal(gv, rv), (gv[:2], rv[:2])


# ---------------------------------------------------------------------------------------------- GEMM and gather
def _gather_inputs(M, N, K, g):
    """a store of two row lengths (2K, the [emb | ada] rows, and K) and N keys from both, with repeats; q [M, K];
    E [N, K] the first K values of each key's row"""
    nk = max(2, min(N, 2000))                  # N = 3000 columns over 2000 keys: repeated keys, tied scores
    long, short = _ints(g, nk // 2, 2 * K), _ints(g, nk - nk // 2, K)
    keys = torch.randint(0, nk, (N,), generator=g)
    keys[N // 2] = nk - 1                      # a key of each length class
    keys[0] = 0
    E = torch.cat([long[:, :K], short])[keys]
    return [long, short], keys, _ints(g, M, K), E


@gpu
@pytest.mark.parametrize("M,N,K", GATHER_SHAPES)
def test_gather_ops_are_exact_on_integer_rows(M, N, K):
    from adapm_b200.ops import gather_gemm, gather_gemm_rank_count, gather_gemm_topk, topk_reference

    g = torch.Generator().manual_seed(M * 31 + N * 7 + K)
    blocks, keys, q, E = _gather_inputs(M, N, K, g)
    tcol = _true_cols(M, N, g)
    ex, mask = _exclusions(M, N, g)
    with _store(blocks) as s:
        dev = s.device
        qd, kd = q.to(dev), keys.to(dev)
        S = q.double().to(dev) @ E.double().to(dev).t()
        assert torch.equal(gather_gemm(s, qd, kd, K).double(), S)
        ts = _true_scores(S, tcol, g)
        cnt = gather_gemm_rank_count(s, qd, kd, K, ts.float(), tcol.to(dev))
        assert torch.equal(cnt.long(), _rank_ref(S, tcol, ts))
        S32, mask = S.float(), mask.to(dev)
        for k in TOPK_KS:
            _same(gather_gemm_topk(s, qd, kd, K, k), topk_reference(S32, k))
        _same(gather_gemm_topk(s, qd, kd, K, 64, exclude=tuple(t.to(dev) for t in ex)), topk_reference(S32, 64, mask))


@gpu
@pytest.mark.parametrize("M,N,K", DENSE_SHAPES)
def test_dense_gemm_rank_count_and_topk_are_exact(M, N, K):
    """gemm_nt_bf16, its rank-count epilogue and gemm_nt_topk on integer matrices; the true column of row 0 is column 0,
    that of row M // 2 the last column, and column N // 3 repeats the true column of row 1 (an exact tie)"""
    from adapm_b200.ops import gemm_nt_bf16, gemm_nt_rank_count, gemm_nt_topk, topk_reference

    g = torch.Generator().manual_seed(M * 13 + N * 5 + K)
    q, e = _ints(g, M, K).cuda(), _ints(g, N, K).cuda()
    tcol = _true_cols(M, N, g)
    if M > 1 and N > 2:
        tcol[1] = 1
        e[N // 3] = e[1]
    S = q.double() @ e.double().t()
    assert torch.equal(gemm_nt_bf16(q, e).double(), S)
    ts = _true_scores(S, tcol, g)
    assert torch.equal(gemm_nt_rank_count(q, e, ts.float(), tcol.cuda()).long(), _rank_ref(S, tcol, ts))
    ex, mask = _exclusions(M, N, g)
    S32 = S.float()
    for k in TOPK_KS:
        _same(gemm_nt_topk(q, e, k), topk_reference(S32, k))
    _same(gemm_nt_topk(q, e, 64, exclude=tuple(t.cuda() for t in ex)), topk_reference(S32, 64, mask.cuda()))


@gpu
@pytest.mark.parametrize("op", ["dense", "gather"])
def test_rank_counts_on_random_operands_within_a_derived_bound(op):
    """random bf16 operands: s_ij carries at most err_ij = 2 K 2^-24 sum_k |q_ik e_jk| of fp32 rounding, whatever the
    summation order. A column is decided for row i when |s_ij - t_i| > err_ij (t_i is the fp32 true score the kernel
    gets); the count lies between the decided greater columns and those plus the undecided ones, and almost every row
    has no undecided column, so the check is close to exact"""
    from adapm_b200.ops import gather_gemm_rank_count, gemm_nt_rank_count

    M, N, K = 300, 300, 64
    g = torch.Generator().manual_seed(5)
    q, e = torch.randn(M, K, generator=g).bfloat16().float(), torch.randn(N, K, generator=g).bfloat16().float()
    tcol = _true_cols(M, N, g)
    with _store([torch.cat([e, torch.randn(N, K, generator=g)], 1)]) as s:
        dev = s.device
        qd, ed, td = q.to(dev), e.to(dev), tcol.to(dev)
        S = qd.double() @ ed.double().t()
        ts = S.gather(1, td.view(-1, 1)).squeeze(1).float()
        if op == "dense":
            got = gemm_nt_rank_count(qd, ed, ts, td).long()
        else:
            got = gather_gemm_rank_count(s, qd, torch.arange(N, device=dev), K, ts, td).long()
        err = 2 * K * 2.0 ** -24 * (qd.double().abs() @ ed.double().abs().t())
        gap = S - ts.double().view(-1, 1)
        other = torch.ones_like(gap, dtype=torch.bool).scatter_(1, td.view(-1, 1), False)
        greater = ((gap > err) & other).sum(1)
        undecided = ((gap.abs() <= err) & other).sum(1)
        assert ((greater <= got) & (got <= greater + undecided)).all()
        assert (undecided == 0).float().mean() >= 0.95, (undecided > 0).sum()


def _e4m3(x):
    return x.to(torch.float8_e4m3fn).contiguous()


def _gemm_e4m3(a8, b8, alpha):
    from adapm_b200 import _C

    M, N, K = a8.shape[0], b8.shape[0], a8.shape[1]
    c = torch.empty(M, N, device=a8.device)
    _C.gemm_nt_e4m3(_stream(), a8.data_ptr(), b8.data_ptr(), M, N, K, c.data_ptr(), N, float(alpha))
    return c


@gpu
@pytest.mark.parametrize("M,N,K", E4M3_SHAPES)
def test_gemm_e4m3_is_exact_on_integers(M, N, K):
    """both operand orders, so that every integer of [-15, 15] is decoded on both sides of the product"""
    g = torch.Generator().manual_seed(M + 3 * N + K)
    wide, narrow = _ints(g, M, K, lim=15).cuda(), _ints(g, N, K, lim=4).cuda()
    S = wide.double() @ narrow.double().t()
    assert torch.equal(_gemm_e4m3(_e4m3(wide), _e4m3(narrow), 1.0).double(), S)
    assert torch.equal(_gemm_e4m3(_e4m3(narrow), _e4m3(wide), 1.0).double(), S.t())


@gpu
def test_gemm_e4m3_applies_alpha_within_a_derived_bound():
    """random e4m3 operands, alpha = 0.3, split K (4096, 6 output tiles): |C - alpha A B^T| <= alpha (K / 32 + 2) 2^-13
    sum_k |a_ik b_jk| (each 32-deep tensor-core step may round at about 14 bits) plus the rounding of the product by
    alpha; a missing or doubled alpha is far outside it"""
    M, N, K, alpha = 200, 300, 4096, 0.3
    g = torch.Generator().manual_seed(7)
    a8, b8 = _e4m3(torch.randn(M, K, generator=g).cuda() * 30), _e4m3(torch.randn(N, K, generator=g).cuda() * 30)
    a, b = a8.double(), b8.double()
    ref = alpha * (a @ b.t())
    bound = alpha * (K / 32 + 2) * 2.0 ** -13 * (a.abs() @ b.abs().t()) + 2.0 ** -23 * ref.abs()
    c = _gemm_e4m3(a8, b8, alpha).double()
    assert ((c - ref).abs() <= bound).all()
    assert ((c - ref).abs() < 0.05 * ref.abs().mean()).float().mean() > 0.99


# ---------------------------------------------------------------------------------------------- distances
PYTHAGOREAN = torch.tensor([[3., 4.], [4., 3.], [5., 12.], [12., 5.], [1., 0.], [0., 1.], [8., 15.], [15., 8.]])


def _dist_rows(p, normalize, n, dim, g):
    """rows [n, dim] on which the metric is exact in fp32"""
    if p == "complex":                         # slot k: an integer multiple of direction k % 8 (moduli 1, 5, 13, 17)
        dirs = PYTHAGOREAN[torch.arange(dim // 2) % 8]
        return (torch.randint(-3, 4, (n, dim // 2, 1), generator=g).float() * dirs).reshape(n, dim)
    if not normalize:
        return _ints(g, n, dim)
    # 1, 4, 16 or 64 entries of +-c, c a power of two: the norm c sqrt(nnz) is a power of two, so the scaled row is dyadic
    rows = torch.zeros(n, dim)
    nnz = 4 ** torch.randint(0, 4, (n,), generator=g)
    c = 2.0 ** torch.randint(-1, 3, (n,), generator=g).float()
    for i in range(n):
        z = int(nnz[i])
        while z > dim:
            z //= 4
        pos = torch.randperm(dim, generator=g)[:z]
        rows[i, pos] = c[i] * (2 * torch.randint(0, 2, (z,), generator=g).float() - 1)
    return rows


def _dist_queries(p, normalize, M, dim, g):
    if p == "complex":
        return _dist_rows(p, False, M, dim, g)
    return _ints(g, M, dim) / 8 if normalize else _ints(g, M, dim)


def _dist_ref(p, normalize, q, e):
    """D [M, N] float32, exact: float64 sums of exactly representable terms; the L2 root is taken in float64 and then
    rounded to float32, which gives the correctly rounded float32 root (53 >= 2 * 24 + 2 bits, so the double rounding
    is harmless), as __fsqrt_rn does"""
    from adapm_b200.ops import complex_dist

    q, e = q.double(), e.double()
    if normalize:
        e = e / e.norm(dim=1, keepdim=True).clamp(min=1e-12)
    if p == "complex":
        return complex_dist(q, e).float()
    if p == 1:
        return torch.cdist(q, e, p=1.0).float()
    sq = (q * q).sum(1, keepdim=True) - 2 * q @ e.t() + (e * e).sum(1).view(1, -1)   # integers or dyadics: exact
    return sq.sqrt().float()


@gpu
@pytest.mark.parametrize("p,normalize,M,N,dim", DIST_CASES)
def test_distance_rank_count_and_topk_are_exact(p, normalize, M, N, dim):
    """gather_dist_rank_count (the true distance from dist_true_kernel, the counts from the tile kernel) and
    gather_dist_topk (k = 1, 63, 64, with padding when N < k) against exact distances; key 0 is an all-zero row
    (under normalize, the 1e-12 clamp) and some rows' true column is its column"""
    from adapm_b200.ops import gather_dist_rank_count, gather_dist_topk, topk_reference

    g = torch.Generator().manual_seed({1: 1, 2: 2, "complex": 3}[p] * 7 + normalize + M * 31 + N * 17 + dim)
    nk = max(2, min(N, 3000))                  # N = 5000 over 3000 keys: repeated keys, tied distances
    rows = _dist_rows(p, normalize, nk, dim, g)
    rows[0] = 0
    keys = torch.randint(0, nk, (N,), generator=g)
    keys[0] = 0
    q = _dist_queries(p, normalize, M, dim, g)
    tcol = _true_cols(M, N, g)
    ex, mask = _exclusions(M, N, g)
    with _store([torch.cat([rows, _ints(g, nk, dim)], 1)]) as s:      # rows of 2 dim: the first dim values count
        dev = s.device
        qd, kd, exd, mask = q.to(dev), keys.to(dev), tuple(t.to(dev) for t in ex), mask.to(dev)
        D = _dist_ref(p, normalize, qd, rows.to(dev)[kd])
        raw, filt = gather_dist_rank_count(s, qd, kd, dim, p, normalize, tcol.to(dev), exd)
        dt = D.gather(1, tcol.to(dev).view(-1, 1))
        better = D < dt
        better.scatter_(1, tcol.to(dev).view(-1, 1), False)
        assert torch.equal(raw, better.sum(1))
        assert torch.equal(filt, (better & ~mask).sum(1))
        for k in TOPK_KS:
            _same(gather_dist_topk(s, qd, kd, dim, k, p, normalize), topk_reference(-D, k))
        _same(gather_dist_topk(s, qd, kd, dim, 64, p, normalize, exclude=exd), topk_reference(-D, 64, mask))


# ---------------------------------------------------------------------------------------------- runners (GPU)
def _run_gemm(op, shape):
    from adapm_b200 import ops

    g = torch.Generator().manual_seed(1)
    M, N, K = shape["M"], shape["N"], shape["K"]
    if op == "gemm_e4m3":
        _gemm_e4m3(_e4m3(_ints(g, M, K).cuda()), _e4m3(_ints(g, N, K).cuda()), 1.0)
        return
    q, e = _ints(g, M, K).cuda(), _ints(g, N, K).cuda()
    if op == "gemm":
        ops.gemm_nt_bf16(q, e)
    elif op == "gemm_rank":
        ops.gemm_nt_rank_count(q, e, torch.zeros(M, device="cuda"), torch.zeros(M, dtype=torch.int64, device="cuda"))
    else:
        ops.gemm_nt_topk(q, e, 10)


def _run_gather(op, shape):
    from adapm_b200 import ops

    g = torch.Generator().manual_seed(1)
    M, N, K = shape["M"], shape["N"], shape["K"]
    blocks, keys, q, _ = _gather_inputs(M, N, K, g)
    with _store(blocks) as s:
        qd, kd = q.to(s.device), keys.to(s.device)
        if op == "gather":
            ops.gather_gemm(s, qd, kd, K)
        elif op == "gather_rank":
            ops.gather_gemm_rank_count(s, qd, kd, K, torch.zeros(M, device=s.device),
                                       torch.zeros(M, dtype=torch.int64, device=s.device))
        else:
            ops.gather_gemm_topk(s, qd, kd, K, 10)
        torch.cuda.synchronize()


def _run_dist(op, shape):
    from adapm_b200 import ops

    g = torch.Generator().manual_seed(1)
    p, nz, M, N, dim = (shape[n] for n in ("p", "normalize", "M", "N", "dim"))
    with _store([_dist_rows(p, nz, N, dim, g)]) as s:
        q, keys = _dist_queries(p, nz, M, dim, g).to(s.device), torch.arange(N, device=s.device)
        if op == "dist_rank":
            ops.gather_dist_rank_count(s, q, keys, dim, p, nz, torch.zeros(M, dtype=torch.int64, device=s.device))
        else:
            ops.gather_dist_topk(s, q, keys, dim, 10, p, nz)
        torch.cuda.synchronize()


RUN = {"gemm": _run_gemm, "gemm_rank": _run_gemm, "gemm_e4m3": _run_gemm, "gemm_topk": _run_gemm,
       "gather": _run_gather, "gather_rank": _run_gather, "gather_topk": _run_gather,
       "dist_rank": _run_dist, "dist_topk": _run_dist}


def _launches_of_every_row():
    """{kernel: the instantiations of its family that its row's shape launches}, for every row, in this process"""
    out = {}
    for r in RETRIEVAL:
        names = launched(lambda: RUN[r.op](r.op, r.shape))
        out[r.kernel] = sorted(n for n in names if family(n) == family(r.kernel))
    return out


_CHILD = f"""
import json, sys
sys.path[:0] = [{os.path.dirname(os.path.abspath(__file__))!r}, {ROOT!r}]
import test_gpu_retrieval
print("LAUNCHES " + json.dumps(test_gpu_retrieval._launches_of_every_row()))
"""


@pytest.fixture(scope="module")
def row_launches():
    """The profiler runs in a fresh process: in a long test session the CUDA activity records of torch.profiler can
    stop arriving after earlier tests (an empty recording, not a wrong one), so that what is checked here does not
    depend on which tests ran before it."""
    import subprocess
    import sys

    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")]
    assert line, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(line[-1][len("LAUNCHES "):])


@gpu
@pytest.mark.parametrize("row", RETRIEVAL, ids=lambda r: r.kernel)
def test_retrieval_row_shape_launches_its_instantiation(row, row_launches):
    same = row_launches[row.kernel]
    assert same == [row.kernel], f"{row.op} at {row.shape} launched {same}, expected only {row.kernel}"
