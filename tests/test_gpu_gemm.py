"""wgmma/TMA GEMM (ops_gemm_wgmma.cu) against torch.matmul on the same bf16-rounded operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 512), (256, 384, 512), (100, 1000, 72), (2048, 14951, 512),
                                   (1, 7, 8), (333, 129, 200), (1000, 5000, 200), (4096, 4096, 1024)])
def test_gemm_nt_bf16_matches_torch(M, N, K):
    from adapm_b200.ops import gemm_nt_bf16

    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g)
    c = gemm_nt_bf16(a, b)
    torch.cuda.synchronize()
    ref = a.to(torch.bfloat16).float() @ b.to(torch.bfloat16).float().t()
    torch.testing.assert_close(c, ref, rtol=1e-3, atol=1e-2 * (K ** 0.5) / 8)


@pytest.mark.parametrize("M,N,K", [(1024, 304, 32768), (200, 130, 4100), (128, 128, 2048)])
def test_gemm_split_k_matches_torch(M, N, K):
    """Few output tiles + long K: the tile kernel spreads the k-blocks of a tile over gridDim.z CTAs that add their
    partial tiles into the zeroed result (the G^T E0 gradient GEMM of the shared-negative SGNS step is the first shape)."""
    from adapm_b200.ops import gemm_nt_bf16

    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g)
    c = gemm_nt_bf16(a, b)
    c2 = gemm_nt_bf16(a, b)            # a second call: the result buffer is zeroed by the call itself
    torch.cuda.synchronize()
    ref = a.to(torch.bfloat16).float() @ b.to(torch.bfloat16).float().t()
    torch.testing.assert_close(c, ref, rtol=1e-3, atol=1e-2 * (K ** 0.5) / 8)
    torch.testing.assert_close(c2, ref, rtol=1e-3, atol=1e-2 * (K ** 0.5) / 8)


def test_gemm_rank_count_epilogue():
    from adapm_b200.ops import gemm_nt_rank_count

    M, N, K = 500, 3000, 128
    g = torch.Generator(device="cuda").manual_seed(1)
    q = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16).float()
    e = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16).float()
    tcol = torch.randint(0, N, (M,), device="cuda", generator=g)
    ts = (q * e[tcol]).sum(1)
    got = gemm_nt_rank_count(q, e, ts, tcol)
    torch.cuda.synchronize()
    scores = q @ e.t()
    scores.scatter_(1, tcol.view(-1, 1), float("-inf"))
    margin = (scores - ts.view(-1, 1)).abs()
    ref = (scores > ts.view(-1, 1)).sum(1)
    # fp32 summation order differs between the tensor cores and torch: only near-ties may flip
    ambiguous = (margin < 1e-3).sum(1)
    assert ((got.long() - ref).abs() <= ambiguous).all()
    assert (got.long() == ref).float().mean() > 0.98


def test_kge_eval_tensor_core_path_matches_fp32():
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, synthetic_triples

    cfg = KGEConfig(num_entities=700, num_relations=11, embed_dim=64, neg_ratio=2, batch_triples=512)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="kgeeval", device=0)
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    tr = synthetic_triples(cfg, 4000, seed=2)
    for ep in range(3):
        for s in range(0, tr.shape[0], cfg.batch_triples):
            model.step(tr[s:s + cfg.batch_triples])
    torch.cuda.synchronize()
    a = model.evaluate(tr[:300], tr, use_tensor_cores=True)
    b = model.evaluate(tr[:300], tr, use_tensor_cores=False)
    assert abs(a["mrr"] - b["mrr"]) < 0.02 and abs(a["hits@10"] - b["hits@10"]) < 0.03, (a, b)
    assert a["mrr"] > 0.05
    kv.finalize()
    server.shutdown()


@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (300, 500, 416), (64, 1000, 80), (2048, 4096, 256)])
def test_gemm_nt_fp8_matches_torch(M, N, K):
    """e4m3 operands on the fp8 wgmma tensor-core path vs the same quantised operands multiplied in fp32."""
    from adapm_b200.ops import gemm_nt_fp8

    g = torch.Generator(device="cuda").manual_seed(K)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g)
    c = gemm_nt_fp8(a, b)
    torch.cuda.synchronize()
    sa, sb = a.abs().amax() / 448.0, b.abs().amax() / 448.0
    aq = (a / sa).to(torch.float8_e4m3fn).float() * sa
    bq = (b / sb).to(torch.float8_e4m3fn).float() * sb
    torch.testing.assert_close(c, aq @ bq.t(), rtol=2e-3, atol=2e-3 * (K ** 0.5))
    # and it is a sane approximation of the fp32 product
    rel = (c - a @ b.t()).norm() / (a @ b.t()).norm()
    assert rel < 0.08


def test_deepfm_trains_on_gpu_with_tensor_core_mlp():
    import adapm_b200 as ad
    from adapm_b200.models.deepfm import DeepFM, DeepFMConfig, synthetic_ctr_batch

    for precision in ("bf16", "fp8"):
        cfg = DeepFMConfig(num_features=26 * 2000, num_fields=26, embed_dim=16, hidden=(128, 128), batch_size=1024,
                           precision=precision)
        server = ad.Server(cfg.row_len, num_keys=cfg.num_features, num_threads=1, rank=0, world=1, backend="cuda",
                           fabric="inproc", job=f"dfm{precision}", device=0)
        kv = ad.Worker(0, server)
        model = DeepFM(server, kv, cfg)
        model.init_model()
        losses = []
        for s in range(60):
            ids, y = synthetic_ctr_batch(cfg, s % 8)
            losses.append(model.step(ids, y))
        kv.finalize()
        server.shutdown()
        assert sum(losses[-10:]) < sum(losses[:10]), (precision, losses[:3], losses[-3:])


def test_fused_gather_gemm_matches_dense():
    """gather (through the directory) + GEMM in one kernel == pull the rows, then multiply."""
    import adapm_b200 as ad
    from adapm_b200.ops import gather_gemm, gather_gemm_rank_count

    nk, d = 3000, 200
    server = ad.Server(2 * d, num_keys=nk, num_threads=1, rank=0, world=1, backend="cuda", fabric="inproc", job="gg", device=0)
    kv = ad.Worker(0, server)
    g = torch.Generator().manual_seed(3)
    rows = torch.randn(nk, 2 * d, generator=g)
    kv.set(torch.arange(nk), rows.clone().view(-1))
    dev = server.device
    keys = torch.randperm(nk, generator=g)[:1777].to(dev)
    q = torch.randn(300, d, generator=g).to(dev)
    c = gather_gemm(server, q, keys, d)
    torch.cuda.synchronize()
    E = rows.to(dev)[keys][:, :d].to(torch.bfloat16).float()
    ref = q.to(torch.bfloat16).float() @ E.t()
    torch.testing.assert_close(c, ref, rtol=1e-3, atol=2e-2)
    tcol = torch.randint(0, keys.numel(), (300,), device=dev)
    ts = (q.to(torch.bfloat16).float() * E[tcol]).sum(1)
    cnt = gather_gemm_rank_count(server, q, keys, d, ts, tcol)
    sc = ref.clone(); sc.scatter_(1, tcol.view(-1, 1), float("-inf"))
    refc = (sc > ts.view(-1, 1)).sum(1)
    amb = ((sc - ts.view(-1, 1)).abs() < 1e-3).sum(1)
    assert ((cnt.long() - refc).abs() <= amb).all()
    kv.finalize(); server.shutdown()


def test_kge_fused_eval_matches_dense_eval():
    import adapm_b200 as ad
    from adapm_b200.models.kge import KGE, KGEConfig, evaluate_fused, synthetic_triples

    cfg = KGEConfig(num_entities=900, num_relations=11, embed_dim=64, neg_ratio=2, batch_triples=512)
    server = ad.Server(cfg.value_lengths(), num_keys=cfg.num_keys, num_threads=1, rank=0, world=1, backend="cuda",
                       fabric="inproc", job="kgefused", device=0)
    kv = ad.Worker(0, server)
    model = KGE(server, kv, cfg)
    model.init_model()
    tr = synthetic_triples(cfg, 3000, seed=4)
    for s in range(0, tr.shape[0], cfg.batch_triples):
        model.step(tr[s:s + cfg.batch_triples])
    torch.cuda.synchronize()
    a = evaluate_fused(model, tr[:400], tr)
    b = model.evaluate(tr[:400], tr, use_tensor_cores=True)
    assert abs(a["mrr"] - b["mrr"]) < 5e-3 and abs(a["hits@10"] - b["hits@10"]) < 1e-2, (a, b)
    assert a["gathered_rows_local"] > 0 and a["gathered_rows_remote"] == 0
    kv.finalize(); server.shutdown()
