"""wgmma GEMM throughput vs cuBLAS (torch.matmul) on the same bf16 operands. CUDA events, 5 warm-up
iterations, an L2 flush (256 MiB write) between timed iterations. Prints one JSON line per shape with the
achieved TFLOP/s and its fraction of the H100 SXM data-sheet dense bf16 rate (989 TFLOP/s at 700 W)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adapm_b200 import _C  # noqa: E402
from adapm_b200.ops import gemm_nt_rank_count  # noqa: E402


def timeit(fn, iters=20):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(5):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    datasheet_bf16_tflops = 989.0
    gpu = torch.cuda.get_device_name()
    shapes = [(2048, 14951, 512, "KGE 1-vs-all eval"), (8192, 400, 416, "DeepFM layer 1"), (4096, 4096, 4096, "square 4k"),
              (8192, 8192, 8192, "square 8k"), (16384, 14951, 512, "KGE eval, large batch")]
    st = torch.cuda.current_stream().cuda_stream
    for M, N, K, name in shapes:
        a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
        c = torch.empty(M, N, dtype=torch.float32, device="cuda")
        mine = timeit(lambda: _C.gemm_nt_bf16(st, a.data_ptr(), b.data_ptr(), M, N, K, c.data_ptr(), N))
        ref = timeit(lambda: torch.matmul(a, b.t()))
        fl = 2.0 * M * N * K
        out = {"shape": [M, N, K], "name": name, "gpu": gpu, "wgmma_ms": mine, "cublas_bf16_out_ms": ref,
               "wgmma_tflops": fl / mine / 1e9, "cublas_tflops": fl / ref / 1e9,
               "frac_of_datasheet_bf16": fl / mine / 1e9 / datasheet_bf16_tflops}
        if M >= 4096 and N >= 4096:
            a8 = a.float().to(torch.float8_e4m3fn); b8 = b.float().to(torch.float8_e4m3fn)
            f8 = timeit(lambda: _C.gemm_nt_e4m3(st, a8.data_ptr(), b8.data_ptr(), M, N, K, c.data_ptr(), N, 1.0))
            out["wgmma_fp8_ms"] = f8
            out["wgmma_fp8_tflops"] = fl / f8 / 1e9
        if "KGE" in name:
            ts = torch.zeros(M, device="cuda"); tc = torch.zeros(M, dtype=torch.int64, device="cuda")
            af, bf = a.float(), b.float()
            out["rank_count_epilogue_ms"] = timeit(lambda: gemm_nt_rank_count(af, bf, ts, tc), iters=10)
            out["note"] = "rank_count timing includes the fp32->bf16 operand casts done by the Python wrapper"
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
