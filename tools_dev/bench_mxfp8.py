"""MX fp8 GEMM (csrc/gemm_mxfp8.cu) vs the bf16 wgmma GEMM, cuBLAS bf16 (torch.mm) and torch._scaled_mm (cuBLASLt
fp8, per-tensor scales) on the DLRM-DCNv2 MLP shapes.  CUDA events, L2 flushed between timings.
    python tools_dev/bench_mxfp8.py > gemm_mxfp8_microbench.jsonl"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hugectr_b200.ops import gemm as G  # noqa: E402
from hugectr_b200.ops import mxfp8 as MX  # noqa: E402

SHAPES = [("top0", 6912, 1024, 3456), ("top1", 6912, 1024, 1024), ("top2", 6912, 512, 1024), ("top3", 6912, 256, 512),
          ("crossU", 6912, 512, 3456), ("bot1", 6912, 256, 512), ("square", 8192, 8192, 8192)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


for name, M, N, K in SHAPES:
    a = (torch.randn(M, K, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(K, N, device="cuda") * 0.05).to(torch.bfloat16)       # [in, out] like the layers
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    (aq, sfa), (bq, sfb) = MX.mx_buffers(M, K, "cuda"), MX.mx_buffers(N, K, "cuda")
    MX.mx_quantize(a, aq, sfa)
    MX.mx_quantize(w, bq, sfb, transposed=True)
    r = {"shape": name, "M": M, "N": N, "K": K}
    r["mxfp8_gemm_us"] = timeit(lambda: MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, out=out))
    r["mx_quant_act_us"] = timeit(lambda: MX.mx_quantize(a, aq, sfa))
    r["mx_quant_wT_us"] = timeit(lambda: MX.mx_quantize(w, bq, sfb, transposed=True))
    r["bf16_wgmma_us"] = timeit(lambda: G.gemm_bf16(a, w, out, b_mn=True))
    r["cublas_bf16_us"] = timeit(lambda: torch.mm(a, w, out=out))
    try:
        a8, w8 = a.to(torch.float8_e4m3fn), w.t().contiguous().to(torch.float8_e4m3fn)
        one = torch.ones((), device="cuda")
        r["cublaslt_fp8_scaled_mm_us"] = timeit(lambda: torch._scaled_mm(a8, w8.t(), one, one, out_dtype=torch.bfloat16))
    except Exception as e:  # noqa: BLE001
        r["cublaslt_fp8_scaled_mm_us"] = f"n/a: {str(e)[:80]}"
    fl = 2.0 * M * N * K
    r["mxfp8_tflops"] = fl / r["mxfp8_gemm_us"] / 1e6
    r["bf16_wgmma_tflops"] = fl / r["bf16_wgmma_us"] / 1e6
    ref = MX.mx_dequantize(aq, sfa, M, K).cuda() @ MX.mx_dequantize(bq, sfb, N, K).cuda().t() if M * N <= 1 << 24 else None
    if ref is not None:
        r["max_err_vs_dequant"] = float((out.float() - ref).abs().max())
    print(json.dumps(r), flush=True)
