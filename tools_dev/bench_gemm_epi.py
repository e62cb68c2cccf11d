"""Device-timed GEMMs with the fused epilogues used by DCNv2 (cross / residual add / relu mask)."""
import json, sys, torch
sys.path.insert(0, "."); sys.path.insert(0, "..")
from hugectr_b200.ops import gemm as G
from bench_gemm import timeit  # noqa
b, w, pd = 6912, 3456, 512
bf = lambda *s: (torch.randn(*s, device="cuda") * 0.1).bfloat16()
H, V, x0, xl, out, T = bf(b, pd), bf(pd, w), bf(b, w), bf(b, w), bf(b, w), bf(b, w)
bias = torch.zeros(w, device="cuda")
U = bf(w, pd)
dH = bf(b, pd)
def rep(tag, ms, flops):
    print(json.dumps(dict(tag=tag, us=round(ms * 1e3, 1), tflops=round(flops / ms / 1e9))), flush=True)
fl = 2 * b * w * pd
for bn in (1128, 1256, 128):
    rep(f"crossV plain bn{bn}", timeit(lambda: G.gemm_bf16(H, V, out, b_mn=True, block_n=bn)), fl)
    rep(f"crossV EPI_CROSS bn{bn}", timeit(lambda: G.gemm_bf16(H, V, out, b_mn=True, bias=bias, x0=x0, xl=xl, aux=T, flags=G.EPI_CROSS, block_n=bn)), fl)
    rep(f"dgrad EPI_ADD bn{bn}", timeit(lambda: G.gemm_bf16(dH, U, out, xl=xl, flags=G.EPI_ADD, block_n=bn)), fl)
    rep(f"dgrad plain bn{bn}", timeit(lambda: G.gemm_bf16(dH, U, out, block_n=bn)), fl)
a = bf(b, 1024); wt = bf(1024, 3456); dy = bf(b, 3456); mask = bf(b, 1024); dx = bf(b, 1024)
for bn in (1128, 1256):
    rep(f"top0 dgrad MASK bn{bn}", timeit(lambda: G.gemm_bf16(dy, wt, dx, mask=mask, flags=G.EPI_MASK, block_n=bn)), 2 * b * 1024 * 3456)
    rep(f"top0 dgrad plain bn{bn}", timeit(lambda: G.gemm_bf16(dy, wt, dx, block_n=bn)), 2 * b * 1024 * 3456)
