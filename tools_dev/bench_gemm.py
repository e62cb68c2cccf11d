"""Device-timed microbenchmark of the wgmma GEMM vs torch.matmul (cuBLAS) on DLRM shapes."""
import json, sys, torch
sys.path.insert(0, ".")
from hugectr_b200.ops import gemm as G

def timeit(fn, iters=20, warm=5):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts)//2]

def main():
    res = []
    b = 6912
    for (M, N, K, tag) in [(b,1024,3456,"top0"),(b,1024,1024,"top1"),(b,512,1024,"top2"),(b,256,512,"top3"),
                           (b,512,3456,"crossU"),(b,3456,512,"crossV"),(b,512,16,"bot0"),(b,256,512,"bot1"),(b,128,256,"bot2"),
                           (8192,8192,8192,"sq8k")]:
        a = torch.randn(M, K, device="cuda").bfloat16(); w = torch.randn(K, N, device="cuda").bfloat16() * 0.05
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        for bn in (128, 256, 1128, 1256):
            t = timeit(lambda: G.gemm_bf16(a, w, out, b_mn=True, block_n=bn))
            res.append(dict(tag=tag, M=M, N=N, K=K, bn=bn, ms=t, tflops=2*M*N*K/t/1e9))
        t = timeit(lambda: torch.matmul(a, w, out=out))
        res.append(dict(tag=tag, M=M, N=N, K=K, bn="cublas", ms=t, tflops=2*M*N*K/t/1e9))
        # wgrad: [K=M rows] x^T dy
        dy = torch.randn(M, N, device="cuda").bfloat16()
        dw = torch.zeros(K, N, device="cuda")
        for sp in (1, 2, 4):
            for bn in (128, 1128, 1256):
                t = timeit(lambda: G.gemm_bf16(a, dy, dw, a_mn=True, b_mn=True, flags=G.EPI_ATOMIC, splits=sp, block_n=bn))
                res.append(dict(tag=tag+"_wgrad", M=K, N=N, K=M, bn=f"split{sp}_bn{bn}", ms=t, tflops=2*M*N*K/t/1e9))
        t = timeit(lambda: torch.matmul(a.t(), dy))
        res.append(dict(tag=tag+"_wgrad", M=K, N=N, K=M, bn="cublas", ms=t, tflops=2*M*N*K/t/1e9))
    for r in res: print(json.dumps(r))
    open("gpurun_out/bench_gemm.jsonl","w").write("\n".join(json.dumps(r) for r in res))

if __name__ == '__main__':
    main()
