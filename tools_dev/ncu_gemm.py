"""One DLRM top-MLP GEMM (6912 x 1024 x 3456, pair tile 256x128) for an ncu --set full capture."""
import sys, torch
sys.path.insert(0, ".")
from hugectr_b200.ops import gemm as G
M, N, K = 6912, 1024, 3456
a = torch.randn(M, K, device="cuda").bfloat16(); w = (torch.randn(K, N, device="cuda") * 0.05).bfloat16()
out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
bias = torch.zeros(N, device="cuda")
for _ in range(6):
    G.gemm_bf16(a, w, out, b_mn=True, bias=bias, flags=G.EPI_RELU, block_n=1128)
torch.cuda.synchronize()
