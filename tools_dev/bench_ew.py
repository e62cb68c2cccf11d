"""Device-timed microbenchmark of the bandwidth-bound kernels (effective GB/s vs the measured copy
roofline in MEASURED_PEAKS.json)."""
import json, sys, torch
sys.path.insert(0, ".")
from hugectr_b200.enums import OPT_STATES_PER_WEIGHT, Optimizer_t as O
from hugectr_b200.ops import dense as D
from hugectr_b200.ops.optim import opt_hp
from hugectr_b200.solver import OptParamsPy

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

def rep(tag, ms, nbytes):
    print(json.dumps(dict(tag=tag, us=round(ms * 1e3, 1), MB=round(nbytes / 1e6, 1),
                          GBps=round(nbytes / ms / 1e6, 1))), flush=True)

b, w = 6912, 3456
bf = lambda *s: torch.randn(*s, device="cuda").bfloat16()
dy, x0, t, dt = bf(b, w), bf(b, w), bf(b, w), bf(b, w)
db = torch.zeros(w, device="cuda")
for dtp in (torch.float32, torch.bfloat16):
    dx0 = torch.zeros(b, w, device="cuda", dtype=dtp)
    e = dx0.element_size()
    for rs in (0, 11, 22, 44, 88):
        rep(f"cross_bwd_ew first {dtp} rs{rs}", timeit(lambda: D.cross_bwd_ew(dy, x0, t, dt, dx0, True, db, row_splits=rs)), b * w * (2 * 4 + e))
        rep(f"cross_bwd_ew accum {dtp} rs{rs}", timeit(lambda: D.cross_bwd_ew(dy, x0, t, dt, dx0, False, db, last=True, row_splits=rs)), b * w * (2 * 4 + 2 * e))
for (r, c) in [(b, 1024), (b, 512), (b, 256), (b, 3456)]:
    x = bf(r, c); o = torch.zeros(c, device="cuda")
    rep(f"colsum {r}x{c}", timeit(lambda: D.colsum_accum(x, o)), r * c * 2)
n = 16_500_000 // 64 * 64
wt, g, w16, s0, s1 = (torch.randn(n, device="cuda"), torch.randn(n, device="cuda"),
                      torch.zeros(n, device="cuda", dtype=torch.bfloat16), torch.ones(n, device="cuda"),
                      torch.ones(n, device="cuda"))
lr_t = torch.full((1,), 0.01, device="cuda"); st = torch.ones(1, dtype=torch.int32, device="cuda")
hp = opt_hp(OptParamsPy(epsilon=1e-8))
for o in (O.SGD, O.AdaGrad, O.Adam, O.Ftrl, O.MomentumSGD, O.Nesterov, O.RMSProp):
    ns = OPT_STATES_PER_WEIGHT[o]
    st0, st1 = s0 if ns >= 1 else None, s1 if ns >= 2 else None
    rep(f"dense_opt {o.name.lower()}", timeit(lambda: D.dense_opt_step(o, wt, g, w16, st0, st1, lr_t, st, hp)),
        n * (4 * (3 + 2 * ns) + 2))
src = bf(b, 128); dst = bf(b, 3456)
rep("copy2d 128->3456 slice", timeit(lambda: D.copy2d(src, dst[:, :128])), b * 128 * 4)
rep("torch copy ref 48MB", timeit(lambda: dt.copy_(dy)), b * w * 4)
rep("torch fp32 copy ref 96MB", timeit(lambda: wt[:n // 2].copy_(g[:n // 2])), n // 2 * 8)
