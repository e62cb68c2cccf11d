"""Device time of every bf16 GEMM of one DLRM-DCNv2 training step: ours (gemm_bf16 on the wgmma kernel) against
torch.mm alone and against gemm_library (torch.mm + the same epilogue in eager PyTorch).

  python tools_dev/bench_gemm.py [--batch 6912] [--iters 20] [--rounds 7] [--out DIR] [--tree DIR]
  python tools_dev/bench_gemm.py --check-bits OTHER_TREE [--tree DIR] [--batch 6912]

The call list is recorded, not hand-written: build_dlrm_dcnv2 (batch --batch, small tables; GEMM shapes depend
on the batch and the dense widths only) runs one eager training step with gemm_bf16 wrapped, and every call is
kept with its M, N, K, operand layouts, epilogue flags, splits, the operands present and their strides.  Each
call is then replayed on fresh random operands of the same shapes and strides; the three arms run
alternately, `iters` launches per timed block, and the median over `rounds` blocks is reported with the
achieved TFLOP/s and GB/s and the floor max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s) from the H100 SXM data
sheet.  Bytes are one pass over every operand and epilogue tensor (fp32 accumulating outputs twice).  `block_n` is
the tile the autotuner picked for ours (gemm_bf16's block_n code).

--tree DIR imports hugectr_b200 from another checkout (built in place), so that two builds can be timed one
process per run in one session.  Without a CUDA device the tool exits with an error and measures nothing.

--check-bits OTHER_TREE times nothing: it replays every recorded call that does not accumulate into its output
(no EPI_ATOMIC, no split K) on the same seeded operands under this tree and under OTHER_TREE, one
process each, and reports per call whether `out` and `aux` are equal bit for bit.  The K order of the
accumulation does not depend on the tile, so two builds that tune to different tiles still agree.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
TENSORS = ("a", "b", "out", "bias", "mask", "x0", "xl", "aux", "colsum")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        info = ""
    return name, info or "unknown"


def record_calls(batch):
    """gemm_bf16 calls of one eager training step, as {tensor name: (shape, stride, dtype)} + scalars."""
    from hugectr_b200.models.dlrm import CRITEO_TB_TABLE_SIZES, build_dlrm_dcnv2
    from hugectr_b200.ops import gemm as G
    m = build_dlrm_dcnv2(batchsize=batch, num_gpus=1, table_sizes=[min(t, 10000) for t in CRITEO_TB_TABLE_SIZES],
                         mixed=True, lr=0.004, use_cuda_graph=False)
    m.compile()
    m.train()
    torch.cuda.synchronize()
    calls, real = [], G.gemm_bf16

    def spy(a, b, out=None, **kw):
        c = {"a_mn": bool(kw.get("a_mn", False)), "b_mn": bool(kw.get("b_mn", False)),
             "flags": int(kw.get("flags", 0)), "splits": int(kw.get("splits", 1)),
             "alpha": float(kw.get("alpha", 1.0))}
        for k, t in [("a", a), ("b", b), ("out", out)] + [(k, kw.get(k)) for k in TENSORS[3:]]:
            if t is not None:
                c[k] = (tuple(t.shape), tuple(t.stride()), str(t.dtype).replace("torch.", ""))
        calls.append(c)
        return real(a, b, out, **kw)

    G.gemm_bf16 = spy
    try:
        m.train()
        torch.cuda.synchronize()
    finally:
        G.gemm_bf16 = real
    del m
    torch.cuda.empty_cache()
    return calls


def make_operands(c, gen):
    ts = {}
    for k in TENSORS:
        if k not in c:
            continue
        shape, stride, dt = c[k]
        dt = getattr(torch, dt)
        t = torch.empty_strided(shape, stride, dtype=dt, device="cuda")
        if k in ("out", "colsum") and dt == torch.float32:
            t.zero_()
        else:
            t.copy_((torch.randn(shape, generator=gen) * (0.1 if k in ("a", "b") else 1.0)).to(dt))
        ts[k] = t
    return ts


def shape_of(c):
    (a0, a1), (b0, b1) = c["a"][0], c["b"][0]
    M, K = (a1, a0) if c["a_mn"] else (a0, a1)
    N = b1 if c["b_mn"] else b0
    return M, N, K


def nbytes(c):
    total = 0
    for k in TENSORS:
        if k in c:
            shape, _, dt = c[k]
            n = 1
            for s in shape:
                n *= s
            total += n * torch.empty(0, dtype=getattr(torch, dt)).element_size()
    if c["flags"] & 4 or c["splits"] > 1:           # EPI_ATOMIC reads the output as well
        shape, _, _ = c["out"]
        total += shape[0] * shape[1] * 4
    return total


def time_arms(arms, iters, rounds):
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            ts[k].append(e0.elapsed_time(e1) / iters)
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()}


def output_digests(batch):
    """sha256 of `out` and `aux` of every non-accumulating recorded call, replayed on seeded operands."""
    from hugectr_b200.ops import gemm as G
    calls = record_calls(batch)
    gen = torch.Generator().manual_seed(0)
    res = []
    for i, c in enumerate(calls):
        ts = make_operands(c, gen)
        if c["flags"] & G.EPI_ATOMIC or c["splits"] > 1:
            continue
        kw = dict(a_mn=c["a_mn"], b_mn=c["b_mn"], flags=c["flags"], splits=c["splits"], alpha=c["alpha"])
        kw.update({k: ts[k] for k in TENSORS[3:] if k in ts and k != "colsum"})
        G.gemm_bf16(ts["a"], ts["b"], ts["out"], **kw)
        torch.cuda.synchronize()
        d = {"call": i, "M": shape_of(c)[0], "N": shape_of(c)[1], "K": shape_of(c)[2], "flags": c["flags"]}
        for k in ("out", "aux"):
            if k in ts:
                d[k] = hashlib.sha256(ts[k].contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
        res.append(d)
    return res


def check_bits(a):
    """Run output_digests under this tree and a.check_bits, one process each, and compare."""
    runs = {}
    for tree in (a.tree, a.check_bits):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--tree", tree, "--batch", str(a.batch),
                            "--digests"], capture_output=True, text=True)
        if r.returncode != 0:
            print(r.stdout[-2000:] + r.stderr[-4000:], file=sys.stderr)
            return 1
        runs[tree] = json.loads(r.stdout.strip().splitlines()[-1])
    mine, other = runs[a.tree], runs[a.check_bits]
    bad = 0
    if len(mine) != len(other):
        print(json.dumps({"error": "different call lists", "calls": [len(mine), len(other)]}))
        return 1
    for x, y in zip(mine, other):
        same = {k: x.get(k) == y.get(k) for k in ("out", "aux") if k in x or k in y}
        bad += not all(same.values())
        print(json.dumps({k: x[k] for k in ("call", "M", "N", "K", "flags")} | {"equal": same}), flush=True)
    summary = {"check_bits": os.path.abspath(a.check_bits), "calls": len(mine), "mismatches": bad}
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "check_bits.json"), "w") as f:
            json.dump(summary, f)
    return 1 if bad else 0


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=6912)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="", help="also write the JSON lines to DIR/bench_gemm.jsonl")
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--check-bits", default="", metavar="OTHER_TREE",
                    help="compare the outputs of every non-accumulating call with OTHER_TREE's, bit for bit")
    ap.add_argument("--digests", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args(argv)
    if a.check_bits and not os.path.isdir(os.path.join(a.check_bits, "hugectr_b200")):
        raise SystemExit(f"bench_gemm: {a.check_bits} holds no hugectr_b200 package")
    if not os.path.isdir(os.path.join(a.tree, "hugectr_b200")):
        raise SystemExit(f"bench_gemm: {a.tree} holds no hugectr_b200 package")
    if not torch.cuda.is_available():
        print("bench_gemm: needs a CUDA device (an H100); nothing was measured", file=sys.stderr)
        return 1
    if a.check_bits:
        return check_bits(a)
    sys.path.insert(0, os.path.abspath(a.tree))
    if a.digests:
        print(json.dumps(output_digests(a.batch)))
        return 0
    from hugectr_b200.ops import gemm as G
    name, info = card()
    head = {"device": name, "power_limit,sm_clock,max_sm_clock": info, "tree": os.path.abspath(a.tree),
            "batch": a.batch}
    print("# " + json.dumps(head), flush=True)
    calls = record_calls(a.batch)
    gen = torch.Generator().manual_seed(0)
    lines, tot = [head], {"ours": 0.0, "mm": 0.0, "library": 0.0, "floor": 0.0}
    for i, c in enumerate(calls):
        ts = make_operands(c, gen)
        M, N, K = shape_of(c)
        kw = dict(a_mn=c["a_mn"], b_mn=c["b_mn"], flags=c["flags"], splits=c["splits"], alpha=c["alpha"])
        kw.update({k: ts[k] for k in TENSORS[3:] if k in ts})
        A = ts["a"].t() if c["a_mn"] else ts["a"]
        B = ts["b"] if c["b_mn"] else ts["b"].t()

        def ours():
            G.IMPL = "tc"
            G.gemm_bf16(ts["a"], ts["b"], ts["out"], **kw)

        def library():
            G.IMPL = "library"
            G.gemm_bf16(ts["a"], ts["b"], ts["out"], **kw)
            G.IMPL = "tc"

        picks, tuned = [], G._tuned_block_n

        def spy_tuned(*args):
            picks.append(tuned(*args))
            return picks[-1]

        G._tuned_block_n = spy_tuned
        try:
            ms = time_arms({"ours": ours, "mm": lambda: torch.mm(A, B), "library": library}, a.iters, a.rounds)
        finally:
            G._tuned_block_n = tuned
        G.IMPL = "tc"
        flop, byt = 2.0 * M * N * K, nbytes(c)
        floor_ms = max(flop / PEAK_FLOPS, byt / PEAK_BW) * 1e3
        r = {"call": i, "M": M, "N": N, "K": K, "a_mn": c["a_mn"], "b_mn": c["b_mn"], "flags": c["flags"],
             "splits": c["splits"], "operands": [k for k in TENSORS[3:] if k in c], "block_n": picks[-1],
             "floor_ms": round(floor_ms, 5),
             "floor_bound": "compute" if flop / PEAK_FLOPS >= byt / PEAK_BW else "memory"}
        for k, t in ms.items():
            r[k] = {"ms": round(t, 5), "tflops": round(flop / t / 1e9, 1), "gbps": round(byt / t / 1e6, 1),
                    "floor_share": round(floor_ms / t, 3)}
            tot[k] += t
        tot["floor"] += floor_ms
        print(json.dumps(r), flush=True)
        lines.append(r)
        del ts
    tot = {k: round(v, 4) for k, v in tot.items()}
    tot["calls"] = len(calls)
    print(json.dumps({"total_ms": tot}), flush=True)
    lines.append({"total_ms": tot})
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_gemm.jsonl"), "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
