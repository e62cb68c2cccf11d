"""Cost of update tracking (EmbeddingTableConfig(track_updates=True)) on the bench.py DLRM-DCNv2 configuration, one
GPU: device-timed steps with every table tracked against none, the stamp kernel's time per step
(torch.profiler), and the time and bytes of a delta export after 100 steps.  Prints one JSON line with the card name
and power limit read in the same run.

  python tools_dev/bench_emb_delta.py [--rounds 2] [--windows 3] [--steps 30]

The configuration is bench.py's one-GPU run: 6912 samples per step, the Criteo-TB tables capped at 10M rows, fp32
AdaGrad state, the "auto" sharding plan, CUDA graph on.  Steps are timed as bench.py times them: ``_run_step()`` over
a device-resident pool of batches, CUDA events around each window.  The two models do not fit the card together, so
each round builds the tracked model, times ``--windows`` windows, tears it down, and does the same for the untracked
model.  Data-parallel tables carry no stamps (they are written whole), so tracking every table tracks the
model-parallel ones."""
import argparse
import gc
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PER_GPU_BATCH = 6912          # bench.py PER_GPU_BATCH
ROW_CAP_1GPU = 10_000_000     # bench.py ROW_CAP_1GPU


def build(track, cap, batch):
    import torch
    from hugectr_b200.models.dlrm import CRITEO_TB_MULTI_HOT, CRITEO_TB_TABLE_SIZES, build_dlrm_dcnv2
    from hugectr_b200.ops import gemm as G
    from hugectr_b200.parallel.comm import Comm
    from hugectr_b200.tools.planner import generate_plan
    G.set_impl("tc")
    tables = [min(t, cap) for t in CRITEO_TB_TABLE_SIZES]
    m = build_dlrm_dcnv2(batchsize=batch, num_gpus=1, table_sizes=tables, mixed=True, lr=0.004, scaler=1.0,
                         shard_plan=generate_plan(tables, CRITEO_TB_MULTI_HOT, 1, plan="auto"),
                         comm=Comm.single(torch.device("cuda", 0)), use_cuda_graph=True)
    for cfg in m.ebc_configs:
        for t in cfg.tables():
            t.track_updates = track
    m.compile()
    return m


class Resident:
    """bench.py's device-timed loop: the reader's pool on the device, every step trains the next batch"""

    def __init__(self, m):
        inp = m.input
        self.m = m
        self.label = m.net_train.tensors[inp.label_name].data
        self.dense = m.net_train.tensors[inp.dense_name].data
        self.slab = m.ebcs_train[0].key_slab
        dev = m.device
        self.pool = [(hb.label.to(dev).view_as(self.label), hb.dense.to(dev).view_as(self.dense).to(self.dense.dtype),
                      hb.keys.to(dev)) for hb in m.reader_train.pool]
        self.i = 0

    def step(self):
        lab, den, keys = self.pool[self.i % len(self.pool)]
        self.i += 1
        self.label.copy_(lab, non_blocking=True)
        self.dense.copy_(den, non_blocking=True)
        self.slab[:keys.numel()].copy_(keys, non_blocking=True)
        self.m._run_step()

    def timed(self, n):
        import torch
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            self.step()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cap-rows", type=int, default=ROW_CAP_1GPU)
    ap.add_argument("--batch", type=int, default=PER_GPU_BATCH)
    ap.add_argument("--steps", type=int, default=30, help="steps per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per model build")
    ap.add_argument("--rounds", type=int, default=2, help="builds of each model, alternated")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    os.environ.setdefault("HCTR_SYNTH_POOL", "64")
    os.environ["HCTR_EMB_STATE_BF16"] = "0"
    times = {"tracked": [], "untracked": []}
    extra = {}
    for r in range(args.rounds):
        for name in ("tracked", "untracked"):
            m = build(name == "tracked", args.cap_rows, args.batch)
            for _ in range(8):                      # eager warm-up, capture, replays (as bench.py)
                m.train()
            run = Resident(m)
            for _ in range(5):
                run.step()
            torch.cuda.synchronize()
            times[name] += [run.timed(args.steps) for _ in range(args.windows)]
            if name == "tracked" and r == args.rounds - 1:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(10):
                        run.step()
                    torch.cuda.synchronize()
                ka = [e for e in prof.key_averages() if "stamp_rows" in e.key]
                extra["stamp_kernel_us_per_step"] = round(sum(e.device_time_total for e in ka) / 10, 2)
                extra["stamp_launches_per_step"] = sum(e.count for e in ka) / 10
                extra["stamp_bytes"] = sum(g.stamp.numel() * 4 for e in m.ebcs_train for g in e.groups
                                           if g.stamp is not None)
                since = m.embedding_clocks()
                for _ in range(100):
                    run.step()
                torch.cuda.synchronize()
                with tempfile.TemporaryDirectory() as d:
                    t0 = time.time()
                    m.embedding_dump_delta(f"{d}/delta", since)
                    secs = time.time() - t0
                    files = [os.path.join(p, f) for p, _, fs in os.walk(d) for f in fs]
                    extra["delta_after_100_steps"] = {
                        "seconds": round(secs, 3), "bytes": sum(os.path.getsize(f) for f in files),
                        "rows": sum(os.path.getsize(f) - 128 for f in files
                                    if os.path.basename(f).startswith("weight")) // (4 * 128)}
            m.close()
            del run, m
            gc.collect()
            torch.cuda.empty_cache()

    def med(v):
        return sorted(v)[len(v) // 2]
    res = {"card": card, "cap_rows": args.cap_rows, "batch": args.batch, "steps_per_window": args.steps,
           "ms_per_step": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "ms_per_step_median": {k: round(med(v), 4) for k, v in times.items()},
           "ms_per_step_spread": {k: round(max(v) - min(v), 4) for k, v in times.items()}, **extra}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
