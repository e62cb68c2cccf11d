"""Multi-process tests: gloo/CPU (world 2) here, NCCL + P2P fused kernels on the GPU box."""
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _run(nproc, args, port, env=None, timeout=300):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(HERE, "dist_worker.py"), *args]
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=e)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


# ----------------------------------------------------------------------------- one 2-rank session for the plain cases
# Interpreter start-up dominates a gloo test (two workers importing torch ~ 6 s): the world-2 cases that need no
# special environment share ONE torchrun session (dist_worker.py `multi`); every test below checks its own marker.
W2_FUZZ = ",".join(str(200 + i) for i in range(6))


@pytest.fixture(scope="module")
def world2(tmp_path_factory):
    d = tmp_path_factory.mktemp("world2")
    specs = ["ebc;mixed;collective", "ebc;column;collective", "model", "equiv;sgd", "equiv;adagrad", "legacy",
             f"ckpt;{d / 'ckpt'}", "dynamic", "sok", f"fuzz;{W2_FUZZ}", "unique;0,1,2,3,5;adagrad",
             "legacy_equiv;distributed;adam;11,12", "legacy_equiv;localized;adam;11,12",
             f"resume;{d / 'r_ebc'};ebc", f"resume;{d / 'r_leg'};legacy", "sok_fuzz;1001,1002,1003,1004,1005,1006"]
    for sub in ("ckpt", "r_ebc", "r_leg"):
        (d / sub).mkdir()
    return _run(2, ["multi"] + specs, 29611, env={"CUDA_VISIBLE_DEVICES": ""}, timeout=1500)


def _in_process(what, args):
    """single-rank cases need no process group: run the worker mode right here"""
    sys.path.insert(0, HERE)
    import dist_worker as W
    from hugectr_b200.parallel.comm import Comm
    comm = Comm.single(torch.device("cpu"))
    fn = {"dynamic": lambda: W.run_dynamic(comm=comm),
          "fuzz": lambda: [W.run_fuzz(sd, comm=comm) for sd in args[0].split(",")],
          "ebcio": lambda: [(os.makedirs(os.path.join(args[0], sd), exist_ok=True),
                             W.run_ebcio(os.path.join(args[0], sd), sd, comm=comm)) for sd in args[1].split(",")]}[what]
    fn()


def _done(out, spec_prefix):
    return any(l.startswith("MULTI_DONE " + spec_prefix) for l in out.splitlines())


@pytest.mark.dist
@pytest.mark.parametrize("plan", ["mixed", "column"])
def test_ebc_collective_gloo(plan, world2):
    assert f"EBC_OK plan={plan}" in world2 and _done(world2, f"ebc;{plan}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["collective", "fused"])
@pytest.mark.parametrize("plan", ["mixed", "column"])
def test_ebc_multi_gpu(plan, mode):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(min(n, 4), ["ebc", plan, mode], 29621)
    assert "EBC_OK" in out


@pytest.mark.gpu
def test_p2p_allreduce():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(min(n, 8), ["allreduce"], 29631)
    assert "ALLREDUCE_OK" in out


@pytest.mark.dist
def test_model_data_parallel_gloo(world2):
    assert "MODEL_OK" in world2 and _done(world2, "model")


@pytest.mark.gpu
def test_model_multi_gpu_overlap_paths():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(min(n, 4), ["model"], 29651)
    assert "MODEL_OK" in out


@pytest.mark.dist
@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
def test_multi_rank_equals_single_process_gloo(opt, world2):
    assert world2.count("EQUIV_OK") >= 2 and _done(world2, f"equiv;{opt}")


@pytest.mark.gpu
def test_multi_gpu_equals_single_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(min(n, 8), ["equiv", "sgd"], 29671)
    assert "EQUIV_OK" in out
    out = _run(min(n, 8), ["equiv", "adagrad"], 29673)
    assert "EQUIV_OK" in out


@pytest.mark.dist
def test_legacy_embeddings_gloo(world2):
    assert "LEGACY_OK" in world2 and _done(world2, "legacy")


@pytest.mark.gpu
def test_legacy_embeddings_multi_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(min(n, 4), ["legacy"], 29691)
    assert "LEGACY_OK" in out


@pytest.mark.dist
def test_hierarchical_exchange_gloo():
    """2 logical nodes x 2 ranks: node-aware two-stage embedding exchange == single process"""
    out = _run(4, ["equiv", "sgd", "2"], 29701, env={"CUDA_VISIBLE_DEVICES": ""})
    assert "EQUIV_OK" in out


@pytest.mark.dist
def test_checkpoint_resharding_gloo(world2):
    """2-rank checkpoint (dense + embedding collection) loads into a single-process model"""
    assert "CKPT_OK" in world2 and _done(world2, "ckpt;")


@pytest.mark.dist
@pytest.mark.parametrize("nproc", [1, 2])
def test_dynamic_tables_in_collection_gloo(nproc, world2, capsys):
    if nproc == 2:
        assert "DYNAMIC_OK" in world2 and _done(world2, "dynamic")
        return
    _in_process("dynamic", [])
    assert "DYNAMIC_OK" in capsys.readouterr().out


@pytest.mark.dist
def test_sok_distributed_lookup_gloo(world2):
    assert "SOK_OK" in world2 and _done(world2, "sok")


@pytest.mark.parametrize("nproc", [1, 2, 3])
def test_randomised_collection_against_bruteforce_oracle_gloo(nproc, world2, capsys):
    """random tables / hotness / combiners / layouts / padded bags / sharding plans vs gather+scatter oracle"""
    seeds = ",".join(str(100 * nproc + i) for i in range(6))
    if nproc == 1:
        _in_process("fuzz", [seeds])
        out = capsys.readouterr().out
    elif nproc == 2:
        out, seeds = "\n".join(l for l in world2.splitlines() if l.startswith("FUZZ_OK 20")), W2_FUZZ
        assert _done(world2, "fuzz;")
    else:
        out = _run(nproc, ["fuzz", seeds], 29751 + nproc, env={"CUDA_VISIBLE_DEVICES": ""})
    assert out.count("FUZZ_OK") == 6, out[-2000:]


@pytest.mark.gpu
@pytest.mark.skipif(not os.environ.get("HCTR_TEST_EXPERIMENTAL"),
                    reason="not yet validated on a GPU box (tools_dev/next_round.sh runs it)")
def test_randomised_collection_against_bruteforce_oracle_gpu():
    n = min(torch.cuda.device_count(), 4)
    seeds = ",".join(str(500 + i) for i in range(8))
    out = _run(n, ["fuzz", seeds], 29761)
    assert out.count("FUZZ_OK") == 8, out[-2000:]


@pytest.mark.dist
@pytest.mark.parametrize("nproc", [1, 3])
def test_parallel_collection_dump_equals_gather_dump_gloo(nproc, tmp_path, capsys):
    """every rank writes its own windows of key / weight / opt files; chunked streamed load restores them"""
    seeds = ",".join(str(40 * nproc + i) for i in range(4))
    if nproc == 1:
        _in_process("ebcio", [str(tmp_path), seeds])
        out = capsys.readouterr().out
    else:
        out = _run(nproc, ["ebcio", str(tmp_path), seeds], 29771 + nproc, env={"CUDA_VISIBLE_DEVICES": ""})
    assert out.count("EBCIO_OK") == 4, out[-2000:]


@pytest.mark.dist
def test_embedding_collection_benchmark_script_gloo():
    """benchmarks/embedding_collection/benchmark.py: the 7-table mixed-width workload (ev 32..256, hotness up
    to 80) planned by plan_tables on 2 gloo ranks; then the SKIP_* ablation switches on one rank"""
    script = os.path.join(os.path.dirname(HERE), "benchmarks", "embedding_collection", "benchmark.py")
    args = ["--workload", "7table_470B_hotness20", "--batch_per_gpu", "16", "--iters", "2", "--warmup", "1",
            "--cap_rows", "300", "--fp32"]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29781", script] + args
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert '"gpus": 2' in r.stdout and '"tables": 7' in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]
    r = subprocess.run([sys.executable, script] + args, capture_output=True, text=True, timeout=600,
                       env=dict(env, SKIP_EMBEDDING="1", SKIP_ALLREDUCE="1", SKIP_H2D="1"))
    assert '"SKIP_EMBEDDING": "1"' in r.stdout and "ablation switches active" in (r.stdout + r.stderr), \
        r.stdout[-1500:] + r.stderr[-1500:]


@pytest.mark.dist
def test_symmetric_heap_failure_is_agreed_on_by_all_ranks_gloo():
    out = _run(3, ["symmfail"], 29791, env={"CUDA_VISIBLE_DEVICES": ""})
    assert "SYMMFAIL_OK" in out, out[-2000:]


@pytest.mark.dist
@pytest.mark.parametrize("nproc,seed", [(2, 11), (4, 12)])
def test_multi_rank_equals_single_process_random_plan_gloo(nproc, seed):
    """whole-model training under a random table / row / column / dp placement == single process (AdaGrad)"""
    out = _run(nproc, ["equiv", "adagrad"], 29800 + seed,
               env={"CUDA_VISIBLE_DEVICES": "", "HCTR_TEST_PLAN_SEED": str(seed)})
    assert "EQUIV_OK" in out, out[-2000:]


@pytest.mark.dist
@pytest.mark.parametrize("nproc,names", [(2, "0,1,2,3,5"), (3, "0,2")])
def test_unique_compression_exchange_gloo(nproc, names, world2):
    """CompressionStrategy.Unique on real processes: the count all-to-all and the variable all-to-alls of 64-bit
    key codes / embedding rows / pre-reduced gradient rows over gloo"""
    if nproc == 2:
        assert "UNIQUE_OK" in world2 and _done(world2, "unique;")
        return
    out = _run(nproc, ["unique", names, "adagrad"], 29741, env={"CUDA_VISIBLE_DEVICES": ""})
    assert "UNIQUE_OK" in out


@pytest.mark.dist
def test_model_with_unique_compression_equals_single_process_gloo():
    """whole model through the public API: ebc.shard(..., compression_strategy={Unique: [...]})"""
    out = _run(2, ["equiv", "adagrad"], 29751, env={"CUDA_VISIBLE_DEVICES": "", "HCTR_TEST_UNIQUE": "1"})
    assert "EQUIV_OK" in out


@pytest.mark.dist
@pytest.mark.parametrize("kind", ["distributed", "localized"])
def test_legacy_embeddings_equal_single_process_gloo(kind, world2):
    assert world2.count("LEGACY_EQUIV_OK") == 4 and _done(world2, f"legacy_equiv;{kind}")


@pytest.mark.dist
@pytest.mark.parametrize("legacy", ["ebc", "legacy"])
def test_multi_rank_exact_resume_gloo(legacy, world2):
    assert world2.count("RESUME_OK") == 2 and any(l.startswith("MULTI_DONE resume;") and l.endswith(";" + legacy)
                                                   for l in world2.splitlines())


@pytest.mark.dist
@pytest.mark.parametrize("nproc", [2, 3])
def test_sok_randomised_lookups_against_dense_oracle_gloo(nproc, world2):
    """random mixes of distributed / localized / dynamic SOK variables, hotness, combiners, weights, padded bags"""
    if nproc == 2:
        assert world2.count("SOK_FUZZ_OK") == 6 and _done(world2, "sok_fuzz;")
        return
    out = _run(nproc, ["sok_fuzz", "1001,1002,1003,1004,1005,1006"], 29781, env={"CUDA_VISIBLE_DEVICES": ""})
    assert out.count("SOK_FUZZ_OK") == 6