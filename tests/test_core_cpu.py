"""core.py: the backend-neutral resource interface (reference HugeCTR/core/core.hpp) over both back-ends."""
import torch

from hugectr_b200 import core as K
from hugectr_b200.parallel.comm import Comm
from hugectr_b200.parallel.emu import run_ranks


def test_single_process_backend():
    c = Comm.single(torch.device("cpu"))
    r = K.as_core(c)
    assert isinstance(r, K.CoreResourceManager) and K.as_core(c) is r and K.as_core(r) is r
    assert (r.get_global_gpu_id(), r.get_global_gpu_count(), r.get_local_gpu_id(), r.get_local_gpu_count()) == (0, 1, 0, 1)
    assert r.get_device_id() == -1 and r.get_comm() is c
    kp = r.get_kernel_param()
    assert kp.num_sms == 132 and kp.warp_size == 32
    g = r.get_local_gpu()
    assert g.get_current_stream_name() == "default"
    g.set_stream("emb")
    assert g.get_current_stream_name() == "emb" and g.get_stream() is None       # (CPU: no streams)


def test_emulated_ranks_backend_and_node_topology():
    def body(c):
        c.local_size = 2                      # two "nodes" of two GPUs
        r = K.as_core(c)
        assert r.get_global_gpu_count() == 4 and r.get_local_gpu_count() == 2
        assert r.get_local_gpu_id() == c.rank % 2
        assert r.get_gpu_global_id_from_local_id(1) == (c.rank // 2) * 2 + 1
        assert r.get_gpu_local_id_from_global_id(3) == 1
        return r.get_global_gpu_id()
    assert run_ranks(4, body, device=torch.device("cpu"), p2p=False) == [0, 1, 2, 3]


def test_embedding_collection_and_sok_go_through_the_interface():
    from hugectr_b200 import sok
    from hugectr_b200.embedding.collection import (EmbeddingCollection, EmbeddingCollectionConfig,
                                                   EmbeddingTableConfig)
    from hugectr_b200.enums import Optimizer_t
    from hugectr_b200.solver import CreateOptimizer
    cpu = torch.device("cpu")
    cfg = EmbeddingCollectionConfig()
    cfg.embedding_lookup(EmbeddingTableConfig("t", 10, 4), "k", "e", "sum")
    core = K.TorchCoreResourceManager(Comm.single(cpu))
    e = EmbeddingCollection(cfg, 2, {"k": 1}, cpu, torch.float32, core, CreateOptimizer(Optimizer_t.SGD))
    assert e.core is core and e.comm is core.get_comm() and (e.rank, e.world) == (0, 1)
    sok.init(Comm.single(cpu))
    assert sok.core().get_global_gpu_count() == sok.num_gpus() == 1 and sok.rank() == 0
