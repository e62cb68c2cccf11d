"""Inference session over a trained checkpoint (the API that survives as remnants in the reference:
InferenceParams / CreateInferenceSession / InferenceModel.predict, HugeCTR/include/inference/*;
HPS itself is removed upstream).  The session rebuilds the graph from its JSON, loads dense weights
and embedding tables and runs the eval network; embeddings may optionally be served through the
GPU hot-row cache (``use_gpu_embedding_cache`` + ``cache_size_percentage``)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from .enums import Check_t, DataReaderType_t
from .model import Model
from .parallel.comm import Comm
from .solver import CreateSolver, DataReaderParams, OptParamsPy


@dataclass
class InferenceParams:
    model_name: str
    max_batchsize: int
    hit_rate_threshold: float = 1.0
    dense_model_file: str = ""
    sparse_model_files: List[str] = field(default_factory=list)
    device_id: int = 0
    use_gpu_embedding_cache: bool = False
    cache_size_percentage: float = 0.2
    i64_input_key: bool = False
    use_mixed_precision: bool = False
    embedding_collection_path: str = ""
    # serve every embedding-collection table as fp8: e4m3 rows with one power-of-two scale per row, quantized
    # while the tables load, dequantized per looked-up row (the dense network still gets fp32 / bf16 inputs)
    fp8_quant: bool = False


class InferenceModel:
    def __init__(self, model_config_path: str, params: InferenceParams, device: Optional[str] = None):
        dev = torch.device(device) if device else (
            torch.device("cuda", params.device_id) if torch.cuda.is_available() else torch.device("cpu"))
        solver = CreateSolver(model_name=params.model_name, batchsize=params.max_batchsize,
                              batchsize_eval=params.max_batchsize, vvgpu=[[params.device_id]],
                              use_mixed_precision=params.use_mixed_precision,
                              i64_input_key=params.i64_input_key, use_cuda_graph=False)
        reader = DataReaderParams(DataReaderType_t.Parquet, source=["synthetic"], eval_source="synthetic",
                                  check_type=Check_t.Non)
        self.model = Model(solver, reader, OptParamsPy(), comm=Comm.single(dev))
        self.model.construct_from_json(model_config_path)
        weighted = [p.top_name for p in self.model.input.data_reader_sparse_param_array if getattr(p, "weighted", False)]
        if weighted:
            # predict() takes keys only: the weights of these inputs would be dropped
            raise ValueError(f"weighted input {weighted[0]}: the inference session does not take per-key weights")
        if params.fp8_quant and not self.model.ebc_configs:
            raise ValueError("fp8_quant quantizes embedding-collection tables; this model has none (legacy "
                             "SparseEmbedding tables keep their storage)")
        self.model.serving, self.model.fp8_quant = True, bool(params.fp8_quant)
        self.model.compile()
        if params.fp8_quant:
            from .utils import logger
            logger.info("fp8_quant: embedding-collection tables served as fp8: "
                        + ", ".join(t.name for e in self.model.ebcs_eval for t in e.tables))
        if params.dense_model_file:
            self.model.load_dense_weights(params.dense_model_file)
        self.hps = {}
        if params.sparse_model_files and params.use_gpu_embedding_cache and self.model.legacy_eval:
            # HPS-style serving: tables stay in the host parameter server, hot rows in the device cache
            from .cache import HpsEmbedding
            from .onnx.hugectr2onnx import load_sparse_model
            for rt, path in zip(self.model.legacy_eval, params.sparse_model_files):
                keys, emb = load_sparse_model(path, rt.vec)
                self.hps[rt.name] = HpsEmbedding(keys, emb, dev, params.cache_size_percentage,
                                                 "mean" if rt.combiner == 1 else "sum")
        elif params.sparse_model_files:
            self.model.load_sparse_weights(params.sparse_model_files)
        if params.embedding_collection_path:
            self.model.embedding_load(params.embedding_collection_path)
        self.params = params
        # {collection id: the until clock of the last delta applied} (update_embedding)
        self.delta_clocks = {}

    def update_embedding(self, path: str):
        """Apply a delta folder written by ``Model.embedding_dump_delta`` in place (new keys of a growing table
        are inserted, fp8 tables quantize the rows as they load).  Deltas apply in clock order: one whose
        ``since`` is after the ``until`` of the last delta applied to a collection leaves a gap and raises
        ValueError, and so does one whose ``until`` is before that clock (it would roll rows back to older values);
        an overlap is fine (rows carry absolute values).  The first delta after the full load is
        accepted whatever its ``since``.  A table the session lacks raises ValueError."""
        from .io.checkpoint import read_delta_info
        m = self.model
        info = read_delta_info(path, m)
        for eid, d in info.items():
            if eid >= len(m.ebcs_train):
                raise ValueError(f"delta {path}: embedding collection {eid} is not in this session")
            have = {t.name for t in m.ebcs_train[eid].tables}
            for n in d["tables"]:
                if n not in have:
                    raise ValueError(f"delta {path}: table {n} of embedding collection {eid} is not in this session")
            last = self.delta_clocks.get(eid)
            if last is not None and d["since"] > last:
                raise ValueError(f"delta {path}: embedding collection {eid} starts after clock {d['since']}, but the "
                                 f"session holds the rows of clock {last}: the deltas in between are missing")
            if last is not None and d["until"] < last:
                raise ValueError(f"delta {path}: embedding collection {eid} ends at clock {d['until']}, but the "
                                 f"session holds the rows of clock {last}: applying it would roll rows back")
        m.embedding_load(path)
        for eid, d in info.items():
            self.delta_clocks[eid] = int(d["until"])

    def predict(self, dense: np.ndarray, keys: np.ndarray) -> np.ndarray:
        """dense [n, dense_dim] float32, keys: feature-major key vector of the batch -> predictions"""
        m = self.model
        n = dense.shape[0]
        b = m.b_eval
        assert n <= b, "batch larger than max_batchsize"
        from .data.batch import HostBatch
        d = torch.zeros(b, m.input.dense_dim)
        d[:n] = torch.from_numpy(np.asarray(dense, dtype="float32"))
        k = torch.as_tensor(keys).to(m.key_dtype)
        hb = HostBatch(torch.zeros(b, m.input.label_dim), d, k, None, n)
        m._load_batch(hb, False)
        for e in m.ebcs_eval:
            e.forward(False)
        for rt in m.legacy_eval:
            if rt.name in self.hps:
                pooled = self.hps[rt.name].lookup(rt.keys_loc.view(rt.b, rt.S, rt.H))
                rt.top_data.copy_(pooled.to(rt.top_data.dtype))
            else:
                rt.forward(False)
        m.net_eval.fprop(False)
        ll = m.net_eval.loss_layers
        pred = ll[0].pred if len(ll) == 1 else torch.cat([l.pred.reshape(b, -1) for l in ll], 1)
        return pred[:n].float().cpu().numpy()


def CreateInferenceSession(model_config_path: str, inference_params: InferenceParams) -> InferenceModel:
    return InferenceModel(model_config_path, inference_params)
