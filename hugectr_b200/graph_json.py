"""Graph JSON round trip: ``Model.graph_to_json`` / ``Model.construct_from_json``.

Format parity: {"layers": [{type:"Data",label,dense,sparse[]}, {type:<Embedding>, bottom, top,
sparse_embedding_hparam{}, optimizer{}}, {type:<Layer>, bottom, top, ...}], "model_name"}
(HugeCTR/src/pybind/add_dense_layer.cpp:67-520 save_graph_to_json, model.cpp:382-437).
EmbeddingCollection configs are stored under an extra "EmbeddingCollection" entry (the reference
cannot serialise them; ours round-trips).
"""
from __future__ import annotations

from .enums import (Activation_t, Embedding_t, Initializer_t, Layer_t, Regularizer_t)
from .solver import (DataReaderSparseParam, DenseLayer, Input, OptParamsPy, SparseEmbedding)

_INIT2S = {Initializer_t.Default: "Default", Initializer_t.Uniform: "Uniform",
           Initializer_t.XavierNorm: "XavierNorm", Initializer_t.XavierUniform: "XavierUniform",
           Initializer_t.Zero: "Zero", Initializer_t.Sinusoidal: "Sinusoidal"}
_S2INIT = {v: k for k, v in _INIT2S.items()}
_ACT2S = {Activation_t.Relu: "Relu", Activation_t.Non: "None"}
_S2ACT = {"Relu": Activation_t.Relu, "None": Activation_t.Non, "Non": Activation_t.Non}


def _one_or_list(v):
    return v[0] if len(v) == 1 else list(v)


def _as_list(v):
    return list(v) if isinstance(v, (list, tuple)) else [v]


def dense_layer_to_json(c: DenseLayer) -> dict:
    t = c.layer_type
    j = {"type": t.name, "bottom": _one_or_list(c.bottom_names), "top": _one_or_list(c.top_names)}
    if t == Layer_t.BatchNorm:
        j["bn_param"] = {"factor": c.factor, "eps": c.eps, "gamma_init": _INIT2S[c.gamma_init_type],
                         "beta_init": _INIT2S[c.beta_init_type]}
    elif t == Layer_t.LayerNorm:
        j["ln_param"] = {"eps": c.eps, "gamma_init": _INIT2S[c.gamma_init_type],
                         "beta_init": _INIT2S[c.beta_init_type]}
    elif t == Layer_t.Dropout:
        j["rate"] = c.dropout_rate
    elif t == Layer_t.SequenceMask:
        j["max_sequence_len_from"] = c.max_sequence_len_from
        j["max_sequence_len_to"] = c.max_sequence_len_to
    elif t == Layer_t.ELU:
        j["elu_param"] = {"alpha": c.elu_alpha}
    elif t == Layer_t.MultiHeadAttention:
        j["num_attention_heads"] = c.num_attention_heads
        j["transpose_b"] = c.transpose_b
    elif t == Layer_t.MLP:
        j["mlp_param"] = {"num_output": c.num_output, "num_outputs": c.num_outputs,
                          "use_bias": c.use_bias, "biases": c.biases,
                          "activation": _ACT2S[c.act_type],
                          "activations": [_ACT2S[a] for a in c.activations],
                          "weight_init": _INIT2S[c.weight_init_type],
                          "bias_init": _INIT2S[c.bias_init_type],
                          "async_wgrad": c.compute_config.async_wgrad,
                          "fuse_wb": c.compute_config.fuse_wb}
    elif t in (Layer_t.InnerProduct, Layer_t.FusedInnerProduct):
        j["fc_param"] = {"num_output": c.num_output, "weight_init": _INIT2S[c.weight_init_type],
                         "bias_init": _INIT2S[c.bias_init_type]}
    elif t == Layer_t.MultiCross:
        j["mc_param"] = {"num_layers": c.num_layers, "projection_dim": c.projection_dim,
                         "weight_init": _INIT2S[c.weight_init_type],
                         "bias_init": _INIT2S[c.bias_init_type]}
    elif t == Layer_t.Reshape:
        if c.selected:
            j["selected"] = c.selected_slots
        j["leading_dim"] = c.leading_dim
        j["time_step"] = c.time_step
        if c.shape:
            j["shape"] = c.shape
            # the reference's converter only understands leading_dim / time_step: spell [-1, d] and
            # [-1, t, d] shapes that way too (hugectr_loader.py:473-491)
            sh = list(c.shape)
            if len(sh) == 2 and sh[0] == -1:
                j["leading_dim"], j["time_step"] = sh[1], 0
            elif len(sh) == 3 and sh[0] == -1:
                j["leading_dim"], j["time_step"] = sh[2], sh[1]
    elif t in (Layer_t.Concat, Layer_t.ReduceSum, Layer_t.ReduceMean):
        j["axis"] = c.axis
    elif t == Layer_t.Slice:
        j["ranges"] = [list(r) for r in c.ranges]
    elif t == Layer_t.WeightMultiply:
        j["weight_dims"] = c.weight_dims
        j["weight_init"] = _INIT2S[c.weight_init_type]
    elif t == Layer_t.FmOrder2:
        j["out_dim"] = c.out_dim
    elif t == Layer_t.Gather:
        j["indices"] = c.indices
    elif t == Layer_t.Select:
        j["dim"] = c.dim
        j["index"] = c.index
    elif t == Layer_t.GRU:
        j["gru_param"] = {"num_output": c.num_output, "batchsize": c.batchsize,
                          "SeqLength": c.SeqLength, "vector_size": c.vector_size,
                          "weight_init": _INIT2S[c.weight_init_type],
                          "bias_init": _INIT2S[c.bias_init_type]}
    elif t == Layer_t.PReLU_Dice:
        j["prelu_dice_param"] = {"alpha": c.elu_alpha, "eps": c.eps}
    elif t == Layer_t.Scale:
        j["scale_param"] = {"axis": c.axis, "factor": c.factor}
    elif t == Layer_t.Softmax:
        j["factor"] = c.factor
    elif t in (Layer_t.BinaryCrossEntropyLoss, Layer_t.CrossEntropyLoss,
               Layer_t.MultiCrossEntropyLoss):
        if t == Layer_t.MultiCrossEntropyLoss:
            j["target_weight"] = c.target_weight_vec
        if c.use_regularizer:
            j["regularizer"] = c.regularizer_type.name
            j["lambda"] = c.lambda_
    return j


def dense_layer_from_json(j: dict) -> DenseLayer:
    name = j["type"]
    alias = {"FusedInnerProduct": "FusedInnerProduct", "ReLUHalf": "ReLU"}
    t = Layer_t[alias.get(name, name)]
    kw = {}
    g = j.get
    if "bn_param" in j:
        p = j["bn_param"]
        kw.update(factor=p["factor"], eps=p["eps"], gamma_init_type=_S2INIT[p["gamma_init"]],
                  beta_init_type=_S2INIT[p["beta_init"]])
    if "ln_param" in j:
        p = j["ln_param"]
        kw.update(eps=p["eps"], gamma_init_type=_S2INIT[p["gamma_init"]],
                  beta_init_type=_S2INIT[p["beta_init"]])
    if "rate" in j:
        kw["dropout_rate"] = j["rate"]
    for k in ("max_sequence_len_from", "max_sequence_len_to", "num_attention_heads", "transpose_b",
              "leading_dim", "time_step", "axis", "weight_dims", "out_dim", "indices", "dim",
              "index", "shape", "factor"):
        if k in j:
            kw[k] = j[k]
    if "elu_param" in j:
        kw["elu_alpha"] = j["elu_param"]["alpha"]
    if "mlp_param" in j:
        p = j["mlp_param"]
        from .solver import DenseLayerComputeConfig
        kw.update(num_output=p.get("num_output", 1), num_outputs=p.get("num_outputs", []),
                  use_bias=p.get("use_bias", True), biases=p.get("biases", []),
                  act_type=_S2ACT[p.get("activation", "Relu")],
                  activations=[_S2ACT[a] for a in p.get("activations", [])],
                  weight_init_type=_S2INIT[p.get("weight_init", "Default")],
                  bias_init_type=_S2INIT[p.get("bias_init", "Default")],
                  compute_config=DenseLayerComputeConfig(p.get("async_wgrad", False),
                                                         p.get("fuse_wb", False)))
    if "fc_param" in j:
        p = j["fc_param"]
        kw.update(num_output=p["num_output"], weight_init_type=_S2INIT[p.get("weight_init", "Default")],
                  bias_init_type=_S2INIT[p.get("bias_init", "Default")])
    if "mc_param" in j:
        p = j["mc_param"]
        kw.update(num_layers=p["num_layers"], projection_dim=p.get("projection_dim", 0),
                  weight_init_type=_S2INIT[p.get("weight_init", "Default")],
                  bias_init_type=_S2INIT[p.get("bias_init", "Default")])
    if "selected" in j:
        kw.update(selected=True, selected_slots=j["selected"])
    if "ranges" in j:
        kw["ranges"] = [tuple(r) for r in j["ranges"]]
    if "weight_init" in j:
        kw["weight_init_type"] = _S2INIT[j["weight_init"]]
    if "gru_param" in j:
        p = j["gru_param"]
        kw.update(num_output=p["num_output"], batchsize=p["batchsize"], SeqLength=p["SeqLength"],
                  vector_size=p["vector_size"])
    if "prelu_dice_param" in j:
        kw.update(elu_alpha=j["prelu_dice_param"]["alpha"], eps=j["prelu_dice_param"]["eps"])
    if "scale_param" in j:
        kw.update(axis=j["scale_param"]["axis"], factor=j["scale_param"]["factor"])
    if "target_weight" in j:
        kw["target_weight_vec"] = j["target_weight"]
    if "regularizer" in j:
        kw.update(use_regularizer=True, regularizer_type=Regularizer_t[j["regularizer"]],
                  lambda_=j.get("lambda", 0.0))
    return DenseLayer(t, _as_list(j["bottom"]), _as_list(j["top"]), **kw)


def model_to_json(model) -> dict:
    layers = []
    inp = model.input
    lab = {"top": _one_or_list(inp.label_names), "label_dim": _one_or_list(inp.label_dims)}
    layers.append({"type": "Data", "label": lab,
                   "dense": {"top": inp.dense_name, "dense_dim": inp.dense_dim},
                   "sparse": [{"top": p.top_name, "type": "DistributedSlot",
                               "nnz_per_slot": p.nnz_per_slot, "is_fixed_length": p.is_fixed_length,
                               "slot_num": p.slot_num, **({"weighted": True} if p.weighted else {}),
                               **({"position_weighted": True} if getattr(p, "position_weighted", False) else {})}
                              for p in inp.data_reader_sparse_param_array]})
    for se in model.sparse_embeddings:
        o = se.optimizer or model.opt_params
        per_gpu = getattr(se, "max_vocabulary_size_per_gpu", 0)
        if per_gpu <= 0 and se.workspace_size_per_gpu_in_mb > 0:      # model.cpp:186-196
            per_gpu = int(se.workspace_size_per_gpu_in_mb * 1024 * 1024 // ((1 + o.num_states) * 4 * se.embedding_vec_size))
        if per_gpu <= 0:
            per_gpu = max(1024, sum(se.slot_size_array or [0]) // max(1, model.world) + 1024)
        hp = {"workspace_size_per_gpu_in_mb": se.workspace_size_per_gpu_in_mb,
              "max_vocabulary_size_global": int(per_gpu * model.world),      # read by hugectr2onnx
              "embedding_vec_size": se.embedding_vec_size, "combiner": se.combiner}
        if se.slot_size_array:
            hp["slot_size_array"] = se.slot_size_array
        layers.append({"type": se.embedding_type.name, "bottom": se.bottom_name,
                       "top": se.sparse_embedding_name, "sparse_embedding_hparam": hp,
                       "optimizer": (se.optimizer or model.opt_params).to_json()})
    for cfg in model.ebc_configs:
        tabs = []
        for t in cfg.tables():
            tj = {"name": t.name, "max_vocabulary_size": t.max_vocabulary_size, "ev_size": t.ev_size,
                  "optimizer": t.opt_params.to_json() if t.opt_params else None}
            if t.dynamic:
                tj.update(init_capacity=t.init_capacity, max_capacity=t.max_capacity)
                if t.evict_strategy is not None:
                    tj["evict_strategy"] = t.evict_strategy
                if t.admit_threshold != 1:
                    tj["admit_threshold"] = t.admit_threshold
                if t.admit_decay_steps != 0:
                    tj["admit_decay_steps"] = t.admit_decay_steps
            if getattr(t, "weight_dtype", "fp32") != "fp32":
                tj["weight_dtype"] = t.weight_dtype
            if t.track_updates:
                tj["track_updates"] = True
            if t.init_param is not None and getattr(t.init_param, "up_bound", 0) > 0:
                tj["init_up_bound"] = float(t.init_param.up_bound)
            tabs.append(tj)
        lks = [{"tables": [t.name for t in lk["tables"]], "bottoms": lk["bottoms"], "top": lk["top"],
                "combiners": lk["combiners"], "batch_major": lk["batch_major"]} for lk in cfg.lookups]
        layers.append({"type": "EmbeddingCollection", "tables": tabs, "lookups": lks,
                       "shard_matrix": cfg.shard_matrix,
                       "shard_strategy": [[k, [list(i) if isinstance(i, tuple) else i for i in items]]
                                          for k, items in (cfg.shard_strategy or [])],
                       "use_exclusive_keys": cfg.use_exclusive_keys,
                       "comm_strategy": cfg.comm_strategy.name,
                       "compression_strategy": {getattr(k, "name", str(k)): [str(x) if not isinstance(x, int) else x for x in v]
                                                for k, v in (cfg.compression_strategy or {}).items()}})
    for c in model.dense_layers:
        if getattr(c, "_auto", False):
            continue
        layers.append(dense_layer_to_json(c))
    out = {"layers": layers}
    if model.solver.model_name:
        out["model_name"] = model.solver.model_name
    return out


def add_from_json(model, graph: dict, include_dense_network: bool = True):
    from .embedding.collection import EmbeddingCollectionConfig, EmbeddingTableConfig
    layers = graph["layers"]
    d = layers[0]
    assert d["type"] == "Data", "first layer of the graph JSON must be Data"
    sparse = [DataReaderSparseParam(s["top"], s["nnz_per_slot"], s["is_fixed_length"], s["slot_num"],
                                    weighted=bool(s.get("weighted", False)),
                                    position_weighted=bool(s.get("position_weighted", False)))
              for s in d.get("sparse", [])]
    lab = d["label"]
    model.add(Input(label_dims=_as_list(lab["label_dim"]), label_names=_as_list(lab["top"]),
                    dense_dim=d["dense"]["dense_dim"], dense_name=d["dense"]["top"],
                    data_reader_sparse_param_array=sparse))
    emb_names = {e.name for e in Embedding_t}
    for j in layers[1:]:
        t = j["type"]
        if t in emb_names:
            hp = j["sparse_embedding_hparam"]
            model.add(SparseEmbedding(Embedding_t[t], hp.get("workspace_size_per_gpu_in_mb", 0),
                                      hp["embedding_vec_size"], hp.get("combiner", "sum"), j["top"],
                                      j["bottom"], hp.get("slot_size_array", []),
                                      OptParamsPy.from_json(j["optimizer"]) if "optimizer" in j else None))
        elif t == "EmbeddingCollection":
            from .enums import CommunicationStrategy, CompressionStrategy
            from .embedding.collection import InitParams
            tabs = {}
            for tt in j["tables"]:
                kw = {k: tt[k] for k in ("init_capacity", "max_capacity", "weight_dtype", "evict_strategy",
                                         "admit_threshold", "admit_decay_steps", "track_updates") if k in tt}
                ip = InitParams(up_bound=tt["init_up_bound"]) if "init_up_bound" in tt else None
                tabs[tt["name"]] = EmbeddingTableConfig(
                    tt["name"], tt["max_vocabulary_size"], tt["ev_size"],
                    OptParamsPy.from_json(tt["optimizer"]) if tt.get("optimizer") else None, ip, **kw)
            cfg = EmbeddingCollectionConfig(j.get("use_exclusive_keys", False),
                                            CommunicationStrategy[j.get("comm_strategy", "Uniform")])
            for lk in j["lookups"]:
                if lk["batch_major"]:
                    cfg.embedding_lookup([tabs[n] for n in lk["tables"]], lk["bottoms"], lk["top"],
                                         lk["combiners"])
                else:
                    cfg.embedding_lookup(tabs[lk["tables"][0]], lk["bottoms"][0], lk["top"],
                                         lk["combiners"][0])
            if j.get("shard_matrix") is not None:
                ss = [(k, [tuple(i) if isinstance(i, list) else i for i in items])
                      for k, items in j["shard_strategy"]]
                comp = {CompressionStrategy[k]: v for k, v in (j.get("compression_strategy") or {}).items()}
                cfg.shard(j["shard_matrix"], ss, comp or None)
            model.add(cfg)
        elif include_dense_network:
            model.add(dense_layer_from_json(j))
