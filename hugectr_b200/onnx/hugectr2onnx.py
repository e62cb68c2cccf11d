"""ONNX converter (C39).

Parity with onnx_converter/hugectr2onnx/{converter,graph_builder,hugectr_loader}.py: an independent
reader of the checkpoint formats (graph JSON, dense ``.model`` = flat fp32 weights in layer order,
sparse ``key`` / ``emb_vector`` files, hugectr_loader.py:222-237,336-358) that rebuilds the
*inference* graph out of standard operators and exports it.  The graph is a ``torch.nn.Module``
(``InferenceGraph``); serialisation uses ``torch.onnx.export`` (the ``onnx`` python package itself is
not needed for the TorchScript exporter).  Inputs of the exported graph: dense [b, dense_dim] and,
per sparse input, int64 keys [b, slot_num, max_nnz] (convert_embedding=True) -- otherwise the
embedding outputs themselves are graph inputs, like the reference's ``convert_embedding=False``.
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


def load_sparse_model(path: str, vec: int):
    keys = np.fromfile(os.path.join(path, "key"), dtype="<i8")
    emb = np.fromfile(os.path.join(path, "emb_vector"), dtype="<f4").reshape(-1, vec)
    return torch.from_numpy(keys.astype("int64")), torch.from_numpy(emb.copy())


def load_dense_weights(path: str) -> torch.Tensor:
    return torch.from_numpy(np.fromfile(path, dtype="<f4").copy())


def _as_list(v):
    return list(v) if isinstance(v, (list, tuple)) else [v]


class _KeyedEmbedding(nn.Module):
    """key -> row lookup with sum/mean combiner.  When the key space is small (slot-offset keys of the
    legacy embeddings: max key < 2**24) a dense key -> row table is used (a plain Gather, exportable
    to ONNX); otherwise a sorted-key binary search (arbitrary int64 keys, torch-only)."""

    LUT_LIMIT = 1 << 24

    def __init__(self, keys, emb, combiner):
        super().__init__()
        order = torch.argsort(keys)
        keys = keys[order]
        n = keys.numel()
        self.register_buffer("emb", torch.cat([emb[order], torch.zeros(1, emb.shape[1])]))
        self.combiner = combiner
        self.n = n
        self.use_lut = bool(n > 0 and int(keys[-1]) < self.LUT_LIMIT and int(keys[0]) >= 0)
        if self.use_lut:
            lut = torch.full((int(keys[-1]) + 2,), n, dtype=torch.int64)      # last entry: "missing"
            lut[keys] = torch.arange(n, dtype=torch.int64)
            self.register_buffer("lut", lut)
        else:
            self.register_buffer("keys", keys)

    def forward(self, k):                       # k [b, S, H], -1 padded
        n = self.n
        if self.use_lut:
            top = self.lut.numel() - 1
            idx = torch.where((k >= 0) & (k < top), k, torch.full_like(k, top))
            rows = self.lut[idx]
        else:
            pos = torch.searchsorted(self.keys, k.clamp(min=0)).clamp(max=max(n - 1, 0))
            hit = (self.keys[pos] == k) & (k >= 0)
            rows = torch.where(hit, pos, torch.full_like(pos, n))
        v = self.emb[rows]                      # [b, S, H, vec]
        out = v.sum(2)
        if self.combiner == "mean":
            out = out / (k >= 0).sum(2, keepdim=True).clamp(min=1)
        return out


class InferenceGraph(nn.Module):
    def __init__(self, graph: dict, dense_weights: torch.Tensor, sparse_models: Optional[List[str]] = None,
                 convert_embedding: bool = False, ntp: Optional[dict] = None):
        super().__init__()
        self.layers = graph["layers"]
        data = self.layers[0]
        self.dense_name = data["dense"]["top"]
        self.sparse_inputs = [s["top"] for s in data.get("sparse", [])]
        self.emb_layers, self.dense_layers = [], []
        emb_types = ("DistributedSlotSparseEmbeddingHash", "LocalizedSlotSparseEmbeddingHash",
                     "LocalizedSlotSparseEmbeddingOneHot", "HybridSparseEmbedding")
        for l in self.layers[1:]:
            if l["type"] == "EmbeddingCollection":
                continue
            (self.emb_layers if l["type"] in emb_types else self.dense_layers).append(l)
        self.convert_embedding = convert_embedding
        self.embs = nn.ModuleDict()
        if convert_embedding:
            for i, l in enumerate(self.emb_layers):
                hp = l["sparse_embedding_hparam"]
                k, e = load_sparse_model(sparse_models[i], hp["embedding_vec_size"])
                self.embs[l["top"]] = _KeyedEmbedding(k, e, hp.get("combiner", "sum"))
        self.ntp = (ntp or {}).get("layers", {})
        # slice the flat weight vector in layer order
        self.w = nn.ParameterList()
        self.windex: Dict[int, List[int]] = {}
        self._off = 0
        self._flat = dense_weights
        self.shapes: Dict[str, tuple] = {}

    # weights are materialised lazily during the first (shape-discovering) forward
    def _take(self, li, shapes):
        if li in self.windex:
            return [self.w[i] for i in self.windex[li]]
        idx = []
        for shp in shapes:
            n = int(np.prod(shp))
            t = self._flat[self._off:self._off + n].reshape(shp).clone()
            self._off += n
            self.w.append(nn.Parameter(t, requires_grad=False))
            idx.append(len(self.w) - 1)
        self.windex[li] = idx
        return [self.w[i] for i in idx]

    def forward(self, dense, *extra):
        t = {self.dense_name: dense}
        if self.convert_embedding:
            for l, keys in zip(self.emb_layers, extra):
                t[l["top"]] = self.embs[l["top"]](keys)
        else:
            for l, e in zip(self.emb_layers, extra):
                t[l["top"]] = e
        if not self.emb_layers:          # EmbeddingCollection graphs: tops are passed as inputs
            names = [tp for l in self.layers[1:] if l["type"] == "EmbeddingCollection"
                     for tp in [lk["top"] for lk in l["lookups"]]]
            for n, e in zip(names, extra):
                t[n] = e
        out = None
        for li, l in enumerate(self.dense_layers):
            ty = l["type"]
            bots = [t[b] for b in _as_list(l["bottom"]) if b in t]
            tops = _as_list(l["top"])
            x = bots[0] if bots else None
            if ty in ("InnerProduct", "FusedInnerProduct"):
                n = l["fc_param"]["num_output"]
                W, b = self._take(li, [(x.shape[-1], n), (1, n)])
                y = x @ W + b
                if ty == "FusedInnerProduct":
                    y = F.relu(y)
            elif ty == "MLP":
                p = l["mlp_param"]
                outs = p["num_outputs"]
                acts = p.get("activations") or [p.get("activation", "Relu")] * len(outs)
                biases = p.get("biases") or [p.get("use_bias", True)] * len(outs)
                shapes, k = [], x.shape[-1]
                for n, hb in zip(outs, biases):
                    shapes.append((k, n))
                    if hb:
                        shapes.append((1, n))
                    k = n
                ws = self._take(li, shapes)
                y, wi = x, 0
                for n, a, hb in zip(outs, acts, biases):
                    y = y @ ws[wi]
                    wi += 1
                    if hb:
                        y = y + ws[wi]
                        wi += 1
                    if a == "Relu":
                        y = F.relu(y)
            elif ty == "MultiCross":
                p = l["mc_param"]
                L, pd, w = p["num_layers"], p.get("projection_dim", 0), x.shape[-1]
                if pd > 0:
                    ws = self._take(li, [s for _ in range(L) for s in ((w, pd), (pd, w), (1, w))])
                    y = x
                    for i in range(L):
                        y = x * ((y @ ws[3 * i]) @ ws[3 * i + 1] + ws[3 * i + 2]) + y
                else:
                    ws = self._take(li, [s for _ in range(L) for s in ((1, w), (1, w))])
                    y = x
                    for i in range(L):
                        y = x * (y @ ws[2 * i].reshape(-1, 1)) + ws[2 * i + 1] + y
            elif ty == "Interaction":
                mlp, emb = bots
                z = torch.cat([mlp.unsqueeze(1), emb], 1)
                zz = torch.bmm(z, z.transpose(1, 2))
                n = z.shape[1]
                li_, lj_ = torch.tril_indices(n, n, -1)
                y = torch.cat([mlp, zz[:, li_, lj_], torch.zeros_like(mlp[:, :1])], 1)
            elif ty == "WeightMultiply":
                (W,) = self._take(li, [tuple(l["weight_dims"])])
                y = (x.unsqueeze(2) * W).reshape(x.shape[0], -1)
            elif ty == "BatchNorm":
                n = x.shape[-1]
                g, b = self._take(li, [(1, n), (1, n)])
                st = None
                for k_, v in self.ntp.items():
                    if len(v["mean"]) == n and st is None:
                        st = v
                mean = torch.tensor(st["mean"]) if st else torch.zeros(n)
                var = torch.tensor(st["var"]) if st else torch.ones(n)
                y = (x - mean) / torch.sqrt(var + l["bn_param"]["eps"]) * g + b
            elif ty == "LayerNorm":
                n = x.shape[-1]
                g, b = self._take(li, [(1, n), (1, n)])
                y = F.layer_norm(x, (n,), g.reshape(-1), b.reshape(-1), l["ln_param"]["eps"])
            elif ty == "Reshape":
                if "selected" in l:
                    y = x[:, l["selected"], :].reshape(x.shape[0], -1)
                elif l.get("shape"):
                    y = x.reshape([s if s != -1 else -1 for s in l["shape"]])
                elif l.get("time_step", 0) > 0:
                    y = x.reshape(-1, l["time_step"], l["leading_dim"])
                else:
                    ld = l.get("leading_dim", 0) or int(np.prod(x.shape[1:]))
                    y = x.reshape(-1, ld)
            elif ty in ("Concat", "Concat3D"):
                y = torch.cat(bots, l.get("axis", 1))
            elif ty == "FusedReshapeConcat":            # [b, F+1, e_i] -> history [b*F, E], item [b, E]
                xc = torch.cat(bots, 2)
                f1 = xc.shape[1]
                t[tops[0]] = xc[:, :f1 - 1, :].reshape(-1, xc.shape[2])
                t[tops[1]] = xc[:, f1 - 1, :]
                out = t[tops[1]]
                continue
            elif ty == "FusedReshapeConcatGeneral":
                xc = torch.cat(bots, 2)
                y = xc.reshape(-1, xc.shape[2])
            elif ty == "MaskedSoftmax":
                v = torch.where(bots[1] > 0, x, torch.full_like(x, -10000.0)) if len(bots) > 1 else x
                y = torch.softmax(v, -1)
            elif ty == "SequenceMask":
                lf, lt = int(l["max_sequence_len_from"]), int(l["max_sequence_len_to"])
                a = bots[0].reshape(-1).float()
                b2 = bots[1].reshape(-1).float()
                mf = torch.arange(lf).view(1, -1, 1) < a.view(-1, 1, 1)
                mt = torch.arange(lt).view(1, 1, -1) < b2.view(-1, 1, 1)
                y = (mf & mt).unsqueeze(1).to(bots[0].dtype)
            elif ty == "Slice":
                ys = [x[..., a:b] for a, b in l["ranges"]]
                for n, v in zip(tops, ys):
                    t[n] = v
                continue
            elif ty in ("ReLU", "ReLUHalf"): y = F.relu(x)
            elif ty == "Sigmoid": y = torch.sigmoid(x)
            elif ty == "ELU": y = F.elu(x, l["elu_param"]["alpha"])
            elif ty == "Dropout" or ty == "Cast": y = x
            elif ty == "Add":
                y = bots[0]
                for b_ in bots[1:]:
                    y = y + b_
            elif ty == "Sub": y = bots[0] - bots[1]
            elif ty in ("ElementwiseMultiply", "DotProduct"):
                y = bots[0]
                for b_ in bots[1:]:
                    y = y * b_
            elif ty == "FmOrder2":
                v = x.reshape(x.shape[0], -1, l["out_dim"])
                s = v.sum(1)
                y = 0.5 * (s * s - (v * v).sum(1))
            elif ty == "ReduceSum": y = x.sum(l.get("axis", 1), keepdim=True)
            elif ty == "ReduceMean": y = x.mean(l.get("axis", 1), keepdim=True)
            elif ty == "Softmax":
                v = x if len(bots) == 1 else torch.where(bots[1] > 0, x, torch.full_like(x, -10000.0))
                y = torch.softmax(v, -1)
            elif ty == "MatrixMultiply": y = torch.matmul(bots[0], bots[1])
            elif ty == "Select": y = torch.index_select(x, l["dim"], torch.tensor(l["index"]))
            elif ty == "Gather": y = x[l["indices"]]
            elif ty == "Scale":
                f = int(l["scale_param"]["factor"])
                y = x.repeat_interleave(f, 1 if l["scale_param"]["axis"] == 0 else 0)
            elif ty == "PReLU_Dice":
                ex = x.mean(0, keepdim=True)
                var = (x * x).mean(0, keepdim=True) - ex * ex
                ps = torch.sigmoid((x - ex) / torch.sqrt(var + l["prelu_dice_param"]["eps"]))
                y = ps * x + (1 - ps) * l["prelu_dice_param"]["alpha"] * x
            elif ty == "MultiHeadAttention":
                q, k, v = bots[:3]
                h = l.get("num_attention_heads", 1)
                b_, sf, hd = q.shape
                dh = hd // h
                qh = q.reshape(b_, sf, h, dh).transpose(1, 2)
                kh = k.reshape(b_, -1, h, dh).transpose(1, 2)
                vh = v.reshape(b_, -1, h, dh).transpose(1, 2)
                s = qh @ kh.transpose(-1, -2) / math.sqrt(dh)
                if len(bots) > 3:
                    s = torch.where(bots[3] > 0, s, torch.full_like(s, -10000.0))
                y = (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(b_, sf, hd)
            elif ty in ("BinaryCrossEntropyLoss", "MultiCrossEntropyLoss"):
                out = torch.sigmoid(x)
                t[tops[0]] = out
                continue
            elif ty == "CrossEntropyLoss":
                out = torch.softmax(x, -1)
                t[tops[0]] = out
                continue
            else:
                raise NotImplementedError(f"hugectr2onnx: layer {ty} is not supported")
            t[tops[0]] = y
            out = y
        return out


def convert(onnx_model_path: str, graph_config: str, dense_model: str, convert_embedding: bool = False,
            sparse_models: Optional[List[str]] = None, ntp_file: Optional[str] = None,
            graph_name: str = "hugectr", batch_size: int = 2) -> InferenceGraph:
    graph = json.load(open(graph_config))
    for s in graph["layers"][0].get("sparse", []):
        if s.get("position_weighted"):
            # (checked before the dense file is read: the position weights follow the network's parameters in it)
            raise ValueError(f"position-weighted input {s['top']}: the ONNX export does not carry the position "
                             "weights")
    ntp = json.load(open(ntp_file)) if ntp_file and os.path.exists(ntp_file) else None
    g = InferenceGraph(graph, load_dense_weights(dense_model), sparse_models or [], convert_embedding, ntp)
    data = graph["layers"][0]
    dense = torch.zeros(batch_size, data["dense"]["dense_dim"])
    extras = []
    sp = {s["top"]: s for s in data.get("sparse", [])}
    for s in sp.values():
        if s.get("weighted"):
            raise ValueError(f"weighted input {s['top']}: the ONNX export does not carry per-key weights")
    for l in g.emb_layers:
        s = sp[l["bottom"]]
        nnz = s["nnz_per_slot"]
        H = max(nnz) if isinstance(nnz, list) else nnz
        if convert_embedding:
            extras.append(torch.zeros(batch_size, s["slot_num"], H, dtype=torch.int64))
        else:
            extras.append(torch.zeros(batch_size, s["slot_num"], l["sparse_embedding_hparam"]["embedding_vec_size"]))
    for l in graph["layers"][1:]:
        if l["type"] == "EmbeddingCollection":
            tabs = {t_["name"]: t_ for t_ in l["tables"]}
            for lk in l["lookups"]:
                w = sum(tabs[n]["ev_size"] for n in lk["tables"])
                extras.append(torch.zeros(batch_size, w))
    g.eval()
    with torch.no_grad():
        g(dense, *extras)                      # materialise weights / validate shapes
    if g._off != g._flat.numel():
        raise RuntimeError(f"dense model has {g._flat.numel()} weights, the graph consumed {g._off}")
    try:
        torch.onnx.export(g, (dense, *extras), onnx_model_path, opset_version=17,
                          input_names=["dense"] + [f"in{i}" for i in range(len(extras))],
                          output_names=["output"], dynamo=False)
    except Exception as e:  # exporter not usable in this environment: keep the torch graph
        torch.save({"graph": graph, "state": g.state_dict()}, onnx_model_path + ".pt")
        g.export_error = str(e)
    return g
