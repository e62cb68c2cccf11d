# %% [markdown]
# # hugectr_b200 quick start
#
# Generate a Criteo-shaped synthetic Parquet data set, train a DCN through the HugeCTR API (`import hugectr`), evaluate,
# checkpoint, reload the checkpoint into an inference session and export the model to ONNX.
# The notebook was executed on CPU (the same script runs unchanged on an H100: one process per GPU under `torchrun`).

# %%
import os
import numpy as np
import hugectr
from hugectr.tools import DataGenerator, DataGeneratorParams
print(hugectr.__version__)

# %% [markdown]
# ## 1. Data: `hugectr.tools.DataGenerator` (power-law keys, 26 one-hot slots, 13 dense features)

# %%
slots = [2000] * 26
gp = DataGeneratorParams(format=hugectr.DataReaderType_t.Parquet, label_dim=1, dense_dim=13, num_slot=26,
                         i64_input_key=True, source="./data/file_list.txt", eval_source="./data/file_list_test.txt",
                         slot_size_array=slots, dist_type=hugectr.Distribution_t.PowerLaw,
                         power_law_type=hugectr.PowerLaw_t.Short, num_files=2, eval_num_files=1,
                         num_samples_per_file=8192)
DataGenerator(gp).generate()
print(open("./data/file_list.txt").read())

# %% [markdown]
# ## 2. Model: solver, reader, optimizer, `model.add(...)`, `compile()`, `summary()`

# %%
solver = hugectr.CreateSolver(batchsize=512, batchsize_eval=512, lr=0.002, vvgpu=[[0]], repeat_dataset=True,
                              i64_input_key=True, max_eval_batches=8)
reader = hugectr.DataReaderParams(hugectr.DataReaderType_t.Parquet, source=["./data/file_list.txt"],
                                  eval_source="./data/file_list_test.txt", check_type=hugectr.Check_t.Non,
                                  slot_size_array=slots)
model = hugectr.Model(solver, reader, hugectr.CreateOptimizer(hugectr.Optimizer_t.Adam))
model.add(hugectr.Input(label_dim=1, label_name="label", dense_dim=13, dense_name="dense",
                        data_reader_sparse_param_array=[hugectr.DataReaderSparseParam("data1", 1, True, 26)]))
model.add(hugectr.SparseEmbedding(hugectr.Embedding_t.DistributedSlotSparseEmbeddingHash, 64, 16, "sum",
                                  "sparse_embedding1", "data1"))
model.add(hugectr.DenseLayer(hugectr.Layer_t.Reshape, ["sparse_embedding1"], ["reshape1"], leading_dim=416))
model.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["reshape1", "dense"], ["concat1"]))
model.add(hugectr.DenseLayer(hugectr.Layer_t.MultiCross, ["concat1"], ["multicross1"], num_layers=2))
model.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["concat1"], ["fc1"], num_output=256))
model.add(hugectr.DenseLayer(hugectr.Layer_t.ReLU, ["fc1"], ["relu1"]))
model.add(hugectr.DenseLayer(hugectr.Layer_t.Concat, ["relu1", "multicross1"], ["concat2"]))
model.add(hugectr.DenseLayer(hugectr.Layer_t.InnerProduct, ["concat2"], ["fc2"], num_output=1))
model.add(hugectr.DenseLayer(hugectr.Layer_t.BinaryCrossEntropyLoss, ["fc2", "label"], ["loss"]))
model.compile()
model.summary()

# %% [markdown]
# ## 3. Train with periodic evaluation (AUC), snapshot every 150 iterations
#
# (The generator's labels are random: the loss falls by memorisation and the evaluation AUC stays at 0.5 -- the point
# here is the API flow, not the metric.)

# %%
model.graph_to_json("dcn.json")
model.fit(max_iter=300, display=100, eval_interval=150, snapshot=150, snapshot_prefix="dcn")
print(sorted(f for f in os.listdir(".") if f.startswith("dcn")))

# %% [markdown]
# ## 4. Inference session over the checkpoint

# %%
from hugectr.inference import CreateInferenceSession, InferenceParams
sess = CreateInferenceSession("dcn.json", InferenceParams(
    model_name="dcn", max_batchsize=512, dense_model_file="dcn_dense_150.model",
    sparse_model_files=["dcn0_sparse_150.model"], i64_input_key=True))
batch = model.get_data_reader_eval()
import pyarrow.parquet as pq
files = open("./data/file_list_test.txt").read().split()[1:]
df = pq.read_table(files[0]).to_pandas().iloc[:512]
dense = df[[f"C{i + 1}" for i in range(13)]].to_numpy(dtype="float32")
keys = df[[f"S{i + 1}" for i in range(26)]].to_numpy(dtype="int64")
offsets = np.concatenate([[0], np.cumsum(slots)[:-1]])
pred = sess.predict(dense, (keys + offsets).reshape(-1))
print("predictions", pred[:8].round(4).reshape(-1), " mean", float(pred.mean()).__round__(4))

# %% [markdown]
# ## 5. ONNX export (`hugectr2onnx.converter.convert`)
#
# The converter rebuilds the inference graph from the graph JSON + model files and hands it to `torch.onnx.export`.
# Without the `onnx` package (as in the environment this notebook was executed in) it keeps the torch graph next to
# the requested path instead; either way the returned graph reproduces the model's predictions.

# %%
import torch
import hugectr2onnx
g = hugectr2onnx.converter.convert(onnx_model_path="dcn.onnx", graph_config="dcn.json",
                                   dense_model="dcn_dense_150.model", convert_embedding=True,
                                   sparse_models=["dcn0_sparse_150.model"])
print(sorted(f for f in os.listdir(".") if f.startswith("dcn.onnx")))
with torch.no_grad():
    out = g(torch.from_numpy(dense), torch.from_numpy(keys + offsets).view(512, 26, 1))
print("converter graph vs inference session: max |diff| =", float((out.reshape(-1) - torch.from_numpy(pred).reshape(-1)).abs().max()))
