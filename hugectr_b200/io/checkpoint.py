"""Checkpoint formats (SURVEY 3.6) -- byte compatible with the reference:

  dense   <prefix>_dense_<iter>.model        raw fp32 master weights, layer creation order, each layer in
                                              set_weight order (MLP W0,b0,W1,b1..; MultiCross U,V,b per
                                              layer; FC W,b), weights [in,out] row-major
                                              (core23_network.cpp:113-141,301-314)
          <prefix>_opt_dense_<iter>.model    raw optimizer state(s): state0 for all params, then state1
          <prefix>_dense_<iter>.model.ntp.json   non-trainable params (BatchNorm running stats)
  sparse  <prefix><i>_sparse_<iter>.model/   directory: key (int64 each), slot_id (uint64 each,
          (legacy embeddings)                 Localized only), emb_vector (fp32 x vec)
                                              (distributed_slot_sparse_embedding_hash.cu:802-955)
          <prefix><i>_opt_sparse_<iter>.model concatenated raw per-state tensors
  EBC     <path>/embedding_collection_<id>/meta_data   int[5]{ntables,key_type,emb_type,0,0},
                                              int table_ids[], size_t key_nums[], int ev_lens[]
          key<tid> / weight<tid> / opt<tid>   128-byte head int[32]{type(1 key,2 weight,3 opt), table_id}
                                              then payload; load re-shards by key % num_shards
                                              (parameter_IO.cpp:179-580, data_info.hpp:19-22)
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from ..utils import logger
from .filesystem import FileSystemBuilder

FILE_HEAD_NBYTES = 128
META_HEAD_NBYTES = 20


def _fs(path, model=None):
    params = getattr(getattr(model, "reader_params", None), "data_source_params", None)
    return FileSystemBuilder.build_by_path(path, params)


# ------------------------------------------------------------------------------------ dense
def dense_paths(prefix: str, it: int):
    return (f"{prefix}_dense_{it}.model", f"{prefix}_opt_dense_{it}.model")


def save_dense(model, prefix: str, it: int):
    wpath, opath = dense_paths(prefix, it)
    if model.comm.rank == 0:
        fs = _fs(wpath, model)
        fs.write(wpath, model.arena.dump_flat().numpy().astype("<f4").tobytes())
        states = [model.arena.dump_state(s) for s in (model.opt_s0, model.opt_s1) if s is not None]
        fs.write(opath, b"".join(s.numpy().astype("<f4").tobytes() for s in states))
        ntp = {}
        for k, v in vars(model.arena).items():
            if k.startswith("_bn_state_"):
                ntp[k[len("_bn_state_"):]] = {"mean": v["mean"].cpu().tolist(),
                                              "var": v["var"].cpu().tolist()}
        if ntp:
            fs.write(wpath + ".ntp.json", json.dumps({"layers": ntp}).encode())
    model.comm.barrier()


def load_dense_weights(model, path: str):
    raw = _fs(path, model).read(path)
    flat = torch.from_numpy(np.frombuffer(raw, dtype="<f4").copy())
    if flat.numel() != model.arena.num_params:
        raise RuntimeError(f"dense model file has {flat.numel()} parameters, the network needs "
                           f"{model.arena.num_params}")
    model.arena.load_flat(flat)
    ntp = path + ".ntp.json"
    if os.path.exists(ntp):
        d = json.loads(open(ntp).read())["layers"]
        for k, v in d.items():
            st = getattr(model.arena, "_bn_state_" + k, None)
            if st is not None:
                st["mean"].copy_(torch.tensor(v["mean"]))
                st["var"].copy_(torch.tensor(v["var"]))


def load_dense_opt_states(model, path: str):
    raw = _fs(path, model).read(path)
    flat = torch.from_numpy(np.frombuffer(raw, dtype="<f4").copy())
    n = model.arena.num_params
    states = [s for s in (model.opt_s0, model.opt_s1) if s is not None]
    if flat.numel() != n * len(states):
        raise RuntimeError("dense optimizer state file does not match the optimizer / network")
    for i, s in enumerate(states):
        model.arena.load_state(s, flat[i * n:(i + 1) * n])


# ------------------------------------------------------------------------------------ legacy sparse
def sparse_paths(prefix: str, i: int, it: int):
    return (f"{prefix}{i}_sparse_{it}.model", f"{prefix}{i}_opt_sparse_{it}.model")


def save_sparse(model, prefix: str, it: int):
    for i, rt in enumerate(model.legacy_train):
        d, o = sparse_paths(prefix, i, it)
        rt.dump_parameters(d)
        rt.dump_opt_states(o)


def load_sparse_weights(model, paths):
    if isinstance(paths, dict):
        for name, p in paths.items():
            rt = [r for r in model.legacy_train if r.name == name]
            if not rt:
                raise KeyError(f"no sparse embedding named {name}")
            rt[0].load_parameters(p)
    else:
        for rt, p in zip(model.legacy_train, paths):
            rt.load_parameters(p)


def load_sparse_opt_states(model, paths):
    if isinstance(paths, dict):
        for name, p in paths.items():
            [r for r in model.legacy_train if r.name == name][0].load_opt_states(p)
    else:
        for rt, p in zip(model.legacy_train, paths):
            rt.load_opt_states(p)


def train_state_path(prefix: str, it: int):
    return f"{prefix}_train_state_{it}.json"


def save_train_state(model, prefix: str, it: int):
    """What the reference's snapshot leaves out (SURVEY 5.4): optimizer step count, iteration and
    learning-rate schedule position, so that ``Model.resume`` continues exactly where the run stopped."""
    if model.comm.rank != 0:
        return
    st = {"iteration": int(getattr(model, "_iter", it)), "snapshot": int(it),
          "optimizer_step": int(model.step_t.item()) if hasattr(model, "step_t") else int(it),
          "lr_scheduler": model.lr_sched.state_dict() if hasattr(model, "lr_sched") else {},
          "world_size": int(model.world)}
    _fs(prefix, model).write(train_state_path(prefix, it), json.dumps(st).encode())


def latest_snapshot(prefix: str, model=None):
    """largest <it> for which <prefix>_dense_<it>.model exists (any file system), or None"""
    import re
    d, base = (prefix.rsplit("/", 1) + [""])[:2] if "/" in prefix else ("", prefix)
    try:
        names = _fs(prefix, model).list_dir(d)
    except (FileNotFoundError, OSError):
        return None
    its = []
    for n in names:
        m = re.fullmatch(re.escape(base) + r"_dense_(\d+)\.model", n)
        if m:
            its.append(int(m.group(1)))
    return max(its) if its else None


def resume(model, prefix: str, it=None) -> int:
    """Load everything ``save_params_to_files(prefix, it)`` wrote -- dense weights + optimizer state,
    legacy sparse models + their optimizer states, embedding collections (weights + optimizer state) and
    the training counters -- and return the iteration to continue from.  ``it=None``: latest snapshot."""
    if it is None:
        it = latest_snapshot(prefix, model)
        if it is None:
            raise FileNotFoundError(f"no snapshot with prefix {prefix}")
    fs = _fs(prefix, model)
    d, o = dense_paths(prefix, it)
    load_dense_weights(model, d)
    if fs.exists(o):
        load_dense_opt_states(model, o)
    sp = [sparse_paths(prefix, i, it) for i in range(len(model.legacy_train))]
    if sp:
        load_sparse_weights(model, [a for a, _ in sp])
        if all(fs.exists(b) for _, b in sp):
            load_sparse_opt_states(model, [b for _, b in sp])
    if model.ebcs_train and fs.exists(f"{prefix}_ebc_{it}"):
        embedding_load(model, f"{prefix}_ebc_{it}")
    sp_state = train_state_path(prefix, it)
    if fs.exists(sp_state):
        st = json.loads(fs.read(sp_state).decode())
        model._iter = int(st["iteration"])
        model.step_t.fill_(int(st["optimizer_step"]))
        model.lr_sched.step = max(int(st.get("lr_scheduler", {}).get("step", 0)), model._iter)
    else:                                   # a snapshot written by the reference: counters from its name
        model._iter = int(it)
        model.step_t.fill_(int(it))
        model.lr_sched.step = int(it)
    model._graph = None
    return model._iter


def save_model(model, prefix: str, it: int):
    save_train_state(model, prefix, it)
    save_sparse(model, prefix, it)
    save_dense(model, prefix, it)
    if model.ebcs_train:
        embedding_dump(model, f"{prefix}_ebc_{it}", None)
    logger.info(f"Dumping dense weights / optimizer states / sparse models with prefix {prefix} iter {it}")


# ------------------------------------------------------------------------------------ EBC
def _file_head(ftype: int, table_id: int) -> bytes:
    head = np.zeros(FILE_HEAD_NBYTES // 4, dtype="<i4")
    head[0], head[1] = ftype, table_id
    return head.tobytes()


def _gather_table(model, ebc, name, parts=None):
    """rank 0 gets the whole table: (keys int64 [n], weights [n, ev], states); ``parts``: this rank's shards in
    the form of ``dump_table_local`` (default: all of them)"""
    parts = ebc.dump_table_local(name) if parts is None else parts
    allp = model.comm.all_gather_object(parts) if model.world > 1 else [parts]
    if model.comm.rank != 0:
        return None
    t = ebc.tmap[name]
    ev = t.ev_size
    seen = {}
    for rank_parts in allp:
        for (keys, w, c0, sts, kind) in rank_parts:
            if kind == "dp" and seen.get(("dp", c0)):
                continue                       # replicated: take one copy
            seen[("dp", c0)] = kind == "dp"
            seen.setdefault("chunks", []).append((keys, w, c0, sts))
    chunks = seen.get("chunks", [])
    allkeys = torch.unique(torch.cat([c[0] for c in chunks])) if chunks else torch.zeros(0, dtype=torch.int64)
    n = allkeys.numel()
    W = torch.zeros(n, ev)
    S = [torch.zeros(n, ev), torch.zeros(n, ev)]
    has_state = [False, False]
    for (keys, w, c0, sts) in chunks:
        pos = torch.searchsorted(allkeys, keys)
        W[pos, c0:c0 + w.shape[1]] = w
        for i, st in enumerate(sts):
            if st is not None:
                S[i][pos, c0:c0 + w.shape[1]] = st
                has_state[i] = True
    return allkeys, W, [S[i] if has_state[i] else None for i in range(2)]


def _parallel_plan(model, ebc, name):
    """Layout of one table in the shared key / weight / opt files for the parallel writer: every distinct
    local row set (static row shard s of k, or one dynamic shard) gets a contiguous row range; each
    (row set, column window) is written by exactly one rank (the lowest that holds it: data-parallel
    replicas are written once).  Returns None when a row set's column windows do not tile the full
    width (the gather path handles those)."""
    meta = ebc.table_parts(name)
    allm = model.comm.all_gather_object(meta) if model.world > 1 else [meta]
    ev = ebc.tmap[name].ev_size
    rowsets, writers, seen = {}, [], set()
    for r, m in enumerate(allm):
        for i, p in enumerate(m):
            rid = ("d", r, i) if p["dynamic"] else ("s", p["s"], p["k"], p["rows"])
            if p["dynamic"] and p["width"] != ev:
                return None
            if rid not in rowsets:
                rowsets[rid] = dict(rows=p["rows"], keyw=(r, i), cols=0)
            if (rid, p["col0"]) in seen:
                continue
            seen.add((rid, p["col0"]))
            rowsets[rid]["cols"] += p["width"]
            writers.append(dict(rank=r, idx=i, rid=rid, col0=p["col0"], width=p["width"]))
    # column windows are written through a shared memory map; across hosts (network file systems flush
    # whole pages of a mapping) only contiguous full-width row windows, written with pwrite, are safe
    multi_host = int(getattr(model.comm, "num_nodes", 1) or 1) > 1 or \
        os.environ.get("HCTR_EBC_DUMP_MULTIHOST", "0") == "1"
    if multi_host and any(w["width"] != ev for w in writers):
        return None
    off = 0
    for rs in rowsets.values():
        if rs["cols"] != ev:
            return None
        rs["off"] = off
        off += rs["rows"]
    nstate = max([p["nstate"] for m in allm for p in m] or [0])
    return dict(n=off, ev=ev, rowsets=rowsets, writers=writers, nstate=nstate)


def _dump_table_parallel(model, ebc, name, tid, folder, plan, kd):
    """Every rank writes its own row / column windows straight into the shared files (the role of the
    reference's MPI-IO writer, parameter_IO.cpp:37-250): no table is ever gathered on one rank."""
    n, ev, ns = plan["n"], plan["ev"], plan["nstate"]
    kb = np.dtype(kd).itemsize
    files = {"key": (f"{folder}/key{tid}", 1, n * kb), "weight": (f"{folder}/weight{tid}", 2, n * ev * 4)}
    if ns:
        files["opt"] = (f"{folder}/opt{tid}", 3, ns * n * ev * 4)
    if model.comm.rank == 0:
        for (fp, ftype, nbytes) in files.values():
            with open(fp, "wb") as f:
                f.write(_file_head(ftype, tid))
                f.truncate(FILE_HEAD_NBYTES + nbytes)
    model.comm.barrier()
    rank = model.comm.rank
    mine = [w for w in plan["writers"] if w["rank"] == rank]
    keyw = {rs["keyw"][1] for rs in plan["rowsets"].values() if rs["keyw"][0] == rank}
    need = {w["idx"] for w in mine} | keyw
    if need and n > 0:
        parts = ebc.dump_table_local(name, only=need)

        def pwrite_rows(path, arr, row_off, row_bytes):
            """contiguous rows [row_off, ...) of a [n, row_bytes] payload: plain positional writes"""
            buf = memoryview(np.ascontiguousarray(arr)).cast("B")
            fd = os.open(path, os.O_WRONLY)
            try:
                pos, off0 = 0, FILE_HEAD_NBYTES + row_off * row_bytes
                while pos < len(buf):
                    pos += os.pwrite(fd, buf[pos:pos + (1 << 30)], off0 + pos)
            finally:
                os.close(fd)
        for rs in plan["rowsets"].values():
            if rs["keyw"][0] == rank and rs["rows"]:
                pwrite_rows(files["key"][0], parts[rs["keyw"][1]][0].numpy().astype(kd), rs["off"], kb)
        strided = [w for w in mine if w["width"] != ev and plan["rowsets"][w["rid"]]["rows"]]
        mw = mo = None
        if strided:        # column windows of a column-sharded table (single host): strided map writes
            mw = np.memmap(files["weight"][0], dtype="<f4", mode="r+", offset=FILE_HEAD_NBYTES, shape=(n, ev))
            mo = np.memmap(files["opt"][0], dtype="<f4", mode="r+", offset=FILE_HEAD_NBYTES,
                           shape=(ns, n, ev)) if ns else None
        for w in mine:
            rs = plan["rowsets"][w["rid"]]
            if not rs["rows"]:
                continue
            keys, W, c0, sts, kind = parts[w["idx"]]
            lo, hi = rs["off"], rs["off"] + rs["rows"]
            if w["width"] == ev:
                pwrite_rows(files["weight"][0], W.numpy().astype("<f4"), lo, ev * 4)
                for i, st in enumerate(sts):
                    if st is not None and ns:
                        pwrite_rows(files["opt"][0], st.numpy().astype("<f4"), i * n + lo, ev * 4)
            else:
                mw[lo:hi, c0:c0 + W.shape[1]] = W.numpy()
                for i, st in enumerate(sts):
                    if st is not None and mo is not None:
                        mo[i, lo:hi, c0:c0 + W.shape[1]] = st.numpy()
        for m in (mw, mo):
            if m is not None:
                m.flush()
    model.comm.barrier()
    return n


def embedding_dump(model, path: str, table_names=None):
    fs = _fs(path, model)
    from .filesystem import LocalFileSystem
    if isinstance(fs, LocalFileSystem) and os.environ.get("HCTR_EBC_DUMP", "parallel") == "parallel":
        return _embedding_dump_parallel(model, path, table_names, fs)
    for eid, ebc in enumerate(model.ebcs_train):
        names = [t.name for t in ebc.tables]
        sel = [n for n in names if table_names is None or n in table_names]
        ids = sorted(names.index(n) for n in sel)
        folder = f"{path}/embedding_collection_{eid}"
        tabs = {}
        for tid in ids:
            tabs[tid] = _gather_table(model, ebc, names[tid])
        if model.comm.rank == 0:
            _write_ebc_folder(model, fs, folder, ebc, ids, tabs)
        model.comm.barrier()


def _write_ebc_folder(model, fs, folder, ebc, ids, tabs):
    """(rank 0) one collection's folder from whole tables ``tabs`` {table id: (keys, weights, states)}"""
    fs.create_dir(folder)
    head = np.zeros(5, dtype="<i4")
    head[0] = len(ids)
    head[1] = 1 if model.key_dtype == torch.int64 else 0
    head[2] = 0   # fp32 values
    meta = head.tobytes() + np.asarray(ids, dtype="<i4").tobytes() + \
        np.asarray([tabs[t][0].numel() for t in ids], dtype="<u8").tobytes() + \
        np.asarray([ebc.tables[t].ev_size for t in ids], dtype="<i4").tobytes()
    fs.write(f"{folder}/meta_data", meta)
    kd = "<i8" if model.key_dtype == torch.int64 else "<u4"
    for tid in ids:
        keys, W, S = tabs[tid]
        fs.write(f"{folder}/key{tid}", _file_head(1, tid) + keys.numpy().astype(kd).tobytes())
        fs.write(f"{folder}/weight{tid}", _file_head(2, tid) + W.numpy().astype("<f4").tobytes())
        st = [s for s in S if s is not None]
        if st:
            fs.write(f"{folder}/opt{tid}", _file_head(3, tid) +
                     b"".join(s.numpy().astype("<f4").tobytes() for s in st))


# a delta's clocks: the stamps are int32
DELTA_CLOCK_LIMIT = 1 << 31


def embedding_dump_delta(model, path: str, since=None, table_names=None):
    """Write, for every table with ``track_updates`` (of ``table_names``, when given), the keys whose rows were
    stamped after ``since[collection id]`` (0 when absent) with their current fp32 values, in the
    ``embedding_collection_<id>/`` layout, and ``delta.json`` with each collection's ``since`` / ``until``
    clocks, tracked tables and data-parallel tables (written whole).  Every rank takes part.  Returns the
    clocks at the time of the dump {collection id: clock}: the ``since`` of the next delta."""
    clocks = model.embedding_clocks()
    for eid, c in clocks.items():
        if c >= DELTA_CLOCK_LIMIT:
            raise RuntimeError(f"embedding collection {eid}: clock {c} reached 2^31, beyond the int32 row stamps")
    since = {eid: int((since or {}).get(eid, 0)) for eid in clocks}
    fs = _fs(path, model)
    info = {}
    for eid, ebc in enumerate(model.ebcs_train):
        names = [t.name for t in ebc.tables]
        tracked = [n for n in names if ebc.tmap[n].track_updates and (table_names is None or n in table_names)]
        ids = [names.index(n) for n in tracked]
        tabs = {}
        for tid in ids:
            n = names[tid]
            parts = ebc.delta_table_local(n, since[eid])
            if ebc.placement[n].col_factor > 1:
                # a key whose row any column slice stamped is written with its full row: every slice reads the
                # union of the stamped keys (the slices of a key are updated in the same steps, so they agree)
                mine = [p[0] for p in parts]
                allk = model.comm.all_gather_object(mine) if model.world > 1 else [mine]
                keys = [k for r in allk for k in r]
                keys = torch.unique(torch.cat(keys)) if keys else torch.zeros(0, dtype=torch.int64)
                parts = ebc.delta_table_local(n, since[eid], keys=keys)
            tabs[tid] = _gather_table(model, ebc, n, parts)
        if model.comm.rank == 0:
            _write_ebc_folder(model, fs, f"{path}/embedding_collection_{eid}", ebc, ids, tabs)
        info[str(eid)] = {"since": since[eid], "until": clocks[eid], "tables": tracked,
                          "data_parallel": [n for n in tracked if ebc.placement[n].kind == "dp"]}
    if model.comm.rank == 0:
        fs.write(f"{path}/delta.json", json.dumps({"collections": info}, indent=1).encode())
    model.comm.barrier()
    return clocks


def read_delta_info(path: str, model=None) -> dict:
    """{collection id: {since, until, tables, data_parallel}} of a folder written by embedding_dump_delta"""
    fs = _fs(path, model)
    if not fs.exists(f"{path}/delta.json"):
        raise ValueError(f"{path}: no delta.json, not a folder written by embedding_dump_delta")
    return {int(k): v for k, v in json.loads(fs.read(f"{path}/delta.json").decode())["collections"].items()}


def _embedding_dump_parallel(model, path, table_names, fs):
    kd = "<i8" if model.key_dtype == torch.int64 else "<u4"
    for eid, ebc in enumerate(model.ebcs_train):
        names = [t.name for t in ebc.tables]
        ids = sorted(names.index(n) for n in names if table_names is None or n in table_names)
        folder = f"{path}/embedding_collection_{eid}"
        if model.comm.rank == 0:
            fs.create_dir(folder)
        model.comm.barrier()
        knums = {}
        for tid in ids:
            plan = _parallel_plan(model, ebc, names[tid])
            logger.debug(f"embedding_dump table {names[tid]}: " + ("gather on rank 0" if plan is None else
                         f"parallel, {plan['n']} rows, {len(plan['writers'])} windows"))
            if plan is not None:
                knums[tid] = _dump_table_parallel(model, ebc, names[tid], tid, folder, plan, kd)
                continue
            tab = _gather_table(model, ebc, names[tid])       # irregular layout: gather on rank 0
            if model.comm.rank == 0:
                keys, W, S = tab
                fs.write(f"{folder}/key{tid}", _file_head(1, tid) + keys.numpy().astype(kd).tobytes())
                fs.write(f"{folder}/weight{tid}", _file_head(2, tid) + W.numpy().astype("<f4").tobytes())
                st = [x for x in S if x is not None]
                if st:
                    fs.write(f"{folder}/opt{tid}", _file_head(3, tid) +
                             b"".join(x.numpy().astype("<f4").tobytes() for x in st))
                knums[tid] = keys.numel()
        if model.comm.rank == 0:
            head = np.zeros(5, dtype="<i4")
            head[0] = len(ids)
            head[1] = 1 if model.key_dtype == torch.int64 else 0
            meta = head.tobytes() + np.asarray(ids, dtype="<i4").tobytes() + \
                np.asarray([knums[t] for t in ids], dtype="<u8").tobytes() + \
                np.asarray([ebc.tables[t].ev_size for t in ids], dtype="<i4").tobytes()
            fs.write(f"{folder}/meta_data", meta)
        model.comm.barrier()


def iter_ebc_folder(folder: str, chunk_rows: int = 1 << 22):
    """Streams a local EBC folder: yields (table_id, keys int64 [m], W [m, ev], states|None) in chunks of
    at most ``chunk_rows`` rows through memory maps, so a rank never holds a whole table on the host."""
    with open(f"{folder}/meta_data", "rb") as f:
        meta = f.read()
    head = np.frombuffer(meta[:META_HEAD_NBYTES], dtype="<i4")
    n, key_type = int(head[0]), int(head[1])
    off = META_HEAD_NBYTES
    ids = np.frombuffer(meta[off:off + 4 * n], dtype="<i4"); off += 4 * n
    knums = np.frombuffer(meta[off:off + 8 * n], dtype="<u8"); off += 8 * n
    evs = np.frombuffer(meta[off:off + 4 * n], dtype="<i4")
    kd = "<i8" if key_type == 1 else "<u4"
    for tid, kn, ev in zip(ids, knums, evs):
        tid, kn, ev = int(tid), int(kn), int(ev)
        if kn == 0:
            continue
        mk = np.memmap(f"{folder}/key{tid}", dtype=kd, mode="r", offset=FILE_HEAD_NBYTES, shape=(kn,))
        mw = np.memmap(f"{folder}/weight{tid}", dtype="<f4", mode="r", offset=FILE_HEAD_NBYTES, shape=(kn, ev))
        mo = None
        op = f"{folder}/opt{tid}"
        if os.path.exists(op):
            ns = (os.path.getsize(op) - FILE_HEAD_NBYTES) // (kn * ev * 4)
            mo = np.memmap(op, dtype="<f4", mode="r", offset=FILE_HEAD_NBYTES, shape=(ns, kn, ev))
        for lo in range(0, kn, chunk_rows):
            hi = min(kn, lo + chunk_rows)
            S = None if mo is None else [torch.from_numpy(np.array(mo[i, lo:hi])) for i in range(mo.shape[0])]
            yield (tid, torch.from_numpy(np.asarray(mk[lo:hi]).astype("int64")),
                   torch.from_numpy(np.array(mw[lo:hi])), S)


def read_ebc_folder(folder: str, fs=None):
    fs = fs or FileSystemBuilder.build_by_path(folder)
    meta = fs.read(f"{folder}/meta_data")
    head = np.frombuffer(meta[:META_HEAD_NBYTES], dtype="<i4")
    n, key_type = int(head[0]), int(head[1])
    off = META_HEAD_NBYTES
    ids = np.frombuffer(meta[off:off + 4 * n], dtype="<i4"); off += 4 * n
    knums = np.frombuffer(meta[off:off + 8 * n], dtype="<u8"); off += 8 * n
    evs = np.frombuffer(meta[off:off + 4 * n], dtype="<i4")
    kd = "<i8" if key_type == 1 else "<u4"
    out = {}
    for tid, kn, ev in zip(ids, knums, evs):
        tid, kn, ev = int(tid), int(kn), int(ev)
        kraw = fs.read(f"{folder}/key{tid}")[FILE_HEAD_NBYTES:]
        wraw = fs.read(f"{folder}/weight{tid}")[FILE_HEAD_NBYTES:]
        keys = torch.from_numpy(np.frombuffer(kraw, dtype=kd).astype("int64"))
        W = torch.from_numpy(np.frombuffer(wraw, dtype="<f4").copy()).view(int(kn), int(ev))
        S = None
        if fs.exists(f"{folder}/opt{tid}"):
            oraw = fs.read(f"{folder}/opt{tid}")[FILE_HEAD_NBYTES:]
            o = torch.from_numpy(np.frombuffer(oraw, dtype="<f4").copy())
            ns = o.numel() // max(1, int(kn) * int(ev))
            S = [o[i * kn * ev:(i + 1) * kn * ev].view(int(kn), int(ev)) for i in range(int(ns))]
        out[int(tid)] = (keys, W, S)
    return out


def embedding_load(model, path: str, table_names=None):
    fs = _fs(path, model)
    from .filesystem import LocalFileSystem
    local = isinstance(fs, LocalFileSystem)
    chunk = int(os.environ.get("HCTR_EBC_LOAD_CHUNK_ROWS", str(1 << 22)))
    for eid, ebc in enumerate(model.ebcs_train):
        folder = f"{path}/embedding_collection_{eid}"
        if local:
            names = [t.name for t in ebc.tables]
            for tid, keys, W, S in iter_ebc_folder(folder, chunk):
                if table_names is None or names[tid] in table_names:
                    ebc.load_table_rows(names[tid], keys, W, S)
            ebc.check_quantized()
            continue
        tabs = read_ebc_folder(folder, fs)
        names = [t.name for t in ebc.tables]
        for tid, (keys, W, S) in tabs.items():
            n = names[tid]
            if table_names is not None and n not in table_names:
                continue
            ebc.load_table_rows(n, keys, W, S)
        ebc.check_quantized()
    model.comm.barrier()
