"""``CompressionStrategy.Unique`` for model-parallel lookups on the collective (NCCL / gloo) path.

What it is (reference: HugeCTR/embedding/data_distributor/data_compression_operators.cu:30-601 -- segmented
unique of the keys per table before the exchange; model_parallel_embedding.cpp "DenseModelParallel" /
"DenseModelParallelWithReduction" groups; common.cpp:320-400 picks it per table): instead of shipping the whole
key block and receiving one pooled vector per sample, a requester sends every DISTINCT key of the step once,
receives one embedding row per distinct key, and pools locally; backward, it pre-reduces the gradient of every
distinct key and ships one gradient row per key.  Traffic scales with the number of distinct keys instead of
batch x hotness -- the win for "dense" (concat) lookups and for heavily repeated ids.

Design here: ONE exchange for all Unique lookups of a collection.  A key travels as a 64-bit code
``owner << 56 | lookup << 48 | key``; ``torch.unique`` of the codes yields the distinct set already grouped by
owner, a count all-to-all sizes the variable all-to-all of codes and of rows.  Owners de-duplicate again across
requesters before the optimizer (one update per row and step).  The counts are read on the host (one sync per
direction), so a model with Unique lookups runs its step eagerly -- the reference synchronises at the same place.

The peer-memory (fused) path does not use this: there the exchange is posted NVLink stores of pooled vectors
issued by the owner kernels; ``EmbeddingCollection`` keeps Unique tables on that path and says so once.
"""
from __future__ import annotations

from typing import List

import torch

from . import ops as E

KEY_BITS, LK_BITS = 48, 8
KEY_MASK = (1 << KEY_BITS) - 1


class UniqueExchange:
    def __init__(self, ebc, lookup_ids: List[int]):
        self.e = ebc
        self.ids = list(lookup_ids)
        assert len(self.ids) < (1 << LK_BITS), "too many Unique lookups in one collection"
        assert ebc.world < 128
        self.max_ev = max(ebc.glookups[g]["ev"] for g in self.ids)
        self._saved = None

    # ------------------------------------------------------------------ helpers
    def _a2a_counts(self, send_counts: torch.Tensor) -> List[int]:
        W = self.e.world
        recv = torch.empty(W, 1, dtype=torch.int64, device=send_counts.device)
        self.e.comm.all_to_all(recv, send_counts.view(W, 1).contiguous())
        return [int(x) for x in recv.view(-1).tolist()]

    def _a2a_v(self, send: torch.Tensor, send_counts: List[int], recv_counts: List[int], width: int = 1):
        out = torch.empty(sum(recv_counts) * width, dtype=send.dtype, device=send.device)
        self.e.comm.all_to_all_v(out, send.reshape(-1), [c * width for c in recv_counts],
                                 [c * width for c in send_counts])
        return out

    def _local_rows(self, lk: torch.Tensor, key: torch.Tensor):
        """(group, flat row index in that group's table, ev) of every received (lookup, key); rows of keys
        outside the table are -1"""
        e = self.e
        res = []
        for j, gi in enumerate(self.ids):
            sel = (lk == j).nonzero().view(-1)
            if sel.numel() == 0:
                continue
            gl = e.glookups[gi]
            loc = gl.get("unique_local")
            assert loc is not None, f"rank {e.rank} received keys of table {gl['table']} it does not hold"
            grp, sl = loc
            r = torch.div(key[sel], sl["k"], rounding_mode="floor")
            row = torch.where(r < sl["rows"], r + sl["row_off"], torch.full_like(r, -1))
            res.append((sel, grp, row, sl["ev"]))
        return res

    # ------------------------------------------------------------------ forward
    def forward(self):
        e = self.e
        b, W, dev = e.b, e.world, e.device
        codes, spans = [], []
        for j, gi in enumerate(self.ids):
            gl = e.glookups[gi]
            keys = e.key_views[gl["bottom"]].reshape(-1).long()
            owners = gl["unique_owners"]                      # GPU of row shard s = key % k
            k = len(owners)
            own = torch.as_tensor(owners, dtype=torch.int64, device=dev)[keys.clamp(min=0) % k]
            code = (own << (KEY_BITS + LK_BITS)) | (j << KEY_BITS) | (keys & KEY_MASK)
            codes.append(torch.where(keys >= 0, code, torch.full_like(code, -1)))
            spans.append(keys.numel())
        allc = torch.cat(codes)
        valid = allc >= 0
        uniq, inv_v = torch.unique(allc[valid], return_inverse=True)       # sorted: grouped by owner
        inv = torch.full_like(allc, -1)
        inv[valid] = inv_v
        send_counts_t = torch.bincount(uniq >> (KEY_BITS + LK_BITS), minlength=W)[:W]
        recv_counts = self._a2a_counts(send_counts_t)
        send_counts = [int(x) for x in send_counts_t.tolist()]
        got = self._a2a_v(uniq, send_counts, recv_counts)
        # ---- owner: one embedding row per received code
        lk = (got >> KEY_BITS) & ((1 << LK_BITS) - 1)
        key = got & KEY_MASK
        vec = torch.zeros(got.numel(), self.max_ev, dtype=e.act_dtype, device=dev)
        located = self._local_rows(lk, key)
        for sel, grp, row, ev in located:
            tmp = torch.empty(row.numel(), grp.pitch, dtype=e.act_dtype, device=dev)
            E.gather_rows(grp.table, grp.pitch, row, tmp)
            vec[sel, :ev] = tmp[:, :ev]
        back = self._a2a_v(vec, recv_counts, send_counts, self.max_ev).view(-1, self.max_ev)
        # ---- requester: expand + pool
        off = 0
        for j, gi in enumerate(self.ids):
            gl = e.glookups[gi]
            H, ev = gl["hotness"], gl["ev"]
            idx = inv[off:off + spans[j]]
            off += spans[j]
            rows = back[idx.clamp(min=0), :ev].float() * (idx >= 0).unsqueeze(-1)
            rows = rows.view(b, H, ev)
            tp = e.tops[gl["top"]]
            t2d = e.top_data[tp["name"]].reshape(b, -1) if not tp.get("alias") else e.top_data[tp["name"]]
            if gl["combiner"] == "concat":
                t2d[:, gl["col"]:gl["col"] + H * ev].copy_(rows.reshape(b, H * ev).to(t2d.dtype))
            else:
                pooled = rows.sum(1)
                if gl["combiner"] in ("mean", "average"):
                    pooled = pooled / float(H)           # kernel convention; _rescale_mean fixes short bags
                t2d[:, gl["col"]:gl["col"] + ev].copy_(pooled.to(t2d.dtype))
        self._saved = (inv, spans, uniq.numel(), send_counts, recv_counts, located, got.numel())

    # ------------------------------------------------------------------ backward
    def backward(self, lr_t, step_t):
        e = self.e
        if self._saved is None:
            return
        inv, spans, n_uniq, send_counts, recv_counts, located, n_got = self._saved
        self._saved = None
        b, dev = e.b, e.device
        acc = torch.zeros(n_uniq, self.max_ev, dtype=torch.float32, device=dev)
        off = 0
        for j, gi in enumerate(self.ids):
            gl = e.glookups[gi]
            H, ev = gl["hotness"], gl["ev"]
            idx = inv[off:off + spans[j]]
            off += spans[j]
            tp = e.tops[gl["top"]]
            g2d = e.top_grad[tp["name"]].reshape(b, -1) if not tp.get("alias") else e.top_grad[tp["name"]]
            if gl["combiner"] == "concat":
                g = g2d[:, gl["col"]:gl["col"] + H * ev].float().reshape(b * H, ev)
            else:
                g = g2d[:, gl["col"]:gl["col"] + ev].float()
                if gl["combiner"] in ("mean", "average"):
                    g = g / float(H)
                g = g.unsqueeze(1).expand(b, H, ev).reshape(b * H, ev)
            ok = idx >= 0
            acc[:, :ev].index_add_(0, idx[ok], g[ok])
        # one pre-reduced gradient row per distinct key, in the activation dtype like every other exchange
        got = self._a2a_v(acc.to(e.act_dtype), send_counts, recv_counts, self.max_ev).view(n_got, self.max_ev)
        for sel, grp, row, ev in located:
            ok = row >= 0
            if not bool(ok.any()):
                continue
            g = torch.zeros(int(ok.sum()), grp.pitch, dtype=torch.float32, device=dev)
            g[:, :ev] = got[sel[ok], :ev].float()
            if grp.stamp is not None:
                grp.stamp[row[ok]] = getattr(e, "_shared", e).evict_clock.to(torch.int32)
            E.update_rows(grp.opt.optimizer_type, grp.table, grp.s0, grp.s1, grp.pitch, row[ok], g,
                          e._hp(grp.opt), lr_t, step_t)

    def wire_elems(self):
        """(codes sent, rows received) of the last forward -- for tests / traffic accounting"""
        if self._saved is None:
            return None
        return self._saved[2], sum(self._saved[3])
