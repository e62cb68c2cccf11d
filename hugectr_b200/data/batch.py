"""Host-side batch container shared by all readers.

Layout handed to the model (per rank, ``b`` = samples of this rank):
  label  [b, label_dim] fp32      dense [b, dense_dim] fp32
  keys   1-D, *feature-major*: for sparse param p (in Input order) a block [b, S_p * H_p]
         (slot_num x max nnz per slot), padded with -1 for variable-length slots
  nnz    optional 1-D int32: for param p a block [S_p, b] with the valid count per (slot, sample)
  weights optional 1-D fp32 in the layout of keys: the weight of every key of a weighted input (1 for
         the keys of unweighted inputs); None when no input is weighted
All tensors are pinned so the H2D copies are asynchronous.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch


@dataclass
class HostBatch:
    label: torch.Tensor
    dense: torch.Tensor
    keys: torch.Tensor
    nnz: Optional[torch.Tensor] = None
    num_valid: int = -1   # < b for an incomplete last batch
    copied: object = None  # CUDA event recorded after the last async H2D copy out of this batch
    _event: object = None  # the event object is created once per batch and re-recorded
    raw: Optional[torch.Tensor] = None   # device-split readers: the batch's raw records (pinned uint8) ...
    raw_skew: int = 0                    # ... starting at this byte offset; label / dense / keys are None
    splitter: object = None              # RawSplit: knows how to turn ``raw`` into the three tensors on the device
    weights: Optional[torch.Tensor] = None

    def mark_copied(self):
        """Called by the consumer right after it queued its asynchronous H2D copies: ring-buffer
        readers wait on this before they hand the staging slot back to their producer threads."""
        if torch.cuda.is_available():
            if self._event is None:
                self._event = torch.cuda.Event()
            self._event.record()
            self.copied = self._event

    def wait_copied(self):
        if self.copied is not None:
            self.copied.synchronize()
            self.copied = None

    def pin(self):
        if torch.cuda.is_available():
            for n in ("label", "dense", "keys", "nnz", "weights"):
                t = getattr(self, n)
                if t is not None and not t.is_pinned():
                    setattr(self, n, t.pin_memory())
        return self

    def h2d_bytes(self) -> int:
        if self.raw is not None:
            return int(self.splitter.batch * self.splitter.rec_bytes)
        return sum(t.numel() * t.element_size() for t in (self.label, self.dense, self.keys, self.nnz, self.weights)
                   if t is not None)


def power_law_keys(n: int, vocab: int, alpha: float, gen: torch.Generator, dtype=torch.int64):
    """Inverse-CDF power-law sampler of the reference DataGenerator
    (HugeCTR/include/data_generator.hpp:109-131): x in [1, vocab+1) with pdf ~ x^-alpha."""
    u = torch.rand(n, generator=gen, dtype=torch.float64)
    if vocab <= 1:
        return torch.zeros(n, dtype=dtype)
    if abs(alpha - 1.0) < 1e-9:
        x = torch.exp(u * torch.log(torch.tensor(float(vocab + 1), dtype=torch.float64)))
    else:
        a = 1.0 - alpha
        lo, hi = 1.0, float(vocab + 1) ** a
        x = ((hi - lo) * u + lo) ** (1.0 / a)
    k = torch.clamp(x.floor().long() - 1, 0, vocab - 1)
    return k.to(dtype)
