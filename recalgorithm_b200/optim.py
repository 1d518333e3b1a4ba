"""Adam on embedding tables with IndexedSlices gradients (SURVEY 8f.3) -- the step right after the hot path.

``TableAdam(tables, lr, lazy=False)`` reproduces ``tf.train.AdamOptimizer(lr, 0.9, 0.999, 1e-8)`` applied to a table
whose gradient is IndexedSlices (DeepFM/deepfm.py:246-250): duplicates summed first, m/v decayed and the variable
updated for EVERY row each step [TF-internal, SURVEY A.8].  ``lazy=True`` is DIEN's LazyAdamOptimizer
(DIEN/dien.py:328): only the referenced rows move.  De-duplication, row sums, updates and the dense sweep are kernels of
libctr_b200.so (ctr_adam_indexed_slices: claim / merge / update, no sort and no host round trip).

``Ftrl(var_list, learning_rate)`` is ``tf.train.FtrlOptimizer`` on dense gradients (the Wide & Deep wide part,
WideAndDeep/wide_and_deep.py:254-257): TF's dense ApplyFtrl on every element of every variable (``ctr_ftrl_apply``).
"""
from __future__ import annotations

import math

import torch

from . import _lib, autograd, ops


class TableAdam:
    """``fused_backward=True`` registers the optimizer on the tables: the backward of ``autograd.lookup_fm2`` then applies the
    row updates itself (``ctr_embed_fm2_bwd_adam``: no IndexedSlices values are written to or re-read from HBM) and ``step()``
    only completes the step (TF's dense decay of the untouched rows when ``lazy=False``).  One lookup backward per step."""

    def __init__(self, tables: "autograd.EmbeddingTables", lr: float, beta1: float = 0.9, beta2: float = 0.999,
                 eps: float = 1e-8, lazy: bool = False, fused_backward: bool = False):
        self.tables, self.lr, self.b1, self.b2, self.eps, self.lazy = tables, lr, beta1, beta2, eps, lazy
        self.fused_backward = fused_backward
        self._fused_applied = False
        self._dup = None
        if fused_backward:
            tables._fused_opt = self
        w = tables.weight
        # the two moments of a row live side by side ((V, 2, D): one DRAM page per row instead of two -- the random row
        # updates are bound by the row-activation rate, not the bus); self.m / self.v are views
        self.mv = torch.zeros((w.shape[0], 2, w.shape[1]), dtype=torch.float32, device=w.device)
        self.m, self.v = self.mv[:, 0, :], self.mv[:, 1, :]
        self._ss = 2 * w.shape[1]
        self.t = 0
        self._bitmap = None if lazy else torch.zeros(((tables.num_rows + 31) // 32,), dtype=torch.int32, device=w.device)
        self._slot = torch.full((tables.num_rows,), -1, dtype=torch.int32, device=w.device)   # -1 between steps
        self._n_unique = torch.zeros((1,), dtype=torch.int64, device=w.device)
        self._dup_list = None

    def apply_fused(self, tile, d_tile, d_fm2, ids) -> None:
        """Called by the lookup's backward (fused_backward=True): backward + row update in one pass."""
        if self._fused_applied:
            raise RuntimeError("TableAdam(fused_backward=True) supports one lookup backward per step(); use the unfused optimizer")
        tb = self.tables
        w = tb.weight
        B, F, D = tile.shape
        self.t += 1
        lr_t = self.lr * math.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
        self._n_unique.zero_()
        if self._bitmap is not None:
            self._bitmap.zero_()
        if self._dup is None or self._dup[0].shape != (B, F, D):
            self._dup = (torch.empty((B, F, D), dtype=torch.float32, device=w.device),
                         torch.empty((B * F + 1,), dtype=torch.int32, device=w.device))
        ops._chk(tile, torch.float32, "tile"); ops._chk(d_tile, torch.float32, "d_tile", (B, F, D)); ops._chk(ids, torch.int64, "ids", (B, F))
        if d_fm2 is not None:
            d_fm2 = d_fm2.reshape(B)
        ops._chk(d_fm2, torch.float32, "d_fm2", (B,))
        _lib.check(_lib.lib().ctr_embed_fm2_bwd_adam(ops._ptr(tile), ops._ptr(d_tile), ops._ptr(d_fm2), tb.field_row_offset.data_ptr(),
                                                     ops._ptr(ids), B, F, D, w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                                     self._ss, self._slot.data_ptr(), self._dup[0].data_ptr(), self._dup[1].data_ptr(), lr_t,
                                                     self.b1, self.b2, self.eps, ops._ptr(self._bitmap), self._n_unique.data_ptr(),
                                                     ops._stream()))
        self._fused_applied = True

    def step(self) -> None:
        """Consume tables.grad_slices (every backward since the last zero_grad) and apply one Adam step.  Nothing is read
        back to the host; `last_unique_rows()` fetches the number of distinct rows the step touched."""
        tb = self.tables
        w = tb.weight
        V, D = w.shape
        L = _lib.lib()
        if self.fused_backward:
            if not self._fused_applied:
                raise RuntimeError("TableAdam(fused_backward=True).step() without a lookup backward since the last step")
            lr_t = self.lr * math.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
            if not self.lazy:
                _lib.check(L.ctr_adam_dense_rest(w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self._ss, V, D, lr_t, self.b1,
                                                 self.b2, self.eps, ops._ptr(self._bitmap), ops._stream()))
            self._fused_applied = False
            tb.zero_grad()
            return
        self.t += 1
        lr_t = self.lr * math.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
        self._n_unique.zero_()
        if self._bitmap is not None:
            self._bitmap.zero_()
        if tb.grad_slices:
            if len(tb.grad_slices) == 1:
                ids, vals = tb.grad_slices[0].ids, tb.grad_slices[0].values
            else:                       # several backward passes: one IndexedSlices with all their entries (TF sums them too)
                ids = torch.cat([sl.ids for sl in tb.grad_slices]); vals = torch.cat([sl.values for sl in tb.grad_slices])
            ids, vals = ids.contiguous(), vals.contiguous()
            off = tb.grad_slices[0].field_row_offset
            B, F = ids.shape
            if self._dup_list is None or self._dup_list.numel() != B * F + 1:
                self._dup_list = torch.empty((B * F + 1,), dtype=torch.int32, device=w.device)
            _lib.check(L.ctr_adam_indexed_slices(w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self._ss, off.data_ptr(), F, D,
                                                 ids.data_ptr(), vals.data_ptr(), B, self._slot.data_ptr(),
                                                 self._dup_list.data_ptr(), lr_t, self.b1, self.b2, self.eps,
                                                 ops._ptr(self._bitmap), self._n_unique.data_ptr(), ops._stream()))
        if not self.lazy:
            _lib.check(L.ctr_adam_dense_rest(w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self._ss, V, D, lr_t, self.b1,
                                             self.b2, self.eps, ops._ptr(self._bitmap), ops._stream()))
        tb.zero_grad()

    def last_unique_rows(self) -> int:
        return int(self._n_unique.item())


class ShardedTableAdam:
    """The same optimizer on a row-sharded table (``sharded.ShardedEmbeddingTables``): every rank updates the rows it owns
    from the (row, gradient) entries the other ranks pushed into its receive queues.  ``step()`` first completes the
    exchange (``tables.finish_push()``: stream sync + barrier, and it RAISES if any rank's queue overflowed -- dropped
    entries would otherwise be silently lost gradients) and ends with a barrier so that the next forward pulls updated rows."""

    def __init__(self, tables, lr: float, beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8, lazy: bool = False):
        self.tables, self.lr, self.b1, self.b2, self.eps, self.lazy = tables, lr, beta1, beta2, eps, lazy
        w = tables.weight
        self.mv = torch.zeros((w.shape[0], 2, w.shape[1]), dtype=torch.float32, device=w.device)     # interleaved, see TableAdam
        self.m, self.v = self.mv[:, 0, :], self.mv[:, 1, :]
        self._ss = 2 * w.shape[1]
        self._dup_list = torch.empty((tables.G * tables.capacity + 1,), dtype=torch.int32, device=w.device)
        self.t = 0
        self._bitmap = None if lazy else torch.zeros(((tables.local_rows + 31) // 32,), dtype=torch.int32, device=w.device)
        self._slot = torch.full((tables.local_rows,), -1, dtype=torch.int32, device=w.device)
        self._n_unique = torch.zeros((1,), dtype=torch.int64, device=w.device)

    def step(self, barrier: bool = True, finish_push: bool = True) -> None:
        tb = self.tables
        if finish_push:
            tb.finish_push()
        w = tb.weight
        V, D = w.shape
        self.t += 1
        lr_t = self.lr * math.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
        L = _lib.lib()
        self._n_unique.zero_()
        if self._bitmap is not None:
            self._bitmap.zero_()
        _lib.check(L.ctr_adam_rows_dedup(w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self._ss, V, D, tb.recv_rows.data_ptr(),
                                         tb.recv_vals.data_ptr(), tb.recv_counts.data_ptr(), tb.G, tb.capacity,
                                         self._slot.data_ptr(), self._dup_list.data_ptr(), lr_t, self.b1, self.b2, self.eps,
                                         ops._ptr(self._bitmap), self._n_unique.data_ptr(), ops._stream()))
        if not self.lazy:
            _lib.check(L.ctr_adam_dense_rest(w.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self._ss, V, D, lr_t, self.b1,
                                             self.b2, self.eps, ops._ptr(self._bitmap), ops._stream()))
        if barrier:
            torch.cuda.current_stream().synchronize()
            tb.dist.barrier(group=tb.group)

    def last_unique_rows(self) -> int:
        return int(self._n_unique.item())


class Ftrl:
    """``tf.train.FtrlOptimizer(learning_rate, learning_rate_power, initial_accumulator_value, l1_regularization_strength,
    l2_regularization_strength)`` applied to variables whose ``.grad`` is dense (SURVEY A.12): slots ``accum`` (starts at
    initial_accumulator_value) and ``linear`` (starts at 0) per variable, one ``ctr_ftrl_apply`` per variable and step.
    l2_shrinkage_regularization_strength (TF's ApplyFtrlV2) is not implemented."""

    def __init__(self, var_list, learning_rate: float, learning_rate_power: float = -0.5, initial_accumulator_value: float = 0.1,
                 l1_regularization_strength: float = 0.0, l2_regularization_strength: float = 0.0,
                 l2_shrinkage_regularization_strength: float = 0.0):
        if initial_accumulator_value < 0.0:
            raise ValueError(f"initial_accumulator_value {initial_accumulator_value} needs to be positive or zero")
        if learning_rate_power > 0.0:
            raise ValueError(f"learning_rate_power {learning_rate_power} needs to be negative or zero")
        if l1_regularization_strength < 0.0:
            raise ValueError(f"l1_regularization_strength {l1_regularization_strength} needs to be positive or zero")
        if l2_regularization_strength < 0.0:
            raise ValueError(f"l2_regularization_strength {l2_regularization_strength} needs to be positive or zero")
        if l2_shrinkage_regularization_strength != 0.0:
            raise ValueError("l2_shrinkage_regularization_strength is not implemented (only TF's ApplyFtrl, shrinkage 0)")
        self.var_list = list(var_list)
        self.lr, self.lr_power = float(learning_rate), float(learning_rate_power)
        self.l1, self.l2 = float(l1_regularization_strength), float(l2_regularization_strength)
        self._slots = {id(v): {"accum": torch.full_like(v.data, float(initial_accumulator_value)), "linear": torch.zeros_like(v.data)}
                       for v in self.var_list}

    def get_slot(self, var, name: str) -> torch.Tensor:
        return self._slots[id(var)][name]

    def step(self) -> None:
        """One FTRL step on every variable that has a gradient; raises if none has (as minimize does)."""
        have = [v for v in self.var_list if v.grad is not None]
        if not have:
            raise ValueError(f"No gradients provided for any variable: {[tuple(v.shape) for v in self.var_list]}")
        for v in have:
            sl = self._slots[id(v)]
            ops.ftrl_apply(v.data, sl["accum"], sl["linear"], v.grad.contiguous(), self.lr, self.lr_power, self.l1, self.l2)

    def zero_grad(self) -> None:
        for v in self.var_list:
            v.grad = None
