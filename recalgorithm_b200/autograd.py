"""torch.autograd glue: each Function is one forward and one backward call into the C ABI.

The gradient of an embedding table is NOT a dense tensor: like TensorFlow's gather gradient
(``IndexedSlices``; the reference's optimizer consumes exactly that -- DeepFM/deepfm.py:246-250,
SURVEY A.8) it is the pair (ids, row values), attached to the table variable as ``grad_slices``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from . import ops


@dataclass
class IndexedSlices:
    """values[b, f, :] is the gradient of row field_row_offset[f] + ids[b, f] (ids < 0 / out of range: dropped)."""
    values: torch.Tensor            # (B, F, D)
    ids: torch.Tensor               # (B, F) int64, per-field local ids
    field_row_offset: torch.Tensor  # (F+1,) int64

    def to_dense(self, num_rows: int) -> torch.Tensor:
        dense = torch.zeros((num_rows, self.values.shape[-1]), dtype=self.values.dtype, device=self.values.device)
        return ops.embed_scatter_add(dense, self.field_row_offset, self.ids, self.values)


class EmbeddingTables:
    """F per-field embedding tables stored back to back in one (V_total, D) buffer.

    Mirrors the variables ``fc.embedding_column`` creates implicitly (one ``embedding_weights`` per
    column; DeepFM/deepfm.py:83-89) but keeps them contiguous so one kernel serves all fields.
    """

    def __init__(self, rows_per_field, dim: int, device="cuda", init: Optional[str] = "truncated_normal",
                 generator: Optional[torch.Generator] = None):
        rows = torch.as_tensor(rows_per_field, dtype=torch.int64)
        self.num_fields = int(rows.numel())
        self.dim = int(dim)
        off = torch.zeros(self.num_fields + 1, dtype=torch.int64)
        off[1:] = torch.cumsum(rows, 0)
        self.num_rows = int(off[-1])
        self.field_row_offset = off.to(device)
        self.weight = torch.empty((self.num_rows, self.dim), dtype=torch.float32, device=device)
        if init == "truncated_normal":          # embedding_column default: truncated_normal(0, 1/sqrt(D))  [SURVEY A.5 / note 4]
            torch.nn.init.trunc_normal_(self.weight, mean=0.0, std=self.dim ** -0.5, a=-2 * self.dim ** -0.5,
                                        b=2 * self.dim ** -0.5, generator=generator)
        self.grad_slices: List[IndexedSlices] = []
        self._anchor = torch.zeros((), device=device, requires_grad=True)   # lets autograd reach backward()

    def zero_grad(self):
        self.grad_slices.clear()


def _ids64_for(ids: torch.Tensor):
    """IndexedSlices carry int64 ids (TF's sparse ids); int32 inputs are widened by the forward kernel itself."""
    return torch.empty(ids.shape, dtype=torch.int64, device=ids.device) if ids.dtype == torch.int32 else None


class _LookupFM2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, tables: EmbeddingTables, ids: torch.Tensor, want_fm2: bool):
        ctx.set_materialize_grads(False)            # an unused output arrives as None in backward, not as a zero-filled (B,F,D)
        ids64 = _ids64_for(ids)
        tile, fm2 = ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids, want_tile=True, want_fm2=want_fm2,
                                      ids64_out=ids64)
        ctx.tables, ctx.ids, ctx.want_fm2 = tables, (ids if ids64 is None else ids64), want_fm2
        ctx.save_for_backward(tile)
        if want_fm2:
            return tile, fm2
        return tile

    @staticmethod
    def backward(ctx, d_tile, d_fm2=None):
        (tile,) = ctx.saved_tensors
        if d_tile is None and d_fm2 is None:        # nothing upstream depends on the lookup: no IndexedSlices
            return None, None, None, None
        if d_tile is not None:
            d_tile = d_tile.contiguous()
        if d_fm2 is not None:
            d_fm2 = d_fm2.contiguous()
        fused = getattr(ctx.tables, "_fused_opt", None)
        if fused is not None:                       # optim.TableAdam(fused_backward=True): the row update happens right here
            fused.apply_fused(tile, d_tile, d_fm2 if ctx.want_fm2 else None, ctx.ids)
            return None, None, None, None
        if not ctx.want_fm2 and d_tile is not None:
            values = d_tile                                      # plain gather: the IndexedSlices values ARE the upstream gradient
        else:
            values = ops.embed_fm2_bwd(tile, d_tile, d_fm2 if ctx.want_fm2 else None)
        ctx.tables.grad_slices.append(IndexedSlices(values, ctx.ids, ctx.tables.field_row_offset))
        return None, None, None, None


def lookup_fm2(tables: EmbeddingTables, ids: torch.Tensor):
    """(B,F) ids -> (tile (B,F,D), fm2 logit (B,1)); differentiable w.r.t. the tables (IndexedSlices)."""
    return _LookupFM2.apply(tables._anchor, tables, ids, True)


def lookup(tables: EmbeddingTables, ids: torch.Tensor):
    """(B,F) ids -> tile (B,F,D)."""
    return _LookupFM2.apply(tables._anchor, tables, ids, False)


class _LookupFM2Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, wlin, tables: EmbeddingTables, ids: torch.Tensor):
        ctx.set_materialize_grads(False)
        ids64 = _ids64_for(ids)
        wl = wlin.contiguous()
        tile, fm2, lin = ops.embed_fm2_lin_fwd(tables.weight, tables.field_row_offset, ids, wl, ids64_out=ids64)
        ctx.tables, ctx.ids = tables, (ids if ids64 is None else ids64)
        ctx.save_for_backward(tile, wl)
        return fm2, lin

    @staticmethod
    def backward(ctx, d_fm2, d_lin):
        tile, wl = ctx.saved_tensors
        values, d_wlin = ops.embed_fm2_lin_bwd(tile, wl, None if d_fm2 is None else d_fm2.contiguous(),
                                               None if d_lin is None else d_lin.contiguous())
        ctx.tables.grad_slices.append(IndexedSlices(values, ctx.ids, ctx.tables.field_row_offset))
        return d_wlin.reshape(wl.shape), None, None


def lookup_fm2_linear(tables: EmbeddingTables, ids: torch.Tensor, wlin: torch.Tensor):
    """(B,F) ids -> (fm2 logit (B,1), lin (B,1) = input_layer output (B, F*D) @ wlin): the lookup, DeepFM's second-order
    term and a dense(1, use_bias=False) consumer of the concatenated embeddings in one kernel each way -- the tile is
    written once (for the backward) and never re-streamed by the consumer.  wlin: (F*D, 1) or (F*D,), requires_grad."""
    return _LookupFM2Linear.apply(wlin, tables, ids)


class _SigmoidCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logit_a, logit_b, labels):
        loss, d = ops.sigmoid_ce(logit_a.contiguous(), None if logit_b is None else logit_b.contiguous(), labels.contiguous())
        ctx.save_for_backward(d)
        ctx.shapes = (logit_a.shape, None if logit_b is None else logit_b.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        (d,) = ctx.saved_tensors
        gd = d * g                                              # g is the scalar upstream gradient (1 for loss.backward())
        return gd.reshape(ctx.shapes[0]), (None if ctx.shapes[1] is None else gd.reshape(ctx.shapes[1])), None


def sigmoid_cross_entropy_mean(logit_a: torch.Tensor, labels: torch.Tensor, logit_b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """reduce_mean(sigmoid_cross_entropy_with_logits(labels, logit_a [+ logit_b])) (DeepFM/deepfm.py:214,235) with its gradient
    computed by the same launch; returns the scalar loss."""
    return _SigmoidCE.apply(logit_a, logit_b, labels)


class _CrossStack(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, xl, w, b):
        x0c = x0.contiguous()
        xlc = None if xl is None else xl.contiguous()
        wc, bc = w.contiguous(), b.contiguous()
        ctx.save_for_backward(x0c, wc, bc, *([] if xlc is None else [xlc]))
        ctx.has_xl = xlc is not None
        return ops.cross_fwd(x0c, wc, bc, xl_in=xlc)

    @staticmethod
    def backward(ctx, g):
        saved = ctx.saved_tensors
        x0, w, b = saved[:3]
        xl = saved[3] if ctx.has_xl else None
        dx0, dxl, dw, db = ops.cross_bwd(x0, w, b, g.contiguous(), xl_in=xl)
        return dx0, dxl, dw, db


def cross_stack(x0: torch.Tensor, w: torch.Tensor, b: torch.Tensor, xl: Optional[torch.Tensor] = None) -> torch.Tensor:
    """All L cross layers (DCN/dcn.py:157-160) in one launch.  w, b: (L, d)."""
    return _CrossStack.apply(x0, xl, w, b)


class _LookupCross(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, tables: EmbeddingTables, ids, w, b):
        ctx.set_materialize_grads(False)            # `g_x0` is None when only the cross output is consumed (and vice versa)
        wc, bc = w.contiguous(), b.contiguous()
        x0, out = ops.embed_cross_fwd(tables.weight, tables.field_row_offset, ids, wc, bc)
        ctx.tables, ctx.ids = tables, (ids if ids.dtype == torch.int64 else ids.long())
        ctx.save_for_backward(x0, wc, bc)
        return out, x0

    @staticmethod
    def backward(ctx, g, g_x0=None):
        x0, w, b = ctx.saved_tensors
        dw = db = None
        if g is not None:
            dx0, _, dw, db = ops.cross_bwd(x0, w, b, g.contiguous())
            if g_x0 is not None:                     # x0 also feeds the deep tower (DCN/dcn.py:163): both gradients reach the tables
                dx0 = dx0 + g_x0
        else:
            dx0 = g_x0.contiguous()
        B, F = ctx.ids.shape
        # the lookup backward of a plain gather: the IndexedSlices values ARE dx0 viewed (B,F,D)
        ctx.tables.grad_slices.append(IndexedSlices(dx0.view(B, F, -1), ctx.ids, ctx.tables.field_row_offset))
        return None, None, None, dw, db


def lookup_cross(tables: EmbeddingTables, ids: torch.Tensor, w: torch.Tensor, b: torch.Tensor):
    """`net = input_layer(...)` + the cross loop (DCN/dcn.py:153-160) in one launch: (B,F) ids -> (x_L (B,F*D), x0 (B,F*D)).
    x0 (the gathered input) is returned for the deep tower (`dcn.py:163`); gradients w.r.t. both outputs reach the tables."""
    return _LookupCross.apply(tables._anchor, tables, ids, w, b)


class _CIN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, xk, filt, want_pooled):
        x0c, xkc, fc_ = x0.contiguous(), xk.contiguous(), filt.contiguous()
        ctx.save_for_backward(x0c, xkc, fc_)
        ctx.want_pooled = want_pooled
        if want_pooled:
            out, pooled = ops.cin_fwd(x0c, xkc, fc_, want_pooled=True)
            return out, pooled
        return ops.cin_fwd(x0c, xkc, fc_)

    @staticmethod
    def backward(ctx, g_out, g_pooled=None):
        x0, xk, filt = ctx.saved_tensors
        if g_out is None:
            g_out = torch.zeros((x0.shape[0], filt.shape[1], x0.shape[2]), dtype=x0.dtype, device=x0.device)
        if g_pooled is not None:
            g_out = g_out + g_pooled.unsqueeze(-1)          # pooled = sum_d out
        dx0, dxk, dw = ops.cin_bwd(x0, xk, filt, g_out.contiguous())
        return dx0, dxk, dw, None


def cin(x0, xk, filt, want_pooled=False):
    """One CIN layer on the tensor cores: (B,m,D),(B,hk,D),(hk*m,H) -> (B,H,D) [, sum over D (B,H)]."""
    return _CIN.apply(x0, xk, filt, want_pooled)


class _DinAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, query, keys, keys_length, is_softmax, w1, b1, w2, b2, w3, b3):
        args = [t.contiguous() for t in (query, keys)] + [keys_length.contiguous()] + \
               [t.contiguous() for t in (w1, b1, w2, b2, w3, b3)]
        ctx.is_softmax = bool(is_softmax)
        out, att = ops.din_attention_fwd(*args, is_softmax=ctx.is_softmax, want_weights=True)
        ctx.save_for_backward(*args, att)
        return out

    @staticmethod
    def backward(ctx, g):
        *args, att = ctx.saved_tensors
        dq, dk, dws = ops.din_attention_bwd(*args, g.contiguous(), is_softmax=ctx.is_softmax, att_w=att)
        return (dq, dk, None, None, *dws)


def din_attention(query, keys, keys_length, w1, b1, w2, b2, w3, b3, is_softmax=False):
    return _DinAttention.apply(query, keys, keys_length, is_softmax, w1, b1, w2, b2, w3, b3)


class _Senet(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, w2):
        xc, w1c, w2c = x.contiguous(), w1.contiguous(), w2.contiguous()
        ctx.save_for_backward(xc, w1c, w2c)
        return ops.senet_fwd(xc, w1c, w2c)

    @staticmethod
    def backward(ctx, g):
        return ops.senet_bwd(*ctx.saved_tensors, g.contiguous())


def senet(x, w1, w2):
    return _Senet.apply(x, w1, w2)


class _Bilinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, type_):
        xc, wc = x.contiguous(), w.contiguous()
        ctx.save_for_backward(xc, wc)
        ctx.type_ = type_
        return ops.bilinear_fwd(xc, wc, type_)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        dx, dw = ops.bilinear_bwd(x, w, ctx.type_, g.contiguous())
        return dx, dw, None


def bilinear(x, w, type_):
    return _Bilinear.apply(x, w, type_)


# ------------------------------------------------------------------------------------ SURVEY 8f.4: FM2 siblings
class _LookupBI(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, tables: EmbeddingTables, ids: torch.Tensor):
        ctx.set_materialize_grads(False)
        tile, bi = ops.embed_bi_fwd(tables.weight, tables.field_row_offset, ids)
        ctx.tables, ctx.ids = tables, ids
        ctx.save_for_backward(tile)
        return tile, bi

    @staticmethod
    def backward(ctx, d_tile, d_bi):
        (tile,) = ctx.saved_tensors
        d_tile = d_tile.contiguous() if d_tile is not None else None
        d_bi = d_bi.contiguous() if d_bi is not None else torch.zeros((tile.shape[0], tile.shape[2]), device=tile.device)
        values = ops.embed_bi_bwd(tile, d_tile, d_bi)
        ctx.tables.grad_slices.append(IndexedSlices(values, ctx.ids, ctx.tables.field_row_offset))
        return None, None, None


def lookup_bi(tables: EmbeddingTables, ids: torch.Tensor):
    """(B,F) ids -> (tile (B,F,D), NFM bi-interaction vector (B,D)); differentiable w.r.t. the tables (IndexedSlices)."""
    return _LookupBI.apply(tables._anchor, tables, ids)


class _LookupFwBI(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, kernel_mf, kernel_fm, bias_mf, bias_fm, tables: EmbeddingTables, ids: torch.Tensor, field_group):
        ctx.set_materialize_grads(False)            # an unused tile gradient arrives as None and goes down as NULL d_tile
        ids64 = _ids64_for(ids)
        kernel_mf, kernel_fm, bias_mf, bias_fm = (t.contiguous() for t in (kernel_mf, kernel_fm, bias_mf, bias_fm))
        tile, h = ops.embed_fwbi_fwd(tables.weight, tables.field_row_offset, ids, field_group, kernel_mf, kernel_fm, bias_mf,
                                     bias_fm, ids64_out=ids64)
        ctx.tables, ctx.ids, ctx.field_group = tables, (ids if ids64 is None else ids64), field_group
        ctx.save_for_backward(tile, kernel_mf, kernel_fm)
        return tile, h

    @staticmethod
    def backward(ctx, d_tile, d_h):
        tile, kernel_mf, kernel_fm = ctx.saved_tensors
        if d_tile is None and d_h is None:
            return (None,) * 8
        d_tile = d_tile.contiguous() if d_tile is not None else None
        d_h = d_h.contiguous() if d_h is not None else torch.zeros((tile.shape[0], tile.shape[2]), device=tile.device)
        values, *dw = ops.fwbi_bwd(tile, d_tile, d_h, ctx.field_group, kernel_mf, kernel_fm)
        ctx.tables.grad_slices.append(IndexedSlices(values, ctx.ids, ctx.tables.field_row_offset))
        return (None, *dw, None, None, None)


def lookup_fwbi(tables: EmbeddingTables, ids: torch.Tensor, field_group, kernel_mf: torch.Tensor, kernel_fm: torch.Tensor,
                bias_mf: torch.Tensor, bias_fm: torch.Tensor):
    """(B,F) ids -> (tile (B,F,D), FLEN field-wise bi-interaction h (B,D)); field_group: F group indices in [0, M),
    M = len(kernel_fm).  Differentiable w.r.t. the tables (IndexedSlices) and the four weights."""
    return _LookupFwBI.apply(tables._anchor, kernel_mf, kernel_fm, bias_mf, bias_fm, tables, ids, tuple(field_group))


class _FwBI(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tile, kernel_mf, kernel_fm, bias_mf, bias_fm, field_group):
        tile, kernel_mf, kernel_fm, bias_mf, bias_fm = (t.contiguous() for t in (tile, kernel_mf, kernel_fm, bias_mf, bias_fm))
        ctx.save_for_backward(tile, kernel_mf, kernel_fm)
        ctx.field_group = field_group
        return ops.fwbi_fwd(tile, field_group, kernel_mf, kernel_fm, bias_mf, bias_fm)

    @staticmethod
    def backward(ctx, g):
        tile, kernel_mf, kernel_fm = ctx.saved_tensors
        return (*ops.fwbi_bwd(tile, None, g.contiguous(), ctx.field_group, kernel_mf, kernel_fm), None)


def fwbi(tile: torch.Tensor, field_group, kernel_mf: torch.Tensor, kernel_fm: torch.Tensor, bias_mf: torch.Tensor,
         bias_fm: torch.Tensor) -> torch.Tensor:
    """FLEN field-wise bi-interaction of a (B,F,D) tile -> h (B,D) (see lookup_fwbi)."""
    return _FwBI.apply(tile, kernel_mf, kernel_fm, bias_mf, bias_fm, tuple(field_group))


class _FwFM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tile, r):
        tile, r = tile.contiguous(), r.contiguous()
        ctx.save_for_backward(tile, r)
        return ops.fwfm_fwd(tile, r)

    @staticmethod
    def backward(ctx, g):
        tile, r = ctx.saved_tensors
        return ops.fwfm_bwd(tile, r, g.contiguous())


def fwfm(tile: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    return _FwFM.apply(tile, r)


class _AFM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tile, w, b, h):
        tile, w, b, h = tile.contiguous(), w.contiguous(), b.contiguous(), h.contiguous()
        ctx.save_for_backward(tile, w, b, h)
        return ops.afm_fwd(tile, w, b, h)

    @staticmethod
    def backward(ctx, g):
        tile, w, b, h = ctx.saved_tensors
        return ops.afm_bwd(tile, w, b, h, g.contiguous())


def afm(tile: torch.Tensor, w: torch.Tensor, b: torch.Tensor, h: torch.Tensor) -> torch.Tensor:
    return _AFM.apply(tile, w, b, h)


class _BstTransformer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, queries, keys, values, keys_length, heads, max_length, use_pos, *params):
        d = queries.shape[-1]
        packed = ops.bst_pack_params(dict(zip(ops.BST_PARAM_ORDER, params)), d, heads, max_length)
        queries, keys, values = queries.contiguous(), keys.contiguous(), values.contiguous()
        ctx.save_for_backward(queries, keys, values, keys_length, packed)
        ctx.cfg = (heads, max_length, use_pos, d)
        return ops.bst_transformer_fwd(queries, keys, values, keys_length, packed, heads, max_length, use_pos)

    @staticmethod
    def backward(ctx, g):
        queries, keys, values, keys_length, packed = ctx.saved_tensors
        heads, max_length, use_pos, d = ctx.cfg
        dq, dk, dv, dp = ops.bst_transformer_bwd(queries, keys, values, keys_length, packed, g.contiguous(), heads, max_length, use_pos)
        grads = ops.bst_unpack_params(dp, d, heads, max_length)
        return (dq, dk, dv, None, None, None, None) + tuple(grads[n] for n in ops.BST_PARAM_ORDER)


def bst_transformer(queries, keys, values, keys_length, params: dict, heads: int, max_length: int, use_position_embedding=True):
    """params: dict with the names of ops.BST_PARAM_ORDER."""
    return _BstTransformer.apply(queries, keys, values, keys_length, heads, max_length, use_position_embedding,
                                 *[params[n] for n in ops.BST_PARAM_ORDER])


class _FFM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tile):
        tile = tile.contiguous()
        ctx.save_for_backward(tile)
        return ops.ffm_fwd(tile)

    @staticmethod
    def backward(ctx, g):
        (tile,) = ctx.saved_tensors
        return ops.ffm_bwd(tile, g.contiguous())


def ffm(tile: torch.Tensor) -> torch.Tensor:
    """(B, F, F-1, K) field/slot tile -> FFM second-order logit (B,1)."""
    return _FFM.apply(tile)


class _PNN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e, wlin, wprod, bias, method):
        e, wlin, wprod, bias = e.contiguous(), wlin.contiguous(), wprod.contiguous(), bias.contiguous()
        out = ops.pnn_fwd(e, wlin, wprod, bias, method)
        ctx.save_for_backward(e, wlin, wprod, out)           # out carries the relu mask of the backward
        ctx.method = method
        return out

    @staticmethod
    def backward(ctx, g):
        e, wlin, wprod, out = ctx.saved_tensors
        d_e, d_wlin, d_wprod, d_bias = ops.pnn_bwd(e, wlin, wprod, out, g.contiguous(), ctx.method)
        return d_e, d_wlin, d_wprod, d_bias, None


def pnn(e: torch.Tensor, wlin: torch.Tensor, wprod: torch.Tensor, bias: torch.Tensor, method: int) -> torch.Tensor:
    """PNN product layer: (B,F,K) field embeddings -> relu(lz + lp + bias) (B,N); method 0 = IPNN, 1 = OPNN."""
    return _PNN.apply(e, wlin, wprod, bias, method)


class _DIEN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seq, seq_len, target, nh, cell, *params):
        na = seq.shape[-1]
        packed = ops.dien_pack_params(params, na, nh)
        seq, target = seq.contiguous(), target.contiguous()
        final, scores, ws = ops.dien_fwd(seq, seq_len, target, packed, nh, cell)
        ctx.save_for_backward(seq, seq_len, target, packed, ws)     # ws: the forward's states and attention weights
        ctx.cfg = (nh, cell)
        ctx.mark_non_differentiable(scores)
        return final, scores

    @staticmethod
    def backward(ctx, g, _g_scores):
        seq, seq_len, target, packed, ws = ctx.saved_tensors
        nh, cell = ctx.cfg
        d_seq, d_tgt, d_p = ops.dien_bwd(seq, seq_len, target, packed, g.contiguous(), nh, cell, ws)
        return (d_seq, None, d_tgt, None, None) + tuple(ops.dien_unpack_params(d_p, seq.shape[-1], nh))


def dien(seq, seq_len, target, params, nh: int, cell: int):
    """DIEN seq_encoder (DIEN/dien.py:198-229): (final_state (B,nh), attention scores (B,T), forward only); params in
    ops.DIEN_PARAM_ORDER; cell 0 = AGRU, 1 = AUGRU."""
    return _DIEN.apply(seq, seq_len, target, nh, cell, *params)


class _DIENAux(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seq, seq_len, target, neg_seq, w_aux, nh, cell, T_neg, *params):
        na = seq.shape[-1]
        packed = ops.dien_pack_params(params, na, nh)
        seq, target, neg_seq, w_aux = seq.contiguous(), target.contiguous(), neg_seq.contiguous(), w_aux.contiguous()
        final, scores, aux, ws = ops.dien_fwd_aux(seq, seq_len, target, neg_seq, packed, w_aux, nh, cell, T_neg)
        ctx.save_for_backward(seq, seq_len, target, neg_seq, packed, w_aux, ws)
        ctx.cfg = (nh, cell, T_neg)
        ctx.mark_non_differentiable(scores)
        ctx.set_materialize_grads(False)            # an unused output's gradient arrives as None and goes down as zeros
        return final, scores, aux

    @staticmethod
    def backward(ctx, g_final, _g_scores, g_aux):
        seq, seq_len, target, neg_seq, packed, w_aux, ws = ctx.saved_tensors
        nh, cell, T_neg = ctx.cfg
        g_final = torch.zeros((seq.shape[0], nh), dtype=seq.dtype, device=seq.device) if g_final is None else g_final.contiguous()
        g_aux = torch.zeros((), dtype=seq.dtype, device=seq.device) if g_aux is None else g_aux.reshape(()).contiguous()
        d_seq, d_neg, d_tgt, d_p, d_w = ops.dien_bwd_aux(seq, seq_len, target, neg_seq, packed, w_aux, g_final, g_aux, nh, cell,
                                                         T_neg, ws)
        return (d_seq, None, d_tgt, d_neg, d_w, None, None, None) + tuple(ops.dien_unpack_params(d_p, seq.shape[-1], nh))


def dien_aux(seq, seq_len, target, neg_seq, w_aux, params, nh: int, cell: int, T_neg: int):
    """DIEN seq_encoder plus the auxiliary loss (DIEN/dien.py:198-229, 256-300, the paper's sign): (final_state (B,nh),
    attention scores (B,T), forward only, aux_loss ()); one backward serves both differentiable outputs."""
    return _DIENAux.apply(seq, seq_len, target, neg_seq, w_aux, nh, cell, T_neg, *params)


class _ResidualUnit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w0, b0, w1, b1):
        x, w0, b0, w1, b1 = (t.contiguous() for t in (x, w0, b0, w1, b1))
        out = ops.residual_unit_fwd(x, w0, b0, w1, b1)
        ctx.save_for_backward(x, w0, b0, w1, b1, out)        # out carries the outer relu mask; h is recomputed from x
        return out

    @staticmethod
    def backward(ctx, g):
        return ops.residual_unit_bwd(*ctx.saved_tensors, g.contiguous())


def residual_unit(x: torch.Tensor, w0: torch.Tensor, b0: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor) -> torch.Tensor:
    """DeepCrossing residual unit: relu(x + relu(x . w0 + b0) . w1 + b1), (B,d) -> (B,d)."""
    return _ResidualUnit.apply(x, w0, b0, w1, b1)


class _AutoInt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w_query, w_key, w_value, w_res, heads, dk):
        x, w_query, w_key, w_value, w_res = (t.contiguous() for t in (x, w_query, w_key, w_value, w_res))
        out = ops.autoint_fwd(x, w_query, w_key, w_value, w_res, heads, dk)
        ctx.save_for_backward(x, w_query, w_key, w_value, w_res, out)   # Q, K, V and the attention are recomputed
        ctx.cfg = (heads, dk)
        return out

    @staticmethod
    def backward(ctx, g):
        return ops.autoint_bwd(*ctx.saved_tensors, g.contiguous(), *ctx.cfg) + (None, None)


def autoint_interacting(x: torch.Tensor, w_query: torch.Tensor, w_key: torch.Tensor, w_value: torch.Tensor,
                        w_res: torch.Tensor, heads: int, dk: int) -> torch.Tensor:
    """AutoInt interacting layer: relu(concat_h softmax(Q_h K_h^T) V_h + x . w_res), (B,F,d) -> (B,F,heads*dk)."""
    return _AutoInt.apply(x, w_query, w_key, w_value, w_res, int(heads), int(dk))


class _MMoE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w_experts, b_experts, w_gates):
        x, w_experts, b_experts, w_gates = (t.contiguous() for t in (x, w_experts, b_experts, w_gates))
        towers, gates = ops.mmoe_fwd(x, w_experts, b_experts, w_gates)
        ctx.save_for_backward(x, w_experts, b_experts, w_gates, gates)   # the expert outputs are recomputed from x
        ctx.mark_non_differentiable(gates)
        return towers, gates

    @staticmethod
    def backward(ctx, g_towers, _g_gates):
        return ops.mmoe_bwd(*ctx.saved_tensors, g_towers.contiguous())


def mmoe(x: torch.Tensor, w_experts: torch.Tensor, b_experts: torch.Tensor, w_gates: torch.Tensor):
    """MMoE expert-gate layer: (towers (T,B,H), gates (T,B,E), forward only) from x (B,d), w_experts (E,d,H), b_experts (E,H)
    and w_gates (T,d,E)."""
    return _MMoE.apply(x, w_experts, b_experts, w_gates)


class _PLE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction):
        x, w_experts, b_experts, w_gates = (t.contiguous() for t in (x, w_experts, b_experts, w_gates))
        out, gates = ops.ple_fwd(x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction)
        ctx.save_for_backward(x, w_experts, b_experts, w_gates, gates)   # the expert outputs are recomputed from x
        ctx.counts = (experts_per_task, num_experts_in_shared, extraction)
        ctx.mark_non_differentiable(gates)
        return out, gates

    @staticmethod
    def backward(ctx, g_out, _g_gates):
        return (*ops.ple_bwd(*ctx.saved_tensors, g_out.contiguous(), *ctx.counts), None, None, None)


def ple(x: torch.Tensor, w_experts: torch.Tensor, b_experts: torch.Tensor, w_gates: torch.Tensor, experts_per_task,
        num_experts_in_shared: int, extraction: bool):
    """PLE expert-gate block: (out, gates (B,GC), forward only) from x (B,d), w_experts (E,d,H), b_experts (E,H) and
    w_gates (d,GC); out is (B,H) for the extraction network and (T,B,H) for the final layer (see ops.ple_fwd)."""
    return _PLE.apply(x, w_experts, b_experts, w_gates, tuple(int(v) for v in experts_per_task), int(num_experts_in_shared),
                      bool(extraction))
