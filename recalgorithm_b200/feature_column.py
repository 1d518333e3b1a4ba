"""Host-side mirror of the ``tf.feature_column`` calls the reference makes around the lookup (row L of SURVEY.md 8a/8b).

Same names and argument meaning as the reference's ``create_feature_columns()`` / ``model_fn`` code
(DeepFM/deepfm.py:44-99,180-190; DCN/dcn.py:84-107,149-153; DIN/din.py:92-114,201-214):

    userid   = fc.categorical_column_with_vocabulary_file('userid', '.../userid.txt')
    userid_e = fc.embedding_column(userid, 16)
    shared   = fc.shared_embedding_columns([feedid, his_seq], 16, combiner='mean')
    x        = fc.input_layer(features, [userid_e, ...])            # (B, sum d), columns sorted by NAME
    seq, n   = fc.sequence_input_layer(features, [shared[1]])       # (B, T, D), (B,)
    cross    = fc.indicator_column(fc.crossed_column([userid, manual_tag_list], hash_bucket_size=100000))
    wide     = fc.indicator_dense(features, [cross], units=1, name="wide_part_variables")   # (B, 1)

``features`` is what ``io.parse_example`` returns (ragged byte strings per key, dense floats for numeric keys).
String -> id mapping runs on the host (vocabulary dict); everything after it is one kernel call per column
(``ctr_bag_lookup_fwd``, mean combiner, empty bag -> zeros) writing straight into its slice of the (B, sum d) row.
Semantics that live inside TensorFlow, not in the reference tree, follow SURVEY Appendix A.3-A.6 and stay
"parity unpinned" (DESIGN.md section 2).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import layers, ops
from .io import FixedLenFeature, VarLenFeature, VocabularyFile


# ------------------------------------------------------------------ column types
@dataclass(eq=False)
class CategoricalColumn:
    key: str
    vocabulary: VocabularyFile
    is_sequence: bool = False

    @property
    def name(self):
        return self.key

    @property
    def num_buckets(self):
        return len(self.vocabulary)


@dataclass(eq=False)
class NumericColumn:
    key: str
    shape: Tuple[int, ...] = (1,)
    default_value: float = 0.0

    @property
    def name(self):
        return self.key


@dataclass(eq=False)
class EmbeddingColumn:
    categorical_column: CategoricalColumn
    dimension: int
    combiner: str = "mean"
    shared_name: Optional[str] = None           # set by shared_embedding_columns

    @property
    def name(self):
        return f"{self.categorical_column.key}_shared_embedding" if self.shared_name else f"{self.categorical_column.key}_embedding"

    @property
    def variable_name(self):
        # <scope>/input_layer/<key>_embedding/embedding_weights ; shared: .../<sorted keys joined by _>_shared_embedding
        return (f"input_layer/{self.shared_name}/embedding_weights" if self.shared_name
                else f"input_layer/{self.categorical_column.key}_embedding/embedding_weights")


@dataclass(eq=False)
class CrossedColumn:
    """tf.feature_column.crossed_column over categorical columns: hashes the keys' vocabulary ids (SURVEY A.11)."""
    keys: Tuple[CategoricalColumn, ...]
    hash_bucket_size: int
    hash_key: int = ops.CROSS_HASH_KEY

    @property
    def name(self):
        return "_X_".join(sorted(k.key for k in self.keys))

    @property
    def num_buckets(self):
        return self.hash_bucket_size


@dataclass(eq=False)
class IndicatorColumn:
    categorical_column: object                  # CategoricalColumn | CrossedColumn

    @property
    def name(self):
        return f"{self.categorical_column.name}_indicator"


def categorical_column_with_vocabulary_file(key, vocabulary_file, vocabulary_size=None, num_oov_buckets=0, default_value=None):
    if num_oov_buckets or default_value is not None or vocabulary_size is not None:
        raise ValueError("only the reference's usage is supported: vocabulary_size=None, num_oov_buckets=0, default_value=None")
    vocab = vocabulary_file if isinstance(vocabulary_file, VocabularyFile) else VocabularyFile(vocabulary_file)
    return CategoricalColumn(key, vocab)


def sequence_categorical_column_with_vocabulary_file(key, vocabulary_file, **kw):
    col = categorical_column_with_vocabulary_file(key, vocabulary_file, **kw)
    col.is_sequence = True
    return col


def numeric_column(key, shape=(1,), default_value=None):
    return NumericColumn(key, tuple(shape), 0.0 if default_value is None else float(default_value))


def embedding_column(categorical_column, dimension, combiner="mean"):
    if combiner != "mean":
        raise ValueError("only combiner='mean' (the reference's) is implemented")
    return EmbeddingColumn(categorical_column, int(dimension), combiner)


def shared_embedding_columns(categorical_columns, dimension, combiner="mean"):
    """Returned in INPUT order (DIN relies on [0] = target, [1] = history: DIN/din.py:113-114); one table serves all."""
    shared = "_".join(sorted(c.key for c in categorical_columns)) + "_shared_embedding"
    return [EmbeddingColumn(c, int(dimension), combiner, shared_name=shared) for c in categorical_columns]


def crossed_column(keys, hash_bucket_size, hash_key=None):
    """The cross of 2 to 4 categorical columns (WideAndDeep/wide_and_deep.py:121).  Raw-string keys (TF hashes their strings
    with Fingerprint64) and crosses of crosses are not implemented."""
    keys = list(keys) if keys is not None else []
    if not hash_bucket_size or hash_bucket_size <= 1:
        raise ValueError(f"hash_bucket_size must be > 1. hash_bucket_size: {hash_bucket_size}")
    if len(keys) < 2:
        raise ValueError(f"keys must be a list with length > 1. Given: {keys}")
    if len(keys) > 4:
        raise ValueError(f"crossed_column: at most 4 keys are implemented, got {len(keys)}")
    for k in keys:
        if not isinstance(k, CategoricalColumn):
            raise ValueError(f"crossed_column: keys must be categorical columns (string keys are not implemented), got {k!r}")
    if int(hash_bucket_size) >= 2 ** 31:
        raise ValueError(f"crossed_column: hash_bucket_size must be < 2**31, got {hash_bucket_size}")
    # sparse_cross_hashed takes `hash_key if hash_key else _DEFAULT_HASH_KEY`: None and 0 both mean the default
    return CrossedColumn(tuple(keys), int(hash_bucket_size), int(hash_key) if hash_key else ops.CROSS_HASH_KEY)


def indicator_column(categorical_column):
    return IndicatorColumn(categorical_column)


def _base_columns(c) -> List[CategoricalColumn]:
    """The categorical columns a feature column reads (a crossed column reads each of its keys)."""
    base = c if isinstance(c, (CategoricalColumn, CrossedColumn)) else c.categorical_column
    return list(base.keys) if isinstance(base, CrossedColumn) else [base]


def make_parse_example_spec(feature_columns) -> Dict[str, object]:
    """tf.feature_column.make_parse_example_spec (SURVEY A.3)."""
    spec: Dict[str, object] = {}
    for c in feature_columns:
        if isinstance(c, NumericColumn):
            spec[c.key] = FixedLenFeature(c.shape, "float", c.default_value)
        else:
            for base in _base_columns(c):
                spec[base.key] = VarLenFeature("bytes")
    return spec


# ------------------------------------------------------------------ runtime
class _BagLookup(torch.autograd.Function):
    """One embedding column: ragged ids -> (B, D) slice of the output row; gradient = IndexedSlices on the table."""

    @staticmethod
    def forward(ctx, table, ids, offsets, out, out_col, slices_sink):
        ops.bag_lookup_fwd(table.data, ids, offsets, out=out, out_col=out_col)
        ctx.meta = (table, ids, offsets, out_col, slices_sink)
        ctx.mark_dirty(out)
        return out

    @staticmethod
    def backward(ctx, g):
        table, ids, offsets, out_col, sink = ctx.meta
        V, D = table.shape
        row_grads = ops.bag_lookup_bwd(g.contiguous(), out_col, V, D, ids, offsets)
        sink.append((table, ids, row_grads))                 # IndexedSlices: (rows = ids, values); ids < 0 carry zeros
        return None, None, None, g, None, None


@dataclass
class LookupContext:
    """Collects the IndexedSlices gradients produced by input_layer calls during one backward pass."""
    slices: List[Tuple[torch.nn.Parameter, torch.Tensor, torch.Tensor]] = field(default_factory=list)

    def to_dense(self) -> Dict[int, torch.Tensor]:
        out: Dict[int, torch.Tensor] = {}
        for table, ids, vals in self.slices:
            g = out.setdefault(id(table), torch.zeros_like(table.data))
            valid = (ids >= 0) & (ids < table.shape[0])
            g.index_add_(0, ids[valid], vals[valid])
        return out


def _ids_of(col: CategoricalColumn, values) -> np.ndarray:
    """Vocabulary ids of a ragged feature's values; values that are already int64 ids (parse_example_native) pass through."""
    if isinstance(values, np.ndarray) and values.dtype == np.int64:
        return values
    return col.vocabulary.lookup(values) if len(values) else np.zeros((0,), np.int64)


def _ragged_ids(col: CategoricalColumn, features, device) -> Tuple[torch.Tensor, torch.Tensor]:
    values, offsets = features[col.key]
    ids = _ids_of(col, values)
    return torch.from_numpy(np.ascontiguousarray(ids)).to(device), torch.from_numpy(np.asarray(offsets, np.int64)).to(device)


def pad_ragged(values: np.ndarray, offsets: np.ndarray, width: int, fill: int = -1) -> np.ndarray:
    """Ragged rows values[offsets[b]:offsets[b+1]] -> (B, width) int64, left aligned, padded with `fill` (one vectorised
    scatter: a Python loop over B = 4096 rows costs more than the DIN step it feeds)."""
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    B = lens.size
    if B and int(lens.max()) > width:
        raise ValueError(f"pad_ragged: a row holds {int(lens.max())} values, width is {width}")
    out = np.full((B, width), fill, np.int64)
    n = int(offsets[-1] - offsets[0]) if B else 0
    if n:
        row = np.repeat(np.arange(B, dtype=np.int64), lens)
        col = np.arange(n, dtype=np.int64) - np.repeat(offsets[:-1] - offsets[0], lens)
        out[row, col] = np.asarray(values)[offsets[0]:offsets[-1]]
    return out


def single_valued_ids(features, categorical_columns) -> np.ndarray:
    """(B, F) int64 id matrix of F single-valued categorical columns, in the order given, -1 where the value is missing /
    out of vocabulary -- the input of the fused lookup (autograd.lookup_fm2 / lookup / lookup_bi)."""
    cols = [c if isinstance(c, CategoricalColumn) else c.categorical_column for c in categorical_columns]
    B = len(features[cols[0].key][1]) - 1
    ids = np.full((B, len(cols)), -1, np.int64)
    for f, c in enumerate(cols):
        values, offsets = features[c.key]
        lens = np.diff(np.asarray(offsets))
        if np.any(lens > 1):
            raise ValueError(f"single_valued_ids: column {c.key} is multi-valued; use input_layer (bag lookup) for it")
        ids[lens == 1, f] = _ids_of(c, values)
    return ids


def parse_example_native(buf, offsets, lengths, feature_columns, read_feature_lists: bool = False, num_threads: int = 0):
    """``tf.parse_example(batch, make_parse_example_spec(feature_columns))`` + the vocabulary lookups in one native call
    (libctr_feed.so, include/ctr_feed.h): records are ``buf[offsets[b] : offsets[b] + lengths[b]]`` (see
    io.native.read_tfrecord_file).  Returns the same ``features`` dict input_layer / sequence_input_layer / indicator_dense
    take, with categorical entries already mapped: key -> (ids int64, row_offsets int64 (B+1,))."""
    from .io import native
    cats, dense = {}, {}
    for c in feature_columns:
        if isinstance(c, NumericColumn):
            dense[c.key] = (int(np.prod(c.shape)), float(c.default_value))
        else:
            for base in _base_columns(c):
                cats[base.key] = base.vocabulary.native()
    out = native.parse_examples(buf, offsets, lengths, cats, dense, read_feature_lists=read_feature_lists, num_threads=num_threads)
    for c in feature_columns:
        if isinstance(c, NumericColumn):
            out[c.key] = out[c.key].reshape((out[c.key].shape[0],) + tuple(c.shape))
    return out


def _table_for(col: EmbeddingColumn) -> torch.nn.Parameter:
    V, D = col.categorical_column.num_buckets, col.dimension
    std = D ** -0.5                                           # embedding_column default: truncated_normal(0, 1/sqrt(D))
    init = lambda shape: torch.nn.init.trunc_normal_(torch.empty(shape), 0.0, std, -2 * std, 2 * std)
    st = layers.default_store()
    saved, st.scope = st.scope, []                            # shared tables live outside the caller's scope path
    try:
        if col.shared_name:
            return st.get_variable(col.variable_name, (V, D), initializer=init)
    finally:
        st.scope = saved
    return layers.get_variable(col.variable_name, (V, D), initializer=init)


def input_layer(features, feature_columns, ctx: Optional[LookupContext] = None, device="cuda") -> torch.Tensor:
    """fc.input_layer: (B, sum d) with the columns concatenated in order of ``column.name`` (SURVEY A.6 / parity note 1).
    Indicator columns are refused here -- use ``indicator_dense`` (a (B, sum V) multi-hot is never materialised)."""
    cols = sorted(feature_columns, key=lambda c: c.name)
    if any(isinstance(c, IndicatorColumn) for c in cols):
        raise ValueError("indicator columns: use feature_column.indicator_dense(features, columns, units=1)")
    widths = [c.dimension if isinstance(c, EmbeddingColumn) else int(np.prod(c.shape)) for c in cols]
    B = None
    for c in cols:
        B = (len(features[c.categorical_column.key][1]) - 1) if isinstance(c, EmbeddingColumn) else features[c.key].shape[0]
        break
    out = torch.zeros((B, sum(widths)), dtype=torch.float32, device=device)
    sink = ctx.slices if ctx is not None else []
    col0 = 0
    for c, w in zip(cols, widths):
        if isinstance(c, NumericColumn):
            out[:, col0:col0 + w] = torch.from_numpy(np.asarray(features[c.key], np.float32).reshape(B, w)).to(device)
        else:
            table = _table_for(c)
            ids, offsets = _ragged_ids(c.categorical_column, features, device)
            out = _BagLookup.apply(table, ids, offsets, out, col0, sink)
        col0 += w
    return out


def sequence_input_layer(features, feature_columns, ctx: Optional[LookupContext] = None, device="cuda"):
    """tf.contrib.feature_column.sequence_input_layer: (B, T_max_in_batch, sum d) zero padded + sequence_length (B,) int64.
    Every VALUE of the ragged feature is one step (single-valued lookup per step)."""
    cols = sorted(feature_columns, key=lambda c: c.name)
    outs, lengths = [], None
    for c in cols:
        if not isinstance(c, EmbeddingColumn):
            raise ValueError("sequence_input_layer only accepts (shared) embedding columns")
        values, offsets = features[c.categorical_column.key]
        offsets = np.asarray(offsets, np.int64)
        lens = np.diff(offsets)
        B, T = len(lens), int(lens.max()) if len(lens) else 0
        table = _table_for(c)
        ids = _ids_of(c.categorical_column, values)
        padded = pad_ragged(ids, offsets, max(T, 1))            # -1 -> zero vector == zero padding
        flat_ids = torch.from_numpy(padded.reshape(-1)).to(device)
        step_off = torch.arange(flat_ids.numel() + 1, dtype=torch.int64, device=device)
        buf = torch.zeros((flat_ids.numel(), c.dimension), dtype=torch.float32, device=device)
        sink = ctx.slices if ctx is not None else []
        emb = _BagLookup.apply(table, flat_ids, step_off, buf, 0, sink).reshape(B, max(T, 1), c.dimension)[:, :T]
        outs.append(emb)
        lengths = torch.from_numpy(lens.astype(np.int64)).to(device)
    return (outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)), lengths


def indicator_dense(features, indicator_columns, units: int = 1, name: str = "fm_first_order_dense", device="cuda") -> torch.Tensor:
    """``tf.layers.dense(fc.input_layer(features, indicator_columns), 1, name=name)`` (DeepFM/deepfm.py:180-181) without the
    (B, sum V) multi-hot: a multi-hot times a one-column kernel is the sum of the kernel rows of the present ids.
    The kernel variable has the reference's shape (sum V, 1) with the columns' blocks in NAME order; bias (1,) zeros."""
    if units != 1:
        raise ValueError("only units=1 (the reference's first-order term) is implemented")
    cols = sorted(indicator_columns, key=lambda c: c.name)
    crossed = [isinstance(c.categorical_column, CrossedColumn) for c in cols]
    if any(crossed):
        if not all(crossed):
            raise ValueError("indicator_dense: a list that mixes crossed and plain indicator columns is not implemented")
        return _crossed_dense(features, cols, name, device)
    sizes = [c.categorical_column.num_buckets for c in cols]
    with layers.variable_scope(name):
        kernel = layers.get_variable("kernel", (sum(sizes), 1))
        bias = layers.get_variable("bias", (1,), initializer=lambda s: torch.zeros(s))
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=device)
    B = len(features[cols[0].categorical_column.key][1]) - 1
    ids = torch.full((B, len(cols)), -1, dtype=torch.int64)
    for f, c in enumerate(cols):
        values, offsets = features[c.categorical_column.key]
        offsets = np.asarray(offsets)
        if np.any(np.diff(offsets) > 1):
            raise ValueError("indicator_dense: multi-valued indicator columns are not implemented")
        got = _ids_of(c.categorical_column, values)
        has = np.diff(offsets) == 1
        col_ids = np.full((B,), -1, np.int64)
        col_ids[has] = got
        ids[:, f] = torch.from_numpy(col_ids)
    return _FirstOrder.apply(kernel, bias, off, ids.to(device))


class _FirstOrder(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kernel, bias, off, ids):
        ctx.save_for_backward(off, ids)
        ctx.shape = kernel.shape
        # the bias is added on the device: reading it back (bias.item()) would be a host sync on every forward and would
        # make the step impossible to capture in a CUDA graph
        return ops.first_order_fwd(kernel.data.reshape(-1).contiguous(), off, ids, 0.0) + bias.data.reshape(1, 1)

    @staticmethod
    def backward(ctx, g):
        off, ids = ctx.saved_tensors
        rows = off[1:] - off[:-1]
        valid = (ids >= 0) & (ids < rows[None, :])
        gr = (ids + off[:-1][None, :])[valid]
        dk = torch.zeros(ctx.shape, dtype=g.dtype, device=g.device)
        dk.index_add_(0, gr, g.expand(-1, ids.shape[1])[valid].unsqueeze(-1))   # tiny (sum V, 1) dense(1) kernel gradient
        return dk, g.sum().reshape(1), None, None


def crossed_ragged_ids(features, col: CrossedColumn) -> Tuple[np.ndarray, np.ndarray]:
    """The keys of a crossed column as one ragged block: values (nnz,) int64 vocabulary ids (OOV -1 kept) and offsets (K, B+1)
    int64, key k of sample b = values[offsets[k,b] : offsets[k,b+1]] (the input of ctr_crossed_indicator_fwd / _bwd)."""
    vals, offs, base = [], [], 0
    for k in col.keys:
        values, offsets = features[k.key]
        offsets = np.asarray(offsets, np.int64)
        vals.append(np.asarray(_ids_of(k, values), np.int64))
        offs.append(offsets + base)
        base += len(vals[-1])
    if len({len(o) for o in offs}) != 1:
        raise ValueError(f"crossed column {col.name}: its keys hold different batch sizes")
    return np.concatenate(vals), np.stack(offs)


def _crossed_dense(features, cols, name, device) -> torch.Tensor:
    """indicator_dense over crossed indicator columns (WideAndDeep/wide_and_deep.py:208-210): one (sum buckets, 1) kernel with
    the columns' blocks in name order; each block is one hashed gather-sum per sample, and the crossed ids never exist."""
    sizes = [c.categorical_column.num_buckets for c in cols]
    with layers.variable_scope(name):
        kernel = layers.get_variable("kernel", (sum(sizes), 1))
        bias = layers.get_variable("bias", (1,), initializer=lambda s: torch.zeros(s))
    blocks, lo = [], 0
    for c, nb in zip(cols, sizes):
        values, offsets = crossed_ragged_ids(features, c.categorical_column)
        blocks.append((torch.from_numpy(values).to(device), torch.from_numpy(offsets).to(device), lo, nb, c.categorical_column.hash_key))
        lo += nb
    return _CrossedDense.apply(kernel, bias, blocks)


class _CrossedDense(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kernel, bias, blocks):
        ctx.blocks, ctx.shape = blocks, kernel.shape
        w = kernel.data.reshape(-1)
        out = None
        for values, offsets, lo, nb, hash_key in blocks:
            # the bias goes into the first block's launch (read on the device); later blocks add a zero bias
            b = bias.data if out is None else torch.zeros((1,), dtype=torch.float32, device=w.device)
            y = ops.crossed_indicator_fwd(values, offsets, nb, w[lo:lo + nb], b, hash_key)
            out = y if out is None else out + y
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dk, db = [], None
        for values, offsets, lo, nb, hash_key in ctx.blocks:
            d, b = ops.crossed_indicator_bwd(values, offsets, nb, g, hash_key, want_bias=db is None)
            dk.append(d)
            db = b if db is None else db
        dk = dk[0] if len(dk) == 1 else torch.cat(dk)
        return dk.reshape(ctx.shape), db, None
