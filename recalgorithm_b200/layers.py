"""Host-side mirror of the reference's layer interface (the drop-in boundary, SURVEY.md section 8b).

The reference has no package API: each ``model_fn`` calls plain Python functions that create their
parameters by side effect with ``tf.get_variable`` inside ``tf.variable_scope`` blocks.  The functions
below keep those names, argument meanings, variable names/shapes and error behaviour, so that a
``model_fn`` body ported to this engine reads like the reference's own:

    with variable_scope("cross_part"):                 # DCN/dcn.py:156-160
        cross_vec = concat_all
        for i in range(params["num_cross_layer"]):
            cross_vec = cross_layer(x0=concat_all, xl=cross_vec, index=i)

Each call is one launch of the matching sm_90a kernel (through recalgorithm_b200.autograd); there
is no other implementation behind these names.
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict, List, Optional, Tuple

import torch

from . import autograd

AUTO_REUSE = "AUTO_REUSE"


class VariableStore:
    """Name-keyed parameter registry mirroring TF1 variable scopes (``tf.get_variable`` semantics:
    create on first use with the default glorot-uniform initializer, reuse afterwards)."""

    def __init__(self, device="cuda", seed: Optional[int] = None):
        self.device = torch.device(device)
        self.vars: Dict[str, torch.nn.Parameter] = {}
        self.scope: List[str] = []
        self.gen = torch.Generator(device="cpu")
        if seed is not None:
            self.gen.manual_seed(seed)

    def full_name(self, name: str) -> str:
        return "/".join(self.scope + [name])

    def get_variable(self, name: str, shape, initializer=None) -> torch.nn.Parameter:
        full = self.full_name(name)
        shape = tuple(int(s) for s in shape)
        if full in self.vars:
            v = self.vars[full]
            if tuple(v.shape) != shape:
                raise ValueError(f"Trying to share variable {full}, but specified shape {shape} and found shape {tuple(v.shape)}.")
            return v
        if initializer is None:                         # tf.get_variable default: glorot_uniform_initializer
            if len(shape) >= 2:
                rf = 1
                for s in shape[:-2]:
                    rf *= s
                fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
            else:
                fan_in = fan_out = shape[0] if shape else 1
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            data = (torch.rand(shape, generator=self.gen) * 2 - 1) * lim
        elif callable(initializer):
            data = initializer(shape)
        else:
            data = torch.as_tensor(initializer, dtype=torch.float32).reshape(shape)
        v = torch.nn.Parameter(data.to(torch.float32).to(self.device).contiguous())
        self.vars[full] = v
        return v

    def assign(self, values: Dict[str, "torch.Tensor"]):
        """Inject weights by their TF variable names (parity is defined on injected weights)."""
        for k, val in values.items():
            t = torch.as_tensor(val, dtype=torch.float32).to(self.device).contiguous()
            if k in self.vars:
                if tuple(self.vars[k].shape) != tuple(t.shape):
                    raise ValueError(f"{k}: shape {tuple(t.shape)} != {tuple(self.vars[k].shape)}")
                self.vars[k].data.copy_(t)
            else:
                self.vars[k] = torch.nn.Parameter(t)

    def parameters(self):
        return list(self.vars.values())


_default_store: Optional[VariableStore] = None


def default_store() -> VariableStore:
    global _default_store
    if _default_store is None:
        _default_store = VariableStore()
    return _default_store


def set_default_store(store: VariableStore) -> VariableStore:
    global _default_store
    _default_store = store
    return store


@contextlib.contextmanager
def variable_scope(name: str, reuse=None):
    st = default_store()
    st.scope.append(name)
    try:
        yield
    finally:
        st.scope.pop()


def get_variable(name, shape, dtype=None, initializer=None):
    return default_store().get_variable(name, shape, initializer)


# --------------------------------------------------------------------------------------------------- DCN
def cross_layer(x0: torch.Tensor, xl: torch.Tensor, index: int) -> torch.Tensor:
    """dcn cross layer -- same signature as DCN/cross_layer.py:4.  Variables ``wl_{index}``, ``bl_{index}`` of shape
    (d, 1), default (glorot-uniform) initialised -- the bias is NOT zero-initialised in the reference (:18-19)."""
    dimension = int(x0.shape[-1])
    wl = get_variable(name=f"wl_{index}", shape=(dimension, 1))
    bl = get_variable(name=f"bl_{index}", shape=(dimension, 1))
    return autograd.cross_stack(x0, wl.reshape(1, dimension), bl.reshape(1, dimension), xl=None if xl is x0 else xl)


def cross_network(x0: torch.Tensor, num_cross_layer: int) -> torch.Tensor:
    """The whole loop of DCN/dcn.py:157-160 (``for i: cross_vec = cross_layer(x0, cross_vec, i)``) in ONE launch;
    creates exactly the variables the loop would create."""
    dimension = int(x0.shape[-1])
    if num_cross_layer == 0:
        return x0
    ws = [get_variable(name=f"wl_{i}", shape=(dimension, 1)) for i in range(num_cross_layer)]
    bs = [get_variable(name=f"bl_{i}", shape=(dimension, 1)) for i in range(num_cross_layer)]
    w = torch.cat([t.reshape(1, dimension) for t in ws], 0)
    b = torch.cat([t.reshape(1, dimension) for t in bs], 0)
    return autograd.cross_stack(x0, w, b)


def _cross_v2_variables(dimension: int, index, projection_dim):
    with variable_scope(f"cross_v2_{index}"):
        if projection_dim is None:
            w, u = get_variable("kernel", (dimension, dimension)), None
        else:
            w = get_variable("kernel_v", (dimension, projection_dim))
            u = get_variable("kernel_u", (projection_dim, dimension))
        b = get_variable("bias", (dimension,), initializer=lambda s: torch.zeros(s))
    return w, u, b


def _projection_dim(projection_dim):
    if projection_dim is None:
        return None
    r = int(projection_dim)
    if r < 1:
        raise ValueError(f"projection_dim must be at least 1 (None selects the full-rank layer), got {projection_dim!r}")
    return r


def cross_layer_v2(x0: torch.Tensor, xl: torch.Tensor, index: int, projection_dim=None) -> torch.Tensor:
    """One DCN-V2 cross layer (Wang et al., WWW 2021, arXiv:2008.13535, eq. 1-2), same call shape as cross_layer:
    ``x0 * (xl . W + bias) + xl`` with W = ``kernel`` (d, d), or at low rank W = ``kernel_v . kernel_u``.

    The reference tree has no DCN-V2 code, so the variable names are this project's choice: in the caller's scope, a scope
    ``cross_v2_{index}`` holding ``kernel`` (d, d) -- or, when ``projection_dim`` r is given, ``kernel_v`` (d, r) and
    ``kernel_u`` (r, d), the paper's V and U^T -- all glorot-uniform, and ``bias`` (d,) zeros.  ``projection_dim`` goes
    through ``int()`` (a string width works)."""
    r = _projection_dim(projection_dim)
    w, u, b = _cross_v2_variables(int(x0.shape[-1]), index, r)
    return autograd.cross_v2(x0, w[None], None if u is None else u[None], b[None], r or 0, xl=None if xl is x0 else xl)


def cross_network_v2(x0: torch.Tensor, num_cross_layer, projection_dim=None) -> torch.Tensor:
    """``for i: x = cross_layer_v2(x0, x, i, projection_dim)`` over ``num_cross_layer`` layers in one call each way; creates
    exactly the variables the loop would create.  ``num_cross_layer = 0`` returns x0 and launches nothing."""
    n, r = int(num_cross_layer), _projection_dim(projection_dim)
    if n == 0:
        return x0
    vs = [_cross_v2_variables(int(x0.shape[-1]), i, r) for i in range(n)]
    w = torch.stack([v[0] for v in vs])
    u = None if r is None else torch.stack([v[1] for v in vs])
    return autograd.cross_v2(x0, w, u, torch.stack([v[2] for v in vs]), r or 0)


_MIX_ACTIVATIONS = ("tanh", "identity")


def cross_network_mix(x0: torch.Tensor, num_cross_layer, num_experts=4, low_rank=32, activation="tanh") -> torch.Tensor:
    """DCN-Mix cross network (Wang et al., WWW 2021, arXiv:2008.13535, eq. 3-4): ``num_cross_layer`` layers, each a
    softmax-gated mixture of ``num_experts`` low-rank experts, ``x_{l+1} = x0 * (sum_i p_i g(g(x_l V_i) C_i) U_i + bias)
    + x_l`` with ``p = softmax(x_l gate)`` and g = tanh (``activation="tanh"``) or the identity, in one call each way.

    The reference tree has no DCN-Mix code, so the variable names are this project's choice: in the caller's scope,
    ``cross_mix_{l}/expert_{i}/kernel_v`` (d, r), ``kernel_c`` (r, r) and ``kernel_u`` (r, d) -- the paper's V_i, C_i^T and
    U_i^T, one 2-D variable per expert matrix so that glorot-uniform sees its own fans -- and ``cross_mix_{l}/bias`` (d,)
    zeros; the paper's gates carry no layer index, so one ``cross_mix_gates/kernel`` (d, K), glorot-uniform, serves every
    layer.  The integer arguments go through ``int()``; ``num_cross_layer = 0`` returns x0 with no variable and no launch."""
    n, K, r = int(num_cross_layer), int(num_experts), int(low_rank)
    if activation not in _MIX_ACTIVATIONS:
        raise ValueError(f"activation must be one of {_MIX_ACTIVATIONS}, got {activation!r}")
    if n < 0:
        raise ValueError(f"num_cross_layer must be at least 0, got {num_cross_layer!r}")
    if K < 1 or r < 1:
        raise ValueError(f"num_experts and low_rank must be at least 1, got {num_experts!r} and {low_rank!r}")
    if K > 16 or K * r > 128:
        raise ValueError(f"num_experts must be at most 16 and num_experts * low_rank at most 128, got {K} * {r}")
    if n == 0:
        return x0
    d = int(x0.shape[-1])
    vs, cs, us, bs = [], [], [], []
    for l in range(n):
        with variable_scope(f"cross_mix_{l}"):
            for i in range(K):
                with variable_scope(f"expert_{i}"):
                    vs.append(get_variable("kernel_v", (d, r)))
                    cs.append(get_variable("kernel_c", (r, r)))
                    us.append(get_variable("kernel_u", (r, d)))
            bs.append(get_variable("bias", (d,), initializer=lambda s: torch.zeros(s)))
    with variable_scope("cross_mix_gates"):
        gate = get_variable("kernel", (d, K))
    stack = lambda ts, *shape: torch.stack(ts).reshape(n, K, *shape)
    return autograd.cross_mix(x0, stack(vs, d, r), stack(cs, r, r), stack(us, r, d), torch.stack(bs), gate, activation)


# --------------------------------------------------------------------------------------------------- xDeepFM
def cin_layer(x0: torch.Tensor, xk: torch.Tensor, hk_1, index: int, return_pooled: bool = False):
    """xdeepfm CIN layer -- same signature as xDeepFM/cin_layer.py:4.  x0 (B,m,D), xk (B,hk,D) -> (B,hk_1,D).
    ``hk_1`` may arrive as a *string* (the reference splits a comma flag, xdeepfm.py:253).  Variable
    ``cin_layer_{index}_filter`` of shape (1, hk*m, hk_1).  ``return_pooled`` additionally returns sum over D
    (the ``tf.reduce_sum(x, axis=-1)`` of xdeepfm.py:173) from the same kernel."""
    hk_1 = int(hk_1)
    m = int(x0.shape[1])
    hk = int(xk.shape[1])
    filters = get_variable(name=f"cin_layer_{index}_filter", shape=(1, hk * m, hk_1))
    return autograd.cin(x0, xk, filters[0], want_pooled=return_pooled)


# --------------------------------------------------------------------------------------------------- DIN
def din_attention(query: torch.Tensor, keys: torch.Tensor, keys_length: torch.Tensor, is_softmax: bool = False):
    """DIN attention unit -- same signature as DIN/din_attention.py:4.  Dense layers ``f1_att`` (4H->64, relu),
    ``f2_att`` (64->32, relu), ``f3_att`` (32->1) with AUTO_REUSE: variables <name>/kernel, <name>/bias (zeros)."""
    H = int(query.shape[-1])
    params = []
    for name, (fi, fo) in (("f1_att", (4 * H, 64)), ("f2_att", (64, 32)), ("f3_att", (32, 1))):
        with variable_scope(name, reuse=AUTO_REUSE):
            params.append(get_variable("kernel", (fi, fo)))
            params.append(get_variable("bias", (fo,), initializer=lambda s: torch.zeros(s)))
    return autograd.din_attention(query, keys, keys_length.to(torch.int64), *params, is_softmax=is_softmax)


# --------------------------------------------------------------------------------------------------- FiBiNET
def senet(input: torch.Tensor, embedding_dim: int, reduction_ratio: int) -> torch.Tensor:
    """SENET -- same signature as FiBiNET/senet.py:4.  NB the reference reduces from ``embedding_dim``
    (``reduction_dim = embedding_dim // reduction_ratio``, :18), not from the field count."""
    F = int(input.shape[1])
    reduction_dim = embedding_dim // reduction_ratio
    assert reduction_dim < embedding_dim, "reduction_dim must be less than embedding_dim"
    w1 = get_variable(name="senet_w1", shape=(F, reduction_dim))
    w2 = get_variable(name="senet_w2", shape=(reduction_dim, F))
    return autograd.senet(input, w1, w2)


def bilinear_interaction_layer(input: torch.Tensor, embedding_dim: int, type: str, name: str) -> torch.Tensor:
    """Bilinear interaction -- same signature as FiBiNET/bilinear_interaction_layer.py:5.  Output is
    (B, (F-1)(F-2)/2, K): the reference enumerates ``combinations(range(F-1), 2)`` (:24,29,33)."""
    F = int(input.shape[1])
    if type == "all":
        w = get_variable(name=f"{name}_w_all", shape=(embedding_dim, embedding_dim))
    elif type == "each":
        w = get_variable(name=f"{name}_w_each", shape=(F - 1, embedding_dim, embedding_dim))
    elif type == "interaction":
        w = get_variable(name=f"{name}_w_interaction", shape=(F * (F - 1) // 2, embedding_dim, embedding_dim))
    else:
        raise ValueError(f"Bilinear Interaction type must be in ['all','each','interaction'], got '{type}'")
    return autograd.bilinear(input, w, type)


# --------------------------------------------------------------------------------------------------- DeepFM
def fm_second_order(tables: autograd.EmbeddingTables, ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The lookup + FM second-order block of DeepFM/deepfm.py:184-200 in one kernel: per-field ids (B,F) ->
    (fields_embeddings as a (B,F,K) tile, fm_second_order_logit (B,1))."""
    return autograd.lookup_fm2(tables, ids)


# --------------------------------------------------------------------------------------------------- NFM / FwFM / AFM (8f.4)
def bi_interaction(tables: autograd.EmbeddingTables, ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The lookup + bi-interaction pooling block of NFM/nfm.py:155-168 in one kernel: per-field ids (B,F) ->
    (fields_embeddings (B,F,K), nfm (B,K)) -- the vector the reference then feeds to batch-norm / dropout / the DNN."""
    return autograd.lookup_bi(tables, ids)


def fwfm_second_order(fields_embeddings: torch.Tensor) -> torch.Tensor:
    """FwFM/fwfm.py:145-158: creates ``fields_pair_strength/fields_pair_strength_weight`` (F(F-1)/2,) and returns
    ``fwfm_second_order_logit`` (B,1) for the (B,F,K) field embeddings."""
    F = int(fields_embeddings.shape[1])
    with variable_scope("fields_pair_strength"):
        r = get_variable("fields_pair_strength_weight", shape=(F * (F - 1) // 2,))
    return autograd.fwfm(fields_embeddings, r)


FWBI_MAX_GROUPS = 8


def _fwbi_variables(field_groups, F: int, D: int):
    """Numbers the group keys by first appearance and creates ``field_wise_bi_interaction/{kernel_mf, kernel_fm, bias_mf,
    bias_fm}`` in the caller's scope."""
    keys = list(field_groups)
    if len(keys) != F:
        raise ValueError(f"field_groups has {len(keys)} entries but there are {F} fields")
    number = {}
    groups = tuple(number.setdefault(k, len(number)) for k in keys)
    M = len(number)
    if M > FWBI_MAX_GROUPS:
        raise ValueError(f"field_groups has {M} distinct groups; the field-wise bi-interaction supports at most "
                         f"{FWBI_MAX_GROUPS}")
    with variable_scope("field_wise_bi_interaction"):
        kmf = get_variable("kernel_mf", (M * (M - 1) // 2,), initializer=lambda s: torch.ones(s))
        kfm = get_variable("kernel_fm", (M,), initializer=lambda s: torch.full(s, 0.5))
        bmf = get_variable("bias_mf", (D,), initializer=lambda s: torch.zeros(s))
        bfm = get_variable("bias_fm", (D,), initializer=lambda s: torch.zeros(s))
    return groups, (kmf, kfm, bmf, bfm)


def field_wise_bi_interaction(fields_embeddings: torch.Tensor, field_groups) -> torch.Tensor:
    """FLEN field-wise bi-interaction (Chen et al., arXiv:1911.04690) of the (B,F,D) field embeddings -> h (B,D).

    ``field_groups`` gives each field's group key; group m is the m-th distinct key in order of first appearance (at most
    8).  h = sum_{i<j} kernel_mf[pair(i,j)] p_i p_j + bias_mf + sum_m kernel_fm[m] (p_m^2 - q_m) + bias_fm, p_m / q_m the
    sums of the group's embeddings / squared embeddings.  The reference tree has no FLEN file, so the variable names are
    this project's choice: ``field_wise_bi_interaction/kernel_mf`` (M(M-1)/2,) ones, ``kernel_fm`` (M,) 0.5, ``bias_mf`` and
    ``bias_fm`` (D,) zeros, in the caller's scope."""
    groups, w = _fwbi_variables(field_groups, int(fields_embeddings.shape[1]), int(fields_embeddings.shape[2]))
    return autograd.fwbi(fields_embeddings, groups, *w)


def field_wise_bi_interaction_lookup(tables: autograd.EmbeddingTables, ids: torch.Tensor, field_groups):
    """The lookup and field_wise_bi_interaction in one kernel each way: per-field ids (B,F) -> (fields_embeddings (B,F,D),
    h (B,D)); same variables as field_wise_bi_interaction."""
    groups, w = _fwbi_variables(field_groups, int(ids.shape[1]), tables.dim)
    return autograd.lookup_fwbi(tables, ids, groups, *w)


def afm_attention(fields_embeddings: torch.Tensor, embedding_dim: int, attention_factor: int) -> torch.Tensor:
    """AFM/afm.py:152-186: attention-weighted sum of the pairwise hadamard products, (B,K).  Creates
    ``attention_part/attention_{w,b,h}`` with the reference's shapes; ``p`` and the final matmul (afm.py:187-188) stay
    with the caller."""
    with variable_scope("attention_part"):
        w = get_variable(name="attention_w", shape=(embedding_dim, attention_factor))
        b = get_variable(name="attention_b", shape=(attention_factor,))
        h = get_variable(name="attention_h", shape=(attention_factor, 1))
    return autograd.afm(fields_embeddings, w, b, h)


# --------------------------------------------------------------------------------------------------- BST (8f.4)
def bst_transformer(queries: torch.Tensor, keys: torch.Tensor, values: torch.Tensor, keys_length: torch.Tensor, heads: int,
                    index: int, max_length: int, use_position_embedding: bool = True) -> torch.Tensor:
    """Transformer block -- same signature as BST/transformer_layer.py:6.  Variables carry the names TF gives them inside
    the caller's scope (``transformer_part`` in BST/bst.py:184): ``position_embedding`` (shared by every block),
    ``w_{q,k,v,o}_{index}``, ``LayerNorm[/_n]/{beta,gamma}`` and ``dense[/_n]/{kernel,bias}`` with TF's uniquifying suffixes
    for block ``index`` (two layer norms and one dense per block)."""
    d = int(queries.shape[-1])
    suffix = lambda base, n: base if n == 0 else f"{base}_{n}"
    ones, zeros = (lambda s: torch.ones(s)), (lambda s: torch.zeros(s))
    p = {"position_embedding": get_variable(name="position_embedding", shape=(max_length, d)),
         "w_q": get_variable(name=f"w_q_{index}", shape=(heads, d, d)), "w_k": get_variable(name=f"w_k_{index}", shape=(heads, d, d)),
         "w_v": get_variable(name=f"w_v_{index}", shape=(heads, d, d)), "w_o": get_variable(name=f"w_o_{index}", shape=(heads * d, d))}
    with variable_scope(suffix("LayerNorm", 2 * index)):
        p["ln1_beta"] = get_variable("beta", (d,), initializer=zeros); p["ln1_gamma"] = get_variable("gamma", (d,), initializer=ones)
    with variable_scope(suffix("dense", index)):
        p["dense_kernel"] = get_variable("kernel", (d, d)); p["dense_bias"] = get_variable("bias", (d,), initializer=zeros)
    with variable_scope(suffix("LayerNorm", 2 * index + 1)):
        p["ln2_beta"] = get_variable("beta", (d,), initializer=zeros); p["ln2_gamma"] = get_variable("gamma", (d,), initializer=ones)
    return autograd.bst_transformer(queries, keys, values, keys_length.to(torch.int64), p, heads, max_length, use_position_embedding)


# --------------------------------------------------------------------------------------------------- PNN
def pnn_product_layer(fields_embeddings: torch.Tensor, num_fields: int, embedding_dim: int, output_dimension: int,
                      product_method: str = "IPNN") -> torch.Tensor:
    """The product layer of PNN/pnn.py:125-181 in one kernel each way: ``fields_embeddings`` (B, F*K) (the input_layer
    outputs concatenated, or (B,F,K)) -> ``product_final`` = relu(lz + lp + bias) (B, output_dimension).

    Creates ``linear_part/linear_w`` (F*K, N), then ``product_part/inner_product_w`` (N, F) when ``product_method`` is
    exactly ``"IPNN"`` and ``product_part/outer_product_w`` (N, K, K) for ANY other value (the reference's ``else`` branch,
    :160 -- ``"ipnn"`` builds the OPNN variable, with no error), then ``bias`` (N,) in the caller's scope.  All four are
    default (glorot-uniform) initialised; the bias is not zero.  The reference's ``weight_regularizer``
    (``l2_regularizer(scale)`` on the three weight matrices, :137,150,164) adds ``scale * sum(w**2) / 2`` per weight to the
    loss when scale > 0 and nothing at the default 0.0: it is a loss-side term the caller adds in torch (see
    examples/model_bodies.py), no kernel."""
    F, K, N = int(num_fields), int(embedding_dim), int(output_dimension)
    method = 0 if product_method == "IPNN" else 1
    with variable_scope("linear_part"):
        linear_w = get_variable("linear_w", shape=(F * K, N))
    with variable_scope("product_part"):
        if method == 0:
            wprod = get_variable("inner_product_w", shape=(N, F))
        else:
            wprod = get_variable("outer_product_w", shape=(N, K, K))
    bias = get_variable("bias", shape=(N,))
    e = fields_embeddings.reshape(-1, F, K)
    return autograd.pnn(e, linear_w, wprod, bias, method)


# --------------------------------------------------------------------------------------------------- DIEN
def dien_interest_evolution(sequnence_input: torch.Tensor, sequnence_length: torch.Tensor, target_input: torch.Tensor,
                            gru_output_units, custom_gru_type: str = "AGRU", return_attention_scores: bool = False):
    """The seq_encoder block of DIEN/dien.py:198-229 in one kernel each way: the GRU interest extractor over every position,
    the attention ``softmax_t(h_t . (W e_a))`` with positions t >= length masked, and the AGRU / AUGRU interest evolution over
    the first ``length`` positions.  Returns ``final_state`` (B, nh), and also the attention scores (B, T, 1) (forward only,
    what the reference logs) when ``return_attention_scores``.

    Creates, in the caller's scope (``seq_encoder`` in the reference), the variables TF gives them:
    ``rnn/gru_cell/{gates,candidate}/{kernel,bias}`` (tf.nn.rnn_cell.GRUCell: gate bias ones, candidate bias zeros),
    ``attention_project_matrix`` (nh, na), and the custom cell's ``rnn/{gates,candidate}/{kernel,bias}`` (gate bias ones,
    custom_grucell.py:66-68).  Kernels are glorot-uniform.  ``custom_gru_type == "AUGRU"`` selects AUGRU; ANY other value
    selects AGRU (dien.py:220-223).  ``gru_output_units`` may arrive as a string."""
    nh, na, cell, params = _dien_variables(sequnence_input, gru_output_units, custom_gru_type)
    final_state, scores = autograd.dien(sequnence_input, sequnence_length.to(torch.int64), target_input, params, nh, cell)
    if return_attention_scores:
        return final_state, scores.unsqueeze(-1)
    return final_state


def _dien_variables(sequnence_input, gru_output_units, custom_gru_type):
    """The nine variables of the seq_encoder block in the caller's scope (ops.DIEN_PARAM_ORDER) -> (nh, na, cell, params)."""
    nh = int(gru_output_units)
    na = int(sequnence_input.shape[-1])
    cell = 1 if custom_gru_type == "AUGRU" else 0
    ones, zeros = (lambda s: torch.ones(s)), (lambda s: torch.zeros(s))
    with variable_scope("rnn"):
        with variable_scope("gru_cell"):
            with variable_scope("gates"):
                gk = get_variable("kernel", (na + nh, 2 * nh)); gb = get_variable("bias", (2 * nh,), initializer=ones)
            with variable_scope("candidate"):
                ck = get_variable("kernel", (na + nh, nh)); cb = get_variable("bias", (nh,), initializer=zeros)
    att = get_variable("attention_project_matrix", (nh, na))
    with variable_scope("rnn"):
        with variable_scope("gates"):
            egk = get_variable("kernel", (2 * nh, 2 * nh)); egb = get_variable("bias", (2 * nh,), initializer=ones)
        with variable_scope("candidate"):
            eck = get_variable("kernel", (2 * nh, nh)); ecb = get_variable("bias", (nh,), initializer=zeros)
    return nh, na, cell, (gk, gb, ck, cb, att, egk, egb, eck, ecb)


def dien_interest_evolution_aux(sequnence_input: torch.Tensor, sequnence_length: torch.Tensor, target_input: torch.Tensor,
                                neg_sequnence_input: torch.Tensor, aux_project_matrix: torch.Tensor, gru_output_units,
                                custom_gru_type: str = "AGRU", negative_sample_number=3,
                                return_attention_scores: bool = False):
    """dien_interest_evolution plus DIEN's auxiliary loss (DIEN/dien.py:256-300) over the same extractor states h_t, one
    kernel set each way.  Returns ``(final_state, aux_loss)``, or ``(final_state, attention_scores (B, T, 1), aux_loss)``
    when ``return_attention_scores``.

    ``aux_loss = -(1/B) sum_b sum_{t < len-1} [log sig(h_t . W^T x_{t+1}) + sum_n log(1 - sig(h_t . W^T neg_{t,n}))]`` with
    W = ``aux_project_matrix`` (na, nh): the paper's next-behaviour loss, i.e. the negative of the reference's aux_loss, in
    the numerically stable softplus form.  ``neg_sequnence_input`` (B, (T-1)*negative_sample_number, na) holds the
    negatives of position t in rows t*T_neg .. t*T_neg + T_neg - 1 (the reshape at :279); the caller samples them, e.g.
    through the shared ``feedid`` table.  ``aux_project_matrix`` is an argument because the reference creates it in
    model_fn's own ``aux_loss`` scope; the nine seq_encoder variables are created in the caller's scope exactly as by
    dien_interest_evolution.  ``negative_sample_number`` may arrive as a string, like ``gru_output_units``."""
    T_neg = int(negative_sample_number)
    nh, na, cell, params = _dien_variables(sequnence_input, gru_output_units, custom_gru_type)
    B, T = sequnence_input.shape[:2]
    want = (B, (T - 1) * T_neg, na)
    if tuple(neg_sequnence_input.shape) != want:
        raise ValueError(f"neg_sequnence_input: expected shape {want} ((B, (T-1)*negative_sample_number, na)), "
                         f"got {tuple(neg_sequnence_input.shape)}")
    if tuple(aux_project_matrix.shape) != (na, nh):
        raise ValueError(f"aux_project_matrix: expected shape {(na, nh)}, got {tuple(aux_project_matrix.shape)}")
    final_state, scores, aux_loss = autograd.dien_aux(sequnence_input, sequnence_length.to(torch.int64), target_input,
                                                      neg_sequnence_input, aux_project_matrix, params, nh, cell, T_neg)
    if return_attention_scores:
        return final_state, scores.unsqueeze(-1), aux_loss
    return final_state, aux_loss


# --------------------------------------------------------------------------------------------------- DeepCrossing
def residual_unit(input: torch.Tensor, internal_dim=None, index=None) -> torch.Tensor:
    """DeepCrossing residual unit -- same signature as DeepCrossing/residual_unit.py:4, one kernel each way:
    ``relu(input + dense(relu(dense(input, internal_dim)), output_dim))`` with ``output_dim`` the input's last dimension.

    Creates, in the caller's scope (``residual_module`` in the reference), the variables of the two ``tf.layers.dense``
    calls: ``dense_{index}_0/kernel`` (d, internal_dim), ``dense_{index}_0/bias`` (internal_dim,), ``dense_{index}_1/kernel``
    (internal_dim, d), ``dense_{index}_1/bias`` (d,).  Kernels are glorot-uniform and both biases start at zero.  As in the
    reference, ``internal_dim`` goes through ``int()`` (a string width works, None raises) and ``index=None`` names the
    variables ``dense_None_0`` / ``dense_None_1``."""
    output_dim = int(input.shape[-1])
    internal_dim = int(internal_dim)
    zeros = lambda s: torch.zeros(s)
    with variable_scope(f"dense_{index}_0"):
        w0 = get_variable("kernel", (output_dim, internal_dim)); b0 = get_variable("bias", (internal_dim,), initializer=zeros)
    with variable_scope(f"dense_{index}_1"):
        w1 = get_variable("kernel", (internal_dim, output_dim)); b1 = get_variable("bias", (output_dim,), initializer=zeros)
    return autograd.residual_unit(input, w0, b0, w1, b1)


# --------------------------------------------------------------------------------------------------- AutoInt
def interacting_layer(input: torch.Tensor, att_embedding_size=None, head_num=None, index=None) -> torch.Tensor:
    """AutoInt interacting layer (Song et al., CIKM 2019, arXiv:1810.11921, eq. 5-8), one kernel each way: multi-head
    self-attention over the fields of ``input`` (B, F, d) with a residual projection and relu, -> (B, F, head_num *
    att_embedding_size).

    The reference tree has no AutoInt file, so the variable names are this project's choice: in the caller's scope, a scope
    ``interacting_layer_{index}`` holding ``query``, ``key``, ``value`` and ``res``, each (d, head_num *
    att_embedding_size) with the store's default glorot-uniform initializer; head h owns columns h * att_embedding_size ..
    (h + 1) * att_embedding_size - 1.  The widths go through ``int()`` (a string width works, None raises)."""
    d = int(input.shape[-1])
    dk, H = int(att_embedding_size), int(head_num)
    with variable_scope(f"interacting_layer_{index}"):
        wq, wk, wv, wr = (get_variable(n, (d, H * dk)) for n in ("query", "key", "value", "res"))
    return autograd.autoint_interacting(input, wq, wk, wv, wr, H, dk)


# --------------------------------------------------------------------------------------------------- MMoE
def mmoe_experts_gates(concat_all_input: torch.Tensor, num_experts, expert_hidden_units, num_tasks,
                       return_gates: bool = False):
    """MMoE experts, gates and gated sums -- MMOE/mmoe.py:207-236, one kernel each way: returns the ``num_tasks`` towers
    ``sum_e softmax_e(x . gate_t)[e] relu(x . expert_e + bias_e)`` as contiguous (B, expert_hidden_units) tensors, and with
    ``return_gates`` also the gate weights (the reference's ``gate_log``) as a list of (B, num_experts) tensors.

    Creates, in the caller's scope, the variables of the reference's ``tf.layers.dense`` calls: ``experts/expert_{i}/kernel``
    (d, expert_hidden_units) glorot-uniform and ``experts/expert_{i}/bias`` zeros for i < num_experts, then
    ``gates/gate_{i}/kernel`` (d, num_experts) glorot-uniform and no bias for i < num_tasks -- gates are named by task
    index, not by task name.  The three sizes go through ``int()``.  The variables are stacked into the packed (E,d,H),
    (E,H) and (T,d,E) layout of the kernels on every call; torch.stack routes the gradients back to each variable."""
    E, H, T = int(num_experts), int(expert_hidden_units), int(num_tasks)
    d = int(concat_all_input.shape[-1])
    zeros = lambda s: torch.zeros(s)
    kernels, biases, gate_kernels = [], [], []
    with variable_scope("experts"):
        for i in range(E):
            with variable_scope(f"expert_{i}"):
                kernels.append(get_variable("kernel", (d, H)))
                biases.append(get_variable("bias", (H,), initializer=zeros))
    with variable_scope("gates"):
        for i in range(T):
            with variable_scope(f"gate_{i}"):
                gate_kernels.append(get_variable("kernel", (d, E)))
    towers, gates = autograd.mmoe(concat_all_input, torch.stack(kernels), torch.stack(biases), torch.stack(gate_kernels))
    towers = list(towers.unbind(0))
    if return_gates:
        return towers, list(gates.unbind(0))
    return towers


# --------------------------------------------------------------------------------------------------- PLE
def _ple_sizes(task_names, num_experts_per_task, num_experts_in_shared, expert_hidden_units):
    task_names = list(task_names)
    n = [int(v) for v in num_experts_per_task]
    if len(task_names) != len(n):
        raise ValueError(f"task_names has {len(task_names)} entries but num_experts_per_task has {len(n)}: the all-gate "
                         "width and the task outputs depend on both")
    return task_names, n, int(num_experts_in_shared), int(expert_hidden_units)


def _expert(name, d, H, kernels, biases):
    with variable_scope(name):
        kernels.append(get_variable("kernel", (d, H)))
        biases.append(get_variable("bias", (H,), initializer=lambda s: torch.zeros(s)))


def _ple_call(x, task_expert_lists, shared, gate_kernels, n, S, extraction):
    """Stacks the variables into the packed layout ([task 0 .. task T-1, shared] experts, gate kernels by columns)."""
    kernels = [k for ks, _ in task_expert_lists for k in ks] + shared[0]
    biases = [b for _, bs in task_expert_lists for b in bs] + shared[1]
    return autograd.ple(x, torch.stack(kernels), torch.stack(biases), torch.cat(gate_kernels, dim=1), n, S, extraction)


def extraction_network(input: torch.Tensor, task_names, num_experts_per_task, num_experts_in_shared, expert_hidden_units,
                       name) -> torch.Tensor:
    """PLE extraction network -- same signature as PLE/extraction_network.py:4, one kernel each way: the sum of every
    task's gated output (over its own experts, then the shared ones) and the all-gate's output (over all experts), (B, H).

    Creates, in scope ``name``, the variables of the reference's ``tf.layers.dense`` calls in its order: the shared experts
    ``shared_expert_{i}``, then per task its experts ``task_specific_expert_{task}_{i}`` and its gate ``gate_{task}``
    (width n_t + S), then ``all_gate`` (width sum n_t + S).  Expert kernels are glorot-uniform with zero biases; gates have
    a glorot-uniform kernel and no bias.  The sizes go through ``int()``.  ``task_names`` and ``num_experts_per_task`` must
    have the same length (ValueError otherwise: the reference's zip would drop tasks and size its all-gate wrongly)."""
    task_names, n, S, H = _ple_sizes(task_names, num_experts_per_task, num_experts_in_shared, expert_hidden_units)
    d = int(input.shape[-1])
    shared, tasks, gates = ([], []), [], []
    with variable_scope(name):
        for i in range(S):
            _expert(f"shared_expert_{i}", d, H, *shared)
        for task, nt in zip(task_names, n):
            ks, bs = [], []
            for i in range(nt):
                _expert(f"task_specific_expert_{task}_{i}", d, H, ks, bs)
            tasks.append((ks, bs))
            with variable_scope(f"gate_{task}"):
                gates.append(get_variable("kernel", (d, nt + S)))
        with variable_scope("all_gate"):
            gates.append(get_variable("kernel", (d, sum(n) + S)))
    return _ple_call(input, tasks, shared, gates, n, S, True)[0]


def ple_final_experts_gates(input: torch.Tensor, task_names, num_experts_per_task, num_experts_in_shared,
                            expert_hidden_units, return_gates: bool = False):
    """PLE's last layer -- PLE/ple.py:185-226, one kernel each way: per task, the gated sum over its own experts and the
    shared ones, returned as T contiguous (B, H) tensors (the tower inputs), and with ``return_gates`` also each task's
    gate weights (B, n_t + S).

    Creates the reference's variables in its order: ``shared_experts_final/shared_expert_final_{i}``, then per task its
    experts ``task_specific_experts_final/task_specific_expert_final_{task}_{i}`` and its gate
    ``task_specific_experts_final/task_gate_final/gate_final_{task}``.  Initialisers, the int() sizes and the length check
    are those of extraction_network."""
    task_names, n, S, H = _ple_sizes(task_names, num_experts_per_task, num_experts_in_shared, expert_hidden_units)
    d = int(input.shape[-1])
    shared, tasks, gates = ([], []), [], []
    with variable_scope("shared_experts_final"):
        for i in range(S):
            _expert(f"shared_expert_final_{i}", d, H, *shared)
    with variable_scope("task_specific_experts_final"):
        for task, nt in zip(task_names, n):
            ks, bs = [], []
            for i in range(nt):
                _expert(f"task_specific_expert_final_{task}_{i}", d, H, ks, bs)
            tasks.append((ks, bs))
            with variable_scope("task_gate_final"), variable_scope(f"gate_final_{task}"):
                gates.append(get_variable("kernel", (d, nt + S)))
    out, p = _ple_call(input, tasks, shared, gates, n, S, False)
    out = list(out.unbind(0))
    if return_gates:
        return out, list(p.split([nt + S for nt in n], dim=1))
    return out


# --------------------------------------------------------------------------------------------------- DIN loss-side term
def mini_batch_aware_regularization(embedding_tensors, l2_lambda: float) -> torch.Tensor:
    """DIN/din.py:254-257 (SURVEY parity note 7): ``l2_lambda * tf.nn.l2_loss(concat(tensors, -1)) / batch`` -- an L2 on the
    looked-up ACTIVATIONS, so its gradient ``l2_lambda * e / B`` reaches the tables through the lookup backward
    (``d_tile`` of ctr_embed_fm2_bwd / ctr_bag_lookup_bwd) like any other upstream gradient.  Torch plumbing, no kernel."""
    x = torch.cat(list(embedding_tensors), dim=-1)
    return l2_lambda * 0.5 * x.pow(2).sum() / x.shape[0]


# --------------------------------------------------------------------------------------------------- FFM
def ffm_table_dim(num_fields: int, embedding_dim: int) -> int:
    """Row width of the id-major FFM table: (F-1)*K padded up to the next width the fused 128-bit gather takes (a power of
    two in 4..128) -- the reference's default config (7 fields, K = 8: 48 floats) becomes 64, the padding is zeros."""
    d = (num_fields - 1) * embedding_dim
    p = 4
    while p < d:
        p *= 2
    if p > 128:
        raise ValueError(f"(F-1)*embedding_dim = {d} exceeds the 128-float row of the fused lookup")
    return p


def ffm_second_order(tables: autograd.EmbeddingTables, ids: torch.Tensor, embedding_dim: int) -> torch.Tensor:
    """FFM/ffm.py:128-160 in two kernels: `tables` holds, per field, rows of (F-1)*K floats (zero padded to
    ``ffm_table_dim(F, K)``) -- the reference's ``{name}_embedding`` variable of shape (F-1, |V_i|, K) stored id-major
    (``EmbeddingTables([...], dim=ffm_table_dim(F, K))``; `ffm_table_from_reference` converts) -- looked up by the fused
    gather, then the field-aware pair sum.  Returns (B,1).  Single-valued fields only (the reference's mean-combined
    ``manual_tag_list`` bag is outside this entry point: look it up with ``ctr_bag_lookup_*`` per slot)."""
    B, F = ids.shape
    d = (F - 1) * embedding_dim
    if tables.dim != ffm_table_dim(F, embedding_dim):
        raise ValueError(f"tables.dim must be ffm_table_dim(F, K) = {ffm_table_dim(F, embedding_dim)}, got {tables.dim}")
    tile = autograd.lookup(tables, ids)                       # (B, F, padded (F-1)*K)
    if tables.dim != d:
        tile = tile[:, :, :d].contiguous()
    return autograd.ffm(tile.reshape(B, F, F - 1, embedding_dim))


def ffm_table_from_reference(embedding_variables) -> torch.Tensor:
    """[(F-1, |V_i|, K) per field] (the reference's variables, ffm.py:129-136) -> the (sum |V_i|, ffm_table_dim) id-major table."""
    F = embedding_variables[0].shape[0] + 1
    K = embedding_variables[0].shape[2]
    t = torch.cat([e.permute(1, 0, 2).reshape(e.shape[1], -1) for e in embedding_variables], dim=0)
    pad = ffm_table_dim(F, K) - t.shape[1]
    return (torch.nn.functional.pad(t, (0, pad)) if pad else t).contiguous()
