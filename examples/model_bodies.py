"""The bodies of the reference's model_fns between "inputs looked up" and "logit", rewritten on this repo's host API.

Each function follows its reference file line by line (cited); the interaction layers keep the reference's names, scopes and
signatures (recalgorithm_b200.layers), the lookup is the fused kernel (autograd.lookup / lookup_fm2), and the dense tail --
out of scope for the library (DESIGN.md section 7) -- is plain torch with variables created under the same TF names through
`dense()` below (glorot kernel, zero bias, like tf.layers.dense).  batch-norm / dropout / Dice of the tails are left out.

tests/test_gpu_model_bodies.py runs every body forward + backward once and checks that gradients reach the tables
(IndexedSlices) and every variable.
"""
from __future__ import annotations

import torch

from recalgorithm_b200 import autograd
from recalgorithm_b200 import feature_column as fc
from recalgorithm_b200 import layers as L


def dense(x: torch.Tensor, units: int, activation=None, use_bias: bool = True, name: str = "dense") -> torch.Tensor:
    """tf.layers.dense: variables <scope>/<name>/kernel (in, units), <scope>/<name>/bias (units,)."""
    with L.variable_scope(name):
        kernel = L.get_variable("kernel", (x.shape[-1], units))
        y = x @ kernel
        if use_bias:
            y = y + L.get_variable("bias", (units,), initializer=lambda s: torch.zeros(s))
    return activation(y) if activation is not None else y


def deepfm_logit(tables: autograd.EmbeddingTables, ids: torch.Tensor, fm_first_order_logit: torch.Tensor, hidden_units=(64, 32)):
    """DeepFM/deepfm.py:178-214.  fm_first_order_logit comes from feature_column.indicator_dense (deepfm.py:180-181)."""
    fields_embeddings, fm_second_order_logit = L.fm_second_order(tables, ids)            # :184-200, one kernel
    with L.variable_scope("fm_deep"):                                                      # :203-211
        net = fields_embeddings.reshape(ids.shape[0], -1)                                 # tf.concat(fields_embeddings, axis=1)
        for i, unit in enumerate(hidden_units):
            net = dense(net, unit, activation=torch.relu, name=f"dense_{i}" if i else "dense")
        deep_logit = dense(net, 1, name="deep_logit")
    return fm_first_order_logit + fm_second_order_logit + deep_logit                      # tf.add_n(...), :214


def dcn_logit(dense_input: torch.Tensor, category_input: torch.Tensor, num_cross_layer: int = 3, hidden_units=(64, 32)):
    """DCN/dcn.py:147-169.  category_input: (B, sum d) flat output of the lookup."""
    concat_all = torch.cat([dense_input, category_input], dim=-1)                         # :155
    with L.variable_scope("cross_part"):                                                  # :157-160
        cross_vec = concat_all
        for i in range(num_cross_layer):
            cross_vec = L.cross_layer(x0=concat_all, xl=cross_vec, index=i)
    with L.variable_scope("dnn_part"):                                                    # :162-165
        dnn_vec = concat_all
        for i, unit in enumerate(hidden_units):
            dnn_vec = dense(dnn_vec, unit, activation=torch.relu, name=f"dnn_dense_{i}")
    with L.variable_scope("output_part"):                                                 # :167-169
        return dense(torch.cat([cross_vec, dnn_vec], dim=-1), 1)


def xdeepfm_logit(dense_input: torch.Tensor, x0: torch.Tensor, cin_layer_feature_maps=("16", "16"), hidden_units=(64, 32)):
    """xDeepFM/xdeepfm.py:152-185.  x0: (B, m, D) tile; layer widths arrive as strings like in the reference (:253)."""
    B = x0.shape[0]
    category_input = x0.reshape(B, -1)
    with L.variable_scope("linear_part"):                                                 # :160-163
        linear_vec = torch.cat([dense_input, category_input], dim=-1)
        linear_logit = dense(linear_vec, 1)
    with L.variable_scope("cin_part"):                                                    # :166-175
        xk, p_plus = x0, []
        for i, features_map_num in enumerate(cin_layer_feature_maps):
            xk, pooled = L.cin_layer(x0, xk, features_map_num, i + 1, return_pooled=True)   # pooled = reduce_sum(x, axis=-1), fused
            p_plus.append(pooled)
        cin_logit = dense(torch.cat(p_plus, dim=-1), 1, use_bias=False)
    with L.variable_scope("dnn_part"):                                                    # :178-182
        dnn_vec = linear_vec
        for i, unit in enumerate(hidden_units):
            dnn_vec = dense(dnn_vec, unit, activation=torch.relu, name=f"dense_{i}")
        dnn_logit = dense(dnn_vec, 1, use_bias=False, name="dnn_logit")
    return linear_logit + cin_logit + dnn_logit                                           # :185


def din_logit(dense_input, category_input, target_input, sequnence_input, sequnence_length, use_softmax=False, hidden_units=(64, 32)):
    """DIN/din.py:199-238 (Dice / PReLU / batch-norm of the fcn tail left out)."""
    with L.variable_scope("attention_part"):                                              # :216-218
        attention_output = L.din_attention(target_input, sequnence_input, sequnence_length, is_softmax=use_softmax)
    concat_all = torch.cat([dense_input, category_input, target_input, attention_output], dim=-1)   # :221
    with L.variable_scope("fcn"):                                                         # :224-238
        net = concat_all
        for i, unit in enumerate(hidden_units):
            net = torch.relu(dense(net, unit, name=f"dense_{i}" if i else "dense"))
        return dense(net, 1, name="logit"), attention_output


def fibinet_logit(dense_input, category_input, embedding_dim: int, reduction_ratio: int = 2, bilinear_interaction_type: str = "all",
                  hidden_units=(64, 32)):
    """FiBiNET/fibinet.py:156-199.  category_input: (B, F, K)."""
    with L.variable_scope("linear_part"):                                                 # :166-168
        linear_logit = dense(dense_input, 1)
    with L.variable_scope("senet_part"):                                                  # :171-174
        senet_output = L.senet(category_input, embedding_dim=embedding_dim, reduction_ratio=reduction_ratio)
    with L.variable_scope("bilinear_interaction_part"):                                   # :177-187
        bi_orginal = L.bilinear_interaction_layer(category_input, embedding_dim=embedding_dim, type=bilinear_interaction_type, name="orginal")
        bi_senet = L.bilinear_interaction_layer(senet_output, embedding_dim=embedding_dim, type=bilinear_interaction_type, name="senet")
        bi_total = torch.cat([bi_orginal, bi_senet], dim=-1).reshape(category_input.shape[0], -1)
    with L.variable_scope("dnn_part"):                                                    # :189-197
        net = bi_total
        for i, unit in enumerate(hidden_units):
            net = dense(net, unit, activation=torch.relu, name=f"dense_{i}" if i else "dense")
        fibinet = dense(net, 1, name="logit")
    return linear_logit + fibinet                                                         # :199


def pnn_logit(fields_embeddings, num_fields: int, embedding_dim: int, output_dimension: int = 1024, product_method: str = "IPNN",
              hidden_units=(64, 32), weight_regularizer: float = 0.0):
    """PNN/pnn.py:125-193.  fields_embeddings: (B, F*K) concatenated input_layer outputs (or the (B, F, K) tile).  Returns
    (logit, regularization_loss): the reference's l2_regularizer(scale) on linear_w and the product weight (:137,150,164)
    contributes scale * sum(w**2) / 2 per weight to REGULARIZATION_LOSSES when scale > 0, and nothing at the default 0.0."""
    product_final = L.pnn_product_layer(fields_embeddings, num_fields, embedding_dim, output_dimension,
                                        product_method=product_method)                        # :125-181, one kernel
    with L.variable_scope("fcn"):                                                         # :184-193 (TF names dense, dense_1, ...)
        net = product_final
        for i, unit in enumerate(hidden_units):
            net = dense(net, unit, activation=torch.relu, name=f"dense_{i}" if i else "dense")
        logit = dense(net, 1, name=f"dense_{len(hidden_units)}" if hidden_units else "dense")
    reg = logit.new_zeros(())
    if weight_regularizer > 0:
        store = L.default_store()
        prod = "product_part/inner_product_w" if product_method == "IPNN" else "product_part/outer_product_w"
        for name in ("linear_part/linear_w", prod):
            reg = reg + weight_regularizer * 0.5 * store.vars[store.full_name(name)].pow(2).sum()
    return logit, reg


def dien_logit(dense_input, category_input, target_input, sequnence_input, sequnence_length, gru_output_units=8,
               custom_gru_type: str = "AGRU", hidden_units=(64, 32), use_auxiliary_loss: bool = False,
               neg_sequnence_input=None, negative_sample_number=3):
    """DIEN/dien.py:179-254 (Dice / PReLU / batch-norm of the fcn tail left out, as for DIN).  Returns (logit,
    attention_scores (B, T, 1)); with ``use_auxiliary_loss`` (:256-300), (logit, attention_scores, aux_loss), where
    aux_loss is the paper's sign (the negative of the reference's) and the training loss is ce + aux_loss (:316-317).
    neg_sequnence_input (B, (T-1)*negative_sample_number, na) are the caller's negatives, looked up like the history."""
    if use_auxiliary_loss:
        na, nh = int(sequnence_input.shape[-1]), int(gru_output_units)
        with L.variable_scope("aux_loss"):                                                # :264, 268
            w_aux = L.get_variable("aux_project_matrix", (na, nh))
    with L.variable_scope("seq_encoder"):                                                 # :199-229, one kernel each way
        if use_auxiliary_loss:
            final_state, attention_scores, aux_loss = L.dien_interest_evolution_aux(
                sequnence_input, sequnence_length, target_input, neg_sequnence_input, w_aux, gru_output_units,
                custom_gru_type=custom_gru_type, negative_sample_number=negative_sample_number, return_attention_scores=True)
        else:
            final_state, attention_scores = L.dien_interest_evolution(sequnence_input, sequnence_length, target_input,
                                                                      gru_output_units, custom_gru_type=custom_gru_type,
                                                                      return_attention_scores=True)
        concat_all = torch.cat([dense_input, category_input, target_input, final_state], dim=-1)   # :237
        with L.variable_scope("fcn"):                                                     # :240-254 (TF names dense, dense_1, ...)
            net = concat_all
            for i, unit in enumerate(hidden_units):
                net = dense(net, unit, name=f"dense_{i}" if i else "dense")
            logit = dense(net, 1, name=f"dense_{len(hidden_units)}" if hidden_units else "dense")
    if use_auxiliary_loss:
        return logit, attention_scores, aux_loss
    return logit, attention_scores


def deepcrossing_logit(dense_input, category_input, residual_internal_dim=256, residual_network_num=2):
    """DeepCrossing/deepcrossing.py:152-159: the residual units over concat_all in scope residual_module, then dense(net, 1)
    outside it.  The reference's best result.md row is residual_internal_dim 256 with 2 units."""
    concat_all = torch.cat([dense_input, category_input], dim=-1)                         # :152
    with L.variable_scope("residual_module"):                                             # :154-157, one kernel each way per unit
        net = concat_all
        for i in range(residual_network_num):
            net = L.residual_unit(net, residual_internal_dim, index=i)
    return dense(net, 1)                                                                  # :159


def autoint_logit(dense_input, fields_embeddings, att_layer_num=3, att_head_num=2, att_embedding_size=8):
    """AutoInt (Song et al., CIKM 2019, arXiv:1810.11921; the reference README lists it as a to-do, so there is no reference
    file to follow): each dense feature m becomes the field x_m v_m with v = `dense_embedding` (n_dense, d), concatenated
    with the categorical field embeddings (B, F, d); then att_layer_num interacting layers (each opens its own
    interacting_layer_{i} scope), a flatten and dense(1)."""
    v = L.get_variable("dense_embedding", (dense_input.shape[-1], fields_embeddings.shape[-1]))
    net = torch.cat([dense_input.unsqueeze(-1) * v, fields_embeddings], dim=1)
    for i in range(att_layer_num):                                                        # one kernel each way per layer
        net = L.interacting_layer(net, att_embedding_size, att_head_num, index=i)
    return dense(net.reshape(net.shape[0], -1), 1)


def flen_logit(tables: autograd.EmbeddingTables, ids: torch.Tensor, field_groups, first_order_logit: torch.Tensor,
               hidden_units=(64, 32)):
    """FLEN (Chen et al., arXiv:1911.04690; the reference README lists it as a to-do, so there is no reference file to
    follow): the fused lookup and field-wise bi-interaction h (B, D) in one kernel each way, a DNN over the flattened
    embeddings, dense(concat([h, dnn]), 1), plus the first-order logit (feature_column.indicator_dense, as for DeepFM).
    The paper's DiceFactor dropout is left out."""
    fields_embeddings, h = L.field_wise_bi_interaction_lookup(tables, ids, field_groups)
    with L.variable_scope("dnn_part"):
        net = fields_embeddings.reshape(ids.shape[0], -1)
        for i, unit in enumerate(hidden_units):
            net = dense(net, unit, activation=torch.relu, name=f"dense_{i}")
    with L.variable_scope("output_part"):
        return dense(torch.cat([h, net], dim=-1), 1) + first_order_logit


def mmoe_logits(dense_input, category_input, labels, task_names=("read_comment", "like", "click_avatar"), num_experts=3,
                expert_hidden_units=512, hidden_units=(512, 256, 128)):
    """MMOE/mmoe.py:205-263: experts, gates and gated sums in one kernel each way, then one tower_layer per task
    (MMOE/tower_layer.py: relu dense stack, tower_{task}_logit; its batch norm and dropout left out) in scope tower, and the
    sum of the per-task mean sigmoid cross-entropies.  labels maps task name -> (B, 1).  Returns (logits, total_loss)."""
    concat_all_input = torch.cat([dense_input, category_input], dim=-1)                   # :205
    towers = L.mmoe_experts_gates(concat_all_input, num_experts, expert_hidden_units, len(task_names))   # :208-236
    logits, n_dense = [], 0
    with L.variable_scope("tower"):
        for x, task_name in zip(towers, task_names):                                      # :241-246
            net = x
            for unit in hidden_units:                                                     # TF uniquifies dense, dense_1, ...
                net = dense(net, unit, activation=torch.relu, name=f"dense_{n_dense}" if n_dense else "dense")
                n_dense += 1
            logits.append(dense(net, 1, name=f"tower_{task_name}_logit"))
    losses = [torch.nn.functional.binary_cross_entropy_with_logits(logit, labels[task_name])          # :261-263
              for logit, task_name in zip(logits, task_names)]
    return logits, sum(losses[1:], losses[0])


def ple_logits(dense_input, category_input, labels, task_names=("read_comment", "like", "click_avatar"),
               num_extract_network=1, num_experts_per_task=(5, 5, 5), num_experts_in_shared=10, expert_hidden_units=256,
               hidden_units=(512, 256, 128)):
    """PLE/ple.py:160-254: num_extract_network extraction networks, then the final experts and gates, each in one kernel
    each way; one tower_layer per task (MMOE/tower_layer.py, which ple.py imports: relu dense stack, tower_{task}_logit; its batch norm and
    dropout left out) in scope tower, and the sum of the per-task mean sigmoid cross-entropies.  labels maps task name ->
    (B, 1).  Returns (logits, total_loss)."""
    net = torch.cat([dense_input, category_input], dim=-1)                                # :169
    for i in range(num_extract_network):                                                  # :172-180
        net = L.extraction_network(net, task_names, num_experts_per_task, num_experts_in_shared, expert_hidden_units,
                                   f"extract_network_{i}")
    towers = L.ple_final_experts_gates(net, task_names, num_experts_per_task, num_experts_in_shared,
                                       expert_hidden_units)                               # :185-226
    logits, n_dense = [], 0
    with L.variable_scope("tower"):
        for x, task_name in zip(towers, task_names):                                      # :229-235
            for unit in hidden_units:                                                     # TF uniquifies dense, dense_1, ...
                x = dense(x, unit, activation=torch.relu, name=f"dense_{n_dense}" if n_dense else "dense")
                n_dense += 1
            logits.append(dense(x, 1, name=f"tower_{task_name}_logit"))
    losses = [torch.nn.functional.binary_cross_entropy_with_logits(logit, labels[task_name])          # :251-254
              for logit, task_name in zip(logits, task_names)]
    return logits, sum(losses[1:], losses[0])


def wide_and_deep_logit(features, wide_part_feature_columns, deep_part_feature_columns, hidden_units=(512, 256, 128),
                        ctx=None):
    """WideAndDeep/wide_and_deep.py:207-225.  The wide part is the crossed indicator columns' dense(1) (one hashed gather-sum
    kernel per column each way) in scope wide_part; its variables are what optim.Ftrl trains (:254-257).  The deep part is
    input_layer plus the relu dense stack in scope deep_part (its dropout and batch norm left out); the embedding tables'
    IndexedSlices gradients go to ctx (feature_column.LookupContext)."""
    with L.variable_scope("wide_part", reuse=L.AUTO_REUSE):                               # :208-210
        wide_logit = fc.indicator_dense(features, wide_part_feature_columns, units=1, name="wide_part_variables")
    with L.variable_scope("deep_part"):                                                   # :213-222 (TF names dense, dense_1, ...)
        net = fc.input_layer(features, deep_part_feature_columns, ctx=ctx)
        for i, unit in enumerate(hidden_units):
            net = dense(net, unit, activation=torch.relu, name=f"dense_{i}" if i else "dense")
        deep_logit = dense(net, 1, name=f"dense_{len(hidden_units)}" if hidden_units else "dense")
    return wide_logit + deep_logit                                                        # :225
