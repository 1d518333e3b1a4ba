"""CPU tests of the PLE host layers (layers.extraction_network, layers.ple_final_experts_gates) with the launch stubbed:
variable names, shapes and initialisers, the packed layout handed to the kernels, and the task-count check."""
import math

import pytest
import torch

from recalgorithm_b200 import autograd
from recalgorithm_b200 import layers as L

TASKS = ("read_comment", "like", "click_avatar")


@pytest.fixture
def captured(monkeypatch):
    calls = []

    def fake(x, we, be, wg, n, S, extraction):
        calls.append(dict(x=x, we=we, be=be, wg=wg, n=tuple(n), S=S, extraction=extraction))
        B, H = x.shape[0], we.shape[2]
        return (torch.zeros((B, H)) if extraction else torch.zeros((len(n), B, H))), torch.zeros((B, wg.shape[1]))

    monkeypatch.setattr(autograd, "ple", fake)
    L.set_default_store(L.VariableStore(device="cpu", seed=0))
    return calls


def _glorot(v, fan_in, fan_out):
    m = float(v.detach().abs().max())
    return 0 < m <= math.sqrt(6.0 / (fan_in + fan_out))


def test_extraction_network_variables_and_packing(captured):
    x = torch.randn(4, 82)
    out = L.extraction_network(x, TASKS, [5, "5", 5.0], "10", 256, "extract_network_0")
    assert out.shape == (4, 256)
    store = L.default_store()
    p = "extract_network_0/"
    want = ([f"{p}shared_expert_{i}/{v}" for i in range(10) for v in ("kernel", "bias")] +
            [n for t in TASKS for n in [f"{p}task_specific_expert_{t}_{i}/{v}" for i in range(5) for v in ("kernel", "bias")]
             + [f"{p}gate_{t}/kernel"]] + [f"{p}all_gate/kernel"])
    assert list(store.vars) == want
    for name, v in store.vars.items():
        if name.endswith("bias"):
            assert v.shape == (256,) and torch.count_nonzero(v) == 0, name
        elif "expert" in name:
            assert v.shape == (82, 256) and _glorot(v, 82, 256), name
    assert store.vars[f"{p}gate_like/kernel"].shape == (82, 15)
    assert store.vars[f"{p}all_gate/kernel"].shape == (82, 25)
    (c,) = captured
    assert c["n"] == (5, 5, 5) and c["S"] == 10 and c["extraction"] is True
    assert c["we"].shape == (25, 82, 256) and c["be"].shape == (25, 256) and c["wg"].shape == (82, 70)
    # packed order: task experts in task order, then the shared experts; gates by columns, all_gate last
    assert torch.equal(c["we"][0], store.vars[f"{p}task_specific_expert_read_comment_0/kernel"])
    assert torch.equal(c["we"][14], store.vars[f"{p}task_specific_expert_click_avatar_4/kernel"])
    assert torch.equal(c["we"][15], store.vars[f"{p}shared_expert_0/kernel"])
    assert torch.equal(c["wg"][:, 15:30], store.vars[f"{p}gate_like/kernel"])
    assert torch.equal(c["wg"][:, 45:], store.vars[f"{p}all_gate/kernel"])


def test_final_layer_variables_and_outputs(captured):
    x = torch.randn(3, 256)
    outs, gates = L.ple_final_experts_gates(x, TASKS[:2], [2, 1], 1, 7, return_gates=True)
    assert len(outs) == 2 and all(o.shape == (3, 7) and o.is_contiguous() for o in outs)
    assert [tuple(g.shape) for g in gates] == [(3, 3), (3, 2)]
    want = (["shared_experts_final/shared_expert_final_0/kernel", "shared_experts_final/shared_expert_final_0/bias"] +
            [f"task_specific_experts_final/task_specific_expert_final_read_comment_{i}/{v}" for i in range(2)
             for v in ("kernel", "bias")] +
            ["task_specific_experts_final/task_gate_final/gate_final_read_comment/kernel",
             "task_specific_experts_final/task_specific_expert_final_like_0/kernel",
             "task_specific_experts_final/task_specific_expert_final_like_0/bias",
             "task_specific_experts_final/task_gate_final/gate_final_like/kernel"])
    assert list(L.default_store().vars) == want
    (c,) = captured
    assert c["extraction"] is False and c["we"].shape == (4, 256, 7) and c["wg"].shape == (256, 5)
    # a second call reuses the variables
    L.ple_final_experts_gates(x, TASKS[:2], [2, 1], 1, 7)
    assert len(L.default_store().vars) == len(want)


@pytest.mark.parametrize("layer", ["extraction", "final"])
def test_task_count_mismatch_is_refused(captured, layer):
    x = torch.randn(2, 8)
    with pytest.raises(ValueError, match="num_experts_per_task"):
        if layer == "extraction":
            L.extraction_network(x, TASKS, [1, 1], 1, 4, "n")
        else:
            L.ple_final_experts_gates(x, TASKS[:1], [1, 1], 1, 4)
    assert not captured and not L.default_store().vars
