"""GPU parity of the Wide & Deep wide part on the fixtures executed from the reference's own lines (tests/golden/wide):
feature_column.indicator_dense over the crossed column (ctr_crossed_indicator_fwd / _bwd) with the run's kernel and bias
injected, against its literal-multi-hot logits and dense(1) gradients; and ctr_ftrl_apply on buffers at any float offset.
Sorts after test_gpu_tc_variants.py, like test_gpu_wide_ftrl.py."""
import glob
import os

import numpy as np
import pytest
import torch

import _wide_fixture as WF
from _util import TOL, assert_close, dev

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(WF.G, "*.npz")))


@pytest.mark.parametrize("name", FIXTURES)
def test_wide_layer_on_fixture(name):
    from recalgorithm_b200 import feature_column as fc, layers as L
    z, col, features, kernel = WF.load(name)
    st = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    try:
        st.assign({"wide_part/wide_part_variables/kernel": kernel, "wide_part/wide_part_variables/bias": z["bias"]})
        with L.variable_scope("wide_part", reuse=L.AUTO_REUSE):
            logit = fc.indicator_dense(features, [col], units=1, name="wide_part_variables")
        assert set(st.vars) == {"wide_part/wide_part_variables/kernel", "wide_part/wide_part_variables/bias"}
        assert_close(logit, z["wide_logit_f64"], TOL, f"{name}: wide logit")
        logit.backward(dev(z["g"]).reshape(-1, 1))
        torch.cuda.synchronize()
        k, b = st.vars["wide_part/wide_part_variables/kernel"], st.vars["wide_part/wide_part_variables/bias"]
        assert np.array_equal(k.grad.reshape(-1).cpu().numpy(), z["d_kernel_f64"].astype(np.float32)), f"{name}: d_kernel"
        assert float(b.grad) == float(np.sum(z["g"], dtype=np.float64))
        if name.endswith("no_tags"):
            assert torch.all(logit.detach() == float(z["bias"][0]))
    finally:
        L.set_default_store(L.VariableStore())


@pytest.mark.parametrize("n", [1, 3, 5, 1003])
@pytest.mark.parametrize("offsets", [(0, 0, 0, 0), (1, 1, 1, 1), (3, 3, 3, 3), (0, 1, 2, 3), (2, 0, 2, 1)])
def test_ftrl_on_views_at_any_float_offset(n, offsets):
    """ctr_ftrl_apply on views that start 0-3 floats past a 16-byte boundary, with shared and with differing offsets, against
    the float64 dense ApplyFtrl; the elements around each view stay untouched."""
    import _wide_ref as R
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(n + 10 * sum(offsets))
    init = [rng.uniform(-0.05, 0.05, n), np.full(n, 0.1) + rng.uniform(0, 0.5, n), rng.uniform(-1, 1, n), rng.standard_normal(n)]
    bases, views = [], []
    for o, a in zip(offsets, init):
        base = torch.full((n + 8,), 7.0, device="cuda")
        base[o:o + n] = dev(a.astype(np.float32))
        bases.append(base)
        views.append(base[o:o + n])
    for p, l1, l2 in ((-0.5, 0.0, 0.0), (-0.3, 0.01, 0.5)):
        want = R.ftrl(*(v.cpu().double().numpy() for v in views), 0.05, p, l1, l2)
        if l1 > 0 and np.any(np.abs(np.abs(want[2]) - l1) <= 1e-5 * l1):
            continue
        ops.ftrl_apply(views[0], views[1], views[2], views[3], 0.05, p, l1, l2)
        torch.cuda.synchronize()
        for got, w, what in zip(views[:3], want, ("var", "accum", "linear")):
            assert_close(got, w, TOL, f"n={n} offsets={offsets} p={p} {what}")
    for o, base in zip(offsets, bases):
        outside = torch.cat([base[:o], base[o + n:]])
        assert torch.all(outside == 7.0)
