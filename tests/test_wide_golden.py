"""CPU tests of the Wide & Deep wide part against the fixtures executed from the reference's own lines
(tools/make_golden_wide.py over WideAndDeep/wide_and_deep.py:121-122,208-210): the fixture digests, the regenerated kernel,
the column name, and the NumPy restatement (tests/_wide_ref.py) fed through the host layer's key block
(feature_column.crossed_ragged_ids) against the literal multi-hot logits and dense(1) gradients."""
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import _wide_fixture as WF
import _wide_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(WF.G, "*.npz")))


def test_fixtures_present():
    assert FIXTURES == ["wide_B16", "wide_B64", "wide_B8_no_tags"]


@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_equals_reference_run(name):
    from recalgorithm_b200 import feature_column as fc
    z, col, features, kernel = WF.load(name)
    assert col.name == str(z["column_name"]) == "manual_tag_list_X_userid_indicator"
    values, offsets = fc.crossed_ragged_ids(features, col.categorical_column)
    nb = int(z["hash_bucket_size"])
    cr = R.crossed_ids(values, offsets, nb)
    got = R.wide_fwd(cr, kernel.astype(np.float64), float(z["bias"][0]))
    assert np.array_equal(got, z["wide_logit_f64"])                   # multiples of 2^-12: every sum is exact
    assert np.abs(z["wide_logit_f32"] - got).max() <= 1e-6 * max(1.0, np.abs(got).max())
    dk, db = R.wide_bwd(cr, z["g"], nb)
    assert np.array_equal(dk, z["d_kernel_f64"]) and db == float(np.sum(z["g"], dtype=np.float64))


def test_no_tags_fixture_is_the_bias():
    """manual_tag_list parsed empty (parity note 8): no sample has a cross, the reference's logit is the bias and the kernel
    gradient is zero."""
    z = np.load(os.path.join(WF.G, "wide_B8_no_tags.npz"), allow_pickle=False)
    assert z["manual_tag_list_offsets"][-1] == 0
    assert np.all(z["wide_logit_f32"] == z["bias"][0]) and not z["d_kernel_f64"].any()


def _digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def test_fixtures_match_reference_digests(tmp_path):
    """Every array of every fixture is bit-identical to the recorded run over the reference.  With RECALG_REFERENCE set to a
    reference checkout (the `algorithm` directory), the generator re-runs into a temporary directory and must reproduce
    the same digests."""
    want = json.load(open(os.path.join(WF.G, "reference_digests.json")))
    assert sorted(want) == sorted(n + ".npz" for n in FIXTURES)
    for name in want:
        with np.load(os.path.join(WF.G, name), allow_pickle=False) as z:
            assert {k: _digest(z[k]) for k in z.files} == want[name], name
    ref = os.environ.get("RECALG_REFERENCE")
    if not ref:
        return
    code = ("import sys, json; sys.path.insert(0, 'tools'); import make_golden_wide as m; "
            f"print(json.dumps(m.gen_wide({str(tmp_path)!r})))")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr
    assert json.loads(out.stdout.strip().splitlines()[-1]) == want


def test_crossed_column_hash_key_zero_is_the_default():
    """sparse_cross_hashed uses `hash_key if hash_key else _DEFAULT_HASH_KEY`: 0 and None both give 0xDECAFCAFFE."""
    from recalgorithm_b200 import feature_column as fc
    a = fc.categorical_column_with_vocabulary_file("a", [b"x"])
    b = fc.categorical_column_with_vocabulary_file("b", [b"y"])
    assert fc.crossed_column([a, b], 10, hash_key=0).hash_key == 0xDECAFCAFFE
    assert fc.crossed_column([a, b], 10).hash_key == 0xDECAFCAFFE
    assert fc.crossed_column([a, b], 10, hash_key=3).hash_key == 3
