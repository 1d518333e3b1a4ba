"""Loads a Wide & Deep wide-part fixture (tests/golden/wide, written by tools/make_golden_wide.py) as the host layer takes it:
the two categorical columns over the fixture's vocabularies, the crossed indicator column, the parsed-features dict, and the
injected kernel regenerated from its seed."""
import hashlib
import os

import numpy as np

import _wide_ref as R

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide")


def load(name):
    from recalgorithm_b200 import feature_column as fc
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    userid = fc.categorical_column_with_vocabulary_file("userid", list(z["userid_vocab"]))
    tags = fc.categorical_column_with_vocabulary_file("manual_tag_list", list(z["manual_tag_list_vocab"]))
    col = fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=int(z["hash_bucket_size"])))
    features = {k: (list(z[k + "_values"]), z[k + "_offsets"]) for k in ("userid", "manual_tag_list")}
    nb = int(z["hash_bucket_size"])
    kernel = R.fixture_kernel(nb, int(z["kernel_seed"])).reshape(nb, 1)
    assert hashlib.sha256(kernel.tobytes()).hexdigest() == str(z["kernel_sha256"]), "regenerated kernel differs from the run's"
    return z, col, features, kernel
