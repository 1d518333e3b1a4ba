"""recalgorithm_b200 -- Hopper-native (sm_90a, H100) hot path of tangxyw/RecAlgorithm.

Only the path named in BASELINE.json lives here: the per-field embedding lookup and the
feature-interaction layers (FM2, cross, CIN, DIN attention, SENET/bilinear), as hand-written CUDA
behind a C ABI (include/ctr_b200.h) with a Python host side that mirrors the reference's own
layer signatures (recalgorithm_b200.layers); plus the steps either side of it (SURVEY 8f): the native feeder
(io.native / input_fn, include/ctr_feed.h) and Adam on the IndexedSlices (optim).
"""
from . import _lib  # noqa: F401

__all__ = ["_lib", "ops", "autograd", "layers", "feature_column", "sharded", "optim", "input_fn", "io", "build"]
