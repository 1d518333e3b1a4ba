"""CPU tests: the C-ABI library loads and exports exactly what include/ctr_b200.h declares."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    hdr = open(os.path.join(ROOT, "include", "ctr_b200.h")).read()
    return set(re.findall(r"\b(ctr_[a-z0-9_]+)\s*\(", hdr))


def test_library_exports_every_declared_symbol():
    from recalgorithm_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    handle = _lib.lib()                         # raises AttributeError if a declared symbol is missing
    declared = header_symbols()
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (ctr_[a-z0-9_]+)", out))
    assert declared <= exported, declared - exported
    assert handle.ctr_version() == 1


def test_argument_validation_happens_before_any_launch():
    """Bad arguments are rejected on the host with an error string (no GPU needed, no compute call)."""
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    assert h.ctr_embed_fm2_fwd(None, None, None, 1, 1, 3, None, None, None) == _lib.CTR_ERR_UNSUPPORTED
    assert b"D=3" in h.ctr_last_error()
    assert h.ctr_cross_fwd(None, None, None, None, 4, 0, 1, None, None) == _lib.CTR_ERR_INVALID_ARG
    with pytest.raises(_lib.CtrInvalidArgument):
        _lib.check(h.ctr_cross_fwd(None, None, None, None, 4, 8, 99, None, None))


def test_no_cpu_fallback():
    """The product path refuses CPU tensors instead of silently computing on the host."""
    import torch
    from recalgorithm_b200 import ops
    t = torch.zeros((4, 8))
    with pytest.raises(RuntimeError):
        ops.embed_fm2_fwd(t, torch.tensor([0, 4]), torch.zeros((2, 1), dtype=torch.int64))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "recalgorithm_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f


def test_every_compute_entry_rejects_null_pointers_with_an_error_string():
    """All-NULL pointers with plausible and with zero sizes: every kernel entry point returns a negative code and explains
    itself through ctr_last_error() -- no launch, no crash (this runs without a GPU)."""
    import ctypes
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    helpers = {"ctr_version", "ctr_last_error", "ctr_kernel_launches", "ctr_device_info", "ctr_enable_peer_access",
               "ctr_bilinear_set_rr", "ctr_cin_fwd_workspace_bytes", "ctr_cin_bwd_workspace_bytes",
               "ctr_bst_param_count", "ctr_peer_free", "ctr_ipc_close", "ctr_vmm_free", "ctr_vmm_alloc", "ctr_vmm_import",
               "ctr_vmm_granularity"}
    checked = 0
    for name, (res, args) in sorted(_lib.SIGNATURES.items()):
        if name in helpers:
            continue
        for size in (4, 0):
            vals = []
            for a in args:
                if a in (ctypes.c_float, ctypes.c_double):
                    vals.append(0.0)
                elif a in (ctypes.c_int, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_longlong):
                    vals.append(size)
                else:
                    vals.append(None)                                 # every pointer (and stream) argument
            rc = getattr(h, name)(*vals)
            assert isinstance(rc, int) and rc < 0, (name, size, rc)
            assert rc in (_lib.CTR_ERR_INVALID_ARG, _lib.CTR_ERR_UNSUPPORTED), (name, size, rc)
            assert h.ctr_last_error().startswith(name.encode()), (name, h.ctr_last_error())
            checked += 1
    assert checked >= 2 * 45                                          # 48 compute entry points today


@pytest.mark.parametrize("header", ["ctr_b200.h", "ctr_feed.h"])
def test_public_headers_are_plain_c_and_cxx(header):
    """The drop-in boundary is a C ABI: both headers must compile on their own as strict C99 and as C++17 (extern "C")."""
    path = os.path.join(ROOT, "include", header)
    for cmd in (["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", path],
                ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", path]):
        out = subprocess.run(cmd, capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
    src = open(path).read()
    assert 'extern "C"' in src and "#ifdef __cplusplus" in src and "torch" not in src.lower().replace("pytorch", "")
