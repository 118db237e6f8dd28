"""The C-ABI shared library loads without a GPU and exports every symbol include/distegnn_b200.h
declares; the Python binding table covers them all; the host-only entry points work."""
import ctypes
import os
import re

from distegnn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols(header="distegnn_b200.h"):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"DISTEGNN_API\s+[\w\s\*]+?\b(distegnn_\w+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    syms = declared_symbols()
    for must in ["distegnn_build_csr", "distegnn_edge_layer_fwd", "distegnn_virtual_layer_fwd",
                 "distegnn_node_layer_fwd", "distegnn_virtual_update_fwd", "distegnn_embed_fwd",
                 "distegnn_param_layout", "distegnn_last_error", "distegnn_abi_version",
                 # SURVEY §8(b) minimum export set: the collective
                 "distegnn_comm_init", "distegnn_comm_connect", "distegnn_allreduce_packed", "distegnn_comm_destroy"]:
        assert must in syms
    # the production header holds production entry points only; cross-check twins live in the testing header
    assert not [s for s in syms if s.endswith(("_simt", "_tf32", "_t16", "_cs")) or "selftest" in s]


def test_testing_library_exports_every_twin():
    from tests import twin_backend
    lib = ctypes.CDLL(twin_backend.TESTING_LIB_PATH)
    twins = declared_symbols("distegnn_b200_testing.h")
    assert twins and set(twins) == set(twin_backend.TWIN_SIGNATURES)
    for name in twins:
        assert hasattr(lib, name), f"{name} declared in the testing header but not exported"
    prod = ctypes.CDLL(_lib.LIB_PATH)
    assert not [n for n in twins if hasattr(prod, n)], "twins leaked into the production library"


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in the header but not exported"


def test_python_binding_table_matches_header():
    bound = set(_lib.SIGNATURES) | {"distegnn_last_error"}
    assert bound == set(declared_symbols())


def test_host_only_entry_points():
    lib = _lib.load()
    assert lib.distegnn_abi_version() == 3 == _lib.ABI_VERSION
    offs, total = _lib.param_layout(2, 8, 2)
    assert total > 0 and offs["E_W1A"] == 0
    # error convention: negative code + message, ValueError on the Python side for bad arguments
    o = (ctypes.c_int64 * len(_lib.P_FIELDS))()
    t = ctypes.c_int64(0)
    rc = lib.distegnn_param_layout(2, 99, 0, o, ctypes.byref(t))
    assert rc == -1 and b"virtual_channels" in lib.distegnn_last_error()
    assert lib.distegnn_comm_handle_bytes() == 64
    assert lib.distegnn_allreduce_packed(None, None, 4, None) == -1 and b"null comm" in lib.distegnn_last_error()
    try:
        _lib.param_layout(2, 99, 0)
        assert False
    except ValueError:
        pass


def test_backend_has_every_method_the_host_code_calls():
    """Static guard (no GPU): every `be.<method>(` used by the host-side modules exists on the CUDA backend class and on
    the torch stand-in used by the CPU tests."""
    import os
    import re
    from distegnn_b200 import backend
    from tests.shadow_backend import ShadowBackend
    root = os.path.dirname(os.path.abspath(backend.__file__))
    used = set(re.findall(r"\bbe\.(\w+)\(", open(os.path.join(root, "fast_egnn.py")).read()))
    cls = [v for v in vars(backend).values() if isinstance(v, type) and v.__name__.endswith("Backend")][0]
    missing = sorted(m for m in used if not hasattr(cls, m))
    assert not missing, f"CudaBackend lacks {missing}"
    missing = sorted(m for m in used if not hasattr(ShadowBackend, m))
    assert not missing, f"ShadowBackend lacks {missing}"
