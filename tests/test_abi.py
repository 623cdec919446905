"""C-ABI boundary checks that need no GPU: the library builds / loads, exports exactly what
include/aurora_b200.h declares, and refuses to work without a device (no CPU fallback)."""

import ctypes as C
import os
import re

import numpy as np
import pytest

from aurora_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "aurora_b200.h")


@pytest.fixture(scope="module")
def lib():
    from aurora_b200.build import build_native

    build_native()          # nvcc cross-compiles for sm_90a without a GPU
    return N.load()


def _declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(aur_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported(lib):
    declared = _declared_symbols()
    assert len(declared) >= 15
    assert sorted(N.EXPORTS) == declared, "aurora_b200/_native.py:EXPORTS and include/aurora_b200.h disagree"
    raw = C.CDLL(N.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), f"{name} declared in the header but not exported by the .so"


def test_abi_version_3_and_error_string(lib):
    """Version 3: aur_stats grew by last_candidates / last_candidates_max, so a caller built against version 2 passes a
    struct the library would write past.  The library, the header and the ctypes binding must agree on it."""
    declared = int(re.search(r"#define AUR_ABI_VERSION (\d+)", open(HEADER).read()).group(1))
    assert lib.aur_abi_version() == N.ABI_VERSION == declared == 3
    assert isinstance(lib.aur_last_error(), bytes)


def _header_struct_fields(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, flags=re.S).group(1)
    ctypes_of = {"int64_t": C.c_int64, "int32_t": C.c_int32, "float": C.c_float, "double": C.c_double}
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(nm.strip(), ctypes_of[ctype]) for nm in names.split(",")]
    return fields


def test_stats_struct_matches_the_header():
    """aur_stats as the header declares it, field by field (ABI 3 added last_candidates / last_candidates_max): the
    ctypes mirror must agree in names, types and therefore offsets, or every stats read is garbage."""
    assert N.AurStats._fields_ == _header_struct_fields("aur_stats")
    assert N.AurStats.last_candidates.offset == 56 and N.AurStats.last_candidates_max.offset == 64
    assert C.sizeof(N.AurStats) == 72


def test_stats_without_a_search_report_no_candidates(lib):
    """aur_get_stats rejects a null index; the new fields exist and start at zero in a zeroed struct."""
    st = N.AurStats()
    assert lib.aur_get_stats(None, C.byref(st)) == N.AUR_ERR_INVALID
    assert st.last_candidates == 0 and st.last_candidates_max == 0


def test_header_cites_reference_interfaces():
    src = open(HEADER).read()
    for needle in ("weaviate_client.py:252-259", "weaviate_client.py:167-186", "similarity.py:84-98",
                   "weaviate_client.py:244-249", "weaviate_client.py:172"):
        assert needle in src


def test_invalid_arguments_are_rejected_without_touching_a_device(lib):
    h = C.c_void_p()
    assert lib.aur_open(None, C.byref(h)) == N.AUR_ERR_INVALID
    cfg = N.AurConfig(device=0, dim=0, dtype=0, reserved=0, capacity=10)
    assert lib.aur_open(C.byref(cfg), C.byref(h)) == N.AUR_ERR_INVALID
    cfg = N.AurConfig(device=0, dim=64, dtype=7, reserved=0, capacity=10)
    assert lib.aur_open(C.byref(cfg), C.byref(h)) == N.AUR_ERR_INVALID
    assert b"dtype" in lib.aur_last_error()
    assert lib.aur_search(None, None, 1, 1, None, None, None, None) == N.AUR_ERR_INVALID
    # a subset search's allow-list is checked before the handle is read (the handle here is a fake pointer)
    q, sc, ids = np.zeros(64, np.uint16), np.empty(1, np.float32), np.empty(1, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert lib.aur_search_subset(C.c_void_p(1), p(q), 1, 1, None, 3, p(sc), p(ids)) == N.AUR_ERR_INVALID
    assert b"allow_ids / n_allow" in lib.aur_last_error()
    assert lib.aur_search_subset(C.c_void_p(1), p(q), 1, 1, None, -1, p(sc), p(ids)) == N.AUR_ERR_INVALID
    assert b"n_allow < 0" in lib.aur_last_error()
    assert lib.aur_close(None) == N.AUR_OK


def test_no_cpu_fallback(lib):
    """Without a CUDA device every compute entry point fails with AUR_ERR_NO_DEVICE."""
    if lib.aur_device_count() > 0:
        pytest.skip("a GPU is present; the no-device behaviour is exercised on the CPU box")
    from aurora_b200.engine import Index, cosine_pairs

    with pytest.raises(N.AuroraError) as e:
        Index(64, 128)
    assert e.value.code == N.AUR_ERR_NO_DEVICE
    with pytest.raises(N.AuroraError) as e:
        cosine_pairs(np.ones((2, 4), np.float32), np.ones((2, 4), np.float32))
    assert e.value.code == N.AUR_ERR_NO_DEVICE


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(N, "_lib", None)
    monkeypatch.setattr(N, "LIB_PATH", "/nonexistent/libaurora_b200.so")
    with pytest.raises(N.NativeLibraryMissing) as e:
        N.load()
    assert "no CPU fallback" in str(e.value)


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "aurora_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f"{fn} imports the oracle"
