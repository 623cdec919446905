"""aur_hybrid_search_multi's refusals that happen before any shard or store is read or any device is touched: NULL
arrays and entries, the shard count, handles listed twice, and the fetch / k_out / fusion / weight checks it shares
with aur_hybrid_search.  The handles are fake pointers, so a check that read one would crash instead of failing."""

import ctypes as C

import numpy as np
import pytest

from aurora_b200 import _native as N


@pytest.fixture(scope="module")
def lib():
    from aurora_b200.build import build_native

    build_native()
    return N.load()


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _fake(*xs):
    return (C.c_void_p * len(xs))(*xs)


def test_rejections_before_any_handle_is_read(lib):
    nq = 2
    qv = np.zeros((nq, 8), np.uint16)
    qt, qo = np.array([1, 2], np.int32), np.array([0, 1, 2], np.int64)
    out_s, out_i, out_c = np.empty(64), np.empty(64, np.int64), np.empty(64, np.float32)
    snaps = np.empty(130, np.int64)

    def call(shards, stores, n, fetch=4, k_out=8, fusion=N.FUSION_RANKED, wd=(0.5, 0.5), ws=(0.5, 0.5), qv_=qv,
             scores=out_s):
        wd, ws = np.array(wd, np.float64), np.array(ws, np.float64)
        return lib.aur_hybrid_search_multi(shards, stores, n, None if qv_ is None else _vp(qv_), nq, fetch, _vp(qt),
                                           _vp(qo), None, None, _vp(wd), _vp(ws), fusion, k_out,
                                           None if scores is None else _vp(scores), _vp(out_i), _vp(out_c), _vp(snaps))

    two = lambda: (_fake(0x1000, 0x2000), _fake(0x3000, 0x4000))              # noqa: E731
    # NULL arrays
    assert call(None, _fake(0x3000), 1) == N.AUR_ERR_INVALID
    assert call(_fake(0x1000), None, 1) == N.AUR_ERR_INVALID
    assert call(*two(), 2, qv_=None) == N.AUR_ERR_INVALID
    assert call(*two(), 2, scores=None) == N.AUR_ERR_INVALID
    # the shard count
    assert call(_fake(0x1000), _fake(0x3000), 0) == N.AUR_ERR_INVALID
    many = [0x10000 + 64 * i for i in range(65)]
    assert call(_fake(*many), _fake(*[m + 0x100000 for m in many]), 65) == N.AUR_ERR_INVALID
    assert b"n must be" in lib.aur_last_error()
    # NULL entries
    assert call(_fake(0x1000, None), _fake(0x3000, 0x4000), 2) == N.AUR_ERR_INVALID
    assert b"NULL" in lib.aur_last_error()
    assert call(_fake(0x1000, 0x2000), _fake(None, 0x4000), 2) == N.AUR_ERR_INVALID
    assert b"NULL" in lib.aur_last_error()
    # a handle listed twice
    assert call(_fake(0x1000, 0x2000, 0x1000), _fake(0x3000, 0x4000, 0x5000), 3) == N.AUR_ERR_INVALID
    assert b"twice" in lib.aur_last_error()
    assert call(_fake(0x1000, 0x2000, 0x6000), _fake(0x3000, 0x4000, 0x4000), 3) == N.AUR_ERR_INVALID
    assert b"twice" in lib.aur_last_error()
    # fetch, k_out, fusion and weights, as aur_hybrid_search checks them
    assert call(*two(), 2, fetch=0, k_out=1) == N.AUR_ERR_INVALID
    assert call(*two(), 2, fetch=129, k_out=1) == N.AUR_ERR_UNSUPPORTED
    assert call(*two(), 2, k_out=0) == N.AUR_ERR_INVALID
    assert call(*two(), 2, k_out=9) == N.AUR_ERR_INVALID
    assert call(*two(), 2, fusion=2) == N.AUR_ERR_INVALID
    assert call(*two(), 2, wd=(0.5, np.nan)) == N.AUR_ERR_INVALID
    assert call(*two(), 2, ws=(np.inf, 0.5)) == N.AUR_ERR_INVALID
    assert b"finite" in lib.aur_last_error()
    # a bad keyword query is refused by the keyword search's own checks, still before any handle is read
    bad_off = np.array([0, 2, 1], np.int64)
    assert lib.aur_hybrid_search_multi(*two(), 2, _vp(qv), nq, 4, _vp(qt), _vp(bad_off), None, None,
                                       _vp(np.full(nq, 0.5)), _vp(np.full(nq, 0.5)), N.FUSION_RANKED, 8, _vp(out_s),
                                       _vp(out_i), _vp(out_c), _vp(snaps)) == N.AUR_ERR_INVALID
