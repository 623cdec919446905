"""Exact comparison of a search with the oracle.  The engine's final ranking is an fp64 re-score of the stored rows, so
a search through aur_search_dev with scores64 is held to:
  - ids bit-exact;
  - scores64 within dim * 2^-52 * 4 of the oracle's fp64 score (a cosine is at most 1 in magnitude, and an fp64 dot
    product of dim terms with fp64 norms and one division errs by a few dim ulps at most);
  - the float32 scores equal to scores64 rounded to float32, exactly;
  - padding (id -1, score -inf in both) exactly where the oracle pads.
A wrong |q|, a dropped element of the row or a neighbour's row in the gather all move the fp64 score by far more."""

from __future__ import annotations

import numpy as np

from aurora_b200.engine import DeviceBuffer
from oracle import cosine_topk as O


def dev_search(ix, Q, k, q_user=None, q_org=None):
    """aur_search_dev on the index's own stream: (ids [nq,k] int64, scores [nq,k] float32, scores64 [nq,k] float64)."""
    q = ix._rows_buffer(Q)
    nq = q.shape[0]
    dq = DeviceBuffer(q.nbytes).upload(q)
    ds, di, d64 = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8), DeviceBuffer(nq * k * 8)
    du = None if q_user is None else DeviceBuffer(nq * 4).upload(np.ascontiguousarray(q_user, dtype=np.int32))
    do = None if q_org is None else DeviceBuffer(nq * 4).upload(np.ascontiguousarray(q_org, dtype=np.int32))
    ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr, d64.ptr, q_user_ptr=du.ptr if du else 0, q_org_ptr=do.ptr if do else 0)
    ix.sync()
    return (di.download(np.empty((nq, k), np.int64)), ds.download(np.empty((nq, k), np.float32)),
            d64.download(np.empty((nq, k), np.float64)))


def _check_ids_and_padding(ids, oids):
    bad = np.argwhere(ids != oids)
    assert bad.size == 0, (f"{len(bad)} id mismatches, first at {tuple(bad[0])}: got {ids[tuple(bad[0])]} "
                           f"want {oids[tuple(bad[0])]}")


def check_exact(got, Q, C, k, want=None, **oracle_kw):
    """got = dev_search(...); want = the oracle's (ids, scores, scores64), computed here unless given.  Returns want."""
    ids, sc, s64 = got
    if want is None:
        want = O.cosine_topk(Q, C, k, return_f64=True, **oracle_kw)
    oids, _, o64 = want
    _check_ids_and_padding(ids, oids)
    pad = oids < 0
    assert (s64[pad] == -np.inf).all() and (sc[pad] == -np.inf).all(), "padding must be (-1, -inf)"
    tol = np.asarray(Q).shape[1] * 2.0 ** -52 * 4
    err = np.abs(s64[~pad] - o64[~pad])
    assert err.size == 0 or float(err.max()) <= tol, f"fp64 score error {float(err.max()):.3e} > {tol:.3e}"
    assert np.array_equal(sc, s64.astype(np.float32)), "float32 scores are not the fp64 scores rounded"
    return want


def check_host_exact(got, Q, C, k, **oracle_kw):
    """Host entry points return float32 scores only: ids bit-exact, padding exact, and each score within one float32
    rounding of the oracle's fp64 score (both sides round an fp64 value that agrees to a few dim ulps)."""
    ids, sc = got
    want = O.cosine_topk(Q, C, k, return_f64=True, **oracle_kw)
    oids, _, o64 = want
    _check_ids_and_padding(ids, oids)
    pad = oids < 0
    assert (sc[pad] == -np.inf).all(), "padding must be (-1, -inf)"
    ulp = np.spacing(np.abs(o64[~pad]).astype(np.float32))
    err = np.abs(sc[~pad].astype(np.float64) - o64[~pad])
    assert err.size == 0 or bool((err <= ulp).all()), f"float32 score off by more than one rounding: {float(err.max()):.3e}"
    return want
