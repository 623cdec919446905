"""numpy restatement of brute-force cosine top-k.  TEST INFRASTRUCTURE ONLY.

What it restates
----------------
The reference delegates vector search to Weaviate 1.27.6 (cosine distance, flat
scan below ``flatSearchCutoff``; ``docker-compose.yaml:461``) -- not vendored, not
runnable here.  Its call sites are
``server/routes/knowledge_base/weaviate_client.py:252-259`` (hybrid, dense leg) and
``server/routes/incident_feedback/weaviate_client.py:286-297`` (``near_text``;
``similarity = 1 - distance``).  The arithmetic of one score is the reference's own
``_cosine_similarity`` (``server/services/correlation/strategies/similarity.py:84-98``)
restated in ``oracle/ref_cosine.py``; this module is the same arithmetic vectorised:

    s_ij = (q_i . c_j) / (|q_i| |c_j|)          fp64, zero norm -> 0.0
    order by (s desc, id asc), first k          (Weaviate returns best-first)

Tenant scope follows weaviate_client.py:244-249: a row is visible to a query iff
``row.user == q.user OR (q.org is set AND row.org == q.org)``.

Exactness: candidates are selected with an fp64 BLAS product (k + slack kept, widened
to every row within ``TIE_MARGIN`` of the k-th when the kept set ends inside a tie
group) and then re-scored with extended precision (``np.longdouble``) accumulation,
so the fp64 score of a row does not depend on its position in the matrix
(bit-identical duplicate rows tie exactly and fall back to ``id asc``, however many
there are).

Pinned by tests/test_oracle_golden.py: element-wise against golden vectors made by
the real reference function, and cfg1's top-5 against the pure-Python flat scan.
"""

from __future__ import annotations

import numpy as np

PAD_ID = -1
PAD_SCORE = -np.inf


# --------------------------------------------------------------------------- bf16
def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> bf16, returned as uint16 bit patterns."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    lsb = (u >> np.uint32(16)) & np.uint32(1)
    rounded = u + np.uint32(0x7FFF) + lsb
    out = (rounded >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(x)
    if nan.any():
        out = np.where(nan, np.uint16(0x7FC0), out)
    return out


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(b, dtype=np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def round_to_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 array whose values are exactly representable in bf16."""
    return bf16_bits_to_f32(f32_to_bf16_bits(x))


# ------------------------------------------------------------------------ scoring
def _norms64(x64: np.ndarray) -> np.ndarray:
    return np.sqrt(np.einsum("ij,ij->i", x64, x64))


def cosine_matrix(Q: np.ndarray, C: np.ndarray, clamp: bool = False) -> np.ndarray:
    """Full [nq, N] fp64 cosine matrix (small cases)."""
    Q64 = np.asarray(Q, dtype=np.float64)
    C64 = np.asarray(C, dtype=np.float64)
    qn, cn = _norms64(Q64), _norms64(C64)
    dots = Q64 @ C64.T
    denom = qn[:, None] * cn[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(denom > 0, dots / denom, 0.0)
    if clamp:
        s = np.clip(s, 0.0, 1.0)
    return s


def exact_cosine(q: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """Position-independent fp64 cosine of one query against a few rows."""
    ql = np.asarray(q, dtype=np.longdouble)
    rl = np.asarray(rows, dtype=np.longdouble)
    dots = (rl * ql[None, :]).sum(axis=1, dtype=np.longdouble)
    qq = (ql * ql).sum(dtype=np.longdouble)
    rr = (rl * rl).sum(axis=1, dtype=np.longdouble)
    dots64 = dots.astype(np.float64)
    denom = np.sqrt(np.float64(qq)) * np.sqrt(rr.astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(denom > 0, dots64 / denom, 0.0)


def visible_mask(row_user, row_org, q_user: int, q_org: int) -> np.ndarray:
    """weaviate_client.py:244-249: user_id == u OR org_id == o (org optional)."""
    m = np.asarray(row_user) == q_user
    if q_org is not None and q_org >= 0:
        m = m | (np.asarray(row_org) == q_org)
    return m


# The fp64 selection keeps k + slack rows per query.  When its last kept score is within this margin of the k-th, a
# group of (near-)tied rows may have been cut at an arbitrary point, so the candidates are widened to every row scoring
# within the margin of the k-th before the exact re-rank orders them by id.  The margin only has to be far above the
# error of an fp64 cosine (~1e-15), so that rows tied in exact arithmetic are never split by it.  A larger margin only
# adds candidates, which the exact re-rank then orders: correctness does not depend on how many rows it pulls in.
TIE_MARGIN = 1e-9


def _chunk_scores(Q64, qn, C, lo, hi, qsel, live, row_user, row_org, q_user, q_org):
    """fp64 cosine of the queries ``qsel`` against rows [lo, hi); invisible rows -inf."""
    Cc = C[lo:hi].astype(np.float64)
    denom = qn[qsel][:, None] * _norms64(Cc)[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(denom > 0, (Q64[qsel] @ Cc.T) / denom, 0.0)
    if live is not None:
        s[:, ~np.asarray(live[lo:hi], dtype=bool)] = -np.inf
    if q_user is not None:
        for j, i in enumerate(qsel):
            qo = None if q_org is None else int(q_org[i])
            s[j, ~visible_mask(row_user[lo:hi], row_org[lo:hi], int(q_user[i]), qo)] = -np.inf
    return s


def cosine_topk(Q, C, k: int, ids=None, live=None, row_user=None, row_org=None,
                q_user=None, q_org=None, clamp: bool = False, slack: int = 16,
                chunk: int = 131072, return_f64: bool = False):
    """Brute-force cosine top-k.

    Q [nq, D], C [N, D] (any float dtype; pass bf16-rounded fp32 to model a bf16
    store).  ``ids`` int64 [N] external ids (default: row numbers); ``live`` bool [N]
    tombstone mask; ``row_user/row_org/q_user/q_org`` int codes for the tenant scope
    (all None = unfiltered).  Returns ``(ids [nq,k] int64, scores [nq,k] float32)``
    best-first, padded with (PAD_ID, PAD_SCORE) when fewer than k rows are visible.
    ``return_f64``: also return the fp64 scores [nq,k] the float32 ones were rounded
    from (same padding), as a third element.
    """
    Q = np.asarray(Q)
    C = np.asarray(C)
    nq, N = Q.shape[0], C.shape[0]
    ids = np.arange(N, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    out_ids = np.full((nq, k), PAD_ID, dtype=np.int64)
    out_sc = np.full((nq, k), PAD_SCORE, dtype=np.float32)
    out64 = np.full((nq, k), PAD_SCORE, dtype=np.float64)
    if N == 0 or nq == 0 or k == 0:
        return (out_ids, out_sc, out64) if return_f64 else (out_ids, out_sc)

    Q64 = Q.astype(np.float64)
    qn = _norms64(Q64)
    keep = min(N, k + slack)
    cand_rows = np.zeros((nq, 0), dtype=np.int64)
    cand_sc = np.zeros((nq, 0), dtype=np.float64)
    allq = np.arange(nq)
    for lo in range(0, N, chunk):
        hi = min(N, lo + chunk)
        s = _chunk_scores(Q64, qn, C, lo, hi, allq, live, row_user, row_org, q_user, q_org)
        rows = np.broadcast_to(np.arange(lo, hi, dtype=np.int64), s.shape)
        cand_sc = np.concatenate([cand_sc, s], axis=1)
        cand_rows = np.concatenate([cand_rows, rows], axis=1)
        if cand_sc.shape[1] > keep:
            part = np.argpartition(-cand_sc, keep - 1, axis=1)[:, :keep]
            cand_sc = np.take_along_axis(cand_sc, part, axis=1)
            cand_rows = np.take_along_axis(cand_rows, part, axis=1)

    # queries whose kept set ends inside a tie group with the k-th: collect the whole group
    fin = np.isfinite(cand_sc)
    kth = -np.sort(-np.where(fin, cand_sc, -np.inf), axis=1)[:, min(k, keep) - 1]
    smin = np.where(fin, cand_sc, np.inf).min(axis=1)
    cut = np.nonzero((fin.sum(axis=1) == keep) & (keep < N) & (smin >= kth - TIE_MARGIN))[0]
    extra = {}
    for lo in range(0, N, chunk):
        if cut.size == 0:
            break
        hi = min(N, lo + chunk)
        s = _chunk_scores(Q64, qn, C, lo, hi, cut, live, row_user, row_org, q_user, q_org)
        for j, i in enumerate(cut):
            near = np.nonzero(s[j] >= kth[i] - TIE_MARGIN)[0] + lo
            extra[i] = np.union1d(extra.get(i, near[:0]), near)

    for i in range(nq):
        valid = np.isfinite(cand_sc[i])
        rows = cand_rows[i][valid]
        if rows.size == 0:
            continue
        if i in extra:
            rows = np.union1d(rows, extra[i])
        ex = exact_cosine(Q[i], C[rows])
        if clamp:
            ex = np.clip(ex, 0.0, 1.0)
        rid = ids[rows]
        order = np.lexsort((rid, -ex))[:k]
        out_ids[i, : order.size] = rid[order]
        out_sc[i, : order.size] = ex[order].astype(np.float32)
        out64[i, : order.size] = ex[order]
    return (out_ids, out_sc, out64) if return_f64 else (out_ids, out_sc)


# --------------------------------------------------------- timed CPU baseline ("port")
def flat_search_f32(Q: np.ndarray, C: np.ndarray, k: int):
    """What a CPU flat cosine index does per batch: normalise, sgemm, select, sort.

    fp32 throughout (Weaviate stores fp32 vectors), BLAS threads = all host cores.
    Used only as bench.py's ``cpu_baseline`` / ``--impl reference`` leg.
    """
    Qf = np.asarray(Q, dtype=np.float32)
    Cf = np.asarray(C, dtype=np.float32)
    qn = np.linalg.norm(Qf, axis=1, keepdims=True)
    cn = np.linalg.norm(Cf, axis=1, keepdims=True)
    Qn = np.divide(Qf, qn, out=np.zeros_like(Qf), where=qn > 0)
    Cn = np.divide(Cf, cn, out=np.zeros_like(Cf), where=cn > 0)
    s = Qn @ Cn.T
    kk = min(k, s.shape[1])
    part = np.argpartition(-s, kk - 1, axis=1)[:, :kk]
    ps = np.take_along_axis(s, part, axis=1)
    order = np.lexsort((part, -ps), axis=1)
    return np.take_along_axis(part, order, axis=1).astype(np.int64), np.take_along_axis(ps, order, axis=1)
