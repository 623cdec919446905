"""fp64 numpy restatement of the BM25 keyword leg over a CSR corpus (the scoring contract of DESIGN.md section 10).

It is ``aurora_b200.bm25.BM25Index.search`` on its loop path, bit for bit, in array form:
  * N, df and total_len over every live document (zero-token documents count in N); avgdl = total_len / N, or 1.0;
  * idf = math.log(1.0 + (N - df + 0.5) / (df + 0.5)) per term (math.log, not np.log: the libm call the loop path makes);
  * a query's terms in the order given (the caller passes sorted(set(tokenize(q))) as vocabulary ids), terms without a
    live posting skipped, repeats ignored;
  * contribution idf * tf * (K1 + 1.0) / (tf + K1 * (1.0 - B + B * dl / avgdl)), elementwise fp64 numpy (one IEEE
    operation per numpy operation, no contraction), added term after term to a score that starts at 0.0;
  * top-k by (score desc, id asc) over the documents with a matching term that pass the filters (tenant scope
    row_user == u or (o >= 0 and row_org == o), allow-list); padding id -1 / score -inf.

``Corpus`` builds the inverted lists once, so sampled queries over a 1M-document corpus take milliseconds each.
"""

from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np

K1, B = 1.2, 0.75


class Corpus:
    """CSR corpus: document i has term_ids / tfs [offsets[i], offsets[i+1]); ``live`` masks tombstones; ``n_rows``
    limits it to a published prefix."""

    def __init__(self, term_ids, tfs, offsets, ids, live=None, row_user=None, row_org=None, n_rows: Optional[int] = None):
        offsets = np.asarray(offsets, dtype=np.int64)
        n = len(offsets) - 1 if n_rows is None else int(n_rows)
        offsets = offsets[: n + 1]
        self.ids = np.asarray(ids, dtype=np.int64)[:n]
        self.live = np.ones(n, dtype=bool) if live is None else np.asarray(live, dtype=bool)[:n]
        self.user = np.zeros(n, np.int32) if row_user is None else np.asarray(row_user, dtype=np.int32)[:n]
        self.org = np.full(n, -1, np.int32) if row_org is None else np.asarray(row_org, dtype=np.int32)[:n]
        t = np.asarray(term_ids, dtype=np.int64)[: offsets[-1]]
        f = np.asarray(tfs, dtype=np.int64)[: offsets[-1]]
        row = np.repeat(np.arange(n, dtype=np.int64), np.diff(offsets))
        self.dl = np.bincount(row, weights=f, minlength=n).astype(np.int64) if n else np.zeros(0, np.int64)
        keep = self.live[row]
        t, f, row = t[keep], f[keep], row[keep]
        order = np.argsort(t, kind="stable")
        self._t, self._f, self._row = t[order], f[order], row[order]
        self._terms, self._starts = np.unique(self._t, return_index=True)
        self._ends = np.append(self._starts[1:], len(self._t))
        self.N = int(self.live.sum())
        self.total_len = int(self.dl[self.live].sum())

    def postings(self, term: int):
        i = np.searchsorted(self._terms, term)
        if i >= len(self._terms) or self._terms[i] != term:
            return None
        s, e = self._starts[i], self._ends[i]
        return self._row[s:e], self._f[s:e]

    def scores(self, q_terms: Sequence[int]):
        """(rows, scores) of every live document with at least one of the query's terms, unfiltered."""
        n_docs = self.N
        if n_docs == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.float64)
        avgdl = self.total_len / n_docs if self.total_len else 1.0
        acc = np.zeros(len(self.ids), dtype=np.float64)
        hit = np.zeros(len(self.ids), dtype=bool)
        seen = set()
        for term in q_terms:
            term = int(term)
            if term in seen:
                continue
            seen.add(term)
            p = self.postings(term)
            if p is None:
                continue
            rows, tf_i = p
            df = len(rows)
            idf = math.log(1.0 + (n_docs - df + 0.5) / (df + 0.5))
            tf = tf_i.astype(np.float64)
            dl = self.dl[rows].astype(np.float64)
            acc[rows] = acc[rows] + idf * tf * (K1 + 1.0) / (tf + K1 * (1.0 - B + B * dl / avgdl))
            hit[rows] = True
        rows = np.nonzero(hit)[0]
        return rows, acc[rows]

    def topk(self, q_terms: Sequence[int], k: int, q_user: Optional[int] = None, q_org: int = -1, allow_ids=None):
        """(ids [k] int64, scores [k] float64) of one query."""
        rows, sc = self.scores(q_terms)
        if q_user is not None:
            ok = (self.user[rows] == q_user) | ((q_org >= 0) & (self.org[rows] == q_org))
            rows, sc = rows[ok], sc[ok]
        if allow_ids is not None:
            ok = np.isin(self.ids[rows], np.asarray(allow_ids, dtype=np.int64))
            rows, sc = rows[ok], sc[ok]
        ids = self.ids[rows]
        order = np.lexsort((ids, -sc))[:k]
        out_i = np.full(k, -1, dtype=np.int64)
        out_s = np.full(k, -np.inf, dtype=np.float64)
        out_i[: len(order)] = ids[order]
        out_s[: len(order)] = sc[order]
        return out_i, out_s


def bm25_topk(corpus: Corpus, q_terms, q_offsets, k: int, q_user=None, q_org=None, allow_ids=None):
    """Batched form of ``Corpus.topk`` with the C ABI's query layout: (ids [nq,k], scores [nq,k])."""
    q_offsets = np.asarray(q_offsets, dtype=np.int64)
    nq = len(q_offsets) - 1
    ids = np.full((nq, k), -1, dtype=np.int64)
    scores = np.full((nq, k), -np.inf, dtype=np.float64)
    for q in range(nq):
        terms = np.asarray(q_terms)[q_offsets[q]:q_offsets[q + 1]]
        u = None if q_user is None else int(q_user[q])
        o = -1 if q_org is None else int(q_org[q])
        ids[q], scores[q] = corpus.topk(terms, k, u, o, allow_ids)
    return ids, scores
