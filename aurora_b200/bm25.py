"""Sparse leg of the hybrid query + ranked fusion (SURVEY.md section 8 a2 / (f)1).

The reference asks Weaviate for ``collection.query.hybrid(query, alpha, fusion_type=HybridFusion.RANKED)``
(server/routes/knowledge_base/weaviate_client.py:252-259): a BM25F keyword search and a vector search
whose ranked lists are fused as ``sum_legs weight_leg / (rank + 60)`` with ``weight = alpha`` for the
vector leg and ``1 - alpha`` for the keyword leg.  Both live inside the Weaviate server (Go, CPU) --
not in /root/reference -- so this restates Weaviate 1.27's documented behaviour: BM25 with k1 = 1.2,
b = 0.75, "word" tokenisation (lower-case, split on non-alphanumerics), idf = ln(1 + (N - n + 0.5) /
(n + 0.5)); rankedFusion with the constant 60 and 0-based ranks.  Unpinned: the reference has no test
at this boundary (SURVEY.md section 8c).  ``BM25Index`` is the host index (the path of the test doubles and
the definition the device is held to); ``DeviceBM25`` keeps the vocabulary and tokenisation on the host and the
postings, scoring and top-k in the GPU keyword store (csrc/keyword.cu, DESIGN.md section 10).  ``ranked_fusion`` and
``relative_score_fusion`` (Weaviate's other fusion, HybridFusion.RELATIVE_SCORE) define the fused score; the device
fusion of ``DeviceBM25.search_batch(..., dense=...)`` (csrc/hybrid.cu, DESIGN.md section 11) equals them bit for bit.
"""

from __future__ import annotations

import math
import re
from collections import Counter, defaultdict
from typing import Callable, Dict, Iterable, List, Optional, Tuple

_WORD = re.compile(r"[0-9a-z]+")
K1, B, RANK_CONSTANT = 1.2, 0.75, 60.0
VECTORISE_FROM = 256      # posting lists at least this long are scored as numpy arrays (cached per term), shorter ones in a Python loop


def tokenize(text: str) -> List[str]:
    return _WORD.findall(text.lower())


class BM25Index:
    """Inverted index over one text field per document id."""

    def __init__(self):
        self._postings: Dict[str, Dict[int, int]] = defaultdict(dict)   # term -> {doc id: tf}
        self._doc_terms: Dict[int, Counter] = {}
        self._doc_len: Dict[int, int] = {}
        self._total_len = 0
        self._arrays: Dict[str, tuple] = {}      # term -> (doc ids ascending, tf, doc lengths) for long posting lists; dropped on mutation

    def __len__(self) -> int:
        return len(self._doc_len)

    def add(self, doc_id: int, text: str) -> None:
        if doc_id in self._doc_len:
            self.remove(doc_id)                       # upsert
        terms = Counter(tokenize(text))
        self._doc_terms[doc_id] = terms
        n = sum(terms.values())
        self._doc_len[doc_id] = n
        self._total_len += n
        for t, tf in terms.items():
            self._postings[t][doc_id] = tf
            self._arrays.pop(t, None)

    def remove(self, doc_id: int) -> bool:
        terms = self._doc_terms.pop(doc_id, None)
        if terms is None:
            return False
        self._total_len -= self._doc_len.pop(doc_id)
        for t in terms:
            plist = self._postings.get(t)
            self._arrays.pop(t, None)
            if plist is not None:
                plist.pop(doc_id, None)
                if not plist:
                    del self._postings[t]
        return True

    def _term_arrays(self, term: str, plist: Dict[int, int]):
        a = self._arrays.get(term)
        if a is None:
            import numpy as np

            ids = np.fromiter(plist.keys(), dtype=np.int64, count=len(plist))
            order = np.argsort(ids, kind="stable")
            ids = ids[order]
            tf = np.fromiter(plist.values(), dtype=np.float64, count=len(plist))[order]
            dl = np.fromiter((self._doc_len[int(d)] for d in ids), dtype=np.float64, count=len(ids))
            a = self._arrays[term] = (ids, tf, dl)
        return a

    def search(self, query: str, limit: int, allow: Optional[Callable[[int], bool]] = None,
               allowed: Optional[set] = None, allowed_sorted=None) -> List[Tuple[int, float]]:
        """Top-``limit`` (doc id, BM25 score), best first; ties by ascending id.  The pre-filter (tenant scope,
        metadata filter) comes as ``allowed`` -- a set of visible doc ids, intersected with every posting list at C
        speed (``allowed_sorted``: the same ids as an ascending int64 array, when the caller keeps one) -- or as a
        predicate ``allow``: documents outside do not exist for this query."""
        n_docs = len(self._doc_len)
        if n_docs == 0 or limit <= 0:
            return []
        avgdl = self._total_len / n_docs if self._total_len else 1.0
        scores: Dict[int, float] = defaultdict(float)
        doc_len = self._doc_len
        long_ids, long_contrib = [], []
        allowed_arr = allowed_sorted        # the same ids as `allowed`, ascending int64 (callers that keep one per tenant)
        for term in sorted(set(tokenize(query))):          # fixed order: equal indexes give bit-equal scores
            plist = self._postings.get(term)
            if not plist:
                continue
            idf = math.log(1.0 + (n_docs - len(plist) + 0.5) / (len(plist) + 0.5))
            if len(plist) >= VECTORISE_FROM and (allowed is None or len(allowed) >= VECTORISE_FROM):
                # a common word: its posting list is scored as arrays (a Python loop over 10^5 postings costs tens of
                # milliseconds per query; Weaviate's BM25 is native code)
                import numpy as np

                ids, tf, dl = self._term_arrays(term, plist)
                if allowed is not None:
                    if allowed_arr is None:
                        allowed_arr = np.fromiter(allowed, dtype=np.int64, count=len(allowed))
                        allowed_arr.sort()
                    if len(allowed_arr) <= len(ids):         # both ascending: look the shorter one up in the longer one
                        pos = np.minimum(np.searchsorted(ids, allowed_arr), len(ids) - 1)
                        pos = pos[ids[pos] == allowed_arr]
                        ids, tf, dl = ids[pos], tf[pos], dl[pos]
                    else:
                        pos = np.minimum(np.searchsorted(allowed_arr, ids), len(allowed_arr) - 1)
                        keep = allowed_arr[pos] == ids
                        ids, tf, dl = ids[keep], tf[keep], dl[keep]
                long_ids.append(ids)
                long_contrib.append(idf * tf * (K1 + 1.0) / (tf + K1 * (1.0 - B + B * dl / avgdl)))
                continue
            docs = plist.keys() & allowed if allowed is not None else plist.keys()
            for doc in docs:
                tf = plist[doc]
                scores[doc] += idf * tf * (K1 + 1.0) / (tf + K1 * (1.0 - B + B * doc_len[doc] / avgdl))
        if long_ids:
            import numpy as np

            if scores:                                      # the short lists' sums join as one more block, first in line
                long_ids.insert(0, np.fromiter(scores.keys(), dtype=np.int64, count=len(scores)))
                long_contrib.insert(0, np.fromiter(scores.values(), dtype=np.float64, count=len(scores)))
            all_ids = np.concatenate(long_ids)
            uniq, inv = np.unique(all_ids, return_inverse=True)
            total = np.bincount(inv, weights=np.concatenate(long_contrib), minlength=len(uniq))
            if allow is not None:
                keep = np.fromiter((bool(allow(int(d))) for d in uniq), dtype=bool, count=len(uniq))
                uniq, total = uniq[keep], total[keep]
            if len(uniq) > 4 * limit:                       # narrow before the exact (score desc, id asc) sort
                kth = np.partition(total, len(total) - limit)[len(total) - limit]
                keep = total >= kth
                uniq, total = uniq[keep], total[keep]
            order = np.lexsort((uniq, -total))[:limit]
            return [(int(uniq[i]), float(total[i])) for i in order]
        if allow is not None:
            scores = {d: v for d, v in scores.items() if allow(d)}
        return sorted(scores.items(), key=lambda kv: (-kv[1], kv[0]))[:limit]


def build_csr(vocab: Dict[str, int], texts: Iterable[str]):
    """Documents -> (term ids int32, tf int32, offsets int64 [n + 1]) with term ids ascending inside each document.
    New words get the next free id in ``vocab`` (grow-only)."""
    import numpy as np

    terms: List[int] = []
    tfs: List[int] = []
    offsets = [0]
    for text in texts:
        counts = Counter(tokenize(text))
        row = []
        for t, tf in counts.items():
            tid = vocab.get(t)
            if tid is None:
                tid = vocab[t] = len(vocab)
            row.append((tid, tf))
        row.sort()
        terms.extend(t for t, _ in row)
        tfs.extend(f for _, f in row)
        offsets.append(len(terms))
    return np.asarray(terms, dtype=np.int32), np.asarray(tfs, dtype=np.int32), np.asarray(offsets, dtype=np.int64)


def query_csr(vocab: Dict[str, int], queries: Iterable[str]):
    """Queries -> (term ids int32, offsets int64 [nq + 1]): each query's ``sorted(set(tokenize(q)))`` -- the loop
    path's summation order -- with words the vocabulary never saw dropped (they have no posting)."""
    import numpy as np

    terms: List[int] = []
    offsets = [0]
    for q in queries:
        terms.extend(vocab[t] for t in sorted(set(tokenize(q))) if t in vocab)
        offsets.append(len(terms))
    return np.asarray(terms, dtype=np.int32), np.asarray(offsets, dtype=np.int64)


class DeviceBM25:
    """The keyword leg on the GPU (``engine.KeywordIndex``), with ``BM25Index``'s surface plus ``search_batch``.

    Scores and order are those of ``BM25Index.search`` on its loop path, bit for bit (DESIGN.md section 10).  Holds the
    vocabulary (word -> int32 term id, grow-only; a reloaded knowledge base rebuilds it from the texts) and tenant codes
    per document, so a tenant scope is applied on the device like the dense leg's."""

    def __init__(self, capacity: int = 1 << 20, device: int = 0, postings_capacity: int = 0, store=None):
        if store is None:
            from .engine import KeywordIndex

            store = KeywordIndex(capacity, postings_capacity=postings_capacity, device=device)
        self.store = store
        self.vocab: Dict[str, int] = {}
        self._docs: set = set()

    def __len__(self) -> int:
        return len(self._docs)

    def add(self, doc_id: int, text: str, user_code: int = 0, org_code: int = -1) -> None:
        self.add_many([doc_id], [text], [user_code], [org_code])

    def add_many(self, doc_ids, texts, user_codes=None, org_codes=None) -> None:
        """Upsert documents in one call (one device append)."""
        import numpy as np

        doc_ids = np.asarray(doc_ids, dtype=np.int64)
        if len(doc_ids) == 0:
            return
        terms, tfs, offsets = build_csr(self.vocab, texts)
        self.store.add(doc_ids, terms, tfs, offsets, user_codes, org_codes)
        self._docs.update(int(d) for d in doc_ids)

    def remove(self, doc_id: int) -> bool:
        return self.remove_many([doc_id]) > 0

    def remove_many(self, doc_ids) -> int:
        import numpy as np

        ids = [int(d) for d in doc_ids]
        if not ids:
            return 0
        self._docs.difference_update(ids)
        return self.store.remove(np.asarray(ids, dtype=np.int64))

    def compact(self) -> int:
        return self.store.compact()

    def stats(self) -> dict:
        return self.store.stats()

    def search(self, query: str, limit: int, allow: Optional[Callable[[int], bool]] = None,
               allowed: Optional[set] = None, allowed_sorted=None) -> List[Tuple[int, float]]:
        """``BM25Index.search``: top-``limit`` (doc id, score), best first, ties by ascending id; ``allowed`` (a set of
        ids) or ``allow`` (a predicate, resolved over the stored ids) pre-filter the documents."""
        if limit <= 0 or not self._docs:
            return []
        allow_ids = None
        if allowed_sorted is not None:
            allow_ids = allowed_sorted
        elif allowed is not None:
            allow_ids = list(allowed)
        if allow is not None:
            base = self._docs if allow_ids is None else set(int(d) for d in allow_ids)
            allow_ids = [d for d in base if allow(d)]
        return self._run([query], limit, None, None, allow_ids)[0]

    def search_batch(self, queries: List[str], limit: int, q_user=None, q_org=None, dense=None) -> List[list]:
        """All queries in one device search; ``q_user`` / ``q_org``: per-query tenant codes (row_user == u or, for
        org >= 0, row_org == o), None = unscoped.

        ``dense = (index, vectors, w_dense, fusion, k_out)``: the whole hybrid query in one device call
        (``engine.hybrid_search``): the keyword leg's top-``limit`` stays in HBM and is fused there with the dense leg's
        top-``limit`` of ``vectors`` over the ``engine.Index`` ``index`` (same scopes), weights ``w_dense`` (per query)
        and ``1 - w_dense``, ``fusion`` an ``AUR_FUSION_*`` value.  Each query's list then holds its best ``k_out``
        pairs ``(id, (fused score, dense cosine or None))``."""
        if not queries:
            return []
        if dense is not None:
            return self._run_hybrid(queries, limit, q_user, q_org, *dense)
        if limit <= 0 or not self._docs:
            return [[] for _ in queries]
        return self._run(queries, limit, q_user, q_org, None)

    def _run_hybrid(self, queries, fetch, q_user, q_org, index, vectors, w_dense, fusion, k_out):
        from .engine import hybrid_search

        q_terms, q_off = query_csr(self.vocab, queries)
        ids, scores, cosine, _ = hybrid_search(index, self.store, vectors, fetch, q_terms, q_off, w_dense, None, fusion,
                                               k_out, q_user, q_org)
        out = []
        for row_i, row_s, row_c in zip(ids, scores, cosine):
            n = int((row_i >= 0).sum())
            out.append([(int(d), (float(s), None if c != c else float(c)))
                        for d, s, c in zip(row_i[:n].tolist(), row_s[:n].tolist(), row_c[:n].tolist())])
        return out

    def _run(self, queries, limit, q_user, q_org, allow_ids):
        q_terms, q_off = query_csr(self.vocab, queries)
        ids, scores, _ = self.store.search(q_terms, q_off, int(limit), q_user, q_org, allow_ids)
        out = []
        for row_i, row_s in zip(ids, scores):
            n = int((row_i >= 0).sum())
            out.append([(int(d), float(s)) for d, s in zip(row_i[:n], row_s[:n])])
        return out


def ranked_fusion(legs: Iterable[Tuple[float, List[int]]], limit: int) -> List[Tuple[int, float]]:
    """Weaviate rankedFusion: ``legs`` = (weight, ids best-first); score(id) = sum over legs of
    weight / (rank + 60), rank 0-based.  Returns the top ``limit`` (id, fused score), ties by id."""
    fused: Dict[int, float] = defaultdict(float)
    for weight, ids in legs:
        if weight <= 0.0:
            continue
        for rank, doc in enumerate(ids):
            fused[doc] += weight / (rank + RANK_CONSTANT)
    return sorted(fused.items(), key=lambda kv: (-kv[1], kv[0]))[:limit]


def relative_score_fusion(legs: Iterable[Tuple[float, List[Tuple[int, float]]]], limit: int) -> List[Tuple[int, float]]:
    """Weaviate relativeScoreFusion: ``legs`` = (weight, [(id, score)] best-first); each leg's scores are min-max
    normalised over its own list, score(id) = sum over legs of weight * (s - lo) / (hi - lo) (weight when hi == lo),
    summed in leg order from 0.0 in fp64.  A leg with weight <= 0 or no entries takes no part.  Returns the top ``limit``
    (id, fused score), ties by id.  The hi == lo rule, the fp64 arithmetic and the id tie-break are this project's
    reading of Weaviate's documentation (parity unpinned, DESIGN.md section 11)."""
    fused: Dict[int, float] = defaultdict(float)
    for weight, entries in legs:
        if weight <= 0.0 or not entries:
            continue
        scores = [s for _, s in entries]
        lo, hi = min(scores), max(scores)
        for doc, s in entries:
            fused[doc] += weight if hi == lo else weight * ((s - lo) / (hi - lo))
    return sorted(fused.items(), key=lambda kv: (-kv[1], kv[0]))[:limit]
