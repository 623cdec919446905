"""Test helpers for the GPU keyword store: a host mirror of what the store holds (an append log with tombstones, the
layout oracle/bm25_topk.py reads), seeded Zipf corpora, and the bit-exact comparison with the oracle."""

import numpy as np

from oracle.bm25_topk import Corpus, bm25_topk


class Mirror:
    """Rows as the device store appends them: upserts and removes tombstone the old row."""

    def __init__(self):
        self.terms, self.tfs, self.offsets = [np.zeros(0, np.int32)], [np.zeros(0, np.int32)], [0]
        self.ids, self.user, self.org = [], [], []
        self.live = []
        self.row_of = {}

    def add(self, ids, terms, tfs, offsets, user=None, org=None):
        n = len(ids)
        base = self.offsets[-1]
        self.terms.append(np.asarray(terms, np.int32))
        self.tfs.append(np.asarray(tfs, np.int32))
        self.offsets.extend((base + np.asarray(offsets[1:], np.int64)).tolist())
        for i, d in enumerate(ids):
            d = int(d)
            if d in self.row_of:
                self.live[self.row_of[d]] = False
            self.row_of[d] = len(self.ids)
            self.ids.append(d)
            self.live.append(True)
            self.user.append(0 if user is None else int(user[i]))
            self.org.append(-1 if org is None else int(org[i]))
        assert len(self.offsets) == len(self.ids) + 1 and n >= 0

    def remove(self, ids):
        for d in ids:
            r = self.row_of.pop(int(d), None)
            if r is not None:
                self.live[r] = False

    def compact(self):
        keep = [r for r in range(len(self.ids)) if self.live[r]]
        t, f, off = self.csr()
        nt, nf, no = [], [], [0]
        for r in keep:
            nt.append(t[off[r]:off[r + 1]])
            nf.append(f[off[r]:off[r + 1]])
            no.append(no[-1] + off[r + 1] - off[r])
        self.terms, self.tfs, self.offsets = nt or [np.zeros(0, np.int32)], nf or [np.zeros(0, np.int32)], no
        self.ids = [self.ids[r] for r in keep]
        self.user = [self.user[r] for r in keep]
        self.org = [self.org[r] for r in keep]
        self.live = [True] * len(keep)
        self.row_of = {d: i for i, d in enumerate(self.ids)}

    def csr(self):
        return np.concatenate(self.terms), np.concatenate(self.tfs), np.asarray(self.offsets, np.int64)

    def corpus(self, n_rows=None):
        t, f, off = self.csr()
        return Corpus(t, f, off, self.ids, self.live, self.user, self.org, n_rows=n_rows)


def zipf_docs(rng, n, vocab=5000, mean_len=40, a=1.3, min_len=0):
    """n documents as CSR (term ids ascending, tf) of Zipf-distributed words."""
    lens = np.maximum(min_len, rng.poisson(mean_len, n))
    words = (rng.zipf(a, int(lens.sum())) - 1) % vocab
    terms, tfs, offsets = [], [], [0]
    pos = 0
    for ln in lens:
        u, c = np.unique(words[pos:pos + ln], return_counts=True)
        pos += ln
        terms.append(u.astype(np.int32))
        tfs.append(c.astype(np.int32))
        offsets.append(offsets[-1] + len(u))
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int32)   # noqa: E731
    return cat(terms), cat(tfs), np.asarray(offsets, np.int64)


def zipf_queries(rng, nq, vocab=5000, lo=2, hi=8, a=1.3):
    terms, offsets = [], [0]
    for _ in range(nq):
        m = int(rng.integers(lo, hi + 1))
        q = np.unique((rng.zipf(a, m) - 1) % vocab)
        terms.append(q.astype(np.int32))
        offsets.append(offsets[-1] + len(q))
    return np.concatenate(terms), np.asarray(offsets, np.int64)


def assert_matches_oracle(store, mirror, q_terms, q_off, k, q_user=None, q_org=None, allow_ids=None, sample=None):
    """Search the store and hold every answer (or the sampled queries) to the oracle over exactly the prefix the search
    reports: ids bit-exact, fp64 scores bit-identical, padding (-1, -inf)."""
    ids, scores, snap = store.search(q_terms, q_off, k, q_user, q_org, allow_ids)
    corpus = mirror.corpus(n_rows=snap)
    qs = range(len(q_off) - 1) if sample is None else sample
    for q in qs:
        sl = slice(q_off[q], q_off[q + 1])
        wi, ws = bm25_topk(corpus, q_terms[sl], np.array([0, q_off[q + 1] - q_off[q]]), k,
                           None if q_user is None else q_user[q:q + 1], None if q_org is None else q_org[q:q + 1], allow_ids)
        assert np.array_equal(ids[q], wi[0]), (q, ids[q][:8], wi[0][:8])
        assert np.array_equal(scores[q].view(np.int64), ws[0].view(np.int64)), (q, scores[q][:4], ws[0][:4])
    return ids, scores, snap
