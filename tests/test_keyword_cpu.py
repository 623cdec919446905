"""The BM25 keyword store's host side, without a GPU: the fp64 oracle (oracle/bm25_topk.py) equals BM25Index.search on
its loop path bit for bit, DeviceBM25's vocabulary / CSR construction, and the aur_kw_* argument checks."""

import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.bm25 import BM25Index, build_csr, query_csr, tokenize
from oracle.bm25_topk import Corpus, bm25_topk

WORDS = ["disk", "full", "cpu", "spike", "oom", "kill", "pod", "node", "error", "timeout", "db", "latency", "x1", "42"]


class Mirror:
    """Append log of the documents as the device store keeps them: upserts tombstone, removes tombstone."""

    def __init__(self):
        self.vocab = {}
        self.terms, self.tfs, self.offsets = [], [], [0]
        self.ids, self.live, self.user, self.org = [], [], [], []
        self.row_of = {}

    def add(self, doc_id, text, user=0, org=-1):
        if doc_id in self.row_of:
            self.live[self.row_of[doc_id]] = False
        t, f, _ = build_csr(self.vocab, [text])
        self.terms += t.tolist()
        self.tfs += f.tolist()
        self.offsets.append(len(self.terms))
        self.row_of[doc_id] = len(self.ids)
        self.ids.append(doc_id)
        self.live.append(True)
        self.user.append(user)
        self.org.append(org)

    def remove(self, doc_id):
        r = self.row_of.pop(doc_id, None)
        if r is not None:
            self.live[r] = False

    def corpus(self):
        return Corpus(self.terms, self.tfs, self.offsets, self.ids, self.live, self.user, self.org)


@pytest.fixture(scope="module", autouse=True)
def loop_path():
    """Every BM25Index here scores on its loop path: the contract's definition."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        yield


text_st = st.lists(st.sampled_from(WORDS), min_size=0, max_size=12).map(" ".join)
op_st = st.tuples(st.sampled_from(["add", "add", "add", "remove"]), st.integers(0, 15), text_st,
                  st.integers(0, 3), st.integers(-1, 2))


@settings(max_examples=80, deadline=None)
@given(ops=st.lists(op_st, min_size=1, max_size=40), query=text_st, scope=st.integers(-1, 3), k=st.integers(1, 20))
def test_oracle_equals_loop_path(ops, query, scope, k):
    host, mirror = BM25Index(), Mirror()
    codes = {}
    for op, doc, text, user, org in ops:
        if op == "add":
            host.add(doc, text)
            mirror.add(doc, text, user, org)
            codes[doc] = (user, org)
        else:
            host.remove(doc)
            mirror.remove(doc)
            codes.pop(doc, None)
    cp = mirror.corpus()
    q_terms, q_off = query_csr(mirror.vocab, [query])
    if scope < 0:
        allowed, q_user, q_org = None, None, None
    else:
        qo = scope - 1                                          # -1 = no org
        allowed = {d for d, (u, o) in codes.items() if u == scope or (qo >= 0 and o == qo)}
        q_user, q_org = np.array([scope], np.int32), np.array([qo], np.int32)
    want = host.search(query, k, allowed=allowed)
    ids, scores = bm25_topk(cp, q_terms, q_off, k, q_user, q_org)
    got = [(int(i), float(s)) for i, s in zip(ids[0], scores[0]) if i >= 0]
    assert got == want                                            # ids and fp64 scores bit-identical
    assert all(i == -1 and s == -np.inf for i, s in zip(ids[0][len(got):], scores[0][len(got):]))


@settings(max_examples=30, deadline=None)
@given(docs=st.lists(text_st, min_size=1, max_size=20), allow=st.sets(st.integers(0, 19)), query=text_st)
def test_oracle_allow_list_equals_loop_path(docs, allow, query):
    host, mirror = BM25Index(), Mirror()
    for i, t in enumerate(docs):
        host.add(i, t)
        mirror.add(i, t)
    q_terms, q_off = query_csr(mirror.vocab, [query])
    ids, scores = bm25_topk(mirror.corpus(), q_terms, q_off, 8, allow_ids=sorted(allow))
    got = [(int(i), float(s)) for i, s in zip(ids[0], scores[0]) if i >= 0]
    assert got == host.search(query, 8, allowed=set(allow))


def test_build_csr_vocabulary_and_order():
    vocab = {}
    t, f, off = build_csr(vocab, ["b a b", "", "c a", "A-b!"])
    assert vocab == {"b": 0, "a": 1, "c": 2}                    # first-seen order, grow-only
    assert off.tolist() == [0, 2, 2, 4, 6]
    assert t.tolist() == [0, 1, 1, 2, 0, 1]                     # ascending ids inside each document
    assert f.tolist() == [2, 1, 1, 1, 1, 1]
    assert t.dtype == np.int32 and f.dtype == np.int32 and off.dtype == np.int64
    t2, _, _ = build_csr(vocab, ["d b"])
    assert vocab["d"] == 3 and t2.tolist() == [0, 3]
    q, qo = query_csr(vocab, ["c b c zzz", "zzz", "a"])
    assert q.tolist() == [0, 2, 1] and qo.tolist() == [0, 2, 2, 3]   # sorted(set(tokenize)) by word, unknown dropped


def test_build_csr_large_tf():
    vocab = {}
    t, f, off = build_csr(vocab, ["w " * 70000])
    assert t.tolist() == [0] and f.tolist() == [70000] and sum(1 for _ in tokenize("w " * 3)) == 3


def test_keyword_abi_rejects_bad_arguments():
    from aurora_b200.build import build_native

    build_native()
    lib = N.load()
    h = C.c_void_p()
    assert lib.aur_kw_open(0, 100, 0, None) == N.AUR_ERR_INVALID
    assert lib.aur_kw_open(0, 0, 0, C.byref(h)) == N.AUR_ERR_INVALID
    assert lib.aur_kw_open(0, 100, -1, C.byref(h)) == N.AUR_ERR_INVALID
    assert lib.aur_kw_close(None) == N.AUR_OK
    assert lib.aur_kw_add(None, None, None, None, None, None, None, 1) == N.AUR_ERR_INVALID
    assert lib.aur_kw_remove(None, None, 0, None) == N.AUR_ERR_INVALID
    assert lib.aur_kw_compact(None, None) == N.AUR_ERR_INVALID
    assert lib.aur_kw_get_stats(None, None) == N.AUR_ERR_INVALID
    out_s, out_i = np.empty(4), np.empty(4, np.int64)
    off = np.array([0, 0], np.int64)
    args = lambda k, nq=1: (None, None, off.ctypes.data_as(C.c_void_p), nq, k, None, None, None, 0,   # noqa: E731
                            out_s.ctypes.data_as(C.c_void_p), out_i.ctypes.data_as(C.c_void_p), None)
    assert lib.aur_kw_search(*args(1)) == N.AUR_ERR_INVALID
    assert b"null" in lib.aur_last_error()


def test_keyword_store_needs_a_device():
    lib = N.load()
    if lib.aur_device_count() > 0:
        pytest.skip("a GPU is present; the no-device behaviour is exercised on the CPU box")
    from aurora_b200.engine import KeywordIndex

    with pytest.raises(N.AuroraError) as e:
        KeywordIndex(128)
    assert e.value.code == N.AUR_ERR_NO_DEVICE
    with pytest.raises(N.AuroraError) as e:
        bm25.DeviceBM25(128)
    assert e.value.code == N.AUR_ERR_NO_DEVICE


def test_header_declares_the_keyword_stats_layout():
    import os
    import re

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "aurora_b200.h")).read()
    body = re.search(r"typedef struct aur_kw_stats \{(.*?)\} aur_kw_stats;", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S), re.S).group(1)
    names = [n.strip() for decl in body.split(";") if decl.strip() for n in decl.split(None, 1)[1].split(",")]
    assert names == [f for f, _ in N.AurKwStats._fields_]
    assert C.sizeof(N.AurKwStats) == 64
    assert re.search(r"#define AUR_ABI_VERSION 3\b", hdr)
