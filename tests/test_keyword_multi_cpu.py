"""The sharded keyword store's host side, without a GPU: aur_kw_search_multi's argument checks, MultiKeywordIndex's
id-mod-n routing over a recording double of KeywordIndex, the per-shard capacity rule it shares with MultiIndex, and
the fp64 k-way merge that folds the stores' lists."""

import ctypes as C

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import MultiIndex, MultiKeywordIndex, shard_capacity


@pytest.fixture(scope="module")
def lib():
    from aurora_b200.build import build_native

    build_native()
    return N.load()


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def test_search_multi_rejects_bad_store_lists_without_touching_a_device(lib):
    """Fake store pointers: every refusal happens before a store is dereferenced or a device is asked for."""
    qt, qo = np.array([1, 2], np.int32), np.array([0, 2], np.int64)
    out_s, out_i, snaps = np.empty(4), np.empty(4, np.int64), np.empty(65, np.int64)

    def call(stores, n, nq=1, k=4):
        return lib.aur_kw_search_multi(stores, n, _vp(qt), _vp(qo), nq, k, None, None, None, 0, _vp(out_s), _vp(out_i),
                                       _vp(snaps))

    fake = lambda *xs: (C.c_void_p * len(xs))(*xs)                     # noqa: E731
    assert call(None, 1) == N.AUR_ERR_INVALID
    assert call(fake(0x1000), 0) == N.AUR_ERR_INVALID
    assert call(fake(*range(0x1000, 0x1000 + 65 * 64, 64)), 65) == N.AUR_ERR_INVALID
    assert b"n_stores" in lib.aur_last_error()
    assert call(fake(0x1000, None, 0x2000), 3) == N.AUR_ERR_INVALID
    assert b"NULL" in lib.aur_last_error()
    assert call(fake(0x1000, 0x2000, 0x1000), 3) == N.AUR_ERR_INVALID
    assert b"twice" in lib.aur_last_error()
    # a well-formed store list with a bad query is refused by aur_kw_search's own checks, still before any store is read
    assert call(fake(0x1000, 0x2000), 2, nq=0) == N.AUR_ERR_INVALID
    assert call(fake(0x1000, 0x2000), 2, k=129) == N.AUR_ERR_UNSUPPORTED
    assert lib.aur_kw_search_multi(fake(0x1000), 1, _vp(qt), None, 1, 4, None, None, None, 0, _vp(out_s), _vp(out_i),
                                   None) == N.AUR_ERR_INVALID


class RecordingStore:
    """KeywordIndex's surface on the host: keeps every call and the documents it was given."""

    def __init__(self, capacity, postings_capacity, device):
        self.capacity, self.postings_capacity, self.device = capacity, postings_capacity, device
        self.calls = []
        self.docs = {}        # id -> (terms, tfs, user, org)
        self.dead = 0

    def add(self, ids, term_ids, tfs, offsets, user_codes=None, org_codes=None):
        assert offsets[0] == 0 and len(offsets) == len(ids) + 1 and offsets[-1] == len(term_ids) == len(tfs)
        self.calls.append(("add", list(map(int, ids)), np.asarray(offsets).tolist()))
        for i, d in enumerate(ids):
            if int(d) in self.docs:
                self.dead += 1
            sl = slice(offsets[i], offsets[i + 1])
            self.docs[int(d)] = (list(map(int, term_ids[sl])), list(map(int, tfs[sl])),
                                 0 if user_codes is None else int(user_codes[i]), -1 if org_codes is None else int(org_codes[i]))

    def remove(self, ids):
        self.calls.append(("remove", list(map(int, ids))))
        n = sum(1 for d in ids if self.docs.pop(int(d), None) is not None)
        self.dead += n
        return n

    def compact(self):
        self.calls.append(("compact",))
        n, self.dead = self.dead, 0
        return n

    def stats(self):
        live = len(self.docs)
        used = sum(len(t) for t, _, _, _ in self.docs.values())
        return {"docs": live + self.dead, "live": live, "capacity": self.capacity, "postings_used": used,
                "postings_allocated": used + 100, "total_len": sum(sum(f) for _, f, _, _ in self.docs.values()),
                "last_launches": 4, "last_ms": 0.5 + self.device, "last_terms": 3 + self.device, "last_spilled": 0}


def _docs(rng, n, vocab=50):
    terms, tfs, off = [], [], [0]
    for _ in range(n):
        t = np.unique(rng.integers(0, vocab, int(rng.integers(0, 6))))
        terms += t.tolist()
        tfs += rng.integers(1, 4, len(t)).tolist()
        off.append(len(terms))
    return np.array(terms, np.int32), np.array(tfs, np.int32), np.array(off, np.int64)


def _multi(n):
    return MultiKeywordIndex(1000, devices=list(range(n)), postings_capacity=5000,
                             store_factory=lambda cap, post, dev: RecordingStore(cap, post, dev))


@pytest.mark.parametrize("n", [1, 3, 8])
def test_documents_land_on_store_id_mod_n_with_rebased_offsets(n):
    rng = np.random.default_rng(n)
    mk = _multi(n)
    ids = rng.permutation(400)[:120].astype(np.int64)
    t, f, off = _docs(rng, len(ids))
    user, org = rng.integers(0, 5, len(ids)).astype(np.int32), rng.integers(-1, 3, len(ids)).astype(np.int32)
    mk.add(ids, t, f, off, user, org)
    for s, st in enumerate(mk.stores):
        assert st.device == s and st.capacity == shard_capacity(1000, n) and st.postings_capacity == shard_capacity(5000, n)
        mine = [int(d) for d in ids if d % n == s]
        assert sorted(st.docs) == sorted(mine)
        if mine:
            assert st.calls[0][1] == mine                                   # one append per store, batch order kept
        else:
            assert st.calls == []                                           # an empty store is not called
    for i, d in enumerate(ids):
        sl = slice(off[i], off[i + 1])
        assert mk.stores[d % n].docs[int(d)] == (t[sl].tolist(), f[sl].tolist(), int(user[i]), int(org[i]))


def test_upserts_and_removes_reach_the_owner():
    rng = np.random.default_rng(5)
    mk = _multi(3)
    ids = np.arange(30, dtype=np.int64)
    mk.add(ids, *_docs(rng, 30))
    up = np.array([4, 7, 29, 12], np.int64)
    t, f, off = _docs(rng, 4)
    mk.add(up, t, f, off)
    for i, d in enumerate(up):
        st = mk.stores[d % 3]
        assert st.docs[int(d)][:2] == (t[off[i]:off[i + 1]].tolist(), f[off[i]:off[i + 1]].tolist())
        assert int(d) in st.calls[-1][1]
    assert all(int(d) not in mk.stores[s].calls[-1][1] for d in up for s in range(3) if s != d % 3)
    gone = np.array([0, 1, 2, 3, 100, 29], np.int64)                       # 100: unknown, still routed to its owner
    assert mk.remove(gone) == 5
    for s, st in enumerate(mk.stores):
        assert st.calls[-1] == ("remove", [int(d) for d in gone if d % 3 == s])
    assert mk.compact() == 4 + 5


def test_stats_are_summed_with_a_list_per_store():
    rng = np.random.default_rng(2)
    mk = _multi(4)
    mk.add(np.arange(50, dtype=np.int64), *_docs(rng, 50))
    mk.remove(np.arange(0, 50, 7))
    s = mk.stats()
    per = [st.stats() for st in mk.stores]
    assert s["stores"] == per and len(per) == 4
    for key in ("docs", "live", "capacity", "postings_used", "postings_allocated", "total_len"):
        assert s[key] == sum(p[key] for p in per), key
    assert s["live"] == 50 - len(range(0, 50, 7)) and s["docs"] == 50
    assert s["last_launches"] == 16 and s["last_ms"] == 3.5 and s["last_terms"] == 6


@pytest.mark.parametrize("cap", [1, 63, 64, 1000, 4096, 1 << 20, 100_000_007])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_shard_capacity_is_multi_index_s_rule(cap, n):
    per = (cap + n - 1) // n
    assert shard_capacity(cap, n) == per + max(64, per // 8)
    seen = []

    class Shard:
        def __init__(self, c):
            seen.append(c)

        def close(self):
            pass

    MultiIndex(16, cap, devices=list(range(n)), shard_factory=lambda d, c, dev: Shard(c)).close()
    assert seen == [per + max(64, per // 8)] * n


def test_fp64_merge_orders_by_score_then_id(lib):
    """Scores one ulp apart in fp64 (one float32 value) keep their fp64 order; exact ties go by id; padding last."""
    one = 1.0
    up = np.nextafter(one, 2.0)
    assert np.float32(up) == np.float32(one)
    sc = np.array([[[one, 0.5, -np.inf]], [[up, one, 0.5]]])                # two lists, one query, k_in 3
    ids = np.array([[[3, 1, -1]], [[9, 2, 0]]], np.int64)
    out_s, out_i = np.empty((1, 6)), np.empty((1, 6), np.int64)
    assert lib.aur_merge_topk_host_f64(_vp(sc), _vp(ids), 2, 1, 3, 6, _vp(out_s), _vp(out_i)) == 0
    assert out_i[0].tolist() == [9, 2, 3, 0, 1, -1]
    assert out_s[0].view(np.int64).tolist() == np.array([up, one, one, 0.5, 0.5, -np.inf]).view(np.int64).tolist()
    rng = np.random.default_rng(0)
    for n_lists, nq, k_in, k_out in ((3, 7, 5, 5), (8, 20, 32, 32), (2, 4, 6, 9), (64, 3, 4, 10)):
        base = np.round(rng.standard_normal((n_lists, nq, k_in)), 1)
        sc = base + rng.integers(0, 3, base.shape) * 2.0 ** -45           # near-ties below float32 resolution
        ids = rng.permutation(n_lists * nq * k_in).reshape(n_lists, nq, k_in).astype(np.int64)
        for l in range(n_lists):
            for q in range(nq):
                o = np.lexsort((ids[l, q], -sc[l, q]))
                sc[l, q], ids[l, q] = sc[l, q][o], ids[l, q][o]
                if rng.random() < 0.3:
                    cut = rng.integers(0, k_in + 1)
                    ids[l, q, cut:], sc[l, q, cut:] = -1, -np.inf
        out_s, out_i = np.empty((nq, k_out)), np.empty((nq, k_out), np.int64)
        assert lib.aur_merge_topk_host_f64(_vp(sc), _vp(ids), n_lists, nq, k_in, k_out, _vp(out_s), _vp(out_i)) == 0
        I, S = np.concatenate(list(ids), axis=1), np.concatenate(list(sc), axis=1)
        order = np.lexsort((np.where(I < 0, np.iinfo(np.int64).max, I), -S), axis=1)
        wi, ws = np.take_along_axis(I, order, axis=1), np.take_along_axis(S, order, axis=1)
        if k_out > wi.shape[1]:
            wi = np.concatenate([wi, np.full((nq, k_out - wi.shape[1]), -1)], axis=1)
            ws = np.concatenate([ws, np.full((nq, k_out - ws.shape[1]), -np.inf)], axis=1)
        wi, ws = wi[:, :k_out], ws[:, :k_out]
        ws[wi < 0] = -np.inf
        assert np.array_equal(out_i, wi) and np.array_equal(out_s.view(np.int64), ws.view(np.int64))
    assert lib.aur_merge_topk_host_f64(None, None, 1, 1, 1, 1, None, None) == N.AUR_ERR_INVALID
