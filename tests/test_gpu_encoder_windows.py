"""Texts longer than the position table on the device: aur_encode_texts and aur_encode_append_texts_multi against
oracle/window_mean.py applied to the window vectors Encoder.encode_packed gives, bit for bit (fp32 and bf16).  A text's
window vectors do not depend on which sequences share their batch (test_gpu_encoder_multi.py shows it), so the oracle
may take them from any batching."""

import ctypes as C
import json
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from aurora_b200 import _native as N
from aurora_b200.encoder import Encoder, EncoderConfig, TextEncoder, encode_append_multi
from aurora_b200.engine import Index, MultiIndex, shard_capacity, to_bf16_bits
from oracle import bert_encoder as B
from oracle.cosine_topk import bf16_bits_to_f32, cosine_topk
from oracle.window_mean import fold_texts

SMALL = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=64, pool="cls")
SMALL_MEAN_RAW = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=64, pool="mean", normalize=False)
MINILM = B.BertConfig(hidden=384, layers=6, heads=12, inter=1536, max_pos=128, pool="mean")   # head dim 32
MINILM_RAW = B.BertConfig(hidden=384, layers=2, heads=12, inter=1536, max_pos=128, pool="cls", normalize=False)
BGE = B.BGE_BASE


def _mirror(c: B.BertConfig) -> EncoderConfig:
    return EncoderConfig(hidden=c.hidden, layers=c.layers, heads=c.heads, inter=c.inter, vocab=c.vocab, max_pos=c.max_pos,
                         type_vocab=c.type_vocab, ln_eps=c.ln_eps, pool=c.pool, normalize=c.normalize)


_WEIGHTS = {}


def _encoder(c, max_tokens=4096, max_seqs=64, device=0) -> Encoder:
    if c not in _WEIGHTS:
        _WEIGHTS.clear()
        _WEIGHTS[c] = B.init_weights(c, seed=7, bf16=True)
    enc = Encoder(_mirror(c), max_tokens=max_tokens, max_seqs=max_seqs, device=device)
    enc.load_weights(_WEIGHTS[c])
    return enc


def _texts(c, wins, seed):
    """Windows of texts with wins[j] windows each, as aur_tokenize_windows lays them out: every window but a text's
    last is max_pos long, the last 3 .. max_pos; (tokens, cu_seqlens, cu_texts)."""
    rng = np.random.default_rng(seed)
    cls_id, sep_id, lo = (101, 102, 1000) if c.vocab > 2000 else (1, 2, 3)
    seqs = []
    for w in wins:
        for k in range(w):
            n = c.max_pos if k < w - 1 else int(rng.integers(3, c.max_pos + 1))
            s = rng.integers(lo, c.vocab, size=n).astype(np.int32)
            s[0], s[-1] = cls_id, sep_id
            seqs.append(s)
    cu = np.zeros(len(seqs) + 1, np.int32)
    cu[1:] = np.cumsum([len(s) for s in seqs])
    ct = np.zeros(len(wins) + 1, np.int32)
    ct[1:] = np.cumsum(wins)
    return np.concatenate(seqs), cu, ct


def _oracle(enc, c, tok, cu, ct):
    v = enc.encode([tok[cu[i]:cu[i + 1]] for i in range(len(cu) - 1)])           # window vectors, any batching
    f = fold_texts(v, ct, c.normalize)
    return f, to_bf16_bits(f)


WINS = [1, 3, 1, 2, 5, 1, 1, 7, 2, 1]


@pytest.mark.parametrize("c", [SMALL, SMALL_MEAN_RAW, MINILM, MINILM_RAW, BGE],
                         ids=["dh64-cls-norm", "dh64-mean-raw", "dh32-mean-norm", "dh32-cls-raw", "bge-base"])
def test_encode_texts_is_the_oracle_over_the_window_vectors(c):
    enc = _encoder(c, max_tokens=8192 if c is BGE else 4096)
    tok, cu, ct = _texts(c, WINS if c is not BGE else [1, 2, 9, 1, 3], seed=c.hidden + c.layers)
    f_ref, b_ref = _oracle(enc, c, tok, cu, ct)
    f = enc.encode_texts(tok, cu, ct)
    b = enc.encode_texts(tok, cu, ct, bf16=True)
    assert np.array_equal(f.view(np.uint32), f_ref.view(np.uint32))
    assert np.array_equal(b, b_ref)
    one = np.nonzero(np.diff(ct) == 1)[0]                                           # one-window texts: aur_encode's vector
    direct = enc.encode_packed(tok, cu)
    assert np.array_equal(f[one].view(np.uint32), direct[ct[one]].view(np.uint32))
    assert np.array_equal(b[one], enc.encode_packed(tok, cu, bf16=True)[ct[one]])
    enc.close()


def test_fitting_texts_launch_what_aur_encode_launches():
    enc = _encoder(SMALL)
    tok, cu, ct = _texts(SMALL, [1] * 12, seed=3)
    enc.encode_packed(tok, cu)
    plain = enc.stats()["launches"]
    enc.encode_texts(tok, cu, ct)
    assert enc.stats()["launches"] == plain
    tok, cu, ct = _texts(SMALL, [1, 2, 1], seed=4)
    enc.encode_texts(tok, cu, ct)
    assert enc.stats()["launches"] == plain + 1                                     # + window_fold_kernel
    enc.close()


def test_a_text_spanning_many_batches_gives_the_bits_of_one_batch():
    big = _encoder(MINILM, max_tokens=8192, max_seqs=64)
    tiny = _encoder(MINILM, max_tokens=2 * MINILM.max_pos, max_seqs=1)             # one window per batch
    two = _encoder(MINILM, max_tokens=3 * MINILM.max_pos, max_seqs=3)
    tok, cu, ct = _texts(MINILM, [9, 1, 4, 1, 1, 6], seed=5)
    want = big.encode_texts(tok, cu, ct)
    for e in (tiny, two):
        assert np.array_equal(e.encode_texts(tok, cu, ct).view(np.uint32), want.view(np.uint32))
        assert np.array_equal(e.encode_texts(tok, cu, ct, bf16=True), to_bf16_bits(want))
    # the fused append with per-call limits that cut every text's windows apart stores the same rows
    a, b = Index(MINILM.hidden, 64), Index(MINILM.hidden, 64)
    ids = np.arange(len(ct) - 1, dtype=np.int64)
    encode_append_multi([big], [a], tok, cu, ids, None, None, 2 * MINILM.max_pos, 1, cu_texts=ct)
    encode_append_multi([big], [b], tok, cu, ids, cu_texts=ct)
    assert np.array_equal(a.read_rows(0, len(ids))[0], to_bf16_bits(want))
    assert np.array_equal(b.read_rows(0, len(ids))[0], to_bf16_bits(want))
    for x in (a, b, big, tiny, two):
        x.close()


# ---------------------------------------------------------------------- multi-shard append
def _exports(index):
    return [sh.export_raw() for sh in (index.shards if isinstance(index, MultiIndex) else [index])]


def _calls(c, n):
    """Two calls: the first repeats an id, leaves the last shard empty (n > 1) and gives shard 0 one 9-window text as
    its whole share; the second upserts ids of the first and reaches every shard.  Tenant codes on every row."""
    out = []
    rng = np.random.default_rng(n)
    wins1 = [9, 1, 2, 1, 3, 1, 1, 4]
    ids1 = np.array([0] + [n * i + 1 for i in range(1, 8)], np.int64)            # id mod n: 0, then 1 (n > 1)
    ids1[6] = ids1[2]
    wins2 = [1, 2, 1, 5, 1, 1, 3]
    ids2 = np.concatenate([ids1[[1, 3]], 50 + np.arange(5)]).astype(np.int64)
    for k, (wins, ids) in enumerate(((wins1, ids1), (wins2, ids2))):
        tok, cu, ct = _texts(c, wins, seed=10 * n + k)
        out.append((tok, cu, ct, ids, rng.integers(0, 5, len(ids)).astype(np.int32), rng.integers(-1, 3, len(ids)).astype(np.int32)))
    return out


CASES = [(n, dtype, limits) for n in (1, 2, 3) for dtype in ("bf16", "int8") for limits in ((0, 0), (200, 3))]


@pytest.mark.parametrize("n,dtype,limits", CASES, ids=[f"n{n}-{d}-{l[0]}" for n, d, l in CASES])
def test_multi_texts_append_stores_encode_texts_rows(n, dtype, limits):
    enc = _encoder(SMALL)
    encs = [enc] + [enc.replicate(0) for _ in range(n - 1)]
    fused = MultiIndex(SMALL.hidden, 256, devices=[0] * n, dtype=dtype)
    host = MultiIndex(SMALL.hidden, 256, devices=[0] * n, dtype=dtype)
    for k, (tok, cu, ct, ids, u, o) in enumerate(_calls(SMALL, n)):
        encode_append_multi(encs, fused.shards, tok, cu, ids, u, o, *limits, cu_texts=ct)
        host.add(enc.encode_texts(tok, cu, ct, bf16=True), ids, u, o)
        if k == 0 and n > 1:
            assert fused.shards[0].stats()["rows"] == 1                            # one 9-window text is shard 0's share
            assert n == 2 or fused.shards[2].stats()["rows"] == 0                   # an empty share
    for s, (x, y) in enumerate(zip(_exports(fused), _exports(host))):
        for name, u_, v_ in zip(("rows", "ids", "user", "org", "live"), x, y):
            assert np.array_equal(u_, v_), f"shard {s}: {name} differ"
    # each shard's rows are in input order
    tok, cu, ct, ids, _, _ = _calls(SMALL, n)[0]
    for s, sh in enumerate(fused.shards):
        mine = [int(i) for i in ids if i % n == s]
        assert sh.read_rows(0, len(mine))[1].tolist() == mine
    for x in [fused, host] + encs[1:] + [enc]:
        x.close()


@pytest.mark.skipif(N.load().aur_device_count() < 2, reason="needs two GPUs")
def test_one_shard_per_gpu():
    enc = _encoder(SMALL, device=0)
    rep = enc.replicate(1)
    fused = MultiIndex(SMALL.hidden, 256, devices=[0, 1])
    host = MultiIndex(SMALL.hidden, 256, devices=[0, 1])
    for tok, cu, ct, ids, u, o in _calls(SMALL, 2):
        encode_append_multi([enc, rep], fused.shards, tok, cu, ids, u, o, 200, 3, cu_texts=ct)
        host.add(enc.encode_texts(tok, cu, ct, bf16=True), ids, u, o)
    for x, y in zip(_exports(fused), _exports(host)):
        assert all(np.array_equal(u_, v_) for u_, v_ in zip(x, y))
    for x in (fused, host, rep, enc):
        x.close()


def _call(encs, shards, tok, cu, ct, ids, n_texts=None, limits=(0, 0)):
    n = len(shards)
    eh = (C.c_void_p * n)(*[e._h.value for e in encs])
    sh = (C.c_void_p * n)(*[s._h.value for s in shards])
    tok, cu, ct = (np.ascontiguousarray(a, np.int32) for a in (tok, cu, ct))
    ids = np.ascontiguousarray(ids, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)      # noqa: E731
    return N.load().aur_encode_append_texts_multi(eh, sh, n, p(tok), p(cu), len(cu) - 1, p(ct),
                                                  len(ct) - 1 if n_texts is None else n_texts, p(ids), None, None, *limits)


def test_rejections_leave_every_shard_and_encoder_untouched():
    enc = _encoder(SMALL, max_tokens=1024, max_seqs=16)
    rep = enc.replicate(0)
    mi = MultiIndex(SMALL.hidden, 30, devices=[0, 0])
    room = shard_capacity(30, 2) - 2                                               # shard 0 holds ids 0 and 2 below
    shards, encs = mi.shards, [enc, rep]
    tok, cu, ct = _texts(SMALL, [1, 3, 2, 1], seed=8)
    ids = np.arange(4, dtype=np.int64)
    assert _call(encs, shards, tok, cu, ct, ids) == N.AUR_OK                        # something to keep unchanged
    state = lambda: ([s.stats()["rows"] for s in shards], [e.stats() for e in encs], [s.export_raw()[0].tobytes() for s in shards])   # noqa: E731
    before = state()
    bad_tok = tok.copy()
    bad_tok[-1] = SMALL.vocab
    many_t, many_cu, many_ct = _texts(SMALL, [2] * (room + 1), seed=9)
    cases = [
        ("cu_texts[0] != 0", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, np.array([1, 1, 4, 6, 7]), ids)),
        ("a text with no window", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, np.array([0, 1, 1, 6, 7]), ids)),
        ("decreasing", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, np.array([0, 4, 3, 6, 7]), ids)),
        ("last != n_seq", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, np.array([0, 1, 4, 6, 6]), ids)),
        ("n_texts != cu_texts", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, ct, ids, n_texts=3)),
        ("bad token id", N.AUR_ERR_INVALID, lambda: _call(encs, shards, bad_tok, cu, ct, ids)),
        ("negative id", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, ct, np.array([0, 1, -2, 3]))),
        ("room counted in texts", N.AUR_ERR_NOMEM,
         lambda: _call(encs, shards, many_t, many_cu, many_ct, 2 * np.arange(room + 1))),
        ("window longer than a call", N.AUR_ERR_NOMEM, lambda: _call(encs, shards, tok, cu, ct, ids, limits=(32, 0))),
        ("limit above the workspace", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, ct, ids, limits=(2048, 0))),
    ]
    for name, code, fn in cases:
        assert fn() == code, (name, N.load().aur_last_error())
        assert state() == before, name
    e_before = enc.stats()
    with pytest.raises(N.AuroraError):                                              # aur_encode_texts checks the same way
        enc.encode_texts(tok, cu, np.array([0, 1, 1, 6, 7]))
    assert enc.stats() == e_before
    assert _call(encs, shards, tok, cu, ct, ids, limits=(128, 2)) == N.AUR_OK       # still usable afterwards
    # room is counted in texts: as many two-window texts as shard 0 has rows left fit
    left = shard_capacity(30, 2) - shards[0].stats()["rows"]
    assert _call(encs, shards, many_t[:many_cu[2 * left]], many_cu[:2 * left + 1], many_ct[:left + 1], 2 * np.arange(left)) == N.AUR_OK
    assert shards[0].stats()["rows"] == shard_capacity(30, 2)
    for x in (mi, rep, enc):
        x.close()


# ---------------------------------------------------------------------- the knowledge base
def _kb_encoder():
    from aurora_b200.wordpiece import NativeTokenizer, basic_tokenize

    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "chunker_ref.json"), encoding="utf-8"))
    docs = [d for d in gold["documents"] if d["chunks"]]
    finding = ("Discovery finding: kube-system/coredns pod restarts on node ip-10-0-3-17.ec2.internal; " +
               " ".join(f"10.0.{i % 7}.{i} sha256:{i * 7919:08x} /var/log/pods/coredns-{i}.log" for i in range(260)))
    words = sorted({w for d in docs for ch in d["chunks"] for w in basic_tokenize(ch["heading_context"] + " " + ch["content"])} |
                   set(basic_tokenize(finding)))
    pieces = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + [w for w in words if len(w) <= 100]
    c = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=len(pieces), max_pos=512, pool="cls")
    enc = Encoder(_mirror(c), max_tokens=4096, max_seqs=32)
    enc.load_weights(B.init_weights(c, seed=11, bf16=True))
    return TextEncoder(enc, NativeTokenizer(pieces)), docs, finding


def _live(index):
    out = {}
    for rows, ids, user, org, live in _exports(index):
        for i in np.nonzero(live > 0)[0]:
            out[int(ids[i])] = (rows[i].tobytes(), int(user[i]), int(org[i]))
    return out


def test_knowledge_base_ingests_over_long_texts_on_the_device(tmp_path, monkeypatch):
    from aurora_b200 import retriever as R

    te, docs, finding = _kb_encoder()
    assert len(te._windows(finding)) >= 3
    guard = {"on": True}                                                            # off only while a snapshot's rows load
    for cls in (Index, MultiIndex):
        orig = cls.add

        def add(self, *a, _orig=orig, **k):
            if guard["on"]:
                raise AssertionError("host vectors must not be added")
            return _orig(self, *a, **k)
        monkeypatch.setattr(cls, "add", add)

    def load(path):
        guard["on"] = False
        try:
            return R.KnowledgeBase.load(path, te, capacity=1024, **({} if loader is None else {"index_loader": loader}))
        finally:
            guard["on"] = True
    for name, factory, loader in (("single", None, None),
                                  ("multi", lambda d, c: MultiIndex(d, c, devices=[0, 0, 0]),
                                   lambda p, cap: MultiIndex.load(p, capacity=cap, devices=[0, 0, 0]))):
        kw = {} if factory is None else {"index_factory": factory}
        kb = R.KnowledgeBase(te, capacity=1024, **kw)
        snap = str(tmp_path / name)
        all_docs = [(f"u{i % 2}", f"doc-{d['name']}", d["name"], d["chunks"]) for i, d in enumerate(docs)]
        all_docs.append(("u1", "finding-1", "discovery.json", [{"chunk_index": 0, "content": finding, "heading_context": ""}]))
        for i, d in enumerate(all_docs):
            if i == 2:
                kb.save(snap)
                kb.attach_wal(os.path.join(snap, "mutations.log"))
            assert kb.insert(*d, org_id="o1") == len(d[3])
        hits = kb.query(finding, 1, user_id="u1", alpha=1.0)
        assert hits and hits[0].properties["document_id"] == "finding-1" and hits[0].metadata.score > 0.999
        # the stored row is encode()'s vector for the same text, as bf16
        q = te.encode([finding])
        assert q[0].tobytes() == te._enc.encode_texts(*te._tok.encode_windows([finding], 512))[0].tobytes()
        rows = _live(kb.index)
        again = load(snap)
        assert again.attach_wal(os.path.join(snap, "mutations.log")) == len(all_docs) - 2
        assert _live(again.index) == rows
        kb.save(str(tmp_path / (name + "-2")))
        assert _live(load(str(tmp_path / (name + "-2"))).index) == rows


def test_searches_while_over_long_texts_are_ingested():
    """A writer inserts over-long texts through the multi-shard append while three readers search every shard; every
    answer equals the oracle's top-k over exactly the prefix aur_search_ex reports."""
    from aurora_b200 import retriever as R

    te, docs, finding = _kb_encoder()
    kb = R.KnowledgeBase(te, capacity=2048, index_factory=lambda d, c: MultiIndex(d, c, devices=[0, 0, 0]))
    k = 6
    Q = bf16_bits_to_f32(to_bf16_bits(te.encode([finding[:300], "runbook restart", finding[-2000:]])))
    rng = np.random.default_rng(2)
    parts = finding.split(" ")
    texts = [" ".join(rng.choice(parts, size=int(rng.integers(400, 1500)))) for _ in range(40)]
    errors, done, answers = [], threading.Event(), []

    def writer():
        try:
            for i in range(0, len(texts), 4):
                kb.insert("u1", f"doc{i}", "f.txt", [{"chunk_index": j, "content": t, "heading_context": ""}
                                                      for j, t in enumerate(texts[i:i + 4])])
        except Exception as e:      # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader():
        try:
            mine = []
            while not done.is_set() or len(mine) < 2:
                for s, sh in enumerate(kb.index.shards):
                    ids, sc, snap = sh.search_snapshot(Q, k)
                    mine.append((s, snap, ids, sc))
            answers.append(mine)
        except Exception as e:      # pragma: no cover
            errors.append(e)

    ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errors, errors[0]
    ex = _exports(kb.index)
    snaps = set()
    for mine in answers:
        for s, snap, ids, sc in mine:
            rows, rid, _, _, live = ex[s]
            snaps.add(snap)
            if snap == 0:
                assert (ids == -1).all()
                continue
            oids, osc = cosine_topk(Q, bf16_bits_to_f32(rows[:snap]), k, ids=rid[:snap])
            assert np.array_equal(ids, oids), (s, snap)
            fin = np.isfinite(osc)
            assert np.array_equal(np.isfinite(sc), fin) and float(np.max(np.abs(sc[fin] - osc[fin]), initial=0)) <= 1e-6
    assert len(snaps) >= 3
    assert sum(sh.stats()["live"] for sh in kb.index.shards) == len(texts)
