"""Encoder replicas (aur_encoder_replicate) and the multi-shard fused ingest (aur_encode_append_multi) of a multi-GPU
knowledge base.  Nothing here has a tolerance: a replica's forward is its source's bit for bit, and the rows a shard
holds after the multi-shard append are, id for id and bit for bit, the rows the host route (encode, bf16 on the host,
MultiIndex.add) and a single shard's aur_encode_append store.  That rests on a sequence's output not depending on which
sequences share its batch (GEMM rows, per-sequence attention items, per-row LayerNorm, per-sequence pooling), which the
row comparisons below show rather than assume.  Everything runs on GPU 0 (MultiIndex(devices=[0, 0, 0])) except the
cases that need two GPUs."""

import ctypes as C
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

SMALL = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")
MINILM = B.MINILM_L6            # head dim 32: the padded wqkv / wo layouts
BGE = B.BGE_BASE


def _mirror(cfg_o: B.BertConfig) -> EncoderConfig:
    return EncoderConfig(hidden=cfg_o.hidden, layers=cfg_o.layers, heads=cfg_o.heads, inter=cfg_o.inter, vocab=cfg_o.vocab,
                         max_pos=cfg_o.max_pos, type_vocab=cfg_o.type_vocab, ln_eps=cfg_o.ln_eps, pool=cfg_o.pool,
                         normalize=cfg_o.normalize)


_WEIGHTS = {}


def _encoder(cfg_o, max_tokens=4096, max_seqs=64, device=0, seed=7) -> Encoder:
    key = (cfg_o, seed)
    if key not in _WEIGHTS:
        _WEIGHTS.clear()
        _WEIGHTS[key] = B.init_weights(cfg_o, seed=seed, bf16=True)
    enc = Encoder(_mirror(cfg_o), max_tokens=max_tokens, max_seqs=max_seqs, device=device)
    enc.load_weights(_WEIGHTS[key])
    return enc


def _two_gpus() -> bool:
    return N.load().aur_device_count() >= 2


def _ragged(cfg_o, n, seed, max_len=300):
    return B.synth_batch(cfg_o, n, seed, mean_len=max_len / 3, std_len=max_len / 4, min_len=1, max_len=max_len)


def _seqs(tok, cu):
    return [tok[cu[i]:cu[i + 1]] for i in range(len(cu) - 1)]


def _pack(seqs):
    cu = np.zeros(len(seqs) + 1, np.int32)
    cu[1:] = np.cumsum([len(s) for s in seqs])
    return (np.concatenate(seqs).astype(np.int32) if seqs else np.zeros(0, np.int32)), cu


def _exports(index):
    shards = index.shards if isinstance(index, MultiIndex) else [index]
    return [sh.export_raw() for sh in shards]


def _live_rows(index):
    """id -> (row bytes, user code, org code) of every live row."""
    out = {}
    for rows, ids, user, org, live in _exports(index):
        for i in np.nonzero(live > 0)[0]:
            out[int(ids[i])] = (rows[i].tobytes(), int(user[i]), int(org[i]))
    return out


def _assert_same_exports(a, b):
    for s, (x, y) in enumerate(zip(_exports(a), _exports(b))):
        for name, u, v in zip(("rows", "ids", "user", "org", "live"), x, y):
            assert np.array_equal(u, v), f"shard {s}: {name} differ"


# ---------------------------------------------------------------------- replicas
@pytest.mark.parametrize("cfg_o", [SMALL, MINILM], ids=["dh64", "dh32"])
def test_replica_forward_is_the_source_forward(cfg_o):
    tok, cu = _ragged(cfg_o, 13, seed=3)
    src = _encoder(cfg_o)
    want_f32, want_bf16 = src.encode_packed(tok, cu), src.encode_packed(tok, cu, bf16=True)
    rep = src.replicate(0)
    src.close()                                              # the replica lives on without its source
    rep2 = rep.replicate(0)                                   # a replica of a replica
    for r in (rep, rep2):
        assert np.array_equal(r.encode_packed(tok, cu).view(np.uint32), want_f32.view(np.uint32))
        assert np.array_equal(r.encode_packed(tok, cu, bf16=True), want_bf16)
    rep.close()
    assert np.array_equal(rep2.encode_packed(tok, cu, bf16=True), want_bf16)
    rep2.close()


def test_replicate_rejects_a_partly_loaded_encoder_and_a_bad_device():
    w = B.init_weights(SMALL, seed=7, bf16=True)
    with Encoder(_mirror(SMALL), max_tokens=1024, max_seqs=8) as enc:
        enc.load_weights({k: v for k, v in w.items() if k != "l1.wo"})
        with pytest.raises(N.AuroraError) as e:
            enc.replicate(0)
        assert e.value.code == N.AUR_ERR_INVALID and "l1.wo" in str(e.value)
        enc.load_weights({"l1.wo": w["l1.wo"]})
        with pytest.raises(N.AuroraError) as e:
            enc.replicate(N.load().aur_device_count())
        assert e.value.code == N.AUR_ERR_INVALID
        h = C.c_void_p()
        assert N.load().aur_encoder_replicate(enc._h, 0, None) == N.AUR_ERR_INVALID
        assert N.load().aur_encoder_replicate(None, 0, C.byref(h)) == N.AUR_ERR_INVALID and not h.value


# ---------------------------------------------------------------------- rows unchanged
def _calls(cfg_o, seed):
    """Two ingest calls over 3 shards: the first leaves shard 2 empty and repeats an id; the second upserts ids of the
    first, repeats one inside the call and reaches every shard.  Tenant codes on every row."""
    tok1, cu1 = _ragged(cfg_o, 20, seed)
    ids1 = np.array([3 * i + (i % 2) for i in range(20)], np.int64)          # id mod 3 in {0, 1}
    ids1[7] = ids1[2]
    tok2, cu2 = _ragged(cfg_o, 15, seed + 1)
    ids2 = np.concatenate([ids1[[0, 4, 9]], 100 + np.arange(12)]).astype(np.int64)
    ids2[10] = ids2[5]
    rng = np.random.default_rng(seed)
    return [(tok, cu, ids, rng.integers(0, 5, len(ids)).astype(np.int32), rng.integers(-1, 3, len(ids)).astype(np.int32))
            for tok, cu, ids in ((tok1, cu1, ids1), (tok2, cu2, ids2))]


CASES = [(SMALL, dtype, share, limits) for dtype in ("bf16", "int8") for share in ("shared", "replicas")
         for limits in ((0, 0), (600, 3))] + [(MINILM, "bf16", "replicas", (700, 4)), (BGE, "int8", "replicas", (1500, 5))]


@pytest.mark.parametrize("cfg_o,dtype,share,limits", CASES,
                         ids=[f"{'small' if c is SMALL else 'minilm' if c is MINILM else 'bge'}-{d}-{s}-{l[0]}"
                              for c, d, s, l in CASES])
def test_multi_append_stores_the_host_routes_rows(cfg_o, dtype, share, limits):
    enc = _encoder(cfg_o, max_tokens=4096, max_seqs=64)
    encs = [enc, enc, enc] if share == "shared" else [enc, enc.replicate(0), enc.replicate(0)]
    fused = MultiIndex(cfg_o.hidden, 256, devices=[0, 0, 0], dtype=dtype)
    host = MultiIndex(cfg_o.hidden, 256, devices=[0, 0, 0], dtype=dtype)
    single = Index(cfg_o.hidden, 256, dtype=dtype)
    for tok, cu, ids, u, o in _calls(cfg_o, seed=11):
        encode_append_multi(encs, fused.shards, tok, cu, ids, u, o, *limits)
        host.add(to_bf16_bits(enc.encode(_seqs(tok, cu))), ids, u, o)            # the host route
        enc.encode_append(single, tok, cu, ids, u, o)                            # one shard, one aur_encode_append
    _assert_same_exports(fused, host)
    assert [sh.stats()["rows"] for sh in fused.shards][2] > 0
    assert _live_rows(fused) == _live_rows(single)
    for s, (rows, ids, _, _, _) in enumerate(_exports(fused)):
        assert np.all(ids % 3 == s)
    # the shard stats and the pool agree on what was appended
    assert sum(sh.stats()["live"] for sh in fused.shards) == single.stats()["live"]
    for ix in (fused, host, single):
        ix.close()


def test_multi_append_with_one_shard_is_encode_append():
    enc = _encoder(SMALL, max_tokens=1024, max_seqs=8)
    tok, cu = _ragged(SMALL, 30, seed=5)
    ids = np.arange(30, dtype=np.int64)
    a, b = Index(SMALL.hidden, 64), Index(SMALL.hidden, 64)
    encode_append_multi([enc], [a], tok, cu, ids)
    seqs = _seqs(tok, cu)
    i = 0
    while i < len(seqs):                      # the greedy workspace batches, one aur_encode_append each
        j, t = i, 0
        while j < len(seqs) and j - i < 8 and t + len(seqs[j]) <= 1024:
            t += len(seqs[j]); j += 1
        enc.encode_append(b, *_pack(seqs[i:j]), ids[i:j])
        i = j
    _assert_same_exports(a, b)


# ---------------------------------------------------------------------- rejections
def _state(shards, encs):
    return [sh.stats()["rows"] for sh in shards], [e.stats() for e in encs]


def _call(encs, shards, tok, cu, ids, n=None, limits=(0, 0)):
    n = len(shards) if n is None else n
    eh = (C.c_void_p * max(n, 1))(*[e._h.value for e in encs][:n])
    sh = (C.c_void_p * max(n, 1))(*[s._h.value for s in shards][:n])
    tok = np.ascontiguousarray(tok, np.int32)
    cu = np.ascontiguousarray(cu, np.int32)
    ids = np.ascontiguousarray(ids, np.int64)
    return N.load().aur_encode_append_multi(eh, sh, n, tok.ctypes.data_as(C.c_void_p), cu.ctypes.data_as(C.c_void_p),
                                            len(cu) - 1, ids.ctypes.data_as(C.c_void_p), None, None, *limits)


def test_rejections_leave_every_shard_and_encoder_untouched():
    enc = _encoder(SMALL, max_tokens=1024, max_seqs=16)
    rep = enc.replicate(0)
    mi = MultiIndex(SMALL.hidden, 60, devices=[0, 0, 0])
    shards = mi.shards
    tok, cu = _ragged(SMALL, 12, seed=9, max_len=200)
    ids = np.arange(12, dtype=np.int64)
    encode_append_multi([enc, rep, enc], shards, tok, cu, ids)                   # something to keep unchanged
    encs = [enc, rep, enc]
    other = Encoder(_mirror(B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="mean")),
                    max_tokens=1024, max_seqs=16)
    other.load_weights(B.init_weights(SMALL, seed=7, bf16=True))
    unloaded = Encoder(_mirror(SMALL), max_tokens=1024, max_seqs=16)
    f32 = Index(SMALL.hidden, 64, dtype="f32")
    narrow = Index(256, 64)
    before = _state(shards, encs)
    per = shard_capacity(60, 3)
    bad_tok = tok.copy()
    bad_tok[-1] = SMALL.vocab                                                      # last token of the last sequence
    long_tok, long_cu = _pack([np.full(150, 5, np.int32)])
    many = np.ones(per + 1, np.int32)
    cases = [
        ("bad token id", N.AUR_ERR_INVALID, lambda: _call(encs, shards, bad_tok, cu, ids)),
        ("shard 0 over capacity", N.AUR_ERR_NOMEM,
         lambda: _call(encs, shards, many, np.arange(per + 2, dtype=np.int32), 3 * np.arange(per + 1))),
        ("encoder configs differ", N.AUR_ERR_INVALID, lambda: _call([enc, other, enc], shards, tok, cu, ids)),
        ("encoder not loaded", N.AUR_ERR_INVALID, lambda: _call([enc, enc, unloaded], shards, tok, cu, ids)),
        ("f32 shard", N.AUR_ERR_INVALID, lambda: _call(encs, [shards[0], f32, shards[2]], tok, cu, ids)),
        ("dim differs", N.AUR_ERR_INVALID, lambda: _call(encs, [shards[0], shards[1], narrow], tok, cu, ids)),
        ("n = 0", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, ids, n=0)),
        ("n = 65", N.AUR_ERR_INVALID, lambda: _call(encs * 22, shards * 22, tok, cu, ids, n=65)),
        ("repeated shard", N.AUR_ERR_INVALID, lambda: _call(encs, [shards[0], shards[1], shards[0]], tok, cu, ids)),
        ("negative id", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, np.where(ids == 11, -1, ids))),
        ("longer than a call", N.AUR_ERR_NOMEM, lambda: _call(encs, shards, long_tok, long_cu, [4], limits=(100, 0))),
        ("limit above the workspace", N.AUR_ERR_INVALID, lambda: _call(encs, shards, tok, cu, ids, limits=(2048, 0))),
        ("empty sequence", N.AUR_ERR_INVALID,
         lambda: _call(encs, shards, tok, np.concatenate([cu[:1], cu]), np.arange(13))),
    ]
    for name, code, fn in cases:
        assert fn() == code, (name, N.load().aur_last_error())
        assert _state(shards, encs) == before, name
    assert f32.stats()["rows"] == 0 and narrow.stats()["rows"] == 0
    assert _call(encs, shards, tok, cu, ids, limits=(300, 2)) == N.AUR_OK      # still usable afterwards
    for x in (other, unloaded, f32, narrow, mi, rep, enc):
        x.close()


@pytest.mark.skipif(not _two_gpus(), reason="needs two GPUs")
def test_two_gpus_replicas_and_rows():
    enc = _encoder(MINILM, max_tokens=4096, max_seqs=64, device=0)
    rep = enc.replicate(1)
    tok, cu = _ragged(MINILM, 17, seed=4)
    assert np.array_equal(rep.encode_packed(tok, cu, bf16=True), enc.encode_packed(tok, cu, bf16=True))
    fused = MultiIndex(MINILM.hidden, 256, devices=[0, 1])
    host = MultiIndex(MINILM.hidden, 256, devices=[0, 1])
    before = _state(fused.shards, [enc, rep])
    assert _call([rep, enc], fused.shards, tok, cu, np.arange(17)) == N.AUR_ERR_INVALID   # encoders on the wrong devices
    assert _state(fused.shards, [enc, rep]) == before
    for tok_, cu_, ids, u, o in _calls(MINILM, seed=12):
        encode_append_multi([enc, rep], fused.shards, tok_, cu_, ids, u, o, 900, 4)
        host.add(to_bf16_bits(enc.encode(_seqs(tok_, cu_))), ids, u, o)
    _assert_same_exports(fused, host)
    for x in (fused, host, rep, enc):
        x.close()


# ---------------------------------------------------------------------- the knowledge base
WORDS = ["disk", "pressure", "node", "restart", "payment", "service", "latency", "spikes", "rotate", "database",
         "credentials", "kafka", "consumer", "lag", "alert", "runbook", "every", "ninety", "days", "memory", "pod",
         "timeout", "network", "failover", "dns", "queue", "depth", "cpu", "throttle", "backup"]
PIECES = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
KB_CFG = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=len(PIECES), max_pos=64, pool="cls")


def _docs(seed, n_docs=6):
    rng = np.random.default_rng(seed)
    docs = []
    for d in range(n_docs):
        chunks = [{"chunk_index": c, "content": " ".join(rng.choice(WORDS, size=int(rng.integers(3, 40)))),
                   "heading_context": "Ops" if c % 2 else ""} for c in range(int(rng.integers(3, 9)))]
        docs.append((f"u{d % 3}", f"doc{seed}-{d}", "f.md", chunks, f"o{d % 2}"))
    docs[1][3][0]["content"] = " ".join(rng.choice(WORDS, size=150))         # longer than the 64-token position table
    return docs


def _text_encoder(devices=(0,)):
    from aurora_b200.wordpiece import NativeTokenizer

    enc = _encoder(KB_CFG, max_tokens=2048, max_seqs=32)
    return TextEncoder(enc, NativeTokenizer(PIECES)).replicate(devices)


class _HostRoute:
    """The encoder as a multi-GPU knowledge base used it before replicas: no can_append, so insert_objects encodes,
    then appends host vectors with MultiIndex.add."""

    def __init__(self, te):
        self.dim, self._te = te.dim, te

    def encode(self, texts):
        return self._te.encode(texts)


def _shape(objs):
    return [(o.uuid, o.metadata.score, None if o.metadata.distance is None else o.metadata.distance) for o in objs]


def test_knowledge_base_over_replicas_matches_a_single_shard(tmp_path):
    from aurora_b200 import retriever as R
    from aurora_b200.filters import Filter

    te = _text_encoder()
    multi = R.KnowledgeBase(te, capacity=512, index_factory=lambda d, c: MultiIndex(d, c, devices=[0, 0, 0]))
    single = R.KnowledgeBase(te, capacity=512)
    host = R.KnowledgeBase(_HostRoute(te), capacity=512, index_factory=lambda d, c: MultiIndex(d, c, devices=[0, 0, 0]))
    assert te.can_append(multi.index) and te.can_append(single.index)
    snap = str(tmp_path / "snap")
    docs = _docs(1) + _docs(2)
    for i, d in enumerate(docs):
        if i == 4:
            multi.save(snap)
            multi.attach_wal(os.path.join(snap, "mutations.log"))
        for kb in (multi, single, host):
            assert kb.insert(*d[:4], org_id=d[4]) == len(d[3])
    assert len(te._windows(docs[1][3][0]["content"])) >= 2
    rows = _live_rows(single.index)
    # (per id: the over-long chunk is appended after its batch's other rows on the fused path, in place on the host route)
    assert _live_rows(multi.index) == rows == _live_rows(host.index) and len(rows) == sum(len(d[3]) for d in docs)
    queries = ["disk pressure node", "kafka consumer lag alert", "nothing matches here", "payment service latency"]
    for q in queries:
        for a in (None, 0.5):
            for u, o in ((None, None), ("u1", "o0")):
                assert _shape(multi.query(q, 5, user_id=u, org_id=o, alpha=a)) == _shape(single.query(q, 5, user_id=u, org_id=o, alpha=a))
        # filtered and batched hybrid searches over three shards are held to the same three shards filled through the
        # host route, not to the single shard: a single shard ranks its dense list by the exact fp64 cosine, while the
        # shards' lists are merged by (fp32 cosine, id) (DESIGN.md section 7).  This random-init encoder puts every
        # cosine near 0.9997, so two rows whose cosines round to the same float32 are common; they may swap ranks, and
        # ranked fusion then scores them differently.  The unscoped queries above happen to meet no such tie.
        f = Filter.by_property("org_id").equal("o1") & Filter.by_property("document_id").like("doc1-*")
        assert _shape(multi.query(q, 5, filters=f, alpha=0.5)) == _shape(host.query(q, 5, filters=f, alpha=0.5))
    reqs = [(f"u{i % 3}", q, 4, a, f"o{i % 2}") for i, q in enumerate(queries) for a in (None, 0.3)]
    assert [_shape(r) for r in multi.query_batch(reqs)] == [_shape(r) for r in host.query_batch(reqs)]
    # a freshly loaded replicated knowledge base replays the log through the same ingest and stores the same rows
    again = R.KnowledgeBase.load(snap, te, capacity=512,
                                 index_loader=lambda p, cap: MultiIndex.load(p, capacity=cap, devices=[0, 0, 0]))
    assert again.attach_wal(os.path.join(snap, "mutations.log")) == len(docs) - 4
    assert _live_rows(again.index) == rows


def test_searches_while_the_replicated_knowledge_base_ingests():
    """Readers search every shard (aur_search_ex reports the prefix it saw) and query the knowledge base while a writer
    inserts documents through the multi-shard append.  Every shard answer must equal the oracle's top-k over exactly
    the prefix it reports; keys are unique, so no row of a prefix is ever tombstoned."""
    from aurora_b200 import retriever as R

    te = _text_encoder()
    kb = R.KnowledgeBase(te, capacity=2048, index_factory=lambda d, c: MultiIndex(d, c, devices=[0, 0, 0]))
    k = 6
    Q = bf16_bits_to_f32(to_bf16_bits(te.encode(["disk pressure node", "kafka lag", "payment latency spikes"])))
    docs = [d for s in range(3, 9) for d in _docs(s)]
    errors, done, answers = [], threading.Event(), []

    def writer():
        try:
            for d in docs:
                kb.insert(*d[:4], org_id=d[4])
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
                kb.query("disk pressure node", 3, alpha=0.5)
            answers.append(mine)
        except Exception as e:      # pragma: no cover
            errors.append(e)

    ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errors, errors[0]
    ex = _exports(kb.index)
    seen = set()
    for mine in answers:
        for s, snap, ids, sc in mine:
            rows, rid, _, _, live = ex[s]
            assert live[:snap].all()
            seen.add((s, snap))
            if snap == 0:
                assert (ids == -1).all()
                continue
            oids, osc = cosine_topk(Q, bf16_bits_to_f32(rows[:snap]), k, ids=rid[:snap])
            assert np.array_equal(ids, oids), (s, snap)
            fin = np.isfinite(osc)
            assert np.array_equal(np.isfinite(sc), fin) and float(np.max(np.abs(sc[fin] - osc[fin]), initial=0)) <= 1e-6
    assert len({snap for _, snap in seen}) >= 3                                   # the readers really overlapped the writer
    assert sum(sh.stats()["live"] for sh in kb.index.shards) == sum(len(d[3]) for d in docs)
