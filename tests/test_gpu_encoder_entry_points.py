"""The encoder's token-id and text ingest entry points against what they are stated to be (include/aurora_b200.h):
aur_encode_text_append is aur_tokenize followed by aur_encode_append_multi with n = 1 and the same per-call limits, row
for row and bit for bit; and aur_encode_append rejects every malformed call before any device work, leaving the shard
and the encoder as they were."""

import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from aurora_b200 import _native as N
from aurora_b200.encoder import Encoder, EncoderConfig, encode_append_multi
from aurora_b200.engine import Index
from aurora_b200.wordpiece import NativeTokenizer
from oracle import bert_encoder as B

WORDS = ["disk", "pressure", "node", "restart", "payment", "service", "latency", "spikes", "rotate", "database",
         "credentials", "kafka", "consumer", "lag", "alert", "runbook", "every", "ninety", "days", "memory", "pod",
         "timeout", "network", "failover", "dns", "queue", "depth", "cpu", "throttle", "backup"]
PIECES = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
TEXT_CFG = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=len(PIECES), max_pos=64, pool="cls")
SMALL = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")


def _mirror(c: B.BertConfig) -> EncoderConfig:
    return EncoderConfig(hidden=c.hidden, layers=c.layers, heads=c.heads, inter=c.inter, vocab=c.vocab, max_pos=c.max_pos,
                         type_vocab=c.type_vocab, ln_eps=c.ln_eps, pool=c.pool, normalize=c.normalize)


def _encoder(c, max_tokens, max_seqs, load=True) -> Encoder:
    enc = Encoder(_mirror(c), max_tokens=max_tokens, max_seqs=max_seqs)
    if load:
        enc.load_weights(B.init_weights(c, seed=7, bf16=True))
    return enc


def _export(ix):
    return [a.copy() for a in ix.export_raw()]


def _same_export(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _forward_stats(st):
    """The encoder stats that describe the last forward (not its time)."""
    return {k: st[k] for k in ("tokens", "seqs", "launches", "gemm_flops", "attn_flops")}


# ---------------------------------------------------------------------- aur_encode_text_append
def _text_append(enc, tok, ix, texts, ids, u, o, max_len, max_tokens_per_call, max_seqs_per_call):
    blob, offs = tok._pack(list(texts))
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)    # noqa: E731
    return N.load().aur_encode_text_append(enc._h, tok._h, ix._h, blob, vp(offs), len(texts), max_len, max_tokens_per_call,
                                           max_seqs_per_call, vp(ids), vp(u), vp(o), 0)


def _chunks(seed, n=23):
    rng = np.random.default_rng(seed)
    texts = [" ".join(rng.choice(WORDS, size=int(rng.integers(1, 45)))) for _ in range(n)]
    texts[9] = " ".join(rng.choice(WORDS, size=150))                       # longer than the 64-token position table
    ids = np.arange(1000, 1000 + n, dtype=np.int64)
    ids[-2] = ids[3]                                                        # a repeated id: its last occurrence stays
    return texts, ids, rng.integers(0, 4, n).astype(np.int32), rng.integers(-1, 3, n).astype(np.int32)


@pytest.mark.parametrize("limits", [(200, 5), (64, 1), (2048, 32)], ids=["batches", "one-per-batch", "workspace"])
def test_text_append_is_tokenize_then_multi_append(limits):
    max_len = TEXT_CFG.max_pos
    enc = _encoder(TEXT_CFG, max_tokens=2048, max_seqs=32)
    tok = NativeTokenizer(PIECES)
    texts, ids, u, o = _chunks(seed=sum(limits))
    got, want = Index(TEXT_CFG.hidden, 64), Index(TEXT_CFG.hidden, 64)

    assert _text_append(enc, tok, got, texts, ids, u, o, max_len, *limits) == N.AUR_OK, N.load().aur_last_error()
    got_stats = _forward_stats(enc.stats())
    t, cu = tok.encode_packed(texts, max_len)
    encode_append_multi([enc], [want], t, cu, ids, u, o, *limits)
    assert _same_export(_export(got), _export(want))
    assert got_stats == _forward_stats(enc.stats())                        # the same last batch
    if limits[0] < int(cu[-1]):
        assert got_stats["seqs"] < len(texts)                              # several batches were cut

    rows, rid, user, org, live = got.export_raw()
    assert live.sum() == len(set(ids.tolist())) and len(rid) == len(texts)
    assert tok.lengths([texts[9]])[0] > max_len and cu[10] - cu[9] == max_len   # the long text was truncated
    row = np.nonzero((rid == ids[9]) & (live > 0))[0]
    assert len(row) == 1
    alone = enc.encode_packed(t[cu[9]:cu[10]], np.array([0, max_len], np.int32), bf16=True)
    assert np.array_equal(rows[row[0]], alone[0])
    assert int(user[row[0]]) == u[9] and int(org[row[0]]) == o[9]
    for ix in (got, want):
        ix.close()
    enc.close()


def test_text_append_rejections_leave_the_shard_untouched():
    enc = _encoder(TEXT_CFG, max_tokens=512, max_seqs=8)
    tok = NativeTokenizer(PIECES)
    texts, ids, u, o = _chunks(seed=5, n=12)
    ix = Index(TEXT_CFG.hidden, 64)
    assert _text_append(enc, tok, ix, texts[:4], ids[:4], u[:4], o[:4], 64, 512, 8) == N.AUR_OK
    before = _export(ix)
    cases = [
        ("max_len 1", (1, 512, 8)),
        ("max_len 513", (513, 1024, 8)),
        ("token limit below max_len", (64, 63, 8)),
        ("no sequence per call", (64, 512, 0)),
        ("token limit above the workspace", (64, 1024, 8)),
        ("sequence limit above the workspace", (64, 512, 9)),
    ]
    for name, (max_len, mt, ms) in cases:
        assert _text_append(enc, tok, ix, texts, ids, u, o, max_len, mt, ms) == N.AUR_ERR_INVALID, name
        assert _same_export(_export(ix), before), name
    ix.close()
    enc.close()


def _pack(lens, rng, vocab=SMALL.vocab):
    cu = np.zeros(len(lens) + 1, np.int32)
    cu[1:] = np.cumsum(lens)
    tok = rng.integers(3, vocab, size=int(cu[-1])).astype(np.int32)
    return tok, cu


# ---------------------------------------------------------------------- aur_encode with both outputs
def test_encode_with_both_outputs_gives_each_outputs_vectors():
    """One output is copied straight into the caller's buffer, both are staged on the host: the same vectors either way."""
    enc = _encoder(SMALL, max_tokens=512, max_seqs=4)
    tok, cu = _pack([17, 60, 25], np.random.default_rng(4))
    f32, bf16 = np.empty((3, SMALL.hidden), np.float32), np.empty((3, SMALL.hidden), np.uint16)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)    # noqa: E731
    N.check(N.load().aur_encode(enc._h, vp(tok), vp(cu), 3, vp(f32), vp(bf16)))
    assert np.array_equal(f32.view(np.uint32), enc.encode_packed(tok, cu).view(np.uint32))
    assert np.array_equal(bf16, enc.encode_packed(tok, cu, bf16=True))
    enc.close()


# ---------------------------------------------------------------------- aur_encode_append rejections
# name, code, the rejected call.  Every row but the two marked ones leaves the encoder's stats untouched at the parent
# commit too, where the no-room and negative-id rows were only found by aur_add_dev, after the forward had run.
REJECTIONS = [
    ("parameters missing", N.AUR_ERR_INVALID, lambda c: c.unloaded.encode_append(c.ix, c.tok, c.cu, c.ids)),
    ("f32 shard", N.AUR_ERR_INVALID, lambda c: c.enc.encode_append(c.f32, c.tok, c.cu, c.ids)),
    ("dim differs", N.AUR_ERR_INVALID, lambda c: c.enc.encode_append(c.narrow, c.tok, c.cu, c.ids)),
    ("n_seq > max_seqs", N.AUR_ERR_NOMEM, lambda c: c.enc.encode_append(c.ix, *_pack([5] * 5, c.rng), np.arange(20, 25))),
    ("tokens > max_tokens", N.AUR_ERR_NOMEM, lambda c: c.enc.encode_append(c.ix, *_pack([300, 250], c.rng), np.arange(20, 22))),
    ("shard without room", N.AUR_ERR_NOMEM,                                           # stats untouched: new
     lambda c: c.enc.encode_append(c.ix, *_pack([9, 11, 13, 15], c.rng), np.arange(20, 24))),
    ("negative id", N.AUR_ERR_INVALID,                                                 # stats untouched: new
     lambda c: c.enc.encode_append(c.ix, c.tok, c.cu, np.array([10, -1, 12]))),
    ("token id out of range", N.AUR_ERR_INVALID, lambda c: c.enc.encode_append(c.ix, c.bad_tok, c.cu, c.ids)),
    ("empty sequence", N.AUR_ERR_INVALID,
     lambda c: c.enc.encode_append(c.ix, c.tok, np.concatenate([c.cu[:1], c.cu]), np.arange(10, 14))),
]


@pytest.mark.parametrize("name,code,call", REJECTIONS, ids=[r[0].replace(" > ", " over ").replace(" ", "-") for r in REJECTIONS])
def test_encode_append_rejection_leaves_shard_and_encoder_untouched(name, code, call):
    c = SimpleNamespace(rng=np.random.default_rng(3))
    c.enc = _encoder(SMALL, max_tokens=512, max_seqs=4)
    c.unloaded = _encoder(SMALL, max_tokens=512, max_seqs=4, load=False)
    c.ix, c.f32, c.narrow = Index(SMALL.hidden, 8), Index(SMALL.hidden, 8, dtype="f32"), Index(256, 8)
    c.enc.encode_append(c.ix, *_pack([40, 7, 90], c.rng), np.arange(3))
    c.enc.encode_append(c.ix, *_pack([33, 21], c.rng), np.arange(3, 5))       # 5 of 8 rows used
    c.tok, c.cu = _pack([17, 60, 25], c.rng)
    c.ids = np.arange(10, 13, dtype=np.int64)
    c.bad_tok = c.tok.copy()
    c.bad_tok[c.cu[1] + 3] = SMALL.vocab
    shards = (c.ix, c.f32, c.narrow)
    before = [_export(s) for s in shards]
    stats = c.enc.stats(), c.unloaded.stats()
    with pytest.raises(N.AuroraError) as e:
        call(c)
    assert e.value.code == code, str(e.value)
    assert all(_same_export(_export(s), b) for s, b in zip(shards, before))
    assert (c.enc.stats(), c.unloaded.stats()) == stats
    c.enc.encode_append(c.ix, c.tok, c.cu, c.ids)                              # still usable afterwards
    assert c.ix.stats()["rows"] == 8
    for x in (c.narrow, c.f32, c.ix, c.unloaded, c.enc):
        x.close()
