"""Small end-to-end run for `compute-sanitizer --tool memcheck` (seconds under the tool):
tensor-core + generic search with partial query blocks, deletes, repeated launches; a tiny encoder forward
with fused ingest; text added to, searched in and closed with a keyword store and its vocabulary.  Exits non-zero on a
parity mismatch."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N
from aurora_b200.encoder import Encoder, EncoderConfig
from aurora_b200.engine import Index, KeywordIndex, KeywordVocab
from oracle import bert_encoder as B
from oracle import cosine_topk as O

rng = np.random.default_rng(0)
for d in (768, 1024):
    n = 6000
    C = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    with Index(d, n + 64) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.remove(np.arange(0, n, 97, dtype=np.int64))
        live = np.ones(n, bool); live[::97] = False
        for nq, k in ((1, 5), (130, 32), (300, 64)):
            Q = O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))
            want = O.cosine_topk(Q, C, k, live=live)
            for kern in (N.KERNEL_AUTO, N.KERNEL_TC1, N.KERNEL_SIMT):
                ix.set_kernel(kern)
                for _ in range(3):
                    ids, sc = ix.search(Q, k)
                assert np.array_equal(ids, want[0]), (d, nq, k, kern)
        # round 2: mixed tenant scopes through the per-row bit masks, a resolved pre-filter, compaction, a batch
        # past 256 queries (query super-blocks), results written straight into the caller's buffers
        ru, ro = rng.integers(0, 5, n).astype(np.int32), rng.integers(-1, 2, n).astype(np.int32)
    with Index(d, n + 64) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), ru, ro)
        Q = O.round_to_bf16(rng.standard_normal((70, d)).astype(np.float32))
        qu, qo = rng.integers(0, 5, 70).astype(np.int32), rng.integers(-1, 2, 70).astype(np.int32)
        ids, sc = ix.search(Q, 16, qu, qo)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        assert np.array_equal(ids, O.cosine_topk(Q, C, 16, row_user=ru, row_org=ro, q_user=qu, q_org=qo)[0])
        allow = np.arange(0, n, 3, dtype=np.int64)
        live = np.zeros(n, bool); live[::3] = True
        assert np.array_equal(ix.search_subset(Q, 16, allow)[0], O.cosine_topk(Q, C, 16, live=live)[0])
        ix.remove(np.arange(0, n, 2, dtype=np.int64))
        assert ix.compact() == n // 2
        live = np.ones(n, bool); live[::2] = False
        Qb = O.round_to_bf16(rng.standard_normal((600, d)).astype(np.float32))
        assert np.array_equal(ix.search(Qb, 10)[0], O.cosine_topk(Qb, C, 10, live=live)[0])
    print("search ok", d, flush=True)

cfg_o = B.BertConfig(hidden=128, layers=1, heads=2, inter=256, vocab=120, max_pos=512, pool="mean")
w = B.init_weights(cfg_o, seed=7, bf16=True)
tok, cu = B.synth_batch(cfg_o, 5, 3, mean_len=150, std_len=120, min_len=1, max_len=400)
cfg = EncoderConfig(hidden=128, layers=1, heads=2, inter=256, vocab=120, max_pos=512, pool="mean")
with Encoder(cfg, max_tokens=2048, max_seqs=8) as enc, Index(128, 32) as ix:
    enc.load_weights(w)
    got = enc.encode_packed(tok, cu)
    ref = B.encode(cfg_o, w, tok, cu)
    assert np.abs(got - ref).max() < 1e-2
    enc.encode_append(ix, tok, cu, np.arange(5, dtype=np.int64))
    assert ix.stats()["live"] == 5
print("encoder ok (attention v2)")


vocab, store = KeywordVocab(0), KeywordIndex(64)
store.add_text(vocab, np.arange(3, dtype=np.int64), ["alpha beta", "gamma alpha delta", "beta beta epsilon"])
ids, _, snap = store.search(np.array([1, 2], np.int32), np.array([0, 1, 2], np.int64), 2)   # beta; gamma
assert snap == 3 and ids[0].tolist() == [2, 0] and ids[1].tolist() == [1, -1], ids
store.close(); vocab.close()
print("keyword ok")
