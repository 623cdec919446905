"""CPU: the numpy BERT restatement (oracle/bert_encoder.py) against vectors produced by the
installed transformers.BertModel (tests/golden/bert_ref.json, made by oracle/gen_golden_bert.py)."""

import json
import os

import numpy as np
import pytest

from oracle import bert_encoder as B

GOLD = os.path.join(os.path.dirname(__file__), "golden", "bert_ref.json")


def _cases():
    with open(GOLD) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_oracle_matches_hf_bertmodel(case):
    if case["name"] == "bge_base":
        pytest.skip("covered by minilm_l6 on CPU; bge_base weights take ~20 s to seed (run in the gpu suite)")
    cfg = B.BertConfig(**case["cfg"])
    w = B.init_weights(cfg, seed=7, bf16=True)
    tok = np.asarray(case["tokens"], dtype=np.int32)
    cu = np.asarray(case["cu_seqlens"], dtype=np.int32)
    got = B.encode(cfg, w, tok, cu)
    np.testing.assert_allclose(got, np.asarray(case["pooled"]), rtol=0, atol=1e-9)


def test_synth_batch_matches_fixture_inputs():
    c = _cases()[0]
    cfg = B.BertConfig(**c["cfg"])
    tok, cu = B.synth_batch(cfg, c["n_seq"], c["seed"], **c["batch"])
    assert tok.tolist() == c["tokens"] and cu.tolist() == c["cu_seqlens"]


def test_pooling_modes_and_empty_sequence():
    cfg = B.BertConfig(hidden=8, layers=1, heads=2, inter=16, vocab=10, max_pos=8, pool="mean", normalize=False)
    hid = np.arange(5 * 8, dtype=np.float64).reshape(5, 8)
    cu = np.array([0, 2, 2, 5])
    out = B.pool(cfg, hid, cu)
    np.testing.assert_allclose(out[0], hid[0:2].mean(axis=0))
    assert not out[1].any()                       # empty sequence -> zero vector
    np.testing.assert_allclose(out[2], hid[2:5].mean(axis=0))
    cls = B.pool(B.BertConfig(hidden=8, layers=1, heads=2, inter=16, vocab=10, max_pos=8, pool="cls", normalize=True), hid, cu)
    np.testing.assert_allclose(np.linalg.norm(cls[2]), 1.0)
    np.testing.assert_allclose(cls[2], hid[2] / np.linalg.norm(hid[2]))


def test_gelu_is_erf_form():
    x = np.array([-3.0, -1.0, 0.0, 0.5, 2.0])
    np.testing.assert_allclose(B.gelu(x), [-0.00404969409489031, -0.15865525393145702, 0.0, 0.34573123063700656, 1.9544997361036416], atol=1e-12)  # torch.nn.functional.gelu (float64)


def test_bf16_store_mode_rounds_where_the_gpu_stores():
    """encode_tokens(bf16_stores=True): every hidden state is a bf16 value, it stays close to the unrounded forward
    (the roundings are small, but real), and under constant_row_weights a token with a constant embedding row comes
    out as exactly bf16(ln2_b)."""
    from oracle.cosine_topk import round_to_bf16

    cfg = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")
    w = B.init_weights(cfg, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg, 4, 3, mean_len=40, std_len=30, min_len=1, max_len=128)
    exact = B.encode_tokens(cfg, w, tok, cu)
    stored = B.encode_tokens(cfg, w, tok, cu, bf16_stores=True)
    assert np.array_equal(stored, round_to_bf16(stored.astype(np.float32)))
    assert not np.array_equal(stored, round_to_bf16(exact.astype(np.float32)))
    assert np.abs(stored - exact).max() <= 0.1
    cos = (stored * exact).sum(1) / np.linalg.norm(stored, axis=1) / np.linalg.norm(exact, axis=1)
    assert cos.min() >= 0.999

    cfg1 = B.BertConfig(**{**cfg.__dict__, "layers": 1})
    w1 = constant_row_weights(cfg1)
    out = B.encode_tokens(cfg1, w1, np.array([1, 5, 5, 7], np.int32), np.array([0, 4], np.int32), bf16_stores=True)
    assert np.array_equal(out[1:3], np.broadcast_to(w1["l0.ln2_b"], (2, cfg.hidden)))


def constant_row_weights(cfg):
    """Weights under which token 5's embedding-LayerNorm input is a constant row (pos / type rows zero, word row 5
    constant) and every later LayerNorm input of that token is constant too: all layer matrices and biases zero, LN
    biases constant vectors.  Its final hidden state is then exactly bf16(ln2_b), with eps 1e-12."""
    w = B.init_weights(cfg, seed=3, bf16=True)
    w["pos_emb"][:] = 0.0
    w["type_emb"][:] = 0.0
    w["word_emb"][5] = 0.3984375                               # a bf16 value
    w["emb_ln_b"][:] = 0.5
    for l in range(cfg.layers):
        for n in ("wqkv", "bqkv", "wo", "bo", "wi", "bi", "wo2", "bo2"):
            w[f"l{l}.{n}"][:] = 0.0
        w[f"l{l}.ln1_b"][:] = -0.25
        w[f"l{l}.ln2_b"][:] = 0.75
    return w
