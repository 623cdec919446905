"""GPU bring-up of the encoder kernels against numpy / the oracle (run on an H100).

    python tools/bringup_encoder.py [--stage gemm|attn|tiny|bge|perf]
"""
import argparse
import ctypes as C
import math
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N
from aurora_b200.encoder import Encoder, EncoderConfig
from aurora_b200.engine import to_bf16_bits
from oracle import bert_encoder as B
from oracle.cosine_topk import bf16_bits_to_f32, round_to_bf16


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def gelu(x):
    return B.gelu(x.astype(np.float64))


def stage_gemm():
    lib = N.load()
    rng = np.random.default_rng(0)
    for g in (1, 2):
      for (m, n, k, epi) in [(128, 256, 64, 0), (200, 256, 128, 0), (300, 128, 192, 0), (1000, 768, 768, 2),
                           (1000, 2304, 768, 0), (777, 3072, 768, 1), (640, 768, 3072, 2), (500, 384, 384, 1),
                           (4096, 3072, 768, 1), (23163, 2304, 768, 0), (23163, 3072, 768, 1), (23163, 768, 3072, 2)]:
          a = round_to_bf16(rng.standard_normal((m, k)).astype(np.float32))
          w = round_to_bf16((rng.standard_normal((n, k)) / math.sqrt(k)).astype(np.float32))
          bias = rng.standard_normal(n).astype(np.float32)
          resid = round_to_bf16(rng.standard_normal((m, n)).astype(np.float32))
          out = np.zeros((m, n), dtype=np.uint16)
          ms = C.c_float()
          N.check(lib.aur_debug_gemm(0, ptr(to_bf16_bits(a)), ptr(to_bf16_bits(w)), ptr(bias), ptr(to_bf16_bits(resid)),
                                   m, n, k, epi, g, ptr(out), C.byref(ms)))
          ref = a.astype(np.float64) @ w.astype(np.float64).T + bias
          if epi == 1:
              ref = gelu(ref)
          if epi == 2:
              ref = ref + resid
          got = bf16_bits_to_f32(out).astype(np.float64)
          err = np.abs(got - ref).max()
          tol = np.abs(ref).max() * 2 ** -8 + 1e-3
          tf = 2.0 * m * n * k / (ms.value * 1e-3) / 1e12
          print(f"gemm g={g} m={m} n={n} k={k} epi={epi}: max|err|={err:.4f} (tol {tol:.4f}) {ms.value*1e3:.1f} us {tf:.1f} TF/s", flush=True)
          assert err <= tol, "GEMM mismatch"


def attn_ref(qkv, cu, heads, hidden):
    T = qkv.shape[0]
    out = np.zeros((T, hidden))
    dh = hidden // heads
    for s in range(len(cu) - 1):
        lo, hi = cu[s], cu[s + 1]
        x = qkv[lo:hi].astype(np.float64)
        for h in range(heads):
            q = x[:, h * dh:(h + 1) * dh]; k = x[:, hidden + h * dh: hidden + (h + 1) * dh]
            v = x[:, 2 * hidden + h * dh: 2 * hidden + (h + 1) * dh]
            a = q @ k.T / math.sqrt(dh)
            a = np.exp(a - a.max(axis=1, keepdims=True)); a /= a.sum(axis=1, keepdims=True)
            out[lo:hi, h * dh:(h + 1) * dh] = a @ v
    return out


def stage_attn():
    lib = N.load()
    rng = np.random.default_rng(1)
    for heads, lens in [(2, [5]), (2, [128]), (2, [129, 1, 64]), (12, [300, 17, 512, 384, 200]), (4, [512] * 3)]:
        hidden = heads * 64
        cu = np.zeros(len(lens) + 1, dtype=np.int32); cu[1:] = np.cumsum(lens)
        T = int(cu[-1])
        qkv = round_to_bf16((rng.standard_normal((T, 3 * hidden)) * 1.5).astype(np.float32))
        out = np.zeros((T, hidden), dtype=np.uint16)
        ms = C.c_float()
        N.check(lib.aur_debug_attention(0, ptr(to_bf16_bits(qkv)), ptr(cu), len(lens), heads, hidden, ptr(out), C.byref(ms)))
        ref = attn_ref(qkv, cu, heads, hidden)
        got = bf16_bits_to_f32(out).astype(np.float64)
        err = np.abs(got - ref).max()
        print(f"attn heads={heads} lens={lens}: max|err|={err:.4f} {ms.value*1e3:.1f} us", flush=True)
        assert err < 0.03, "attention mismatch"


def run_encoder(cfg_o, n_seq, seed, batch_kw, max_tokens=8192):
    cfg = EncoderConfig(hidden=cfg_o.hidden, layers=cfg_o.layers, heads=cfg_o.heads, inter=cfg_o.inter, vocab=cfg_o.vocab,
                        max_pos=cfg_o.max_pos, type_vocab=cfg_o.type_vocab, ln_eps=cfg_o.ln_eps, pool=cfg_o.pool,
                        normalize=cfg_o.normalize)
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, n_seq, seed, **batch_kw)
    with Encoder(cfg, max_tokens=max_tokens, max_seqs=max(n_seq, 8)) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(tok, cu)
        hid = bf16_bits_to_f32(enc.hidden_states()).astype(np.float64)
        st = enc.stats()
    t0 = time.time()
    ref_h = B.encode_tokens(cfg_o, w, tok, cu, dtype=np.float32 if cfg_o.hidden > 256 else np.float64)
    ref = B.pool(cfg_o, ref_h.astype(np.float64), cu)
    herr = np.abs(hid - ref_h).max()
    perr = np.abs(got - ref).max()
    cos = (got * ref).sum(axis=1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    print(f"encoder H={cfg_o.hidden} L={cfg_o.layers} n_seq={n_seq} tokens={len(tok)}: hidden max|err|={herr:.4f} "
          f"pooled max|err|={perr:.5f} min cos={cos.min():.6f}  gpu {st['total_ms']:.3f} ms (oracle {time.time()-t0:.1f} s)", flush=True)
    return perr, cos.min()


def stage_tiny():
    cfg = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=64, pool="cls")
    perr, cos = run_encoder(cfg, 5, 11, dict(mean_len=20, std_len=12, min_len=2, max_len=64))
    assert cos > 0.999
    cfg = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="mean")
    perr, cos = run_encoder(cfg, 7, 12, dict(mean_len=200, std_len=150, min_len=1, max_len=512))
    assert cos > 0.999


def stage_bge():
    perr, cos = run_encoder(B.BGE_BASE, 6, 15, dict(mean_len=100, std_len=80, min_len=4, max_len=512))
    assert cos > 0.999


def stage_perf():
    cfg_o = B.BGE_BASE
    cfg = EncoderConfig()
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    with Encoder(cfg, max_tokens=65536, max_seqs=256) as enc:
        enc.load_weights(w)
        for n_seq in (16, 64, 160):
            tok, cu = B.synth_batch(cfg_o, n_seq, 1003)
            for _ in range(3):
                enc.encode_packed(tok, cu)
            st = enc.stats()
            fl = st["gemm_flops"] + st["attn_flops"]
            print(f"perf n_seq={n_seq} tokens={st['tokens']}: {st['total_ms']:.3f} ms  {n_seq/st['total_ms']*1e3:.0f} chunks/s  "
                  f"{fl/st['total_ms']/1e9:.1f} TF/s (gemm {st['gemm_flops']/1e12:.2f} TF, attn {st['attn_flops']/1e12:.2f} TF) launches {st['launches']}", flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", default="all")
    a = ap.parse_args()
    stages = {"gemm": stage_gemm, "attn": stage_attn, "tiny": stage_tiny, "bge": stage_bge, "perf": stage_perf}
    for name, fn in stages.items():
        if a.stage in ("all", name):
            print(f"== {name}", flush=True)
            fn()
    print("bringup_encoder OK")
