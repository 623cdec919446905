"""One bge-base forward over a synthetic cfg3 batch, for ncu / timing (run on an H100).

    python tools/profile_encoder.py [n_seq] [reps]
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200.encoder import Encoder, EncoderConfig

n_seq = int(sys.argv[1]) if len(sys.argv) > 1 else 64
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
cfg = EncoderConfig()
rng = np.random.default_rng(7)
lens = np.clip(np.rint(rng.normal(384, 96, n_seq)), 16, 512).astype(np.int64)
cu = np.zeros(n_seq + 1, np.int32); cu[1:] = np.cumsum(lens)
tok = rng.integers(1000, cfg.vocab, size=int(cu[-1])).astype(np.int32)
with Encoder(cfg, max_tokens=int(cu[-1]) + 128, max_seqs=n_seq) as enc:
    # device-side random weights would need another entry point; small std-0.02 host init per tensor
    h, i = cfg.hidden, cfg.inter
    shapes = {"word_emb": (cfg.vocab, h), "pos_emb": (cfg.max_pos, h), "type_emb": (cfg.type_vocab, h), "emb_ln_g": (h,), "emb_ln_b": (h,)}
    for l in range(cfg.layers):
        for k, s in {"wqkv": (3 * h, h), "bqkv": (3 * h,), "wo": (h, h), "bo": (h,), "ln1_g": (h,), "ln1_b": (h,), "wi": (i, h),
                     "bi": (i,), "wo2": (h, i), "bo2": (h,), "ln2_g": (h,), "ln2_b": (h,)}.items():
            shapes[f"l{l}.{k}"] = s
    for name, s in shapes.items():
        a = (1.0 + 0.1 * rng.standard_normal(s)) if name.endswith("_g") else 0.02 * rng.standard_normal(s)
        enc.load_weights({name: a.astype(np.float32)})
    for _ in range(reps):
        enc.encode_packed(tok, cu)
        st = enc.stats()
        fl = st["gemm_flops"] + st["attn_flops"]
        print(f"n_seq={n_seq} tokens={st['tokens']}: {st['total_ms']:.3f} ms {n_seq / st['total_ms'] * 1e3:.0f} chunks/s "
              f"{fl / st['total_ms'] / 1e9:.1f} TF/s launches {st['launches']}", flush=True)
