"""One vector per text from its windows' vectors, restated in numpy: what aur_encode_texts and
aur_encode_append_texts_multi give a text whose tokenisation spans w windows (window_fold_kernel, csrc/encoder_simt.cu).

v_1 .. v_w are the fp32 window vectors as the encoder pools them (each normalised when the encoder normalises).
  w = 1: the text's vector is v_1.
  w >= 2: s = fl32(..fl32(v_1 + v_2) .. + v_w), in window order, one rounding per add; m = fl32(s / w).
    normalize: every square m_i^2 is exact in fp64; lane sums r_c = m_c^2 + m_{c+32}^2 + ... in increasing i, for
    c = 0 .. 31 (hidden is a multiple of 32), then q = r_0 + r_1 + ... + r_31, each add one fp64 rounding.
    q > 0: out_i = fl32(fl64(m_i / fl64(sqrt(q)))); otherwise out = m.  Without normalize, out = m.
The bf16 row is out rounded to nearest even (engine.to_bf16_bits).
"""

from __future__ import annotations

import numpy as np

LANES = 32


def fold_windows(v: np.ndarray, normalize: bool) -> np.ndarray:
    """fp32 window vectors [w, hidden] -> the text's fp32 vector [hidden]."""
    v = np.ascontiguousarray(v, dtype=np.float32)
    if v.ndim != 2 or v.shape[0] < 1 or v.shape[1] % LANES:
        raise ValueError("window vectors [w >= 1, hidden], hidden a multiple of 32")
    if v.shape[0] == 1:
        return v[0].copy()
    s = v[0].copy()
    for j in range(1, v.shape[0]):
        s = s + v[j]                                            # float32 + float32: one rounding
    m = s / np.float32(v.shape[0])
    if not normalize:
        return m
    sq = m.astype(np.float64) ** 2                              # exact: 24-bit significands, 48-bit product
    r = np.zeros(LANES, dtype=np.float64)
    for k in range(0, sq.size, LANES):                          # per lane, in increasing dim
        r = r + sq[k:k + LANES]
    q = 0.0
    for c in range(LANES):                                      # the lane sums in lane order
        q = float(np.float64(q) + r[c])
    if not q > 0.0:
        return m
    return (m.astype(np.float64) / np.sqrt(np.float64(q))).astype(np.float32)


def fold_texts(v: np.ndarray, cu_texts: np.ndarray, normalize: bool) -> np.ndarray:
    """fp32 window vectors [windows, hidden] and cu_texts [n_texts + 1] -> text vectors [n_texts, hidden] fp32."""
    cu_texts = np.asarray(cu_texts, dtype=np.int64)
    out = np.empty((cu_texts.size - 1, np.shape(v)[1]), dtype=np.float32)
    for j in range(out.shape[0]):
        out[j] = fold_windows(v[cu_texts[j]:cu_texts[j + 1]], normalize)
    return out
