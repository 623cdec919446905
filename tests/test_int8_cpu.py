"""The int8 row format (AUR_I8) without a device: the quantization rule of oracle/quantize.py, the argument checks of
engine.Index(dtype="int8") that come before the library is opened, and the header's enum value."""

from __future__ import annotations

import os
import re

import numpy as np
import pytest

from aurora_b200 import _native as N
from oracle import quantize as Qz
from oracle.cosine_topk import f32_to_bf16_bits

HERE = os.path.dirname(os.path.abspath(__file__))


def _bits(vals):
    return f32_to_bf16_bits(np.asarray(vals, dtype=np.float32)).reshape(1, -1)


def test_half_even_ties():
    # amax = 254: q = x * 127 / 254 = x / 2, so odd integers land exactly on .5 and round to even
    x = [254.0, 1.0, 3.0, 5.0, -1.0, -3.0, 7.0, 0.0]
    q, fin = Qz.quantize_rows(_bits(x))
    assert fin.all()
    assert q[0].tolist() == [127, 0, 2, 2, 0, -2, 4, 0]


def test_amax_element_is_127_and_bounds():
    rng = np.random.default_rng(3)
    bits = f32_to_bf16_bits(rng.standard_normal((200, 96)).astype(np.float32) * rng.uniform(1e-3, 1e3, (200, 1)).astype(np.float32))
    q, fin = Qz.quantize_rows(bits)
    assert fin.all()
    assert (np.abs(q.astype(np.int32)) <= 127).all()
    assert (np.abs(q.astype(np.int32)).max(axis=1) == 127).all()


def test_negative_amax_element():
    q, _ = Qz.quantize_rows(_bits([-2.0, 1.0, 0.5, 0.0]))
    assert q[0].tolist() == [-127, 64, 32, 0]      # 63.5 -> 64 (even), 31.75 -> 32


def test_zero_row():
    q, fin = Qz.quantize_rows(np.zeros((2, 32), np.uint16))
    assert fin.all() and not q.any()


def test_subnormals_and_largest_finite():
    tiny = np.array([0x0001, 0x0002, 0x8003, 0x0000], np.uint16).reshape(1, -1)      # bf16 subnormals
    q, fin = Qz.quantize_rows(tiny)
    assert fin.all()
    assert q[0].tolist() == [42, 85, -127, 0]      # 127 / 3 = 42.33, 254 / 3 = 84.67
    big = np.array([0x7F7F, 0xFF7F, 0x3F80, 0x0000], np.uint16).reshape(1, -1)       # +-max finite bf16, 1.0
    q, fin = Qz.quantize_rows(big)
    assert fin.all() and q[0].tolist() == [127, -127, 0, 0]


def test_non_finite_rows_are_zeros():
    rows = np.stack([_bits([1.0, np.nan, 2.0, 0.0])[0], _bits([np.inf, 1.0, 0.0, 0.0])[0], _bits([-np.inf, 0, 0, 0])[0],
                     _bits([1.0, 2.0, 3.0, 4.0])[0]])
    q, fin = Qz.quantize_rows(rows)
    assert fin.tolist() == [False, False, False, True]
    assert not q[:3].any()


def test_idempotent():
    rng = np.random.default_rng(5)
    bits = f32_to_bf16_bits(rng.standard_normal((300, 64)).astype(np.float32))
    q, _ = Qz.quantize_rows(bits)
    q2, _ = Qz.quantize_rows(Qz.int8_to_bf16_bits(q))
    assert np.array_equal(q, q2)
    assert np.array_equal(Qz.bf16_bits_to_f64(Qz.int8_to_bf16_bits(q)), q.astype(np.float64))


def test_header_enum():
    src = open(os.path.join(HERE, "..", "include", "aurora_b200.h")).read()
    m = re.search(r"typedef enum aur_dtype \{([^}]*)\}", src)
    assert m and re.search(r"AUR_I8\s*=\s*2", m.group(1))
    assert N.AUR_I8 == 2
    assert re.search(r"#define AUR_ABI_VERSION 3\b", src)


def test_index_argument_refusals():
    from aurora_b200.engine import Index

    with pytest.raises(ValueError, match="dim % 16"):
        Index(72, 64, dtype="int8")
    with pytest.raises(ValueError, match="dtype"):
        Index(64, 64, dtype="i8")
