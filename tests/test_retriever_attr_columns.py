"""KnowledgeBase's attribute columns (the device-filter path) on a recording CPU double: a property gets a column the
first time a filter names it, inserts keep it current, and a property whose values cannot be coded gives its column
back for the next property."""

from __future__ import annotations

import numpy as np

from aurora_b200 import retriever as R
from aurora_b200.filters import Filter
from tests.doubles import HashEmbedder, OracleIndex


class RecordingIndex(OracleIndex):
    dtype = 0                                           # a bf16 shard

    def __init__(self, dim, capacity):
        super().__init__(dim, capacity)
        self.codes = {}                                 # column -> {id: code}

    def set_attrs(self, col, ids, codes):
        self.codes.setdefault(col, {}).update(zip(np.asarray(ids).tolist(), np.asarray(codes).tolist()))

    def search_filtered(self, queries, k, programs, q_program=None, max_list_rows=0):
        raise AssertionError("not searched here")


def _kb():
    kb = R.KnowledgeBase(HashEmbedder(16), capacity=64, index_factory=lambda d, c: RecordingIndex(d, c))
    kb.insert_objects([(f"k{i}", {"tag": f"t{i % 3}"}, "x") for i in range(6)], "u")
    return kb


def test_columns_follow_inserts_and_unhashable_values_free_their_slot():
    kb = _kb()
    prog = kb._device_program(Filter.by_property("tag").equal("t1"), False, None, None)
    assert prog is not None
    col = kb._attr_cols["tag"].col
    assert col == 2 and col not in kb._attr_free
    assert kb.index.codes[col] == {i: i % 3 for i in range(6)}
    kb.insert_objects([("k9", {"tag": "t7"}, "y")], "u")                    # inserts keep the column current
    assert kb.index.codes[col][6] == 3
    kb.insert_objects([("k10", {"tag": ["a", "list"]}, "z")], "u")          # no code for a list
    assert "tag" not in kb._attr_cols and col in kb._attr_free
    assert kb._device_program(Filter.by_property("tag").equal("t1"), False, None, None) is None   # host path from now on
    assert kb._device_program(Filter.by_property("other").equal(1), False, None, None) is not None
    assert kb._attr_cols["other"].col == 3
    n_free = len(kb._attr_free)
    for i in range(n_free):                            # every slot the pool holds can be used, the returned one included
        assert kb._device_program(Filter.by_property(f"p{i}").equal(1), False, None, None) is not None
    assert not kb._attr_free and col in {c.col for c in kb._attr_cols.values()}
