"""filters.compile_program: a filter tree compiled to a postfix program over per-row codes answers what
``_Expr.matches`` answers, row by row.  The program is evaluated here in numpy exactly as csrc/filter.cu evaluates it
(bit code + 1 of a leaf's bitmap slice, a bit stack for AND / OR)."""

from __future__ import annotations

import numpy as np
import pytest

from aurora_b200.filters import (FILTER_AND, FILTER_LEAF, MAX_LEAVES, AttrColumn, Filter, compile_program,
                                 pack_programs)


def run_programs(tokens, offsets, bitmap, cols):
    """[n_programs, n_rows] bool: the device's evaluation (filter_count_kernel) restated in numpy."""
    bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little").astype(bool)
    n = len(next(iter(cols.values())))
    out = []
    for p in range(len(offsets) - 1):
        stack = []
        for kind, col, off, ln in tokens[offsets[p]:offsets[p + 1]]:
            if kind == FILTER_LEAF:
                idx = cols[col] + 1
                ok = (idx >= 0) & (idx < ln)
                v = np.zeros(n, bool)
                v[ok] = bits[off + idx[ok]]
                stack.append(v)
            else:
                b, a = stack.pop(), stack.pop()
                stack.append(a & b if kind == FILTER_AND else a | b)
        assert len(stack) == 1
        out.append(stack[0])
    return np.array(out)


def _table(rng, n):
    words = ["alpha", "beta", "gamma", "delta", "a?c", "x[y]"]
    rows = []
    for i in range(n):
        p = {}
        r = rng.random()
        if r < 0.7:
            p["document_id"] = (f"discovery:{rng.integers(20)}" if rng.random() < 0.5 else
                                f"doc-{rng.choice(words)}-{rng.integers(5)}")
        elif r < 0.8:
            p["document_id"] = None
        if rng.random() < 0.8:
            p["org_id"] = f"o{rng.integers(6)}"
        if rng.random() < 0.75:
            p["n"] = int(rng.integers(-3, 12)) if rng.random() < 0.9 else None
        if rng.random() < 0.85:
            p["created_at"] = f"2026-0{rng.integers(1, 10)}-{rng.integers(10, 29)}T{rng.integers(10, 24)}:00:00+00:00"
        if rng.random() < 0.6:
            p["mixed"] = int(rng.integers(4)) if rng.random() < 0.5 else str(rng.choice(words))
        rows.append(p)
    return rows


def _leaf(rng):
    prop = rng.choice(["document_id", "org_id", "n", "created_at", "mixed", "ghost"])
    F = Filter.by_property(str(prop))
    if prop == "document_id":
        return rng.choice([F.like("discovery:*"), F.like("doc-?????-*"), F.like("doc-[ab]*"), F.equal(None),
                           F.not_equal("discovery:3"), F.like("*[0-4]")])
    if prop == "org_id":
        return F.equal(f"o{rng.integers(7)}") if rng.random() < 0.7 else F.not_equal(f"o{rng.integers(7)}")
    if prop == "n":
        return rng.choice([F.less_than(int(rng.integers(10))), F.greater_than(int(rng.integers(10))), F.equal(3),
                           F.equal(3.0), F.not_equal(None)])
    if prop == "created_at":
        return rng.choice([F.less_than("2026-05-01"), F.greater_than("2026-03-15T12"), F.like("2026-0[1-3]-*")])
    if prop == "mixed":
        return rng.choice([F.equal(1), F.equal("beta"), F.like("a?c"), F.not_equal(2), F.equal(True)])
    return rng.choice([F.equal("x"), F.less_than(5), F.like("*"), F.not_equal(None)])


def _tree(rng, n_leaves):
    if n_leaves == 1:
        return _leaf(rng)
    left = int(rng.integers(1, n_leaves))
    a, b = _tree(rng, left), _tree(rng, n_leaves - left)
    return a & b if rng.random() < 0.5 else a | b


def _codes(columns, rows):
    return {c.col: np.array([c.code(p) for p in rows], np.int32) for c in columns.values()}


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_equal_matches(seed):
    rng = np.random.default_rng(seed)
    rows = _table(rng, 400)
    names = ["document_id", "org_id", "n", "created_at", "mixed", "ghost"]
    columns = {nm: AttrColumn(nm, 2 + i) for i, nm in enumerate(names)}
    cols = _codes(columns, rows)
    exprs = [_tree(rng, int(n)) for n in [1, 2, 3, 5, 8, 13, 21, 32] + list(rng.integers(1, 33, size=8))]
    programs = [compile_program(e, columns) for e in exprs]
    got = run_programs(*pack_programs(programs), cols)
    for e, g in zip(exprs, got):
        want = np.array([e.matches(p) for p in rows])
        assert np.array_equal(g, want), e.desc


def test_bitmaps_extend_over_new_values():
    rng = np.random.default_rng(11)
    rows = _table(rng, 200)
    columns = {nm: AttrColumn(nm, 2 + i) for i, nm in enumerate(["document_id", "org_id", "n"])}
    e = (Filter.by_property("org_id").equal("o2") & Filter.by_property("document_id").like("discovery:*")) | \
        Filter.by_property("n").greater_than(7)
    before = compile_program(e, columns)
    _codes(columns, rows)                               # the table's values get codes after the first compile
    more = rows + [{"org_id": "o2", "document_id": "discovery:new"}, {"n": 99}, {"org_id": "o9"}]
    cols = _codes(columns, more)
    got = run_programs(*pack_programs([compile_program(e, columns), before]), cols)
    want = np.array([e.matches(p) for p in more])
    assert np.array_equal(got[0], want)
    assert len(before[0][0][1]) == 1                    # the first program knew only "absent"


def test_tenant_clause_over_tenant_codes():
    rng = np.random.default_rng(3)
    n = 300
    user = rng.integers(-1, 5, size=n).astype(np.int32)
    org = rng.integers(-1, 4, size=n).astype(np.int32)
    rows = _table(rng, n)
    columns = {"org_id": AttrColumn("org_id", 2)}
    cols = {0: user, 1: org, **_codes(columns, rows)}
    f = Filter.by_property("org_id").not_equal("o1")
    for u, o in [(2, 1), (-2, 3), (4, -1), (-2, -1), (0, 0)]:
        tokens, offsets, bm = pack_programs([compile_program(None, columns, tenant=(u, o)),
                                             compile_program(f, columns, tenant=(u, o))])
        got = run_programs(tokens, offsets, bm, cols)
        scope = (user == u) | ((o >= 0) & (org == o))
        assert np.array_equal(got[0], scope)
        assert np.array_equal(got[1], scope & np.array([f.matches(p) for p in rows]))


def test_leaf_that_raises_raises_in_compile():
    rows = [{"n": 3}, {"n": "three"}, {}]
    columns = {"n": AttrColumn("n", 2)}
    _codes(columns, rows)
    e = Filter.by_property("n").less_than(5)
    with pytest.raises(TypeError):
        [e.matches(p) for p in rows]
    with pytest.raises(TypeError):
        compile_program(e, columns)


def test_limits():
    columns = {"a": AttrColumn("a", 2)}
    e = Filter.by_property("a").equal(0)
    for i in range(1, MAX_LEAVES):
        e = e | Filter.by_property("a").equal(i)
    compile_program(e, columns)
    with pytest.raises(ValueError):
        compile_program(e | Filter.by_property("a").equal(-1), columns)
    with pytest.raises(ValueError):                     # 31 leaves + the tenant clause's two
        compile_program(e, columns, tenant=(0, 0))
    with pytest.raises(KeyError):
        compile_program(Filter.by_property("b").equal(1), columns)
    with pytest.raises(TypeError):
        AttrColumn("a", 2).code({"a": [1, 2]})
    assert AttrColumn("a", 2).code({}) == -1


def test_string_equality_from_the_dictionary_and_bounded_cache():
    """eq / ne against a str over JSON scalars come from the dictionary; any other column evaluates _eval per value.
    Both equal matches; the leaf cache keeps at most CACHE_LEAVES bitmaps per column."""
    rows = [{"u": f"user{i % 40}"} for i in range(300)] + [{"u": None}, {}, {"u": 3}, {"u": True}, {"u": 1.0}]
    plain = AttrColumn("u", 2)
    cols = {2: np.array([plain.code(p) for p in rows], np.int32)}

    class Loose(str):               # a str subclass: equal to a plain str of the same text
        pass
    mixed = AttrColumn("u", 3)
    rows2 = rows + [{"u": Loose("user7")}]
    cols[3] = np.array([mixed.code(p) for p in rows2], np.int32)
    for value in ("user7", "nobody", "user39"):
        for op in ("equal", "not_equal"):
            e = getattr(Filter.by_property("u"), op)(value)
            got = run_programs(*pack_programs([compile_program(e, {"u": plain})]), {2: cols[2]})[0]
            assert np.array_equal(got, np.array([e.matches(p) for p in rows]))
            got = run_programs(*pack_programs([compile_program(e, {"u": mixed})]), {3: cols[3]})[0]
            assert np.array_equal(got, np.array([e.matches(p) for p in rows2]))
    assert not plain._bits                                  # the dictionary path caches nothing
    for i in range(AttrColumn.CACHE_LEAVES + 40):
        compile_program(Filter.by_property("u").like(f"user{i}*"), {"u": plain})
    assert len(plain._bits) == AttrColumn.CACHE_LEAVES
