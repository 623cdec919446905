"""Minimal stand-in for ``weaviate.classes.query.Filter`` / ``HybridFusion``.

The reference builds its tenant and discovery scopes with this algebra
(server/routes/knowledge_base/weaviate_client.py:244-249, :301-304, :380-385;
server/chat/background/rca_prompt_builder.py:286-289): ``by_property(p).equal(v)``,
``.like("prefix*")``, ``.less_than(v)``, combined with ``&`` and ``|``.  Only what those
call sites use is implemented.  ``_eval`` is the one definition of what a filter matches: the
host path runs it per metadata row, and ``compile_program`` runs it once per distinct property
value to build the bitmaps a device program tests row codes against.  An expression is a plain tree
(``to_json`` / ``from_json``) so it can cross the engine daemon's socket.
"""

from __future__ import annotations

import fnmatch
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

_LEAF_OPS = ("eq", "ne", "like", "lt", "gt")


def _eval(tree: List[Any], p: Dict[str, Any]) -> bool:
    op = tree[0]
    if op == "and":
        return _eval(tree[1], p) and _eval(tree[2], p)
    if op == "or":
        return _eval(tree[1], p) or _eval(tree[2], p)
    name, value = tree[1], tree[2]
    got = p.get(name)
    if op == "eq":
        return got == value
    if op == "ne":
        return got != value
    if op == "like":   # Weaviate LIKE: '*' any run of characters, '?' exactly one
        return isinstance(got, str) and fnmatch.fnmatchcase(got, value)
    if op == "lt":
        return got is not None and got < value
    if op == "gt":
        return got is not None and got > value
    raise ValueError(f"unknown filter operator {op!r}")


def _desc(tree: List[Any]) -> str:
    op = tree[0]
    if op in ("and", "or"):
        return f"({_desc(tree[1])} {op.upper()} {_desc(tree[2])})"
    sym = {"eq": "==", "ne": "!=", "like": "LIKE", "lt": "<", "gt": ">"}[op]
    return f"{tree[1]} {sym} {tree[2]!r}"


class _Expr:
    def __init__(self, tree: List[Any]):
        self.tree = tree

    @property
    def desc(self) -> str:
        return _desc(self.tree)

    def matches(self, props: Dict[str, Any]) -> bool:
        return bool(_eval(self.tree, props))

    def __and__(self, other: "_Expr") -> "_Expr":
        return _Expr(["and", self.tree, other.tree])

    def __or__(self, other: "_Expr") -> "_Expr":
        return _Expr(["or", self.tree, other.tree])

    def __repr__(self) -> str:
        return f"Filter[{self.desc}]"

    # ---- wire format (engine daemon) -------------------------------------------------
    def to_json(self) -> List[Any]:
        return self.tree

    @staticmethod
    def from_json(tree: Optional[List[Any]]) -> Optional["_Expr"]:
        if tree is None:
            return None

        def check(t):
            if not isinstance(t, (list, tuple)) or len(t) != 3:
                raise ValueError("malformed filter expression")
            if t[0] in ("and", "or"):
                return [t[0], check(t[1]), check(t[2])]
            if t[0] not in _LEAF_OPS or not isinstance(t[1], str):
                raise ValueError("malformed filter expression")
            return [t[0], t[1], t[2]]

        return _Expr(check(tree))

    # ---- tenant terms ----------------------------------------------------------------
    def required_equalities(self) -> Dict[str, Any]:
        """Property == value terms every match must satisfy (the AND-spine of the tree); used to
        narrow the metadata scan before the full predicate runs."""
        out: Dict[str, Any] = {}

        def walk(t):
            if t[0] == "and":
                walk(t[1]); walk(t[2])
            elif t[0] == "eq":
                out.setdefault(t[1], t[2])

        walk(self.tree)
        return out


# ---------------------------------------------------------------------- device programs
# A filter runs on the GPU as a postfix program over per-row int32 codes (include/aurora_b200.h, aur_search_filtered):
# every property a filter names becomes a code column whose dictionary maps each exact Python value to a code (-1 =
# absent), and a leaf becomes a bitmap over those codes, computed by ``_eval`` itself once per distinct value -- so the
# device answers what ``_Expr.matches`` answers, row by row, whatever the operator and the value types.
FILTER_LEAF, FILTER_AND, FILTER_OR = 0, 1, 2
MAX_LEAVES = 32
_PLAIN = (str, int, float, bool, type(None))   # value types whose equality with a str is str identity (JSON scalars)


class AttrColumn:
    """One property as a device code column: ``values[c]`` is the value behind code c.  Leaf bitmaps are cached, at
    most CACHE_LEAVES per column (least recently used out), and extended only over the values added since they were
    computed.  ``eq`` / ``ne`` against a str over a column of JSON scalars come straight from the dictionary instead: no
    other such value equals a str, so the one code of that exact string is the whole answer."""

    CACHE_LEAVES = 256

    def __init__(self, name: str, col: int):
        self.name, self.col = name, int(col)
        self.values: List[Any] = []
        self._codes: Dict[Any, int] = {}
        self._bits: "OrderedDict[Any, np.ndarray]" = OrderedDict()
        self._plain = True              # every value's type is exactly one of _PLAIN

    def code(self, props: Dict[str, Any]) -> int:
        """The code of ``props``' value of this property (-1: the property is absent); new values get the next code.
        Values are told apart by type as well (1, 1.0 and True are three codes); an unhashable value raises TypeError."""
        if self.name not in props:
            return -1
        v = props[self.name]
        key = (type(v), v)
        c = self._codes.get(key)
        if c is None:
            c = self._codes[key] = len(self.values)
            self.values.append(v)
            self._plain = self._plain and type(v) in _PLAIN
        return c

    def leaf_bits(self, op: str, value: Any) -> np.ndarray:
        """bits[c + 1] = the leaf ``[op, name, value]`` on a row whose code is c (bits[0]: absent); never modified
        afterwards (an extension is a new array)."""
        if op in ("eq", "ne") and type(value) is str and self._plain:
            bits = np.zeros(len(self.values) + 1, dtype=bool)
            c = self._codes.get((str, value))
            if c is not None:
                bits[c + 1] = True
            return ~bits if op == "ne" else bits       # absent: None == value is False, None != value True
        tree = [op, self.name, value]
        try:
            key = (op, type(value), value)
            hash(key)
        except TypeError:
            key = None
        bits = self._bits.get(key) if key is not None else None
        if bits is not None:
            self._bits.move_to_end(key)
        known = 0 if bits is None else len(bits) - 1
        if bits is None or known < len(self.values):
            new = [bool(_eval(tree, {self.name: v})) for v in self.values[known:]]
            if bits is None:
                bits = np.array([bool(_eval(tree, {}))] + new, dtype=bool)
            else:
                bits = np.concatenate([bits, np.array(new, dtype=bool)])
            if key is not None:
                self._bits[key] = bits
                if len(self._bits) > self.CACHE_LEAVES:
                    self._bits.popitem(last=False)
        return bits


def compile_program(expr: Optional["_Expr"], columns: Dict[str, AttrColumn],
                    tenant: Optional[Tuple[int, int]] = None) -> Tuple[List[Tuple[int, np.ndarray]], List[int]]:
    """``expr`` AND the tenant clause ``row_user == u OR (o >= 0 AND row_org == o)`` (``tenant`` = (u, o) codes; None =
    no clause) as a postfix program: (leaves [(column, bits)], tokens) where a token >= 0 names a leaf and
    -1 / -2 stand for AND / OR.  Raises when a leaf evaluation raises, when a property has no column in ``columns`` and
    when the program would have more than MAX_LEAVES leaves.  ``pack_programs`` turns programs into the C arrays."""
    leaves: List[Tuple[int, np.ndarray]] = []
    toks: List[int] = []

    def leaf(col: int, bits: np.ndarray) -> None:
        toks.append(len(leaves))
        leaves.append((col, bits))

    def walk(t) -> None:
        if t[0] in ("and", "or"):
            walk(t[1]); walk(t[2])
            toks.append(-1 if t[0] == "and" else -2)
            return
        if t[0] not in _LEAF_OPS:
            raise ValueError(f"unknown filter operator {t[0]!r}")
        c = columns[t[1]]
        leaf(c.col, c.leaf_bits(t[0], t[2]))

    if expr is not None:
        walk(expr.tree)
    if tenant is not None:
        u, o = int(tenant[0]), int(tenant[1])
        leaf(0, np.arange(u + 2) == u + 1 if u >= -1 else np.zeros(0, bool))
        leaf(1, np.arange(o + 2) == o + 1 if o >= 0 else np.zeros(0, bool))
        toks.append(-2)
        if expr is not None:
            toks.append(-1)
    if not leaves:
        raise ValueError("empty filter program")
    if len(leaves) > MAX_LEAVES:
        raise ValueError(f"filter has {len(leaves)} leaves; the device evaluates at most {MAX_LEAVES}")
    return leaves, toks


def pack_programs(programs):
    """Programs of ``compile_program`` as aur_search_filtered's arrays: (tokens int32 [n, 4], offsets int32
    [len + 1], bitmap uint32).  Every leaf's bitmap starts on a word boundary."""
    rows: List[List[int]] = []
    offsets = [0]
    chunks: List[np.ndarray] = []
    words = 0
    for leaves, toks in programs:
        placed = []
        for col, bits in leaves:
            b = np.zeros(-(-max(len(bits), 1) // 32) * 32, dtype=bool)
            b[:len(bits)] = bits
            placed.append((col, words * 32, len(bits)))
            chunks.append(np.packbits(b, bitorder="little").view(np.uint32))
            words += len(b) // 32
        for t in toks:
            rows.append([FILTER_LEAF, *placed[t]] if t >= 0 else [FILTER_AND if t == -1 else FILTER_OR, 0, 0, 0])
        offsets.append(len(rows))
    tokens = np.asarray(rows, dtype=np.int32).reshape(-1, 4)
    bitmap = np.concatenate(chunks) if chunks else np.zeros(1, np.uint32)
    return np.ascontiguousarray(tokens), np.asarray(offsets, dtype=np.int32), np.ascontiguousarray(bitmap, dtype=np.uint32)


class _Property:
    def __init__(self, name: str):
        self.name = name

    def equal(self, value: Any) -> _Expr:
        return _Expr(["eq", self.name, value])

    def not_equal(self, value: Any) -> _Expr:
        return _Expr(["ne", self.name, value])

    def like(self, pattern: str) -> _Expr:
        return _Expr(["like", self.name, pattern])

    def less_than(self, value: Any) -> _Expr:
        return _Expr(["lt", self.name, value])

    def greater_than(self, value: Any) -> _Expr:
        return _Expr(["gt", self.name, value])


class Filter:
    @staticmethod
    def by_property(name: str) -> _Property:
        return _Property(name)

    from_json = staticmethod(_Expr.from_json)


class HybridFusion:
    RANKED = "FUSION_TYPE_RANKED"
    RELATIVE_SCORE = "FUSION_TYPE_RELATIVE_SCORE"
