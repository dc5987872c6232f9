"""Atlas-style pre-filters for the vector index: filter fields -> 64-bit row tags, MQL predicates -> sa_filter words.

An Atlas vector index declares some document fields as ``{"type": "filter", "path": ...}``; a ``$vectorSearch`` can then
restrict its top-k to the documents whose fields match an MQL ``filter``.  Here the index keeps one 64-bit tag per row
(include/sa_api.h, sa_corpus_bind_tags) and the scan applies each query's predicate in the normal form ``sa_filter``
(all_of, none_of, any_of[0], any_of[1]) before a row can enter a candidate list, so the answer stays exact over the
rows the filter admits.

``FilterSchema`` maps (field, value) pairs to tag bits; ``compile_filter`` turns an MQL document into the normal form.
Pure Python and numpy: nothing here needs a GPU.
"""
from __future__ import annotations

import numpy as np

MAX_PAIRS = 63          # bits 0..62 name (field, value) pairs ...
NEVER_BIT = 63          # ... bit 63 is carried by no row: a filter requiring it matches nothing
NEVER = np.uint64(1) << np.uint64(NEVER_BIT)
MATCH_ALL = np.zeros(4, dtype=np.uint64)
_RANGE_OPS = ("$gt", "$gte", "$lt", "$lte")


def _value_key(field: str, v):
    """A filter value as a category: strings, bools and ints (bool and int are different categories, as in MQL)."""
    if isinstance(v, bool):
        return ("bool", v)
    if isinstance(v, (int, np.integer)):
        return ("int", int(v))
    if isinstance(v, str):
        return ("str", v)
    raise ValueError(f"filter field {field!r}: value {v!r} of type {type(v).__name__} is not a string, bool or int")


def _row_values(field: str, row: dict) -> list:
    """The category keys a row carries for a field: one per array element, none when missing or null."""
    v = row.get(field) if row else None
    if v is None:
        return []
    items = v if isinstance(v, (list, tuple)) else [v]
    return [_value_key(field, x) for x in items if x is not None]


class FilterSchema:
    """The filter fields of an index and the bit of every (field, value) pair seen so far, assigned in first-seen row
    order (within a row: field order, then array order).  At most 63 pairs; bit 63 is NEVER."""

    def __init__(self, fields):
        self.fields = tuple(fields)
        if len(set(self.fields)) != len(self.fields):
            raise ValueError(f"filter fields repeat: {self.fields}")
        self.bits: dict[tuple[str, tuple], int] = {}

    def __len__(self) -> int:
        return len(self.bits)

    def bit(self, field: str, value) -> int | None:
        """The bit of (field, value), or None if no row carried it."""
        return self.bits.get((field, _value_key(field, value)))

    def tags(self, rows) -> np.ndarray:
        """Tags (uint64 [len(rows)]) of metadata dicts, assigning bits to new pairs.  If the new pairs would exceed 63,
        ValueError names the field and nothing is assigned."""
        new: dict[tuple[str, tuple], int] = {}
        per_row = []
        for row in rows:
            keys = []
            for f in self.fields:
                for vk in _row_values(f, row):
                    pair = (f, vk)
                    if pair not in self.bits and pair not in new:
                        if len(self.bits) + len(new) >= MAX_PAIRS:
                            raise ValueError(f"filter field {f!r}: value {vk[1]!r} would be distinct (field, value) "
                                             f"pair number {MAX_PAIRS + 1}; an index holds at most {MAX_PAIRS}")
                        new[pair] = len(self.bits) + len(new)
                    keys.append(pair)
            per_row.append(keys)
        self.bits.update(new)
        out = np.zeros(len(per_row), dtype=np.uint64)
        for i, keys in enumerate(per_row):
            t = 0
            for pair in keys:
                t |= 1 << self.bits[pair]
            out[i] = t
        return out

    def to_json(self) -> dict:
        order = sorted(self.bits.items(), key=lambda kv: kv[1])
        return {"fields": list(self.fields), "bits": [[f, vk[0], vk[1]] for (f, vk), _ in order]}

    @classmethod
    def from_json(cls, d: dict) -> "FilterSchema":
        s = cls(d["fields"])
        for i, (f, kind, v) in enumerate(d["bits"]):
            s.bits[(f, (kind, v))] = i
        return s


class _Form:
    def __init__(self):
        self.all_of = 0
        self.none_of = 0
        self.any_of: list[int] = []


def _bits_of(schema: FilterSchema, field: str, values) -> int:
    m = 0
    for v in values:
        if v is None:
            raise ValueError(f"filter on {field!r}: null values are not supported")
        b = schema.bit(field, v)
        if b is not None:
            m |= 1 << b
    return m


def _as_list(field: str, op: str, v) -> list:
    if not isinstance(v, (list, tuple)):
        raise ValueError(f"filter on {field!r}: {op} takes an array")
    return list(v)


def _field_atom(schema: FilterSchema, field: str, cond, form: _Form) -> None:
    if field not in schema.fields:
        raise ValueError(f"filter on {field!r}: not a filter field of this index (declared: {list(schema.fields)})")
    ops = cond if isinstance(cond, dict) else {"$eq": cond}
    if isinstance(cond, dict) and not cond:
        raise ValueError(f"filter on {field!r}: empty condition")
    for op, v in ops.items():
        if op in _RANGE_OPS:
            raise ValueError(f"filter on {field!r}: range operator {op} is not supported (categories only)")
        if op == "$eq":
            if v is None:
                raise ValueError(f"filter on {field!r}: $eq: null is not supported")
            if isinstance(v, (list, tuple, dict)):
                raise ValueError(f"filter on {field!r}: equality with an array or document is not supported")
            b = schema.bit(field, v)
            form.all_of |= (1 << b) if b is not None else (1 << NEVER_BIT)
        elif op == "$ne":
            if v is None or isinstance(v, (list, tuple, dict)):
                raise ValueError(f"filter on {field!r}: $ne takes a string, bool or int")
            form.none_of |= _bits_of(schema, field, [v])
        elif op == "$in":
            m = _bits_of(schema, field, _as_list(field, op, v))
            form.any_of.append(m if m else 1 << NEVER_BIT)
        elif op == "$nin":
            form.none_of |= _bits_of(schema, field, _as_list(field, op, v))
        elif op == "$not":
            if not isinstance(v, dict) or len(v) != 1 or next(iter(v)) not in ("$eq", "$in"):
                raise ValueError(f"filter on {field!r}: $not is supported over $eq or $in only")
            (inner, x), = v.items()
            if inner == "$eq":
                if x is None or isinstance(x, (list, tuple, dict)):
                    raise ValueError(f"filter on {field!r}: $not: {{$eq}} takes a string, bool or int")
                form.none_of |= _bits_of(schema, field, [x])
            else:
                form.none_of |= _bits_of(schema, field, _as_list(field, "$in", x))
        else:
            raise ValueError(f"filter on {field!r}: operator {op} is not supported")


def _positive_mask(schema: FilterSchema, doc, where: str) -> int:
    """A positive atom ({f: v}, {f: {$eq: v}}, {f: {$in: [...]}}) as the mask of bits any one of which satisfies it."""
    if not isinstance(doc, dict) or len(doc) != 1 or next(iter(doc)).startswith("$"):
        raise ValueError(f"{where}: each branch must be a single-field $eq / $in condition")
    (field, cond), = doc.items()
    f = _Form()
    if isinstance(cond, dict) and set(cond) - {"$eq", "$in"}:
        raise ValueError(f"{where}: each branch must be a single-field $eq / $in condition")
    if isinstance(cond, dict) and len(cond) != 1:
        raise ValueError(f"{where}: each branch must be a single-field $eq / $in condition")
    _field_atom(schema, field, cond, f)
    if f.all_of:
        return f.all_of & ~(1 << NEVER_BIT)
    return f.any_of[0] & ~(1 << NEVER_BIT)


def _compile(schema: FilterSchema, doc, form: _Form) -> None:
    if not isinstance(doc, dict):
        raise ValueError(f"a filter is an MQL document, not {type(doc).__name__}")
    for key, val in doc.items():
        if key == "$and":
            for part in _as_list("$and", "$and", val):
                _compile(schema, part, form)
        elif key == "$or":
            m = 0
            for branch in _as_list("$or", "$or", val):
                m |= _positive_mask(schema, branch, "$or")
            form.any_of.append(m if m else 1 << NEVER_BIT)
        elif key == "$nor":
            for branch in _as_list("$nor", "$nor", val):
                form.none_of |= _positive_mask(schema, branch, "$nor")
        elif key.startswith("$"):
            raise ValueError(f"operator {key} is not supported at the top level")
        else:
            _field_atom(schema, key, val, form)


def compile_filter(schema: FilterSchema, mql) -> np.ndarray:
    """An MQL filter document -> the sa_filter words uint64 [4] = (all_of, none_of, any_of[0], any_of[1]).

    Supported, with MQL's array semantics ({f: v} on an array field means "contains v"): implicit equality and $eq
    (all_of); $ne, $nin, $not over $eq / $in, and $nor of such atoms (none_of); $in (one any_of clause); $or of positive
    $eq / $in atoms on any fields (one any_of clause); $and and implicit conjunction.  $in: [] and an unseen value under
    $eq or $in match nothing (NEVER); $ne / $nin of an unseen value add no constraint.  Everything else -- range
    operators, $eq: null, undeclared fields, more than two any_of clauses, $or over conjunctions -- raises ValueError."""
    form = _Form()
    _compile(schema, mql if mql is not None else {}, form)
    if len(form.any_of) > 2:
        raise ValueError(f"filter needs {len(form.any_of)} $in / $or clauses; at most 2 are supported")
    any_of = form.any_of + [0] * (2 - len(form.any_of))
    return np.array([form.all_of, form.none_of, any_of[0], any_of[1]], dtype=np.uint64)


def filter_pass(tags: np.ndarray, f: np.ndarray) -> np.ndarray:
    """The normal form evaluated in numpy (bool [n]): the predicate the kernels apply, for host-side checks."""
    t = np.asarray(tags, dtype=np.uint64)
    f = np.asarray(f, dtype=np.uint64)
    z = np.uint64(0)
    ok = ((t & f[0]) == f[0]) & ((t & f[1]) == z)
    for a in (f[2], f[3]):
        ok &= (a == z) | ((t & a) != z)
    return ok
