"""A list item whose first value is an array that starts with an object with nested values and later holds an element that is not
an object: toon.py tries that array as columnar without a type check (toon.py:400-404), so the key sets of the rows before that
element decide between "not columnar" (the item is encoded) and the reference's AttributeError.  The token-parallel kernel body
(csrc/json_tp.h, on the CPU warp emulator, tools/toon_emu.py) with its resolving pass behind the first one, as toon_tp_kernel runs
them, must reach the oracle's verdict itself, without handing the unit to the sequential encoder."""
import itertools
import json
import os
import sys

import pytest

from oracle import toon_ref

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import toon_emu  # noqa: E402

FALLBACK = 7


def oracle(text):
    """(0, TOON text) or (4, None) for the reference's AttributeError, without the "strictly smaller" rule."""
    try:
        return 0, toon_ref.encode(toon_ref.loads_strict(text))
    except toon_ref.ToonCrash:
        return 4, None


def mixed_family():
    """A first row with a nested value, later rows with the same, permuted, fewer, more or other keys, and an element that is not an
    object at every position; glbvs / yacxa have the same 32-bit FNV-1a hash."""
    row0 = {"id": 1, "meta": {"k": 1}, "name": "x"}
    later = [
        {"id": 2, "meta": {"k": 2}, "name": "y"},                  # same keys
        {"name": "z", "id": 3, "meta": [1, 2]},                    # same keys, other order
        {"id": 4, "name": "w"},                                    # a key missing
        {"id": 5, "meta": 1, "name": "v", "extra": True},          # a key more
        {"id": 6, "meta": 2, "nome": "u"},                         # same count, one key differs
    ]
    nondict = [7, "s", [1, 2], None]
    out = []
    for n_rows in range(0, 4):
        for rows in itertools.product(range(len(later)), repeat=n_rows):
            for nd in nondict[:2] if n_rows > 1 else nondict:
                arr = [row0] + [later[r] for r in rows] + [nd]
                out.append([{"rows": arr, "z": 1}])
                out.append({"items": [{"rows": arr + [row0]}, 3]})
                out.append({"rows": arr})                               # not a list item: the array is encoded as list items
    a = {"glbvs": {"x": 1}, "q": 1}
    b = {"yacxa": {"x": 2}, "q": 2}
    out.append([{"rows": [a, b, 1]}])                                   # different keys, equal hashes
    out.append([{"rows": [a, dict(a), 1]}])
    out.append([{"rows": [{}, {"a": 1}, 1]}])                            # empty first row: never columnar
    out.append([{"rows": [{"a": {"b": 1}}, {"a": 2}, 1]}, {"rows": [{"a": [1]}, {"b": 2}, 1]}])
    return out


@pytest.mark.parametrize("order", [0, 1])
def test_mixed_list_item_arrays_resolved_against_the_oracle(order):
    n_crash = n_conv = 0
    for doc in mixed_family():
        text = json.dumps(doc)
        exp = oracle(text)
        st, got, why, _, _ = toon_emu.toon_tp(text, unlimited=True, order=order)
        assert st != FALLBACK, (text, why)
        assert (st, got if st == 0 else None) == exp, (text, st, got, exp)
        n_crash += exp[0] == 4
        n_conv += exp[0] == 0
    assert n_crash > 20 and n_conv > 20, (n_crash, n_conv)
