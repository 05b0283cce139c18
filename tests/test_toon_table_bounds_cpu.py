"""Table rounds of the token-parallel TOON kernel at the edges of its staging buffers, on the CPU warp emulator.

Rows of an array of objects are checked (an_rows) and written (em_rows) 32 at a time, one lane per row.  A round's source
bytes are staged in the warp's staging buffer (json_tp.h ROW_SRC = 4 608 B; an_rows stages up to 4 576) and its output in
Shared::row_out (ROW_OUT = 3 840 B), as long as they fit:
  * rows whose sizes put the end of the staged source anywhere around ROW_SRC: the round takes only the leading rows that fit;
  * a single row longer than ROW_SRC: that round is one row, read straight from global memory (R = 1);
  * rounds whose output exceeds ROW_OUT: written straight to global memory.
Every document runs in both lane orders and at all 16 alignments to the 16-byte grid, against the oracle."""
import json

import pytest

import hostsim_util as hs
from oracle import toon_ref

ROW_SRC, ROW_OUT = 4608, 3840


def _doc(rows, compact):
    return json.dumps({"rows": rows, "n": len(rows)}, separators=(",", ":") if compact else (", ", ": "))


def table_bounds_docs():
    """(name, JSON text) pairs covering the staging boundaries of a table round."""
    docs = []
    # rows of a fixed size: 30 rows of ~150 B fill ROW_SRC; sizes around ROW_SRC / k put the cut after k rows
    for per_row in (ROW_SRC // 32 - 4, ROW_SRC // 31, ROW_SRC // 30, ROW_SRC // 16 + 1, ROW_SRC // 2 - 20, ROW_SRC // 2 + 20):
        fill = max(per_row - 40, 1)
        rows = [{"id": i, "v": "x" * (fill - len(str(i))), "ok": i % 3 == 0} for i in range(70)]
        docs.append((f"fixed{per_row}", _doc(rows, True)))
    # rows whose sizes vary, so that the staged prefix ends at every row position of a round
    rows = [{"id": i, "name": f"user{i}", "note": "lorem ipsum, " * (1 + (i * 7) % 23)} for i in range(200)]
    docs.append(("varying", _doc(rows, False)))
    # one row longer than ROW_SRC among short ones (first, middle, last row)
    for at in (0, 17, 39):
        rows = [{"k": i, "s": ("y" * (ROW_SRC + 300)) if i == at else f"s{i}"} for i in range(40)]
        docs.append((f"long_row_at{at}", _doc(rows, True)))
    # a table of long rows only: every round is one row
    rows = [{"k": i, "s": "z" * (ROW_SRC + 17 * i)} for i in range(5)]
    docs.append(("all_long", _doc(rows, True)))
    # rounds of 32 staged rows whose output exceeds ROW_OUT (~128 B of output per row), and rounds just below it
    for val in (ROW_OUT // 32 + 8, ROW_OUT // 32 - 8, ROW_OUT // 30):
        rows = [{"a": "w" * val, "b": i} for i in range(100)]
        docs.append((f"out{val}", _doc(rows, True)))
    # quoted cells (commas, leading blanks) make the output longer than the plain text
    rows = [{"a": " lead, comma " + "q" * 100, "b": -i * 1.5} for i in range(64)]
    docs.append(("quoted", _doc(rows, False)))
    # dense tokens: more than one window of TOK_WIN = 192 tokens per 1 KiB step of the tokenizer (its masks are rebuilt per window)
    docs.append(("dense_ints", json.dumps({"v": [i % 10 for i in range(3000)], "s": ["a", "b"] * 400}, separators=(",", ":"))))
    rows = [{"a": i % 10, "b": "x", "c": i % 2 == 0} for i in range(300)]
    docs.append(("dense_rows", _doc(rows, True)))
    return docs


DOCS = table_bounds_docs()


@pytest.mark.parametrize("name,text", DOCS, ids=[n for n, _ in DOCS])
def test_table_rounds_at_staging_bounds(name, text):
    exp = toon_ref.process_text(text, 0, 1 << 30)
    assert exp is not None, name
    for shift in range(16):
        for lane_order in (0, 1):
            st, got = hs.toon_tp(text, report_errors=False, order=lane_order | (shift << 4))
            assert st == 0 and got == exp, (name, shift, lane_order, st)
