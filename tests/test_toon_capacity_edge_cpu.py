"""toon_encoder keeps a conversion only when the TOON text is strictly smaller than the input, and every encoder gets that rule as a
capacity of n - 1 bytes.  These tests put documents exactly at the edge of that decision: padded with spaces (at the head, at the
tail, between tokens) to n = L - 1, L, L + 1 and L + 2 bytes, where L is the TOON length of oracle/toon_ref.py, on the host builds
of the sequential encoder (csrc/json_toon.h, the source toon_kernel compiles; with and without giving up at the first byte past
the capacity) and of the token-parallel kernel body (csrc/json_tp.h on the warp emulator; both lane orders, two alignments).

The trimming family: a columnar array as the first field of a list item whose header key holds raw newlines.  The reference
strips every header line after the first (toon.py:405-413), so trailing whitespace the encoder has already written is taken back
at the next newline.  When that whitespace crosses the capacity and the final text still fits, the text is strictly smaller and
must be converted.  Each such document is swept over every length from its compact form to past the whitespace it trims.

tests/test_toon_capacity_edge_gpu.py runs the same corpora through the C ABI and the Python API on the GPU."""
import json
import os
import random

import pytest

import hostsim_util as hs
from mcp_context_forge_b200 import synth
from oracle import toon_ref

TS_CONVERTED, TS_NOT_SMALLER, TS_NOT_JSON, TS_VALUE_ERROR, TS_ATTR_ERROR, HANDED_OVER = 0, 1, 2, 3, 4, 7
FB_KEY_ESCAPE = 2                                     # csrc/json_tp.h FB_*
FB_REASONS = range(1, 9)
EDGE = (-1, 0, 1, 2)                                  # n - L
WHERE = ("tail", "head", "mid")
TP_ORDERS = (0, 1, 7 << 4, 1 | (13 << 4))             # lane order (bit 0) x the unit's offset in the 16-byte grid (bits 4..)
GOLD = os.path.join(os.path.dirname(__file__), "golden", "toon.json")

# every code point outside ASCII that str.isspace (and so str.strip) takes, and the two ASCII ones a JSON key may carry
SPACES = [" ", "\t", "\x85", "\xa0", "\u1680"] + [chr(c) for c in range(0x2000, 0x200B)] + ["\u2028", "\u2029", "\u202f", "\u205f", "\u3000"]


# ------------------------------------------------------------------------------------------------------------------- the oracle
def oracle(doc: str):
    """(status, TOON text or None) of the reference for `doc` with every error reported: the text when it is strictly smaller."""
    try:
        obj = toon_ref.loads_strict(doc)
    except (ValueError, TypeError):
        return TS_NOT_JSON, None
    try:
        t = toon_ref.encode(obj)
    except toon_ref.ToonCrash:
        return TS_ATTR_ERROR, None
    except ValueError:
        return TS_VALUE_ERROR, None
    exp = (TS_CONVERTED, t) if len(t.encode("utf-8")) < len(doc.encode("utf-8")) else (TS_NOT_SMALLER, None)
    assert exp[1] == toon_ref.process_text(doc, min_size=0, max_size=1 << 30)
    return exp


def agrees(got, exp, report_errors: bool) -> bool:
    """An encoder that stops at the first byte past the capacity may report a later error as "not smaller"; the text is the same."""
    if report_errors or exp[0] in (TS_CONVERTED, TS_NOT_JSON):
        return got == exp
    return got[1] is None and got[0] in (TS_NOT_SMALLER, TS_VALUE_ERROR, TS_ATTR_ERROR)


# ------------------------------------------------------------------------------------------------------------- padding to n bytes
def compact(doc: str):
    """(doc without the whitespace between its tokens, offsets just after its structural characters)."""
    out, gaps, in_str, esc = [], [], False, False
    for ch in doc:
        if in_str:
            out.append(ch)
            if esc:
                esc = False
            elif ch == "\\":
                esc = True
            elif ch == '"':
                in_str = False
        elif ch not in " \t\n\r":
            out.append(ch)
            in_str = ch == '"'
            if ch in "[{,:":
                gaps.append(len(out))
    return "".join(out), gaps


def pad(doc: str, gaps, k: int, where: str) -> str:
    if where == "tail":
        return doc + " " * k
    if where == "head":
        return " " * k + doc
    g = gaps[len(gaps) // 2]
    return doc[:g] + " " * k + doc[g:]


def toon_len(doc: str) -> int:
    return len(toon_ref.encode(toon_ref.loads_strict(doc)).encode("utf-8"))


# ------------------------------------------------------------------------------------------------------------------ the corpus
def golden_docs():
    with open(GOLD, encoding="utf-8") as f:
        g = json.load(f)
    docs = [c["json"] for c in g["encode"] if "toon" in c]
    for block in g["plugin"]:
        for c in block["cases"]:
            res = c["result"]
            for item in res.get("content", []) if isinstance(res, dict) else []:
                if isinstance(item, dict) and isinstance(item.get("text"), str):
                    docs.append(item["text"])
    return docs


def synth_docs():
    out = []
    for size in (160, 700, 3000):
        for seed in range(3):
            out += [synth.payload("A", size, seed=seed), synth.payload("B", size, seed=seed)]
            out.append(json.dumps({"doc": synth.payload("C", size, seed=seed), "n": seed}))
    return out


def larger_docs():
    """Documents whose TOON text outgrows the JSON: list items nested in list items, each level indented further."""
    rng = random.Random(11)
    out = []
    for _ in range(40):
        v = rng.randint(0, 99)
        for d in range(rng.randint(2, 7)):
            v = {"k%d" % d: [v, {"x": [1, [2, v]]}] if rng.random() < 0.5 else [{"a": v, "b": [v]}]}
        out.append(json.dumps(v, separators=(",", ":")))
    return out


def lifted(doc: str):
    """An object document with a string field in front, long enough to take the document past the plugin's 100-byte minimum."""
    c, _ = compact(doc)
    if not c.startswith("{") or c == "{}" or len(c.encode("utf-8")) >= 100:
        return None
    return '{"_pad":"' + "p" * (110 - len(c)) + '",' + c[1:]


def base_docs():
    """Documents that parse and encode, each once."""
    seen, out = set(), []
    for d in golden_docs() + synth_docs() + larger_docs():
        for x in (d, lifted(d)):
            if x is None or x in seen or oracle(x)[0] not in (TS_CONVERTED, TS_NOT_SMALLER):
                continue
            seen.add(x)
            out.append(x)
    return out


def edge_corpus():
    """[(document, n - L)]: every base document padded to each edge length its compact form allows, at each place."""
    out = []
    for d in base_docs():
        c, gaps = compact(d)
        C, L = len(c.encode("utf-8")), toon_len(c)
        for e in EDGE:
            if L + e < C:
                continue
            for where in WHERE:
                if where != "mid" or gaps:
                    out.append((pad(c, gaps, L + e - C, where), e))
    return out


# ------------------------------------------------------------------------------------------------------------ the trimming family
def trim_doc(ws: str, depth: int, lines: int, reps: int, trimmed: int, blank: bool, rows: int, after: bool, other_key: bool) -> str:
    """A columnar array as the first field of a list item, `depth` list items deep.  Its header key starts with the marker "hdrQ"
    and holds `lines` short lines (they make the TOON text grow against the JSON), `trimmed` lines ending in `reps` times `ws`, an
    all-whitespace line when `blank`, and a last line "z"."""
    key = "hdrQ" + "\nk" * lines + "".join("\n" + ws + "t%d" % i + ws * reps for i in range(trimmed)) + ("\n" + ws * 3 if blank else "") + "\nz"
    row_keys = ["b", key] if other_key else [key]
    item = {"team": [{k: 10 * r + j for j, k in enumerate(row_keys)} for r in range(rows)]}
    if after:
        item["n"] = 7
    doc = [item]
    for lvl in range(depth):
        doc = {"users%d" % lvl: doc} if lvl % 2 == 0 else [doc]
        if lvl:
            doc = {"w": doc} if isinstance(doc, list) else [doc]
    return json.dumps(doc, separators=(",", ":"), ensure_ascii=False)


def trim_peak(doc: str):
    """(L, peak, trimmed): the TOON length, the most bytes the encoder has written at any point (the last whitespace of a stripped
    header line is written, then taken back at its newline) and the bytes so taken back.  A capacity of n - 1 with L < n <= peak is where the bytes written cross it and
    the final text still fits."""
    obj = json.loads(doc)
    toon = toon_ref.encode(obj)
    lines = toon.split("\n")
    h = next(i for i, ln in enumerate(lines) if "hdrQ" in ln)
    keys = []

    def find(x):
        if isinstance(x, dict):
            for k, v in x.items():
                if k == "team":
                    keys.extend(v[0].keys())
                find(v)
        elif isinstance(x, list):
            for v in x:
                find(v)
    find(obj)
    pieces = ",".join(keys).split("\n")
    peak = L = len(toon.encode("utf-8"))
    end = sum(len(ln.encode("utf-8")) + 1 for ln in lines[:h]) + len(lines[h].encode("utf-8"))   # where line h ends
    trimmed = 0
    for j in range(1, len(pieces) - 1):                  # the lines that end in a newline of the header
        end += 1 + len(lines[h + j].encode("utf-8"))
        p = pieces[j]
        if p.strip():                                    # (an all-whitespace line is never written)
            t = len(p[len(p.rstrip()):].encode("utf-8"))
            peak, trimmed = max(peak, end + t), trimmed + t
    return L, peak, trimmed


def trim_family():
    """[(document, compact length, L, peak)] with L < peak and the window L < n <= peak reachable from the compact length: for each
    whitespace code point and shape, the first line count and whitespace run (searched from small to large) that gives one."""
    shapes = [dict(depth=1, trimmed=1, blank=False, rows=1, after=False, other_key=False),
              dict(depth=1, trimmed=1, blank=False, rows=1, after=True, other_key=True),
              dict(depth=2, trimmed=3, blank=True, rows=1, after=True, other_key=False),
              dict(depth=3, trimmed=2, blank=False, rows=2, after=False, other_key=True),
              dict(depth=3, trimmed=1, blank=True, rows=3, after=True, other_key=False)]
    out = []
    for i, ws in enumerate(SPACES):
        for shape in shapes[i % 2::2] if i % 3 else shapes:
            found = None
            for reps in (4, 8, 16, 32, 64, 128, 256, 320):
                for lines in range(0, 200, 4):
                    d = trim_doc(ws, lines=lines, reps=reps, **shape)
                    C = len(d.encode("utf-8"))
                    L, peak, _ = trim_peak(d)
                    if max(C, L + 1) <= peak:
                        found = (d, C, L, peak)
                        break
                if found:
                    break
            assert found, (ascii(ws), shape)
            out.append(found)
    return out


def trim_sweep():
    """[(document, L, peak)]: each family member at every length from its compact form to L + (bytes trimmed) + 2."""
    out = []
    for d, C, L, peak in trim_family():
        c, gaps = compact(d)
        trimmed = trim_peak(d)[2]
        assert peak <= L + trimmed
        for n in range(C, L + trimmed + 3):
            out.append((pad(c, gaps, n - C, WHERE[n % 3]), L, peak))
    return out


DEEP = '{"a":[{"i":1,"b":[{"i":2,"c":[{"d":7,"e":[1,[2,[3]]]}]}]},{"i":3,"e":[{"i":4,"f":[4]}]}]}'


def error_docs():
    """Documents whose TOON output outgrows the input early (list items nested in list items) and that hold a quoted control
    character further on: in a value, in a key, in a table row, in a list."""
    out = []
    for tail in ('"z":"x\\u0001y"', '"q\\u001fk":1', '"t":[{"r":"ok"},{"r":"\\u0007"}]', '"m":0,"l":[[1],"\\u0000"]'):
        out.append(DEEP[:-1] + "," + tail + "}")
        out.append("[" + DEEP + ",{" + tail + "}]")
    return out


# ------------------------------------------------------------------------------------------------------------------ the routes
def seq_host(doc: str, stop: bool):
    return hs.toon_host(doc, stop_on_over=stop)


def run_host_routes(docs, exps, key_escape_only=False):
    """Every host route over docs against exps; returns {"tp_converted": units the token-parallel body converted itself, ...}."""
    stats = {"tp_converted": 0, "tp_not_smaller": 0, "handed": 0}
    for i, (d, e) in enumerate(zip(docs, exps)):
        for stop in (False, True):
            got = seq_host(d, stop)
            assert agrees(got, e, not stop), ("sequential", stop, d[:160], got[0], e[0])
        for report in (True, False):
            o = TP_ORDERS[(i + 2 * report) % len(TP_ORDERS)]
            got = hs.toon_tp(d, report_errors=report, order=o)
            if got[0] == HANDED_OVER:
                why = hs.toon_tp.last_reason
                assert why == FB_KEY_ESCAPE if key_escape_only else why in FB_REASONS, (d[:160], why)
                stats["handed"] += 1
                continue
            assert agrees(got, e, report), ("token-parallel", report, o, d[:160], got[0], e[0])
            if got[0] == TS_CONVERTED:
                stats["tp_converted"] += 1
            elif got[0] == TS_NOT_SMALLER:
                stats["tp_not_smaller"] += 1
    return stats


# ------------------------------------------------------------------------------------------------------------------- the tests
@pytest.fixture(scope="module")
def edge():
    corpus = edge_corpus()
    return corpus, [oracle(d) for d, _ in corpus]


def test_edge_corpus_reaches_every_edge_length(edge):
    corpus, exps = edge
    at = {e: [x[0] for (_, ee), x in zip(corpus, exps) if ee == e] for e in EDGE}
    assert all(len(v) >= 600 for v in at.values()), {e: len(v) for e, v in at.items()}
    # at n = L the text is not strictly smaller, at n = L + 1 it is
    assert set(at[-1]) == set(at[0]) == {TS_NOT_SMALLER} and set(at[1]) == set(at[2]) == {TS_CONVERTED}
    assert sum(len(compact(d)[0]) > toon_len(d) + 2 for d in base_docs()) >= 50      # documents too large to reach the edge exist
    assert sum(toon_len(d) > len(compact(d)[0]) for d in base_docs()) >= 40          # and ones whose TOON text outgrows the JSON


def test_edge_corpus_on_every_host_route(edge):
    corpus, exps = edge
    stats = run_host_routes([d for d, _ in corpus], exps)
    # units the token-parallel body decided itself at the edge, on both sides
    assert stats["tp_converted"] >= 1000 and stats["tp_not_smaller"] >= 600, stats


def test_trimmed_header_whitespace_across_the_capacity():
    """Regression: header whitespace written past the capacity and then stripped left the unit "not smaller" although the final
    text fits."""
    sweep = trim_sweep()
    docs = [d for d, _, _ in sweep]
    exps = [oracle(d) for d in docs]
    window = 0
    for (d, L, peak), e in zip(sweep, exps):
        n = len(d.encode("utf-8"))
        assert len(toon_ref.encode(json.loads(d)).encode("utf-8")) == L
        assert e[0] == (TS_CONVERTED if n > L else TS_NOT_SMALLER)
        window += L < n <= peak
    assert window >= 500, window
    run_host_routes(docs, exps, key_escape_only=True)


def test_trim_family_covers_every_whitespace_code_point():
    fam = trim_family()
    assert all(ch.isspace() for ch in SPACES[:2]) and set(SPACES[2:]) == {chr(c) for c in range(0x80, 0x110000) if chr(c).isspace()}
    assert all(L < peak and max(C, L + 1) <= peak for _, C, L, peak in fam)
    assert any('"n":7' in d for d, _, _, _ in fam) and any('"n":7' not in d for d, _, _, _ in fam)


def test_errors_after_the_output_outgrew_the_input():
    """A control character that must be quoted raises in the reference whatever the size: reported as a ValueError with errors
    reported, even though the output passed the capacity long before."""
    for d in error_docs():
        c, gaps = compact(d)
        for k in range(0, 48, 3):
            doc = pad(c, gaps, k, WHERE[k % 3])
            assert oracle(doc) == (TS_VALUE_ERROR, None), doc
            assert seq_host(doc, False) == (TS_VALUE_ERROR, None), doc
            assert seq_host(doc, True)[1] is None
            for o in TP_ORDERS:
                st, _ = hs.toon_tp(doc, report_errors=True, order=o)
                assert st == TS_VALUE_ERROR or (st == HANDED_OVER and hs.toon_tp.last_reason in FB_REASONS), (doc, st)
    assert toon_len(DEEP) > len(DEEP) + 20
