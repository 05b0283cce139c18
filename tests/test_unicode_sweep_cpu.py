"""Every code point and every short UTF-8 sequence against CPython: the corpus builders of the Unicode sweeps, and a reduced
sweep on the host build of the kernels' headers (tests/hostsim).

The kernels work on UTF-8 bytes and must reproduce decisions CPython makes on `str` code points: the scan and substitution
kernels' byte classes, lead-byte prefilters and look-behind (re_backend.cpp, scan_core.h), the TOON encoder's Unicode `\\d` and
`str.isspace()` tables and its strict UTF-8 check (json_toon.h, json_tp.h), and the masking kernel's re-escaping and key handling
(json_mask.h, masking.py).  Every expected value here comes from CPython itself (`re`, `str`, `bytes.decode`) or from the oracles
pinned to the reference (oracle/toon_ref.py, oracle/mask_ref.py), never from regex_frontend's interval sets or another kernel.

The full sweeps (every one of the 0x110000 code points, every 1-3 byte sequence) run on the GPU in test_unicode_sweep_gpu.py,
which imports its corpora from here.  The reduced sweep here covers all of plane 0, every range boundary of the tables the sweeps
exercise, and every 97th code point above U+FFFF; the token-parallel kernel body, which runs on a slow warp emulator here, sees a
smaller subset still."""
import os
import random
import re
import unicodedata

import numpy as np
import pytest

from mcp_context_forge_b200 import masking
from oracle import mask_ref, toon_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_CP = 0x110000
SURROGATES = range(0xD800, 0xE000)
N_SCALARS = N_CP - len(SURROGATES)


# ---------------------------------------------------------------------------------------------------------------------
# code points
# ---------------------------------------------------------------------------------------------------------------------
_ALL = None


def all_chars() -> str:
    """Every code point, surrogates included, as one str: index == code point."""
    global _ALL
    if _ALL is None:
        _ALL = "".join(map(chr, range(N_CP)))
    return _ALL


def char_ranges(pattern: str):
    """Inclusive ranges of the code points one `re` pattern matches as a single character (finditer over every code point)."""
    out = []
    for m in re.finditer(pattern + "+", all_chars()):
        out.append((m.start(), m.end() - 1))
    return out


def digit_ranges():
    return char_ranges(r"\d")


def space_ranges():
    out = []
    for c in range(N_CP):
        if chr(c).isspace():
            if out and out[-1][1] == c - 1:
                out[-1] = (out[-1][0], c)
            else:
                out.append((c, c))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# §1 scan: one-character patterns and context patterns over every code point, three templates each
# ---------------------------------------------------------------------------------------------------------------------
CASED_RANGES = [("a", "z"), ("À", "ɏ"), ("Ͱ", "Ͽ"), ("Ѐ", "ԯ"), ("Ḁ", "῿"), ("Ⰰ", "ⳳ"), ("Ꙁ", "ꟿ"), ("Ａ", "ｚ"),
                ("\U00010400", "\U0001044F"), ("\U0001E900", "\U0001E943")]
ONE_CHAR = ([r"\w", r"\W", r"\d", r"\D", r"\s", r"\S", r".", r"(?s).", r"[^a]", r"(?a)\w", r"(?a)\s"]
            + ["(?i)" + c for c in "ksißσµωθ"]
            + [f"(?i)[{lo}-{hi}]" for lo, hi in CASED_RANGES] + [f"(?i)[^{lo}-{hi}]" for lo, hi in CASED_RANGES])
# patterns whose answer depends on the neighbour: checked with a `search` per unit
CONTEXT = [r"\Ba", r"(?m)^a", r"a\b", r"a$", r"(?m)a$"]
SCAN_PATTERNS = ONE_CHAR + CONTEXT
TEMPLATES = ("c", "c+a", "a+c")                     # unit 3 * i + t holds code point i in template t


def scan_units(cps):
    """Three units per code point, then one empty unit (on which even `(?s).` misses)."""
    out = []
    for c in cps:
        ch = chr(c)
        out += [ch, ch + "a", "a" + ch]
    return out + [""]


_TABLES = {}


def one_char_table(pattern: str) -> np.ndarray:
    """bool[0x110000]: does `pattern` match the one-character string chr(c)?  One finditer of `pattern+` over every code point
    (each pattern is one atom; test_one_char_shortcut_equals_search holds this to a `search` per character)."""
    t = _TABLES.get(pattern)
    if t is None:
        t = np.zeros(N_CP, dtype=bool)
        for m in re.finditer(pattern + "+", all_chars()):
            t[m.start():m.end()] = True
        _TABLES[pattern] = t
    return t


def scan_expected(cps) -> np.ndarray:
    """uint64 bitmaps (bit i = SCAN_PATTERNS[i]) of the units scan_units(cps) builds."""
    cps = np.asarray(cps, dtype=np.int64)
    n = len(cps)
    exp = np.zeros(3 * n + 1, dtype=np.uint64)
    a = ord("a")
    for i, p in enumerate(ONE_CHAR):
        t = one_char_table(p)
        m = t[cps]
        bit = np.uint64(1 << i)
        exp[0:3 * n:3] |= np.where(m, bit, np.uint64(0))
        ma = m | t[a]
        exp[1:3 * n:3] |= np.where(ma, bit, np.uint64(0))
        exp[2:3 * n:3] |= np.where(ma, bit, np.uint64(0))
    units = scan_units(cps.tolist())
    for j, p in enumerate(CONTEXT):
        s = re.compile(p).search
        bit = 1 << (len(ONE_CHAR) + j)
        exp |= np.fromiter((bit if s(u) else 0 for u in units), dtype=np.uint64, count=len(units))
    return exp


def first_scan_mismatch(cps, got: np.ndarray, exp: np.ndarray):
    """(pattern, code point, template, got, expected) of the first differing bit, or None."""
    diff = np.nonzero(got != exp)[0]
    if not len(diff):
        return None
    k = int(diff[0])
    x = int(got[k]) ^ int(exp[k])
    i = (x & -x).bit_length() - 1
    cp, template = (hex(cps[k // 3]), TEMPLATES[k % 3]) if k < 3 * len(cps) else (None, "empty")
    return SCAN_PATTERNS[i], cp, template, bool(int(got[k]) >> i & 1), bool(int(exp[k]) >> i & 1)


def bits_seen(exp: np.ndarray):
    """(OR of the bitmaps, OR of their complements): which patterns matched somewhere and which missed somewhere."""
    full = np.uint64((1 << len(SCAN_PATTERNS)) - 1)
    return int(np.bitwise_or.reduce(exp)), int(np.bitwise_or.reduce(~exp & full))


# ---------------------------------------------------------------------------------------------------------------------
# the reduced code point set
# ---------------------------------------------------------------------------------------------------------------------
def edge_code_points():
    """The UTF-8 length and surrogate edges, every plane's ends, the \\d and isspace ranges' lo-1 / lo / hi / hi+1, and every
    code point where one of the one-character patterns changes its answer (and the one before it)."""
    pts = {0, 0x7F, 0x80, 0x7FF, 0x800, 0xFFFF, 0x10000, 0x10FFFF, 0xD7FF, 0xD800, 0xDBFF, 0xDC00, 0xDFFF, 0xE000}
    for p in range(17):
        pts |= {p << 16, (p << 16) + 1, (p << 16) | 0xFFFF, ((p << 16) | 0xFFFF) - 1}
    for lo, hi in digit_ranges() + space_ranges():
        pts |= {lo - 1, lo, hi, hi + 1}
    for p in ONE_CHAR:
        t = one_char_table(p)
        ch = np.nonzero(t[1:] != t[:-1])[0] + 1
        pts |= set(ch.tolist()) | set((ch - 1).tolist())
    return {c for c in pts if 0 <= c < N_CP}


def reduced_code_points():
    return sorted(set(range(0x10000)) | set(range(0x10000, N_CP, 97)) | edge_code_points())


def is_scalar(c):
    return not 0xD800 <= c < 0xE000


# ---------------------------------------------------------------------------------------------------------------------
# §2 substitution: runs of 64 consecutive code points, an ASCII separator every 16
# ---------------------------------------------------------------------------------------------------------------------
SUB_RULES = [(r"(\w+)", r"[\1]"), (r"\s+", "_"), (r"(?i)(k|s)", r"<\1>"), (r"[^\x00-\x7f]", ""), (r"(\d)(\D)", r"\2\1"), (r"\b", "|")]
SEPARATORS = " ,\n-"


def sub_units(first_cps):
    """One unit per start code point: 64 consecutive code points (surrogates included), a separator after every 16."""
    out = []
    for k, c0 in enumerate(first_cps):
        parts = []
        for q in range(4):
            parts.append("".join(map(chr, range(c0 + 16 * q, min(c0 + 16 * q + 16, N_CP)))))
            parts.append(SEPARATORS[(k + q) % 4])
        out.append("".join(parts))
    return out


def sub_expected(rules, text):
    """re.subn of each rule in order: (text, total count)."""
    n = 0
    for p, r in rules:
        text, k = re.subn(p, r, text)
        n += k
    return text, n


# ---------------------------------------------------------------------------------------------------------------------
# §3 TOON: every scalar in every quoting-relevant position, raw and escaped, as values, keys and table headers
# ---------------------------------------------------------------------------------------------------------------------
VALUE_TEMPLATES = ["{}", "x{}", "{}x", "x{}x", "1{}", "0{}", "1.{}", "1e{}", "1e+{}", "0.{}"]
KEY_TEMPLATES = ["{}", "a{}", "{}a"]
TOON_SHAPES = ["values", "object", "table"]          # array of 64 strings, object of 64 keys, two rows of such an object


def escape_cp(c: int) -> str:
    """JSON escape of one code point: \\uXXXX, or a surrogate pair for an astral one."""
    if c < 0x10000:
        return "\\u%04x" % c
    c -= 0x10000
    return "\\u%04x\\u%04x" % (0xD800 + (c >> 10), 0xDC00 + (c & 0x3FF))


def raw_cp(c: int) -> str:
    """The code point as it stands in a JSON string written without \\u escapes (only '"' and '\\\\' must be escaped)."""
    return {0x22: '\\"', 0x5C: "\\\\"}.get(c, chr(c))


def json_str(template: str, c: int, escaped: bool) -> str:
    pre, post = template.split("{}")
    return '"' + pre + (escape_cp(c) if escaped else raw_cp(c)) + post + '"'


def toon_doc(shape: str, template: str, cps, escaped: bool) -> str:
    strs = [json_str(template, c, escaped) for c in cps]
    if shape == "values":
        return "[" + ",".join(strs) + "]"
    row = lambda v: "{" + ",".join(f"{s}:{v + i}" for i, s in enumerate(strs)) + "}"      # noqa: E731
    return row(0) if shape == "object" else "[" + row(0) + "," + row(100) + "]"


def toon_groups(cps):
    """Code points of one sweep in documents: 64 per group, and each code point below 0x20 alone."""
    ctl = [c for c in cps if c < 0x20]
    rest = [c for c in cps if c >= 0x20 and is_scalar(c)]
    return [[c] for c in ctl] + [rest[i:i + 64] for i in range(0, len(rest), 64)]


def toon_expected(doc: str):
    """(status, text) of include/cfgpu.h for an unlimited output: 0 = toon_ref's text, 2 = not JSON, 3 / 4 = the reference raises
    ValueError / AttributeError (CF_TOON_REPORT_ERRORS)."""
    try:
        obj = toon_ref.loads_strict(doc)
    except ValueError:
        return 2, None
    try:
        return 0, toon_ref.encode(obj)
    except ValueError:
        return 3, None
    except toon_ref.ToonCrash:
        return 4, None


def toon_corpus(groups):
    """[(doc bytes, expected (status, text or None), escaped, shape, template, group)].  A converted document is padded with
    trailing spaces until its TOON form is strictly smaller, so that its text is really compared.  The raw and the escaped
    document of one group parse to the same value: toon_ref runs once for both (the parse of each is compared)."""
    out = []
    for g in groups:
        for shape in TOON_SHAPES:
            for template in (VALUE_TEMPLATES if shape == "values" else KEY_TEMPLATES):
                raw = toon_doc(shape, template, g, False)
                esc = toon_doc(shape, template, g, True)
                st, text = toon_expected(raw)
                if st == 2:                                   # a raw control character: the escaped form has its own answer
                    est = toon_expected(esc)
                else:
                    assert toon_ref.loads_strict(esc) == toon_ref.loads_strict(raw)
                    est = (st, text)
                for doc, (s, t), e in ((raw, (st, text), False), (esc, est, True)):
                    b = doc.encode("utf-8")
                    if s == 0:
                        b += b" " * max(0, len(t.encode("utf-8")) - len(b) + 1)
                    out.append((b, (s, t), e, shape, template, g))
    return out


FB_KEY_ESCAPE, FB_DUP_HASH = 2, 5                  # csrc/json_tp.h


def handover_reasons(doc: bytes):
    """The reasons for which the token-parallel kernel may hand one of these documents to the sequential encoder: a key that holds
    an escape, and a collision in the duplicate-key screen.  A document without a backslash never reports FB_KEY_ESCAPE."""
    return {FB_KEY_ESCAPE, FB_DUP_HASH} if b"\\" in doc else {FB_DUP_HASH}


def toon_edge_hits(corpus):
    """{(table, lo, hi, which)} of the \\d / isspace range edges (lo-1, lo, hi, hi+1) the corpus places in a document."""
    cps = set()
    for _, _, _, _, _, g in corpus:
        cps.update(g)
    hits = set()
    for name, ranges in (("digit", digit_ranges()), ("space", space_ranges())):
        for lo, hi in ranges:
            for which, c in (("lo-1", lo - 1), ("lo", lo), ("hi", hi), ("hi+1", hi + 1)):
                if c in cps:
                    hits.add((name, lo, hi, which))
    return hits


def assert_control_answers(corpus):
    """A raw control character is not JSON; escaped, it raises ValueError unless it is \\n, \\r or \\t, which are quoted.  (In a
    table the reference writes the header's keys without that check: toon_ref has the answer there.)"""
    seen = 0
    for b, (s, _), escaped, shape, _, g in corpus:
        if len(g) == 1 and g[0] < 0x20 and (shape != "table" or not escaped):
            seen += 1
            if not escaped:
                assert s == 2, (b, s)
            else:
                assert s == (0 if chr(g[0]) in "\n\r\t" else 3), (b, s)
    assert seen == 32 * (2 * len(VALUE_TEMPLATES) + 3 * len(KEY_TEMPLATES))


# ---------------------------------------------------------------------------------------------------------------------
# §4 strict UTF-8: short byte sequences in a string, at every offset from the 32-byte lane window and across a 1 KiB step
# ---------------------------------------------------------------------------------------------------------------------
TAIL_BYTES = [b for b in range(0x20, 0x100) if b not in (0x22, 0x5C)]
BOUNDARY_SECOND = (0x80, 0x9F, 0xA0, 0xBF)
FOUR_TAIL = (0x7F, 0x80, 0xBF, 0xC0)
LANE = 32
# unit positions of the sequence's first byte: 0..35 bytes into a 32-byte-aligned lane window, and the 8 positions around the
# first 1 KiB step boundary (units are laid out so that they start on a 32-byte boundary)
OFFSETS = [2 * LANE + o for o in range(36)] + [1024 - 4 + k for k in range(8)]
HEAD = b'{"s":"'
TAIL = b'"}'


def utf8_sequences():
    """[(seq, offset index or None)]: None = at every offset (the 1- and 2-byte sets and the boundary second bytes); the other 3- and
    4-byte sequences take offset i mod len(OFFSETS) from their index i in this list, so that each offset is still reached."""
    out = [(bytes([a]), None) for a in range(0x80, 0x100)]
    out += [(bytes([a, b]), None) for a in range(0x80, 0x100) for b in TAIL_BYTES]
    seqs = [bytes([a, b, c]) for a in range(0xE0, 0xF0) for b in TAIL_BYTES for c in TAIL_BYTES]
    seqs += [bytes([a, b, c, d]) for a in range(0xF0, 0xF8) for b in TAIL_BYTES for c in FOUR_TAIL for d in FOUR_TAIL]
    out += [(q, None if q[1] in BOUNDARY_SECOND else i % len(OFFSETS)) for i, q in enumerate(seqs)]
    return out


def closing_quote_sequences():
    """Every lead byte directly followed by the closing quote, at every offset."""
    return [(bytes([a]), None) for a in range(0x80, 0x100)]


def utf8_body(seq: bytes, pos: int, quote_after: bool = False) -> bytes:
    """{"s":"<pad><seq><pad>"} with seq at unit position `pos`, padded with trailing spaces so that unit + terminator is a
    multiple of 64 bytes (every unit of a packed batch then starts on a lane window)."""
    pre = b"a" * (pos - len(HEAD))
    body = HEAD + pre + seq + (b"" if quote_after else b"b" * 7) + TAIL
    return body + b" " * (-(len(body) + 1) % 64)


def utf8_units(seqs, quote_after=False, reduce=1):
    """[(body, seq, offset index)] of utf8_sequences() or closing_quote_sequences() entries; `reduce` keeps every reduce-th unit."""
    out = []
    k = 0
    for seq, at in seqs:
        for j in (range(len(OFFSETS)) if at is None else (at,)):
            if k % reduce == 0:
                out.append((utf8_body(seq, OFFSETS[j], quote_after), seq, j))
            k += 1
    return out


def utf8_valid(seq: bytes) -> bool:
    try:
        seq.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def utf8_offset_coverage(units):
    """{offset index: (valid bodies, invalid bodies)}."""
    cov = {j: [0, 0] for j in range(len(OFFSETS))}
    for body, seq, j in units:
        cov[j][0 if utf8_valid(seq) else 1] += 1
    return cov


def utf8_toon_expected(body: bytes):
    """(status, text): not JSON when the body is not UTF-8, else toon_ref's answer (the body's TOON form is always smaller)."""
    try:
        s = body.decode("utf-8")
    except UnicodeDecodeError:
        return 2, None
    return toon_expected(s)


def utf8_mask_expected(body: bytes):
    """The masked body from mask_ref, or None where serde_json rejects it."""
    try:
        return mask_ref.mask_json_bytes(body, 10)
    except ValueError:
        return None


# ---------------------------------------------------------------------------------------------------------------------
# §5 masking
# ---------------------------------------------------------------------------------------------------------------------
def mask_escape_docs(cps):
    """Every scalar in a string value, raw and escaped, 64 per document ({"k":["<c0>", ...]}), and every lone surrogate escaped
    alone ({"k":"\\udXXX"})."""
    scal = [c for c in cps if is_scalar(c)]
    docs = []
    for i in range(0, len(scal), 64):
        g = scal[i:i + 64]
        for escaped in (False, True):
            if not escaped and g[0] < 0x20:                        # raw controls: one per document (serde rejects them)
                docs += ['{"k":["' + raw_cp(c) + '"]}' for c in g if c < 0x20]
                g = [c for c in g if c >= 0x20]
            docs.append('{"k":[' + ",".join(json_str("{}", c, escaped) for c in g) + "]}")
    docs += ['{"k":"' + escape_cp(c) + '"}' for c in cps if not is_scalar(c)]
    return [d.encode("utf-8") for d in docs]


def mask_key_order_docs(cps, seed=7):
    """Objects of 64 keys in shuffled order: every group of 64 consecutive scalars, and groups drawn from U+E000..U+FFFF and
    above U+FFFF together (where UTF-16 order and code point order disagree) and from the whole range."""
    rng = random.Random(seed)
    scal = [c for c in cps if is_scalar(c) and c >= 0x20]
    groups = [scal[i:i + 64] for i in range(0, len(scal), 64)]
    hi = [c for c in scal if c >= 0xE000]
    for _ in range(max(64, len(scal) // 4096)):
        groups.append(rng.sample(hi, 64))
        groups.append(rng.sample(scal, 64))
    docs = []
    for g in groups:
        g = list(g)
        rng.shuffle(g)
        esc = rng.random() < 0.5
        docs.append(("{" + ",".join(f'{json_str("{}", c, esc)}:{i}' for i, c in enumerate(g)) + "}").encode("utf-8"))
    return docs


def mask_expected(doc: bytes):
    try:
        return mask_ref.mask_json_bytes(doc, 10)
    except ValueError:
        return None


KEY_CLASS_TEMPLATES = ["{}", "pass{}word", "API{}Key"]


def key_class_keys(cps):
    return [t.format(chr(c)) for c in cps if is_scalar(c) for t in KEY_CLASS_TEMPLATES]


def cased_code_points():
    """Code points that some case mapping changes (str.lower or str.upper), about 2.8 k."""
    return [c for c in range(N_CP) if is_scalar(c) and (chr(c).lower() != chr(c) or chr(c).upper() != chr(c))]


def probe_texts():
    """The non-JSON fallback's probes: for each sensitive key and each position j holding a letter, key[:j] + c + key[j+1:] for
    every cased code point c and every ASCII code point."""
    subs = sorted(set(cased_code_points()) | set(range(0x80)))
    out = []
    for k in masking.SENSITIVE_KEYS:
        for j, ch in enumerate(k):
            if ch.isalpha():
                out += [k[:j] + chr(c) + k[j + 1:] for c in subs]
    return out


def probe_expected(s: str) -> bool:
    low = s.lower()
    return any(k in low for k in masking.SENSITIVE_KEYS)


# =====================================================================================================================
# tests on the host build
# =====================================================================================================================
@pytest.fixture(scope="module")
def reduced():
    return reduced_code_points()


def test_one_char_shortcut_equals_search():
    """The finditer shortcut of one_char_table against a `search` on every sampled one-character string, for every pattern."""
    rng = random.Random(1)
    sample = sorted(set(rng.sample(range(N_CP), 20000)) | edge_code_points())
    for p in ONE_CHAR:
        t = one_char_table(p)
        s = re.compile(p).search
        bad = [hex(c) for c in sample if bool(s(chr(c))) != bool(t[c])]
        assert not bad, (p, bad[:8])


def test_scan_sweep_on_the_host_build(reduced, monkeypatch):
    import hostsim_util as hs

    exp = scan_expected(reduced)
    matched, missed = bits_seen(exp)
    full = (1 << len(SCAN_PATTERNS)) - 1
    assert matched == full and missed == full, [p for i, p in enumerate(SCAN_PATTERNS) if not (matched & missed) >> i & 1]
    for pair in ("0", "1"):
        monkeypatch.setenv("CF_PAIR_FILTER", pair)
        prog = hs.HostProgram()
        for p in SCAN_PATTERNS:
            prog.add(p)
        got, _ = prog.scan(scan_units(reduced))
        assert first_scan_mismatch(reduced, np.array(got, dtype=np.uint64), exp) is None, (pair, first_scan_mismatch(reduced, np.array(got, dtype=np.uint64), exp))


def test_substitution_sweep_on_the_host_build(reduced):
    import hostsim_util as hs
    from mcp_context_forge_b200 import regex_frontend as fe

    starts = sorted({c - c % 64 for c in reduced})
    units = sub_units(starts)
    prog = hs.HostProgram()
    for p, r in SUB_RULES:
        prog.add(p, 0, ordered=True, repl=fe.template_parts(r, re.compile(p)))
    matched = [0] * len(SUB_RULES)
    for u in units:
        text = u
        for k, rule in enumerate(SUB_RULES):
            got = prog.sub(k, u)
            assert got == sub_expected([rule], u), (rule, u)
            matched[k] += got[1] > 0
            t2 = prog.sub(k, text)
            assert t2 == sub_expected([rule], text), (rule, text)
            text = t2[0]
        assert text == sub_expected(SUB_RULES, u)[0], u
    assert all(m > 0 for m in matched), matched


def test_toon_sweep_on_the_host_build(reduced):
    """The sequential encoder on every document of the reduced sweep; the token-parallel body (warp emulator) on the groups that
    hold a \\d or isspace range edge, raw and escaped."""
    import hostsim_util as hs

    corpus = toon_corpus(toon_groups(reduced))
    assert_control_answers(corpus)
    hits = toon_edge_hits(corpus)
    plane0 = [(n, lo, hi, w) for n, ranges in (("digit", digit_ranges()), ("space", space_ranges())) for lo, hi in ranges
              for w in ("lo-1", "lo", "hi", "hi+1")]
    assert set(plane0) <= hits, sorted(set(plane0) - hits)[:4]
    edges = {c for lo, hi in digit_ranges() + space_ranges() for c in (lo - 1, lo, hi, hi + 1)}
    n_tp = 0
    for b, exp, escaped, shape, template, g in corpus:
        st, text = hs.toon_host(b)
        assert (st, text) == exp, (b[:120], st, exp[0])
        if edges.intersection(g) and (shape == "values" or not escaped):
            st, text = hs.toon_tp(b)
            if st == 7:
                assert hs.toon_tp.last_reason in handover_reasons(b), (b[:120], hs.toon_tp.last_reason)
            else:
                assert (st, text) == exp, (b[:120], st, exp[0])
            n_tp += 1
    assert n_tp > 500


TP_LEADS = (0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xED, 0xEF, 0xF0, 0xF4, 0xF5)


def test_strict_utf8_sweep_on_the_host_build():
    """Every 1-byte sequence and every lead byte before the closing quote at every offset; the 2- to 4-byte sets thinned out.
    The sequential encoder and the masking parser on all of them, the token-parallel body on the boundary second bytes."""
    import hostsim_util as hs

    seqs = utf8_sequences()
    units = (utf8_units([s for s in seqs if len(s[0]) == 1]) + utf8_units(closing_quote_sequences(), quote_after=True)
             + utf8_units([s for s in seqs if len(s[0]) > 1], reduce=37))
    cov = utf8_offset_coverage(units)
    assert all(v > 0 and iv > 0 for v, iv in cov.values()), cov
    n_tp = 0
    for i, (body, seq, j) in enumerate(units):
        exp = utf8_toon_expected(body)
        assert hs.toon_host(body) == exp, (seq.hex(), OFFSETS[j])
        m = utf8_mask_expected(body)
        st, out = hs.mask_host(body)
        assert (st, out) == ((0, m) if m is not None else (2, None)), (seq.hex(), OFFSETS[j], st)
        if len(seq) > 1 and seq[1] in BOUNDARY_SECOND + (0x7F, 0xC0) and seq[0] in TP_LEADS:
            st, text = hs.toon_tp(body)
            assert st != 7 and (st, text) == exp, (seq.hex(), OFFSETS[j], st)
            n_tp += 1
    assert n_tp > 200


def test_masking_sweep_on_the_host_build(reduced):
    import hostsim_util as hs

    docs = mask_escape_docs(reduced) + mask_key_order_docs(reduced)
    n_ok = 0
    for d in docs:
        m = mask_expected(d)
        st, out = hs.mask_host(d)
        assert (st, out) == ((0, m) if m is not None else (2, None)), (d[:120], st)
        n_ok += m is not None
    assert n_ok > len(docs) // 2
    keys = key_class_keys(reduced)
    bad = [k for k in keys if hs.key_sensitive_host(k) != mask_ref.is_sensitive_key(k)]
    assert not bad, [ascii(k) for k in bad[:8]]
    assert 0 < sum(mask_ref.is_sensitive_key(k) for k in keys) < len(keys)


def test_fallback_probes_on_the_host_build():
    """masking._probe_pattern's 13 probes, compiled like non_json_fallback_batch compiles them, on every probe text."""
    import hostsim_util as hs

    texts = probe_texts()
    assert len(texts) > 13 * 2000
    prog = hs.HostProgram()
    for k in masking.SENSITIVE_KEYS:
        prog.add(masking._probe_pattern(k))
    got, _ = prog.scan(texts)
    bad = [ascii(t) for t, g in zip(texts, got) if bool(g) != probe_expected(t)]
    assert not bad, bad[:8]
    assert 0 < sum(1 for g in got if g) < len(texts)


# ---------------------------------------------------------------------------------------------------------------------
# §6 the generated tables
# ---------------------------------------------------------------------------------------------------------------------
def header_ranges():
    with open(os.path.join(ROOT, "mcp_context_forge_b200", "csrc", "unicode_tables.h"), encoding="utf-8") as f:
        src = f.read()
    vals = {}
    for name in ("ND_LO", "ND_HI", "WS_LO", "WS_HI"):
        vals[name] = [int(x, 16) for x in re.search(r"#define CFU_%s (.*)" % name, src).group(1).split(",")]
    version = re.search(r"\(Unicode ([0-9.]+)\)", src).group(1)
    return version, list(zip(vals["ND_LO"], vals["ND_HI"])), list(zip(vals["WS_LO"], vals["WS_HI"]))


def test_unicode_tables_match_this_interpreter():
    """csrc/unicode_tables.h holds the \\d and str.isspace() ranges of the interpreter the gateway runs on."""
    version, nd, ws = header_ranges()
    if version != unicodedata.unidata_version:
        pytest.skip(f"unicode_tables.h is generated from Unicode {version}; this interpreter has {unicodedata.unidata_version}")
    assert nd == digit_ranges()
    assert ws == space_ranges()
