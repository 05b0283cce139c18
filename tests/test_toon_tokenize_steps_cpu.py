"""The token-parallel tokenizer (csrc/json_tp.h tokenize / tok_batch) at its lane and step edges, on the CPU warp emulator.

The tokenizer reads a unit in 1 KiB steps, 32 bytes per lane, on a 16-byte grid, and checks UTF-8 step by step (the three bytes in
front of a lane or a step carried in): where a byte lands depends on the unit's alignment.  Every case here is placed so that its interesting bytes straddle
a lane boundary or a step boundary at each of the 16 alignments, and run in both lane orders.  Each result is held to the
sequential encoder (json_toon.h: status and text), to the TOON oracle, and, when the unit is handed over, to a stable reason.

Cases: multi-byte UTF-8 in short and long strings; invalid sequences (truncated leads, stray continuations, overlongs, surrogates,
bytes F5 and up); non-ASCII bytes outside strings; a hand-over reason found before a later invalid string; units that end 1-15
bytes into a step; decimals at the edges of the number grammar and of the canonical form, also crossing a lane or step boundary;
strings of random lead / continuation / ASCII bytes against the sequential validator."""
import pytest

import hostsim_util as hs
from oracle import toon_ref

FALLBACK = 7
FB_NUM_EXACT = 1
STEP = 1024


def _place(feature: bytes, hot: int, target: int, lead: int) -> bytes:
    """{"p":"<pad>","x":<feature>} with feature[hot] at virtual offset `target` (unit offset + lead)."""
    head = b'{"p":"'
    mid = b'","x":'
    pad = target - lead - len(head) - len(mid) - hot
    assert pad >= 0
    return head + b"a" * pad + mid + feature + b"}"


def _check(text: bytes, lead: int, order: int):
    """One run of the warp kernel body against the sequential encoder and the oracle; returns (status, reason)."""
    o = (order & 1) | (lead << 4)
    st_seq, out_seq = hs.toon_host(text, unlimited=True)
    st, out = hs.toon_tp(text, unlimited=True, order=o)
    reason = hs.toon_tp.last_reason
    if st == FALLBACK:
        assert st_seq in (0, 1, 3, 4), (text[-80:], st_seq)
    else:
        assert (st, out) == (st_seq, out_seq), (text[-80:], lead, order)
    try:
        s = text.decode("utf-8")
    except UnicodeDecodeError:
        s = None
    if s is not None:
        exp = toon_ref.process_text(s, 0, 1 << 30)
        st2, got = hs.toon_tp(text, report_errors=False, order=o)
        if st2 != FALLBACK:
            assert (got if st2 == 0 else None) == exp, (text[-80:], lead, order)
    return st, reason


def _sweep(feature: bytes, hot: int):
    """feature[hot] on the 1 KiB step boundary and on a lane boundary inside a step, 1-3 bytes before each, all 16 alignments."""
    seen = set()
    for base in (STEP, STEP + 5 * 32, 2 * STEP + 31 * 32):
        for k in (1, 2, 3):
            for lead in range(16):
                text = _place(feature, hot, base - k + (hot == 0), lead)
                seen.add(_check(text, lead, lead & 1))
    return seen


LONG = 120          # longer than LONG_HI: the whole-warp string checks


def _string(content: bytes, at: int = 0):
    """A JSON string holding `content`; hot index = content's first byte (after `at` bytes of ASCII)."""
    return b'"' + b"x" * at + content + b"x" * 7 + b'"', 1 + at


VALID_UTF8 = [b"\xc3\xa9", b"\xe2\x82\xac", b"\xf0\x9d\x84\x9e", b"\xed\x9f\xbf", b"\xf4\x8f\xbf\xbf", b"\xe0\xa0\x80", b"\xf0\x90\x80\x80"]
INVALID_UTF8 = [
    b"\xc3",                    # truncated 2-byte lead
    b"\xe2\x82",                # truncated 3-byte lead
    b"\xf0\x9d\x84",            # truncated 4-byte lead
    b"\x80",                    # stray continuation
    b"\xbf\xbf",                # stray continuations
    b"\xc0\xaf",                # overlong (C0)
    b"\xc1\xbf",                # overlong (C1)
    b"\xe0\x80\xaf",            # overlong 3-byte
    b"\xf0\x80\x80\xaf",        # overlong 4-byte
    b"\xed\xa0\x80",            # surrogate D800
    b"\xed\xbf\xbf",            # surrogate DFFF
    b"\xf4\x90\x80\x80",        # above U+10FFFF
    b"\xf5\x80\x80\x80",        # F5 lead
    b"\xff",                    # FF
]


@pytest.mark.parametrize("seq", VALID_UTF8, ids=lambda b: b.hex())
@pytest.mark.parametrize("at", [0, LONG])
def test_valid_multibyte_across_boundaries(seq, at):
    # hot = the sequence's second byte, so that the sequence itself is split
    f, h = _string(seq * 3, at)
    sts = {st for st, _ in _sweep(f, h + 1)}
    assert sts <= {0, 1, FALLBACK}, sts


@pytest.mark.parametrize("seq", INVALID_UTF8, ids=lambda b: b.hex())
@pytest.mark.parametrize("at", [0, LONG])
def test_invalid_utf8_across_boundaries(seq, at):
    f, h = _string(b"\xc3\xa9" + seq, at)
    assert {st for st, _ in _sweep(f, h + 2)} == {2}


@pytest.mark.parametrize("seq", [b"\xc3\xa9", b"\x80", b"\xe2\x82\xac"], ids=lambda b: b.hex())
def test_non_ascii_outside_strings(seq):
    for f, h in ((b"[1," + seq + b"]", 3), (b"1" + seq, 1), (seq + b"1", 0), (b'["a"' + seq + b"]", 4)):
        assert {st for st, _ in _sweep(f, h)} == {2}


def test_first_handover_reason_comes_before_a_later_bad_string():
    # a decimal the exact formatter must print, then (over 32 tokens later: another token batch, and for the longer gaps another
    # 1 KiB step) a string with invalid UTF-8: the first attempt stops at the decimal, as the tokenizer reaches it first
    num = b"1.234567890123456"                        # 16 significant digits
    for lead in range(16):
        for order in (0, 1):
            for gap in (40, 300, 600):
                fill = b",".join(b"%d" % i for i in range(gap))
                for bad in (b"x\xed\xa0\x80y", b"x" * 100 + b"\xed\xa0\x80y"):
                    text = b'{"n":' + num + b',"p":[' + fill + b'],"s":"' + bad + b'"}'
                    st, out = hs.toon_tp(text, unlimited=True, order=(order & 1) | (lead << 4))
                    assert st == FALLBACK and hs.toon_tp.last_reason == FB_NUM_EXACT, (lead, order, gap, st)
                    assert hs.toon_host(text, unlimited=True)[0] == 2


@pytest.mark.parametrize("k", range(1, 16))
def test_units_ending_inside_a_step(k):
    for lead in range(16):
        n = 2 * STEP + k - lead
        for tail in (b"1.25]", b"7]", b'"\xc3\xa9"]', b"true]", b'"ab"]'):
            body = b'["' + b"b" * (n - 5 - len(tail) - 2) + b'", ' + tail
            text = body + b" " * (n - len(body))
            assert len(text) == n
            st, _ = _check(text, lead, k & 1)
            assert st in (0, 1), (k, lead, tail, st)


DECIMALS = [
    b"-0.0", b"0.0", b"0.50", b"10.000", b"-10.000", b"100.25", b"87.25", b"-0.5", b"0.05", b"0.000125",
    b"123456789.012345",                    # 15 significant digits
    b"1234567890.123456",                   # 16: exact formatter
    b"0.0000123456789012345678",            # tiny and long: exact formatter
    b"0.0001234567890123",                  # 15 significant digits after 3 zeros
    b"-1234567.00000000000000",             # 7 significant digits once the zeros go
    b"01.5", b"00.5", b"-01.5", b"1.", b".5", b"-.5", b"1.5e3", b"1.5E-3", b"1e5", b"1.5.5", b"1.5-3", b"--1.5", b"1-5", b"1.x5",
]


@pytest.mark.parametrize("num", DECIMALS, ids=lambda b: b.decode())
def test_decimals_across_boundaries(num):
    for f, h in ((b"[" + num + b",1]", 1), (b"[" + num + b",1]", 1 + len(num) // 2), (b"[" + num + b",1]", len(num))):
        for st, reason in _sweep(f, h):
            if st == FALLBACK:
                assert reason == FB_NUM_EXACT, (num, reason)


@pytest.mark.parametrize("num", DECIMALS, ids=lambda b: b.decode())
def test_decimals_as_table_values(num):
    rows = b",".join(b'{"id":%d,"score":%s}' % (i, num) for i in range(40))
    text = b'{"rows":[' + rows + b"]}"
    for lead in range(16):
        st, reason = _check(text, lead, lead & 1)
        if st == FALLBACK:
            assert reason == FB_NUM_EXACT, (num, reason)


def test_random_bytes_in_strings_match_the_sequential_validator():
    # strings of random bytes drawn from the lead / continuation / ASCII classes, short and long, at random alignments: the
    # step-wise check must fail exactly the units the sequential encoder's string validator fails
    import random
    rng = random.Random(20261018)
    pool = [0x20, 0x41, 0x7E, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xED, 0xEF, 0xF0, 0xF3, 0xF4, 0xF5, 0xFF]
    valid = [b"\xc3\xa9", b"\xe2\x82\xac", b"\xf0\x9d\x84\x9e", b"\xed\x9f\xbf", b"abc"]
    n_bad = 0
    for it in range(1500):
        parts = []
        for _ in range(rng.randrange(1, 60)):
            parts.append(rng.choice(valid) if rng.random() < 0.9 else bytes([rng.choice(pool)]))
        body = b"".join(parts)
        pad = rng.randrange(0, 1100)
        text = b'{"p":"' + b"a" * pad + b'","s":"' + body + b'","t":[1,2]}'
        lead = rng.randrange(16)
        st_seq, out_seq = hs.toon_host(text, unlimited=True)
        st, out = hs.toon_tp(text, unlimited=True, order=(it & 1) | (lead << 4))
        if st != FALLBACK:
            assert (st, out) == (st_seq, out_seq), (body, pad, lead)
        n_bad += st_seq == 2
    assert n_bad > 100
