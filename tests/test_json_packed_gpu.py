"""The JSON kernels at batch sizes where one warp walks several units (units_per_warp in cfjson.cu: 1, 4 and 32 units per
warp for about 200, 6 000 and 40 000 units on an H100), with hostile neighbours in every warp: empty, 1-byte, invalid and
64 KiB units, nesting 63 / 64 / 65, hard numbers, escapes and surrogate pairs.  cf_mask_host (max_depth 10 and 3),
cf_toon_host on the default path (token-parallel kernel + sequential hand-over) and with CF_TOON_SEQUENTIAL are compared
with the oracles (oracle/mask_ref.py, oracle/toon_ref.py), never with another GPU path.  A unit beyond the documented
device limits (a number whose exact conversion needs more than 3200 bits; for the TOON encoders also nesting > 64) must report
UNSUPPORTED (6) instead; masking parses serde_json's 127 levels, so it holds the nested units to the oracle.

A second corpus reaches every reason (json_tp.h FB_*) for which the token-parallel kernel hands a unit to the sequential
encoder: with CF_TOON_NO_HANDOVER the reason is reported, on the default path the unit gets the oracle's answer."""
import ctypes
import random
import struct

import numpy as np
import pytest

from mcp_context_forge_b200 import engine
from oracle import mask_ref, toon_ref

TOON_REPORT_ERRORS, TOON_SEQUENTIAL, TOON_NO_HANDOVER = 1, 8, 16
TS_FALLBACK = 7
PAD = " " * 48            # trailing whitespace: the TOON form of a small document is then smaller, so it is really compared

DEPTH_LIMIT = 64
BIG_BITS = 3200


def nested(kind, d):
    """A document nested d levels deep: arrays, objects or both alternating."""
    if kind == "arr":
        return "[" * d + "1" + "]" * d
    if kind == "obj":
        return '{"a": ' * d + "1" + "}" * d
    head = "".join('[' if i % 2 else '{"k": ' for i in range(d))
    return head + "1" + "".join(']' if i % 2 else '}' for i in reversed(range(d)))


def hard_numbers(rng):
    nums = []
    for _ in range(80):                                  # repr of random bit patterns
        x = struct.unpack("<d", rng.getrandbits(64).to_bytes(8, "little"))[0]
        if x == x and abs(x) != float("inf"):
            nums.append(repr(x))
    nums += ["9007199254740993", "9007199254740993.0", "1.00000000000000011102230246251565404236316680908203125",
             "1.00000000000000011102230246251565404236316680908203124", "2.4703282292062327e-324", "2.4703282292062328e-324",
             "4.9406564584124654e-324", "5e-324", "2.2250738585072011e-308", "2.2250738585072014e-308", "2.225073858507201e-308",
             "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "0.1", "0.30000000000000004", "1e23",
             "8.98846567431158e307", "-0", "-0.0", "0e5", "0.0e-5", "1E+2", "-1e-7", "123456789012345678", "1e400", "-1e400",
             "1e-400", "-1e-400", "123.456e-400", "0.000001e400", "1e-320", "4503599627370496.5", "4503599627370497.5"]
    for _ in range(40):                                  # 15 to 17 significant digits
        nd = rng.choice([15, 16, 17])
        m = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        nums.append(f"{m[0]}.{m[1:]}e{rng.randint(-330, 300)}")
        nums.append(f"{'-' if rng.random() < 0.5 else ''}0.{'0' * rng.randint(0, 5)}{m}")
    for v in (2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1, 2 ** 64 - 1, 2 ** 64, 2 ** 64 + 1, 10 ** 19, 10 ** 20):
        nums += [str(v), str(-v)]
    return nums


def big_integers():
    """(text, beyond the device limit?) integers just under and just over the 3200-bit capacity of the exact formatter."""
    out = []
    for v in (2 ** BIG_BITS - 1, 2 ** (BIG_BITS - 8), 10 ** 960, 2 ** BIG_BITS, 2 ** BIG_BITS + 1, 10 ** 970):
        out.append((str(v), v.bit_length() > BIG_BITS))
    return out


def long_mantissas(rng):
    """(text, beyond the device limit?) in-range numbers whose exact conversion runs close to the 3200-bit workspace: about
    900 to 963 significant digits with a negative exponent (the conversion scales the digits to 66 + 3.33 * |exponent| bits
    when they have fewer), and digit strings of more than 3200 bits, which are beyond the limit whatever their exponent."""
    out = []
    for nd, e in ((900, -895), (900, -840), (930, -925), (960, -900), (963, -903)):
        m = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        assert int(m).bit_length() <= BIG_BITS and 66 + (-e * 3402 >> 10) <= BIG_BITS - 32
        out.append((f"{m}e{e}", False))
        out.append((f"{m[:nd + e]}.{m[nd + e:]}", False))                # the same value without an exponent
    for nd, e in ((965, -960), (970, -900), (1000, -990)):
        m = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        assert int(m).bit_length() > BIG_BITS
        out.append((f"{m}e{e}", True))
        out.append((f"-{m[:nd + e]}.{m[nd + e:]}", True))
    return out


def big_json(rng, target, sensitive):
    rows = []
    n = 0
    while n < target:
        r = {"id": len(rows), "name": "user-%d" % rng.randrange(10 ** 6), "score": rng.random() * 100, "ok": rng.random() < 0.5}
        if sensitive:
            r["password"] = "pw%d" % len(rows)
        rows.append(r)
        n += 90
    import json

    return json.dumps({"rows": rows, "note": "x"})


def hostile_pool(seed):
    """[(unit bytes, beyond the device limits?)]; "toon": beyond the TOON encoders' limits only."""
    import json

    rng = random.Random(seed)
    pool = [(b"", False), (b"1", False), (b"{", False), (b" ", False), (b"x", False), (b'"', False),
            (b'{"a":1,}', False), (b"[01]", False), (b"\xff", False), (b'{"a":', False), (b'{"a" 1}', False), (b"[1] 2", False),
            (b'"\xc3"', False), (b'{"password": "\xed\xa0\x80"}', False)]
    for kind in ("arr", "obj", "mix"):
        for d in (63, 64, 65):
            pool.append(((nested(kind, d) + PAD).encode(), "toon" if d > DEPTH_LIMIT else False))   # masking parses serde_json's 127 levels
    pool.append(((nested("obj", 64)[:-1] + PAD).encode(), False))           # unterminated at depth 64
    for x in hard_numbers(rng):
        pool.append((('{"n": ' + x + ', "v": [' + x + ', 1], "rows": [{"a": ' + x + ', "b": 2}, {"a": 3, "b": ' + x + '}]}' + PAD).encode(), False))
    for x, beyond in big_integers() + long_mantissas(rng):
        pool.append((('{"n": ' + x + '}' + PAD).encode(), beyond))
        pool.append((("[" + x + ", 1]" + PAD).encode(), beyond))
    for s in ('\\ud83d\\ude00', '\\u00e9\\u65e5', 'a\\nb\\tc\\"d\\\\e\\/f', '\\u0000', '\\u001f x', '\\b\\f\\r', 'é日\U0001F600', '\\ud83d\\ude00' * 40):
        pool.append((('{"s": "' + s + '", "' + s + '": 1, "token": "' + s + '"}' + PAD).encode("utf-8"), False))
        pool.append((('["' + s + '", "' + s + '"]' + PAD).encode("utf-8"), False))
    pool.append((big_json(rng, 65536, False).encode(), False))
    pool.append((big_json(rng, 65536, True).encode(), False))
    pool.append((('["' + "é" * 32768 + '"]').encode(), False))
    pool.append((("[" + ", ".join(str(i) for i in range(12000)) + "]").encode(), False))
    return pool


def plain_unit(rng, i):
    """An ordinary small tool result, between the hostile units."""
    rows = [{"id": i * 10 + k, "name": "n%d" % rng.randrange(1000), "v": round(rng.random(), 3)} for k in range(rng.randint(0, 4))]
    import json

    return (json.dumps({"result": rows, "secret": "s%d" % i, "page": i}) + PAD).encode()


def batch_units(n, pool, seed):
    """n units: the hostile pool spread over the whole batch (every warp gets some) with ordinary units between them."""
    rng = random.Random(seed)
    out = []
    k = 0
    for i in range(n):
        if rng.random() < 0.5:
            out.append(pool[(k * 7919 + seed) % len(pool)])
            k += 1
        else:
            out.append((plain_unit(rng, i), False))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# oracles (cached per distinct unit: the pool repeats)
# ---------------------------------------------------------------------------------------------------------------------
_TOON, _MASK = {}, {}


def toon_oracle(b):
    if b not in _TOON:
        try:
            s = b.decode("utf-8")
        except UnicodeDecodeError:
            _TOON[b] = None
        else:
            _TOON[b] = toon_ref.process_text(s, 0, 1 << 30)
    return _TOON[b]


def mask_oracle(b, md):
    if (b, md) not in _MASK:
        try:
            _MASK[(b, md)] = mask_ref.mask_json_bytes(b, md)
        except (ValueError, RecursionError):
            _MASK[(b, md)] = None
    return _MASK[(b, md)]


# ---------------------------------------------------------------------------------------------------------------------
# device calls
# ---------------------------------------------------------------------------------------------------------------------
def toon_call(ctx, units, flags):
    """cf_toon_host with explicit flags: (status int32[n], out_len uint32[n], texts)."""
    stream, offs = engine.pack_units(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    out = np.empty(max(len(stream), 1), dtype=np.uint8)
    out_len = np.empty(n, dtype=np.uint32)
    status = np.empty(n, dtype=np.int32)
    with ctx.lock:
        ctx.check(ctx.lib.cf_toon_host(ctx.h, batch.h, flags, ctypes.cast(ctypes.c_char_p(stream), ctypes.c_void_p), len(stream), offs.ctypes.data, n,
                                       out.ctypes.data, out_len.ctypes.data, status.ctypes.data), "cf_toon_host")
    texts = [out[int(offs[i]):int(offs[i]) + int(out_len[i])].tobytes().decode("utf-8") if status[i] == engine.TOON_CONVERTED else None for i in range(n)]
    return status, out_len, texts


def check_toon(units, flags):
    ctx = engine.Context.get()
    st, _, texts = toon_call(ctx, [u for u, _ in units], flags)
    bad = []
    for i, ((u, beyond), s, t) in enumerate(zip(units, st, texts)):
        if beyond:
            ok = s == engine.TOON_UNSUPPORTED
        else:
            ok = s != engine.TOON_UNSUPPORTED and t == toon_oracle(u)
        if not ok:
            bad.append((i, u[:100], int(s), (t or "")[:100], (toon_oracle(u) or "")[:100] if not beyond else "UNSUPPORTED"))
    assert not bad, (len(bad), bad[:4])
    return st


def check_mask(units, md):
    ctx = engine.Context.get()
    stream, offs = engine.pack_units([u for u, _ in units])
    st, outs = engine.mask_host(engine.Batch(ctx, len(stream), len(units)), stream, offs, md)
    bad = []
    for i, ((u, beyond), s, o) in enumerate(zip(units, st, outs)):
        if beyond is True:          # past the workspace: UNSUPPORTED, unless the number is out of binary64's range (the crate's ValueError)
            ok = s == (engine.MASK_PARSE_ERROR if mask_oracle(u, md) is None else engine.MASK_UNSUPPORTED) and o is None
        else:
            ok = s != engine.MASK_UNSUPPORTED and o == mask_oracle(u, md)
        if not ok:
            bad.append((i, u[:100], int(s), (o or b"")[:100], (mask_oracle(u, md) or b"")[:100] if beyond is not True else "UNSUPPORTED"))
    assert not bad, (len(bad), bad[:4])
    return st


SIZES = [200, 6000, 40000]           # 1, 4 and 32 units per warp on a 132-SM H100


@pytest.fixture(scope="module")
def pool():
    return hostile_pool(1)


def test_long_mantissas_on_the_cpu_build():
    """The exact decimal conversion (json_toon.h, shared by the TOON and masking kernels) built for the CPU: digit strings of
    up to 3199 bits convert exactly when their exponent needs no more workspace (regression: a shift by zero bits of a
    100-word number was refused, and such in-range numbers came back UNSUPPORTED); longer digit strings are UNSUPPORTED."""
    import hostsim_util as hs

    for x, beyond in long_mantissas(random.Random(2)):
        u = ('{"n": ' + x + ', "m": [' + x + ']}' + PAD).encode()
        for md in (10, 3):
            st, out = hs.mask_host(u, md)
            assert (st == 6) if beyond else (st == 0 and out == mask_oracle(u, md)), (x[:20], len(x), md, st)
        st, out = hs.toon_host(u)
        assert (st == 6) if beyond else (st == 0 and out == toon_oracle(u)), (x[:20], len(x), st)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_mask_packed_warps_vs_serde_limits(pool, n):
    """Masking at serde_json's limits: the 65-level units mask like the oracle, integers beyond the 3200-bit workspace are out of
    binary64's range (the crate's ValueError), and only in-range literals past the workspace are UNSUPPORTED."""
    units = batch_units(n, pool, n)
    for md in (10, 3):
        st = check_mask(units, md)
        assert (st == engine.MASK_OK).sum() > n // 3
        assert (st == engine.MASK_UNSUPPORTED).sum() >= 1 if n >= 6000 else True


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("mode", ["default", "sequential"])
def test_toon_packed_warps_vs_oracle(pool, n, mode):
    units = batch_units(n, pool, n + 1)
    st = check_toon(units, TOON_REPORT_ERRORS | (TOON_SEQUENTIAL if mode == "sequential" else 0))
    assert (st == engine.TOON_CONVERTED).sum() > n // 3


@pytest.mark.gpu
def test_every_hostile_unit_once_at_serde_limits(pool):
    """The whole pool in one small batch (one unit per warp), so that no unit of it can escape the comparison by chance; masking
    held to serde_json's limits as in test_mask_packed_warps_vs_serde_limits, TOON to its 64 levels."""
    check_mask(pool, 10)
    check_toon(pool, TOON_REPORT_ERRORS)
    check_toon(pool, TOON_REPORT_ERRORS | TOON_SEQUENTIAL)


# ---------------------------------------------------------------------------------------------------------------------
# hand-over reasons of the token-parallel kernel
# ---------------------------------------------------------------------------------------------------------------------
FB = {"NUM_EXACT": 1, "KEY_ESCAPE": 2, "TOK_CAP": 3, "KH_CAP": 4, "DUP_HASH": 5, "ROW_ORDER": 6, "MIXED_ITEM": 7, "TOO_LONG": 8}


def fallback_corpus():
    """{reason: [units that the token-parallel kernel hands over for that reason]}.  Every FB_* reason is reachable."""
    return {
        # a number whose TOON form needs the exact big-integer formatter (num_canon cannot shorten it on the fast path)
        "NUM_EXACT": ['{"n": 1.5e300, "m": 2}' + PAD, '{"n": 123456789012345678901234567890}' + PAD, '[0.1e1, 2]' + PAD],
        "KEY_ESCAPE": ['{"a\\nb": 1, "c": 2}' + PAD, '{"k\\u00e9y": [1, 2]}' + PAD],
        # more significant tokens than the scratch holds (len / 2 + 64): empty containers are one token per byte and a half
        "TOK_CAP": ["[" + "[]," * 1000 + "[]]" + PAD, "[" + "{}," * 600 + "{}]"],
        # more keys in the open objects than the duplicate screen's stack holds (256)
        "KH_CAP": ["{" + ", ".join('"k%d": %d' % (i, i) for i in range(300)) + "}" + PAD],
        "DUP_HASH": ['{"a": 1, "b": 2, "a": 3}' + PAD, '[{"x": 1, "y": 2}, {"x": 1, "x": 2}]' + PAD],
        # a table whose later rows list the first row's keys in another order
        "ROW_ORDER": ['[{"a": 1, "b": 2}, {"b": 3, "a": 4}]' + PAD, '{"t": [{"p": "x", "q": 1, "r": true}, {"p": "y", "r": false, "q": 2}]}' + PAD],
        # the first field of a list item is an array whose first element is an object with a nested value and a later element
        # is not an object (whether toon.py's columnar attempt raises decides the answer)
        "MIXED_ITEM": ['[{"k": [{"a": [1]}, 2]}, 5]' + PAD, '{"l": [{"k": [{"a": {"b": 1}}, "s"], "m": 1}, 3]}' + PAD],
        # a string longer than a token's 20-bit length field
        "TOO_LONG": ['["' + "a" * (1 << 20) + '"]', '{"s": "' + "é" * (1 << 19) + '", "n": 1}'],
    }


def test_fallback_corpus_reaches_each_reason_in_the_warp_emulator():
    """The kernel body on the CPU warp emulator (tests/hostsim): each unit of the corpus is handed over for its reason."""
    import hostsim_util as hs

    corpus = fallback_corpus()
    assert set(corpus) == set(FB)
    for name, units in corpus.items():
        for u in units:
            st, _ = hs.toon_tp(u)
            assert (st, hs.toon_tp.last_reason) == (TS_FALLBACK, FB[name]), (name, u[:80], st, hs.toon_tp.last_reason)


@pytest.mark.gpu
def test_fallback_reasons_on_the_device_and_their_answers():
    ctx = engine.Context.get()
    corpus = fallback_corpus()
    units, reasons = [], []
    for name, us in corpus.items():
        for u in us:
            units.append(u.encode())
            reasons.append(FB[name])
    st, out_len, _ = toon_call(ctx, units, TOON_REPORT_ERRORS | TOON_NO_HANDOVER)
    assert [int(s) for s in st] == [TS_FALLBACK] * len(units)
    assert [int(x) for x in out_len] == reasons
    check_toon([(u, False) for u in units], TOON_REPORT_ERRORS)
    check_toon([(u, False) for u in units], TOON_REPORT_ERRORS | TOON_SEQUENTIAL)
