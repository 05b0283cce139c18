"""GPU: mask_kernel held to the oracle (oracle/mask_ref.py, serde_json's behaviour restated) where a one-lane JSON re-serialiser
usually goes wrong:
  * floats — the shortest round-trip digits of every binary64 power of two and its two neighbours, each written three ways, the exact
    integers 2^64 .. 2^1023, float32 powers of two and random float32 values (a power of two's round-trip interval is half as wide
    below it as above, so the nearest p-digit decimal can miss while the one on the other side hits);
  * values that are never printed — numbers out of binary64's range and lone surrogates under a sensitive key, below the depth cap,
    overwritten by a duplicate key: serde_json parses the whole document first, so each one fails the call;
  * nesting at 64 .. 200 levels, either side of serde_json's limit of 127;
  * outputs up to ten times their input, beside thousands of ordinary bodies packed several to a warp.
Every case runs through the drop-in module's batch API and through cf_run_batch(SCAN | MASK) with host buffers and resident.
tests/test_mask_edges_cpu.py runs the same bodies on the host build of csrc/json_mask.h."""
import importlib
import json
import math
import random

import numpy as np
import pytest

from mcp_context_forge_b200 import synth
from oracle import mask_ref

pytestmark = pytest.mark.gpu

PER_BODY = 16                               # numbers per float body: each one takes the big-integer path on one lane


# ------------------------------------------------------------------------------------------------------------- case generators
def float_literals():
    out = []
    for k in range(-1074, 1024):
        x = math.ldexp(1.0, k)
        for v in (math.nextafter(x, 0.0), x, math.nextafter(x, math.inf)):
            if v == 0.0 or math.isinf(v):
                continue
            out += [repr(v), "%.17e" % v, "%.25e" % v]
        if k >= 64:
            out.append(str(2 ** k))                 # beyond u64: the float path
    for k in range(-149, 128):                      # float32 powers of two, written as float32's shortest digits
        out.append(repr(float(np.float32(math.ldexp(1.0, k)))))
        out.append(str(np.float32(math.ldexp(1.0, k))))
    bits = np.random.default_rng(20240917).integers(0, 1 << 32, size=10000, dtype=np.uint64).astype(np.uint32)
    for f in bits.view(np.float32):
        if np.isfinite(f):
            out.append(repr(float(f)))
    return ["-" + t if i % 5 == 3 and t[0] != "-" else t for i, t in enumerate(out)]


def float_bodies():
    lits = float_literals()
    return [("[" + ",".join(lits[i:i + PER_BODY]) + "]").encode() for i in range(0, len(lits), PER_BODY)]


UNPRINTED_VALUES = ["1e400", "1e309", "-2e308", "1" * 310, '"\\ud800"', '"\\udbff"', '"\\udc00"', '"x\\udfff"', '"\\udc00\\ud800"']
UNPRINTED_PLACES = ['{"password":%s}', '{"a":[[[[[[[[[[[%s]]]]]]]]]]]}', '{"a":%s,"a":1}', '{"token":[1,%s]}', '{"b":{"a":[%s],"a":2}}']
# in range, near the edge the range check screens (10^308 <= value < 10^309 takes the exact conversion)
IN_RANGE_VALUES = ["1e308", "1.5e308", "0.15e309", "15" + "0" * 307, "9" * 308, "-1e308", "1e-400", "0e999", '"\\ud83d\\ude00"']


def unprinted_bodies():
    return [(p % v).encode() for p in UNPRINTED_PLACES for v in UNPRINTED_VALUES]


def in_range_bodies():
    return [(p % v).encode() for p in UNPRINTED_PLACES for v in IN_RANGE_VALUES]


def nest(depth: int, kind: str, inner: str = "0") -> str:
    opens, closes = [], []
    for i in range(depth):
        obj = kind == "obj" or (kind == "mix" and i % 2)
        opens.append('{"k%d":' % i if obj else "[")
        closes.append("}" if obj else "]")
    return "".join(opens) + inner + "".join(reversed(closes))


NEST_DEPTHS = (64, 65, 100, 126, 127, 128, 129, 200)


def nesting_bodies():
    out = [nest(d, k).encode() for d in NEST_DEPTHS for k in ("arr", "obj", "mix")]
    out += [('{"token":%s}' % nest(d, "mix")).encode() for d in (100, 126, 127)]
    out += [('{"x":%s}' % nest(d, "arr", '"\\ud800"')).encode() for d in (100, 127)]
    return out


def _fill(elem: str, size: int, wrap) -> str:
    n = 1
    while len(wrap(",".join([elem] * (n * 2)))) <= size:
        n *= 2
    lo, hi = n, n * 2
    while lo + 1 < hi:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if len(wrap(",".join([elem] * mid))) <= size else (lo, mid)
    return wrap(",".join([elem] * lo))


GROWTH_SIZES = (17, 16 << 10, 256 << 10)
# (element, wrapper, max_depth): nested-too-deep markers for short values, and numbers serde_json prints longer
GROWTH_SHAPES = [("0", lambda s: "[" + s + "]", 1), ("0", lambda s: "[" * 10 + s + "]" * 10, 10), ("[]", lambda s: '{"k":[' + s + "]}", 2),
                 ("1e15", lambda s: "[" + s + "]", 10), ("-0", lambda s: "[" + s + "]", 10)]


def growth_cases():
    """(body, max_depth) pairs: every shape at every size."""
    return [(_fill(e, size, w).encode(), md) for e, w, md in GROWTH_SHAPES for size in GROWTH_SIZES]


def expected(body: bytes, max_depth: int):
    try:
        return mask_ref.mask_json_bytes(body, max_depth)
    except ValueError:
        return None


# Key names holding a backslash or the text of a JSON escape.  A name handed over as a str (mask_sensitive_data, the header
# masking) is classified as written: "pass\\word" is not "password", and "pass\\u0077ord" is not either.  In a JSON body the
# same names arrive escaped and are decoded first.
BACKSLASH_KEYS = ["pass\\word", "pass\\\\word", "\\password", "password\\", "api\\_key", "API\\u004bey", "pass\\u0077ord", "to\\ken",
                  "secret\\n", "\\u0074oken", "jwt\\", "\\", "x\\", "\\\"token", "pass\\/word", "to\\u006ben"]


def packed_with_neighbours(special, n_plain: int = 3000, seed: int = 7):
    """`special` bodies at random places among n_plain ordinary synth bodies (several to a warp once the batch is this large)."""
    rng = random.Random(seed)
    bodies = [synth.payload("B" if i % 3 else "A", rng.choice([300, 700, 1500]), seed=i).encode() for i in range(n_plain)]
    where = sorted(rng.sample(range(n_plain + len(special)), len(special)))
    for pos, b in zip(where, special):
        bodies.insert(pos, b)
    return bodies, where


# ------------------------------------------------------------------------------------------------------------------- GPU runs
@pytest.fixture(scope="module")
def mod():
    return importlib.import_module("request_logging_masking_native_extension")


@pytest.fixture(scope="module")
def chain():
    from mcp_context_forge_b200 import engine

    ctx = engine.Context.get(0)
    prog = engine.Program()
    prog.add_literal("zqxj")
    prog.compile(ctx)
    return ctx, prog


def check_all_paths(mod, chain, bodies, max_depth: int):
    from mcp_context_forge_b200 import engine
    from mcp_context_forge_b200._native import CF_STAGE_MASK, CF_STAGE_SCAN, CF_V_MASKED

    exp = [expected(b, max_depth) for b in bodies]
    got = mod.mask_sensitive_json_bytes_batch(bodies, max_depth)
    bad = [i for i, (g, e) in enumerate(zip(got, exp)) if g != e]
    assert not bad, [(bodies[i][:80], got[i] and got[i][:80], exp[i] and exp[i][:80]) for i in bad[:5]]
    ctx, prog = chain
    stream, offs = engine.pack_units(bodies)
    batch = engine.Batch(ctx, len(stream), len(bodies))
    for host in (True, False):
        v, out, oo, _ = engine.run_batch(prog, batch, np.frombuffer(stream, dtype=np.uint8) if host else None, offs,
                                         CF_STAGE_SCAN | CF_STAGE_MASK, mask_max_depth=max_depth)
        for i, e in enumerate(exp):
            masked = bool(v["flags"][i] & CF_V_MASKED)
            assert masked == (e is not None), (i, host, bodies[i][:80])
            assert int(v["aux"][i]) == (engine.MASK_OK if e is not None else engine.MASK_PARSE_ERROR), (i, host)
            assert int(v["out_len"][i]) == (len(e) if e is not None else 0), (i, host)
            assert out[int(oo[i]):int(oo[i + 1])].tobytes() == (e if e is not None else b""), (i, host, bodies[i][:80])
        assert int(oo[-1]) == sum(len(e) for e in exp if e is not None)
    return exp


def test_floats_print_shortest_round_trip_digits(mod, chain):
    bodies = float_bodies()
    assert len(bodies) > 1500
    exp = check_all_paths(mod, chain, bodies, 10)
    assert all(e is not None for e in exp)


def test_values_never_printed_still_fail_the_parse(mod, chain):
    bodies = unprinted_bodies()
    for md in (10, 1):
        exp = check_all_paths(mod, chain, bodies, md)
        assert all(e is None for e in exp)
    exp = check_all_paths(mod, chain, in_range_bodies(), 10)
    assert all(e is not None for e in exp)


@pytest.mark.parametrize("max_depth", [10, 1, 127])
def test_nesting_either_side_of_the_recursion_limit(mod, chain, max_depth):
    bodies = nesting_bodies()
    exp = check_all_paths(mod, chain, bodies, max_depth)
    assert [e is None for e in exp[:3 * len(NEST_DEPTHS)]] == [d > 127 for d in NEST_DEPTHS for _ in range(3)]
    assert exp[3 * len(NEST_DEPTHS)] == b'{"token":"******"}'


def test_outputs_much_larger_than_their_input_among_packed_neighbours(mod, chain):
    cases = growth_cases()
    by_depth = {}
    for b, md in cases:
        by_depth.setdefault(md, []).append(b)
    for md, special in by_depth.items():
        bodies, where = packed_with_neighbours(special, seed=md)
        exp = check_all_paths(mod, chain, bodies, md)
        assert any(len(exp[i]) > 5 * len(bodies[i]) + 32 for i in where)      # outgrows the room of the first pass
    assert max(len(expected(b, md)) / len(b) for b, md in cases) > 9


def test_literals_beyond_the_workspace_fail_loudly(mod):
    with pytest.raises(RuntimeError, match="3200-bit"):
        mod.mask_sensitive_json_bytes_batch([b"[1.5]", b"[0." + b"1" * 1200 + b"]"])


def test_backslash_key_names_are_classified_as_written(mod):
    data = {k: "v" for k in BACKSLASH_KEYS}
    assert mod.mask_sensitive_data(data) == mask_ref.mask_value(data)
    assert mod.mask_sensitive_headers(data) == mask_ref.mask_headers(data)
    bodies = [json.dumps({k: "v"}).encode() for k in BACKSLASH_KEYS]
    assert mod.mask_sensitive_json_bytes_batch(bodies) == [expected(b, 10) for b in bodies]
