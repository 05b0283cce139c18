"""The bodies of tests/test_mask_edges_gpu.py (float binade edges, values that are never printed, nesting either side of serde_json's
limit, outputs up to ten times their input) on the host build of csrc/json_mask.h — the source mask_kernel compiles — sized per unit
like cf_mask_host sizes it (5 * len + 32 bytes, then a retry into the length the unit asked for), and through the masking module
with its launches on the CPU simulator."""
import importlib

import pytest

import hostsim_batcher
import hostsim_util as hs
import test_mask_edges_gpu as tg


@pytest.fixture()
def mod(monkeypatch):
    hostsim_batcher.install(monkeypatch)
    return importlib.import_module("request_logging_masking_native_extension")


def check(bodies, max_depth):
    exp = [tg.expected(b, max_depth) for b in bodies]
    bad = []
    for b, e in zip(bodies, exp):
        st, got = hs.mask_host(b, max_depth)
        if got != e or st != (0 if e is not None else 2):
            bad.append((b[:80], st, got and got[:80], e and e[:80]))
    assert not bad, bad[:5]
    return exp


def test_floats_print_shortest_round_trip_digits():
    exp = check(tg.float_bodies(), 10)
    assert all(e is not None for e in exp)


def test_power_of_two_edges_take_the_far_side_decimal():
    # the nearest 16-digit decimal of these falls below the round-trip interval; serde_json prints the one above
    for lit, want in [("5.960464477539063e-08", b"[5.960464477539063e-8]"), ("5.684341886080802e-14", b"[5.684341886080802e-14]"),
                      ("6.189700196426902e+26", b"[6.189700196426902e26]")]:
        assert hs.mask_host(("[" + lit + "]").encode())[1] == want


def test_values_never_printed_still_fail_the_parse():
    for md in (10, 1):
        assert all(e is None for e in check(tg.unprinted_bodies(), md))
    assert all(e is not None for e in check(tg.in_range_bodies(), 10))


@pytest.mark.parametrize("max_depth", [10, 1, 127])
def test_nesting_either_side_of_the_recursion_limit(max_depth):
    exp = check(tg.nesting_bodies(), max_depth)
    assert [e is None for e in exp[:3 * len(tg.NEST_DEPTHS)]] == [d > 127 for d in tg.NEST_DEPTHS for _ in range(3)]


def test_outputs_much_larger_than_their_input():
    for b, md in tg.growth_cases():
        e = tg.expected(b, md)
        st, first = hs.mask_host(b, md, retry=False)
        if len(e) > 5 * len(b) + 32:
            assert (st, first) == (hs.MASK_OVERFLOW, len(e)), (b[:40], md)     # the first pass reports the exact length it needs
        else:
            assert (st, first) == (0, e)
        assert hs.mask_host(b, md) == (0, e)
    assert {len(tg.expected(b, md)) - 5 * len(b) for b, md in tg.growth_cases()} >= {32, 33}


def test_module_batches_on_the_simulator(mod):
    for md, bodies in [(10, tg.float_bodies()[::7] + tg.unprinted_bodies() + tg.in_range_bodies()), (1, tg.nesting_bodies())]:
        assert mod.mask_sensitive_json_bytes_batch(bodies, md) == [tg.expected(b, md) for b in bodies]
    for b, md in tg.growth_cases():
        assert mod.mask_sensitive_json_bytes(b, md) == tg.expected(b, md)
    with pytest.raises(ValueError):
        mod.mask_sensitive_json_bytes(b'{"password":1e400}')
    with pytest.raises(RuntimeError, match="3200-bit"):
        mod.mask_sensitive_json_bytes_batch([b"[1.5]", b"[0." + b"1" * 1200 + b"]"])


def test_backslash_key_names_are_classified_as_written():
    """A raw key name's backslash is a character, not an escape (regression: "pass\\word" was classified as "password"); the same
    names escaped in a JSON body are decoded first."""
    from oracle import mask_ref

    for k in tg.BACKSLASH_KEYS:
        assert hs.key_sensitive_host(k) == mask_ref.is_sensitive_key(k), k
    assert any(mask_ref.is_sensitive_key(k) for k in tg.BACKSLASH_KEYS) and not all(mask_ref.is_sensitive_key(k) for k in tg.BACKSLASH_KEYS)
    import json

    check([json.dumps({k: "v", "n": [k]}).encode() for k in tg.BACKSLASH_KEYS], 10)
