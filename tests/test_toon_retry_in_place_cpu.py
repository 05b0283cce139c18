"""The in-place retry of the token-parallel TOON kernel body (csrc/json_tp.h toon_unit, on the CPU warp emulator, tools/toon_emu.py): a
unit whose first attempt stops at a mixed list-item array (FB_MIXED_ITEM) is analyzed in resolve mode and emitted again over the token
array it already has.  The result must be the one of the separate resolving pass that tokenizes the unit again (the first attempt, then
the resolving pass when the first attempt returns FB_MIXED_ITEM): same status, reason, out_len and bytes, in both lane orders and at
several 16-byte alignments, over the mixed list-item family, bench.py's payloads, the hand-over corpus of the GPU suite and the recorded
differential fuzz cases (whose recorded answers of the reference's toon.py the result must also equal unless the unit is handed over)."""
import gzip
import json
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import fuzz_toon_tp  # noqa: E402
import toon_emu  # noqa: E402
from test_json_packed_gpu import fallback_corpus  # noqa: E402
from test_toon_mixed_items_cpu import mixed_family  # noqa: E402

FALLBACK, FB_MIXED_ITEM, FB_KH_CAP = 7, 7, 4
CONFIGS = [0, 1, 3 << 4, 1 | (9 << 4), 14 << 4]          # toon_emu `order`: bit 0 the lane order, bits 4.. the text's shift from the 16-byte grid


def two_pass(text, **kw):
    """The unit as the kernel used to encode it: the first attempt, then for FB_MIXED_ITEM the resolving pass from the unit's bytes."""
    st, txt, why, n, _ = toon_emu.run(text, toon_emu.FIRST, **kw)
    if st == FALLBACK and why == FB_MIXED_ITEM:
        return toon_emu.run(text, toon_emu.RESOLVE, **kw)[:4], True
    return (st, txt, why, n), False


def check(texts, configs, kinds=((True, True), (False, False))):
    """Every text in every config and every (unlimited, report_errors) kind; returns how many runs went through the retry."""
    retried = 0
    for text in texts:
        for order in configs:
            for unlimited, rep in kinds:
                kw = {"order": order, "unlimited": unlimited, "report_errors": rep}
                exp, r = two_pass(text, **kw)
                got = toon_emu.run(text, toon_emu.IN_PLACE, **kw)[:4]
                assert got == exp, (text[:200], kw, got, exp)
                retried += r
    return retried


def kh_cap_in_resolve_mode():
    """A mixed list-item array whose first row (100 keys, one nested value) is kept on the key stack in resolve mode, so that the keys of
    the second row's nested object no longer fit (FB_KH_CAP), while the first attempt, which keeps no first row, fits them."""
    row0 = {"n": {"x": 1}, **{f"k{i}": i for i in range(99)}}
    row1 = {"n": {f"m{i}": i for i in range(200)}, **{f"k{i}": i for i in range(99)}}
    return json.dumps([{"rows": [row0, row1, 1]}])


@pytest.mark.parametrize("order", CONFIGS)
def test_mixed_family_in_place_equals_two_passes(order):
    texts = [json.dumps(d) for d in mixed_family()] + [json.dumps(d, indent=2) for d in mixed_family()[::7]]
    assert check(texts, [order]) > 500


def test_bench_payloads_in_place_equal_two_passes():
    # the product's settings (kept only when strictly smaller, errors not reported): four of bench.py's five nested-config payloads with a
    # mixed list-item array reach it before they outgrow their input
    assert check(bench.make_payloads(), [0, 1 | (7 << 4)], kinds=((False, False),)) == 2 * 4


def test_hand_over_corpus_in_place_equals_two_passes():
    corpus = fallback_corpus()
    assert check([u for us in corpus.values() for u in us if len(u) < 65536], [0, 1 | (5 << 4)]) >= 2 * 2 * len(corpus["MIXED_ITEM"])
    for u in [u for us in corpus.values() for u in us if len(u) >= 65536]:           # the long-token units: one config each
        assert check([u], [1 | (11 << 4)], kinds=((False, True),)) == 0


def test_kh_cap_during_the_retry_is_handed_over():
    text = kh_cap_in_resolve_mode()
    for order in (0, 1 | (6 << 4)):
        assert toon_emu.run(text, toon_emu.FIRST, order=order)[:3] == (FALLBACK, None, FB_MIXED_ITEM)
        assert toon_emu.run(text, toon_emu.IN_PLACE, order=order)[:3] == (FALLBACK, None, FB_KH_CAP)
    assert check([text], [0, 1 | (6 << 4)]) == 4


def test_recorded_fuzz_cases_in_place():
    """The cases of tests/golden/fuzz_toon.json.gz, regenerated as tools/fuzz_vs_reference.py generates them (the alignment it drew for
    each case included), in both lane orders."""
    with gzip.open(os.path.join(ROOT, "tests", "golden", "fuzz_toon.json.gz"), "rt", encoding="utf-8") as f:
        rec = json.load(f)
    seed, n, which = rec["args"]
    assert which == "gen1" and len(rec["answers"]) == int(n)
    rng = random.Random(int(seed))
    case = fuzz_toon_tp.make_gen(rng)
    compared = 0
    for ans in rec["answers"]:
        t = case()
        if ans is None or (ans[0] == 2 and any(0xD800 <= ord(c) <= 0xDFFF for c in t)):
            continue                                                  # skipped by the fuzz tool too (no shift is drawn for them)
        shift = rng.randrange(16) << 4
        for order in (shift, shift | 1):
            exp, _ = two_pass(t, unlimited=True, order=order)
            got = toon_emu.run(t, toon_emu.IN_PLACE, unlimited=True, order=order)[:4]
            assert got == exp, (t[:200], order, got, exp)
            if got[0] != FALLBACK:
                assert (got[0], got[1]) == (ans[0], ans[1]), (t[:200], got, ans)
                compared += 1
    assert compared > 5000, compared
