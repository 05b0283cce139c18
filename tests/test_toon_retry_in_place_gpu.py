"""Mixed list-item arrays retried in place by toon_tp_kernel (see test_toon_retry_in_place_cpu.py), on the GPU: the mixed list-item
family, bench.py's payload mix and a unit whose retry runs out of key-stack room (FB_KH_CAP), packed in their natural order, reversed
and sorted, through cf_toon_host and through cf_run_batch with host buffers and resident.  No unit is left at status 7 and every text
equals the oracle's; with CF_TOON_NO_HANDOVER the kernel makes the first attempt only, so a mixed unit reports FB_MIXED_ITEM as the
emulated first attempt does."""
import json
import os
import sys

import numpy as np
import pytest

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine
from oracle import toon_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import toon_emu  # noqa: E402
from test_toon_mixed_items_cpu import mixed_family  # noqa: E402
from test_toon_retry_in_place_cpu import kh_cap_in_resolve_mode  # noqa: E402

pytestmark = pytest.mark.gpu
REPORT_ERRORS, NO_HANDOVER = 1, 16
FALLBACK, FB_MIXED_ITEM, FB_KH_CAP = 7, 7, 4


def corpus():
    return [json.dumps(d, indent=2) for d in mixed_family()] + bench.make_payloads() + [kh_cap_in_resolve_mode()]


def packed(texts, packing):
    if packing == "reversed":
        return texts[::-1]
    if packing == "sorted":
        return sorted(texts)
    return list(texts)


def toon_host(texts, flags):
    """cf_toon_host: [(status, reason or TOON text)] per unit."""
    ctx = engine.Context.get()
    stream, offs = engine.pack_units([engine.encode_unit(t) for t in texts])
    status, got, out_len = engine.toon_host_flags(engine.Batch(ctx, len(stream), len(texts)), stream, offs, flags)
    return [(int(s), int(k) if g is None else g.decode()) for s, g, k in zip(status, got, out_len)]


@pytest.fixture(scope="module")
def expected():
    return {t: toon_ref.process_text(t, 0, 1 << 30) for t in corpus()}


@pytest.mark.parametrize("packing", ["natural", "reversed", "sorted"])
@pytest.mark.parametrize("flags", [0, REPORT_ERRORS])
def test_toon_host(expected, packing, flags):
    texts = packed(corpus(), packing)
    for t, (st, got) in zip(texts, toon_host(texts, flags)):
        assert st != FALLBACK, t[:200]
        assert (got if st == 0 else None) == expected[t], t[:200]


@pytest.mark.parametrize("packing", ["natural", "reversed", "sorted"])
def test_run_batch_host_buffers_and_resident(expected, packing):
    texts = packed(corpus(), packing)
    ctx = engine.Context.get()
    stream, offs = engine.pack_units([engine.encode_unit(t) for t in texts])
    batch = engine.Batch(ctx, len(stream), len(texts))
    v, out, oo, _ = engine.run_batch(None, batch, stream, offs, N.CF_STAGE_TOON)
    out = out[:int(oo[-1])].tobytes()
    for i, t in enumerate(texts):
        assert int(v["aux"][i]) != FALLBACK, t[:200]
        got = out[int(oo[i]):int(oo[i + 1])].decode() if v["flags"][i] & N.CF_V_TOON else None
        assert got == expected[t], t[:200]
    v2, none, oo2, _ = engine.run_batch(None, batch, None, offs, N.CF_STAGE_TOON, outputs_resident=True)
    assert none is None and v2.tobytes() == v.tobytes() and np.array_equal(oo2, oo)
    assert engine.device_output(ctx).tobytes() == out


def test_no_handover_reports_the_first_attempt():
    texts = [json.dumps(d, indent=2) for d in mixed_family()] + [kh_cap_in_resolve_mode()]
    got = toon_host(texts, REPORT_ERRORS | NO_HANDOVER)
    n_mixed = 0
    for t, (st, why) in zip(texts, got):
        est, _, ewhy, _, _ = toon_emu.run(t, toon_emu.FIRST)
        if est == FALLBACK:
            assert (st, why) == (FALLBACK, ewhy), t[:200]
            n_mixed += ewhy == FB_MIXED_ITEM
        else:
            assert st == est, t[:200]
    assert n_mixed > 500 and got[-1] == (FALLBACK, FB_MIXED_ITEM)
    # without the flag the retry of the last unit runs out of key-stack room and the sequential encoder answers
    st, txt = toon_host([texts[-1]], REPORT_ERRORS)[0]
    assert toon_emu.run(texts[-1], toon_emu.IN_PLACE)[:3] == (FALLBACK, None, FB_KH_CAP)
    assert (txt if st == 0 else None) == toon_ref.process_text(texts[-1], 0, 1 << 30)
