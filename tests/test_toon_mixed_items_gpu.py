"""Mixed list-item arrays (see test_toon_mixed_items_cpu.py) through the whole TOON stage on the GPU: the first token-parallel pass,
the resolving pass for the units it hands over as mixed, the sequential encoder for the rest.  Every result equals the oracle, as do
the results of bench.py's payload mix."""
import json
import os
import sys

import pytest

from mcp_context_forge_b200 import engine
from oracle import toon_ref

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from test_toon_mixed_items_cpu import mixed_family  # noqa: E402

pytestmark = pytest.mark.gpu
REPORT_ERRORS, FALLBACK = 1, 7


def toon(texts, flags):
    ctx = engine.Context.get()
    enc = [engine.encode_unit(t) for t in texts]
    stream, offs = engine.pack_units(enc)
    status, got, _ = engine.toon_host_flags(engine.Batch(ctx, len(stream), len(enc)), stream, offs, flags)
    return [(int(s), None if g is None else g.decode()) for s, g in zip(status, got)]


@pytest.mark.parametrize("flags", [0, REPORT_ERRORS])
def test_mixed_list_items_and_bench_mix(flags):
    texts = [json.dumps(d, indent=2) for d in mixed_family()] + bench.make_payloads()
    for t, (st, got) in zip(texts, toon(texts, flags)):
        assert st != FALLBACK, t[:200]
        assert got == toon_ref.process_text(t, 0, 1 << 30), t[:200]
