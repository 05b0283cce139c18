"""GPU parity of the token-parallel TOON kernel (toon_tp_kernel, csrc/json_tp.h) through the C ABI: the default cf_toon_host
path (token-parallel + sequential hand-over) must equal the sequential encoder (CF_TOON_SEQUENTIAL) unit for unit on a
seeded fuzz corpus, and the tabular bench shape must stay on the fast path."""
import json
import os
import random
import sys

import pytest

from mcp_context_forge_b200 import engine, synth
from oracle import toon_ref

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import fuzz_toon_tp  # noqa: E402

pytestmark = pytest.mark.gpu
SEQ, NOFB = 8, 16


def toon(texts, flags):
    ctx = engine.Context.get()
    enc = [engine.encode_unit(t) for t in texts]
    stream, offs = engine.pack_units(enc)
    status, got, out_len = engine.toon_host_flags(engine.Batch(ctx, len(stream), len(enc)), stream, offs, flags)
    return [(int(s), g) for s, g in zip(status, got)], status, out_len


@pytest.mark.parametrize("rep", [0, 1])
def test_fuzz_token_parallel_equals_sequential(rep):
    rng = random.Random(77 + rep)
    case = fuzz_toon_tp.make_gen(rng)
    texts = [case() for _ in range(20000)]
    a, _, _ = toon(texts, rep | SEQ)
    b, _, _ = toon(texts, rep)
    bad = []
    for t, x, y in zip(texts, a, b):
        if x == y:
            continue
        if not rep and x[0] in (1, 3, 4) and y[0] in (1, 3, 4):
            continue
        bad.append((t[:200], x, y))
    assert not bad, bad[:3]
    _, st, why = toon(texts, rep | NOFB)
    handed = int((st == 7).sum())
    assert 0 < handed < len(texts) // 3          # the hand-over exists and is the minority even on this adversarial corpus


def test_bench_shapes_fast_path_and_oracle():
    texts = [synth.payload("A", 16384, seed=s) for s in range(96)] + [synth.payload("A", 2048, seed=s) for s in range(64)] + [synth.payload("A", 262144, seed=s) for s in range(4)]
    texts += [json.dumps({"doc": synth.payload("C", 16384, seed=s), "n": s}) for s in range(32)]
    res, st, _ = toon(texts, NOFB)
    assert int((st == 7).sum()) == 0
    for t, (s, got) in zip(texts, res):
        assert (got.decode("utf-8") if s == 0 else None) == toon_ref.process_text(t, 0, 1 << 30)
