"""cf_run_batch's regex_filter rewriting: the substitution runs beside the TOON kernel and one gather places every produced text.
Checked against CPython `re` (the oracle), against cf_sub_host on the same batch, and host-buffer outputs against resident outputs,
at rewritten-unit counts from none to every unit, with per-unit stage sets, a rewrite that outgrows the first scratch bound, a rule
that deletes a whole unit, the exact output capacity, and an error return followed by a normal call on the same context."""
import ctypes
import json
import random
import re

import numpy as np
import pytest

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import toon_ref

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes")]
# "@" grows 100x: a unit of 3 000 "@" (300 000 bytes out) outgrows the first pass's 64 L + 64 KiB and runs again with 8x the room
BIG = [("@", 0, "Z" * 100), ("DELETE-THIS-UNIT", 0, "")]
SUB_TOON = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
SUB_ONLY = N.CF_STAGE_SCAN | N.CF_STAGE_SUB


def program(subs):
    p = engine.Program()
    for pat, f in HARMFUL:
        p.add_search(pat, f)
    for pat, f, r in subs:
        p.add_sub(pat, f, r)
    return p.compile(engine.Context.get())


class Oracle:
    """Expected results per distinct unit text (units repeat from small pools, so every text is computed once)."""

    def __init__(self, subs):
        self.rules = ref.regex_compile_rules([{"search": s, "replace": r} for s, _, r in subs])
        self.subs = subs
        self.cache = {}

    def __call__(self, u):
        if u not in self.cache:
            dirty = any(p.search(u) for p, _ in self.rules)
            bits = ref.scan_bitmaps([u], HARMFUL, [], [(p, f) for p, f, _ in self.subs])[0]
            self.cache[u] = (bits, dirty, ref.regex_apply_str(self.rules, u).encode() if dirty else None, toon_ref.process_text(u, 0, 1 << 30))
        return self.cache[u]


def pools():
    rng = random.Random(7)
    clean = [synth.payload("A", rng.randrange(600, 3000), seed=s) for s in range(10)] + \
            [synth.payload("B", rng.randrange(600, 2500), seed=s) for s in range(4)] + \
            [synth.payload("C", rng.randrange(300, 2000), seed=s, hit_rate=0.0) for s in range(6)] + ["", "x", "Kill him now"]
    dirty = [json.dumps({"rows": [{"id": i, "t": "crap" if i % 7 == 0 else "ok"} for i in range(k)]}) for k in (3, 20, 45)] + \
            ["this is crap", "crud", "crap crud crap", "a crapcrudcrap b " * 30, json.dumps({"note": "total crud", "n": 5}),
             synth.payload("C", 1500, seed=3, hit_rate=0.0) + " crap", "é crap 日本 crud 😀"]
    return clean, dirty


CLEAN, DIRTY = pools()


def make_units(n, n_dirty, seed):
    rng = random.Random(seed)
    where = set(rng.sample(range(n), n_dirty))
    return [DIRTY[rng.randrange(len(DIRTY))] if i in where else CLEAN[rng.randrange(len(CLEAN))] for i in range(n)]


def check(oracle, units, mask, stages, v, out, oo):
    """Verdicts and texts of one call against the oracle; returns the indices of the rewritten units."""
    rewritten = []
    for i, u in enumerate(units):
        bits, dirty, sub_text, toon_text = oracle(u)
        st = int(stages[i]) if stages is not None else 0xFF
        flags, got = int(v["flags"][i]), out[int(oo[i]):int(oo[i + 1])].tobytes()
        assert int(v["match_bitmap"][i]) == bits, i
        assert int(v["out_len"][i]) == len(got), i
        if dirty and st & N.CF_STAGE_SUB:
            rewritten.append(i)
            assert flags & N.CF_V_REWRITTEN and not flags & N.CF_V_TOON, (i, flags)
            assert got == sub_text, i
            toon_here = bool(mask & N.CF_STAGE_TOON)
            assert bool(flags & N.CF_V_RESUBMIT) == (toon_here and bool(st & N.CF_STAGE_TOON)), (i, flags)
            if toon_here:
                assert int(v["aux"][i]) == engine.TOON_SKIPPED, i
        elif mask & N.CF_STAGE_TOON and st & N.CF_STAGE_TOON:
            assert not flags & (N.CF_V_REWRITTEN | N.CF_V_RESUBMIT), i
            assert (got.decode() if flags & N.CF_V_TOON else None) == toon_text, i
        else:
            assert flags == 0 and got == b"", (i, flags)
            if mask & N.CF_STAGE_TOON:
                assert int(v["aux"][i]) == engine.TOON_SKIPPED, i
    return rewritten


def run_all_ways(prog, oracle, units, mask, stages=None):
    """Host buffers, then the resident batch with resident outputs: byte-equal, both right, and the rewritten texts equal
    cf_sub_host's on the same batch."""
    ctx = engine.Context.get()
    stream, offs = engine.pack_units([engine.encode_unit(u) for u in units])
    batch = engine.Batch(ctx, len(stream), len(units))
    v, out, oo, _ = engine.run_batch(prog, batch, stream, offs, mask, stages)
    out = out[:int(oo[-1])].copy()
    rewritten = check(oracle, units, mask, stages, v, out, oo)
    v2, none, oo2, _ = engine.run_batch(prog, batch, None, offs, mask, stages, outputs_resident=True)
    assert none is None and v2.tobytes() == v.tobytes() and np.array_equal(oo2, oo)
    assert engine.device_output(ctx).tobytes() == out.tobytes()
    if rewritten:
        for i, g in zip(rewritten, engine.sub_host(prog, batch, rewritten)):
            assert g == out[int(oo[i]):int(oo[i + 1])].tobytes(), i
    return v, out, oo, rewritten


@pytest.mark.parametrize("mask", [SUB_TOON, SUB_ONLY], ids=["with_toon", "without_toon"])
@pytest.mark.parametrize("n,n_dirty", [(600, 0), (600, 1), (700, 255), (700, 256), (2400, 2000), (400, 400)])
def test_rewritten_unit_counts(mask, n, n_dirty):
    prog = program(SUBS)
    oracle = Oracle(SUBS)
    units = make_units(n, n_dirty, seed=n * 1000 + n_dirty)
    _v, _out, _oo, rewritten = run_all_ways(prog, oracle, units, mask)
    assert len(rewritten) == n_dirty


def test_unit_stages_mix_sub_and_toon():
    prog = program(SUBS)
    oracle = Oracle(SUBS)
    rng = random.Random(11)
    units = make_units(1500, 500, seed=3)
    choices = [N.CF_STAGE_SUB, N.CF_STAGE_TOON, N.CF_STAGE_SUB | N.CF_STAGE_TOON, 0, N.CF_STAGE_SCAN]
    stages = np.array([rng.choice(choices) for _ in units], dtype=np.uint8)
    v, _out, _oo, rewritten = run_all_ways(prog, oracle, units, SUB_TOON, stages)
    resubmit = [i for i in range(len(units)) if v["flags"][i] & N.CF_V_RESUBMIT]
    assert resubmit and len(resubmit) < len(rewritten)        # both kinds of rewritten unit occur
    assert any(v["flags"][i] & N.CF_V_TOON for i in range(len(units)))


def test_regrow_and_whole_unit_deletion():
    prog = program(BIG)
    oracle = Oracle(BIG)
    units = (CLEAN[10:] + ["@" * 3000, "DELETE-THIS-UNIT", "x@y", "@" * 200, json.dumps({"a": "@", "b": [1, 2]}), "DELETE-THIS-UNIT and more"]) * 3
    for mask in (SUB_TOON, SUB_ONLY):
        v, out, oo, rewritten = run_all_ways(prog, oracle, units, mask)
        big = [i for i in rewritten if units[i] == "@" * 3000]
        gone = [i for i in rewritten if units[i] == "DELETE-THIS-UNIT"]
        assert big and all(int(v["out_len"][i]) == 300000 for i in big)
        assert gone and all(int(v["out_len"][i]) == 0 and v["flags"][i] & N.CF_V_REWRITTEN for i in gone)


def test_output_capacity_is_checked_before_any_write():
    ctx = engine.Context.get()
    prog = program(SUBS)
    units = make_units(900, 300, seed=5)
    stream, offs = engine.pack_units([engine.encode_unit(u) for u in units])
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    v0, out0, oo0, _ = engine.run_batch(prog, batch, stream, offs, SUB_TOON)
    need = int(oo0[-1])
    for cap, want in ((need - 1, N.CF_E_CAPACITY), (need, N.CF_OK)):
        v = np.zeros(n, dtype=engine.VERDICT_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        buf = np.full(need + 64, 0xAB, dtype=np.uint8)
        got_need = ctypes.c_uint64(0)
        with ctx.lock:
            rc = ctx.lib.cf_run_batch(ctx.h, prog.h, batch.h, None, len(stream), offs.ctypes.data, n, SUB_TOON, None, 0, 10, v.ctypes.data, None,
                                      buf.ctypes.data, cap, oo.ctypes.data, ctypes.byref(got_need))
        assert rc == want and got_need.value == need, (cap, rc)
        if rc == N.CF_OK:
            assert buf[:need].tobytes() == out0[:need].tobytes() and v.tobytes() == v0.tobytes() and np.array_equal(oo, oo0)
            assert (buf[need:] == 0xAB).all()
        else:
            assert (buf == 0xAB).all()                              # refused before anything reached out_bytes


def test_too_large_then_a_normal_call_on_the_same_context():
    """Resident offsets that disagree with the batch (same unit count and total) size a unit's scratch too small: its rewrite
    outgrows even the worst case computed from them, the call returns CF_E_TOO_LARGE, and the next call on the context is right."""
    ctx = engine.Context.get()
    prog = program(BIG)
    oracle = Oracle(BIG)
    units = ["@" * 2000, "xy"] + CLEAN[10:16]
    stream, offs = engine.pack_units([engine.encode_unit(u) for u in units])
    batch = engine.Batch(ctx, len(stream), len(units))
    batch.upload(stream, offs)
    wrong = offs.copy()
    wrong[1] = 3                                                 # unit 0 claims 2 bytes, unit 1 the rest
    for mask in (SUB_TOON, SUB_ONLY):
        with pytest.raises(N.CfError) as exc:
            engine.run_batch(prog, batch, None, wrong, mask, outputs_resident=True)
        assert exc.value.code == N.CF_E_TOO_LARGE and "exceeds the worst-case bound" in str(exc.value)
        v, _none, oo, _ = engine.run_batch(prog, batch, None, offs, mask, outputs_resident=True)
        check(oracle, units, mask, None, v, engine.device_output(ctx), oo)
        v, out, oo, _ = engine.run_batch(prog, batch, stream, offs, mask)
        check(oracle, units, mask, None, v, out, oo)
