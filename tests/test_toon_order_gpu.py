"""The TOON first pass takes its units in cost order (toon_order_kernel + a radix sort, csrc/cfjson.cu): the order may change which
warp encodes a unit, never what the unit becomes.  Checked here: the same units in natural, reversed and shape-sorted packings give
identical per-unit results through cf_toon_host and cf_run_batch (host buffers and resident); every unit's status and length are
written exactly once at batch sizes around the CTA width; per-unit stage sets; and units at the key's edges (all keys equal,
saturated keys, empty and 1-byte units, units shorter than the key's window, a 64 KiB unit, a prose head before a nested tail)."""
import functools
import json
import random
import re

import numpy as np
import pytest
import torch

import bench
from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import toon_ref

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
SUBS = [("crap", 0, "crud")]
SENTINEL = 0x5A5A5A5A


def nested(depth: int, seed: int) -> str:
    rng = random.Random(seed)
    v = {"leaf": rng.randrange(1000), "s": "x" * rng.randrange(5)}
    for d in range(depth):
        v = {f"k{d}": v, "n": d, "a": [d, {"b": d}]}
    return json.dumps(v, separators=(",", ":"))


def edge_units() -> list:
    cfg = json.loads(synth.payload("B", 6000, seed=9))
    return [
        "", "x", "{", "[", "{}", "[]", "1", '{"a":1}', '[{"a":1},{"a":2}]', '[{"a":1}, {"a":2}]',
        "[" * 300 + "]" * 300,                                      # saturates the key, deeper than the encoder's stack
        "[" * 40 + "1" + "]" * 40,
        "[" + ",".join(["[]"] * 1500) + "]",                         # bracket-dense, key clamped
        nested(30, 1), nested(60, 2),
        synth.payload("B", 65536, seed=4), synth.payload("A", 65536, seed=4),   # 64 KiB units
        synth.payload("A", 600, seed=5), synth.payload("B", 700, seed=5),       # shorter than the key's window
        json.dumps({"doc": synth.payload("C", 3000, seed=6, hit_rate=0.0), "cfg": cfg}, separators=(",", ":")),   # prose head, nested tail
        '{"note": "total crap", "n": 5}',
    ]


@functools.lru_cache(maxsize=1)
def corpus() -> list:
    return bench.make_payloads() + edge_units()


def weight(t: str) -> int:
    return t.count("{") + t.count("[")


def packings(units):
    n = len(units)
    return {"natural": list(range(n)), "reversed": list(range(n))[::-1],
            "sorted": sorted(range(n), key=lambda i: -weight(units[i]))}


def toon_host(units):
    ctx = engine.Context.get()
    stream, offs = engine.pack_units(units)
    status, texts = engine.toon_host(engine.Batch(ctx, len(stream), len(units)), stream, offs)
    return [(int(s), t) for s, t in zip(status, texts)]


def run_batch(prog, units, unit_stages=None, stage_mask=N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON):
    """per unit (flags, out_len, aux, bytes) from a host-buffer call, then from a resident one on the same batch"""
    ctx = engine.Context.get()
    stream, offs = engine.pack_units([engine.encode_unit(u) for u in units])
    batch = engine.Batch(ctx, len(stream), len(units))
    res = []
    for resident in (False, True):
        v, out, oo, _ = engine.run_batch(prog, batch, None if resident else stream, offs, stage_mask, unit_stages=unit_stages, outputs_resident=resident)
        if resident:
            out = engine.device_output(ctx)
        res.append([(int(v["flags"][i]), int(v["out_len"][i]), int(v["aux"][i]), out[int(oo[i]):int(oo[i + 1])].tobytes()) for i in range(len(units))])
    return res


@pytest.fixture(scope="module")
def prog():
    p = engine.Program()
    for pat, f in HARMFUL:
        p.add_search(pat, f)
    for pat, f, r in SUBS:
        p.add_sub(pat, f, r)
    return p.compile(engine.Context.get())


def unpermute(res, perm):
    out = [None] * len(perm)
    for k, i in enumerate(perm):
        out[i] = res[k]
    return out


def test_order_independent_toon_host():
    units = corpus()
    got = {name: unpermute(toon_host([units[i] for i in perm]), perm) for name, perm in packings(units).items()}
    assert got["natural"] == got["reversed"] == got["sorted"]
    assert sum(1 for s, _ in got["natural"] if s == engine.TOON_CONVERTED) > len(units) // 2
    rng = random.Random(3)
    for i in rng.sample(range(len(units) - len(edge_units())), 24) + list(range(len(units) - len(edge_units()), len(units))):
        s, t = got["natural"][i]
        assert (t.decode() if s == engine.TOON_CONVERTED else None) == toon_ref.process_text(units[i], 0, 1 << 30), i


def test_order_independent_run_batch(prog):
    units = corpus()
    got = {name: [unpermute(r, perm) for r in run_batch(prog, [units[i] for i in perm])] for name, perm in packings(units).items()}
    for name in ("natural", "reversed", "sorted"):
        host, resident = got[name]
        assert host == resident, name
        assert host == got["natural"][0], name
    flags = [f for f, _, _, _ in got["natural"][0]]
    assert any(f & N.CF_V_TOON for f in flags) and any(f & N.CF_V_REWRITTEN for f in flags)
    for i in range(len(units) - len(edge_units()), len(units)):
        f, _, _, b = got["natural"][0][i]
        if not f & N.CF_V_REWRITTEN:
            assert (b.decode() if f & N.CF_V_TOON else None) == toon_ref.process_text(units[i], 0, 1 << 30), i


def test_equal_keys_and_saturated_keys():
    tab = [synth.payload("A", 3000 + 37 * s, seed=s) for s in range(64)]                 # every key equal
    dense = ["[" * (20 + s) + "]" * (20 + s) for s in range(40)] + [nested(25 + s, s) for s in range(24)]   # keys at the clamp
    for units in (tab, dense, tab + dense):
        got = {name: unpermute(toon_host([units[i] for i in perm]), perm) for name, perm in packings(units).items()}
        assert got["natural"] == got["reversed"] == got["sorted"]
        for i in range(0, len(units), 7):
            s, t = got["natural"][i]
            assert (t.decode() if s == engine.TOON_CONVERTED else None) == toon_ref.process_text(units[i], 0, 1 << 30), i


@pytest.mark.parametrize("n", [1, 7, 8, 9, 2111, 2113, 32771])
def test_every_unit_written_once(n):
    pool = [synth.payload("A", 300, seed=1), synth.payload("B", 400, seed=2), synth.payload("C", 250, seed=3, hit_rate=0.0), "", "x", "[]",
            "[" * 80 + "]" * 80, nested(12, 4), '{"a":[1,2,{"b":3}]}']
    rng = random.Random(n)
    units = [pool[rng.randrange(len(pool))] for _ in range(n)]
    ctx = engine.Context.get()
    stream, offs = engine.pack_units(units)
    batch = engine.Batch(ctx, len(stream), n)
    batch.upload(stream, offs)
    d_out = torch.empty(len(stream) + 16, dtype=torch.uint8, device="cuda")
    d_len = torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
    d_st = torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
    ctx.check(ctx.lib.cf_toon(ctx.h, batch.h, 0, d_out.data_ptr(), d_len.data_ptr(), d_st.data_ptr(), None), "cf_toon")
    torch.cuda.synchronize()
    st, ln = d_st.cpu().numpy(), d_len.cpu().numpy()
    assert not (st == SENTINEL).any() and not (ln == SENTINEL).any()
    expect = {p: toon_ref.process_text(p, 0, 1 << 30) for p in pool}
    out = d_out.cpu().numpy()
    for i in range(0, n, max(1, n // 300)):
        o = int(offs[i])
        got = out[o:o + int(ln[i])].tobytes().decode() if st[i] == engine.TOON_CONVERTED else None
        assert got == expect[units[i]], i


def test_per_unit_stages(prog):
    units = corpus()
    rng = random.Random(11)
    toon_half = np.array([rng.random() < 0.5 for _ in units])
    stages = np.where(toon_half, N.CF_STAGE_SCAN | N.CF_STAGE_TOON, N.CF_STAGE_SCAN).astype(np.uint8)
    mask = N.CF_STAGE_SCAN | N.CF_STAGE_TOON
    all_toon = run_batch(prog, units, stage_mask=mask)[0]
    for res in run_batch(prog, units, unit_stages=stages, stage_mask=mask):
        for i, r in enumerate(res):
            if toon_half[i]:
                assert r == all_toon[i], i
            else:
                assert r[2] == engine.TOON_SKIPPED and not r[0] & N.CF_V_TOON and r[1] == 0, i


def test_sequential_encoder_refuses_per_unit_stages(prog):
    """CF_TOON_SEQUENTIAL reaches the run, whose sequential encoder takes no per-unit stage masks: cf_run_batch refuses the pair
    before anything is queued, and the same batch then runs as before."""
    units = corpus()
    stream, offs = engine.pack_units([engine.encode_unit(u) for u in units])
    batch = engine.Batch(engine.Context.get(), len(stream), len(units))
    stages = np.full(len(units), N.CF_STAGE_SCAN | N.CF_STAGE_TOON, dtype=np.uint8)
    with pytest.raises(N.CfError) as err:
        engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_TOON, unit_stages=stages, toon_flags=N.CF_TOON_SEQUENTIAL)
    assert err.value.code == N.CF_E_BADARG
    v, _, _, _ = engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_TOON,
                                  toon_flags=N.CF_TOON_SEQUENTIAL | N.CF_TOON_REPORT_ERRORS)
    assert [int(a) for a in v["aux"]] == [s for s, _ in toon_host(units)]
