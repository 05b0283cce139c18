"""GPU: BASELINE configs[2] — the pattern scan and request_logging_masking on ONE upload, `cf_run_batch(CF_STAGE_SCAN | CF_STAGE_MASK)`
(include/cfgpu.h): bitmaps as the scan alone gives them, masked bodies as the oracle (lib.rs:276-360 restated) gives them, units that do
not parse flagged and left without an output.  (File name: runs last in the suite.)"""
import json
import re

import numpy as np
import pytest

from mcp_context_forge_b200 import engine, synth
from mcp_context_forge_b200._native import CF_STAGE_MASK, CF_STAGE_SCAN, CF_STAGE_SUB, CF_V_MASKED, CF_V_REWRITTEN
from oracle import hook_chain_ref as ref
from oracle import mask_ref

pytestmark = pytest.mark.gpu


def test_scan_and_masking_on_one_upload():
    ctx = engine.Context.get(0)
    prog = engine.Program()
    pats = [(p, re.I) for ps in ref.DEFAULT_LEXICONS.values() for p in ps]
    for p, f in pats:
        prog.add_search(p, f)
    prog.compile(ctx)
    bodies = [synth.payload("B", 16384, seed=s) for s in range(24)] + [synth.payload("A", 16384, seed=s) for s in range(8)]
    bodies += ['{"password":"secret","note":"I want to kill myself","nested":{"authToken":"abc","count":3}}', '{"a":1,}', "[01]", "", '{"level":{"nested":{}}}',
               '[0.30000000000000004,5e-324,1e23,-0]', '{"Cookie":"jwt_token=abc","text":"how to make a bomb \\u00e9"}', synth.payload("B", 262144, seed=3)]
    stream, offs = engine.pack_units(bodies)
    batch = engine.Batch(ctx, len(stream), len(bodies))
    for max_depth in (10, 2):
        v, out, oo, _ = engine.run_batch(prog, batch, np.frombuffer(stream, dtype=np.uint8), offs, CF_STAGE_SCAN | CF_STAGE_MASK, mask_max_depth=max_depth)
        exp_bm = ref.scan_bitmaps(bodies, pats, [], [])
        for i, b in enumerate(bodies):
            assert int(v["match_bitmap"][i]) == exp_bm[i], i
            try:
                exp = mask_ref.mask_json_bytes(b.encode(), max_depth)
            except ValueError:
                exp = None
            got = out[int(oo[i]):int(oo[i + 1])].tobytes() if v["flags"][i] & CF_V_MASKED else None
            assert got == exp, (i, max_depth)
            assert int(v["out_len"][i]) == (len(exp) if exp is not None else 0)
        assert int(oo[-1]) == sum(int(x) for x in v["out_len"])
    # the masking stage alone (no program) on the batch that is already resident: same outputs
    v, out, oo = v.copy(), out[: int(oo[-1])].copy(), oo.copy()          # (`out` is the batch's reusable buffer)
    v2, out2, oo2, _ = engine.run_batch(None, batch, None, offs, CF_STAGE_MASK, mask_max_depth=2)
    assert (v2["flags"] == (v["flags"] & CF_V_MASKED)).all() and (oo2 == oo).all() and (out2[: int(oo2[-1])] == out).all()


def test_scan_sub_and_masking_verdicts_match_the_oracles():
    """`cf_run_batch(SCAN | SUB | MASK)`: the substitution only decides the verdicts (rewritten texts are not returned in masking
    mode), the masked bodies are the output.  Per unit, from the oracles (CPython `re`, oracle/mask_ref.py): match_bitmap = word 0 of
    the bitmap; CF_V_REWRITTEN when a rule matches and the unit's stages allow SUB; CF_V_MASKED when the body masks; out_len = the
    masked length when masked, else the rewritten length when rewritten, else 0; aux = the CF_MASK_* status."""
    # A fresh context, so that its run's substitution arena starts at 1 MiB.  A dirty unit asks the arena for two buffers of
    # min(worst, 64 L + 64 KiB) bytes; "zqx" -> 4000 bytes grows a 16 KiB unit's worst case far beyond 64 L + 64 KiB, so each dirty
    # 16 KiB body asks for 2 x (64 x 16 KiB + 64 KiB) = 2.1 MiB > 1 MiB: the first call defers it to the synchronous substitution.
    ctx = engine.Context(0)
    searches = [(p, re.I) for ps in ref.DEFAULT_LEXICONS.values() for p in ps]
    literals = [f"wq{k:03d}v" for k in range(60)]                 # with the searches: the rules' bits sit in bitmap word 1
    subs = [("crap", 0, "crud"), ("crud", 0, "yikes"), ("zqx", 0, "Z" * 4000)]
    prog = engine.Program()
    for p, f in searches:
        prog.add_search(p, f)
    for w in literals:
        prog.add_literal(w)
    for p, f, r in subs:
        prog.add_sub(p, f, r)
    prog.compile(ctx)
    assert prog.words == 2
    rules = [(re.compile(p, f), r) for p, f, r in subs]
    big = lambda s, extra: json.dumps({"password": "hunter2", "note": extra, "data": synth.payload("A", 16384, seed=s)})   # noqa: E731
    bodies = [big(0, "zqx once")[:-1], big(1, "zqx, zqx and crap"), big(2, "no rule here"), big(3, "zqx but SUB is left out"),
              synth.payload("B", 3000, seed=1), json.dumps({"token": "crap", "x": [1, 2, {"apiKey": "crud"}]}), '{"a": "crap",}',
              json.dumps({"text": "I want to kill myself", "ids": ["wq007v", "wq059v"]}), "", '{"Cookie": "zqx=1"}', "[1, 2, 3]",
              json.dumps({"secret": "zqx", "list": list(range(50))})]
    stages = np.array([CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_MASK] * len(bodies), dtype=np.uint8)
    for i in (3, 5, 11):                                          # dirty units whose stages leave SUB out
        stages[i] = CF_STAGE_SCAN | CF_STAGE_MASK
    stream, offs = engine.pack_units(bodies)
    bits = ref.scan_bitmaps(bodies, searches, literals, [(p, f) for p, f, _ in subs])
    exp_v = []
    for i, b in enumerate(bodies):
        try:
            masked = mask_ref.mask_json_bytes(b.encode(), 10)
        except ValueError:
            masked = None
        dirty = bool(stages[i] & CF_STAGE_SUB) and any(c.search(b) for c, _ in rules)
        out_len = len(masked) if masked is not None else len(ref.regex_apply_str(rules, b).encode()) if dirty else 0
        flags = (CF_V_REWRITTEN if dirty else 0) | (CF_V_MASKED if masked is not None else 0)
        exp_v.append((bits[i] & ((1 << 64) - 1), flags, out_len, engine.MASK_OK if masked is not None else engine.MASK_PARSE_ERROR, 0, masked))
    assert sum(1 for e in exp_v if e[1] & CF_V_REWRITTEN) >= 4 and sum(1 for e in exp_v if e[1] == CF_V_REWRITTEN) >= 2   # rewritten, not masked
    batch = engine.Batch(ctx, len(stream), len(bodies))
    for host in (True, False):                                    # host buffers (the deferring call), then the resident batch
        v, out, oo, full = engine.run_batch(prog, batch, np.frombuffer(stream, dtype=np.uint8) if host else None, offs,
                                            CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_MASK, unit_stages=stages, mask_max_depth=10, want_full_bitmaps=True)
        assert engine.bitmaps_to_ints(full, len(bodies), prog.words) == bits
        for i, (bm, flags, out_len, aux, reserved, masked) in enumerate(exp_v):
            assert (int(v["match_bitmap"][i]), int(v["flags"][i]), int(v["out_len"][i]), int(v["aux"][i]), int(v["reserved"][i])) == \
                (bm, flags, out_len, aux, reserved), (i, host)
            assert out[int(oo[i]):int(oo[i + 1])].tobytes() == (masked if masked is not None else b""), (i, host)
        assert int(oo[-1]) == sum(len(e[5]) for e in exp_v if e[5] is not None)
