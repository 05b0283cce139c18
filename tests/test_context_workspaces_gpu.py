"""One context, every entry point that takes device workspace from it, in one sequence whose batches grow, shrink and then grow past
the headroom of the context's run: cf_run_batch (SCAN|SUB; SCAN|SUB|TOON with host buffers and with the outputs left in HBM;
SCAN|MASK with bodies that outgrow the mask's first room), cf_toon on a torch stream, cf_toon_host on the default, sequential and
parse-only routes, cf_sub_host with a rewrite that outgrows its first scratch bound, cf_scan_host, cf_json_index_host and
cf_classify_keys_host.  Every result is checked against the oracles, and the device buffer a CF_RUN_OUTPUTS_RESIDENT call leaves
behind must keep its bytes through the calls include/cfgpu.h says do not gather into it."""
import ctypes
import json
import re

import numpy as np
import pytest

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import mask_ref, toon_ref
from test_resident_and_reuse_gpu import plain_index

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
DENY = ["innovative", "groundbreaking", "revolutionary"]
# "~" -> 200 bytes: a unit of 1000 of them rewrites to 200 000 bytes, more than its first scratch bound of 64 L + 64 KiB
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes"), ("~", 0, "-" * 200)]
RULES = ref.regex_compile_rules([{"search": s, "replace": r} for s, _, r in SUBS])
REPORT_ERRORS, PARSE_ONLY, SEQUENTIAL = 1, 4, 8
SENSITIVE_KEYS = ["password", "authToken", "token_count", "X-Api-Key", "name", "secret_name", "client_secret", "port"]


def wave(k, seed):
    """k tool results of each payload shape, then rewritten units (one over 64 KiB, one past its first scratch bound, one inside
    JSON), a hit, an empty unit and two bodies whose masked output at max_depth 2 outgrows 5 len + 32 bytes."""
    units = [synth.payload("A", 2000 + 400 * (i % 5), seed=seed + i) for i in range(k)]
    units += [synth.payload("B", 1500, seed=seed + i) for i in range(k)]
    units += [synth.payload("C", 3000, seed=seed + i, hit_rate=2e-3) for i in range(k)]
    units += ["this is crap", "Kill him now", "crap " * 20000, "~" * 1000, json.dumps({"rows": [{"id": i, "t": "crap"} for i in range(20)]}), ""]
    units += ['{"k":[' + ",".join(["[]"] * m) + "]}" for m in (40, 400)]
    return units


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def toon_oracle(u):
    return toon_ref.process_text(u, 0, 1 << 30)


def mask_oracle(u, max_depth):
    try:
        return mask_ref.mask_json_bytes(u.encode(), max_depth)
    except ValueError:
        return None


def oracle_bits(units):
    return ref.scan_bitmaps(units, HARMFUL, DENY, [(p, f) for p, f, _ in SUBS])


def resident_output(ctx):
    p, nb = ctypes.c_void_p(), ctypes.c_uint64(0)
    ctx.check(ctx.lib.cf_run_batch_device_output(ctx.h, ctypes.byref(p), ctypes.byref(nb)), "cf_run_batch_device_output")
    return p.value, nb.value


def read_device(ctx, p, nbytes):
    out = np.empty(nbytes, dtype=np.uint8)
    ctx.check(ctx.lib.cf_copy_to_host(ctx.h, out.ctypes.data, p, nbytes), "cf_copy_to_host")
    return out.tobytes()


def check_chain(units, v, out, oo, full, toon):
    assert engine.bitmaps_to_ints(full, len(units), 1) == oracle_bits(units)
    for i, u in enumerate(units):
        txt = out[int(oo[i]):int(oo[i + 1])].tobytes().decode()
        if v["flags"][i] & N.CF_V_REWRITTEN:
            assert txt == ref.regex_apply_str(RULES, u), i
        elif toon:
            assert (txt if v["flags"][i] & N.CF_V_TOON else None) == toon_oracle(u), i
        else:
            assert txt == "", i
    assert [i for i in range(len(units)) if v["flags"][i] & N.CF_V_REWRITTEN] == [i for i, u in enumerate(units) if any(r.search(u) for r, _ in RULES)]
    assert max(int(oo[i + 1] - oo[i]) for i in range(len(units))) > 1 << 16


def is_json(u):
    try:
        json.loads(u)
        return True
    except ValueError:
        return False


def run_sequence(ctx, prog, units):
    import torch

    stream, offs = engine.pack_units(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    # cf_run_batch SCAN|SUB: rewrites only, a deferred unit finished by cf_run_finish among them
    v, out, oo, full = engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_SUB, want_full_bitmaps=True)
    check_chain(units, v, out, oo, full, toon=False)
    # SCAN|SUB|TOON with host buffers, then with the texts left in HBM
    chain = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
    v, out, oo, full = engine.run_batch(prog, batch, stream, offs, chain, want_full_bitmaps=True)
    check_chain(units, v, out, oo, full, toon=True)
    texts = out[:int(oo[-1])].tobytes()
    v2, _, oo2, _ = engine.run_batch(prog, batch, stream, offs, chain, outputs_resident=True)
    assert v2.tobytes() == v.tobytes() and np.array_equal(oo2, oo)
    assert engine.device_output(ctx).tobytes() == texts
    resident = resident_output(ctx)
    # cf_toon on a torch stream, into tensors allocated on the current stream
    s = torch.cuda.Stream()
    d_out = torch.zeros(len(stream), dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    batch.upload(stream, offs, cuda_stream=s.cuda_stream)
    with ctx.lock:
        ctx.check(ctx.lib.cf_toon(ctx.h, batch.h, REPORT_ERRORS, ptr(d_out), ptr(d_len), ptr(d_st), ctypes.c_void_p(s.cuda_stream)), "cf_toon")
    s.synchronize()
    o, ln, st = d_out.cpu().numpy(), d_len.cpu().numpy(), d_st.cpu().numpy()
    exp_toon = [toon_oracle(u) for u in units]
    assert [o[int(offs[i]):int(offs[i]) + int(ln[i])].tobytes().decode() if st[i] == engine.TOON_CONVERTED else None for i in range(n)] == exp_toon
    assert sum(t is not None for t in exp_toon) >= 3
    # cf_sub_host: the "~" unit outgrows its first bound (the regrowth loop) and engine.sub_host's first 64 KiB of output
    dirty = [i for i, u in enumerate(units) if any(r.search(u) for r, _ in RULES)]
    subs = engine.sub_host(prog, batch, dirty)
    assert [x.decode() for x in subs] == [ref.regex_apply_str(RULES, units[i]) for i in dirty]
    assert max(len(x) for x in subs) > 64 * 1000 + (1 << 16)
    # cf_scan_host, cf_json_index_host, cf_classify_keys_host
    assert engine.bitmaps_to_ints(engine.scan_host(prog, batch, stream, offs), n, 1) == oracle_bits(units)
    index = engine.json_index_host(batch, stream, offs)
    assert [[int(p) & 0x7FFFFFFF for p, _ in t] for t, _ in index] == [plain_index(u.encode()) for u in units]
    assert engine.classify_keys_host(batch, SENSITIVE_KEYS) == [mask_ref.is_sensitive_key(k) for k in SENSITIVE_KEYS]
    # none of these gathers into the resident output buffer
    assert resident_output(ctx) == resident and read_device(ctx, *resident) == texts
    # cf_toon_host on every route
    for flags in (REPORT_ERRORS, SEQUENTIAL | REPORT_ERRORS):
        _, got, _ = engine.toon_host_flags(batch, stream, offs, flags)
        assert [None if t is None else t.decode() for t in got] == exp_toon, flags
    status, _, _ = engine.toon_host_flags(batch, stream, offs, PARSE_ONLY)
    assert [int(x) for x in status] == [0 if is_json(u) else 1 for u in units]
    # SCAN|MASK at two depths: the masking workspace is reused, and at depth 2 the last two bodies outgrow their first room
    for md in (10, 2):
        v, out, oo, full = engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_MASK, mask_max_depth=md, want_full_bitmaps=True)
        assert engine.bitmaps_to_ints(full, n, 1) == oracle_bits(units)
        exp = [mask_oracle(u, md) for u in units]
        assert [out[int(oo[i]):int(oo[i + 1])].tobytes() if v["flags"][i] & N.CF_V_MASKED else None for i in range(n)] == exp, md
    assert all(len(exp[i]) > 5 * len(units[i]) + 32 for i in (n - 2, n - 1))


def test_one_context_grows_shrinks_and_grows_past_its_run():
    ctx = engine.Context(0)                      # a fresh context: its run and scratch start empty
    prog = engine.Program()
    for p, f in HARMFUL:
        prog.add_search(p, f)
    for w in DENY:
        prog.add_literal(w)
    for p, f, r in SUBS:
        prog.add_sub(p, f, r)
    prog.compile(ctx)
    assert prog.words == 1
    small, medium, large = wave(2, 100), wave(16, 0), wave(40, 200)
    assert len(large) > 1.25 * len(medium) and len(engine.pack_units(large)[0]) > 1.25 * len(engine.pack_units(medium)[0]) + 4096
    for units in (medium, small, large):
        run_sequence(ctx, prog, units)
