"""The device-resident entry points (cf_scan, cf_toon, cf_run_enqueue, cf_json_index, cf_run_batch with the batch or the outputs
left in HBM), one long-lived Batch that takes uploads of very different sizes one after the other (what the product's
batchers do), and the host-side cache of a batch's unit lengths in cf_sub_host across a freed and re-allocated batch.
Everything is checked against the oracles and against the host-buffer entry points on a fresh batch."""
import ctypes
import gc
import json
import re
import weakref

import numpy as np
import pytest

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import mask_ref, toon_ref

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
DENY = ["innovative", "groundbreaking", "revolutionary"]
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes")]
RULES = ref.regex_compile_rules([{"search": s, "replace": r} for s, _, r in SUBS])
MORE = ["zq%03d" % i for i in range(80)]          # W = 2 bitmap words


def program(extra=()):
    p = engine.Program()
    for pat, f in HARMFUL:
        p.add_search(pat, f)
    for w in DENY + list(extra):
        p.add_literal(w)
    for pat, f, r in SUBS:
        p.add_sub(pat, f, r)
    return p.compile(engine.Context.get())


def oracle_bits(units, extra=()):
    return ref.scan_bitmaps(units, HARMFUL, DENY + list(extra), [(p, f) for p, f, _ in SUBS])


def toon_oracle(u):
    return toon_ref.process_text(u, 0, 1 << 30)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def wave():
    """Tool results of one wave: TOON-convertible JSON, plain texts with hits, rewritten units (one inside JSON), a rewrite
    larger than 64 KiB, an empty unit."""
    units = [synth.payload("A", 3000, seed=s) for s in range(6)] + [synth.payload("B", 2000, seed=s) for s in range(2)]
    units += ["this is crap", "Kill him now", "zq042 and zq079", json.dumps({"rows": [{"id": i, "t": "crap"} for i in range(20)]}),
              "crap " * 20000, "", "innovative crud", synth.payload("C", 5000, seed=3, hit_rate=1e-3)]
    units += [synth.payload("A", 1500, seed=s + 10) for s in range(6)]
    return units


# ---------------------------------------------------------------------------------------------------------------------
# device-resident entry points
# ---------------------------------------------------------------------------------------------------------------------
def test_cf_scan_into_torch_bitmaps_matches_host_scan():
    import torch

    ctx = engine.Context.get()
    prog = program(MORE)
    units = wave()
    stream, offs = engine.pack_units(units)
    n, W = len(units), prog.words
    assert W == 2
    batch = engine.Batch(ctx, len(stream), n)
    host = engine.scan_host(prog, batch, stream, offs)
    dev = torch.full((n * W,), -1, dtype=torch.int64, device="cuda")
    batch2 = engine.Batch(ctx, len(stream), n)
    batch2.upload(stream, offs)
    with ctx.lock:
        ctx.check(ctx.lib.cf_scan(ctx.h, prog.h, batch2.h, ptr(dev), None), "cf_scan")
    torch.cuda.synchronize()
    got = dev.cpu().numpy().view(np.uint64)
    assert np.array_equal(got, host)
    assert engine.bitmaps_to_ints(got, n, W) == oracle_bits(units, MORE)


def _toon_buffers(nbytes, n):
    import torch

    return (torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda"), torch.full((n,), 0x7777, dtype=torch.int32, device="cuda"),
            torch.full((n,), -1, dtype=torch.int32, device="cuda"))


def _toon_texts(out, out_len, status, offs):
    o, ln, st = out.cpu().numpy(), out_len.cpu().numpy().view(np.uint32), status.cpu().numpy()
    return st, [o[int(offs[i]):int(offs[i]) + int(ln[i])].tobytes().decode() if st[i] == engine.TOON_CONVERTED else None for i in range(len(st))]


def test_cf_toon_and_run_enqueue_device_resident():
    import torch

    ctx = engine.Context.get()
    prog = program(MORE)
    units = wave()
    stream, offs = engine.pack_units(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    batch.upload(stream, offs)
    out, out_len, status = _toon_buffers(len(stream), n)
    with ctx.lock:
        ctx.check(ctx.lib.cf_toon(ctx.h, batch.h, 1, ptr(out), ptr(out_len), ptr(status), None), "cf_toon")
    torch.cuda.synchronize()
    st, texts = _toon_texts(out, out_len, status, offs)
    assert texts == [toon_oracle(u) for u in units]
    assert (st == engine.TOON_CONVERTED).sum() >= 8
    # cf_run_enqueue: scan + TOON on the resident batch; units whose stage mask leaves out TOON come back SKIPPED
    stages = np.array([N.CF_STAGE_SCAN | (N.CF_STAGE_TOON if i % 3 else 0) for i in range(n)], dtype=np.uint8)
    d_stages = torch.from_numpy(stages).cuda()
    bm = torch.full((n * prog.words,), -1, dtype=torch.int64, device="cuda")
    v = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
    oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    out = torch.zeros(len(stream), dtype=torch.uint8, device="cuda")
    run = engine.Run(ctx, n, len(stream))
    run.enqueue(prog, batch, N.CF_STAGE_SCAN | N.CF_STAGE_TOON, d_stages, 1, v, oo, out, bm)
    assert run.finish() == 0
    v, oo, out = v.cpu().numpy().view(engine.VERDICT_DTYPE), oo.cpu().numpy(), out.cpu().numpy()
    assert engine.bitmaps_to_ints(bm.cpu().numpy().view(np.uint64), n, prog.words) == oracle_bits(units, MORE)
    for i, u in enumerate(units):
        if stages[i] & N.CF_STAGE_TOON:
            assert (out[oo[i]:oo[i + 1]].tobytes().decode() if v["flags"][i] & N.CF_V_TOON else None) == toon_oracle(u), i
        else:
            assert v["aux"][i] == engine.TOON_SKIPPED, i


def test_cf_json_index_device_resident_matches_host_entry_point():
    import torch

    ctx = engine.Context.get()
    docs = [synth.payload("A", 3000, seed=1), synth.payload("B", 2000, seed=2), "", "[1, 2", '"abc', '{"a": "x\\"y", "b": [true, null]}', " 7 "]
    stream, offs = engine.pack_units(docs)
    n = len(docs)
    host = engine.json_index_host(engine.Batch(ctx, len(stream), n), stream, offs, classify=True)
    batch = engine.Batch(ctx, len(stream), n)
    batch.upload(stream, offs)
    toks = torch.zeros((len(stream) + 64) * 2, dtype=torch.int32, device="cuda")
    counts = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    with ctx.lock:
        ctx.check(ctx.lib.cf_json_index(ctx.h, batch.h, 1, ptr(toks), ptr(counts), None), "cf_json_index")
    torch.cuda.synchronize()
    t = toks.cpu().numpy().view(np.uint32).reshape(-1, 2)
    c = counts.cpu().numpy().view(np.uint32)
    for i in range(n):
        k = int(c[i]) & 0x7FFFFFFF
        assert np.array_equal(t[int(offs[i]):int(offs[i]) + k], host[i][0]), i
        assert bool(int(c[i]) >> 31) == host[i][1], i
        assert [int(p) & 0x7FFFFFFF for p, _ in host[i][0]] == plain_index(docs[i].encode())


def plain_index(doc):
    """Token positions of the structural index, by a plain byte walk (the scanner of __graft_entry__.smoke)."""
    expect, in_str, prev_other, run = [], False, False, 0
    for i, c in enumerate(doc):
        real_quote = c == 0x22 and run % 2 == 0
        run = run + 1 if c == 0x5C else 0
        if in_str:
            if real_quote:
                expect.append(i)
                in_str = False
            prev_other = False
        elif real_quote:
            expect.append(i)
            in_str, prev_other = True, False
        elif c in b"{}[]:,":
            expect.append(i)
            prev_other = False
        elif c in b" \t\n\r":
            prev_other = False
        else:
            if not prev_other:
                expect.append(i)
            prev_other = True
    return expect


# ---------------------------------------------------------------------------------------------------------------------
# cf_run_batch: host buffers, resident batch, resident outputs, exact capacity
# ---------------------------------------------------------------------------------------------------------------------
STAGES = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON


def _check_wave_against_oracles(units, v, out, oo, full, W):
    assert engine.bitmaps_to_ints(full, len(units), W) == oracle_bits(units, MORE)
    for i, u in enumerate(units):
        txt = out[int(oo[i]):int(oo[i + 1])].tobytes().decode()
        if v["flags"][i] & N.CF_V_REWRITTEN:
            assert txt == ref.regex_apply_str(RULES, u), i
        else:
            assert (txt if v["flags"][i] & N.CF_V_TOON else None) == toon_oracle(u), i
    rewritten = [i for i in range(len(units)) if v["flags"][i] & N.CF_V_REWRITTEN]
    assert rewritten == [i for i, u in enumerate(units) if RULES[0][0].search(u) or RULES[1][0].search(u)]
    assert max(int(oo[i + 1] - oo[i]) for i in rewritten) > (1 << 16)          # took the CF_E_CAPACITY retry of cf_sub_host
    assert any(v["flags"][i] & N.CF_V_TOON for i in range(len(units)))


def test_run_batch_resident_paths_equal_the_host_buffer_call():
    ctx = engine.Context.get()
    prog = program(MORE)
    units = wave()
    stream, offs = engine.pack_units(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    v0, out0, oo0, full0 = engine.run_batch(prog, batch, stream, offs, STAGES, want_full_bitmaps=True)
    out0 = out0[:int(oo0[-1])].copy()
    _check_wave_against_oracles(units, v0, out0, oo0, full0, prog.words)
    # the batch already on the device (stream = NULL)
    v1, out1, oo1, full1 = engine.run_batch(prog, batch, None, offs, STAGES, want_full_bitmaps=True)
    assert v1.tobytes() == v0.tobytes() and np.array_equal(oo1, oo0) and np.array_equal(full1, full0)
    assert out1[:int(oo1[-1])].tobytes() == out0.tobytes()
    # outputs left in HBM, with and without a fresh upload
    for sp in (stream, None):
        v2, none, oo2, full2 = engine.run_batch(prog, batch, sp, offs, STAGES, want_full_bitmaps=True, outputs_resident=True)
        assert none is None
        assert v2.tobytes() == v0.tobytes() and np.array_equal(oo2, oo0) and np.array_equal(full2, full0)
        assert engine.device_output(ctx).tobytes() == out0.tobytes()


def test_run_batch_output_capacity_is_exact():
    ctx = engine.Context.get()
    prog = program(MORE)
    units = wave()
    stream, offs = engine.pack_units(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    v0, out0, oo0, _ = engine.run_batch(prog, batch, stream, offs, STAGES)
    need = int(oo0[-1])
    ref_bytes = out0[:need].tobytes()
    for cap, want_rc in ((need - 1, N.CF_E_CAPACITY), (need, N.CF_OK)):
        v = np.zeros(n, dtype=engine.VERDICT_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        buf = np.full(need + 64, 0xAB, dtype=np.uint8)
        got_need = ctypes.c_uint64(0)
        with ctx.lock:
            rc = ctx.lib.cf_run_batch(ctx.h, prog.h, batch.h, ctypes.cast(ctypes.c_char_p(stream), ctypes.c_void_p), len(stream), offs.ctypes.data, n, STAGES,
                                      None, 0, 10, v.ctypes.data, None, buf.ctypes.data, cap, oo.ctypes.data, ctypes.byref(got_need))
        assert rc == want_rc, (cap, rc)
        assert got_need.value == need
        if rc == N.CF_OK:
            assert buf[:need].tobytes() == ref_bytes and v.tobytes() == v0.tobytes()
            assert (buf[need:] == 0xAB).all()                           # nothing written past out_cap


# ---------------------------------------------------------------------------------------------------------------------
# one Batch, uploads of very different sizes
# ---------------------------------------------------------------------------------------------------------------------
def _all_results(prog, batch, units):
    stream, offs = engine.pack_units(units)
    bits = engine.bitmaps_to_ints(engine.scan_host(prog, batch, stream, offs), len(units), prog.words)
    dirty = [i for i, b in enumerate(bits) if b >> (len(HARMFUL) + len(DENY))]
    subs = engine.sub_host(prog, batch, dirty)
    toon = engine.toon_host(batch, stream, offs)
    masks = {md: engine.mask_host(batch, stream, offs, md) for md in (10, 3)}
    index = engine.json_index_host(batch, stream, offs, classify=True)
    return bits, dirty, subs, toon, masks, index


def _diff(a, b):
    """Indices where two equally long result lists differ (a short assertion message on failure)."""
    assert len(a) == len(b)
    return [i for i, (x, y) in enumerate(zip(a, b)) if not (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y)][:5]


def _same(a, b):
    bits_a, dirty_a, subs_a, (ts_a, tt_a), masks_a, idx_a = a
    bits_b, dirty_b, subs_b, (ts_b, tt_b), masks_b, idx_b = b
    assert not _diff(bits_a, bits_b) and dirty_a == dirty_b and not _diff(subs_a, subs_b)
    assert np.array_equal(ts_a, ts_b) and not _diff(tt_a, tt_b)
    for md in masks_a:
        assert np.array_equal(masks_a[md][0], masks_b[md][0]) and not _diff(masks_a[md][1], masks_b[md][1])
    assert not _diff([t for t, _ in idx_a], [t for t, _ in idx_b]) and [u for _, u in idx_a] == [u for _, u in idx_b]


def _against_oracles(units, res):
    bits, dirty, subs, (ts, tt), masks, index = res
    assert not _diff(bits, oracle_bits(units))
    assert not _diff([s.decode() for s in subs], [ref.regex_apply_str(RULES, units[i]) for i in dirty])
    assert not _diff([t.decode() if t is not None else None for t in tt], [toon_oracle(u) for u in units])
    for md, (_, outs) in masks.items():
        exp = []
        for u in units:
            try:
                exp.append(mask_ref.mask_json_bytes(u.encode(), md))
            except ValueError:
                exp.append(None)
        assert not _diff(outs, exp), md
    assert not _diff([[int(p) & 0x7FFFFFFF for p, _ in t] for t, _ in index], [plain_index(u.encode()) for u in units])


def test_one_batch_takes_large_then_small_then_one_byte_uploads():
    ctx = engine.Context.get()
    prog = program()
    # the first 64 KiB of the large upload are dense with hits (and the JSON after them has some too): after a smaller upload
    # they are the bytes right behind its end, inside its last scan tile, where the tail re-arm must have put 0xFF again
    dense = "Kill him now, I want to die; this is crap. suicide innovative crud " * 1000
    large = [dense, json.dumps({"token": "t", "rows": [{"a": i, "b": "kill him", "c": "crap"} for i in range(300)]})]
    large += [synth.payload("A", 2000, seed=s) for s in range(300)] + [synth.payload("C", 4000, seed=s, hit_rate=2e-3) for s in range(40)]
    # hits and JSON in the very last bytes of the large upload too
    large += ["x " * 3000 + "this is crap and I want to die", json.dumps({"password": "p", "rows": [{"a": i, "b": "suicide"} for i in range(50)]})]
    small = ["crap", '{"a": 1, "token": "t"}', "Kill him", "[1, 2, 3]" + " " * 40, ""]
    tiny = ["1"]
    total = len(engine.pack_units(large)[0])
    shared = engine.Batch(ctx, total, len(large))
    for units in (large, small, tiny, large, tiny):
        got = _all_results(prog, shared, units)
        stream, _ = engine.pack_units(units)
        fresh = _all_results(prog, engine.Batch(ctx, len(stream), len(units)), units)
        _same(got, fresh)
        _against_oracles(units, got)


# ---------------------------------------------------------------------------------------------------------------------
# cf_sub_host's cache of unit lengths after a batch is freed and another one takes its place
# ---------------------------------------------------------------------------------------------------------------------
def test_sub_sizing_follows_a_new_batch_at_a_freed_batch_address():
    """cf_sub_host keeps the host copy of a batch's offsets to size each unit's scratch.  A batch freed and re-created at the
    same address, after as many uploads and with as many units, must not reuse the old batch's unit lengths."""
    ctx = engine.Context.get()
    p = engine.Program()
    p.add_sub("a", 0, "bb")
    p.add_sub("b", 0, "cc")
    p.compile(ctx)
    rules = ref.regex_compile_rules([{"search": "a", "replace": "bb"}, {"search": "b", "replace": "cc"}])
    # grow the substitution scratch first: a wrongly sized unit could then only land inside the allocation (wrong output).
    # `bb` stays alive to the end, so that the batches below cannot take its place: the only lengths a stale cache entry
    # could then hold are b1's short ones.
    big = ["a" * 200000, "b" * 200000]
    s, o = engine.pack_units(big)
    bb = engine.Batch(ctx, len(s), 2)
    bb.upload(s, o)
    assert [x.decode() for x in engine.sub_host(p, bb, [0, 1])] == [ref.regex_apply_str(rules, u) for u in big]
    first = ["a", "xa"]
    s, o = engine.pack_units(first)
    b1 = engine.Batch(ctx, 4096, 2)
    assert b1.h.value != bb.h.value
    b1.upload(s, o)
    assert [x.decode() for x in engine.sub_host(p, b1, [0, 1])] == [ref.regex_apply_str(rules, u) for u in first]
    addr = b1.h.value
    del b1
    keep = []
    for _ in range(8):
        b2 = engine.Batch(ctx, 1 << 16, 2)
        if b2.h.value == addr:
            break
        keep.append(b2)
    assert b2.h.value == addr, "no new batch took the freed batch's place"
    # as many uploads and units as b1 had, but a unit 1500 times longer: sized from b1's lengths, the chained rewrite of
    # that unit would run over its two scratch buffers and come back wrong
    second = ["a", "a" * 3000]
    s, o = engine.pack_units(second)
    b2.upload(s, o)
    assert [x.decode() for x in engine.sub_host(p, b2, [0, 1])] == [ref.regex_apply_str(rules, u) for u in second]
    del bb


def test_run_batch_texts_outlive_their_batch():
    """The texts run_batch returns are a view of the Batch's page-locked output buffer.  The view keeps that buffer alive: the texts
    of a Batch that was dropped right after the call (a temporary argument) read back whole, and the buffer is freed with the last view."""
    ctx = engine.Context.get()
    texts = [synth.payload("A", 2048, seed=s) for s in range(16)] + [synth.payload("B", 2048, seed=s) for s in range(4)]
    stream, offs = engine.pack_units(texts)
    batch = engine.Batch(ctx, len(stream), len(texts))
    v, out, oo, _ = engine.run_batch(None, batch, stream, offs, N.CF_STAGE_TOON)
    pin = weakref.ref(batch._out_pin)
    del batch
    gc.collect()
    assert pin() is not None
    got = [out[int(oo[i]):int(oo[i + 1])].tobytes().decode() if v["aux"][i] == engine.TOON_CONVERTED else None for i in range(len(texts))]
    assert got == [toon_ref.process_text(t, 0, 1 << 30) for t in texts]
    assert any(got)
    del out
    gc.collect()
    assert pin() is None
