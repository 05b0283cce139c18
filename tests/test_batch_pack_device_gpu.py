"""cf_batch_pack_device (engine.Batch.pack_device): a batch built from texts already in device memory must be the batch
cf_batch_upload makes of the same units.  Every consumer of a batch is run on both and must give the same bytes: cf_scan (full
bitmaps), cf_toon, cf_json_index, and cf_run_enqueue with SCAN|SUB|TOON and with SCAN|MASK.  Also covered: re-submitting a run's
rewritten units to TOON on the device (CF_V_RESUBMIT) against the oracle and the host route, pack + enqueue captured in one CUDA
graph, and the refusals, which must leave nothing queued."""
import json
import random

import numpy as np
import pytest
import torch

import test_run_async_gpu as ra
from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import toon_ref

pytestmark = pytest.mark.gpu

FULL = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
SCAN_MASK = N.CF_STAGE_SCAN | N.CF_STAGE_MASK
INDEX_CLASSIFY = 1                                         # CF_INDEX_CLASSIFY


def enc(units):
    return [engine.encode_unit(u) for u in units]


def device_source(units, misalign=0):
    """The units back to back (no terminators) in a CUDA uint8 tensor, starting `misalign` bytes into it, and their int64 offsets."""
    e = enc(units)
    raw = b"\xee" * misalign + b"".join(e) + b"\xee" * 3
    src = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda() if raw else torch.zeros(1, dtype=torch.uint8, device="cuda")
    offs = np.zeros(len(e) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in e], out=offs[1:])
    return src, torch.from_numpy(offs + misalign).cuda(), int(offs[-1])


def stream():
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    return s


def consumers(ch, batch, n, nbytes, s):
    """Every consumer of the batch on stream s: scan bitmaps, TOON statuses and texts, structural index, and two runs."""
    ctx, L = batch.ctx, batch.ctx.lib
    W = ch.prog.words
    bm = torch.zeros(n * W, dtype=torch.int64, device="cuda")
    tout = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    tlen = torch.zeros(n, dtype=torch.int32, device="cuda")
    tst = torch.zeros(n, dtype=torch.int32, device="cuda")
    toks = torch.zeros(2 * max(nbytes, 1), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    with ctx.lock:
        ctx.check(L.cf_scan(ctx.h, ch.prog.h, batch.h, bm.data_ptr(), s.cuda_stream), "cf_scan")
        ctx.check(L.cf_toon(ctx.h, batch.h, 0, tout.data_ptr(), tlen.data_ptr(), tst.data_ptr(), s.cuda_stream), "cf_toon")
        ctx.check(L.cf_json_index(ctx.h, batch.h, INDEX_CLASSIFY, toks.data_ptr(), cnt.data_ptr(), s.cuda_stream), "cf_json_index")
    s.synchronize()
    res = {"bitmaps": bm.cpu().numpy().tobytes(), "toon_status": tst.cpu().numpy().tolist(), "runs": {}}
    tl, tb, cn, tk = tlen.cpu().numpy(), tout.cpu().numpy(), cnt.cpu().numpy(), toks.cpu().numpy().reshape(-1, 2)
    for mask in (FULL, SCAN_MASK):
        run = engine.Run(ctx, n, nbytes)
        bufs = ra.Bufs(n, W, 6 * nbytes + 4096)
        run.enqueue(ch.prog, batch, mask, None, 0, bufs.v, bufs.oo, bufs.out, bufs.bm, stream=s)
        assert run.finish() == 0
        v, texts, rbm, oo = bufs.results()
        res["runs"][mask] = (v.tobytes(), texts, rbm.tobytes(), oo.tobytes())
    res["toon_raw"] = (tl.tobytes(), tst.cpu().numpy().tobytes())
    res["_tb"], res["_cnt"], res["_tk"] = tb, cn, tk
    return res


def texts_of(res, offsets):
    """Per unit: the TOON text when converted, the index tokens and the count, read at the batch's offsets."""
    tl = np.frombuffer(res["toon_raw"][0], dtype=np.int32)
    tst = res["toon_status"]
    toon = [res["_tb"][int(offsets[i]):int(offsets[i]) + int(tl[i])].tobytes() if tst[i] == engine.TOON_CONVERTED else None for i in range(len(tst))]
    idx = [(int(res["_cnt"][i]), res["_tk"][int(offsets[i]):int(offsets[i]) + (int(res["_cnt"][i]) & 0x7FFFFFFF)].tobytes()) for i in range(len(tst))]
    return toon, idx


def assert_same(ch, units, misalign=0, batch=None):
    """Pack `units` from a device tensor (into `batch` when given) and upload them into a fresh batch: every consumer agrees."""
    ctx = engine.Context.get()
    stream_bytes, offs = ra.pack(units)
    n, nbytes = len(units), len(stream_bytes)
    s = stream()
    up = engine.Batch(ctx, nbytes, n)
    up.upload(stream_bytes, offs, cuda_stream=s.cuda_stream)
    a = consumers(ch, up, n, nbytes, s)
    src, d_off, src_bytes = device_source(units, misalign)
    pk = batch or engine.Batch(ctx, nbytes, n)
    pk.pack_device(src, d_off, stream=s, src_bytes=src_bytes)
    assert int(ctx.lib.cf_batch_units(pk.h)) == n and int(ctx.lib.cf_batch_bytes(pk.h)) == nbytes
    b = consumers(ch, pk, n, nbytes, s)
    assert a["bitmaps"] == b["bitmaps"]
    assert a["toon_raw"][1] == b["toon_raw"][1]
    assert texts_of(a, offs) == texts_of(b, offs)
    for mask in (FULL, SCAN_MASK):
        va, ta, bma, ooa = a["runs"][mask]
        vb, tb, bmb, oob = b["runs"][mask]
        assert va == vb and bma == bmb and ooa == oob, mask
        assert ta == tb, mask
    return a


@pytest.fixture(scope="module")
def chain():
    return ra.Chain(ra.HARMFUL, ra.SUBS + ra.TEMPLATES)


def mix16k(n, hit_rate=1e-2, seed=0):
    """bench.py's payload shapes at its 16 KiB size: API records, nested configs and prose in a JSON body."""
    pool = []
    for i in range(9):
        shape = "ABC"[i % 3]
        if shape == "C":
            pool.append(json.dumps({"title": f"document {i}", "lang": "en", "body": synth.payload("C", 16384 - 64, seed=i, hit_rate=hit_rate)},
                                   ensure_ascii=False, separators=(",", ":")))
        else:
            pool.append(synth.payload(shape, 16384 if shape == "A" else 9800, seed=i, hit_rate=hit_rate))
    rng = random.Random(seed)
    return [rng.choice(ra.DIRTY) if rng.random() < 0.1 else rng.choice(pool) for _ in range(n)]


def by_length(lo, hi):
    """One unit of every length in [lo, hi]: JSON-ish text with the rules' and lexicons' words, so all consumers have work."""
    base = '{"a": "crap kill them", "b": [1, 2.5, "x"], "c": "bob@example.com crud"} I want to die ' * 4
    return [base[:k] for k in range(lo, hi + 1)]


def test_bench_mix(chain):
    assert_same(chain, mix16k(40))


def test_every_length_and_alignment(chain):
    assert_same(chain, by_length(0, 70) + [""] * 3 + by_length(0, 20)[::-1])


@pytest.mark.parametrize("misalign", range(1, 16))
def test_misaligned_source(chain, misalign):
    assert_same(chain, by_length(0, 40)[::3] + mix16k(3, seed=misalign), misalign=misalign)


def test_coarse_boundaries(chain):
    """Units of exactly 4096 bytes, units whose terminator is the last byte of a 4 KiB page, and words the scan matches on both sides
    of every coarse boundary: a wrong coarse[] entry attributes a match to the wrong unit and shows in the bitmaps."""
    word = "crap kill them "
    exact = [(word * 300)[:4096]] * 3
    page_end = [word + "x" * (4095 - 2 * len(word)) + word] * 3            # 4095 bytes + terminator: ends on a 4 KiB boundary
    straddle, pos = [], 3 * 4096 + 3 * 4097                               # after page_end and exact below
    for _ in range(12):                                                   # a unit ends with the word right before a boundary,
        gap = 4096 - pos % 4096                                           # the next one starts with it right after
        ln = max(gap - 1, len(word))
        u = ("." * (ln - len(word)) + word)[:ln]
        straddle.append(u)
        pos += len(u.encode()) + 1
        straddle.append(word.strip())
        pos += len(word.strip()) + 1
    units = page_end + exact + straddle + ["", "", word] + exact
    a = assert_same(chain, units)
    hits = [int.from_bytes(a["bitmaps"][8 * i * chain.prog.words:8 * i * chain.prog.words + 8], "little") for i in range(len(units))]
    assert all(hits[i] for i in range(len(units)) if units[i])                # every non-empty unit has a match of its own


def test_large_single_unit_and_non_ascii(chain):
    big = json.dumps({"rows": [{"id": i, "t": "crap é 日本 😀" if i % 7 == 0 else "fine"} for i in range(4000)]}, ensure_ascii=False)
    assert len(big.encode()) > 65536
    assert_same(chain, [big])
    assert_same(chain, ["é crap 日本 crud 😀", "lone \ud800 surrogate crap", json.dumps({"k": "\udfff x"}), "\x00\x01 ctrl", "ß" * 33, big[:70001]],
                misalign=3)


def test_pack_after_a_longer_upload_rearms_the_tail(chain):
    ctx = engine.Context.get()
    long_units = mix16k(30, seed=4)
    st, of = ra.pack(long_units)
    batch = engine.Batch(ctx, len(st), 100)
    batch.upload(st, of)
    torch.cuda.synchronize()
    assert_same(chain, by_length(0, 60) + mix16k(2, seed=5), batch=batch)


def rewrite_chain():
    """regex_filter rules that rewrite inside JSON strings: literals, templates with group references, and one that grows the text."""
    return ra.Chain(ra.HARMFUL, ra.SUBS + ra.TEMPLATES + [("yikes", 0, "redacted-redacted-redacted-redacted")])


def resubmit_units():
    rows = [json.dumps({"rows": [{"id": i, "t": "crap" if i % 3 == k % 3 else "ok", "m": f"u{i}@mail.com"} for i in range(10 + k)]}) for k in range(6)]
    return mix16k(30, seed=8) + rows + [json.dumps({"note": "mail bob@example.com about the crup", "n": 5}), json.dumps(["crud", "crap", 1])] + ["not json crap"]


def toon_run(ctx, batch, n, nbytes, d_us, s):
    run = engine.Run(ctx, n, nbytes)
    bufs = ra.Bufs(n, 1, 2 * nbytes + 4096)
    run.enqueue(None, batch, N.CF_STAGE_TOON, d_us, 0, bufs.v, bufs.oo, bufs.out, None, stream=s)
    assert run.finish() == 0
    v, texts, _bm, oo = bufs.results()
    return v, texts


def test_resubmit_rewritten_units_on_the_device():
    """SCAN|SUB|TOON flags the units a rule rewrote with CF_V_RESUBMIT; the run's own out / out_offsets are packed into a second batch
    with no host copy, and TOON runs over it with unit stages set on the device from the flag.  The TOON texts must be the oracle's
    toon.encode of the oracle's rewritten text, and the same as downloading, packing on the host and uploading."""
    ch = rewrite_chain()
    ctx = engine.Context.get()
    units = resubmit_units()
    n = len(units)
    st, of = ra.pack(units)
    s = stream()
    b1 = engine.Batch(ctx, len(st), n)
    b1.upload(st, of, cuda_stream=s.cuda_stream)
    run = engine.Run(ctx, n, len(st))
    cap = 4 * len(st) + 4096
    bufs = ra.Bufs(n, ch.prog.words, cap)
    run.enqueue(ch.prog, b1, FULL, None, 0, bufs.v, bufs.oo, bufs.out, bufs.bm, stream=s)
    assert run.finish() == 0
    total = run.gathered_bytes
    v1, texts1, _bm, oo1 = bufs.results()
    assert total == int(oo1[-1])
    resub = [i for i in range(n) if int(v1["flags"][i]) & N.CF_V_RESUBMIT]
    assert len(resub) >= 8 and any(len(texts1[i]) > len(engine.encode_unit(units[i])) for i in resub)

    b2 = engine.Batch(ctx, total + n, n)
    with torch.cuda.stream(s):
        flags = bufs.v.view(n, 24)[:, 8]
        d_us = ((flags & N.CF_V_RESUBMIT) != 0).to(torch.uint8) * N.CF_STAGE_TOON
    b2.pack_device(bufs.out, bufs.oo, stream=s, src_bytes=total)
    v2, texts2 = toon_run(ctx, b2, n, total + n, d_us, s)

    for i in range(n):
        if i in resub:
            rewritten = ref.regex_apply_str(ch.rules, units[i]).encode()
            assert texts1[i] == rewritten, i
            want = toon_ref.process_text(rewritten.decode(), 0, 1 << 30)
            got = texts2[i].decode() if int(v2["flags"][i]) & N.CF_V_TOON else None
            assert got == want, i
            assert int(v2["aux"][i]) != engine.TOON_SKIPPED
        else:
            assert int(v2["aux"][i]) == engine.TOON_SKIPPED and texts2[i] == b"", i

    # the host route: download the run's texts, pack them on the host, upload, same stages
    hs, ho = engine.pack_units(texts1)
    b3 = engine.Batch(ctx, len(hs), n)
    b3.upload(hs, ho, cuda_stream=s.cuda_stream)
    v3, texts3 = toon_run(ctx, b3, n, len(hs), d_us, s)
    assert v2.tobytes() == v3.tobytes() and texts2 == texts3


def test_pack_and_enqueue_captured_in_one_graph(chain):
    """Pack + enqueue captured after a warm-up; replays over new source content of the same unit count and byte count, in other
    orders, each equal to the upload path."""
    ctx = engine.Context.get()
    base = ra.bench_mix(1e-2, distinct=9, n=100, seed=21)
    contents = [base[::-1], base[41:] + base[:41], sorted(base)]
    src, d_off, src_bytes = device_source(base, misalign=5)
    n, nbytes = len(base), src_bytes + len(base)
    batch = engine.Batch(ctx, nbytes, n)
    run = engine.Run(ctx, n, nbytes)
    bufs = ra.Bufs(n, chain.prog.words, 2 * nbytes)
    s = stream()

    def step(st):
        batch.pack_device(src, d_off, n, stream=st, src_bytes=src_bytes)
        run.enqueue(chain.prog, batch, FULL, None, 0, bufs.v, bufs.oo, bufs.out, bufs.bm, stream=st)

    step(s)                                                              # warm-up: the run's workspaces and arena reach their size
    assert run.finish() == 0
    ra.check(chain, base, FULL, None, (bufs.results(), 0))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step(torch.cuda.current_stream())
    for units in contents:
        nsrc, noff, nb = device_source(units, misalign=5)
        assert nb == src_bytes
        with torch.cuda.stream(s):
            src.copy_(nsrc)
            d_off.copy_(noff)
            g.replay()
        assert run.finish() == 0
        got = bufs.results()
        (want, _need) = ra.run_async(chain, units, FULL)
        assert got[0].tobytes() == want[0].tobytes() and got[1] == want[1] and np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])


def test_refusals_queue_nothing(chain):
    ctx = engine.Context.get()
    units = ra.bench_mix(1e-2, distinct=6, n=40, seed=3)
    st, of = ra.pack(units)
    n = len(units)
    batch = engine.Batch(ctx, len(st), n)
    batch.upload(st, of)
    big = units + ["x" * 100]
    src, d_off, sb = device_source(big)
    L = ctx.lib
    for args, code in (((0, d_off.data_ptr(), n, sb), N.CF_E_BADARG),
                       ((src.data_ptr(), 0, n, sb), N.CF_E_BADARG),
                       ((src.data_ptr(), d_off.data_ptr(), 0, sb), N.CF_E_BADARG),
                       ((src.data_ptr(), d_off.data_ptr(), n + 1, sb), N.CF_E_CAPACITY),          # n over max_units
                       ((src.data_ptr(), d_off.data_ptr(), n, len(st) - n + 1), N.CF_E_CAPACITY),  # src_bytes + n over the stream capacity
                       ((src.data_ptr(), d_off.data_ptr(), n, 1 << 63), N.CF_E_CAPACITY)):
        assert L.cf_batch_pack_device(ctx.h, batch.h, *args, None) == code, args
    with pytest.raises(N.CfError) as exc:
        batch.pack_device(src, d_off, stream=0)                           # n + 1 units over max_units, src_bytes read from the device
    assert exc.value.code == N.CF_E_CAPACITY
    with pytest.raises(ValueError):
        batch.pack_device(src, d_off[:3], n=n, src_bytes=sb)
    with pytest.raises(ValueError):
        batch.pack_device(src[:10], d_off, n=n, src_bytes=sb)
    torch.cuda.synchronize()
    v, out, oo, _ = engine.run_batch(chain.prog, batch, None, of, FULL)   # the batch still holds what was uploaded
    rv, rout, roo, _ = engine.run_batch(chain.prog, engine.Batch(ctx, len(st), n), st, of, FULL)
    assert v.tobytes() == rv.tobytes() and np.array_equal(oo, roo) and out[:int(oo[-1])].tobytes() == rout[:int(roo[-1])].tobytes()
