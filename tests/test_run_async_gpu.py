"""cf_run_enqueue / cf_run_finish (engine.Run): the fused chain enqueued on the caller's stream, verdicts and texts left on the device.
Every result is checked against two independent references: the stage-by-stage ABI (cf_scan_host, cf_sub_host on the units the
bitmaps select, cf_toon_host) and the CPU oracle (CPython `re`, oracle/toon_ref.py).  Covered: the bench's payload mix at three hit
rates, per-unit stages, more than 64 patterns, template rules with group references, units deferred to cf_run_finish (a rewrite that
outgrows its first bound, an arena too small for the dirty units), the output capacity, two runs in flight on two streams, a CUDA
graph capture of the enqueue replayed over new content, and ShardedChain's device all-gather on a one-rank NCCL group."""
import json
import random
import re
import socket

import numpy as np
import pytest
import torch

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from mcp_context_forge_b200.regex_frontend import template_parts
from oracle import hook_chain_ref as ref
from oracle import toon_ref

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes")]
TEMPLATES = [(r"(\w+)@(\w+)\.com", 0, r"<\2 at \1>"), (r"cr(a|u)p", 0, r"[\g<0>/\1]")]
WIDE = [(f"zq{k:03d}x", 0) for k in range(70)]              # with HARMFUL: more than 64 patterns, W = 2
GROW = [("a", 0, "Z" * 200)]                                # 2 000 "a" -> 400 000 bytes: past the first bound of 64 L + 64 KiB
FULL = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
DIRTY = [json.dumps({"rows": [{"id": i, "t": "crap" if i % 3 == 0 else "ok"} for i in range(12)]}), "this is crap", "crap crud crap",
         json.dumps({"note": "mail bob@example.com about the crup", "n": 5}), "é crap 日本 crud 😀 zq007x", "zq069x and zq001x"]


class Chain:
    """A compiled program and its oracle (per distinct unit text: full bitmap, dirty, rewritten text, TOON text)."""

    def __init__(self, searches, subs):
        self.searches, self.subs = searches, subs
        p = engine.Program()
        for pat, f in searches:
            p.add_search(pat, f)
        self.sub_bits = [p.add_sub(pat, f, template_parts(r, re.compile(pat, f))) for pat, f, r in subs]
        self.prog = p.compile(engine.Context.get())
        self.rules = [(re.compile(pat, f), r) for pat, f, r in subs]
        self.cache = {}

    def oracle(self, u):
        if u not in self.cache:
            bits = ref.scan_bitmaps([u], self.searches, [], [(p, f) for p, f, _ in self.subs])[0]
            dirty = any(c.search(u) for c, _ in self.rules)
            self.cache[u] = (bits, dirty, ref.regex_apply_str(self.rules, u).encode() if dirty else None, toon_ref.process_text(u, 0, 1 << 30))
        return self.cache[u]


def bench_mix(hit_rate, distinct=24, n=160, seed=0):
    """The bench's payload shapes (A: API records, B: nested configs, C: prose in a JSON body) at its hit rate, plus rewrite units."""
    pool = []
    for i in range(distinct):
        shape = "ABC"[i % 3]
        if shape == "C":
            pool.append(json.dumps({"title": f"document {i}", "body": synth.payload("C", 6000, seed=i, hit_rate=hit_rate)}, ensure_ascii=False))
        else:
            pool.append(synth.payload(shape, 6000 if shape == "A" else 3600, seed=i, hit_rate=hit_rate))
    rng = random.Random(seed)
    return [rng.choice(DIRTY) if rng.random() < 0.1 else rng.choice(pool) for _ in range(n)]


def pack(units):
    return engine.pack_units([engine.encode_unit(u) for u in units])


class Bufs:
    def __init__(self, n, W, cap):
        self.v = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
        self.oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        self.out = torch.full((max(cap, 1),), 0xAB, dtype=torch.uint8, device="cuda")
        self.bm = torch.zeros(n * W, dtype=torch.int64, device="cuda")

    def results(self):
        v = self.v.cpu().numpy().view(engine.VERDICT_DTYPE)
        oo = self.oo.cpu().numpy().view(np.uint64)
        out = self.out.cpu().numpy()
        return v, [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(len(v))], self.bm.cpu().numpy().view(np.uint64), oo


def enqueue(run, ch, batch, bufs, mask, d_us, stream):
    run.enqueue(ch.prog, batch, mask, d_us, 0, bufs.v, bufs.oo, bufs.out, bufs.bm, stream=stream)


def run_async(ch, units, mask, stages=None, arena=1 << 20, cap=None):
    ctx = engine.Context.get()
    stream, offs = pack(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    run = engine.Run(ctx, n, len(stream), arena)
    bufs = Bufs(n, ch.prog.words, 2 * len(stream) + 4096 if cap is None else cap)
    d_us = torch.from_numpy(stages).cuda() if stages is not None else None
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    batch.upload(stream, offs, cuda_stream=s.cuda_stream)
    enqueue(run, ch, batch, bufs, mask, d_us, s)
    need = run.finish()
    return bufs.results(), need


def stage_by_stage(ch, units, mask, stages=None):
    """The same chain through the synchronous per-stage entry points."""
    ctx = engine.Context.get()
    stream, offs = pack(units)
    n, W = len(units), ch.prog.words
    batch = engine.Batch(ctx, len(stream), n)
    bm = engine.scan_host(ch.prog, batch, stream, offs)
    st = [0xFF] * n if stages is None else [int(x) for x in stages]
    sub_bits = ch.sub_bits if mask & N.CF_STAGE_SUB else []
    dirty = [i for i in range(n) if st[i] & N.CF_STAGE_SUB and any(int(bm[i * W + b // 64]) >> (b % 64) & 1 for b in sub_bits)]
    subs = dict(zip(dirty, engine.sub_host(ch.prog, batch, dirty)))
    tst, tt = engine.toon_host(batch, stream, offs, report_errors=False) if mask & N.CF_STAGE_TOON else (None, None)
    v = np.zeros(n, dtype=engine.VERDICT_DTYPE)
    texts = []
    for i in range(n):
        flags, aux, text = 0, 0, b""
        toon_here = bool(mask & N.CF_STAGE_TOON and st[i] & N.CF_STAGE_TOON)
        if i in subs:
            flags, text = N.CF_V_REWRITTEN | (N.CF_V_RESUBMIT if toon_here else 0), subs[i]
        if mask & N.CF_STAGE_TOON:
            aux = engine.TOON_SKIPPED if flags & N.CF_V_RESUBMIT or not toon_here else int(tst[i])
            if aux == engine.TOON_CONVERTED and not flags & N.CF_V_REWRITTEN:
                flags, text = flags | N.CF_V_TOON, tt[i]
        v[i] = (int(bm[i * W]), flags, len(text), aux, 0)
        texts.append(text)
    return v, texts, bm


def check(ch, units, mask, stages, got):
    (v, texts, bm, oo), need = got
    assert need == 0
    rv, rtexts, rbm = stage_by_stage(ch, units, mask, stages)
    assert v.tobytes() == rv.tobytes()
    assert texts == rtexts
    assert np.array_equal(bm, rbm)
    W = ch.prog.words
    for i, u in enumerate(units):                            # the oracle
        bits, dirty, sub_text, toon_text = ch.oracle(u)
        st = int(stages[i]) if stages is not None else 0xFF
        assert sum(int(bm[i * W + w]) << (64 * w) for w in range(W)) == bits, i
        flags = int(v["flags"][i])
        if dirty and st & N.CF_STAGE_SUB and mask & N.CF_STAGE_SUB:
            assert flags & N.CF_V_REWRITTEN and texts[i] == sub_text, i
        elif mask & N.CF_STAGE_TOON and st & N.CF_STAGE_TOON:
            assert (texts[i].decode() if flags & N.CF_V_TOON else None) == toon_text, i
        else:
            assert flags == 0 and texts[i] == b"", i
    assert int(oo[-1]) == sum(len(t) for t in texts)
    return v


def random_stages(n, seed):
    rng = random.Random(seed)
    choices = [N.CF_STAGE_SUB, N.CF_STAGE_TOON, N.CF_STAGE_SUB | N.CF_STAGE_TOON, 0, N.CF_STAGE_SCAN]
    return np.array([rng.choice(choices) for _ in range(n)], dtype=np.uint8)


@pytest.mark.parametrize("with_stages", [False, True], ids=["all_stages", "unit_stages"])
@pytest.mark.parametrize("hit_rate", [0.0, 1e-4, 1e-2])
def test_parity_on_the_bench_mix(hit_rate, with_stages):
    ch = Chain(HARMFUL, SUBS)
    units = bench_mix(hit_rate, seed=int(hit_rate * 1e4) + with_stages)
    stages = random_stages(len(units), 5) if with_stages else None
    v = check(ch, units, FULL, stages, run_async(ch, units, FULL, stages))
    assert any(v["flags"] & N.CF_V_REWRITTEN) and any(v["flags"] & N.CF_V_TOON)


@pytest.mark.parametrize("mask", [FULL, N.CF_STAGE_SCAN | N.CF_STAGE_SUB, N.CF_STAGE_SCAN | N.CF_STAGE_TOON], ids=["full", "no_toon", "no_sub"])
def test_parity_more_than_64_patterns_and_templates(mask):
    ch = Chain(HARMFUL + WIDE, SUBS + TEMPLATES)
    assert ch.prog.words == 2
    units = bench_mix(1e-2, distinct=9, n=120, seed=3) + DIRTY * 4
    for stages in (None, random_stages(len(units), 9)):
        check(ch, units, mask, stages, run_async(ch, units, mask, stages))


def test_deferred_units_are_finished():
    ch = Chain(HARMFUL, GROW + SUBS)
    clean = [json.dumps({"id": i, "v": [1, 2, i], "w": "xyz" * i}) for i in range(8)]   # no "a" anywhere
    units = ["a" * 2000, "crap", "xay", json.dumps({"k": "a", "v": [1, 2]}), "no hit here!"] * 6 + clean * 3
    cap = 6 * 400000 + (1 << 20)
    (v, _t, _b, _o), _n = got = run_async(ch, units, FULL, cap=cap)   # outgrows the first bound: deferred, finished by cf_run_finish
    check(ch, units, FULL, None, got)
    assert all(int(v["out_len"][i]) == 400000 for i, u in enumerate(units) if u == "a" * 2000)
    for arena in (0, 4096):                                           # the arena holds none / a few of the dirty units
        check(ch, units, FULL, None, run_async(ch, units, FULL, arena=arena, cap=cap))


def test_too_large_is_still_reported():
    """Host offsets that disagree with the batch size a unit's scratch below what its rewrite needs: cf_run_batch (an enqueue and a
    finish on the context's run) returns CF_E_TOO_LARGE from the deferred unit's synchronous substitution."""
    ch = Chain(HARMFUL, GROW)
    ctx = engine.Context.get()
    units = ["a" * 2000, "xy", "crap"]
    stream, offs = pack(units)
    batch = engine.Batch(ctx, len(stream), len(units))
    batch.upload(stream, offs)
    wrong = offs.copy()
    wrong[1] = 3
    with pytest.raises(N.CfError) as exc:
        engine.run_batch(ch.prog, batch, None, wrong, FULL, outputs_resident=True)
    assert exc.value.code == N.CF_E_TOO_LARGE
    v, out, oo, _ = engine.run_batch(ch.prog, batch, stream, offs, FULL)
    assert int(v["out_len"][0]) == 400000 and out[:200].tobytes() == b"Z" * 200


def test_output_capacity():
    ch = Chain(HARMFUL, SUBS)
    units = bench_mix(1e-2, distinct=6, n=60, seed=4)
    (_v, texts, _b, oo), _ = run_async(ch, units, FULL)
    need = int(oo[-1])
    (v1, _t1, _b1, oo1), got = run_async(ch, units, FULL, cap=need - 1)
    assert got == need
    rv, rtexts, _ = stage_by_stage(ch, units, FULL)
    assert v1.tobytes() == rv.tobytes() and int(oo1[-1]) == need          # verdicts and offsets are valid, nothing was gathered
    check(ch, units, FULL, None, run_async(ch, units, FULL, cap=need))


def test_two_runs_in_flight():
    ch = Chain(HARMFUL, SUBS + TEMPLATES)
    ctx = engine.Context.get()
    sets = [bench_mix(1e-2, distinct=9, n=90, seed=7), bench_mix(1e-4, distinct=12, n=140, seed=8) + DIRTY]
    state = []
    for units in sets:
        stream, offs = pack(units)
        batch = engine.Batch(ctx, len(stream), len(units))
        run = engine.Run(ctx, len(units), len(stream))
        bufs = Bufs(len(units), ch.prog.words, 2 * len(stream))
        state.append((units, stream, offs, batch, run, bufs, torch.cuda.Stream()))
    torch.cuda.synchronize()
    for units, stream, offs, batch, run, bufs, s in state:             # both enqueued before either is finished
        batch.upload(stream, offs, cuda_stream=s.cuda_stream)
        enqueue(run, ch, batch, bufs, FULL, None, s)
    for units, _s, _o, _b, run, bufs, _st in reversed(state):
        need = run.finish()
        check(ch, units, FULL, None, (bufs.results(), need))


def test_enqueue_captured_in_a_cuda_graph():
    """Capture fails when the enqueue synchronises or allocates; two replays over new content of the same shape are both right."""
    ch = Chain(HARMFUL, SUBS + TEMPLATES)
    ctx = engine.Context.get()
    base = bench_mix(1e-2, distinct=9, n=100, seed=11)
    contents = [base, base[::-1], base[37:] + base[:37]]                 # same units and bytes, other order
    stream, offs = pack(base)
    n = len(base)
    batch = engine.Batch(ctx, len(stream), n)
    run = engine.Run(ctx, n, len(stream))
    bufs = Bufs(n, ch.prog.words, 2 * len(stream))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    batch.upload(stream, offs, cuda_stream=s.cuda_stream)
    enqueue(run, ch, batch, bufs, FULL, None, s)                           # warm-up: workspaces and the arena reach their size
    need = run.finish()
    check(ch, base, FULL, None, (bufs.results(), need))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enqueue(run, ch, batch, bufs, FULL, None, torch.cuda.current_stream())
    for units in contents[1:]:
        st, of = pack(units)
        assert len(st) == len(stream)
        with torch.cuda.stream(s):
            batch.upload(st, of, cuda_stream=s.cuda_stream)
            g.replay()
        need = run.finish()
        check(ch, units, FULL, None, (bufs.results(), need))


def test_sharded_chain_all_gathers_device_verdicts():
    import torch.distributed as dist

    from mcp_context_forge_b200.dist import ShardedChain

    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        ch = Chain(HARMFUL, SUBS)
        units = bench_mix(1e-2, distinct=9, n=80, seed=13)
        stages = random_stages(len(units), 2)
        sc = ShardedChain(ch.prog, device=torch.cuda.current_device())
        parts = sc.partition([len(u.encode()) for u in units])
        full, mine, out, oo = sc.run(units, parts, FULL, stages)
        stream, offs = pack(units)
        batch = engine.Batch(engine.Context.get(), len(stream), len(units))
        v, rout, roo, _ = engine.run_batch(ch.prog, batch, stream, offs, FULL, stages)
        assert mine == list(range(len(units)))
        assert full.tobytes() == v.tobytes()
        assert np.array_equal(oo, roo) and out.tobytes() == rout[:int(roo[-1])].tobytes()
    finally:
        dist.destroy_process_group()


def test_graph_replays_with_more_dirty_units_than_the_capture():
    """A replay that needs more arena than the warm-up defers the units that do not fit; the finish behind it grows the run's arena,
    and the graph (which still holds the old one) stays right on the replays after it."""
    ch = Chain(HARMFUL, SUBS)
    ctx = engine.Context.get()
    dirty, clean = "crap " * 60, "okay " * 60                             # same length: every content below has the same shape
    light = [dirty] + [clean] * 99
    heavy = [dirty if i % 5 < 3 else clean for i in range(100)]
    stream, offs = pack(light)
    batch = engine.Batch(ctx, len(stream), len(light))
    run = engine.Run(ctx, len(light), len(stream), 1024)                 # holds the light content's one dirty unit (640 bytes)
    bufs = Bufs(len(light), ch.prog.words, 2 * len(stream))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    batch.upload(stream, offs, cuda_stream=s.cuda_stream)
    enqueue(run, ch, batch, bufs, FULL, None, s)
    need = run.finish()
    check(ch, light, FULL, None, (bufs.results(), need))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enqueue(run, ch, batch, bufs, FULL, None, torch.cuda.current_stream())
    for units in (heavy, heavy[::-1], light, heavy):
        st, of = pack(units)
        with torch.cuda.stream(s):
            batch.upload(st, of, cuda_stream=s.cuda_stream)
            g.replay()
        need = run.finish()
        check(ch, units, FULL, None, (bufs.results(), need))


def test_substitution_limit_of_a_deferred_unit_is_an_error():
    """A deferred unit whose rewrite would pass 4 GB: the synchronous substitution's limit is reported as an error by cf_run_batch
    (its code, as before) and by cf_run_finish (CF_E_TOO_LARGE), never taken for an output buffer that is too small."""
    ch = Chain(HARMFUL, [("a", 0, "Z" * 5000)])
    ctx = engine.Context.get()
    units = ["a" * (1 << 20), "xyz", "crap"]
    stream, offs = pack(units)
    batch = engine.Batch(ctx, len(stream), len(units))
    with pytest.raises(N.CfError) as exc:
        engine.run_batch(ch.prog, batch, stream, offs, FULL)
    assert exc.value.code == N.CF_E_CAPACITY and "beyond 4 GB" in str(exc.value)
    with pytest.raises(N.CfError) as exc:
        run_async(ch, units, FULL)
    assert exc.value.code == N.CF_E_TOO_LARGE and "beyond 4 GB" in str(exc.value)


def test_short_tensors_are_refused():
    ch = Chain(HARMFUL, SUBS)
    ctx = engine.Context.get()
    units = DIRTY * 3
    stream, offs = pack(units)
    n = len(units)
    batch = engine.Batch(ctx, len(stream), n)
    batch.upload(stream, offs)
    run = engine.Run(ctx, n, len(stream))
    bufs = Bufs(n, ch.prog.words, 2 * len(stream))
    for name, short in (("verdicts", dict(verdicts=bufs.v[:-1])), ("out_offsets", dict(out_offsets=bufs.oo[:-1])),
                        ("bitmaps_full", dict(bitmaps_full=bufs.bm[:-1]))):
        args = dict(verdicts=bufs.v, out_offsets=bufs.oo, out=bufs.out, bitmaps_full=bufs.bm)
        args.update(short)
        with pytest.raises(ValueError, match=name):
            run.enqueue(ch.prog, batch, FULL, None, 0, **args)
