"""GPU: request_logging_masking through cf_run_enqueue / cf_run_finish (engine.Run with CF_STAGE_MASK): the masking kernel, the
verdicts, the offsets, the gather and the re-masking of the bodies that outgrow their first room, all on the caller's stream.  Every
result is checked against cf_run_batch on the same batch (engine.run_batch) and against the oracle (oracle/mask_ref.py).  Covered: the
bench's shapes and the edge bodies of tests/test_mask_edges_gpu.py at two depths, outputs many times their input among packed
neighbours, SCAN | SUB | MASK with units deferred to cf_run_finish, a CUDA graph capture replayed over new bodies, two runs in flight,
the output capacity, the refusals, and ShardedChain's device path on a one-rank NCCL group."""
import json
import os
import re

import numpy as np
import pytest
import torch

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from oracle import hook_chain_ref as ref
from oracle import mask_ref
from test_mask_edges_gpu import float_bodies, growth_cases, nesting_bodies, packed_with_neighbours, unprinted_bodies

pytestmark = pytest.mark.gpu

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
SM = N.CF_STAGE_SCAN | N.CF_STAGE_MASK
ZZ_BODIES = ['{"password":"secret","note":"I want to kill myself","nested":{"authToken":"abc","count":3}}', '{"a":1,}', "[01]", "",
             '{"level":{"nested":{}}}', '[0.30000000000000004,5e-324,1e23,-0]', '{"Cookie":"jwt_token=abc","text":"how to make a bomb \\u00e9"}']


def _b(x):
    return x if isinstance(x, bytes) else x.encode()


def expected(body, max_depth):
    try:
        return mask_ref.mask_json_bytes(_b(body), max_depth)
    except ValueError:
        return None


def growth(max_depth):
    return [b for b, md in growth_cases() if md == max_depth]


def corpus():
    """synth shapes A / B, the bodies of test_zz_run_batch_mask_gpu.py and the edge bodies of test_mask_edges_gpu.py."""
    bodies = [synth.payload("B", 16384, seed=s) for s in range(12)] + [synth.payload("A", 16384, seed=s) for s in range(6)] + ZZ_BODIES
    bodies += nesting_bodies() + unprinted_bodies() + float_bodies()[::40] + growth(10) + growth(2)
    return [_b(b) for b in bodies]


_progs = {}


def scan_prog():
    if "scan" not in _progs:
        p = engine.Program()
        for pat, f in HARMFUL:
            p.add_search(pat, f)
        _progs["scan"] = p.compile(engine.Context.get())
    return _progs["scan"]


class Bufs:
    def __init__(self, n, W, cap):
        self.v = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
        self.oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        self.out = torch.full((max(cap, 1),), 0xAB, dtype=torch.uint8, device="cuda")
        self.bm = torch.zeros(n * W, dtype=torch.int64, device="cuda")

    def results(self):
        v = self.v.cpu().numpy().view(engine.VERDICT_DTYPE)
        oo = self.oo.cpu().numpy().view(np.uint64)
        return v, oo, self.out.cpu().numpy()[: int(oo[-1])].tobytes()


class Async:
    """One Run, its batch and its device buffers, enqueued on a side stream."""

    def __init__(self, bodies, cap=None, arena=1 << 20, W=1):
        self.ctx = engine.Context.get()
        self.stream, self.offs = engine.pack_units(bodies)
        self.n = len(bodies)
        self.batch = engine.Batch(self.ctx, len(self.stream), self.n)
        self.run = engine.Run(self.ctx, self.n, len(self.stream), arena)
        self.bufs = Bufs(self.n, W, 12 * len(self.stream) + 4096 if cap is None else cap)
        self.s = torch.cuda.Stream()
        self.s.wait_stream(torch.cuda.current_stream())

    def upload(self, bodies=None):
        stream, offs = (self.stream, self.offs) if bodies is None else engine.pack_units(bodies)
        self.batch.upload(stream, offs, cuda_stream=self.s.cuda_stream)

    def enqueue(self, prog, stage_mask, max_depth, d_us=None, stream=None):
        scan = stage_mask & (N.CF_STAGE_SCAN | N.CF_STAGE_SUB)
        self.run.enqueue(prog, self.batch, stage_mask, d_us, 0, self.bufs.v, self.bufs.oo, self.bufs.out, self.bufs.bm if scan else None,
                         stream=self.s if stream is None else stream, mask_max_depth=max_depth)

    def __call__(self, prog, stage_mask, max_depth, d_us=None):
        self.upload()
        self.enqueue(prog, stage_mask, max_depth, d_us)
        return self.run.finish()


def sync(prog, bodies, stage_mask, max_depth, stages=None):
    """cf_run_batch on the same bodies: (verdicts, out_offsets, bytes)."""
    stream, offs = engine.pack_units(bodies)
    batch = engine.Batch(engine.Context.get(), len(stream), len(bodies))
    v, out, oo, _ = engine.run_batch(prog, batch, np.frombuffer(stream, dtype=np.uint8), offs, stage_mask, unit_stages=stages, mask_max_depth=max_depth)
    return v.copy(), oo.copy(), out[: int(oo[-1])].tobytes()


def check_oracle(bodies, max_depth, got):
    v, oo, out = got
    for i, b in enumerate(bodies):
        e = expected(b, max_depth)
        assert bool(v["flags"][i] & N.CF_V_MASKED) == (e is not None), (i, max_depth, b[:80])
        assert int(v["aux"][i]) == (engine.MASK_OK if e is not None else engine.MASK_PARSE_ERROR), (i, max_depth)
        assert out[int(oo[i]):int(oo[i + 1])] == (e if e is not None else b""), (i, max_depth, b[:80])
    assert int(oo[-1]) == sum(len(e) for e in (expected(b, max_depth) for b in bodies) if e is not None)


def assert_same(got, want):
    assert got[0].tobytes() == want[0].tobytes()
    assert np.array_equal(got[1], want[1])
    assert got[2] == want[2]


@pytest.mark.parametrize("max_depth", [10, 2])
@pytest.mark.parametrize("stage_mask", [SM, N.CF_STAGE_MASK], ids=["scan_mask", "mask"])
def test_parity_with_run_batch_and_the_oracle(stage_mask, max_depth):
    bodies = corpus()
    prog = scan_prog() if stage_mask & N.CF_STAGE_SCAN else None
    a = Async(bodies)
    assert a(prog, stage_mask, max_depth) == 0
    got = a.bufs.results()
    assert_same(got, sync(prog, bodies, stage_mask, max_depth))
    check_oracle(bodies, max_depth, got)
    assert any(len(expected(b, max_depth) or b"") > 5 * len(b) + 32 for b in bodies)     # some body outgrew the first room


def test_overflow_is_masked_again_on_the_device():
    """Bodies whose output outgrows 5 len + 32 bytes, packed among ordinary neighbours, come out exact; the re-masking is one launch
    that runs whether or not a body overflows, so such a batch costs the launches of one without overflow."""
    for md in (1, 10):
        special = growth(md)
        bodies, where = packed_with_neighbours(special, n_plain=800, seed=md)
        plain = [b for i, b in enumerate(bodies) if i not in set(where)]
        plain = plain + plain[: len(special)]
        assert any(len(expected(bodies[i], md)) > 5 * len(bodies[i]) + 32 for i in where)
        assert all(len(expected(b, md) or b"") <= 5 * len(b) + 32 for b in plain)
        counts = []
        for bs in (bodies, plain):
            a = Async(bs)
            a.upload()
            torch.cuda.synchronize()
            before = a.ctx.kernel_launches
            a.enqueue(None, N.CF_STAGE_MASK, md)
            counts.append(a.ctx.kernel_launches - before)
            assert a.run.finish() == 0
            got = a.bufs.results()
            check_oracle(bs, md, got)
            assert_same(got, sync(None, bs, N.CF_STAGE_MASK, md))
        # first pass, verdicts, offset scan, gather, re-masking
        assert counts == [5, 5]


def test_scan_sub_mask_with_deferred_units():
    """SCAN | SUB | MASK (test_zz_run_batch_mask_gpu.py's second case) on a fresh Run with a 1 MiB arena: each dirty 16 KiB body asks the
    arena for more than it holds, so the enqueue defers it and cf_run_finish completes it, then redoes the verdicts, the offsets, the
    gather and the re-masking of the overflow bodies against the new offsets.  Records as cf_run_batch and the oracles give them."""
    ctx = engine.Context.get()
    literals = [f"wq{k:03d}v" for k in range(60)]
    subs = [("crap", 0, "crud"), ("crud", 0, "yikes"), ("zqx", 0, "Z" * 4000)]
    prog = engine.Program()
    for p, f in HARMFUL:
        prog.add_search(p, f)
    for w in literals:
        prog.add_literal(w)
    for p, f, r in subs:
        prog.add_sub(p, f, r)
    prog.compile(ctx)
    rules = [(re.compile(p, f), r) for p, f, r in subs]
    big = lambda s, extra: json.dumps({"password": "hunter2", "note": extra, "data": synth.payload("A", 16384, seed=s)})   # noqa: E731
    bodies = [big(0, "zqx once")[:-1], big(1, "zqx, zqx and crap"), big(2, "no rule here"), big(3, "zqx but SUB is left out"),
              synth.payload("B", 3000, seed=1), json.dumps({"token": "crap", "x": [1, 2, {"apiKey": "crud"}]}), '{"a": "crap",}',
              json.dumps({"text": "I want to kill myself", "ids": ["wq007v", "wq059v"]}), "", '{"Cookie": "zqx=1"}', "[1, 2, 3]",
              json.dumps({"secret": "zqx", "list": list(range(50))})]
    bodies = [_b(b) for b in bodies] + growth(10)[:3]
    stages = np.array([N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_MASK] * len(bodies), dtype=np.uint8)
    for i in (3, 5, 11):
        stages[i] = SM
    stage_mask = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_MASK
    a = Async(bodies, W=prog.words)
    assert a(prog, stage_mask, 10, torch.from_numpy(stages).cuda()) == 0
    got = a.bufs.results()
    assert_same(got, sync(prog, bodies, stage_mask, 10, stages))
    v, oo, out = got
    for i, b in enumerate(bodies):
        text = b.decode()
        masked = expected(b, 10)
        dirty = bool(stages[i] & N.CF_STAGE_SUB) and any(c.search(text) for c, _ in rules)
        out_len = len(masked) if masked is not None else len(ref.regex_apply_str(rules, text).encode()) if dirty else 0
        flags = (N.CF_V_REWRITTEN if dirty else 0) | (N.CF_V_MASKED if masked is not None else 0)
        assert (int(v["flags"][i]), int(v["out_len"][i])) == (flags, out_len), i
        assert out[int(oo[i]):int(oo[i + 1])] == (masked if masked is not None else b""), i
    assert sum(1 for i in range(len(bodies)) if v["flags"][i] == N.CF_V_REWRITTEN) >= 2
    assert any(len(expected(b, 10)) > 5 * len(b) + 32 for b in growth(10)[:3])


def test_enqueue_captured_in_a_cuda_graph():
    """Capture fails when the enqueue synchronises or allocates; two replays over other bodies of the same shape, overflow bodies
    included, are both right."""
    base = corpus()
    contents = [base, base[::-1], base[37:] + base[:37]]
    prog = scan_prog()
    a = Async(base)
    assert a(prog, SM, 10) == 0                                          # warm-up: the masking workspace is allocated here
    assert_same(a.bufs.results(), sync(prog, base, SM, 10))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=a.s):
        a.enqueue(prog, SM, 10, stream=torch.cuda.current_stream())
    for bodies in contents[1:]:
        with torch.cuda.stream(a.s):
            a.upload(bodies)
            g.replay()
        assert a.run.finish() == 0
        got = a.bufs.results()
        assert_same(got, sync(prog, bodies, SM, 10))
        check_oracle(bodies, 10, got)


def test_two_runs_in_flight_mask_and_toon():
    ctx = engine.Context.get()
    subs = [("crap", 0, "crud"), ("crud", 0, "yikes")]
    tprog = engine.Program()
    for p, f in HARMFUL:
        tprog.add_search(p, f)
    for p, f, r in subs:
        tprog.add_sub(p, f, r)
    tprog.compile(ctx)
    full = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
    mbodies = corpus()
    tbodies = [_b(synth.payload("AB"[i % 2], 4000, seed=i)) for i in range(60)] + [b"this is crap", b'{"a":"crud","b":[1,2]}']
    ma, ta = Async(mbodies), Async(tbodies, W=tprog.words)
    torch.cuda.synchronize()
    ma.upload()
    ma.enqueue(None, N.CF_STAGE_MASK, 10)
    ta.upload()
    ta.enqueue(tprog, full, 10)
    assert ta.run.finish() == 0 and ma.run.finish() == 0
    assert_same(ma.bufs.results(), sync(None, mbodies, N.CF_STAGE_MASK, 10))
    assert_same(ta.bufs.results(), sync(tprog, tbodies, full, 10))
    assert any(ta.bufs.results()[0]["flags"] & N.CF_V_TOON)


def test_output_capacity():
    """An `out` too small: finish returns the size it needs and leaves `out` untouched (the re-masking writes nothing either); with
    that size the same enqueue gives the whole result."""
    bodies = [_b(b) for b in ZZ_BODIES] + growth(10)
    need = len(sync(None, bodies, N.CF_STAGE_MASK, 10)[2])
    a = Async(bodies, cap=need - 1)
    assert a(None, N.CF_STAGE_MASK, 10) == need
    assert bool((a.bufs.out == 0xAB).all())
    a.bufs.out = torch.full((need,), 0xAB, dtype=torch.uint8, device="cuda")
    assert a(None, N.CF_STAGE_MASK, 10) == 0
    got = a.bufs.results()
    assert_same(got, sync(None, bodies, N.CF_STAGE_MASK, 10))
    check_oracle(bodies, 10, got)


def test_refusals_come_before_any_launch():
    bodies = [_b(b) for b in ZZ_BODIES] + growth(2)
    a = Async(bodies)
    a.upload()
    torch.cuda.synchronize()
    lib, ctx = a.ctx.lib, a.ctx
    before = ctx.kernel_launches
    rc = lib.cf_run_enqueue(ctx.h, None, a.batch.h, a.run.h, N.CF_STAGE_MASK, None, 0, a.bufs.v.data_ptr(), None, a.bufs.oo.data_ptr(),
                            a.bufs.out.data_ptr(), a.bufs.out.numel(), a.s.cuda_stream)
    assert rc == N.CF_E_BADARG and "cf_run_set_mask" in lib.cf_last_error(ctx.h).decode()
    with pytest.raises(N.CfError) as exc:
        a.enqueue(None, N.CF_STAGE_MASK | N.CF_STAGE_TOON, 2)
    assert exc.value.code == N.CF_E_BADARG
    assert ctx.kernel_launches == before
    a.enqueue(None, N.CF_STAGE_MASK, 2)
    assert a.run.finish() == 0
    got = a.bufs.results()
    assert_same(got, sync(None, bodies, N.CF_STAGE_MASK, 2))
    check_oracle(bodies, 2, got)


def test_sharded_chain_masks_on_the_device_path(tmp_path):
    import torch.distributed as dist

    from mcp_context_forge_b200.dist import ShardedChain

    store = dist.FileStore(os.path.join(str(tmp_path), "store"), 1)
    dist.init_process_group("nccl", store=store, rank=0, world_size=1)
    try:
        prog = scan_prog()
        bodies = [b.decode() for b in corpus()[:200]]
        sc = ShardedChain(prog, device=torch.cuda.current_device())
        parts = sc.partition([len(_b(u)) for u in bodies])
        full, mine, out, oo = sc.run(bodies, parts, SM, mask_max_depth=2)
        assert sc.run_dev is not None                                    # the shard went through cf_run_enqueue
        v, roo, rout = sync(prog, [_b(u) for u in bodies], SM, 2)
        assert mine == list(range(len(bodies)))
        assert full.tobytes() == v.tobytes()
        assert np.array_equal(oo, roo) and out.tobytes() == rout
    finally:
        dist.destroy_process_group()
