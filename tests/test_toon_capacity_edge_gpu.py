"""GPU: the documents of tests/test_toon_capacity_edge_cpu.py at the edge of toon_encoder's "strictly smaller" decision (n = L - 1
.. L + 2, and the trimming family swept across its window) through every route that takes the decision: cf_toon_host on the default
route, with CF_TOON_REPORT_ERRORS, CF_TOON_SEQUENTIAL and CF_TOON_NO_HANDOVER; cf_run_batch(CF_STAGE_TOON); engine.Run; the
toon_encoder plugin and BatchedPluginManager at the plugin's default min_size_bytes.  Every answer is compared with the oracle
(oracle/toon_ref.py), never with another GPU route.

The edge documents sit among ordinary neighbours in launches of about 200, 6 000 and 40 000 units, where the sequential kernel's
warps walk 1, 4 and 32 units each (cfjson.cu units_per_warp on an H100) and the token-parallel kernel meets the boundary at many
unit alignments."""
import asyncio
import os
import random
import tempfile
import time

import numpy as np
import pytest
import torch

import test_toon_capacity_edge_cpu as E
from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine, synth
from mcp_context_forge_b200 import framework as fw
from mcp_context_forge_b200.manager import BatchedPluginManager
from mcp_context_forge_b200.plugins.toon_encoder import ToonEncoderPlugin
from oracle import toon_ref

pytestmark = pytest.mark.gpu

REPORT_ERRORS, SEQUENTIAL, NO_HANDOVER = 1, 8, 16
PACKINGS = (100, 3000, None)          # edge documents per launch, as many neighbours beside them: 200, 6 000 and 40 000 units
TOTAL_UNITS = 40000
PLUGIN_MIN = 100                      # ToonEncoderPlugin's default min_size_bytes
CTX = fw.PluginContext(global_context=fw.GlobalContext(request_id="t"))
YAML = """
plugins:
  - name: "ToonEncoder"
    kind: "mcp_context_forge_b200.plugins.toon_encoder.ToonEncoderPlugin"
    hooks: ["tool_post_invoke"]
    mode: "sequential"
    priority: 900
plugin_settings:
  plugin_timeout: 120
"""


# --------------------------------------------------------------------------------------------------------------------- corpora
@pytest.fixture(scope="module")
def corpus():
    """(documents, oracle answers, trimming-family flags): the edge corpus, the trimming sweep and the error documents."""
    docs = [d for d, _ in E.edge_corpus()]
    n_edge = len(docs)
    docs += [d for d, _, _ in E.trim_sweep()]
    n_trim = len(docs) - n_edge
    for d in E.error_docs():
        c, gaps = E.compact(d)
        docs += [E.pad(c, gaps, k, E.WHERE[k % 3]) for k in range(0, 48, 3)]
    trim = [n_edge <= i < n_edge + n_trim for i in range(len(docs))]
    return docs, [E.oracle(d) for d in docs], trim


NEIGHBOURS = [synth.payload("AB"[i % 2], 300 + 97 * i, seed=i) for i in range(48)]
NEIGHBOUR_EXP = [E.oracle(d) for d in NEIGHBOURS]


def packed(idx, n_units, seed):
    """Unit list: the corpus indices `idx` at random places among neighbours (negative entries -1 - k: neighbour k)."""
    rng = random.Random(seed)
    units = [-1 - rng.randrange(len(NEIGHBOURS)) for _ in range(max(n_units - len(idx), 0))]
    for i in idx:
        units.insert(rng.randrange(len(units) + 1), i)
    return units


def launches(n_docs):
    """[(packing, unit list)] covering the corpus once per packing."""
    out = []
    for per in PACKINGS:
        if per is None:
            out.append(("40000", packed(list(range(n_docs)), max(TOTAL_UNITS, n_docs + 1000), 3)))
            continue
        for lo in range(0, n_docs, per):
            idx = list(range(lo, min(lo + per, n_docs)))
            out.append((str(2 * per), packed(idx, 2 * per, lo)))
    return out


# ---------------------------------------------------------------------------------------------------------------------- routes
def toon_host(ctx, stream, offs, n, flags):
    status, texts, out_len = engine.toon_host_flags(engine.Batch(ctx, len(stream), n), stream, offs, flags)
    return [(int(s), None if t is None else t.decode("utf-8")) for s, t in zip(status, texts)], out_len.tolist()


def from_verdicts(v, raw, oo):
    res = []
    for i in range(len(v)):
        s = int(v["aux"][i])
        assert bool(v["flags"][i] & N.CF_V_TOON) == (s == 0), (i, s)
        res.append((s, raw[int(oo[i]):int(oo[i + 1])].decode("utf-8") if s == 0 else None))
    return res


def run_batch(ctx, stream, offs, n):
    batch = engine.Batch(ctx, len(stream), n)
    v, out, oo, _ = engine.run_batch(None, batch, stream, offs, N.CF_STAGE_TOON)
    return from_verdicts(v, out[:int(oo[-1])].tobytes(), oo)


def run_enqueue(ctx, stream, offs, n):
    batch = engine.Batch(ctx, len(stream), n)
    run = engine.Run(ctx, n, len(stream))
    v = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
    oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    out = torch.full((max(len(stream), 1),), 0xAB, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    batch.upload(stream, offs, cuda_stream=s.cuda_stream)
    run.enqueue(None, batch, N.CF_STAGE_TOON, None, 0, v, oo, out, stream=s)
    assert run.finish() == 0
    return from_verdicts(v.cpu().numpy().view(engine.VERDICT_DTYPE), out.cpu().numpy().tobytes(), oo.cpu().numpy().view(np.uint64))


ROUTES = {"default": lambda c, s, o, n: toon_host(c, s, o, n, 0), "report-errors": lambda c, s, o, n: toon_host(c, s, o, n, REPORT_ERRORS),
          "sequential": lambda c, s, o, n: toon_host(c, s, o, n, SEQUENTIAL),
          "no-handover": lambda c, s, o, n: toon_host(c, s, o, n, REPORT_ERRORS | NO_HANDOVER),
          "run_batch": lambda c, s, o, n: (run_batch(c, s, o, n), None), "run": lambda c, s, o, n: (run_enqueue(c, s, o, n), None)}
REPORTS = {"report-errors", "no-handover"}


@pytest.mark.parametrize("route", list(ROUTES))
def test_capacity_edge_on_the_c_abi(corpus, route):
    t0 = time.perf_counter()
    docs, exps, trim = corpus
    ctx = engine.Context.get()
    report = route in REPORTS
    compared, handed = 0, 0
    for packing, units in launches(len(docs)):
        texts = [docs[u] if u >= 0 else NEIGHBOURS[-1 - u] for u in units]
        stream, offs = engine.pack_units([engine.encode_unit(t) for t in texts])
        got, why = ROUTES[route](ctx, stream, offs, len(units))
        for j, (u, g) in enumerate(zip(units, got)):
            e = exps[u] if u >= 0 else NEIGHBOUR_EXP[-1 - u]
            if route == "no-handover" and g[0] == E.HANDED_OVER:
                assert why[j] == E.FB_KEY_ESCAPE if u >= 0 and trim[u] else why[j] in E.FB_REASONS, (packing, texts[j][:160], why[j])
                handed += 1
                continue
            assert E.agrees(g, e, report), (route, packing, texts[j][:160], g[0], e[0], (g[1] or "")[:80], (e[1] or "")[:80])
            compared += u >= 0
    if route == "no-handover":                       # the units the token-parallel kernel decides itself
        assert compared > 1000 * len(PACKINGS) and handed > 0
    else:
        assert compared == len(docs) * len(PACKINGS) and handed == 0
    print(f"\n{route}: {len(docs)} edge documents x {len(PACKINGS)} packings, {compared} compared, {handed} handed over, "
          f"{time.perf_counter() - t0:.1f}s")


def plugin_docs(corpus):
    docs, _, trim = corpus
    out = [(d, t) for d, t in zip(docs, trim) if len(d.encode("utf-8")) >= PLUGIN_MIN]
    out += [(d, False) for d in E.base_docs()[:50] if len(d.encode("utf-8")) < PLUGIN_MIN]   # below the minimum: left alone
    return [d for d, _ in out], [toon_ref.process_text(d) for d, _ in out], [t for _, t in out]


def check_items(docs, exps, trim, results):
    """Every item against the oracle; returns (items converted, of them trimming-family ones)."""
    n_conv = n_window = 0
    for d, e, t, r in zip(docs, exps, trim, results):
        if e is None:
            assert r.modified_payload is None, d[:160]
            continue
        assert r.modified_payload is not None, d[:160]
        item = r.modified_payload.result["content"][0]
        assert item["text"] == e and item["annotations"] == {"format": "toon"}, d[:160]
        n_conv += 1
        n_window += t
    return n_conv, n_window


def test_capacity_edge_through_the_plugin(corpus):
    docs, exps, trim = plugin_docs(corpus)
    plug = ToonEncoderPlugin(fw.PluginConfig(name="toon", kind="x", hooks=["tool_post_invoke"]))

    async def many():
        return await asyncio.gather(*[plug.tool_post_invoke(fw.ToolPostInvokePayload(name="t", result={"content": [{"type": "text", "text": d}]}), CTX)
                                      for d in docs])

    n_conv, n_trim = check_items(docs, exps, trim, asyncio.new_event_loop().run_until_complete(many()))
    assert n_conv > len(docs) // 3 and n_trim > 1000, (n_conv, n_trim)


def test_capacity_edge_through_the_batched_manager(corpus):
    docs, exps, trim = plugin_docs(corpus)
    with tempfile.TemporaryDirectory() as td:
        cfg = os.path.join(td, "plugins.yaml")
        with open(cfg, "w") as f:
            f.write(YAML)
        mgr = BatchedPluginManager(cfg, timeout=120)
        loop = asyncio.new_event_loop()
        loop.run_until_complete(mgr.initialize())
        n_conv = n_trim = 0
        for lo in range(0, len(docs), 4000):
            part = slice(lo, lo + 4000)

            async def wave():
                return await asyncio.gather(*[mgr.invoke_hook("tool_post_invoke", fw.ToolPostInvokePayload(name="t", result={"content": [{"type": "text", "text": d}]}),
                                                              fw.GlobalContext(request_id=f"r{i}")) for i, d in enumerate(docs[part])])

            a, b = check_items(docs[part], exps[part], trim[part], [r[0] for r in loop.run_until_complete(wave())])
            n_conv, n_trim = n_conv + a, n_trim + b
        loop.run_until_complete(mgr.shutdown())
    assert n_conv > len(docs) // 3 and n_trim > 1000, (n_conv, n_trim)
