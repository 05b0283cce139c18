"""bench.py's batch (bench.make_payloads) as request bodies through the pattern scan and request_logging_masking (SCAN|MASK, max_depth
10) with host buffers on both sides, timed three ways:

  sync      engine.run_batch in a loop: pinned packed stream in, verdicts and masked bodies back in pinned memory; every call waits for
            its upload, its kernels and its downloads (cf_run_batch)
  pipelined two engine.Run / Batch slots: the H2D of batch k+1 runs on a copy stream while the chain of batch k runs on the compute
            stream, and the D2H of batch k-1's verdicts, offsets and masked bodies runs on a third stream behind it (cf_run_enqueue /
            cf_run_finish)
  graph     one engine.Run whose enqueue was captured in a CUDA graph: per step the H2D, one replay, cf_run_finish and the D2H, one
            after the other on one stream

All three process the same batch --steps times after --warmup steps.  The last step's verdicts, offsets and masked bodies of the three
must be byte-identical, and a sample of the masked bodies must equal oracle/mask_ref.py.  Rates are payloads per second of wall clock
around the whole loop, ending in a device synchronise.

    python tools/run_mask_async_bench.py [--units 32768] [--steps 20] [--warmup 3] [--out DIR]

Prints one JSON document with the card's name, power limit and max SM clock (read in the same run).  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from run_async_bench import card  # noqa: E402  (tools/ is this script's directory)

MAX_DEPTH = 10


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON document to DIR/run_mask_async_bench.json")
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from mcp_context_forge_b200 import engine
    from mcp_context_forge_b200._native import CF_STAGE_MASK, CF_STAGE_SCAN, CF_V_MASKED
    from mcp_context_forge_b200.plugins.harmful_content_detector import DEFAULT_LEXICONS
    from oracle import mask_ref

    if not torch.cuda.is_available():
        raise SystemExit("run_mask_async_bench.py: no CUDA device")
    STAGES = CF_STAGE_SCAN | CF_STAGE_MASK
    ctx = engine.Context.get(0)
    prog = engine.Program()
    for pats in DEFAULT_LEXICONS.values():
        for pat in pats:
            prog.add_search(pat, re.I)
    prog.compile(ctx)
    payloads = bench.make_payloads()
    n = args.units
    units = [payloads[i % len(payloads)] for i in range(n)]
    stream, offs = engine.pack_units(units)
    nbytes = len(stream)
    h_stream = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    h_stream.numpy()[:] = np.frombuffer(stream, dtype=np.uint8)
    h_np = h_stream.numpy()

    def timed(step, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = step(steps)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    # ---- sync: cf_run_batch per step
    batch = engine.Batch(ctx, nbytes, n)

    def sync_loop(steps):
        for _ in range(steps):
            v, out, oo, _ = engine.run_batch(prog, batch, h_np, offs, STAGES, mask_max_depth=MAX_DEPTH)
        return v.tobytes(), oo.tobytes(), out[:int(oo[-1])].tobytes()

    sync_loop(args.warmup)
    sync_s, ref = timed(sync_loop, args.steps)
    del batch
    v_ref = np.frombuffer(ref[0], dtype=engine.VERDICT_DTYPE)
    oo_ref = np.frombuffer(ref[1], dtype=np.uint64)
    oracle_ok = True
    for i in (0, 1, 2, n // 2, n - 1):
        got = ref[2][int(oo_ref[i]):int(oo_ref[i + 1])] if v_ref["flags"][i] & CF_V_MASKED else None
        try:
            exp = mask_ref.mask_json_bytes(engine.encode_unit(units[i]), MAX_DEPTH)
        except ValueError:
            exp = None
        oracle_ok = oracle_ok and got == exp
    cap = int(oo_ref[-1]) + 4096

    # ---- pipelined: two slots
    dev = torch.device("cuda", 0)
    h2d, comp, d2h = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    W = prog.words
    slots = []
    for _ in range(2):
        slots.append({"batch": engine.Batch(ctx, nbytes, n), "run": engine.Run(ctx, n, nbytes),
                      "v": torch.empty(n * 24, dtype=torch.uint8, device=dev), "oo": torch.empty(n + 1, dtype=torch.int64, device=dev),
                      "out": torch.empty(cap, dtype=torch.uint8, device=dev), "bm": torch.empty(n * W, dtype=torch.int64, device=dev),
                      "hv": torch.empty(n * 24, dtype=torch.uint8, pin_memory=True), "hoo": torch.empty(n + 1, dtype=torch.int64, pin_memory=True),
                      "hout": torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                      "up": torch.cuda.Event(), "done": torch.cuda.Event(), "copied": torch.cuda.Event()})
    torch.cuda.synchronize()

    def enqueue(sl, stream):
        sl["run"].enqueue(prog, sl["batch"], STAGES, None, 0, sl["v"], sl["oo"], sl["out"], sl["bm"], stream=stream, mask_max_depth=MAX_DEPTH)

    def finish(sl):
        if sl["run"].finish():
            raise SystemExit("output buffer too small")

    def collect(sl):
        """After the slot's finish: its verdicts and offsets, then its masked bodies, on the D2H stream."""
        with torch.cuda.stream(d2h):
            sl["hv"].copy_(sl["v"], non_blocking=True)
            sl["hoo"].copy_(sl["oo"], non_blocking=True)
        d2h.synchronize()
        total = int(sl["hoo"][-1])
        with torch.cuda.stream(d2h):
            sl["hout"][:total].copy_(sl["out"][:total], non_blocking=True)
            sl["copied"].record(d2h)
        return total

    def result(sl, total):
        return sl["hv"].numpy().tobytes(), sl["hoo"].numpy().tobytes(), sl["hout"].numpy()[:total].tobytes()

    def pipelined(steps):
        pending = None
        for k in range(steps):
            sl = slots[k & 1]
            h2d.wait_event(sl["done"])                          # the slot's batch is no longer read by the chain of step k - 2
            sl["batch"].upload(h_np, offs, cuda_stream=h2d.cuda_stream)
            sl["up"].record(h2d)
            comp.wait_event(sl["up"])
            comp.wait_event(sl["copied"])                       # step k - 2's bodies have left the slot's buffers
            enqueue(sl, comp)
            sl["done"].record(comp)
            if pending is not None:                             # step k - 1: finished while step k runs, its D2H behind it
                finish(pending)
                pending["total"] = collect(pending)
            pending = sl
        finish(pending)
        pending["total"] = collect(pending)
        d2h.synchronize()
        return result(pending, pending["total"])

    pipelined(args.warmup)
    pipe_s, pipe_out = timed(pipelined, args.steps)

    # ---- graph: slot 0's run (warmed up above) captured once, replayed per step
    sl = slots[0]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enqueue(sl, torch.cuda.current_stream())

    def graph_loop(steps):
        for _ in range(steps):
            with torch.cuda.stream(s):
                sl["batch"].upload(h_np, offs, cuda_stream=s.cuda_stream)
                g.replay()
            finish(sl)
            with torch.cuda.stream(s):
                sl["hv"].copy_(sl["v"], non_blocking=True)
                sl["hoo"].copy_(sl["oo"], non_blocking=True)
            s.synchronize()
            total = int(sl["hoo"][-1])
            with torch.cuda.stream(s):
                sl["hout"][:total].copy_(sl["out"][:total], non_blocking=True)
            s.synchronize()
        return result(sl, total)

    graph_loop(args.warmup)
    graph_s, graph_out = timed(graph_loop, args.steps)

    equal = pipe_out == ref and graph_out == ref
    rate = lambda t: {"payloads_per_s": n * args.steps / t, "ms_per_step": 1e3 * t / args.steps}   # noqa: E731
    doc = {"card": card(), "units": n, "payload_bytes": bench.PAYLOAD_BYTES, "stream_bytes": nbytes, "masked_bytes": int(oo_ref[-1]),
           "masked_units": int(((v_ref["flags"] & CF_V_MASKED) != 0).sum()), "steps": args.steps, "stages": "SCAN|MASK", "max_depth": MAX_DEPTH,
           "outputs_equal": equal, "oracle_sample_ok": oracle_ok,
           "sync_cf_run_batch": rate(sync_s), "pipelined_two_runs": rate(pipe_s), "graph_one_run": rate(graph_s)}
    print(json.dumps(doc, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "run_mask_async_bench.json"), "w") as f:
            json.dump(doc, f, indent=1)
    return 0 if equal and oracle_ok else 1


if __name__ == "__main__":
    sys.exit(main())
