"""The bench batch (bench.make_payloads, bench.SUBS, SCAN|SUB|TOON) with host buffers on both sides, timed two ways:

  sync      engine.run_batch in a loop: pinned packed stream in, verdicts and texts back in pinned memory; every call waits for its
            upload, its kernels and its downloads (cf_run_batch)
  pipelined two engine.Run / Batch slots: the H2D of batch k+1 runs on a copy stream while the chain of batch k runs on the compute
            stream, and the D2H of batch k-1's verdicts, offsets and texts runs on a third stream behind it (cf_run_enqueue /
            cf_run_finish)

Both loops process the same batch --steps times after --warmup steps; the last step's verdicts, offsets and texts of the two loops
must be byte-identical.  Rates are payloads per second of wall clock around the whole loop, ending in a device synchronise.

    python tools/run_async_bench.py [--units 32768] [--steps 20] [--warmup 3] [--hit-rate 1e-4] [--out DIR]

Prints one JSON document with the card's name, power limit and max SM clock (read in the same run).  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--hit-rate", type=float, default=1e-4)
    ap.add_argument("--out", help="also write the JSON document to DIR/run_async_bench.json")
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from mcp_context_forge_b200 import engine
    from mcp_context_forge_b200._native import CF_STAGE_SCAN, CF_STAGE_SUB, CF_STAGE_TOON
    from mcp_context_forge_b200.plugins.harmful_content_detector import DEFAULT_LEXICONS

    if not torch.cuda.is_available():
        raise SystemExit("run_async_bench.py: no CUDA device")
    STAGES = CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_TOON
    ctx = engine.Context.get(0)
    prog = engine.Program()
    for pats in DEFAULT_LEXICONS.values():
        for pat in pats:
            prog.add_search(pat, re.I)
    for s, f, r in bench.SUBS:
        prog.add_sub(s, f, r)
    prog.compile(ctx)
    payloads = bench.make_payloads(hit_rate=args.hit_rate)
    n = args.units
    stream, offs = engine.pack_units([payloads[i % len(payloads)] for i in range(n)])
    nbytes = len(stream)
    h_stream = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    h_stream.numpy()[:] = np.frombuffer(stream, dtype=np.uint8)
    h_np = h_stream.numpy()

    # ---- sync: cf_run_batch per step
    batch = engine.Batch(ctx, nbytes, n)
    last = {}

    def step_sync():
        v, out, oo, _ = engine.run_batch(prog, batch, h_np, offs, STAGES)
        last["sync"] = (v, out, oo)

    for _ in range(args.warmup):
        step_sync()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step_sync()
    torch.cuda.synchronize()
    sync_s = time.perf_counter() - t0
    v_s, out_s, oo_s = last["sync"]
    ref = (v_s.tobytes(), oo_s.tobytes(), out_s[:int(oo_s[-1])].tobytes())
    del batch

    # ---- pipelined: two slots
    dev = torch.device("cuda", 0)
    h2d, comp, d2h = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    W = prog.words
    cap = nbytes + 4096
    slots = []
    for _ in range(2):
        slots.append({"batch": engine.Batch(ctx, nbytes, n), "run": engine.Run(ctx, n, nbytes),
                      "v": torch.empty(n * 24, dtype=torch.uint8, device=dev), "oo": torch.empty(n + 1, dtype=torch.int64, device=dev),
                      "out": torch.empty(cap, dtype=torch.uint8, device=dev), "bm": torch.empty(n * W, dtype=torch.int64, device=dev),
                      "hv": torch.empty(n * 24, dtype=torch.uint8, pin_memory=True), "hoo": torch.empty(n + 1, dtype=torch.int64, pin_memory=True),
                      "hout": torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                      "up": torch.cuda.Event(), "done": torch.cuda.Event(), "copied": torch.cuda.Event()})
    torch.cuda.synchronize()

    def collect(sl):
        """After the slot's finish: its verdicts and offsets, then its texts, on the D2H stream (behind nothing but other copies)."""
        with torch.cuda.stream(d2h):
            sl["hv"].copy_(sl["v"], non_blocking=True)
            sl["hoo"].copy_(sl["oo"], non_blocking=True)
        d2h.synchronize()
        total = int(sl["hoo"][-1])
        with torch.cuda.stream(d2h):
            sl["hout"][:total].copy_(sl["out"][:total], non_blocking=True)
            sl["copied"].record(d2h)
        return total

    def pipelined(steps):
        pending = None
        for k in range(steps):
            sl = slots[k & 1]
            h2d.wait_event(sl["done"])                          # the slot's batch is no longer read by the chain of step k - 2
            sl["batch"].upload(h_np, offs, cuda_stream=h2d.cuda_stream)
            sl["up"].record(h2d)
            comp.wait_event(sl["up"])
            comp.wait_event(sl["copied"])                       # step k - 2's texts have left the slot's buffers
            sl["run"].enqueue(prog, sl["batch"], STAGES, None, 0, sl["v"], sl["oo"], sl["out"], sl["bm"], stream=comp)
            sl["done"].record(comp)
            if pending is not None:                             # step k - 1: finished while step k runs, its D2H behind it
                if pending["run"].finish():
                    raise SystemExit("output buffer too small")
                pending["total"] = collect(pending)
            pending = sl
        if pending["run"].finish():
            raise SystemExit("output buffer too small")
        pending["total"] = collect(pending)
        d2h.synchronize()
        return pending

    pipelined(args.warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sl = pipelined(args.steps)
    torch.cuda.synchronize()
    pipe_s = time.perf_counter() - t0
    got = (sl["hv"].numpy().tobytes(), sl["hoo"].numpy().tobytes(), sl["hout"].numpy()[:sl["total"]].tobytes())
    equal = got == ref

    doc = {"card": card(), "units": n, "payload_bytes": bench.PAYLOAD_BYTES, "stream_bytes": nbytes, "hit_rate": args.hit_rate, "steps": args.steps,
           "stages": "SCAN|SUB|TOON", "outputs_equal": equal,
           "sync_cf_run_batch": {"payloads_per_s": n * args.steps / sync_s, "ms_per_step": 1e3 * sync_s / args.steps},
           "pipelined_two_runs": {"payloads_per_s": n * args.steps / pipe_s, "ms_per_step": 1e3 * pipe_s / args.steps},
           "speedup": sync_s / pipe_s}
    print(json.dumps(doc, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "run_async_bench.json"), "w") as f:
            json.dump(doc, f, indent=1)
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
