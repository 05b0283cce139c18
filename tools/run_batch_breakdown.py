"""Where the time of one resident cf_run_batch goes, at bench.py's batch (32 768 x 16 KiB, bench.make_payloads).

For SCAN|TOON and SCAN|SUB|TOON at hit rates 0, 1e-4 and 1e-2: the wall time of each call (cf_run_batch is synchronous), the scan and
TOON kernels from the library's own event pairs (cf_profile_collect_each), and post = wall - scan - TOON, the time the call spends
outside those two kernels.  Median and spread (min / max) over --steps calls.  Then, in a separate run per case, a torch.profiler trace
(written to --out) from which the CUDA launches, memcpys and runtime calls per cf_run_batch are counted.

    python tools/run_batch_breakdown.py --out DIR [--steps 20] [--units 32768]

Prints one JSON document and writes it to DIR/run_batch_breakdown.json.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import collections
import ctypes
import json
import os
import re
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HIT_RATES = (0.0, 1e-4, 1e-2)


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001 - reported, not fatal
        return {"error": str(exc)[:200]}


def spread(xs) -> dict:
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the JSON result and the profiler traces")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--trace-steps", type=int, default=5)
    args = ap.parse_args()
    if args.steps < 10:
        ap.error("--steps must be at least 10")
    os.makedirs(args.out, exist_ok=True)

    import numpy as np
    import torch

    import bench
    from mcp_context_forge_b200 import engine
    from mcp_context_forge_b200._native import CF_STAGE_SCAN, CF_STAGE_SUB, CF_STAGE_TOON, CF_V_REWRITTEN, CF_V_TOON
    from mcp_context_forge_b200.plugins.harmful_content_detector import DEFAULT_LEXICONS

    if not torch.cuda.is_available():
        raise SystemExit("run_batch_breakdown.py: no CUDA device")
    ctx = engine.Context.get(0)
    lib = ctx.lib
    prog = engine.Program()                      # bench.py's program: the harmful lexicons + the regex_filter rules
    for pats in DEFAULT_LEXICONS.values():
        for pat in pats:
            prog.add_search(pat, re.I)
    for s, f, r in bench.SUBS:
        prog.add_sub(s, f, r)
    prog.compile(ctx)
    masks = {"SCAN|TOON": CF_STAGE_SCAN | CF_STAGE_TOON, "SCAN|SUB|TOON": CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_TOON}

    result = {"gpu": gpu_info(), "units": args.units, "steps": args.steps, "cases": []}
    for hr in HIT_RATES:
        payloads = bench.make_payloads(hit_rate=hr)
        units = [payloads[i % len(payloads)] for i in range(args.units)]
        stream, offs = engine.pack_units(units)
        batch = engine.Batch(ctx, len(stream), args.units)
        batch.upload(np.frombuffer(stream, dtype=np.uint8), offs)
        torch.cuda.synchronize()
        for mname, mask in masks.items():
            def call():
                return engine.run_batch(prog, batch, None, offs, mask, outputs_resident=True)[0]

            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            walls = []
            ctx.check(lib.cf_profile_begin(ctx.h, 2 * args.steps), "profile_begin")
            for _ in range(args.steps):
                t0 = time.perf_counter()
                v = call()
                walls.append((time.perf_counter() - t0) * 1e3)
            each = (ctypes.c_double * (2 * args.steps))()
            kn = ctypes.c_uint32()
            ctx.check(lib.cf_profile_collect_each(ctx.h, each, 2 * args.steps, ctypes.byref(kn)), "profile_collect_each")
            ctx.check(lib.cf_profile_begin(ctx.h, 0), "profile_end")
            if kn.value != 2 * args.steps:
                raise SystemExit(f"run_batch_breakdown.py: expected {2 * args.steps} kernel timings, got {kn.value}")
            scan = [each[2 * i] for i in range(args.steps)]
            toon = [each[2 * i + 1] for i in range(args.steps)]
            post = [w - s - t for w, s, t in zip(walls, scan, toon)]

            # separate run under the profiler: what one call enqueues
            acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
            with torch.profiler.profile(activities=acts) as prof:
                for _ in range(args.trace_steps):
                    call()
                torch.cuda.synchronize()
            tag = f"{mname.replace('|', '_')}_hr{hr:g}"
            trace = os.path.join(args.out, f"trace_{tag}.json")
            prof.export_chrome_trace(trace)
            with open(trace, encoding="utf-8") as f:
                evs = json.load(f)
            evs = evs.get("traceEvents", evs) if isinstance(evs, dict) else evs
            counts = {"kernel": collections.Counter(), "gpu_memcpy": collections.Counter(), "gpu_memset": collections.Counter(),
                      "cuda_runtime": collections.Counter()}
            for e in evs:
                if e.get("ph") == "X" and e.get("cat") in counts:
                    counts[e["cat"]][e["name"]] += 1
            per_call = {cat: {k: n / args.trace_steps for k, n in sorted(c.items())} for cat, c in counts.items()}
            result["cases"].append({
                "stages": mname, "hit_rate": hr,
                "rewritten_units": int(((v["flags"] & CF_V_REWRITTEN) != 0).sum()),
                "toon_units": int(((v["flags"] & CF_V_TOON) != 0).sum()),
                "wall_ms": spread(walls), "scan_ms": spread(scan), "toon_ms": spread(toon), "post_ms": spread(post),
                "per_call": {"launches": sum(per_call["kernel"].values()), "memcpys": sum(per_call["gpu_memcpy"].values()),
                             "memsets": sum(per_call["gpu_memset"].values()), **per_call},
                "trace": os.path.basename(trace)})
            c = result["cases"][-1]
            print(f"{mname:14s} hr={hr:<6g} rewritten={c['rewritten_units']:5d}  wall {c['wall_ms']['median']:7.3f} ms  scan {c['scan_ms']['median']:6.3f}  "
                  f"toon {c['toon_ms']['median']:7.3f}  post {c['post_ms']['median']:6.3f} [{c['post_ms']['min']:.3f}, {c['post_ms']['max']:.3f}]  "
                  f"launches/call {c['per_call']['launches']:g}  memcpys/call {c['per_call']['memcpys']:g}", file=sys.stderr)
        del batch
    with open(os.path.join(args.out, "run_batch_breakdown.json"), "w", encoding="utf-8") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
