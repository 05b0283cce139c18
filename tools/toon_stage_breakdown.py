"""Where the TOON stage's time goes, by payload shape: cf_toon on a device-resident batch of bench.py's payloads.

For each case (shapes A tabular, B nested config, P prose-in-JSON alone, each tiled from bench.make_payloads()'s own payloads of
that shape, the bench mix itself, and mix_sorted = the mix's texts packed by shape, B then A then P) it times, with CUDA events over
warmed launches:
  flags = 0                the whole stage: token-parallel kernel (mixed list-item arrays retried in place) + the sequential encoder for
                           the units it hands over
  CF_TOON_NO_HANDOVER      the token-parallel kernel alone, first attempts only; the difference is the hand-over tail: the sequential
                           encoder's launch, plus the in-place retries' share of the kernel
and reports median / min / max in ms, and how many units the token-parallel kernel handed over.

usage: python tools/toon_stage_breakdown.py [--units 32768] [--reps 15] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from mcp_context_forge_b200 import engine  # noqa: E402

CF_TOON_NO_HANDOVER = 16     # include/cfgpu.h: handed-over units stay at status 7
TS_FALLBACK = 7


def shape_of(i: int) -> str:
    """bench.make_payloads()'s shape of payload i (the same golden-ratio draw over bench.MIX)."""
    r = (i * 0.61803398875) % 1.0
    acc = 0.0
    for s, w in bench.MIX:
        acc += w
        if r < acc:
            return s
    return "A"


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(",")) if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(), "?", "?")
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def time_case(ctx, texts, reps: int) -> dict:
    lib = ctx.lib
    stream, offs = engine.pack_units([t.encode() for t in texts])
    n = len(texts)
    batch = engine.Batch(ctx, len(stream), n)
    batch.upload(stream, offs)
    d_out = torch.empty(len(stream) + 16, dtype=torch.uint8, device="cuda")
    d_len = torch.empty(n, dtype=torch.int32, device="cuda")
    d_st = torch.empty(n, dtype=torch.int32, device="cuda")
    res = {"units": n, "bytes": len(stream)}
    for name, flags in (("stage", 0), ("tp_kernel", CF_TOON_NO_HANDOVER)):
        def launch():
            ctx.check(lib.cf_toon(ctx.h, batch.h, flags, d_out.data_ptr(), d_len.data_ptr(), d_st.data_ptr(), None), "cf_toon")
        for _ in range(3):
            launch()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res[name] = {"median_ms": float(np.median(ms)), "min_ms": min(ms), "max_ms": max(ms)}
        if flags == CF_TOON_NO_HANDOVER:
            res["handed_over"] = int((d_st == TS_FALLBACK).sum())
    res["handover_tail_ms"] = res["stage"]["median_ms"] - res["tp_kernel"]["median_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("toon_stage_breakdown.py: no CUDA device")
    ctx = engine.Context.get(0)
    payloads = bench.make_payloads()
    by_shape = {}
    for i, p in enumerate(payloads):
        by_shape.setdefault(shape_of(i), []).append(p)
    cases = {name: [base[i % len(base)] for i in range(args.units)]
             for name, base in (("A", by_shape["A"]), ("B", by_shape["B"]), ("P", by_shape["C"]), ("mix", payloads))}
    # the mix's own texts packed by shape, nested configs first: what the first pass costs when no CTA mixes shapes
    rank = {"B": 0, "A": 1, "C": 2}
    cases["mix_sorted"] = [payloads[i % len(payloads)]
                           for i in sorted(range(args.units), key=lambda i: rank[shape_of(i % len(payloads))])]
    out = {"card": card(), "cases": {}}
    print(json.dumps(out["card"]))
    for name, texts in cases.items():
        r = time_case(ctx, texts, args.reps)
        out["cases"][name] = r
        print(f"{name:4s} units {r['units']}  stage {r['stage']['median_ms']:.3f} ms [{r['stage']['min_ms']:.3f}, {r['stage']['max_ms']:.3f}]  "
              f"tp kernel {r['tp_kernel']['median_ms']:.3f} ms [{r['tp_kernel']['min_ms']:.3f}, {r['tp_kernel']['max_ms']:.3f}]  "
              f"hand-over tail {r['handover_tail_ms']:.3f} ms  handed over {r['handed_over']}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
