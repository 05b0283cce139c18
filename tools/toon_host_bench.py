"""Steady-state time of the per-plugin TOON path, engine.toon_host (cf_toon_host: upload, encode, texts back in the input's layout),
which GpuBatcher.toon and the toon_encoder drop-in call.  bench.py does not measure it.

Shapes at bench.py's sizes, 2 048 to 32 768 units of 2 to 256 KiB: A (tabular) and B (nested config) at 2 and 16 KiB, M (bench.py's
mixed 2 / 16 / 256 KiB tabular payloads, 80 / 19 / 1 % by count) and A at 256 KiB.  Each case warms up, then times --calls calls
with torch.cuda.synchronize around each; the median and min per call are printed with the card's name and power limit.

    python tools/toon_host_bench.py [--calls 10] [--root TREE] [--out result.json]

--root imports the package from another checkout of this repository (built in place), so that two builds can be timed by one
command."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

CASES = [("A", 2048, 32768), ("A", 16384, 32768), ("B", 2048, 32768), ("B", 16384, 16384), ("M", 0, 32768), ("A", 262144, 2048)]


def texts_of(synth, shape, size, n):
    if shape == "M":
        pool = {k: [synth.payload("A", k, seed=s).encode() for s in range(8)] for k in (2048, 16384, 262144)}
        return [pool[262144 if i % 100 == 0 else 16384 if i % 5 == 0 else 2048][i % 8] for i in range(n)]
    base = [synth.payload(shape, size, seed=s).encode() for s in range(64)]
    return [base[i % 64] for i in range(n)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch

    from mcp_context_forge_b200 import engine, synth

    ctx = engine.Context.get()
    rows = []
    for shape, size, n in CASES:
        stream, offs = engine.pack_units(texts_of(synth, shape, size, n))
        batch = engine.Batch(ctx, len(stream), n)
        converted = 0
        for _ in range(args.warmup):
            converted = int((engine.toon_host(batch, stream, offs)[0] == engine.TOON_CONVERTED).sum())
        ms = []
        for _ in range(args.calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            engine.toon_host(batch, stream, offs)
            torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
        rows.append({"shape": shape, "payload_bytes": size, "units": n, "stream_mib": round(len(stream) / (1 << 20), 1), "converted": converted,
                     "median_ms": round(statistics.median(ms), 2), "min_ms": round(min(ms), 2)})
        print(f"{shape} {size:7d} B x {n:6d}  {rows[-1]['stream_mib']:7.1f} MiB  converted {converted:6d}  median {rows[-1]['median_ms']:8.2f} ms  "
              f"min {rows[-1]['min_ms']:8.2f} ms", flush=True)
        del batch
    res = {"device": card(), "root": os.path.abspath(args.root), "calls": args.calls, "rows": rows}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
