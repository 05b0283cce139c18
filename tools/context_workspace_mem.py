"""Device memory one context holds after each step of a sequence that reaches every entry point taking device workspace from it.

The sequence runs three times, on batches of about --mib MiB, then a quarter of that, then 1.5 times it (past the headroom of the
context's run): cf_run_batch SCAN|SUB, SCAN|SUB|TOON with host buffers and with the outputs left in HBM, cf_toon on a torch stream,
cf_sub_host, cf_scan_host, cf_json_index_host, cf_classify_keys_host, cf_toon_host (default, sequential, parse-only) and cf_run_batch
SCAN|MASK.  After each step the device's used memory (torch.cuda.mem_get_info) is printed relative to the fresh context, in MiB.  At
64 MiB batches the workspaces are far above the 2 MiB allocation granularity, so a buffer that one build keeps and another does not
shows in the column.

    python tools/context_workspace_mem.py [--mib 64] [--root TREE] [--out result.json]

--root imports the package from another checkout of this repository (built in place), so that two builds can be compared from one
command.  The numbers are device-wide: other processes on the same GPU show in them too."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import re
import sys

STEPS = ["run_batch SCAN|SUB", "run_batch SCAN|SUB|TOON", "run_batch SCAN|SUB|TOON resident", "cf_toon (torch stream)", "cf_sub_host",
         "cf_scan_host", "cf_json_index_host", "cf_classify_keys_host", "cf_toon_host", "cf_toon_host SEQUENTIAL", "cf_toon_host PARSE_ONLY",
         "run_batch SCAN|MASK"]
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes"), ("~", 0, "-" * 200)]


def units_of(synth, target_bytes):
    """Distinct tool results of every shape (JSON tabular and nested, prose with hits, rewritten units, bodies whose masked output
    outgrows their first room), repeated up to target_bytes."""
    base = [synth.payload("A", 4000, seed=s) for s in range(40)] + [synth.payload("B", 3000, seed=s) for s in range(40)]
    base += [synth.payload("C", 4000, seed=s, hit_rate=2e-3) for s in range(40)]
    base += ["this is crap", "Kill him now", "crap " * 2000, "~" * 1000, json.dumps({"rows": [{"id": i, "t": "crap"} for i in range(20)]}), ""]
    base += ['{"k":[' + ",".join(["[]"] * m) + "]}" for m in (40, 400)]
    per = sum(len(u.encode()) + 1 for u in base)
    return base * max(1, round(target_bytes / per))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=float, default=64.0)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    import torch

    from mcp_context_forge_b200 import _native as N
    from mcp_context_forge_b200 import engine, synth
    from oracle import hook_chain_ref as ref

    def used():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info()
        return total - free

    torch.cuda.init()
    base = used()
    ctx = engine.Context(0)
    prog = engine.Program()
    for p in (p for pats in ref.DEFAULT_LEXICONS.values() for p in pats):
        prog.add_search(p, re.I)
    for w in ("innovative", "groundbreaking", "revolutionary"):
        prog.add_literal(w)
    for p, f, r in SUBS:
        prog.add_sub(p, f, r)
    prog.compile(ctx)
    start = used()
    rows = []
    for phase, scale in (("grow", 1.0), ("shrink", 0.25), ("grow past", 1.5)):
        units = units_of(synth, int(args.mib * scale * (1 << 20)))
        stream, offs = engine.pack_units(units)
        n = len(units)
        batch = engine.Batch(ctx, len(stream), n)
        chain = N.CF_STAGE_SCAN | N.CF_STAGE_SUB | N.CF_STAGE_TOON
        dirty = [i for i, u in enumerate(units) if "crap" in u or "crud" in u or "~" in u]

        def toon_dev():
            s = torch.cuda.Stream()
            out = torch.empty(len(stream), dtype=torch.uint8, device="cuda")
            ln = torch.empty(n, dtype=torch.int32, device="cuda")
            st = torch.empty(n, dtype=torch.int32, device="cuda")
            s.wait_stream(torch.cuda.current_stream())
            batch.upload(stream, offs, cuda_stream=s.cuda_stream)
            ctx.check(ctx.lib.cf_toon(ctx.h, batch.h, 1, out.data_ptr(), ln.data_ptr(), st.data_ptr(), ctypes.c_void_p(s.cuda_stream)), "cf_toon")
            s.synchronize()

        def toon_host(flags):
            out, ln, st = np.empty(len(stream), np.uint8), np.empty(n, np.uint32), np.empty(n, np.int32)
            ctx.check(ctx.lib.cf_toon_host(ctx.h, batch.h, flags, ctypes.cast(ctypes.c_char_p(stream), ctypes.c_void_p), len(stream), offs.ctypes.data, n,
                                           out.ctypes.data, ln.ctypes.data, st.ctypes.data), "cf_toon_host")

        steps = [lambda: engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_SUB),
                 lambda: engine.run_batch(prog, batch, stream, offs, chain),
                 lambda: (engine.run_batch(prog, batch, stream, offs, chain, outputs_resident=True), engine.device_output(ctx)),
                 toon_dev,
                 lambda: engine.sub_host(prog, batch, dirty),
                 lambda: engine.scan_host(prog, batch, stream, offs),
                 lambda: engine.json_index_host(batch, stream, offs),
                 lambda: engine.classify_keys_host(batch, ["password", "authToken", "token_count", "name"] * 64),
                 lambda: toon_host(1), lambda: toon_host(8 | 1), lambda: toon_host(4),
                 lambda: engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SCAN | N.CF_STAGE_MASK, mask_max_depth=2)]
        for name, step in zip(STEPS, steps):
            step()
            rows.append({"phase": phase, "batch_mib": round(len(stream) / (1 << 20), 1), "units": n, "step": name,
                         "used_mib": round((used() - start) / (1 << 20), 1)})
            print(f"{phase:10s} {rows[-1]['batch_mib']:7.1f} MiB {n:7d} units  {name:34s} {rows[-1]['used_mib']:9.1f} MiB", flush=True)
        del batch
    res = {"device": torch.cuda.get_device_name(0), "context_and_program_mib": round((start - base) / (1 << 20), 1), "rows": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
