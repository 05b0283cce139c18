"""Where the token-parallel TOON kernel's cycles go inside a unit, by phase and payload shape.

Builds libcfgpu.so with -DCF_TOON_PHASES into a scratch directory (the library in the tree is not touched), then runs cf_toon over
the same cases as tools/toon_stage_breakdown.py (shapes A tabular, B nested config, P prose-in-JSON, and the bench mix, 32 768 units
each) and prints, per case, the clock64() cycles per unit each phase took (summed over the warps, lane 0's clock):
  tokenize      bytes -> token array
  an_generic    analyze's generic bracket walk (an_batch)       an_table   analyze's table rows (an_rows)
  em_generic    emit's generic walk (em_batch)                  em_table   emit's table rows (em_rows)
  resolve       the in-place retry of mixed list-item arrays (its analyze and emit count here only)
and, on a second line per case, tokenize split into its parts (cycles per unit and share of tokenize):
  load          the step's loads and the source window's shift
  masks         mask algebra and the warp scans (separators, open strings, token ranks)
  ring          the per-kind ring passes (brackets, strings, scalar runs)
  classify      tok_batch without the long-string checks
  long          tok_batch's per-string pass over long non-ASCII / escaped strings (warp_escapes, first / last code point)
The timing itself costs cycles (clock reads, one atomic per phase call), so the numbers are for comparing phases and builds, not
for adding up to the stage time.

--build-only DIR builds into DIR and stops; --so DIR/libcfgpu.so then times that library instead of building one.

usage: python tools/toon_phase_breakdown.py [--units 32768] [--reps 5] [--build-only DIR | --so LIB] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import concurrent.futures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

PHASES = ("tokenize", "an_generic", "an_table", "em_generic", "em_table", "resolve")   # json_tp.h PH_*
TK_PHASES = ("load", "masks", "ring", "batch", "long")                                # json_tp.h PH_TK_* (batch includes long)
TK_SHOWN = ("load", "masks", "ring", "classify", "long")


def build_variant(outdir: str) -> str:
    from mcp_context_forge_b200 import build
    os.makedirs(outdir, exist_ok=True)
    flags = build.NVCC_FLAGS + ["-DCF_TOON_PHASES", "-I", build.INC]

    def compile_one(src):
        obj = os.path.join(outdir, os.path.splitext(src)[0] + ".o")
        subprocess.run([build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, src), "-o", obj], check=True)
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=len(build.SOURCES)) as ex:
        objs = list(ex.map(compile_one, build.SOURCES))
    so = os.path.join(outdir, "libcfgpu.so")
    subprocess.run([build._nvcc()] + build.ARCH + ["-shared", "-cudart", "static", "-o", so] + objs, check=True)
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--build-only", metavar="DIR")
    ap.add_argument("--so", metavar="LIB")
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if args.build_only:
        print(build_variant(args.build_only))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("toon_phase_breakdown.py: no CUDA device")
    so = args.so or build_variant(tempfile.mkdtemp(prefix="toon_phases_"))
    from mcp_context_forge_b200 import _native
    _native.SO_PATH = so                       # before anything loads the library
    import bench
    from mcp_context_forge_b200 import engine
    import toon_stage_breakdown as tsb

    ctx = engine.Context.get(0)
    lib = ctx.lib
    read = ctypes.CDLL(so).cf_toon_phase_cycles
    read.restype = ctypes.c_int
    read.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
    cyc = (ctypes.c_ulonglong * (len(PHASES) + len(TK_PHASES)))()

    payloads = bench.make_payloads()
    by_shape = {}
    for i, p in enumerate(payloads):
        by_shape.setdefault(tsb.shape_of(i), []).append(p)
    cases = {name: [base[i % len(base)] for i in range(args.units)]
             for name, base in (("A", by_shape["A"]), ("B", by_shape["B"]), ("P", by_shape["C"]), ("mix", payloads))}
    out = {"card": tsb.card(), "units": args.units, "reps": args.reps, "cases": {}}
    print(json.dumps(out["card"]))
    print(f"{'case':5s}" + "".join(f"{p:>12s}" for p in PHASES) + f"{'total':>12s}   (cycles per unit)")
    for name, texts in cases.items():
        stream, offs = engine.pack_units([t.encode() for t in texts])
        n = len(texts)
        batch = engine.Batch(ctx, len(stream), n)
        batch.upload(stream, offs)
        d_out = torch.empty(len(stream) + 16, dtype=torch.uint8, device="cuda")
        d_len = torch.empty(n, dtype=torch.int32, device="cuda")
        d_st = torch.empty(n, dtype=torch.int32, device="cuda")

        def launch():
            ctx.check(lib.cf_toon(ctx.h, batch.h, 0, d_out.data_ptr(), d_len.data_ptr(), d_st.data_ptr(), None), "cf_toon")
        launch()
        torch.cuda.synchronize()
        assert read(cyc) == 0
        for _ in range(args.reps):
            launch()
        torch.cuda.synchronize()
        assert read(cyc) == 0
        per = {p: cyc[k] / (args.reps * n) for k, p in enumerate(PHASES)}
        tk = {p: cyc[len(PHASES) + k] / (args.reps * n) for k, p in enumerate(TK_PHASES)}
        tk["classify"] = tk.pop("batch") - tk["long"]
        tot = sum(per.values())
        ttk = per["tokenize"]
        out["cases"][name] = {"cycles_per_unit": per, "share": {p: (v / tot if tot else 0.0) for p, v in per.items()},
                              "tokenize_cycles_per_unit": tk, "tokenize_share": {p: (v / ttk if ttk else 0.0) for p, v in tk.items()}}
        print(f"{name:5s}" + "".join(f"{per[p]:12.0f}" for p in PHASES) + f"{tot:12.0f}")
        print(f"{'':5s}" + "".join(f"{100 * per[p] / tot if tot else 0:11.1f}%" for p in PHASES))
        print(f"{'':5s}  tokenize:" + "".join(f"  {p} {tk[p]:.0f} ({100 * tk[p] / ttk if ttk else 0:.1f}%)" for p in TK_SHOWN), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
