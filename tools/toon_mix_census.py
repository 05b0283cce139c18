"""What the token-parallel TOON encoder does with bench.py's payload mix, by shape (CPU only).

Runs bench.make_payloads()'s distinct payloads through json_tp.h's per-unit pipeline on the CPU warp emulator
(tools/toon_emu.py) and reports per shape: the first attempt's statuses and hand-over reasons (status 7, FB_* of json_tp.h), the
statuses toon_tp_kernel ends with, a unit that stops at a mixed list-item array being analyzed and emitted again in place (status 7
there = handed to the sequential encoder), the warp collectives per unit (ballots, shuffles and syncs: the serial steps of a warp) of
the first attempt and what the in-place retries add to them, and the emulator's time per unit of the kernel's run.  The bench batch
tiles the distinct payloads evenly, so their shares are the batch's.  Emulator times are CPU times; they rank shapes, they are not GPU
times.

usage: python tools/toon_mix_census.py
"""
import collections
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import toon_emu  # noqa: E402
from toon_stage_breakdown import shape_of  # noqa: E402

STATUS = {0: "converted", 1: "not_smaller", 2: "not_json", 3: "value_error", 4: "attr_error", 6: "unsupported", 7: "handed_over"}
REASON = {1: "FB_NUM_EXACT", 2: "FB_KEY_ESCAPE", 3: "FB_TOK_CAP", 4: "FB_KH_CAP", 5: "FB_DUP_HASH", 6: "FB_ROW_ORDER", 7: "FB_MIXED_ITEM", 8: "FB_TOO_LONG"}
NAMES = {"A": "A tabular", "B": "B nested config", "C": "P prose-in-JSON"}


def main():
    toon_emu.lib()
    payloads = bench.make_payloads()
    new = lambda: {"n": 0, "coll": 0, "coll2": 0, "retried": 0, "sec": 0.0, "status": collections.Counter(), "reason": collections.Counter(),
                   "final": collections.Counter()}
    agg = collections.defaultdict(new)
    for i, p in enumerate(payloads):
        a = agg[shape_of(i)]
        st, _, why, c1 = toon_emu.toon_pass(p.encode(), False)
        t0 = time.perf_counter()
        fin, _, _, _, c = toon_emu.toon_tp(p.encode())
        a["sec"] += time.perf_counter() - t0
        a["coll"] += c1
        a["coll2"] += c - c1
        a["n"] += 1
        a["retried"] += st == toon_emu.TS_FALLBACK and why == toon_emu.FB_MIXED_ITEM
        a["status"][STATUS.get(st, st)] += 1
        a["final"][STATUS.get(fin, fin)] += 1
        if st == 7:
            a["reason"][REASON.get(why, why)] += 1
    total = sum(a["n"] for a in agg.values())
    handed1 = handed = retried = 0
    print(f"{'shape':18s} {'share':>6s} {'coll./unit':>11s} {'+retries':>9s} {'emu ms/unit':>12s}  first attempt: statuses; hand-over reasons | kernel's result")
    for s in sorted(agg):
        a = agg[s]
        handed1 += a["status"]["handed_over"]
        handed += a["final"]["handed_over"]
        retried += a["retried"]
        print(f"{NAMES.get(s, s):18s} {a['n'] / total:6.0%} {a['coll'] // a['n']:11d} {a['coll2'] // a['n']:9d} {a['sec'] / a['n'] * 1e3:12.1f}  "
              f"{dict(a['status'])}; {dict(a['reason'])} | {dict(a['final'])}")
    print(f"handed over by the first attempt: {handed1} of {total} distinct payloads ({handed1 / total:.2%} of the bench batch), "
          f"{retried} of them retried in place as mixed list-item arrays; to the sequential encoder: {handed} ({handed / total:.2%})")


if __name__ == "__main__":
    main()
