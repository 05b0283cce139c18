"""What the token-parallel TOON encoder does with bench.py's payload mix, by shape (CPU only).

Runs bench.make_payloads()'s distinct payloads through json_tp.h's per-unit pipeline on the CPU warp emulator
(tools/toon_emu.py) as toon_tp_kernel runs it (first pass; the resolving pass for units handed over as mixed list-item arrays)
and reports per shape: the first pass's statuses and hand-over reasons (status 7, FB_* of json_tp.h), the statuses after the
resolving pass (status 7 there = handed to the sequential encoder), the warp collectives per unit (ballots, shuffles and
syncs: the serial steps of a warp) and the emulator's time per unit.  The bench batch tiles the distinct payloads evenly, so
their shares are the batch's.  Emulator times are CPU times; they rank shapes, they are not GPU times.

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
    new = lambda: {"n": 0, "coll": 0, "coll2": 0, "sec": 0.0, "status": collections.Counter(), "reason": collections.Counter(), "final": collections.Counter()}
    agg = collections.defaultdict(new)
    for i, p in enumerate(payloads):
        a = agg[shape_of(i)]
        t0 = time.perf_counter()
        st, _, why, c1 = toon_emu.toon_pass(p.encode(), False)
        fin, c2 = st, 0
        if st == toon_emu.TS_FALLBACK and why == toon_emu.FB_MIXED_ITEM:
            fin, _, _, c2 = toon_emu.toon_pass(p.encode(), True)
        a["sec"] += time.perf_counter() - t0
        a["coll"] += c1
        a["coll2"] += c2
        a["n"] += 1
        a["status"][STATUS.get(st, st)] += 1
        a["final"][STATUS.get(fin, fin)] += 1
        if st == 7:
            a["reason"][REASON.get(why, why)] += 1
    total = sum(a["n"] for a in agg.values())
    handed1 = handed = 0
    print(f"{'shape':18s} {'share':>6s} {'coll./unit':>11s} {'+resolving':>11s} {'emu ms/unit':>12s}  first pass: statuses; hand-over reasons | after resolving")
    for s in sorted(agg):
        a = agg[s]
        handed1 += a["status"]["handed_over"]
        handed += a["final"]["handed_over"]
        print(f"{NAMES.get(s, s):18s} {a['n'] / total:6.0%} {a['coll'] // a['n']:11d} {a['coll2'] // a['n']:11d} {a['sec'] / a['n'] * 1e3:12.1f}  "
              f"{dict(a['status'])}; {dict(a['reason'])} | {dict(a['final'])}")
    print(f"handed over by the first pass: {handed1} of {total} distinct payloads ({handed1 / total:.2%} of the bench batch); "
          f"to the sequential encoder: {handed} ({handed / total:.2%})")


if __name__ == "__main__":
    main()
