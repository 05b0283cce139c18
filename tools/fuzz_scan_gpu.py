"""Random-pattern differential test of the GPU scan (both prefilter kernels) against CPython `re`.
usage: [CF_PAIR_FILTER=0|1] python -u tools/fuzz_scan_gpu.py [first_seed] [rounds]   (needs an H100)"""
import random
import re
import sys
import time

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from mcp_context_forge_b200 import engine
from mcp_context_forge_b200.regex_frontend import UnsupportedPattern
from test_regex_fuzz_cpu import ALPH, pattern

seed0 = int(sys.argv[1]) if len(sys.argv) > 1 else 0
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 100
ctx = engine.Context.get()
t0, npat, nbad, skipped = time.time(), 0, 0, 0
for rd in range(rounds):
    rng = random.Random(seed0 * 100000 + rd)
    prog = engine.Program()
    pats = []
    for _ in range(rng.randint(1, 12)):
        p, fl = pattern(rng)
        try:
            c = re.compile(p, fl)
        except re.error:
            continue
        try:
            prog.add_search(p, fl)
        except UnsupportedPattern:
            continue
        pats.append((p, fl, c))
    if not pats:
        continue
    try:
        prog.compile(ctx)
    except Exception as exc:
        if "too large" in str(exc):
            skipped += 1
            continue
        raise
    # units of very different lengths so that matches straddle lanes, chains, tiles and unit boundaries
    units = []
    for _ in range(400):
        n = rng.choice([0, 1, 3, 17, 31, 32, 33, 63, 64, 65, 200, 2047, 2048, 2049, 5000])
        units.append("".join(rng.choice(ALPH) for _ in range(rng.randint(0, n))))
    got = engine.scan_units(prog, units)
    npat += len(pats)
    for u, g in zip(units, got):
        exp = 0
        for i, (_, _, c) in enumerate(pats):
            if c.search(u):
                exp |= 1 << i
        if g != exp:
            i = ((g ^ exp) & -(g ^ exp)).bit_length() - 1
            print("MISMATCH", seed0, rd, repr(pats[i][0]), pats[i][1], repr(u[:80]), len(u), "got", (g >> i) & 1)
            nbad += 1
            break
print("rounds", rounds, "patterns", npat, "rounds with mismatches", nbad, "skipped (too large)", skipped, "seconds", round(time.time() - t0, 1))
