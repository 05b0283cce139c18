"""Both scan kernels (byte and pair prefilter) against the oracle (CPython `re` / `in`), at the places where a persistent
TMA-ring scan goes wrong: a match exactly on a tile edge, on the stage-ring wrap and on lane-chunk edges, with a multi-byte
character or a unit terminator right in front of it; a candidate-dense stream that overflows the candidate queue; bitmaps
of 1, 2 and 4 words; an always-matching pattern; random patterns.

The library reads CF_SCAN_RESERVE_SMS once, in cf_init, and a Context is cached per process, so each configuration runs in a
worker process of its own (this file, `--worker`).  The parent writes the corpora, runs the worker with the configuration's
environment, and compares the bitmaps the worker saved with the oracle, which it computes once per corpus.

The geometry below must equal the kernels' (checked without a GPU), so that the planted matches land on their real tile,
lane and stage-ring edges."""
import json
import os
import random
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from mcp_context_forge_b200 import _native, engine  # noqa: E402
from oracle import hook_chain_ref as ref  # noqa: E402

CSRC = os.path.join(ROOT, "mcp_context_forge_b200", "csrc")

# scan_kernel's geometry (csrc/cf_internal.h) and the depth of its TMA stage ring per prefilter (csrc/cfgpu.cu)
WARPS = 16
LANE_BYTES = 64
TILE = WARPS * 32 * LANE_BYTES
BYTE_STAGES = 3
PAIR_STAGES = 2

HARMFUL = [(p, re.I) for pats in ref.DEFAULT_LEXICONS.values() for p in pats]
DENY = ["innovative", "groundbreaking", "revolutionary"]
SUBS = [("crap", 0, "crud"), ("crud", 0, "yikes")]
EXTRA_SEARCH = [(r"\Bkill", re.I), (r"\bDROP\b", re.I)]
ALWAYS = (r"x*", 0)                                   # matches every unit: the fill_bitmaps_kernel path


def literals(n):
    return ["zq%03d" % i for i in range(n)]


# name -> (search patterns, literals, sub rules): W = 1, 2 (with an always-matching pattern) and 4 bitmap words
PROGRAMS = {
    "w1": (HARMFUL + EXTRA_SEARCH, DENY, SUBS),
    "w2": (HARMFUL + EXTRA_SEARCH + [ALWAYS], DENY + literals(80), SUBS),
    "w4": (HARMFUL + EXTRA_SEARCH, DENY + literals(200), SUBS),
}


# ---------------------------------------------------------------------------------------------------------------------
# corpora
# ---------------------------------------------------------------------------------------------------------------------
TERM = None                                           # "the unit starts here": the byte in front is the 0xFF terminator
CTXS = [" ", "é", "日", "\U0001F600", "\n", TERM]
WORDS = ["suicide", "kill", "DROP", "innovative", "zq079", "zq199"]
TAIL = " ok."
FILL = ("lorem ipsum dolor sit amet, consectetur adipiscing elit; sed do eiusmod tempor incididunt ut labore et dolore "
        "magna aliqua. ") * 8
EDGE_DS = list(range(-12, 5))                         # match start = edge + d
EDGE_TILES = 5                                        # tile edges 1..5: the first three, and (with one CTA) the ring wrap of 2 and 3 stages


def filler(n):
    reps = n // len(FILL) + 1
    return (FILL * reps)[:n]


def lane_ms(tile, lb):
    """Lane-chunk indices inside a tile whose start gets a planted match: the first lanes, the warp edge, the last lane."""
    return [1, 2, 31, 32, 33, tile // lb - 1]


def edge_stream(tile, lb, d, counter):
    """Units of one stream in which a match starts at every tile edge k*tile + d (k = 1..EDGE_TILES) and at the lane-chunk
    edges m*lb + d of every tile.  Returns (units as str, placements [(offset, word, ctx)]).  The (word, context) pairs cycle
    through every combination over the whole corpus, separately for tile edges and lane edges (`counter` carries the two
    cycles from stream to stream)."""
    targets = []
    for t in range(EDGE_TILES + 1):
        if t:
            targets.append(t * tile + d)
        targets += [t * tile + m * lb + d for m in lane_ms(tile, lb)]
    targets.sort()
    units, placements, pos = [], [], 0               # pos = stream offset where the next unit starts
    for o in targets:
        kind = 0 if o % tile == d % tile and o >= tile + d else 1     # tile edge / lane-chunk edge: separate cycles
        i = counter[kind]
        counter[kind] += 1
        word = WORDS[i % len(WORDS)]
        ctx = CTXS[(i // len(WORDS)) % len(CTXS)]
        if ctx is TERM:
            pad = o - 1 - pos                         # a filler unit that ends right in front of the match
            assert pad >= 0, (o, pos)
            units.append(filler(pad))
            units.append(word + TAIL)
        else:
            n = o - pos - len(ctx.encode())
            assert n >= 0, (o, pos)
            units.append(filler(n) + ctx + word + TAIL)
        placements.append((o, word, ctx))
        pos = o + len(word) + len(TAIL) + 1
    units.append(filler(tile // 3))
    return units, placements


def edge_corpus(tile, lb):
    """One stream per d in EDGE_DS: [(units, placements)]."""
    counter = [0, 0]
    return [edge_stream(tile, lb, d, counter) for d in EDGE_DS]


def dense_base():
    """The 16 distinct units of the candidate-dense corpus (a prefilter candidate every few bytes)."""
    rng = random.Random(7)
    words = ["kill", "bomb", "crap", "crud", "killer", "skill", "innovative", "suicid", "bombs", "kil", "k1ll",
             "assault", "Kill yourself", "self-harm", "I hate", "innovativ"]
    base = []
    for _ in range(16):
        parts, n = [], 0
        while n < 16000:
            w = rng.choice(words)
            parts.append(w)
            n += len(w) + 1
        base.append(" ".join(parts))
    return base


DENSE_UNITS = 2048
FUZZ_SEEDS = [7000, 7001, 7002, 7003]


def fuzz_round(seed):
    """Random patterns (test_regex_fuzz_cpu.pattern, drawn as its rounds draw them) that the front end accepts, and units of
    very different lengths so that matches straddle lanes, tiles and unit boundaries.  Returns (patterns, units)."""
    from mcp_context_forge_b200.regex_frontend import UnsupportedPattern, compile_ast
    from test_regex_fuzz_cpu import ALPH, pattern

    rng = random.Random(seed)
    pats = []
    for _ in range(rng.randint(1, 12)):
        p, fl = pattern(rng)
        try:
            re.compile(p, fl)
            compile_ast(p, fl, "search")
        except (re.error, UnsupportedPattern):
            continue
        pats.append((p, fl))
    units = []
    for _ in range(400):
        n = rng.choice([0, 1, 3, 17, 31, 32, 33, 63, 64, 65, 200, 2047, 2048, 2049, 5000, 20000])
        units.append("".join(rng.choice(ALPH) for _ in range(rng.randint(0, n))))
    return pats, units


def configurations(sms=132):
    """Each prefilter's kernel on the full persistent grid (all corpora), and again with one CTA (edge corpus only).  On the
    full grid an edge stream of a few tiles gives each CTA one tile, so its stage ring never wraps; with one CTA, tile k sits
    in stage k mod stages and the planted edges k = 1..5 cross the ring wrap of the byte filter's 3 stages and the pair
    filter's 2."""
    cfgs = []
    for name, pair in (("byte", False), ("pair", True)):
        env = {"CF_PAIR_FILTER": int(pair)}
        cfgs.append({"id": name, "pair": pair, "edge_only": False, "env": env})
        cfgs.append({"id": name + "-one-cta", "pair": pair, "edge_only": True, "env": dict(env, CF_SCAN_RESERVE_SMS=sms - 1)})
    cfgs.append({"id": "default-reserve-4", "pair": False, "edge_only": False, "env": {"CF_SCAN_RESERVE_SMS": 4, "CF_PAIR_FILTER": 0}})
    # one CTA owns every tile of the candidate-dense corpus: its share of the candidate queue overflows
    cfgs.append({"id": "default-one-cta", "pair": False, "edge_only": False, "env": {"CF_SCAN_RESERVE_SMS": sms - 1, "CF_PAIR_FILTER": 0}})
    return cfgs


CONFIG_IDS = [c["id"] for c in configurations()]


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks
# ---------------------------------------------------------------------------------------------------------------------
def test_geometry_matches_the_library():
    """The corpora's geometry is the kernels' (read from the source), and the built library holds exactly the two kernels."""
    hdr = open(os.path.join(CSRC, "cf_internal.h"), encoding="utf-8").read()
    assert int(re.search(r"uint32_t SCAN_WARPS = (\d+);", hdr).group(1)) == WARPS
    assert int(re.search(r"uint32_t SCAN_LANE_BYTES = (\d+);", hdr).group(1)) == LANE_BYTES
    src = open(os.path.join(CSRC, "cfgpu.cu"), encoding="utf-8").read()
    pair_st, byte_st = re.search(r"constexpr uint32_t STAGES = PAIR \? (\d+) : (\d+);", src).groups()
    assert (int(byte_st), int(pair_st)) == (BYTE_STAGES, PAIR_STAGES)
    cuobjdump = next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)), None)
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", _native.SO_PATH], capture_output=True, text=True, check=True).stdout
    kernels = sorted(set(re.findall(r"Function (\S*scan_kernel\S*):", out)))
    assert kernels == ["_Z11scan_kernelILj0EEv10ScanParams14CUtensorMap_st", "_Z11scan_kernelILj1EEv10ScanParams14CUtensorMap_st"], kernels


def test_edge_corpus_places_every_match_where_intended():
    tile, lb = TILE, LANE_BYTES
    seen = set()
    for d, (units, placements) in zip(EDGE_DS, edge_corpus(tile, lb)):
        stream, offs = engine.pack_units(units)
        starts = set(int(x) for x in offs[:-1])
        want = sorted([k * tile + d for k in range(1, EDGE_TILES + 1)] +
                      [t * tile + m * lb + d for t in range(EDGE_TILES + 1) for m in lane_ms(tile, lb)])
        assert [o for o, _, _ in placements] == want
        for o, word, ctx in placements:
            assert stream[o:o + len(word)] == word.encode(), (o, word)
            if ctx is TERM:
                assert stream[o - 1] == 0xFF and o in starts
            else:
                c = ctx.encode()
                assert stream[o - len(c):o] == c and o not in starts
            if o % tile == (d % tile) and o >= tile + d:
                seen.add((word, ctx))
    # every (word, context) pair sits on some tile edge
    assert seen == {(w, c) for w in WORDS for c in CTXS}


# ---------------------------------------------------------------------------------------------------------------------
# GPU: parent side
# ---------------------------------------------------------------------------------------------------------------------
def _oracle(prog, units):
    search, lits, subs = PROGRAMS[prog]
    return ref.scan_bitmaps(units, search, lits, [(p, f) for p, f, _ in subs])


class Corpora:
    """Files of every corpus under one directory, and their oracle bitmaps (computed once, shared by the configurations)."""

    def __init__(self, root):
        self.root = root
        self.files = {}
        self.expect = {}
        self.units = {}

    def _write(self, key, units):
        if key not in self.files:
            stream, offs = engine.pack_units(units)
            path = os.path.join(self.root, key.replace("/", "_"))
            np.save(path + ".stream.npy", np.frombuffer(stream, dtype=np.uint8))
            np.save(path + ".offs.npy", offs)
            self.files[key] = path
            self.units[key] = units
        return self.files[key]

    def oracle(self, key, prog, fn):
        if (key, prog) not in self.expect:
            self.expect[(key, prog)] = fn(self.units[key])
        return self.expect[(key, prog)]

    def jobs(self, cfg):
        """[(program spec, corpus key, corpus path, oracle function)] for one configuration."""
        out = []
        for i, (units, _) in enumerate(edge_corpus(TILE, LANE_BYTES)):
            key = f"edge-{i}"
            path = self._write(key, units)
            for prog in PROGRAMS:
                out.append((prog, key, path, lambda u, p=prog: _oracle(p, u)))
        if cfg["edge_only"]:
            return out
        base = dense_base()
        path = self._write("dense", [base[i % 16] for i in range(DENSE_UNITS)])
        if ("dense", "w1") not in self.expect:
            exp = _oracle("w1", base)
            self.expect[("dense", "w1")] = [exp[i % 16] for i in range(DENSE_UNITS)]
        out.append(("w1", "dense", path, None))
        for seed in FUZZ_SEEDS:
            pats, units = fuzz_round(seed)
            key = f"fuzz-{seed}"
            path = self._write(key, units)
            comp = [re.compile(p, f) for p, f in pats]
            out.append(({"search": pats}, key, path,
                        lambda u, c=comp: [sum(1 << i for i, x in enumerate(c) if x.search(s)) for s in u]))
        return out


@pytest.fixture(scope="module")
def corpora(tmp_path_factory):
    return Corpora(str(tmp_path_factory.mktemp("scan_corpora")))


def _run_worker(job, env_over, tmp_path, timeout=600):
    jf = os.path.join(str(tmp_path), "job.json")
    with open(jf, "w") as f:
        json.dump(job, f)
    env = dict(os.environ)
    for k in ("CF_SCAN_RESERVE_SMS", "CF_PAIR_FILTER"):
        env.pop(k, None)
    env.update({k: str(v) for k, v in env_over.items()})
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", jf], env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stderr[-4000:]
    with open(os.path.join(str(tmp_path), "result.json")) as f:
        return json.load(f)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(CONFIG_IDS)), ids=CONFIG_IDS)
def test_variant_matches_oracle(idx, corpora, tmp_path):
    cfg = configurations(_sm_count())[idx]
    jobs = corpora.jobs(cfg)
    job = {"out": str(tmp_path), "scans": [{"name": f"s{i}", "program": prog, "corpus": path} for i, (prog, _, path, _) in enumerate(jobs)]}
    res = _run_worker(job, cfg["env"], tmp_path)
    assert res["error"] is None, res["error"]
    # the programs took the prefilter (byte / pair) the configuration names
    assert set(res["prefilter"].values()) == {1 if cfg["pair"] else 0}, res["prefilter"]
    data = np.load(os.path.join(str(tmp_path), "bitmaps.npz"))
    checked = 0
    for i, (prog, key, _, fn) in enumerate(jobs):
        exp = corpora.oracle(key, prog if isinstance(prog, str) else f"fuzz{key}", fn)
        W = int(res["words"][f"s{i}"])
        got = engine.bitmaps_to_ints(data[f"s{i}"], len(exp), W)
        bad = [(k, hex(g), hex(e)) for k, (g, e) in enumerate(zip(got, exp)) if g != e]
        assert not bad, (cfg["id"], prog if isinstance(prog, str) else "fuzz", key, bad[:5])
        checked += len(exp)
    assert checked > 1000
    if cfg["id"] == "default-one-cta":
        assert res["dense_candidates"] > (1 << 20)        # far more than one CTA's share of the candidate queue


# ---------------------------------------------------------------------------------------------------------------------
# GPU: worker side (a fresh process per configuration)
# ---------------------------------------------------------------------------------------------------------------------
def _worker(job_file):
    with open(job_file) as f:
        job = json.load(f)
    res = {"error": None, "prefilter": {}, "words": {}}
    try:
        ctx = engine.Context(0)
    except engine.N.CfError as exc:
        res["error"] = str(exc)
    if res["error"] is None:
        progs = {}
        out = {}
        for sc in job["scans"]:
            spec = sc["program"]
            key = spec if isinstance(spec, str) else json.dumps(spec)
            if key not in progs:
                search, lits, subs = PROGRAMS[spec] if isinstance(spec, str) else (spec["search"], [], [])
                p = engine.Program()
                for q, fl in search:
                    p.add_search(q, fl)
                for w in lits:
                    p.add_literal(w)
                for q, fl, r in subs:
                    p.add_sub(q, fl, r)
                res["prefilter"][key] = int(p.compile_host().prefilter)
                progs[key] = p.compile(ctx)
            p = progs[key]
            stream = np.load(sc["corpus"] + ".stream.npy")
            offs = np.load(sc["corpus"] + ".offs.npy")
            batch = engine.Batch(ctx, len(stream), len(offs) - 1)
            out[sc["name"]] = engine.scan_host(p, batch, stream, offs)
            res["words"][sc["name"]] = p.words
            if sc["corpus"].endswith("dense"):
                res["dense_candidates"] = ctx.scan_counters()[0]
        np.savez(os.path.join(job["out"], "bitmaps.npz"), **out)
    with open(os.path.join(job["out"], "result.json"), "w") as f:
        json.dump(res, f)


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--worker":
    _worker(sys.argv[2])
