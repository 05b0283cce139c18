"""The regex_filter substitution kernel (sub_kernel, csrc/cfgpu.cu) against CPython `re`, with random rule programs and with
units built to hit the places where the kernel works differently from a sequential `re.sub`:

- a rule that cannot match "" examines 512 start positions per warp iteration (SUB_WIN) and resolves overlaps across
  iterations; a rule that can examines 256, each with a first match and a must-advance match.  Matches are planted at
  512*j + d and 256*j + d (d = -20..20), with a 2-, 3- or 4-byte character straddling the edge in front of the match or
  inside it, and matches long enough to run across two or three windows;
- rule r + 1 reads rule r's output from a ping-pong scratch pair, and a program of more than 32 rules (SUB_LAUNCH_RULES)
  continues in further launches from the record the previous launch left for each unit;
- each unit's scratch is sized from a worst-case growth bound: rules whose output reaches it, many units side by side.

Every random program goes through the kernel's three callers: engine.sub_host (cf_sub_host) with a shuffled selection,
SearchReplacePlugin (the scan bitmap picks the units it rewrites), and engine.run_batch with CF_STAGE_SUB, alone and with
CF_STAGE_TOON and per-unit stages.  A failure prints the rules (pattern, flags, template) and an excerpt of the unit around
the first difference, enough to reproduce it.  The random rounds count what they covered and assert it, so they cannot pass
without reaching the window edges."""
import asyncio
import bisect
import itertools
import json
import os
import random
import re
import re._parser as sre_parse  # type: ignore[import]
import tempfile

import numpy as np
import pytest

from mcp_context_forge_b200 import _native as N
from mcp_context_forge_b200 import engine
from mcp_context_forge_b200.regex_frontend import UnsupportedPattern, template_parts
from oracle import hook_chain_ref as ref
from oracle import toon_ref
from test_regex_fuzz_cpu import ALPH, sub_pattern

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFGPU = os.path.join(ROOT, "mcp_context_forge_b200", "csrc", "cfgpu.cu")

SUB_WIN = 512                   # start positions per warp iteration of a rule that cannot match ""
NULL_WIN = 256                  # ... of a rule that can
LAUNCH_RULES = 32               # rules per sub_kernel launch
EDGE_DS = list(range(-20, 21))  # planted match start = window edge + d
EDGE_JS = (1, 2, 3, 4)          # window edges j * window of a planted unit
NEAR = 20                       # a match "at" an edge starts within this many bytes of it
WIDE = ["é", "日", "\U0001F600"]  # 2-, 3- and 4-byte characters
TEXT_ALPH = ALPH + WIDE
ASCII = [c for c in ALPH if ord(c) < 128]
BLEN = {c: len(c.encode()) for c in TEXT_ALPH}
FLAG_NAMES = ((re.I, "i"), (re.M, "m"), (re.S, "s"))


# ---------------------------------------------------------------------------------------------------------------------
# rules and programs
# ---------------------------------------------------------------------------------------------------------------------
class Rule:
    """One regex_filter rule: `re.compile(pattern, flags).sub(template, text)`."""

    def __init__(self, pattern, flags, template):
        self.pattern, self.flags, self.template = pattern, flags, template
        self.c = re.compile(pattern, flags)
        self.parts = template_parts(template, self.c)
        self.nullable = sre_parse.parse(pattern, flags).getwidth()[0] == 0
        self.refs = any(isinstance(p, int) for p in self.parts)

    def word(self):
        """The rule as a regex_filter config entry, its flags written inline."""
        f = "".join(ch for fl, ch in FLAG_NAMES if self.flags & fl)
        return {"search": (f"(?{f})" if f else "") + self.pattern, "replace": self.template}

    def __repr__(self):
        f = "|".join("re." + ch.upper() for fl, ch in FLAG_NAMES if self.flags & fl) or "0"
        return f"({self.pattern!r}, {f}, {self.template!r})"


def plain_rule(p, fl, tmpl):
    try:
        return Rule(p, fl, tmpl)
    except re.error:
        return None


def engine_rule(p, fl, tmpl):
    """The rule if the GPU front end and back end take it (the ones they refuse are documented limits, as in the CPU fuzz)."""
    r = plain_rule(p, fl, tmpl)
    if r is None:
        return None
    try:
        prog = engine.Program()
        prog.add_sub(p, fl, r.parts)
        prog.compile_host()
    except UnsupportedPattern:
        return None
    except N.CfError as exc:
        if exc.code in (N.CF_E_UNSUPPORTED, N.CF_E_TOO_LARGE):
            return None
        raise
    return r


def tractable(p, fl):
    """True when CPython's backtracking stays near-linear on long units: at most one unbounded repeat, and no repeat of more
    than one iteration or alternation inside such a repeat.  (`(\\S[^a]*?|9)*?`, `((k|k))*^9` or `\\w*\\w*x` take `re` minutes
    on a long unit, so there would be no oracle; the GPU engine has no such limit.)"""
    unbounded = 0

    def walk(sub, in_repeat):
        nonlocal unbounded
        for op, av in sub:
            if op in (sre_parse.MAX_REPEAT, sre_parse.MIN_REPEAT, sre_parse.POSSESSIVE_REPEAT):
                lo, hi, body = av
                unbounded += hi == sre_parse.MAXREPEAT
                if hi > 1 and in_repeat:
                    return False
                if not walk(body, in_repeat or hi > 1):
                    return False
            elif op == sre_parse.SUBPATTERN:
                if not walk(av[-1], in_repeat):
                    return False
            elif op == sre_parse.BRANCH:
                if in_repeat or not all(walk(alt, in_repeat) for alt in av[1]):
                    return False
        return True

    return walk(sre_parse.parse(p, fl), False) and unbounded <= 1


def rand_template(rng, c):
    pieces = ["-", "<", ">", "é", "日", "\U0001F600", "\\\\", ""] + [f"\\{g}" for g in range(1, c.groups + 1)] + ["\\g<0>"]
    return "".join(rng.choice(pieces) for _ in range(rng.randint(0, 4)))


def rand_program(rng, make=engine_rule):
    """1-8 random rules (capturing groups, rules that can match "", templates with \\N and \\g<0>, random I/M/S flags) from
    the CPU fuzz's generator, keeping the patterns `re` can run on long units."""
    rules, want = [], rng.randint(1, 8)
    for _ in range(8 * want):
        if len(rules) == want:
            break
        p, fl = sub_pattern(rng)
        try:
            c = re.compile(p, fl)
        except re.error:
            continue
        if not tractable(p, fl):
            continue
        r = make(p, fl, rand_template(rng, c))
        if r is not None:
            rules.append(r)
    return rules


def build_program(rules):
    prog = engine.Program()
    for r in rules:
        prog.add_sub(r.pattern, r.flags, r.parts)
    return prog


# ---------------------------------------------------------------------------------------------------------------------
# units
# ---------------------------------------------------------------------------------------------------------------------
def rand_text(rng, n_chars, alph=TEXT_ALPH):
    return "".join(rng.choices(alph, k=n_chars))


def filler(rng, nbytes):
    """Random text of exactly `nbytes` UTF-8 bytes."""
    chars = rng.choices(TEXT_ALPH, k=nbytes)
    k = bisect.bisect_right(list(itertools.accumulate(BLEN[c] for c in chars)), nbytes)
    head = chars[:k]
    return "".join(head) + "".join(rng.choices(ASCII, k=nbytes - sum(BLEN[c] for c in head)))


def sample_matches(rng, rule):
    """Non-empty texts `re` matches for the rule, taken from random texts."""
    for _ in range(4):
        t = rand_text(rng, 60)
        out = [m.group() for m in rule.c.finditer(t) if m.end() > m.start()]
        if out:
            return out
    return []


def long_match(rng, rule, samples, min_bytes):
    """A match of at least `min_bytes` bytes, from 700-character texts over one letter, over the letters of the rule's short
    matches, or over a few random letters (None when none turns up)."""
    seen = sorted({ch for m in samples for ch in m})
    alphs = [[ch] for ch in TEXT_ALPH] + ([seen] * 3 if seen else []) + [rng.sample(TEXT_ALPH, rng.randint(2, 4)) for _ in range(4)]
    for a in alphs:
        t = "".join(rng.choices(a, k=700))
        for m in rule.c.finditer(t):
            if len(m.group().encode()) >= min_bytes:
                return m.group()
    return None


class Plant:
    """One planted copy: match text `m` of `rule` at byte `off` (char `ci`) of its unit; `edge` is the edge of a `win`-byte window
    it was aimed at, `wide` the (byte offset, length) of the character meant to straddle the edge ("pre" / "inside" modes)."""

    def __init__(self, rule, m, off, ci, win, edge, mode, wide):
        self.rule, self.m, self.off, self.ci, self.win, self.edge, self.mode, self.wide = rule, m, off, ci, win, edge, mode, wide


def planted_unit(rng, rule, m, win, targets, pre, mode):
    """A unit with `pre` + `m` placed so that m's first byte sits at each byte offset of `targets` (ascending), random text
    between.  Returns (unit, [Plant] of the copies `re` really matches there) or None when the copies do not fit."""
    mb, pb = m.encode(), pre.encode()
    parts, pos, nch, placed = [], 0, 0, []
    for edge, o in targets:
        gap = o - len(pb) - pos
        if gap < 0:
            return None
        f = filler(rng, gap)
        parts += [f, pre, m]
        ci = nch + len(f) + len(pre)
        wide = None
        if mode == "pre":
            wide = (o - len(pb), len(pb))
        elif mode == "inside":
            q = next(i for i, ch in enumerate(m) if len(ch.encode()) > 1)
            wide = (o + len(m[:q].encode()), len(m[q].encode()))
        placed.append((edge, o, ci, wide))
        nch = ci + len(m)
        pos = o + len(mb)
    parts.append(filler(rng, rng.randint(0, 60)))
    unit = "".join(parts)
    plants = []
    for edge, o, ci, wide in placed:
        mm = rule.c.match(unit, ci)
        if mm and mm.end() > ci:
            plants.append(Plant(rule, m, o, ci, win, edge, mode, wide))
    return unit, plants


def plants_for_rule(rng, rule, d_cycle):
    """Planted units for one rule: per window size (512, and 256 when the rule can match ""), a copy at edge + d for every
    edge j = 1..4, a copy behind a wide character that straddles the edge, a copy whose own wide character straddles it,
    and one match long enough to cross one or more edges."""
    out = []
    samples = sample_matches(rng, rule)
    for win in ([SUB_WIN, NULL_WIN] if rule.nullable else [SUB_WIN]):
        fits = [m for m in samples if len(m.encode()) + 4 < win - 2 * NEAR]
        if fits:
            m = rng.choice(fits)
            d = next(d_cycle)
            out.append(planted_unit(rng, rule, m, win, [(j * win, j * win + d) for j in EDGE_JS], "", "d"))
            ch = rng.choice(WIDE)
            k = rng.randint(1, len(ch.encode()) - 1)             # ch covers [edge - k, edge - k + len): it straddles the edge
            out.append(planted_unit(rng, rule, m, win, [(j * win, j * win + len(ch.encode()) - k) for j in EDGE_JS], ch, "pre"))
            wide = [m for m in fits if any(len(ch.encode()) > 1 for ch in m)]
            if wide:
                m = rng.choice(wide)
                q = next(i for i, ch in enumerate(m) if len(ch.encode()) > 1)
                qb, L = len(m[:q].encode()), len(m[q].encode())
                k = rng.randint(1, L - 1)
                out.append(planted_unit(rng, rule, m, win, [(j * win, j * win - qb - k) for j in EDGE_JS], "", "inside"))
        g = long_match(rng, rule, samples, win + NEAR + 1)            # from edge + d, d >= -NEAR, it runs past the next edge
        if g is not None:
            edge = win * rng.choice((1, 2))
            out.append(planted_unit(rng, rule, g, win, [(edge, edge + next(d_cycle))], "", "cross"))
    return [u for u in out if u is not None]


def json_unit(rng):
    return json.dumps([{"id": i, "name": rand_text(rng, rng.randint(1, 8)), "ok": i % 2 == 0} for i in range(rng.randint(2, 6))], ensure_ascii=False)


def program_units(rng, rules, d_cycle):
    """(units, plants): short random units, long random units, planted units per rule, a few JSON documents."""
    units = [rand_text(rng, rng.randint(0, 40)) for _ in range(32)] + ["", "\n", filler(rng, rng.randint(600, 20000))]
    plants = []
    for r in rules:
        for u, ps in plants_for_rule(rng, r, d_cycle):
            units.append(u)
            plants.append(ps)
    units += [json_unit(rng) for _ in range(3)]
    return units, plants


# ---------------------------------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------------------------------
def byte_offsets(s):
    """Byte offset of every character boundary of s (len(s) + 1 entries)."""
    cp = np.frombuffer(s.encode("utf-32-le", "surrogatepass"), dtype=np.uint32)
    lens = 1 + (cp >= 0x80) + (cp >= 0x800) + (cp >= 0x10000)
    out = np.zeros(len(s) + 1, dtype=np.int64)
    np.cumsum(lens, out=out[1:])
    return out


def edge_stats(rule, s, stats):
    """Counts the rule's non-empty matches in s that start within NEAR bytes of a window edge of the kernel, and those that cross
    an edge.  Windows are positions of the text the rule reads: 512 for a rule that cannot match "", 256 for one that can."""
    win = NULL_WIN if rule.nullable else SUB_WIN
    if len(s) * 4 < win - NEAR:
        return
    spans = np.array([m.span() for m in rule.c.finditer(s) if m.end() > m.start()], dtype=np.int64).reshape(-1, 2)
    if not len(spans):
        return
    bo = byte_offsets(s)
    a, e = bo[spans[:, 0]], bo[spans[:, 1]]
    k = (a + win // 2) // win                                      # nearest edge
    stats["near_edge"] += int(np.count_nonzero((k >= 1) & (np.abs(a - k * win) <= NEAR)))
    stats["cross_edge"] += int(np.count_nonzero((a // win + 1) * win < e))


def apply_rules(rules, u, stats=None):
    s = u
    for r in rules:
        if stats is not None:
            edge_stats(r, s, stats)
        s = r.c.sub(r.template, s)
    return s


def excerpt(got, exp, u):
    """Where got and exp first differ, with the unit around the same place."""
    i = next((i for i, (x, y) in enumerate(zip(got, exp)) if x != y), min(len(got), len(exp)))
    lo = max(i - 40, 0)
    ub = engine.encode_unit(u)
    return (f"unit ({len(ub)} bytes) {ub[lo:i + 40]!r}; first difference at byte {i} of {len(exp)}: "
            f"got {got[lo:i + 40]!r}, expected {exp[lo:i + 40]!r}")


def fail(where, rules, u, got, exp):
    pytest.fail(f"{where}: rules {rules}\n{excerpt(got, exp, u)}", pytrace=False)


def run(coro):
    return asyncio.new_event_loop().run_until_complete(coro)


# ---------------------------------------------------------------------------------------------------------------------
# the three callers of the kernel, each compared with the oracle
# ---------------------------------------------------------------------------------------------------------------------
def check_sub_host(ctx, prog, rules, units, exp, rng):
    """cf_sub_host on a selection of every matched unit plus unmatched ones (which must come back unchanged), shuffled, with
    one unit listed twice."""
    enc = [engine.encode_unit(u) for u in units]
    stream, offs = engine.pack_units(enc)
    batch = engine.Batch(ctx, len(stream), len(units))
    batch.upload(stream, offs)
    matched = [i for i, u in enumerate(units) if any(r.c.search(u) for r in rules)]
    unmatched = sorted(set(range(len(units))) - set(matched))
    sel = matched + rng.sample(unmatched, min(4, len(unmatched))) + [rng.randrange(len(units))]
    rng.shuffle(sel)
    for i, g in zip(sel, engine.sub_host(prog, batch, sel)):
        if g != exp[i]:
            fail(f"cf_sub_host (selection of {len(sel)})", rules, units[i], g, exp[i])
        if i in unmatched:
            assert g == enc[i]
    return len(unmatched)


def check_run_batch(ctx, prog, rules, units, exp, rng, with_toon):
    """cf_run_batch with CF_STAGE_SUB, or CF_STAGE_SUB | CF_STAGE_TOON with a random stage set per unit: the verdict bits,
    CF_V_REWRITTEN exactly on the units the scan selects (and that asked for SUB), out_len and the bytes.  A rule that can
    match "" has its bit set on every unit (it only selects the units the kernel visits; `\\B` finds nothing in "", yet the
    unit is visited): such a unit is reported rewritten, with the oracle's text."""
    enc = [engine.encode_unit(u) for u in units]
    stream, offs = engine.pack_units(enc)
    batch = engine.Batch(ctx, len(stream), len(units))
    stages = None
    mask = N.CF_STAGE_SUB
    if with_toon:
        mask |= N.CF_STAGE_TOON
        stages = np.array([rng.choice([N.CF_STAGE_SUB, N.CF_STAGE_TOON, N.CF_STAGE_SUB | N.CF_STAGE_TOON, 0]) for _ in units], dtype=np.uint8)
    v, out, oo, _ = engine.run_batch(prog, batch, stream, offs, mask, stages)
    raw = out[: int(oo[-1])].tobytes()
    for i, u in enumerate(units):
        hits = [r.nullable or bool(r.c.search(u)) for r in rules]
        st = int(stages[i]) if stages is not None else N.CF_STAGE_SUB
        bits = int(v["match_bitmap"][i])
        assert [bool(bits >> k & 1) for k in range(min(len(rules), 64))] == hits[:64], (rules, u[:80])
        flags, got = int(v["flags"][i]), raw[int(oo[i]):int(oo[i + 1])]
        rewritten = bool(st & N.CF_STAGE_SUB) and any(hits)
        assert bool(flags & N.CF_V_REWRITTEN) == rewritten, (rules, u[:80], st, flags)
        if rewritten:
            assert int(v["out_len"][i]) == len(exp[i]), (rules, u[:80])
            if got != exp[i]:
                fail(f"cf_run_batch stages {mask:#x}, unit stage {st:#x}", rules, u, got, exp[i])
            assert bool(flags & N.CF_V_RESUBMIT) == bool(st & N.CF_STAGE_TOON)
        elif st & N.CF_STAGE_TOON:
            t = toon_ref.process_text(u, 0, 1 << 30)
            assert (got.decode() if flags & N.CF_V_TOON else None) == t, (rules, u[:80])
        else:
            assert flags == 0 and int(v["out_len"][i]) == 0 and got == b""


def check_plugin(rules, units, exp):
    """SearchReplacePlugin with the rules as a config (flags inline): the GpuBatcher scans, then rewrites the units some rule matched."""
    from mcp_context_forge_b200 import framework as fw
    from mcp_context_forge_b200.plugins.regex_filter import SearchReplacePlugin

    words = [r.word() for r in rules]
    plug = SearchReplacePlugin(fw.PluginConfig(name="rf", kind="x", config={"words": words}))
    for u, g, e in zip(units, run(plug._apply(units)), exp):
        if g != e:
            fail("SearchReplacePlugin", rules, u, engine.encode_unit(g), engine.encode_unit(e))


def check_all(ctx, rules, units, rng, stats=None, sub_host=True, run_batch=(False, True)):
    """Every caller of the kernel on these rules and units; `run_batch` lists the cf_run_batch variants (with TOON or not)."""
    exp_s = [apply_rules(rules, u, stats) for u in units]
    exp = [engine.encode_unit(e) for e in exp_s]
    prog = build_program(rules).compile(ctx)
    n_unmatched = check_sub_host(ctx, prog, rules, units, exp, rng) if sub_host else 0
    for with_toon in run_batch:
        check_run_batch(ctx, prog, rules, units, exp, rng, with_toon)
    check_plugin(rules, units, exp_s)
    return n_unmatched


# ---------------------------------------------------------------------------------------------------------------------
# random rule programs
# ---------------------------------------------------------------------------------------------------------------------
ROUNDS = {"byte": (300, 70000), "pair": (100, 80000)}     # programs, first seed


@pytest.mark.gpu
@pytest.mark.parametrize("prefilter", ["byte", "pair"])
def test_random_rule_programs(prefilter, monkeypatch):
    """Random programs of 1-8 rules, each on short, long and planted units, through cf_sub_host, cf_run_batch (with and without
    TOON on alternate programs) and the plugin.  `pair`: CF_PAIR_FILTER=1, so the scan that picks the units to rewrite is the
    pair-prefilter variant (cf_sub_host, which takes its selection from the caller, is left to the `byte` rounds)."""
    monkeypatch.setenv("CF_PAIR_FILTER", "1" if prefilter == "pair" else "0")
    ctx = engine.Context.get()
    n_programs, seed0 = ROUNDS[prefilter]
    stats = {"programs": 0, "nullable": 0, "templates": 0, "planted": 0, "unmatched": 0, "near_edge": 0, "cross_edge": 0}
    d_cycle = itertools.cycle(EDGE_DS)
    for k in range(n_programs):
        rng = random.Random(seed0 + k)
        rules = rand_program(rng)
        if not rules:
            continue
        units, plants = program_units(rng, rules, d_cycle)
        assert build_program(rules).compile_host().prefilter == (prefilter == "pair")
        stats["unmatched"] += check_all(ctx, rules, units, rng, stats, sub_host=prefilter == "byte", run_batch=(k % 2 == 1,))
        stats["programs"] += 1
        stats["nullable"] += any(r.nullable for r in rules)
        stats["templates"] += any(r.refs for r in rules)
        stats["planted"] += sum(len(p) for p in plants)
    scale = n_programs / ROUNDS["byte"][0]
    assert stats["programs"] >= 300 * scale, stats
    assert stats["nullable"] >= 50 * scale and stats["templates"] >= 50 * scale, stats
    assert stats["near_edge"] >= 2000 * scale and stats["cross_edge"] >= 500 * scale, stats
    assert prefilter == "pair" or stats["unmatched"] >= stats["programs"], stats


# ---------------------------------------------------------------------------------------------------------------------
# rule chains and programs of more than 32 rules
# ---------------------------------------------------------------------------------------------------------------------
TOKENS = [chr(ord("a") + i) for i in range(26)] + [chr(0x3B1 + i) for i in range(25)] + [chr(0x4E00 + i) for i in range(60)]
CHAIN_FILL = list("0123456789 -+=") + ["€", "\U0001F600"]


def tok(k):
    """Token k of a chain: a, bb, c, dd, ...: the text grows and shrinks along the chain; one-, two- and three-byte letters."""
    return TOKENS[k] * (1 + k % 2)


def chain(n, identity_every=0, last=None):
    """Rule k rewrites tok(k) to tok(k + 1), so rule k + 1 matches what rule k wrote; every `identity_every`-th rule is instead
    tok(k) -> tok(k) (a match that changes nothing), followed by the rewrite as the next rule.  `last` replaces the final
    rule's replacement (e.g. "": the chain ends in nothing)."""
    rules, k = [], 0
    while len(rules) < n:
        if identity_every and len(rules) % identity_every == identity_every - 1:
            rules.append(Rule(re.escape(tok(k)), 0, tok(k)))
            continue
        rules.append(Rule(re.escape(tok(k)), 0, tok(k + 1)))
        k += 1
    if last is not None:
        rules[-1] = Rule(rules[-1].pattern, 0, last)
    return rules


def chain_units(rng, rules):
    toks = sorted({r.pattern for r in rules})
    toks = [re.sub(r"\\(.)", r"\1", t) for t in toks]

    def fill(n):
        return "".join(rng.choices(CHAIN_FILL, k=n))

    units = ["", "no tokens 123", fill(30)]
    for t in toks:                                    # enters the chain at one rule: every earlier rule (or launch) finds nothing
        units.append(fill(rng.randint(0, 5)) + t * rng.randint(1, 4) + fill(rng.randint(0, 5)))
        units.append(t)
    units.append("".join(rng.choice(toks) + fill(rng.randint(0, 2)) for _ in range(200)))
    units.append("".join(rng.choices(toks, k=60)))  # tokens only
    long = []
    for j in EDGE_JS:                                 # tokens across the 512-byte window edges
        long.append(fill(SUB_WIN - 3 - len("".join(long).encode()) % SUB_WIN) + "".join(rng.choices(toks, k=4)))
    units.append("".join(long))
    return units


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 7, 31, 32, 33, 64, 65, 100])
def test_rule_chains(n):
    """Chains where each rule rewrites what the previous one wrote, through every caller.  More than 32 rules run as several
    launches; units that only a later launch changes continue from the stream, the others from the scratch pair."""
    ctx = engine.Context.get()
    rng = random.Random(500 + n)
    for rules in (chain(n), chain(n, identity_every=3), chain(n, last="")):
        units = chain_units(rng, rules)
        if rules[-1].template == "":
            units += ["".join(rng.choices([re.sub(r"\\(.)", r"\1", r.pattern) for r in rules], k=k)) for k in (1, 5, 40)]
        check_all(ctx, rules, units, rng)
    rules = chain(n, last="")
    prog = build_program(rules).compile(ctx)
    whole = "".join(tok(k) for k in range(n))        # every rule matches, the end result is empty
    stream, offs = engine.pack_units([whole, tok(0), "x"])
    batch = engine.Batch(ctx, len(stream), 3)
    v, out, oo, _ = engine.run_batch(prog, batch, stream, offs, N.CF_STAGE_SUB)
    assert [int(f) & N.CF_V_REWRITTEN for f in v["flags"]] == [N.CF_V_REWRITTEN, N.CF_V_REWRITTEN, 0]
    assert int(oo[-1]) == 0 and apply_rules(rules, whole) == ""


@pytest.mark.gpu
def test_identity_rules_count_as_matches():
    """a -> a changes nothing, yet the unit was matched: cf_run_batch reports it rewritten (with the same text)."""
    ctx = engine.Context.get()
    rules = [Rule("a", 0, "a"), Rule("(b)", 0, r"\1"), Rule("c*", 0, r"\g<0>")]
    units = ["a", "b", "xyz", "", "aaa bbb", "\U0001F600a\U0001F600", "q" * 1000 + "a"]
    check_all(ctx, rules, units, random.Random(1))
    stream, offs = engine.pack_units(units)
    batch = engine.Batch(ctx, len(stream), len(units))        # owns the page-locked buffer `out` is a view of
    v, out, oo, _ = engine.run_batch(build_program(rules[:2]).compile(ctx), batch, stream, offs, N.CF_STAGE_SUB)
    raw = out[: int(oo[-1])].tobytes()
    for i, u in enumerate(units):
        assert bool(v["flags"][i] & N.CF_V_REWRITTEN) == ("a" in u or "b" in u)
        if v["flags"][i] & N.CF_V_REWRITTEN:
            assert raw[int(oo[i]):int(oo[i + 1])] == u.encode()


EARLY, LATE = [tok(k) for k in range(12)], [tok(k) for k in range(12, 24)]


def many_rules(n, rng):
    """n rules: token rewrites in random directions (including identities and deletions), some with flags and templates.  The
    rules of the first launch read and write the EARLY tokens, those of later launches the LATE ones, so a unit can change in
    the first launch only, in later ones only, in both or in none."""
    words = []
    for k in range(n):
        pool = EARLY if k < LAUNCH_RULES else LATE
        t = rng.choice(pool)
        kind = k % 4
        if kind == 0:
            words.append({"search": re.escape(t), "replace": rng.choice(pool)})
        elif kind == 1:
            words.append({"search": f"(?i)({re.escape(t)})+", "replace": rng.choice(["", r"<\1>", r"\g<0>", rng.choice(pool)])})
        elif kind == 2:
            words.append({"search": f"{re.escape(t)}[0-9]*", "replace": rng.choice([t, "", "日"])})
        else:
            words.append({"search": re.escape(t), "replace": t})
    return words


def count_units(rng):
    fill = ["1", "2", " ", "+"]
    units = ["", "1 2 3", "".join(rng.choices(fill, k=40))]
    for toks in (EARLY, LATE, EARLY + LATE):
        units += ["".join(rng.choices(toks + fill + CHAIN_FILL, k=rng.randint(1, 30))) for _ in range(25)]
        units.append("".join(rng.choices(toks + fill, k=900)))
    return units


def manager_for(words, td):
    from mcp_context_forge_b200.cpex_compat.framework import HookPayloadPolicy
    from mcp_context_forge_b200.manager import BatchedPluginManager

    cfg = os.path.join(td, "plugins.yaml")
    with open(cfg, "w", encoding="utf-8") as f:
        f.write("plugins:\n  - name: \"ReplaceBadWordsPlugin\"\n"
                "    kind: \"mcp_context_forge_b200.plugins.regex_filter.SearchReplacePlugin\"\n"
                "    hooks: [\"tool_pre_invoke\"]\n    mode: \"sequential\"\n    priority: 150\n    config:\n      words:\n")
        for w in words:
            f.write(f"        - {{search: {json.dumps(w['search'])}, replace: {json.dumps(w['replace'])}}}\n")
        f.write("plugin_settings:\n  plugin_timeout: 120\n")
    pol = {"tool_pre_invoke": HookPayloadPolicy(writable_fields=frozenset({"name", "args", "headers"}))}
    return BatchedPluginManager(cfg, timeout=120, hook_policies=pol)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [32, 33, 64, 100])
def test_rule_counts_through_plugin_and_manager(n):
    """regex_filter configs of exactly 32 rules and of more (33, 64, 100): the plugin and the batched manager (YAML config)
    give the oracle's output; cf_sub_host and cf_run_batch on the same program do too."""
    from mcp_context_forge_b200 import framework as fw

    rng = random.Random(900 + n)
    words = many_rules(n, rng)
    oracle = ref.regex_compile_rules(words)
    assert len(oracle) == n
    units = count_units(rng)
    check_all(engine.Context.get(), [Rule(w["search"], 0, w["replace"]) for w in words], units, rng)
    with tempfile.TemporaryDirectory() as td:
        m = manager_for(words, td)
        loop = asyncio.new_event_loop()
        loop.run_until_complete(m.initialize())
        payloads = [fw.ToolPreInvokePayload(name="t", args={"a": units[i], "b": units[-1 - i], "n": i}) for i in range(len(units) // 2)]
        gcs = [fw.GlobalContext(request_id=f"r{i}") for i in range(len(payloads))]
        async def wave():
            return await asyncio.gather(*[m.invoke_hook("tool_pre_invoke", p, g) for p, g in zip(payloads, gcs)])

        res = loop.run_until_complete(wave())
        for p, (r, _) in zip(payloads, res):
            exp = ref.regex_apply_dict(oracle, p.args)
            got = r.modified_payload.args if r.modified_payload is not None else p.args
            assert got == exp, (n, p.args)
        loop.run_until_complete(m.shutdown())


# ---------------------------------------------------------------------------------------------------------------------
# output at the scratch bound
# ---------------------------------------------------------------------------------------------------------------------
W40 = "日本語" * 4 + "語" + "!"                        # 40 bytes, 14 characters
assert len(W40.encode()) == 40

BOUND_PROGRAMS = {
    # a rule that can match "" gets L + 1 empty matches on a unit of L ASCII bytes, each replaced by 40 bytes
    "nullable-literal": [Rule("x*", 0, W40)],
    "nullable-lazy-literal": [Rule("x*?", 0, W40)],
    "nullable-g0": [Rule("a*", 0, r"\g<0>\g<0>\g<0>")],
    "nullable-lazy-g0": [Rule("(?:ab|a)*?", 0, r"\g<0>\g<0>\g<0>")],
    "nullable-class-g0": [Rule("[^x]*", 0, r"\g<0>\g<0>\g<0>"), Rule("(x)?", 0, r"[\1\g<0>]")],
    # eight rules of one character -> four bytes, each matching what the previous one wrote: 4^8 = 65536x
    "chain-8x4": [Rule(re.escape(TOKENS[k]), 0, TOKENS[k + 1] * 4) for k in range(8)],
    "chain-8x4-wide": [Rule("é", 0, "\U0001F600"), Rule("\U0001F600", 0, "éé")] + [Rule(re.escape(TOKENS[k]), 0, TOKENS[k + 1] * 4) for k in range(6)],
    # case-insensitive rules where a character is 2 or 3 bytes (ſ, İ, K = Kelvin sign) but one code point
    "ignorecase": [Rule("s", re.I, "ſſ"), Rule("ſ", re.I, "\u212a\u212a"), Rule("k", re.I, "İİ"), Rule("i\u0307|İ", re.I, "\U0001F600"),
                   Rule("(k+)", re.I, r"\1\1")],
}
BOUND_ALPH = {
    "nullable-literal": "xab日", "nullable-lazy-literal": "xab日", "nullable-g0": "ab日", "nullable-lazy-g0": "abx", "nullable-class-g0": "xay",
    "chain-8x4": TOKENS[:3], "chain-8x4-wide": ["é", "\U0001F600", "a", "b"], "ignorecase": ["s", "S", "ſ", "k", "K", "\u212a", "i", "I", "İ", "ı", "\u0307", " "],
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BOUND_PROGRAMS))
def test_output_at_scratch_bound(name):
    """Rules whose output reaches the scratch bound cf_sub_host computes, on many units in one call so that their scratch
    areas are adjacent: a bound that is too small is an error, and a neighbour's text would show any stray write."""
    ctx = engine.Context.get()
    rng = random.Random(sum(map(ord, name)))
    rules = BOUND_PROGRAMS[name]
    alph = list(BOUND_ALPH[name])
    big = name.startswith("chain")
    lens = [0, 1, 2, 3] if big else [0, 1, 2, 5, 17, 100, 700]
    units = []
    for L in lens:
        for _ in range(12 if big else 20):
            units.append("".join(rng.choices(alph, k=L)))
    for ch in alph[:3]:                                   # runs of one character: all-x and no-x units for `x*`
        units += [ch * L for L in ([1, 2, 4] if big else [1, 2, 255, 256, 257, 600, 3000])]
    rng.shuffle(units)
    check_all(ctx, rules, units, rng)


# ---------------------------------------------------------------------------------------------------------------------
# without a GPU: the generator and the kernel constants it aims at
# ---------------------------------------------------------------------------------------------------------------------
def test_window_constants_match_kernel():
    """The window sizes and the rules per launch this file plants around are the ones sub_kernel uses."""
    with open(CFGPU, encoding="utf-8") as f:
        src = f.read()
    assert int(re.search(r"\bSUB_WIN = (\d+);", src).group(1)) == SUB_WIN
    assert int(re.search(r"\bSUB_LAUNCH_RULES = (\d+);", src).group(1)) == LAUNCH_RULES
    body = src[src.index("sub_kernel(const __grid_constant__ SubParams P)"):src.index("__global__ void sub_compact_kernel")]
    nullable, plain = body[body.index("if (R.nullable)"):].split("} else", 1)
    # a rule that can match "": 8 positions per lane, SUB_WIN / 2 per iteration; otherwise 16 per lane, SUB_WIN per iteration
    assert "wbase += SUB_WIN / 2" in nullable and "(uint64_t)lane * 8" in nullable and 32 * 8 == NULL_WIN == SUB_WIN // 2
    assert "wbase += SUB_WIN)" in plain and "(uint64_t)lane * 16" in plain and 32 * 16 == SUB_WIN
    # the rule counts tested: one launch, exactly full, one rule into a second launch, two full launches and into a fourth
    assert {32, 33, 64, 100} <= {LAUNCH_RULES, LAUNCH_RULES + 1, 2 * LAUNCH_RULES, 100} and 100 > 3 * LAUNCH_RULES


def test_planted_matches_sit_at_their_offsets():
    """Every planted copy starts at the byte it was aimed at, `re` matches the rule there, and the wide character of the
    "pre" and "inside" units really straddles the window edge.  Every d = -20..20 and every mode turns up."""
    d_cycle = itertools.cycle(EDGE_DS)
    seen_d, modes, wins = set(), {"d": 0, "pre": 0, "inside": 0, "cross": 0}, set()
    for seed in range(80):
        rng = random.Random(3000 + seed)
        for r in rand_program(rng, make=plain_rule):
            for unit, plants in plants_for_rule(rng, r, d_cycle):
                ub = unit.encode()
                for p in plants:
                    mb = p.m.encode()
                    assert len(unit[:p.ci].encode()) == p.off and ub[p.off:p.off + len(mb)] == mb, (r, p.mode)
                    mm = r.c.match(unit, p.ci)
                    assert mm is not None and mm.end() > p.ci, (r, p.mode)
                    assert p.edge % p.win == 0 and p.win in ((SUB_WIN, NULL_WIN) if r.nullable else (SUB_WIN,))
                    if p.mode in ("d", "cross"):
                        assert abs(p.off - p.edge) <= NEAR
                        seen_d.add(p.off - p.edge)
                    else:
                        s, L = p.wide
                        assert s < p.edge < s + L and L > 1 and len(ub[s:s + L].decode()) == 1, (r, p.mode)
                        assert s + L == p.off if p.mode == "pre" else p.off <= s and s + L <= p.off + len(mb)
                    if p.mode == "cross":
                        assert p.off + len(mb) > p.edge + p.win
                    modes[p.mode] += 1
                    wins.add(p.win)
    assert seen_d == set(EDGE_DS), sorted(set(EDGE_DS) - seen_d)
    assert min(modes.values()) >= 20 and wins == {SUB_WIN, NULL_WIN}, modes


def test_tractable_keeps_cpython_fast():
    assert tractable(r"a\w*b", 0) and tractable(r"(x{1,3}|y)?z+", re.I) and tractable(r"(ab)*?c", 0)
    assert not tractable(r"\w*\w*x", 0) and not tractable(r"((k|k))*^9", 0) and not tractable(r"(\S[^a]*?|9)*?", 0)
