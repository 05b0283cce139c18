"""The full Unicode sweeps through the C ABI on the GPU: every code point through the scan kernel (both prefilters) and the
substitution kernel, every scalar in every quoting-relevant TOON position on four routes, every short UTF-8 sequence at every
lane-window offset through the TOON and masking kernels, and the masking kernel's escaping, key order, key classes and
non-JSON probes.  The corpora and CPython's answers come from test_unicode_sweep_cpu.py; nothing here is compared with
another GPU path.  Each test prints its counts."""
import re
import time

import pytest

import test_unicode_sweep_cpu as U
from mcp_context_forge_b200 import engine, masking
from mcp_context_forge_b200 import regex_frontend as fe
from mcp_context_forge_b200._native import CF_STAGE_MASK, CF_STAGE_TOON, CF_V_MASKED
from oracle import mask_ref

pytestmark = pytest.mark.gpu

MAX_STREAM = 32 << 20                                  # bytes per launch
TOON_REPORT_ERRORS, TOON_SEQUENTIAL, TOON_NO_HANDOVER, HANDED_OVER = 1, 8, 16, 7


def chunks(units, max_bytes=MAX_STREAM):
    """Consecutive slices of `units` (bytes) whose packed stream stays within max_bytes."""
    i = 0
    while i < len(units):
        j, n = i, 0
        while j < len(units) and (j == i or n + len(units[j]) + 1 <= max_bytes):
            n += len(units[j]) + 1
            j += 1
        yield units[i:j]
        i = j


# ---------------------------------------------------------------------------------------------------------------------
# §1 scan
# ---------------------------------------------------------------------------------------------------------------------
_SCAN_EXP = {}


def plane_expected(plane):
    if plane not in _SCAN_EXP:
        _SCAN_EXP[plane] = U.scan_expected(range(plane << 16, (plane + 1) << 16))
    return _SCAN_EXP[plane]


@pytest.mark.parametrize("pair", [0, 1])
def test_scan_every_code_point(pair, monkeypatch):
    t0 = time.perf_counter()
    monkeypatch.setenv("CF_PAIR_FILTER", str(pair))
    ctx = engine.Context.get()
    prog = engine.Program()
    for p in U.SCAN_PATTERNS:
        prog.add_search(p)
    assert prog.compile_host().prefilter == pair
    prog.compile(ctx)
    assert prog.words == 1
    n_cp = n_units = matched = missed = 0
    for plane in range(17):
        cps = list(range(plane << 16, (plane + 1) << 16))
        units = U.scan_units(cps)
        stream, offs = engine.pack_units(units)
        got = engine.scan_host(prog, engine.Batch(ctx, len(stream), len(units)), stream, offs)
        exp = plane_expected(plane)
        bad = U.first_scan_mismatch(cps, got, exp)
        assert bad is None, bad
        a, b = U.bits_seen(exp)
        matched, missed = matched | a, missed | b
        n_cp += len(cps)
        n_units += len(units)
    full = (1 << len(U.SCAN_PATTERNS)) - 1
    assert n_cp == U.N_CP and matched == full and missed == full
    print(f"\nscan pair={pair}: {n_cp} code points, {n_units} units, {len(U.SCAN_PATTERNS)} patterns, {time.perf_counter() - t0:.1f}s")


# ---------------------------------------------------------------------------------------------------------------------
# §2 substitution
# ---------------------------------------------------------------------------------------------------------------------
SUB_CHUNK = 4096


def test_substitution_every_code_point():
    """Each rule as its own program and all six as one ordered chain, through engine.sub_host after a scan, against re.subn.  A
    unit the scan does not flag must come back unchanged and have no match."""
    t0 = time.perf_counter()
    ctx = engine.Context.get()
    units = U.sub_units(range(0, U.N_CP, 64))
    counts = {}
    for rules in [[r] for r in U.SUB_RULES] + [U.SUB_RULES]:
        prog = engine.Program()
        for p, r in rules:
            prog.add_sub(p, 0, fe.template_parts(r, re.compile(p)))
        prog.compile(ctx)
        total = 0
        for lo in range(0, len(units), SUB_CHUNK):
            part = units[lo:lo + SUB_CHUNK]
            stream, offs = engine.pack_units(part)
            batch = engine.Batch(ctx, len(stream), len(part))
            bm = engine.scan_host(prog, batch, stream, offs)
            got = engine.sub_host(prog, batch, list(range(len(part))))
            for u, g, b in zip(part, got, bm):
                text, n = U.sub_expected(rules, u)
                assert g.decode("utf-8", "surrogatepass") == text, (rules, ascii(u), ascii(g.decode("utf-8", "surrogatepass")), ascii(text))
                assert b or n == 0, (rules, ascii(u))
                total += n
        counts[" ; ".join(p for p, _ in rules) if len(rules) > 1 else rules[0][0]] = total
    assert all(counts.values()), counts
    print(f"\nsubstitution: {len(units)} units of 64 code points, {len(counts)} programs, matches {counts}, {time.perf_counter() - t0:.1f}s")


# ---------------------------------------------------------------------------------------------------------------------
# TOON and masking calls
# ---------------------------------------------------------------------------------------------------------------------
def toon_call(ctx, docs, flags):
    """cf_toon_host with explicit flags over `docs` (launches of at most MAX_STREAM bytes): [(status, text or None)], [out_len]."""
    res, lens = [], []
    for part in chunks(docs):
        stream, offs = engine.pack_units(part)
        status, texts, out_len = engine.toon_host_flags(engine.Batch(ctx, len(stream), len(part)), stream, offs, flags)
        res += [(int(s), None if t is None else t.decode("utf-8")) for s, t in zip(status, texts)]
        lens += out_len.tolist()
    return res, lens


def toon_run_batch(ctx, docs):
    """cf_run_batch(CF_STAGE_TOON): [(status, text or None)]."""
    res = []
    for part in chunks(docs):
        stream, offs = engine.pack_units(part)
        v, out, oo, _ = engine.run_batch(None, engine.Batch(ctx, len(stream), len(part)), stream, offs, CF_STAGE_TOON, toon_flags=TOON_REPORT_ERRORS)
        raw = out[: int(oo[-1])].tobytes()
        res += [(int(s), raw[int(oo[i]):int(oo[i + 1])].decode("utf-8") if s == 0 else None) for i, s in enumerate(v["aux"])]
    return res


def toon_routes(ctx, docs, exps):
    """The four routes on `docs` against `exps` [(status, text)]: returns {route: units compared}.  Without hand-over a unit may
    instead report one of the reasons U.handover_reasons allows for it."""
    seen = {}
    for name, flags in (("default", TOON_REPORT_ERRORS), ("sequential", TOON_REPORT_ERRORS | TOON_SEQUENTIAL),
                        ("no-handover", TOON_REPORT_ERRORS | TOON_NO_HANDOVER), ("run_batch", None)):
        if flags is None:
            got, why = toon_run_batch(ctx, docs), None
        else:
            got, why = toon_call(ctx, docs, flags)
        handed = 0
        for i, (d, e, g) in enumerate(zip(docs, exps, got)):
            if name == "no-handover" and g[0] == HANDED_OVER:
                assert why[i] in U.handover_reasons(d), (name, d[:160], why[i])
                handed += 1
                continue
            assert g == e, (name, d[:160], g[0], e[0], (g[1] or "")[:80], (e[1] or "")[:80])
        seen[name] = len(docs) - handed
    return seen


def mask_routes(ctx, docs, exps):
    """cf_mask_host and cf_run_batch(CF_STAGE_MASK) against `exps` (masked bytes, or None for a parse error)."""
    for part_lo, part in _indexed_chunks(docs):
        stream, offs = engine.pack_units(part)
        batch = engine.Batch(ctx, len(stream), len(part))
        st, outs = engine.mask_host(batch, stream, offs, 10)
        v, out, oo, _ = engine.run_batch(None, batch, stream, offs, CF_STAGE_MASK, mask_max_depth=10)
        raw = out[: int(oo[-1])].tobytes()
        for i, d in enumerate(part):
            e = exps[part_lo + i]
            assert (int(st[i]), outs[i]) == ((engine.MASK_OK, e) if e is not None else (engine.MASK_PARSE_ERROR, None)), ("cf_mask_host", d[:160], int(st[i]))
            g = raw[int(oo[i]):int(oo[i + 1])] if v["flags"][i] & CF_V_MASKED else None
            assert g == e and int(v["aux"][i]) == int(st[i]), ("cf_run_batch", d[:160], int(v["aux"][i]))


def _indexed_chunks(docs):
    lo = 0
    for part in chunks(docs):
        yield lo, part
        lo += len(part)


# ---------------------------------------------------------------------------------------------------------------------
# §3 TOON
# ---------------------------------------------------------------------------------------------------------------------
def test_toon_every_scalar_in_every_position():
    t0 = time.perf_counter()
    ctx = engine.Context.get()
    groups = U.toon_groups(range(U.N_CP))
    assert sum(len(g) for g in groups) == U.N_SCALARS
    n_docs, seen = 0, {}
    hits = set()
    for lo in range(0, len(groups), 1024):
        corpus = U.toon_corpus(groups[lo:lo + 1024])
        if lo == 0:
            U.assert_control_answers(corpus)
        hits |= U.toon_edge_hits(corpus)
        docs = [c[0] for c in corpus]
        for k, v in toon_routes(ctx, docs, [c[1] for c in corpus]).items():
            seen[k] = seen.get(k, 0) + v
        n_docs += len(docs)
    want = {(n, lo, hi, w) for n, ranges in (("digit", U.digit_ranges()), ("space", U.space_ranges())) for lo, hi in ranges
            for w in ("lo-1", "lo", "hi", "hi+1")}
    assert want <= hits, sorted(want - hits)[:4]
    assert seen["default"] == seen["sequential"] == seen["run_batch"] == n_docs and seen["no-handover"] > n_docs // 2, seen
    print(f"\ntoon: {U.N_SCALARS} scalars, {n_docs} documents, routes {seen}, {time.perf_counter() - t0:.1f}s")


# ---------------------------------------------------------------------------------------------------------------------
# §4 strict UTF-8
# ---------------------------------------------------------------------------------------------------------------------
def test_strict_utf8_every_short_sequence():
    t0 = time.perf_counter()
    ctx = engine.Context.get()
    seqs = U.utf8_sequences()
    cov = {j: [0, 0] for j in range(len(U.OFFSETS))}
    n_units = 0
    slices = [(seqs[i:i + 20000], False) for i in range(0, len(seqs), 20000)] + [(U.closing_quote_sequences(), True)]
    for part, quote_after in slices:
        units = U.utf8_units(part, quote_after)
        for j, (v, iv) in U.utf8_offset_coverage(units).items():
            cov[j][0] += v
            cov[j][1] += iv
        docs = [u[0] for u in units]
        toon_routes(ctx, docs, [U.utf8_toon_expected(d) for d in docs])
        mask_routes(ctx, docs, [U.utf8_mask_expected(d) for d in docs])
        n_units += len(units)
    assert all(v > 0 and iv > 0 for v, iv in cov.values()), cov
    print(f"\nstrict UTF-8: {len(seqs)} sequences + {len(U.closing_quote_sequences())} before the quote, {n_units} units, "
          f"{len(U.OFFSETS)} offsets, 4 TOON routes + 2 masking routes, {time.perf_counter() - t0:.1f}s")


# ---------------------------------------------------------------------------------------------------------------------
# §5 masking
# ---------------------------------------------------------------------------------------------------------------------
def test_masking_escapes_and_key_order():
    t0 = time.perf_counter()
    ctx = engine.Context.get()
    docs = U.mask_escape_docs(range(U.N_CP)) + U.mask_key_order_docs(range(U.N_CP))
    exps = [U.mask_expected(d) for d in docs]
    mask_routes(ctx, docs, exps)
    assert sum(e is None for e in exps) >= 2048 + 32 and sum(e is not None for e in exps) > len(docs) // 2
    print(f"\nmasking escapes + key order: {len(docs)} documents, {time.perf_counter() - t0:.1f}s")


def test_key_classes_every_scalar():
    t0 = time.perf_counter()
    ctx = engine.Context.get()
    keys = U.key_class_keys(range(U.N_CP))
    assert len(keys) == 3 * U.N_SCALARS
    n_sens = 0
    for lo in range(0, len(keys), 1 << 20):
        part = keys[lo:lo + (1 << 20)]
        enc = [engine.encode_unit(k) for k in part]
        got = engine.classify_keys_host(engine.Batch(ctx, sum(len(e) + 1 for e in enc), len(enc)), enc)
        exp = [mask_ref.is_sensitive_key(k) for k in part]
        if got != exp:
            i = next(i for i, (g, e) in enumerate(zip(got, exp)) if g != e)
            pytest.fail(f"key {ascii(part[i])}: kernel {got[i]}, mask_ref {exp[i]}")
        n_sens += sum(exp)
    assert 0 < n_sens < len(keys)
    print(f"\nkey classes: {len(keys)} keys, {n_sens} sensitive, {time.perf_counter() - t0:.1f}s")


def test_fallback_probes_every_cased_code_point():
    t0 = time.perf_counter()
    texts = U.probe_texts()
    got = masking.non_json_fallback_batch([t.encode("utf-8") for t in texts])
    bad = [ascii(t) for t, g in zip(texts, got) if (g == masking.NON_JSON_MASKED) != U.probe_expected(t)]
    assert not bad, bad[:8]
    n_hit = sum(U.probe_expected(t) for t in texts)
    assert 0 < n_hit < len(texts)
    print(f"\nfallback probes: {len(texts)} texts, {n_hit} sensitive, {time.perf_counter() - t0:.1f}s")
