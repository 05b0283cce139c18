"""Differential fuzz of the drop-in PLUGINS (their host logic — unit extraction, verdict -> result assembly, findings
order, payload rebuilding — on the engine's CPU simulator) against the REFERENCE'S OWN plugin classes, imported unmodified from /root/reference:
regex_filter, deny_filter, harmful_content_detector, sql_sanitizer, code_safety_linter, toon_encoder.  Random configurations (from pools that
include rules matching "", group-reference templates, invalid patterns, IGNORECASE Unicode traps) and random payload shapes (nested dicts /
lists / non-strings, every hook each plugin implements).  A configuration the engine rejects loudly (UnsupportedPattern) is skipped and counted.
With --record the reference itself is run and its answers are stored (tools/ref_answers.py); without it they are read back from tests/golden/.
usage: python tools/fuzz_plugins_vs_reference.py [seed] [rounds] [--record]"""
import asyncio
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_golden  # noqa: E402
from ref_answers import Answers  # noqa: E402

WORDS = ["kill", "myself", "suicide", "self-harm", "want", "to", "die", "him", "her", "them", "someone", "shoot", "stab", "eradicate", "people", "racial", "slur", "hate", "speech", "crap",
         "crud", "innovative", "groundbreaking", "revolutionary", "the", "a", "of", "x", "Kill", "KILL", "ſuicide", "Kill", "é", "ß", "naïve", "日本語", "\U0001f600", "12", "_", "-", ".",
         ",", "\n", "DROP", "drop table t", "DELETE FROM t", "delete from t where x=1", "UPDATE t SET a=1", "update t set a=1 where b=2", "-- comment", "/* c */", "select * from t",
         "eval(", "exec (", "os.system('x')", "subprocess.run([", "rm -rf /", "'; --", "\"%s\" % x", "f\"{x}\"", "{} + {}", "buy now", "free", "xxy", "user@example.com", "555-1234", "a b",
         "zzz", "TRUNCATE", "alter", "GRANT all", "where", "#", "/*", "*/", "--", ";", "bell\x07", "\x01"]
SEPS = [" ", " ", " ", "", "  ", "\n", "-", "_", ".", "é", "1", "\t", ", "]
RULES = [("crap", "crud"), ("crud", "yikes"), (r"\bkill\b", "[k]"), ("(unclosed", "x"), (r"\d+", "#"), (r"cr[au]p+", "X"), (r"a|ab|abc", "<>"), ("a*", "-"), (r"(a)|b", r"[\1]"), (r"x*", "."),
         (r"(\w+)@(\w+)\.com", r"\2 at \1"), (r"\s+", " "), (r"(?i)kill", "K"), (r"é", "e"), (r"(?P<n>\d)(\d)", r"\g<n>-\2"), (r"^", ">"), (r"$", "<"), (r"\b", "|"), (r"[^\W\d_]+", "w"),
         (r"(a)\1", "bad"), (r"(?=x)", "la"), ("", "+"), (r"日本", "JP"), (r".", "d"), (r"\.", "dot")]
DENY = ["innovative", "groundbreaking", "revolutionary", "a b", "é", "x", "", "zzz", "kill", "Kill", "日本", "\n", "free", "--"]
HARM_CFG = [None, {"block_on": ["violence"]}, {"categories": {"spam": ["buy now", r"\bfree\b"], "x": ["x+y"]}, "block_on": ["spam"]}, {"block_on": []}, {"block_on": ["self_harm", "hate"]},
            {"categories": {"k": [r"k\w+l", "é+"], "w": [r"\bwhere\b"]}, "block_on": ["k", "w", "violence"]}]
import re as _re  # noqa: E402

HARM_CFG += [{"categories": {"c": [_re.compile("Kill"), _re.compile("him", _re.I), "Her"], "d": [_re.compile(r"k.ll\s+h", _re.S | _re.I), _re.compile(r"^die", _re.M)]}, "block_on": ["c", "d"]},
             {"categories": {"e": [_re.compile(r"\bé\w*", _re.I), _re.compile(r"ſ", _re.I), _re.compile(r"(?i)K")]}, "block_on": ["e"]}]
SQL_CFG = [None, {"block_on_violation": False}, {"block_on_violation": False, "require_parameterization": True, "fields": ["sql", "query"]}, {"strip_comments": False},
           {"fields": ["q"], "blocked_statements": [r"\bDROP\b", r"(?i)truncate\s+table"]}, {"require_parameterization": True}, {"block_delete_without_where": False, "block_update_without_where": False}]
CODE_CFG = [None, {"blocked_patterns": [r"curl\s+\S+\s*\|\s*sh", r"(?i)\bdrop\b", r"import\s+os"]}, {"blocked_patterns": []}, {"blocked_patterns": [r"rm\s+-rf", r"é+"]}]
TOON_CFG = [{"min_size_bytes": 10}, {"min_size_bytes": 10, "max_size_bytes": 300}, {"min_size_bytes": 10, "add_format_marker": False}, {"min_size_bytes": 40, "exclude_tools": ["other"]}, {"min_size_bytes": 10, "skip_on_error": False},
            {"min_size_bytes": 10, "skip_on_error": False, "add_format_marker": False}]


def text(rng, n=None):
    return "".join(rng.choice(WORDS) + rng.choice(SEPS) for _ in range(rng.randint(0, 7) if n is None else n))


def value(rng, depth):
    r = rng.random()
    if depth <= 0 or r < 0.45:
        return text(rng)
    if r < 0.55:
        return rng.choice([None, 5, 2.5, True, b"bytes".decode(), ""])
    if r < 0.75:
        return [value(rng, depth - 1) for _ in range(rng.randint(0, 3))]
    return {rng.choice(["sql", "query", "q", "text", "a", "b", "k1", "note", "content"]): value(rng, depth - 1) for _ in range(rng.randint(0, 4))}


def norm(r):
    v = r.violation.model_dump(include={"reason", "description", "code", "details"}) if r.violation is not None else None
    mp = r.modified_payload
    md = {k: x for k, x in (r.metadata or {}).items() if k != "conversion_time_ms"}
    res = getattr(mp, "result", None) if mp is not None else "-"
    if hasattr(res, "model_dump"):
        res = res.model_dump()
    return json.loads(json.dumps({"cont": r.continue_processing, "violation": v, "args": getattr(mp, "args", None) if mp is not None else "-", "result": res,
                                  "metadata": md}, default=str, sort_keys=True))


def main() -> int:
    record = "--record" in sys.argv
    argv = [a for a in sys.argv[1:] if a != "--record"]
    seed = int(argv[0]) if len(argv) > 0 else 1
    rounds = int(argv[1]) if len(argv) > 1 else 40
    answers = Answers("plugins", [seed, rounds], record)
    gen_golden.install_shims()
    import pytest
    from cpex.framework import GlobalContext, PluginConfig, PluginContext, PromptPosthookPayload, PromptPrehookPayload, ToolPostInvokePayload, ToolPreInvokePayload
    if record:
        from plugins.code_safety_linter.code_safety_linter import CodeSafetyLinterPlugin as RCode
        from plugins.deny_filter.deny import DenyListPlugin as RDeny
        from plugins.harmful_content_detector.harmful_content_detector import HarmfulContentDetectorPlugin as RHarm
        from plugins.regex_filter.search_replace import SearchReplacePlugin as RRegex
        from plugins.sql_sanitizer.sql_sanitizer import SQLSanitizerPlugin as RSql
        from plugins.toon_encoder.toon_encoder import ToonEncoderPlugin as RToon
    else:
        RCode = RDeny = RHarm = RRegex = RSql = RToon = None

    import hostsim_batcher
    from mcp_context_forge_b200.plugins.code_safety_linter import CodeSafetyLinterPlugin
    from mcp_context_forge_b200.plugins.deny_filter import DenyListPlugin
    from mcp_context_forge_b200.plugins.harmful_content_detector import HarmfulContentDetectorPlugin
    from mcp_context_forge_b200.plugins.regex_filter import SearchReplacePlugin
    from mcp_context_forge_b200.plugins.sql_sanitizer import SQLSanitizerPlugin
    from mcp_context_forge_b200.plugins.toon_encoder import ToonEncoderPlugin
    from mcp_context_forge_b200.regex_frontend import UnsupportedPattern

    hostsim_batcher.install(pytest.MonkeyPatch())
    ctx = PluginContext(global_context=GlobalContext(request_id="fuzz"))
    rng = random.Random(seed)
    loop = asyncio.new_event_loop()
    t0 = time.time()
    n = bad = rejected = raised = 0

    def payloads(kind):
        out = []
        for _ in range(24):
            if kind == "args":
                a = value(rng, 3)
                out.append(a if isinstance(a, dict) and rng.random() < 0.9 else {"k": text(rng), "sql": text(rng), "n": 7} if rng.random() < 0.8 else None)
            else:
                r = rng.random()
                out.append(text(rng) if r < 0.3 else value(rng, 3) if r < 0.7 else {"content": [{"type": "text", "text": json.dumps(value(rng, 3), ensure_ascii=False)}, {"type": "image", "data": "A"}], "isError": False})
        return out

    for rd in range(rounds):
        plan = [
            ("regex_filter", RRegex, SearchReplacePlugin, {"words": [{"search": s, "replace": r} for s, r in rng.sample(RULES, rng.randint(0, 4))]}, ["prompt_pre_fetch", "tool_pre_invoke", "tool_post_invoke", "prompt_post_fetch"]),
            ("deny_filter", RDeny, DenyListPlugin, {"words": rng.sample(DENY, rng.randint(0, 4))}, ["prompt_pre_fetch"]),
            ("harmful", RHarm, HarmfulContentDetectorPlugin, rng.choice(HARM_CFG), ["prompt_pre_fetch", "tool_post_invoke"]),
            ("sql_sanitizer", RSql, SQLSanitizerPlugin, rng.choice(SQL_CFG), ["prompt_pre_fetch", "tool_pre_invoke"]),
            ("code_safety", RCode, CodeSafetyLinterPlugin, rng.choice(CODE_CFG), ["tool_post_invoke"]),
            ("toon_encoder", RToon, ToonEncoderPlugin, rng.choice(TOON_CFG), ["tool_post_invoke"]),
        ]
        for name, rcls, ocls, cfg, hooks in plan:
            pc = PluginConfig(name=name, kind="x", hooks=hooks, config=cfg)
            ref = rcls(pc) if record else None
            try:
                ours = ocls(pc)
            except UnsupportedPattern:
                rejected += 1
                continue
            for hook in hooks:
                for p in payloads("args" if hook in ("prompt_pre_fetch", "tool_pre_invoke") else "result"):
                    if hook == "prompt_post_fetch":                                       # a rendered prompt: messages with text content
                        msgs = {"messages": [{"role": rng.choice(["user", "assistant"]), "content": {"type": "text", "text": text(rng)}} for _ in range(rng.randint(0, 4))]}
                        mk = lambda: PromptPosthookPayload(prompt_id="p", result=json.loads(json.dumps(msgs)))   # noqa: E731
                    elif hook == "prompt_pre_fetch":
                        mk = lambda: PromptPrehookPayload(prompt_id="p", args=p)          # noqa: E731
                    elif hook == "tool_pre_invoke":
                        mk = lambda: ToolPreInvokePayload(name="t", args=p)              # noqa: E731
                    else:
                        mk = lambda: ToolPostInvokePayload(name="t", result=p)           # noqa: E731
                    try:
                        pa, pb = mk(), mk()
                    except Exception:  # noqa: BLE001 - a payload shape the model rejects
                        continue
                    def reference():
                        try:
                            return norm(loop.run_until_complete(getattr(ref, hook)(pa, ctx)))
                        except Exception as exc:  # noqa: BLE001 - the reference raises: so must the drop-in
                            return {"raises": type(exc).__name__, "message": str(exc)}

                    exp = answers(reference)
                    try:
                        got = norm(loop.run_until_complete(getattr(ours, hook)(pb, ctx)))
                    except Exception as exc:  # noqa: BLE001
                        got = {"raises": type(exc).__name__, "message": str(exc)}
                    n += 1
                    raised += "raises" in exp
                    if exp != got:
                        bad += 1
                        if bad <= 6:
                            print("BAD", name, hook, repr(cfg)[:300], "\n  payload  ", repr(p)[:400], "\n  reference", json.dumps(exp, ensure_ascii=False)[:500],
                                  "\n  drop-in  ", json.dumps(got, ensure_ascii=False)[:500])
            if callable(getattr(ours, "get_stats", None)):      # toon_encoder's counters after the same calls
                n += 1
                exp = answers(lambda: ref.get_stats() if callable(getattr(ref, "get_stats", None)) else None)
                if exp is not None and exp != json.loads(json.dumps(ours.get_stats())):
                    bad += 1
                    if bad <= 6:
                        print("BAD stats", name, repr(cfg), exp, ours.get_stats())
    answers.finish()
    print(f"seed={seed} rounds={rounds} hook_calls={n} configs_rejected_loudly={rejected} reference_raised={raised} bad={bad} time={time.time() - t0:.1f}s")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
