"""The whole product chain against the whole reference chain.  One YAML, two managers: the sequential `PluginManager` loading
the REFERENCE'S OWN plugin classes (kind: plugins.regex_filter.search_replace.SearchReplacePlugin, ... imported unmodified from /root/reference)
and `BatchedPluginManager` loading this repo's drop-ins (kind: mcp_context_forge_b200.plugins....) on the engine's CPU simulator — same priorities,
modes, conditions and hook policies, random waves of concurrent requests on the three hooks of the path, violations as results and as
exceptions.  Every request's (continue_processing, modified payload, violation, metadata) or raised error must be equal.
With --record the reference itself is run and its answers are stored (tools/ref_answers.py); without it they are read back from tests/golden/
(fuzz_chain.json.gz, or NAME.json.gz with --answers NAME).  --device runs the batched manager's launches on the GPU instead of the simulator.
usage: python tools/fuzz_chain_vs_reference.py [seed] [rounds] [requests per wave] [--record | --device] [--answers NAME]"""
import asyncio
import json
import os
import random
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_golden  # noqa: E402
from ref_answers import Answers, canon, split_argv  # noqa: E402

OURS = {"harm": "mcp_context_forge_b200.plugins.harmful_content_detector.HarmfulContentDetectorPlugin", "deny": "mcp_context_forge_b200.plugins.deny_filter.DenyListPlugin",
        "regex": "mcp_context_forge_b200.plugins.regex_filter.SearchReplacePlugin", "sql": "mcp_context_forge_b200.plugins.sql_sanitizer.SQLSanitizerPlugin",
        "code": "mcp_context_forge_b200.plugins.code_safety_linter.CodeSafetyLinterPlugin", "repair": "mcp_context_forge_b200.plugins.json_repair.JSONRepairPlugin",
        "toon": "mcp_context_forge_b200.plugins.toon_encoder.ToonEncoderPlugin"}
REFS = {"harm": "plugins.harmful_content_detector.harmful_content_detector.HarmfulContentDetectorPlugin", "deny": "plugins.deny_filter.deny.DenyListPlugin",
        "regex": "plugins.regex_filter.search_replace.SearchReplacePlugin", "sql": "plugins.sql_sanitizer.sql_sanitizer.SQLSanitizerPlugin",
        "code": "plugins.code_safety_linter.code_safety_linter.CodeSafetyLinterPlugin", "repair": "plugins.json_repair.json_repair.JSONRepairPlugin",
        "toon": "plugins.toon_encoder.toon_encoder.ToonEncoderPlugin"}
WORDS = ["hello", "crap", "crud", "innovative", "kill him", "suicide", "normal text", "Kill her", "revolutionary idea", "I want to die", "racial slur", "fine", "DROP table t -- crap",
         "select 1 /* c */", "delete from t", "eval(x)", "rm -rf /", "é", "ſuicide", "日本語", "user@example.com", "12", "update t set a=1", "groundbreaking", "x", "", "bell\x07"]


def config(rng):
    """One random chain: which plugins, their modes / priorities / configs (the same dict rendered with either set of `kind`s)."""
    rules = [["crap", "crud"], ["crud", "yikes"], ["(?i)(kill) (him|her)", r"\2 <\1>"], [r"\d+", "#"], ["a*", "-"], [r"(\w+)@(\w+)\.com", r"\2 at \1"], [r"\s+", " "], ["é", "e"]]
    mode = lambda: rng.choice(["sequential", "sequential", "transform", "audit", "enforce", "enforce_ignore_error", "permissive", "fire_and_forget", "concurrent", "disabled"])   # noqa: E731
    plugs = [
        {"k": "harm", "hooks": ["prompt_pre_fetch", "tool_post_invoke"], "mode": mode(), "priority": rng.choice([96, 40, 500]),
         "config": rng.choice([{}, {"block_on": ["violence"]}, {"categories": {"spam": ["buy now", r"\bfine\b"]}, "block_on": ["spam", "self_harm"]}])},
        {"k": "deny", "hooks": ["prompt_pre_fetch"], "mode": mode(), "priority": 100, "config": {"words": rng.sample(["innovative", "groundbreaking", "revolutionary", "é", "x"], rng.randint(0, 3))}},
        {"k": "regex", "hooks": ["prompt_pre_fetch", "tool_pre_invoke", "tool_post_invoke"], "mode": mode(), "priority": rng.choice([150, 50, 97]),
         "config": {"words": [{"search": s, "replace": r} for s, r in rng.sample(rules, rng.randint(1, 4))]}},
        {"k": "sql", "hooks": ["prompt_pre_fetch", "tool_pre_invoke"], "mode": mode(), "priority": 45, "config": rng.choice([{"block_on_violation": False}, {}, {"strip_comments": False}])},
        {"k": "code", "hooks": ["tool_post_invoke"], "mode": mode(), "priority": rng.choice([120, 30]), "config": {}},
        {"k": "repair", "hooks": ["tool_post_invoke"], "mode": mode(), "priority": 145, "config": {}},
        {"k": "toon", "hooks": ["tool_post_invoke"], "mode": mode(), "priority": 900, "config": rng.choice([{"min_size_bytes": 10}, {}, {"min_size_bytes": 10, "add_format_marker": False}, {"min_size_bytes": 10, "skip_on_error": False}]),
         "conditions": rng.choice([None, [{"tools": ["t", "u"]}]])},
    ]
    conds = [None, None, None, [{"tools": ["t", "u"]}], [{"server_ids": ["s1"]}], [{"tenant_ids": ["acme"]}], [{"user_patterns": ["ali"]}], [{"prompts": ["p"]}, {"tools": ["other"]}],
             [{"server_ids": ["s2"], "tools": ["t"]}], [{"user_patterns": ["bob*", "zed"]}]]
    for p in plugs:
        p["on_error"] = rng.choice(["fail", "fail", "ignore", "disable"])
        if "conditions" not in p:
            p["conditions"] = rng.choice(conds)
    return [p for p in plugs if rng.random() < 0.8]


def render(plugs, kinds, fail_all=False):
    import yaml

    out = []
    for p in plugs:
        d = {"name": p["k"], "kind": kinds[p["k"]], "hooks": p["hooks"], "mode": p["mode"], "priority": p["priority"], "config": p["config"], "on_error": p["on_error"]}
        if p.get("conditions"):
            d["conditions"] = p["conditions"]
        out.append(d)
    return yaml.safe_dump({"plugins": out, "plugin_settings": {"plugin_timeout": 120, "fail_on_plugin_error": fail_all}})


def main() -> int:
    argv, record, device, name = split_argv(sys.argv[1:])
    seed = int(argv[0]) if len(argv) > 0 else 1
    rounds = int(argv[1]) if len(argv) > 1 else 20
    nreq = int(argv[2]) if len(argv) > 2 else 60
    answers = Answers("chain", [seed, rounds, nreq], record, name)
    gen_golden.install_shims(reference=record)
    import logging

    import pytest

    import hostsim_batcher
    import test_manager_gpu as tm
    from mcp_context_forge_b200 import framework as fw, synth
    from mcp_context_forge_b200.manager import BatchedPluginManager
    from mcp_context_forge_b200.regex_frontend import UnsupportedPattern

    logging.disable(logging.ERROR)
    if not device:
        hostsim_batcher.install(pytest.MonkeyPatch())
    rng = random.Random(seed)
    loop = asyncio.new_event_loop()
    t0 = time.time()
    n = bad = rejected = slow = 0
    for rd in range(rounds):
        plugs = config(rng)
        with tempfile.TemporaryDirectory() as td:
            a, b = os.path.join(td, "ref.yaml"), os.path.join(td, "ours.yaml")
            fail_all = rng.random() < 0.2
            open(a, "w").write(render(plugs, REFS, fail_all))
            open(b, "w").write(render(plugs, OURS, fail_all))
            seq = fw.PluginManager(a, timeout=120, hook_policies=tm.POL) if record else None
            bat = BatchedPluginManager(b, timeout=120, hook_policies=tm.POL, max_wave=rng.choice([8192, 8192, 7, 1, 33]), window_us=rng.choice([0, 0, 50, 400]))
            if record:
                loop.run_until_complete(seq.initialize())
            try:
                loop.run_until_complete(bat.initialize())
            except (UnsupportedPattern, RuntimeError) as exc:
                if "Unsupported" not in repr(exc) and "unsupported" not in repr(exc):
                    raise
                rejected += 1
                continue
            pre, tpre, post = [], [], []
            for i in range(nreq):
                args = {f"k{j}": " ".join(rng.choice(WORDS) for _ in range(rng.randint(1, 6))) for j in range(rng.randint(0, 3))}
                if rng.random() < 0.15:
                    args["n"] = rng.randint(0, 9)
                pre.append(fw.PromptPrehookPayload(prompt_id="p", args=args))
                tpre.append(fw.ToolPreInvokePayload(name="t", args=dict(args)))
                r = rng.random()
                if r < 0.45:
                    text = synth.payload("A", rng.choice([300, 1500]), seed=i + rd * 1000) if rng.random() < 0.6 else json.dumps({"note": rng.choice(WORDS), "x": [1, 2, {"y": rng.choice(WORDS)}]})
                    result = {"content": [{"type": "text", "text": text}, {"type": "text", "text": rng.choice(WORDS) * 3}], "summary": rng.choice(WORDS) + " crap"}
                elif r < 0.6:
                    result = rng.choice(["{'a': 1, 'b': [1, 2,],}", '{"a": "crap", "b": [1, 2, 3]}', "[1, 2, 3,] crap", '"k": "kill him"', "{'x': 'eval(1)'}", "[1,2,3]", "not json " + rng.choice(WORDS)])
                elif r < 0.8:
                    result = " ".join(rng.choice(WORDS) for _ in range(rng.randint(0, 8)))
                else:
                    result = rng.choice([{"text": rng.choice(WORDS), "other": rng.choice(WORDS)}, None, 5, [rng.choice(WORDS)], {"a": {"b": rng.choice(WORDS)}, "c": [rng.choice(WORDS), 3]}])
                post.append(fw.ToolPostInvokePayload(name=rng.choice(["t", "u", "other"]), result=result))
            gcs = [fw.GlobalContext(request_id=f"r{i}", server_id=rng.choice([None, "s1", "s2"]), tenant_id=rng.choice([None, "acme", "other"]), user=rng.choice([None, "alice", "bob7", "zed"]))
                   for i in range(nreq)]
            for hook, pls in (("prompt_pre_fetch", pre), ("tool_pre_invoke", tpre), ("tool_post_invoke", post)):
                for vae in (False, True):
                    async def wave(m):
                        return await asyncio.gather(*[m.invoke_hook(hook, p, g, None, vae) for p, g in zip(pls, gcs)], return_exceptions=True)
                    x = answers(lambda: [tm.norm(u) for u in loop.run_until_complete(wave(seq))])
                    y = loop.run_until_complete(wave(bat))
                    for i, (u, v) in enumerate(zip(x, y)):
                        n += 1
                        if u != canon(tm.norm(v)):
                            bad += 1
                            if bad <= 5:
                                print("BAD", hook, "vae", vae, "\n  chain    ", [(p["k"], p["mode"], p["priority"]) for p in plugs], "\n  payload  ", repr(pls[i])[:400], "\n  reference", repr(u)[:600],
                                      "\n  product  ", repr(tm.norm(v))[:600])
            slow += bat.slow_path_calls
    answers.finish()
    print(f"seed={seed} chains={rounds} rejected_loudly={rejected} requests={n} compared={n} slow_path_calls={slow} bad={bad} time={time.time() - t0:.1f}s")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
