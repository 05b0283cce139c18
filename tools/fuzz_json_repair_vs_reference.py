"""Differential fuzz of the json_repair drop-in (on the engine's CPU simulator: JSON kernel source for "does it parse",
substitution routines for the trailing-comma rule) against the REFERENCE'S OWN plugins/json_repair/json_repair.py, imported unmodified from
/root/reference (orjson stood in for by the strict stdlib parser; texts that would expose an orjson / json delta are skipped).
With --record the reference itself is run and its answers are stored (tools/ref_answers.py); without it they are read back from tests/golden/.
usage: python tools/fuzz_json_repair_vs_reference.py [seed] [cases] [--record]"""
import os
import random
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_golden  # noqa: E402
from fuzz_toon_tp import make_gen  # noqa: E402
from ref_answers import Answers  # noqa: E402

_DELTA = re.compile(r"\d{18,}|[eE][+-]?\d{3,}|\\u[dD][89a-fA-F]|NaN|Infinity")


def main() -> int:
    record = "--record" in sys.argv
    argv = [a for a in sys.argv[1:] if a != "--record"]
    seed = int(argv[0]) if len(argv) > 0 else 1
    n = int(argv[1]) if len(argv) > 1 else 3000
    answers = Answers("json_repair", [seed, n], record)
    gen_golden.install_shims()
    import pytest
    from cpex.framework import GlobalContext, PluginConfig, PluginContext, ToolPostInvokePayload

    import hostsim_batcher
    import test_json_repair as tj
    from mcp_context_forge_b200.plugins.json_repair import JSONRepairPlugin

    hostsim_batcher.install(pytest.MonkeyPatch())
    if record:
        from plugins.json_repair.json_repair import JSONRepairPlugin as RefPlugin

        ref = RefPlugin(PluginConfig(name="jr", kind="x", hooks=["tool_post_invoke"]))
    ctx = PluginContext(global_context=GlobalContext(request_id="fuzz"))

    def reference(t):
        r = gen_golden.run(ref.tool_post_invoke(ToolPostInvokePayload(name="t", result=t), ctx))
        return {"continue_processing": r.continue_processing, "out_result": r.modified_payload.result if r.modified_payload is not None else None,
                "modified": r.modified_payload is not None, "metadata": r.metadata or {}}

    rng = random.Random(seed)
    case = make_gen(rng)
    t0 = time.time()
    cases = []
    while len(cases) < n:
        t = case()
        k = rng.random()
        if k < 0.25:
            t = t.replace('"', "'")
        elif k < 0.5:
            t = re.sub(r"([}\]])", lambda m: rng.choice([",", ", ", ",\n", "", ""]) + m.group(1), t)
        elif k < 0.6 and t.startswith("{") and t.endswith("}"):
            t = t[1:-1]
        t = rng.choice(["", "", " ", "\n", " ", "\t"]) + t + rng.choice(["", "", " ", "\r\n", "　"])
        if _DELTA.search(t) or any(0xD800 <= ord(c) <= 0xDFFF for c in t) or t.count("[") + t.count("{") > 60:
            continue
        cases.append({"result": t, **answers(lambda: reference(t))})
    try:
        for i in range(0, len(cases), 500):
            tj.check_dropin(cases[i:i + 500], JSONRepairPlugin)
    except AssertionError as exc:
        print("BAD", str(exc)[:1500])
        return 1
    answers.finish()
    print(f"seed={seed} cases={len(cases)} repaired={sum(c['modified'] for c in cases)} bad=0 time={time.time() - t0:.1f}s")
    return 0


if __name__ == "__main__":
    sys.exit(main())
