"""The reference's own evidence, replayed without its tree: the recorded outcome of its own test files run against this repo
(tests/golden/reference_tests_run_*.json, made by tools/run_reference_tests.py; the executor scenarios they hold are restated in
tests/test_executor_reference_cases.py) and the differential fuzzers, whose reference answers are stored under tests/golden/fuzz_*.json.gz
(tools/ref_answers.py).  The executor restatement, the drop-in plugins and the kernels' source run live on the engine's CPU simulator."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_committed_run_records_have_no_unexplained_failure():
    for name in ("framework", "dropin"):
        with open(os.path.join(ROOT, "tests", "golden", f"reference_tests_run_{name}.json")) as f:
            s = json.load(f)
        assert s["passed"] > 0 and all(v["bucket"] != "other" for v in s["not_passed_detail"].values())


@pytest.mark.parametrize("tool,args", [("fuzz_vs_reference.py", ["5", "4000"]), ("fuzz_mask_vs_reference.py", ["5", "8000", "800"]), ("fuzz_json_repair_vs_reference.py", ["5", "4000"]),
                                       ("fuzz_plugins_vs_reference.py", ["5", "12"]), ("fuzz_chain_vs_reference.py", ["5", "8", "40"])])
def test_live_differential_fuzz_against_the_reference(tool, args):
    """A short run of each differential fuzzer (kernel source on the host build / warp emulator, drop-ins and the batched chain on the CPU
    simulator) against the reference's answers for the same seeded inputs, recorded from the reference's own modules."""
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), *args], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and " bad=0" in p.stdout, (p.stdout[-2000:], p.stderr[-2000:])
