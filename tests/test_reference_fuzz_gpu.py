"""The differential fuzzers replayed on the device: each tool's --device mode runs the same seeded inputs through the CUDA kernels
(cf_toon_host on every route, cf_run_batch, cf_mask_host, classify_keys_kernel) and through the drop-ins and the batched manager launching
for real, against the reference's answers recorded from its own modules (tests/golden/fuzz_*.json.gz, tools/ref_answers.py).  The CPU suite
replays the same recordings on the kernels' host build and the simulator (tests/test_reference_own_tests_cpu.py); the device build differs
in more than the compiler (shift and conversion semantics, local-memory limits, launch geometry, the order units are claimed in)."""
import gzip
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (tool, positional arguments as the recording stores them, recording, answers it holds, floor on compared=): the floor is what the
# host build / simulator replay of the same recording compares, so a run that skips work fails
RUNS = [
    ("fuzz_vs_reference.py", ["5", "4000", "gen1"], "fuzz_toon", 4000, 3921),
    ("fuzz_vs_reference.py", ["11", "10000", "gen2"], "fuzz_toon_gen2", 10000, 10000),
    ("fuzz_vs_reference.py", ["17", "10000", "gen2"], "fuzz_toon_gen2_s17", 10000, 10000),
    ("fuzz_vs_reference.py", ["12", "20000", "gen1"], "fuzz_toon_gen1_large", 20000, 19544),
    ("fuzz_mask_vs_reference.py", ["5", "8000", "800"], "fuzz_mask", 7964, 8163),
    ("fuzz_mask_vs_reference.py", ["13", "40000", "4000"], "fuzz_mask_large", 38067, 39066),
    ("fuzz_json_repair_vs_reference.py", ["5", "4000"], "fuzz_json_repair", 4000, 4000),
    ("fuzz_json_repair_vs_reference.py", ["14", "20000"], "fuzz_json_repair_large", 20000, 20000),
    ("fuzz_plugins_vs_reference.py", ["5", "12"], "fuzz_plugins", 3084, 3084),
    ("fuzz_plugins_vs_reference.py", ["15", "60"], "fuzz_plugins_large", 14940, 14940),
    ("fuzz_chain_vs_reference.py", ["5", "8", "40"], "fuzz_chain", 48, 1920),
    ("fuzz_chain_vs_reference.py", ["16", "40", "40"], "fuzz_chain_large", 240, 9600),
]
IDS = [name for _, _, name, _, _ in RUNS]


def _counts(stdout: str) -> dict:
    return {k: int(v) for k, v in re.findall(r"\b(\w+)=(\d+)\b", stdout.strip().splitlines()[-1])}


@pytest.mark.gpu
@pytest.mark.parametrize("tool,args,name,n_answers,floor", RUNS, ids=IDS)
def test_fuzz_replay_on_the_device(tool, args, name, n_answers, floor):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), *args, "--device", "--answers", name], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and " bad=0" in p.stdout, (p.stdout[-3000:], p.stderr[-3000:])
    c = _counts(p.stdout)
    assert c["bad"] == 0 and c["compared"] >= floor, c
    if tool == "fuzz_vs_reference.py":
        # the hand-over to the sequential encoder happened, not for every unit, and the exact number formatter was among its reasons
        assert 0 < c["handed_over"] < c["compared"] and c["handed_over_num_exact"] > 0, c


def test_device_table_matches_the_recordings():
    """Every recording the table names exists and holds the arguments and answer count the table passes (a stale table fails here, not on
    the device)."""
    for tool, args, name, n_answers, floor in RUNS:
        assert os.path.exists(os.path.join(ROOT, "tools", tool)), tool
        with gzip.open(os.path.join(ROOT, "tests", "golden", f"{name}.json.gz"), "rt", encoding="utf-8") as f:
            stored = json.load(f)
        assert stored["args"] == args and len(stored["answers"]) == n_answers, (name, stored["args"], len(stored["answers"]))
        assert floor > 0, name
