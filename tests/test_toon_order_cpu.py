"""The TOON first pass's cost key (json_tp.h order_events, summed by toon_order_kernel over a unit's first ORDER_WINDOW bytes) on
the CPU: the very header the kernel compiles, built into a small host library, against a plain Python restatement of the rule, and
on bench.py's payloads, where it must put every nested-config payload strictly above every tabular and prose one."""
import ctypes
import os
import random
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import toon_stage_breakdown  # noqa: E402

WINDOW = 2048

# the kernel's walk in 32-bit words (bytes past the window are zero, the word before the unit is zero)
SHIM = r"""
#include "json_tp.h"
extern "C" uint32_t order_key(const uint8_t* s, uint32_t len) {
  const uint32_t win = len < cftp::ORDER_WINDOW ? len : cftp::ORDER_WINDOW;
  uint32_t prev = 0, ev = 0;
  for (uint32_t i = 0; i < win; i += 4) {
    uint32_t w = 0;
    for (uint32_t k = 0; k < 4 && i + k < win; ++k) w |= (uint32_t)s[i + k] << (8 * k);
    ev += cftp::order_events(prev, w);
    prev = w;
  }
  return ev < 255u ? ev : 255u;
}
extern "C" uint32_t order_window() { return cftp::ORDER_WINDOW; }
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("order_key")
    src, so = d / "shim.cpp", d / "liborderkey.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-w", "-DCF_WARP_EMU", "-I", os.path.join(ROOT, "mcp_context_forge_b200", "csrc"),
                           str(src), os.path.join(ROOT, "tests", "hostsim", "warp_emu.cpp"), "-o", str(so)])
    L = ctypes.CDLL(str(so))
    L.order_key.restype = ctypes.c_uint32
    L.order_window.restype = ctypes.c_uint32
    return L


def key_ref(b: bytes) -> int:
    """'{' and '[' bytes of the first WINDOW bytes, minus each '{' right after "}," or "}, ", clamped to 8 bits."""
    w = b[:WINDOW]
    ev = sum(1 for c in w if c in b"{[")
    ev -= sum(1 for i, c in enumerate(w) if c == ord("{") and (w[max(0, i - 2):i] == b"}," or w[max(0, i - 3):i] == b"}, "))
    return min(ev, 255)


def key(lib, b: bytes) -> int:
    return int(lib.order_key(b, len(b)))


def test_window(lib):
    assert lib.order_window() == WINDOW


def test_rule_matches_restatement(lib):
    rng = random.Random(5)
    alphabet = b'{}[],: "a\\\n'
    cases = [b"", b"{", b"[", b"},{", b"}, {", b"},  {", b"} ,{", b"{" * 300, b"[" * 4000, b"x" * (WINDOW - 1) + b"{[", b"{" + b"},{" * 1000]
    for _ in range(3000):
        n = rng.choice([rng.randrange(0, 16), rng.randrange(0, 300), rng.randrange(1500, 2600)])
        cases.append(bytes(rng.choice(alphabet) for _ in range(n)))
    for c in cases:
        assert key(lib, c) == key_ref(c), c[:80]


def test_rows_of_a_table_do_not_count(lib):
    rows = ",".join('{"id":%d,"n":"x"}' % i for i in range(50))
    assert key(lib, ('{"results":[' + rows + "]}").encode()) == 3
    assert key(lib, ('{"results": [' + rows.replace(",{", ", {") + "]}").encode()) == 3
    assert key(lib, ('{"a":{"b":{"c":[1,[2,[3]]]}}}').encode()) == 6


def test_bench_payloads_nested_strictly_above(lib):
    by = {}
    for i, p in enumerate(bench.make_payloads()):
        by.setdefault(toon_stage_breakdown.shape_of(i), []).append(key(lib, p.encode()))
    assert set(by) == {"A", "B", "C"}
    assert min(by["B"]) > max(by["A"] + by["C"])
