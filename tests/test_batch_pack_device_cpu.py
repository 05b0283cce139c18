"""The offsets and coarse unit index cf_batch_pack_device builds on the device (cf::packed_offset / cf::packed_coarse in
scan_core.h), in their host build, held to a restatement of cf_batch_upload's host sweep over the offsets the same units get when
they are packed on the host.  Random offset arrays with empty units, units that end or start on a 4 KiB boundary, units of exactly
4096 bytes, single units, and sources whose first unit does not start at 0.

The host build is a small shared library compiled here from scan_core.h with g++ (the header is plain C++ on the host), into the
test session's temporary directory."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mcp_context_forge_b200", "csrc")
COARSE_SHIFT = 12
SHIM = r"""
#include "scan_core.h"
// offsets[0 .. n], coarse[0 .. (src_bytes + n) >> COARSE_SHIFT] of a batch packed from src_off, as the device kernels compute them
extern "C" void pack_index(const uint64_t* src_off, uint32_t n, uint64_t src_bytes, uint64_t* offsets, uint32_t* coarse) {
  const uint64_t nbytes = src_bytes + n;
  for (uint32_t i = 0; i <= n; ++i) offsets[i] = cf::packed_offset(src_off, i, nbytes);
  for (uint64_t k = 0; k <= nbytes >> cf::COARSE_SHIFT; ++k) coarse[k] = cf::packed_coarse(src_off, n, nbytes, k);
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("pack_index")
    src, so = d / "pack_index.cpp", d / "libpack_index.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", str(so), str(src)])
    lib = ctypes.CDLL(str(so))
    lib.pack_index.restype = None
    lib.pack_index.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def upload_sweep(offsets, nbytes):
    """cf_batch_upload's coarse index: for every 4 KiB position, the last unit whose start is at or before it."""
    n = len(offsets) - 1
    coarse, u = [], 0
    for k in range((nbytes >> COARSE_SHIFT) + 1):
        pos = k << COARSE_SHIFT
        while u + 1 < n and offsets[u + 1] <= pos:
            u += 1
        coarse.append(u)
    return coarse


def host_pack(lengths, base):
    """(source offsets, src_bytes, the offsets pack_units gives the same units)."""
    src = np.zeros(len(lengths) + 1, dtype=np.uint64)
    np.cumsum(np.asarray(lengths, dtype=np.uint64), out=src[1:])
    packed = [int(src[i]) + i for i in range(len(lengths) + 1)]
    return src + np.uint64(base), int(src[-1]), packed


def pack_index(lib, src_off, n, src_bytes):
    nbytes = src_bytes + n
    offs = np.zeros(n + 1, dtype=np.uint64)
    coarse = np.zeros((nbytes >> COARSE_SHIFT) + 1, dtype=np.uint32)
    lib.pack_index(src_off.ctypes.data, n, src_bytes, offs.ctypes.data, coarse.ctypes.data)
    return [int(x) for x in offs], [int(x) for x in coarse]


def lengths_for(rng, kind, n):
    if kind == "random":
        return [rng.choice([0, 0, 1, 7, 100, 4095, 4096, 4097, rng.randrange(20000)]) for _ in range(n)]
    if kind == "empty":
        return [0] * n
    if kind == "page":                      # unit + terminator = 4096: every unit starts on a 4 KiB boundary
        return [4095] * n
    if kind == "exact":
        return [4096] * n
    if kind == "mixed_boundaries":          # runs of empty units right at, before and after coarse boundaries
        out, pos = [], 0
        while len(out) < n:
            gap = 4096 - (pos % 4096)
            ln = rng.choice([gap - 1, max(gap - 2, 0), gap, 0, 0, rng.randrange(9000)])
            out.append(ln)
            pos += ln + 1
        return out
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["random", "empty", "page", "exact", "mixed_boundaries"])
@pytest.mark.parametrize("n", [1, 2, 3, 17, 300])
def test_packed_offsets_and_coarse_match_the_upload_sweep(shim, kind, n):
    rng = random.Random(n * 31 + len(kind))
    for trial in range(6):
        base = rng.choice([0, 1, 13, 4096, 1 << 33])
        src_off, src_bytes, packed = host_pack(lengths_for(rng, kind, n), base)
        offs, coarse = pack_index(shim, src_off, n, src_bytes)
        assert offs == packed, (kind, n, trial)
        assert offs[-1] == src_bytes + n
        assert coarse == upload_sweep(packed, src_bytes + n), (kind, n, trial)


def test_offsets_that_are_not_monotone_stay_inside_the_stream(shim):
    """Garbage offsets give wrong units, never a position past the stream or a unit index past the batch."""
    rng = random.Random(5)
    for _ in range(200):
        n = rng.randrange(1, 40)
        src_off = np.array([rng.randrange(1 << 20) for _ in range(n + 1)], dtype=np.uint64)
        src_bytes = rng.randrange(1 << 16)
        offs, coarse = pack_index(shim, src_off, n, src_bytes)
        assert all(0 <= o <= src_bytes + n for o in offs)
        assert all(0 <= c < n for c in coarse)
