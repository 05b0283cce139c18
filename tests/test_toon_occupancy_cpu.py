"""Residency of the token-parallel TOON kernel, checked on the built library without a GPU.

toon_tp_kernel is latency-bound: a warp works through its unit in serial, dependent steps, and the warps resident on an SM are
what hides that latency.  It is built for TP_CTAS_PER_SM CTAs per SM (its launch bounds); this test reads the kernel's
register count and stack frame from `cuobjdump --dump-resource-usage` of libcfgpu.so and its launch shape from cf_toon_tp_config
(a test hook of the library, not part of the C API), and fails
when either the registers or the shared memory would no longer let that many CTAs share an H100 SM, so that a change which
silently drops back to fewer resident warps shows up here."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from mcp_context_forge_b200 import _native

# H100 (sm_90) per-SM limits
REGS_PER_SM = 65536
REG_ALLOC_UNIT = 256            # registers are allocated per warp in units of 256 (8 per thread)
SMEM_PER_SM = 228 * 1024
SMEM_RESERVED_PER_CTA = 1024    # the runtime's reservation per resident CTA
MIN_WARPS_PER_SM = 24


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip("cuobjdump not found")


def _launch_config():
    lib = ctypes.CDLL(_native.SO_PATH)
    w, c, s = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    lib.cf_toon_tp_config(ctypes.byref(w), ctypes.byref(c), ctypes.byref(s))
    return w.value, c.value, s.value


def _resource_usage():
    out = subprocess.run([_cuobjdump(), "--dump-resource-usage", _native.SO_PATH], capture_output=True, text=True, check=True).stdout
    m = re.search(r"Function \S*toon_tp_kernel\S*:\s*\n\s*(REG:.*)", out)
    assert m, "toon_tp_kernel not found in the library's resource usage"
    return {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", m.group(1))}


def test_launch_shape_keeps_24_warps_per_sm():
    warps, ctas, _ = _launch_config()
    assert warps * ctas >= MIN_WARPS_PER_SM


def test_registers_fit_the_ctas_per_sm():
    warps, ctas, _ = _launch_config()
    ru = _resource_usage()
    per_warp = -(-ru["REG"] * 32 // REG_ALLOC_UNIT) * REG_ALLOC_UNIT
    assert per_warp * warps * ctas <= REGS_PER_SM, f"{ru['REG']} registers per thread allow fewer than {ctas} CTAs of {warps} warps per SM"


def test_shared_memory_fits_the_ctas_per_sm():
    warps, ctas, smem = _launch_config()
    ru = _resource_usage()
    # SHARED is the static shared memory as cuobjdump reports it (on sm_90 it includes the 1 KiB reservation)
    static = max(ru["SHARED"] - SMEM_RESERVED_PER_CTA, 0)
    per_cta = smem + static + SMEM_RESERVED_PER_CTA
    assert ctas * per_cta <= SMEM_PER_SM, f"{per_cta} B of shared memory per CTA allow fewer than {ctas} CTAs per SM"


# The launch bounds make ptxas spill rather than exceed the register budget, so the register check above holds by construction;
# what a change that needs more registers costs shows up as spills, in the stack frame.  136 B today: 72 B of the emitter's own
# locals (the Emit object the out-of-line escx takes by reference, uint_dec's digits) and the tokenizer's spilled carries.
MAX_STACK_BYTES = 136


def test_stack_frame_does_not_grow():
    ru = _resource_usage()
    assert ru["STACK"] <= MAX_STACK_BYTES, f"toon_tp_kernel's stack frame grew to {ru['STACK']} B: registers are spilling"
