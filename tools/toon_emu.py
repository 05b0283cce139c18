"""ctypes access to tools/toon_emu.cpp: the token-parallel TOON kernel body on the CPU warp emulator, as toon_tp_kernel runs it (the
first attempt, and the in-place retry of a unit that stops at a mixed list-item array), plus the separate resolving pass that retry
replaced.  The library is compiled with g++ into a temporary directory on first use."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRCS = [os.path.join(ROOT, "tools", "toon_emu.cpp"), os.path.join(ROOT, "tests", "hostsim", "warp_emu.cpp")]
FB_MIXED_ITEM, TS_FALLBACK = 7, 7
FIRST, RESOLVE, IN_PLACE = 0, 1, 2          # toon_emu.cpp's modes
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="toon_emu_"), "libtoonemu.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-DCF_WARP_EMU", "-o", so] + SRCS)
        _lib = ctypes.CDLL(so)
    return _lib


def run(text, mode: int, unlimited: bool = False, report_errors: bool = True, order: int = 0):
    """One emulated run in toon_emu.cpp's `mode`: (status, toon_text_or_None, fallback reason, out_len, warp collectives)."""
    b = text if isinstance(text, bytes) else text.encode("utf-8", "surrogatepass")
    cap = len(b) * 6 + 4096 if unlimited else max(len(b) - 1, 0)
    out = ctypes.create_string_buffer(max(cap, 1))
    n, why, coll = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_ulonglong()
    st = lib().toon_emu_unit(b, len(b), out, cap, ctypes.byref(n), 1 if report_errors else 0, order, mode, ctypes.byref(why), ctypes.byref(coll))
    assert st >= 0, st
    return st, (out.raw[: n.value].decode("utf-8", "surrogatepass") if st == 0 else None), why.value, n.value, coll.value


def toon_pass(text, resolve_mixed: bool, **kw):
    """One pass over the unit from its bytes, the first attempt or the resolving pass: (status, toon_text_or_None, fallback reason,
    warp collectives)."""
    st, txt, why, _, coll = run(text, RESOLVE if resolve_mixed else FIRST, **kw)
    return st, txt, why, coll


def toon_tp(text, **kw):
    """The unit as toon_tp_kernel encodes it, a mixed list-item array retried in place: (status, toon_text_or_None, fallback reason,
    out_len, warp collectives)."""
    return run(text, IN_PLACE, **kw)
