"""ctypes access to tools/toon_emu.cpp: the token-parallel TOON kernel body on the CPU warp emulator, first pass and the resolving
pass for mixed list-item arrays, as toon_tp_kernel runs them.  The library is compiled with g++ into a temporary directory on first use."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRCS = [os.path.join(ROOT, "tools", "toon_emu.cpp"), os.path.join(ROOT, "tests", "hostsim", "warp_emu.cpp")]
FB_MIXED_ITEM, TS_FALLBACK = 7, 7
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="toon_emu_"), "libtoonemu.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-DCF_WARP_EMU", "-o", so] + SRCS)
        _lib = ctypes.CDLL(so)
    return _lib


def toon_pass(text, resolve_mixed: bool, unlimited: bool = False, report_errors: bool = True, order: int = 0):
    """One pass: (status, toon_text_or_None, fallback reason, warp collectives)."""
    b = text if isinstance(text, bytes) else text.encode("utf-8", "surrogatepass")
    cap = len(b) * 6 + 4096 if unlimited else max(len(b) - 1, 0)
    out = ctypes.create_string_buffer(max(cap, 1))
    n, why, coll = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_ulonglong()
    st = lib().toon_emu_unit(b, len(b), out, cap, ctypes.byref(n), 1 if report_errors else 0, order, 1 if resolve_mixed else 0, ctypes.byref(why),
                             ctypes.byref(coll))
    assert st >= 0, st
    return st, (out.raw[: n.value].decode("utf-8", "surrogatepass") if st == 0 else None), why.value, coll.value


def toon_tp(text, **kw):
    """Both passes as on the device: (status, text, reason, collectives of the first pass, collectives of the resolving pass or 0)."""
    st, txt, why, c1 = toon_pass(text, False, **kw)
    if st == TS_FALLBACK and why == FB_MIXED_ITEM:
        st, txt, why, c2 = toon_pass(text, True, **kw)
        return st, txt, why, c1, c2
    return st, txt, why, c1, 0
