"""ctypes access to tests/hostsim/libcfhostsim.so (TEST-ONLY CPU simulation of the scan tables)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "tests", "hostsim", "libcfhostsim.so")
SRCS = [
    os.path.join(ROOT, "tests", "hostsim", "host_sim.cpp"),
    os.path.join(ROOT, "mcp_context_forge_b200", "csrc", "cf_host.cpp"),
    os.path.join(ROOT, "mcp_context_forge_b200", "csrc", "re_backend.cpp"),
    os.path.join(ROOT, "tests", "hostsim", "warp_emu.cpp"),
]


def build(force=False):
    deps = SRCS + [os.path.join(ROOT, "mcp_context_forge_b200", "csrc", h) for h in ("scan_core.h", "re_backend.h", "cf_host.h", "json_toon.h", "json_mask.h", "json_index.h", "json_tp.h", "warp_prims.h", "unicode_tables.h")] + [os.path.join(ROOT, "tests", "hostsim", "warp_emu.h")]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-DCF_WARP_EMU", "-o", SO] + SRCS)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.cf_builder_last_error.restype = ctypes.c_char_p
    return _lib


class HostProgram:
    """Builder wrapper mirroring mcp_context_forge_b200.engine.Program but running on the CPU simulator."""

    def __init__(self):
        from mcp_context_forge_b200 import regex_frontend as fe

        self.fe = fe
        self.L = lib()
        self.b = ctypes.c_void_p()
        assert self.L.cf_builder_new(ctypes.byref(self.b)) == 0
        ws = np.array(fe.word_set(), dtype=np.uint32).reshape(-1)
        assert self.L.cf_builder_set_word_set(self.b, ws.ctypes.data_as(ctypes.c_void_p), len(ws) // 2) == 0
        self.n = 0

    def add_ast(self, ast, ordered=False, repl=None):
        a = np.array(ast, dtype=np.uint32)
        idx = ctypes.c_uint32()
        rc = self.L.cf_builder_add_pattern(self.b, a.ctypes.data_as(ctypes.c_void_p), len(a), 1 if ordered else 0, ctypes.byref(idx))
        assert rc == 0, self.err()
        if ordered and isinstance(repl, list):            # template parts: literal strings and group indices
            lit, parts = self.fe.encode_template(repl)
            pa = np.array(parts, dtype=np.uint32)
            rc = self.L.cf_builder_set_template(self.b, idx, lit, len(lit), pa.ctypes.data_as(ctypes.c_void_p), len(pa) // 3)
            assert rc == 0, self.err()
        elif ordered:
            r = (repl or "").encode("utf-8", "surrogatepass")
            assert self.L.cf_builder_set_replacement(self.b, idx, r, len(r)) == 0
        self.n += 1
        return idx.value

    def add(self, pattern, flags=0, ordered=False, repl=None):
        groups = isinstance(repl, list) and any(isinstance(p, int) for p in repl)
        return self.add_ast(self.fe.compile_ast(pattern, flags, "sub" if ordered else "search", groups=groups), ordered, repl)

    def err(self):
        return self.L.cf_builder_last_error(self.b).decode()

    def compile(self):
        stats = (ctypes.c_uint32 * 8)()
        rc = self.L.cf_builder_compile_host(self.b, stats)
        if rc:
            raise RuntimeError(f"compile rc={rc}: {self.err()}")
        return list(stats)

    def scan(self, units):
        """units: list[str] -> list[int] bitmaps (python ints), stats"""
        enc = [u.encode("utf-8", "surrogatepass") for u in units]
        stream = b"".join(e + b"\xff" for e in enc)
        offs = np.zeros(len(enc) + 1, dtype=np.uint64)
        np.cumsum([len(e) + 1 for e in enc], out=offs[1:])
        W = (self.n + 63) // 64
        bm = np.zeros(len(enc) * W, dtype=np.uint64)
        st = np.zeros(2, dtype=np.uint64)
        rc = self.L.cfh_scan(self.b, stream, ctypes.c_uint64(len(stream)), offs.ctypes.data_as(ctypes.c_void_p), len(enc),
                             bm.ctypes.data_as(ctypes.c_void_p), st.ctypes.data_as(ctypes.c_void_p))
        if rc:
            raise RuntimeError(f"scan rc={rc}: {self.err()}")
        out = []
        for i in range(len(enc)):
            v = 0
            for w in range(W):
                v |= int(bm[i * W + w]) << (64 * w)
            out.append(v)
        return out, [int(x) for x in st]

    def sub(self, ordered_index, text):
        e = text.encode("utf-8", "surrogatepass")
        cap = len(e) * 8 + 1024
        buf = ctypes.create_string_buffer(cap)
        olen = ctypes.c_uint64()
        nm = ctypes.c_uint64()
        rc = self.L.cfh_sub(self.b, ordered_index, e, ctypes.c_uint64(len(e)), buf, ctypes.c_uint64(cap), ctypes.byref(olen), ctypes.byref(nm))
        if rc:
            raise RuntimeError(f"sub rc={rc}: {self.err()}")
        return buf.raw[: olen.value].decode("utf-8", "surrogatepass"), nm.value

    def __del__(self):
        try:
            self.L.cf_builder_free(self.b)
        except Exception:
            pass


TOON_STATUS = {0: "converted", 1: "not_smaller", 2: "not_json", 3: "value_error", 4: "attr_error", 6: "unsupported"}


def toon_host(text: str, unlimited: bool = False, indexed: bool = False, stop_on_over: bool = False):
    """(status, toon_text_or_None) from the shared json_toon.h pipeline compiled for the CPU.
    unlimited=True lifts the product's "strictly smaller" capacity so the encoder output itself can
    be compared with the reference's toon.encode.  indexed=True parses through the structural index +
    token-driven builder (json_index.h — the path the CUDA kernels take) instead of the sequential parser.
    stop_on_over=True (sequential parser only) gives up once the output is past the capacity, as toon_kernel does when errors
    are not reported."""
    b = text if isinstance(text, bytes) else text.encode("utf-8", "surrogatepass")
    cap = len(b) * 6 + 4096 if unlimited else max(len(b) - 1, 0)
    out = ctypes.create_string_buffer(max(cap, 1))
    n = ctypes.c_uint32()
    if indexed:
        st = lib().cfh_toon_indexed(b, len(b), out, cap, ctypes.byref(n))
    else:
        st = lib().cfh_toon(b, len(b), out, cap, ctypes.byref(n), 1 if stop_on_over else 0)
    return st, (out.raw[: n.value].decode("utf-8", "surrogatepass") if st == 0 else None)


def toon_tp(text, unlimited: bool = False, report_errors: bool = True, order: int = 0):
    """(status, toon_text_or_None) from the TOKEN-PARALLEL warp kernel body (json_tp.h) run on the 32-fibre warp
    emulator.  status 7 = the unit is handed to the sequential encoder."""
    b = text if isinstance(text, bytes) else text.encode("utf-8", "surrogatepass")
    cap = len(b) * 6 + 4096 if unlimited else max(len(b) - 1, 0)
    out = ctypes.create_string_buffer(max(cap, 1))
    n = ctypes.c_uint32()
    why = ctypes.c_uint32()
    st = lib().cfh_toon_tp(b, len(b), out, cap, ctypes.byref(n), 1 if report_errors else 0, order, ctypes.byref(why))
    toon_tp.last_reason = why.value
    return st, (out.raw[: n.value].decode("utf-8", "surrogatepass") if st == 0 else None)


def index_equiv(data: bytes):
    """(code, status_sequential, status_indexed): code 0 = the sequential parser and index+builder agree."""
    a, b = ctypes.c_int(), ctypes.c_int()
    rc = lib().cfh_index_equiv(data, len(data), ctypes.byref(a), ctypes.byref(b))
    return rc, a.value, b.value


def json_index(data: bytes):
    """Token list of the structural index: [(pos, is_close_quote, aux)], unterminated flag."""
    n = len(data)
    pos = (ctypes.c_uint32 * (n + 1))()
    aux = (ctypes.c_uint32 * (n + 1))()
    unt = ctypes.c_int()
    L = lib()
    L.cfh_json_index.restype = ctypes.c_uint32
    nt = L.cfh_json_index(data, n, pos, aux, ctypes.byref(unt))
    return [(pos[i] & 0x7FFFFFFF, bool(pos[i] >> 31), aux[i]) for i in range(nt)], bool(unt.value)


MASK_OVERFLOW = 7


def mask_host(payload: bytes, max_depth: int = 10, indexed: bool = False, retry: bool = True):
    """(status, masked_bytes_or_None) from the shared json_mask.h pipeline compiled for the CPU, sized like cf_mask_host sizes a
    unit: 5 * len + 32 bytes of room, and a unit that reports MS_OVERFLOW (7) run again into exactly the length it asked for.
    retry=False returns the first pass as it is: (7, needed length) for a unit that outgrew its room."""
    fn = lib().cfh_mask_indexed if indexed else lib().cfh_mask
    cap = len(payload) * 5 + 32
    for _ in range(2):
        out = ctypes.create_string_buffer(max(cap, 1))
        n = ctypes.c_uint32()
        st = fn(payload, len(payload), max_depth, out, cap, ctypes.byref(n))
        if st != MASK_OVERFLOW or not retry:
            break
        cap = n.value
    if st == MASK_OVERFLOW:
        return st, n.value
    return st, (out.raw[: n.value] if st == 0 else None)


def key_sensitive_host(key: str) -> bool:
    b = key.encode("utf-8", "surrogatepass")
    return bool(lib().cfh_key_sensitive(b, len(b)))
