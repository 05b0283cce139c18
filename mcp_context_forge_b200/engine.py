"""Host-side engine objects over the C ABI (include/cfgpu.h): Context, Program, Batch.

These are thin: packing of Python strings into the packed-stream layout, pattern front-end calls,
and error translation.  All data-path work happens in libcfgpu.so on the GPU.
"""
from __future__ import annotations

import ctypes
import threading
from ctypes import byref, c_uint32, c_uint64, c_void_p
from typing import Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _native as N
from . import regex_frontend as fe

TERM = b"\xff"


def encode_unit(u: Union[str, bytes]) -> bytes:
    """UTF-8 with 'surrogatepass' so every Python str (even with lone surrogates) has a byte form
    whose decoding reproduces the same code points the reference's `re` sees."""
    return u if isinstance(u, bytes) else u.encode("utf-8", "surrogatepass")


def pack_units(units: Sequence[Union[str, bytes]]) -> Tuple[bytes, np.ndarray]:
    """Pack units into the stream layout of include/cfgpu.h: unit 0xFF unit 0xFF ..., uint64 offsets."""
    enc = [encode_unit(u) for u in units]
    stream = TERM.join(enc) + TERM if enc else b""
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        np.cumsum(np.fromiter((len(e) + 1 for e in enc), dtype=np.uint64, count=len(enc)), out=offs[1:])
    return stream, offs


class Context:
    """One per (process, device).  Not thread-safe: calls are serialised with a lock."""

    _instances: dict = {}
    _ilock = threading.Lock()

    def __init__(self, device: int = 0):
        self.lib = N.load()
        self.h = c_void_p()
        rc = self.lib.cf_init(device, byref(self.h))
        if rc != N.CF_OK:
            msg = self.lib.cf_last_error(self.h).decode() if self.h else "no CUDA device / driver"
            raise N.CfError(rc, f"cf_init(device={device}) failed: {msg}")
        self.device = device
        self.lock = threading.RLock()

    @classmethod
    def get(cls, device: int = 0) -> "Context":
        with cls._ilock:
            ctx = cls._instances.get(device)
            if ctx is None:
                ctx = cls._instances[device] = Context(device)
            return ctx

    def check(self, rc: int, what: str) -> None:
        if rc != N.CF_OK:
            raise N.CfError(rc, f"{what}: {self.lib.cf_last_error(self.h).decode()}")

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.cf_kernel_launches(self.h))

    def scan_counters(self) -> Tuple[int, int]:
        out = (c_uint64 * 2)()
        self.check(self.lib.cf_scan_counters(self.h, out), "cf_scan_counters")
        return int(out[0]), int(out[1])


class Program:
    """A set of patterns compiled for the GPU.  Pattern i owns bit i of every verdict bitmap."""

    def __init__(self):
        self.lib = N.load()
        self.b = c_void_p()
        rc = self.lib.cf_builder_new(byref(self.b))
        if rc != N.CF_OK:
            raise N.CfError(rc, "cf_builder_new")
        ws = np.asarray(fe.word_set(), dtype=np.uint32).reshape(-1)
        self._check_b(self.lib.cf_builder_set_word_set(self.b, ws.ctypes.data, len(ws) // 2), "word set")
        self.n_patterns = 0
        self.n_ordered = 0
        self.h: Optional[c_void_p] = None
        self.ctx: Optional[Context] = None

    def _check_b(self, rc: int, what: str) -> None:
        if rc != N.CF_OK:
            raise N.CfError(rc, f"{what}: {self.lib.cf_builder_last_error(self.b).decode()}")

    def _add(self, ast: List[int], flags: int) -> int:
        a = np.asarray(ast, dtype=np.uint32)
        idx = c_uint32()
        self._check_b(self.lib.cf_builder_add_pattern(self.b, a.ctypes.data, len(a), flags, byref(idx)), "add_pattern")
        self.n_patterns += 1
        return idx.value

    def add_search(self, pattern: str, flags: int = 0) -> int:
        """`re.compile(pattern, flags).search(unit)` existence bit."""
        return self._add(fe.compile_ast(pattern, flags, "search"), N.CF_PAT_SEARCH)

    def add_literal(self, word: str) -> int:
        """`word in unit` existence bit (deny_filter)."""
        return self._add(fe.literal_ast(word), N.CF_PAT_SEARCH)

    def add_sub(self, pattern: str, flags: int, replacement) -> int:
        """One regex_filter rule: `re.compile(pattern, flags).sub(replacement, unit)`.  `replacement` is the EXPANDED template:
        a literal string, or the flat list of literal strings and group indices `regex_frontend.template_parts` returns."""
        if isinstance(replacement, str):
            replacement = [replacement] if replacement else []
        refs = any(isinstance(p, int) for p in replacement)
        idx = self._add(fe.compile_ast(pattern, flags, "sub", groups=refs), N.CF_PAT_ORDERED)
        if refs:
            lit, parts = fe.encode_template(replacement)
            pa = np.asarray(parts, dtype=np.uint32)
            self._check_b(self.lib.cf_builder_set_template(self.b, idx, lit, len(lit), pa.ctypes.data, len(pa) // 3), "set_template")
        else:
            r = encode_unit("".join(replacement))
            self._check_b(self.lib.cf_builder_set_replacement(self.b, idx, r, len(r)), "set_replacement")
        self.n_ordered += 1
        return idx

    def compile_host(self) -> N.CompileStats:
        st = N.CompileStats()
        self._check_b(self.lib.cf_builder_compile_host(self.b, byref(st)), "compile")
        return st

    def compile(self, ctx: Context) -> "Program":
        self.compile_host()
        h = c_void_p()
        with ctx.lock:
            ctx.check(self.lib.cf_compile(ctx.h, self.b, byref(h)), "cf_compile")
        self.h, self.ctx = h, ctx
        return self

    @property
    def words(self) -> int:
        return (self.n_patterns + 63) // 64 or 1

    def __del__(self):
        try:
            if self.h:
                self.lib.cf_free_prog(self.h)
            self.lib.cf_builder_free(self.b)
        except Exception:
            pass


class PinnedBuffer:
    """Page-locked host memory (cf_host_alloc) as a numpy uint8 array: the D2H of the produced texts runs at the PCIe rate
    instead of through the driver's bounce buffer."""

    def __init__(self, ctx: Context, nbytes: int):
        self.ctx = ctx
        self.p = c_void_p()
        self.nbytes = nbytes
        with ctx.lock:
            ctx.check(ctx.lib.cf_host_alloc(ctx.h, nbytes, byref(self.p)), "cf_host_alloc")

    @property
    def array(self) -> np.ndarray:
        """A view of the buffer that keeps the buffer alive: texts sliced from it stay readable after the Batch that held it is gone
        or has grown a bigger one."""
        view = (ctypes.c_uint8 * self.nbytes).from_address(self.p.value)
        view.owner = self
        return np.frombuffer(view, dtype=np.uint8)

    def __del__(self):
        try:
            self.ctx.lib.cf_host_free(self.ctx.h, self.p)
        except Exception:
            pass


class Batch:
    """Device-resident packed stream (grown on demand by the caller creating a bigger one)."""

    def __init__(self, ctx: Context, max_bytes: int, max_units: int):
        self.ctx = ctx
        self.h = c_void_p()
        with ctx.lock:
            ctx.check(ctx.lib.cf_batch_create(ctx.h, max_bytes, max_units, byref(self.h)), "cf_batch_create")
        self.max_bytes, self.max_units = max_bytes, max_units

    def upload(self, stream, offsets: np.ndarray, cuda_stream: int = 0) -> None:
        n = len(offsets) - 1
        sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
        nbytes = int(offsets[-1])
        with self.ctx.lock:
            self.ctx.check(self.ctx.lib.cf_batch_upload(self.ctx.h, self.h, sp, nbytes, offsets.ctypes.data, n, cuda_stream), "cf_batch_upload")

    def pack_device(self, src, offsets, n: Optional[int] = None, stream=0, src_bytes: Optional[int] = None) -> None:
        """cf_batch_pack_device: fill the batch from texts already in device memory, unit i = src[offsets[i] .. offsets[i+1]), with
        the result cf_batch_upload of the same units would give.  A Run's `out` / `out_offsets` can be packed as they are, with
        src_bytes=run.gathered_bytes.

        src: a contiguous CUDA uint8 tensor or a raw device pointer.  offsets: a CUDA int64 tensor of at least n + 1 entries (n
        defaults to its length - 1), or a raw device pointer with `n` given.  `stream`: a torch.cuda.Stream or a raw cudaStream_t.
        src_bytes = offsets[n] - offsets[0].  Given, it is taken as it is and the call only enqueues (it may be captured in a CUDA
        graph).  When None it is read from the device: the device is synchronised and offsets[0] and offsets[n] are copied back,
        so that form is neither asynchronous nor capturable.  The source must stay untouched until the work on `stream` has run."""
        if isinstance(offsets, int):
            if n is None:
                raise ValueError("offsets given as a raw pointer: pass n")
        else:
            import torch

            if offsets.dtype != torch.int64:
                raise ValueError(f"offsets must be an int64 tensor, not {offsets.dtype}")
            if n is None:
                n = offsets.numel() - 1
            if offsets.numel() < n + 1:
                raise ValueError(f"offsets holds {offsets.numel()} entries; {n} units need {n + 1}")
        if not isinstance(src, int):
            import torch

            if src.dtype != torch.uint8:
                raise ValueError(f"src must be a uint8 tensor, not {src.dtype}")
        po, ps = _dev_ptr(offsets), _dev_ptr(src)
        if src_bytes is None and n > 0:
            import torch

            torch.cuda.synchronize()
            ends = np.zeros(2, dtype=np.uint64)
            with self.ctx.lock:
                self.ctx.check(self.ctx.lib.cf_copy_to_host(self.ctx.h, ends.ctypes.data, po, 8), "cf_copy_to_host")
                self.ctx.check(self.ctx.lib.cf_copy_to_host(self.ctx.h, ends.ctypes.data + 8, po + 8 * n, 8), "cf_copy_to_host")
            src_bytes = int(ends[1]) - int(ends[0])
            if not isinstance(src, int) and src.numel() < int(ends[1]):
                raise ValueError(f"src holds {src.numel()} bytes; offsets[{n}] = {int(ends[1])}")
        elif src_bytes is not None and not isinstance(src, int) and src.numel() < src_bytes:
            raise ValueError(f"src holds {src.numel()} bytes; src_bytes = {src_bytes}")
        st = getattr(stream, "cuda_stream", stream)
        with self.ctx.lock:
            self.ctx.check(self.ctx.lib.cf_batch_pack_device(self.ctx.h, self.h, ps, po, n, src_bytes or 0, st or None), "cf_batch_pack_device")

    def __del__(self):
        try:
            self.ctx.lib.cf_batch_free(self.h)
        except Exception:
            pass


def bitmaps_to_ints(bm: np.ndarray, n: int, W: int) -> List[int]:
    if W == 1:
        return [int(x) for x in bm[:n]]
    out = []
    for i in range(n):
        v = 0
        for w in range(W):
            v |= int(bm[i * W + w]) << (64 * w)
        out.append(v)
    return out


def scan_host(prog: Program, batch: Batch, stream, offsets: np.ndarray) -> np.ndarray:
    """End-to-end scan through the C ABI with host buffers (H2D + kernels + D2H, synchronous).
    Returns a uint64 array of n_units * W bitmap words."""
    ctx = batch.ctx
    n = len(offsets) - 1
    W = prog.words
    out = np.empty(n * W, dtype=np.uint64)
    sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
    with ctx.lock:
        ctx.check(ctx.lib.cf_scan_host(ctx.h, prog.h, batch.h, sp, int(offsets[-1]), offsets.ctypes.data, n, out.ctypes.data), "cf_scan_host")
    return out


def scan_units(prog: Program, units: Sequence[Union[str, bytes]], ctx: Optional[Context] = None) -> List[int]:
    """Convenience: pack, scan on the GPU, return one Python int bitmap per unit."""
    ctx = ctx or prog.ctx or Context.get()
    if prog.h is None:
        prog.compile(ctx)
    if not units:
        return []
    stream, offs = pack_units(units)
    batch = Batch(ctx, len(stream), len(units))
    bm = scan_host(prog, batch, stream, offs)
    return bitmaps_to_ints(bm, len(units), prog.words)


def sub_host(prog: Program, batch: Batch, unit_indices: Sequence[int]) -> List[bytes]:
    """Apply the program's substitution rules (in order) to the listed units of the batch that was
    last uploaded/scanned.  Returns the rewritten bytes of each listed unit (cf_sub_host)."""
    ctx = batch.ctx
    n = len(unit_indices)
    if n == 0:
        return []
    sel = np.asarray(unit_indices, dtype=np.uint32)
    offs = np.zeros(n + 1, dtype=np.uint64)
    need = c_uint64(0)
    cap = 1 << 16
    while True:
        out = np.empty(cap, dtype=np.uint8)
        with ctx.lock:
            rc = ctx.lib.cf_sub_host(ctx.h, prog.h, batch.h, sel.ctypes.data, n, out.ctypes.data, cap, offs.ctypes.data, byref(need))
        if rc == N.CF_E_CAPACITY and need.value > cap:
            cap = int(need.value)
            continue
        ctx.check(rc, "cf_sub_host")
        break
    raw = out.tobytes()
    return [raw[int(offs[i]):int(offs[i + 1])] for i in range(n)]


TOON_CONVERTED, TOON_NOT_SMALLER, TOON_NOT_JSON, TOON_VALUE_ERROR, TOON_ATTR_ERROR, TOON_UNSUPPORTED, TOON_SKIPPED = 0, 1, 2, 3, 4, 6, 8

VERDICT_DTYPE = np.dtype([("match_bitmap", "<u8"), ("flags", "<u4"), ("out_len", "<u4"), ("aux", "<i4"), ("reserved", "<u4")])   # cf_verdict, 24 bytes


def run_batch(prog: Optional[Program], batch: Batch, stream, offsets: np.ndarray, stage_mask: int, unit_stages: Optional[np.ndarray] = None,
              toon_flags: int = 0, mask_max_depth: int = 10, want_full_bitmaps: bool = False, outputs_resident: bool = False):
    """cf_run_batch: ONE upload of the packed stream, every requested stage on the resident batch, verdicts + only the produced
    texts back.  Returns (verdicts[VERDICT_DTYPE], out uint8[], out_offsets uint64[n+1], full bitmaps or None).
    `outputs_resident`: the produced texts stay in HBM (CF_RUN_OUTPUTS_RESIDENT; `out` is None, fetch with device_output())."""
    ctx = batch.ctx
    n = len(offsets) - 1
    nbytes = int(offsets[-1])
    verdicts = np.zeros(n, dtype=VERDICT_DTYPE)
    out_offs = np.zeros(n + 1, dtype=np.uint64)
    W = prog.words if prog is not None else 1
    full = np.zeros(n * W, dtype=np.uint64) if want_full_bitmaps else None
    need = c_uint64(0)
    if outputs_resident:
        sp = None if stream is None else (stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p))
        us = np.ascontiguousarray(unit_stages, dtype=np.uint8) if unit_stages is not None else None
        with ctx.lock:
            rc = ctx.lib.cf_run_batch(ctx.h, prog.h if prog is not None else None, batch.h, sp, nbytes, offsets.ctypes.data, n, stage_mask,
                                      us.ctypes.data if us is not None else None, toon_flags | N.CF_RUN_OUTPUTS_RESIDENT, mask_max_depth, verdicts.ctypes.data,
                                      full.ctypes.data if full is not None else None, None, 0, out_offs.ctypes.data, byref(need))
        ctx.check(rc, "cf_run_batch")
        return verdicts, None, out_offs, full
    # the output buffer lives with the Batch, is page-locked and only grows.  NOTE: the returned `out` is a view of it — it is
    # overwritten by the next run_batch on this Batch (callers slice/copy what they keep).
    pin = getattr(batch, "_out_pin", None)
    cap = max(nbytes, 1 << 12) if pin is None else pin.nbytes
    if pin is None:
        pin = batch._out_pin = PinnedBuffer(ctx, cap)
    out = pin.array
    if stream is None:                                   # resident run: the batch already holds these units
        sp = None
    else:
        sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
    us = None
    if unit_stages is not None:
        us = np.ascontiguousarray(unit_stages, dtype=np.uint8)
    while True:
        if len(out) < cap:
            batch._out_pin = None                          # free before growing
            pin = batch._out_pin = PinnedBuffer(ctx, cap + cap // 4)
            out = pin.array
            cap = len(out)
        with ctx.lock:
            rc = ctx.lib.cf_run_batch(ctx.h, prog.h if prog is not None else None, batch.h, sp, nbytes, offsets.ctypes.data, n, stage_mask,
                                      us.ctypes.data if us is not None else None, toon_flags, mask_max_depth, verdicts.ctypes.data,
                                      full.ctypes.data if full is not None else None, out.ctypes.data, cap, out_offs.ctypes.data, byref(need))
        if rc == N.CF_E_CAPACITY and need.value > cap:
            cap = int(need.value)
            continue
        ctx.check(rc, "cf_run_batch")
        break
    return verdicts, out, out_offs, full


def _dev_ptr(x) -> Optional[int]:
    """Device address of a CUDA torch tensor, or a raw device pointer (int), or None."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if not x.is_cuda or not x.is_contiguous():
        raise ValueError("cf_run buffers must be contiguous CUDA tensors or raw device pointers")
    return x.data_ptr()


class Run:
    """cf_run: the fused chain (scan, regex_filter rewriting, TOON or masking) enqueued on the caller's CUDA stream, with verdicts, offsets and
    texts left in device memory.  `enqueue` returns as soon as the work is queued (it may be captured in a CUDA graph); `finish`
    waits for it.  Each Run holds its own device state, so several can be in flight on different streams.

        run = Run(ctx, max_units, max_bytes)
        batch.upload(stream, offsets, cuda_stream=s)              # on the same stream
        run.enqueue(prog, batch, STAGES, None, 0, verdicts, out_offsets, out, bitmaps_full, stream=s)
        needed = run.finish()                                     # 0, or the capacity `out` needs; CfError on failure

    After a finish that returned 0, `gathered_bytes` is the byte count of the texts in `out` (out_offsets[n]): what
    Batch.pack_device needs to feed them to another run on the device, e.g. to TOON-encode the units flagged CF_V_RESUBMIT.
    """

    def __init__(self, ctx: Context, max_units: int, max_bytes: int, sub_arena_bytes: int = 1 << 20):
        self.ctx = ctx
        self.h = c_void_p()
        with ctx.lock:
            ctx.check(ctx.lib.cf_run_create(ctx.h, max_units, max_bytes, sub_arena_bytes, byref(self.h)), "cf_run_create")
        self._keep = ()
        self.gathered_bytes: Optional[int] = None   # out_offsets[n] of the last finish() that gathered every text into `out`

    def enqueue(self, prog: Optional[Program], batch: Batch, stage_mask: int, d_unit_stages, toon_flags: int, verdicts, out_offsets, out,
                bitmaps_full=None, stream=0, mask_max_depth: int = 10) -> None:
        """verdicts: n * 24 bytes (e.g. a uint8 / int64 tensor), out_offsets: n + 1 uint64, out: the texts' buffer (its byte size is
        the capacity), bitmaps_full: n * W uint64 (allocated here when None and SCAN / SUB run).  Tensor sizes are checked against
        the batch (ValueError); raw device pointers are taken as they are.  `stream`: a torch.cuda.Stream or a raw
        cudaStream_t.  The buffers must stay alive and untouched until finish().
        With CF_STAGE_MASK the bodies are masked at `mask_max_depth`; the first masking enqueue of a Run allocates its masking
        workspace, so it must not be the one captured in a CUDA graph (warm the Run up with one enqueue + finish first)."""
        n = int(self.ctx.lib.cf_batch_units(batch.h))
        scan = bool(stage_mask & (N.CF_STAGE_SCAN | N.CF_STAGE_SUB))
        if bitmaps_full is None and scan:
            import torch

            bitmaps_full = torch.empty(n * prog.words, dtype=torch.int64, device=verdicts.device if hasattr(verdicts, "device") else "cuda")
        if not hasattr(out, "numel"):
            raise ValueError("pass `out` as a CUDA tensor (its byte size is the capacity)")
        cap = out.numel() * out.element_size()
        # the kernels write n records, n + 1 offsets and n * W bitmap words: a short tensor would be written past its end
        for name, t, need in (("verdicts", verdicts, 24 * n), ("out_offsets", out_offsets, 8 * (n + 1)),
                              ("bitmaps_full", bitmaps_full if scan else None, 8 * n * (prog.words if prog is not None else 1)),
                              ("d_unit_stages", d_unit_stages, n)):
            if t is not None and not isinstance(t, int) and t.numel() * t.element_size() < need:
                raise ValueError(f"{name} holds {t.numel() * t.element_size()} bytes; this batch needs {need}")
        st = getattr(stream, "cuda_stream", stream)
        self._keep = (verdicts, out_offsets, out, bitmaps_full, d_unit_stages)
        with self.ctx.lock:
            if stage_mask & N.CF_STAGE_MASK:
                self.ctx.check(self.ctx.lib.cf_run_set_mask(self.ctx.h, self.h, mask_max_depth), "cf_run_set_mask")
            self.ctx.check(self.ctx.lib.cf_run_enqueue(self.ctx.h, prog.h if prog is not None else None, batch.h, self.h, stage_mask, _dev_ptr(d_unit_stages),
                                                       toon_flags, _dev_ptr(verdicts), _dev_ptr(bitmaps_full), _dev_ptr(out_offsets), _dev_ptr(out), cap,
                                                       st or None), "cf_run_enqueue")

    @property
    def bitmaps_full(self):
        """The bitmap buffer of the last enqueue (the one passed in, or the one allocated for it)."""
        return self._keep[3] if self._keep else None

    def finish(self) -> int:
        """Wait for the last enqueue (or a graph replay of it).  Returns 0 when every text was gathered into `out`, and the bytes
        `out` must hold when it was too small (CF_E_CAPACITY: verdicts and out_offsets are valid, `out` is untouched); raises
        CfError on any other failure."""
        need = c_uint64(0)
        self.gathered_bytes = None
        with self.ctx.lock:
            rc = self.ctx.lib.cf_run_finish(self.ctx.h, self.h, byref(need))
        if rc == N.CF_E_CAPACITY and need.value:
            return int(need.value)
        self.ctx.check(rc, "cf_run_finish")
        self.gathered_bytes = int(need.value)
        return 0

    def __del__(self):
        try:
            self.ctx.lib.cf_run_free(self.h)
        except Exception:
            pass


def device_output(ctx: Context) -> np.ndarray:
    """Host copy of the device buffer the last `run_batch(..., outputs_resident=True)` of this context left in HBM."""
    p = c_void_p()
    nb = c_uint64(0)
    with ctx.lock:
        ctx.check(ctx.lib.cf_run_batch_device_output(ctx.h, byref(p), byref(nb)), "cf_run_batch_device_output")
        out = np.empty(nb.value, dtype=np.uint8)
        if nb.value:
            ctx.check(ctx.lib.cf_copy_to_host(ctx.h, out.ctypes.data, p, nb.value), "cf_copy_to_host")
    return out


def toon_host(batch: Batch, stream, offsets: np.ndarray, report_errors: bool = True):
    """cf_toon_host: every unit is one JSON text.  Returns (status int32[n], toon texts as bytes or
    None per unit)."""
    ctx = batch.ctx
    n = len(offsets) - 1
    nbytes = int(offsets[-1])
    out = np.empty(max(nbytes, 1), dtype=np.uint8)
    out_len = np.empty(n, dtype=np.uint32)
    status = np.empty(n, dtype=np.int32)
    sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
    with ctx.lock:
        ctx.check(ctx.lib.cf_toon_host(ctx.h, batch.h, 1 if report_errors else 0, sp, nbytes, offsets.ctypes.data, n, out.ctypes.data, out_len.ctypes.data, status.ctypes.data), "cf_toon_host")
    texts: List[Optional[bytes]] = []
    for i in range(n):
        if status[i] == TOON_CONVERTED:
            o = int(offsets[i])
            texts.append(out[o:o + int(out_len[i])].tobytes())
        else:
            texts.append(None)
    return status, texts


def json_index_host(batch: Batch, stream, offsets: np.ndarray, classify: bool = False):
    """cf_json_index_host: structural index of every unit (one JSON text each).  Returns per unit
    (tokens uint32[k, 2] = (pos | close_quote << 31, aux), unterminated flag)."""
    ctx = batch.ctx
    n = len(offsets) - 1
    nbytes = int(offsets[-1])
    toks = np.zeros((max(nbytes, 1), 2), dtype=np.uint32)
    counts = np.zeros(max(n, 1), dtype=np.uint32)
    sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
    with ctx.lock:
        ctx.check(ctx.lib.cf_json_index_host(ctx.h, batch.h, 1 if classify else 0, sp, nbytes, offsets.ctypes.data, n, toks.ctypes.data, counts.ctypes.data), "cf_json_index_host")
    out = []
    for i in range(n):
        o = int(offsets[i])
        k = int(counts[i]) & 0x7FFFFFFF
        out.append((toks[o:o + k].copy(), bool(int(counts[i]) >> 31)))
    return out


MASK_OK, MASK_PARSE_ERROR, MASK_UNSUPPORTED = 0, 2, 6


def mask_host(batch: Batch, stream, offsets: np.ndarray, max_depth: int = 10):
    """cf_mask_host: every unit is one JSON request body.  Returns (status int32[n], masked bytes or None)."""
    ctx = batch.ctx
    n = len(offsets) - 1
    nbytes = int(offsets[-1])
    status = np.empty(n, dtype=np.int32)
    out_offs = np.zeros(n + 1, dtype=np.uint64)
    need = c_uint64(0)
    cap = nbytes + 4096
    sp = stream.ctypes.data if isinstance(stream, np.ndarray) else ctypes.cast(ctypes.c_char_p(stream), c_void_p)
    while True:
        out = np.empty(cap, dtype=np.uint8)
        with ctx.lock:
            rc = ctx.lib.cf_mask_host(ctx.h, batch.h, sp, nbytes, offsets.ctypes.data, n, max_depth, out.ctypes.data, cap, out_offs.ctypes.data, status.ctypes.data, byref(need))
        if rc == N.CF_E_CAPACITY and need.value > cap:
            cap = int(need.value)
            continue
        ctx.check(rc, "cf_mask_host")
        break
    raw = out.tobytes()
    return status, [raw[int(out_offs[i]):int(out_offs[i + 1])] if status[i] == MASK_OK else None for i in range(n)]


def classify_keys_host(batch: Batch, keys: Sequence[Union[str, bytes]]) -> List[bool]:
    """is_sensitive_key for each key name on the GPU."""
    if not keys:
        return []
    stream, offs = pack_units(keys)
    ctx = batch.ctx
    out = np.empty(len(keys), dtype=np.uint8)
    with ctx.lock:
        ctx.check(ctx.lib.cf_classify_keys_host(ctx.h, batch.h, ctypes.cast(ctypes.c_char_p(stream), c_void_p), len(stream), offs.ctypes.data, len(keys), out.ctypes.data), "cf_classify_keys_host")
    return [bool(x) for x in out]
