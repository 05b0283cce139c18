"""In-tree build of libcfgpu.so (nvcc, sm_90a only).  Used by __graft_entry__.build() and runnable
directly: `python -m mcp_context_forge_b200.build [--force] [-v]`.  nvcc cross-compiles without a GPU.

Every source becomes an object under csrc/_obj/ (git-ignored); objects are rebuilt only when the source or a
header they include changed, the sources compile in parallel, then one link step produces the .so."""
from __future__ import annotations

import concurrent.futures
import os
import re
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
SO = os.path.join(HERE, "libcfgpu.so")
INC = os.path.join(os.path.dirname(HERE), "include")
SOURCES = ["cfgpu.cu", "cfjson.cu", "cfjson_seq.cu", "cf_host.cpp", "re_backend.cpp"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libcfgpu.so cannot be built")


_INC_RE = re.compile(r'^\s*#\s*include\s+"([^"]+)"', re.M)


def _deps(path: str, seen=None) -> set:
    """The source plus every project header it includes (transitively)."""
    seen = seen if seen is not None else set()
    if path in seen or not os.path.exists(path):
        return seen
    seen.add(path)
    with open(path, encoding="utf-8", errors="replace") as f:
        text = f.read()
    for inc in _INC_RE.findall(text):
        for base in (os.path.dirname(path), CSRC, INC):
            cand = os.path.normpath(os.path.join(base, inc))
            if os.path.exists(cand):
                _deps(cand, seen)
                break
    return seen


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def needs_build() -> bool:
    if not os.path.exists(SO):
        return True
    for s in SOURCES:
        obj = os.path.join(OBJ, os.path.splitext(s)[0] + ".o")
        # the object against its sources (a source edited while an earlier build was running is newer than its object but older
        # than the library that build linked), and the library against the object
        if _stale(obj, _deps(os.path.join(CSRC, s))) or _stale(SO, [obj]):
            return True
    return False


def _compile(src: str, verbose: bool) -> str:
    obj = os.path.join(OBJ, os.path.splitext(src)[0] + ".o")
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-I", INC, "-c", os.path.join(CSRC, src), "-o", obj]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n" + proc.stdout + proc.stderr)
    return proc.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return SO
    os.makedirs(OBJ, exist_ok=True)
    todo = [s for s in SOURCES if force or _stale(os.path.join(OBJ, os.path.splitext(s)[0] + ".o"), _deps(os.path.join(CSRC, s)))]
    with concurrent.futures.ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        for log in ex.map(lambda s: _compile(s, verbose), todo):
            if verbose:
                sys.stderr.write(log)
    objs = [os.path.join(OBJ, os.path.splitext(s)[0] + ".o") for s in SOURCES]
    cmd = [_nvcc()] + ARCH + ["-shared", "-cudart", "static", "-o", SO] + objs
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("link failed:\n" + proc.stdout + proc.stderr)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
