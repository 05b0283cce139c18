"""Oracle restatement of the reference TOON encoder and of the plugin's per-item decision.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Written independently of the reference's code
structure: the reference builds child strings and re-prefixes them line by line
(plugins/toon_encoder/toon.py:559-560, 421-422, 432-433); here every function appends finished lines
with an explicit "outer prefix" `pre`, which is also how the CUDA emitter works.  Same outputs,
including the quirks the reference's behaviour pins (SURVEY.md Appendix A-5/A-6):

  encode                      toon.py:82-132      float formatting           toon.py:135-160
  string quoting rules        toon.py:163-222     quoting / escapes          toon.py:249-283
  key encoding                toon.py:286-309     arrays                     toon.py:312-375
  objects as list items       toon.py:378-441     columnar                   toon.py:456-511
  objects                     toon.py:514-565     plugin item decision       toon_encoder.py:237-326

Pinned by tests/golden/toon.json (recorded from the reference's own toon.py / toon_encoder.py, inputs
harvested from the reference's tests/unit/plugins/toon_encoder/*.py plus fuzz).
"""
from __future__ import annotations

import json
import re
from typing import Any, List, Optional, Tuple

_SPECIAL = set('\n\r\t,:[]{}"\\-')
_NUM = re.compile(r"^-?(?:0|[1-9]\d*)(?:\.\d+)?(?:[eE][+-]?\d+)?$")     # toon.py:54 (Unicode \d, `$` quirk)
_LEAD0 = re.compile(r"^0\d+$")                                           # toon.py:57
_KEY = re.compile(r"^[A-Za-z_][A-Za-z0-9_.]*$")                          # toon.py:71 (`$` admits a final "\n")
_RESERVED = ("null", "true", "false")


class ToonCrash(Exception):
    """The reference raises AttributeError here (toon.py:400-404 calling :479-497 on non-dicts)."""


def fmt_float(x: float) -> str:
    if x != x or x in (float("inf"), float("-inf")):
        return "null"
    if x == 0.0:
        return "0"
    if x.is_integer():
        return str(int(x))
    s = "%.15g" % x
    if "e" in s:
        s = ("%.15f" % x).rstrip("0").rstrip(".")
    return s


def needs_quotes(s: str) -> bool:
    if s == "" or s in _RESERVED:
        return True
    if any(c in _SPECIAL for c in s):
        return True
    if _NUM.match(s) or _LEAD0.match(s):
        return True
    if s[0].isspace() or s[-1].isspace():
        return True
    return any(ord(c) < 32 for c in s)


def quote(s: str) -> str:
    out = ['"']
    for c in s:
        if c == "\\":
            out.append("\\\\")
        elif c == '"':
            out.append('\\"')
        elif c == "\n":
            out.append("\\n")
        elif c == "\r":
            out.append("\\r")
        elif c == "\t":
            out.append("\\t")
        elif ord(c) < 32:
            raise ValueError("control character")
        else:
            out.append(c)
    out.append('"')
    return "".join(out)


def enc_str(s: str) -> str:
    return quote(s) if needs_quotes(s) else s


def enc_key(k: str) -> str:
    if k and _KEY.match(k) and k not in _RESERVED:
        return k
    return quote(k)


def simple(v: Any) -> bool:
    return v is None or isinstance(v, (bool, int, float, str))


def enc_prim(v: Any) -> str:
    if v is None:
        return "null"
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, float):
        return fmt_float(v)
    if isinstance(v, str):
        return enc_str(v)
    raise TypeError(type(v).__name__)


def columnar(arr: list) -> Optional[Tuple[str, List[str]]]:
    """(header without prefix, rows without indentation) or None.  Raises ToonCrash where the
    reference's unchecked `.keys()` would raise AttributeError."""
    if not arr:
        return None
    if not isinstance(arr[0], dict):
        raise ToonCrash()
    keys = list(arr[0].keys())
    if not keys:
        return None
    ks = set(keys)
    for o in arr[1:]:
        if not isinstance(o, dict):
            raise ToonCrash()
        if set(o.keys()) != ks:
            return None
    for o in arr:
        if not all(simple(v) for v in o.values()):
            return None
    header = "[%d]{%s}:" % (len(arr), ",".join(keys))          # keys are NOT quoted here (toon.py:501)
    return header, [",".join(enc_prim(o[k]) for k in keys) for o in arr]


def _nl(text: str, pre: str) -> str:
    """A key the reference emits unquoted may contain a raw newline (its `$` admits one final "\\n", toon.py:299-306; columnar header
    fields are never quoted, :501).  The reference builds nested text as strings and re-splits them on "\\n" at every enclosing level
    (:369, :421, :432, :559), so what follows such a newline is a line of its own and receives the prefixes of the ENCLOSING levels —
    `pre` here — but not the indentation the emitting level wrote in front of the key itself."""
    return text.replace("\n", "\n" + pre) if "\n" in text else text


def emit_array(out: List[str], arr: list, pre: str, indent: int, prefix: str, first_prefix: Optional[str] = None) -> None:
    """Lines of one array.  `pre` = spaces contributed by enclosing blocks; `indent` = the
    reference's indent argument (absolute!), `first_prefix` overrides `pre` for the first line
    (used when the array starts on a hyphen line)."""
    p0 = pre if first_prefix is None else first_prefix
    if not arr:
        out.append(f"{p0}{prefix}[0]:")
        return
    if all(isinstance(x, dict) for x in arr):
        col = columnar(arr)
        if col is not None:
            out.append(f"{p0}{prefix}{_nl(col[0], pre)}")
            out.extend(f"{pre}  {r}" for r in col[1])
            return
    if all(simple(x) for x in arr):
        out.append(f"{p0}{prefix}[{len(arr)}]: " + ",".join(enc_prim(x) for x in arr))
        return
    out.append(f"{p0}{prefix}[{len(arr)}]:")
    ci = " " * (2 * (indent + 1))
    for x in arr:
        if simple(x):
            out.append(f"{pre}{ci}- {enc_prim(x)}")
        elif isinstance(x, dict):
            if not x:
                out.append(f"{pre}{ci}-")
            else:
                emit_list_item(out, x, pre, indent + 1)
        else:
            emit_array(out, x, f"{pre}{ci}  ", indent + 2, "", first_prefix=f"{pre}{ci}- ")


def emit_list_item(out: List[str], obj: dict, pre: str, indent: int) -> None:
    ind = " " * (2 * indent)
    fi = " " * (2 * (indent + 1))
    for i, (k, v) in enumerate(obj.items()):
        ek = _nl(enc_key(k), pre)
        lead = f"{pre}{ind}- " if i == 0 else f"{pre}{fi}"
        if isinstance(v, list) and v:
            if i == 0:
                col = columnar(v)
                if col is not None:
                    # toon.py:405-413: the columnar text is split on "\n"; line 0 is "the header", every other line — the rest of a
                    # header with a raw newline included — is "a row": stripped and indented like one
                    hdr = col[0].split("\n")
                    out.append(f"{lead}{ek}{hdr[0]}")
                    out.extend(f"{pre}{fi}  {r.strip()}" for r in hdr[1:] + col[1])
                    continue
            out.append(f"{lead}{ek}:")
            emit_array(out, v, f"{pre}{fi}  ", indent + 2, "")
        elif isinstance(v, dict) and v:
            out.append(f"{lead}{ek}:")
            emit_object(out, v, f"{pre}{fi}  ", indent + 2)
        else:
            ev = "[0]:" if isinstance(v, list) else "" if isinstance(v, dict) else enc_prim(v)
            out.append(f"{lead}{ek}: {ev}")


def emit_object(out: List[str], obj: dict, pre: str, indent: int) -> None:
    for k, v in obj.items():
        ek = _nl(enc_key(k), pre)
        if isinstance(v, list):
            emit_array(out, v, pre, indent, ek)
        elif isinstance(v, dict):
            out.append(f"{pre}{ek}:")
            if v:
                emit_object(out, v, pre + "  ", indent + 1)
        else:
            out.append(f"{pre}{ek}: {enc_prim(v)}")


def encode(obj: Any) -> str:
    """toon.encode(obj); raises ValueError / ToonCrash where the reference raises."""
    if simple(obj):
        return enc_prim(obj)
    out: List[str] = []
    if isinstance(obj, (list, tuple)):
        emit_array(out, list(obj), "", 0, "")
    elif isinstance(obj, dict):
        if not obj:
            return ""
        emit_object(out, obj, "", 0)
    else:
        raise TypeError(type(obj).__name__)
    return "\n".join(out)


def loads_strict(text: str) -> Any:
    """JSON parse with orjson-like strictness (no NaN/Infinity literals).  orjson 3.11.8 is the
    reference's parser (toon_encoder.py:281); differences to stdlib json that matter (ints beyond
    64 bits, lone surrogates) are avoided in test inputs."""
    def bad(c):
        raise ValueError(c)

    def parse_int(t):
        # orjson (yyjson) returns Python ints only inside [-2**63, 2**64-1]; larger integer literals
        # come back as floats (SURVEY.md Appendix A-7; orjson itself is not installable here, so this
        # rule is restated, not observed); one beyond binary64 is rejected like a float literal that overflows
        v = int(t)
        return v if -(2 ** 63) <= v <= 2 ** 64 - 1 else parse_float(t)

    def parse_float(t):
        v = float(t)
        if v in (float("inf"), float("-inf")):
            raise ValueError("number out of range")   # yyjson rejects literals that overflow binary64
        return v
    return json.loads(text, parse_constant=bad, parse_int=parse_int, parse_float=parse_float)


def process_text(text: str, min_size: int = 100, max_size: int = 1024 * 1024, skip_on_error: bool = True) -> Optional[str]:
    """The decision of `_process_content_item` for one text (toon_encoder.py:257-303): the TOON text
    when the item is converted, else None."""
    n = len(text.encode("utf-8"))
    if n < min_size or n > max_size:
        return None
    try:
        parsed = loads_strict(text)
    except (ValueError, TypeError):
        return None
    try:
        toon = encode(parsed)
    except Exception:
        if skip_on_error:
            return None
        raise
    return toon if len(toon.encode("utf-8")) < n else None
