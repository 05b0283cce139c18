# -*- coding: utf-8 -*-
"""GPU implementation of the `request_logging_masking_native_extension` module surface
(/root/reference/crates/request_logging_masking_native_extension/src/lib.rs:307-368, stub
python/request_logging_masking_native_extension/__init__.pyi:13-15):

    mask_sensitive_data(data, max_depth=None)        -> masked copy of dict / list trees
    mask_sensitive_headers(headers)                  -> masked copy of a header dict
    mask_sensitive_json_bytes(payload, max_depth=None) -> bytes (compact JSON, keys sorted)

plus the batch forms the serving path should use (`*_batch`), which put many request bodies into one
packed stream and one kernel launch.  The sensitive-key classifier, the masking walk and the
serde_json-compatible re-serialisation run on the GPU (csrc/json_mask.h).  Cookie splitting for the
`cookie` header is host logic (a handful of bytes per request), restating lib.rs:199-231.
Errors: whatever serde_json rejects (invalid JSON, lone surrogates, numbers out of binary64's range,
nesting deeper than 127 levels) raises ValueError like the crate (the middleware then takes its own
Python path, mcpgateway/middleware/request_logging_middleware.py:299-305); number literals longer than
the device's 3200-bit workspace raise RuntimeError — never a silent different answer.
"""
from __future__ import annotations

import threading
from typing import Any, Dict, List, Optional, Sequence

from . import engine
from .batching import GpuBatcher

MASKED_VALUE = "******"
NESTED_TOO_DEEP = "<nested too deep>"
_RUST_WHITE_SPACE = frozenset("\t\n\x0b\x0c\r \x85\xa0                　")


_own_batch: Optional[engine.Batch] = None
_own_lock = threading.RLock()


def _batch(nbytes: int, nunits: int) -> engine.Batch:
    """The masker's OWN device batch (the plugins' GpuBatcher has its own): a logging middleware thread and the hook chain's event
    loop never overwrite each other's upload.  Callers hold `_own_lock` for the upload + launch + download of one call."""
    global _own_batch
    b = _own_batch
    if b is None or nbytes > b.max_bytes or nunits > b.max_units:
        _own_batch = b = engine.Batch(GpuBatcher.get().ctx, max(nbytes * 2, 1 << 20, b.max_bytes if b else 0), max(nunits * 2, 1024, b.max_units if b else 0))
    return b


def mask_sensitive_json_bytes_batch(payloads: Sequence[bytes], max_depth: Optional[int] = None) -> List[Optional[bytes]]:
    """Masked bytes per payload; None where the crate would raise ValueError (invalid JSON, a number out of binary64's range,
    nesting deeper than 127 levels)."""
    if not payloads:
        return []
    depth = 10 if max_depth is None else int(max_depth)
    stream, offs = engine.pack_units(list(payloads))
    with _own_lock:
        status, outs = engine.mask_host(_batch(len(stream), len(payloads)), stream, offs, depth)
    res: List[Optional[bytes]] = []
    for st, o in zip(status, outs):
        if st == engine.MASK_OK:
            res.append(o)
        elif st == engine.MASK_PARSE_ERROR:
            res.append(None)
        else:
            raise RuntimeError("request_logging_masking(GPU): payload exceeds the device limits (a number literal longer than the 3200-bit "
                               "workspace, or a body over 768 MiB)")
    return res


def mask_sensitive_json_bytes(payload: bytes, max_depth: Optional[int] = None) -> bytes:
    out = mask_sensitive_json_bytes_batch([bytes(payload)], max_depth)[0]
    if out is None:
        raise ValueError("invalid JSON payload")
    return out


def _rust_trim(s: str) -> str:
    a, b = 0, len(s)
    while a < b and s[a] in _RUST_WHITE_SPACE:
        a += 1
    while b > a and s[b - 1] in _RUST_WHITE_SPACE:
        b -= 1
    return s[a:b]


def _mask_cookie_header(cookie_header: str) -> str:
    """lib.rs:199-231."""
    parts = []
    for cookie in cookie_header.split(";"):
        trimmed = _rust_trim(cookie)
        if "=" in trimmed:
            name = _rust_trim(trimmed.split("=", 1)[0])
            low = "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in name)
            if "jwt" in low or "token" in low or "auth" in low or "session" in low:
                parts.append(f"{name}={MASKED_VALUE}")
                continue
        parts.append(trimmed)
    return "; ".join(parts)


def _collect_keys(data: Any, depth: int, keys: Dict[str, bool]) -> None:
    if depth <= 0:
        return
    if isinstance(data, dict):
        for k, v in data.items():
            keys.setdefault(str(k), False)
            _collect_keys(v, depth - 1, keys)
    elif isinstance(data, list):
        for v in data:
            _collect_keys(v, depth - 1, keys)


def _classify(keys: Dict[str, bool]) -> None:
    names = list(keys)
    if not names:
        return
    enc = [n.encode("utf-8", "surrogatepass") for n in names]
    nbytes = sum(len(e) + 1 for e in enc)
    with _own_lock:
        flags = engine.classify_keys_host(_batch(nbytes, len(enc)), enc)
    for n, s in zip(names, flags):
        keys[n] = s


def _apply(data: Any, depth: int, keys: Dict[str, bool]) -> Any:
    if depth <= 0:
        return NESTED_TOO_DEEP
    if isinstance(data, dict):
        return {k: (MASKED_VALUE if keys[str(k)] else _apply(v, depth - 1, keys)) for k, v in data.items()}
    if isinstance(data, list):
        return [_apply(v, depth - 1, keys) for v in data]
    return data


def mask_sensitive_data(data: Any, max_depth: Optional[int] = None) -> Any:
    """lib.rs:307-316 / :233-274 — every key name of the tree is classified on the GPU in one launch."""
    depth = 10 if max_depth is None else int(max_depth)
    keys: Dict[str, bool] = {}
    _collect_keys(data, depth, keys)
    _classify(keys)
    return _apply(data, depth, keys)


def mask_sensitive_headers(headers: Any) -> Dict[Any, Any]:
    """lib.rs:318-344."""
    if not isinstance(headers, dict):
        raise TypeError("headers must be a dict")
    keys = {str(k): False for k in headers}
    _classify(keys)
    out = {}
    for k, v in headers.items():
        ks = str(k)
        if keys[ks]:
            out[k] = MASKED_VALUE
        elif ks.lower() == "cookie" and ks.isascii() and isinstance(v, str):
            out[k] = _mask_cookie_header(v)
        elif "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in ks) == "cookie" and isinstance(v, str):
            out[k] = _mask_cookie_header(v)
        else:
            out[k] = v
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# RequestLoggingMiddleware remainder (SURVEY.md §8(f)-4)
# ---------------------------------------------------------------------------------------------------------------------------
# /root/reference/mcpgateway/middleware/request_logging_middleware.py:83-99
SENSITIVE_KEYS = ("password", "passphrase", "secret", "token", "api_key", "apikey", "access_token", "refresh_token", "client_secret", "authorization",
                  "auth_token", "jwt_token", "private_key")
NON_JSON_MASKED = "<contains sensitive data - masked>"
_fallback_prog: Optional[engine.Program] = None


def _probe_pattern(key: str) -> str:
    """`key in text.lower()` as a pattern over the ORIGINAL text: every letter matches itself, its capital and whatever other
    code point `str.lower()` maps to exactly that letter (only U+212A KELVIN SIGN -> 'k'; U+0130 lowers to TWO code points and
    therefore never produces a bare 'i')."""
    out = []
    for c in key:
        if c.isalpha():
            out.append("[" + c + c.upper() + ("\u212a" if c == "k" else "") + "]")
        else:
            out.append("\\" + c if not c.isalnum() and c != "_" else c)
    return "".join(out)


def non_json_fallback_batch(payloads: Sequence[bytes]) -> List[str]:
    """The middleware's non-JSON branch (request_logging_middleware.py:661-667) for many request bodies at once:
    `s = body.decode("utf-8", errors="ignore")`; if any of the 13 SENSITIVE_KEYS occurs in `s.lower()` the body is logged as
    "<contains sensitive data - masked>", else as `s`.  The 13 probes are ONE fused scan over the packed bodies."""
    global _fallback_prog
    if not payloads:
        return []
    texts = [bytes(p).decode("utf-8", errors="ignore") for p in payloads]
    if _fallback_prog is None:
        prog = engine.Program()
        for k in SENSITIVE_KEYS:
            prog.add_search(_probe_pattern(k), 0)
        _fallback_prog = prog
    hits = GpuBatcher.get().scan_groups(_fallback_prog, [texts])[0]
    return [NON_JSON_MASKED if h else t for h, t in zip(hits, texts)]


def mask_sensitive_headers_batch(headers_list: Sequence[Any]) -> List[Dict[Any, Any]]:
    """`mask_sensitive_headers` (lib.rs:318-344) for the header dicts of many requests: every distinct header name of the
    wave is classified in ONE launch."""
    for h in headers_list:
        if not isinstance(h, dict):
            raise TypeError("headers must be a dict")
    keys: Dict[str, bool] = {}
    for h in headers_list:
        for k in h:
            keys.setdefault(str(k), False)
    _classify(keys)
    out = []
    for h in headers_list:
        m = {}
        for k, v in h.items():
            ks = str(k)
            if keys[ks]:
                m[k] = MASKED_VALUE
            elif "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in ks) == "cookie" and isinstance(v, str):
                m[k] = _mask_cookie_header(v)
            else:
                m[k] = v
        out.append(m)
    return out
