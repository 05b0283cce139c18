"""Oracle restatement of the Rust request_logging_masking crate
(/root/reference/crates/request_logging_masking_native_extension/src/lib.rs) — TEST INFRASTRUCTURE ONLY.

  normalize_key_for_masking   lib.rs:79-111       has_non_sensitive_suffix   lib.rs:113-120
  is_sensitive_key            lib.rs:122-187      mask_cookie_header         lib.rs:199-231
  mask_sensitive_data_inner   lib.rs:233-274      mask_json_value_inner      lib.rs:276-305
  mask_sensitive_json_bytes   lib.rs:346-360

The crate cannot be compiled here (no cargo/rustc), so the oracle is pinned by (a) the crate's own unit
tests lib.rs:380-425, (b) vectors recorded from the Python twin the reference ships for the same
algorithm (mcpgateway/middleware/request_logging_middleware.py:125-291 -> tests/golden/masking_twin.json).
The byte format of `mask_sensitive_json_bytes` comes from serde_json 1.0.149 (not vendored): compact,
BTreeMap key order (bytewise), duplicate keys last-wins, i64/u64 integers verbatim, every other number as
the shortest round-trip binary64 in ryu's layout, strings re-escaped.  The reference's own tests mock this
function, so that format is "parity unpinned" (SURVEY.md §8c) and restated from serde_json's documented
behaviour.
"""
from __future__ import annotations

import json
from decimal import Decimal
from typing import Any, List

MASKED = "******"
TOO_DEEP = "<nested too deep>"
SUFFIXES = ("_count", "_counts", "_size", "_length", "_ttl", "_seconds", "_ms", "_id", "_ids", "_name", "_type", "_url", "_uri", "_path", "_status", "_code")
EXACT = {"password", "passphrase", "secret", "token", "api_key", "apikey", "access_token", "refresh_token", "client_secret", "authorization", "auth_token", "jwt_token", "private_key"}
AUTH_TOKENS = {"auth", "authorization", "jwt"}
WORD_TOKENS = {"password", "passphrase", "secret", "token", "apikey", "authorization"}
BIGRAMS = {("api", "key"), ("access", "token"), ("refresh", "token"), ("client", "secret"), ("auth", "token"), ("jwt", "token"), ("private", "key")}


def normalize_key(key: str) -> str:
    out: List[str] = []
    prev_lower_or_digit = False
    prev_underscore = False
    for ch in key:
        is_upper = "A" <= ch <= "Z"
        is_alnum = is_upper or "a" <= ch <= "z" or "0" <= ch <= "9"
        if is_upper and prev_lower_or_digit and not prev_underscore:
            out.append("_")
        if is_alnum:
            out.append(ch.lower() if is_upper else ch)
            prev_underscore = False
        elif not prev_underscore and out:
            out.append("_")
            prev_underscore = True
        prev_lower_or_digit = "a" <= ch <= "z" or "0" <= ch <= "9"
        if is_upper:
            prev_underscore = False
    s = "".join(out)
    return s.rstrip("_")


def is_sensitive_key(key: str) -> bool:
    n = normalize_key(key)
    if not n:
        return False
    has_suffix = any(n.endswith(s) for s in SUFFIXES)
    if n in EXACT:
        return True
    toks = n.split("_")
    if not has_suffix and any(t in AUTH_TOKENS for t in toks):
        return True
    if has_suffix:
        return False
    prev = ""
    for t in (t for t in toks if t):
        if t in WORD_TOKENS or (prev, t) in BIGRAMS:
            return True
        prev = t
    return False


_RUST_WS = set("\t\n\x0b\x0c\r \x85\xa0                　")


def _rust_trim(s: str) -> str:
    a, b = 0, len(s)
    while a < b and s[a] in _RUST_WS:
        a += 1
    while b > a and s[b - 1] in _RUST_WS:
        b -= 1
    return s[a:b]


def _ascii_lower(s: str) -> str:
    return "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in s)


def mask_cookie_header(cookie_header: str) -> str:
    parts = []
    for cookie in cookie_header.split(";"):
        trimmed = _rust_trim(cookie)
        if "=" in trimmed:
            name = _rust_trim(trimmed.split("=", 1)[0])
            low = _ascii_lower(name)
            if "jwt" in low or "token" in low or "auth" in low or "session" in low:
                parts.append(f"{name}={MASKED}")
                continue
        parts.append(trimmed)
    return "; ".join(parts)


def mask_value(data: Any, max_depth: int = 10) -> Any:
    if max_depth <= 0:
        return TOO_DEEP
    if isinstance(data, dict):
        return {k: (MASKED if is_sensitive_key(str(k)) else mask_value(v, max_depth - 1)) for k, v in data.items()}
    if isinstance(data, list):
        return [mask_value(v, max_depth - 1) for v in data]
    return data


def mask_headers(headers: dict) -> dict:
    out = {}
    for k, v in headers.items():
        ks = str(k)
        if is_sensitive_key(ks):
            out[k] = MASKED
        elif _ascii_lower(ks) == "cookie" and isinstance(v, str):
            out[k] = mask_cookie_header(v)
        else:
            out[k] = v
    return out


# ---------------------------------------------------------------- serde_json-compatible bytes path
def ryu_format(x: float) -> str:
    """Shortest round-trip digits (== repr) laid out like ryu's `format_finite`."""
    if x == 0.0:
        return "-0.0" if str(x).startswith("-") else "0.0"
    sign, digits, exp = Decimal(repr(x)).as_tuple()
    ds = "".join(map(str, digits)).rstrip("0") or "0"
    exp += len(digits) - len(ds)
    n, k = len(ds), exp
    kk = n + k
    s = "-" if sign else ""
    if 0 <= k and kk <= 16:
        return s + ds + "0" * k + ".0"
    if 0 < kk <= 16:
        return s + ds[:kk] + "." + ds[kk:]
    if -5 < kk <= 0:
        return s + "0." + "0" * (-kk) + ds
    e = kk - 1
    return s + (ds if n == 1 else ds[0] + "." + ds[1:]) + "e" + str(e)


def _escape(s: str) -> str:
    out = ['"']
    for ch in s:
        o = ord(ch)
        if ch == '"':
            out.append('\\"')
        elif ch == "\\":
            out.append("\\\\")
        elif o == 8:
            out.append("\\b")
        elif o == 12:
            out.append("\\f")
        elif o == 10:
            out.append("\\n")
        elif o == 13:
            out.append("\\r")
        elif o == 9:
            out.append("\\t")
        elif o < 0x20:
            out.append("\\u%04x" % o)
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)


def _ser(v: Any, out: List[str]) -> None:
    if v is None:
        out.append("null")
    elif v is True:
        out.append("true")
    elif v is False:
        out.append("false")
    elif isinstance(v, int):
        out.append(str(v))
    elif isinstance(v, float):
        out.append(ryu_format(v))
    elif isinstance(v, str):
        out.append(_escape(v))
    elif isinstance(v, list):
        out.append("[")
        for i, x in enumerate(v):
            if i:
                out.append(",")
            _ser(x, out)
        out.append("]")
    else:
        out.append("{")
        for i, k in enumerate(sorted(v, key=lambda s: s.encode("utf-8"))):
            if i:
                out.append(",")
            out.append(_escape(k))
            out.append(":")
            _ser(v[k], out)
        out.append("}")


def _depth(v: Any) -> int:
    d, stack = 0, [(v, 1)]
    while stack:
        x, k = stack.pop()
        if isinstance(x, (dict, list)):
            d = max(d, k)
            stack.extend((y, k + 1) for y in (x.values() if isinstance(x, dict) else x))
    return d


def parse_serde(payload: bytes) -> Any:
    text = payload.decode("utf-8")       # invalid UTF-8 -> error, like serde_json::from_slice

    def parse_int(t: str):
        v = int(t)
        if t.startswith("-"):
            return v if v != 0 and v >= -(2 ** 63) else parse_float(t)      # "-0" is the float -0.0 in serde_json
        return v if v <= 2 ** 64 - 1 else parse_float(t)                  # beyond binary64 too: "number out of range"

    def parse_float(t: str):
        v = float(t)
        if v in (float("inf"), float("-inf")):
            raise ValueError("number out of range")
        return v

    def bad(c):
        raise ValueError(c)

    def pairs(kv):
        d = dict(kv)
        if len(d) != len(kv):            # serde_json parsed the values a duplicate key overwrites as well
            _reject_lone_surrogates([x for _, x in kv])
        return d

    v = json.loads(text, parse_int=parse_int, parse_float=parse_float, parse_constant=bad, object_pairs_hook=pairs)
    # serde_json's check_recursion!: remaining_depth starts at 128, each '[' or '{' decrements it and the parse fails when it
    # reaches 0, so 127 nested containers parse and 128 do not.
    if _depth(v) > 127:
        raise ValueError("recursion limit exceeded")
    _reject_lone_surrogates(v)
    return v


def _reject_lone_surrogates(v: Any) -> None:
    """json.loads keeps a \\uD800-\\uDFFF escape that is not half of a pair as a lone surrogate; serde_json rejects it while
    parsing (parse_unicode_escape), wherever the string sits.  A valid pair has become one astral code point by now."""
    stack = [v]
    while stack:
        x = stack.pop()
        if isinstance(x, dict):
            stack.extend(x.keys())
            stack.extend(x.values())
        elif isinstance(x, list):
            stack.extend(x)
        elif isinstance(x, str) and any("\ud800" <= c <= "\udfff" for c in x):
            raise ValueError("lone leading or trailing surrogate in hex escape")


def mask_json_bytes(payload: bytes, max_depth: int = 10) -> bytes:
    """mask_sensitive_json_bytes (lib.rs:346-360); raises ValueError where the crate raises."""
    out: List[str] = []
    _ser(mask_value(parse_serde(payload), max_depth), out)
    return "".join(out).encode("utf-8")
