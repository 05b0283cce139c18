// json_mask.h — request_logging_masking on the JSON DOM of json_toon.h: sensitive-key classifier,
// depth-capped masking walk and serde_json-compatible re-serialisation (sorted keys, shortest
// round-trip floats).  Host + device, one payload per thread; shared verbatim with the CPU tests.
//
// Reference (paths relative to /root/reference):
//   normalize_key_for_masking / has_non_sensitive_suffix / is_sensitive_key
//                                   crates/request_logging_masking_native_extension/src/lib.rs:79-187
//   mask_json_value_inner           lib.rs:276-305        mask_sensitive_json_bytes   lib.rs:346-360
//   output format: serde_json 1.0.149 `to_vec` of a `Value` (BTreeMap objects) — see oracle/mask_ref.py
#pragma once
#include "json_toon.h"

namespace cfm {

using cfj::Big;
using cfj::Dbl;
using cfj::JNode;
using cfj::StrIter;

enum : int { MS_OK = 0, MS_PARSE_ERROR = 2, MS_UNSUPPORTED = 6, MS_OVERFLOW = 7 };

// serde_json's recursion limit: remaining_depth starts at 128 and the parse fails when an opening bracket brings it to 0, so a
// document holds at most 127 nested containers.  The mask path parses exactly that deep; one level more is a parse error.
static const int MASK_MAXD = 127;

// Output cursor of the masking walk.  Past its cap it stops writing but keeps counting, so that a unit whose output outgrows its
// room reports the exact length it needs (saturating at 0xFFFFFFFF).
struct Out {
  uint8_t* p;
  uint32_t n, cap;
  bool over;
  CF_HD void put(uint32_t c) { if (n < cap) p[n++] = (uint8_t)c; else { over = true; if (n != 0xFFFFFFFFu) ++n; } }
  CF_HD void puts(const char* z) { while (*z) put((uint8_t)*z++); }
  CF_HD void put_cp(uint32_t cp) {
    if (cp < 0x80) put(cp);
    else if (cp < 0x800) { put(0xC0 | (cp >> 6)); put(0x80 | (cp & 63)); }
    else if (cp < 0x10000) { put(0xE0 | (cp >> 12)); put(0x80 | ((cp >> 6) & 63)); put(0x80 | (cp & 63)); }
    else { put(0xF0 | (cp >> 18)); put(0x80 | ((cp >> 12) & 63)); put(0x80 | ((cp >> 6) & 63)); put(0x80 | (cp & 63)); }
  }
  CF_HD void put_uint(uint32_t v) {
    uint8_t b[10]; int k = 0;
    do { b[k++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
    while (k) put(b[--k]);
  }
};

// ------------------------------------------------------------------------------------------------
// sensitive-key classifier (streaming over the decoded key; no buffer for the normalised key)
// ------------------------------------------------------------------------------------------------
enum : uint32_t {
  T_OTHER = 0, T_AUTH, T_AUTHORIZATION, T_JWT, T_PASSWORD, T_PASSPHRASE, T_SECRET, T_TOKEN, T_APIKEY,
  T_API, T_KEY, T_ACCESS, T_REFRESH, T_CLIENT, T_PRIVATE, T_SUFFIX   // any of the 16 non-sensitive suffix words
};

CF_HD bool tok_eq(const uint8_t* t, uint32_t n, const char* w) {
  uint32_t i = 0;
  for (; i < n; ++i) { if (!w[i] || (uint8_t)w[i] != t[i]) return false; }
  return w[i] == 0;
}

CF_HD uint32_t classify_token(const uint8_t* t, uint32_t n) {
  if (n > 13) return T_OTHER;
  if (tok_eq(t, n, "auth")) return T_AUTH;
  if (tok_eq(t, n, "authorization")) return T_AUTHORIZATION;
  if (tok_eq(t, n, "jwt")) return T_JWT;
  if (tok_eq(t, n, "password")) return T_PASSWORD;
  if (tok_eq(t, n, "passphrase")) return T_PASSPHRASE;
  if (tok_eq(t, n, "secret")) return T_SECRET;
  if (tok_eq(t, n, "token")) return T_TOKEN;
  if (tok_eq(t, n, "apikey")) return T_APIKEY;
  if (tok_eq(t, n, "api")) return T_API;
  if (tok_eq(t, n, "key")) return T_KEY;
  if (tok_eq(t, n, "access")) return T_ACCESS;
  if (tok_eq(t, n, "refresh")) return T_REFRESH;
  if (tok_eq(t, n, "client")) return T_CLIENT;
  if (tok_eq(t, n, "private")) return T_PRIVATE;
  if (tok_eq(t, n, "count") || tok_eq(t, n, "counts") || tok_eq(t, n, "size") || tok_eq(t, n, "length") || tok_eq(t, n, "ttl") ||
      tok_eq(t, n, "seconds") || tok_eq(t, n, "ms") || tok_eq(t, n, "id") || tok_eq(t, n, "ids") || tok_eq(t, n, "name") ||
      tok_eq(t, n, "type") || tok_eq(t, n, "url") || tok_eq(t, n, "uri") || tok_eq(t, n, "path") || tok_eq(t, n, "status") || tok_eq(t, n, "code"))
    return T_SUFFIX;
  return T_OTHER;
}

CF_HD bool is_bigram(uint32_t a, uint32_t b) {
  return (a == T_API && b == T_KEY) || (a == T_ACCESS && b == T_TOKEN) || (a == T_REFRESH && b == T_TOKEN) ||
         (a == T_CLIENT && b == T_SECRET) || (a == T_AUTH && b == T_TOKEN) || (a == T_JWT && b == T_TOKEN) || (a == T_PRIVATE && b == T_KEY);
}
CF_HD bool is_word(uint32_t t) { return t == T_PASSWORD || t == T_PASSPHRASE || t == T_SECRET || t == T_TOKEN || t == T_APIKEY || t == T_AUTHORIZATION; }

struct KeyClassifier {
  uint8_t tok[16];
  uint32_t tlen, ntok, prev, last;
  bool any_auth, any_word, any_bigram, exact1, exact2, pending_us, empty;
  CF_HD void init() { tlen = ntok = 0; prev = last = T_OTHER; any_auth = any_word = any_bigram = exact1 = exact2 = pending_us = false; empty = true; }
  CF_HD void end_token() {
    if (!tlen) return;
    uint32_t t = classify_token(tok, tlen > 16 ? 16 : tlen);
    if (tlen > 16) t = T_OTHER;
    if (t == T_AUTH || t == T_AUTHORIZATION || t == T_JWT) any_auth = true;
    if (is_word(t)) any_word = true;
    if (ntok >= 1 && is_bigram(prev, t)) any_bigram = true;
    if (ntok == 0) exact1 = is_word(t);
    if (ntok == 1) exact2 = is_bigram(prev, t);
    prev = last = t;
    ++ntok;
    tlen = 0;
  }
  CF_HD void push_char(uint32_t c) {          // c is a lower-case ASCII letter or digit
    if (pending_us) { end_token(); pending_us = false; }
    if (tlen < 16) tok[tlen] = (uint8_t)c;
    ++tlen;
    empty = false;
  }
  CF_HD void push_us() { if (!empty) pending_us = true; }   // committed only if an alnum follows (trailing '_' are trimmed)
  CF_HD bool result() {
    end_token();
    if (ntok == 0) return false;
    const bool has_suffix = ntok >= 2 && last == T_SUFFIX;
    if ((ntok == 1 && exact1) || (ntok == 2 && exact2)) return true;
    if (!has_suffix && any_auth) return true;
    if (has_suffix) return false;
    return any_word || any_bigram;
  }
};

// A key parsed from JSON carries JF_ESC when its text holds escapes; a raw key name (cf_classify_keys_host) never does, so a
// backslash in it is a character of the name.  Only ASCII letters and digits count, so the raw bytes of a multi-byte character
// classify like the character itself (a run of non-alphanumerics is one separator either way).
CF_HD bool key_sensitive(const uint8_t* s, const JNode& key) {
  KeyClassifier kc;
  kc.init();
  StrIter it{s + key.off, s + key.off + key.len};
  const bool esc = (key.t & cfj::JF_ESC) != 0;
  bool prev_lower_or_digit = false, prev_us = false;
  while (!it.done()) {
    const uint32_t ch = esc ? it.next() : *it.p++;
    const bool is_upper = ch >= 'A' && ch <= 'Z';
    const bool is_lower = ch >= 'a' && ch <= 'z';
    const bool is_digit = ch >= '0' && ch <= '9';
    if (is_upper && prev_lower_or_digit && !prev_us) kc.push_us();
    if (is_upper || is_lower || is_digit) { kc.push_char(is_upper ? ch + 32 : ch); prev_us = false; }
    else if (!prev_us && !kc.empty) { kc.push_us(); prev_us = true; }
    prev_lower_or_digit = is_lower || is_digit;
    if (is_upper) prev_us = false;
  }
  return kc.result();
}

// ------------------------------------------------------------------------------------------------
// numbers: serde_json prints i64/u64 verbatim, everything else as the shortest round-trip binary64
// in ryu's layout
// ------------------------------------------------------------------------------------------------
// ds[0..n) significant digits (no trailing zeros unless n == 1), value = 0.ds * 10^kk  (kk = n + k)
CF_HD void emit_ryu_layout(Out& o, bool neg, const uint8_t* ds, int n, int kk) {
  if (neg) o.put('-');
  const int k = kk - n;
  if (k >= 0 && kk <= 16) {
    for (int i = 0; i < n; ++i) o.put(ds[i]);
    for (int i = 0; i < k; ++i) o.put('0');
    o.put('.'); o.put('0');
  } else if (kk > 0 && kk <= 16) {
    for (int i = 0; i < kk; ++i) o.put(ds[i]);
    o.put('.');
    for (int i = kk; i < n; ++i) o.put(ds[i]);
  } else if (kk > -5 && kk <= 0) {
    o.put('0'); o.put('.');
    for (int i = 0; i < -kk; ++i) o.put('0');
    for (int i = 0; i < n; ++i) o.put(ds[i]);
  } else {
    o.put(ds[0]);
    if (n > 1) { o.put('.'); for (int i = 1; i < n; ++i) o.put(ds[i]); }
    o.put('e');
    int e = kk - 1;
    if (e < 0) { o.put('-'); e = -e; }
    o.put_uint((uint32_t)e);
  }
}

struct NumWork { Big* big; Big* big2; uint8_t* digits; uint32_t digits_cap; };

// exact decimal expansion of a finite non-zero binary64: digits D[0..nd), value = 0.D * 10^kk
CF_HD bool exact_digits(const Dbl& d, NumWork& w, uint32_t* nd_out, int* kk_out) {
  Big* X = w.big;
  bool integral = d.e >= 0;
  if (!integral && -d.e < 64) integral = (d.m & ((1ull << (-d.e)) - 1)) == 0;
  uint32_t kfrac = 0;
  if (integral) {
    uint64_t m = d.e >= 0 ? d.m : d.m >> (-d.e);
    X->w[0] = (uint32_t)m; X->w[1] = (uint32_t)(m >> 32);
    X->n = X->w[1] ? 2 : (X->w[0] ? 1 : 0);
    if (d.e > 0 && !X->shl((uint32_t)d.e)) return false;
  } else {
    kfrac = (uint32_t)(-d.e);
    X->w[0] = (uint32_t)d.m; X->w[1] = (uint32_t)(d.m >> 32);
    X->n = X->w[1] ? 2 : 1;
    for (uint32_t i = 0; i < kfrac;) {
      uint32_t step = kfrac - i >= 13 ? 13 : kfrac - i, mul = 1;
      for (uint32_t j = 0; j < step; ++j) mul *= 5;
      if (!X->mul_add(mul, 0)) return false;
      i += step;
    }
  }
  uint32_t nd = cfj::big_to_digits(X, w.digits, w.digits_cap - 24);
  if (nd == 0xFFFFFFFFu || nd == 0) return false;
  *nd_out = nd;
  *kk_out = (int)nd - (int)kfrac;
  return true;
}

// shortest digit string that parses back to exactly `d`: binary search on the precision p.  A probe takes the p-digit decimal
// nearest to `d` (exact round-half-even of the decimal expansion) and, when that one does not parse back to `d`, the p-digit
// decimal on the other side of `d`.  The second one matters at a power of two: there the interval that rounds to `d` is half
// as wide below `d` as above it, so the nearest decimal can fall out of it while the farther one is inside.  "Some p-digit
// decimal parses back" is monotone in p, which keeps the binary search valid, and the nearer of two that both parse back wins.
CF_HD bool shortest_digits(const Dbl& d, NumWork& w, uint8_t* out_ds, int* out_n, int* out_kk) {
  uint32_t nd;
  int kk;
  if (!exact_digits(d, w, &nd, &kk)) return false;
  const uint8_t* D = w.digits;
  uint8_t* txt = w.digits + w.digits_cap - 24;     // "dddddddddddddddddE" scratch lives at the buffer's tail
  // 0 / 1: whether "c[0..p)e(ckk-p)" parses back to d; -1: the workspace is too small
  auto round_trips = [&](const uint8_t* c, int p, int ckk) -> int {
    uint32_t tl = 0;
    for (int i = 0; i < p; ++i) txt[tl++] = c[i];
    txt[tl++] = 'e';
    int ex = ckk - p;
    if (ex < 0) { txt[tl++] = '-'; ex = -ex; }
    uint8_t eb[6]; int en = 0;
    do { eb[en++] = (uint8_t)('0' + ex % 10); ex /= 10; } while (ex);
    while (en) txt[tl++] = eb[--en];
    Dbl back;
    if (!cfj::dec_to_double(txt, tl, &back, w.big2)) return -1;
    return !back.inf && back.m == d.m && (back.e == d.e || back.m == 0);
  };
  int lo = 1, hi = nd < 17 ? (int)nd : 17;          // 17 significant digits always round-trip
  int best_n = 0, best_kk = 0;
  uint8_t best[17];
  while (lo <= hi) {
    const int p = (lo + hi) >> 1;
    uint8_t dn[17], upc[17];                         // D truncated to p digits, and one unit in the p-th digit above it
    int up_kk = kk;
    for (int i = 0; i < p; ++i) dn[i] = upc[i] = D[i];
    bool exact = true, up = false;
    for (uint32_t i = (uint32_t)p; i < nd; ++i) if (D[i] != '0') { exact = false; break; }
    if (!exact) {
      int i = p - 1;
      while (i >= 0 && upc[i] == '9') { upc[i] = '0'; --i; }
      if (i >= 0) upc[i]++; else { for (int j = p - 1; j > 0; --j) upc[j] = upc[j - 1]; upc[0] = '1'; ++up_kk; }
      if (D[p] > '5') up = true;
      else if (D[p] == '5') {
        bool rest = false;
        for (uint32_t i2 = (uint32_t)p + 1; i2 < nd; ++i2) if (D[i2] != '0') { rest = true; break; }
        up = rest || ((D[p - 1] - '0') & 1);
      }
    }
    const uint8_t* c = up ? upc : dn;
    int ckk = up ? up_kk : kk;
    int r = round_trips(c, p, ckk);
    if (r < 0) return false;
    if (!r && !exact) {
      c = up ? dn : upc;
      ckk = up ? kk : up_kk;
      if ((r = round_trips(c, p, ckk)) < 0) return false;
    }
    if (r) { best_n = p; best_kk = ckk; for (int i = 0; i < p; ++i) best[i] = c[i]; hi = p - 1; }
    else lo = p + 1;
  }
  if (!best_n) return false;
  while (best_n > 1 && best[best_n - 1] == '0') --best_n;
  for (int i = 0; i < best_n; ++i) out_ds[i] = best[i];
  *out_n = best_n;
  *out_kk = best_kk;
  return true;
}

CF_HD int emit_number_serde(Out& o, const uint8_t* s, const JNode& nd, NumWork& w) {
  const uint8_t* t = s + nd.off;
  const uint32_t len = nd.len;
  const bool neg = (nd.t & cfj::JF_NEG) != 0;
  const uint8_t* dg = t + (neg ? 1 : 0);
  const uint32_t dl = len - (neg ? 1 : 0);
  if (!(nd.t & (cfj::JF_FRAC | cfj::JF_EXP))) {
    bool fits = dl < 19;
    if (!fits && dl <= 20) {
      const char* lim = neg ? "9223372036854775808" : "18446744073709551615";
      const uint32_t ll = neg ? 19 : 20;
      if (dl < ll) fits = true;
      else if (dl == ll) { fits = true; for (uint32_t i = 0; i < ll; ++i) { if (dg[i] < (uint8_t)lim[i]) break; if (dg[i] > (uint8_t)lim[i]) { fits = false; break; } } }
    }
    if (fits && !(neg && dl == 1 && dg[0] == '0')) { for (uint32_t i = 0; i < len; ++i) o.put(t[i]); return MS_OK; }
  }
  // float: cheap exact path when the literal has <= 15 significant digits and a tame exponent
  {
    uint8_t ds[16];
    int n = 0, point_shift = 0;
    bool seen_dot = false, any = false, overflow_digits = false;
    uint32_t p = 0;
    for (; p < dl; ++p) {
      const uint8_t c = dg[p];
      if (c == '.') { seen_dot = true; continue; }
      if (c == 'e' || c == 'E') break;
      if (seen_dot) --point_shift;
      if (!any && c == '0') continue;
      any = true;
      if (n < 16) ds[n] = c;
      ++n;
      if (n > 15 && c != '0') overflow_digits = true;
    }
    long long ex = 0;
    if (p < dl) {
      ++p;
      bool en = false;
      if (p < dl && (dg[p] == '+' || dg[p] == '-')) { en = dg[p] == '-'; ++p; }
      for (; p < dl; ++p) if (ex < 100000) ex = ex * 10 + (dg[p] - '0');
      if (en) ex = -ex;
    }
    if (!any) { if (neg) o.put('-'); o.put('0'); o.put('.'); o.put('0'); return MS_OK; }   // +-0.0
    if (!overflow_digits) {
      int total = n;                                   // digits read (may include trailing zeros beyond 15: all '0')
      int nn = n > 15 ? 15 : n;
      while (nn > 1 && ds[nn - 1] == '0') --nn;
      const long long kk = (long long)total + point_shift + ex;   // value = 0.ds * 10^kk
      if (kk > -290 && kk < 290) { emit_ryu_layout(o, neg, ds, nn, (int)kk); return MS_OK; }
    }
  }
  Dbl d;
  if (!cfj::dec_to_double(t, len, &d, w.big)) return MS_UNSUPPORTED;
  if (d.inf) return MS_PARSE_ERROR;                    // serde_json: "number out of range"
  if (d.m == 0) { if (neg) o.put('-'); o.put('0'); o.put('.'); o.put('0'); return MS_OK; }
  uint8_t ds[17];
  int n, kk;
  if (!shortest_digits(d, w, ds, &n, &kk)) return MS_UNSUPPORTED;
  emit_ryu_layout(o, d.neg, ds, n, kk);
  return MS_OK;
}

// serde_json parses the whole document before masking it, so a number out of binary64's range fails the call wherever it sits,
// printed, masked, below the depth cap or overwritten by a duplicate key: the mask path's parser runs this on every number.  Every literal under 10^308 is in range; one of 10^309 or more is not; only those in [10^308, 10^309) need the
// exact conversion.  MS_OK, MS_PARSE_ERROR ("number out of range") or MS_UNSUPPORTED (longer than the workspace).
CF_HD int number_in_range(const uint8_t* t, uint32_t len, uint32_t fl, NumWork& w) {
  if (!(fl & cfj::JF_EXP) && len <= 308) return MS_OK;   // at most 308 integer digits
  long long kk = 0;                                      // value in [10^(kk-1), 10^kk)
  bool dot = false, any = false;
  uint32_t p = (fl & cfj::JF_NEG) ? 1 : 0;
  for (; p < len; ++p) {
    const uint8_t c = t[p];
    if (c == '.') { dot = true; continue; }
    if (c == 'e' || c == 'E') break;
    if (!any) { if (c == '0') { if (dot) --kk; continue; } any = true; }
    if (!dot) ++kk;
  }
  if (!any) return MS_OK;                                // +-0
  if (p < len) {
    ++p;
    bool en = false;
    if (p < len && (t[p] == '+' || t[p] == '-')) { en = t[p] == '-'; ++p; }
    long long ex = 0;
    for (; p < len; ++p) if (ex < 100000) ex = ex * 10 + (t[p] - '0');
    kk += en ? -ex : ex;
  }
  if (kk <= 308) return MS_OK;
  if (kk >= 310) return MS_PARSE_ERROR;
  Dbl d;
  if (!cfj::dec_to_double(t, len, &d, w.big)) return MS_UNSUPPORTED;
  return d.inf ? MS_PARSE_ERROR : MS_OK;
}

CF_HD void emit_json_string(Out& o, const uint8_t* s, const JNode& nd) {
  StrIter it{s + nd.off, s + nd.off + nd.len};
  o.put('"');
  while (!it.done()) {
    const uint32_t cp = it.next();
    switch (cp) {
      case '"': o.put('\\'); o.put('"'); break;
      case '\\': o.put('\\'); o.put('\\'); break;
      case 8: o.put('\\'); o.put('b'); break;
      case 12: o.put('\\'); o.put('f'); break;
      case 10: o.put('\\'); o.put('n'); break;
      case 13: o.put('\\'); o.put('r'); break;
      case 9: o.put('\\'); o.put('t'); break;
      default:
        if (cp < 0x20) { o.put('\\'); o.put('u'); o.put('0'); o.put('0'); o.put("0123456789abcdef"[cp >> 4]); o.put("0123456789abcdef"[cp & 15]); }
        else o.put_cp(cp);
    }
  }
  o.put('"');
}

// key order of serde_json's BTreeMap<String, Value>: bytewise on UTF-8 == code point order
CF_HD bool key_less(const uint8_t* s, const JNode& a, const JNode& b) {
  StrIter ia{s + a.off, s + a.off + a.len}, ib{s + b.off, s + b.off + b.len};
  while (!ia.done() && !ib.done()) {
    uint32_t ca = ia.next(), cb = ib.next();
    if (ca != cb) return ca < cb;
  }
  return ia.done() && !ib.done();
}

CF_HD void sort_keys(const uint8_t* s, const JNode* N, uint32_t* a, uint32_t n) {   // heapsort
  if (n < 2) return;
  for (uint32_t start = n / 2; start-- > 0;) {
    uint32_t root = start;
    while (true) {
      uint32_t child = 2 * root + 1;
      if (child >= n) break;
      if (child + 1 < n && key_less(s, N[a[child]], N[a[child + 1]])) ++child;
      if (!key_less(s, N[a[root]], N[a[child]])) break;
      uint32_t t = a[root]; a[root] = a[child]; a[child] = t;
      root = child;
    }
  }
  for (uint32_t end = n - 1; end > 0; --end) {
    uint32_t t = a[0]; a[0] = a[end]; a[end] = t;
    uint32_t root = 0;
    while (true) {
      uint32_t child = 2 * root + 1;
      if (child >= end) break;
      if (child + 1 < end && key_less(s, N[a[child]], N[a[child + 1]])) ++child;
      if (!key_less(s, N[a[root]], N[a[child]])) break;
      uint32_t t2 = a[root]; a[root] = a[child]; a[child] = t2;
      root = child;
    }
  }
}

struct MFrame { uint32_t node, cur, i, seg; int depth; };   // depth = max_depth available to the children

// emit value `v` given the depth budget `depth` of the call mask_json_value_inner(v, depth)
CF_HD int mask_emit(const uint8_t* s, const JNode* N, Out& o, int max_depth, uint32_t* idx, uint32_t idx_cap, NumWork& w) {
  MFrame st[MASK_MAXD + 1];
  int sp = 0;
  uint32_t idx_used = 0;
  // returns true when a frame was pushed
  auto value = [&](uint32_t v, int depth, int* err) -> bool {
    if (depth <= 0) { o.puts("\"<nested too deep>\""); return false; }
    const uint32_t t = N[v].t & cfj::J_TYPE;
    switch (t) {
      case cfj::J_NULL: o.puts("null"); return false;
      case cfj::J_TRUE: o.puts("true"); return false;
      case cfj::J_FALSE: o.puts("false"); return false;
      case cfj::J_STR: emit_json_string(o, s, N[v]); return false;
      case cfj::J_NUM: { int r = emit_number_serde(o, s, N[v], w); if (r) *err = r; return false; }
      case cfj::J_ARR:
        o.put('[');
        if (N[v].len == 0) { o.put(']'); return false; }
        st[sp++] = MFrame{v, N[v].off, 0, 0, depth - 1};
        return true;
      default: {   // object
        o.put('{');
        const uint32_t n = N[v].len;
        if (n == 0) { o.put('}'); return false; }
        if (idx_used + n > idx_cap) { *err = MS_UNSUPPORTED; return false; }
        uint32_t* a = idx + idx_used;
        uint32_t k = 0;
        for (uint32_t m = N[v].off; m; m = N[m].next) a[k++] = m;
        sort_keys(s, N, a, n);
        st[sp++] = MFrame{v, 0, 0, idx_used, depth - 1};
        idx_used += n;
        return true;
      }
    }
  };
  int err = 0;
  value(0, max_depth, &err);
  while (sp > 0 && !err) {
    MFrame& f = st[sp - 1];
    const bool is_obj = (N[f.node].t & cfj::J_TYPE) == cfj::J_OBJ;
    if (is_obj) {
      if (f.i >= N[f.node].len) { o.put('}'); --sp; continue; }
      const uint32_t k = idx[f.seg + f.i];
      if (f.i) o.put(',');
      ++f.i;
      emit_json_string(o, s, N[k]);
      o.put(':');
      if (key_sensitive(s, N[k])) { o.puts("\"******\""); continue; }
      const int depth = f.depth;
      if (sp > MASK_MAXD) { err = MS_UNSUPPORTED; break; }
      value(k + 1, depth, &err);
    } else {
      if (f.cur == 0) { o.put(']'); --sp; continue; }
      const uint32_t x = f.cur;
      if (f.i) o.put(',');
      ++f.i;
      f.cur = N[x].next;
      const int depth = f.depth;
      if (sp > MASK_MAXD) { err = MS_UNSUPPORTED; break; }
      value(x, depth, &err);
    }
  }
  return err;
}

CF_HD int mask_finish(int pr, const uint8_t* s, const JNode* nodes, uint32_t* idx, uint32_t idx_cap, uint8_t* out, uint32_t out_cap,
                      uint32_t* out_len, int max_depth, NumWork& w);

// serde_json's parse: nesting up to its recursion limit, and every number in binary64's range
struct RangeCheck {
  NumWork* w;
  CF_HD int operator()(const uint8_t* t, uint32_t len, uint32_t fl) const {
    const int r = number_in_range(t, len, fl, *w);
    return r == MS_OK ? cfj::PARSE_OK : r == MS_PARSE_ERROR ? cfj::PARSE_ERROR : cfj::PARSE_UNSUPPORTED;
  }
};

// Whole per-unit pipeline: mask_sensitive_json_bytes(payload, max_depth).
CF_HD int mask_process(const uint8_t* s, uint32_t n, JNode* nodes, uint32_t node_cap, uint32_t* idx, uint32_t idx_cap, uint8_t* out,
                       uint32_t out_cap, uint32_t* out_len, int max_depth, NumWork& w) {
  uint32_t count = 0;
  RangeCheck check{&w};
  int pr = cfj::json_parse_t<MASK_MAXD, cfj::PARSE_ERROR>(s, n, nodes, node_cap, &count, check);
  return mask_finish(pr, s, nodes, idx, idx_cap, out, out_cap, out_len, max_depth, w);
}

// the part after the parse (pr = PARSE_* of whichever parser built `nodes`).  MS_OVERFLOW: the output did not fit in out_cap
// bytes, and *out_len is the length it needs.
CF_HD int mask_finish(int pr, const uint8_t* s, const JNode* nodes, uint32_t* idx, uint32_t idx_cap, uint8_t* out, uint32_t out_cap,
                      uint32_t* out_len, int max_depth, NumWork& w) {
  if (pr == cfj::PARSE_ERROR) return MS_PARSE_ERROR;
  if (pr == cfj::PARSE_UNSUPPORTED) return MS_UNSUPPORTED;
  Out o;
  o.p = out; o.n = 0; o.cap = out_cap; o.over = false;
  int err = mask_emit(s, nodes, o, max_depth, idx, idx_cap, w);
  if (err) return err;
  if (o.over && o.n == 0xFFFFFFFFu) return MS_UNSUPPORTED;
  *out_len = o.n;
  return o.over ? MS_OVERFLOW : MS_OK;
}

}  // namespace cfm
