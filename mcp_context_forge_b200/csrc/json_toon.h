// json_toon.h — strict JSON -> flat DOM -> TOON text, one payload per (GPU) thread.
// Plain sequential C++ that compiles for host and device (the CPU unit tests run the very same code
// through tests/hostsim; the CUDA kernel toon_kernel in cfgpu.cu calls toon_process per unit).
//
// Reference semantics (paths relative to /root/reference):
//   parse      orjson.loads                               plugins/toon_encoder/toon_encoder.py:281
//   encode     toon.encode and helpers                    plugins/toon_encoder/toon.py:82-565
//   decision   "only if strictly smaller in UTF-8 bytes"  plugins/toon_encoder/toon_encoder.py:295-303
// Quirks reproduced on purpose are listed in SURVEY.md Appendix A-5/A-6 (hyphen anywhere forces
// quotes, columnar header keys are never quoted, list-item indentation compounds, the unchecked
// `.keys()` crash path, `$` admitting a final newline in the key regex, ...).
#pragma once
#include <stdint.h>

#include "scan_core.h"
#include "unicode_tables.h"

namespace cfj {

// ------------------------------------------------------------------------------------------------
// Unicode tables (value lists generated from CPython; one copy per address space)
// ------------------------------------------------------------------------------------------------
static const uint32_t ND_LO_H[] = {CFU_ND_LO};
static const uint32_t ND_HI_H[] = {CFU_ND_HI};
static const uint32_t WS_LO_H[] = {CFU_WS_LO};
static const uint32_t WS_HI_H[] = {CFU_WS_HI};
#ifdef __CUDACC__
static __device__ const uint32_t ND_LO_D[] = {CFU_ND_LO};
static __device__ const uint32_t ND_HI_D[] = {CFU_ND_HI};
static __device__ const uint32_t WS_LO_D[] = {CFU_WS_LO};
static __device__ const uint32_t WS_HI_D[] = {CFU_WS_HI};
#endif
#ifdef __CUDA_ARCH__
#define CFJ_TAB(name) name##_D
#else
#define CFJ_TAB(name) name##_H
#endif

// ASCII classes for the plain-string fast path of parse_string
enum : uint32_t { AC_STOP = 1 /* '"', '\\', control, non-ASCII */, AC_SPECIAL = 2 /* , : [ ] { } - */, AC_KEYCH = 4 /* [A-Za-z0-9_.] */ };
#define CFJ_AC_ROW(b) \
  ((uint8_t)((((b) < 0x20 || (b) >= 0x80 || (b) == '"' || (b) == '\\') ? 1 : 0) | \
             (((b) == ',' || (b) == ':' || (b) == '[' || (b) == ']' || (b) == '{' || (b) == '}' || (b) == '-') ? 2 : 0) | \
             ((((b) >= 'A' && (b) <= 'Z') || ((b) >= 'a' && (b) <= 'z') || ((b) >= '0' && (b) <= '9') || (b) == '_' || (b) == '.') ? 4 : 0)))
#define CFJ_AC_8(b) CFJ_AC_ROW(b), CFJ_AC_ROW((b) + 1), CFJ_AC_ROW((b) + 2), CFJ_AC_ROW((b) + 3), CFJ_AC_ROW((b) + 4), CFJ_AC_ROW((b) + 5), CFJ_AC_ROW((b) + 6), CFJ_AC_ROW((b) + 7)
#define CFJ_AC_64(b) CFJ_AC_8(b), CFJ_AC_8((b) + 8), CFJ_AC_8((b) + 16), CFJ_AC_8((b) + 24), CFJ_AC_8((b) + 32), CFJ_AC_8((b) + 40), CFJ_AC_8((b) + 48), CFJ_AC_8((b) + 56)
#define CFJ_AC_ALL CFJ_AC_64(0), CFJ_AC_64(64), CFJ_AC_64(128), CFJ_AC_64(192)
static const uint8_t ACLS_H[256] = {CFJ_AC_ALL};
#ifdef __CUDACC__
static __device__ const uint8_t ACLS_D[256] = {CFJ_AC_ALL};
#endif

CF_HD bool is_nd(uint32_t cp) {            // \d of a str pattern
  if (cp < 0x80) return cp >= '0' && cp <= '9';
  uint32_t lo = 0, hi = CFU_ND_COUNT;
  while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (CFJ_TAB(ND_LO)[mid] <= cp) lo = mid; else hi = mid; }
  return cp >= CFJ_TAB(ND_LO)[lo] && cp <= CFJ_TAB(ND_HI)[lo];
}
CF_HD bool is_pyspace(uint32_t cp) {       // str.isspace()
  for (uint32_t i = 0; i < CFU_WS_COUNT; ++i) if (cp >= CFJ_TAB(WS_LO)[i] && cp <= CFJ_TAB(WS_HI)[i]) return true;
  return false;
}

// ------------------------------------------------------------------------------------------------
// DOM
// ------------------------------------------------------------------------------------------------
struct alignas(16) JNode { uint32_t t, off, len, next; };   // one 128-bit load/store per node
enum : uint32_t { J_NULL = 0, J_FALSE = 1, J_TRUE = 2, J_NUM = 3, J_STR = 4, J_ARR = 5, J_OBJ = 6, J_KEY = 7, J_TYPE = 0xF };
enum : uint32_t { JF_ESC = 0x100, JF_NEG = 0x100, JF_FRAC = 0x200, JF_EXP = 0x400,
                  // string properties computed while the parser validates the string (one pass, no re-scan at emit time)
                  JF_Q = 0x800 /* toon._needs_quotes(s) */, JF_CTRLERR = 0x1000 /* a char toon._quote_string rejects */,
                  JF_KEYOK = 0x2000 /* valid unquoted TOON key */ };
//   scalar   : off/len = raw text span (strings: between the quotes)
//   container: off = index of first child (0 = none), len = number of children; for objects the
//              children are J_KEY nodes, the value of key k is node k+1, keys are chained by .next
//   array elements are chained by .next; an object value's .next holds the hash of its key
static const int MAXD = 64;                // nesting depth handled on the device (deeper -> TS_UNSUPPORTED)

enum : int { PARSE_OK = 0, PARSE_ERROR = 1, PARSE_UNSUPPORTED = 2 };

CF_HD bool j_ws(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
CF_HD int hexv(uint32_t c) {
  if (c >= '0' && c <= '9') return (int)c - '0';
  c |= 0x20;
  if (c >= 'a' && c <= 'f') return (int)c - 'a' + 10;
  return -1;
}

// Incremental evaluation of the reference's string predicates over the decoded code points
// (toon.py:163-222 _needs_quotes, :276-279 the control characters _quote_string rejects, :286-309 key rule).
struct StrProps {
  uint32_t count, first, last;
  int num;            // number-like automaton state (toon.py:54); -1 = failed
  bool lead0, special, ctrl, ctrl_bad, key_ok, key_nl, r1, r2, r3;
  CF_HD void init() { count = first = last = 0; num = 0; lead0 = true; special = ctrl = ctrl_bad = key_nl = false; key_ok = true; r1 = r2 = r3 = true; }
  CF_HD void feed(uint32_t cp) {
    if (count == 0) first = cp;
    last = cp;
    if (cp < 32) { ctrl = true; if (cp != '\n' && cp != '\r' && cp != '\t') ctrl_bad = true; }
    if (cp == '\n' || cp == '\r' || cp == '\t' || cp == ',' || cp == ':' || cp == '[' || cp == ']' || cp == '{' || cp == '}' || cp == '"' || cp == '\\' || cp == '-') special = true;
    const bool d = (cp >= '0' && cp <= '9') || (cp >= 0x80 && (num > 0 || lead0) && is_nd(cp));
    if (count == 0) lead0 = (cp == '0'); else lead0 = lead0 && d;
    switch (num) {
      case 0: num = (cp == '0') ? 1 : (cp >= '1' && cp <= '9') ? 2 : -1; break;
      case 1: num = (cp == '.') ? 3 : (cp == 'e' || cp == 'E') ? 5 : -1; break;
      case 2: num = d ? 2 : (cp == '.') ? 3 : (cp == 'e' || cp == 'E') ? 5 : -1; break;
      case 3: num = d ? 4 : -1; break;
      case 4: num = d ? 4 : (cp == 'e' || cp == 'E') ? 5 : -1; break;
      case 5: num = (cp == '+') ? 6 : d ? 7 : -1; break;   // '-' already forces quotes through `special`
      case 6: num = d ? 7 : -1; break;
      case 7: num = d ? 7 : -1; break;
      default: break;
    }
    // key rule ^[A-Za-z_][A-Za-z0-9_.]*$ where `$` also admits one final "\n"
    if (key_nl) key_ok = false;
    const bool al = (cp >= 'A' && cp <= 'Z') || (cp >= 'a' && cp <= 'z') || cp == '_';
    if (count == 0) { if (!al) key_ok = false; }
    else if (!(al || (cp >= '0' && cp <= '9') || cp == '.')) { if (cp == '\n') key_nl = true; else key_ok = false; }
    if (count >= 4 || cp != (uint32_t)(uint8_t)"null"[count]) r1 = false;
    if (count >= 4 || cp != (uint32_t)(uint8_t)"true"[count]) r2 = false;
    if (count >= 5 || cp != (uint32_t)(uint8_t)"false"[count]) r3 = false;
    ++count;
  }
  CF_HD uint32_t flags() const {
    const bool reserved = (r1 && count == 4) || (r2 && count == 4) || (r3 && count == 5);
    const bool numlike = (num == 1 || num == 2 || num == 4 || num == 7);
    uint32_t f = 0;
    if (count == 0 || reserved || special || numlike || (lead0 && count >= 2) || ctrl || is_pyspace(first) || is_pyspace(last)) f |= JF_Q;
    if (ctrl_bad) f |= JF_CTRLERR;
    if (count > 0 && key_ok && !reserved) f |= JF_KEYOK;
    return f;
  }
};

// Validate one JSON string starting at the opening quote; returns false on any error.  On success
// *pos is just past the closing quote.  Hash (FNV-1a) is over the DECODED UTF-8 bytes.
CF_HD bool parse_string(const uint8_t* s, uint32_t n, uint32_t* pos, uint32_t* flags, uint32_t* hash) {
  // Fast path: the string is plain printable ASCII without escapes and does not start with a digit
  // (so the number-like rules cannot apply).  Four bytes per step: the loads and class lookups of a
  // step are independent, which is what a lone GPU thread needs (no speculation across the branch).
  {
    const uint32_t b = *pos + 1;
    uint32_t q = b, h = 2166136261u, orb = 0, andb = 0xFF;
    const uint8_t* T = CFJ_TAB(ACLS);
    bool plain = false;
    if (b < n && !(s[b] >= '0' && s[b] <= '9')) {
      while (true) {
        if (q + 4 <= n) {
          const uint32_t c0 = s[q], c1 = s[q + 1], c2 = s[q + 2], c3 = s[q + 3];
          const uint32_t k0 = T[c0], k1 = T[c1], k2 = T[c2], k3 = T[c3];
          if (!((k0 | k1 | k2 | k3) & AC_STOP)) {
            orb |= k0 | k1 | k2 | k3; andb &= k0 & k1 & k2 & k3;
            h = (h ^ c0) * 16777619u; h = (h ^ c1) * 16777619u; h = (h ^ c2) * 16777619u; h = (h ^ c3) * 16777619u;
            q += 4;
            continue;
          }
        }
        // tail: one byte at a time up to the stopping byte
        while (q < n) {
          const uint32_t c = s[q], k = T[c];
          if (k & AC_STOP) { plain = (c == '"'); break; }
          orb |= k; andb &= k; h = (h ^ c) * 16777619u; ++q;
        }
        break;
      }
    }
    if (plain) {
      const uint32_t count = q - b;
      uint32_t f = 0;
      if (count == 0) f = JF_Q;
      else {
        const uint32_t first = s[b], last = s[q - 1];
        const bool reserved = (count == 4 && ((first == 'n' && s[b + 1] == 'u' && s[b + 2] == 'l' && s[b + 3] == 'l') ||
                                              (first == 't' && s[b + 1] == 'r' && s[b + 2] == 'u' && s[b + 3] == 'e'))) ||
                              (count == 5 && first == 'f' && s[b + 1] == 'a' && s[b + 2] == 'l' && s[b + 3] == 's' && s[b + 4] == 'e');
        if (reserved || (orb & AC_SPECIAL) || first == ' ' || last == ' ') f |= JF_Q;   // ' ' is the only printable-ASCII str.isspace() char
        const bool al = (first >= 'A' && first <= 'Z') || (first >= 'a' && first <= 'z') || first == '_';
        if (al && (andb & AC_KEYCH) && !reserved) f |= JF_KEYOK;
      }
      *pos = q + 1;
      *flags = f;
      *hash = h;
      return true;
    }
  }
  uint32_t p = *pos + 1, h = 2166136261u, fl = 0;
  StrProps sp_;
  sp_.init();
  while (true) {
    if (p >= n) return false;
    uint32_t c = s[p];
    if (c == '"') break;
    if (c < 0x20) return false;
    if (c == '\\') {
      fl |= JF_ESC;
      if (p + 1 >= n) return false;
      uint32_t e = s[p + 1];
      uint32_t cp;
      switch (e) {
        case '"': cp = '"'; break;   case '\\': cp = '\\'; break; case '/': cp = '/'; break;
        case 'b': cp = 8; break;     case 'f': cp = 12; break;    case 'n': cp = 10; break;
        case 'r': cp = 13; break;    case 't': cp = 9; break;
        case 'u': {
          if (p + 6 > n) return false;
          int a = hexv(s[p + 2]), b = hexv(s[p + 3]), c2 = hexv(s[p + 4]), d = hexv(s[p + 5]);
          if ((a | b | c2 | d) < 0) return false;
          cp = (uint32_t)((a << 12) | (b << 8) | (c2 << 4) | d);
          if (cp >= 0xDC00 && cp <= 0xDFFF) return false;                  // lone low surrogate
          if (cp >= 0xD800 && cp <= 0xDBFF) {
            if (p + 12 > n || s[p + 6] != '\\' || s[p + 7] != 'u') return false;
            int a2 = hexv(s[p + 8]), b2 = hexv(s[p + 9]), c3 = hexv(s[p + 10]), d2 = hexv(s[p + 11]);
            if ((a2 | b2 | c3 | d2) < 0) return false;
            uint32_t lo = (uint32_t)((a2 << 12) | (b2 << 8) | (c3 << 4) | d2);
            if (lo < 0xDC00 || lo > 0xDFFF) return false;
            cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            p += 6;
          }
          p += 4;
          break;
        }
        default: return false;
      }
      p += 2;
      sp_.feed(cp);
      // hash the UTF-8 encoding of cp
      if (cp < 0x80) { h = (h ^ cp) * 16777619u; }
      else if (cp < 0x800) { h = (h ^ (0xC0 | (cp >> 6))) * 16777619u; h = (h ^ (0x80 | (cp & 63))) * 16777619u; }
      else if (cp < 0x10000) { h = (h ^ (0xE0 | (cp >> 12))) * 16777619u; h = (h ^ (0x80 | ((cp >> 6) & 63))) * 16777619u; h = (h ^ (0x80 | (cp & 63))) * 16777619u; }
      else { h = (h ^ (0xF0 | (cp >> 18))) * 16777619u; h = (h ^ (0x80 | ((cp >> 12) & 63))) * 16777619u; h = (h ^ (0x80 | ((cp >> 6) & 63))) * 16777619u; h = (h ^ (0x80 | (cp & 63))) * 16777619u; }
      continue;
    }
    if (c < 0x80) { h = (h ^ c) * 16777619u; sp_.feed(c); ++p; continue; }
    // strict UTF-8
    uint32_t need, mn;
    if (c >= 0xC2 && c <= 0xDF) { need = 1; mn = 0x80; }
    else if (c >= 0xE0 && c <= 0xEF) { need = 2; mn = 0x800; }
    else if (c >= 0xF0 && c <= 0xF4) { need = 3; mn = 0x10000; }
    else return false;
    if (p + need >= n) return false;
    uint32_t cp = c & (0x3F >> need);
    h = (h ^ c) * 16777619u;
    for (uint32_t k = 1; k <= need; ++k) {
      uint32_t cc = s[p + k];
      if ((cc & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (cc & 0x3F);
      h = (h ^ cc) * 16777619u;
    }
    if (cp < mn || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    sp_.feed(cp);
    p += need + 1;
  }
  *pos = p + 1;
  *flags = fl | sp_.flags();
  *hash = h;
  return true;
}

// Iterator over the decoded code points of a (validated) JSON string span.
struct StrIter {
  const uint8_t* p;
  const uint8_t* e;
  CF_HD bool done() const { return p >= e; }
  CF_HD uint32_t next() {
    uint32_t c = *p;
    if (c == '\\') {
      uint32_t x = p[1];
      p += 2;
      switch (x) {
        case 'b': return 8; case 'f': return 12; case 'n': return 10; case 'r': return 13; case 't': return 9;
        case 'u': {
          uint32_t cp = (uint32_t)((hexv(p[0]) << 12) | (hexv(p[1]) << 8) | (hexv(p[2]) << 4) | hexv(p[3]));
          p += 4;
          if (cp >= 0xD800 && cp <= 0xDBFF) {
            uint32_t lo = (uint32_t)((hexv(p[2]) << 12) | (hexv(p[3]) << 8) | (hexv(p[4]) << 4) | hexv(p[5]));
            p += 6;
            cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
          }
          return cp;
        }
        default: return x;   // " \ /
      }
    }
    if (c < 0x80) { ++p; return c; }
    uint32_t need = c >= 0xF0 ? 3u : c >= 0xE0 ? 2u : 1u;
    uint32_t cp = c & (0x3F >> need);
    for (uint32_t k = 1; k <= need; ++k) cp = (cp << 6) | (p[k] & 0x3F);
    p += need + 1;
    return cp;
  }
};

CF_HD bool keys_equal(const uint8_t* s, const JNode& a, const JNode& b) {
  if (!((a.t | b.t) & JF_ESC)) {
    if (a.len != b.len) return false;
    const uint8_t* x = s + a.off;
    const uint8_t* y = s + b.off;
    uint32_t i = 0;
    for (; i + 4 <= a.len; i += 4) {    // independent loads, one branch per four bytes
      const uint32_t d = (uint32_t)(x[i] ^ y[i]) | (uint32_t)(x[i + 1] ^ y[i + 1]) | (uint32_t)(x[i + 2] ^ y[i + 2]) | (uint32_t)(x[i + 3] ^ y[i + 3]);
      if (d) return false;
    }
    for (; i < a.len; ++i) if (x[i] != y[i]) return false;
    return true;
  }
  StrIter ia{s + a.off, s + a.off + a.len}, ib{s + b.off, s + b.off + b.len};
  while (!ia.done() && !ib.done()) if (ia.next() != ib.next()) return false;
  return ia.done() && ib.done();
}

// JSON number grammar from *pos (at '-' or a digit); on success *pos is just past it and *fl holds JF_NEG/FRAC/EXP.
CF_HD bool scan_number(const uint8_t* s, uint32_t n, uint32_t* ppos, uint32_t* pfl) {
  uint32_t pos = *ppos, fl = 0;
  if (s[pos] == '-') { fl |= JF_NEG; ++pos; if (pos >= n) return false; }
  if (s[pos] == '0') ++pos;
  else if (s[pos] >= '1' && s[pos] <= '9') { while (pos < n && s[pos] >= '0' && s[pos] <= '9') ++pos; }
  else return false;
  if (pos < n && s[pos] == '.') {
    fl |= JF_FRAC; ++pos;
    if (pos >= n || s[pos] < '0' || s[pos] > '9') return false;
    while (pos < n && s[pos] >= '0' && s[pos] <= '9') ++pos;
  }
  if (pos < n && (s[pos] == 'e' || s[pos] == 'E')) {
    fl |= JF_EXP; ++pos;
    if (pos < n && (s[pos] == '+' || s[pos] == '-')) ++pos;
    if (pos >= n || s[pos] < '0' || s[pos] > '9') return false;
    while (pos < n && s[pos] >= '0' && s[pos] <= '9') ++pos;
  }
  *ppos = pos; *pfl = fl;
  return true;
}

// Parse `s[0..n)` (a whole JSON document, surrounding whitespace allowed) into nodes[0..cap).
// Token-at-a-time.  (A byte-at-a-time flat state machine was tried to cut warp divergence and was
// slower, so the straightforward form stays.)
// All per-container running state (child count, last child, kind, the key hashes of the open objects)
// lives in thread-local arrays: a read-after-write through the node array in HBM costs an L2 round
// trip per token, local memory stays in L1.  Nodes are written once, when complete.
static const uint32_t KH_CAP = 512;        // key hashes of all currently open objects (an object whose hashes did not fit -> slow dedupe)
CF_HD int json_parse(const uint8_t* s, uint32_t n, JNode* nodes, uint32_t cap, uint32_t* out_count) {
  uint32_t pos = 0, nn = 0;
  uint32_t st_node[MAXD], st_last[MAXD], st_len[MAXD], st_kh[MAXD];
  uint32_t kh[KH_CAP];
  uint32_t khn = 0;                 // used entries of kh
  uint64_t khbad = 0;               // bit d: the object at depth d has keys whose hashes did not fit
  uint64_t objbits = 0;             // bit d: the container at depth d is an object
  int sp = 0;
  bool member = false;              // the value being parsed belongs to an object member
  uint32_t member_hash = 0;
  enum { M_VALUE, M_KEY, M_AFTER } mode = M_VALUE;
  while (pos < n && j_ws(s[pos])) ++pos;
  while (true) {
    if (mode == M_VALUE || mode == M_KEY) {
      if (pos >= n) return PARSE_ERROR;
      if (nn + 2 > cap) return PARSE_UNSUPPORTED;
      uint32_t c = s[pos];
      uint32_t idx = nn;
      if (mode == M_KEY) {
        if (c != '"') return PARSE_ERROR;
        uint32_t fl, h, p0 = pos;
        if (!parse_string(s, n, &pos, &fl, &h)) return PARSE_ERROR;
        nodes[nn++] = JNode{J_KEY | fl, p0 + 1, pos - p0 - 2, 0};
        if (st_last[sp - 1]) nodes[st_last[sp - 1]].next = idx; else nodes[st_node[sp - 1]].off = idx;
        st_last[sp - 1] = idx;
        st_len[sp - 1]++;
        if (khn < KH_CAP) kh[khn++] = h; else khbad |= 1ull << (sp - 1);
        while (pos < n && j_ws(s[pos])) ++pos;
        if (pos >= n || s[pos] != ':') return PARSE_ERROR;
        ++pos;
        while (pos < n && j_ws(s[pos])) ++pos;
        member = true;          // the value node follows immediately and carries the key hash in .next
        member_hash = h;
        mode = M_VALUE;
        continue;
      }
      const uint32_t keep_next = member ? member_hash : 0;
      if (!member && sp > 0) {   // array element: chain
        if (st_last[sp - 1]) nodes[st_last[sp - 1]].next = idx; else nodes[st_node[sp - 1]].off = idx;
        st_last[sp - 1] = idx;
        st_len[sp - 1]++;
      }
      member = false;
      if (c == '{' || c == '[') {
        if (sp >= MAXD) return PARSE_UNSUPPORTED;
        nodes[nn++] = JNode{c == '{' ? (uint32_t)J_OBJ : (uint32_t)J_ARR, 0, 0, keep_next};
        st_node[sp] = idx; st_last[sp] = 0; st_len[sp] = 0; st_kh[sp] = khn;
        if (c == '{') objbits |= 1ull << sp; else objbits &= ~(1ull << sp);
        ++sp;
        ++pos;
        while (pos < n && j_ws(s[pos])) ++pos;
        if (pos < n && s[pos] == (c == '{' ? '}' : ']')) { ++pos; --sp; mode = M_AFTER; }
        else mode = (c == '{') ? M_KEY : M_VALUE;
        continue;
      }
      if (c == '"') {
        uint32_t fl, h, p0 = pos;
        if (!parse_string(s, n, &pos, &fl, &h)) return PARSE_ERROR;
        nodes[nn++] = JNode{J_STR | fl, p0 + 1, pos - p0 - 2, keep_next};
      } else if (c == '-' || (c >= '0' && c <= '9')) {
        uint32_t p0 = pos, fl = 0;
        if (!scan_number(s, n, &pos, &fl)) return PARSE_ERROR;
        nodes[nn++] = JNode{J_NUM | fl, p0, pos - p0, keep_next};
      } else if (c == 't' && pos + 4 <= n && s[pos + 1] == 'r' && s[pos + 2] == 'u' && s[pos + 3] == 'e') {
        nodes[nn++] = JNode{J_TRUE, pos, 4, keep_next}; pos += 4;
      } else if (c == 'f' && pos + 5 <= n && s[pos + 1] == 'a' && s[pos + 2] == 'l' && s[pos + 3] == 's' && s[pos + 4] == 'e') {
        nodes[nn++] = JNode{J_FALSE, pos, 5, keep_next}; pos += 5;
      } else if (c == 'n' && pos + 4 <= n && s[pos + 1] == 'u' && s[pos + 2] == 'l' && s[pos + 3] == 'l') {
        nodes[nn++] = JNode{J_NULL, pos, 4, keep_next}; pos += 4;
      } else return PARSE_ERROR;
      mode = M_AFTER;
      continue;
    }
    // M_AFTER: a value has just been completed
    while (pos < n && j_ws(s[pos])) ++pos;
    if (sp == 0) {
      if (pos != n) return PARSE_ERROR;
      *out_count = nn;
      return PARSE_OK;
    }
    if (pos >= n) return PARSE_ERROR;
    const bool is_obj = (objbits >> (sp - 1)) & 1;
    uint32_t c = s[pos];
    if (c == ',') {
      ++pos;
      while (pos < n && j_ws(s[pos])) ++pos;
      mode = is_obj ? M_KEY : M_VALUE;
      continue;
    }
    if (c != (is_obj ? '}' : ']')) return PARSE_ERROR;
    ++pos;
    --sp;
    const uint32_t cidx = st_node[sp];
    uint32_t clen = st_len[sp];
    if (is_obj) {
      // duplicate keys: the last value wins, the first position stays (Python dict / orjson).
      // Cheap screen on the hashes held in local memory; the node walk only runs when two hashes collide.
      const uint32_t kb = st_kh[sp];
      bool maybe_dup = (khbad >> sp) & 1;
      khbad &= ~(1ull << sp);
      if (!maybe_dup)
        for (uint32_t i = kb + 1; i < khn && !maybe_dup; ++i)
          for (uint32_t j = kb; j < i; ++j) if (kh[j] == kh[i]) { maybe_dup = true; break; }
      khn = kb;
      if (maybe_dup && clen > 1) {
        const uint32_t first = nodes[cidx].off;   // stored when the first key arrived
        uint32_t prev = first;
        for (uint32_t k = nodes[prev].next; k;) {
          uint32_t nxt = nodes[k].next;
          bool dup = false;
          for (uint32_t i = first; i != k; i = nodes[i].next)
            if (nodes[i + 1].next == nodes[k + 1].next && keys_equal(s, nodes[i], nodes[k])) {
              uint32_t hsh = nodes[i + 1].next;
              nodes[i + 1] = nodes[k + 1];
              nodes[i + 1].next = hsh;
              dup = true;
              break;
            }
          if (dup) { nodes[prev].next = nxt; clen--; }
          else prev = k;
          k = nxt;
        }
      }
    }
    nodes[cidx].len = clen;
    mode = M_AFTER;
  }
}

// ------------------------------------------------------------------------------------------------
// Exact decimal <-> binary64 helpers (big integers; only used when the cheap text path cannot
// decide: more than 15 significant digits, exponents, integers beyond 64 bits)
// ------------------------------------------------------------------------------------------------
static const int BIGN = 100;   // 3200 bits
struct Big {
  uint32_t n;
  uint32_t w[BIGN];
  CF_HD void set(uint32_t v) { n = v ? 1 : 0; w[0] = v; }
  CF_HD bool zero() const { return n == 0; }
  CF_HD bool mul_add(uint32_t m, uint32_t a) {   // this = this*m + a; false on overflow
    uint64_t c = a;
    for (uint32_t i = 0; i < n; ++i) { uint64_t t = (uint64_t)w[i] * m + c; w[i] = (uint32_t)t; c = t >> 32; }
    if (c) { if (n >= BIGN) return false; w[n++] = (uint32_t)c; }
    return true;
  }
  CF_HD uint32_t div_small(uint32_t d) {         // this /= d; returns remainder
    uint64_t r = 0;
    for (uint32_t i = n; i-- > 0;) { uint64_t t = (r << 32) | w[i]; w[i] = (uint32_t)(t / d); r = t % d; }
    while (n && w[n - 1] == 0) --n;
    return (uint32_t)r;
  }
  CF_HD bool shl(uint32_t bits) {
    uint32_t ws = bits >> 5, bs = bits & 31;
    if (n == 0) return true;
    const uint32_t carry_word = bs && (w[n - 1] >> (32 - bs)) ? 1u : 0u;   // the top word spills into a new one
    if (n + ws + carry_word > BIGN) return false;                          // exact: a result that fits is never refused
    for (uint32_t i = n; i-- > 0;) w[i + ws] = w[i];
    for (uint32_t i = 0; i < ws; ++i) w[i] = 0;
    n += ws;
    if (bs) {
      uint32_t c = 0;
      for (uint32_t i = ws; i < n; ++i) { uint32_t t = w[i]; w[i] = (t << bs) | c; c = t >> (32 - bs); }
      if (c) w[n++] = c;
    }
    return true;
  }
  CF_HD uint32_t bitlen() const {
    if (!n) return 0;
    uint32_t t = w[n - 1], b = 0;
    while (t) { ++b; t >>= 1; }
    return (n - 1) * 32 + b;
  }
  CF_HD uint32_t bit(uint32_t i) const { return (i >> 5) < n ? (w[i >> 5] >> (i & 31)) & 1u : 0u; }
  CF_HD bool any_below(uint32_t i) const {       // any set bit strictly below position i
    uint32_t ws = i >> 5;
    for (uint32_t k = 0; k < ws && k < n; ++k) if (w[k]) return true;
    if (ws < n && (i & 31)) return (w[ws] & ((1u << (i & 31)) - 1)) != 0;
    return false;
  }
};

// A binary64 as sign, 53-bit integer mantissa m (0 or 2^52 <= m < 2^53 for normals) and exponent e: m * 2^e.
struct Dbl { bool neg; bool inf; uint64_t m; int e; };

// Correctly rounded (nearest-even) conversion of the decimal text to binary64.  Returns false when
// the text needs more capacity than the big-integer workspace offers.
CF_HD bool dec_to_double(const uint8_t* t, uint32_t len, Dbl* out, Big* X) {
  uint32_t p = 0;
  out->neg = false; out->inf = false; out->m = 0; out->e = 0;
  if (p < len && t[p] == '-') { out->neg = true; ++p; }
  X->set(0);
  long long e10 = 0;
  bool seen_dot = false, any = false;
  for (; p < len; ++p) {
    uint32_t c = t[p];
    if (c == '.') { seen_dot = true; continue; }
    if (c == 'e' || c == 'E') break;
    if (!any && c == '0') { if (seen_dot) --e10; continue; }   // leading zeros carry no information
    any = true;
    if (!X->mul_add(10, c - '0')) return false;
    if (seen_dot) --e10;
  }
  if (p < len) {   // exponent
    ++p;
    bool en = false;
    if (p < len && (t[p] == '+' || t[p] == '-')) { en = t[p] == '-'; ++p; }
    long long ex = 0;
    for (; p < len; ++p) { if (ex < 100000) ex = ex * 10 + (t[p] - '0'); }
    e10 += en ? -ex : ex;
  }
  if (X->zero()) return true;                                   // +-0
  uint32_t nd10 = (uint32_t)((X->bitlen() * 1233) >> 12) + 1;   // ~ decimal digits of X
  if (e10 + (long long)nd10 > 330) { out->inf = true; return true; }
  if (e10 + (long long)nd10 < -345) return true;                // underflows to zero
  int bin_e = 0;        // value = X * 2^bin_e (+ sticky)
  bool sticky = false;
  if (e10 >= 0) {
    for (long long i = 0; i < e10; ++i) if (!X->mul_add(10, 0)) return false;
  } else {
    long long q = -e10;
    uint32_t want = 64 + (uint32_t)((q * 3402) >> 10) + 2;      // bits so that the quotient keeps >= 64 bits
    uint32_t have = X->bitlen();
    uint32_t s = want > have ? want - have : 0;
    if (!X->shl(s)) return false;
    bin_e = -(int)s;
    while (q >= 9) { if (X->div_small(1000000000u)) sticky = true; q -= 9; }
    uint32_t d = 1;
    for (; q > 0; --q) d *= 10;
    if (d > 1 && X->div_small(d)) sticky = true;
  }
  // round X * 2^bin_e to 53 bits (or fewer for subnormals)
  int L = (int)X->bitlen();
  int drop = L - 53;
  int e = bin_e + drop;                     // exponent of the kept integer mantissa
  if (e < -1074) { drop += (-1074 - e); e = -1074; }
  uint64_t m = 0;
  if (drop <= 0) {
    for (int i = L - 1; i >= 0; --i) m = (m << 1) | X->bit((uint32_t)i);
    m <<= (uint32_t)(-drop);
  } else {
    if (drop > L) { m = 0; sticky = sticky || !X->zero(); }
    else for (int i = L - 1; i >= drop; --i) m = (m << 1) | X->bit((uint32_t)i);
    bool half = drop <= L && X->bit((uint32_t)(drop - 1));
    bool rest = sticky || X->any_below((uint32_t)(drop - 1));
    if (drop > L) { half = false; }
    if (half && (rest || (m & 1))) ++m;
    if (m == (1ull << 53)) { m >>= 1; ++e; }
  }
  if (m == 0) return true;
  // normalise: value = m * 2^e ; overflow check
  int top = 0; { uint64_t tt = m; while (tt) { ++top; tt >>= 1; } }
  if (e + top > 1024) { out->inf = true; return true; }
  out->m = m;
  out->e = e;
  return true;
}

// Decimal digits of a big integer, most significant first, into buf; returns count (0 for zero).
CF_HD uint32_t big_to_digits(Big* X, uint8_t* buf, uint32_t cap) {
  // generate 9 digits at a time from the least significant end, then reverse
  uint32_t n = 0;
  while (!X->zero()) {
    uint32_t r = X->div_small(1000000000u);
    for (int k = 0; k < 9; ++k) {
      if (n >= cap) return 0xFFFFFFFFu;
      buf[n++] = (uint8_t)('0' + r % 10);
      r /= 10;
      if (X->zero() && r == 0) break;
    }
  }
  for (uint32_t i = 0; i < n / 2; ++i) { uint8_t t = buf[i]; buf[i] = buf[n - 1 - i]; buf[n - 1 - i] = t; }
  return n;
}

// ------------------------------------------------------------------------------------------------
// TOON emitter
// ------------------------------------------------------------------------------------------------
enum : int {
  TS_CONVERTED = 0, TS_NOT_SMALLER = 1, TS_NOT_JSON = 2, TS_VALUE_ERROR = 3 /* control character */,
  TS_ATTR_ERROR = 4 /* the reference's unchecked .keys() */, TS_UNSUPPORTED = 6
};

struct Out {
  uint8_t* p;
  uint32_t n, cap;
  bool over;
  CF_HD void put(uint32_t c) { if (n < cap) p[n++] = (uint8_t)c; else over = true; }
  // copy a span of source bytes; the in-capacity case is unrolled so that a lone GPU thread has
  // several independent loads in flight
  CF_HD void put_span(const uint8_t* b, uint32_t len) {
    if (n + len <= cap) {
      uint8_t* d = p + n;
      uint32_t i = 0;
      for (; i + 4 <= len; i += 4) {
        const uint8_t a0 = b[i], a1 = b[i + 1], a2 = b[i + 2], a3 = b[i + 3];
        d[i] = a0; d[i + 1] = a1; d[i + 2] = a2; d[i + 3] = a3;
      }
      for (; i < len; ++i) d[i] = b[i];
      n += len;
    } else {
      for (uint32_t i = 0; i < len; ++i) put(b[i]);
    }
  }
  CF_HD void puts(const char* z) { while (*z) put((uint8_t)*z++); }
  CF_HD void spaces(uint32_t k) { for (uint32_t i = 0; i < k; ++i) put(' '); }
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

struct Ctx {
  const uint8_t* s;
  const JNode* nodes;
  Out out;
  int err;          // 0 or TS_VALUE_ERROR / TS_ATTR_ERROR / TS_UNSUPPORTED
  bool started;     // a line has been opened already (next line needs a '\n' first)
  bool stop_on_over; // give up as soon as the output cannot be smaller (errors then go unreported: fine when
                    // the caller treats encode errors and "not smaller" alike, i.e. skip_on_error=True)
  Big* big;         // workspace for the exact number path
  uint8_t* digits;  // decimal digit workspace
  uint32_t digits_cap;
};

CF_HD void newline(Ctx& c, uint32_t pre) {
  if (c.started) c.out.put('\n');
  c.started = true;
  c.out.spaces(pre);
}

CF_HD bool is_simple(uint32_t t) { uint32_t k = t & J_TYPE; return k != J_ARR && k != J_OBJ; }

// string value -> TOON (quote only when the reference's _needs_quotes says so; the predicate was
// evaluated by the parser and sits in the node flags)
CF_HD void emit_string(Ctx& c, const JNode& nd, bool force_quote) {
  const uint8_t* b = c.s + nd.off;
  const uint8_t* e = b + nd.len;
  const bool q = force_quote || (nd.t & JF_Q);
  if (q && (nd.t & JF_CTRLERR)) { c.err = TS_VALUE_ERROR; return; }
  if (!(nd.t & JF_ESC)) {
    // no escapes in the source: the decoded text IS the source bytes, and nothing in it needs a TOON
    // escape either (a raw '"' or '\' cannot occur unescaped in JSON)
    if (q) c.out.put('"');
    c.out.put_span(b, nd.len);
    if (q) c.out.put('"');
    return;
  }
  StrIter it{b, e};
  if (!q) { while (!it.done()) c.out.put_cp(it.next()); return; }
  c.out.put('"');
  while (!it.done()) {
    uint32_t cp = it.next();
    if (cp == '\\') { c.out.put('\\'); c.out.put('\\'); }
    else if (cp == '"') { c.out.put('\\'); c.out.put('"'); }
    else if (cp == '\n') { c.out.put('\\'); c.out.put('n'); }
    else if (cp == '\r') { c.out.put('\\'); c.out.put('r'); }
    else if (cp == '\t') { c.out.put('\\'); c.out.put('t'); }
    else c.out.put_cp(cp);
  }
  c.out.put('"');
}

// object key: unquoted iff ^[A-Za-z_][A-Za-z0-9_.]*$ (where `$` admits one final "\n") and not reserved.
// Such a key carries its newline RAW into the output.  The reference builds nested text as strings and re-splits them on "\n" at
// every enclosing level (toon.py:369, :421, :432, :559), so whatever follows the newline is a line of its own and receives the
// prefixes of the enclosing levels — `pre` spaces — but not the indentation the emitting level wrote in front of the key.
CF_HD void emit_key(Ctx& c, const JNode& k, uint32_t pre) {
  const uint8_t* b = c.s + k.off;
  const uint8_t* e = b + k.len;
  if (k.t & JF_KEYOK) {
    if (!(k.t & JF_ESC)) { c.out.put_span(b, k.len); return; }
    StrIter it{b, e};
    while (!it.done()) { const uint32_t cp = it.next(); c.out.put_cp(cp); if (cp == '\n') c.out.spaces(pre); }
    return;
  }
  emit_string(c, k, true);
}

// The header "[n]{k1,k2}:" of a columnar array.  Its fields are never quoted (toon.py:501), so they may carry raw newlines anywhere.
// What follows one is, as above, a line of its own: `hdr_pre` spaces in front — or, when the array is the first field of a list item
// (toon.py:405-413 splits the columnar text and treats every line but the first as "a row"), the line is stripped on both sides
// (str.strip) and indented like the rows (`row_pre`).
struct HeaderSink {
  Ctx& c;
  uint32_t hdr_pre, row_pre;
  bool strip;
  uint32_t piece, ws_tail;
  bool at_start;
  CF_HD void cp(uint32_t x) {
    if (x == '\n') {
      if (strip) {
        if (piece && !c.out.over) c.out.n -= ws_tail;             // rstrip of the line that ends here
        c.out.put('\n'); c.out.spaces(row_pre);
      } else { c.out.put('\n'); c.out.spaces(hdr_pre); }
      ++piece; ws_tail = 0; at_start = true;
      return;
    }
    if (strip && piece) {
      if (is_pyspace(x)) {
        if (at_start) return;                                      // lstrip
        const uint32_t before = c.out.n;
        c.out.put_cp(x);
        ws_tail += c.out.n - before;
        return;
      }
      at_start = false; ws_tail = 0;
    }
    c.out.put_cp(x);
  }
  CF_HD void key(const JNode& k) {
    const uint8_t* b = c.s + k.off;
    if (!(k.t & JF_ESC)) {
      if (!(strip && piece)) { c.out.put_span(b, k.len); return; }  // no escapes: no raw newline, no whitespace handling needed on line 0
      StrIter raw{b, b + k.len};                                    // (without escapes StrIter is a plain UTF-8 decoder)
      while (!raw.done()) cp(raw.next());
      return;
    }
    StrIter it{b, b + k.len};
    while (!it.done()) cp(it.next());
  }
};

// Python's float formatting as used by toon._encode_float, from the exact binary value.
CF_HD void emit_double(Ctx& c, const Dbl& d) {
  if (d.m == 0) { c.out.put('0'); return; }                       // +-0 -> "0"
  // is it an integer?
  bool integral = d.e >= 0;
  if (!integral && -d.e < 64) integral = (d.m & ((1ull << (-d.e)) - 1)) == 0;
  Big* X = c.big;
  if (integral) {
    uint64_t m = d.e >= 0 ? d.m : d.m >> (-d.e);
    X->n = 0; X->w[0] = (uint32_t)m; X->w[1] = (uint32_t)(m >> 32);
    X->n = X->w[1] ? 2 : (X->w[0] ? 1 : 0);
    if (d.e > 0 && !X->shl((uint32_t)d.e)) { c.err = TS_UNSUPPORTED; return; }
    uint32_t nd = big_to_digits(X, c.digits, c.digits_cap);
    if (nd == 0xFFFFFFFFu) { c.err = TS_UNSUPPORTED; return; }
    if (d.neg) c.out.put('-');
    for (uint32_t i = 0; i < nd; ++i) c.out.put(c.digits[i]);
    return;
  }
  // value = m / 2^k = (m * 5^k) / 10^k, k = -e > 0: exact decimal expansion with k fractional digits
  uint32_t k = (uint32_t)(-d.e);
  X->n = 0; X->w[0] = (uint32_t)d.m; X->w[1] = (uint32_t)(d.m >> 32);
  X->n = X->w[1] ? 2 : 1;
  for (uint32_t i = 0; i < k;) {
    uint32_t step = k - i >= 13 ? 13 : k - i;
    uint32_t mul = 1;
    for (uint32_t j = 0; j < step; ++j) mul *= 5;
    if (!X->mul_add(mul, 0)) { c.err = TS_UNSUPPORTED; return; }
    i += step;
  }
  uint32_t nd = big_to_digits(X, c.digits, c.digits_cap - 2);
  if (nd == 0xFFFFFFFFu) { c.err = TS_UNSUPPORTED; return; }
  uint8_t* D = c.digits;                       // N = D[0..nd), value = N * 10^-k  (k >= 1)
  int exp10 = (int)nd - (int)k - 1;            // decimal exponent of the leading digit
  // ---- "%.15g": 15 significant digits, round-half-even on the exact value
  uint8_t sig[18];
  uint32_t ns = nd < 15 ? nd : 15;
  for (uint32_t i = 0; i < ns; ++i) sig[i] = D[i];
  int e15 = exp10;
  if (nd > 15) {
    bool up = false;
    if (D[15] > '5') up = true;
    else if (D[15] == '5') {
      bool rest = false;
      for (uint32_t i = 16; i < nd; ++i) if (D[i] != '0') { rest = true; break; }
      up = rest || ((D[14] - '0') & 1);
    }
    if (up) {
      int i = 14;
      while (i >= 0 && sig[i] == '9') { sig[i] = '0'; --i; }
      if (i >= 0) sig[i]++; else { for (int j = 14; j > 0; --j) sig[j] = sig[j - 1]; sig[0] = '1'; ++e15; }
    }
  }
  if (e15 >= -4 && e15 < 15) {
    // fixed notation; %g strips trailing zeros
    uint32_t nsig = ns;
    while (nsig > 1 && sig[nsig - 1] == '0') --nsig;
    if (d.neg) c.out.put('-');
    if (e15 >= 0) {
      for (int i = 0; i <= e15; ++i) c.out.put(i < (int)nsig ? sig[i] : '0');
      if ((int)nsig > e15 + 1) { c.out.put('.'); for (uint32_t i = (uint32_t)e15 + 1; i < nsig; ++i) c.out.put(sig[i]); }
    } else {
      c.out.put('0'); c.out.put('.');
      for (int i = 0; i < -e15 - 1; ++i) c.out.put('0');
      for (uint32_t i = 0; i < nsig; ++i) c.out.put(sig[i]);
    }
    return;
  }
  // ---- %g would use an exponent: the reference falls back to "%.15f", strips zeros, then a final '.'
  int ni = (int)nd - (int)k;                   // digits before the decimal point (<= 0: the integer part is 0)
  // fractional digit j (0-based) is D[ni + j] when ni + j >= 0, else '0'
  uint8_t f[16];
  for (int j = 0; j < 15; ++j) { int idx = ni + j; f[j] = (j < (int)k && idx >= 0) ? D[idx] : (uint8_t)'0'; }
  bool carry = false;
  if (k > 15) {
    int idx16 = ni + 15;
    uint8_t d16 = idx16 >= 0 ? D[idx16] : (uint8_t)'0';
    bool up = false;
    if (d16 > '5') up = true;
    else if (d16 == '5') {
      bool rest = false;
      for (int i = idx16 + 1; i < (int)nd; ++i) if (i >= 0 && D[i] != '0') { rest = true; break; }
      up = rest || ((f[14] - '0') & 1);
    }
    if (up) {
      int i = 14;
      while (i >= 0 && f[i] == '9') { f[i] = '0'; --i; }
      if (i >= 0) f[i]++; else carry = true;
    }
  }

  bool int_grew = false;
  if (carry) {                                   // propagate into the integer digits D[0..ni)
    int i = ni - 1;
    while (i >= 0 && D[i] == '9') { D[i] = '0'; --i; }
    if (i >= 0) D[i]++; else int_grew = true;
  }
  int nf = 15;
  while (nf > 0 && f[nf - 1] == '0') --nf;
  if (d.neg) c.out.put('-');
  if (int_grew) c.out.put('1');
  if (ni > 0) { for (int i = 0; i < ni; ++i) c.out.put(D[i]); }
  else if (!int_grew) c.out.put('0');
  if (nf) { c.out.put('.'); for (int i = 0; i < nf; ++i) c.out.put(f[i]); }
}

CF_HD void emit_number(Ctx& c, const JNode& nd) {
  const uint8_t* t = c.s + nd.off;
  uint32_t len = nd.len;
  bool neg = (nd.t & JF_NEG) != 0;
  const uint8_t* dg = t + (neg ? 1 : 0);
  uint32_t dl = len - (neg ? 1 : 0);
  if (!(nd.t & (JF_FRAC | JF_EXP))) {
    // integer literal: Python int when it fits i64 / u64 (orjson), else a float
    bool fits = dl < 19;
    if (!fits && dl <= 20) {
      const char* lim = neg ? "9223372036854775808" : "18446744073709551615";
      uint32_t ll = neg ? 19 : 20;
      if (dl < ll) fits = true;
      else if (dl == ll) { fits = true; for (uint32_t i = 0; i < ll; ++i) { if (dg[i] < (uint8_t)lim[i]) break; if (dg[i] > (uint8_t)lim[i]) { fits = false; break; } } }
    }
    if (fits) {
      if (dl == 1 && dg[0] == '0') { c.out.put('0'); return; }     // "-0" -> int 0
      c.out.put_span(t, len);
      return;
    }
  } else if (!(nd.t & JF_EXP)) {
    // cheap exact path: [-]INT.FRAC with at most 15 significant digits — binary64 round-trips such
    // decimals, so "%.15g" / str(int(x)) reproduce the text digits and no arithmetic is needed
    uint32_t dot = 0;
    while (dg[dot] != '.') ++dot;
    uint32_t fe = dl;
    while (fe > dot + 1 && dg[fe - 1] == '0') --fe;        // FRAC without trailing zeros
    const uint32_t nfrac = fe - dot - 1;
    const bool int_zero = (dot == 1 && dg[0] == '0');
    uint32_t lead_fz = 0;
    if (int_zero) while (lead_fz < nfrac && dg[dot + 1 + lead_fz] == '0') ++lead_fz;
    const uint32_t sigd = int_zero ? nfrac - lead_fz : dot + nfrac;
    const bool tiny_long = int_zero && lead_fz >= 4 && nfrac > 15;   // "%.15f" would have to round
    if (sigd <= 15 && !tiny_long) {
      if (nfrac == 0) {                                    // integral float -> str(int(x)); +-0.0 -> "0"
        if (int_zero) { c.out.put('0'); return; }
        if (neg) c.out.put('-');
        c.out.put_span(dg, dot);
        return;
      }
      if (neg) c.out.put('-');
      c.out.put_span(dg, dot + 1 + nfrac);
      return;
    }
  }
  // exact path
  Dbl d;
  if (!dec_to_double(t, len, &d, c.big)) { c.err = TS_UNSUPPORTED; return; }
  if (d.inf) { c.err = TS_NOT_JSON; return; }   // yyjson/orjson reject numbers that overflow to infinity
  emit_double(c, d);
}

CF_HD void emit_prim(Ctx& c, uint32_t idx) {
  const JNode& nd = c.nodes[idx];
  switch (nd.t & J_TYPE) {
    case J_NULL: c.out.puts("null"); break;
    case J_TRUE: c.out.puts("true"); break;
    case J_FALSE: c.out.puts("false"); break;
    case J_NUM: emit_number(c, nd); break;
    case J_STR: emit_string(c, nd, false); break;
    default: break;
  }
}

// find the value node of the member of object `obj` whose key equals key node `k` (0 if absent)
CF_HD uint32_t find_member(const Ctx& c, uint32_t obj, uint32_t k) {
  uint32_t h = c.nodes[k + 1].next;
  for (uint32_t m = c.nodes[obj].off; m; m = c.nodes[m].next)
    if (c.nodes[m + 1].next == h && keys_equal(c.s, c.nodes[m], c.nodes[k])) return m + 1;
  return 0;
}

// same, trying the member at `*cursor` first (rows of a table almost always repeat the key order)
CF_HD uint32_t find_member_hint(const Ctx& c, uint32_t obj, uint32_t k, uint32_t* cursor) {
  const uint32_t m = *cursor;
  if (m && c.nodes[m + 1].next == c.nodes[k + 1].next && keys_equal(c.s, c.nodes[m], c.nodes[k])) { *cursor = c.nodes[m].next; return m + 1; }
  return find_member(c, obj, k);
}

enum : int { COL_YES = 1, COL_YES_ALIGNED = 2, COL_NO = 0, COL_CRASH = -1 };
// toon.py:456-511 called on `arr` (non-empty).  COL_YES_ALIGNED: additionally every row lists the keys in
// the first row's order, so the emitter can walk the members without looking anything up.
// Evaluation order matters for parity: a non-dict row raises only if no earlier row already returned None.
CF_HD int columnar_check(const Ctx& c, uint32_t arr) {
  const JNode* N = c.nodes;
  const uint32_t first = N[arr].off;
  const JNode f = N[first];
  if ((f.t & J_TYPE) != J_OBJ) return COL_CRASH;
  if (f.len == 0) return COL_NO;
  bool aligned = true, simple = true;
  for (uint32_t k = f.off; k; k = N[k].next) if (!is_simple(N[k + 1].t)) simple = false;
  for (uint32_t x = f.next; x; ) {
    const JNode r = N[x];
    if ((r.t & J_TYPE) != J_OBJ) return COL_CRASH;
    if (r.len != f.len) return COL_NO;
    uint32_t cur = r.off;
    for (uint32_t k = f.off; k; k = N[k].next) {
      const uint32_t before = cur;
      const uint32_t v = find_member_hint(c, x, k, &cur);
      if (!v) return COL_NO;
      if (v != before + 1) aligned = false;
      if (!is_simple(N[v].t)) simple = false;
    }
    x = r.next;
  }
  if (!simple) return COL_NO;
  return aligned ? COL_YES_ALIGNED : COL_YES;
}

// "[n]{k1,k2}:" then one row per element at `row_pre` spaces
CF_HD void emit_columnar(Ctx& c, uint32_t arr, uint32_t row_pre, bool aligned, uint32_t hdr_pre, bool strip) {
  const JNode* N = c.nodes;
  uint32_t first = N[arr].off;
  c.out.put('['); c.out.put_uint(N[arr].len); c.out.put(']'); c.out.put('{');
  HeaderSink hs{c, hdr_pre, row_pre, strip, 0, 0, false};
  bool f0 = true;
  for (uint32_t k = N[first].off; k; k = N[k].next) { if (!f0) hs.cp(','); f0 = false; hs.key(N[k]); }
  hs.cp('}'); hs.cp(':');
  for (uint32_t x = first; x && !c.err && !(c.out.over && c.stop_on_over); x = N[x].next) {
    newline(c, row_pre);
    bool f1 = true;
    if (aligned) {
      for (uint32_t m = N[x].off; m; m = N[m].next) {
        if (!f1) c.out.put(',');
        f1 = false;
        emit_prim(c, m + 1);
      }
      continue;
    }
    uint32_t cur = N[x].off;
    for (uint32_t k = N[first].off; k; k = N[k].next) {
      if (!f1) c.out.put(',');
      f1 = false;
      emit_prim(c, find_member_hint(c, x, k, &cur));
    }
  }
}

struct Frame { uint32_t kind, node, cur, pre, indent, i; };
enum : uint32_t { FR_OBJ = 0, FR_ARR_ITEMS = 1, FR_LIST_ITEM = 2 };

// Emit an array whose line start (indentation + optional key prefix) is already written.
// Returns true when the array pushed a frame for its items (complex form).
CF_HD bool begin_array(Ctx& c, uint32_t arr, uint32_t pre, uint32_t indent, Frame* st, int* sp) {
  const JNode* N = c.nodes;
  uint32_t n = N[arr].len;
  if (n == 0) { c.out.puts("[0]:"); return false; }
  bool all_obj = true, all_simple = true;
  for (uint32_t x = N[arr].off; x; x = N[x].next) {
    uint32_t k = N[x].t & J_TYPE;
    if (k != J_OBJ) all_obj = false;
    if (k == J_OBJ || k == J_ARR) all_simple = false;
  }
  if (all_obj) {
    const int cc = columnar_check(c, arr);
    if (cc >= COL_YES) { emit_columnar(c, arr, pre + 2, cc == COL_YES_ALIGNED, pre, false); return false; }
  }
  c.out.put('['); c.out.put_uint(n); c.out.put(']'); c.out.put(':');
  if (all_simple) {
    c.out.put(' ');
    bool f0 = true;
    for (uint32_t x = N[arr].off; x; x = N[x].next) { if (!f0) c.out.put(','); f0 = false; emit_prim(c, x); }
    return false;
  }
  if (*sp >= MAXD) { c.err = TS_UNSUPPORTED; return false; }
  st[(*sp)++] = Frame{FR_ARR_ITEMS, arr, N[arr].off, pre, indent, 0};
  return true;
}

CF_HD void toon_emit(Ctx& c, uint32_t root) {
  const JNode* N = c.nodes;
  Frame st[MAXD];
  int sp = 0;
  uint32_t rk = N[root].t & J_TYPE;
  if (rk != J_ARR && rk != J_OBJ) { emit_prim(c, root); return; }
  if (rk == J_ARR) { c.started = true; begin_array(c, root, 0, 0, st, &sp); }
  else { if (N[root].len == 0) return; st[sp++] = Frame{FR_OBJ, root, N[root].off, 0, 0, 0}; }
  while (sp > 0 && !c.err && !(c.out.over && c.stop_on_over)) {
    Frame& f = st[sp - 1];
    if (f.cur == 0) { --sp; continue; }
    if (f.kind == FR_OBJ) {                                   // toon.py:514-565
      uint32_t k = f.cur, v = k + 1;
      f.cur = N[k].next;
      uint32_t pre = f.pre, indent = f.indent;
      newline(c, pre);
      emit_key(c, N[k], pre);
      uint32_t vt = N[v].t & J_TYPE;
      if (vt == J_ARR) begin_array(c, v, pre, indent, st, &sp);
      else if (vt == J_OBJ) {
        c.out.put(':');
        if (N[v].len) { if (sp >= MAXD) { c.err = TS_UNSUPPORTED; break; } st[sp++] = Frame{FR_OBJ, v, N[v].off, pre + 2, indent + 1, 0}; }
      } else { c.out.put(':'); c.out.put(' '); emit_prim(c, v); }
    } else if (f.kind == FR_ARR_ITEMS) {                      // toon.py:349-375
      uint32_t x = f.cur;
      f.cur = N[x].next;
      uint32_t pre = f.pre, indent = f.indent, ci = 2 * (indent + 1);
      uint32_t xt = N[x].t & J_TYPE;
      if (xt == J_OBJ) {
        if (N[x].len == 0) { newline(c, pre + ci); c.out.put('-'); }
        else { if (sp >= MAXD) { c.err = TS_UNSUPPORTED; break; } st[sp++] = Frame{FR_LIST_ITEM, x, N[x].off, pre, indent + 1, 0}; }
      } else if (xt == J_ARR) {
        newline(c, pre + ci); c.out.put('-'); c.out.put(' ');
        begin_array(c, x, pre + ci + 2, indent + 2, st, &sp);
      } else { newline(c, pre + ci); c.out.put('-'); c.out.put(' '); emit_prim(c, x); }
    } else {                                                  // FR_LIST_ITEM  toon.py:378-441
      uint32_t k = f.cur, v = k + 1, i = f.i;
      f.cur = N[k].next;
      f.i = i + 1;
      uint32_t pre = f.pre, indent = f.indent, ind = 2 * indent, fi = 2 * (indent + 1);
      newline(c, pre + (i == 0 ? ind : fi));
      if (i == 0) { c.out.put('-'); c.out.put(' '); }
      emit_key(c, N[k], pre);
      if (c.err) break;                                         // the key is encoded first (toon.py:396): its ValueError precedes the .keys() crash below
      uint32_t vt = N[v].t & J_TYPE;
      if (vt == J_ARR && N[v].len) {
        if (i == 0) {
          int cc = columnar_check(c, v);
          if (cc == COL_CRASH) { c.err = TS_ATTR_ERROR; break; }
          if (cc >= COL_YES) { emit_columnar(c, v, pre + fi + 2, cc == COL_YES_ALIGNED, pre, true); continue; }
        }
        c.out.put(':');
        newline(c, pre + fi + 2);
        begin_array(c, v, pre + fi + 2, indent + 2, st, &sp);
      } else if (vt == J_OBJ && N[v].len) {
        c.out.put(':');
        if (sp >= MAXD) { c.err = TS_UNSUPPORTED; break; }
        st[sp++] = Frame{FR_OBJ, v, N[v].off, pre + fi + 2, indent + 2, 0};
      } else {
        c.out.put(':'); c.out.put(' ');
        if (vt == J_ARR) c.out.puts("[0]:");
        else if (vt != J_OBJ) emit_prim(c, v);
      }
    }
  }
}

CF_HD int toon_finish(int pr, const uint8_t* s, const JNode* nodes, uint8_t* out, uint32_t out_cap, uint32_t* out_len, Big* big,
                      uint8_t* digits, uint32_t digits_cap, bool stop_on_over);

// Whole per-unit pipeline.  The product passes out_cap = n - 1: a conversion is only kept when it is
// strictly smaller than the n input bytes, so a longer TOON text can be abandoned mid-way.  Returns a TS_* status; *out_len is valid for TS_CONVERTED.
CF_HD int toon_process(const uint8_t* s, uint32_t n, JNode* nodes, uint32_t node_cap, uint8_t* out, uint32_t out_cap,
                       uint32_t* out_len, Big* big, uint8_t* digits, uint32_t digits_cap, bool stop_on_over) {
  uint32_t count = 0;
  int pr = json_parse(s, n, nodes, node_cap, &count);
  return toon_finish(pr, s, nodes, out, out_cap, out_len, big, digits, digits_cap, stop_on_over);
}

// the part after the parse (pr = PARSE_* of whichever parser built `nodes`)
CF_HD int toon_finish(int pr, const uint8_t* s, const JNode* nodes, uint8_t* out, uint32_t out_cap, uint32_t* out_len, Big* big,
                      uint8_t* digits, uint32_t digits_cap, bool stop_on_over) {
  if (pr == PARSE_ERROR) return TS_NOT_JSON;
  if (pr == PARSE_UNSUPPORTED) return TS_UNSUPPORTED;
  Ctx c;
  c.s = s; c.nodes = nodes;
  c.out.p = out; c.out.n = 0; c.out.cap = out_cap; c.out.over = false;
  c.err = 0; c.started = false; c.stop_on_over = stop_on_over;
  c.big = big; c.digits = digits; c.digits_cap = digits_cap;
  toon_emit(c, 0);
  if (c.err) return c.err;
  if (c.out.over) return TS_NOT_SMALLER;
  *out_len = c.out.n;
  return TS_CONVERTED;
}

}  // namespace cfj
