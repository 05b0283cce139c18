// scan_core.h — data layout + the per-candidate verification routine shared by the CUDA scan
// kernel (cfgpu.cu) and the host-side table simulator used only by the CPU unit tests
// (host_sim.cpp).  Everything here is plain C++ that compiles for host and device.
//
// Reference semantics being implemented (all relative to /root/reference):
//   * harmful_content_detector: `pat.search(text)` for each IGNORECASE pattern
//       plugins/harmful_content_detector/harmful_content_detector.py:92-107
//   * deny_filter: `word in value`                      plugins/deny_filter/deny.py:59-60
//   * regex_filter: `pattern.sub(replacement, value)`   plugins/regex_filter/search_replace.py:127-130
// A "unit" is one Python `str` handed to those calls, UTF-8 encoded.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define CF_HD __host__ __device__ __forceinline__
#else
#define CF_HD inline
#endif

namespace cf {

// ---------------------------------------------------------------------------------------------
// Packed stream layout (HBM and host):
//   stream = unit_0 0xFF unit_1 0xFF ... unit_{n-1} 0xFF          (0xFF never occurs in UTF-8)
//   offsets[i] = byte offset of unit_i, offsets[n] = total length including terminators
//   unit_i = stream[offsets[i] .. offsets[i+1]-1)   (the byte at offsets[i+1]-1 is its 0xFF)
// On the device the stream is preceded by CF_FRONT_PAD bytes of 0xFF and followed by 0xFF up to a
// multiple of the scan tile plus one extra tile, so tile loads never need bounds checks.
// ---------------------------------------------------------------------------------------------
static const uint8_t  TERM      = 0xFF;
static const uint32_t FRONT_PAD = 256;

// Coarse unit index of a batch: coarse[k] = the unit that holds stream byte k << COARSE_SHIFT, for k in [0, nbytes >> COARSE_SHIFT].
static const uint32_t COARSE_SHIFT = 12;

// A batch packed from device memory (cf_batch_pack_device): unit i is src[src_off[i] .. src_off[i+1]) of the source, and starts in the
// stream at its source offset rebased to unit 0 plus one terminator per unit before it.  Clamped to the stream's `nbytes`, so that
// offsets that are not monotone give wrong units but never a position past the stream.
CF_HD uint64_t packed_offset(const uint64_t* src_off, uint32_t i, uint64_t nbytes) {
  const uint64_t o = src_off[i] - src_off[0] + i;
  return o < nbytes ? o : nbytes;
}
// coarse[k] of that batch: the last unit i in [0, n) whose packed offset is <= k << COARSE_SHIFT (an upper-bound binary search over
// units 1 .. n-1), which is what cf_batch_upload's host sweep finds for monotone offsets.  Always in [0, n).
CF_HD uint32_t packed_coarse(const uint64_t* src_off, uint32_t n, uint64_t nbytes, uint64_t k) {
  const uint64_t pos = k << COARSE_SHIFT;
  uint32_t lo = 1, hi = n;   // the first unit in [1, n) that starts after pos, or n
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (packed_offset(src_off, mid, nbytes) <= pos) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

// previous-character contexts (needed by \b, \B, ^, \A)
enum : uint32_t { P_START = 0, P_WORD = 1, P_NL = 2, P_OTHER = 3 };

static const uint32_t DEAD = 0;         // DFA state 0 is the dead state
static const uint32_t ACC_SHIFT = 16;   // transition entry = next_state | acc_index << 16

// Tables for one anchored DFA over code-point classes.
struct DfaTables {
  const uint16_t* ascii_cls;    // [128] class of each ASCII code point
  const uint32_t* range_start;  // [nranges] first code point of each non-ASCII range (sorted, [0]=0x80)
  const uint16_t* range_cls;    // [nranges] class of that range
  const uint8_t*  cls_ctx;      // [ncls] P_WORD / P_NL / P_OTHER for a char of this class
  const uint32_t* trans;        // [nstates * ncols]; ncols = ncls + 1, column ncls = end-of-text
  const uint64_t* accsets;      // [naccs * W] pattern bitmaps; acc index 0 = empty set
  uint32_t nranges;
  uint32_t ncols;
  uint32_t W;                   // u64 words per verdict bitmap
  uint32_t start_state[4];      // indexed by previous-character context
  uint32_t start_adv[4];        // ordered DFAs only: the same, but a zero-length match at the start position does not count
  uint32_t nl_cls, nlf_cls;     // class of '\n'; class that stands for "the '\n' that is the unit's LAST character" (a non-MULTILINE `$`
                                // holds in front of it) or NO_CLS when no pattern needs the distinction
};
static const uint32_t NO_CLS = 0xFFFFFFFFu;
// column of the character that was just classified: the final newline of the unit gets its own class when the program asks for it
CF_HD uint32_t final_nl(const DfaTables& t, uint32_t col, bool last_char) { return (col == t.nl_cls && last_char && t.nlf_cls != NO_CLS) ? t.nlf_cls : col; }

// Decode one UTF-8 scalar (generalised: surrogates ED A0..BF xx are accepted, Python's
// 'surrogatepass').  `p < end` is required.  Never reads at or beyond `end`.
CF_HD uint32_t utf8_decode(const uint8_t* s, uint64_t p, uint64_t end, uint32_t* len) {
  uint32_t b0 = s[p];
  if (b0 < 0x80) { *len = 1; return b0; }
  uint32_t need = (b0 >= 0xF0) ? 4u : (b0 >= 0xE0) ? 3u : (b0 >= 0xC0) ? 2u : 1u;
  if (need == 1 || p + need > end) { *len = 1; return 0xFFFD; }  // stray continuation / truncated
  uint32_t cp = b0 & (0xFFu >> (need + 1));
  for (uint32_t k = 1; k < need; ++k) cp = (cp << 6) | (s[p + k] & 0x3Fu);
  *len = need;
  return cp;
}

CF_HD uint32_t classify(const DfaTables& t, uint32_t cp) {
  if (cp < 0x80) return t.ascii_cls[cp];
  uint32_t lo = 0, hi = t.nranges;  // last range with start <= cp
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (t.range_start[mid] <= cp) lo = mid; else hi = mid;
  }
  return t.range_cls[lo];
}

// Context of the character that ends right before byte position p (p > ustart).
CF_HD uint32_t prev_context(const DfaTables& t, const uint8_t* s, uint64_t ustart, uint64_t p) {
  uint64_t q = p - 1;
  while (q > ustart && (s[q] & 0xC0) == 0x80 && p - q < 4) --q;
  uint32_t len;
  uint32_t cp = utf8_decode(s, q, p, &len);
  return t.cls_ctx[classify(t, cp)];
}

// Run the anchored DFA from byte position p of the unit [ustart, uend); OR the bitmaps of all
// patterns that match starting exactly at p (any end) into bits[0..W).  Returns the number of
// DFA steps (for statistics).  Search semantics: existence only.
CF_HD uint32_t verify_search(const DfaTables& t, const uint8_t* s, uint64_t ustart, uint64_t uend,
                             uint64_t p, uint64_t* bits) {
  uint32_t ctx = (p == ustart) ? (uint32_t)P_START : prev_context(t, s, ustart, p);
  uint32_t S = t.start_state[ctx];
  uint64_t q = p;
  uint32_t steps = 0;
  while (S != DEAD) {
    uint32_t col, len = 0;
    if (q >= uend) col = t.ncols - 1;
    else col = final_nl(t, classify(t, utf8_decode(s, q, uend, &len)), q + 1 == uend);
    uint32_t e = t.trans[(uint64_t)S * t.ncols + col];
    uint32_t a = e >> ACC_SHIFT;
    if (a) for (uint32_t w = 0; w < t.W; ++w) bits[w] |= t.accsets[(uint64_t)a * t.W + w];
    S = e & 0xFFFFu;
    ++steps;
    if (q >= uend) break;
    q += len;
  }
  return steps;
}

// Leftmost-first match of ONE ordered (priority) DFA anchored at p.  Transition entries carry
// bit 16 = "a match ends before this character".  Returns the match end (byte offset) or
// UINT64_MAX when nothing matches at p.  This is Python's backtracking preference order
// (plugins/regex_filter/search_replace.py:130 -> re.Pattern.sub).
// `must_advance`: the match may not be empty (what `re.sub` asks for at the position right after an empty match:
// Modules/_sre/sre.c pattern_subx `state.must_advance = (state.ptr == state.start)`); a lower-priority non-empty
// alternative is then taken if there is one, exactly like sre's backtracking.
CF_HD uint64_t match_first(const DfaTables& t, const uint8_t* s, uint64_t ustart, uint64_t uend,
                           uint64_t p, bool must_advance = false) {
  uint32_t ctx = (p == ustart) ? (uint32_t)P_START : prev_context(t, s, ustart, p);
  uint32_t S = must_advance ? t.start_adv[ctx] : t.start_state[ctx];
  uint64_t q = p, last = ~0ull;
  while (S != DEAD) {
    uint32_t col, len = 0;
    if (q >= uend) col = t.ncols - 1;
    else col = final_nl(t, classify(t, utf8_decode(s, q, uend, &len)), q + 1 == uend);
    uint32_t e = t.trans[(uint64_t)S * t.ncols + col];
    if (e >> ACC_SHIFT) last = q;
    S = e & 0xFFFFu;
    if (q >= uend) break;
    q += len;
  }
  return last;
}

// ---------------------------------------------------------------------------------------------
// Capture pass for replacement templates with group references (`\\1`, `\\g<name>`): a Pike VM over the rule's Thompson NFA
// (re_backend.h NfaOut), anchored at p — the start the ordered DFA found — with the DFA's own character classes, assertion
// semantics (previous-character context + class of the next character) and priority order, so it finds the very match the
// DFA found and, with it, the group spans Python's backtracking matcher reports for it (a group inside a repeat keeps the span
// of its last participating iteration; a group that never took part stays unset -> "" in the template, Python >= 3.5).
// One thread per NFA instruction and position at most: O(match length x NFA size), no backtracking.
// ---------------------------------------------------------------------------------------------
enum : uint32_t { N_CHAR = 0, N_SPLIT = 1, N_ASSERT = 2, N_MATCH = 3, N_SAVE = 4 };
static const uint32_t CAP_UNSET = 0xFFFFFFFFu;
struct NfaView {
  const uint32_t* code;       // 3 words per instruction
  const uint32_t* setbits;
  uint32_t ninst, start, wpc, nslots;   // nslots = 2 * (groups + 1); slots 0/1 = the whole match
};
CF_HD uint64_t pike_scratch_words(uint32_t ninst, uint32_t nslots) { return (uint64_t)ninst * (1 + 2 + 2ull * nslots + 6) + nslots; }

CF_HD bool assert_holds(uint32_t kind, uint32_t P, uint32_t col, uint32_t eot_col, const uint8_t* cls_ctx, uint32_t nlf_cls) {
  const bool eot = col == eot_col;
  const bool nw = !eot && cls_ctx[col] == P_WORD, nnl = !eot && cls_ctx[col] == P_NL;
  switch (kind) {
    case 1: return (P == P_WORD) != nw;                                   // \b
    case 2: if (P == P_START && eot) return false; return (P == P_WORD) == nw;   // \B (sre: never on an empty string)
    case 3: return P == P_START;                                          // \A
    case 4: return P == P_START || P == P_NL;                             // ^ (MULTILINE)
    case 5: return eot;                                                   // \Z
    case 7: return eot || col == nlf_cls;                                 // $ without MULTILINE: also before a final newline
    case 6: return eot || nnl;                                            // $ (MULTILINE)
  }
  return false;
}

// Threads of one position: pcs[k], caps[k * nslots ..].  `add` follows the epsilon edges from pc in priority order.
struct PikeList { uint32_t* pcs; uint32_t* caps; uint32_t n; };
CF_HD void pike_add(const DfaTables& t, const NfaView& N, PikeList& L, uint32_t pc0, uint32_t pos, uint32_t P, uint32_t col,
                    uint32_t* cur, uint32_t* visited, uint32_t stamp, uint32_t* stack) {
  uint32_t sp = 0;
  stack[sp++] = pc0; stack[sp++] = CAP_UNSET;                 // {pc, CAP_UNSET} = explore, {slot, old value + marker} = restore
  while (sp) {
    const uint32_t b = stack[--sp], a = stack[--sp];
    if (b != CAP_UNSET) { cur[a] = b == CAP_UNSET - 1 ? CAP_UNSET : b; continue; }      // restore a capture slot
    if (visited[a] == stamp) continue;
    visited[a] = stamp;
    const uint32_t w = N.code[3 * a], op = w & 0xFF, arg = w >> 8, x = N.code[3 * a + 1], y = N.code[3 * a + 2];
    switch (op) {
      case N_CHAR: case N_MATCH: {
        L.pcs[L.n] = a;
        for (uint32_t k = 0; k < N.nslots; ++k) L.caps[(uint64_t)L.n * N.nslots + k] = cur[k];
        ++L.n;
        break;
      }
      case N_SPLIT: stack[sp++] = y; stack[sp++] = CAP_UNSET; stack[sp++] = x; stack[sp++] = CAP_UNSET; break;
      case N_ASSERT: if (assert_holds(arg, P, col, t.ncols - 1, t.cls_ctx, t.nlf_cls)) { stack[sp++] = x; stack[sp++] = CAP_UNSET; } break;
      case N_SAVE:
        stack[sp++] = arg; stack[sp++] = cur[arg] == CAP_UNSET ? CAP_UNSET - 1 : cur[arg];
        cur[arg] = pos;
        stack[sp++] = x; stack[sp++] = CAP_UNSET;
        break;
    }
  }
}

// caps_out[0 .. nslots): byte offsets relative to the unit (CAP_UNSET = group did not take part).  Returns false when nothing
// matches at p (cannot happen for a start the DFA accepted).  Offsets must fit 32 bits (units are < 4 GB).
CF_HD bool pike_captures(const DfaTables& t, const NfaView& N, const uint8_t* s, uint64_t ustart, uint64_t uend, uint64_t p,
                         bool must_advance, uint32_t* scratch, uint32_t* caps_out) {
  uint32_t* visited = scratch;
  PikeList A, B;
  A.pcs = visited + N.ninst; B.pcs = A.pcs + N.ninst;
  A.caps = B.pcs + N.ninst; B.caps = A.caps + (uint64_t)N.ninst * N.nslots;
  uint32_t* stack = B.caps + (uint64_t)N.ninst * N.nslots;
  uint32_t* cur = stack + 6ull * N.ninst;
  for (uint32_t k = 0; k < N.ninst; ++k) visited[k] = 0;
  for (uint32_t k = 0; k < N.nslots; ++k) cur[k] = CAP_UNSET;
  uint32_t stamp = 0;
  uint32_t P = (p == ustart) ? (uint32_t)P_START : prev_context(t, s, ustart, p);
  uint64_t q = p;
  uint32_t len = 0;
  uint32_t col = q >= uend ? t.ncols - 1 : final_nl(t, classify(t, utf8_decode(s, q, uend, &len)), q + 1 == uend);
  A.n = 0;
  cur[0] = (uint32_t)(p - ustart);
  pike_add(t, N, A, N.start, (uint32_t)(q - ustart), P, col, cur, visited, ++stamp, stack);
  bool matched = false;
  while (A.n) {
    const uint64_t q2 = q + len;
    uint32_t len2 = 0, col2 = t.ncols - 1, P2 = P_OTHER;
    if (col != t.ncols - 1) {
      P2 = t.cls_ctx[col];
      if (q2 < uend) col2 = final_nl(t, classify(t, utf8_decode(s, q2, uend, &len2)), q2 + 1 == uend);
    }
    B.n = 0;
    ++stamp;
    for (uint32_t k = 0; k < A.n; ++k) {
      const uint32_t pc = A.pcs[k], w = N.code[3 * pc], op = w & 0xFF;
      if (op == N_MATCH) {
        if (must_advance && q == p) continue;               // sre: an empty match at the start fails SUCCESS and backtracks
        for (uint32_t j = 0; j < N.nslots; ++j) caps_out[j] = A.caps[(uint64_t)k * N.nslots + j];
        caps_out[1] = (uint32_t)(q - ustart);
        matched = true;
        break;                                              // lower-priority threads are cut
      }
      if (col != t.ncols - 1 && ((N.setbits[(uint64_t)(w >> 8) * N.wpc + (col >> 5)] >> (col & 31)) & 1u)) {
        for (uint32_t j = 0; j < N.nslots; ++j) cur[j] = A.caps[(uint64_t)k * N.nslots + j];
        pike_add(t, N, B, N.code[3 * pc + 1], (uint32_t)(q2 - ustart), P2, col2, cur, visited, stamp, stack);
      }
    }
    if (col == t.ncols - 1) break;
    PikeList T = A; A = B; B = T;
    q = q2; len = len2; P = P2; col = col2;
  }
  return matched;
}

// Prefilter.  Five 5-bit fields per byte value, five pattern buckets per field:
//   E[b] = P3<<20 | P2<<15 | P1<<10 | P0<<5 | N
//   N  : bucket k admits b as the byte BEFORE a match start (\b, ^ contexts; 0xFF = start of unit)
//   Pj : bucket k admits b as byte j of a match
//   acc' = ((acc << 5) | 31) & E[b]            (the shift is a multiply-add: acc * 32 + 31)
// After feeding byte p, (acc & F_HIT) != 0  <=>  some bucket admits a match starting at p-3
// (a 5-byte window: previous byte + first four match bytes).  No false negatives.
// 25 bits leave room to advance TWO bytes per step in the scan kernel:
//   acc'' = ((acc << 10) | 1023) & ((E[b0] << 5) | 31) & (E[b1] | F_HIT << 5)
// keeps the first byte's candidate field in bits 25-29 and the second byte's in bits 20-24.
static const uint32_t F_BITS = 5, F_FILL = 31u, F_HIT = 0x01F00000u, F_BUCKETS = 5;
static const uint32_t F_LOOKBACK = 4;   // bytes fed before the first owned position
static const uint32_t F_START_OFF = 3;  // candidate start = fed position - 3
CF_HD uint32_t filter_step(uint32_t acc, uint32_t e) { return ((acc << F_BITS) | F_FILL) & e; }

// Pair prefilter (large rule sets).  The byte filter admits a window when every position's byte is in
// that position's SET; with many patterns per bucket the sets fill up and the filter stops filtering.
// The pair filter keys each position on the byte AND its predecessor, hashed to PF_SLOTS table slots:
//   T[h(x, y)] = P3<<24 | P2<<16 | P1<<8 | P0,  eight buckets per field,
//   Pj bucket k : some pattern of bucket k has byte y at match position j preceded by byte x
//                 (j = 0: x is the byte before the match; 0xFF = start of unit)
//   acc' = ((acc << 8) | 0xFF) & T[h(prev, cur)];   (acc & PF_HIT) != 0 after feeding byte p
//   <=> some bucket admits a match starting at p-3.  Same window (5 bytes), same candidate position,
//   no false negatives (hash collisions only add admitted pairs).
static const uint32_t PF_SLOTS = 1024, PF_BUCKETS = 8, PF_HIT = 0xFF000000u, PF_MULT = 0x9E3779B1u;
CF_HD uint32_t pair_hash(uint32_t prev, uint32_t cur) {
  const uint32_t u = (prev | (cur << 8)) * 0x00010001u;     // {prev, cur, prev, cur}: one PRMT on the GPU
  return (u * PF_MULT) >> 22;
}
CF_HD uint32_t pair_step(uint32_t acc, uint32_t e) { return ((acc << 8) | 0xFFu) & e; }

}  // namespace cf
