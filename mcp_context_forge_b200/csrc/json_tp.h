// json_tp.h — token-parallel JSON -> TOON, one WARP per payload, no DOM.
//
// The reference work this replaces (paths relative to /root/reference):
//   orjson.loads + toon.encode + "keep only if strictly smaller"   plugins/toon_encoder/toon_encoder.py:277-303
//   encoder rules                                                    plugins/toon_encoder/toon.py:82-565
//
// Shape of the computation (DESIGN.md §4.4).  Everything is written so that each LANE runs sequential code over
// data it owns (its 32 bytes, its token, its table row): the first version put lane i on byte i of one 32-byte chunk
// and paid ~16 warp-instructions per input byte (profiles/r02_toon_tp_v1_lines.txt).
//   tokenize   1 KiB per step, lane l owns bytes [32 l, 32 l + 32) as eight 32-bit words: SWAR byte-class flags ->
//              per-lane 32-bit masks (quote, backslash, brackets, comma, colon, blank, ...), escape parity and the
//              in-string state carried across lanes by ballots / warp scans -> SIGNIFICANT tokens (brackets, strings at
//              their closing quote, scalar starts; commas and colons are only counted in front of the next token).
//              32 tokens at a time, lane i <-> token i: scalars / strings validated and classified (orjson's accept
//              set), 8-byte tokens stored to HBM scratch.
//   analyze    over the token array.  Generic mode: 32 tokens, ONE warp-uniform walk over the batch's brackets keeps the
//              container stack (grammar, child counts, duplicate-key screen, table detection against the first row) and
//              patches each opener with {child count, layout mode}.  Table mode: once the first row of an array of
//              objects is known, every later row is checked by its own lane against the first row's token pattern.
//   emit       over the token array.  Generic mode: the bracket walk carries the TOON frames (layout mode, prefix width,
//              indent level), piece lengths -> warp prefix sum -> parallel writes.  Table mode: one lane per table row.
// Whatever the fast path does not cover (duplicate keys, escaped keys, permuted table rows, numbers that need the exact
// big-integer formatter, ...) is reported as TS_FALLBACK and re-done by the sequential per-thread encoder (json_toon.h) —
// still on the GPU, never on the CPU.
#pragma once
#include <stdint.h>

#include "json_index.h"
#include "json_toon.h"
#include "warp_prims.h"

namespace cftp {

using cfj::TS_ATTR_ERROR;
using cfj::TS_CONVERTED;
using cfj::TS_NOT_JSON;
using cfj::TS_NOT_SMALLER;
using cfj::TS_UNSUPPORTED;
using cfj::TS_VALUE_ERROR;
enum : int { TS_FALLBACK = 7 };      // internal: bits 8.. carry the reason (FB_*), stripped at the ABI
enum : uint32_t { FB_NUM_EXACT = 1, FB_KEY_ESCAPE = 2, FB_TOK_CAP = 3, FB_KH_CAP = 4, FB_DUP_HASH = 5, FB_ROW_ORDER = 6, FB_MIXED_ITEM = 7, FB_TOO_LONG = 8 };

// ---- phase timing: build option CF_TOON_PHASES, off in the shipped library (tools/toon_phase_breakdown.py builds it) ----
// Lane 0 of each warp adds the clock64() cycles of each phase to the warp's row of toon_phase_cycles (warp slots wrap around at
// PH_WARPS).  Column PH_N is the warp's "inside the resolve retry" flag: the retry's cycles count once, in PH_RESOLVE.
// The PH_TK_* columns split PH_TOKENIZE: the step's loads and window shift, the mask algebra and warp scans, the per-kind ring
// passes, the classification batches (tok_batch, the long-string checks included) and, inside them, the whole-warp long-string
// checks alone.
enum : uint32_t { PH_TOKENIZE = 0, PH_AN_GENERIC = 1, PH_AN_TABLE = 2, PH_EM_GENERIC = 3, PH_EM_TABLE = 4, PH_RESOLVE = 5,
                  PH_TK_LOAD = 6, PH_TK_MASKS = 7, PH_TK_RING = 8, PH_TK_BATCH = 9, PH_TK_LONG = 10, PH_N = 11 };
#if defined(CF_TOON_PHASES) && defined(__CUDACC__)
static const uint32_t PH_WARPS = 1u << 16;
__device__ unsigned long long toon_phase_cycles[PH_WARPS * (PH_N + 1)];
TP_FN unsigned long long* ph_row() { return toon_phase_cycles + ((blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) % PH_WARPS) * (PH_N + 1); }
TP_FN void ph_add(uint32_t k, unsigned long long t0) {
  const unsigned long long t1 = clock64();
  if (tpw::lane() == 0 && (k == PH_RESOLVE || !ph_row()[PH_N])) atomicAdd(ph_row() + k, t1 - t0);
}
TP_FN void ph_in_retry(bool on) { if (tpw::lane() == 0) ph_row()[PH_N] = on ? 1ull : 0ull; }
#define TP_PHASE(k, ...) do { const unsigned long long ph_t0_ = clock64(); __VA_ARGS__; ph_add((k), ph_t0_); } while (0)
// a sub-phase whose code may `break` out of the enclosing loop: TP_MARK(t) starts it, TP_LAP(k, t) adds its cycles and restarts t
#define TP_MARK(t) unsigned long long t = clock64()
#define TP_LAP(k, t) do { ph_add((k), (t)); (t) = clock64(); } while (0)
#else
TP_FN void ph_in_retry(bool) {}
#define TP_PHASE(k, ...) do { __VA_ARGS__; } while (0)
#define TP_MARK(t) do {} while (0)
#define TP_LAP(k, t) do {} while (0)
#endif

// ---- tokens --------------------------------------------------------------------------------------------------------
enum : uint32_t { K_OPEN_OBJ = 0, K_OPEN_ARR = 1, K_CLOSE_OBJ = 2, K_CLOSE_ARR = 3, K_STR = 4, K_KEY = 5, K_NUM = 6, K_LIT = 7 };
struct GTok { uint32_t pos, w; };                 // w = kind:3 | flags:5 | commas:2 | colons:2 | len:20
static const uint32_t GT_MAXLEN = (1u << 20) - 1;
// flags (5 bits)
enum : uint32_t { SF_Q = 1, SF_ESCX = 2, SF_CTRLERR = 4 };        // K_STR: needs quotes / needs transcoding / holds a char TOON cannot quote
enum : uint32_t { KF_KEYOK = 1 };                                 // K_KEY: valid unquoted key
enum : uint32_t { AM_EMPTY = 0, AM_COLUMNAR = 1, AM_INLINE = 2, AM_ITEMS = 3, AF_MIXED = 4 /* first element an object, some later one not, verdict unknown */,
                  AF_CRASH = 8 /* toon._try_columnar_encoding(arr) raises AttributeError */ };   // K_OPEN_ARR (patched at its closer)
TP_FN uint32_t gt_kind(uint32_t w) { return w & 7u; }
TP_FN uint32_t gt_flags(uint32_t w) { return (w >> 3) & 31u; }
TP_FN uint32_t gt_nc(uint32_t w) { return (w >> 8) & 3u; }        // commas in front of the token (saturating at 3)
TP_FN uint32_t gt_nk(uint32_t w) { return (w >> 10) & 3u; }       // colons in front of the token
TP_FN uint32_t gt_len(uint32_t w) { return w >> 12; }
TP_FN uint32_t gt_make(uint32_t kind, uint32_t fl, uint32_t nc, uint32_t nk, uint32_t len) { return kind | (fl << 3) | (nc << 8) | (nk << 10) | (len << 12); }
TP_FN uint32_t gt_patch(uint32_t w, uint32_t kind, uint32_t fl, uint32_t len) { return (w & 0xF00u) | kind | (fl << 3) | (len << 12); }

// ring record meta (tokenizer -> classification batch)
enum : uint32_t { RM_KIND = 7u, RM_NCOMMA_SH = 3, RM_NCOLON_SH = 5, RM_SPECIAL = 1u << 7, RM_NONKEY = 1u << 8, RM_HI = 1u << 9, RM_BS = 1u << 10,
                  RM_OPENEND = 1u << 11 /* scalar run reaches past the next lane's 32 bytes: length still unknown */,
                  RM_ALLDIGIT = 1u << 12 /* scalar run consists of ASCII digits only */ };

// ---- per-warp shared memory ----------------------------------------------------------------------------------------
// Shared + the staging buffer (STAGE) is what one warp owns: 9 488 B, so that three 8-warp CTAs fit an SM (cfjson.cu TP_SMEM).
// Storage no two phases use at once is shared: tokenize keeps its ring's meta words behind the source window in the staging
// buffer, and emit's table rounds stage their output over the analyze-only fields (row_out).
static const uint32_t RING = 256, MAXD = 64, KH_CAP = 256;
static const uint32_t TOK_WIN = 192;      // tokens of one 1 KiB step pushed through the ring at a time (a window never overtakes the 32-token batches)
static const uint32_t UNSET = 0xFFFFFFFFu;
struct Shared {
  unsigned long long sbar_bar;         // mbarrier of the staging buffer's bulk TMA loads (initialised by the kernel)
  uint32_t sbar_phase;
  uint32_t utf8_bad;                   // tokenize: unit position of the first byte where its UTF-8 fails (UNSET: none so far)
  // analyze: container stack            | emit: frame stack (same storage)
  uint32_t open_idx[MAXD];             // token index of the opener      | frame mode
  uint32_t cnt[MAXD];                  // children (values) so far       | children so far
  uint32_t cfl[MAXD];                  // C_* flags                      | prefix width
  uint32_t khbase[MAXD];               // base of the key hashes         | indent level
  // tokenize and analyze only: from row0_idx to the end, emit's table rounds stage their output here (row_out)
  uint32_t row0_idx[MAXD];             // arrays: 1 + token index of the first element when it is an object
  uint32_t row0_n[MAXD];               // arrays: member count of that first object once it closed
  uint32_t open_w[MAXD];               // analyze: the opener's token word (its separator bits survive the patch)
  uint32_t kh[KH_CAP];                 // key hashes of the open objects (stack)
  uint32_t ring_pos[RING], ring_len[RING];   // tokenize | analyze: ring_pos[j], ring_len[j] = the key whose hash is kh[j]
  TP_FN uint8_t* row_out() { return reinterpret_cast<uint8_t*>(row0_idx); }
};
enum : uint32_t {
  C_OBJ = 1,
  // arrays
  C_ALL_SIMPLE = 2,      // no element is a container
  C_ALL_OBJ = 4,         // every element is an object
  C_KEYSET_OK = 8,       // every object element so far has the first one's key set (toon.py:487-490)
  C_ROWS_SIMPLE = 64,    // every member value of every object element so far is a primitive (toon.py:493-495)
  C_ND_SEEN = 128,       // a non-object element followed an object first element (the unchecked .keys() of toon.py:488)
  C_CRASH = 256,         // ... and arrived before any key-set mismatch: _try_columnar_encoding raises AttributeError
  C_PERMUTED = 512,      // some row lists the first row's keys in another order (columnar output needs a gather)
  C_ROW0_SIMPLE = 1024,  // the first row's values are primitives: its j-th key is token row0 + 1 + 2j
  C_ITEM_HEAD = 2048,    // the first member of an object that is an element of an array: as a list item's first value, toon.py:400-404
                         // tries the array as columnar without a type check, so only here does AF_CRASH / AF_MIXED matter
  C_R0KEYS = 8192,       // (resolve_mixed) the first row is not simple; its keys stay at kh / ring_pos / ring_len[khbase - row0_n ..)
                         // (the later rows' keys are hashed from khbase on) so that every later row's key set is compared with it
  // objects
  C_ALIGNED = 16,        // keys equal the first row's, position by position
  C_VALS_SIMPLE = 32,    // all member values are primitives
  C_DIFFSET = 4096       // some key does not occur in the first row at all
};

// Per-warp staging buffer (shared memory on the GPU): lane-strided byte accesses to global memory cost one L1 wavefront per
// lane (profiles/r02_toon_tp_v2_ncu.txt: the kernel was bound by exactly that), so whatever a lane reads byte by byte is
// first brought in with coalesced 16-byte loads, and table rows are written to global memory through it the same way.
static const uint32_t STAGE = 4608;          // bytes per warp
static const uint32_t WIN = 2048;            // tokenizer: the last two 1 KiB steps of source text, then the ring's meta words (RING of them)
// table rows: source bytes of a round (the staging buffer) | its output (Shared::row_out, 3 840 B); an A-shaped row of ~150 source
// bytes writes ~95, so a round of 30 rows fits both
static const uint32_t ROW_SRC = STAGE, ROW_OUT = (uint32_t)(sizeof(Shared) - 16 - 4 * 4 * MAXD);
static_assert(WIN + 4 * RING <= STAGE, "tokenizer window + ring meta fit the staging buffer");
static_assert(ROW_OUT == 3 * 4 * MAXD + 4 * KH_CAP + 2 * 4 * RING, "row_out spans row0_idx .. the end of Shared");
static_assert(sizeof(Shared) % 16 == 0 && (16 + 4 * 4 * MAXD) % 16 == 0, "row_out and the staging buffer behind Shared stay 16-byte aligned");

// stage[0..) <- s[a0 .. a1) where a0 is rounded down to the 16-byte grid; returns the unit position of stage[0] (can be negative)
// On the GPU the copy is ONE bulk TMA transfer (cp.async.bulk global -> shared, SASS UBLKCP) completing on the warp's mbarrier.
struct StageBar { uint64_t bar; uint32_t phase; };     // lives in the warp's shared memory (Shared::sbar)
TP_FN int64_t stage_load(uint8_t* stage, const uint8_t* s, uint32_t a0, uint32_t a1, StageBar& sb) {
  const uint32_t lead = (uint32_t)((uintptr_t)(s + a0) & 15u);
  const uint8_t* g = s + a0 - lead;
  const uint32_t bytes = a1 - a0 + lead;
#ifdef __CUDA_ARCH__
  const uint32_t b16 = (bytes + 15u) & ~15u;
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&sb.bar), dst = (uint32_t)__cvta_generic_to_shared(stage);
  const uint32_t parity = sb.phase;
  tpw::sync();                                                          // every lane is done with the buffer's previous contents
  if (tpw::lane() == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // generic-proxy accesses to the buffer are ordered before the async-proxy write
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(b16) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(g), "r"(b16), "r"(bar) : "memory");
    sb.phase = parity ^ 1u;
  }
  uint32_t ok;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
  tpw::sync();
#else
  (void)sb;
  for (uint32_t o = tpw::lane() * 16; o < bytes; o += 512) *reinterpret_cast<uint4*>(stage + o) = *reinterpret_cast<const uint4*>(g + o);
  tpw::sync();
#endif
  return (int64_t)a0 - (int64_t)lead;
}
// out[dst .. dst+len) <- stage[0 .. len), coalesced (16-byte stores on the aligned middle)
TP_FN void stage_flush(uint8_t* out, uint32_t dst, const uint8_t* stage, uint32_t len) {
  const uint32_t l = tpw::lane();
  uint8_t* g = out + dst;
  const uint32_t head = (uint32_t)((16u - ((uintptr_t)g & 15u)) & 15u);
  const uint32_t h = head < len ? head : len;
  if (l < h) g[l] = stage[l];
  if ((h & 15u) == 0 || true) {
    // stage + h is not 16-byte aligned in general: assemble each 16-byte store from byte reads of shared memory
    const uint32_t mid = (len - h) & ~15u;
    for (uint32_t o = l * 16; o < mid; o += 512) {
      const uint8_t* p = stage + h + o;
      uint4 v;
      v.x = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
      v.y = (uint32_t)p[4] | ((uint32_t)p[5] << 8) | ((uint32_t)p[6] << 16) | ((uint32_t)p[7] << 24);
      v.z = (uint32_t)p[8] | ((uint32_t)p[9] << 8) | ((uint32_t)p[10] << 16) | ((uint32_t)p[11] << 24);
      v.w = (uint32_t)p[12] | ((uint32_t)p[13] << 8) | ((uint32_t)p[14] << 16) | ((uint32_t)p[15] << 24);
      *reinterpret_cast<uint4*>(g + h + o) = v;
    }
    const uint32_t t0 = h + mid;
    if (t0 + l < len) g[t0 + l] = stage[t0 + l];
  }
  tpw::sync();
}

// byte classes (scalar-run scan of the rare paths; the tokenizer itself uses SWAR flag words)
enum : uint32_t { BC_QUOTE = 2, BC_STRUCT = 4, BC_WS = 32 };
TP_FN uint32_t byte_class(uint32_t b) {
  uint32_t k = 0;
  if (b == '"') k |= BC_QUOTE;
  if (b == '{' || b == '}' || b == '[' || b == ']' || b == ':' || b == ',') k |= BC_STRUCT;
  if (b == ' ' || b == '\t' || b == '\n' || b == '\r') k |= BC_WS;
  return k;
}

#ifdef __CUDACC__
TP_FN uint32_t bits_below(uint32_t i) { return __funnelshift_lc(0xFFFFFFFFu, 0u, i); }   // bits 0..i-1 (one SHF; the shift clamps at 32)
#else
TP_FN uint32_t bits_below(uint32_t i) { return i >= 32 ? 0xFFFFFFFFu : ((1u << i) - 1u); }   // bits 0..i-1
#endif
TP_FN uint32_t range_mask(uint32_t lo, uint32_t hi) { return bits_below(hi) & ~bits_below(lo); }   // bits lo..hi-1
TP_FN uint32_t sat3(uint32_t v) { return v > 3u ? 3u : v; }

// ---- SWAR over 4 bytes of a 32-bit word: the result has 0x80 in every byte that satisfies the predicate ----
TP_FN uint32_t swar_eq(uint32_t w, uint32_t c) { const uint32_t x = w ^ (c * 0x01010101u); return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u; }
// lo <= byte <= hi for bytes below 0x80 (x7 = w & 0x7F7F7F7F; bytes >= 0x80 must be masked out by the caller)
TP_FN uint32_t swar_range7(uint32_t x7, uint32_t lo, uint32_t hi) { return (x7 + (0x80u - lo) * 0x01010101u) & ~(x7 + (0x7Fu - hi) * 0x01010101u) & 0x80808080u; }
TP_FN uint32_t gather4(uint32_t f) { return (((f >> 7) * 0x00204081u) >> 21) & 15u; }   // flags at bits 7,15,23,31 -> nibble

// ---- cost key of a unit (toon_order_kernel, cfjson.cu): the first pass runs units heaviest first ----
// Estimate of the events the generic bracket walk handles in the 4 bytes of w (prev = the 4 bytes before them, 0 before the
// unit): every '{' and '[', except a '{' right after "}," or "}, " -- the next row of an array of objects, which table mode
// checks lane-parallel.  Brackets inside strings count too: the key only orders the units, it never changes a result.
static const uint32_t ORDER_WINDOW = 2048;   // bytes of a unit the key reads
TP_FN uint32_t order_events(uint32_t prev, uint32_t w) {
  const uint32_t p1 = (w << 8) | (prev >> 24), p2 = (w << 16) | (prev >> 16), p3 = (w << 24) | (prev >> 8);   // byte j <- byte j-1, j-2, j-3
  const uint32_t open = swar_eq(w | 0x20202020u, '{');                                  // '{' or '[' ('[' | 0x20 == '{')
  const uint32_t close_comma = swar_eq(p2, '}') & swar_eq(p1, ',');
  const uint32_t row = swar_eq(w, '{') & (close_comma | (swar_eq(p3, '}') & swar_eq(p2, ',') & swar_eq(p1, ' ')));
  return tpw::popc(open) - tpw::popc(row);
}

struct LaneMasks { uint32_t q, bs, ob, cb, curly, cm, co, ws, ctrl, hi, special, nonkey, digit; };   // bit j <-> byte j of the lane's 32 bytes
TP_FN void build_masks(const uint32_t* w, LaneMasks& M) {
  M.q = M.bs = M.ob = M.cb = M.curly = M.cm = M.co = M.ws = M.ctrl = M.hi = M.special = M.nonkey = M.digit = 0;
  uint32_t f_bs[8], f_ctrl[8], any_bs = 0, any_ctrl = 0, any_hi = 0;
#pragma unroll
  for (uint32_t k = 0; k < 8; ++k) {
    const uint32_t x = w[k], sh = 4 * k;
    const uint32_t hi = x & 0x80808080u, x7 = x & 0x7F7F7F7Fu;
    const uint32_t q = swar_eq(x, '"'), bs = swar_eq(x, '\\'), cm = swar_eq(x, ','), co = swar_eq(x, ':'), sp = swar_eq(x, ' ');
    const uint32_t x20 = x | 0x20202020u;
    const uint32_t ob = swar_eq(x20, '{'), cb = swar_eq(x20, '}');                    // '[' | 0x20 == '{', ']' | 0x20 == '}'
    const uint32_t br = ob | cb;
    const uint32_t curly = br & (x << 2);                                             // bit 5 of the byte: '{' '}' have it, '[' ']' do not
    const uint32_t ctrl = ~((x7 + 0x60606060u) | x) & 0x80808080u;                    // byte < 0x20
    uint32_t ws = sp;
    if (ctrl) ws |= ctrl & (swar_eq(x, '\t') | swar_eq(x, '\n') | swar_eq(x, '\r'));
    const uint32_t special = br | cm | co | swar_eq(x, '-');
    // [A-Za-z0-9_.]: folding to lower case maps '@' to '`' (below 'a') and '[' '\\' ']' '^' '_' to '{' '|' '}' '~' 0x7F (above 'z')
    const uint32_t x7l = x20 & 0x7F7F7F7Fu;
    const uint32_t digit = swar_range7(x7, '0', '9') & ~hi;
    const uint32_t keych = ((swar_range7(x7l, 'a', 'z') & ~hi) | digit | swar_eq(x, '_') | swar_eq(x, '.'));
    f_bs[k] = bs; f_ctrl[k] = ctrl; any_bs |= bs; any_ctrl |= ctrl; any_hi |= hi;
    M.q |= gather4(q) << sh; M.ob |= gather4(ob) << sh; M.cb |= gather4(cb) << sh; M.curly |= gather4(curly) << sh;
    M.cm |= gather4(cm) << sh; M.co |= gather4(co) << sh; M.ws |= gather4(ws) << sh;
    M.special |= gather4(special) << sh; M.nonkey |= gather4(keych ^ 0x80808080u) << sh; M.digit |= gather4(digit) << sh;
  }
  // rare classes: only gathered when the lane has any such byte
  if (any_bs) {
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) M.bs |= gather4(f_bs[k]) << (4 * k);
  }
  if (any_ctrl) {
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) M.ctrl |= gather4(f_ctrl[k]) << (4 * k);
  }
  if (any_hi) {
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) M.hi |= gather4(w[k] & 0x80808080u) << (4 * k);
  }
}

// Which bytes are escaped (preceded by an odd-length run of backslashes)?  simdjson's carry trick on the lane's 32-bit
// backslash mask; e_in = the lane's first byte is escaped; *e_out = the first byte after the lane is.
TP_FN uint32_t find_escaped(uint32_t bs, uint32_t e_in, uint32_t* e_out) {
  bs &= ~e_in;
  const uint32_t follows = (bs << 1) | e_in;
  const uint32_t EVEN = 0x55555555u;
  const uint32_t odd_starts = bs & ~EVEN & ~follows;
  const uint32_t sum = odd_starts + bs;
  *e_out = sum < bs ? 1u : 0u;                      // carry out of bit 31
  const uint32_t invert = sum << 1;
  return (EVEN ^ invert) & follows;
}

// ---- scalars ---------------------------------------------------------------------------------------------------------
// Number literal t[0..len) (already grammar-checked, flags from cfj::scan_number): the text toon._encode_float / str(int)
// produce is, on the cheap path, a PREFIX of the literal (possibly without its '-').  Returns false when the exact
// big-integer formatter is needed (json_toon.h emit_number's exact path).
TP_FN bool num_canon(const uint8_t* t, uint32_t len, uint32_t fl, uint32_t* eoff, uint32_t* elen) {
  const bool neg = (fl & cfj::JF_NEG) != 0;
  const uint8_t* dg = t + (neg ? 1 : 0);
  const uint32_t dl = len - (neg ? 1 : 0);
  if (!(fl & (cfj::JF_FRAC | cfj::JF_EXP))) {
    if (dl >= 19) return false;                                  // may leave the i64/u64 range: exact path decides
    if (dl == 1 && dg[0] == '0') { *eoff = neg ? 1 : 0; *elen = 1; return true; }   // "-0" -> int 0
    *eoff = 0; *elen = len;
    return true;
  }
  if (fl & cfj::JF_EXP) return false;
  uint32_t dot = 0;
  while (dg[dot] != '.') ++dot;
  uint32_t fe = dl;
  while (fe > dot + 1 && dg[fe - 1] == '0') --fe;
  const uint32_t nfrac = fe - dot - 1;
  const bool int_zero = (dot == 1 && dg[0] == '0');
  uint32_t lead_fz = 0;
  if (int_zero) while (lead_fz < nfrac && dg[dot + 1 + lead_fz] == '0') ++lead_fz;
  const uint32_t sigd = int_zero ? nfrac - lead_fz : dot + nfrac;
  const bool tiny_long = int_zero && lead_fz >= 4 && nfrac > 15;
  if (sigd > 15 || tiny_long) return false;
  if (nfrac == 0) {
    if (int_zero) { *eoff = neg ? 1 : 0; *elen = 1; return true; }     // +-0.0 -> "0"
    *eoff = 0; *elen = (neg ? 1 : 0) + dot;
    return true;
  }
  *eoff = 0; *elen = (neg ? 1 : 0) + dot + 1 + nfrac;
  return true;
}

// ---- strings ---------------------------------------------------------------------------------------------------------
TP_FN bool is_reserved(const uint8_t* b, uint32_t len) {
  if (len == 4) return (b[0] == 'n' && b[1] == 'u' && b[2] == 'l' && b[3] == 'l') || (b[0] == 't' && b[1] == 'r' && b[2] == 'u' && b[3] == 'e');
  if (len == 5) return b[0] == 'f' && b[1] == 'a' && b[2] == 'l' && b[3] == 's' && b[4] == 'e';
  return false;
}
// escapes other than \" \\ \n \r \t need transcoding (the TOON text differs from the JSON text)
TP_SLOW bool has_complex_escape(const uint8_t* b, uint32_t len) {
  for (uint32_t i = 0; i + 1 < len; ++i)
    if (b[i] == '\\') {
      const uint32_t e = b[i + 1];
      if (!(e == '"' || e == '\\' || e == 'n' || e == 'r' || e == 't')) return true;
      ++i;
    }
  return false;
}
TP_FN uint32_t fnv1a(const uint8_t* b, uint32_t len) {
  uint32_t h = 2166136261u;
  for (uint32_t i = 0; i < len; ++i) h = (h ^ b[i]) * 16777619u;
  return h;
}

// decoded length / bytes of a string that needs transcoding (JSON escapes -> TOON text), quoted or not
TP_SLOW uint32_t escx_len(const uint8_t* b, uint32_t len, bool quoted) {       // cold (strings with escapes): out of line, the kernel's hot code stays small
  cfj::StrIter it{b, b + len};
  uint32_t n = quoted ? 2u : 0u;
  while (!it.done()) {
    const uint32_t cp = it.next();
    if (quoted && (cp == '\\' || cp == '"' || cp == '\n' || cp == '\r' || cp == '\t')) n += 2;
    else n += cp < 0x80 ? 1u : cp < 0x800 ? 2u : cp < 0x10000 ? 3u : 4u;
  }
  return n;
}

// ---- output ----------------------------------------------------------------------------------------------------------
struct Emit {
  uint8_t* out;
  uint32_t cap, o;
  TP_FN void put(uint32_t c) { if (o < cap) out[o] = (uint8_t)c; ++o; }
  TP_FN void span(const uint8_t* b, uint32_t len) {
    if (o + len <= cap) {
      // eight independent loads in flight, then the stores: a lone lane cannot hide the load latency any other way
      uint8_t* d = out + o;
      uint32_t i = 0;
      for (; i + 8 <= len; i += 8) {
        const uint8_t a0 = b[i], a1 = b[i + 1], a2 = b[i + 2], a3 = b[i + 3], a4 = b[i + 4], a5 = b[i + 5], a6 = b[i + 6], a7 = b[i + 7];
        d[i] = a0; d[i + 1] = a1; d[i + 2] = a2; d[i + 3] = a3; d[i + 4] = a4; d[i + 5] = a5; d[i + 6] = a6; d[i + 7] = a7;
      }
      for (; i < len; ++i) d[i] = b[i];
      o += len;
    } else for (uint32_t i = 0; i < len; ++i) put(b[i]);
  }
  TP_FN void spaces(uint32_t k) { for (uint32_t i = 0; i < k; ++i) put(' '); }
  TP_FN void uint_dec(uint32_t v) {
    uint8_t b[10]; int k = 0;
    do { b[k++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
    while (k) put(b[--k]);
  }
  TP_FN void cp(uint32_t c) {
    if (c < 0x80) put(c);
    else if (c < 0x800) { put(0xC0 | (c >> 6)); put(0x80 | (c & 63)); }
    else if (c < 0x10000) { put(0xE0 | (c >> 12)); put(0x80 | ((c >> 6) & 63)); put(0x80 | (c & 63)); }
    else { put(0xF0 | (c >> 18)); put(0x80 | ((c >> 12) & 63)); put(0x80 | ((c >> 6) & 63)); put(0x80 | (c & 63)); }
  }
  TP_SLOW void escx(const uint8_t* b, uint32_t len, bool quoted) {
    cfj::StrIter it{b, b + len};
    if (quoted) put('"');
    while (!it.done()) {
      const uint32_t c = it.next();
      if (quoted && c == '\\') { put('\\'); put('\\'); }
      else if (quoted && c == '"') { put('\\'); put('"'); }
      else if (quoted && c == '\n') { put('\\'); put('n'); }
      else if (quoted && c == '\r') { put('\\'); put('r'); }
      else if (quoted && c == '\t') { put('\\'); put('t'); }
      else cp(c);
    }
    if (quoted) put('"');
  }
};
TP_FN uint32_t dec_digits(uint32_t v) { uint32_t d = 1; while (v >= 10) { v /= 10; ++d; } return d; }

// frame modes of emit
enum : uint32_t { M_ROOT = 0, M_OBJ = 1, M_LIST_ITEM = 2, M_ROW = 3, M_ARR_ITEMS = 4, M_ARR_INLINE = 5, M_ARR_COL = 6, M_DEAD = 7 /* empty container */ };

// A non-object element arrives in an array whose first element is an object (row0 = 1 + its token index, row0_n its member
// count).  toon._try_columnar_encoding would call .keys() on it unless an earlier row already returned None.
TP_FN uint32_t nondict_element(uint32_t afl, uint32_t row0, uint32_t row0_n) {
  afl &= ~C_ALL_OBJ;
  if (row0 && !(afl & C_ND_SEEN)) {
    afl |= C_ND_SEEN;
    if ((afl & C_KEYSET_OK) && (afl & (C_ROW0_SIMPLE | C_R0KEYS)) && row0_n != 0 && row0_n != UNSET) afl |= C_CRASH;
  }
  return afl;
}
TP_FN bool key_equals(const uint8_t* s, const GTok r, const uint8_t* b, uint32_t len) {
  if (gt_kind(r.w) != K_KEY || gt_len(r.w) != len) return false;
  const uint8_t* a = s + r.pos;
  for (uint32_t i = 0; i < len; ++i) if (a[i] != b[i]) return false;
  return true;
}

// rare paths of the classification batch, kept out of line (instruction-cache footprint of the hot loop)
TP_SLOW uint32_t scalar_end(const uint8_t* s, uint32_t n, uint32_t e) {
  while (e < n) { const uint32_t k = byte_class(s[e]); if (k & (BC_STRUCT | BC_WS | BC_QUOTE)) break; ++e; }
  return e;
}
TP_SLOW bool string_slow(const uint8_t* s, uint32_t n, uint32_t pos, uint32_t len, uint32_t* sf) {
  uint32_t p = pos - 1, h = 0;
  return cfj::parse_string(s, n, &p, sf, &h) && p == pos + len + 1;
}

TP_FN uint32_t utf8_first_cp(const uint8_t* b) {
  const uint32_t c = b[0];
  if (c < 0x80) return c;
  const uint32_t need = c >= 0xF0 ? 3u : c >= 0xE0 ? 2u : 1u;
  uint32_t cp = c & (0x3Fu >> need);
  for (uint32_t k = 1; k <= need; ++k) cp = (cp << 6) | (b[k] & 0x3Fu);
  return cp;
}
static const uint32_t LONG_HI = 96;      // non-ASCII / escaped strings at least this long: escapes checked by the whole warp, UTF-8 by utf8_bad

// Escapes of a long string s[a .. a+len), whole warp: every unescaped backslash must start one of JSON's two-character escapes
// (a \uXXXX escape makes the caller take the sequential validator: its code point decides the predicates).
// Returns a bit set: 1 invalid escape, 2 some \u escape, 4 an escape TOON writes differently (\/ \b \f), 8 \b or \f (a control
// character toon._quote_string rejects).
enum : uint32_t { XE_BAD = 1, XE_U = 2, XE_COMPLEX = 4, XE_CTRL = 8 };
TP_SLOW uint32_t warp_escapes(const uint8_t* s, uint32_t a, uint32_t len) {
  const uint32_t l = tpw::lane();
  uint32_t res = 0, e_in = 0, pend = 0;                 // e_in: the chunk's first byte is escaped; pend: it is an escape's code character
  for (uint32_t base = 0; base < len; base += 32) {
    const uint32_t i = base + l;
    const uint32_t c = i < len ? (uint32_t)s[a + i] : 0u;
    const uint32_t bs = tpw::ballot(c == '\\');
    uint32_t e_out;
    const uint32_t escaped = find_escaped(bs, e_in, &e_out);
    const uint32_t start = bs & ~escaped;                // backslashes that open an escape
    const uint32_t code = (start << 1) | pend;            // their code characters
    if ((code >> l) & 1u) {
      if (i >= len) res |= XE_BAD;                        // the string ends on a lone backslash (cannot happen: the quote would be escaped)
      else if (c == 'u') res |= XE_U;
      else if (c == '/') res |= XE_COMPLEX;
      else if (c == 'b' || c == 'f') res |= XE_COMPLEX | XE_CTRL;
      else if (!(c == '"' || c == '\\' || c == 'n' || c == 'r' || c == 't')) res |= XE_BAD;
    }
    pend = start >> 31;
    e_in = e_out;
  }
  if (pend) res |= XE_BAD;
  for (uint32_t d = 16; d; d >>= 1) res |= tpw::shfl(res, (l + d) & 31u);   // OR over the lanes (butterfly by rotation)
  return res;
}

// ----------------------------------------------------------------------------------------------------------------------
// tokenize, classification batch: raw tokens ring[head .. head+m) -> validated GTok toks[ntok ..); la_ncolon = colons in
// front of the token that follows the batch (a string followed by a colon is a key)
// ----------------------------------------------------------------------------------------------------------------------
struct TokState { uint32_t ntok; int status; };
// the ring's meta words live behind the tokenizer's source window in the staging buffer (its positions and lengths in Shared)
TP_FN uint32_t* ring_meta(uint8_t* stage) { return reinterpret_cast<uint32_t*>(stage + WIN); }
TP_FN const uint32_t* ring_meta(const uint8_t* stage) { return reinterpret_cast<const uint32_t*>(stage + WIN); }
// win[0..WIN) holds the unit's bytes [wlo, wlo + WIN) (unit positions; wlo may be "negative" = wrapped, see in_window)
TP_FN const uint8_t* in_window(const uint8_t* s, const uint8_t* win, uint32_t wlo, uint32_t pos, uint32_t len) {
  const uint32_t d = pos - wlo;                       // wraps to a huge value when pos < wlo
  return (d < WIN && len <= WIN - d) ? win + d : s + pos;
}
// Strict UTF-8 over the step's bytes in the window (stage[1024, 2048)), lane l on its 32 bytes and the three in front of them (the
// previous step's last ones for lane 0: stage[1021, 1024)); bytes outside [lead, vend) count as blanks.  A byte must be a
// continuation byte exactly when one of the three bytes before it is a lead that reaches it, leads are C2..F4, and the second byte
// of E0 / ED / F0 / F4 sequences is range-checked (no overlongs, no surrogates, nothing above U+10FFFF): what cfj::parse_string
// checks one code point at a time.  The first failing position of the unit goes to sh.utf8_bad; tok_batch raises it at the
// string that holds it, so the unit's status is the one a string-by-string check gives.  (Outside strings, a non-ASCII byte
// fails its scalar run anyway.)
// SWAR, four bytes per step of the lane's walk: 0x80 in every byte of x (bytes b0) that breaks a rule, pw = the word in front.
TP_FN uint32_t utf8_bad_bytes(uint32_t x, uint32_t pw) {
  const uint32_t p1 = (x << 8) | (pw >> 24), p2 = (x << 16) | (pw >> 16), p3 = (x << 24) | (pw >> 8);   // b1, b2, b3 of each byte
  const uint32_t cont = swar_eq(x & 0xC0C0C0C0u, 0x80u);
  const uint32_t must = swar_eq(p1 & 0xC0C0C0C0u, 0xC0u) | swar_eq(p2 & 0xE0E0E0E0u, 0xE0u) | swar_eq(p3 & 0xF0F0F0F0u, 0xF0u);
  // leads C0, C1 and F5..FF (F5 and up: the low seven bits plus 0x0B carry into bit 7)
  const uint32_t bad_lead = x & ~cont & (swar_eq(x & 0xFEFEFEFEu, 0xC0u) | (x & ((x & 0x7F7F7F7Fu) + 0x0B0B0B0Bu)));
  // second bytes: after E0 at least A0 (bit 5), after ED at most 9F, after F0 at least 90 (bit 4 or 5), after F4 at most 8F
  const uint32_t b5 = x << 2, b45 = (x << 2) | (x << 3);
  const uint32_t second = cont & ((swar_eq(p1, 0xE0u) & ~b5) | (swar_eq(p1, 0xEDu) & b5) | (swar_eq(p1, 0xF0u) & ~b45) | (swar_eq(p1, 0xF4u) & b45));
  return ((cont ^ must) | bad_lead | second) & 0x80808080u;
}
// the bytes of x (at virtual offsets [pos, pos + 4)) outside [lo, hi) -> blanks
TP_SLOW uint32_t utf8_blank(uint32_t x, int64_t pos, uint32_t lo, uint32_t hi) {
  for (uint32_t j = 0; j < 4; ++j)
    if (pos + j < (int64_t)lo || pos + j >= (int64_t)hi) x = (x & ~(0xFFu << (8 * j))) | (0x20u << (8 * j));
  return x;
}
TP_FN void step_utf8_walk(const uint8_t* stage, Shared& sh, uint32_t v, uint32_t lead, uint32_t vend, bool mine) {
  const uint32_t l = tpw::lane();
  uint32_t first = UNSET;
  if (mine) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(stage + 1024 + 32 * l);
    const bool edge = v < lead + 4 || v + 32 > vend;         // some byte of the lane or of the word in front is not the unit's
    uint32_t pw = p[-1];                                     // lane 0: the previous step's last word
    if (edge) pw = utf8_blank(pw, (int64_t)v - 4, lead, vend);
#pragma unroll 1
    for (uint32_t k = 0; k < 8; ++k) {
      uint32_t x = p[k];
      if (edge) x = utf8_blank(x, (int64_t)v + 4 * k, lead, vend);
      const uint32_t bad = utf8_bad_bytes(x, pw);
      if (bad) { first = v + 4 * k + ((tpw::ffs(bad) - 1) >> 3) - lead; break; }
      pw = x;
    }
  }
  for (uint32_t d = 16; d; d >>= 1) { const uint32_t o = tpw::shfl(first, (l + d) & 31u); first = o < first ? o : first; }
  if (l == 0 && sh.utf8_bad == UNSET) sh.utf8_bad = first;
  tpw::sync();
}
// ASCII steps (the common case) pay two shared loads, a shuffle and a vote; only steps with a non-ASCII byte walk their bytes.
// (Out of line, the walk measured slower on every payload shape: the call spills the tokenizer's carries around it.)
TP_FN void step_utf8(const uint8_t* stage, Shared& sh, uint32_t v, uint32_t lead, uint32_t vend) {
  const uint32_t l = tpw::lane();
  const uint4 a = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l), b = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l + 16);
  const uint32_t hi = (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) & 0x80808080u;
  uint32_t tail = tpw::shfl_up(b.w, 1);               // the three bytes in front of the lane (their lead bytes may reach into it)
  if (l == 0) tail = *reinterpret_cast<const uint32_t*>(stage + 1020);
  const bool mine = hi != 0 || (tail & 0x80808000u) != 0;
  if (tpw::any(mine)) step_utf8_walk(stage, sh, v, lead, vend, mine);
}

TP_FN void tok_batch(const uint8_t* s, uint32_t n, GTok* toks, uint32_t tok_cap, Shared& sh, TokState& st, uint32_t head, uint32_t m, uint32_t la_ncolon,
                     const uint8_t* win, uint32_t wlo) {
  const uint32_t l = tpw::lane();
  const bool act = l < m;
  uint32_t pos = 0, len = 0, meta = 0;
  if (act) { const uint32_t r = (head + l) & (RING - 1); pos = sh.ring_pos[r]; len = sh.ring_len[r]; meta = ring_meta(win)[r]; }
  uint32_t kind = meta & RM_KIND;
  const uint32_t ncomma = (meta >> RM_NCOMMA_SH) & 3u, ncolon = (meta >> RM_NCOLON_SH) & 3u;
  uint32_t nxt_ncolon = tpw::shfl_down(ncolon, 1);
  if (l + 1 >= m) nxt_ncolon = la_ncolon;
  bool bad = false, unsup = false, long_hi = false;
  uint32_t fb = 0, fl = 0;
  const bool isK = act && kind == K_STR && ncolon == 0 && nxt_ncolon >= 1;
  if (act && kind == K_NUM) {                       // scalar run starting at pos
    if (meta & RM_OPENEND) len = scalar_end(s, n, pos + len) - pos;        // the run left its lane and the next: find its end
    const uint8_t* b = in_window(s, win, wlo, pos, len);
    const uint32_t c0 = b[0];
    if (c0 == 't') { if (len == 4 && b[1] == 'r' && b[2] == 'u' && b[3] == 'e') kind = K_LIT; else bad = true; }
    else if (c0 == 'f') { if (len == 5 && b[1] == 'a' && b[2] == 'l' && b[3] == 's' && b[4] == 'e') kind = K_LIT; else bad = true; }
    else if (c0 == 'n') { if (len == 4 && b[1] == 'u' && b[2] == 'l' && b[3] == 'l') kind = K_LIT; else bad = true; }
    else if ((meta & RM_ALLDIGIT) && len < 19 && (len == 1 || c0 != '0')) { /* plain integer: the text is its own TOON form */ }
    else if (c0 == '-' || (c0 >= '0' && c0 <= '9')) {
      uint32_t p = 0, nf = 0;
      if (!cfj::scan_number(b, len, &p, &nf) || p != len) bad = true;
      else {
        uint32_t eoff, elen;
        if (num_canon(b, len, nf, &eoff, &elen)) { pos += eoff; len = elen; }
        else fb = FB_NUM_EXACT;                     // exact formatter: sequential encoder
      }
    } else bad = true;
  } else if (act && kind == K_STR) {
    // only the first / last bytes (and up to five for the reserved words) are looked at on the fast path
    const uint8_t* b = in_window(s, win, wlo, pos, len);
    if (len > GT_MAXLEN) fb = FB_TOO_LONG;
    else if ((meta & (RM_HI | RM_BS)) && len >= LONG_HI && !(b[0] >= '0' && b[0] <= '9')) long_hi = true;   // whole-warp validation below
    else if ((meta & (RM_BS | RM_HI)) || (len && b[0] >= '0' && b[0] <= '9')) {
      // escapes, non-ASCII or number-like candidates: the sequential validator decides (same function as json_toon.h)
      uint32_t sf = 0;
      if (!string_slow(s, n, pos, len, &sf)) bad = true;
      else if (isK) { if (sf & cfj::JF_ESC) fb = FB_KEY_ESCAPE; if (sf & cfj::JF_KEYOK) fl |= KF_KEYOK; }
      else {
        if (sf & cfj::JF_Q) fl |= SF_Q;
        if (sf & cfj::JF_CTRLERR) fl |= SF_CTRLERR;
        if ((sf & cfj::JF_ESC) && has_complex_escape(s + pos, len)) fl |= SF_ESCX;
      }
    } else {
      const bool res = is_reserved(b, len);
      if (isK) {
        const uint32_t f0 = len ? b[0] : 0u;
        const bool al = (f0 >= 'A' && f0 <= 'Z') || (f0 >= 'a' && f0 <= 'z') || f0 == '_';
        if (len && al && !(meta & RM_NONKEY) && !res) fl |= KF_KEYOK;
      } else if (len == 0 || res || (meta & RM_SPECIAL) || b[0] == ' ' || b[len - 1] == ' ') fl |= SF_Q;
    }
    if (isK) kind = K_KEY;
  }
  // long non-ASCII or escaped strings, one after the other: UTF-8 was checked step by step (Shared::utf8_bad, the first failing
  // position of the unit: a string that holds it, closing quote included, is not JSON; a failure in front of it stopped an earlier
  // batch), escapes by the whole warp; what is left of the predicates needs the first and the last code point only (no digit in
  // front: not number-like)
  TP_MARK(t_long);
  for (uint32_t lm = tpw::ballot(long_hi); lm; lm &= lm - 1) {
    const uint32_t j = tpw::ffs(lm) - 1;
    const uint32_t jpos = tpw::shfl(pos, j), jlen = tpw::shfl(len, j), jmeta = tpw::shfl(meta, j);
    const bool ok = !(jmeta & RM_HI) || sh.utf8_bad - jpos > jlen;
    const uint32_t xe = (jmeta & RM_BS) ? warp_escapes(s, jpos, jlen) : 0u;
    if (l == j) {
      if (!ok || (xe & XE_BAD)) bad = true;
      else if (xe & XE_U) {                              // \uXXXX: the decoded code points decide — sequential validator
        uint32_t sf = 0;
        if (!string_slow(s, n, pos, len, &sf)) bad = true;
        else if (isK) fb = FB_KEY_ESCAPE;
        else {
          if (sf & cfj::JF_Q) fl |= SF_Q;
          if (sf & cfj::JF_CTRLERR) fl |= SF_CTRLERR;
          if (has_complex_escape(s + pos, len)) fl |= SF_ESCX;
        }
      } else if (isK) { if (meta & RM_BS) fb = FB_KEY_ESCAPE; }   // (a key with non-ASCII bytes is never a valid unquoted key: fl stays 0)
      else if (meta & RM_BS) {
        // two-character escapes only: each decodes to a character that forces quotes (" \ \n \r \t, \b \f) except \/
        const uint8_t* g = s + pos;
        uint32_t q = len - 1;
        while (q && (g[q] & 0xC0u) == 0x80u) --q;
        bool quoting = (meta & RM_SPECIAL) || (xe & XE_CTRL) != 0;
        if (!quoting) {                                  // any escape other than \/ ?  (scan by this lane only when still undecided)
          for (uint32_t i = 0; i + 1 < len; ++i) if (g[i] == '\\') { if (g[i + 1] != '/') { quoting = true; break; } ++i; }
        }
        const uint32_t fc = g[0] == '\\' ? (g[1] == '/' ? (uint32_t)'/' : 0u) : utf8_first_cp(g);      // 0: an escape that quotes anyway
        const bool last_esc = q >= 1 && len >= 2 && ((g[len - 2] == '\\') && true);                     // conservatively handled below
        uint32_t lc = utf8_first_cp(g + q);
        (void)last_esc;
        if (quoting || (fc && cfj::is_pyspace(fc)) || cfj::is_pyspace(lc)) fl |= SF_Q;
        if (xe & XE_CTRL) fl |= SF_CTRLERR | SF_Q;
        if (xe & XE_COMPLEX) fl |= SF_ESCX;
      } else {
        const uint8_t* g = s + pos;
        uint32_t q = len - 1;
        while (q && (g[q] & 0xC0u) == 0x80u) --q;
        if ((meta & RM_SPECIAL) || cfj::is_pyspace(utf8_first_cp(g)) || cfj::is_pyspace(utf8_first_cp(g + q))) fl |= SF_Q;
      }
    }
  }
  TP_LAP(PH_TK_LONG, t_long);
  if (len > GT_MAXLEN) { if (kind == K_NUM || kind == K_LIT) unsup = true; else if (!fb) fb = FB_TOO_LONG; len = 0; }
  if (st.ntok + m > tok_cap) fb = FB_TOK_CAP;
  else if (act) { GTok t; t.pos = pos; t.w = gt_make(kind, fl, ncomma, ncolon, kind <= K_CLOSE_ARR ? 0u : len); toks[st.ntok + l] = t; }
  st.ntok += m;
  const bool any_bad = tpw::any(bad), any_unsup = tpw::any(unsup);
  const uint32_t fbm = tpw::ballot(fb != 0);
  if (any_bad) st.status = TS_NOT_JSON;
  else if (any_unsup) st.status = TS_UNSUPPORTED;
  else if (fbm) st.status = TS_FALLBACK | (int)(tpw::shfl(fb, tpw::ffs(fbm) - 1) << 8);
}

// ----------------------------------------------------------------------------------------------------------------------
// tokenize: s[0..n) -> toks[0..*ntok_out).  Returns 0 or a TS_* status (warp-uniform).
// The unit is walked in 1 KiB steps on a 16-byte-aligned grid (the bytes in front of s and behind s+n that fall into the
// first / last step count as blanks; the caller guarantees 15 readable bytes in front and 1 KiB behind).
// ----------------------------------------------------------------------------------------------------------------------
TP_FN int tokenize(const uint8_t* s, uint32_t n, GTok* toks, uint32_t tok_cap, Shared& sh, uint8_t* stage, uint32_t* ntok_out) {
  const uint32_t l = tpw::lane();
  const uint32_t ltm = tpw::lt_mask();
  TokState st; st.ntok = 0; st.status = 0;
  uint32_t* rmeta = ring_meta(stage);
  const uint32_t lead = (uint32_t)((uintptr_t)s & 15u);
  const uint8_t* s0 = s - lead;                       // 16-byte aligned
  const uint32_t vend = n + lead;
  // carries between steps (warp-uniform), the one-bit ones and the open string's classes packed into one word (registers are what
  // limits the resident warps): bit 0 inside a string, bit 1 the next byte is escaped, bit 2 a scalar run continues, bits 4..7 classes
  uint32_t c_bits = 0, c_sep = 0 /* commas | colons << 16 since the last token */;
  uint32_t c_open = 0;                                // string open across steps: position of its opening quote
  uint32_t head = 0, rcount = 0;
  if (l == 0) sh.utf8_bad = UNSET;
  tpw::sync();
  for (uint32_t vb = 0; vb < vend; vb += 1024) {
    TP_MARK(t_tk);
    const uint32_t v = vb + 32 * l;                   // virtual offset of this lane's first byte
    // source window for the classification batches: [previous step | this step]
    {
      uint4 c0;                                       // lanes past the end: blanks
      c0.x = c0.y = c0.z = c0.w = 0x20202020u;
      uint4 c1 = c0;
      if (v < vend) { c0 = *reinterpret_cast<const uint4*>(s0 + v); c1 = *reinterpret_cast<const uint4*>(s0 + v + 16); }
      const uint4 p0 = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l), p1 = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l + 16);
      tpw::sync();
      *reinterpret_cast<uint4*>(stage + 32 * l) = p0; *reinterpret_cast<uint4*>(stage + 32 * l + 16) = p1;
      *reinterpret_cast<uint4*>(stage + 1024 + 32 * l) = c0; *reinterpret_cast<uint4*>(stage + 1024 + 32 * l + 16) = c1;
      tpw::sync();
    }
    step_utf8(stage, sh, v, lead, vend);
    TP_LAP(PH_TK_LOAD, t_tk);
    const uint32_t wlo = vb - 1024 - lead;             // unit position of stage[0] (wraps for the first step: nothing lies there)
    // The step's masks are rebuilt for every window of TOK_WIN tokens, from its bytes in the staging buffer and the carries at the
    // step's start, so that none of them is live across the classification batches (tok_batch): 80 registers hold either, not both.
    // A step with more than one window (over TOK_WIN tokens in 1 KiB) is rare; it pays the mask algebra once more per window.
    const uint32_t c_bits0 = c_bits, c_sep0 = c_sep, c_open0 = c_open;
    for (uint32_t done = 0;; done += TOK_WIN) {
      c_bits = c_bits0; c_sep = c_sep0; c_open = c_open0;
      uint32_t w[8];
      {
        const uint4 a = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l), b = *reinterpret_cast<const uint4*>(stage + 1024 + 32 * l + 16);
        w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
      }
      uint32_t valid = 0;
      if (v < vend) {
        valid = 0xFFFFFFFFu;
        if (v < lead) valid &= ~bits_below(lead - v);
        if (v + 32 > vend) valid &= bits_below(vend - v);
      }
      LaneMasks M;
      build_masks(w, M);
      if (valid != 0xFFFFFFFFu) {
        M.q &= valid; M.bs &= valid; M.ob &= valid; M.cb &= valid; M.curly &= valid; M.cm &= valid; M.co &= valid; M.ctrl &= valid; M.hi &= valid;
        M.special &= valid; M.nonkey &= valid; M.digit &= valid; M.ws |= ~valid;
      }
      // ---- escapes: which quotes are real
      uint32_t quotes = M.q;
      if (tpw::any(M.bs != 0) || (c_bits & 2u)) {
        uint32_t eo;
        find_escaped(M.bs, 0, &eo);
        uint32_t e_in = tpw::shfl_up(eo, 1);
        if (l == 0) e_in = (c_bits >> 1) & 1u;
        if (tpw::any(M.bs == 0xFFFFFFFFu)) {            // a whole lane of backslashes: its carry-out depends on its carry-in
          uint32_t e = (c_bits >> 1) & 1u;
          for (uint32_t k = 0; k < 32; ++k) {
            const uint32_t bk = tpw::shfl(M.bs, k);
            uint32_t ek;
            find_escaped(bk, e, &ek);
            if (l == k) e_in = e;
            e = ek;
          }
        }
        uint32_t eo2;
        const uint32_t escaped = find_escaped(M.bs, e_in, &eo2);
        quotes &= ~escaped;
        c_bits = (c_bits & ~2u) | (tpw::shfl(eo2, 31) << 1);
      }
      // ---- in-string state
      const uint32_t par = tpw::ballot(tpw::popc(quotes) & 1u);
      const uint32_t is_in = ((c_bits & 1u) ^ (tpw::popc(par & ltm) & 1u)) ? 0xFFFFFFFFu : 0u;   // this lane starts inside a string
      c_bits ^= tpw::popc(par) & 1u;
      uint32_t x = quotes;
      x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
      const uint32_t instr = x ^ is_in;                 // opening quote included, closing quote excluded
      const uint32_t openq = quotes & instr, closeq = quotes & ~instr;
      const uint32_t content = instr & ~openq;
      const bool ctl_bad = (M.ctrl & content) != 0;      // raw control character inside a string
      const uint32_t outside = ~instr & ~closeq;
      const uint32_t st_all = M.ob | M.cb | M.cm | M.co;
      const uint32_t comma_out = M.cm & outside, colon_out = M.co & outside;
      const uint32_t other = outside & ~st_all & ~M.ws;
      uint32_t prev_other = tpw::shfl_up(other >> 31, 1);
      if (l == 0) prev_other = (c_bits >> 2) & 1u;
      c_bits = (c_bits & ~4u) | (tpw::shfl(other >> 31, 31) << 2);
      const uint32_t starts = other & ~((other << 1) | prev_other);
      const uint32_t brackets = (M.ob | M.cb) & outside;
      const uint32_t T = brackets | closeq | starts;
      if (tpw::any(ctl_bad)) { st.status = TS_NOT_JSON; break; }
      const uint32_t m_special = M.special & content, m_nonkey = M.nonkey & content, m_hi = M.hi & content, m_bs = M.bs & content;
      // ---- separators in front of each lane's first token: segmented scan over the lanes
      uint32_t sep_in;
      {
        const uint32_t after = T ? ~bits_below(32 - tpw::clz(T)) : 0xFFFFFFFFu;
        uint32_t r = T ? 1u : 0u, vv = tpw::popc(comma_out & after) | (tpw::popc(colon_out & after) << 16);
  #pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
          const uint32_t r2 = tpw::shfl_up(r, d), v2 = tpw::shfl_up(vv, d);
          if (l >= d) { if (!r) vv += v2; r |= r2; }
        }
        uint32_t rin = tpw::shfl_up(r, 1), vin = tpw::shfl_up(vv, 1);
        if (l == 0) { rin = 0; vin = 0; }
        sep_in = vin + (rin ? 0u : c_sep);
        const uint32_t r31 = tpw::shfl(r, 31), v31 = tpw::shfl(vv, 31);
        c_sep = v31 + (r31 ? 0u : c_sep);
        if ((c_sep & 0xFFFFu) > 3u) c_sep = (c_sep & 0xFFFF0000u) | 3u;
        if ((c_sep >> 16) > 3u) c_sep = (c_sep & 0xFFFFu) | (3u << 16);
      }
      // ---- the string that is open at each lane's start: position of its opening quote + classes seen so far
      uint32_t so_pos, so_cls;
      {
        uint32_t r = quotes ? 1u : 0u, pp = 0, cc;
        if (quotes) {                                    // only meaningful when the lane ends inside a string it opened
          const uint32_t ob = 31 - tpw::clz(quotes), after = ~bits_below(ob + 1);
          pp = v + ob;
          cc = ((m_special & after) ? 1u : 0u) | ((m_nonkey & after) ? 2u : 0u) | ((m_hi & after) ? 4u : 0u) | ((m_bs & after) ? 8u : 0u);
        } else cc = (m_special ? 1u : 0u) | (m_nonkey ? 2u : 0u) | (m_hi ? 4u : 0u) | (m_bs ? 8u : 0u);
  #pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
          const uint32_t r2 = tpw::shfl_up(r, d), p2 = tpw::shfl_up(pp, d), c2 = tpw::shfl_up(cc, d);
          if (l >= d && !r) { pp = p2; cc |= c2; r = r2; }
        }
        uint32_t rin = tpw::shfl_up(r, 1), pin = tpw::shfl_up(pp, 1), cin = tpw::shfl_up(cc, 1);
        if (l == 0) { rin = 0; pin = 0; cin = 0; }
        so_pos = rin ? pin : c_open;
        so_cls = rin ? cin : (cin | (c_bits >> 4));
        const uint32_t r31 = tpw::shfl(r, 31), p31 = tpw::shfl(pp, 31), c31 = tpw::shfl(cc, 31);
        if (!r31) c_bits |= c31 << 4; else { c_open = p31; c_bits = (c_bits & 15u) | (c31 << 4); }
      }
      // ---- tokens of this lane through the ring (TOK_WIN at a time), one pass per token kind so that the lanes of a pass
      // run the same code: slot = rank of the token in text order, separators = commas / colons since the previous token
      const uint32_t cntT = tpw::popc(T);
      const uint32_t incl = tpw::scan_incl(cntT);
      const uint32_t lane_off = incl - cntT, total = tpw::shfl(incl, 31);
      uint32_t other_nx = tpw::shfl_down(other, 1);       // the next lane's scalar bytes: a run may continue there
      if (l == 31) other_nx = 0xFFFFFFFFu;                // unknown: treated as "continues" -> RM_OPENEND
      TP_LAP(PH_TK_MASKS, t_tk);
      if (done >= total) break;                          // no (more) tokens in this step
      {
        const uint32_t win = total - done > TOK_WIN ? TOK_WIN : total - done;
        const uint32_t lo = done > lane_off ? done - lane_off : 0u, hi = done + win > lane_off ? done + win - lane_off : 0u;   // ranks [lo, hi) of this lane
  #define TP_TOKEN_PROLOGUE(MASK)                                                                               \
        for (uint32_t tm = (MASK); tm;) {                                                                       \
          const uint32_t j = tpw::ffs(tm) - 1;                                                                  \
          tm &= tm - 1;                                                                                         \
          const uint32_t below = bits_below(j), rank = tpw::popc(T & below);                                    \
          if (rank < lo || rank >= hi) continue;                                                                \
          const uint32_t pt = T & below;                                                                        \
          uint32_t between = below, nc = sep_in & 0xFFFFu, nk = sep_in >> 16;                                   \
          if (pt) { between = below & ~bits_below(32 - tpw::clz(pt)); nc = 0; nk = 0; }                         \
          nc = sat3(nc + tpw::popc(comma_out & between));                                                       \
          nk = sat3(nk + tpw::popc(colon_out & between));                                                       \
          uint32_t meta = (nc << RM_NCOMMA_SH) | (nk << RM_NCOLON_SH), tpos = v + j - lead, tlen = 0;           \
          const uint32_t r = (head + rcount + (lane_off + rank - done)) & (RING - 1);
  #define TP_TOKEN_EPILOGUE                                                                                     \
          sh.ring_pos[r] = tpos; sh.ring_len[r] = tlen; rmeta[r] = meta;                                        \
        }
        TP_TOKEN_PROLOGUE(brackets)
          meta |= ((M.ob >> j) & 1u) ? (((M.curly >> j) & 1u) ? K_OPEN_OBJ : K_OPEN_ARR) : (((M.curly >> j) & 1u) ? K_CLOSE_OBJ : K_CLOSE_ARR);
        TP_TOKEN_EPILOGUE
        TP_TOKEN_PROLOGUE(closeq)
          const uint32_t qb = quotes & below;
          uint32_t span = below, cls = so_cls, op = so_pos;
          if (qb) { const uint32_t ob = 31 - tpw::clz(qb); op = v + ob; span = below & ~bits_below(ob + 1); cls = 0; }
          tpos = op + 1 - lead; tlen = (v + j) - op - 1;
          meta |= K_STR;
          if ((cls & 1u) | (m_special & span)) meta |= RM_SPECIAL;
          if ((cls & 2u) | (m_nonkey & span)) meta |= RM_NONKEY;
          if ((cls & 4u) | (m_hi & span)) meta |= RM_HI;
          if ((cls & 8u) | (m_bs & span)) meta |= RM_BS;
        TP_TOKEN_EPILOGUE
        TP_TOKEN_PROLOGUE(starts)
          meta |= K_NUM;
          const uint32_t e = ~other & ~bits_below(j + 1);          // first byte after the run, within the lane
          if (e) { tlen = tpw::ffs(e) - 1 - j; if (!(range_mask(j, j + tlen) & ~M.digit)) meta |= RM_ALLDIGIT; }
          else if (~other_nx) tlen = 32 - j + tpw::ffs(~other_nx) - 1;   // ends in the next lane
          else { tlen = 32 - j; meta |= RM_OPENEND; }
        TP_TOKEN_EPILOGUE
  #undef TP_TOKEN_PROLOGUE
  #undef TP_TOKEN_EPILOGUE
        rcount += win;
        tpw::sync();
        TP_LAP(PH_TK_RING, t_tk);
        while (rcount >= 33 && !st.status) {
          const uint32_t la = (rmeta[(head + 32) & (RING - 1)] >> RM_NCOLON_SH) & 3u;
          tok_batch(s, n, toks, tok_cap, sh, st, head, 32, la, stage, wlo);
          head += 32; rcount -= 32;
        }
        tpw::sync();
        TP_LAP(PH_TK_BATCH, t_tk);
      }
      if (st.status || done + TOK_WIN >= total) break;
    }
    if (st.status) break;
  }
  if (!st.status) {
    const uint32_t steps = (vend + 1023) / 1024;
    const uint32_t wlo = (steps - 1) * 1024 - 1024 - lead;
    if ((c_bits & 1u) || (c_sep & 0xFFFFu) || (c_sep >> 16)) st.status = TS_NOT_JSON;     // unterminated string / separators after the last token
    while (rcount && !st.status) {
      const uint32_t m = rcount > 32 ? 32u : rcount;
      const uint32_t la = rcount > 32 ? ((rmeta[(head + 32) & (RING - 1)] >> RM_NCOLON_SH) & 3u) : 0u;
      TP_PHASE(PH_TK_BATCH, tok_batch(s, n, toks, tok_cap, sh, st, head, m, la, stage, wlo));
      head += m; rcount -= m;
    }
  }
  *ntok_out = st.ntok;
  return st.status;
}

// ----------------------------------------------------------------------------------------------------------------------
// analyze: grammar + container stack over the token array; patches every opener with {child count, layout mode}
// ----------------------------------------------------------------------------------------------------------------------
struct AnState {
  uint32_t sp, root_cnt, last_was_key;
  int status;
};
TP_FN bool table_candidate(const Shared& sh, uint32_t top) {
  const uint32_t tfl = sh.cfl[top];
  return !(tfl & C_OBJ) && sh.cnt[top] > 0 && (tfl & C_KEYSET_OK) && (tfl & C_ROW0_SIMPLE) && !(tfl & C_ND_SEEN) && sh.row0_n[top] != UNSET && sh.row0_n[top] != 0;
}

// Generic mode: tokens [i, i+m) with one walk over their brackets.  Returns the number of tokens consumed: the walk stops in
// front of a row opener `{` of a table candidate (unless it is the batch's first token and `force`), so that table mode can
// take over.
template <bool RESOLVE_MIXED>
TP_FN uint32_t an_batch(const uint8_t* s, GTok* toks, uint32_t tok_cap, Shared& sh, AnState& st, uint32_t i, uint32_t m, bool force) {
  const uint32_t l = tpw::lane();
  const uint32_t ltm = tpw::lt_mask();
  const bool act = l < m;
  GTok t; t.pos = 0; t.w = K_CLOSE_ARR;
  if (act) t = toks[i + l];
  const uint32_t kind = gt_kind(t.w), ncomma = gt_nc(t.w), ncolon = gt_nk(t.w), len = gt_len(t.w), pos = t.pos;
  bool bad = false;
  uint32_t fb = 0;
  const bool isV = act && kind >= K_STR && kind != K_KEY;           // value that is not a container
  uint32_t evm = tpw::ballot(act && kind <= K_CLOSE_ARR);
  const uint32_t Km = tpw::ballot(act && kind == K_KEY), Vm = tpw::ballot(isV);
  uint32_t prevK = tpw::shfl_up(kind == K_KEY ? 1u : 0u, 1);
  if (l == 0) prevK = st.last_was_key;
  const uint32_t hash = (act && kind == K_KEY) ? fnv1a(s + pos, len) : 0u;   // every key of the batch at once (the walk below is serial)
  uint32_t sp = st.sp, root_cnt = st.root_cnt;
  bool ubad = false, uunsup = false;
  uint32_t ufb = 0;                  // warp-uniform verdicts of the walk
  uint32_t cur = 0, consumed = m;
  // The entry on top of the stack lives in (warp-uniform) registers during the walk; shared memory holds the entries below it and
  // is brought up to date when a container is pushed and at the end of the batch.
  uint32_t T_oi = 0, T_cnt = 0, T_cfl = 0, T_khb = 0, T_r0i = 0, T_r0n = UNSET, T_ow = 0;
  if (sp) { const uint32_t k = sp - 1; T_oi = sh.open_idx[k]; T_cnt = sh.cnt[k]; T_cfl = sh.cfl[k]; T_khb = sh.khbase[k]; T_r0i = sh.row0_idx[k]; T_r0n = sh.row0_n[k]; T_ow = sh.open_w[k]; }
  tpw::sync();                       // every lane has its copy before lane 0 may overwrite the slot (push / write-back)
  while (true) {
    const uint32_t e = evm ? tpw::ffs(evm) - 1 : m;
    const uint32_t run = range_mask(cur, e);
    if (run) {
      const bool inrun = (run >> l) & 1u;
      if (sp == 0) {                       // a scalar document: exactly one token, no separators
        if (inrun && (kind == K_KEY || ncomma || ncolon || root_cnt + tpw::popc(run & ltm) != 0)) bad = true;
        root_cnt += tpw::popc(run);
      } else {
        const uint32_t c0 = T_cnt;
        const bool isobj = (T_cfl & C_OBJ) != 0;
        const uint32_t Vr = Vm & run, Kr = Km & run;
        const uint32_t ord = c0 + tpw::popc(Vr & ltm);
        if (inrun) {
          if (isobj) {
            if (kind == K_KEY) { if (ncolon != 0 || ncomma != (ord > 0 ? 1u : 0u)) bad = true; }
            else if (ncolon != 1 || ncomma != 0 || !prevK) bad = true;
          } else if (kind == K_KEY || ncolon != 0 || ncomma != (ord > 0 ? 1u : 0u)) bad = true;
        }
        T_cnt = c0 + tpw::popc(Vr);
        if (!isobj && Vr) T_cfl = nondict_element(T_cfl, T_r0i, T_r0n);
        if (isobj && Kr) {
          // duplicate-key screen on the hashes (a repeated hash, real duplicate or not, goes to the sequential encoder)
          const uint32_t kb = T_khb;
          const bool mine = inrun && kind == K_KEY;
          if (mine) { if (kb + ord >= KH_CAP) fb = FB_KH_CAP; else { sh.kh[kb + ord] = hash; if (RESOLVE_MIXED) { sh.ring_pos[kb + ord] = pos; sh.ring_len[kb + ord] = len; } } }
          tpw::sync();
          if (mine && kb + ord < KH_CAP) for (uint32_t j = kb; j < kb + ord; ++j) if (sh.kh[j] == hash) { fb = FB_DUP_HASH; break; }
          // table detection: the keys of every later row against the first row's, position by position
          if (sp >= 2) {
            const uint32_t par = sp - 2, pfl = sh.cfl[par];
            if (!(pfl & C_OBJ) && (pfl & C_KEYSET_OK) && (pfl & C_ROW0_SIMPLE) && !(pfl & C_ND_SEEN) && sh.row0_n[par] != UNSET && T_oi + 1 != sh.row0_idx[par]) {
              const uint32_t r0 = sh.row0_idx[par] - 1, rn = sh.row0_n[par];
              bool mism = false, diff = false;
              if (mine) {
                if (ord >= rn || !key_equals(s, toks[r0 + 1 + 2 * ord], s + pos, len)) {
                  mism = true;
                  diff = true;                               // out of place: does the first row have this key at all?
                  for (uint32_t j = 0; j < rn; ++j) if (key_equals(s, toks[r0 + 1 + 2 * j], s + pos, len)) { diff = false; break; }
                }
              }
              const bool anym = tpw::any(mism), anyd = tpw::any(diff);
              if (anym) T_cfl = (T_cfl & ~C_ALIGNED) | (anyd ? C_DIFFSET : 0u);
            } else if (RESOLVE_MIXED && (pfl & C_R0KEYS) && (pfl & C_KEYSET_OK) && !(pfl & C_ND_SEEN)) {
              // a later row of an array whose first row is not simple: is each key one of the first row's?
              const uint32_t rn = sh.row0_n[par], r0k = sh.khbase[par] - rn;
              bool diff = false;
              if (mine) {
                const auto same = [&](uint32_t j) {            // hash and length screen in shared memory, then the bytes
                  if (sh.kh[r0k + j] != hash || sh.ring_len[r0k + j] != len) return false;
                  const uint8_t* a = s + sh.ring_pos[r0k + j];
                  for (uint32_t q = 0; q < len; ++q) if (a[q] != s[pos + q]) return false;
                  return true;
                };
                if (ord >= rn || !same(ord)) {
                  diff = true;
                  for (uint32_t j = 0; j < rn; ++j) if (same(j)) { diff = false; break; }
                }
              }
              if (tpw::any(diff)) T_cfl |= C_DIFFSET;
            }
          }
          tpw::sync();
        }
      }
    }
    if (e >= m) break;
    // ---- the bracket at lane e
    const uint32_t ek = tpw::shfl(kind, e), ew = tpw::shfl(t.w, e), eprevK = tpw::shfl(prevK, e);
    const uint32_t ecomma = gt_nc(ew), ecolon = gt_nk(ew);
    const uint32_t eidx = i + e;
    if (ek <= K_OPEN_ARR) {
      uint32_t newkb = 0;
      bool item_head = false;
      if (sp == 0) { if (ecomma || ecolon || root_cnt) ubad = true; ++root_cnt; }
      else {
        const uint32_t ord = T_cnt;
        const bool isobj = (T_cfl & C_OBJ) != 0;
        if (ek == K_OPEN_OBJ && (e > 0 || !force) && !isobj && T_cnt > 0 && (T_cfl & C_KEYSET_OK) && (T_cfl & C_ROW0_SIMPLE) && !(T_cfl & C_ND_SEEN) &&
            T_r0n != UNSET && T_r0n != 0) { consumed = e; break; }   // a table row: table mode takes it from here
        if (isobj) { if (ecolon != 1 || ecomma != 0 || !eprevK) ubad = true; }
        else if (ecolon != 0 || ecomma != (ord > 0 ? 1u : 0u)) ubad = true;
        T_cfl &= ~C_ALL_SIMPLE;
        if (isobj) T_cfl &= ~C_VALS_SIMPLE;
        else if (ek == K_OPEN_ARR) T_cfl = nondict_element(T_cfl, T_r0i, T_r0n);
        newkb = T_khb + (isobj ? ord + 1 : 0u);
        T_cnt = ord + 1;
        if (!isobj && ord == 0 && ek == K_OPEN_OBJ) T_r0i = eidx + 1;
        if (RESOLVE_MIXED) item_head = ek == K_OPEN_ARR && isobj && ord == 0 && sp >= 2 && !(sh.cfl[sp - 2] & C_OBJ);
      }
      if (sp >= MAXD) { uunsup = true; break; }
      if (sp && l == 0) { const uint32_t k = sp - 1; sh.open_idx[k] = T_oi; sh.cnt[k] = T_cnt; sh.cfl[k] = T_cfl; sh.khbase[k] = T_khb; sh.row0_idx[k] = T_r0i; sh.row0_n[k] = T_r0n; sh.open_w[k] = T_ow; }
      T_oi = eidx; T_cnt = 0; T_khb = newkb < KH_CAP ? newkb : KH_CAP;
      T_cfl = ek == K_OPEN_OBJ ? (C_OBJ | C_ALIGNED | C_VALS_SIMPLE) : (C_ALL_SIMPLE | C_ALL_OBJ | C_KEYSET_OK | C_ROWS_SIMPLE | (item_head ? C_ITEM_HEAD : 0u));
      T_r0i = 0; T_r0n = UNSET; T_ow = gt_make(ek, 0, ecomma, ecolon, 0);
      ++sp;
      tpw::sync();
    } else {
      if (sp == 0) { ubad = true; break; }
      const uint32_t tfl = T_cfl, nn = T_cnt, oi = T_oi;
      const bool isobj = (tfl & C_OBJ) != 0;
      if ((ek == K_CLOSE_OBJ) != isobj || ecomma || ecolon) ubad = true;
      if (nn > GT_MAXLEN) ufb = FB_TOO_LONG;
      uint32_t pk, pf;
      if (isobj) { pk = K_OPEN_OBJ; pf = 0; }
      else {
        const bool col = (tfl & C_ALL_OBJ) && (tfl & C_KEYSET_OK) && (tfl & C_ROWS_SIMPLE) && T_r0n != 0;
        const uint32_t mode = nn == 0 ? AM_EMPTY : col ? AM_COLUMNAR : (tfl & C_ALL_SIMPLE) ? AM_INLINE : AM_ITEMS;
        if (col && (tfl & C_PERMUTED)) ufb = FB_ROW_ORDER;          // the rows need a gather: sequential encoder
        uint32_t xf = 0;
        // the second pass leaves the verdict open only for a first row whose keys were not kept (too many open keys), unless a row
        // count already differed
        if (T_r0i && !(tfl & C_ALL_OBJ))
          xf = (tfl & C_CRASH) ? AF_CRASH : (!(tfl & (C_ROW0_SIMPLE | C_R0KEYS)) && (!RESOLVE_MIXED || (tfl & C_KEYSET_OK)) && T_r0n != 0) ? AF_MIXED : 0u;
        pk = K_OPEN_ARR; pf = mode | xf;
      }
      if (l == 0 && oi < tok_cap) toks[oi].w = gt_patch(T_ow, pk, pf, nn & GT_MAXLEN);
      --sp;
      if (sp) {                                                      // the parent comes back into the registers
        const uint32_t k = sp - 1;
        T_oi = sh.open_idx[k]; T_cnt = sh.cnt[k]; T_cfl = sh.cfl[k]; T_khb = sh.khbase[k]; T_r0i = sh.row0_idx[k]; T_r0n = sh.row0_n[k]; T_ow = sh.open_w[k];
        tpw::sync();
        if (isobj && !(T_cfl & C_OBJ)) {                             // an object element of an array closed: table bookkeeping
          if (!(tfl & C_VALS_SIMPLE)) T_cfl &= ~C_ROWS_SIMPLE;
          if (oi + 1 == T_r0i) {                                     // the first row
            if (tfl & C_VALS_SIMPLE) T_cfl |= C_ROW0_SIMPLE;
            else if (RESOLVE_MIXED && (T_cfl & C_ITEM_HEAD) && nn != 0 && T_khb + 2 * nn <= KH_CAP) { T_cfl |= C_R0KEYS; T_khb += nn; }   // keep its keys
            T_r0n = nn;
          } else if (T_r0n != UNSET && (T_cfl & C_KEYSET_OK) && !(T_cfl & C_ND_SEEN)) {
            // same key set?  (no duplicate keys here — those went to the sequential encoder — so equal counts + every key found = equal sets)
            if (nn != T_r0n || (tfl & C_DIFFSET)) T_cfl &= ~C_KEYSET_OK;
            else if (!(tfl & C_ALIGNED)) T_cfl |= C_PERMUTED;
          }
        }
      }
    }
    cur = e + 1;
    evm &= evm - 1;
  }
  if (sp && l == 0) { const uint32_t k = sp - 1; sh.open_idx[k] = T_oi; sh.cnt[k] = T_cnt; sh.cfl[k] = T_cfl; sh.khbase[k] = T_khb; sh.row0_idx[k] = T_r0i; sh.row0_n[k] = T_r0n; sh.open_w[k] = T_ow; }
  tpw::sync();
  st.sp = sp; st.root_cnt = root_cnt;
  if (consumed) st.last_was_key = tpw::shfl(kind == K_KEY ? 1u : 0u, consumed - 1);
  // verdicts of lanes past the stop point do not count (their tokens are walked again)
  const uint32_t live = bits_below(consumed);
  const bool any_bad = (tpw::ballot(bad) & live) != 0 || ubad;
  const uint32_t fbm = tpw::ballot(fb != 0) & live;
  if (any_bad) st.status = TS_NOT_JSON;
  else if (uunsup) st.status = TS_UNSUPPORTED;
  else if (fbm) st.status = TS_FALLBACK | (int)(tpw::shfl(fb, tpw::ffs(fbm) - 1) << 8);
  else if (ufb) st.status = TS_FALLBACK | (int)(ufb << 8);
  return consumed;
}

// Table mode: token i opens a row of the array on top of the stack whose first row (rn members, primitives only) closed.
// Lane r checks row r against the first row's token pattern; returns the number of leading rows that conform (each of
// S = 2 + 2 rn tokens) after patching their openers and counting them as children.  *staged_only: every row the round took
// conforms, and the round was only cut short because the rows behind them did not fit the staging buffer.
TP_FN uint32_t an_rows(const uint8_t* s, GTok* toks, uint32_t ntok, Shared& sh, uint8_t* stage, AnState& st, uint32_t i, bool* staged_only) {
  const uint32_t l = tpw::lane();
  const uint32_t top = st.sp - 1;
  const uint32_t rn = sh.row0_n[top], r0 = sh.row0_idx[top] - 1, S = 2 + 2 * rn;
  const uint32_t avail = (ntok - i) / S;
  uint32_t R = avail > 32 ? 32u : avail;
  const uint32_t R0 = R;
  const uint32_t t0 = i + l * S;
  // source bytes of the candidate rows -> staging buffer (as many leading rows as fit)
  const uint32_t a0 = toks[i].pos;
  uint32_t rend = l < R ? toks[t0 + S - 1].pos + 1 : 0xFFFFFFFFu;
  const uint32_t fits = tpw::ballot(l < R && rend >= a0 && rend - a0 <= STAGE - 32);
  const uint32_t Rf = fits == 0xFFFFFFFFu ? 32u : tpw::ffs(~fits) - 1;
  const uint8_t* sb = s;                               // base such that sb + pos addresses the row bytes
  if (Rf) {
    R = Rf;
    const uint32_t a1 = tpw::shfl(rend, R - 1);
    sb = stage - stage_load(stage, s, a0, a1, *reinterpret_cast<StageBar*>(&sh.sbar_bar));
  }
  bool ok = l < R;
  if (ok) {
    const uint32_t w0 = toks[t0].w, wc = toks[t0 + S - 1].w;
    ok = gt_kind(w0) == K_OPEN_OBJ && gt_nc(w0) == 1 && gt_nk(w0) == 0 && gt_kind(wc) == K_CLOSE_OBJ && gt_nc(wc) == 0 && gt_nk(wc) == 0;
    for (uint32_t kb = 0; kb < rn && ok; kb += 4) {            // four members per step: their token loads are issued together
      GTok a[4]; uint32_t vw[4];
#pragma unroll
      for (uint32_t q = 0; q < 4; ++q) { const uint32_t k = kb + q < rn ? kb + q : rn - 1; a[q] = toks[t0 + 1 + 2 * k]; vw[q] = toks[t0 + 2 + 2 * k].w; }
#pragma unroll
      for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t k = kb + q < rn ? kb + q : rn - 1;
        ok = ok && gt_nc(a[q].w) == (k ? 1u : 0u) && gt_nk(a[q].w) == 0 && gt_kind(vw[q]) >= K_STR && gt_kind(vw[q]) != K_KEY && gt_nc(vw[q]) == 0 &&
             gt_nk(vw[q]) == 1 && gt_kind(a[q].w) == K_KEY && a[q].pos >= a0 && a[q].pos + gt_len(a[q].w) <= rend &&
             key_equals(s, toks[r0 + 1 + 2 * k], sb + a[q].pos, gt_len(a[q].w));
      }
    }
  }
  const uint32_t good = tpw::ballot(ok);
  const uint32_t ngood = good == 0xFFFFFFFFu ? 32u : tpw::ffs(~good) - 1;
  if (l < ngood) toks[t0].w = gt_patch(toks[t0].w, K_OPEN_OBJ, 0, rn);
  if (ngood) {
    tpw::sync();
    if (l == 0) sh.cnt[top] = sh.cnt[top] + ngood;
    tpw::sync();
    st.last_was_key = 0;
  }
  *staged_only = ngood == R && R < R0;
  return ngood;
}

template <bool RESOLVE_MIXED>
TP_FN int analyze(const uint8_t* s, GTok* toks, uint32_t ntok, uint32_t tok_cap, Shared& sh, uint8_t* stage) {
  AnState st; st.sp = 0; st.root_cnt = 0; st.last_was_key = 0; st.status = 0;
  uint32_t i = 0;
  bool force = false;
  while (i < ntok && !st.status) {
    if (!force && st.sp > 0 && table_candidate(sh, st.sp - 1) && gt_kind(toks[i].w) == K_OPEN_OBJ) {
      const uint32_t S = 2 + 2 * sh.row0_n[st.sp - 1];
      bool staged_only;
      uint32_t g;
      TP_PHASE(PH_AN_TABLE, g = an_rows(s, toks, ntok, sh, stage, st, i, &staged_only));
      i += g * S;
      if (g < 32 && !staged_only) force = true;       // the next row (if it is one) does not conform: generic walk
      continue;
    }
    const uint32_t m = ntok - i > 32 ? 32u : ntok - i;
    uint32_t c;
    TP_PHASE(PH_AN_GENERIC, c = an_batch<RESOLVE_MIXED>(s, toks, tok_cap, sh, st, i, m, force));
    force = false;
    i += c;
  }
  if (!st.status && (st.sp != 0 || st.root_cnt != 1)) st.status = TS_NOT_JSON;
  return st.status;
}

// ----------------------------------------------------------------------------------------------------------------------
// emit: tokens -> TOON text
// ----------------------------------------------------------------------------------------------------------------------
struct Piece {
  uint32_t l0;        // literal before the line break: 0 or ':'
  uint32_t nl;        // 1 = line break + `spaces` blanks, 2 = blanks only (first line of the document)
  uint32_t spaces;
  uint32_t l1, l1n;   // literal after the indentation (up to 2 chars, low byte first)
  uint32_t body;      // B_*
  uint32_t tail;      // array header tail: T_*
};
enum : uint32_t { B_NONE = 0, B_SPAN = 1, B_QSPAN = 2, B_ESCX = 3, B_QESCX = 4, B_ARR = 5 };
enum : uint32_t { T_COLON = 0, T_COLON_SP = 1, T_COLUMNAR = 2 };
TP_FN uint32_t lit2(char a, char b) { return (uint32_t)(uint8_t)a | ((uint32_t)(uint8_t)b << 8); }

struct EmState {
  uint32_t sp, ocur;
  int status;
  bool over;
  uint32_t col_first, col_rows, col_rn;    // set when a batch stopped behind a table header: first row token, rows, members per row
};

// text of one primitive value token (string / number / literal) as a table cell: length, then bytes
TP_FN uint32_t cell_len(const uint8_t* s, const GTok t, uint32_t* err) {
  const uint32_t kind = gt_kind(t.w), fl = gt_flags(t.w), len = gt_len(t.w);
  if (kind != K_STR) return len;
  const bool q = (fl & SF_Q) != 0;
  if (q && (fl & SF_CTRLERR)) *err = TS_VALUE_ERROR;
  if (fl & SF_ESCX) return escx_len(s + t.pos, len, q);
  return len + (q ? 2u : 0u);
}
TP_FN void cell_put(Emit& em, const uint8_t* s, const GTok t) {
  const uint32_t kind = gt_kind(t.w), fl = gt_flags(t.w), len = gt_len(t.w);
  if (kind != K_STR) { em.span(s + t.pos, len); return; }
  const bool q = (fl & SF_Q) != 0;
  if (fl & SF_ESCX) { em.escx(s + t.pos, len, q); return; }
  if (q) em.put('"');
  em.span(s + t.pos, len);
  if (q) em.put('"');
}

static const uint32_t SPAN_LOADS = 8;     // long spans (em_batch): bytes each lane loads before it stores them

// Generic mode: tokens [i, i+m).  Returns the number consumed: the batch ends right behind the header of a table.
TP_FN uint32_t em_batch(const uint8_t* s, const GTok* toks, uint32_t ntok, uint8_t* out, uint32_t out_cap, Shared& sh, EmState& st, uint32_t i, uint32_t m,
                        bool report_errors) {
  const uint32_t l = tpw::lane();
  const uint32_t ltm = tpw::lt_mask();
  uint32_t* f_mode = sh.open_idx; uint32_t* f_cnt = sh.cnt; uint32_t* f_pre = sh.cfl; uint32_t* f_ind = sh.khbase;
  uint32_t sp = st.sp;
  bool act = l < m;
  GTok t; t.pos = 0; t.w = K_CLOSE_ARR;
  if (act) t = toks[i + l];
  const uint32_t kind = gt_kind(t.w), fl = gt_flags(t.w), len = gt_len(t.w);
  uint32_t nk = tpw::shfl_down(kind, 1);                         // kind of the following token
  if (l + 1 >= m) nk = i + m < ntok ? gt_kind(toks[i + m].w) : (uint32_t)K_CLOSE_ARR;
  Piece pc; pc.l0 = 0; pc.nl = 0; pc.spaces = 0; pc.l1 = 0; pc.l1n = 0; pc.body = B_NONE; pc.tail = T_COLON;
  uint32_t err = 0;                                             // per-lane TS_* error of this token
  const bool isV = act && kind >= K_STR && kind != K_KEY;
  uint32_t evm = tpw::ballot(act && kind <= K_CLOSE_ARR);
  const uint32_t Vm = tpw::ballot(isV);
  uint32_t cur = 0, consumed = m;
  st.col_rows = 0;
  // the frame on top of the stack lives in (warp-uniform) registers during the walk
  uint32_t F_mode = M_ROOT, F_pre = 0, F_ind = 0, F_cnt = 0;
  if (sp) { const uint32_t k = sp - 1; F_mode = f_mode[k]; F_pre = f_pre[k]; F_ind = f_ind[k]; F_cnt = f_cnt[k]; }
  tpw::sync();
  while (true) {
    const uint32_t e = evm ? tpw::ffs(evm) - 1 : m;
    const uint32_t run = range_mask(cur, e);
    if (run) {
      const bool inrun = (run >> l) & 1u;
      if (sp == 0) { if (inrun) pc.body = B_SPAN; }
      else {
        const uint32_t mode = F_mode, pre = F_pre, ind = F_ind, c0 = F_cnt;
        const uint32_t Vr = Vm & run;
        const uint32_t ord = c0 + tpw::popc(Vr & ltm);
        if (inrun) {
          if (kind == K_KEY) {
            if (mode == M_OBJ) { pc.nl = (pre == 0 && ord == 0 && sp == 1) ? 2u : 1u; pc.spaces = pre; pc.body = B_SPAN; }
            else if (mode == M_LIST_ITEM) {
              pc.nl = 1; pc.spaces = pre + (ord == 0 ? 2 * ind : 2 * (ind + 1));
              if (ord == 0) { pc.l1 = lit2('-', ' '); pc.l1n = 2; }
              pc.body = B_SPAN;
            }
          } else {
            pc.body = B_SPAN;
            if (mode == M_OBJ || mode == M_LIST_ITEM) { pc.l1 = lit2(':', ' '); pc.l1n = 2; }
            else if (mode == M_ROW || mode == M_ARR_INLINE) { if (ord > 0) { pc.l1 = ','; pc.l1n = 1; } }
            else if (mode == M_ARR_ITEMS) { pc.nl = 1; pc.spaces = pre + 2 * (ind + 1); pc.l1 = lit2('-', ' '); pc.l1n = 2; }
          }
        }
        F_cnt = c0 + tpw::popc(Vr);
      }
    }
    if (e >= m) break;
    const uint32_t ek = tpw::shfl(kind, e);
    if (ek <= K_OPEN_ARR) {
      const uint32_t ew = tpw::shfl(t.w, e), enk = tpw::shfl(nk, e);
      const uint32_t en = gt_len(ew), efl = gt_flags(ew);
      uint32_t pmode = M_ROOT, pre = 0, ind = 0, ord = 0;
      if (sp > 0) { pmode = F_mode; pre = F_pre; ind = F_ind; ord = F_cnt; F_cnt = ord + 1; }
      uint32_t nmode = M_DEAD, npre = 0, nind = 0;
      Piece q; q.l0 = 0; q.nl = 0; q.spaces = 0; q.l1 = 0; q.l1n = 0; q.body = B_NONE; q.tail = T_COLON;
      uint32_t eerr = 0;
      bool table = false;
      if (ek == K_OPEN_OBJ) {
        if (pmode == M_ROOT) { nmode = M_OBJ; npre = 0; nind = 0; }
        else if (pmode == M_OBJ) { q.l1 = ':'; q.l1n = 1; nmode = M_OBJ; npre = pre + 2; nind = ind + 1; }
        else if (pmode == M_ARR_ITEMS) {
          if (en == 0) { q.nl = 1; q.spaces = pre + 2 * (ind + 1); q.l1 = '-'; q.l1n = 1; }
          else { nmode = M_LIST_ITEM; npre = pre; nind = ind + 1; }
        } else if (pmode == M_LIST_ITEM) {
          if (en == 0) { q.l1 = lit2(':', ' '); q.l1n = 2; }
          else { q.l1 = ':'; q.l1n = 1; nmode = M_OBJ; npre = pre + 2 * (ind + 1) + 2; nind = ind + 2; }
        } else if (pmode == M_ARR_COL) { q.nl = 1; q.spaces = pre; nmode = M_ROW; }
        if (en == 0) nmode = M_DEAD;
      } else {
        const uint32_t amode = efl & 3u;
        uint32_t apre = pre, aind = ind;                           // arguments of begin_array
        bool col_on_hyphen = false;
        q.body = B_ARR;
        if (pmode == M_ARR_ITEMS) { const uint32_t ci = 2 * (ind + 1); q.nl = 1; q.spaces = pre + ci; q.l1 = lit2('-', ' '); q.l1n = 2; apre = pre + ci + 2; aind = ind + 2; }
        else if (pmode == M_LIST_ITEM) {
          const uint32_t fi = 2 * (ind + 1);
          if (en == 0) { q.l1 = lit2(':', ' '); q.l1n = 2; }
          else {
            if (ord == 0) {                                       // toon.py:400-404: columnar attempt without a type check
              if (enk != K_OPEN_OBJ) eerr = TS_ATTR_ERROR;
              else if (efl & AF_CRASH) eerr = TS_ATTR_ERROR;
              else if (efl & AF_MIXED) eerr = TS_FALLBACK | (FB_MIXED_ITEM << 8);
              else if (amode == AM_COLUMNAR) col_on_hyphen = true;
            }
            apre = pre + fi + 2; aind = ind + 2;
            if (!col_on_hyphen) { q.l0 = ':'; q.nl = 1; q.spaces = apre; }
          }
        }
        if (amode == AM_EMPTY) q.tail = T_COLON;
        else if (amode == AM_COLUMNAR) { q.tail = T_COLUMNAR; nmode = M_ARR_COL; npre = apre + 2; nind = aind; table = true; }
        else if (amode == AM_INLINE) { q.tail = T_COLON_SP; nmode = M_ARR_INLINE; }
        else { q.tail = T_COLON; nmode = M_ARR_ITEMS; npre = apre; nind = aind; }
        if (col_on_hyphen) npre = apre;
      }
      if (l == e) { pc = q; err = eerr; }
      if (sp >= MAXD) { st.status = TS_UNSUPPORTED; break; }
      if (sp && l == 0) { const uint32_t k = sp - 1; f_mode[k] = F_mode; f_pre[k] = F_pre; f_ind[k] = F_ind; f_cnt[k] = F_cnt; }
      F_mode = nmode; F_pre = npre; F_ind = nind; F_cnt = 0;
      ++sp;
      tpw::sync();
      if (table && !eerr) {                                        // rows are written one lane per row (em_rows)
        consumed = e + 1;
        st.col_first = i + e + 1; st.col_rows = en; st.col_rn = gt_len(toks[i + e + 1].w);
        break;
      }
    } else {
      --sp;
      if (sp) { const uint32_t k = sp - 1; F_mode = f_mode[k]; F_pre = f_pre[k]; F_ind = f_ind[k]; F_cnt = f_cnt[k]; tpw::sync(); }
    }
    cur = e + 1;
    evm &= evm - 1;
  }
  if (sp && l == 0) { const uint32_t k = sp - 1; f_mode[k] = F_mode; f_pre[k] = F_pre; f_ind[k] = F_ind; f_cnt[k] = F_cnt; }
  tpw::sync();
  st.sp = sp;
  if (st.status) return consumed;
  if (l >= consumed) { act = false; pc.l0 = 0; pc.nl = 0; pc.l1n = 0; pc.body = B_NONE; err = 0; }

  // ---- piece lengths
  uint32_t blen = 0;
  const uint8_t* src = s + t.pos;
  if (act && pc.body == B_SPAN) {
    if (kind == K_KEY) { if (!(fl & KF_KEYOK)) pc.body = B_QSPAN; }
    else if (kind == K_STR) {
      const bool q = (fl & SF_Q) != 0;
      if (q && (fl & SF_CTRLERR)) err = TS_VALUE_ERROR;
      pc.body = (fl & SF_ESCX) ? (q ? B_QESCX : B_ESCX) : (q ? B_QSPAN : B_SPAN);
    }
  }
  uint32_t hk = 0;                                              // columnar header: number of keys
  if (act) {
    if (pc.body == B_SPAN) blen = len;
    else if (pc.body == B_QSPAN) blen = len + 2;
    else if (pc.body == B_ESCX || pc.body == B_QESCX) blen = escx_len(src, len, pc.body == B_QESCX);
    else if (pc.body == B_ARR) {
      blen = 2 + dec_digits(len) + (pc.tail == T_COLON_SP ? 2u : 1u);
      if (pc.tail == T_COLUMNAR) {
        hk = gt_len(toks[i + l + 1].w);                         // members of the first row
        blen += 2 + (hk - 1);
        for (uint32_t j = 0; j < hk; ++j) blen += gt_len(toks[i + l + 2 + 2 * j].w);
      }
    }
  }
  const uint32_t plen = act ? ((pc.l0 ? 1u : 0u) + (pc.nl == 1 ? 1u : 0u) + (pc.nl ? pc.spaces : 0u) + pc.l1n + blen) : 0u;
  const uint32_t incl = tpw::scan_incl(plen);
  const uint32_t off = st.ocur + incl - plen;
  const uint32_t total = tpw::shfl(incl, 31);
  // first error / first overflow in token order
  const uint32_t errm = tpw::ballot(err != 0), ovm = tpw::ballot(plen && off + plen > out_cap);
  if (errm) {
    const uint32_t fe = tpw::ffs(errm) - 1;
    const bool ov_first = ovm && (tpw::ffs(ovm) - 1) < fe;
    if (report_errors || !(st.over || ov_first)) { st.status = (int)tpw::shfl(err, fe); return consumed; }
  }
  if (ovm) { st.over = true; if (!report_errors) { st.status = TS_NOT_SMALLER; return consumed; } }
  // ---- write
  const bool longspan = act && (pc.body == B_SPAN || pc.body == B_QSPAN) && len >= 64;
  if (act && plen) {
    Emit em; em.out = out; em.cap = out_cap; em.o = off;
    if (pc.l0) em.put(pc.l0);
    if (pc.nl == 1) em.put('\n');
    if (pc.nl) em.spaces(pc.spaces);
    if (pc.l1n >= 1) em.put(pc.l1 & 0xFF);
    if (pc.l1n >= 2) em.put((pc.l1 >> 8) & 0xFF);
    if (pc.body == B_SPAN) { if (!longspan) em.span(src, len); }
    else if (pc.body == B_QSPAN) { em.put('"'); if (!longspan) em.span(src, len); else em.o += len; em.put('"'); }
    else if (pc.body == B_ESCX || pc.body == B_QESCX) em.escx(src, len, pc.body == B_QESCX);
    else if (pc.body == B_ARR) {
      em.put('['); em.uint_dec(len); em.put(']');
      if (pc.tail == T_COLUMNAR) {
        em.put('{');
        for (uint32_t j = 0; j < hk; ++j) { const GTok k = toks[i + l + 2 + 2 * j]; if (j) em.put(','); em.span(s + k.pos, gt_len(k.w)); }
        em.put('}'); em.put(':');
      } else { em.put(':'); if (pc.tail == T_COLON_SP) em.put(' '); }
    }
  }
  uint32_t lm = tpw::ballot(longspan);
  while (lm) {                                                  // long spans: the whole warp copies
    const uint32_t j = tpw::ffs(lm) - 1;
    lm &= lm - 1;
    const uint32_t jpos = tpw::shfl(t.pos, j), jlen = tpw::shfl(len, j);
    const uint32_t jdst = tpw::shfl(off + plen - blen + (pc.body == B_QSPAN ? 1u : 0u), j);
    // SPAN_LOADS bytes per lane per round, every load issued before the round's stores: `out` may alias `s` as far as the compiler
    // knows, so a load behind a store waits for it, and one byte per round paid a full L2 round trip per 32 bytes of a long string
    for (uint32_t b = 0; b < jlen; b += 32 * SPAN_LOADS) {
      uint8_t v[SPAN_LOADS];
#pragma unroll
      for (uint32_t q = 0; q < SPAN_LOADS; ++q) { const uint32_t k = b + 32 * q + l; v[q] = k < jlen ? s[jpos + k] : (uint8_t)0; }
#pragma unroll
      for (uint32_t q = 0; q < SPAN_LOADS; ++q) { const uint32_t k = b + 32 * q + l; if (k < jlen && jdst + k < out_cap) out[jdst + k] = v[q]; }
    }
  }
  st.ocur += total;
  return consumed;
}

// Table mode: `rows` rows of rn members each (2 + 2 rn tokens per row, primitives only) starting at token `first`;
// every lane writes one row per round: line break, prefix, cells joined by commas.  The round's source bytes come in and its
// output goes out through the staging buffer (coalesced), as long as they fit.
TP_FN void em_rows(const uint8_t* s, const GTok* toks, uint8_t* out, uint32_t out_cap, Shared& sh, uint8_t* stage, EmState& st, bool report_errors) {
  const uint32_t l = tpw::lane();
  const uint32_t rn = st.col_rn, S = 2 + 2 * rn, pre = sh.cfl[st.sp - 1];     // f_pre of the table frame = row prefix
  uint32_t rb = 0;
  while (rb < st.col_rows) {
    uint32_t R = st.col_rows - rb > 32 ? 32u : st.col_rows - rb;
    const uint32_t r = rb + l;
    const uint32_t t0 = st.col_first + r * S;
    // stage the source bytes of as many leading rows of the round as fit
    const uint32_t a0 = toks[st.col_first + rb * S].pos;
    const uint32_t rend = l < R ? toks[t0 + S - 1].pos + 1 : 0xFFFFFFFFu;
    const uint32_t fits = tpw::ballot(l < R && rend >= a0 && rend - a0 <= ROW_SRC - 32);
    const uint32_t Rf = fits == 0xFFFFFFFFu ? 32u : tpw::ffs(~fits) - 1;
    const uint8_t* sb = s;
    if (Rf) {
      R = Rf;
      sb = stage - stage_load(stage, s, a0, tpw::shfl(rend, R - 1), *reinterpret_cast<StageBar*>(&sh.sbar_bar));
    } else R = 1;                                        // one over-long row at a time, straight from global memory
    const bool act = l < R;
    uint32_t plen = 0, err = 0;
    if (act) {
      plen = 1 + pre + (rn - 1);
      for (uint32_t kb = 0; kb < rn; kb += 4) {
        GTok c[4];
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) c[q] = toks[t0 + 2 + 2 * (kb + q < rn ? kb + q : rn - 1)];
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) if (kb + q < rn) plen += cell_len(sb, c[q], &err);
      }
    }
    const uint32_t incl = tpw::scan_incl(plen);
    const uint32_t off = st.ocur + incl - plen;
    const uint32_t total = tpw::shfl(incl, 31);
    const uint32_t errm = tpw::ballot(err != 0), ovm = tpw::ballot(plen && off + plen > out_cap);
    if (errm) {
      const uint32_t fe = tpw::ffs(errm) - 1;
      const bool ov_first = ovm && (tpw::ffs(ovm) - 1) < fe;
      if (report_errors || !(st.over || ov_first)) { st.status = (int)tpw::shfl(err, fe); return; }
    }
    if (ovm) { st.over = true; if (!report_errors) { st.status = TS_NOT_SMALLER; return; } }
    const bool staged_out = Rf && total <= ROW_OUT && !st.over;
    if (act) {
      Emit em;
      if (staged_out) { em.out = sh.row_out() - st.ocur; em.cap = st.ocur + ROW_OUT; }
      else { em.out = out; em.cap = out_cap; }
      em.o = off;
      em.put('\n');
      em.spaces(pre);
      for (uint32_t k = 0; k < rn; ++k) { if (k) em.put(','); cell_put(em, sb, toks[t0 + 2 + 2 * k]); }
    }
    if (staged_out) { tpw::sync(); stage_flush(out, st.ocur, sh.row_out(), total); }
    st.ocur += total;
    rb += R;
  }
}

TP_FN int emit(const uint8_t* s, const GTok* toks, uint32_t ntok, uint8_t* out, uint32_t out_cap, uint32_t* out_len, Shared& sh, uint8_t* stage, bool report_errors) {
  EmState st; st.sp = 0; st.ocur = 0; st.status = 0; st.over = false; st.col_first = 0; st.col_rows = 0; st.col_rn = 0;
  uint32_t i = 0;
  while (i < ntok && !st.status) {
    const uint32_t m = ntok - i > 32 ? 32u : ntok - i;
    TP_PHASE(PH_EM_GENERIC, i += em_batch(s, toks, ntok, out, out_cap, sh, st, i, m, report_errors));
    if (!st.status && st.col_rows) {
      TP_PHASE(PH_EM_TABLE, em_rows(s, toks, out, out_cap, sh, stage, st, report_errors));
      i = st.col_first + st.col_rows * (2 + 2 * st.col_rn);       // the table's closing bracket comes next
    }
  }
  if (st.status) return st.status;
  if (st.over || st.ocur > out_cap) return TS_NOT_SMALLER;
  *out_len = st.ocur;
  return TS_CONVERTED;
}

// analyze + emit over the token array tokenize produced.
// RESOLVE_MIXED: decide mixed list-item arrays whose first row is not simple (C_R0KEYS) instead of returning FB_MIXED_ITEM.  Its key
// bookkeeping would slow every nested unit down, so a unit is first analyzed without it, and with it only when that attempt stops at
// such an array (toon_unit's retry).
template <bool RESOLVE_MIXED>
TP_FN int toon_tokens(const uint8_t* s, GTok* toks, uint32_t ntok, uint32_t tok_cap, uint8_t* out, uint32_t out_cap, uint32_t* out_len, Shared& sh,
                      uint8_t* stage, bool report_errors) {
  const int st = analyze<RESOLVE_MIXED>(s, toks, ntok, tok_cap, sh, stage);
  if (st) return st;
  tpw::sync();
  return emit(s, toks, ntok, out, out_cap, out_len, sh, stage, report_errors);
}
// The retry in resolve mode, out of line: 2 % of the bench mix's units take it, and inlined beside the first attempt it made the tabular and
// prose units' code larger and those shapes slower (DESIGN.md §6).
TP_SLOW int toon_tokens_resolve(const uint8_t* s, GTok* toks, uint32_t ntok, uint32_t tok_cap, uint8_t* out, uint32_t out_cap, uint32_t* out_len,
                                Shared& sh, uint8_t* stage, bool report_errors) {
  return toon_tokens<true>(s, toks, ntok, tok_cap, out, out_cap, out_len, sh, stage, report_errors);
}

// Whole per-unit pipeline (all 32 lanes call it with the same arguments).  out_cap = n - 1 in the product (a
// conversion is only kept when strictly smaller).  Returns a TS_* status, TS_FALLBACK (| reason << 8) when the sequential
// encoder has to redo the unit.
// `stage` = STAGE bytes of per-warp scratch, 16-byte aligned (shared memory on the GPU).
// retry_mixed: a unit whose first attempt stops at a mixed list-item array (exactly FB_MIXED_ITEM) is analyzed again in resolve mode
// and emitted again, over the SAME token array.  That array is a valid input to a second analyze: analyze patches an opener from a
// word it rebuilds out of the separator bits alone (gt_patch keeps them and replaces kind, flags and length), so a patched opener
// reads as the tokenizer's; an_rows patches row openers the same way, and nothing else writes into the array after tokenize.
// Every Shared field analyze reads was written earlier in the same walk, and every bulk copy into `stage` has completed when
// stage_load returns, so the mbarrier's phase stays in step.  The failed emit's output is overwritten and out_len is set by a
// successful emit only.
TP_FN int toon_unit(const uint8_t* s, uint32_t n, GTok* toks, uint32_t tok_cap, uint8_t* out, uint32_t out_cap, uint32_t* out_len, Shared& sh,
                    uint8_t* stage, bool report_errors, bool retry_mixed = false) {
  uint32_t ntok = 0;
  int st;
  TP_PHASE(PH_TOKENIZE, st = tokenize(s, n, toks, tok_cap, sh, stage, &ntok));
  if (st) return st;
  tpw::sync();
  st = toon_tokens<false>(s, toks, ntok, tok_cap, out, out_cap, out_len, sh, stage, report_errors);
  if (retry_mixed && st == (TS_FALLBACK | (int)(FB_MIXED_ITEM << 8))) {
    tpw::sync();
    ph_in_retry(true);
    TP_PHASE(PH_RESOLVE, st = toon_tokens_resolve(s, toks, ntok, tok_cap, out, out_cap, out_len, sh, stage, report_errors));
    ph_in_retry(false);
  }
  return st;
}

}  // namespace cftp
