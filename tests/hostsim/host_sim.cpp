// host_sim.cpp — CPU simulation of the scan / sub kernels' table-driven algorithm.
// TEST-ONLY: built into tests/hostsim/libcfhostsim.so and loaded only by tests/ (-m "not gpu")
// to validate the compiled tables (prefilter + DFAs, shared scan_core.h routines) against
// CPython `re` on a box with no GPU.  The product library (libcfgpu.so) does not contain this.
#include <string.h>

#include <vector>

#include "../../mcp_context_forge_b200/csrc/cf_host.h"
#include "../../mcp_context_forge_b200/csrc/scan_core.h"

static cf::DfaTables tables_of(const cfre::DfaOut& d) {
  cf::DfaTables t;
  t.ascii_cls = d.ascii_cls.data();
  t.range_start = d.range_start.data();
  t.range_cls = d.range_cls.data();
  t.cls_ctx = d.cls_ctx.data();
  t.trans = d.trans.data();
  t.accsets = d.accsets.data();
  t.nranges = (uint32_t)d.range_start.size();
  t.ncols = d.ncols;
  t.W = d.W;
  for (int i = 0; i < 4; ++i) { t.start_state[i] = d.start_state[i]; t.start_adv[i] = d.start_adv[i]; }
  t.nl_cls = d.nl_cls; t.nlf_cls = d.nlf_cls;
  return t;
}

extern "C" {

int cfh_scan(cf_builder* b, const uint8_t* stream, uint64_t nbytes, const uint64_t* offsets,
             uint32_t n, uint64_t* bitmaps, uint64_t* stats) {
  int rc = cf_builder_compile_host(b, nullptr);
  if (rc) return rc;
  const cfre::CompileOut& co = b->out;
  cf::DfaTables t = tables_of(co.search);
  uint32_t W = t.W;
  for (uint32_t u = 0; u < n; ++u)
    for (uint32_t w = 0; w < W; ++w) bitmaps[(uint64_t)u * W + w] = co.always_bits[w];
  std::vector<uint8_t> pad(cf::FRONT_PAD + nbytes + 64, cf::TERM);
  memcpy(pad.data() + cf::FRONT_PAD, stream, nbytes);
  const uint8_t* s = pad.data() + cf::FRONT_PAD;   // s[-FRONT_PAD..] valid
  uint32_t acc = 0;
  uint64_t ncand = 0, nsteps = 0;
  const bool pairs = co.filter.use_pairs;
  // feed from LOOKBACK bytes before the stream to START_OFF bytes after (the last start is nbytes-1)
  for (int64_t p = -(int64_t)cf::F_LOOKBACK; p < (int64_t)nbytes + (int64_t)cf::F_START_OFF; ++p) {
    if (pairs) {
      acc = cf::pair_step(acc, co.filter.pairT[cf::pair_hash(s[p - 1], s[p])]);
      if (!(acc & cf::PF_HIT)) continue;
    } else {
      acc = cf::filter_step(acc, co.filter.E[s[p]]);
      if (!(acc & cf::F_HIT)) continue;
    }
    int64_t start = p - (int64_t)cf::F_START_OFF;
    if (start < 0 || start >= (int64_t)nbytes) continue;
    if ((s[start] & 0xC0) == 0x80) continue;   // not a character boundary
    ++ncand;
    // unit lookup: largest u with offsets[u] <= start
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) / 2; if (offsets[mid] <= (uint64_t)start) lo = mid; else hi = mid; }
    uint64_t ustart = offsets[lo], uend = offsets[lo + 1] - 1;
    nsteps += cf::verify_search(t, s, ustart, uend, (uint64_t)start, bitmaps + (uint64_t)lo * W);
  }
  if (stats) { stats[0] = ncand; stats[1] = nsteps; }
  return CF_OK;
}

// Apply ONE ordered rule (index into the ordered list, in add order) to one unit, Python
// `pattern.sub(repl, unit)` semantics for patterns that cannot match the empty string.
int cfh_sub(cf_builder* b, uint32_t ordered_index, const uint8_t* unit, uint64_t len,
            uint8_t* out, uint64_t cap, uint64_t* out_len, uint64_t* n_matches) {
  int rc = cf_builder_compile_host(b, nullptr);
  if (rc) return rc;
  if (ordered_index >= b->out.ordered.size()) return CF_E_BADARG;
  // find the pattern index of this ordered rule
  uint32_t pat = 0, seen = 0;
  for (; pat < b->ordered.size(); ++pat) if (b->ordered[pat] && seen++ == ordered_index) break;
  const std::vector<uint8_t>& repl = b->repl[pat];
  cf::DfaTables t = tables_of(b->out.ordered[ordered_index]);
  const uint32_t* E = b->out.ordered_filter[ordered_index].E;
  std::vector<uint8_t> pad(cf::FRONT_PAD + len + 64, cf::TERM);
  memcpy(pad.data() + cf::FRONT_PAD, unit, len);
  const uint8_t* s = pad.data() + cf::FRONT_PAD;
  uint64_t o = 0, cur = 0, nm = 0;
  auto put = [&](const uint8_t* p, uint64_t k) {
    if (o + k <= cap) memcpy(out + o, p, k);
    o += k;
  };
  // the replacement of one match: the literal, or the template with this match's group texts (the same cf::pike_captures the
  // kernel's lane 0 runs)
  const std::vector<uint32_t>& tm = b->tmpl[pat];
  const cfre::NfaOut& nf = b->out.ordered_nfa[ordered_index];
  cf::NfaView nv;
  nv.code = nf.code.data(); nv.setbits = nf.setbits.data(); nv.ninst = nf.ninst; nv.start = nf.start; nv.wpc = nf.wpc; nv.nslots = 2 * (nf.ngroups + 1);
  std::vector<uint32_t> pike(cf::pike_scratch_words(nv.ninst, nv.nslots)), caps(nv.nslots);
  auto put_repl = [&](uint64_t sp, bool adv) {
    if (tm.empty()) { put(repl.data(), repl.size()); return; }
    for (auto& c : caps) c = cf::CAP_UNSET;
    cf::pike_captures(t, nv, s, 0, len, sp, adv, pike.data(), caps.data());
    for (size_t k = 0; k + 2 < tm.size(); k += 3) {
      if (tm[k] == 0) put(repl.data() + tm[k + 1], tm[k + 2]);
      else if (caps[2 * tm[k + 1]] != cf::CAP_UNSET && caps[2 * tm[k + 1] + 1] != cf::CAP_UNSET && caps[2 * tm[k + 1] + 1] >= caps[2 * tm[k + 1]])
        put(s + caps[2 * tm[k + 1]], caps[2 * tm[k + 1] + 1] - caps[2 * tm[k + 1]]);
    }
  };
  if (b->out.info[pat].min_len_chars == 0) {
    // a rule that can match "": the sequential statement of sub_kernel's nullable branch (= sre's pattern_subx loop)
    bool adv = false;
    for (uint64_t sp = 0; sp <= len;) {
      if (sp < len && (s[sp] & 0xC0) == 0x80) { ++sp; continue; }
      uint64_t e = cf::match_first(t, s, 0, len, sp, adv);
      if (e == ~0ull) { adv = false; ++sp; continue; }
      put(s + cur, sp - cur);
      put_repl(sp, adv);
      ++nm;
      cur = e;
      adv = (e == sp);
      sp = e;            // after an empty match the same position is tried again with must_advance
    }
    put(s + cur, len - cur);
    *out_len = o;
    if (n_matches) *n_matches = nm;
    return o <= cap ? CF_OK : CF_E_CAPACITY;
  }
  uint32_t acc = 0;
  for (int64_t p = -(int64_t)cf::F_LOOKBACK; p < (int64_t)len + (int64_t)cf::F_START_OFF; ++p) {
    acc = cf::filter_step(acc, E[s[p]]);
    if (!(acc & cf::F_HIT)) continue;
    int64_t start = p - (int64_t)cf::F_START_OFF;
    if (start < 0 || start >= (int64_t)len) continue;
    if ((uint64_t)start < cur) continue;            // inside the previous match
    if ((s[start] & 0xC0) == 0x80) continue;
    uint64_t e = cf::match_first(t, s, 0, len, (uint64_t)start);
    if (e == ~0ull) continue;
    put(s + cur, (uint64_t)start - cur);
    put_repl((uint64_t)start, false);
    cur = e;
    ++nm;
  }
  put(s + cur, len - cur);
  *out_len = o;
  if (n_matches) *n_matches = nm;
  return o <= cap ? CF_OK : CF_E_CAPACITY;
}

}  // extern "C"

// ---- TOON: run the shared json_toon.h pipeline on the CPU (same code the CUDA kernel calls) ----
#include "../../mcp_context_forge_b200/csrc/json_toon.h"
// stop_on_over: give up at the first check past the capacity, as toon_kernel does without CF_TOON_REPORT_ERRORS
extern "C" int cfh_toon(const uint8_t* text, uint32_t n, uint8_t* out, uint32_t out_cap, uint32_t* out_len, int stop_on_over) {
  std::vector<cfj::JNode> nodes(n / 2 + 4);
  cfj::Big big;
  std::vector<uint8_t> digits(1240);
  *out_len = 0;
  return cfj::toon_process(text, n, nodes.data(), (uint32_t)nodes.size(), out, out_cap, out_len, &big, digits.data(), (uint32_t)digits.size(),
                           stop_on_over != 0);
}

// ---- masking: shared json_mask.h pipeline on the CPU ----
#include "../../mcp_context_forge_b200/csrc/json_mask.h"
extern "C" int cfh_mask(const uint8_t* text, uint32_t n, int max_depth, uint8_t* out, uint32_t out_cap, uint32_t* out_len) {
  std::vector<cfj::JNode> nodes(n / 2 + 4);
  std::vector<uint32_t> idx(n / 2 + 4);
  cfj::Big big;
  std::vector<uint8_t> digits(1240);
  cfm::NumWork w{&big, &big, digits.data(), (uint32_t)digits.size()};
  *out_len = 0;
  return cfm::mask_process(text, n, nodes.data(), (uint32_t)nodes.size(), idx.data(), (uint32_t)idx.size(), out, out_cap, out_len, max_depth, w);
}
extern "C" int cfh_key_sensitive(const uint8_t* key, uint32_t n) {
  cfj::JNode k{cfj::J_KEY, 0, n, 0};   // raw (unescaped) key bytes
  return cfm::key_sensitive(key, k) ? 1 : 0;
}

// ---- structural index + token-driven DOM builder (json_index.h), the path the CUDA kernels take ----
#include "../../mcp_context_forge_b200/csrc/json_index.h"
static int indexed_parse(const uint8_t* text, uint32_t n, std::vector<cfj::JNode>& nodes, uint32_t* count) {
  std::vector<cfx::Tok> tok(n + 1);
  bool unt = false;
  const uint32_t nt = cfx::index_host(text, n, tok.data(), &unt);
  for (uint32_t t = 0; t < nt; ++t) tok[t].aux = cfx::classify_token(text, n, tok[t].pos);
  return cfx::json_build(text, n, tok.data(), nt, unt, nodes.data(), (uint32_t)nodes.size(), count);
}
// 0 = both parsers agree (same status and, when it parsed, identical node arrays); else a diagnostic code
extern "C" int cfh_index_equiv(const uint8_t* text, uint32_t n, int* status_seq, int* status_idx) {
  std::vector<cfj::JNode> a(n / 2 + 4), b(n / 2 + 4);
  uint32_t ca = 0, cb = 0;
  const int pa = cfj::json_parse(text, n, a.data(), (uint32_t)a.size(), &ca);
  const int pb = indexed_parse(text, n, b, &cb);
  *status_seq = pa; *status_idx = pb;
  if (pa != pb) return 1;
  if (pa != cfj::PARSE_OK) return 0;
  if (ca != cb) return 2;
  for (uint32_t i = 0; i < ca; ++i)
    if (a[i].t != b[i].t || a[i].off != b[i].off || a[i].len != b[i].len) return 3;
  // .next: sibling links and, for object member values, the key hash (28 bits kept by the index path)
  for (uint32_t i = 0; i < ca; ++i) {
    const bool member_value = i > 0 && (a[i - 1].t & cfj::J_TYPE) == cfj::J_KEY;
    if (member_value) { if ((a[i].next & 0x0FFFFFFFu) != (b[i].next & 0x0FFFFFFFu)) return 4; }
    else if (a[i].next != b[i].next) return 5;
  }
  return 0;
}
// token list of the index alone: pos (bit 31 = closing quote); returns the count, *unterminated as flag
extern "C" uint32_t cfh_json_index(const uint8_t* text, uint32_t n, uint32_t* pos_out, uint32_t* aux_out, int* unterminated) {
  std::vector<cfx::Tok> tok(n + 1);
  bool unt = false;
  const uint32_t nt = cfx::index_host(text, n, tok.data(), &unt);
  for (uint32_t t = 0; t < nt; ++t) { pos_out[t] = tok[t].pos; aux_out[t] = cfx::classify_token(text, n, tok[t].pos); }
  *unterminated = unt ? 1 : 0;
  return nt;
}
extern "C" int cfh_toon_indexed(const uint8_t* text, uint32_t n, uint8_t* out, uint32_t out_cap, uint32_t* out_len) {
  std::vector<cfj::JNode> nodes(n / 2 + 4);
  cfj::Big big;
  std::vector<uint8_t> digits(1240);
  uint32_t cnt = 0;
  *out_len = 0;
  const int pr = indexed_parse(text, n, nodes, &cnt);
  return cfj::toon_finish(pr, text, nodes.data(), out, out_cap, out_len, &big, digits.data(), (uint32_t)digits.size(), false);
}
// (json_build keeps the 64-level stack and has no number range check: this twin agrees with cfh_mask on bodies inside both)
extern "C" int cfh_mask_indexed(const uint8_t* text, uint32_t n, int max_depth, uint8_t* out, uint32_t out_cap, uint32_t* out_len) {
  std::vector<cfj::JNode> nodes(n / 2 + 4);
  std::vector<uint32_t> idx(n / 2 + 4);
  cfj::Big big;
  std::vector<uint8_t> digits(1240);
  cfm::NumWork w{&big, &big, digits.data(), (uint32_t)digits.size()};
  uint32_t cnt = 0;
  *out_len = 0;
  const int pr = indexed_parse(text, n, nodes, &cnt);
  return cfm::mask_finish(pr, text, nodes.data(), idx.data(), (uint32_t)idx.size(), out, out_cap, out_len, max_depth, w);
}

// ---- token-parallel TOON (json_tp.h): the warp-per-unit kernel body, run on the 32-fibre warp emulator ----
#include "../../mcp_context_forge_b200/csrc/json_tp.h"
#include "warp_emu.h"
// order: 0 ascending / 1 descending lane schedule.  Returns the TS_* status (7 = sequential fallback requested).
extern "C" int cfh_toon_tp(const uint8_t* text, uint32_t n, uint8_t* out, uint32_t out_cap, uint32_t* out_len, int report_errors, int order,
                           uint32_t* ntok_out) {
  // the kernel reads whole 1 KiB steps on a 16-byte grid: give it the padding the device buffers have; `order` bits 4.. shift the
  // unit's alignment inside the 16-byte grid
  std::vector<uint8_t> buf(64 + n + 2048, 0xFF);
  const uint32_t shift = ((uint32_t)order >> 4) & 15u;
  uint8_t* base = buf.data() + 32;
  base += (16 - ((uintptr_t)base & 15u)) & 15u;
  uint8_t* s = base + shift;
  memcpy(s, text, n);
  std::vector<cftp::GTok> toks(n / 2 + 64);
  std::vector<cftp::Shared> sh(1);
  std::vector<uint8_t> stage_buf(cftp::STAGE + 64);
  uint8_t* stage = stage_buf.data() + ((16 - ((uintptr_t)stage_buf.data() & 15u)) & 15u);
  int status[32];
  uint32_t olen[32];
  for (int i = 0; i < 32; ++i) { status[i] = -1; olen[i] = 0; }
  wemu::run_warp([&](uint32_t lane) {
    uint32_t ol = 0;
    status[lane] = cftp::toon_unit(s, n, toks.data(), (uint32_t)toks.size(), out, out_cap, &ol, sh[0], stage, report_errors != 0);
    olen[lane] = ol;
  }, order & 1);
  for (int i = 1; i < 32; ++i) if (status[i] != status[0] || olen[i] != olen[0]) return -100 - i;   // the status must be warp-uniform
  *out_len = olen[0];
  if (ntok_out) *ntok_out = (uint32_t)status[0] >> 8;   // fallback reason (diagnostics)
  return status[0] & 0xFF;
}
