// re_backend.cpp — see re_backend.h.  Host-only C++ (no CUDA), compiled into libcfgpu.so and into
// the CPU-test helper library.
#include "re_backend.h"

#include <algorithm>
#include <map>
#include <deque>
#include <queue>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "scan_core.h"

namespace cfre {

static const int CF_E_UNSUPPORTED = -3;
static const int CF_E_TOO_LARGE = -4;
static const int CF_E_BADARG = -2;

namespace {

struct Node {
  uint32_t op = A_EMPTY;
  std::vector<Node> kids;
  CharSet set;
  uint32_t mn = 0, mx = 0, greedy = 1, kind = 0;
};

bool parse_node(const std::vector<uint32_t>& w, size_t& pos, Node& out, int depth) {
  if (pos >= w.size() || depth > 2000) return false;
  out.op = w[pos++];
  switch (out.op) {
    case A_EMPTY: return true;
    case A_SET: {
      if (pos >= w.size()) return false;
      uint32_t n = w[pos++];
      if (pos + 2ull * n > w.size()) return false;
      for (uint32_t i = 0; i < n; ++i) {
        Interval iv{w[pos], w[pos + 1]};
        pos += 2;
        if (iv.lo > iv.hi || iv.hi > 0x10FFFF) return false;
        if (!out.set.empty() && iv.lo <= out.set.back().hi) return false;
        out.set.push_back(iv);
      }
      return true;
    }
    case A_CAT:
    case A_ALT: {
      if (pos >= w.size()) return false;
      uint32_t n = w[pos++];
      if (n > w.size()) return false;
      out.kids.resize(n);
      for (uint32_t i = 0; i < n; ++i)
        if (!parse_node(w, pos, out.kids[i], depth + 1)) return false;
      return true;
    }
    case A_REPEAT: {
      if (pos + 3 > w.size()) return false;
      out.mn = w[pos++]; out.mx = w[pos++]; out.greedy = w[pos++];
      if (out.mx != REPEAT_INF && out.mx < out.mn) return false;
      out.kids.resize(1);
      return parse_node(w, pos, out.kids[0], depth + 1);
    }
    case A_ASSERT:
      if (pos >= w.size()) return false;
      out.kind = w[pos++];
      return out.kind >= AS_WORD_B && out.kind <= AS_END_DOLLAR;
    case A_GROUP:
      if (pos >= w.size()) return false;
      out.kind = w[pos++];
      if (out.kind == 0 || out.kind > 99) return false;
      out.kids.resize(1);
      return parse_node(w, pos, out.kids[0], depth + 1);
    default: return false;
  }
}

enum : uint8_t { I_CHAR, I_SPLIT, I_ASSERT, I_MATCH, I_SAVE };   // I_SAVE: kind = capture slot (an epsilon edge for the DFAs)
struct Inst { uint8_t op; int x = -1, y = -1; int set = -1; uint32_t kind = 0; int pat = -1; };

struct Prog {
  std::vector<Inst> insts;
  std::vector<CharSet> sets;
  std::map<std::vector<uint32_t>, int> set_ids;
  std::vector<int> start;          // per pattern
  size_t limit = 30000;
  bool overflow = false;

  int add(const Inst& i) {
    if (insts.size() >= limit) { overflow = true; return 0; }
    insts.push_back(i);
    return (int)insts.size() - 1;
  }
  int set_id(const CharSet& s) {
    std::vector<uint32_t> key;
    for (auto& iv : s) { key.push_back(iv.lo); key.push_back(iv.hi); }
    auto it = set_ids.find(key);
    if (it != set_ids.end()) return it->second;
    int id = (int)sets.size();
    sets.push_back(s);
    set_ids[key] = id;
    return id;
  }
  // continuation-passing Thompson construction: returns the entry pc of `n` followed by `next`
  int comp(const Node& n, int next) {
    if (overflow) return next;
    switch (n.op) {
      case A_EMPTY: return next;
      case A_SET: { Inst i; i.op = I_CHAR; i.set = set_id(n.set); i.x = next; return add(i); }
      case A_CAT: {
        int cur = next;
        for (size_t k = n.kids.size(); k-- > 0;) cur = comp(n.kids[k], cur);
        return cur;
      }
      case A_ALT: {
        if (n.kids.empty()) return next;
        std::vector<int> s(n.kids.size());
        for (size_t k = 0; k < n.kids.size(); ++k) s[k] = comp(n.kids[k], next);
        int cur = s.back();
        for (size_t k = n.kids.size() - 1; k-- > 0;) {
          Inst i; i.op = I_SPLIT; i.x = s[k]; i.y = cur; cur = add(i);
        }
        return cur;
      }
      case A_ASSERT: { Inst i; i.op = I_ASSERT; i.kind = n.kind; i.x = next; return add(i); }
      case A_GROUP: {
        Inst c; c.op = I_SAVE; c.kind = 2 * n.kind + 1; c.x = next;
        int body = comp(n.kids[0], add(c));
        Inst o; o.op = I_SAVE; o.kind = 2 * n.kind; o.x = body;
        return add(o);
      }
      case A_REPEAT: {
        const Node& c = n.kids[0];
        int cur;
        if (n.mx == REPEAT_INF) {
          Inst sp; sp.op = I_SPLIT;
          int L = add(sp);
          int body = comp(c, L);
          if (overflow) return next;
          insts[L].x = n.greedy ? body : next;
          insts[L].y = n.greedy ? next : body;
          cur = L;
        } else {
          cur = next;
          uint32_t k = n.mx - n.mn;
          if (k > 2000) { overflow = true; return next; }
          for (uint32_t i = 0; i < k; ++i) {
            int body = comp(c, cur);
            Inst sp; sp.op = I_SPLIT;
            sp.x = n.greedy ? body : next;
            sp.y = n.greedy ? next : body;
            cur = add(sp);
          }
        }
        if (n.mn > 2000) { overflow = true; return next; }
        for (uint32_t i = 0; i < n.mn; ++i) cur = comp(c, cur);
        return cur;
      }
    }
    return next;
  }
};

// ---------------------------------------------------------------------------------------------
// Code-point classes: the coarsest partition of [0, 0x10FFFF] on which every SET, the \w set and
// '\n' are constant.
// ---------------------------------------------------------------------------------------------
struct Classes {
  uint32_t ncls = 0;
  uint32_t nl_cls = 0, nlf_cls = 0xFFFFFFFFu;   // class of '\n'; class of "the '\n' that is the unit's last character" (only when some `$` needs it)
  std::vector<uint16_t> ascii_cls;
  std::vector<uint32_t> range_start;
  std::vector<uint16_t> range_cls;
  std::vector<uint8_t> cls_ctx;
  std::vector<std::vector<uint8_t>> set_has;   // [set][cls]
  // UTF-8 first-byte information per class (for the prefilter)
  std::vector<std::vector<uint8_t>> ascii_members;  // [cls][128] 0/1
  std::vector<std::vector<uint8_t>> lead[5];        // lead[L][cls][256], L = 2..4
};

static bool in_set(const CharSet& s, uint32_t cp) {
  size_t lo = 0, hi = s.size();
  while (lo < hi) {
    size_t mid = (lo + hi) / 2;
    if (s[mid].hi < cp) lo = mid + 1; else hi = mid;
  }
  return lo < s.size() && s[lo].lo <= cp;
}

static uint32_t utf8_lead(uint32_t cp) {
  if (cp < 0x800) return 0xC0 | (cp >> 6);
  if (cp < 0x10000) return 0xE0 | (cp >> 12);
  return 0xF0 | (cp >> 18);
}

static int build_classes(const Prog& prog, const CharSet& word, Classes& C, std::string* err) {
  std::vector<uint32_t> cuts = {0, 0x80, 0x800, 0x10000, 0x110000, '\n', '\n' + 1};
  auto add_set = [&](const CharSet& s) {
    for (auto& iv : s) { cuts.push_back(iv.lo); cuts.push_back(iv.hi + 1); }
  };
  for (auto& s : prog.sets) add_set(s);
  add_set(word);
  std::sort(cuts.begin(), cuts.end());
  cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
  size_t nsets = prog.sets.size();
  size_t sigw = (nsets + 2 + 63) / 64;
  std::map<std::vector<uint64_t>, uint32_t> sig2cls;
  std::vector<uint32_t> piece_cls(cuts.size() - 1);
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    uint32_t cp = cuts[i];
    std::vector<uint64_t> sig(sigw, 0);
    for (size_t s = 0; s < nsets; ++s)
      if (in_set(prog.sets[s], cp)) sig[s >> 6] |= 1ull << (s & 63);
    bool w = in_set(word, cp), nl = (cp == '\n');
    if (w) sig[nsets >> 6] |= 1ull << (nsets & 63);
    if (nl) sig[(nsets + 1) >> 6] |= 1ull << ((nsets + 1) & 63);
    auto it = sig2cls.find(sig);
    uint32_t c;
    if (it == sig2cls.end()) {
      c = (uint32_t)sig2cls.size();
      sig2cls[sig] = c;
      C.cls_ctx.push_back(w ? cf::P_WORD : nl ? cf::P_NL : cf::P_OTHER);
      C.set_has.resize(nsets);
      for (size_t s = 0; s < nsets; ++s) C.set_has[s].push_back((sig[s >> 6] >> (s & 63)) & 1);
    } else c = it->second;
    piece_cls[i] = c;
  }
  C.ncls = (uint32_t)sig2cls.size();
  if (C.ncls >= 4000) { if (err) *err = "too many character classes"; return CF_E_TOO_LARGE; }
  C.ascii_cls.assign(128, 0);
  C.ascii_members.assign(C.ncls, std::vector<uint8_t>(128, 0));
  for (int L = 2; L <= 4; ++L) C.lead[L].assign(C.ncls, std::vector<uint8_t>(256, 0));
  for (size_t i = 0; i + 1 < cuts.size(); ++i) {
    uint32_t a = cuts[i], b = cuts[i + 1] - 1, c = piece_cls[i];
    if (a < 0x80) {
      for (uint32_t cp = a; cp <= b; ++cp) { C.ascii_cls[cp] = (uint16_t)c; C.ascii_members[c][cp] = 1; }
    } else {
      if (C.range_cls.empty() || C.range_cls.back() != c) {
        C.range_start.push_back(a);
        C.range_cls.push_back((uint16_t)c);
      }
      int L = a < 0x800 ? 2 : a < 0x10000 ? 3 : 4;   // pieces never straddle a length boundary
      for (uint32_t lb = utf8_lead(a); lb <= utf8_lead(b); ++lb) C.lead[L][c][lb] = 1;
    }
  }
  if (C.range_start.empty() || C.range_start[0] != 0x80) {
    if (err) *err = "internal: class ranges"; return CF_E_BADARG;
  }
  C.nl_cls = C.ascii_cls['\n'];
  // A non-MULTILINE `$` (AS_END_DOLLAR) holds at the end of the text AND before a final "\n".  The automata see one character of
  // look-ahead, so "a newline that is the last character" becomes a character class of its own: it behaves like '\n' everywhere,
  // the matchers substitute it for '\n' at the last position (scan_core.h), and `$` tests for it.  Only built when some `$` needs it.
  bool need_nlf = false;
  for (auto& in : prog.insts) if (in.op == I_ASSERT && in.kind == AS_END_DOLLAR) need_nlf = true;
  if (need_nlf) {
    C.nlf_cls = C.ncls++;
    C.cls_ctx.push_back(cf::P_NL);
    for (size_t s = 0; s < nsets; ++s) C.set_has[s].push_back(C.set_has[s][C.nl_cls]);
    C.ascii_members.push_back(std::vector<uint8_t>(128, 0));
    C.ascii_members.back()['\n'] = 1;
    for (int L = 2; L <= 4; ++L) C.lead[L].push_back(std::vector<uint8_t>(256, 0));
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// DFA construction with lazy epsilon closure (assertions are evaluated with the previous-char
// context stored in the state and the class of the next char, i.e. at transition time).
// ---------------------------------------------------------------------------------------------
struct DfaBuilder {
  const Prog& prog;
  const Classes& C;
  bool ordered;
  uint32_t npat, W;
  size_t max_states;
  std::vector<uint8_t> needs_ctx;   // per pc: an ASSERT is epsilon-reachable
  std::map<std::pair<uint32_t, std::vector<int>>, uint32_t> ids;
  std::vector<std::pair<uint32_t, std::vector<int>>> states;
  std::vector<uint32_t> trans;
  std::map<std::vector<uint64_t>, uint32_t> accids;
  std::vector<uint64_t> accsets;
  bool overflow = false;
  // scratch
  std::vector<uint32_t> visited;
  uint32_t stamp = 0;
  std::vector<int> out_chars;
  std::vector<int> out_match;
  bool cut = false;
  bool no_empty = false;            // must-advance start state: a zero-length match is not a match and cuts nothing

  DfaBuilder(const Prog& p, const Classes& c, bool ord, uint32_t np, size_t maxs)
      : prog(p), C(c), ordered(ord), npat(np), W(ord ? 1 : (np + 63) / 64), max_states(maxs) {
    if (W == 0) W = 1;
    visited.assign(prog.insts.size(), 0);
    compute_needs_ctx();
    states.push_back({cf::P_OTHER, {}});   // DEAD = 0
    ids[states[0]] = 0;
    accsets.assign(W, 0);                  // acc index 0 = empty
    accids[std::vector<uint64_t>(W, 0)] = 0;
  }

  void compute_needs_ctx() {
    size_t n = prog.insts.size();
    needs_ctx.assign(n, 0);
    // iterate to fixpoint (graph is small)
    bool changed = true;
    while (changed) {
      changed = false;
      for (size_t i = 0; i < n; ++i) {
        if (needs_ctx[i]) continue;
        const Inst& in = prog.insts[i];
        bool v = false;
        if (in.op == I_ASSERT) v = true;
        else if (in.op == I_SPLIT) v = (in.x >= 0 && needs_ctx[in.x]) || (in.y >= 0 && needs_ctx[in.y]);
        else if (in.op == I_SAVE) v = in.x >= 0 && needs_ctx[in.x];
        if (v) { needs_ctx[i] = 1; changed = true; }
      }
    }
  }

  bool holds(uint32_t kind, uint32_t P, uint32_t col) const {
    bool eot = (col == C.ncls);
    bool nw = !eot && C.cls_ctx[col] == cf::P_WORD;
    bool nnl = !eot && C.cls_ctx[col] == cf::P_NL;
    switch (kind) {
      case AS_WORD_B: return (P == cf::P_WORD) != nw;
      // sre: `if (state->beginning == state->end) return 0;` for AT_NON_BOUNDARY on an empty string
      case AS_NOT_WORD_B: if (P == cf::P_START && eot) return false; return (P == cf::P_WORD) == nw;
      case AS_BEGIN_STRING: return P == cf::P_START;
      case AS_BEGIN_LINE: return P == cf::P_START || P == cf::P_NL;
      case AS_END_STRING: return eot;
      case AS_END_DOLLAR: return eot || col == C.nlf_cls;
      case AS_END_LINE: return eot || nnl;
    }
    return false;
  }

  void addthread(int pc, uint32_t P, uint32_t col) {
    // iterative DFS preserving priority order (x before y)
    std::vector<int> stack;
    stack.push_back(pc);
    while (!stack.empty() && !cut) {
      int p = stack.back(); stack.pop_back();
      if (visited[p] == stamp) continue;
      visited[p] = stamp;
      const Inst& in = prog.insts[p];
      switch (in.op) {
        case I_CHAR: out_chars.push_back(p); break;
        case I_MATCH: if (no_empty) break; out_match.push_back(in.pat); if (ordered) cut = true; break;
        case I_ASSERT: if (holds(in.kind, P, col)) stack.push_back(in.x); break;
        case I_SPLIT: stack.push_back(in.y); stack.push_back(in.x); break;
        case I_SAVE: stack.push_back(in.x); break;
      }
    }
  }

  // P carries P_ADV for the must-advance start states (sre: `state->must_advance && ptr == state->start` fails the SUCCESS
  // opcode and backtracks, Modules/_sre/sre_lib.h SRE_OP_SUCCESS): only the closure at the start position is affected.
  static const uint32_t P_ADV = 4;
  void closure(const std::vector<int>& kernel, uint32_t P, uint32_t col) {
    ++stamp; out_chars.clear(); out_match.clear(); cut = false;
    no_empty = (P & P_ADV) != 0;
    for (int pc : kernel) { if (cut) break; addthread(pc, P & 3u, col); }
    no_empty = false;
  }

  uint32_t get_state(uint32_t P, std::vector<int>& kernel) {
    if (kernel.empty()) return cf::DEAD;
    if (!ordered) { std::sort(kernel.begin(), kernel.end()); kernel.erase(std::unique(kernel.begin(), kernel.end()), kernel.end()); }
    bool need = false;
    for (int pc : kernel) if (needs_ctx[pc]) { need = true; break; }
    if (!need) P = (P & P_ADV) | cf::P_OTHER;
    auto key = std::make_pair(P, kernel);
    auto it = ids.find(key);
    if (it != ids.end()) return it->second;
    if (states.size() >= max_states) { overflow = true; return cf::DEAD; }
    uint32_t id = (uint32_t)states.size();
    states.push_back(key);
    ids[key] = id;
    return id;
  }

  uint32_t acc_index(const std::vector<int>& matches) {
    if (matches.empty()) return 0;
    if (ordered) return 1;
    std::vector<uint64_t> bm(W, 0);
    for (int p : matches) bm[p >> 6] |= 1ull << (p & 63);
    auto it = accids.find(bm);
    if (it != accids.end()) return it->second;
    uint32_t id = (uint32_t)(accsets.size() / W);
    accsets.insert(accsets.end(), bm.begin(), bm.end());
    accids[bm] = id;
    return id;
  }

  // Build all states reachable from the given start kernels.  Returns start ids per context.
  void build(const std::vector<int>& start_kernel, uint32_t start_state[4], uint32_t* start_adv = nullptr) {
    uint32_t ncols = C.ncls + 1;
    if (ordered) { accsets.assign(2, 0); accsets[1] = 1; }
    for (uint32_t P = 0; P < 4; ++P) {
      std::vector<int> k = start_kernel;
      start_state[P] = get_state(P, k);
    }
    if (start_adv) for (uint32_t P = 0; P < 4; ++P) {
      std::vector<int> k = start_kernel;
      start_adv[P] = get_state(P | P_ADV, k);
    }
    size_t done = 1;
    trans.assign(ncols, 0);   // DEAD row
    std::vector<int> nk;
    while (done < states.size() && !overflow) {
      uint32_t sid = (uint32_t)done++;
      uint32_t P = states[sid].first;
      std::vector<int> kernel = states[sid].second;   // copy: `states` may reallocate
      trans.resize((size_t)(sid + 1) * ncols, 0);
      for (uint32_t col = 0; col < ncols; ++col) {
        closure(kernel, P, col);
        uint32_t acc = acc_index(out_match);
        uint32_t next = cf::DEAD;
        if (col < C.ncls) {
          nk.clear();
          ++stamp;   // reuse `visited` as "already in nk" marker for ordered dedupe
          for (int pc : out_chars) {
            const Inst& in = prog.insts[pc];
            if (C.set_has[in.set][col]) {
              if (visited[in.x] != stamp) { visited[in.x] = stamp; nk.push_back(in.x); }
            }
          }
          next = get_state(C.cls_ctx[col], nk);
        }
        if (acc >= 65536 || next >= 65536) { overflow = true; break; }
        trans[(size_t)sid * ncols + col] = next | (acc << cf::ACC_SHIFT);
      }
    }
  }

  void emit(DfaOut& o, const uint32_t start_state[4], const uint32_t* start_adv = nullptr) const {
    for (int i = 0; i < 4; ++i) o.start_adv[i] = start_adv ? start_adv[i] : 0;
    o.ascii_cls = C.ascii_cls; o.range_start = C.range_start; o.range_cls = C.range_cls;
    o.cls_ctx = C.cls_ctx; o.trans = trans; o.accsets = accsets;
    o.ncols = C.ncls + 1; o.nstates = (uint32_t)states.size(); o.W = W;
    o.nl_cls = C.nl_cls; o.nlf_cls = C.nlf_cls;
    for (int i = 0; i < 4; ++i) o.start_state[i] = start_state[i];
  }
};

// ---------------------------------------------------------------------------------------------
// Prefilter derivation: per pattern, the byte sets admissible before the match (N) and at match
// byte positions 0..2 (A, B, C), over-approximated from its anchored DFA.
// ---------------------------------------------------------------------------------------------
struct ByteSet {
  uint64_t w[4] = {0, 0, 0, 0};
  void set(uint32_t b) { w[b >> 6] |= 1ull << (b & 63); }
  bool get(uint32_t b) const { return (w[b >> 6] >> (b & 63)) & 1; }
  void all() { w[0] = w[1] = w[2] = w[3] = ~0ull; }
  void merge(const ByteSet& o) { for (int i = 0; i < 4; ++i) w[i] |= o.w[i]; }
  int count() const { int c = 0; for (int i = 0; i < 4; ++i) c += __builtin_popcountll(w[i]); return c; }
  int union_count(const ByteSet& o) const { int c = 0; for (int i = 0; i < 4; ++i) c += __builtin_popcountll(w[i] | o.w[i]); return c; }
};
static const int NPOS = 4;   // match-byte positions covered by the prefilter
struct SlotSet {                      // subset of the cf::PF_SLOTS pair-hash slots
  uint64_t w[cf::PF_SLOTS / 64];
  SlotSet() { memset(w, 0, sizeof(w)); }
  void set(uint32_t i) { w[i >> 6] |= 1ull << (i & 63); }
  bool get(uint32_t i) const { return (w[i >> 6] >> (i & 63)) & 1; }
  void all() { memset(w, 0xFF, sizeof(w)); }
  void merge(const SlotSet& o) { for (size_t i = 0; i < cf::PF_SLOTS / 64; ++i) w[i] |= o.w[i]; }
};
struct PatFilter { ByteSet N, pos[NPOS]; SlotSet pair[NPOS]; };

static void explore(const DfaBuilder& B, const Classes& C, uint32_t state, int bytepos,
                    std::vector<uint8_t>& seen, PatFilter& f) {
  if (bytepos >= NPOS || state == cf::DEAD) return;
  size_t key = (size_t)state * NPOS + bytepos;
  if (seen[key]) return;
  seen[key] = 1;
  uint32_t ncols = C.ncls + 1;
  for (uint32_t col = 0; col < ncols; ++col) {
    uint32_t e = B.trans[(size_t)state * ncols + col];
    if (e >> cf::ACC_SHIFT) for (int k = bytepos; k < NPOS; ++k) f.pos[k].all();
    uint32_t t = e & 0xFFFF;
    if (col == C.ncls || t == cf::DEAD) continue;
    bool any_ascii = false;
    for (uint32_t b = 0; b < 128; ++b) if (C.ascii_members[col][b]) { f.pos[bytepos].set(b); any_ascii = true; }
    if (any_ascii) explore(B, C, t, bytepos + 1, seen, f);
    for (int L = 2; L <= 4; ++L) {
      bool any = false;
      for (uint32_t b = 0xC0; b < 0x100; ++b) if (C.lead[L][col][b]) { f.pos[bytepos].set(b); any = true; }
      if (!any) continue;
      for (int j = 1; j < L && bytepos + j < NPOS; ++j)
        for (uint32_t b = 0x80; b < 0xC0; ++b) f.pos[bytepos + j].set(b);
      explore(B, C, t, bytepos + L, seen, f);
    }
  }
}

static bool alive(const DfaBuilder& B, const Classes& C, uint32_t state) {
  if (state == cf::DEAD) return false;
  uint32_t ncols = C.ncls + 1;
  for (uint32_t col = 0; col < ncols; ++col) if (B.trans[(size_t)state * ncols + col]) return true;
  return false;
}

// Pair sets by forward data flow over the pattern's anchored DFA: reach[s] = bytes that can immediately
// precede the transition out of state s at the current byte position.  Multi-byte characters are
// over-approximated (any continuation byte may follow a lead or another continuation byte).
static void add_pairs(SlotSet& ps, const ByteSet& prev, const ByteSet& cur) {
  for (uint32_t x = 0; x < 256; ++x) {
    if (!prev.get(x)) continue;
    for (uint32_t y = 0; y < 256; ++y) if (cur.get(y)) ps.set(cf::pair_hash(x, y));
  }
}
static void pattern_pairs(const DfaBuilder& B, const Classes& C, const uint32_t ss[4], const ByteSet ctxN[4], PatFilter& f) {
  const uint32_t ncols = C.ncls + 1;
  const size_t ns = B.states.size();
  ByteSet conts;
  for (uint32_t b = 0x80; b < 0xC0; ++b) conts.set(b);
  // code points of every small non-ASCII class (empty = none or too many to enumerate)
  std::vector<std::vector<uint32_t>> nonascii_cps(C.ncls);
  {
    std::vector<uint64_t> total(C.ncls, 0);
    const size_t nr = C.range_start.size();
    for (size_t i = 0; i < nr; ++i) {
      const uint32_t lo = C.range_start[i], hi = i + 1 < nr ? C.range_start[i + 1] - 1 : 0x10FFFFu;
      total[C.range_cls[i]] += (uint64_t)hi - lo + 1;
    }
    for (size_t i = 0; i < nr; ++i) {
      const uint32_t cls = C.range_cls[i];
      if (total[cls] > 256) continue;
      const uint32_t lo = C.range_start[i], hi = i + 1 < nr ? C.range_start[i + 1] - 1 : 0x10FFFFu;
      for (uint32_t cp = lo; cp <= hi; ++cp) nonascii_cps[cls].push_back(cp);
    }
  }
  // reach[j][s]: possible previous bytes when state s is entered with j match bytes consumed
  std::vector<std::vector<ByteSet>> reach(NPOS + 4, std::vector<ByteSet>(ns));
  std::vector<std::vector<uint8_t>> live(NPOS + 4, std::vector<uint8_t>(ns, 0));
  for (int P = 0; P < 4; ++P) {
    if (ss[P] == cf::DEAD || ctxN[P].count() == 0) continue;
    reach[0][ss[P]].merge(ctxN[P]);
    live[0][ss[P]] = 1;
  }
  bool open_from[NPOS + 1] = {false, false, false, false, false};   // a match can be complete before byte j: anything follows
  for (int j = 0; j < NPOS; ++j) {
    for (size_t s = 0; s < ns; ++s) {
      if (!live[j][s]) continue;
      const ByteSet& R = reach[j][s];
      for (uint32_t col = 0; col < ncols; ++col) {
        const uint32_t e = B.trans[s * ncols + col];
        if (e >> cf::ACC_SHIFT) open_from[j] = true;
        const uint32_t t = e & 0xFFFF;
        if (col == C.ncls || t == cf::DEAD) continue;
        ByteSet asc;
        bool any_ascii = false;
        for (uint32_t b = 0; b < 128; ++b) if (C.ascii_members[col][b]) { asc.set(b); any_ascii = true; }
        if (any_ascii) {
          add_pairs(f.pair[j], R, asc);
          reach[j + 1][t].merge(asc);
          live[j + 1][t] = 1;
        }
        // non-ASCII members of the class: exact byte sequences when the class is small (the case-fold partners
        // of ASCII letters: K, long s, dotless i ...), over-approximated continuation bytes otherwise
        if (col < C.ncls && !nonascii_cps[col].empty()) {
          for (uint32_t cp : nonascii_cps[col]) {
            uint8_t u[4];
            int L = 0;
            if (cp < 0x800) { u[0] = 0xC0 | (cp >> 6); u[1] = 0x80 | (cp & 63); L = 2; }
            else if (cp < 0x10000) { u[0] = 0xE0 | (cp >> 12); u[1] = 0x80 | ((cp >> 6) & 63); u[2] = 0x80 | (cp & 63); L = 3; }
            else { u[0] = 0xF0 | (cp >> 18); u[1] = 0x80 | ((cp >> 12) & 63); u[2] = 0x80 | ((cp >> 6) & 63); u[3] = 0x80 | (cp & 63); L = 4; }
            ByteSet one;
            one.set(u[0]);
            add_pairs(f.pair[j], R, one);
            for (int k = 1; k < L && j + k < NPOS; ++k) f.pair[j + k].set(cf::pair_hash(u[k - 1], u[k]));
            if (j + L < NPOS + 4) { reach[j + L][t].set(u[L - 1]); live[j + L][t] = 1; }
          }
          continue;
        }
        for (int L = 2; L <= 4; ++L) {
          ByteSet leads;
          bool any = false;
          for (uint32_t b = 0xC0; b < 0x100; ++b) if (C.lead[L][col][b]) { leads.set(b); any = true; }
          if (!any) continue;
          add_pairs(f.pair[j], R, leads);
          for (int k = 1; k < L && j + k < NPOS; ++k) add_pairs(f.pair[j + k], k == 1 ? leads : conts, conts);
          if (j + L < NPOS + 4) { reach[j + L][t].merge(conts); live[j + L][t] = 1; }
        }
      }
    }
    if (open_from[j]) for (int k = j; k < NPOS; ++k) f.pair[k].all();
  }
}

static int pattern_filter(const Prog& prog, const Classes& C, int pat, PatFilter& f, std::string* err) {
  DfaBuilder B2(prog, C, false, (uint32_t)pat + 1, 20000);
  uint32_t ss[4];
  std::vector<int> k = {prog.start[pat]};
  B2.build(k, ss);
  if (B2.overflow) { if (err) *err = "pattern DFA too large"; return CF_E_TOO_LARGE; }
  std::vector<uint8_t> seen(B2.states.size() * NPOS, 0);
  bool al[4];
  for (int P = 0; P < 4; ++P) {
    al[P] = alive(B2, C, ss[P]);
    // `seen` is shared: start states may coincide
    explore(B2, C, ss[P], 0, seen, f);
  }
  if (al[cf::P_START]) f.N.set(cf::TERM);
  for (uint32_t b = 0; b < 128; ++b) if (al[C.cls_ctx[C.ascii_cls[b]]]) f.N.set(b);
  if (al[cf::P_WORD] || al[cf::P_OTHER]) for (uint32_t b = 0x80; b < 0xC0; ++b) f.N.set(b);
  // the same "byte before the match" sets, per start context, for the pair filter
  ByteSet ctxN[4];
  if (al[cf::P_START]) ctxN[cf::P_START].set(cf::TERM);
  for (uint32_t b = 0; b < 128; ++b) { const uint32_t cx = C.cls_ctx[C.ascii_cls[b]]; if (al[cx]) ctxN[cx].set(b); }
  for (uint32_t b = 0x80; b < 0xC0; ++b) { if (al[cf::P_WORD]) ctxN[cf::P_WORD].set(b); if (al[cf::P_OTHER]) ctxN[cf::P_OTHER].set(b); }
  pattern_pairs(B2, C, ss, ctxN, f);
  return 0;
}

// Rough byte-frequency prior for JSON / prose payloads; only the RANKING of bucket layouts depends on
// it (a bad prior costs prefilter candidates, never correctness).
static const double* byte_prior() {
  static double f[256];
  static bool init = false;
  if (init) return f;
  for (int b = 0; b < 256; ++b) f[b] = b >= 0x80 ? 0.0004 : (b < 0x20 ? 0.0005 : 0.003);
  const char* letters = "etaoinsrhdlcumfpgwybvkxjqz";
  const double lf[26] = {.100, .072, .065, .060, .058, .056, .052, .050, .042, .034, .034, .026, .024,
                         .021, .019, .017, .016, .015, .015, .012, .009, .006, .002, .001, .001, .001};
  for (int i = 0; i < 26; ++i) { f[(uint8_t)letters[i]] = lf[i]; f[(uint8_t)(letters[i] - 32)] = lf[i] * 0.06; }
  for (int d = '0'; d <= '9'; ++d) f[d] = 0.012;
  f[' '] = 0.12; f['"'] = 0.04; f[','] = 0.02; f[':'] = 0.02; f['.'] = 0.01; f['_'] = 0.008; f['-'] = 0.005;
  f['\n'] = 0.005; f[0xFF] = 0.0001;
  init = true;
  return f;
}

// Partition the patterns into at most `nb` buckets minimising the expected candidates per byte of the BYTE
// filter (sum over buckets of P(N) * prod P(pos_k) under the prior); the pair filter reuses the partition
// logic with its own bucket count (patterns that share byte sets share pairs).  Returns the total cost.
static double partition_patterns(const std::vector<PatFilter>& pf, size_t nb, std::vector<std::vector<int>>& groups) {
  size_t n = pf.size();
  const double* prior = byte_prior();
  auto mass = [&](const ByteSet& s) {
    double m = 0;
    for (int b = 0; b < 256; ++b) if (s.get(b)) m += prior[b];
    return m;
  };
  // expected candidates per byte of one bucket: P(N) * prod P(pos_k) under independent bytes
  auto cost = [&](const PatFilter& f) {
    double c = mass(f.N);
    for (int k = 0; k < NPOS; ++k) c *= mass(f.pos[k]);
    return c;
  };
  auto merged = [](const PatFilter& a, const PatFilter& b) {
    PatFilter m = a;
    m.N.merge(b.N);
    for (int k = 0; k < NPOS; ++k) m.pos[k].merge(b.pos[k]);
    return m;
  };
  struct Bk { PatFilter f; std::vector<int> pats; };
  std::vector<Bk> bks;
  if (n <= 160) {
    for (size_t i = 0; i < n; ++i) { Bk b; b.f = pf[i]; b.pats.push_back((int)i); bks.push_back(b); }
  } else {
    // very large rule sets: seed 64 groups by the smallest byte a match can start with (agglomeration is cubic)
    std::vector<int> of_byte(256, -1);
    for (size_t i = 0; i < n; ++i) {
      uint32_t b0 = 0;
      while (b0 < 255 && !pf[i].pos[0].get(b0)) ++b0;
      const uint32_t key = b0 & 63;
      if (of_byte[key] < 0) { of_byte[key] = (int)bks.size(); bks.push_back(Bk()); }
      Bk& b = bks[of_byte[key]];
      b.f = b.pats.empty() ? pf[i] : merged(b.f, pf[i]);
      b.pats.push_back((int)i);
    }
  }
  // greedy agglomeration ...
  while (bks.size() > nb) {
    size_t bi = 0, bj = 1; double best = 1e300;
    for (size_t i = 0; i < bks.size(); ++i)
      for (size_t j = i + 1; j < bks.size(); ++j) {
        double d = cost(merged(bks[i].f, bks[j].f)) - cost(bks[i].f) - cost(bks[j].f);
        if (d < best) { best = d; bi = i; bj = j; }
      }
    bks[bi].f = merged(bks[bi].f, bks[bj].f);
    bks[bi].pats.insert(bks[bi].pats.end(), bks[bj].pats.begin(), bks[bj].pats.end());
    bks.erase(bks.begin() + bj);
  }
  // ... then single-pattern moves while they lower the total
  auto rebuild = [&](Bk& b) {
    b.f = PatFilter();
    for (int p : b.pats) b.f = merged(b.f, pf[p]);
  };
  auto total = [&]() { double t = 0; for (auto& b : bks) if (!b.pats.empty()) t += cost(b.f); return t; };
  const int rounds = n > 160 ? 1 : 16;   // bound compile time for very large rule sets
  for (int round = 0; round < rounds; ++round) {
    bool moved = false;
    for (size_t from = 0; from < bks.size(); ++from)
      for (size_t pi = 0; pi < bks[from].pats.size(); ++pi) {
        int pat = bks[from].pats[pi];
        double base = total();
        size_t best_to = from; double best_t = base;
        for (size_t to = 0; to < bks.size(); ++to) {
          if (to == from) continue;
          Bk sf = bks[from], st = bks[to];
          bks[from].pats.erase(bks[from].pats.begin() + pi);
          rebuild(bks[from]);
          bks[to].pats.push_back(pat);
          rebuild(bks[to]);
          double t = total();
          if (t < best_t * (1 - 1e-9)) { best_t = t; best_to = to; }
          bks[from] = sf; bks[to] = st;
        }
        if (best_to != from) {
          bks[from].pats.erase(bks[from].pats.begin() + pi);
          rebuild(bks[from]);
          bks[best_to].pats.push_back(pat);
          rebuild(bks[best_to]);
          moved = true;
          --pi;
        }
      }
    if (!moved) break;
  }
  groups.clear();
  for (auto& b : bks) groups.push_back(b.pats);
  return total();
}

// expected candidates per byte above which the pair filter (slower per byte, far more selective) takes over:
// past it the byte filter spends more time verifying candidates than the pair filter loses on its lower scan rate
static const double PAIR_MODE_COST = 3e-3;

static void assign_buckets(const std::vector<PatFilter>& pf, FilterOut& fo, bool allow_pairs) {
  const size_t n = pf.size();
  fo.bucket_of_pattern.assign(n, 0);
  std::vector<std::vector<int>> groups;
  fo.byte_cost = partition_patterns(pf, cf::F_BUCKETS, groups);
  memset(fo.E, 0, sizeof(fo.E));
  for (size_t k = 0; k < groups.size(); ++k) {
    ByteSet N, pos[NPOS];
    for (int p : groups[k]) {
      fo.bucket_of_pattern[p] = (int)k;
      N.merge(pf[p].N);
      for (int j = 0; j < NPOS; ++j) pos[j].merge(pf[p].pos[j]);
    }
    for (uint32_t b = 0; b < 256; ++b) {
      uint32_t e = 0;
      if (N.get(b)) e |= 1u << k;
      for (int j = 0; j < NPOS; ++j)
        if (pos[j].get(b)) e |= 1u << ((j + 1) * cf::F_BITS + k);
      fo.E[b] |= e;
    }
  }
  fo.use_pairs = false;
  fo.pairT.clear();
  const char* force = getenv("CF_PAIR_FILTER");      // "1" / "0" force the choice (tests, measurements)
  bool want = allow_pairs && fo.byte_cost > PAIR_MODE_COST;
  if (allow_pairs && force && (force[0] == '0' || force[0] == '1')) want = force[0] == '1';
  if (getenv("CF_DBG_FILTER")) fprintf(stderr, "byte filter cost %.3g (n=%zu) -> %s\n", fo.byte_cost, n, want ? "pairs" : "bytes");
  if (!want) return;
  std::vector<std::vector<int>> pg;
  partition_patterns(pf, cf::PF_BUCKETS, pg);
  fo.use_pairs = true;
  fo.pairT.assign(cf::PF_SLOTS, 0);
  for (size_t k = 0; k < pg.size(); ++k)
    for (int p : pg[k])
      for (int j = 0; j < NPOS; ++j)
        for (uint32_t sl = 0; sl < cf::PF_SLOTS; ++sl)
          if (pf[p].pair[j].get(sl)) fo.pairT[sl] |= 1u << (8 * j + k);
}

static bool nullable_no_assert(const Prog& prog, int start) {
  std::vector<uint8_t> seen(prog.insts.size(), 0);
  std::vector<int> st = {start};
  while (!st.empty()) {
    int p = st.back(); st.pop_back();
    if (seen[p]) continue;
    seen[p] = 1;
    const Inst& in = prog.insts[p];
    if (in.op == I_MATCH) return true;
    if (in.op == I_SPLIT) { st.push_back(in.x); st.push_back(in.y); }
    if (in.op == I_SAVE) st.push_back(in.x);
  }
  return false;
}

static uint32_t min_len(const Prog& prog, int start) {
  // 0-1 BFS over the NFA: CHAR edges cost 1, everything else 0 (assertions treated as passable)
  std::vector<uint32_t> dist(prog.insts.size(), 0xFFFFFFFFu);
  std::deque<int> dq;
  dist[start] = 0; dq.push_back(start);
  while (!dq.empty()) {
    int p = dq.front(); dq.pop_front();
    const Inst& in = prog.insts[p];
    auto relax = [&](int q, uint32_t w) {
      if (q < 0) return;
      if (dist[p] + w < dist[q]) { dist[q] = dist[p] + w; if (w) dq.push_back(q); else dq.push_front(q); }
    };
    switch (in.op) {
      case I_MATCH: return dist[p];
      case I_CHAR: relax(in.x, 1); break;
      case I_ASSERT: relax(in.x, 0); break;
      case I_SAVE: relax(in.x, 0); break;
      case I_SPLIT: relax(in.x, 0); relax(in.y, 0); break;
    }
  }
  return 0xFFFFFFFFu;
}

// The instructions reachable from `start`, renumbered in discovery order, with per-rule set numbering.
static void export_nfa(const Prog& prog, const Classes& C, int start, NfaOut& o) {
  std::vector<int> id(prog.insts.size(), -1), order, st = {start};
  while (!st.empty()) {
    int p = st.back(); st.pop_back();
    if (p < 0 || id[p] >= 0) continue;
    id[p] = (int)order.size();
    order.push_back(p);
    const Inst& in = prog.insts[p];
    if (in.op == I_SPLIT) { st.push_back(in.y); st.push_back(in.x); }
    else if (in.op != I_MATCH) st.push_back(in.x);
  }
  std::map<int, uint32_t> setmap;
  o.wpc = (C.ncls + 31) / 32;
  o.ninst = (uint32_t)order.size();
  o.start = 0;
  o.ngroups = 0;
  o.code.assign((size_t)o.ninst * 3, 0);
  for (size_t k = 0; k < order.size(); ++k) {
    const Inst& in = prog.insts[order[k]];
    uint32_t arg = 0, x = in.x >= 0 ? (uint32_t)id[in.x] : 0, y = 0;
    switch (in.op) {
      case I_CHAR: {
        auto it = setmap.find(in.set);
        if (it == setmap.end()) {
          uint32_t sid = (uint32_t)setmap.size();
          it = setmap.insert({in.set, sid}).first;
          o.setbits.resize((size_t)(sid + 1) * o.wpc, 0);
          for (uint32_t c = 0; c < C.ncls; ++c) if (C.set_has[in.set][c]) o.setbits[(size_t)sid * o.wpc + (c >> 5)] |= 1u << (c & 31);
        }
        arg = it->second;
        break;
      }
      case I_SPLIT: y = in.y >= 0 ? (uint32_t)id[in.y] : 0; break;
      case I_ASSERT: arg = in.kind; break;
      case I_SAVE: arg = in.kind; if (in.kind / 2 > o.ngroups) o.ngroups = in.kind / 2; break;
      case I_MATCH: break;
    }
    o.code[3 * k] = (uint32_t)in.op | (arg << 8);
    o.code[3 * k + 1] = x;
    o.code[3 * k + 2] = y;
  }
  if (o.setbits.empty()) o.setbits.assign(o.wpc, 0);
}

}  // namespace

int compile(const std::vector<PatternIn>& pats, const std::vector<uint8_t>& want_ordered,
            const CharSet& word_set, CompileOut* out, std::string* err) {
  if (pats.empty()) { if (err) *err = "no patterns"; return CF_E_BADARG; }
  if (want_ordered.size() != pats.size()) { if (err) *err = "want_ordered size"; return CF_E_BADARG; }
  Prog prog;
  for (size_t i = 0; i < pats.size(); ++i) {
    Node root;
    size_t pos = 0;
    if (!parse_node(pats[i].ast, pos, root, 0) || pos != pats[i].ast.size()) {
      if (err) *err = "malformed AST for pattern " + std::to_string(i);
      return CF_E_BADARG;
    }
    Inst m; m.op = I_MATCH; m.pat = (int)i;
    int mpc = prog.add(m);
    int s = prog.comp(root, mpc);
    if (prog.overflow) { if (err) *err = "pattern " + std::to_string(i) + ": NFA too large"; return CF_E_TOO_LARGE; }
    prog.start.push_back(s);
  }
  Classes C;
  int rc = build_classes(prog, word_set, C, err);
  if (rc) return rc;

  uint32_t npat = (uint32_t)pats.size();
  out->info.resize(npat);
  uint32_t W = (npat + 63) / 64;
  out->always_bits.assign(W, 0);
  for (uint32_t i = 0; i < npat; ++i) {
    out->info[i].min_len_chars = min_len(prog, prog.start[i]);
    // A substitution rule that can match "" (with or without assertions) is applied to every unit: its verdict bit only selects
    // the units the substitution kernel visits, and "matches somewhere, possibly at the very end" is not worth a scan of its own.
    out->info[i].nullable_always = nullable_no_assert(prog, prog.start[i]) || (want_ordered[i] && out->info[i].min_len_chars == 0);
    if (out->info[i].nullable_always) out->always_bits[i >> 6] |= 1ull << (i & 63);
  }

  // union search DFA (patterns that always match are left out of the automaton: their bit is
  // constant, and keeping them would make every byte a prefilter candidate)
  {
    DfaBuilder B(prog, C, false, npat, 60000);
    std::vector<int> k;
    for (uint32_t i = 0; i < npat; ++i) if (!out->info[i].nullable_always) k.push_back(prog.start[i]);
    uint32_t ss[4] = {0, 0, 0, 0};
    if (!k.empty()) B.build(k, ss); else B.trans.assign(C.ncls + 1, 0);
    if (B.overflow) { if (err) *err = "search DFA too large (state explosion)"; return CF_E_TOO_LARGE; }
    B.emit(out->search, ss);
  }
  // prefilter
  std::vector<PatFilter> pf(npat);
  for (uint32_t i = 0; i < npat; ++i) {
    if (out->info[i].nullable_always) continue;   // empty filter: never a candidate
    rc = pattern_filter(prog, C, (int)i, pf[i], err);
    if (rc) return rc;
  }
  assign_buckets(pf, out->filter, true);

  // ordered (leftmost-first) DFAs
  for (uint32_t i = 0; i < npat; ++i) {
    if (!want_ordered[i]) continue;
    DfaBuilder B(prog, C, true, npat, 60000);
    std::vector<int> k = {prog.start[i]};
    uint32_t ss[4], sa[4];
    B.build(k, ss, sa);
    if (B.overflow) { if (err) *err = "ordered DFA too large for pattern " + std::to_string(i); return CF_E_TOO_LARGE; }
    DfaOut d;
    B.emit(d, ss, sa);
    out->ordered.push_back(std::move(d));
    std::vector<PatFilter> one(1);
    one[0] = pf[i];
    FilterOut fo;
    assign_buckets(one, fo, false);
    out->ordered_filter.push_back(fo);
    NfaOut nfa;
    export_nfa(prog, C, prog.start[i], nfa);
    out->ordered_nfa.push_back(std::move(nfa));
  }
  return 0;
}

}  // namespace cfre
