// cfgpu.cu — device half of libcfgpu.so (include/cfgpu.h): contexts, table upload, batches and
// the sm_90a kernels of the plugin hook-chain hot path.
//
// Kernel inventory
//   prep_kernel      per scan: bitmap initialisation (always-match bits), tile -> first-unit index
//   scan_kernel      the fused multi-pattern scan (harmful + deny + regex_filter dirty detection):
//                    persistent CTAs, TMA (cp.async.bulk) tile ring in shared memory, per byte one
//                    LDS + 4 integer ops shift-AND prefilter, rare candidates verified by an
//                    anchored class DFA (scan_core.h) cooperatively within the warp.
// This is HBM-bound byte work: no tensor cores by design.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <new>
#include <string>
#include <vector>


#include "cf_internal.h"

// ------------------------------------------------------------------------------------------------
// device helpers: mbarrier + 1-D TMA bulk copy
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// --- the same primitives on 32-bit absolute shared addresses (no generic->shared conversion, true LDS) ---
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d_a(uint32_t dst, const CUtensorMap* tmap, int32_t x, int32_t y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(tmap), "r"(x), "r"(y), "r"(bar)
      : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// 2-D tiled TMA load (rows of 128 bytes, SWIZZLE_128B): one instruction per tile
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tmap, int32_t x, int32_t y, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}

// ------------------------------------------------------------------------------------------------
// scan pipeline: fill (only when some pattern matches every unit) -> scan_kernel -> verify_kernel
// ------------------------------------------------------------------------------------------------
__global__ void fill_bitmaps_kernel(uint64_t* __restrict__ bitmaps, const uint64_t* __restrict__ always,
                                    uint32_t W, uint64_t total) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) bitmaps[i] = always[i % W];
}

struct ScanParams {
  const uint8_t* stream;     // device pointer to stream byte 0 (FRONT_PAD bytes of 0xFF precede it)
  uint64_t nbytes;           // stream length including terminators
  uint64_t ntiles;
  const uint64_t* offsets;
  const uint32_t* coarse;    // coarse[k] = unit containing stream byte k << cf::COARSE_SHIFT
  uint32_t n_units;
  const uint32_t* E;
  cf::DfaTables dfa;
  unsigned long long* bitmaps;
  unsigned long long* queue;      // candidate start positions; CTA c owns [c*qcap_cta, (c+1)*qcap_cta)
  unsigned long long* qstate;     // [0] = candidates found, [1] = DFA steps (statistics, this scan)
  unsigned long long* qstate_next; // the pair the NEXT scan will use; CTA 0 zeroes it
  uint32_t qcap_cta;
  uint32_t dfa_bytes;             // bytes needed to stage the DFA tables in shared memory (0 = too big)
  uint32_t dfa_trans_bytes, dfa_acc_bytes;
  uint32_t mulc;                  // 1024 (kept out of the instruction stream on purpose)
};

// Verify one candidate start: run the anchored class DFA from `start` until it dies or reaches the
// unit's 0xFF terminator; unit boundaries come from the terminators themselves.  The unit INDEX is
// only needed when something matched: one probe of the 4 KiB-granular coarse index + a short walk.
__device__ __forceinline__ uint32_t unit_of(const ScanParams& P, uint64_t pos) {
  uint32_t u = P.coarse[pos >> cf::COARSE_SHIFT];
  while (P.offsets[u + 1] <= pos) ++u;
  return u;
}

__device__ __noinline__ void verify_candidate(const ScanParams& P, const cf::DfaTables& t, uint64_t start, uint32_t& steps) {
  if (start >= P.nbytes) return;                       // pad region
  const uint8_t* __restrict__ s = P.stream;
  const uint32_t b0 = s[start];
  if ((b0 & 0xC0) == 0x80) return;                     // not a character boundary
  uint32_t ctx;
  if (s[start - 1] == cf::TERM) ctx = cf::P_START;     // FRONT_PAD makes s[-1] valid for unit 0
  else ctx = cf::prev_context(t, s, start >= 4 ? start - 4 : 0, start); // backward scan stops at any non-continuation byte (no wrap-around in unit 0)
  uint32_t S = t.start_state[ctx];
  uint64_t q = start;
  const bool small = t.W <= 2;
  unsigned long long bits0 = 0, bits1 = 0;
  uint32_t unit = 0xFFFFFFFFu;
  while (S != cf::DEAD) {
    uint32_t col, len = 0;
    const bool eot = s[q] == cf::TERM;
    if (eot) col = t.ncols - 1;
    else col = cf::final_nl(t, cf::classify(t, cf::utf8_decode(s, q, q + 4, &len)), s[q + 1] == cf::TERM);
    uint32_t e = t.trans[(uint64_t)S * t.ncols + col];
    uint32_t a = e >> cf::ACC_SHIFT;
    if (a) {
      if (small) {
        bits0 |= t.accsets[(uint64_t)a * t.W];
        if (t.W == 2) bits1 |= t.accsets[(uint64_t)a * 2 + 1];
      } else {
        if (unit == 0xFFFFFFFFu) unit = unit_of(P, start);
        for (uint32_t w = 0; w < t.W; ++w) {
          unsigned long long v = t.accsets[(uint64_t)a * t.W + w];
          if (v) atomicOr(&P.bitmaps[(uint64_t)unit * t.W + w], v);
        }
      }
    }
    S = e & 0xFFFFu;
    ++steps;
    if (eot) break;
    q += len;
  }
  if (bits0 | bits1) {
    unit = unit_of(P, start);
    if (bits0) atomicOr(&P.bitmaps[(uint64_t)unit * t.W], bits0);
    if (bits1) atomicOr(&P.bitmaps[(uint64_t)unit * t.W + 1], bits1);
  }
}

static const uint32_t WQ = 32;          // per-warp candidate staging slots in shared memory
static const uint32_t SCAN_SMEM = 227 * 1024;   // whole opt-in shared memory of the SM (1 CTA per SM)

// Small per-CTA bookkeeping that lives next to the tile stages.
static const uint32_t MAX_STAGES = 5;   // mbarrier slots: at least the stages of either filter's ring
struct ScanMisc {
  alignas(8) unsigned long long wq[SCAN_WARPS][WQ];
  uint32_t wq_n[SCAN_WARPS];
  uint32_t cq_n;                   // candidates in this CTA's global queue segment
  alignas(8) uint64_t full[MAX_STAGES];
  alignas(8) uint64_t empty[MAX_STAGES];
};

// append one candidate (called by the few lanes that found one; divergent context)
__device__ __noinline__ void push_candidate(ScanMisc& sm, const ScanParams& P, uint32_t warp, uint64_t pos) {
  uint32_t slot = atomicAdd(&sm.wq_n[warp], 1u);
  if (slot < WQ) { sm.wq[warp][slot] = pos; return; }
  // staging full (pathologically dense candidates): go straight to the CTA queue
  uint32_t g = atomicAdd(&sm.cq_n, 1u);
  if (g < P.qcap_cta) P.queue[(uint64_t)blockIdx.x * P.qcap_cta + g] = pos;
  else { uint32_t st = 0; verify_candidate(P, P.dfa, pos, st); }   // queue full: verify in place
}

// warp-cooperative flush of the staging slots into the CTA's queue segment
__device__ __forceinline__ void flush_candidates(ScanMisc& sm, const ScanParams& P, uint32_t warp, uint32_t lane) {
  uint32_t n = sm.wq_n[warp];
  if (n > WQ) n = WQ;
  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(&sm.cq_n, n);
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (lane < n) {
    unsigned long long pos = sm.wq[warp][lane];
    if (base + lane < P.qcap_cta) P.queue[(uint64_t)blockIdx.x * P.qcap_cta + base + lane] = pos;
    else { uint32_t st = 0; verify_candidate(P, P.dfa, pos, st); }
  }
  __syncwarp();
  if (lane == 0) sm.wq_n[warp] = 0;
  __syncwarp();
}

// Prefilter tables in shared memory, "lane-private bank" layout at a 64 KiB-aligned ABSOLUTE shared
// address T.  Each byte value b owns a 256-byte row: lanes' copies of E1[b] in the first half, of F[b]
// in the second:   E1(b, l) = T + (b << 8) + (l << 2)        F(b, l) = T + (b << 8) + 128 + (l << 2)
//   * bank = l for every lookup -> conflict-free for any input bytes
//   * the full 32-bit shared address is produced by ONE PRMT: bytes {l<<2 (|0x80), b, T>>16, 0} taken from
//     the data word and a per-lane constant -> no address arithmetic in the loop
//   * TWO bytes advance per step:  acc = (acc * 1024 + 1023) & F[b0] & E1[b1]
//       F[b]  = (E[b] << 5) | 31          first byte of the pair, pre-shifted
//       E1[b] = E[b] | 0x3E000000         second byte; keeps the first byte's candidate field (bits 25-29)
//     one IMAD (FMA pipe; the multiplier is kept out of the immediate field so that ptxas cannot turn it
//     back into an ALU-pipe shift) + one 3-input LOP3 per two bytes.
static const uint32_t HIT2 = 0x3FF00000u;   // candidate fields of both bytes of a pair

__device__ __forceinline__ uint32_t lds_abs(uint32_t addr) {
  uint32_t v;
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t pair_step(uint32_t acc, uint32_t f0, uint32_t e1, uint32_t mulc) {
  uint32_t t;
  asm("mad.lo.u32 %0, %1, %2, 1023;" : "=r"(t) : "r"(acc), "r"(mulc));
  return t & f0 & e1;
}

// two bytes (k, k+1) of `word`
#define FEEDP(word, k, H)                                                                        \
  {                                                                                              \
    const uint32_t a0_ = __byte_perm((word), laneKF, 0x7604 | ((k) << 4));       /* F[b_k]   */  \
    const uint32_t a1_ = __byte_perm((word), laneK, 0x7604 | (((k) + 1) << 4));  /* E1[b_k+1] */ \
    acc = pair_step(acc, lds_abs(a0_), lds_abs(a1_), mulc);                                      \
    H |= acc;                                                                                    \
  }

// rare path, lane-local: re-run one 16-byte group one byte at a time with position tracking
// (data still in registers; E[b] is recovered from the E1 copy)
#define REFEED(word, k, bit)                                                                    \
  {                                                                                             \
    const uint32_t a_ = __byte_perm((word), laneK, 0x7604 | ((k) << 4));                        \
    acc = ((acc << 5) | 31u) & (lds_abs(a_) & 0x01FFFFFFu);                                     \
    m |= ((acc & 0x01F00000u) ? 1u : 0u) << (bit);                                              \
  }
#define REFEED4(word, b0) REFEED(word, 0, (b0)) REFEED(word, 1, (b0) + 1) REFEED(word, 2, (b0) + 2) REFEED(word, 3, (b0) + 3)
#define REGROUP(prevword, v, gpos)                                                              \
  {                                                                                             \
    uint32_t acc = 0, m = 0;                                                                    \
    REFEED4(prevword, 0)                                                                        \
    m = 0;                                                                                      \
    REFEED4((v).x, 0) REFEED4((v).y, 4) REFEED4((v).z, 8) REFEED4((v).w, 12)                    \
    while (m) {                                                                                 \
      const uint32_t k_ = __ffs(m) - 1;                                                         \
      m &= m - 1;                                                                               \
      push_candidate(sm, P, warp, (gpos) + k_ - 3);                                             \
    }                                                                                           \
  }

// ---- pair prefilter (scan_core.h; chosen at compile time of the rule set when the byte filter would admit
// too many windows).  Table: PF_SLOTS rows of 128 bytes, lane-private banks again:
//   T(h, l) = tbl + (h << 7) + (l << 2),   h = pair_hash(previous byte, byte)
// Per byte: PRMT {prev, cur, prev, cur} -> IMAD (hash) -> SHF -> IMAD (address) -> LDS -> IMAD (acc*256+255) -> LOP3.
template <uint32_t K>
__device__ __forceinline__ uint32_t pair_u(uint32_t pw, uint32_t w) {
  if (K == 0) return __byte_perm(pw, w, 0x4343);                                 // last byte of the previous word, first of this
  return __byte_perm(w, 0u, (K << 12) | ((K - 1) << 8) | (K << 4) | (K - 1));
}
__device__ __forceinline__ uint32_t pairq_step(uint32_t acc, uint32_t u, uint32_t lane_base, uint32_t mulc) {
  const uint32_t h = (u * cf::PF_MULT) >> 22;
  const uint32_t e = lds_abs(h * 128u + lane_base);
  uint32_t t;
  asm("mad.lo.u32 %0, %1, %2, 255;" : "=r"(t) : "r"(acc), "r"(mulc));
  return t & e;
}
// look-back: bytes 1..3 of `w` (byte 0 only serves as the first predecessor); hits belong to the previous owner
#define QFEED_LB(ACCV, w)                                             \
  ACCV = pairq_step(ACCV, pair_u<1>(0u, (w)), lane_base, mulc);       \
  ACCV = pairq_step(ACCV, pair_u<2>(0u, (w)), lane_base, mulc);       \
  ACCV = pairq_step(ACCV, pair_u<3>(0u, (w)), lane_base, mulc);
#define QFEED4(ACCV, pw, w, H)                                        \
  ACCV = pairq_step(ACCV, pair_u<0>((pw), (w)), lane_base, mulc); H |= ACCV; \
  ACCV = pairq_step(ACCV, pair_u<1>(0u, (w)), lane_base, mulc); H |= ACCV;   \
  ACCV = pairq_step(ACCV, pair_u<2>(0u, (w)), lane_base, mulc); H |= ACCV;   \
  ACCV = pairq_step(ACCV, pair_u<3>(0u, (w)), lane_base, mulc); H |= ACCV;
// rare path: exact positions inside one 16-byte group
#define QREFEED(pw, w, K, bit)                                        \
  acc_ = pairq_step(acc_, pair_u<K>((pw), (w)), lane_base, mulc);     \
  m_ |= ((acc_ & cf::PF_HIT) ? 1u : 0u) << (bit);
#define QREFEED4(pw, w, b0) QREFEED(pw, w, 0, (b0)) QREFEED(pw, w, 1, (b0) + 1) QREFEED(pw, w, 2, (b0) + 2) QREFEED(pw, w, 3, (b0) + 3)
#define QREGROUP(prevword, v, gpos)                                   \
  {                                                                   \
    uint32_t acc_ = 0, m_ = 0;                                        \
    QFEED_LB(acc_, (prevword))                                        \
    QREFEED4((prevword), (v).x, 0) QREFEED4((v).x, (v).y, 4) QREFEED4((v).y, (v).z, 8) QREFEED4((v).z, (v).w, 12) \
    while (m_) {                                                      \
      const uint32_t k_ = __ffs(m_) - 1;                              \
      m_ &= m_ - 1;                                                   \
      push_candidate(sm, P, warp, (gpos) + k_ - 3);                   \
    }                                                                 \
  }

// PAIR = 0: byte prefilter; PAIR = 1: pair prefilter.  Geometry: SCAN_WARPS, SCAN_LANE_BYTES (cf_internal.h).
template <uint32_t PAIR>
__global__ void __launch_bounds__(SCAN_WARPS * 32, 1) scan_kernel(const __grid_constant__ ScanParams P,
                                                                    const __grid_constant__ CUtensorMap tmap) {
  // TMA ring depth: 3 for the byte filter (4 measured slower, DESIGN §6); the pair filter's 128 KiB table leaves room for 2
  constexpr uint32_t STAGES = PAIR ? 2 : 3;
  static_assert(STAGES <= MAX_STAGES, "one full / empty mbarrier pair per stage");
  constexpr uint32_t NS = SCAN_LANE_BYTES / 16;     // 16-byte slots per lane per tile
  static_assert(NS == 4, "the feeds below are written for 64 bytes per lane");
  constexpr uint32_t LPR = 128 / SCAN_LANE_BYTES;   // lanes per 128-byte row
  constexpr int32_t TROWS = SCAN_BOX_ROWS;          // a tile is one TMA box
  constexpr int32_t ROW0 = cf::FRONT_PAD / 128;     // stream byte 0 is row FRONT_PAD/128 of the buffer
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- carve shared memory: table at the first 64 KiB boundary, tile stages + misc around it.
  // Stage s lives at absolute shared address stage_abs(s): the first NA stages in the gap before the
  // table, the rest behind it (pure arithmetic: no pointer array, so the tile reads stay true LDS).
  const uint32_t abs0 = smem_u32(smem_raw);
  constexpr uint32_t TBL_BYTES = PAIR ? cf::PF_SLOTS * 128u : 0x10000u;
  // byte filter: the one-PRMT address needs a 64 KiB-aligned table; the pair table only needs its 1 KiB alignment
  const uint32_t tbl_abs = PAIR ? ((abs0 + 1023u) & ~1023u) : ((abs0 + 0xFFFFu) & ~0xFFFFu);
  const uint32_t a_base = (abs0 + 1023u) & ~1023u;               // free space before the table
  const uint32_t b_base = tbl_abs + TBL_BYTES;                   // free space after it
  const uint32_t na_fit = (tbl_abs - a_base) / SCAN_TILE;
  const uint32_t NA = na_fit < STAGES ? na_fit : STAGES;
  uint32_t a_end = a_base + NA * SCAN_TILE, b_end = b_base + (STAGES - NA) * SCAN_TILE;
  uint32_t misc_abs;
  if (a_end + sizeof(ScanMisc) <= tbl_abs) misc_abs = a_end; else { misc_abs = b_end; b_end += (uint32_t)sizeof(ScanMisc); }
  if (b_end > abs0 + SCAN_SMEM) __trap();                        // cannot happen: both rings are sized for 227 KiB
  auto stage_abs = [&](uint32_t sidx) -> uint32_t { return sidx < NA ? a_base + sidx * SCAN_TILE : b_base + (sidx - NA) * SCAN_TILE; };
  ScanMisc& sm = *reinterpret_cast<ScanMisc*>(smem_raw + (misc_abs - abs0));
  const uint32_t full_abs = misc_abs + (uint32_t)offsetof(ScanMisc, full);
  const uint32_t empty_abs = misc_abs + (uint32_t)offsetof(ScanMisc, empty);
  uint32_t* tbl = reinterpret_cast<uint32_t*>(smem_raw + (tbl_abs - abs0));
  const uint32_t laneK = (lane << 2) | tbl_abs;                  // tbl_abs has zero low 16 bits
  const uint32_t laneKF = laneK | 0x80u;                         // second half of each row: the F copies
  const uint32_t mulc = P.mulc;                                  // 1024 (pair filter: 256), deliberately not an immediate
  const uint32_t lane_base = tbl_abs + (lane << 2);              // pair filter: T(h, lane) = lane_base + (h << 7)
  (void)laneKF; (void)lane_base;

  auto load_tile = [&](uint32_t slot_, uint32_t tile_) {
    mbar_expect_tx_a(full_abs + 8 * slot_, SCAN_TILE);
    tma_load_2d_a(stage_abs(slot_), &tmap, 0, ROW0 + (int32_t)tile_ * TROWS, full_abs + 8 * slot_);
  };

  const uint32_t first = blockIdx.x, stride = gridDim.x, ntiles = (uint32_t)P.ntiles;
  if (tid < SCAN_WARPS) sm.wq_n[tid] = 0;
  if (tid == 0) {
    sm.cq_n = 0;
    if (blockIdx.x == 0) { P.qstate_next[0] = 0; P.qstate_next[1] = 0; }
    for (uint32_t s = 0; s < STAGES; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], SCAN_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // prologue: put STAGES-1 tiles in flight right away; the table fill below overlaps their latency
    for (uint32_t j = 0; j < STAGES - 1; ++j) {
      const uint32_t tj = first + j * stride;
      if (tj < ntiles) load_tile(j, tj);
    }
  }
  if (PAIR) {
    for (uint32_t i = tid; i < cf::PF_SLOTS * 32; i += SCAN_WARPS * 32) tbl[i] = P.E[i >> 5];   // row h: 32 lane copies of T[h]
  } else {
    for (uint32_t i = tid; i < 256 * 32; i += SCAN_WARPS * 32) {
      const uint32_t e = P.E[i >> 5];
      tbl[(i >> 5) * 64 + (i & 31)] = e | 0x3E000000u;            // E1
      tbl[(i >> 5) * 64 + 32 + (i & 31)] = (e << 5) | 31u;        // F
    }
  }
  __syncthreads();

  // per-lane swizzled offsets of its 16-byte slots and of the word holding its look-back bytes
  const uint32_t g = warp * 32 + lane, row = g / LPR, xr = row & 7, c0 = (g % LPR) * NS;
  uint32_t off[NS];
#pragma unroll
  for (uint32_t j = 0; j < NS; ++j) off[j] = row * 128 + (((c0 + j) ^ xr) << 4);
  const uint32_t gp = g ? g - 1 : 0, rowp = gp / LPR;
  const uint32_t ob = rowp * 128 + (((((gp % LPR) * NS) + NS - 1) ^ (rowp & 7)) << 4) + 12;
  // lane 0 of the CTA takes its look-back word (last 4 bytes of the previous tile) from HBM/L2,
  // fetched one iteration ahead
  const uint8_t* back_ptr = P.stream + (uint64_t)first * SCAN_TILE - 4;
  const uint64_t back_step = (uint64_t)stride * SCAN_TILE;
  uint32_t back_next = 0;
  if (tid == 0 && first < ntiles) back_next = *reinterpret_cast<const uint32_t*>(back_ptr);

  // ring bookkeeping kept incrementally (no div/mod in the loop)
  uint32_t slot = 0, phase = 0;                  // consumer side
  uint32_t pslot = STAGES - 1, pphase = 1;       // producer side: slot / parity of tile it + STAGES - 1
  uint32_t pj = STAGES - 1;                      // its index in this CTA's tile sequence
  for (uint32_t t = first; t < ntiles; t += stride) {
    if (tid == 0) {   // keep STAGES-1 tiles in flight
      const uint32_t tj = t + (STAGES - 1) * stride;
      if (tj < ntiles) {
        if (pj >= STAGES) mbar_wait_a(empty_abs + 8 * pslot, pphase);
        load_tile(pslot, tj);
      }
    }
    if (++pslot == STAGES) { pslot = 0; pphase ^= 1; }
    ++pj;
    uint32_t back = back_next;
    back_ptr += back_step;
    if (tid == 0 && t + stride < ntiles) back_next = *reinterpret_cast<const uint32_t*>(back_ptr);
    mbar_wait_a(full_abs + 8 * slot, phase);

    // this lane's 64 bytes (+ the word holding its 4 look-back bytes)
    const uint32_t chunk = g * SCAN_LANE_BYTES;   // tile-relative
    const uint32_t base = stage_abs(slot);
    if (g) back = lds32(base + ob);
    uint4 v[NS];
#pragma unroll
    for (uint32_t j = 0; j < NS; ++j) v[j] = lds128(base + off[j]);
    __syncwarp();
    if (lane == 0) mbar_arrive_a(empty_abs + 8 * slot);   // slot may be refilled: data is in registers
    if (++slot == STAGES) { slot = 0; phase ^= 1; }

    uint32_t h[NS];
    if (PAIR) {
      // two independent chains (bytes 0-31 and 32-63), one byte per step
      uint32_t accA = 0, accB = 0;
      h[0] = h[1] = h[2] = h[3] = 0;
      QFEED_LB(accA, back)
      QFEED_LB(accB, v[1].w)
      QFEED4(accA, back, v[0].x, h[0]) QFEED4(accB, v[1].w, v[2].x, h[2])
      QFEED4(accA, v[0].x, v[0].y, h[0]) QFEED4(accB, v[2].x, v[2].y, h[2])
      QFEED4(accA, v[0].y, v[0].z, h[0]) QFEED4(accB, v[2].y, v[2].z, h[2])
      QFEED4(accA, v[0].z, v[0].w, h[0]) QFEED4(accB, v[2].z, v[2].w, h[2])
      QFEED4(accA, v[0].w, v[1].x, h[1]) QFEED4(accB, v[2].w, v[3].x, h[3])
      QFEED4(accA, v[1].x, v[1].y, h[1]) QFEED4(accB, v[3].x, v[3].y, h[3])
      QFEED4(accA, v[1].y, v[1].z, h[1]) QFEED4(accB, v[3].y, v[3].z, h[3])
      QFEED4(accA, v[1].z, v[1].w, h[1]) QFEED4(accB, v[3].z, v[3].w, h[3])
    } else {
      // two independent shift-AND chains per lane (bytes 0-31 and 32-63) for instruction-level
      // parallelism; the second chain re-feeds the last word of the first half as its look-back
      uint32_t accA = 0, accB = 0, dA = 0, dB = 0;
      h[0] = h[1] = h[2] = h[3] = 0;
#define FEEDA(word, k, H) { uint32_t acc = accA; FEEDP(word, k, H) accA = acc; }
#define FEEDB(word, k, H) { uint32_t acc = accB; FEEDP(word, k, H) accB = acc; }
#define FEED2(wa, wb, k, HA, HB) FEEDA(wa, k, HA) FEEDB(wb, k, HB)
#define FEED2x4(wa, wb, HA, HB) FEED2(wa, wb, 0, HA, HB) FEED2(wa, wb, 2, HA, HB)
      FEED2x4(back, v[1].w, dA, dB)
      FEED2x4(v[0].x, v[2].x, h[0], h[2]) FEED2x4(v[0].y, v[2].y, h[0], h[2]) FEED2x4(v[0].z, v[2].z, h[0], h[2]) FEED2x4(v[0].w, v[2].w, h[0], h[2])
      FEED2x4(v[1].x, v[3].x, h[1], h[3]) FEED2x4(v[1].y, v[3].y, h[1], h[3]) FEED2x4(v[1].z, v[3].z, h[1], h[3]) FEED2x4(v[1].w, v[3].w, h[1], h[3])
#undef FEED2x4
#undef FEED2
#undef FEEDA
#undef FEEDB
      (void)dA; (void)dB;
    }

    // rare path: an admissible 5-byte window ended in one of this lane's 16-byte groups
    uint32_t hany = 0;
#pragma unroll
    for (uint32_t j = 0; j < NS; ++j) hany |= h[j];
    constexpr uint32_t HITM = PAIR ? cf::PF_HIT : HIT2;
    const bool anyhit = (hany & HITM) != 0;
    if (__any_sync(0xFFFFFFFFu, anyhit)) {
      if (anyhit) {
        const uint64_t cpos = (uint64_t)t * SCAN_TILE + chunk;   // stream offset of this lane's first byte
#pragma unroll
        for (uint32_t j = 0; j < NS; ++j)
          if (h[j] & HITM) {
            if (PAIR) QREGROUP((j ? v[j ? j - 1 : 0].w : back), v[j], cpos + 16 * j)
            else REGROUP((j ? v[j ? j - 1 : 0].w : back), v[j], cpos + 16 * j)
          }
      }
      __syncwarp();
      if (sm.wq_n[warp] >= WQ / 2) flush_candidates(sm, P, warp, lane);
    }
  }
  __syncwarp();
  if (sm.wq_n[warp]) flush_candidates(sm, P, warp, lane);
  __syncthreads();   // every tile this CTA requested has been consumed; table + tile buffers are free

  // ---- tail: verify this CTA's candidates, DFA tables staged over the (now idle) prefilter table
  const uint32_t ncand = sm.cq_n;
  if (ncand == 0) return;
  const uint32_t nq = ncand < P.qcap_cta ? ncand : P.qcap_cta;
  cf::DfaTables T = P.dfa;
  if (P.dfa_bytes && P.dfa_bytes <= 0x10000u) {
    uint8_t* dst = reinterpret_cast<uint8_t*>(tbl);
    uint32_t off_ = 0;
    auto stage_tbl = [&](const void* src, uint32_t bytes) -> const void* {
      const uint32_t words = (bytes + 3) / 4;
      const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
      uint32_t* d32 = reinterpret_cast<uint32_t*>(dst + off_);
      for (uint32_t i = tid; i < words; i += SCAN_WARPS * 32) d32[i] = s32[i];
      const void* r = dst + off_;
      off_ += (words * 4 + 15) & ~15u;
      return r;
    };
    T.ascii_cls = (const uint16_t*)stage_tbl(P.dfa.ascii_cls, 128 * 2);
    T.range_start = (const uint32_t*)stage_tbl(P.dfa.range_start, P.dfa.nranges * 4);
    T.range_cls = (const uint16_t*)stage_tbl(P.dfa.range_cls, P.dfa.nranges * 2);
    T.cls_ctx = (const uint8_t*)stage_tbl(P.dfa.cls_ctx, P.dfa.ncols - 1);
    T.trans = (const uint32_t*)stage_tbl(P.dfa.trans, P.dfa_trans_bytes);
    T.accsets = (const uint64_t*)stage_tbl(P.dfa.accsets, P.dfa_acc_bytes);
    __syncthreads();
  }
  uint32_t steps = 0;
  const unsigned long long* q = P.queue + (uint64_t)blockIdx.x * P.qcap_cta;
  for (uint32_t i = lane * SCAN_WARPS + warp; i < nq; i += SCAN_WARPS * 32)   // spread over warps: less divergence
    verify_candidate(P, T, q[i], steps);
  for (int o = 16; o; o >>= 1) steps += __shfl_xor_sync(0xFFFFFFFFu, steps, o);
  if (lane == 0 && steps) atomicAdd(&P.qstate[1], (unsigned long long)steps);
  if (tid == 0) atomicAdd(&P.qstate[0], (unsigned long long)ncand);
}

// ------------------------------------------------------------------------------------------------
// regex_filter substitution (rare path: only units the scan flagged as containing some rule match).
// One warp per selected unit; rules are applied one after another on the unit's current text
// (plugins/regex_filter/search_replace.py:127-130), each rule = Python `pattern.sub(repl, text)`:
// leftmost-first, non-overlapping matches; a rule that can match "" follows re.sub's empty-match rules.  Every write is clamped
// to the unit's scratch bound, so a bound that is too small is reported (CF_E_TOO_LARGE) instead of overwriting a neighbour.
// ------------------------------------------------------------------------------------------------
static const uint32_t SUB_LAUNCH_RULES = 32;    // rules per sub_kernel launch; longer programs continue in further launches
static const uint32_t SUB_WIN = 512;            // start positions examined per warp iteration
static const uint32_t SUB_WARPS = 4;

struct SubRule {
  cf::DfaTables dfa;
  const uint32_t* E;
  const uint8_t* repl;
  uint32_t repl_len;
  uint32_t nullable;          // the rule can match "": every position is a candidate, re.sub's must_advance rule applies
  // replacement template with group references (n_parts == 0: `repl` is the literal replacement)
  const uint32_t* parts;      // {kind, a, b} triples; literals live in `repl`
  cf::NfaView nfa;
  uint32_t n_parts;
};

struct SubParams {
  const uint8_t* stream;
  const uint64_t* offsets;
  const uint32_t* sel;        // selected unit indices
  const uint64_t* soff;       // per selected unit: offset of its scratch area (two buffers of `bound` bytes)
  const uint64_t* bound;
  uint8_t* scratch;
  uint64_t* rec;              // per selected unit: [0] = text offset in scratch (~0: unchanged, SUB_OVERFLOW), [1] = length
  uint32_t* pike;             // per selected unit: pike_words of Pike-VM scratch (rules with group references only); NULL with
                              // pike_words != 0: in the unit's scratch area, behind its two buffers
  uint64_t pike_words;
  uint32_t n_sel;
  const uint32_t* n_dev;      // not NULL: the number of selected units is on the device (the grid covers n_sel)
  uint32_t n_rules;
  uint32_t first_rule;        // program index of rules[0]
  uint32_t resume;            // 0: start from the stream; 1: continue from `rec` (a previous launch's rules)
  SubRule rules[SUB_LAUNCH_RULES];
};

// dst[pos, pos + n) = src[0, n), clamped to dst[0, cap): an output longer than its scratch area never reaches a neighbour's
__device__ __forceinline__ void warp_put(uint8_t* dst, uint64_t pos, uint64_t cap, const uint8_t* src, uint64_t n, uint32_t lane) {
  const uint64_t m = pos < cap ? (n < cap - pos ? n : cap - pos) : 0;
  for (uint64_t i = lane; i < m; i += 32) dst[pos + i] = src[i];
}

// One replacement at dst[pos] (clamped to cap) for the match of rule R that starts at sp: the literal, or the template with the group
// texts of THIS match (captures by lane 0's Pike VM pass, spans broadcast through shared memory).  Returns the length of the replacement.
__device__ __forceinline__ uint64_t emit_replacement(const SubRule& R, const uint8_t* src, uint64_t len, uint64_t sp, bool must_advance, uint8_t* dst,
                                                     uint64_t pos, uint64_t cap, uint32_t lane, uint32_t* caps_s, uint32_t* pike) {
  if (R.n_parts == 0) { warp_put(dst, pos, cap, R.repl, R.repl_len, lane); return R.repl_len; }
  __syncwarp();
  if (lane == 0) {
    for (uint32_t k = 0; k < R.nfa.nslots; ++k) caps_s[k] = cf::CAP_UNSET;
    cf::pike_captures(R.dfa, R.nfa, src, 0, len, sp, must_advance, pike, caps_s);
  }
  __syncwarp();
  uint64_t o = 0;
  for (uint32_t k = 0; k < R.n_parts; ++k) {
    const uint32_t kind = R.parts[3 * k], a = R.parts[3 * k + 1], b = R.parts[3 * k + 2];
    if (kind == 0) { warp_put(dst, pos + o, cap, R.repl + a, b, lane); o += b; }
    else {
      const uint32_t g0 = caps_s[2 * a], g1 = caps_s[2 * a + 1];
      if (g0 != cf::CAP_UNSET && g1 != cf::CAP_UNSET && g1 >= g0) { warp_put(dst, pos + o, cap, src + g0, g1 - g0, lane); o += g1 - g0; }
    }
  }
  return o;
}

__global__ void __launch_bounds__(SUB_WARPS * 32) sub_kernel(const __grid_constant__ SubParams P) {
  __shared__ uint32_t mlen_s[SUB_WARPS][SUB_WIN];
  __shared__ uint32_t caps_all[SUB_WARPS][64];
  const uint32_t lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
  const uint32_t w = blockIdx.x * SUB_WARPS + wic;
  if (w >= (P.n_dev ? *P.n_dev : P.n_sel)) return;
  uint32_t* mlen = mlen_s[wic];
  uint32_t* caps_s = caps_all[wic];
  uint32_t* pike = nullptr;
  if (P.pike_words) pike = P.pike ? P.pike + (uint64_t)w * P.pike_words : reinterpret_cast<uint32_t*>(P.scratch + P.soff[w] + 2 * P.bound[w]);
  const uint32_t u = P.sel[w];
  const uint8_t* src = P.stream + P.offsets[u];
  uint64_t len = P.offsets[u + 1] - P.offsets[u] - 1;
  const uint64_t cap = P.bound[w];                          // bytes of each buffer of the pair: every write is clamped to it
  uint8_t* bufs[2] = {P.scratch + P.soff[w], P.scratch + P.soff[w] + cap};
  uint32_t which = 0;
  bool changed = false;
  if (P.resume) {          // continue from the previous launch: the stream, or the buffer of the pair it wrote last
    const uint64_t at = P.rec[2 * (uint64_t)w];
    if (at == SUB_OVERFLOW) return;
    if (at != ~0ull) {
      src = P.scratch + at;
      len = P.rec[2 * (uint64_t)w + 1];
      which = src == bufs[0] ? 1 : 0;
      changed = true;
    }
  }

  for (uint32_t r = 0; r < P.n_rules; ++r) {
    const SubRule& R = P.rules[r];
    uint8_t* dst = bufs[which];
    uint64_t out_pos = 0, copied = 0, cur = 0;
    uint32_t nmatch = 0;
    if (R.nullable) {
      // Every character boundary of [0, len] is a candidate (no prefilter).  Per position: e1 = the leftmost-first match, and, when
      // that is the empty match, e2 = the best NON-empty match there — what sre finds when it retries the position with
      // must_advance after an empty match (pattern_subx).  mlen = e1 - sp, mlen2 = e2 - sp (0: there is none).
      uint32_t* mlen2 = mlen + SUB_WIN / 2;                 // 256 positions per iteration in this mode
      for (uint64_t wbase = 0; wbase <= len; wbase += SUB_WIN / 2) {
        const uint64_t b0 = wbase + (uint64_t)lane * 8;
        uint32_t has = 0;
        for (uint32_t k = 0; k < 8; ++k) {
          const uint64_t sp = b0 + k;
          if (sp > len || (sp < len && (src[sp] & 0xC0) == 0x80)) continue;
          const uint64_t e1 = cf::match_first(R.dfa, src, 0, len, sp);
          if (e1 == ~0ull) continue;
          uint32_t m1 = (uint32_t)(e1 - sp), m2 = 0;
          if (e1 == sp) {
            const uint64_t e2 = cf::match_first(R.dfa, src, 0, len, sp, true);
            if (e2 != ~0ull) m2 = (uint32_t)(e2 - sp);
          }
          mlen[lane * 8 + k] = m1; mlen2[lane * 8 + k] = m2;
          has |= 1u << k;
        }
        __syncwarp();
        for (uint32_t L = 0; L < 32; ++L) {
          uint32_t mk = __shfl_sync(0xFFFFFFFFu, has, L);
          while (mk) {
            const uint32_t k = __ffs(mk) - 1;
            mk &= mk - 1;
            const uint64_t sp = wbase + (uint64_t)L * 8 + k;
            if (sp < cur) continue;                     // inside the previous match
            const uint32_t m1 = mlen[L * 8 + k], m2 = mlen2[L * 8 + k];
            warp_put(dst, out_pos, cap, src + copied, sp - copied, lane);
            out_pos += sp - copied;
            out_pos += emit_replacement(R, src, len, sp, false, dst, out_pos, cap, lane, caps_s, pike);
            ++nmatch;
            if (m1 == 0 && m2) {                        // empty match, then the non-empty one at the same position
              out_pos += emit_replacement(R, src, len, sp, true, dst, out_pos, cap, lane, caps_s, pike);
              ++nmatch;
            }
            copied = cur = sp + (m1 ? m1 : m2);
          }
        }
        __syncwarp();
      }
    } else
    for (uint64_t wbase = 0; wbase < len; wbase += SUB_WIN) {
      // prefilter the 16 start positions owned by this lane (5-byte window: start-1 .. start+3)
      const uint64_t b0 = wbase + (uint64_t)lane * 16;
      uint32_t acc = 0, cand = 0;
      for (int k = -1; k < 19; ++k) {
        const int64_t pos = (int64_t)b0 + k;
        const uint32_t byte = (pos < 0 || (uint64_t)pos >= len) ? (uint32_t)cf::TERM : (uint32_t)src[pos];
        acc = cf::filter_step(acc, R.E[byte]);
        if (k >= 3 && (acc & cf::F_HIT)) cand |= 1u << (k - 3);
      }
      uint32_t has = 0;
      for (uint32_t k = 0; k < 16; ++k) mlen[lane * 16 + k] = 0;
      while (cand) {
        const uint32_t k = __ffs(cand) - 1;
        cand &= cand - 1;
        const uint64_t sp = b0 + k;
        if (sp >= len || (src[sp] & 0xC0) == 0x80) continue;
        const uint64_t e = cf::match_first(R.dfa, src, 0, len, sp);
        if (e != ~0ull && e > sp) { mlen[lane * 16 + k] = (uint32_t)(e - sp); has |= 1u << k; }
      }
      __syncwarp();
      // resolve overlaps left to right (uniform across the warp) and emit
      for (uint32_t L = 0; L < 32; ++L) {
        uint32_t mk = __shfl_sync(0xFFFFFFFFu, has, L);
        while (mk) {
          const uint32_t k = __ffs(mk) - 1;
          mk &= mk - 1;
          const uint64_t sp = wbase + (uint64_t)L * 16 + k;
          if (sp < cur) continue;                       // inside the previous match
          const uint32_t ml = mlen[L * 16 + k];
          warp_put(dst, out_pos, cap, src + copied, sp - copied, lane);
          out_pos += sp - copied;
          out_pos += emit_replacement(R, src, len, sp, false, dst, out_pos, cap, lane, caps_s, pike);
          copied = cur = sp + ml;
          ++nmatch;
        }
      }
      __syncwarp();
    }
    if (nmatch) {
      warp_put(dst, out_pos, cap, src + copied, len - copied, lane);
      out_pos += len - copied;
      if (out_pos > cap) {           // the scratch bound was too small for this rule's output: the host reports the unit and the rule
        if (lane == 0) { P.rec[2 * (uint64_t)w] = SUB_OVERFLOW; P.rec[2 * (uint64_t)w + 1] = P.first_rule + r; }
        return;
      }
      __syncwarp();
      __threadfence_block();
      src = dst;
      len = out_pos;
      which ^= 1;
      changed = true;
    }
  }
  __syncwarp();                      // every lane has read this unit's `rec` (resume) before lane 0 rewrites it
  if (lane == 0) {
    P.rec[2 * (uint64_t)w] = changed ? (uint64_t)(src - P.scratch) : ~0ull;
    P.rec[2 * (uint64_t)w + 1] = len;
  }
}

// Scratch bound of a unit of `len` bytes: worst = its worst-case growth through all rules.  A rule with matches of >= ml characters
// (so >= ml bytes) turns L bytes into at most L * ceil(repl / ml); a rule that can match "" has at most L + 1 empty and L non-empty
// matches; a template emits its literals and each referenced group (at most the match itself) per match.  Over a long program that
// product is far above what any text needs (a -> bb, bb -> c, ... doubles it at every other rule), so the first pass gives a unit at
// most 64 L + 64 KiB.  Host (cf_sub_device) and device (sub_select_kernel) share the formula.
__host__ __device__ inline double sub_worst(uint64_t len, const RuleGrowth* g, uint32_t nr) {
  double bd = (double)len;
  for (uint32_t r = 0; r < nr; ++r) {
    const uint32_t ml = g[r].minlen;
    if (g[r].n_parts) {
      const double nmatch = ml ? bd / ml + 1.0 : 2.0 * bd + 1.0;
      bd = bd * (1.0 + g[r].nrefs) + nmatch * (double)g[r].lit_len;
    } else if (ml == 0) bd += (2.0 * bd + 1.0) * (double)g[r].repl_len;
    else { const double f = (double)((g[r].repl_len + ml - 1) / ml); if (f > 1.0) bd *= f; }
  }
  return bd + 16.0;
}
__host__ __device__ inline uint64_t sub_round16(double x) { return ((uint64_t)x + 15) & ~15ull; }
__host__ __device__ inline uint64_t sub_first_bound(uint64_t len, double worst) {
  const double cap = 64.0 * (double)len + 65536.0;
  return sub_round16(worst < cap ? worst : cap);
}

// cf_run_enqueue: the dirty units (a CF_PAT_ORDERED bit set, SUB allowed by the unit's stages), their first-pass bounds, and their two
// scratch buffers (+ Pike-VM words) from the run's arena by an atomic cursor.  The units that fit are compacted with a warp ballot
// into sel / soff / bound (slot[u] = selection index); the others are deferred to cf_run_finish.  The cursor's final value is what
// the call needed: every dirty unit adds to it, fitting or not.
__global__ void __launch_bounds__(256) sub_select_kernel(const uint64_t* __restrict__ bm, uint32_t W, const uint64_t* __restrict__ rule_mask,
                                                         const uint8_t* __restrict__ unit_stages, const uint64_t* __restrict__ offsets, uint32_t n,
                                                         const RuleGrowth* __restrict__ g, uint32_t nr, uint64_t pike_bytes, uint64_t arena_bytes,
                                                         RunStatus* st, uint32_t* __restrict__ slot, uint32_t* __restrict__ sel,
                                                         uint64_t* __restrict__ soff, uint64_t* __restrict__ bound) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  bool dirty = false, fit = false;
  uint64_t off = 0, bd = 0;
  if (u < n && (!unit_stages || (unit_stages[u] & CF_STAGE_SUB)))
    for (uint32_t w = 0; w < W; ++w)
      if (bm[(uint64_t)u * W + w] & rule_mask[w]) { dirty = true; break; }
  if (dirty) {
    const uint64_t len = offsets[u + 1] - offsets[u] - 1;
    bd = sub_first_bound(len, sub_worst(len, g, nr));
    const uint64_t need = 2 * bd + pike_bytes;
    off = atomicAdd(reinterpret_cast<unsigned long long*>(&st->arena_used), (unsigned long long)need);
    fit = off + need <= arena_bytes;
  }
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, fit);
  uint32_t base = 0;
  if (lane == 0 && m) base = atomicAdd(&st->n_sel, (uint32_t)__popc(m));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (u >= n) return;
  if (fit) {
    const uint32_t w = base + __popc(m & ((1u << lane) - 1u));
    sel[w] = u;
    soff[w] = off;
    bound[w] = bd;
    slot[u] = w;
  } else slot[u] = dirty ? RUN_DEFER_PENDING : RUN_NOT_DIRTY;
}

__global__ void sub_compact_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets,
                                   const uint32_t* __restrict__ sel, const uint8_t* __restrict__ scratch,
                                   const uint64_t* __restrict__ rec, const uint64_t* __restrict__ out_off,
                                   uint8_t* __restrict__ out, uint32_t n_sel) {
  const uint32_t w = blockIdx.x;
  if (w >= n_sel) return;
  const uint64_t n = rec[2 * (uint64_t)w + 1];
  const uint8_t* src = rec[2 * (uint64_t)w] == ~0ull ? stream + offsets[sel[w]] : scratch + rec[2 * (uint64_t)w];
  uint8_t* dst = out + out_off[w];
  for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------------------
// host API
// ------------------------------------------------------------------------------------------------
template <typename T>
static int upload(cf_ctx* ctx, const std::vector<T>& v, const T** out, std::vector<void*>& allocs) {
  void* d = nullptr;
  size_t bytes = (v.size() ? v.size() : 1) * sizeof(T);
  bytes = (bytes + 15) & ~(size_t)15;   // the scan kernel stages tables into shared memory in whole 32-bit words (compute-sanitizer memcheck, round 2)
  CF_CUDA(ctx, cudaMalloc(&d, bytes));
  allocs.push_back(d);
  if (!v.empty()) CF_CUDA(ctx, cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = (const T*)d;
  return CF_OK;
}

static int upload_dfa(cf_ctx* ctx, const cfre::DfaOut& d, DevDfa& o) {
  int rc;
  if ((rc = upload(ctx, d.ascii_cls, &o.t.ascii_cls, o.allocs))) return rc;
  if ((rc = upload(ctx, d.range_start, &o.t.range_start, o.allocs))) return rc;
  if ((rc = upload(ctx, d.range_cls, &o.t.range_cls, o.allocs))) return rc;
  if ((rc = upload(ctx, d.cls_ctx, &o.t.cls_ctx, o.allocs))) return rc;
  if ((rc = upload(ctx, d.trans, &o.t.trans, o.allocs))) return rc;
  if ((rc = upload(ctx, d.accsets, &o.t.accsets, o.allocs))) return rc;
  o.trans_bytes = d.trans.size() * 4;
  o.acc_bytes = d.accsets.size() * 8;
  auto r16 = [](uint64_t b) { return (b + 15) & ~15ull; };
  o.stage_bytes = r16(256) + r16(d.range_start.size() * 4) + r16(d.range_cls.size() * 2) + r16(d.ncols) +
                  r16(o.trans_bytes) + r16(o.acc_bytes) + 64;
  o.t.nranges = (uint32_t)d.range_start.size();
  o.t.ncols = d.ncols;
  o.t.W = d.W;
  for (int i = 0; i < 4; ++i) { o.t.start_state[i] = d.start_state[i]; o.t.start_adv[i] = d.start_adv[i]; }
  o.t.nl_cls = d.nl_cls; o.t.nlf_cls = d.nlf_cls;
  return CF_OK;
}

// ---- the substitution pass shared by cf_sub_host and cf_run_batch (cf_internal.h)
// Descriptors of a pass, one H2D from pinned staging into ctx->sub_desc: soff[n] | bound[n] | sel[n]; then rec[2n] comes back in one D2H.
static size_t sub_desc_bytes(uint32_t n) { return ((size_t)n * 20 + 15) & ~(size_t)15; }
static const uint32_t* sub_desc_sel(const cf_ctx* ctx, uint32_t n) { return (const uint32_t*)((const uint64_t*)ctx->sub_desc.p + 2 * (size_t)n); }
size_t cf_sub_stage_bytes(uint32_t n_sel) { return sub_desc_bytes(n_sel) + (size_t)n_sel * 16; }

// the sub_kernel launches of one pass: SUB_LAUNCH_RULES rules per launch; each further launch continues every unit from the record
// the previous one left
static int sub_launch_rules(cf_ctx* ctx, const cf_prog* p, SubParams& SP, cudaStream_t st) {
  const uint32_t nr = (uint32_t)p->ordered.size();
  for (uint32_t r0 = 0; r0 < nr; r0 += SUB_LAUNCH_RULES) {
    SP.first_rule = r0;
    SP.resume = r0 > 0;
    SP.n_rules = std::min(nr - r0, SUB_LAUNCH_RULES);
    for (uint32_t i = 0; i < SP.n_rules; ++i) {
      const uint32_t r = r0 + i;
      SubRule& S = SP.rules[i];
      S.dfa = p->ordered[r].t;
      S.E = p->d_ordered_E[r];
      S.repl = p->d_repl[r];
      S.repl_len = p->repl_len[r];
      S.nullable = p->ordered_minlen[r] == 0;
      const cf_prog::RuleTmpl& T = p->tmpl[r];
      S.parts = T.d_parts;
      S.n_parts = T.n_parts;
      S.nfa.code = T.d_code; S.nfa.setbits = T.d_sets;
      S.nfa.ninst = T.ninst; S.nfa.start = 0; S.nfa.wpc = T.wpc; S.nfa.nslots = T.nslots;
    }
    sub_kernel<<<(SP.n_sel + SUB_WARPS - 1) / SUB_WARPS, SUB_WARPS * 32, 0, st>>>(SP);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
  }
  return CF_OK;
}

int cf_sub_enqueue(cf_ctx* ctx, cf_prog* p, cf_batch* b, cf_run* run, const uint64_t* d_bitmaps, const uint8_t* d_unit_stages, cudaStream_t st) {
  const uint32_t n = b->n;
  const uint64_t pike_bytes = ((uint64_t)p->pike_words * 4 + 15) & ~15ull;
  sub_select_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_bitmaps, p->W, p->d_rule_mask, d_unit_stages, b->d_offsets, n, p->d_growth,
                                                     (uint32_t)p->ordered.size(), pike_bytes, run->arena_bytes, run->d_status, run->d_slot,
                                                     run->d_sel, run->d_soff, run->d_bound);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  // the launches are sized for every unit; warps past the device's count of selected units exit at once
  SubParams SP;
  SP.stream = b->d_buf + cf::FRONT_PAD;
  SP.offsets = b->d_offsets;
  SP.sel = run->d_sel; SP.soff = run->d_soff; SP.bound = run->d_bound;
  SP.scratch = run->d_arena;
  SP.rec = run->d_rec;
  SP.pike = nullptr; SP.pike_words = p->pike_words;
  SP.n_sel = n;
  SP.n_dev = &run->d_status->n_sel;
  return sub_launch_rules(ctx, p, SP, st);
}

int cf_sub_device(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint64_t* h_offsets, const uint32_t* units, uint32_t n_sel, cudaStream_t st,
                  uint8_t* h_stage, const uint64_t** rec_out) {
  const uint32_t nr = (uint32_t)p->ordered.size();
  if (nr == 0) { ctx->err = "program has no substitution rules"; return CF_E_BADARG; }
  uint64_t* soff = (uint64_t*)h_stage;
  uint64_t* bound = soff + n_sel;
  uint32_t* sel = (uint32_t*)(bound + n_sel);
  uint64_t* rec = (uint64_t*)(h_stage + sub_desc_bytes(n_sel));
  // Scratch: two buffers of bound[i] bytes per selected unit, first sub_first_bound.  The kernel clamps every write to the unit's bound
  // and reports a unit whose output outgrew it; that unit runs again with 8x the room, up to worst[i].  Outgrowing worst[i] itself is
  // an internal error (CF_E_TOO_LARGE), never a write into a neighbour's scratch.
  std::vector<double> worst(n_sel);
  for (uint32_t i = 0; i < n_sel; ++i) {
    if (units[i] >= b->n) { ctx->err = "unit index out of range"; return CF_E_BADARG; }
    sel[i] = units[i];
    uint64_t len = h_offsets[units[i] + 1] - h_offsets[units[i]] - 1;
    worst[i] = sub_worst(len, p->growth.data(), nr);
    bound[i] = sub_first_bound(len, worst[i]);
  }
  int rc;
  // grow-only scratch of the context: no cudaMalloc / cudaFree per call
  if ((rc = cf_dev_reserve(ctx, ctx->sub_desc, sub_desc_bytes(n_sel))) || (rc = cf_dev_reserve(ctx, ctx->sub_rec, (size_t)n_sel * 16))) return rc;
  uint64_t* d_desc = (uint64_t*)ctx->sub_desc.p;
  SubParams SP;
  SP.stream = b->d_buf + cf::FRONT_PAD;
  SP.offsets = b->d_offsets;
  SP.soff = d_desc; SP.bound = d_desc + n_sel; SP.sel = sub_desc_sel(ctx, n_sel);
  SP.rec = (uint64_t*)ctx->sub_rec.p;
  SP.n_sel = n_sel;
  SP.n_dev = nullptr;
  SP.pike = nullptr; SP.pike_words = p->pike_words;
  if (SP.pike_words) {
    if ((uint64_t)n_sel * SP.pike_words * 4 > (4ull << 30)) { ctx->err = "capture scratch exceeds 4 GiB (too many units for a rule with group references)"; return CF_E_CAPACITY; }
    if ((rc = cf_dev_reserve(ctx, ctx->sub_pike, (size_t)n_sel * SP.pike_words * 4))) return rc;
    SP.pike = (uint32_t*)ctx->sub_pike.p;
  }
  for (bool again = true; again;) {        // one pass, and another while some unit outgrew a bound below its worst case
    again = false;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n_sel; ++i) { soff[i] = total; total += 2 * bound[i]; }
    if (total > (8ull << 30)) { ctx->err = "substitution scratch exceeds 8 GiB"; return CF_E_CAPACITY; }
    if ((rc = cf_dev_reserve(ctx, ctx->sub_scratch, total))) return rc;
    SP.scratch = (uint8_t*)ctx->sub_scratch.p;
    CF_CUDA(ctx, cudaMemcpyAsync(d_desc, h_stage, sub_desc_bytes(n_sel), cudaMemcpyHostToDevice, st));
    if ((rc = sub_launch_rules(ctx, p, SP, st))) return rc;
    CF_CUDA(ctx, cudaMemcpyAsync(rec, SP.rec, (size_t)n_sel * 16, cudaMemcpyDeviceToHost, st));
    CF_CUDA(ctx, cudaStreamSynchronize(st));
    for (uint32_t i = 0; i < n_sel; ++i) {
      if (rec[2 * (size_t)i] != SUB_OVERFLOW) continue;
      const double grown = std::min(worst[i], 8.0 * (double)bound[i]);
      if ((double)bound[i] >= worst[i]) {
        ctx->err = "substitution of unit " + std::to_string(units[i]) + " (selection index " + std::to_string(i) + "): the output of rule " +
                   std::to_string(rec[2 * (size_t)i + 1]) + " exceeds the worst-case bound of its scratch";
        return CF_E_TOO_LARGE;
      }
      if (grown > 4e9) { ctx->err = "substitution rules expand a unit beyond 4 GB"; return CF_E_CAPACITY; }
      bound[i] = sub_round16(grown);
      again = true;
    }
  }
  *rec_out = rec;
  return CF_OK;
}

extern "C" {

int cf_init(int device_ordinal, cf_ctx** out) {
  if (!out) return CF_E_BADARG;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device_ordinal >= n) return CF_E_NOGPU;
  cf_ctx* ctx = new (std::nothrow) cf_ctx();
  if (!ctx) return CF_E_NOMEM;
  ctx->device = device_ordinal;
  *out = ctx;
  CF_CUDA(ctx, cudaSetDevice(device_ordinal));
  cudaDeviceProp prop;
  CF_CUDA(ctx, cudaGetDeviceProperties(&prop, device_ordinal));
  ctx->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) { ctx->err = "libcfgpu.so is built for sm_90a (Hopper, compute capability 9.0) only"; return CF_E_NOGPU; }
  CF_CUDA(ctx, cudaMalloc(&ctx->d_qstate, 4 * sizeof(uint64_t)));
  CF_CUDA(ctx, cudaMemset(ctx->d_qstate, 0, 4 * sizeof(uint64_t)));
  CF_CUDA(ctx, cudaMalloc(&ctx->d_queue, (size_t)ctx->qcap * sizeof(uint64_t)));
  if (const char* e = getenv("CF_SCAN_RESERVE_SMS")) ctx->scan_reserve_sms = (uint32_t)atoi(e);
  CF_CUDA(ctx, cudaFuncSetAttribute(scan_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SCAN_SMEM));
  CF_CUDA(ctx, cudaFuncSetAttribute(scan_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SCAN_SMEM));
  CF_CUDA(ctx, cf_toon_tp_allow_smem());
  return CF_OK;
}

void cf_shutdown(cf_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaFree(ctx->d_qstate);
  cudaFree(ctx->d_queue);
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  cf_run_free(ctx->run);
  delete ctx;   // frees the DevBuf scratch, on the device set above
}

const char* cf_last_error(cf_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

uint64_t cf_kernel_launches(const cf_ctx* ctx) { return ctx ? ctx->launches : 0; }

int cf_compile(cf_ctx* ctx, cf_builder* b, cf_prog** out) {
  if (!ctx || !b || !out) return CF_E_BADARG;
  int rc = cf_builder_compile_host(b, nullptr);
  if (rc) { ctx->err = b->err; return rc; }
  for (size_t i = 0; i < b->pats.size(); ++i)
    if (b->ordered[i] && !b->has_repl[i]) { ctx->err = "ordered pattern without replacement"; return CF_E_BADARG; }
  CF_CUDA(ctx, cudaSetDevice(ctx->device));
  cf_prog* p = new (std::nothrow) cf_prog();
  if (!p) return CF_E_NOMEM;
  p->ctx = ctx;
  p->npat = (uint32_t)b->pats.size();
  p->W = b->out.search.W;
  *out = p;
  if ((rc = upload_dfa(ctx, b->out.search, p->search))) return rc;
  p->use_pairs = b->out.filter.use_pairs;
  if (p->use_pairs) {   // large rule set: the pair prefilter's table instead of the byte table (scan_core.h)
    CF_CUDA(ctx, cudaMalloc(&p->d_E, cf::PF_SLOTS * 4));
    CF_CUDA(ctx, cudaMemcpy(p->d_E, b->out.filter.pairT.data(), cf::PF_SLOTS * 4, cudaMemcpyHostToDevice));
  } else {
    CF_CUDA(ctx, cudaMalloc(&p->d_E, 256 * 4));
    CF_CUDA(ctx, cudaMemcpy(p->d_E, b->out.filter.E, 256 * 4, cudaMemcpyHostToDevice));
  }
  CF_CUDA(ctx, cudaMalloc(&p->d_always, p->W * 8));
  CF_CUDA(ctx, cudaMemcpy(p->d_always, b->out.always_bits.data(), p->W * 8, cudaMemcpyHostToDevice));
  for (uint64_t v : b->out.always_bits) if (v) p->any_always = true;
  p->search_empty = true;
  for (int i = 0; i < 256; ++i) if (b->out.filter.E[i]) p->search_empty = false;
  size_t oi = 0;
  for (size_t i = 0; i < b->pats.size(); ++i) {
    if (!b->ordered[i]) continue;
    p->ordered.emplace_back();
    if ((rc = upload_dfa(ctx, b->out.ordered[oi], p->ordered.back()))) return rc;
    uint32_t* dE = nullptr;
    CF_CUDA(ctx, cudaMalloc(&dE, 256 * 4));
    CF_CUDA(ctx, cudaMemcpy(dE, b->out.ordered_filter[oi].E, 256 * 4, cudaMemcpyHostToDevice));
    p->d_ordered_E.push_back(dE);
    p->ordered_pat.push_back((int)i);
    uint8_t* dr = nullptr;
    size_t rl = b->repl[i].size();
    CF_CUDA(ctx, cudaMalloc(&dr, rl ? rl : 1));
    if (rl) CF_CUDA(ctx, cudaMemcpy(dr, b->repl[i].data(), rl, cudaMemcpyHostToDevice));
    p->d_repl.push_back(dr);
    p->repl_len.push_back((uint32_t)rl);
    p->ordered_minlen.push_back(b->out.info[i].min_len_chars);
    cf_prog::RuleTmpl T;
    if (!b->tmpl[i].empty()) {
      const cfre::NfaOut& nf = b->out.ordered_nfa[oi];
      T.ninst = nf.ninst; T.wpc = nf.wpc; T.nslots = 2 * (nf.ngroups + 1); T.n_parts = (uint32_t)(b->tmpl[i].size() / 3);
      for (uint32_t k = 0; k < T.n_parts; ++k) { if (b->tmpl[i][3 * k] == 1) ++T.nrefs; else T.lit_len += b->tmpl[i][3 * k + 2]; }
      CF_CUDA(ctx, cudaMalloc(&T.d_code, nf.code.size() * 4));
      CF_CUDA(ctx, cudaMemcpy(T.d_code, nf.code.data(), nf.code.size() * 4, cudaMemcpyHostToDevice));
      CF_CUDA(ctx, cudaMalloc(&T.d_sets, nf.setbits.size() * 4));
      CF_CUDA(ctx, cudaMemcpy(T.d_sets, nf.setbits.data(), nf.setbits.size() * 4, cudaMemcpyHostToDevice));
      CF_CUDA(ctx, cudaMalloc(&T.d_parts, b->tmpl[i].size() * 4));
      CF_CUDA(ctx, cudaMemcpy(T.d_parts, b->tmpl[i].data(), b->tmpl[i].size() * 4, cudaMemcpyHostToDevice));
    }
    p->tmpl.push_back(T);
    p->growth.push_back({p->ordered_minlen.back(), (uint32_t)rl, T.n_parts, T.nrefs, T.lit_len});
    if (T.n_parts) p->pike_words = std::max(p->pike_words, (uint32_t)cf::pike_scratch_words(T.ninst, T.nslots));
    ++oi;
  }
  std::vector<uint64_t> rule_mask(p->W, 0);
  for (int pi : p->ordered_pat) rule_mask[(size_t)pi / 64] |= 1ull << (pi % 64);
  CF_CUDA(ctx, cudaMalloc(&p->d_rule_mask, p->W * 8));
  CF_CUDA(ctx, cudaMemcpy(p->d_rule_mask, rule_mask.data(), p->W * 8, cudaMemcpyHostToDevice));
  if (!p->growth.empty()) {
    CF_CUDA(ctx, cudaMalloc(&p->d_growth, p->growth.size() * sizeof(RuleGrowth)));
    CF_CUDA(ctx, cudaMemcpy(p->d_growth, p->growth.data(), p->growth.size() * sizeof(RuleGrowth), cudaMemcpyHostToDevice));
  }
  return CF_OK;
}

void cf_free_prog(cf_prog* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  for (void* a : p->search.allocs) cudaFree(a);
  for (auto& d : p->ordered) for (void* a : d.allocs) cudaFree(a);
  for (auto* e : p->d_ordered_E) cudaFree(e);
  for (auto* r : p->d_repl) cudaFree(r);
  for (auto& t : p->tmpl) { cudaFree(t.d_code); cudaFree(t.d_sets); cudaFree(t.d_parts); }
  cudaFree(p->d_E);
  cudaFree(p->d_always);
  cudaFree(p->d_rule_mask);
  cudaFree(p->d_growth);
  delete p;
}

uint32_t cf_prog_words(const cf_prog* p) { return p ? p->W : 0; }
uint32_t cf_prog_patterns(const cf_prog* p) { return p ? p->npat : 0; }

static uint64_t ntiles_for(uint64_t nbytes, uint32_t tile) { return (nbytes + 2 + tile - 1) / tile; }

// Freed batch handles are kept (up to BATCH_POOL of them) and handed out again, the last freed first: a batch created right after
// another was freed takes its address.  Whatever is keyed on a batch handle must therefore key on cf_batch::generation as well
// (cf_sub_host's copy of the offsets does).  The pool is never destroyed, so a handle freed during process exit still finds it.
static const size_t BATCH_POOL = 16;
static std::mutex& batch_pool_mu() { static std::mutex* m = new std::mutex; return *m; }
static std::vector<cf_batch*>& batch_pool() { static std::vector<cf_batch*>* v = new std::vector<cf_batch*>; return *v; }

static cf_batch* batch_alloc() {
  {
    std::lock_guard<std::mutex> g(batch_pool_mu());
    std::vector<cf_batch*>& pool = batch_pool();
    if (!pool.empty()) {
      cf_batch* b = pool.back();
      pool.pop_back();
      return new (b) cf_batch();
    }
  }
  return new (std::nothrow) cf_batch();
}

static void batch_release(cf_batch* b) {
  b->~cf_batch();
  {
    std::lock_guard<std::mutex> g(batch_pool_mu());
    std::vector<cf_batch*>& pool = batch_pool();
    if (pool.size() < BATCH_POOL) { pool.push_back(b); return; }
  }
  if (alignof(cf_batch) > __STDCPP_DEFAULT_NEW_ALIGNMENT__) ::operator delete(b, std::align_val_t(alignof(cf_batch)));
  else ::operator delete(b);
}

int cf_batch_create(cf_ctx* ctx, uint64_t max_stream_bytes, uint32_t max_units, cf_batch** out) {
  if (!ctx || !out) return CF_E_BADARG;
  CF_CUDA(ctx, cudaSetDevice(ctx->device));
  cf_batch* b = batch_alloc();
  if (!b) return CF_E_NOMEM;
  b->ctx = ctx;
  *out = b;
  b->cap_bytes = max_stream_bytes;
  b->cap_units = max_units;
  uint64_t total = cf::FRONT_PAD + (ntiles_for(max_stream_bytes, MAX_TILE) + 1) * (uint64_t)MAX_TILE;
  CF_CUDA(ctx, cudaMalloc(&b->d_buf, total));
  CF_CUDA(ctx, cudaMemset(b->d_buf, 0xFF, total));
  CF_CUDA(ctx, cudaMalloc(&b->d_offsets, ((uint64_t)max_units + 1) * 8));
  CF_CUDA(ctx, cudaMalloc(&b->d_coarse, ((max_stream_bytes >> cf::COARSE_SHIFT) + 2) * 4));
  // tensor map for the scan kernel's tile loads
  typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CF_CUDA(ctx, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) { ctx->err = "cuTensorMapEncodeTiled unavailable"; return CF_E_CUDA; }
  cuuint64_t gdim[2] = {128, total / 128};
  cuuint64_t gstride[1] = {128};
  cuuint32_t box[2] = {128, SCAN_BOX_ROWS};
  cuuint32_t estr[2] = {1, 1};
  CUresult cr = ((encode_fn)fn)(&b->tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, b->d_buf, gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) { ctx->err = "cuTensorMapEncodeTiled failed: " + std::to_string((int)cr); return CF_E_CUDA; }
  return CF_OK;
}

int cf_host_alloc(cf_ctx* ctx, uint64_t bytes, void** out) {
  if (!ctx || !out || !bytes) return CF_E_BADARG;
  *out = nullptr;
  CF_CUDA(ctx, cudaSetDevice(ctx->device));
  CF_CUDA(ctx, cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return CF_OK;
}
void cf_host_free(cf_ctx* ctx, void* p) {
  (void)ctx;
  if (p) cudaFreeHost(p);
}

void cf_batch_free(cf_batch* b) {
  if (!b) return;
  cudaSetDevice(b->ctx->device);
  cudaFree(b->d_buf);
  cudaFree(b->d_offsets);
  cudaFree(b->d_coarse);
  batch_release(b);
}

uint32_t cf_batch_units(const cf_batch* b) { return b ? b->n : 0; }
uint64_t cf_batch_bytes(const cf_batch* b) { return b ? b->nbytes : 0; }

// cf_batch::generation of a batch's new contents (cf_batch_upload, cf_batch_pack_device)
static uint64_t next_batch_generation() {
  static std::atomic<uint64_t> serial{0};
  return ++serial;
}

int cf_batch_upload(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes,
                    const uint64_t* offsets, uint32_t n_units, void* cuda_stream) {
  if (!ctx || !b || !stream || !offsets || !n_units) return CF_E_BADARG;
  if (stream_bytes > b->cap_bytes || n_units > b->cap_units) { ctx->err = "batch capacity exceeded"; return CF_E_CAPACITY; }
  if (offsets[0] != 0 || offsets[n_units] != stream_bytes) { ctx->err = "offsets[0] must be 0 and offsets[n] the stream length"; return CF_E_BADARG; }
  cudaStream_t st = (cudaStream_t)cuda_stream;
  uint8_t* d_stream = b->d_buf + cf::FRONT_PAD;
  // small transfers first (offsets and the coarse index usually come from pageable memory: staged copies that
  // would otherwise queue behind the big one), then the stream itself
  CF_CUDA(ctx, cudaMemcpyAsync(b->d_offsets, offsets, ((uint64_t)n_units + 1) * 8, cudaMemcpyHostToDevice, st));
  {  // coarse unit index (host sweep over offsets; tiny next to the stream copy)
    const uint64_t nc = (stream_bytes >> cf::COARSE_SHIFT) + 1;
    b->h_coarse.resize(nc);
    uint32_t u = 0;
    for (uint64_t k = 0; k < nc; ++k) {
      const uint64_t pos = k << cf::COARSE_SHIFT;
      while (u + 1 < n_units && offsets[u + 1] <= pos) ++u;
      b->h_coarse[k] = u;
    }
    CF_CUDA(ctx, cudaMemcpyAsync(b->d_coarse, b->h_coarse.data(), nc * 4, cudaMemcpyHostToDevice, st));
  }
  // re-arm the tail padding that a previous, longer upload may have overwritten
  const uint64_t end = (ntiles_for(b->nbytes > stream_bytes ? b->nbytes : stream_bytes, MAX_TILE) + 1) * (uint64_t)MAX_TILE;
  CF_CUDA(ctx, cudaMemsetAsync(d_stream + stream_bytes, 0xFF, end - stream_bytes, st));
  CF_CUDA(ctx, cudaMemcpyAsync(d_stream, stream, stream_bytes, cudaMemcpyHostToDevice, st));
  b->nbytes = stream_bytes;
  b->n = n_units;
  b->generation = next_batch_generation();
  return CF_OK;
}
}  // extern "C"

// cf_batch_pack_device: offsets[i] (i <= n) and coarse[k] (k < nc) of the packed batch, one thread per entry, from the source offsets
__global__ void __launch_bounds__(256) pack_index_kernel(const uint64_t* __restrict__ src_off, uint32_t n, uint64_t nbytes, uint64_t nc,
                                                         uint64_t* __restrict__ offsets, uint32_t* __restrict__ coarse) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t <= n) offsets[t] = cf::packed_offset(src_off, (uint32_t)t, nbytes);
  if (t < nc) coarse[t] = cf::packed_coarse(src_off, n, nbytes, t);
}

// ... and the stream: unit i's bytes and its terminator, one warp per unit.  Every write is clamped to stream[0, nbytes).
__global__ void __launch_bounds__(256) pack_copy_kernel(const uint8_t* __restrict__ src, const uint64_t* __restrict__ src_off, uint32_t n,
                                                        uint64_t nbytes, uint8_t* __restrict__ stream) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (u >= n) return;
  const uint64_t at = cf::packed_offset(src_off, u, nbytes);
  const uint64_t len = min(src_off[u + 1] - src_off[u], nbytes - at);
  warp_copy_span(stream, at, src + src_off[u], len, lane);
  if (lane == 0 && at + len < nbytes) stream[at + len] = cf::TERM;
}

extern "C" {
int cf_batch_pack_device(cf_ctx* ctx, cf_batch* b, const uint8_t* d_src, const uint64_t* d_src_offsets, uint32_t n_units, uint64_t src_bytes,
                         void* cuda_stream) {
  if (!ctx || !b || !d_src || !d_src_offsets || !n_units) return CF_E_BADARG;
  if (n_units > b->cap_units || src_bytes > b->cap_bytes || src_bytes + n_units > b->cap_bytes) { ctx->err = "batch capacity exceeded"; return CF_E_CAPACITY; }
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const uint64_t nbytes = src_bytes + n_units;
  const uint64_t nc = (nbytes >> cf::COARSE_SHIFT) + 1;
  uint8_t* d_stream = b->d_buf + cf::FRONT_PAD;
  // the tail padding, as cf_batch_upload re-arms it; the kernels write nothing at or past nbytes
  const uint64_t end = (ntiles_for(b->nbytes > nbytes ? b->nbytes : nbytes, MAX_TILE) + 1) * (uint64_t)MAX_TILE;
  CF_CUDA(ctx, cudaMemsetAsync(d_stream + nbytes, 0xFF, end - nbytes, st));
  const uint64_t idx_threads = nc > (uint64_t)n_units + 1 ? nc : (uint64_t)n_units + 1;
  pack_index_kernel<<<(unsigned)((idx_threads + 255) / 256), 256, 0, st>>>(d_src_offsets, n_units, nbytes, nc, b->d_offsets, b->d_coarse);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  pack_copy_kernel<<<(n_units + 7) / 8, 256, 0, st>>>(d_src, d_src_offsets, n_units, nbytes, d_stream);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  b->nbytes = nbytes;
  b->n = n_units;
  b->generation = next_batch_generation();
  return CF_OK;
}

int cf_scan(cf_ctx* ctx, cf_prog* p, cf_batch* b, uint64_t* d_bitmaps, void* cuda_stream) {
  if (!ctx || !p || !b || !d_bitmaps || !b->n) return CF_E_BADARG;
  return cf_scan_launch(ctx, p, b, d_bitmaps, (cudaStream_t)cuda_stream, ctx->d_queue, ctx->d_qstate, &ctx->qphase);
}
}  // extern "C"

int cf_scan_launch(cf_ctx* ctx, cf_prog* p, cf_batch* b, uint64_t* d_bitmaps, cudaStream_t st, uint64_t* queue, uint64_t* qstate, uint32_t* qphase) {
  const uint64_t ntiles = ntiles_for(b->nbytes, SCAN_TILE);
  const uint64_t total = (uint64_t)b->n * p->W;
  if (p->any_always) {
    fill_bitmaps_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_bitmaps, p->d_always, p->W, total);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
  } else {
    CF_CUDA(ctx, cudaMemsetAsync(d_bitmaps, 0, total * 8, st));
  }
  if (p->search_empty) return CF_OK;
  ScanParams P;
  P.stream = b->d_buf + cf::FRONT_PAD;
  P.nbytes = b->nbytes;
  P.ntiles = ntiles;
  P.offsets = b->d_offsets;
  P.coarse = b->d_coarse;
  P.n_units = b->n;
  P.E = p->d_E;
  P.dfa = p->search.t;
  P.bitmaps = (unsigned long long*)d_bitmaps;
  P.queue = (unsigned long long*)queue;
  P.qstate = (unsigned long long*)qstate + 2 * *qphase;
  P.qstate_next = (unsigned long long*)qstate + 2 * (*qphase ^ 1);
  *qphase ^= 1;
  P.qcap_cta = ctx->qcap / (uint32_t)ctx->sm_count;
  P.dfa_bytes = p->search.stage_bytes < (1u << 30) ? (uint32_t)p->search.stage_bytes : 0;
  P.dfa_trans_bytes = (uint32_t)p->search.trans_bytes;
  P.dfa_acc_bytes = (uint32_t)p->search.acc_bytes;
  P.mulc = p->use_pairs ? 256 : 1024;
  const auto fn = p->use_pairs ? scan_kernel<1> : scan_kernel<0>;
  uint64_t grid = (uint64_t)ctx->sm_count;   // persistent: one CTA per SM
  if (ctx->scan_reserve_sms && ctx->scan_reserve_sms < grid) grid -= ctx->scan_reserve_sms;
  if (grid > ntiles) grid = ntiles;
  const bool prof = ctx->prof_on && (size_t)ctx->prof_used + 2 <= ctx->prof_ev.size();
  if (prof) cudaEventRecord(ctx->prof_ev[ctx->prof_used], st);
  fn<<<(unsigned)grid, SCAN_WARPS * 32, SCAN_SMEM, st>>>(P, b->tmap);
  if (prof) { cudaEventRecord(ctx->prof_ev[ctx->prof_used + 1], st); ctx->prof_used += 2; }
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  return CF_OK;
}

extern "C" {
int cf_scan_host(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes,
                 const uint64_t* offsets, uint32_t n_units, uint64_t* h_bitmaps) {
  if (!h_bitmaps) return CF_E_BADARG;
  int rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
  if (rc) return rc;
  const size_t bytes = (size_t)n_units * p->W * 8;
  if ((rc = cf_dev_reserve(ctx, ctx->bitmaps, bytes))) return rc;
  uint64_t* d_bm = (uint64_t*)ctx->bitmaps.p;
  if ((rc = cf_scan(ctx, p, b, d_bm, nullptr))) return rc;
  CF_CUDA(ctx, cudaMemcpyAsync(h_bitmaps, d_bm, bytes, cudaMemcpyDeviceToHost, 0));
  CF_CUDA(ctx, cudaStreamSynchronize(0));
  return CF_OK;
}

int cf_sub_host(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint32_t* units, uint32_t n_sel, uint8_t* out_bytes,
                uint64_t out_cap, uint64_t* out_offsets, uint64_t* out_needed) {
  if (!ctx || !p || !b || !units || !n_sel || !out_offsets) return CF_E_BADARG;
  if (p->ordered.empty()) { ctx->err = "program has no substitution rules"; return CF_E_BADARG; }
  if (p->h_offsets_owner != b || p->h_offsets_gen != b->generation || p->h_offsets.size() != (size_t)b->n + 1) {
    // unit lengths are needed on the host to size the scratch area
    p->h_offsets.resize((size_t)b->n + 1);
    CF_CUDA(ctx, cudaMemcpy(p->h_offsets.data(), b->d_offsets, ((size_t)b->n + 1) * 8, cudaMemcpyDeviceToHost));
    p->h_offsets_owner = b;
    p->h_offsets_gen = b->generation;
  }
  int rc;
  if ((rc = cf_stage_reserve(ctx, cf_sub_stage_bytes(n_sel)))) return rc;
  const uint64_t* rec = nullptr;
  if ((rc = cf_sub_device(ctx, p, b, p->h_offsets.data(), units, n_sel, 0, (uint8_t*)ctx->h_stage, &rec))) return rc;
  uint64_t need = 0;
  for (uint32_t i = 0; i < n_sel; ++i) { out_offsets[i] = need; need += rec[2 * (size_t)i + 1]; }
  out_offsets[n_sel] = need;
  if (out_needed) *out_needed = need;
  if (need > out_cap || (!out_bytes && need)) { ctx->err = "output buffer too small"; return CF_E_CAPACITY; }
  if (need) {
    if ((rc = cf_dev_reserve(ctx, ctx->sub_out_offsets, ((size_t)n_sel + 1) * 8)) || (rc = cf_dev_reserve(ctx, ctx->sub_out, need))) return rc;
    uint64_t* d_ooff = (uint64_t*)ctx->sub_out_offsets.p;
    uint8_t* d_out = (uint8_t*)ctx->sub_out.p;
    CF_CUDA(ctx, cudaMemcpy(d_ooff, out_offsets, ((size_t)n_sel + 1) * 8, cudaMemcpyHostToDevice));
    sub_compact_kernel<<<n_sel, 256>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, sub_desc_sel(ctx, n_sel), (const uint8_t*)ctx->sub_scratch.p,
                                       (const uint64_t*)ctx->sub_rec.p, d_ooff, d_out, n_sel);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    CF_CUDA(ctx, cudaMemcpy(out_bytes, d_out, need, cudaMemcpyDeviceToHost));
  }
  return CF_OK;
}

int cf_profile_begin(cf_ctx* ctx, uint32_t max_launches) {
  if (!ctx) return CF_E_BADARG;
  for (auto e : ctx->prof_ev) cudaEventDestroy(e);
  ctx->prof_ev.clear();
  ctx->prof_used = 0;
  ctx->prof_on = max_launches > 0;
  for (uint32_t i = 0; i < 2 * max_launches; ++i) {
    cudaEvent_t e;
    CF_CUDA(ctx, cudaEventCreate(&e));
    ctx->prof_ev.push_back(e);
  }
  return CF_OK;
}

int cf_profile_collect(cf_ctx* ctx, double* total_ms, uint32_t* n_launches) {
  if (!ctx || !total_ms || !n_launches) return CF_E_BADARG;
  double tot = 0;
  uint32_t n = 0;
  for (uint32_t i = 0; i + 1 < ctx->prof_used; i += 2) {
    CF_CUDA(ctx, cudaEventSynchronize(ctx->prof_ev[i + 1]));
    float ms = 0;
    CF_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->prof_ev[i], ctx->prof_ev[i + 1]));
    tot += ms;
    ++n;
  }
  *total_ms = tot;
  *n_launches = n;
  ctx->prof_used = 0;
  return CF_OK;
}

int cf_scan_counters(cf_ctx* ctx, uint64_t out[2]) {
  if (!ctx || !out) return CF_E_BADARG;
  CF_CUDA(ctx, cudaMemcpy(out, ctx->d_qstate + 2 * (ctx->qphase ^ 1), 16, cudaMemcpyDeviceToHost));  // pair used by the last scan
  return CF_OK;
}

}  // extern "C"
