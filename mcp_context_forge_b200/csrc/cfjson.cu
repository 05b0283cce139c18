// cfjson.cu — the JSON kernels of libcfgpu.so and their C-ABI entry points (include/cfgpu.h): structural index
// (json_index.h), toon_encoder (token-parallel json_tp.h + sequential json_toon.h for the units it hands over),
// request_logging_masking (json_mask.h).  Split from cfgpu.cu so that either half rebuilds on its own.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <nvtx3/nvToolsExt.h>

#include "cf_internal.h"
#include "json_index.h"
#include "json_mask.h"
#include "json_toon.h"
#include "json_tp.h"

// ------------------------------------------------------------------------------------------------
// JSON structural index (SURVEY.md §8(f)-2; csrc/json_index.h), one WARP per unit:
//   stage 1   one ballot per byte class and 32 bytes (bytes prefetched eight chunks ahead): escape parity,
//             in-string mask by prefix XOR, structural characters, scalar starts -> token positions
//   stage 1b  (CF_INDEX_CLASSIFY) lane-parallel over the tokens: strings validated + their predicates/hash,
//             scalars validated — the same functions the sequential parser uses
// Measured as a front end of the TOON / masking kernels (index kernel + token-driven DOM build per lane)
// it loses to the sequential per-lane parser at large batches (stage 1b is issue-bound at ~12 warp-instructions
// per byte and the tokens triple the memory traffic), so
// those kernels keep json_parse; the index stands alone as a reusable op (string extraction, length
// guards) and as the first stage of the token-parallel design the next round needs (DESIGN.md §7).
// ------------------------------------------------------------------------------------------------
static const uint32_t IDX_AHEAD = 8;     // chunks of 32 bytes in flight per warp
__device__ __forceinline__ uint32_t warp_index(const uint8_t* __restrict__ s, uint32_t n, cfx::Tok* __restrict__ tk, bool* unterminated,
                                               uint32_t lane, const uint8_t* __restrict__ cls) {
  cfx::IndexCarry cy;
  cy.init();
  uint32_t nt = 0;
  const uint32_t below = (1u << lane) - 1u;
  for (uint32_t base0 = 0; base0 < n; base0 += 32 * IDX_AHEAD) {
    uint32_t cs[IDX_AHEAD];
#pragma unroll
    for (uint32_t k = 0; k < IDX_AHEAD; ++k) {
      const uint32_t p = base0 + 32 * k + lane;
      cs[k] = p < n ? (uint32_t)s[p] : (uint32_t)' ';
    }
#pragma unroll
    for (uint32_t k = 0; k < IDX_AHEAD; ++k) {
      const uint32_t base = base0 + 32 * k;
      if (base >= n) break;
      const uint32_t kc = cls[cs[k]];            // byte class from a 256-byte shared table: 1 LDS instead of ~14 compares
      const uint32_t bs = __ballot_sync(0xFFFFFFFFu, (kc & 1u) != 0);
      const uint32_t qm = __ballot_sync(0xFFFFFFFFu, (kc & 2u) != 0);
      const uint32_t st = __ballot_sync(0xFFFFFFFFu, (kc & 4u) != 0);
      const uint32_t ws = __ballot_sync(0xFFFFFFFFu, (kc & 8u) != 0);
      uint32_t esc = 0;
      if (bs | cy.bs_parity) {
        esc = __ballot_sync(0xFFFFFFFFu, cfx::escaped_bit(bs, lane, cy.bs_parity) != 0);
        cy.bs_parity = cfx::next_bs_parity(bs, cy.bs_parity);
      }
      uint32_t close;
      const uint32_t tm = cfx::index_chunk(qm & ~esc, st, ws, cy, &close);
      if ((tm >> lane) & 1u) {
        cfx::Tok t;
        t.pos = (base + lane) | (((close >> lane) & 1u) ? cfx::T_CLOSE : 0u);
        t.aux = 0;
        tk[nt + __popc(tm & below)] = t;
      }
      nt += __popc(tm);
    }
  }
  *unterminated = cy.in_string != 0;
  return nt;
}

static const uint32_t NTOK_UNTERMINATED = 0x80000000u;
// tokens of unit u at toks + offsets[u] (capacity len + 1: offsets count one terminator per unit); ntok[u] = count | flag
__global__ void __launch_bounds__(128) json_index_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets, uint32_t n_units,
                                                          cfx::Tok* __restrict__ toks, uint32_t* __restrict__ ntok, uint64_t max_len,
                                                          uint32_t flags) {
  __shared__ uint8_t cls[256];       // bit 0 backslash, 1 quote, 2 structural, 3 JSON whitespace
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x)
    cls[i] = (uint8_t)((i == '\\' ? 1u : 0u) | (i == '"' ? 2u : 0u) | (cfx::is_structural(i) ? 4u : 0u) | (cfj::j_ws(i) ? 8u : 0u));
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= n_units) return;
  const uint64_t b = offsets[u];
  const uint64_t len64 = offsets[u + 1] - b - 1;
  if (len64 > max_len) { if (lane == 0) ntok[u] = 0; return; }
  const uint32_t len = (uint32_t)len64;
  cfx::Tok* tk = toks + b;
  bool unt;
  const uint32_t nt = warp_index(stream + b, len, tk, &unt, lane, cls);
  __syncwarp();
  if (flags & CF_INDEX_CLASSIFY)
    for (uint32_t t = lane; t < nt; t += 32) tk[t].aux = cfx::classify_token(stream + b, len, tk[t].pos);
  if (lane == 0) ntok[u] = nt | (unt ? NTOK_UNTERMINATED : 0u);
}

// ------------------------------------------------------------------------------------------------
// toon_encoder, token-parallel (csrc/json_tp.h): one WARP per unit, two passes over the unit's bytes (the second
// one comes from L2), 8-byte tokens through HBM scratch, no DOM.  Units the fast path does not cover get status
// TS_FALLBACK (reason in out_len) and are re-done by the sequential toon_kernel below (TOON_ONLY_FALLBACK).  A unit that stops
// at a mixed list-item array (FB_MIXED_ITEM) is decided by the same warp right away: analyze in resolve mode and emit again over
// the token array it already has (json_tp.h toon_unit).  Resolve mode costs key comparisons the first attempt saves on every
// other unit, and a warp is far quicker than the sequential encoder's one thread per unit.
// The kernel takes its units in cost order (toon_order_kernel + a stable radix sort, heaviest first): a CTA holds its slot
// until its slowest warp is done, and a nested unit costs about three tabular ones, so CTAs that mix shapes idle most of their
// warps.  In cost order each CTA, and at any moment each SM, runs units of one kind.  The sequential encoder keeps the natural
// order: its few units are then spread over many SMs instead of packed into a few CTAs.
// ------------------------------------------------------------------------------------------------
static const uint32_t TP_WARPS = 8;
static const uint32_t TP_TOK_SLACK = 64;               // token capacity of unit u: len/2 + TP_TOK_SLACK
static const uint32_t TP_WARP_SMEM = (uint32_t)sizeof(cftp::Shared) + cftp::STAGE;   // container stack + token ring | staging buffer
// Three CTAs (24 warps) per SM: the kernel is latency-bound (a warp works through its unit in serial, dependent steps), so
// resident warps are what hides the latency.  That needs <= 80 registers per thread and <= 75 KB of shared memory per CTA
// (3 x (75 904 + 1 024 reserved) B of the SM's 228 KB); tests/test_toon_occupancy_cpu.py holds both.
static const uint32_t TP_CTAS_PER_SM = 3;
static const uint32_t TP_SMEM = TP_WARPS * TP_WARP_SMEM;                              // 75 904 B
static_assert(TP_CTAS_PER_SM * (TP_SMEM + 1024) <= 228 * 1024, "TP_CTAS_PER_SM CTAs fit the SM's shared memory");
__global__ void __launch_bounds__(TP_WARPS * 32, TP_CTAS_PER_SM) toon_tp_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets, uint32_t n_units,
                                                                    cftp::GTok* __restrict__ toks, uint8_t* __restrict__ out, uint32_t* __restrict__ out_len,
                                                                    int32_t* __restrict__ status, uint32_t flags, const uint8_t* __restrict__ unit_stages,
                                                                    const uint32_t* __restrict__ order) {
  extern __shared__ __align__(16) uint8_t tp_smem[];
  const uint32_t lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
  const uint32_t slot = blockIdx.x * TP_WARPS + wic;
  if (slot >= n_units) return;
  const uint32_t u = order[slot];
  if (unit_stages && !(unit_stages[u] & CF_STAGE_TOON)) { if (lane == 0) { status[u] = CF_TOON_SKIPPED; out_len[u] = 0; } return; }
  cftp::Shared& sh = *reinterpret_cast<cftp::Shared*>(tp_smem + (size_t)wic * TP_WARP_SMEM);
  uint8_t* stage = tp_smem + (size_t)wic * TP_WARP_SMEM + sizeof(cftp::Shared);
  if (lane == 0) {                                   // the warp's mbarrier for its bulk TMA loads into the staging buffer
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&sh.sbar_bar)));
    sh.sbar_phase = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const uint64_t b = offsets[u];
  const uint64_t len64 = offsets[u + 1] - b - 1;
  if (len64 > 0x7FFFFFFFull) { if (lane == 0) { status[u] = cfj::TS_UNSUPPORTED; out_len[u] = 0; } return; }
  const uint32_t len = (uint32_t)len64;
  cftp::GTok* my = toks + (b >> 1) + (uint64_t)TP_TOK_SLACK * u;
  uint32_t ol = 0;
  // CF_TOON_NO_HANDOVER: the first attempt only, so that a mixed list-item array still reports FB_MIXED_ITEM
  const int st = cftp::toon_unit(stream + b, len, my, len / 2 + TP_TOK_SLACK, out + b, len ? len - 1 : 0, &ol, sh, stage, (flags & 1u) != 0,
                                 !(flags & CF_TOON_NO_HANDOVER));
  if (lane == 0) {
    status[u] = st & 0xFF;
    out_len[u] = (st & 0xFF) == cfj::TS_CONVERTED ? ol : (uint32_t)st >> 8;
  }
}

// cost key of each unit for the first pass's order (json_tp.h order_events over the unit's first ORDER_WINDOW bytes, clamped to
// 8 bits; 0 for units that do not take TOON, empty and oversized ones), one warp per unit with 16-byte loads; idx[u] = u.
// The loads are rounded out to the 16-byte grid: the batch buffer's front and tail padding keep them inside it, and the bytes
// outside the window are zeroed.
__global__ void __launch_bounds__(256) toon_order_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets, uint32_t n_units,
                                                         const uint8_t* __restrict__ unit_stages, uint8_t* __restrict__ key, uint32_t* __restrict__ idx) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= n_units) return;
  const uint64_t b = offsets[u];
  const uint64_t len = offsets[u + 1] - b - 1;
  uint32_t ev = 0;
  if (len && len <= 0x7FFFFFFFull && !(unit_stages && !(unit_stages[u] & CF_STAGE_TOON))) {
    const uint32_t win = len < cftp::ORDER_WINDOW ? (uint32_t)len : cftp::ORDER_WINDOW;
    const uint32_t lead = (uint32_t)((uintptr_t)(stream + b) & 15u);
    const uint4* g = reinterpret_cast<const uint4*>(stream + b - lead);
    const uint32_t nchunks = (lead + win + 15) >> 4;
    uint32_t carry = 0;                                    // the last word of the previous round's lane 31
    for (uint32_t c0 = 0; c0 < nchunks; c0 += 32) {
      const uint32_t c = c0 + lane;
      uint32_t w[4] = {0, 0, 0, 0};
      if (c < nchunks) {
        const uint4 v = g[c];
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
        const int32_t p0 = (int32_t)(16 * c) - (int32_t)lead;   // unit position of the chunk's byte 0
        if (p0 < 0 || p0 + 16 > (int32_t)win) {
#pragma unroll
          for (uint32_t k = 0; k < 16; ++k) {
            const int32_t p = p0 + (int32_t)k;
            if (p < 0 || p >= (int32_t)win) w[k >> 2] &= ~(0xFFu << (8 * (k & 3)));
          }
        }
      }
      uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, w[3], 1);
      if (lane == 0) prev = carry;
      carry = __shfl_sync(0xFFFFFFFFu, w[3], 31);
      ev += cftp::order_events(prev, w[0]) + cftp::order_events(w[0], w[1]) + cftp::order_events(w[1], w[2]) + cftp::order_events(w[2], w[3]);
    }
    ev = __reduce_add_sync(0xFFFFFFFFu, ev);
  }
  if (lane == 0) {
    key[u] = (uint8_t)(ev < 255u ? ev : 255u);
    idx[u] = u;
  }
}

// gather per-unit results (unit u at src + mul*offsets[u] + add*u, out_len[u] bytes) into one contiguous buffer
__global__ void compact_kernel(const uint8_t* __restrict__ src, uint32_t mul, uint32_t add, const uint64_t* __restrict__ offsets,
                               const uint32_t* __restrict__ out_len, const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out,
                               uint32_t n_units) {
  const uint32_t u = blockIdx.x;
  if (u >= n_units) return;
  const uint8_t* s = src + (uint64_t)mul * offsets[u] + (uint64_t)add * u;
  uint8_t* dst = out + out_off[u];
  for (uint32_t i = threadIdx.x; i < out_len[u]; i += blockDim.x) dst[i] = s[i];
}



int cf_dev_reserve(cf_ctx* ctx, cf_ctx::DevBuf& b, size_t need) {
  if (need <= b.cap) return CF_OK;
  cudaFree(b.p);
  b.p = nullptr; b.cap = 0;
  const size_t c = need + need / 4 + 256;
  CF_CUDA(ctx, cudaMalloc(&b.p, c));
  b.cap = c;
  return CF_OK;
}
int cf_stage_reserve(cf_ctx* ctx, size_t need) {
  if (need <= ctx->h_stage_bytes) return CF_OK;
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  ctx->h_stage = nullptr; ctx->h_stage_bytes = 0;
  const size_t c = need + need / 4 + 4096;
  CF_CUDA(ctx, cudaHostAlloc(&ctx->h_stage, c, cudaHostAllocDefault));
  ctx->h_stage_bytes = c;
  return CF_OK;
}
// units per warp for the thread-per-unit JSON kernels: fill the GPU with warps first (about 12 resident
// warps per SM at their register footprint), only then put several units into one warp
static uint32_t units_per_warp(const cf_ctx* ctx, uint32_t n) {
  const uint32_t warps = (uint32_t)ctx->sm_count * 12u;
  uint32_t u = 1;
  while (u < 32 && (n + u - 1) / u > warps) u <<= 1;
  return u;
}
static uint32_t json_blocks(uint32_t n, uint32_t upw) { return ((n + upw - 1) / upw + 1) / 2; }   // two warps per block
extern "C" {
int cf_json_index(cf_ctx* ctx, cf_batch* b, uint32_t flags, cf_json_token* d_tokens, uint32_t* d_counts, void* cuda_stream) {
  if (!ctx || !b || !d_tokens || !d_counts) return CF_E_BADARG;
  if (b->n == 0) return CF_OK;
  static_assert(sizeof(cf_json_token) == sizeof(cfx::Tok), "token layout");
  json_index_kernel<<<(b->n + 3) / 4, 128, 0, (cudaStream_t)cuda_stream>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cfx::Tok*)d_tokens, d_counts,
                                                                            0x7FFFFFFFull, flags);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  return CF_OK;
}

int cf_json_index_host(cf_ctx* ctx, cf_batch* b, uint32_t flags, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets,
                       uint32_t n_units, cf_json_token* tokens, uint32_t* counts) {
  if (!ctx || !b || !tokens || !counts) return CF_E_BADARG;
  int rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
  if (rc) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->d_tok, (size_t)(stream_bytes + 64) * sizeof(cfx::Tok)))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->d_ntok, (size_t)(n_units + 1) * 4))) return rc;
  if ((rc = cf_json_index(ctx, b, flags, (cf_json_token*)ctx->d_tok.p, (uint32_t*)ctx->d_ntok.p, nullptr))) return rc;
  CF_CUDA(ctx, cudaMemcpy(counts, ctx->d_ntok.p, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  CF_CUDA(ctx, cudaMemcpy(tokens, ctx->d_tok.p, (size_t)stream_bytes * sizeof(cfx::Tok), cudaMemcpyDeviceToHost));
  return CF_OK;
}

// TOON device workspace: token / DOM scratch, and the first pass's unit order with the sort behind it (indices | keys in | keys out |
// radix-sort temp storage).  The context's for cf_toon and cf_run_batch, a run's own for cf_run_enqueue.
struct ToonWs {
  void* scratch;
  uint64_t scratch_bytes;
  uint32_t* order;
  uint8_t* sort;
  size_t sort_bytes;
};
static uint64_t toon_scratch_need(uint64_t nbytes, uint32_t n) {
  const uint64_t need = (nbytes / 2 + 4ull * n + 8) * sizeof(cfj::JNode);
  const uint64_t need_tp = (nbytes / 2 + (uint64_t)TP_TOK_SLACK * n + 8) * sizeof(cftp::GTok);
  return need_tp > need ? need_tp : need;
}
static size_t toon_sort_tmp_offset(uint32_t n) { return ((size_t)n * 4 + 2 * (size_t)n + 255) & ~(size_t)255; }
static int toon_sort_temp(cf_ctx* ctx, uint32_t n, cudaStream_t st, size_t* bytes) {
  CF_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(nullptr, *bytes, (const uint8_t*)nullptr, (uint8_t*)nullptr, (const uint32_t*)nullptr,
                                                         (uint32_t*)nullptr, (int)n, 0, 8, st));
  return CF_OK;
}
static int toon_tp_prepare(cf_ctx* ctx) {
  static bool smem_set = false;
  if (!smem_set) {
    CF_CUDA(ctx, cudaFuncSetAttribute(toon_tp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TP_SMEM));
    smem_set = true;
  }
  return CF_OK;
}

// does `ws` hold the TOON stage of batch b (token-parallel path)?  Host-only, no launch.
static int toon_ws_check(cf_ctx* ctx, const cf_batch* b, const ToonWs& ws, cudaStream_t st) {
  size_t sort_tmp = 0;
  int rc;
  if ((rc = toon_sort_temp(ctx, b->n, st, &sort_tmp))) return rc;
  if (toon_scratch_need(b->nbytes, b->n) > ws.scratch_bytes || toon_sort_tmp_offset(b->n) + sort_tmp > ws.sort_bytes) { ctx->err = "TOON workspace too small"; return CF_E_CAPACITY; }
  return CF_OK;
}

// the TOON launches on `st` with a workspace that is already large enough (no allocation, no synchronisation)
static int toon_enqueue(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, const uint8_t* d_unit_stages,
                        cudaStream_t st, const ToonWs& ws) {
  const bool tp = !(flags & (CF_TOON_PARSE_ONLY | CF_TOON_SEQUENTIAL));
  if (!tp && d_unit_stages) { ctx->err = "per-unit stage masks need the token-parallel encoder"; return CF_E_BADARG; }
  // the first pass's unit order: key + stable radix sort over its 8 bits, descending
  const size_t o_kin = (size_t)b->n * 4, o_kout = o_kin + b->n, o_tmp = toon_sort_tmp_offset(b->n);
  size_t sort_tmp = 0;
  int rc;
  if (tp && (rc = toon_sort_temp(ctx, b->n, st, &sort_tmp))) return rc;
  if (toon_scratch_need(b->nbytes, b->n) > ws.scratch_bytes || (tp && o_tmp + sort_tmp > ws.sort_bytes)) { ctx->err = "TOON workspace too small"; return CF_E_CAPACITY; }
  const bool prof = ctx->prof_on && (size_t)ctx->prof_used + 2 <= ctx->prof_ev.size();
  if (prof) cudaEventRecord(ctx->prof_ev[ctx->prof_used], st);
  if (tp) {
    if ((rc = toon_tp_prepare(ctx))) return rc;
    uint8_t* srt = ws.sort;
    toon_order_kernel<<<(b->n + 7) / 8, 256, 0, st>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, d_unit_stages, srt + o_kin, (uint32_t*)srt);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    CF_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(srt + o_tmp, sort_tmp, srt + o_kin, srt + o_kout, (const uint32_t*)srt, ws.order, (int)b->n, 0, 8, st));
    ctx->launches++;
    const uint32_t grid = (b->n + TP_WARPS - 1) / TP_WARPS;
    toon_tp_kernel<<<grid, TP_WARPS * 32, TP_SMEM, st>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cftp::GTok*)ws.scratch, d_out, d_out_len,
                                                         d_status, flags, d_unit_stages, ws.order);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    // the units the fast path handed over: sequential encoder, one unit per warp (they are few)
    if (!(flags & CF_TOON_NO_HANDOVER)) cf_launch_toon_seq(json_blocks(b->n, 1), st, b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cfj::JNode*)ws.scratch, d_out, d_out_len, d_status,
                                                     (flags & 1u) | TOON_ONLY_FALLBACK, 1);
  } else {
    const uint32_t upw = units_per_warp(ctx, b->n);
    cf_launch_toon_seq(json_blocks(b->n, upw), st, b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cfj::JNode*)ws.scratch, d_out, d_out_len,
                                                       d_status, flags & ~TOON_ONLY_FALLBACK, upw);
  }
  if (prof) { cudaEventRecord(ctx->prof_ev[ctx->prof_used + 1], st); ctx->prof_used += 2; }
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  return CF_OK;
}

// the context's TOON workspace (cf_toon, cf_run_batch), grown on demand
static int toon_ctx_ws(cf_ctx* ctx, const cf_batch* b, uint32_t flags, cudaStream_t st, ToonWs* ws) {
  const uint64_t need = toon_scratch_need(b->nbytes, b->n);
  if (need > ctx->toon_scratch_bytes) {
    CF_CUDA(ctx, cudaStreamSynchronize(st));
    cudaFree(ctx->d_toon_scratch);
    ctx->d_toon_scratch = nullptr;
    ctx->toon_scratch_bytes = 0;
    CF_CUDA(ctx, cudaMalloc(&ctx->d_toon_scratch, need + need / 4));
    ctx->toon_scratch_bytes = need + need / 4;
  }
  if (!(flags & (CF_TOON_PARSE_ONLY | CF_TOON_SEQUENTIAL))) {
    size_t sort_tmp = 0;
    int rc;
    if ((rc = toon_sort_temp(ctx, b->n, st, &sort_tmp))) return rc;
    if ((rc = cf_dev_reserve(ctx, ctx->toon_order, (size_t)b->n * 4))) return rc;
    if ((rc = cf_dev_reserve(ctx, ctx->toon_sort, toon_sort_tmp_offset(b->n) + sort_tmp))) return rc;
  }
  *ws = ToonWs{ctx->d_toon_scratch, ctx->toon_scratch_bytes, (uint32_t*)ctx->toon_order.p, (uint8_t*)ctx->toon_sort.p, ctx->toon_sort.cap};
  return CF_OK;
}
static int toon_launch(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, const uint8_t* d_unit_stages,
                       cudaStream_t st) {
  ToonWs ws;
  const int rc = toon_ctx_ws(ctx, b, flags, st, &ws);
  return rc ? rc : toon_enqueue(ctx, b, flags, d_out, d_out_len, d_status, d_unit_stages, st, ws);
}

int cf_toon(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, void* cuda_stream) {
  if (!ctx || !b || !b->n || !d_out || !d_out_len || !d_status) return CF_E_BADARG;
  return toon_launch(ctx, b, flags, d_out, d_out_len, d_status, nullptr, (cudaStream_t)cuda_stream);
}

#ifdef CF_TOON_PHASES
// Phase-timing builds only (json_tp.h TP_PHASE): out[k] = the cycles all warps spent in phase k since the last call, which clears them.
int cf_toon_phase_cycles(unsigned long long* out) {
  const size_t n = (size_t)cftp::PH_WARPS * (cftp::PH_N + 1);
  unsigned long long* h = (unsigned long long*)calloc(n, sizeof(unsigned long long));
  if (!h) return CF_E_NOMEM;
  cudaError_t e = cudaMemcpyFromSymbol(h, cftp::toon_phase_cycles, n * sizeof(unsigned long long));
  for (uint32_t k = 0; k < cftp::PH_N; ++k) out[k] = 0;
  for (size_t w = 0; w < cftp::PH_WARPS; ++w)
    for (uint32_t k = 0; k < cftp::PH_N; ++k) out[k] += h[w * (cftp::PH_N + 1) + k];
  memset(h, 0, n * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(cftp::toon_phase_cycles, h, n * sizeof(unsigned long long));
  free(h);
  return e == cudaSuccess ? CF_OK : CF_E_CUDA;
}
#endif

// Not part of the C API (include/cfgpu.h): the token-parallel kernel's launch shape for tests/test_toon_occupancy_cpu.py, which
// checks it against the built kernel's resource usage without a device.
void cf_toon_tp_config(uint32_t* warps_per_cta, uint32_t* ctas_per_sm, uint32_t* smem_per_cta) {
  if (warps_per_cta) *warps_per_cta = TP_WARPS;
  if (ctas_per_sm) *ctas_per_sm = TP_CTAS_PER_SM;
  if (smem_per_cta) *smem_per_cta = TP_SMEM;
}

int cf_toon_host(cf_ctx* ctx, cf_batch* b, uint32_t flags, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets,
                 uint32_t n_units, uint8_t* out_stream, uint32_t* out_len, int32_t* status) {
  if (!out_stream || !out_len || !status) return CF_E_BADARG;
  int rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
  if (rc) return rc;
  // device: encode in the input's layout, then gather the converted texts so that only they cross PCIe
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[0], stream_bytes + 16))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[1], (size_t)n_units * 4))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[2], (size_t)n_units * 4))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[3], ((size_t)n_units + 1) * 8))) return rc;
  uint8_t* d_out = (uint8_t*)ctx->tmp[0].p;
  uint32_t* d_len = (uint32_t*)ctx->tmp[1].p;
  int32_t* d_st = (int32_t*)ctx->tmp[2].p;
  uint64_t* d_ooff = (uint64_t*)ctx->tmp[3].p;
  rc = cf_toon(ctx, b, flags, d_out, d_len, d_st, nullptr);
  if (rc) return rc;
  CF_CUDA(ctx, cudaMemcpy(out_len, d_len, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  CF_CUDA(ctx, cudaMemcpy(status, d_st, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  if (flags & CF_TOON_PARSE_ONLY) return CF_OK;
  std::vector<uint64_t> ooff((size_t)n_units + 1);
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_units; ++i) { ooff[i] = total; total += out_len[i]; }
  ooff[n_units] = total;
  if (!total) return CF_OK;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[4], total))) return rc;
  if ((rc = cf_stage_reserve(ctx, total))) return rc;
  CF_CUDA(ctx, cudaMemcpy(d_ooff, ooff.data(), ((size_t)n_units + 1) * 8, cudaMemcpyHostToDevice));
  compact_kernel<<<n_units, 128>>>(d_out, 1, 0, b->d_offsets, d_len, d_ooff, (uint8_t*)ctx->tmp[4].p, n_units);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  CF_CUDA(ctx, cudaMemcpy(ctx->h_stage, ctx->tmp[4].p, total, cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < n_units; ++i)
    if (out_len[i]) memcpy(out_stream + offsets[i], (const uint8_t*)ctx->h_stage + ooff[i], out_len[i]);
  return CF_OK;
}

static int cf_mask_resident(cf_ctx* ctx, cf_batch* b, int max_depth, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, int32_t* status,
                            uint64_t* out_needed);
int cf_mask_host(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets, uint32_t n_units,
                 int max_depth, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, int32_t* status, uint64_t* out_needed) {
  if (!ctx || !b || !out_offsets || !status) return CF_E_BADARG;
  int rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
  if (rc) return rc;
  return cf_mask_resident(ctx, b, max_depth, out_bytes, out_cap, out_offsets, status, out_needed);
}
// masking of the batch already uploaded
static int cf_mask_resident(cf_ctx* ctx, cf_batch* b, int max_depth, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, int32_t* status,
                            uint64_t* out_needed) {
  int rc;
  const uint64_t stream_bytes = b->nbytes;
  const uint32_t n_units = b->n;
  const uint64_t nnodes = stream_bytes / 2 + 4ull * n_units + 8;
  const uint64_t need = nnodes * sizeof(cfj::JNode);
  if (need > ctx->toon_scratch_bytes) {
    cudaFree(ctx->d_toon_scratch);
    ctx->d_toon_scratch = nullptr;
    ctx->toon_scratch_bytes = 0;
    CF_CUDA(ctx, cudaMalloc(&ctx->d_toon_scratch, need + need / 4));
    ctx->toon_scratch_bytes = need + need / 4;
  }
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[0], 5 * stream_bytes + 32ull * n_units + 64))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[1], (size_t)n_units * 4))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[2], (size_t)n_units * 4))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[3], ((size_t)n_units + 1) * 8))) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[5], nnodes * 4))) return rc;
  uint8_t* d_arena = (uint8_t*)ctx->tmp[0].p;
  uint32_t* d_len = (uint32_t*)ctx->tmp[1].p;
  int32_t* d_st = (int32_t*)ctx->tmp[2].p;
  uint64_t* d_ooff = (uint64_t*)ctx->tmp[3].p;
  uint32_t* d_idx = (uint32_t*)ctx->tmp[5].p;
  std::vector<uint32_t> lens(n_units);
  const uint32_t upw = units_per_warp(ctx, n_units);
  cf_launch_mask_seq(json_blocks(n_units, upw), b->d_buf + cf::FRONT_PAD, b->d_offsets, n_units, (cfj::JNode*)ctx->d_toon_scratch, d_idx, d_arena, d_len,
                                                 d_st, max_depth, upw, nullptr, nullptr);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  CF_CUDA(ctx, cudaMemcpy(lens.data(), d_len, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  CF_CUDA(ctx, cudaMemcpy(status, d_st, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  // A unit whose output outgrew its 5 * len + 32 bytes (MS_OVERFLOW, lens = the length it needs) is masked again below, straight
  // into its place in the gathered output.  Its offsets count that length already.
  std::vector<uint32_t> retry;
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_units; ++i) {
    if (status[i] == cfm::MS_OVERFLOW) retry.push_back(i);
    out_offsets[i] = total;
    total += lens[i];
  }
  out_offsets[n_units] = total;
  if (out_needed) *out_needed = total;
  if (total > out_cap || (!out_bytes && total)) { ctx->err = "output buffer too small"; return CF_E_CAPACITY; }
  if (total) {
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[4], total))) return rc;
    if ((rc = cf_stage_reserve(ctx, total))) return rc;
    CF_CUDA(ctx, cudaMemcpy(d_ooff, out_offsets, ((size_t)n_units + 1) * 8, cudaMemcpyHostToDevice));
    if (!retry.empty()) {        // the gather copies nothing for them (their text is not in the arena)
      for (uint32_t u : retry) lens[u] = 0;
      CF_CUDA(ctx, cudaMemcpy(d_len, lens.data(), (size_t)n_units * 4, cudaMemcpyHostToDevice));
    }
    compact_kernel<<<n_units, 128>>>(d_arena, 5, 32, b->d_offsets, d_len, d_ooff, (uint8_t*)ctx->tmp[4].p, n_units);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    if (!retry.empty()) {        // the unit list goes to the arena, which the gather has finished reading
      const uint32_t nr = (uint32_t)retry.size();
      uint32_t* d_retry = (uint32_t*)d_arena;
      CF_CUDA(ctx, cudaMemcpy(d_retry, retry.data(), (size_t)nr * 4, cudaMemcpyHostToDevice));
      const uint32_t rupw = units_per_warp(ctx, nr);
      cf_launch_mask_seq(json_blocks(nr, rupw), b->d_buf + cf::FRONT_PAD, b->d_offsets, nr, (cfj::JNode*)ctx->d_toon_scratch, d_idx,
                         (uint8_t*)ctx->tmp[4].p, d_len, d_st, max_depth, rupw, d_retry, d_ooff);
      ctx->launches++;
      CF_CUDA(ctx, cudaGetLastError());
      CF_CUDA(ctx, cudaMemcpy(status, d_st, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
      for (uint32_t u : retry)
        if (status[u] != cfm::MS_OK) { ctx->err = "mask_kernel: a unit retried with the room it asked for did not fit"; return CF_E_CUDA; }
    }
    CF_CUDA(ctx, cudaMemcpy(ctx->h_stage, ctx->tmp[4].p, total, cudaMemcpyDeviceToHost));
    memcpy(out_bytes, ctx->h_stage, total);
  }
  return CF_OK;
}

int cf_classify_keys_host(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets, uint32_t n_units,
                          uint8_t* sensitive) {
  if (!ctx || !b || !sensitive) return CF_E_BADARG;
  int rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
  if (rc) return rc;
  if ((rc = cf_dev_reserve(ctx, ctx->tmp[6], n_units))) return rc;
  uint8_t* d = (uint8_t*)ctx->tmp[6].p;
  cf_launch_classify_keys((n_units + 127) / 128, b->d_buf + cf::FRONT_PAD, b->d_offsets, n_units, d);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  CF_CUDA(ctx, cudaMemcpy(sensitive, d, n_units, cudaMemcpyDeviceToHost));
  return CF_OK;
}


// ------------------------------------------------------------------------------------------------
// the fused chain on the caller's stream (cf_run_enqueue / cf_run_finish, include/cfgpu.h).  Stream st: scan, TOON, verdicts,
// offsets, gather.  The run's side stream: dirty-unit selection + substitution, which need only the scan's bitmaps and so run
// beside the TOON kernel.  Nothing between the first launch and the return reads device memory on the host.
// ------------------------------------------------------------------------------------------------

// verdict records of cf_run_batch's semantics, and per unit the source and length of its produced text (len[n] = 0, so that the
// exclusive scan of len gives out_offsets[0..n]).  A dirty unit whose substitution did not run (RUN_DEFER_PENDING) or outgrew its
// bound (SUB_OVERFLOW) is deferred: appended to `deferred`, slot[u] = RUN_DEFER | its index there, no output yet.  cf_run_finish runs
// the kernel again with def_rec: the deferred units' records from the synchronous substitution (offsets relative to def_base).
__global__ void __launch_bounds__(256) run_verdict_kernel(uint32_t n, uint32_t stage_mask, const uint8_t* __restrict__ unit_stages,
                                                          const uint64_t* __restrict__ bm, uint32_t W, const uint32_t* __restrict__ toon_ls,
                                                          uint32_t* slot, const uint64_t* __restrict__ rec, const uint8_t* arena,
                                                          const uint64_t* __restrict__ def_rec, const uint8_t* def_base, const uint8_t* stream,
                                                          const uint64_t* __restrict__ offsets, const uint8_t* toon_out, uint32_t* __restrict__ deferred,
                                                          RunStatus* st, cf_verdict* __restrict__ v, uint64_t* __restrict__ src, uint64_t* __restrict__ len) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u == n) len[n] = 0;
  if (u >= n) return;
  uint32_t flags = 0, out_len = 0;
  int32_t aux = 0;
  uintptr_t s = 0;
  const bool toon = (stage_mask & CF_STAGE_TOON) && (!unit_stages || (unit_stages[u] & CF_STAGE_TOON));
  const uint32_t sl = slot ? slot[u] : RUN_NOT_DIRTY;
  if (sl != RUN_NOT_DIRTY) {
    flags = CF_V_REWRITTEN | (toon ? CF_V_RESUBMIT : 0u);    // the caller TOON-encodes the rewritten text
    uint64_t at = SUB_OVERFLOW, l = 0;
    const uint8_t* base = arena;
    bool defer = sl == RUN_DEFER_PENDING;
    if (!defer && (sl & RUN_DEFER)) {
      if (def_rec) { at = def_rec[2 * (uint64_t)(sl & ~RUN_DEFER)]; l = def_rec[2 * (uint64_t)(sl & ~RUN_DEFER) + 1]; base = def_base; }
    } else if (!defer) {
      at = rec[2 * (uint64_t)sl];
      l = rec[2 * (uint64_t)sl + 1];
      defer = at == SUB_OVERFLOW;
    }
    if (defer) {
      const uint32_t k = atomicAdd(&st->n_deferred, 1u);
      deferred[k] = u;
      slot[u] = RUN_DEFER | k;
    } else if (at != SUB_OVERFLOW) {
      s = at == ~0ull ? (uintptr_t)(stream + offsets[u]) : (uintptr_t)(base + at);
      out_len = (uint32_t)l;
    }
  }
  if (stage_mask & CF_STAGE_TOON) {
    aux = (flags & CF_V_RESUBMIT) ? CF_TOON_SKIPPED : (int32_t)toon_ls[n + u];
    if (aux == CF_TOON_CONVERTED && !(flags & CF_V_REWRITTEN)) {
      flags |= CF_V_TOON;
      out_len = toon_ls[u];
      s = (uintptr_t)(toon_out + offsets[u]);
    }
  }
  cf_verdict r;
  r.match_bitmap = bm ? bm[(uint64_t)u * W] : 0;
  r.flags = flags;
  r.out_len = out_len;
  r.aux = aux;
  r.reserved = 0;
  v[u] = r;
  src[u] = s;
  len[u] = out_len;
}

// gather of every produced text: dst[out_off[u], out_off[u+1]) = src[u][0, len), one warp per unit.  16-byte stores; 16-byte loads
// when source and destination share their alignment, otherwise aligned 4-byte loads funnel-shifted into place.  Every word loaded
// holds at least one byte of the source span, so no load leaves the span's 4-byte-aligned envelope.  When the total exceeds out_cap
// nothing is written and the status block says so.
__global__ void __launch_bounds__(256) gather_kernel(const uint64_t* __restrict__ out_off, const uint64_t* __restrict__ src, uint8_t* __restrict__ out,
                                                     uint32_t n_units, uint64_t out_cap, RunStatus* st) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t total = out_off[n_units];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->needed = total;
    if (total > out_cap) st->err = CF_E_CAPACITY;
  }
  if (total > out_cap || u >= n_units) return;
  uint64_t n = out_off[u + 1] - out_off[u];
  if (!n) return;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(src[u]);
  uint8_t* d = out + out_off[u];
  const uint64_t head = min(n, (uint64_t)((16u - ((uint32_t)(uintptr_t)d & 15u)) & 15u));
  if (lane < head) d[lane] = s[lane];
  d += head; s += head; n -= head;
  const uint64_t nv = n >> 4;
  uint4* dv = reinterpret_cast<uint4*>(d);
  if (((uint32_t)(uintptr_t)s & 15u) == 0) {
    const uint4* sv = reinterpret_cast<const uint4*>(s);
    for (uint64_t k = lane; k < nv; k += 32) dv[k] = sv[k];
  } else {
    const uint32_t* sw = reinterpret_cast<const uint32_t*>((uintptr_t)s & ~(uintptr_t)3);
    const uint32_t sh = ((uint32_t)(uintptr_t)s & 3u) * 8u;
    for (uint64_t k = lane; k < nv; k += 32) {
      const uint32_t* q = sw + 4 * k;
      const uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3], w4 = sh ? q[4] : 0u;
      dv[k] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
    }
  }
  const uint64_t t = nv << 4;
  if (lane < n - t) d[t + lane] = s[t + lane];
}

// the gather of the run's last enqueue into run->d_out (run->out_cap bytes)
static int run_gather(cf_ctx* ctx, cf_run* run) {
  const uint32_t n = run->batch->n;
  CF_CUDA(ctx, cudaMemsetAsync(&run->d_status->err, 0, sizeof(int32_t), run->st));
  gather_kernel<<<(n + 7) / 8, 256, 0, run->st>>>(run->d_out_offsets, run->d_src, run->d_out, n, run->out_cap, run->d_status);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  return CF_OK;
}

// verdict records, out_offsets (exclusive scan of the lengths) and the gather of the run's last enqueue
static int run_assemble(cf_ctx* ctx, cf_run* run, const uint64_t* def_rec, const uint8_t* def_base) {
  cf_batch* b = run->batch;
  const uint32_t n = b->n;
  run_verdict_kernel<<<(n + 256) / 256, 256, 0, run->st>>>(n, run->stage_mask, run->d_unit_stages, run->d_bitmaps, run->W, run->d_toon_ls,
                                                           run->sub ? run->d_slot : nullptr, run->d_rec, run->enq_arena, def_rec, def_base,
                                                           b->d_buf + cf::FRONT_PAD, b->d_offsets, run->d_toon_out, run->d_deferred, run->d_status,
                                                           run->d_verdicts, run->d_src, run->d_len);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  size_t tmp = 0;
  CF_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const uint64_t*)run->d_len, run->d_out_offsets, (int)n + 1, run->st));
  if (tmp > run->scan_tmp_bytes) { ctx->err = "offset scan workspace too small"; return CF_E_CAPACITY; }
  CF_CUDA(ctx, cub::DeviceScan::ExclusiveSum(run->d_scan_tmp, tmp, (const uint64_t*)run->d_len, run->d_out_offsets, (int)n + 1, run->st));
  ctx->launches++;
  return run_gather(ctx, run);
}

// device -> host copy on the run's side stream (non-blocking and idle once ev_done has completed), so that a finish never waits for
// work the caller has queued on other streams since
static int run_d2h(cf_ctx* ctx, cf_run* run, void* dst, const void* src, size_t bytes) {
  CF_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, run->side));
  CF_CUDA(ctx, cudaStreamSynchronize(run->side));
  return CF_OK;
}

// cf_run_finish without the arena's growth: cf_run_batch may gather again (into a larger buffer) from the arena first.  h_offsets:
// the host copy of the batch's offsets that sizes the deferred units' scratch (NULL: read them from the device).  *out_short is set
// when, and only when, CF_E_CAPACITY means the gather's output buffer: every error of the deferred units' substitution (its own
// CF_E_CAPACITY limits included) is returned as that substitution returned it.
static int run_finish(cf_ctx* ctx, cf_run* run, const uint64_t* h_offsets, uint64_t* needed, bool* out_short) {
  *out_short = false;
  if (!ctx || !run || run->ctx != ctx) return CF_E_BADARG;
  if (!run->batch) { ctx->err = "cf_run_finish: nothing was enqueued on this run"; return CF_E_BADARG; }
  CF_CUDA(ctx, cudaEventSynchronize(run->ev_done));
  int rc;
  if ((rc = run_d2h(ctx, run, run->h_status, run->d_status, sizeof(RunStatus)))) return rc;
  if (const uint32_t nd = run->h_status->n_deferred) {
    // the deferred units through the synchronous substitution (regrowth, CF_E_TOO_LARGE), then verdicts, offsets and gather again
    cf_batch* b = run->batch;
    std::vector<uint32_t> units(nd);
    if ((rc = run_d2h(ctx, run, units.data(), run->d_deferred, (size_t)nd * 4))) return rc;
    std::vector<uint64_t> offs;
    if (!h_offsets) {
      offs.resize((size_t)b->n + 1);
      if ((rc = run_d2h(ctx, run, offs.data(), b->d_offsets, ((size_t)b->n + 1) * 8))) return rc;
      h_offsets = offs.data();
    }
    if ((rc = cf_stage_reserve(ctx, cf_sub_stage_bytes(nd)))) return rc;
    const uint64_t* rec = nullptr;
    if ((rc = cf_sub_device(ctx, run->prog, b, h_offsets, units.data(), nd, run->st, (uint8_t*)ctx->h_stage, &rec))) return rc;
    CF_CUDA(ctx, cudaMemcpyAsync(run->d_def_rec, rec, (size_t)nd * 16, cudaMemcpyHostToDevice, run->st));
    if ((rc = run_assemble(ctx, run, run->d_def_rec, (const uint8_t*)ctx->tmp[8].p))) return rc;
    CF_CUDA(ctx, cudaStreamSynchronize(run->st));
    if ((rc = run_d2h(ctx, run, run->h_status, run->d_status, sizeof(RunStatus)))) return rc;
  }
  if (needed) *needed = run->h_status->needed;
  if (run->h_status->err) { ctx->err = "output buffer too small"; *out_short = true; return CF_E_CAPACITY; }
  return CF_OK;
}

// the arena for the next call: what this one asked for, and a quarter more.  Once an enqueue of this run was captured in a CUDA graph,
// the graph holds the arena's address: the old arena then stays allocated until cf_run_free, so that a replay never writes freed memory.
static int run_grow_arena(cf_ctx* ctx, cf_run* run) {
  const uint64_t used = run->h_status->arena_used;
  if (used <= run->arena_bytes) return CF_OK;
  if (run->ever_captured) run->retired.push_back(run->d_arena);
  else cudaFree(run->d_arena);
  run->d_arena = nullptr;
  run->arena_bytes = 0;
  CF_CUDA(ctx, cudaMalloc(&run->d_arena, used + used / 4));
  run->arena_bytes = used + used / 4;
  return CF_OK;
}

// own_toon == false: the run gets no TOON workspace of its own; cf_run_batch lends it the context's before each enqueue
static int run_create(cf_ctx* ctx, uint32_t max_units, uint64_t max_stream_bytes, uint64_t sub_arena_bytes, bool own_toon, cf_run** out) {
  if (!ctx || !out || !max_units) return CF_E_BADARG;
  *out = nullptr;
  CF_CUDA(ctx, cudaSetDevice(ctx->device));
  cf_run* r = new (std::nothrow) cf_run();
  if (!r) return CF_E_NOMEM;
  r->ctx = ctx;
  r->max_units = max_units;
  r->max_bytes = max_stream_bytes;
  struct Guard { cf_run*& r; ~Guard() { if (r) cf_run_free(r); } } guard{r};   // every error return frees what was made
  const uint32_t n = max_units;
  int rc;
  auto dev = [&](auto** p, size_t bytes) -> int {
    void* q = nullptr;
    CF_CUDA(ctx, cudaMalloc(&q, bytes ? bytes : 16));
    r->allocs.push_back(q);
    *p = reinterpret_cast<std::remove_pointer_t<decltype(p)>>(q);
    return CF_OK;
  };
  if (own_toon) {
    r->toon_scratch_bytes = toon_scratch_need(max_stream_bytes, n);
    size_t sort_tmp = 0;
    if ((rc = toon_sort_temp(ctx, n, nullptr, &sort_tmp))) return rc;
    r->toon_sort_bytes = toon_sort_tmp_offset(n) + sort_tmp;
    if ((rc = dev(&r->d_toon_scratch, r->toon_scratch_bytes)) || (rc = dev(&r->d_toon_order, (size_t)n * 4)) || (rc = dev(&r->d_toon_sort, r->toon_sort_bytes)) ||
        (rc = dev(&r->d_toon_out, max_stream_bytes + 16)) || (rc = dev(&r->d_toon_ls, (size_t)n * 8)))
      return rc;
  }
  CF_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, r->scan_tmp_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n + 1));
  if ((rc = dev(&r->d_queue, (size_t)ctx->qcap * 8)) || (rc = dev(&r->d_qstate, 32)) || (rc = dev(&r->d_slot, (size_t)n * 4)) || (rc = dev(&r->d_sel, (size_t)n * 4)) ||
      (rc = dev(&r->d_soff, (size_t)n * 8)) || (rc = dev(&r->d_bound, (size_t)n * 8)) || (rc = dev(&r->d_rec, (size_t)n * 16)) ||
      (rc = dev(&r->d_deferred, (size_t)n * 4)) || (rc = dev(&r->d_def_rec, (size_t)n * 16)) || (rc = dev(&r->d_src, (size_t)n * 8)) ||
      (rc = dev(&r->d_len, ((size_t)n + 1) * 8)) || (rc = dev(&r->d_scan_tmp, r->scan_tmp_bytes)) || (rc = dev(&r->d_status, sizeof(RunStatus))))
    return rc;
  CF_CUDA(ctx, cudaMemset(r->d_qstate, 0, 32));
  CF_CUDA(ctx, cudaMemset(r->d_status, 0, sizeof(RunStatus)));
  if (sub_arena_bytes) {
    CF_CUDA(ctx, cudaMalloc(&r->d_arena, sub_arena_bytes));
    r->arena_bytes = sub_arena_bytes;
  }
  CF_CUDA(ctx, cudaHostAlloc((void**)&r->h_status, sizeof(RunStatus), cudaHostAllocDefault));
  memset(r->h_status, 0, sizeof(RunStatus));
  int prio_lo = 0, prio_hi = 0;   // the few substitution blocks take SMs as TOON blocks retire instead of queueing behind all of them
  CF_CUDA(ctx, cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  CF_CUDA(ctx, cudaStreamCreateWithPriority(&r->side, cudaStreamNonBlocking, prio_hi));
  for (cudaEvent_t* e : {&r->ev_scan, &r->ev_sub, &r->ev_done}) CF_CUDA(ctx, cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  if ((rc = toon_tp_prepare(ctx))) return rc;
  *out = r;
  r = nullptr;
  return CF_OK;
}
int cf_run_create(cf_ctx* ctx, uint32_t max_units, uint64_t max_stream_bytes, uint64_t sub_arena_bytes, cf_run** out) {
  return run_create(ctx, max_units, max_stream_bytes, sub_arena_bytes, true, out);
}

void cf_run_free(cf_run* run) {
  if (!run) return;
  cudaSetDevice(run->ctx->device);
  if (run->side) cudaStreamSynchronize(run->side);
  for (void* p : run->allocs) cudaFree(p);
  cudaFree(run->d_arena);
  for (void* p : run->retired) cudaFree(p);
  if (run->h_status) cudaFreeHost(run->h_status);
  if (run->side) cudaStreamDestroy(run->side);
  for (cudaEvent_t e : {run->ev_scan, run->ev_sub, run->ev_done}) if (e) cudaEventDestroy(e);
  delete run;
}

int cf_run_enqueue(cf_ctx* ctx, cf_prog* prog, cf_batch* b, cf_run* run, uint32_t stage_mask, const uint8_t* d_unit_stages, uint32_t toon_flags,
                   cf_verdict* d_verdicts, uint64_t* d_bitmaps_full, uint64_t* d_out_offsets, uint8_t* d_out, uint64_t out_cap, void* cuda_stream) {
  if (!ctx || !b || !run || run->ctx != ctx || !d_verdicts || !d_out_offsets || (!d_out && out_cap)) return CF_E_BADARG;
  if (stage_mask & CF_STAGE_MASK) { ctx->err = "cf_run_enqueue runs CF_STAGE_SCAN / SUB / TOON; masking needs cf_run_batch"; return CF_E_BADARG; }
  if (stage_mask & ~(CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_TOON)) { ctx->err = "unknown stage bits"; return CF_E_BADARG; }
  if (stage_mask & CF_STAGE_SUB) stage_mask |= CF_STAGE_SCAN;
  if ((stage_mask & CF_STAGE_SCAN) && (!prog || !d_bitmaps_full)) { ctx->err = "CF_STAGE_SCAN / SUB need a program and d_bitmaps_full"; return CF_E_BADARG; }
  const uint32_t n = b->n;
  if (!n) { ctx->err = "the batch holds no units"; return CF_E_BADARG; }
  if (n > run->max_units || b->nbytes > run->max_bytes) { ctx->err = "the batch exceeds the run's max_units / max_stream_bytes"; return CF_E_CAPACITY; }
  cudaStream_t st = (cudaStream_t)cuda_stream;
  // every check that can fail comes before the first launch, so that an error return leaves nothing queued
  int rc;
  const ToonWs ws{run->d_toon_scratch, run->toon_scratch_bytes, run->d_toon_order, run->d_toon_sort, run->toon_sort_bytes};
  if (stage_mask & CF_STAGE_TOON) {
    if (!run->d_toon_scratch || !run->d_toon_out) { ctx->err = "the run has no TOON workspace"; return CF_E_BADARG; }
    if ((rc = toon_ws_check(ctx, b, ws, st))) return rc;
  }
  size_t scan_tmp = 0;
  CF_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n + 1, st));
  if (scan_tmp > run->scan_tmp_bytes) { ctx->err = "offset scan workspace too small"; return CF_E_CAPACITY; }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CF_CUDA(ctx, cudaStreamIsCapturing(st, &cs));
  if (cs == cudaStreamCaptureStatusActive) run->ever_captured = true;
  run->prog = prog;
  run->batch = b;
  run->st = st;
  run->stage_mask = stage_mask;
  run->d_unit_stages = d_unit_stages;
  run->d_verdicts = d_verdicts;
  run->d_bitmaps = (stage_mask & CF_STAGE_SCAN) ? d_bitmaps_full : nullptr;
  run->d_out_offsets = d_out_offsets;
  run->d_out = d_out;
  run->out_cap = out_cap;
  run->W = prog ? prog->W : 1;
  run->sub = (stage_mask & CF_STAGE_SUB) && !prog->ordered.empty();
  run->enq_arena = run->d_arena;      // a finish after a replay of this enqueue must read the arena the graph holds, even once grown
  CF_CUDA(ctx, cudaMemsetAsync(run->d_status, 0, sizeof(RunStatus), st));
  if ((stage_mask & CF_STAGE_SCAN) && (rc = cf_scan_launch(ctx, prog, b, d_bitmaps_full, st, run->d_queue, run->d_qstate, &run->qphase))) return rc;
  if (run->sub) {
    CF_CUDA(ctx, cudaEventRecord(run->ev_scan, st));
    CF_CUDA(ctx, cudaStreamWaitEvent(run->side, run->ev_scan, 0));
    if ((rc = cf_sub_enqueue(ctx, prog, b, run, d_bitmaps_full, d_unit_stages, run->side))) return rc;
    CF_CUDA(ctx, cudaEventRecord(run->ev_sub, run->side));
  }
  if (stage_mask & CF_STAGE_TOON) {
    if ((rc = toon_enqueue(ctx, b, toon_flags & ~(CF_TOON_PARSE_ONLY | CF_TOON_SEQUENTIAL | CF_RUN_OUTPUTS_RESIDENT), run->d_toon_out, run->d_toon_ls,
                           (int32_t*)(run->d_toon_ls + n), d_unit_stages, st, ws))) return rc;
  }
  if (run->sub) CF_CUDA(ctx, cudaStreamWaitEvent(st, run->ev_sub, 0));
  if ((rc = run_assemble(ctx, run, nullptr, nullptr))) return rc;
  // inside a stream capture the completion event becomes a node of the graph, so that cf_run_finish waits for each replay
  CF_CUDA(ctx, cudaEventRecordWithFlags(run->ev_done, st, cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault));
  return CF_OK;
}

int cf_run_finish(cf_ctx* ctx, cf_run* run, uint64_t* needed) {
  if (needed) *needed = 0;
  bool out_short = false;
  int rc = run_finish(ctx, run, nullptr, needed, &out_short);
  if (rc == CF_E_CAPACITY && !out_short) rc = CF_E_TOO_LARGE;   // a deferred unit's substitution hit one of its limits: not the output buffer
  if (ctx && run && run->ctx == ctx) {
    const int g = run_grow_arena(ctx, run);
    if (g && !rc) return g;
  }
  return rc;
}

// ---- the fused chain with host buffers (include/cfgpu.h): one H2D of the stream, cf_run_enqueue + cf_run_finish on the context's
// run (legacy stream), then verdicts, offsets and only the produced texts cross PCIe back through the context's pinned staging.
// With CF_STAGE_MASK the run (SCAN / SUB, when asked for) gives the verdicts, and the masking kernel then the texts, statuses and offsets.
int cf_run_batch(cf_ctx* ctx, cf_prog* prog, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets, uint32_t n_units,
                 uint32_t stage_mask, const uint8_t* unit_stages, uint32_t toon_flags, int mask_max_depth, cf_verdict* verdicts, uint64_t* bitmaps_full,
                 uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, uint64_t* out_needed) {
  if (!ctx || !b || !offsets || !n_units || !verdicts || !out_offsets) return CF_E_BADARG;
  if ((stage_mask & (CF_STAGE_SCAN | CF_STAGE_SUB)) && !prog) return CF_E_BADARG;
  if ((stage_mask & CF_STAGE_TOON) && (stage_mask & CF_STAGE_MASK)) { ctx->err = "CF_STAGE_TOON and CF_STAGE_MASK both produce the unit's output: two calls"; return CF_E_BADARG; }
  if (stage_mask & CF_STAGE_SUB) stage_mask |= CF_STAGE_SCAN;
  if (!stream && (b->n != n_units || b->nbytes != stream_bytes)) { ctx->err = "resident run: the batch on the device is a different one"; return CF_E_BADARG; }
  struct Nvtx { Nvtx(const char* n) { nvtxRangePushA(n); } ~Nvtx() { nvtxRangePop(); } } nvtx_call("cf_run_batch");   // ranges: assemble (caller) | h2d | kernels | d2h
  // every return, error returns included, waits for the run's streams: nothing the next call's buffers are reused for stays in flight
  struct Drain { cf_ctx* c; ~Drain() { if (c->run) cudaStreamSynchronize(c->run->side); cudaStreamSynchronize(0); } } drain{ctx};
  const bool mask = (stage_mask & CF_STAGE_MASK) != 0;
  stage_mask &= ~CF_STAGE_MASK;
  const bool keep = !mask && (toon_flags & CF_RUN_OUTPUTS_RESIDENT) != 0;
  const uint32_t W = prog ? prog->W : 1;
  int rc;
  if (stream) {
    nvtxRangePushA("cf_run_batch:h2d");
    rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
    nvtxRangePop();
    if (rc) return rc;
  }
  ctx->run_out = nullptr; ctx->run_out_bytes = 0;
  uint64_t total = 0;
  bool fits = true;
  if (mask && !stage_mask) memset(verdicts, 0, (size_t)n_units * sizeof(cf_verdict));    // masking alone: no run
  else {
    if (!ctx->run || ctx->run->max_units < n_units || ctx->run->max_bytes < stream_bytes) {     // the context's run, grown with the batches
      const uint64_t arena = ctx->run ? ctx->run->arena_bytes : (1ull << 20);
      cf_run_free(ctx->run);
      ctx->run = nullptr;
      if ((rc = run_create(ctx, n_units + n_units / 4, stream_bytes + stream_bytes / 4 + 4096, arena, false, &ctx->run))) return rc;
    }
    cf_run* run = ctx->run;
    if (stage_mask & CF_STAGE_TOON) {       // the context's TOON workspace, lent to its run: TOON output in tmp[0], lengths | statuses in tmp[2]
      ToonWs ws;
      if ((rc = toon_ctx_ws(ctx, b, 0, 0, &ws)) || (rc = cf_dev_reserve(ctx, ctx->tmp[0], stream_bytes + 16)) ||
          (rc = cf_dev_reserve(ctx, ctx->tmp[2], (size_t)n_units * 8)))
        return rc;
      run->d_toon_scratch = ws.scratch; run->toon_scratch_bytes = ws.scratch_bytes;
      run->d_toon_order = ws.order; run->d_toon_sort = ws.sort; run->toon_sort_bytes = ws.sort_bytes;
      run->d_toon_out = (uint8_t*)ctx->tmp[0].p;
      run->d_toon_ls = (uint32_t*)ctx->tmp[2].p;
    }
    // pinned staging: unit_stages on the way in; verdicts | out_offsets | bitmaps on the way out
    const size_t o_oo = ((size_t)n_units * sizeof(cf_verdict) + 15) & ~(size_t)15, o_bm = (o_oo + ((size_t)n_units + 1) * 8 + 15) & ~(size_t)15;
    const size_t bm_bytes = (stage_mask & CF_STAGE_SCAN) ? (size_t)n_units * W * 8 : 0;
    if ((rc = cf_stage_reserve(ctx, std::max(o_bm + bm_bytes, (size_t)n_units)))) return rc;
    uint8_t* hs = (uint8_t*)ctx->h_stage;
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[1], (size_t)n_units * sizeof(cf_verdict))) || (rc = cf_dev_reserve(ctx, ctx->tmp[3], ((size_t)n_units + 1) * 8)) ||
        (bm_bytes && (rc = cf_dev_reserve(ctx, ctx->tmp[6], bm_bytes))) ||
        (rc = cf_dev_reserve(ctx, ctx->tmp[4], std::max<uint64_t>(16, keep ? stream_bytes : std::min(out_cap, stream_bytes)))))
      return rc;
    uint8_t* d_us = nullptr;
    if (unit_stages) {
      if ((rc = cf_dev_reserve(ctx, ctx->tmp[7], n_units))) return rc;
      d_us = (uint8_t*)ctx->tmp[7].p;
      memcpy(hs, unit_stages, n_units);
      CF_CUDA(ctx, cudaMemcpyAsync(d_us, hs, n_units, cudaMemcpyHostToDevice, 0));
    }
    cf_verdict* d_v = (cf_verdict*)ctx->tmp[1].p;
    uint64_t* d_oo = (uint64_t*)ctx->tmp[3].p;
    // the device buffer takes what the caller can take (all of it when the texts stay resident); a shortfall of the device buffer alone
    // is made up below by growing it and gathering again.  Masking returns no rewritten texts: the run gathers none, and the
    // CF_E_CAPACITY its finish then reports for rewritten units is expected.
    uint8_t* d_out = mask ? nullptr : (uint8_t*)ctx->tmp[4].p;
    const uint64_t dcap = keep ? ctx->tmp[4].cap : (d_out && out_bytes ? std::min<uint64_t>(ctx->tmp[4].cap, out_cap) : 0);
    nvtxRangePushA("cf_run_batch:kernels");
    rc = cf_run_enqueue(ctx, prog, b, run, stage_mask, d_us, toon_flags, d_v, bm_bytes ? (uint64_t*)ctx->tmp[6].p : nullptr, d_oo, d_out, dcap, nullptr);
    bool out_short = false;
    if (!rc) rc = run_finish(ctx, run, offsets, &total, &out_short);
    nvtxRangePop();
    if (out_short && d_out && (keep || (out_bytes && total <= out_cap))) {
      if ((rc = cf_dev_reserve(ctx, ctx->tmp[4], total))) return rc;
      run->d_out = (uint8_t*)ctx->tmp[4].p;
      run->out_cap = total;
      if ((rc = run_gather(ctx, run))) return rc;
      CF_CUDA(ctx, cudaStreamSynchronize(0));
    }
    const int grown = run_grow_arena(ctx, run);
    if (rc && !out_short) return rc;
    if (grown) return grown;
    Nvtx nvtx_d2h("cf_run_batch:d2h");
    if ((rc = cf_stage_reserve(ctx, o_bm + bm_bytes))) return rc;    // a deferred unit's substitution may have grown the staging
    hs = (uint8_t*)ctx->h_stage;
    CF_CUDA(ctx, cudaMemcpyAsync(hs, d_v, (size_t)n_units * sizeof(cf_verdict), cudaMemcpyDeviceToHost, 0));
    CF_CUDA(ctx, cudaMemcpyAsync(hs + o_oo, d_oo, ((size_t)n_units + 1) * 8, cudaMemcpyDeviceToHost, 0));
    if (bitmaps_full && bm_bytes) CF_CUDA(ctx, cudaMemcpyAsync(hs + o_bm, ctx->tmp[6].p, bm_bytes, cudaMemcpyDeviceToHost, 0));
    fits = keep || (total <= out_cap && (out_bytes || !total));
    if (fits && d_out && !keep && total) CF_CUDA(ctx, cudaMemcpyAsync(out_bytes, ctx->tmp[4].p, total, cudaMemcpyDeviceToHost, 0));
    CF_CUDA(ctx, cudaStreamSynchronize(0));
    memcpy(verdicts, hs, (size_t)n_units * sizeof(cf_verdict));
    memcpy(out_offsets, hs + o_oo, ((size_t)n_units + 1) * 8);
    if (bitmaps_full && bm_bytes) memcpy(bitmaps_full, hs + o_bm, bm_bytes);
  }
  if (mask) {     // the masked bodies are the output: the mask's texts, offsets, size and CF_E_CAPACITY; its statuses patch the records
    std::vector<int32_t> mst(n_units);
    if ((rc = cf_mask_resident(ctx, b, mask_max_depth, out_bytes, out_cap, out_offsets, mst.data(), out_needed))) return rc;
    for (uint32_t i = 0; i < n_units; ++i) {
      verdicts[i].aux = mst[i];
      if (mst[i] == CF_MASK_OK) { verdicts[i].flags |= CF_V_MASKED; verdicts[i].out_len = (uint32_t)(out_offsets[i + 1] - out_offsets[i]); }
    }
    return CF_OK;
  }
  if (out_needed) *out_needed = total;
  if (!fits) { ctx->err = "output buffer too small"; return CF_E_CAPACITY; }
  if (keep) {
    ctx->run_out = total ? (const uint8_t*)ctx->tmp[4].p : nullptr;
    ctx->run_out_bytes = total;
  }
  return CF_OK;
}

int cf_run_batch_device_output(cf_ctx* ctx, const uint8_t** d_out, uint64_t* bytes) {
  if (!ctx || !d_out || !bytes) return CF_E_BADARG;
  *d_out = ctx->run_out;
  *bytes = ctx->run_out_bytes;
  return CF_OK;
}

int cf_copy_to_host(cf_ctx* ctx, void* host_dst, const void* device_src, uint64_t bytes) {
  if (!ctx || (bytes && (!host_dst || !device_src))) return CF_E_BADARG;
  if (bytes) CF_CUDA(ctx, cudaMemcpy(host_dst, device_src, bytes, cudaMemcpyDeviceToHost));
  return CF_OK;
}

int cf_profile_collect_each(cf_ctx* ctx, double* ms, uint32_t cap, uint32_t* n_launches) {
  if (!ctx || !ms || !n_launches) return CF_E_BADARG;
  uint32_t n = 0;
  for (uint32_t i = 0; i + 1 < ctx->prof_used; i += 2) {
    CF_CUDA(ctx, cudaEventSynchronize(ctx->prof_ev[i + 1]));
    float t = 0;
    CF_CUDA(ctx, cudaEventElapsedTime(&t, ctx->prof_ev[i], ctx->prof_ev[i + 1]));
    if (n < cap) ms[n] = t;
    ++n;
  }
  *n_launches = n;
  ctx->prof_used = 0;
  return CF_OK;
}

}  // extern "C"
