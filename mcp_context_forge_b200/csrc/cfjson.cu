// cfjson.cu — the JSON kernels of libcfgpu.so and their C-ABI entry points (include/cfgpu.h): structural index
// (json_index.h), toon_encoder (token-parallel json_tp.h + sequential json_toon.h for the units it hands over),
// request_logging_masking (json_mask.h).  Split from cfgpu.cu so that either half rebuilds on its own.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>
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

static int toon_launch(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, const uint8_t* d_unit_stages,
                       cudaStream_t st) {
  uint64_t need = (b->nbytes / 2 + 4ull * b->n + 8) * sizeof(cfj::JNode);
  const uint64_t need_tp = (b->nbytes / 2 + (uint64_t)TP_TOK_SLACK * b->n + 8) * sizeof(cftp::GTok);
  if (need_tp > need) need = need_tp;
  if (need > ctx->toon_scratch_bytes) {
    CF_CUDA(ctx, cudaStreamSynchronize(st));
    cudaFree(ctx->d_toon_scratch);
    ctx->d_toon_scratch = nullptr;
    ctx->toon_scratch_bytes = 0;
    CF_CUDA(ctx, cudaMalloc(&ctx->d_toon_scratch, need + need / 4));
    ctx->toon_scratch_bytes = need + need / 4;
  }
  const bool tp = !(flags & (CF_TOON_PARSE_ONLY | CF_TOON_SEQUENTIAL));
  // the first pass's unit order: key + stable radix sort over its 8 bits, descending; toon_sort = indices | keys in | keys out | temp
  const size_t o_kin = (size_t)b->n * 4, o_kout = o_kin + b->n, o_tmp = (o_kout + b->n + 255) & ~(size_t)255;
  size_t sort_tmp = 0;
  if (tp) {
    CF_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_tmp, (const uint8_t*)nullptr, (uint8_t*)nullptr, (const uint32_t*)nullptr,
                                                           (uint32_t*)nullptr, (int)b->n, 0, 8, st));
    int rc;
    if ((rc = cf_dev_reserve(ctx, ctx->toon_order, (size_t)b->n * 4))) return rc;
    if ((rc = cf_dev_reserve(ctx, ctx->toon_sort, o_tmp + sort_tmp))) return rc;
  }
  const bool prof = ctx->prof_on && (size_t)ctx->prof_used + 2 <= ctx->prof_ev.size();
  if (prof) cudaEventRecord(ctx->prof_ev[ctx->prof_used], st);
  if (tp) {
    static bool smem_set = false;
    if (!smem_set) {
      CF_CUDA(ctx, cudaFuncSetAttribute(toon_tp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TP_SMEM));
      smem_set = true;
    }
    uint8_t* srt = (uint8_t*)ctx->toon_sort.p;
    uint32_t* order = (uint32_t*)ctx->toon_order.p;
    toon_order_kernel<<<(b->n + 7) / 8, 256, 0, st>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, d_unit_stages, srt + o_kin, (uint32_t*)srt);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    CF_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(srt + o_tmp, sort_tmp, srt + o_kin, srt + o_kout, (const uint32_t*)srt, order, (int)b->n, 0, 8, st));
    ctx->launches++;
    const uint32_t grid = (b->n + TP_WARPS - 1) / TP_WARPS;
    toon_tp_kernel<<<grid, TP_WARPS * 32, TP_SMEM, st>>>(b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cftp::GTok*)ctx->d_toon_scratch, d_out, d_out_len,
                                                         d_status, flags, d_unit_stages, order);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    // the units the fast path handed over: sequential encoder, one unit per warp (they are few)
    if (!(flags & CF_TOON_NO_HANDOVER)) cf_launch_toon_seq(json_blocks(b->n, 1), st, b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cfj::JNode*)ctx->d_toon_scratch, d_out, d_out_len, d_status,
                                                     (flags & 1u) | TOON_ONLY_FALLBACK, 1);
  } else {
    if (d_unit_stages) { ctx->err = "per-unit stage masks need the token-parallel encoder"; return CF_E_BADARG; }
    const uint32_t upw = units_per_warp(ctx, b->n);
    cf_launch_toon_seq(json_blocks(b->n, upw), st, b->d_buf + cf::FRONT_PAD, b->d_offsets, b->n, (cfj::JNode*)ctx->d_toon_scratch, d_out, d_out_len,
                                                       d_status, flags & ~TOON_ONLY_FALLBACK, upw);
  }
  if (prof) { cudaEventRecord(ctx->prof_ev[ctx->prof_used + 1], st); ctx->prof_used += 2; }
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  return CF_OK;
}

int cf_toon(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, void* cuda_stream) {
  if (!ctx || !b || !b->n || !d_out || !d_out_len || !d_status) return CF_E_BADARG;
  return toon_launch(ctx, b, flags, d_out, d_out_len, d_status, nullptr, (cudaStream_t)cuda_stream);
}

int cf_chain(cf_ctx* ctx, cf_prog* prog, cf_batch* b, uint32_t stage_mask, uint32_t toon_flags, uint64_t* d_bitmaps, const uint8_t* d_unit_stages,
             uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, void* cuda_stream) {
  if (!ctx || !b || !b->n) return CF_E_BADARG;
  if (stage_mask & ~(CF_STAGE_SCAN | CF_STAGE_TOON)) { ctx->err = "cf_chain runs CF_STAGE_SCAN / CF_STAGE_TOON; the other stages need cf_run_batch"; return CF_E_BADARG; }
  int rc;
  if (stage_mask & CF_STAGE_SCAN) {
    if (!prog || !d_bitmaps) return CF_E_BADARG;
    if ((rc = cf_scan(ctx, prog, b, d_bitmaps, cuda_stream))) return rc;
  }
  if (stage_mask & CF_STAGE_TOON) {
    if (!d_out || !d_out_len || !d_status) return CF_E_BADARG;
    if ((rc = toon_launch(ctx, b, toon_flags, d_out, d_out_len, d_status, d_unit_stages, (cudaStream_t)cuda_stream))) return rc;
  }
  return CF_OK;
}

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
                                                 d_st, max_depth, upw);
  ctx->launches++;
  CF_CUDA(ctx, cudaGetLastError());
  CF_CUDA(ctx, cudaMemcpy(lens.data(), d_len, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  CF_CUDA(ctx, cudaMemcpy(status, d_st, (size_t)n_units * 4, cudaMemcpyDeviceToHost));
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_units; ++i) { out_offsets[i] = total; total += lens[i]; }
  out_offsets[n_units] = total;
  if (out_needed) *out_needed = total;
  if (total > out_cap || (!out_bytes && total)) { ctx->err = "output buffer too small"; return CF_E_CAPACITY; }
  if (total) {
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[4], total))) return rc;
    if ((rc = cf_stage_reserve(ctx, total))) return rc;
    CF_CUDA(ctx, cudaMemcpy(d_ooff, out_offsets, ((size_t)n_units + 1) * 8, cudaMemcpyHostToDevice));
    compact_kernel<<<n_units, 128>>>(d_arena, 5, 32, b->d_offsets, d_len, d_ooff, (uint8_t*)ctx->tmp[4].p, n_units);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
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


// gather of every text cf_run_batch produced: dst[out_off[u], out_off[u+1]) = src[u][0, len), one warp per unit.  16-byte stores;
// 16-byte loads when source and destination share their alignment, otherwise aligned 4-byte loads funnel-shifted into place.  Every
// word loaded holds at least one byte of the source span, so no load leaves the span's 4-byte-aligned envelope.
__global__ void __launch_bounds__(256) gather_kernel(const uint64_t* __restrict__ out_off, const uint64_t* __restrict__ src, uint8_t* __restrict__ out,
                                                     uint32_t n_units) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= n_units) return;
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

// ---- the fused chain with host buffers (include/cfgpu.h): one H2D of the stream, every stage on the resident batch, then
// verdicts + only the produced texts cross PCIe back.  Legacy stream: scan, TOON, gather.  ctx->side: the substitution of the units a
// rule matched, which needs only the scan's bitmaps and so runs beside the TOON kernel.  Host <-> device copies go through the
// context's pinned staging.
int cf_run_batch(cf_ctx* ctx, cf_prog* prog, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets, uint32_t n_units,
                 uint32_t stage_mask, const uint8_t* unit_stages, uint32_t toon_flags, int mask_max_depth, cf_verdict* verdicts, uint64_t* bitmaps_full,
                 uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, uint64_t* out_needed) {
  if (!ctx || !b || !offsets || !n_units || !verdicts || !out_offsets) return CF_E_BADARG;
  if ((stage_mask & (CF_STAGE_SCAN | CF_STAGE_SUB)) && !prog) return CF_E_BADARG;
  if ((stage_mask & CF_STAGE_TOON) && (stage_mask & CF_STAGE_MASK)) { ctx->err = "CF_STAGE_TOON and CF_STAGE_MASK both produce the unit's output: two calls"; return CF_E_BADARG; }
  if (stage_mask & CF_STAGE_SUB) stage_mask |= CF_STAGE_SCAN;
  if (!stream && (b->n != n_units || b->nbytes != stream_bytes)) { ctx->err = "resident run: the batch on the device is a different one"; return CF_E_BADARG; }
  struct Nvtx { Nvtx(const char* n) { nvtxRangePushA(n); } ~Nvtx() { nvtxRangePop(); } } nvtx_call("cf_run_batch");   // ranges: assemble (caller) | h2d | kernels | d2h
  // every return, error returns included, waits for both streams: nothing the next call's buffers are reused for stays in flight
  struct Drain { cf_ctx* c; ~Drain() { cudaStreamSynchronize(c->side); cudaStreamSynchronize(0); } } drain{ctx};
  const uint32_t W = prog ? prog->W : 1;
  // pinned staging: unit_stages | bitmaps | TOON lengths + statuses | gather descriptors | substitution descriptors
  auto r16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t o_bm = r16(unit_stages ? n_units : 0);
  const size_t o_toon = o_bm + r16((stage_mask & CF_STAGE_SCAN) ? (size_t)n_units * W * 8 : 0);
  const size_t o_gather = o_toon + r16((size_t)n_units * 8);
  const size_t o_sub = o_gather + r16(((size_t)2 * n_units + 1) * 8);
  int rc = cf_stage_reserve(ctx, o_sub + ((stage_mask & CF_STAGE_SUB) ? cf_sub_stage_bytes(n_units) : 0));
  if (rc) return rc;
  uint8_t* hs = (uint8_t*)ctx->h_stage;
  if (stream) {
    nvtxRangePushA("cf_run_batch:h2d");
    rc = cf_batch_upload(ctx, b, stream, stream_bytes, offsets, n_units, nullptr);
    nvtxRangePop();
    if (rc) return rc;
  }
  uint8_t* d_us = nullptr;
  if (unit_stages) {
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[7], n_units))) return rc;
    d_us = (uint8_t*)ctx->tmp[7].p;
    memcpy(hs, unit_stages, n_units);
    CF_CUDA(ctx, cudaMemcpyAsync(d_us, hs, n_units, cudaMemcpyHostToDevice, 0));
  }
  // ---- launches, back to back; each stage's per-unit results come back in one D2H behind it
  nvtxRangePushA("cf_run_batch:kernels");
  const uint64_t* bm = (const uint64_t*)(hs + o_bm);
  uint32_t* tlen = (uint32_t*)(hs + o_toon);
  const int32_t* tst = (const int32_t*)(tlen + n_units);
  if (stage_mask & CF_STAGE_SCAN) {
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[6], (size_t)n_units * W * 8))) return rc;
    if ((rc = cf_scan(ctx, prog, b, (uint64_t*)ctx->tmp[6].p, nullptr))) return rc;
    CF_CUDA(ctx, cudaMemcpyAsync(hs + o_bm, ctx->tmp[6].p, (size_t)n_units * W * 8, cudaMemcpyDeviceToHost, 0));
    CF_CUDA(ctx, cudaEventRecord(ctx->ev_scan, 0));
  }
  if (stage_mask & CF_STAGE_TOON) {
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[0], stream_bytes + 16))) return rc;
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[1], (size_t)n_units * 8))) return rc;     // lengths | statuses
    uint32_t* d_len = (uint32_t*)ctx->tmp[1].p;
    if ((rc = toon_launch(ctx, b, toon_flags & ~(CF_TOON_PARSE_ONLY | CF_TOON_SEQUENTIAL | CF_RUN_OUTPUTS_RESIDENT), (uint8_t*)ctx->tmp[0].p, d_len,
                          (int32_t*)(d_len + n_units), d_us, 0))) return rc;
    CF_CUDA(ctx, cudaMemcpyAsync(tlen, d_len, (size_t)n_units * 8, cudaMemcpyDeviceToHost, 0));
    CF_CUDA(ctx, cudaEventRecord(ctx->ev_toon, 0));
  }
  nvtxRangePop();
  // ---- results of the launches
  Nvtx nvtx_d2h("cf_run_batch:d2h+verdicts");
  for (uint32_t i = 0; i < n_units; ++i) { verdicts[i].match_bitmap = 0; verdicts[i].flags = 0; verdicts[i].out_len = 0; verdicts[i].aux = 0; verdicts[i].reserved = 0; }
  std::vector<uint32_t> dirty;
  if (stage_mask & CF_STAGE_SCAN) {
    CF_CUDA(ctx, cudaEventSynchronize(ctx->ev_scan));
    if (bitmaps_full) memcpy(bitmaps_full, bm, (size_t)n_units * W * 8);
    std::vector<uint64_t> rule_mask(W, 0);
    for (int pi : prog->ordered_pat) rule_mask[(size_t)pi / 64] |= 1ull << (pi % 64);
    for (uint32_t i = 0; i < n_units; ++i) {
      verdicts[i].match_bitmap = bm[(size_t)i * W];
      if ((stage_mask & CF_STAGE_SUB) && (!unit_stages || (unit_stages[i] & CF_STAGE_SUB))) {
        bool d = false;
        for (uint32_t w = 0; w < W; ++w) if (bm[(size_t)i * W + w] & rule_mask[w]) { d = true; break; }
        if (d) dirty.push_back(i);
      }
    }
  }
  // ---- regex_filter rewriting of the (few) units a rule matched, on the side stream while the TOON kernel runs
  const uint64_t* rec = nullptr;
  if (!dirty.empty()) {
    CF_CUDA(ctx, cudaStreamWaitEvent(ctx->side, ctx->ev_scan, 0));
    if ((rc = cf_sub_device(ctx, prog, b, offsets, dirty.data(), (uint32_t)dirty.size(), ctx->side, hs + o_sub, &rec))) return rc;
    CF_CUDA(ctx, cudaEventRecord(ctx->ev_sub, ctx->side));
    CF_CUDA(ctx, cudaStreamWaitEvent(0, ctx->ev_sub, 0));
    for (size_t k = 0; k < dirty.size(); ++k) {
      const uint32_t i = dirty[k];
      verdicts[i].flags |= CF_V_REWRITTEN;
      verdicts[i].out_len = (uint32_t)rec[2 * k + 1];
      if ((stage_mask & CF_STAGE_TOON) && (!unit_stages || (unit_stages[i] & CF_STAGE_TOON))) verdicts[i].flags |= CF_V_RESUBMIT;
    }
  }
  if (stage_mask & CF_STAGE_TOON) {
    CF_CUDA(ctx, cudaEventSynchronize(ctx->ev_toon));
    for (uint32_t i = 0; i < n_units; ++i) {
      const int32_t s = (verdicts[i].flags & CF_V_RESUBMIT) ? CF_TOON_SKIPPED : tst[i];   // the caller encodes the rewritten text
      verdicts[i].aux = s;
      if (s == CF_TOON_CONVERTED && !(verdicts[i].flags & CF_V_REWRITTEN)) { verdicts[i].flags |= CF_V_TOON; verdicts[i].out_len = tlen[i]; }
    }
  }
  // ---- masking on the same upload (sequential kernel; its own gather)
  if (stage_mask & CF_STAGE_MASK) {
    std::vector<int32_t> mst(n_units);
    std::vector<uint64_t> moff((size_t)n_units + 1);
    uint64_t need = 0;
    rc = cf_mask_resident(ctx, b, mask_max_depth, out_bytes, out_cap, moff.data(), mst.data(), &need);
    if (out_needed) *out_needed = need;
    if (rc) return rc;
    for (uint32_t i = 0; i < n_units; ++i) {
      out_offsets[i] = moff[i];
      verdicts[i].aux = mst[i];
      if (mst[i] == CF_MASK_OK) { verdicts[i].flags |= CF_V_MASKED; verdicts[i].out_len = (uint32_t)(moff[i + 1] - moff[i]); }
    }
    out_offsets[n_units] = moff[n_units];
    return CF_OK;
  }
  // ---- pack the outputs: TOON texts (input layout in tmp[0]) and rewritten texts (substitution scratch, or the unit itself) in one
  // gather at their final offsets, then one D2H straight into out_bytes unless they stay resident
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_units; ++i) { out_offsets[i] = total; total += verdicts[i].out_len; }
  out_offsets[n_units] = total;
  if (out_needed) *out_needed = total;
  const bool keep = (toon_flags & CF_RUN_OUTPUTS_RESIDENT) != 0;
  ctx->run_out = nullptr; ctx->run_out_bytes = 0;
  if (!keep && (total > out_cap || (!out_bytes && total))) { ctx->err = "output buffer too small"; return CF_E_CAPACITY; }
  if (total) {
    uint64_t* h_src = (uint64_t*)(hs + o_gather);          // src[n] | out_off[n + 1]: one H2D
    const uintptr_t toon_out = (uintptr_t)ctx->tmp[0].p, d_stream = (uintptr_t)(b->d_buf + cf::FRONT_PAD), scratch = (uintptr_t)ctx->tmp[8].p;
    for (uint32_t i = 0; i < n_units; ++i) h_src[i] = (verdicts[i].flags & CF_V_TOON) ? toon_out + offsets[i] : 0;
    for (size_t k = 0; k < dirty.size(); ++k) h_src[dirty[k]] = rec[2 * k] == ~0ull ? d_stream + offsets[dirty[k]] : scratch + rec[2 * k];
    memcpy(h_src + n_units, out_offsets, ((size_t)n_units + 1) * 8);
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[3], ((size_t)2 * n_units + 1) * 8))) return rc;
    if ((rc = cf_dev_reserve(ctx, ctx->tmp[4], total))) return rc;
    const uint64_t* d_src = (const uint64_t*)ctx->tmp[3].p;
    CF_CUDA(ctx, cudaMemcpyAsync(ctx->tmp[3].p, h_src, ((size_t)2 * n_units + 1) * 8, cudaMemcpyHostToDevice, 0));
    gather_kernel<<<(n_units + 7) / 8, 256, 0, 0>>>(d_src + n_units, d_src, (uint8_t*)ctx->tmp[4].p, n_units);
    ctx->launches++;
    CF_CUDA(ctx, cudaGetLastError());
    if (!keep) CF_CUDA(ctx, cudaMemcpyAsync(out_bytes, ctx->tmp[4].p, total, cudaMemcpyDeviceToHost, 0));
    CF_CUDA(ctx, cudaStreamSynchronize(0));
  }
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
