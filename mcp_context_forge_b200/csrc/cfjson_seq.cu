// cfjson_seq.cu — the sequential (one thread per unit) JSON kernels: toon_kernel (json_toon.h), mask_kernel (json_mask.h) and
// the key classifier.  toon_kernel is what the token-parallel encoder (cfjson.cu, json_tp.h) hands its uncovered units to.
// Own translation unit: these kernels inline the whole parser + exact number formatter and take minutes to compile.
#include "cf_internal.h"
#include "json_mask.h"
#include "json_toon.h"

// toon_encoder: output for unit i goes to out + offsets[i]; a conversion is only produced when it is strictly
// smaller than the input (plugins/toon_encoder/toon_encoder.py:295-303).
__global__ void __launch_bounds__(64) toon_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets,
                                                   uint32_t n_units, cfj::JNode* __restrict__ nodes, uint8_t* __restrict__ out,
                                                   uint32_t* __restrict__ out_len, int32_t* __restrict__ status, uint32_t flags, uint32_t upw) {
  const uint32_t lane = threadIdx.x & 31;
  if (lane >= upw) return;
  const uint32_t u = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * upw + lane;
  if (u >= n_units) return;
  const uint64_t b = offsets[u];
  const uint64_t len64 = offsets[u + 1] - b - 1;
  if (len64 > 0x7FFFFFFFull) { status[u] = cfj::TS_UNSUPPORTED; out_len[u] = 0; return; }
  if ((flags & TOON_ONLY_FALLBACK) && status[u] != CF_TS_FALLBACK) return;
  const uint32_t len = (uint32_t)len64;
  cfj::JNode* my = nodes + (b >> 1) + 4ull * u;
  if (flags & CF_TOON_PARSE_ONLY) {
    uint32_t cnt = 0;
    const int pr = cfj::json_parse(stream + b, len, my, len / 2 + 4, &cnt);
    status[u] = pr; out_len[u] = cnt;
    return;
  }
  cfj::Big big;
  uint8_t digits[1240];
  uint32_t ol = 0;
  const int st = cfj::toon_process(stream + b, len, my, len / 2 + 4, out + b, len ? len - 1 : 0, &ol, &big, digits, sizeof(digits), (flags & 1u) == 0);
  status[u] = st;
  out_len[u] = st == cfj::TS_CONVERTED ? ol : 0;
}

// request_logging_masking: mask_sensitive_json_bytes per unit (csrc/json_mask.h), plus a key classifier
// kernel for the object-level entry points of the drop-in module.  First pass (retry == nullptr): unit u writes into its
// 5 * len + 32 bytes at out + 5 * offsets[u] + 32 * u; a unit whose output needs more room gets MS_OVERFLOW and out_len = the
// length it needs.  Retry pass: the grid covers n_units threads, and thread i < rs->n_retry runs unit retry[i] into exactly
// out_off[u + 1] - out_off[u] bytes at out + out_off[u]; it leaves status and out_len as the first pass wrote them and flags a unit
// that does not fit in rs->mask_err.  Nothing runs when the gather found the output buffer too small (rs->err).
__global__ void __launch_bounds__(64) mask_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets, uint32_t n_units,
                                                   cfj::JNode* __restrict__ nodes, uint32_t* __restrict__ idx, uint8_t* __restrict__ out,
                                                   uint32_t* __restrict__ out_len, int32_t* __restrict__ status, int max_depth, uint32_t upw,
                                                   const uint32_t* __restrict__ retry, const uint64_t* __restrict__ out_off, RunStatus* rs) {
  const uint32_t lane = threadIdx.x & 31;
  if (lane >= upw) return;
  uint32_t u = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * upw + lane;
  if (u >= n_units) return;
  if (retry) {
    if (u >= rs->n_retry || rs->err) return;
    u = retry[u];
  }
  const uint64_t b = offsets[u];
  const uint64_t len64 = offsets[u + 1] - b - 1;
  if (len64 > 0x30000000ull) { status[u] = cfm::MS_UNSUPPORTED; out_len[u] = 0; return; }
  const uint32_t len = (uint32_t)len64;
  cfj::JNode* my = nodes + (b >> 1) + 4ull * u;
  uint32_t* myidx = idx + (b >> 1) + 4ull * u;
  cfj::Big big;
  uint8_t digits[1240];
  cfm::NumWork w{&big, &big, digits, (uint32_t)sizeof(digits)};
  uint8_t* dst = retry ? out + out_off[u] : out + 5 * b + 32ull * u;
  const uint32_t cap = retry ? (uint32_t)(out_off[u + 1] - out_off[u]) : 5 * len + 32;
  uint32_t ol = 0;
  const int st = cfm::mask_process(stream + b, len, my, len / 2 + 4, myidx, len / 2 + 4, dst, cap, &ol, max_depth, w);
  if (retry) {
    if (st != cfm::MS_OK) rs->mask_err = 1;
    return;
  }
  status[u] = st;
  out_len[u] = st == cfm::MS_OK || st == cfm::MS_OVERFLOW ? ol : 0;
}

__global__ void classify_keys_kernel(const uint8_t* __restrict__ stream, const uint64_t* __restrict__ offsets, uint32_t n_units,
                                     uint8_t* __restrict__ sensitive) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const uint64_t b = offsets[u];
  cfj::JNode k{cfj::J_KEY, 0, (uint32_t)(offsets[u + 1] - b - 1), 0};   // raw key text (no JSON escapes)
  sensitive[u] = cfm::key_sensitive(stream + b, k) ? 1 : 0;
}

void cf_launch_toon_seq(uint32_t blocks, cudaStream_t st, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, cfj::JNode* nodes, uint8_t* out,
                        uint32_t* out_len, int32_t* status, uint32_t flags, uint32_t upw) {
  toon_kernel<<<blocks, 64, 0, st>>>(stream, offsets, n_units, nodes, out, out_len, status, flags, upw);
}
void cf_launch_mask_seq(uint32_t blocks, cudaStream_t st, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, cfj::JNode* nodes, uint32_t* idx,
                        uint8_t* out, uint32_t* out_len, int32_t* status, int max_depth, uint32_t upw, const uint32_t* retry, const uint64_t* out_off,
                        RunStatus* rs) {
  mask_kernel<<<blocks, 64, 0, st>>>(stream, offsets, n_units, nodes, idx, out, out_len, status, max_depth, upw, retry, out_off, rs);
}
void cf_launch_classify_keys(uint32_t blocks, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, uint8_t* sensitive) {
  classify_keys_kernel<<<blocks, 128>>>(stream, offsets, n_units, sensitive);
}
