// cf_internal.h — objects shared by the translation units of libcfgpu.so (cfgpu.cu: contexts, batches, scan / substitution
// kernels; cfjson.cu: the JSON kernels — structural index, TOON, masking).  Not part of the ABI (include/cfgpu.h is).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "cf_host.h"
#include "scan_core.h"

// ------------------------------------------------------------------------------------------------
// host-side objects
// ------------------------------------------------------------------------------------------------
// scan_kernel's geometry: 16 warps of 32 lanes, each lane scanning 64 contiguous bytes of a 32 KiB tile (DESIGN §6 has the
// measurement behind these values).  A tile is one TMA box of 128-byte rows.
static const uint32_t SCAN_WARPS = 16;
static const uint32_t SCAN_LANE_BYTES = 64;
static const uint32_t SCAN_TILE = SCAN_WARPS * 32 * SCAN_LANE_BYTES;
static const uint32_t SCAN_BOX_ROWS = SCAN_TILE / 128;
static_assert(SCAN_BOX_ROWS <= 256, "a scan tile must fit one TMA box (at most 256 rows)");
// padding granularity of a batch's buffer: the stream is followed by 0xFF up to a multiple of MAX_TILE plus one more MAX_TILE,
// so the scan's last tile stays inside the allocation (other kernels may read into the padding too)
static const uint32_t MAX_TILE = 64 * 1024;
static_assert(MAX_TILE >= SCAN_TILE, "the padding must cover at least one scan tile");

struct cf_ctx {
  int device = 0;
  int sm_count = 0;
  std::string err;
  uint64_t launches = 0;
  uint64_t* d_qstate = nullptr;     // two {candidates appended, verify steps} pairs, used alternately
  uint32_t qphase = 0;
  uint64_t* d_queue = nullptr;      // candidate start positions
  uint32_t qcap = 1u << 20;
  // grow-only device scratch of the synchronous entry points (cf_dev_reserve: no cudaMalloc per call), freed with the context
  struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { cudaFree(p); }
  };
  // cf_sub_device (cf_sub_host, and cf_run_finish's deferred units): the rewritten texts, a pass's descriptors (soff | bound | sel),
  // its records and the Pike VM's capture words
  DevBuf sub_scratch, sub_desc, sub_rec, sub_pike;
  DevBuf sub_out_offsets, sub_out;  // cf_sub_host's gather of the rewritten texts
  DevBuf verdicts, unit_stages;     // cf_run_batch with host buffers: verdict records, per-unit stage masks on the way in
  // the gather of cf_run_batch (and so of cf_toon_host and cf_mask_host): out offsets and the gathered texts, which no call outlives,
  // except `gathered` after a CF_RUN_OUTPUTS_RESIDENT call: cf_run_batch_device_output hands it out until cf_run_batch runs again
  DevBuf out_offsets, gathered;
  DevBuf bitmaps;                   // pattern bitmaps of cf_scan_host and cf_run_batch, or cf_classify_keys_host's flags
  DevBuf d_tok, d_ntok;             // structural index of the current batch (json_index_kernel)
  void* h_stage = nullptr;          // pinned host staging for gathered results
  size_t h_stage_bytes = 0;
  const uint8_t* run_out = nullptr;   // device buffer of the last CF_RUN_OUTPUTS_RESIDENT call
  uint64_t run_out_bytes = 0;
  cf_run* run = nullptr;              // the run of cf_run_batch, cf_toon and cf_toon_host (ctx_run in cfjson.cu), grown with the batches
  // optional per-launch timing of the dominant kernel (bench.py roofline): event pairs
  std::vector<cudaEvent_t> prof_ev;
  uint32_t prof_used = 0;
  bool prof_on = false;
  uint32_t scan_reserve_sms = 0;   // CF_SCAN_RESERVE_SMS: SMs the persistent scan grid leaves free
};

// the figures of an ordered rule that bound its output's growth (cf_sub_device's `worst`)
struct RuleGrowth { uint32_t minlen, repl_len, n_parts, nrefs, lit_len; };

struct DevDfa {
  cf::DfaTables t;
  std::vector<void*> allocs;
  uint64_t trans_bytes = 0, acc_bytes = 0, stage_bytes = 0;   // sizes for staging in shared memory
};

struct cf_prog {
  cf_ctx* ctx = nullptr;
  uint32_t npat = 0, W = 1;
  DevDfa search;
  uint32_t* d_E = nullptr;         // byte prefilter E[256], or the pair prefilter's T[PF_SLOTS] when use_pairs
  bool use_pairs = false;
  uint64_t* d_always = nullptr;
  bool any_always = false;
  bool search_empty = false;       // every pattern is "always" -> no automaton work at all
  std::vector<DevDfa> ordered;
  std::vector<uint32_t*> d_ordered_E;
  std::vector<int> ordered_pat;    // pattern index of each ordered rule
  std::vector<uint8_t*> d_repl;
  std::vector<uint32_t> repl_len;
  std::vector<uint32_t> ordered_minlen;   // minimum match length (code points) of each ordered rule
  struct RuleTmpl {                       // replacement template with group references (n_parts == 0: literal replacement)
    uint32_t *d_code = nullptr, *d_sets = nullptr, *d_parts = nullptr;
    uint32_t ninst = 0, wpc = 1, nslots = 2, n_parts = 0, nrefs = 0, lit_len = 0;
  };
  std::vector<RuleTmpl> tmpl;             // per ordered rule
  std::vector<RuleGrowth> growth;         // per ordered rule: the figures of the scratch bound (host and device copy; cf_run_enqueue
  RuleGrowth* d_growth = nullptr;         // computes the bound on the device)
  uint64_t* d_rule_mask = nullptr;        // W words: the bits of the CF_PAT_ORDERED patterns
  uint32_t pike_words = 0;                // Pike-VM scratch words per unit of the largest template rule (0: no template rule)
  std::vector<uint64_t> h_offsets;        // host copy of the last batch's offsets (cf_sub_host sizing)
  const void* h_offsets_owner = nullptr;
  uint64_t h_offsets_gen = 0;
};

struct cf_batch {
  cf_ctx* ctx = nullptr;
  uint8_t* d_buf = nullptr;        // FRONT_PAD + stream + tail pad
  uint64_t* d_offsets = nullptr;
  uint32_t* d_coarse = nullptr;    // unit index at every 4 KiB of stream (built on upload, or on the device by a pack)
  std::vector<uint32_t> h_coarse;
  uint64_t cap_bytes = 0;
  uint32_t cap_units = 0;
  uint64_t nbytes = 0;
  uint32_t n = 0;
  uint64_t generation = 0;         // serial of the current upload, unique in the process (0 = none yet): a batch allocated
                                   // at a freed batch's address never repeats its (address, generation) cache key
  CUtensorMap tmap;                // 2-D view of d_buf: rows of 128 B, box = one scan tile, SWIZZLE_128B
};


#define CF_CUDA(ctx, call)                                                                  \
  do {                                                                                      \
    cudaError_t e_ = (call);                                                                \
    if (e_ != cudaSuccess) {                                                                \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                      \
      return CF_E_CUDA;                                                                     \
    }                                                                                       \
  } while (0)


// grow-only device / pinned-host scratch of the *_host entry points (defined in cfjson.cu)
int cf_dev_reserve(cf_ctx* ctx, cf_ctx::DevBuf& b, size_t need);
int cf_stage_reserve(cf_ctx* ctx, size_t need);

// regex_filter substitution of the selected units on stream `st` (cfgpu.cu); the rewritten texts stay on the device.  Unit units[i]
// ends as rec[2i+1] bytes at ctx->sub_scratch.p + rec[2i], or as the unit itself in the batch's stream when rec[2i] == ~0 (no rule
// changed it).  h_offsets: host copy of the batch's offsets (scratch sizing); h_stage: pinned, cf_sub_stage_bytes(n_sel) bytes, and
// *rec points into it.  Returns with the work on `st` done.  Of the context's device buffers only sub_scratch, sub_desc, sub_rec and
// sub_pike are written.
size_t cf_sub_stage_bytes(uint32_t n_sel);
int cf_sub_device(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint64_t* h_offsets, const uint32_t* units, uint32_t n_sel, cudaStream_t st,
                  uint8_t* h_stage, const uint64_t** rec);

static const uint64_t SUB_OVERFLOW = ~1ull;     // record[0] of a unit whose output outgrew its scratch bound (record[1] = the rule)

// ---- cf_run (include/cfgpu.h): the state of one asynchronous chain
// device status block of a run, zeroed at the start of every enqueue
struct RunStatus {
  int32_t err;            // CF_E_CAPACITY when the gathered texts exceed out_cap (the gather is skipped)
  uint32_t n_sel;         // dirty units the enqueue rewrites (selection list length)
  uint32_t n_deferred;    // dirty units left to cf_run_finish
  uint32_t n_retry;       // masked units that outgrew the first pass's room (retry list length)
  uint64_t needed;        // bytes of all gathered texts
  uint64_t arena_used;    // substitution arena bytes the dirty units asked for (fitting or not)
  int32_t mask_err;       // a retried unit did not mask into the exact length its first pass asked for
  uint32_t pad;
};
static const uint32_t RUN_NOT_DIRTY = 0xFFFFFFFFu;    // slot[u]: the unit is not rewritten
static const uint32_t RUN_DEFER_PENDING = 0xFFFFFFFEu;  // ... dirty, did not fit the arena
static const uint32_t RUN_DEFER = 0x80000000u;        // ... deferred, RUN_DEFER | index in the deferred list; otherwise the selection index

struct cf_run {
  cf_ctx* ctx = nullptr;
  uint32_t max_units = 0;
  uint64_t max_bytes = 0;
  std::vector<void*> allocs;
  cudaStream_t side = nullptr;                          // the substitution, beside TOON
  cudaEvent_t ev_scan = nullptr, ev_sub = nullptr, ev_done = nullptr;
  uint64_t* d_queue = nullptr;                          // scan candidate queue and its counters
  uint64_t* d_qstate = nullptr;
  uint32_t qphase = 0;
  void* d_toon_scratch = nullptr;                       // TOON workspace (run_reserve_toon): token / DOM scratch, unit order and its sort
  uint64_t toon_scratch_bytes = 0;
  uint32_t* d_toon_order = nullptr;
  uint8_t* d_toon_sort = nullptr;
  size_t toon_sort_bytes = 0;
  uint8_t* d_toon_out = nullptr;                        // TOON texts in the input's layout
  uint32_t* d_toon_ls = nullptr;                        // TOON (or masking) lengths [n] | statuses [n]
  // masking (cf_run_set_mask): the parser's nodes are the TOON scratch; TOON and masking never share an enqueue
  uint8_t* d_mask_arena = nullptr;                      // first pass: unit u masks into 5 len + 32 bytes at 5 offsets[u] + 32 u
  uint64_t mask_arena_bytes = 0;
  uint32_t* d_mask_retry = nullptr;                     // units that outgrew their room (RunStatus::n_retry of them)
  uint32_t* d_mask_idx = nullptr;                       // the parser's node index
  uint64_t mask_idx_bytes = 0;
  int mask_depth = 0;
  uint32_t* d_slot = nullptr;                           // per unit: RUN_NOT_DIRTY / selection index / RUN_DEFER*
  uint32_t* d_sel = nullptr;                            // per selection index: unit, scratch offset, bound, record
  uint64_t *d_soff = nullptr, *d_bound = nullptr, *d_rec = nullptr;
  uint8_t* d_arena = nullptr;
  uint64_t arena_bytes = 0;
  bool ever_captured = false;                           // an enqueue was captured in a CUDA graph: arenas it may use are kept
  std::vector<void*> retired;                           // ... here, until cf_run_free
  uint8_t* enq_arena = nullptr;                         // the arena the last enqueue (or the graph replaying it) rewrote into
  uint32_t* d_deferred = nullptr;                       // deferred units; d_def_rec: their records after cf_run_finish
  uint64_t* d_def_rec = nullptr;
  uint64_t* d_src = nullptr;                            // per unit: device address of its produced text
  uint64_t* d_len = nullptr;                            // per unit: its length, [n] = 0 (scanned into out_offsets)
  void* d_scan_tmp = nullptr;
  size_t scan_tmp_bytes = 0;
  RunStatus* d_status = nullptr;
  RunStatus* h_status = nullptr;                        // pinned
  // the last enqueue
  cf_prog* prog = nullptr;
  cf_batch* batch = nullptr;
  cudaStream_t st = nullptr;
  uint32_t stage_mask = 0;
  const uint8_t* d_unit_stages = nullptr;
  cf_verdict* d_verdicts = nullptr;
  const uint64_t* d_bitmaps = nullptr;
  uint32_t W = 1;
  bool sub = false;                                     // the substitution ran (d_slot is valid)
  uint64_t* d_out_offsets = nullptr;
  uint8_t* d_out = nullptr;
  uint64_t out_cap = 0;
};

// out[at, at + n) = s[0, n) by the 32 lanes of one warp (gather_kernel, pack_copy_kernel).  16-byte stores; 16-byte loads when source
// and destination share their alignment, otherwise aligned 4-byte loads funnel-shifted into place.  Every word loaded holds at least
// one byte of the source span, so no load leaves the span's 4-byte-aligned envelope; every store stays inside out[at, at + n).
// (The destination is passed as base and offset: that way gather_kernel compiles to the same SASS as with the copy written inline.)
__device__ __forceinline__ void warp_copy_span(uint8_t* out, uint64_t at, const uint8_t* s, uint64_t n, uint32_t lane) {
  uint8_t* d = out + at;
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

// the scan of cf_scan on a given candidate queue / counter pair (cfgpu.cu)
int cf_scan_launch(cf_ctx* ctx, cf_prog* p, cf_batch* b, uint64_t* d_bitmaps, cudaStream_t st, uint64_t* queue, uint64_t* qstate, uint32_t* qphase);
// cf_init's share of cfjson.cu: allows toon_tp_kernel its dynamic shared memory on the current device
cudaError_t cf_toon_tp_allow_smem();
// cf_run_enqueue's substitution on `st` (cfgpu.cu): dirty-unit selection, bounds and arena allocation, then the sub_kernel launches
int cf_sub_enqueue(cf_ctx* ctx, cf_prog* p, cf_batch* b, cf_run* run, const uint64_t* d_bitmaps, const uint8_t* d_unit_stages, cudaStream_t st);

// sequential JSON kernels (cfjson_seq.cu)
namespace cfj { struct JNode; }
static const int CF_TS_FALLBACK = 7;                   // == cftp::TS_FALLBACK (json_tp.h): unit handed to the sequential encoder
static const uint32_t TOON_ONLY_FALLBACK = 0x100u;     // internal flag of toon_kernel: only units with status TS_FALLBACK
void cf_launch_toon_seq(uint32_t blocks, cudaStream_t st, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, cfj::JNode* nodes, uint8_t* out,
                        uint32_t* out_len, int32_t* status, uint32_t flags, uint32_t upw);
void cf_launch_mask_seq(uint32_t blocks, cudaStream_t st, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, cfj::JNode* nodes, uint32_t* idx,
                        uint8_t* out, uint32_t* out_len, int32_t* status, int max_depth, uint32_t upw, const uint32_t* retry, const uint64_t* out_off,
                        RunStatus* rs);
void cf_launch_classify_keys(uint32_t blocks, const uint8_t* stream, const uint64_t* offsets, uint32_t n_units, uint8_t* sensitive);
