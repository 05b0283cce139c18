/* cfgpu.h — C ABI of libcfgpu.so, the H100 (sm_90a) implementation of ContextForge's plugin
 * hook-chain hot path.  Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * What each entry point replaces in the reference (/root/reference):
 *   cf_builder_add_pattern + cf_compile
 *       -> `re.compile(...)` at plugin construction:
 *          plugins/regex_filter/search_replace.py:67-75,
 *          plugins/harmful_content_detector/harmful_content_detector.py:70-87,
 *          plugins/deny_filter/deny.py:43-46
 *   cf_scan / cf_scan_host
 *       -> the per-string matcher loops:
 *          harmful `_scan_text`  plugins/harmful_content_detector/harmful_content_detector.py:92-107
 *          deny `word in value`  plugins/deny_filter/deny.py:59-60
 *          regex_filter "does any rule match" (dirty detection for cf_sub_host)
 *   cf_sub_host
 *       -> `pattern.sub(replacement, value)` applied rule after rule:
 *          plugins/regex_filter/search_replace.py:127-130,147-155
 *   cf_mask_host
 *       -> `mask_sensitive_json_bytes(payload, max_depth)`:
 *          crates/request_logging_masking_native_extension/src/lib.rs:346-360
 *   cf_toon_host
 *       -> `orjson.loads` + `toon.encode` + "only if smaller" of `_process_content_item`:
 *          plugins/toon_encoder/toon_encoder.py:277-303, plugins/toon_encoder/toon.py:82-565
 *   cf_json_index / cf_json_index_host
 *       -> no single reference function: the shared JSON structural index SURVEY.md §8(f)-2 asks for —
 *          what `orjson.loads` (toon_encoder.py:281), `serde_json::from_slice` (lib.rs:353) and the
 *          string walk `_iter_strings` (harmful_content_detector.py:110-139) each recompute per payload
 *
 *   cf_run_batch / cf_run_enqueue + cf_run_finish
 *       -> the whole per-request plugin chain over one uploaded batch (mcpgateway/services/tool_service.py:5866-5872)
 *
 * Environment (read once per process):
 *   CF_SCAN_RESERVE_SMS=k   the persistent scan grid leaves k SMs free (a collective running beside it needs somewhere to go)
 *   CF_PAIR_FILTER=0|1   force the byte / pair prefilter instead of choosing per rule set (tests, measurements)
 *
 * Conventions: every function returns CF_OK (0) or a negative CF_E_* code and never throws.
 * All buffers are caller-owned.  A cf_ctx belongs to one device; calls on one ctx must be
 * serialised by the caller (the Python host holds one ctx per process/GPU).
 *
 * Packed stream layout (host and device), used by every data entry point:
 *     stream  = unit_0 0xFF unit_1 0xFF ... unit_{n-1} 0xFF      (UTF-8; 0xFF never occurs in UTF-8)
 *     offsets = uint64[n+1]; offsets[i] = start of unit_i; offsets[n] = stream length
 *     unit_i  = stream[offsets[i] .. offsets[i+1]-1)
 */
#ifndef CFGPU_H
#define CFGPU_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CF_OK 0
#define CF_E_CUDA (-1)        /* CUDA runtime/driver error; see cf_last_error */
#define CF_E_BADARG (-2)
#define CF_E_UNSUPPORTED (-3) /* valid pattern the engine cannot express (caller must fail loudly) */
#define CF_E_TOO_LARGE (-4)   /* automaton/state explosion or table limits */
#define CF_E_CAPACITY (-5)    /* caller-provided output buffer too small; required size reported */
#define CF_E_NOGPU (-6)       /* no usable CUDA device */
#define CF_E_NOMEM (-7)

#define CF_PAT_SEARCH 0u   /* existence only (harmful / deny) */
#define CF_PAT_ORDERED 1u  /* regex_filter rule: also build the leftmost-first automaton */

typedef struct cf_builder cf_builder;
typedef struct cf_ctx cf_ctx;
typedef struct cf_prog cf_prog;
typedef struct cf_batch cf_batch;

/* ---------------- program construction (host only; usable without a GPU) ---------------- */
int cf_builder_new(cf_builder** out);
void cf_builder_free(cf_builder* b);
const char* cf_builder_last_error(cf_builder* b);
/* code points that are \w (sorted, disjoint inclusive ranges: lo0 hi0 lo1 hi1 ...) */
int cf_builder_set_word_set(cf_builder* b, const uint32_t* ranges, uint32_t nranges);
/* ast: serialized pattern (see csrc/re_backend.h); returns the pattern's bit index */
int cf_builder_add_pattern(cf_builder* b, const uint32_t* ast, uint32_t nwords, uint32_t flags,
                           uint32_t* out_index);
/* literal replacement bytes (UTF-8) for a CF_PAT_ORDERED pattern */
int cf_builder_set_replacement(cf_builder* b, uint32_t pattern_index, const uint8_t* repl, uint32_t len);
/* replacement TEMPLATE with group references (`re.sub` templates `\\1`, `\\g<name>`, `\\g<0>`; the reference passes the
 * configured `replace` string straight to `pattern.sub`, plugins/regex_filter/search_replace.py:130): `parts` holds n_parts
 * triples {kind, a, b} — kind 0: literal bytes literals[a .. a+b), kind 1: the text of group a (0 = the whole match; a group
 * that did not take part contributes nothing).  The pattern's AST must carry its A_GROUP nodes (csrc/re_backend.h). */
int cf_builder_set_template(cf_builder* b, uint32_t pattern_index, const uint8_t* literals, uint32_t literals_len,
                            const uint32_t* parts, uint32_t n_parts);
/* run the host part of compilation now (idempotent); reports table sizes */
typedef struct cf_compile_stats {
  uint32_t n_patterns, words_per_bitmap, n_classes, n_states, n_accsets, n_ordered;
  uint32_t trans_bytes;
  uint32_t prefilter;   /* 0 = byte filter (5-byte window of per-position byte sets), 1 = pair filter (keyed on byte pairs;
                         * chosen when the byte filter would admit too many windows, i.e. large rule sets) */
} cf_compile_stats;
int cf_builder_compile_host(cf_builder* b, cf_compile_stats* out);

/* ---------------- device context / program ----------------
 * Threading (SURVEY 8(b)): a cf_builder belongs to one thread at a time.  A cf_ctx owns a device, its scratch pools and the default
 * stream's work: calls on ONE cf_ctx must be serialised by the caller (the Python binding holds a lock per context; a gateway
 * worker has one context and one launching thread).  Different cf_ctx objects — one per worker process or per GPU — are
 * independent.  A compiled cf_prog is immutable and may be used by any call of the ctx that compiled it; a cf_batch holds ONE
 * upload at a time.  The asynchronous entry points (cf_scan, cf_toon, cf_run_enqueue) only enqueue on the given stream and
 * return. */
int cf_init(int device_ordinal, cf_ctx** out);
void cf_shutdown(cf_ctx* ctx);
const char* cf_last_error(cf_ctx* ctx);
int cf_compile(cf_ctx* ctx, cf_builder* b, cf_prog** out); /* uploads tables to HBM */
void cf_free_prog(cf_prog* p);
uint32_t cf_prog_words(const cf_prog* p);    /* u64 words per verdict bitmap (W) */
uint32_t cf_prog_patterns(const cf_prog* p);

/* ---------------- batches (device-resident packed streams) ---------------- */
int cf_batch_create(cf_ctx* ctx, uint64_t max_stream_bytes, uint32_t max_units, cf_batch** out);
void cf_batch_free(cf_batch* b);
/* async H2D of a packed stream on `cuda_stream` (cudaStream_t, may be NULL) */
int cf_batch_upload(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes,
                    const uint64_t* offsets, uint32_t n_units, void* cuda_stream);
uint32_t cf_batch_units(const cf_batch* b);
uint64_t cf_batch_bytes(const cf_batch* b);
/* Page-locked host memory for the buffers a caller hands to the *_host / cf_run_batch entry points (packed stream in, produced
 * texts out).  Any host pointer works; a pageable one is copied through the driver's bounce buffer at a fraction of the PCIe rate
 * (measured: 306 MB of TOON text per step, 21 ms pageable vs 6 ms pinned). */
int cf_host_alloc(cf_ctx* ctx, uint64_t bytes, void** out);
void cf_host_free(cf_ctx* ctx, void* p);

/* ---------------- stage 1: multi-pattern scan ---------------- */
/* device-resident: d_bitmaps = device pointer to n_units*W uint64 (may be torch-owned memory) */
int cf_scan(cf_ctx* ctx, cf_prog* p, cf_batch* b, uint64_t* d_bitmaps, void* cuda_stream);
/* host buffers: upload + scan + download, synchronous; h_bitmaps = n_units*W uint64 */
int cf_scan_host(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes,
                 const uint64_t* offsets, uint32_t n_units, uint64_t* h_bitmaps);
/* ---------------- stage 2: regex_filter substitution (units the scan flagged) ---------------- */
/* Applies every CF_PAT_ORDERED rule of `p`, in the order added, to the listed units of the batch
 * that was last uploaded (Python `pattern.sub(replacement, value)` rule after rule,
 * plugins/regex_filter/search_replace.py:127-130).  Rewritten units are returned back to back in
 * out_bytes with out_offsets[n_sel+1]; a unit no rule matched comes back unchanged.
 * There is no limit on the number of rules (the kernel takes 32 per launch and continues each unit in the next launch).
 * CF_E_CAPACITY with *out_needed set when out_cap is too small (CF_E_CAPACITY without it: a unit would grow beyond 4 GB).
 * CF_E_TOO_LARGE when a rule's output outgrows the rules' worst-case growth bound (an internal error; cf_last_error names
 * the unit and the rule).  Synchronous. */
int cf_sub_host(cf_ctx* ctx, cf_prog* p, cf_batch* b, const uint32_t* units, uint32_t n_sel, uint8_t* out_bytes,
                uint64_t out_cap, uint64_t* out_offsets, uint64_t* out_needed);

/* ---------------- stage 3: request_logging_masking ---------------- */
/* mask_sensitive_json_bytes(payload, max_depth) per unit (one JSON request body per unit):
 * crates/request_logging_masking_native_extension/src/lib.rs:346-360.  Masked compact JSON of every
 * unit with status CF_MASK_OK is returned back to back in out_bytes / out_offsets[n+1].
 * status: CF_MASK_OK, CF_MASK_PARSE_ERROR (the crate raises ValueError: invalid JSON, a number out of
 * binary64's range anywhere in the document, nesting deeper than serde_json's 127 levels),
 * CF_MASK_UNSUPPORTED (beyond the device limits: a number literal longer than the 3200-bit workspace, or a
 * body over 768 MiB — the caller must fail loudly).  Outputs of any size are returned. */
#define CF_MASK_OK 0
#define CF_MASK_PARSE_ERROR 2
#define CF_MASK_UNSUPPORTED 6
int cf_mask_host(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets, uint32_t n_units,
                 int max_depth, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, int32_t* status, uint64_t* out_needed);
/* is_sensitive_key(key) for a batch of key names (lib.rs:122-187); sensitive[i] = 0/1.  Used by the
 * object-level entry points mask_sensitive_data / mask_sensitive_headers (lib.rs:307-344). */
int cf_classify_keys_host(cf_ctx* ctx, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets,
                          uint32_t n_units, uint8_t* sensitive);

/* ---------------- JSON structural index (reusable op, SURVEY.md 8(f)-2) ---------------- */
/* Per unit (one JSON text), in text order: the positions of every structural character { } [ ] : , outside
 * strings, every string's opening and closing quote (a quote preceded by an odd-length run of backslashes is
 * not a quote), and the first byte of every other run of non-whitespace bytes outside strings (scalars).
 * Tokens of unit i are tokens[offsets[i] .. offsets[i] + (counts[i] & 0x7FFFFFFF)) — the token buffer is indexed
 * like the stream and needs `stream_bytes` entries; counts[i] bit 31 = the text ends inside a string.
 * With CF_INDEX_CLASSIFY each token also carries `aux`: strings are validated (escapes, strict UTF-8, control
 * characters) and get their emit-time predicates + hash, scalars their kind/flags/length; 0xFFFFFFFF = invalid. */
typedef struct cf_json_token { uint32_t pos; /* byte offset in the unit; bit 31 = closing quote */ uint32_t aux; } cf_json_token;
#define CF_INDEX_CLASSIFY 1u
int cf_json_index(cf_ctx* ctx, cf_batch* b, uint32_t flags, cf_json_token* d_tokens, uint32_t* d_counts, void* cuda_stream);
int cf_json_index_host(cf_ctx* ctx, cf_batch* b, uint32_t flags, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets,
                       uint32_t n_units, cf_json_token* tokens, uint32_t* counts);

/* ---------------- stage 4: toon_encoder (JSON text -> TOON text) ---------------- */
/* Per unit (one JSON text): orjson.loads + toon.encode + "keep only if strictly smaller"
 * (plugins/toon_encoder/toon_encoder.py:277-303, toon.py:82-565).  status[i] is one of CF_TOON_*;
 * when CF_TOON_CONVERTED the TOON text is out_stream[offsets[i] .. offsets[i]+out_len[i]). */
#define CF_TOON_CONVERTED 0
#define CF_TOON_NOT_SMALLER 1   /* TOON would not be smaller: item keeps its JSON */
#define CF_TOON_NOT_JSON 2      /* orjson.JSONDecodeError */
#define CF_TOON_VALUE_ERROR 3   /* toon raises ValueError (un-encodable control character) */
#define CF_TOON_ATTR_ERROR 4    /* toon raises AttributeError (unchecked .keys(), toon.py:400-404) */
#define CF_TOON_UNSUPPORTED 6   /* beyond the device limits (nesting > 64, number > 3200 bits): caller must fail loudly */
#define CF_TOON_REPORT_ERRORS 1u /* flags: keep encoding after the output outgrew the input so that VALUE/ATTR
                                   errors are still reported (needed for skip_on_error=False) */
#define CF_TOON_PARSE_ONLY 4u    /* flags, diagnostic: only parse; status = 0 ok / 1 invalid JSON / 2 beyond limits,
                                  * out_len = DOM node count (used by tools/toon_prof.py to time the parser alone) */
#define CF_TOON_SEQUENTIAL 8u    /* flags, diagnostic: skip the token-parallel kernel (csrc/json_tp.h), run every unit through the
                                  * sequential per-thread encoder (the one that otherwise only takes the units the fast path hands over) */
#define CF_TOON_NO_HANDOVER 16u  /* flags, diagnostic: leave the units the token-parallel kernel does not cover at status 7 with the
                                  * reason (json_tp.h FB_*) in out_len instead of re-doing them with the sequential encoder */
/* device-resident (batch already uploaded); d_out has room for the batch's stream bytes */
int cf_toon(cf_ctx* ctx, cf_batch* b, uint32_t flags, uint8_t* d_out, uint32_t* d_out_len, int32_t* d_status, void* cuda_stream);
/* host buffers: upload + encode + download, synchronous */
int cf_toon_host(cf_ctx* ctx, cf_batch* b, uint32_t flags, const uint8_t* stream, uint64_t stream_bytes, const uint64_t* offsets,
                 uint32_t n_units, uint8_t* out_stream, uint32_t* out_len, int32_t* status);

/* ---------------- the fused chain: ONE upload, every stage on the device-resident batch, one call ---------------- */
/* SURVEY.md 8(b) cf_run_batch: what PluginManager.invoke_hook does plugin after plugin over each payload
 * (mcpgateway/services/tool_service.py:5866-5872) — pattern scans (regex_filter dirty detection + deny + harmful),
 * regex_filter rewriting of the units a rule matched, toon_encoder JSON->TOON — over ONE uploaded packed stream.
 * unit_stages[i] (may be NULL = every stage in stage_mask) selects the stages that apply to unit i.
 * Per unit a 24-byte verdict record; the rewritten / re-encoded texts come back packed in out_bytes with out_offsets[n+1]
 * (a unit without output has out_offsets[i+1] == out_offsets[i]).
 *   CF_STAGE_SCAN  verdict.match_bitmap = word 0 of the unit's pattern bitmap (all W words in bitmaps_full when not NULL)
 *   CF_STAGE_SUB   units with a set CF_PAT_ORDERED bit are rewritten rule after rule (cf_sub_host semantics): CF_V_REWRITTEN.
 *                  Such a unit is NOT TOON-encoded in the same call (the reference would encode the rewritten text): the
 *                  caller re-submits it; flags carry CF_V_RESUBMIT when TOON was requested for it.
 *   CF_STAGE_TOON  verdict.aux = CF_TOON_* status; CF_V_TOON when converted (out = the TOON text)
 * stream == NULL runs the stages on the batch that is ALREADY resident (uploaded by cf_batch_upload or a previous call): bench.py's
 * device-resident `value`; offsets must then be the host copy of that batch's offsets.
 *   CF_STAGE_MASK  request_logging_masking on the same upload (verdict.aux = CF_MASK_* status, out = masked JSON);
 *                  not combinable with CF_STAGE_TOON in one call (both produce the unit's output).  Rewritten texts are not
 *                  returned: a rewritten unit that does not mask keeps its rewritten length in out_len and has no output. */
#define CF_STAGE_SCAN 1u
#define CF_STAGE_SUB 2u
#define CF_STAGE_MASK 4u
#define CF_STAGE_TOON 8u
#define CF_V_REWRITTEN 1u
#define CF_V_TOON 2u
#define CF_V_MASKED 4u
#define CF_V_RESUBMIT 8u
#define CF_TOON_SKIPPED 8       /* status of a unit whose unit_stages excluded CF_STAGE_TOON */
#define CF_RUN_OUTPUTS_RESIDENT 32u /* toon_flags of cf_run_batch: leave the produced texts in HBM — gathered at out_offsets in one device
                                     * buffer (cf_run_batch_device_output), rewritten units included — instead of copying them to out_bytes
                                     * (which may then be NULL).  Verdicts and out_offsets come back as usual; the call returns when the
                                     * device work is done.  For consumers that keep working on the device, and bench.py's `value`. */
typedef struct cf_verdict {
  uint64_t match_bitmap;  /* bit i = pattern i matched (first 64 patterns) */
  uint32_t flags;         /* CF_V_* */
  uint32_t out_len;       /* bytes of this unit in out_bytes */
  int32_t aux;            /* stage status: CF_TOON_* / CF_MASK_* */
  uint32_t reserved;
} cf_verdict;
int cf_run_batch(cf_ctx* ctx, cf_prog* prog /* may be NULL without SCAN/SUB */, cf_batch* b, const uint8_t* stream, uint64_t stream_bytes,
                 const uint64_t* offsets, uint32_t n_units, uint32_t stage_mask, const uint8_t* unit_stages, uint32_t toon_flags, int mask_max_depth,
                 cf_verdict* verdicts, uint64_t* bitmaps_full, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets, uint64_t* out_needed);
/* the device buffer of the last CF_RUN_OUTPUTS_RESIDENT call of this ctx (valid until the next cf_run_batch / *_host call) */
int cf_run_batch_device_output(cf_ctx* ctx, const uint8_t** d_out, uint64_t* bytes);
/* synchronous copy of `bytes` device bytes to a host buffer (for callers without a CUDA runtime binding of their own) */
int cf_copy_to_host(cf_ctx* ctx, void* host_dst, const void* device_src, uint64_t bytes);

/* ---------------- the fused chain on the caller's stream: cf_run_enqueue / cf_run_finish ----------------
 * cf_run_batch's SCAN, SUB and TOON stages without a host round trip between launch and completion: the dirty-unit selection, the
 * substitution's scratch bounds and arena allocation, the verdict records, the output offsets and the gather are decided on the
 * device.  cf_run_batch itself is an upload, one enqueue and one finish on a run the context owns (with CF_STAGE_MASK, the masking
 * kernel after them).
 *
 * A cf_run owns every piece of per-call device state (scan queue, TOON scratch and unit order, the dirty-unit list, the substitution
 * descriptors and arena, per-unit gather sources, a status block, a completion event and a side stream), so runs created on one
 * ctx can be in flight at once on different streams.  Memory of a run: 8 x max_stream_bytes of TOON scratch, max_stream_bytes of
 * TOON output, about 170 bytes per unit, 8 MiB of scan queue and the arena.  (The run cf_run_batch uses borrows the context's TOON
 * workspace instead, the one cf_toon uses, so a context holds one.)
 *
 * cf_run_enqueue: the batch must be resident (cf_batch_upload on the same stream, or ordered before it).  d_verdicts (n_units
 * records), d_out_offsets (n_units + 1), d_out (out_cap bytes), d_bitmaps_full (n_units * W words; required with SCAN or SUB) and
 * d_unit_stages (may be NULL) are caller-owned DEVICE memory (torch tensors work).  Stages: CF_STAGE_SCAN, CF_STAGE_SUB (implies
 * SCAN), CF_STAGE_TOON; CF_STAGE_MASK is CF_E_BADARG (masking keeps cf_run_batch).  Results are cf_run_batch's, unit for unit.
 * Between its first launch and its return the call neither synchronises, allocates nor reads device memory on the host, so it
 * can be captured in a CUDA graph.  Warm the run up with one enqueue + finish first, so that the arena has its size; a replay that
 * needs more defers the units that do not fit, and the graph stays valid: once an enqueue of a run was captured, arenas the run
 * outgrows are kept until cf_run_free.  The batch, the program and every buffer passed in must stay untouched until cf_run_finish
 * returns.  Every check that can fail is made before the first launch, so an error return leaves nothing queued.
 *
 * Deferred units: a dirty unit whose two scratch buffers (first-pass bound min(worst, 64 L + 64 KiB) each, as cf_sub_host) do not fit
 * the arena that is left, or whose rewrite outgrows that bound, gets no output in the enqueue.  cf_run_finish completes it with the
 * synchronous substitution (which regrows its room and reports CF_E_TOO_LARGE), patches its record and redoes offsets and gather.
 *
 * cf_run_finish: waits for the run's last enqueue (or a graph replay of it) and reads its status through the run's own non-blocking
 * stream (it waits for nothing else the caller has queued).  Returns CF_OK; CF_E_CAPACITY only when the gathered texts need
 * *needed > out_cap bytes (verdicts and out_offsets are valid, d_out is untouched); CF_E_TOO_LARGE when a deferred unit's substitution
 * exceeds one of its limits (the worst-case bound, a unit beyond 4 GB, scratch beyond 8 GiB: cf_last_error says which); or another
 * error.  *needed (may be NULL) = bytes of all gathered texts, 0 on any error other than CF_E_CAPACITY.  It grows the arena to what
 * the call asked for, for the next call. */
typedef struct cf_run cf_run;
int cf_run_create(cf_ctx* ctx, uint32_t max_units, uint64_t max_stream_bytes, uint64_t sub_arena_bytes, cf_run** out);
void cf_run_free(cf_run* run);
int cf_run_enqueue(cf_ctx* ctx, cf_prog* prog, cf_batch* b, cf_run* run, uint32_t stage_mask, const uint8_t* d_unit_stages, uint32_t toon_flags,
                   cf_verdict* d_verdicts, uint64_t* d_bitmaps_full, uint64_t* d_out_offsets, uint8_t* d_out, uint64_t out_cap, void* cuda_stream);
int cf_run_finish(cf_ctx* ctx, cf_run* run, uint64_t* needed);

/* number of kernels launched by this ctx so far (for bench.py's gpu_launches) */
uint64_t cf_kernel_launches(const cf_ctx* ctx);

/* per-launch CUDA-event timing of the dominant kernel of each stage (scan_kernel for cf_scan),
 * recorded on the launching stream; used by bench.py for roofline.achieved */
int cf_profile_begin(cf_ctx* ctx, uint32_t max_launches); /* 0 disables */
int cf_profile_collect(cf_ctx* ctx, double* total_ms, uint32_t* n_launches);
/* same, one duration per recorded launch, in launch order (cf_scan and the TOON stage record one pair each); resets the list */
int cf_profile_collect_each(cf_ctx* ctx, double* ms, uint32_t cap, uint32_t* n_launches);

/* device-side counters of the last cf_scan / cf_scan_host scan: [0]=prefilter candidates, [1]=DFA verify steps.  cf_run_enqueue
 * (and cf_run_batch, which runs through it) counts on its run's own pair. */
int cf_scan_counters(cf_ctx* ctx, uint64_t out[2]);

#ifdef __cplusplus
}
#endif
#endif /* CFGPU_H */
