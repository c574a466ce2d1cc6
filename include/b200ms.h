/*
 * b200ms.h -- C-ABI of libb200ms.so: the H100 (sm_90a) implementation of Morphik's ColPali
 * late-interaction (MaxSim) scoring path.  Plain pointers and sizes only; no C++/torch types.
 *
 * Drop-in boundary (reference paths relative to the morphik-core repository root):
 *   The reference has no FFI on this path; its scorers are reached through the Python plugin
 *   interface core/vector_store/base_vector_store.py:7-65 (BaseVectorStore).  The host mirror of that
 *   interface lives in morphik-core_b200/store.py and calls this library through ctypes
 *   (INTEGRATION.md shows the binding).  Each entry point below names what it replaces:
 *
 *   b200ms_sign_pack       <- morphik_rust binary_quantize_batch_packed  (morphik_rust/src/binary_ops.rs:147-222,
 *                             core/utils/fast_ops.py:191-227, called from multi_vector_store.py:329-345)
 *   b200ms_pack_pages      <- store_embeddings' per-page quantise + layout (multi_vector_store.py:681-703;
 *                             fast_multivector_store.py:673-707 writes fp32 .npy; values are bf16-exact :674)
 *   b200ms_set_corpus      <- the table scan source: multi_vector_embeddings rows (multi_vector_store.py:240-251)
 *   b200ms_pack_queries    <- _binary_quantize(query) (multi_vector_store.py:731) / torch.from_numpy(q).float()
 *                             (fast_multivector_store.py:554)
 *   b200ms_score           <- SQL public.max_sim over every row (multi_vector_store.py:287-311,746-763) for
 *                             B200MS_B1, and colpali_engine score_multi_vector (fast_multivector_store.py:553-555)
 *                             for B200MS_BF16; B200MS_I8 is new (BASELINE config 3, SURVEY F5)
 *   b200ms_topk            <- ORDER BY similarity DESC LIMIT k (multi_vector_store.py:759) / torch.topk
 *                             (fast_multivector_store.py:556), plus the WHERE document_id IN (...) filter (:752-757)
 *   b200ms_merge_topk      <- (new) merge of per-GPU-shard top-k lists after the NCCL all-gather (SURVEY 8e)
 *   b200ms_search_host     <- MultiVectorStore.query_similar's scoring section with HOST query buffers
 *                             (multi_vector_store.py:721-763): quantise/convert, scan, top-k, results to host
 *   b200ms_search_device   <- same with device-resident inputs/outputs, asynchronous on the caller's stream
 *
 * Conventions: every function returns 0 on success or a negative B200MS_E* code; b200ms_last_error()
 * returns a message for the last failure on that handle (or the last global failure for NULL).
 * A handle is bound to one CUDA device and is NOT thread-safe: the caller serialises calls per handle
 * (the Python store holds a lock and calls through asyncio.to_thread, SURVEY 8b "Threading").
 * Calls on one handle run on the GPU in the order they were made, whatever streams they name: they share the handle's
 * scratch.  Entry points taking a `stream` enqueue on it; b200ms_search_host*, b200ms_sharded_search_host_begin,
 * b200ms_set_corpus* and b200ms_fde_configure* enqueue on the handle's own stream.  A call on stream B therefore waits
 * for the handle's previous call on stream A to finish on the GPU, and so does the caller's later work on B (one event
 * wait, and one event record per call).  Calls of different handles are not ordered against each other.  A stream that is
 * being captured into a CUDA graph is neither ordered nor recorded: capturing the device entry points is not supported.
 * Device buffers passed in are caller-owned (torch tensors); the library only owns small scratch and the blocks of the "corpus storage" section.
 * There is no CPU fallback: without a CUDA device every compute entry point fails with B200MS_ECUDA.
 */
#ifndef B200MS_H_
#define B200MS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MS_VERSION 200 /* 0.2.0: + multi-GPU entry points (b200ms_comm_*, b200ms_allgather_topk, b200ms_sharded_search_*),
                              b200ms_rerank_batch_device, b200ms_fde_configure_ex, B200MS_F8 corpora, option "zero_pad_compat";
                              options "a_in_tmem" / "split4" / "epi_w4" removed with the kernels they selected;
                              + b200ms_last_scan_stats: a search with an allow mask scans only the pages the mask allows */

/* element types */
#define B200MS_F32 0  /* float32 source rows (ingest / query side only)            */
#define B200MS_BF16 1 /* bfloat16 rows, 256 B per 128-d patch vector                */
#define B200MS_I8 2   /* int8 rows, 128 B per patch vector (global symmetric scale) */
#define B200MS_B1 3   /* sign bits, MSB-first, 16 B per patch vector                */
#define B200MS_I32 4  /* int32 scores (I8 / B1 corpora)                             */
#define B200MS_F8 5   /* fp8 e4m3 rows, 128 B per patch vector (global power-of-two scale), f32 scores */

/* error codes */
#define B200MS_OK 0
#define B200MS_EINVAL (-1) /* bad argument                                  */
#define B200MS_ECUDA (-2)  /* CUDA runtime/driver failure or no device       */
#define B200MS_ESTATE (-3) /* call order violated (e.g. score before corpus) */
#define B200MS_ENOMEM (-4) /* scratch allocation failed                      */

#define B200MS_DIM 128        /* embedding dimension of ColPali / ColQwen patch vectors */
#define B200MS_ROW_GROUP 32   /* pages and queries are padded to multiples of 32 rows   */
#define B200MS_MAX_K 4096     /* largest k accepted by b200ms_topk / b200ms_merge_topk  */
#define B200MS_MAX_PER_DOC 64 /* most pages per document the b200ms_*_docs calls return   */

typedef struct b200ms b200ms_t;

int b200ms_version(void);
/* Number of CUDA devices visible (0 without a driver); never fails. */
int b200ms_device_count(void);
int b200ms_create(int device, b200ms_t** out);
int b200ms_destroy(b200ms_t* h);
const char* b200ms_last_error(const b200ms_t* h);

/* ---- layout helpers (host, pure arithmetic) ------------------------------------------------- */
/* Rows a page of `len` true rows occupies in the padded corpus layout: roundup(len, 32); 0 stays 0. */
int64_t b200ms_padded_len(int64_t len);
/* Sum of b200ms_padded_len over page_lens[0..n_pages). */
int64_t b200ms_padded_rows(const int32_t* page_lens, int64_t n_pages);
/* Bytes per row for a corpus dtype (BF16 256 / I8 and F8 128 / B1 16), or 0. */
int64_t b200ms_row_bytes(int dtype);
/* Number of 32-row query groups for queries of the given lengths: sum ceil(len/32) (a 0-length query -> 0). */
int64_t b200ms_query_groups(const int32_t* q_lens, int n_q);

/* ---- quantise / layout (device) ------------------------------------------------------------- */
/* x: device [rows,128] F32|BF16 -> out: device [rows,16] sign bits, bit = (float32(x) > 0), MSB first. */
int b200ms_sign_pack(b200ms_t* h, const void* x, int src_dtype, int64_t rows, uint8_t* out, void* stream);

/* out[i] = popcount(q_bits XOR cand_bits[i]) for one packed 16-byte query row against n packed candidate rows (device,
 * 16-byte aligned): fast_ops.hamming_distance_batch (core/utils/fast_ops.py:242-248, binary_ops.rs:266-292). */
int b200ms_hamming_batch(b200ms_t* h, const uint8_t* q_bits, const uint8_t* cand_bits, int64_t n, uint32_t* out, void* stream);

/* Convert n_pages pages stored back to back at src (device, [sum len,128] F32|BF16) into the padded
 * corpus layout at dst (device): page i occupies padded_len(len_i) rows, the padding rows repeat the
 * page's last true row byte for byte (max-/min-invariant, so scores are unchanged); a page of length 0 occupies no rows.
 * Per element, for every float32 input (a BF16 source is widened exactly first):
 *   BF16: round-to-nearest-even; subnormals are kept; finite values past the largest bf16 round to +-inf; +-inf stay;
 *         every NaN -> 0x7fff (the canonical bf16 NaN, sign dropped).
 *   I8:   rint(fp32 product x * i8_scale) (ties to even) clamped to [-127,127]; +-inf -> +-127; NaN -> 0 (it has no sign
 *         and no magnitude).
 *   F8:   e4m3 of the fp32 product x * i8_scale (so the product is rounded first, then rounded again to e4m3: use a
 *         power-of-two scale, 64 for unit-norm rows, to make the first rounding exact), round-to-nearest-even, saturating:
 *         |x * i8_scale| > 448 and +-inf -> +-448 (0x7e / 0xfe); -0 and negative values that round to 0 -> 0x80;
 *         every NaN -> 0x7f (sign dropped).
 *   B1:   bit = x > 0, so +-0 and every NaN -> 0, +inf -> 1.
 * page_lens is a HOST array. */
int b200ms_pack_pages(b200ms_t* h, const void* src, int src_dtype, const int32_t* page_lens, int64_t n_pages,
                      void* dst, int dst_dtype, float i8_scale, void* stream);

/* Attach a packed corpus (device memory, caller-owned, must stay valid until the next set_corpus/destroy).
 * rows: [b200ms_padded_rows(page_lens), 128] of dtype BF16|I8|F8|B1, 1024-byte aligned.  page_lens (HOST) are the
 * TRUE lengths.  Builds the chunk->page table, the work-unit plan and the TMA descriptor. */
int b200ms_set_corpus(b200ms_t* h, const void* rows, int dtype, const int32_t* page_lens, int64_t n_pages);
/* ---- host-resident corpus: patch rows in pinned host memory, only the rerank candidates cross PCIe ----------------------
 * Replaces the reference's multivector storage outside the ANN index (load_multivector_from_storage,
 * fast_multivector_store.py:545-548, :713-774): the FDE matrix stays in HBM, the packed rows stay in host RAM.
 * set_corpus_host: same layout and arguments as b200ms_set_corpus, but rows_host is pinned, device-mapped host memory
 *   (b200ms_host_alloc; anything else -> B200MS_EINVAL), 16-byte aligned.  Only b200ms_rerank_device /
 *   b200ms_rerank_batch_device score it: every rerank call dedups the valid candidate pages of the whole call, gathers them
 *   over PCIe into a library-owned HBM staging block (rounds of at most option "host_stage_bytes") and runs the same scorers
 *   on it -- scores, ids, counts and tie order are bit-identical to an HBM corpus of the same rows.  Such a call
 *   synchronises the caller's stream once (one small D2H of the plan) and is never graph-captured.  Full scans
 *   (b200ms_score, b200ms_search_*, b200ms_sharded_search_*) return B200MS_ESTATE.  b200ms_fde_encode_corpus reads a bf16
 *   host corpus through the mapping.
 * host_alloc / host_free: cudaHostAlloc(Mapped | Portable) of exactly `bytes` (the caller owns and frees the block; host_free
 *   also accepts a NULL handle, for a block that outlives its handle).
 * last_gather_stats: of the last host-tier rerank call: unique pages gathered, bytes copied (padded rows x row bytes),
 *   gather rounds, and the device time (ms, CUDA events) of the gather kernels; synchronises. */
int b200ms_set_corpus_host(b200ms_t* h, const void* rows_host, int dtype, const int32_t* page_lens, int64_t n_pages);
int b200ms_host_alloc(b200ms_t* h, int64_t bytes, void** out);
int b200ms_host_free(b200ms_t* h, void* p);
int b200ms_last_gather_stats(b200ms_t* h, int64_t* unique_pages, int64_t* bytes, int* rounds, float* ms);
int64_t b200ms_corpus_pages(const b200ms_t* h);
int64_t b200ms_corpus_rows(const b200ms_t* h);

/* ---- corpus storage: a device buffer that grows without a copy, and compaction in place ------------------------------------
 * Replaces what the reference's stores give for free (Postgres rows and .npy objects take INSERT and DELETE ... WHERE
 * document_id at any fill level, multi_vector_store.py:681-703, :929-933): a live corpus in a cudaMalloc'd buffer needs a
 * second buffer to grow or to drop deleted pages, so it could use less than half of the card.
 *
 * A block is a reserved range of device virtual addresses, owned by the library and backed by physical memory in chunks of
 * B200MS_BLOCK_CHUNK_BYTES (a multiple of the device's allocation granularity; there is no option for it).  Its pointer is
 * ordinary device memory for every entry point here (b200ms_pack_pages, b200ms_set_corpus, the FDE calls) and for torch.
 *   block_create:  reserve max_bytes of address space (no physical memory yet).  The base address is 1024-byte aligned.
 *   block_resize:  make exactly the first roundup(bytes, chunk) bytes of the range backed: maps new chunks behind the mapped
 *     ones, or unmaps chunks from the tail and RELEASES them to the driver.  Bytes that stay mapped keep their contents and
 *     their address.  Ordered like every other call of the handle: a shrink waits for the handle's earlier work before it
 *     unmaps (work the caller enqueued on the range by other means is the caller's to wait for).  Growing compares the bytes
 *     it has to add with cudaMemGetInfo first and returns B200MS_ENOMEM without creating anything when they do not fit; a
 *     chunk that cannot be created all the same gives the same code.  Either way the block is left as it was.
 *   block_ptr / block_mapped_bytes: the base address (constant for the block's life) and the backed bytes; NULL -> NULL / 0.
 *   block_destroy: waits like a shrink, releases everything.  b200ms_destroy releases the blocks the caller forgot.
 * B200MS_EINVAL: a NULL handle, out or block, a negative size, bytes > max_bytes, a block of another handle.
 *
 * compact_rows: move n_runs runs of rows down so that they become contiguous from row 0, in order, inside one buffer:
 *   run i = rows [run_start[i], run_start[i] + run_rows[i]), run_start ascending, runs disjoint (HOST arrays, checked; a run
 *   may be empty).  row_bytes is a multiple of 16 (at most 64 MiB), rows 16-byte aligned.  Source and destination overlap; the
 *   result is byte for byte what copying the runs into a second buffer gives, and rows past the last moved row keep whatever
 *   they held.  Asynchronous on cuda_stream; the only scratch is a library-owned bounce buffer of 64 MiB (allocated by the
 *   first call that needs it), never a second copy of the data: the destination is walked in ascending windows, a window whose
 *   sources all lie past its end is gathered directly, the others go through the bounce buffer. */
#define B200MS_BLOCK_CHUNK_BYTES (32 << 20)
typedef struct b200ms_block b200ms_block_t;
int b200ms_block_create(b200ms_t* h, int64_t max_bytes, b200ms_block_t** out);
int b200ms_block_resize(b200ms_t* h, b200ms_block_t* b, int64_t bytes);
void* b200ms_block_ptr(const b200ms_block_t* b);
int64_t b200ms_block_mapped_bytes(const b200ms_block_t* b);
int b200ms_block_destroy(b200ms_t* h, b200ms_block_t* b);
int b200ms_compact_rows(b200ms_t* h, void* rows, int64_t row_bytes, const int64_t* run_start, const int64_t* run_rows,
                        int64_t n_runs, void* cuda_stream);

/* Pack n_q queries stored back to back at q (device, [sum len,128] F32|BF16) into 32-row groups of the
 * corpus dtype at q_packed (device, capacity >= roundup(groups,4)*32 rows; tail rows are zeroed).
 * group_offsets_out (HOST, [n_q+1]) receives the group range of every query.  Returns group count in
 * *n_groups_out. */
int b200ms_pack_queries(b200ms_t* h, const void* q, int src_dtype, const int32_t* q_lens, int n_q, void* q_packed,
                        int dst_dtype, float i8_scale, int32_t* group_offsets_out, int* n_groups_out, void* stream);

/* ---- the hot path ---------------------------------------------------------------------------- */
/* group_scores[g, p] = sum over the (<=32) true tokens of group g of max over the rows of page p of <q_t, d_r>
 *   BF16 / F8 corpus: float32 (fp32 accumulate on wgmma);  I8: int32 exact;  B1: int32 sum_t max_r (128 - hamming).
 *   (A group holds at most 32 tokens, so its I8 score fits int32; a whole query's sum need not -- see b200ms_topk for the
 *   I32 sum rule every selection and reported score follows.)
 * q_packed: device [roundup(n_groups,4)*32, 128] of the corpus dtype; q_lens/group_offsets (HOST) as produced by
 * b200ms_pack_queries.  With both given, the true tokens of each group are the query's (the zero padding rows of a group
 * add +0).  B1 needs them; for BF16 / I8 / F8 they may be NULL, and then every row of q_packed counts as a token, the zero
 * padding rows included (each adds max_r <0, d_r>: 0 on finite pages, NaN on a page whose rows all hold an infinity).
 * Value rule of BF16 and F8 corpora (the "float value rule"; every entry point that scores them follows it):
 *   - sim(q_t, d_r) is the dot product of the PACKED values (bf16, or e4m3 codes widened exactly to f16), rounded to fp32,
 *     with IEEE non-finite arithmetic: 0 * +-inf = NaN, NaN * x = NaN, +inf + -inf = NaN.  The products are exact and
 *     the finite sum is rounded to fp32: to nearest even in its normal range, past it to +-inf, and into its subnormal
 *     range (below 2^-126) toward zero, to a multiple of 2^-149, as the tensor core rounds there.  The order of the fp32 additions is the tensor core's, so a finite result can differ from the
 *     exactly rounded sum by a few fp32 ulps per term (oracle/scoring.py TOL).
 *   - Measured on an NVIDIA H100 80GB HBM3 (700 W limit; wgmma m64n128k16 .bf16, fp32 accumulate), on every bf16 pattern
 *     and on one-hot products of bf16 patterns and powers of two: subnormal bf16 inputs are used as they are, not flushed;
 *     a product that lands in fp32's subnormal range is kept where it is a multiple of 2^-149 (2^-127 .. 2^-149 exact) and
 *     truncated toward zero otherwise (1.0078 * 2^-150 gives 0, 1.5 * 2^-149 gives 2^-149, where round-to-nearest would
 *     give 2^-149 and 2^-148); a product of 2^128 or more gives +-inf.  A product does not overflow on its own: 2^64 * 2^64 + (-2^64) * 2^64 inside one 16-element MMA
 *     step gives 0, not NaN (partial sums across steps are fp32).  e4m3 products lie in [2^-18, 448^2] and are exact.
 *   - The max over a page's TRUE rows is fmaxf's: a NaN row is ignored unless every row is NaN (then the max is NaN).
 *   - The group score sums the query's true tokens only, so a query's score is the IEEE sum of its tokens' maxima:
 *     NaN if some token's max is NaN or if +inf and -inf meet, else +-inf if one occurs, else finite.
 *   - zero_pad_compat (b200ms_set_option) replaces a clamped page's token max m by fmaxf(m, 0), so a NaN max becomes 0 there;
 *     colpali_engine's torch scorer propagates the NaN instead (torch.max over a row holding a NaN is NaN).
 * Reranks, document searches, host-resident corpora and sharded searches score with this kernel, so the rule holds for
 * them; b200ms_explain_device reports the same per-token values.
 * group_scores: device [n_groups_padded, ld] with ld >= n_pages, n_groups_padded = roundup(n_groups,4).
 * Pages with zero rows score 0 (COALESCE(...,0.0), multi_vector_store.py:308).
 * b200ms_score scans every page.  The search entry points below that take an allow mask (b200ms_search_host*,
 * b200ms_search_device*, b200ms_search_docs_device, b200ms_sharded_search_*) scan only the pages some query of the call may
 * see: the work units of the scan are rebuilt from the masks on the device in every call (the masks may change behind the
 * same pointer), without a synchronisation, and the results are bit for bit those of b200ms_score + b200ms_topk.  A query
 * without a mask in the batch (mask index -1) makes the call scan every page.  Corpora whose scan is a single wave of work
 * units keep the full scan. */
int b200ms_score(b200ms_t* h, const void* q_packed, int n_groups, const int32_t* q_lens, const int32_t* group_offsets,
                 int n_q, void* group_scores, int64_t ld, void* stream);

/* Per query: sum[p] = the group scores group_scores[g, p], g in [group_offsets[q], group_offsets[q+1]), added in order to
 * +0; keep the k best pages whose bit is set in allow_mask (device, bit p&31 of word p>>5; NULL = all; bits at
 * p >= n_pages are ignored), ordered by sum DESC then page id ASC (the reference leaves ties unspecified).  The order is
 * total: -0 ties with +0, every NaN ranks above every number (+inf included) and NaNs tie with each other -- as torch.topk
 * and Postgres ORDER BY ... DESC order them.  Columns p >= n_pages (ld > n_pages) are never read.
 * Sums of score_dtype F32 are float32.  Sums of score_dtype I32 (the "I32 sum rule"): the group scores are added in int64
 * and the sum is clamped to +-(2^31 - 1).  Pages whose clamped sums differ are ranked exactly, also where float32 would
 * merge them; pages whose sums lie beyond the bound tie at it (lower page id first).  An int8 query of 1041 or more tokens
 * (1033 or more against -128 codes) can get there: a token scores at most 128 * 127^2 (128 * 127 * 128).
 * Reported score = float32(sum) * scale in fp32, of the clamped sum for I32 (a NaN as 0x7fffffff).  Outputs are device
 * arrays: top_scores/top_ids [n_q, k] (unused slots: -inf / -1), top_counts [n_q].  id_base is added to every page id
 * (global ids of a shard). */
int b200ms_topk(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                const int32_t* group_offsets, int n_q, const uint32_t* allow_mask, int k, float scale, int64_t id_base,
                float* top_scores, int64_t* top_ids, int32_t* top_counts, void* stream);
/* b200ms_topk with one allow-mask PER QUERY (the FDE first stage of a search whose queries carry different filters):
 * allow_masks_dev [n_masks, ceil(n_pages/32)] and mask_index_dev [n_q] (-1 = unfiltered) are DEVICE arrays, as in
 * b200ms_search_device_masked; n_masks = 0: unfiltered.  Everything else as b200ms_topk. */
int b200ms_topk_masked(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                       const int32_t* group_offsets, int n_q, const uint32_t* allow_masks_dev, int n_masks,
                       const int32_t* mask_index_dev, int k, float scale, int64_t id_base, float* top_scores,
                       int64_t* top_ids, int32_t* top_counts, void* cuda_stream);

/* Merge candidate lists (e.g. the all-gathered per-shard top-k): cand_scores/cand_ids device [n_q, m]
 * (entries with id < 0 are ignored) -> best k by (score DESC, id ASC) in the total order of b200ms_topk (-0 == +0, NaN
 * above every number, NaNs tied); a -0 is reported as +0 and a NaN as 0x7fffffff.  m <= 2*B200MS_MAX_K. */
int b200ms_merge_topk(b200ms_t* h, const float* cand_scores, const int64_t* cand_ids, int n_q, int m, int k,
                      float* top_scores, int64_t* top_ids, int32_t* top_counts, void* stream);

/* Whole query step with HOST buffers (pageable or pinned): q_host [sum q_lens,128] float32.  Copies the
 * queries to the device, packs, scores the attached corpus, selects top-k and copies results back;
 * synchronous.  allow_mask_host may be NULL.  score scale: BF16 1.0; B1 1/128; I8 1/(q_scale*corpus_scale). */
int b200ms_search_host(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                       const uint32_t* allow_mask_host, float i8_q_scale, float score_scale, int64_t id_base,
                       float* top_scores_host, int64_t* top_ids_host, int32_t* top_counts_host);

/* b200ms_search_host with ONE allow-mask PER QUERY: allow_masks_host is a [n_masks, ceil(n_pages/32)] matrix of page
 * bitmasks, mask_index_host[i] the row that filters query i (-1 = unfiltered); n_masks = 0 means no filtering at all.
 * The production caller always passes the requesting user's authorised doc_ids (core/services/document_service.py:408-417),
 * so concurrent query_similar calls carry DIFFERENT filters; with per-query masks they still share one pass over the
 * corpus (four 32-token queries fit one 128-row MMA tile and cost the same as one). */
int b200ms_search_host_masked(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                              const uint32_t* allow_masks_host, int n_masks, const int32_t* mask_index_host,
                              float i8_q_scale, float score_scale, int64_t id_base, float* top_scores_host,
                              int64_t* top_ids_host, int32_t* top_counts_host);

/* Same with everything on the device and no synchronisation (enqueued on `stream`).  q_dev: F32|BF16. */
int b200ms_search_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                         const uint32_t* allow_mask_dev, float i8_q_scale, float score_scale, int64_t id_base,
                         float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);

/* b200ms_search_device with one allow-mask per query: allow_masks_dev [n_masks, ceil(n_pages/32)] and mask_index_dev
 * [n_q] (-1 = unfiltered) are DEVICE arrays (see b200ms_search_host_masked). */
int b200ms_search_device_masked(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                                const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                float i8_q_scale, float score_scale, int64_t id_base, float* top_scores_dev,
                                int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);

/* The searches above rank and report I8 / B1 pages by the I32 sum rule of b200ms_topk, and so do the reranks and document
 * calls below.
 * MaxSim over an explicit candidate list (the "rerank" half of a two-stage search, fast_multivector_store.py:545-557;
 * BF16 / F8 scores follow the float value rule of b200ms_score, so do the rerank and document calls below):
 * cand_ids_dev = device array of n_cand page ids (-1, or any id outside [0, n_pages) = unused slot; a page may appear in
 * several slots).  Only those pages are scanned; ties break towards the earlier candidate slot (= better first-stage rank),
 * for every n_cand.  Outputs as b200ms_search_device. */
int b200ms_rerank_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                         const int64_t* cand_ids_dev, int n_cand, int k, float i8_q_scale, float score_scale,
                         float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);

/* b200ms_rerank_device with one candidate list PER QUERY (the two-stage search of a query batch: every query reranks its own
 * first-stage candidates, fast_multivector_store.py:526-557): cand_ids_dev = device [n_q, n_cand] page ids (-1 = unused slot).
 * One launch per 128-token query tile scores that tile's queries against their own lists only; outputs as above. */
int b200ms_rerank_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                               const int64_t* cand_ids_dev, int n_cand, int k, float i8_q_scale, float score_scale,
                               float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);

/* ---- explaining a match (new; no reference counterpart) ---------------------------------------------------------------
 * Per-token MaxSim breakdown of chosen pages: for query q, page slot j, token t
 *   token_scores[q, j, t] = max over the TRUE rows r of page page_ids[q, j] of sim(q_t, d_r)
 *   best_rows[q, j, t]    = the lowest r attaining that max  (0 <= r < page length)
 *   sim_map[q, j, t, r]   = sim(q_t, d_r) for r < min(page length, map_rows)      (sim_map may be NULL)
 * sim() is the search's own per-token value, in the units of the reported score:
 *   BF16 / F8 fp32 dot (times score_scale), I8 int32 dot (times score_scale), B1 (128 - hamming) (times score_scale).
 * The dense dtypes compute it on the scan's tensor-core instructions in the scan's order, so the map holds the very values the
 * scan took its max over: sum_t token_scores[q, j, t] is the score b200ms_rerank_batch_device reports for that page (for
 * I8 / B1 exactly while the int64 sum of the integer token values lies within +-(2^31 - 1); beyond it the rerank reports
 * the bound, by the I32 sum rule of b200ms_topk; for BF16 / F8 up to the order of the float32 sum over tokens), and
 * token_scores == sim_map at best_rows.
 * q_dev: F32 | BF16 rows [sum q_lens, 128]; q_lens HOST; page_ids_dev device int64 [n_q, n_cand] (-1 or outside
 * [0, n_pages) = unused slot; a page may appear in several slots); t_max = max(q_lens).  Outputs are device arrays:
 *   token_scores / best_rows [n_q, n_cand, t_max], sim_map [n_q, n_cand, t_max, map_rows].
 * Every output entry is written.  For an unused slot, a page with no rows, or a token t >= q_lens[q]: score 0,
 * best row -1, map entries -inf.  Map entries at r >= page length are -inf.
 * Queries are packed exactly as b200ms_search_device packs them (same i8_q_scale, same sign rule).
 * A max over rows is fmaxf's (a NaN only when every row is NaN); a tie, +0 and -0 included, reports the lowest row.
 * BF16 / F8 values follow the float value rule of b200ms_score: their token scores add up, NaN and +-inf included, to the
 * rerank's score, since neither counts a query's padding tokens.
 * Host-resident corpora: the named pages are gathered like a rerank's candidates (b200ms_last_gather_stats reports the call)
 * and the outputs are bit-identical to an HBM corpus of the same rows.
 * Option "zero_pad_compat" is ignored: maps are over true rows only.
 * B200MS_EINVAL: NULL or inconsistent arguments, a negative query length, map_rows < 0, n_q * n_cand >= 2^30;
 * B200MS_ESTATE: no corpus attached. */
int b200ms_explain_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                          const int64_t* page_ids_dev, int n_cand, float i8_q_scale, float score_scale,
                          float* token_scores, int32_t* best_rows, float* sim_map, int64_t map_rows, void* stream);

/* ---- grouping results by document (new; no reference counterpart) -------------------------------------------------------
 * The top k DOCUMENTS instead of the top k pages, for callers that want documents: DocumentService.retrieve_docs
 * (core/services/document_service.py:819-851) asks for k chunks and keeps the best chunk per document
 * (_create_document_results, :1759-1763), so a long document whose pages all match fills every slot by itself.
 * page_doc: device int32 [n_pages] (indexed by page id, candidate mode too), the document ordinal of every page; a page
 * whose value is outside [0, n_docs) is never returned (the table is not validated: holes are safe).
 * For query q let L be the flat ranking of the eligible pages in b200ms_topk's order (a page is eligible when its allow bit
 * is set, if a mask is given, and its page_doc is in range).  The result is
 *   - documents in the order of their first page in L, at most k of them;
 *   - for each, its first per_doc pages in L (a document with fewer eligible pages returns fewer);
 *   - every score bit for bit the score the flat call reports for that page (BF16 / F8: the float value rule of
 *     b200ms_score); a document's score is its first page's.
 * Candidate mode: L ranks q's valid slots (id in [0, n_pages)) by score DESC then slot ASC; a page that occupies several
 * slots counts once, at its earliest slot.  With n_docs == n_pages, page_doc[p] == p and per_doc == 1 the result equals
 * the flat call's.  Outputs are device arrays:
 *   doc_page_scores float32 [n_q, k, per_doc] (unused: -inf), doc_page_ids int64 [n_q, k, per_doc] (page id + id_base;
 *   unused: -1), doc_page_counts int32 [n_q, k] (unused documents: 0), doc_counts int32 [n_q].
 * B200MS_EINVAL: NULL outputs or page_doc, k outside [1, 4096], per_doc outside [1, B200MS_MAX_PER_DOC], n_docs < 1 while
 * pages exist, n_docs > n_pages, and the per-call bounds of the flat call;  B200MS_ESTATE: as the flat call (no corpus; a
 * full scan of a host-resident corpus).  Nothing is launched when a call is refused. */
/* over a score matrix, like b200ms_topk (group_offsets HOST, one allow mask or NULL; I32 sums by its I32 sum rule) */
int b200ms_topk_docs(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                     const int32_t* group_offsets, int n_q, const uint32_t* allow_mask, const int32_t* page_doc, int64_t n_docs,
                     int k, int per_doc, float scale, int64_t id_base, float* doc_page_scores, int64_t* doc_page_ids,
                     int32_t* doc_page_counts, int32_t* doc_counts, void* stream);
/* full scan, masks as b200ms_search_device_masked (n_masks = 0: unfiltered) */
int b200ms_search_docs_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k, int per_doc,
                              const int32_t* page_doc, int64_t n_docs, const uint32_t* allow_masks_dev, int n_masks,
                              const int32_t* mask_index_dev, float i8_q_scale, float score_scale, int64_t id_base,
                              float* doc_page_scores, int64_t* doc_page_ids, int32_t* doc_page_counts, int32_t* doc_counts,
                              void* stream);
/* per-query candidate lists, as b200ms_rerank_batch_device */
int b200ms_rerank_docs_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                    const int64_t* cand_ids_dev, int n_cand, int k, int per_doc, const int32_t* page_doc,
                                    int64_t n_docs, float i8_q_scale, float score_scale, float* doc_page_scores,
                                    int64_t* doc_page_ids, int32_t* doc_page_counts, int32_t* doc_counts, void* stream);

/* ---- documents ranked by document-level MaxSim (new; extends the document grouping above) ------------------------------
 * DocumentService.retrieve_docs (_create_document_results, core/services/document_service.py:1759-1763) and
 * b200ms_search_docs_device rank a document by its best page, so a query whose tokens are answered on different pages of
 * one document scores as a partial match everywhere.  These calls score a document as one bag of patch vectors:
 *   S(q, D) = sum over q's true tokens t of M[t, D],   M[t, D] = max over D's counted pages p of m[t, p],
 * m[t, p] being the per-token maximum the scan computes (b200ms_explain_device's token score; 1-bit: with the token's
 * constant).  Float maxima follow fmaxf (a NaN token max loses to any number; -0 ranks below +0), integers the integer
 * max; B[t, D], the page holding M[t, D], is the lower page on a tie.  The M[t, D] are added exactly as a page's token
 * maxima are (the group tree of b200ms_score, then the groups in order; I32 by the I32 sum rule), so a one-page document
 * scores bit for bit its page's b200ms_search_device score.  A page counts when its allow bit is set (masks as
 * b200ms_search_device_masked), its page_doc is in [0, n_docs) and it has rows; a document without a counted page is not
 * returned, so a query may find fewer than k.  Documents are ranked in b200ms_topk's order of S (ties: lower document
 * ordinal).  S only grows with a document's pages: long documents are favoured by definition, and nothing normalises it.
 * zero_pad_compat does not apply.  A query without tokens finds no document.
 * Evidence: for each returned document, its distinct pages B[t, D], each with its share (the M[t, D] it holds, added in
 * token order), largest share first (the order of b200ms_topk's keys; ties: lower page), at most per_doc of them.  I32
 * shares add up to S exactly, float shares within rounding.
 * Outputs (device; unused entries -inf / -1 / 0): doc_scores float32 [n_q, k] (S * score_scale), doc_ids int64 [n_q, k]
 * (document ordinals), page_ids int64 [n_q, k, per_doc] (page id + id_base), page_shares float32 [n_q, k, per_doc] (share *
 * score_scale), page_counts int32 [n_q, k], doc_counts int32 [n_q].
 * Cost: one scan of the counted pages, plus a token table of 8 B x padded query tokens x n_docs in the handle's scratch.  A
 * batch whose table passes 1 GiB runs as several passes of whole queries; a query that alone passes it, or has more than
 * 8192 tokens, is refused with B200MS_EINVAL.  B200MS_EINVAL also for bad arguments as b200ms_search_docs_device;
 * B200MS_ESTATE without a corpus or for a host-resident corpus (every page of a document is read).  Nothing is launched
 * when a call is refused.  Asynchronous on cuda_stream, in the handle's call order (a call on another stream waits
 * for the handle's previous call). */
/* full scan */
int b200ms_search_doc_maxsim_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                                    int per_doc, const int32_t* page_doc, int64_t n_docs, const uint32_t* allow_masks_dev,
                                    int n_masks, const int32_t* mask_index_dev, float i8_q_scale, float score_scale,
                                    int64_t id_base, float* doc_scores, int64_t* doc_ids, int64_t* page_ids,
                                    float* page_shares, int32_t* page_counts, int32_t* doc_counts, void* cuda_stream);
/* two-stage: cand_ids_dev int64 [n_q, n_cand] (-1 = unused slot) are query q's first-stage pages; q is scored over every
 * counted page of their documents (the masks still apply) */
int b200ms_rerank_doc_maxsim_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                          const int64_t* cand_ids_dev, int n_cand, int k, int per_doc, const int32_t* page_doc,
                                          int64_t n_docs, const uint32_t* allow_masks_dev, int n_masks,
                                          const int32_t* mask_index_dev, float i8_q_scale, float score_scale, int64_t id_base,
                                          float* doc_scores, int64_t* doc_ids, int64_t* page_ids, float* page_shares,
                                          int32_t* page_counts, int32_t* doc_counts, void* cuda_stream);

/* ---- diversifying results (new; no reference counterpart) ---------------------------------------------------------------
 * Maximal marginal relevance (MMR) over each query's candidate list: near-copies of a page picked already (a re-uploaded
 * deck, a repeated slide template, the same figure on two pages) give way to pages that add something.  The call needs no
 * query rows: relevance comes from the scores a search already reported, so it follows every search path (full scan,
 * filtered scans, both first stages of the two-stage search, host-resident corpora).
 * Per query q (cand_ids / cand_scores device [n_q, n_cand], as every search and rerank returns them; q_lens HOST):
 *   rel_j  = cand_scores[q, j] / q_lens[q] in fp32 (a mean per query token); q_lens[q] == 0: rel_j = cand_scores[q, j].
 *   sim(j -> s) = fp32(fp32(S) * score_scale) / len_j, every step rounded to fp32, where S = sum over the TRUE rows r of
 *     page j of the max over the TRUE rows r' of page s of dot(j_r, s_r') -- how much of page j page s covers (directional).
 *     The dot is the scan's per-row value on the packed rows (BF16: fp32 wgmma of bf16; F8: e4m3 widened to f16, fp32;
 *     I8: exact s8 dot; B1: 128 - hamming) and the float value rule of b200ms_score holds for BF16 / F8 (max by fmaxf over
 *     true rows, IEEE non-finite arithmetic).  S is an fp32 sum for BF16 / F8 (each 64-row tile of page j summed in row
 *     order, the tiles added in order) and an exact int64 for I8 / B1 (1041 rows at +-127 pass int32).  score_scale is the
 *     one the search reported its scores with (BF16 1, I8 / F8 1/scale^2, B1 1/128), so sim and rel share units.  A page
 *     without rows, on either side, gives sim = 0.
 *   red_j  = fmaxf over the pages picked so far of sim(j -> pick) (a NaN only when every one is NaN).
 *   Pick 1 is the best slot by rel; every later pick the best live slot by
 *     v_j = __fsub_rn(__fmul_rn(lambda_mult, rel_j), __fmul_rn(__fsub_rn(1, lambda_mult), red_j))
 *   in the total order of b200ms_topk (-0 == +0, NaN above every number, NaNs tied), ties to the lower slot.  With
 *   lambda_mult == 1, v_j = rel_j and red is never read (0 * inf cannot make a NaN): the result is the candidates in rel
 *   order, which for a search's own list is its order.
 *   Slots: an id of -1 or outside [0, n_pages) is unused and never picked; a page in several slots counts once, at its
 *   earliest slot (the rule of b200ms_rerank_docs_batch_device).  count = min(k, distinct valid candidates).
 * Outputs (device): out_ids int64 [n_q, k] in pick order, out_scores float32 [n_q, k] (each pick's cand_scores entry bit
 * for bit), out_counts int32 [n_q]; unused entries -1 / -inf.  sims (NULL or float32 [n_q, k, n_cand]): sims[q, i, j] =
 * sim(slot j -> pick i) for every slot j still unpicked after pick i (why a page was demoted, and by which pick); -inf for
 * unused and repeated slots, for pick i itself and the picks before it, and for i >= count.
 * Launches on cuda_stream, without a host synchronisation on an HBM corpus: a setup kernel, then two kernels per further
 * pick (min(k, n_cand) picks at most), and two more for the last row of sims when it is asked for; lambda_mult == 1 without
 * sims is the setup kernel alone.  Option "zero_pad_compat" is ignored.
 * Host-resident corpora: the call's unique candidate pages are gathered once (b200ms_last_gather_stats reports it; the call
 * synchronises cuda_stream), and the results are bit-identical to an HBM corpus of the same rows.  Every pair must be
 * resident together, so a call whose unique candidate pages need more than one gather round (option "host_stage_bytes")
 * is refused with B200MS_EINVAL.
 * B200MS_EINVAL: NULL arguments, lambda_mult NaN or outside [0, 1], score_scale not finite and > 0, k < 1, n_cand outside
 * [1, B200MS_MAX_K], n_q < 1, a negative query length, n_q * n_cand >= 2^30, the host-tier round rule above;
 * B200MS_ESTATE: no corpus attached.  Nothing is launched when a call is refused. */
int b200ms_mmr_device(b200ms_t* h, const int64_t* cand_ids, const float* cand_scores, int n_cand, const int32_t* q_lens,
                      int n_q, int k, float lambda_mult, float score_scale, int64_t* out_ids, float* out_scores,
                      int32_t* out_counts, float* sims, void* cuda_stream);

/* ---- searching with stored pages as the queries (new; no reference counterpart) -------------------------------------------
 * "Pages like this one": DocumentService.retrieve_chunks(query_image=...) (core/services/document_service.py:193, 278-286)
 * embeds a query image as a page-length query; a page that is already stored is the same kind of query, and its packed rows
 * are already here.  These calls take source page ids (HOST int64 [n_src], each in [0, n_pages); anything else is
 * B200MS_EINVAL) and use each page's packed rows as one query, copied as stored -- BF16 rows, I8 codes at the corpus scale,
 * F8 e4m3 codes, B1 sign rows -- with no dequantise / requantise round trip: query q has the page's TRUE row count as its
 * length, padding rows never count, and the value rule of b200ms_score holds unchanged.  A host-resident corpus's source
 * rows are read through the mapping (one PCIe read of the named pages, as b200ms_fde_encode_corpus).
 *   search_pages_device: the full scan of b200ms_search_device_masked for these queries -- the same packing layout, work
 *     units (filtered scans included), b200ms_topk selection, I32 sum rule, tie and NaN order -- with one allow-mask row per
 *     source (allow_masks_dev [n_masks, ceil(n_pages/32)], mask_index_dev [n_src], -1 = unfiltered; n_masks = 0: none).
 *     Masks are the only filter: excluding the source itself, or its document, is a mask bit the caller clears.  Host-resident
 *     corpora: B200MS_ESTATE (use a first stage and rerank_pages_batch_device).
 *   rerank_pages_batch_device: b200ms_rerank_batch_device for these queries over cand_ids_dev [n_src, n_cand] (-1 = unused
 *     slot), tie order by slot as there; a candidate whose page the source's mask row forbids is an unused slot.  Works on
 *     host-resident corpora: the candidates are gathered exactly as b200ms_rerank_batch_device gathers them
 *     (b200ms_last_gather_stats reports them; the source rows are not part of the gather).
 *   Reported score (both): the normalised page-to-page MaxSim on the scale of b200ms_mmr_device's sim(source -> page),
 *     __fdiv_rn(float32(sum) * score_scale, len) with len the source's true row count: the score b200ms_search_device would
 *     report for the source's rows (dequantised: bf16 values, e4m3 values / scale, int8 codes / scale, +-1 for sign bits) divided by
 *     len, so that one number means the same across sources of different lengths.  A NaN stays as reported (0x7fffffff).
 *     score_scale as for the search (BF16 1, I8 / F8 1/scale^2, B1 1/128): the library does not know a quantised corpus's
 *     scale.  I8: the sum follows the I32 sum rule of b200ms_topk -- a row scores at most 128 * 128 * 128 = 2^21 (-128 codes
 *     against -128 rows), so a source of 1024 rows can pass 2^31 - 1 (1033 rows of +-127 codes against -128 rows, 1041
 *     against +-127 rows); such pages are clamped to the bound and tie there, lower page id (slot) first.
 *     A source page with zero rows gets count 0 (every slot -inf / -1).  zero_pad_compat does not apply: its clamp belongs
 *     to the reference's query-vs-page batching, and b200ms_mmr_device's sim has none either.
 *   page_rows_device: the true rows of the source pages back to back into out (device float32 [sum of their lengths, 128]),
 *     each element the packed value widened exactly (bf16; int8 code; e4m3 value; sign bit as +1 / -1) times scale in fp32 --
 *     the float query a first stage (b200ms_fde_encode, b200ms_sign_candidates_device) takes, with scale = 1/corpus scale for
 *     I8 / F8 corpora.
 * B200MS_EINVAL: n_src < 1, a source id outside [0, n_pages) (a page compacted away no longer exists), k outside [1, 4096],
 * NULL outputs, n_masks > 0 without masks and index, n_cand < 1 or n_src * n_cand >= 2^30;  B200MS_ESTATE: no corpus, a
 * full search_pages_device of a host-resident corpus.  Nothing is launched when a call is refused. */
int b200ms_search_pages_device(b200ms_t* h, const int64_t* src_pages_host, int n_src, int k, const uint32_t* allow_masks_dev,
                               int n_masks, const int32_t* mask_index_dev, float score_scale, int64_t id_base,
                               float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* cuda_stream);
int b200ms_rerank_pages_batch_device(b200ms_t* h, const int64_t* src_pages_host, int n_src, const int64_t* cand_ids_dev,
                                     int n_cand, int k, const uint32_t* allow_masks_dev, int n_masks,
                                     const int32_t* mask_index_dev, float score_scale, float* top_scores_dev,
                                     int64_t* top_ids_dev, int32_t* top_counts_dev, void* cuda_stream);
int b200ms_page_rows_device(b200ms_t* h, const int64_t* src_pages_host, int n_src, float scale, float* out, void* cuda_stream);

/* ---- relevance feedback: liked and disliked examples, one fused score (new; no reference counterpart) ---------------------
 * "More like these, less like that": a REQUEST has one or more weighted EXAMPLES, and pages rank by the weighted sum of their
 * scores against every example, all examples of all requests scored in ONE pass over the corpus (or the candidates).
 *   Examples (HOST arrays): n_qe query embeddings first -- rows of q_dev (F32 or BF16, [sum q_lens, 128], as
 *   b200ms_search_device_masked) of q_lens[i] tokens -- then n_src stored pages src_pages_host[j] in [0, n_pages), packed as
 *   b200ms_search_pages_device packs them.  Example i (query examples first, then pages) belongs to request ex_req_host[i] in
 *   [0, n_req) and carries the weight ex_weight_host[i]: finite and != 0, > 0 for "like", < 0 for "unlike".  Every request
 *   needs at least one example of positive weight.
 *   Example score s_e(p): __fdiv_rn(float32(finish_sum(sum of its group scores)) * score_scale, len) -- for a page example
 *     exactly what b200ms_search_pages_device reports (len = its true rows), for a query example b200ms_search_device's score
 *     over its token count (len = T): the mean MaxSim per query row.  I8 / B1: each example's sum follows the I32 sum rule of
 *     b200ms_topk on its own (an int64 sum clamped to +-(2^31 - 1)); the fusion happens after that clamp.  An example of zero
 *     rows or tokens adds no term (a request whose examples all have none scores 0 on every page).
 *   Fused score: acc = 0.0f; for each example e of the request, in example order: acc = __fadd_rn(acc, __fmul_rn(w_e,
 *     s_e(p))) -- no FMA contraction, so numpy float32 reproduces it bit for bit.  The fused rows go through the selection of
 *     b200ms_topk (one group per request, F32, scale 1): its keys, ties towards the lower page (candidate mode: the lower
 *     slot), its NaN order, id_base.  One allow-mask row per REQUEST (allow_masks_dev [n_masks, ceil(n_pages/32)],
 *     mask_index_dev [n_req], -1 = unfiltered; n_masks = 0: none).  Example pages are returned like any other page: a caller
 *     who does not want them clears their bits in the request's mask row.  zero_pad_compat does not apply.
 *   search_examples_device: the full scan (filtered scans included: the pages some request's mask row allows).  Host-resident
 *     corpora: B200MS_ESTATE (use a first stage, union_candidates_device and rerank_examples_batch_device).
 *   rerank_examples_batch_device: over one candidate list per request, cand_ids_dev [n_req, n_cand] (-1 = unused slot);
 *     every example of request r scores r's list, a candidate r's mask row forbids is an unused slot, and the outputs are
 *     [n_req, k] as b200ms_rerank_batch_device's.  Works on host-resident corpora: the candidates are gathered once per
 *     distinct page, exactly as b200ms_rerank_batch_device gathers them (b200ms_last_gather_stats).
 * B200MS_EINVAL: no example, n_req < 1, a request without a positive example, a zero or non-finite weight, ex_req outside
 * [0, n_req), a page id outside [0, n_pages), a negative query length, a query example without F32 / BF16 rows, k outside
 * [1, 4096], NULL outputs, n_masks > 0 without masks and index, n_cand < 1 or (n_req + examples) * n_cand >= 2^30;
 * B200MS_ESTATE: no corpus, a full search_examples_device of a host-resident corpus.  Nothing is launched when a call is
 * refused.
 *   union_candidates_device: the union of first-stage lists, for the rerank above.  Request r owns rows list_off_host[r] ..
 *     list_off_host[r+1] of cand_ids_dev [n_lists, n_cand] (list_off_host [n_req+1] rising from 0 to n_lists); out_dev
 *     [n_req, width] gets r's distinct ids (>= 0; negative ids are unused slots) in first-occurrence order, row-major over
 *     its lists, then -1.  A union of more than width ids keeps the first width.  One CTA per request, deterministic, no
 *     host synchronisation.  B200MS_EINVAL: n_req < 1, n_cand < 1, width < 1, n_lists * n_cand >= 2^30, a bad list_off, NULL
 *     arrays. */
int b200ms_search_examples_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_qe,
                                  const int64_t* src_pages_host, int n_src, const int32_t* ex_req_host,
                                  const float* ex_weight_host, int n_req, int k, const uint32_t* allow_masks_dev, int n_masks,
                                  const int32_t* mask_index_dev, float i8_q_scale, float score_scale, int64_t id_base,
                                  float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* cuda_stream);
int b200ms_rerank_examples_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_qe,
                                        const int64_t* src_pages_host, int n_src, const int32_t* ex_req_host,
                                        const float* ex_weight_host, int n_req, const int64_t* cand_ids_dev, int n_cand,
                                        int k, const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                        float i8_q_scale, float score_scale, float* top_scores_dev, int64_t* top_ids_dev,
                                        int32_t* top_counts_dev, void* cuda_stream);
int b200ms_union_candidates_device(b200ms_t* h, const int64_t* cand_ids_dev, int n_lists, int n_cand,
                                   const int32_t* list_off_host, int n_req, int64_t* out_dev, int width, void* cuda_stream);

/* ---- near-duplicate pages (new; no reference counterpart) -------------------------------------------------------------
 * A workspace fills with copies (a PDF uploaded twice, v3 and v4 of a report, a deck's repeated template pages), and a search
 * then spends its top-k on copies of one page.  These calls compute the duplicate relation as a page -> group table that
 * b200ms_search_docs_device / b200ms_rerank_docs_batch_device take as page_doc with per_doc = 1.
 *   pair_maxsim_device: for each pair i (device int64 pair_a_dev / pair_b_dev [n_pairs], page ids of the attached corpus)
 *     sim_ab_dev[i] = sim(a -> b) and sim_ba_dev[i] = sim(b -> a), float32, where sim(j -> s) is exactly b200ms_mmr_device's
 *     sim: the rows, dot, max rule, summation order (each 64-row block of j in row order, the blocks in order; exact int64 for
 *     I8 / B1) and __fdiv_rn(__fmul_rn(S, score_scale), len_j) -- bit for bit.  sim(b -> a) sums b's column maxima in the
 *     same order, in 64-row blocks of b.  Both come from ONE tensor-core product per pair (dense dtypes: a's 64-row blocks
 *     as the A operand, b's 128-row tiles as B; the epilogue takes row maxima and, over b's true rows, column maxima; 1-bit
 *     corpora: 128 - popc on the CUDA cores).  Maxima commute, so the values do not depend on the schedule.  A page without
 *     rows gives 0 both ways; an id outside [0, n_pages) gives NaN both ways.  Pairs may repeat and may be (a, a).  Pages of
 *     any length work: column maxima of a page past 2048 rows go to per-CTA scratch in the handle.  One CTA per pair in a
 *     grid-stride loop on cuda_stream, no host synchronisation.
 *   duplicate_groups_device: a pair is an EDGE when sim_ab >= threshold and sim_ba >= threshold (the smaller direction; a
 *     NaN never is one), both ids lie in [0, n_pages), a != b, and allow_mask_dev (uint32 page words, NULL = every page) has
 *     both pages.  labels_dev (device int64 [n_pages]) gets, for every allowed page, the smallest page of its connected
 *     component, and -1 for a page the mask excludes (the grouped top-k treats it as a deleted page): a group is never
 *     joined through a page the mask hides.  On the GPU, as a lock-free union-find rather than rounds of min-label hooking
 *     and pointer jumping repeated until nothing changes: one pass hooks each edge's larger root onto its smaller root with
 *     a CAS and retries while the two roots differ.  Every retry of one edge follows the hooking of a root it had found,
 *     and each root is hooked once, so each edge retries at most n_pages - 1 times (the bound is per edge; several edges
 *     can fail on the same hook).  Labels only decrease (atomicMin, also in the path halving of every root search), so no
 *     racing write moves a page back down its path; a second pass points every page at its root.  The result is the unique
 *     minimum label of each component whatever the schedule.  Three launches on cuda_stream, no host synchronisation, no
 *     iteration count to bound.
 *   Neither call suggests a threshold: none has been measured on real ColPali pages.
 * B200MS_EINVAL: n_pairs < 0, NULL arrays with n_pairs > 0, score_scale not finite and > 0, a non-finite threshold, NULL
 * labels_dev;  B200MS_ESTATE: no corpus, a host-resident corpus (both pages of a pair are read from HBM), a corpus dtype
 * without a scorer.  Nothing is launched when a call is refused. */
int b200ms_pair_maxsim_device(b200ms_t* h, const int64_t* pair_a_dev, const int64_t* pair_b_dev, int64_t n_pairs,
                              float score_scale, float* sim_ab_dev, float* sim_ba_dev, void* cuda_stream);
int b200ms_duplicate_groups_device(b200ms_t* h, const int64_t* pair_a_dev, const int64_t* pair_b_dev,
                                   const float* sim_ab_dev, const float* sim_ba_dev, int64_t n_pairs, float threshold,
                                   const uint32_t* allow_mask_dev, int64_t* labels_dev, void* cuda_stream);

/* ---- multi-GPU: document shards, one NCCL all-gather of top-k lists (SURVEY 8e; new relative to the reference) -------------
 * One process per GPU; every rank owns a handle over its shard.  NCCL is bound at run time (dlopen libnccl.so.2, or the
 * path in B200MS_NCCL_LIB); b200ms_comm_available() says whether that worked.
 *   rank 0: b200ms_comm_unique_id(id) -> ship the 128 bytes to every rank by any means (file, socket, MPI, torch) ->
 *   every rank: b200ms_comm_init(h, id, rank, world)      (collective; creates the handle's own communicator)
 *   or b200ms_comm_adopt(h, ncclComm_t, rank, world) to use a communicator the host already has.
 * Exchange layout of one rank's list ("xchg"): [n_q*k int64 global page ids][n_q*k float32 scores] padded to a multiple of
 * 16 bytes = b200ms_xchg_bytes(n_q,k) bytes (so that every rank's block of the gathered buffer is 8-byte aligned), unused
 * entries id -1 / score -inf -- b200ms_search_device can write it in place (top_ids_dev = xchg,
 * top_scores_dev = xchg + n_q*k*8). */
int b200ms_comm_available(void);
int b200ms_comm_unique_id(uint8_t* id128);
int b200ms_comm_init(b200ms_t* h, const uint8_t* id128, int rank, int world);
int b200ms_comm_adopt(b200ms_t* h, void* nccl_comm, int rank, int world);
int b200ms_comm_destroy(b200ms_t* h);
int b200ms_comm_rank(const b200ms_t* h);
int b200ms_comm_world(const b200ms_t* h);
int64_t b200ms_xchg_bytes(int n_q, int k);
/* ncclBroadcast of a device buffer from `root` (e.g. the query rows of a batch) on `stream`. */
int b200ms_bcast_device(b200ms_t* h, void* buf, int64_t bytes, int root, void* stream);
/* ncclSend / ncclRecv of a device buffer to / from rank `peer` (e.g. ingest rows from the coordinating rank to the owner). */
int b200ms_send_device(b200ms_t* h, const void* buf, int64_t bytes, int peer, void* stream);
int b200ms_recv_device(b200ms_t* h, void* buf, int64_t bytes, int peer, void* stream);
/* The one collective of the path: all-gather every rank's xchg block (nccl_comm NULL = the handle's communicator) and merge
 * the world*k candidates per query -> identical top-k on every rank (score DESC, id ASC).  world * k <= 8192. */
int b200ms_allgather_topk(b200ms_t* h, void* nccl_comm, const void* xchg_local_dev, int n_q, int k, float* top_scores_dev,
                          int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);
/* Pipelined sharded search.  _begin enqueues the local scan + top-k (global ids = id_base + local page) on `stream` and the
 * all-gather + merge on the handle's communication stream behind an event, then returns a ticket (>= 0; negative = error);
 * the caller's stream is NOT made to wait for the other ranks, so the next _begin may follow at once (two exchange slots: at
 * most two searches in flight).  The local scores follow the float value rule of b200ms_score.  _end makes `stream` wait for that ticket's merged result in the output buffers given to
 * _begin.  Masks as in b200ms_search_device_masked (n_masks = 0: unfiltered).  Works with world == 1 (no collective). */
int64_t b200ms_sharded_search_begin(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                                    const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                    float i8_q_scale, float score_scale, int64_t id_base, float* top_scores_dev,
                                    int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream);
int b200ms_sharded_search_end(b200ms_t* h, int64_t ticket, void* stream);
/* The same pipeline with HOST query rows (pinned or pageable float32) and host results: _host_begin copies the rows to the
 * device on the handle's stream and returns at once; _host_end blocks until that ticket's merged top-k has been copied back
 * and stores it in the caller's arrays.  Collect ticket t before beginning t+2. */
int64_t b200ms_sharded_search_host_begin(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                                         const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                         float i8_q_scale, float score_scale, int64_t id_base);
int b200ms_sharded_search_host_end(b200ms_t* h, int64_t ticket, float* top_scores_host, int64_t* top_ids_host,
                                   int32_t* top_counts_host);

/* ---- fixed-dimensional encodings (MUVERA FDE): candidate generation in front of the scorer ---------------------------
 * Replaces the `fixed_dimensional_encoding` C++ extension (fast_multivector_store.py:325-331,447-449,521) and the
 * Turbopuffer ANN over its output (:526-532) with an exact encoder and an exhaustive cosine scan.
 * configure: reps repetitions x 2^ksim SimHash partitions x proj_dim AMS-sketch dims = fde_dim floats per item.
 *   simhash [reps,128,ksim] Gaussian, ams_index [reps,128] in [0,proj_dim), ams_sign [reps,128] = +-1 (HOST arrays).
 *   Needs 1 <= reps <= 65535, 1 <= ksim <= 8, 1 <= proj_dim <= 64, proj_dim * 2^ksim <= 512 and a multiple of 8.  Every
 *   argument is checked before anything is uploaded: a call that returns B200MS_EINVAL leaves the previous configuration
 *   in force.
 * encode: items stored back to back at rows (device F32|BF16, [sum len,128]); is_document 0: SUM per partition (query),
 *   1: AVERAGE per partition, empty partition -> 0 (document); out device float32 [n_items, fde_dim].
 * finalize: fp32 FDEs -> bf16 rows of the FDE corpus + 1/||row||.
 * scan: scores[q,p] = <q_fde[q], F[p]> * inv_norm[p]  (cosine ranking);  feed to b200ms_topk (score dtype F32,
 *   group_offsets = 0..n_q) to get the candidate list. */
int b200ms_fde_configure(b200ms_t* h, int reps, int ksim, int proj_dim, float scale, const float* simhash,
                         const int32_t* ams_index, const float* ams_sign);
/* configure + the upstream knobs the reference leaves at their defaults (fast_multivector_store.py:325-331 sets neither):
 *   fill_empty_partitions != 0: an empty document partition takes the projection of the point whose SimHash sign bits are
 *     nearest (Hamming distance, first minimum) instead of zeros;
 *   final_dim > 0: a final count sketch of the whole encoding, out[j] = sum_{i: final_index[i]==j} final_sign[i] * v[i]
 *     (final_index / final_sign: HOST arrays of reps*2^ksim*proj_dim entries; final_dim a multiple of 8) -- fde_dim becomes
 *     final_dim.  The matrices are INPUTS: a caller that holds the upstream extension's matrices passes them here and gets
 *     encodings interchangeable with vectors already stored by the reference. */
int b200ms_fde_configure_ex(b200ms_t* h, int reps, int ksim, int proj_dim, float scale, const float* simhash,
                            const int32_t* ams_index, const float* ams_sign, int fill_empty_partitions, int final_dim,
                            const int32_t* final_index, const float* final_sign);
int64_t b200ms_fde_dim(const b200ms_t* h);
int b200ms_fde_encode(b200ms_t* h, const void* rows, int src_dtype, const int32_t* item_lens, int64_t n_items,
                      int is_document, float* out, void* stream);
/* Document FDEs of pages [first_page, first_page + n_pages) of the attached BF16 corpus, computed from its packed rows
 * (rebuilds the FDE matrix of a corpus loaded from a shard file; at most 65535 pages per call). */
int b200ms_fde_encode_corpus(b200ms_t* h, int64_t first_page, int64_t n_pages, float* out, void* stream);
int b200ms_fde_finalize(b200ms_t* h, const float* fde, int64_t n, void* out_rows, float* inv_norm, void* stream);
int b200ms_fde_scan(b200ms_t* h, const void* fde_rows, const float* inv_norm, int64_t n_pages, const float* q_fde, int n_q,
                    float* scores, int64_t ld, void* stream);

/* ---- sign candidates: asymmetric 1-bit MaxSim over an HBM sign copy of the corpus (new; no reference counterpart) --------
 * A first stage for a two-stage search besides the FDE scan: full-precision queries against the sign bits of every page,
 * then b200ms_rerank_batch_device / b200ms_rerank_docs_batch_device over the candidates.  A sign row is 16 B per patch
 * vector (1/16 of bf16), so the signs of a host-resident corpus many times the size of HBM fit in HBM and are scanned
 * exhaustively; only the candidates cross PCIe.
 *   sign_rows: the sign rows of pages [first_page, first_page + n_pages) of the attached BF16 / I8 / F8 corpus into out
 *     (device, padded rows page_start[first_page] .. page_start[first_page + n_pages], 16 B each, MSB first -- the layout of
 *     a B1 corpus; padding rows repeat the page's last true row).  Bit i of row r = element i of the PACKED row r > 0:
 *     BF16 > +0 (+-0 and NaN give 0), I8 > 0, F8 e4m3 sign clear and magnitude nonzero (NaN 0x7f gives 0).  Signs come from
 *     the packed values, not the float source, so a corpus loaded from a shard file gets the signs of the live one; in I8 /
 *     F8 corpora values that quantised to 0 give 0.  Host-resident rows are read through the mapping (one PCIe read of the
 *     named pages).  B200MS_ESTATE: no corpus, or a B1 corpus (it has no more precise rows to rerank with).
 *   set_sign_rows: attach caller-owned device sign rows (16-byte aligned, n_rows == b200ms_corpus_rows) for the corpus
 *     attached now; every b200ms_set_corpus* detaches them.  A host-resident corpus gets its work units, chunk table and
 *     scan-plan scratch here, on cuda_stream.  B200MS_ESTATE: no corpus, or a B1 corpus.
 *   sign_candidates_device: per query q (q_dev F32 | BF16 rows [sum q_lens, 128], q_lens HOST)
 *       q8 = clamp(rint(fp32(x * i8_q_scale)), -63, 63) per element (ties to even; NaN -> 0, +-inf -> +-63),
 *       S[q, p] = sum over the query's tokens t of max over the TRUE rows r of page p of sum_i q8[t,i] * (bit(r,i) ? +1 : -1),
 *     an exact int32 (a page without rows scores 0, a query without tokens scores 0 everywhere); the candidates are the
 *     n_cand best pages by S among those q's mask allows, in b200ms_topk's order (S DESC, page id ASC), reported score
 *     float32(S) * score_scale.  Outputs (device) cand_scores / cand_ids [n_q, n_cand] (unused: -inf / -1), cand_counts
 *     [n_q]: the candidate layout b200ms_rerank_batch_device takes.  Masks as b200ms_search_device_masked (n_masks = 0:
 *     unfiltered); only the allowed pages are scanned, without a synchronisation.  Works on host-resident corpora.
 *     B200MS_EINVAL: src dtype, n_q < 1, a negative query length, n_cand outside [1, B200MS_MAX_K], i8_q_scale not finite
 *     and > 0, NULL outputs, n_masks > 0 without masks and index;  B200MS_ESTATE: no corpus, or no sign rows attached to it.
 * Nothing is launched when a call is refused. */
int b200ms_sign_rows(b200ms_t* h, int64_t first_page, int64_t n_pages, uint8_t* out, void* cuda_stream);
int b200ms_set_sign_rows(b200ms_t* h, const void* sign_rows, int64_t n_rows, void* cuda_stream);
int b200ms_sign_candidates_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int n_cand,
                                  const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev, float i8_q_scale,
                                  float score_scale, float* cand_scores, int64_t* cand_ids, int32_t* cand_counts,
                                  void* cuda_stream);

/* ---- instrumentation ------------------------------------------------------------------------- */
/* Kernels launched by this handle since creation (bench.py's gpu_launches claim). */
int64_t b200ms_launch_count(const b200ms_t* h);
/* Device time (ms, CUDA events on the launching stream) of the last b200ms_score call's scoring kernels only;
 * synchronises.  Returns a negative error code on failure. */
float b200ms_last_score_ms(b200ms_t* h);
/* Number of scoring calls (b200ms_score or search) recorded so far, and the device times (ms) of the most recent n of
 * them (n <= 256, oldest first; synchronises; returns n or a negative error).  bench.py derives the roofline's
 * `achieved` from these: CUDA events on the launching stream, recorded inside the timed region. */
int64_t b200ms_score_call_count(const b200ms_t* h);
int b200ms_score_times_ms(b200ms_t* h, float* out_ms, int n);
/* Work units and padded rows walked by the handle's last full scan (b200ms_score or a search without candidates): those of
 * the whole corpus, or of the allowed pages when the search scanned a filtered plan; synchronises with that call. */
int b200ms_last_scan_stats(b200ms_t* h, int64_t* units, int64_t* rows);
/* Tuning knobs (0 keeps the default): rows per work unit, CTAs to launch. */
int b200ms_set_tuning(b200ms_t* h, int64_t unit_rows, int max_ctas);
/* Named options:
 *   "b1_tensor"       full scans of 1-bit corpora: 1 = wgmma kernel with in-kernel bit expansion, 0 = POPC kernel, 2 (default)
 *                     = POPC for one or two 32-token query groups, wgmma for three or more (same results bit for bit)
 *   "zero_pad_compat" N > 0: reproduce colpali_engine score_multi_vector's zero-padding quirk with batch size N (128 upstream,
 *                     processing_colpali.py:350-362): a page shorter than the longest page of its batch scores
 *                     sum_t max(max_r <q_t,d_r>, 0).  Rerank calls batch the candidates in first-stage order (exactly the
 *                     reference, fast_multivector_store.py:553-555); full scans batch pages in page-id order.  0 = clean MaxSim
 *                     (default).  Float and int8 corpora only -- SQL max_sim has no padding.
 *   "zero_copy"       1 (default): host entry points move small calls (<= 256 query rows) through mapped pinned memory
 *   "host_graph"      1 (default): small unmasked host searches (pack -> score -> top-k) are captured into a CUDA graph on their
 *                     second use and replayed as one launch; 0 = three plain launches (same results)
 *   "fde_gemm"        1 (default): FDE scan on wgmma when fde_dim % 64 == 0, 0 = SIMT scan
 *   "unit_rows", "max_ctas"   work-unit size (needs a new b200ms_set_corpus) and launch width.
 *   "host_stage_bytes" host-resident corpora: HBM staging budget of one gather round (default 2 GiB, raised to the largest
 *                     page); a rerank call whose unique candidate pages need more runs in rounds (same results). */
int b200ms_set_option(b200ms_t* h, const char* name, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* B200MS_H_ */
