// common.cuh -- handle layout, error plumbing and kernel-launcher prototypes shared by the .cu files.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200ms.h"

namespace bms {

constexpr int kDim = B200MS_DIM;
constexpr int kGroup = B200MS_ROW_GROUP;  // 32 rows: padding granule of pages and queries ("chunk")
constexpr int kTileN = 128;               // patch rows per MMA tile (4 chunks)
constexpr int kTileM = 128;               // query rows per MMA tile (4 groups)

struct DeviceBuf {  // grow-only device scratch
  void* p = nullptr;
  size_t cap = 0;
};
struct PinnedBuf {  // grow-only pinned + device-mapped host block (cudaHostAlloc)
  void* p = nullptr;
  size_t cap = 0;
};
struct DeviceGuard {  // switch to the handle's device for the duration of a call
  int prev = -1;
  explicit DeviceGuard(int dev);
  ~DeviceGuard();
};
struct Comm;  // comm.cu: NCCL communicator + the exchange pipeline of the sharded search

// query groups rounded up to whole 128-row MMA tiles: the row count of a packed query block and of a group-score matrix
inline int64_t groups_padded(int64_t groups) { return (groups + 3) & ~int64_t(3); }

// Candidate list(s) of a search (ids: device int64, -1 = unused slot).
//   ids == NULL           : scan the whole corpus, scores indexed by page id.
//   ids, per_query == 0   : ONE list of n_cand page ids scored by every query, scores indexed by slot.
//   ids, per_query == 1   : one list PER QUERY laid out as [n_q, stride()]: query q owns slots [q*stride, q*stride + n_cand)
//                           and only its own groups are scored against them.
struct CandSpec {
  const int64_t* ids = nullptr;
  int n_cand = 0;
  int per_query = 0;
  int64_t stride() const { return per_query ? (int64_t(n_cand) + 31) & ~int64_t(31) : 0; }
  int64_t n_slots(int n_q) const { return per_query ? stride() * n_q : n_cand; }
};

// Layout of n items (queries, or pages) of lens[i] rows, each padded to whole 32-row groups, as ONE host block that is
// uploaded with one copy or read in place from mapped pinned memory:
//   [ss int64 (n+1) true-row offsets | ds int64 (n+1) padded-row offsets | goff int32 (n+1) group offsets, 16 B aligned |
//    ntok int32 (groups_padded, at least 4) true tokens per group]
// Without groups (pages) the block ends after ds.
struct SearchMeta {
  std::vector<uint8_t> host;
  size_t off_ds = 0, off_goff = 0, off_ntok = 0;  // ss is at offset 0
  int64_t n = 0, rows = 0, padded_rows = 0, groups = 0, groups_padded = 0;
  const int32_t* goff() const { return reinterpret_cast<const int32_t*>(host.data() + off_goff); }
};
// NULL lens or n < 0 give the empty layout (search_core rejects such a request)
SearchMeta build_search_meta(const int32_t* lens, int64_t n, bool with_groups = true);
// true tokens of every group: item i's lens[i] tokens fill groups [goff[i], goff[i+1]) 32 at a time; groups at or past
// n_groups are skipped
void group_tokens(const int32_t* lens, int64_t n, const int32_t* goff, int64_t n_groups, int32_t* ntok);

// Grouping a search's results by document (topk_docs.cu): page_doc int32 [n_pages] (device) maps a page to its document
// ordinal; pages with a value outside [0, n_docs) are never returned.  Outputs (device): scores / ids [n_q, k, per_doc],
// page_counts [n_q, k], doc_counts [n_q].
struct DocSpec {
  const int32_t* page_doc = nullptr;
  int64_t n_docs = 0;
  int per_doc = 1;
  float* scores = nullptr;
  int64_t* ids = nullptr;
  int32_t* page_counts = nullptr;
  int32_t* doc_counts = nullptr;
};

// Document mode of the wgmma scan (doc_maxsim.cu): instead of group scores, every true token row t (32 * group + token) of
// the call keeps table[t, d] = max over the scanned pages p of document d of (token max key << 32 | ~p).  A page counts
// when page_doc[p] is in [0, n_docs) and allow (NULL = all; else row mask_index[group_query[group]], -1 = all, rows
// mask_stride words apart) has its bit.
struct DocScan {
  unsigned long long* table = nullptr;
  int64_t n_docs = 0;
  const int32_t* page_doc = nullptr;
  const int32_t* group_query = nullptr;
  const uint32_t* allow = nullptr;
  const int32_t* mask_index = nullptr;
  int64_t mask_stride = 0;
};

// A document-level MaxSim call (doc_maxsim.cu).  q / q_lens / masks as SearchRequest (n_masks rows; mask_index per query);
// cand != NULL: per-query candidate page lists [n_q, n_cand] whose documents are scored.  Outputs (device): doc_scores /
// doc_ids [n_q, k], ev_scores / ev_ids [n_q, k, per_doc], ev_counts [n_q, k], doc_counts [n_q].
struct DocMaxSimCall {
  const void* q = nullptr;
  int q_dtype = B200MS_F32;
  const int32_t* q_lens = nullptr;  // HOST
  int n_q = 0, k = 0, per_doc = 1;
  const int32_t* page_doc = nullptr;
  int64_t n_docs = 0;
  const uint32_t* allow = nullptr;
  int n_masks = 0;
  const int32_t* mask_index = nullptr;
  const int64_t* cand = nullptr;
  int n_cand = 0;
  float i8_q_scale = 1.f, score_scale = 1.f;
  int64_t id_base = 0;
  float* doc_scores = nullptr;
  int64_t* doc_ids = nullptr;
  float* ev_scores = nullptr;
  int64_t* ev_ids = nullptr;
  int32_t* ev_counts = nullptr;
  int32_t* doc_counts = nullptr;
};
// Largest token table (8 B x padded query tokens x n_docs) one pass of a document-level call builds, and the longest query
// it takes (the evidence kernel holds a query's token maxima in shared memory)
constexpr int64_t kDocTableBytes = int64_t(1) << 30;
constexpr int kDocMaxTokens = 8192;
int doc_maxsim(b200ms_t* h, const DocMaxSimCall& x, cudaStream_t s);

// One search: pack queries -> score -> top-k.  Device pointers, except that q and the outputs may be mapped pinned memory.
struct SearchRequest {
  const void* q = nullptr;  // rows [sum q_lens,128] of q_dtype (F32 | BF16)
  int q_dtype = B200MS_F32;
  const int32_t* q_lens = nullptr;  // HOST
  int n_q = 0;
  int k = 0;
  float i8_q_scale = 1.f;
  float score_scale = 1.f;
  float* top_scores = nullptr;   // [n_q, k]
  int64_t* top_ids = nullptr;    // [n_q, k]
  int32_t* top_counts = nullptr; // [n_q]
  int64_t id_base = 0;
  const uint32_t* allow = nullptr;       // allow-mask bits over the pages (NULL = all); with mask_index: [n_masks, words]
  const int32_t* mask_index = nullptr;   // per query: row of `allow` (-1 = no mask); NULL = the one mask for every query
  CandSpec cand;                         // ids == NULL: full scan
  const DocSpec* docs = nullptr;         // != NULL: the top k documents (per-query candidate lists only) instead of pages
  const int64_t* src_pages = nullptr;    // != NULL (device, [n_q - src_first]): query q >= src_first is corpus page
                                         // src_pages[q - src_first], its packed rows taken as they are stored (q_lens = the
                                         // pages' true lengths); queries before src_first are rows of q (q_dtype) as usual
  int src_first = 0;
  bool page_scale = false;  // a page or example search: scores on b200ms_mmr_device's sim scale, so zero_pad_compat does
                            // not apply to any of its queries
};

// What the scan part of a search (search_scan) leaves for its selection: the candidate lists it scored (cs.ids == NULL: a
// full scan), the score matrix's row stride, its group offsets on the device and its score dtype (F32 | I32)
struct ScanResult {
  CandSpec cs;
  int64_t ld = 0;
  const int32_t* goff_dev = nullptr;
  int sdt = 0;
};

// Results of a search as one block: [n_q*k int64 ids | n_q*k f32 scores | n_q int32 counts], padded to 16 bytes, so that
// a host entry point copies them back with one D2H.  Its first two parts are the exchange layout of the sharded search.
struct ResultBlock {
  size_t n_q, nk;
  ResultBlock(int n_q_, int k) : n_q(size_t(n_q_)), nk(size_t(n_q_) * size_t(k > 0 ? k : 0)) {}
  size_t bytes() const { return (nk * 12 + n_q * 4 + 15) & ~size_t(15); }
  int64_t* ids(void* b) const { return static_cast<int64_t*>(b); }
  float* scores(void* b) const { return reinterpret_cast<float*>(static_cast<uint8_t*>(b) + nk * 8); }
  int32_t* counts(void* b) const { return reinterpret_cast<int32_t*>(static_cast<uint8_t*>(b) + nk * 12); }
  void unpack(const void* b, float* ts, int64_t* ti, int32_t* tc) const {  // -> host arrays
    const uint8_t* p = static_cast<const uint8_t*>(b);
    memcpy(ti, p, nk * 8);
    memcpy(ts, p + nk * 8, nk * 4);
    memcpy(tc, p + nk * 12, n_q * 4);
  }
};

// Exchange layout of one rank's top-k list (what the all-gather moves, and what launch_merge_gathered reads):
//   [n_q*k int64 global page ids][n_q*k float32 scores], padded to a multiple of 16 bytes so that every rank's block of the
//   gathered buffer starts 8-byte aligned (n_q*k*12 alone is not: 1 query x 7 entries = 84 bytes);  unused entries: id -1, -inf.
inline size_t xchg_bytes(int n_q, int k) { return (size_t(n_q) * size_t(k) * 12 + 15) & ~size_t(15); }

// Which chunk ranges a scoring launch walks.  Full scan: the corpus' own unit plan, scores indexed by page id.
// Candidate ("slot") mode: unit j = the chunk range of candidate page j, scores indexed by j.
// Filtered full scan (launch_scan_plan): units over the allowed pages only, counted on the device; scores by page id.
struct UnitPlan {
  const int32_t* start = nullptr;
  const int32_t* end = nullptr;
  int n_units = 0;
  // != NULL: the unit count is this device word, written by an earlier kernel of the stream; n_units is then only an
  // upper bound (it sizes the launch)
  const int32_t* n_units_dev = nullptr;
  // filtered full scan, POPC kernel (one warp per page, no units): the allowed pages in ascending order and their count
  const int64_t* pages = nullptr;
  const int32_t* n_pages_dev = nullptr;
  int slot_mode = 0;
  // zero_pad_compat: bit i set = page i (slot_mode: candidate slot i) is shorter than the longest page of its scoring
  // batch, so its per-token maxima are clamped at 0 like the reference's zero padding does; NULL = clean MaxSim
  const uint32_t* clamp_bits = nullptr;
};

struct Corpus {
  const void* rows = nullptr;
  int dtype = -1;
  int64_t n_pages = 0;
  int64_t n_rows = 0;    // padded rows
  int64_t n_chunks = 0;  // n_rows / 32
  int n_units = 0;
  CUtensorMap tmap;      // [n_rows,128] view, box = {128 B, kTileN rows}, SWIZZLE_128B (BF16 / I8 only)
  bool has_tmap = false;
  bool has_empty = false;  // some page has zero rows (its score is the memset 0)
  int64_t clamp_batch = 0;  // zero_pad_compat batch size the full-scan clamp bitmask (b200ms::clamp_pages) was built for
  bool host = false;        // rows live in mapped pinned host memory (b200ms_set_corpus_host): candidate scoring only
  int64_t max_page_rows = 0;  // largest padded page
  bool scan_tables = false;   // n_units, unit_start, chunk_page and the scan-plan scratch are built (HBM corpora always; a
                              // host-resident one once sign rows are attached to it)
  bool signs = false;               // b200ms_set_sign_rows was called since the corpus was attached (set_corpus* detaches)
  const void* sign_rows = nullptr;  // its device [n_rows, 16 B] sign bits
};

// The packed rows a scoring launch reads: the attached corpus, or -- for a host-resident corpus -- the HBM staging block
// one gather round filled (a packed corpus of its own: pages 0..n, chunk_page and page_start local to the block).
struct CorpusView {
  const void* rows = nullptr;
  int dtype = -1;
  int64_t n_pages = 0;  // candidate ids outside [0, n_pages) are unused slots
  int64_t n_rows = 0;
  const CUtensorMap* tmap = nullptr;  // NULL: no TMA descriptor (1-bit rows)
  const int32_t* chunk_page = nullptr;
  const int64_t* page_start = nullptr;
};

}  // namespace bms

struct b200ms {
  int device = 0;
  int num_sms = 0;
  int smem_optin = 0;  // largest dynamic shared memory one block may opt in to (cudaDevAttrMaxSharedMemoryPerBlockOptin)
  std::string err;
  bms::Corpus corpus;
  // device metadata of the attached corpus
  bms::DeviceBuf chunk_page;   // int32 [n_chunks]   page index of every 32-row chunk
  bms::DeviceBuf unit_start;   // int32 [n_units+1]  first chunk of every work unit (page aligned)
  bms::DeviceBuf page_start;   // int64 [n_pages+1]  first padded row of every page   (B1 kernel, pack)
  bms::DeviceBuf page_len;     // int32 [n_pages]    TRUE row count of every page (zero_pad_compat, FDE from packed rows)
  bms::DeviceBuf clamp_pages;  // uint32 words: zero_pad_compat clamp bit per page (full scan), built lazily
  bms::DeviceBuf clamp_slots;  // uint32 words: clamp bit per candidate slot (rerank), rebuilt per call
  std::vector<int32_t> page_len_host;
  // filtered full scan (scan_plan.cu), sized by set_corpus and rebuilt by every filtered search: the union of the call's
  // masks, per full-plan unit the count and offset of its filtered units, the filtered units, and {units, pages, rows}
  bms::DeviceBuf scan_union, scan_cnt, scan_off, scan_start, scan_end, scan_hdr;
  bms::DeviceBuf scan_word_off, scan_pages;  // 1-bit corpora: per-word offsets into, and the list of, the allowed pages
  bool scan_planned = false;                 // the last full scan walked a filtered plan (b200ms_last_scan_stats)
  // scratch for pack / search
  bms::DeviceBuf meta, meta_b;  // per-call metadata block of a search (one upload) / of a pack call
  bms::DeviceBuf q_raw, q_packed, scores, mask, mask_index, out_all;
  bms::PinnedBuf stage;         // host entry points: [metadata | query rows | results], mapped into the device address space
  bms::DeviceBuf topk_keys, topk_ids;  // first-level (per-slice) top-k candidates
  bms::DeviceBuf docs_best, docs_mask, docs_top, docs_pick;  // grouping by document: per-(query, document) best key / rank,
                                                             // best-page mask, document order, picked pages' keys
  bms::DeviceBuf b1_q_i8, b1_tok_const;  // tensor-core 1-bit scorer: +-1 int8 query tiles and per-token constants
  bms::DeviceBuf f8_q_f16;  // e4m3 corpora: the query rows widened to f16 (A operand of the f16 MMA)
  bms::DeviceBuf cand_pad;  // batched rerank: per-query candidate lists re-laid out with a 32-slot-aligned stride
  bms::DeviceBuf cand_start, cand_end, cand_mask;  // candidate (rerank) mode: per-slot chunk ranges, valid-slot bitmask
  bms::DeviceBuf fde_simhash, fde_ams_index, fde_ams_sign, fde_tmp;  // FDE configuration (device copies) + scratch
  bms::DeviceBuf fde_q_bf16;                      // scan: query FDEs split into bf16 hi/lo rows (wgmma B operand)
  bms::DeviceBuf fde_final_index, fde_final_sign; // optional final count-sketch projection (final_projection_dimension)
  int fde_dim = 0, fde_reps = 0, fde_ksim = 0, fde_proj = 0;
  int fde_inner_dim = 0;   // reps * 2^ksim * proj (before the optional final projection)
  int fde_fill_empty = 0;  // fill_empty_partitions (documents): empty partition <- projection of the nearest point
  int fde_gemm = 1;        // 1: scan on wgmma (fde_scan_wgmma_kernel) when the shape allows, 0: SIMT scan
  float fde_scale = 1.f;
  int zero_copy = 1;       // host entry points: small calls read queries / write results through mapped pinned memory
  bms::Comm* comm = nullptr;
  cudaStream_t stream = nullptr;  // internal stream for *_host entry points
  // the order of the handle's calls across streams (bms::StreamOrder): order_ev is recorded at the end of the last call
  // that enqueued work, on order_stream; order_pending = false once that call is known to be finished
  cudaEvent_t order_ev = nullptr;
  cudaStream_t order_stream = nullptr;
  bool order_pending = false;
  // ring of CUDA-event pairs bracketing the scoring kernels of the most recent b200ms_score / search calls
  static constexpr int kEvRing = 256;
  cudaEvent_t ev0[kEvRing] = {}, ev1[kEvRing] = {};
  int64_t ev_count = 0;  // scoring calls recorded since creation / last reset
  int64_t launches = 0;
  int64_t unit_rows = 4096;
  int max_ctas = 0;
  int b1_tensor = 2;  // 1-bit full scans: 0 = POPC kernel, 1 = wgmma kernel (bits expanded to {0,1} int8 in smem), 2 = by group count
  int zero_pad_batch = 0;  // > 0: reproduce score_multi_vector's zero-padding quirk with this batch size (128 upstream)
  CUtensorMap tmap_q;  // query rows in 16-row boxes; re-encoded only when (pointer, dtype, rows) change
  const void* tmap_q_base = nullptr;
  int tmap_q_dtype = -1;
  int64_t tmap_q_rows = -1;
  // CUDA graphs of the small zero-copy host search (pack -> score -> top-k): key -> executable graph
  struct HostGraph {
    uint64_t key = 0;
    uint64_t generation = 0;
    cudaGraphExec_t exec = nullptr;
    int launches = 0;
    int seen = 0;  // uses of this key so far; the graph is captured on the second one (buffers are warm by then)
    uint64_t last_use = 0;
  };
  std::vector<HostGraph> host_graphs;
  uint64_t generation = 0;   // bumped whenever a scratch buffer moves, the corpus is re-attached or an option changes
  uint64_t graph_clock = 0;
  int host_graph = 1;        // option "host_graph": replay small unmasked host searches as one CUDA graph
  bool capturing = false;    // inside stream capture: no event timing, no allocation
  // host-resident corpus (host_tier.cu): per-call dedup / plan scratch and the HBM staging block of the gathered pages
  int64_t host_stage_bytes = int64_t(2) << 30;  // option "host_stage_bytes": staging budget per gather round
  bms::DeviceBuf ht_bitmap, ht_wpre, ht_uniq, ht_stage_off, ht_hdr, ht_remap, ht_ps, ht_chunk_page, ht_scores;
  bms::DeviceBuf ht_stage;           // staging rows (1024-byte aligned inside the allocation)
  CUtensorMap ht_tmap;               // TMA descriptor of the staging block, re-encoded when the block moves
  const void* ht_tmap_base = nullptr;
  int ht_tmap_dtype = -1;
  int64_t ht_tmap_rows = 0;
  std::vector<cudaEvent_t> ht_ev;    // event pairs around each round's gather (last call)
  int64_t ht_unique = 0, ht_bytes = 0;
  int ht_rounds = 0;
  // corpus storage: the growable blocks created on this handle (block.cu), and b200ms_compact_rows' run tables and bounce
  // buffer (compact.cu)
  std::vector<b200ms_block_t*> blocks;
  bms::DeviceBuf compact_meta, compact_bounce;
  // diversifying results (maxsim_mmr.cu): per-call state of the greedy pick and the round kernels' per-tile partial sums
  bms::DeviceBuf mmr_state, mmr_partials;
  // searching with stored pages as the queries (search_pages.cu): the call's source page ids [, their true-row offsets]
  bms::DeviceBuf src_pages;
  // relevance feedback (search_examples.cu): the call's example table, the requests' and examples' candidate lists (or the
  // examples' mask rows), the fused score rows, and the hash tables of a candidate union
  bms::DeviceBuf ex_meta, ex_lists, ex_fused, ex_union;
  // document-level MaxSim (doc_maxsim.cu): the token table, the document scores and found mask, the candidate calls'
  // document marks and allow rows
  bms::DeviceBuf dm_table, dm_scores, dm_allow;
  // near-duplicate pages (duplicates.cu): per-CTA column maxima of pages too long for shared memory
  bms::DeviceBuf dup_cols;
};

namespace bms {

// Calls on one handle run on the GPU in the order they were made, whatever streams they name: they share the handle's
// scratch.  Every entry point that enqueues work holds one of these, on the stream it enqueues on, for the whole call.  On
// entry the stream waits for the handle's previous call if that call ran on another stream; on exit the handle's event is
// recorded on the stream, or, after finished() (the call synchronised its stream), nothing is left pending.  A stream that
// is being captured into a graph neither waits nor records: an event recorded outside a capture cannot be waited on inside.
class StreamOrder {
 public:
  StreamOrder(b200ms_t* h, cudaStream_t s);
  ~StreamOrder();
  StreamOrder(const StreamOrder&) = delete;
  StreamOrder& operator=(const StreamOrder&) = delete;
  int error() const { return err_; }  // the wait could not be enqueued: the call must not enqueue anything
  void finished() { synced_ = true; }

 private:
  b200ms_t* h_;
  cudaStream_t s_;
  bool active_ = false, synced_ = false;
  int err_ = 0;
};

int set_error(b200ms_t* h, int code, const std::string& msg);
int check_cuda(b200ms_t* h, cudaError_t e, const char* what);
int reserve(b200ms_t* h, DeviceBuf& b, size_t bytes);
int upload(b200ms_t* h, DeviceBuf& b, const void* src, size_t bytes, cudaStream_t s);
int reserve_pinned(b200ms_t* h, PinnedBuf& b, size_t bytes);
// Raise cudaFuncAttributeMaxDynamicSharedMemorySize when static + dynamic shared memory passes the 48 KB default; process-global
// raise-only table per (device, kernel) -- the attribute belongs to the function, not to the handle
int ensure_smem(b200ms_t* h, const void* kernel, int smem, const char* what);
int make_tmap_rows(b200ms_t* h, CUtensorMap* out, const void* base, int dtype, int64_t n_rows, int box_rows,
                   int64_t row_bytes = 0);
void comm_teardown(b200ms_t* h);
void release_blocks(b200ms_t* h);  // block.cu: unmap, release and free every block still alive on the handle
// pack -> score -> top-k of r on stream s (api.cu); m = build_search_meta(r.q_lens, r.n_q).  meta_dev != NULL: m's block
// already sits in device-readable memory at this address (mapped pinned staging) -- no upload; else ONE cudaMemcpyAsync.
int search_core(b200ms_t* h, const SearchRequest& r, const SearchMeta& m, cudaStream_t s, const void* meta_dev = nullptr);
// search_core without the selection: pack -> score, the group scores left in h->scores as *out describes them
int search_scan(b200ms_t* h, const SearchRequest& r, const SearchMeta& m, cudaStream_t s, const void* meta_dev, ScanResult* out);

// Full scan: unit u = chunks [unit_start[u], unit_start[u+1]) of the attached corpus, scores indexed by page id
inline UnitPlan full_scan_plan(const b200ms_t* h) {
  UnitPlan p;
  p.start = static_cast<const int32_t*>(h->unit_start.p);
  p.end = p.start + 1;
  p.n_units = h->corpus.n_units;
  return p;
}

// Score matrix of a call: gp padded query groups (at least 4) by ld items (n_items rounded up to 32, at least 32), 4 bytes each
struct ScoreLayout {
  int64_t gp, ld;
};
inline ScoreLayout score_layout(const SearchMeta& m, int64_t n_items) {
  const int64_t ld = (n_items + 31) & ~int64_t(31);
  return {m.groups_padded > 0 ? m.groups_padded : 4, ld > 0 ? ld : 32};
}
// Zeroes gp x ld scores: the scores no launch writes (the tile kernels skip pages without rows), or all of them when a call
// scores nothing -- every page then scores 0, still a defined ranking
int zero_scores(b200ms_t* h, void* scores, int64_t gp, int64_t ld, cudaStream_t s, const char* what);
// The units a full scan of the attached corpus walks, into *plan: the corpus' own, or with allow masks the filtered plan
// (launch_scan_plan).  Sets h->scan_planned to which one it is (b200ms_last_scan_stats).
int plan_full_scan(b200ms_t* h, const uint32_t* allow, const int32_t* mask_index, int n_q, cudaStream_t s, UnitPlan* plan);

// The attached corpus as the scorers see it
inline CorpusView corpus_view(const b200ms_t* h) {
  const Corpus& c = h->corpus;
  CorpusView v;
  v.rows = c.rows;
  v.dtype = c.dtype;
  v.n_pages = c.n_pages;
  v.n_rows = c.n_rows;
  v.tmap = c.has_tmap ? &c.tmap : nullptr;
  v.chunk_page = static_cast<const int32_t*>(h->chunk_page.p);
  v.page_start = static_cast<const int64_t*>(h->page_start.p);
  return v;
}

// CTAs of a grid-stride launch over n items, per_block items per CTA: enough to cover them, at least 1 and at most per_sm
// per SM
inline int grid_stride_blocks(const b200ms_t* h, int64_t n, int per_block, int per_sm) {
  const int64_t want = (n + per_block - 1) / per_block, cap = int64_t(h->num_sms) * per_sm;
  return int(want < 1 ? 1 : want < cap ? want : cap);
}

// Pages of a host-resident corpus named by ids[0..n_slots) (host_tier.cu): dedup them, gather them into the staging block in
// rounds of at most host_stage_bytes and call round_fn after each round's gather with the block as a corpus view and remap
// (slot -> page of the view; -1 = invalid id or a page of another round).  Sets the gather stats; h->ht_rounds stays 0 when
// no named page has a row.  Synchronises s once.
int gather_host_tier(b200ms_t* h, const int64_t* ids, int64_t n_slots, cudaStream_t s,
                     int (*round_fn)(b200ms_t*, const CorpusView&, const int64_t* remap, int r, int rounds, void* ctx),
                     void* ctx);
// Gather rounds gather_host_tier needs for unique pages of `rows` padded rows in all (0 for none)
int host_tier_rounds(const b200ms_t* h, int64_t rows);
// Candidate scoring of a host-resident corpus: gather_host_tier over the candidate slots, every round scored through
// score_round.
int score_host_tier(b200ms_t* h, const CandSpec& cs, int n_q, int64_t gp, int64_t ld, void* group_scores, cudaStream_t s,
                    int (*score_round)(b200ms_t*, const CorpusView&, const int64_t* unit_ids, void* scores, bool fill,
                                       void* ctx),
                    void* ctx);

// kernel launchers (each returns a b200ms error code and bumps h->launches)
// group_ntok (device, [n_groups_real] or NULL = 32 each): the true tokens of every group; a padding token adds +0
// doc != NULL: document mode (DocScan) -- group_scores and plan.clamp_bits are not used, plan.slot_mode must be 0
int launch_score_wgmma(b200ms_t* h, const CorpusView& v, const UnitPlan& plan, const void* q_packed, int n_groups_real,
                       const int32_t* group_ntok, void* group_scores, int64_t ld, cudaStream_t s, int m_tile_lo = 0,
                       int m_tile_hi = -1, const DocScan* doc = nullptr);
// scan != NULL (full scans, cand_ids == NULL): only the pages scan->pages lists, scores still indexed by page id
int launch_score_b1(b200ms_t* h, const CorpusView& v, const int64_t* cand_ids, int64_t n_cand, const void* q_packed,
                    int n_groups, const int32_t* group_ntok_dev, void* group_scores, int64_t ld, cudaStream_t s, int g_lo,
                    int g_hi, const UnitPlan* scan = nullptr);
int launch_pad_cands(b200ms_t* h, const int64_t* src, int n_cand, int n_lists, int64_t stride, int64_t* dst, cudaStream_t s);
int launch_clamp_slots(b200ms_t* h, const int64_t* cand_ids, int n_cand, int n_lists, int64_t list_stride, int batch,
                       uint32_t* clamp_bits, cudaStream_t s);
int launch_score_b1_wgmma(b200ms_t* h, const UnitPlan& plan, const void* q_bits, const int32_t* group_ntok_dev,
                          int n_groups_real, void* group_scores, int64_t ld, cudaStream_t s, const DocScan* doc = nullptr);
// The A operand of the 1-bit wgmma scan: int8 rows q_i8 [n_rows,128] (1024-byte aligned) and one int32 constant per row,
// in the handle's scratch
int reserve_b1_query(b200ms_t* h, int64_t n_rows, int8_t** q_i8, int32_t** tok_const);
// The 1-bit wgmma scan of the sign rows of v (v.rows: 16 B per row) for prepared A rows: group_scores[g, p] = sum over the
// group's rows t of (tok_const[t] + max over the page's rows r of <q_i8[t], bits(r) as {0,1}>)
int launch_b1_tiles(b200ms_t* h, const CorpusView& v, const UnitPlan& plan, const int8_t* q_i8, const int32_t* tok_const,
                    int n_groups_real, void* group_scores, int64_t ld, cudaStream_t s, const int32_t* group_ntok = nullptr,
                    const DocScan* doc = nullptr);
// Corpus tables a full scan needs (unit_start, chunk_page, scan-plan scratch), enqueued on s; c.n_units is set
int build_scan_tables(b200ms_t* h, Corpus& c, const int64_t* ps_host, cudaStream_t s);
// Scratch of launch_scan_plan for the corpus c (set_corpus reserves it, so that no search grows it)
int reserve_scan_plan(b200ms_t* h, const Corpus& c);
// Work units of a full scan that reads only the pages the call's masks allow (scan_plan.cu), built on stream s without a
// synchronisation: allow / mask_index as in SearchRequest (allow != NULL).  *plan keeps its clamp_bits.
int launch_scan_plan(b200ms_t* h, const uint32_t* allow, const int32_t* mask_index, int n_q, cudaStream_t s, UnitPlan* plan);
// Full-plan units and padded rows the last full scan walked; reads the device words of a filtered plan (the caller has
// waited for the scan)
int read_scan_stats(b200ms_t* h, int64_t* units, int64_t* rows);
int launch_cand_units(b200ms_t* h, const CorpusView& v, const int64_t* cand_ids, int n_cand, int32_t* unit_start,
                      int32_t* unit_end, uint32_t* slot_mask, cudaStream_t s);
int launch_hamming_batch(b200ms_t* h, const void* q, const void* cand, int64_t n, uint32_t* out, cudaStream_t s);
int launch_chunk_page(b200ms_t* h, const int64_t* page_start_dev, int64_t n_pages, int32_t* chunk_page, cudaStream_t s);
int launch_pack_rows(b200ms_t* h, const void* src, int src_dtype, const int64_t* src_start_dev,
                     const int64_t* dst_start_dev, int64_t n_items, int64_t dst_rows, int pad_mode, void* dst,
                     int dst_dtype, float i8_scale, cudaStream_t s);
int launch_topk(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                const int32_t* group_offsets_dev, int n_q, const uint32_t* allow_mask, int k, float scale,
                int64_t id_base, const int64_t* id_map, float* top_scores, int64_t* top_ids, int32_t* top_counts,
                cudaStream_t s, const int32_t* mask_index = nullptr, int64_t mask_stride = 0, int64_t q_stride = 0);
// the top k documents (DocSpec) over a group-score matrix, in the total order of launch_topk.  Full scan (cand == NULL):
// items are pages [0, n_items), filtered as launch_topk filters them (allow, mask_index); candidate mode: per-query lists
// cand [n_q, q_stride] of n_items slots (q_stride a multiple of 32), page ids valid in [0, n_pages).
int launch_topk_docs(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_items, int64_t ld,
                     const int32_t* group_offsets_dev, int n_q, const uint32_t* allow, const int32_t* mask_index,
                     const int64_t* cand, int64_t q_stride, int64_t n_pages, const DocSpec& d, int k, float scale,
                     int64_t id_base, cudaStream_t s);
// merge straight from the all-gathered exchange layout: gathered = world blocks of [n_q*k int64 ids | n_q*k f32 scores]
int launch_merge_gathered(b200ms_t* h, const void* gathered, int world, int n_q, int k, float* top_scores, int64_t* top_ids,
                          int32_t* top_counts, cudaStream_t s);
int launch_fde_encode(b200ms_t* h, const void* rows, int src_dtype, const int64_t* item_start_dev, int n_items,
                      int is_document, float* out, cudaStream_t s, const int32_t* item_len_dev = nullptr);
int launch_fde_finalize(b200ms_t* h, const float* fde, int64_t n, void* out_rows, float* inv_norm, cudaStream_t s);
int launch_fde_scan(b200ms_t* h, const void* F, const float* inv_norm, int64_t n_pages, const float* q_fde, int n_q,
                    float* scores, int64_t ld, cudaStream_t s);
int launch_merge_topk(b200ms_t* h, const float* cand_scores, const int64_t* cand_ids, int n_q, int m, int k,
                      float* top_scores, int64_t* top_ids, int32_t* top_counts, cudaStream_t s);
// search_pages.cu.  src_dev: device page ids of the attached corpus (checked by the caller); ss_dev / ds_dev: [n_src+1] true /
// padded row offsets of the sources (build_search_meta of their lengths).
// The sources' packed rows in the query layout of b200ms_pack_queries: rows [row0, dst_rows) of dst, zero past each source's
// true rows.  ss_dev / ds_dev may be the tail of a longer layout (the sources after some query rows): row0 = ds_dev[0].
int launch_pack_src_pages(b200ms_t* h, const int64_t* src_dev, const int64_t* ss_dev, const int64_t* ds_dev, int64_t n_src,
                          int64_t row0, int64_t dst_rows, void* dst, cudaStream_t s);
// The sources' true rows back to back as float32 [n_rows, 128]: packed value (a sign bit as +-1) times scale
int launch_page_rows(b200ms_t* h, const int64_t* src_dev, const int64_t* ss_dev, int64_t n_src, int64_t n_rows, float scale,
                     float* out, cudaStream_t s);
// Candidate mode: clear the valid bit of every slot whose page its list's allow-mask row (as SearchRequest) forbids
int launch_mask_cand_slots(b200ms_t* h, const int64_t* cand, int64_t n_slots, int64_t stride, const uint32_t* allow,
                           const int32_t* mask_index, uint32_t* slot_mask, cudaStream_t s);
// Reported scores of source q divided by its true length; a source without rows gets count 0
int launch_normalise_pages(b200ms_t* h, const int64_t* src_dev, int n_src, int k, float* scores, int64_t* ids,
                           int32_t* counts, cudaStream_t s);
// search_examples.cu.  One example of a request: its group rows [g0, g1) of the score matrix (g0 == g1: no rows, no term),
// its true rows or tokens, its weight, and the score column of its item 0 (candidate mode: its list's first slot).
struct ExampleItem {
  int32_t g0, g1;
  float len, w;
  int64_t col0;
};
// dst row i = src row idx[i] (row_len elements each); T = int32_t or int64_t
template <typename T>
int launch_gather_rows(b200ms_t* h, const T* src, int64_t row_len, const int32_t* idx, int n_rows, T* dst, cudaStream_t s);
// fused[r * fused_ld + p], p < n_items: sum over request r's examples (items[req_off[r] .. req_off[r+1]), in order) of
// w * (float(finish_sum(its groups' scores at col0 + p)) * score_scale / len), with _rn arithmetic; items whose bit in r's
// allow row (mask_index ? allow row mask_index[r] : allow row r, rows mask_stride words apart; -1 / NULL = all) is clear
// are not read or written.
int launch_fuse_examples(b200ms_t* h, const void* gs, int score_dtype, int64_t ld, const ExampleItem* items,
                         const int32_t* req_off, int n_req, int64_t n_items, const uint32_t* allow, const int32_t* mask_index,
                         int64_t mask_stride, float score_scale, float* fused, int64_t fused_ld, cudaStream_t s);
// out [n_req, width]: request r's distinct page ids (>= 0) over lists list_off[r] .. list_off[r+1] of cand [*, n_cand], in
// first-occurrence order, -1 padded; tables: h->ex_union scratch
int launch_union_candidates(b200ms_t* h, const int64_t* cand, int n_cand, const int32_t* list_off_dev, int n_req,
                            int64_t max_entries, int64_t* out, int width, cudaStream_t s);

}  // namespace bms
