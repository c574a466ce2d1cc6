"""MaxSim at the sizes it is benchmarked at: every page of corpora past 4 GiB against the float64 reference (-m gpu, H100).

Each corpus is a planted corpus of tests/scale_reference.py, built on the GPU through reserve_rows + add_pages so the pack
kernel writes the layout, with more than 1 GiB of packed rows past byte offset 2^32 (checked below): bf16 20 480 pages,
int8 / fp8 40 960, 1-bit 327 680 (its page-level top-k runs 40 slices for k <= 204 and 2 for k = 4096).  One corpus is
resident at a time; a corpus is skipped, with the reason, when the card lacks the memory.  Every page is compared with
scale_reference.reference_scores, computed on the GPU from the packed bytes the scan reads, through oracle.scoring's
assert_scores / assert_ranking / assert_candidate_ranking and their tolerances:
  * full scans of 1, 3, 13 and 40 query groups, default grid and one CTA (its stage ring wraps over the whole corpus); 1-bit
    on the POPC and the wgmma kernel, bit-identical to each other; top-k of 10 and 4096;
  * 256 queries x 32 tokens (bf16 and int8): score_matrix, search_host and search_device;
  * filtered scans: 0.1 / 1 / 10 / 50 % masks, a mask of only the pages past 4 GiB, per-query masks with an unfiltered query --
    ranking against the reference, bit-identical to b200ms_score + masked b200ms_topk, plan = tests/scan_plan_model.py;
  * search_docs_device with 16 pages per document against tests/docs_oracle.py;
  * rerank_batch of 1000 candidates per query, most past 4 GiB, with duplicates and unused slots; explain of pages past 4 GiB;
  * the host tier: an int8 corpus of more than 4 GiB in pinned memory reranks bit-identically to the HBM tier;
  * the sign stage (bf16, int8, fp8): b200ms_sign_rows of every row, past byte 2^32, against the header's rule in torch
    integer ops; every page's exact S (scale_reference.sign_reference) through per-query masks of at most 4096 pages on the
    filtered plan, and the first 4096 candidates of the unmasked batch in the oracle's order.
"""
import ctypes
import gc
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import scale_reference as sr  # noqa: E402
import sign_oracle as so  # noqa: E402
import scan_plan_model as spm  # noqa: E402
import test_gpu_filtered_scan as tfs  # noqa: E402
from docs_oracle import topk_docs_np  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex, _aligned_bytes  # noqa: E402
from oracle.scoring import TOL, assert_candidate_ranking, assert_ranking, assert_scores, slot_scores_of  # noqa: E402

DEV = torch.device("cuda", 0)
SEED = 0
PAGES = {"bf16": 20480, "int8": 40960, "fp8": 40960, "binary": 327680}
DTYPES = list(PAGES)
# 13 queries; the prefixes of 1, 2, 3 and 13 queries are batches of 1, 3, 13 and 40 32-token groups
Q_TOKENS = [32, 40, 300, 130, 33, 7, 1, 64, 256, 20, 31, 96, 65]
PREFIX_GROUPS = {1: 1, 2: 3, 3: 13, 13: 40}
WORK_BYTES = 10 << 30  # build chunks, the reference's products and the score matrices, next to the corpus
FOUR_GIB = 1 << 32


class Scale:
    def __init__(self, dtype):
        self.dtype = dtype
        t0 = time.time()
        self.idx = sr.build(dtype, PAGES[dtype], SEED)
        self.lens = np.asarray(self.idx.page_lens, dtype=np.int64)
        self.starts = np.concatenate([[0], np.cumsum(sr.padded_rows(self.lens))])
        self.qs = sr.queries(dtype, SEED, Q_TOKENS)
        _, self.goff, _, self.q_packed = self.idx.score_groups(self.qs)
        t1 = time.time()
        self.ref = sr.reference_scores(self.idx, self.q_packed, self.goff, Q_TOKENS)
        print(f"\n[scale] {dtype}: {self.idx.n_pages} pages, {self.idx.n_rows_padded * self.idx.row_bytes / 2**30:.2f} GiB of "
              f"rows, built in {t1 - t0:.1f} s, reference of {len(Q_TOKENS)} queries in {time.time() - t1:.1f} s")

    def past_4gib(self):
        """Pages with rows whose first row starts at or past byte 2^32."""
        return np.flatnonzero((self.starts[:-1] * self.idx.row_bytes >= FOUR_GIB) & (self.lens > 0))

    def q_dev(self, n):
        return torch.from_numpy(np.concatenate(self.qs[:n]).astype(np.float32)).to(DEV)


@pytest.fixture(scope="module")
def scale(request):
    dtype = request.param
    rows = int(sr.padded_rows(sr.page_lens(PAGES[dtype], SEED)).sum())
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(DEV)
    need = rows * sr.ROW_BYTES[dtype] + WORK_BYTES
    print(f"\n[scale] {torch.cuda.get_device_name(DEV)}: {free / 2**30:.1f} of {total / 2**30:.1f} GiB free before the "
          f"{dtype} corpus")
    if free < need:
        pytest.skip(f"the {dtype} corpus needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB are free")
    torch.cuda.reset_peak_memory_stats(DEV)
    s = Scale(dtype)
    assert s.idx.n_rows_padded * s.idx.row_bytes > FOUR_GIB + (1 << 30)  # at least 1 GiB of rows past 4 GiB
    yield s
    print(f"\n[scale] {dtype}: torch.cuda.max_memory_allocated = {torch.cuda.max_memory_allocated(DEV) / 2**30:.2f} GiB")
    s.idx.close()
    del s
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ full scans
@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_full_scan_scores_every_page(scale):
    idx, dtype = scale.idx, scale.dtype
    paths = [("b1_tensor", 0), ("b1_tensor", 1)] if dtype == "binary" else [(None, None)]
    by_path = {}
    try:
        for opt, val in paths:
            if opt:
                idx.set_option(opt, val)
            for n, groups in PREFIX_GROUPS.items():
                for max_ctas in ((0, 1) if groups <= 3 else (0,)):
                    idx.set_option("max_ctas", max_ctas)
                    got = idx.score_matrix(scale.qs[:n])
                    assert_scores(dtype, got, scale.ref[:n], f"{dtype} {opt}={val} {groups} groups max_ctas={max_ctas}")
                    by_path.setdefault((n, max_ctas), []).append(got)
    finally:
        idx.set_option("max_ctas", 0)
        if dtype == "binary":
            idx.set_option("b1_tensor", 2)
    for key, outs in by_path.items():  # POPC and wgmma 1-bit kernels: the same integers
        assert all(np.array_equal(o, outs[0]) for o in outs[1:]), key
    for k in (10, 4096):
        ts, ti, tc = idx.search_host(scale.qs, k)
        for qi in range(len(scale.qs)):
            assert_ranking(dtype, ts[qi], ti[qi], tc[qi], scale.ref[qi], k, what=f"{dtype} k={k} q{qi}")


@pytest.mark.parametrize("scale", ["bf16", "int8"], indirect=True)
def test_query_batch_of_256(scale):
    """256 queries x 32 tokens: 64 query tiles, 16 passes of NM = 4 (bf16) or 8 passes of NM = 8 (int8)."""
    idx, dtype = scale.idx, scale.dtype
    lens = [32] * 256
    qs = sr.queries(dtype, SEED, lens, q_seed=256)
    _, goff, _, q_packed = idx.score_groups(qs)
    ref = sr.reference_scores(idx, q_packed, goff, lens)
    assert_scores(dtype, idx.score_matrix(qs), ref, f"{dtype} q256 score_matrix")
    qd = torch.from_numpy(np.concatenate(qs)).to(DEV)
    for k in (10, 4096):
        host = idx.search_host(qs, k)
        dev = tfs.to_np(idx.search_device(qd, lens, k))
        for name, (ts, ti, tc) in (("search_host", host), ("search_device", dev)):
            for qi in range(len(qs)):
                assert_ranking(dtype, ts[qi], ti[qi], tc[qi], ref[qi], k, what=f"{dtype} q256 {name} k={k} q{qi}")


# ------------------------------------------------------------------------------------------------ filtered scans
@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_filtered_scan(scale):
    idx, dtype = scale.idx, scale.dtype
    n = idx.n_pages
    rng = np.random.default_rng(7)
    past = np.zeros(n, bool)
    past[scale.past_4gib()] = True
    masks = {f"{pct}%": rng.random(n) < pct / 100.0 for pct in (0.1, 1, 10, 50)}
    masks["past 4 GiB"] = past
    for name, allow in masks.items():
        words = idx.mask_from_pages(allow)
        for nq in (1, 3):  # 1 group (1-bit: POPC walks the allowed pages) and 13 groups
            got = tfs.to_np(idx.search_device(scale.q_dev(nq), Q_TOKENS[:nq], tfs.K, allow_mask_dev=tfs.dev_words(words)))
            tfs.assert_plan(idx, words, None, f"{dtype} {name}")
            for qi in range(nq):
                assert_ranking(dtype, got[0][qi], got[1][qi], got[2][qi], scale.ref[qi], tfs.K, allow, f"{dtype} {name} q{qi}")
            tfs.assert_bits(got, tfs.reference(idx, scale.qs[:nq], [allow] * nq), f"{dtype} {name} {nq} queries")
    rows = [masks["1%"], past]
    stacked = np.stack([idx.mask_from_pages(r) for r in rows])
    for mask_index in ([0, 1, 0], [1, -1, 0]):
        mi = torch.tensor(mask_index, dtype=torch.int32, device=DEV)
        got = tfs.to_np(idx.search_device(scale.q_dev(3), Q_TOKENS[:3], tfs.K, allow_mask_dev=tfs.dev_words(stacked),
                                          mask_index_dev=mi))
        tfs.assert_plan(idx, stacked, mask_index, f"{dtype} per-query {mask_index}")
        allow = [rows[i] if i >= 0 else np.ones(n, bool) for i in mask_index]
        for qi in range(3):
            assert_ranking(dtype, got[0][qi], got[1][qi], got[2][qi], scale.ref[qi], tfs.K, allow[qi],
                           f"{dtype} per-query {mask_index} q{qi}")
        tfs.assert_bits(got, tfs.reference(idx, scale.qs[:3], allow), f"{dtype} per-query {mask_index}")


# ------------------------------------------------------------------------------------------------ documents
@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_documents(scale):
    """16 pages per document.  int8 / 1-bit: against the docs oracle on the reference scores (exact).  bf16 / fp8: the
    one-group query, whose score_matrix row is the kernel's own float32 score, is held to the reference and then ranked."""
    idx, dtype = scale.idx, scale.dtype
    n = idx.n_pages
    per_page = 16
    page_doc = (torch.arange(n, device=DEV, dtype=torch.int32) // per_page).contiguous()
    n_docs = (n + per_page - 1) // per_page
    exact = TOL[dtype] == 0.0
    nq = 3 if exact else 1
    if exact:
        want_scores = scale.ref[:nq]
    else:
        own = idx.score_matrix(scale.qs[:1])
        assert_scores(dtype, own, scale.ref[:1], f"{dtype} one-group query")
        want_scores = own.astype(np.float32)
    k, per_doc = 10, 3
    ts, ti, pc, dc = tfs.to_np(idx.search_docs_device(scale.q_dev(nq), Q_TOKENS[:nq], k, per_doc, page_doc, n_docs))
    pd_np = page_doc.cpu().numpy()
    for qi in range(nq):
        _, ids, counts, nd = topk_docs_np(want_scores[qi], pd_np, n_docs, k, per_doc)
        assert int(dc[qi]) == nd and np.array_equal(pc[qi], counts) and np.array_equal(ti[qi], ids), (dtype, qi)
        used = ids >= 0
        if exact:
            assert_scores(dtype, ts[qi][used], scale.ref[qi][ids[used]], f"{dtype} docs q{qi}")
        else:
            assert np.array_equal(ts[qi][used], want_scores[qi][ids[used]]), (dtype, qi)


# ------------------------------------------------------------------------------------------------ candidates
def candidate_lists(scale, n_q, n_cand, seed):
    """Mostly pages past 4 GiB, some from anywhere, an empty page, duplicates and -1 slots."""
    rng = np.random.default_rng(seed)
    past, n = scale.past_4gib(), scale.idx.n_pages
    cand = np.where(rng.random((n_q, n_cand)) < 0.9, rng.choice(past, (n_q, n_cand)), rng.integers(0, n, (n_q, n_cand)))
    empty = np.flatnonzero(scale.lens == 0)
    cand[:, 3] = cand[:, 1]
    cand[:, n_cand - 1] = cand[:, 0]
    cand[:, 5] = -1
    cand[:, 600] = -1
    cand[:, 7] = empty[-1]
    cand[:, 8] = n - 1
    return np.ascontiguousarray(cand, dtype=np.int64)


@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_rerank_and_explain_past_4gib(scale):
    idx, dtype = scale.idx, scale.dtype
    n_q, n = 3, idx.n_pages
    cand = candidate_lists(scale, n_q, 1000, 11)
    qd = scale.q_dev(n_q)
    for k in (10, 1000):
        ts, ti, tc = tfs.to_np(idx.rerank_batch(qd, Q_TOKENS[:n_q], torch.from_numpy(cand).to(DEV), k))
        for qi in range(n_q):
            assert_candidate_ranking(dtype, ts[qi], ti[qi], tc[qi], slot_scores_of(scale.ref[qi], cand[qi]), cand[qi], n, k,
                                     f"{dtype} rerank k={k} q{qi}")
    # explain: the last pages, pages of edge lengths and random pages, all past 4 GiB
    past = scale.past_4gib()
    edge = [p for p in past if scale.lens[p] % 32 in (0, 1, 31) or scale.lens[p] < 8][:6]
    pages = np.asarray(sorted(set([int(past[-1]), int(past[-2]), int(past[0])] + edge +
                                  np.random.default_rng(12).choice(past, 8).tolist())), dtype=np.int64)
    tsx, br, _ = idx.explain(scale.qs[:n_q], pages)
    tsx, br = tfs.to_np((tsx, br))
    assert_scores(dtype, tsx.astype(np.float64).sum(axis=2), scale.ref[:n_q, pages], f"{dtype} explain token sums")
    rows_u8 = idx.packed_rows()
    q_u8 = scale.q_packed.reshape(-1, idx.row_bytes)
    for j, p in enumerate(pages):
        L = int(scale.lens[p])
        sims = sr.token_maxima(dtype, rows_u8, int(scale.starts[p]), L, q_u8, scale.goff, Q_TOKENS[:n_q])
        for qi, sim in enumerate(sims):
            T = Q_TOKENS[qi]
            b = br[qi, j, :T]
            assert ((b >= 0) & (b < L)).all(), (dtype, qi, int(p))
            best, at = sim.max(axis=1), sim[np.arange(T), b]
            slack = TOL[dtype] * np.maximum(np.abs(best), 1e-3) if TOL[dtype] else 0.0
            assert (at >= best - slack).all(), (dtype, qi, int(p), np.flatnonzero(at < best - slack)[:5])


# ------------------------------------------------------------------------------------------------ host tier
@pytest.mark.parametrize("scale", ["int8"], indirect=True)
def test_host_tier_rerank_is_bit_identical(scale):
    idx = scale.idx
    host = MaxSimIndex(dtype="int8", tier="host")
    try:
        host.reserve_rows(idx.n_rows_padded)
    except nat.NativeError as e:
        host.close()
        pytest.skip(f"no pinned host block of {idx.n_rows_padded * idx.row_bytes / 2**30:.1f} GiB: {e}")
    try:
        host.append_packed(idx.packed_rows(), idx._page_lens)
        assert host.n_rows_padded * host.row_bytes > FOUR_GIB + (1 << 30)
        qd = scale.q_dev(3)
        for seed in (21, 22):
            cand = torch.from_numpy(candidate_lists(scale, 3, 1000, seed)).to(DEV)
            for k in (10, 1000):
                want = tfs.to_np(idx.rerank_batch(qd, Q_TOKENS[:3], cand, k))
                got = tfs.to_np(host.rerank_batch(qd, Q_TOKENS[:3], cand, k))
                tfs.assert_bits(got, want, f"host tier k={k} seed={seed}")
        assert host.gather_stats()["unique_pages"] > 0
    finally:
        host.close()


# ------------------------------------------------------------------------------------------------ sign stage
def sign_candidates(idx, queries, n_cand, masks=None, index=None):
    """b200ms_sign_candidates_device at q_scale 127 and score_scale 1 (scores are float32(S)) -> host arrays."""
    src = torch.from_numpy(np.concatenate(queries).astype(np.float32)).to(DEV)
    lens = [len(q) for q in queries]
    n_q = len(lens)
    ts = torch.empty((n_q, n_cand), dtype=torch.float32, device=DEV)
    ti = torch.empty((n_q, n_cand), dtype=torch.int64, device=DEV)
    tc = torch.empty((n_q,), dtype=torch.int32, device=DEV)
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    idx.h.check(nat.lib.b200ms_sign_candidates_device(
        idx.h.ptr, vp(src), nat.F32, nat.i32_array(lens), n_q, n_cand, vp(masks), 0 if masks is None else masks.shape[0],
        vp(index), ctypes.c_float(127.0), ctypes.c_float(1.0), vp(ts), vp(ti), vp(tc),
        ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)), "b200ms_sign_candidates_device")
    return tfs.to_np((ts, ti, tc))


def assert_sign_order(got, S, allowed, what):
    ts, ti, tc = got
    want = so.topk(S, len(ti), allowed)
    assert int(tc) == len(want) and ti[:len(want)].tolist() == want, what
    assert np.array_equal(ts[:len(want)], S[want].astype(np.float32)), what
    assert (ti[len(want):] == -1).all(), what


@pytest.mark.parametrize("scale", ["bf16", "int8", "fp8"], indirect=True)
def test_sign_stage_past_4gib(scale):
    idx, dtype = scale.idx, scale.dtype
    n, rows = idx.n_pages, idx.n_rows_padded
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    signs = _aligned_bytes(rows * 16, DEV, 16)
    try:
        idx.h.check(nat.lib.b200ms_sign_rows(idx.h.ptr, 0, n, ctypes.c_void_p(signs.data_ptr()), stream), "b200ms_sign_rows")
        want_rows = sr.sign_rows_of(dtype, idx.packed_rows())
        got_rows = signs.view(rows, 16)
        past = FOUR_GIB // idx.row_bytes
        assert torch.equal(got_rows[:past], want_rows[:past]) and torch.equal(got_rows[past:], want_rows[past:])
        idx.h.check(nat.lib.b200ms_set_sign_rows(idx.h.ptr, ctypes.c_void_p(signs.data_ptr()), rows, stream),
                    "b200ms_set_sign_rows")
        S = sr.sign_reference(want_rows, scale.lens, [so.quantise_query(q, 127.0) for q in scale.qs])
        del want_rows
        # every page once: query 0 under disjoint masks of at most 4096 pages (more units than SMs: the filtered plan)
        perm = np.random.default_rng(3).permutation(n)
        parts = np.array_split(perm, -(-n // 4096))
        allow = np.zeros((len(parts), n), bool)
        for m, part in enumerate(parts):
            allow[m, part] = True
        masks = torch.from_numpy(np.stack([idx.mask_from_pages(a) for a in allow]).view(np.int32)).to(DEV)
        index = torch.arange(len(parts), dtype=torch.int32, device=DEV)
        ts, ti, tc = sign_candidates(idx, [scale.qs[0]] * len(parts), 4096, masks, index)
        for m in range(len(parts)):
            assert_sign_order((ts[m], ti[m], tc[m]), S[0], allow[m], f"{dtype} mask {m}")
        assert np.array_equal(np.sort(np.concatenate([ti[m, :tc[m]] for m in range(len(parts))])), np.arange(n))
        # the unmasked batch of the module's 13 queries
        ts, ti, tc = sign_candidates(idx, scale.qs, 4096)
        for qi in range(len(scale.qs)):
            assert_sign_order((ts[qi], ti[qi], tc[qi]), S[qi], None, f"{dtype} q{qi}")
        print(f"\n[scale] {dtype}: sign stage checked on {n} pages, {rows * 16 / 2**20:.0f} MiB of sign rows, {len(parts)} masks")
    finally:
        torch.cuda.synchronize(DEV)
        idx._attached = False
        idx._attach()  # set_corpus detaches the sign rows before their buffer goes
        del signs
