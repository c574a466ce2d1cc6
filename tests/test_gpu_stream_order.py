"""Calls on one handle, in flight on different streams at once (run with -m gpu on an H100).

Every case of tests/stream_order_cases.py issues call A on stream S1 and, as soon as A returns, call B on stream S2 (or on
the handle's own stream, which the *_host entry points, set_corpus* and fde_configure* use).  Both share the handle's
scratch: packed queries, score matrices, metadata uploads, top-k and grouping buffers, FDE scratch, the corpus tables.  The
library orders a handle's calls in the order they were made, so both calls must return, bit for bit, what they return when
run alone -- every score, id, count, token score, best row, map entry and FDE value.  All these paths are deterministic for
a fixed launch shape.

A is long and multi-launch so that B's kernels are queued while A's still run: a full scan of 8192 pages x 512 rows (1 GiB
in bf16) by 48 queries x 32 tokens (12 query tiles, three passes of four resident tiles), reranks and explanations of 64
candidates per query, host-tier reranks that gather their pages over PCIe, FDE encodings of the whole corpus.  B uses other
queries, candidates and masks than A, so a call that reads the other's scratch returns something else.

The alone runs of the first case are anchored to oracle.scoring for every corpus dtype.
"""
import copy
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import stream_order_cases as soc  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex, _aligned_bytes  # noqa: E402
from oracle.scoring import TOL, assert_scores, oracle_scores  # noqa: E402

DEV = torch.device("cuda", 0)
N_PAGES, HOST_PAGES, PAGE_ROWS = 8192, 2048, 512
OTHER_PAGES, OTHER_ROWS = 512, 256  # the corpus set_corpus* attaches in mid-flight
LENS = {"a": [32] * 48, "b": [20, 33, 7, 64]}
N_CAND = {"a": 64, "b": 40}
B_IDS = 400  # B's candidate ids stay below this, so they name pages of the other corpus too
K, PER_DOC, MAP_ROWS = 16, 2, 16
# FDE configurations: (seed, reps, ksim, proj_dim, final_dim); "main" and "ex" end in a final projection (scratch fde_tmp)
FDE = {"main": (11, 20, 4, 8, 512), "plain": (12, 10, 3, 16, 0), "ex": (13, 8, 3, 8, 256)}


def vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def cstream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def unit_rows(gen, n, dtype):
    x = torch.randn((n, nat.DIM), generator=gen, device=DEV)
    return (x / x.norm(dim=1, keepdim=True)).to(dtype)


def make_index(kind, rows, n_pages, page_rows):
    dtype, b1, tier = soc.KINDS[kind]
    idx = MaxSimIndex(dtype=dtype, tier=tier)
    if b1 is not None:
        idx.set_option("b1_tensor", b1)
    idx.add_pages(list(rows.split(page_rows)))
    idx._attach()
    assert idx.n_pages == n_pages
    return idx


def fde_configure(h, name):
    seed, reps, ksim, proj, final = FDE[name]
    rng = np.random.default_rng(seed)
    sh = rng.standard_normal((reps, nat.DIM, ksim)).astype(np.float32)
    ai = rng.integers(0, proj, size=(reps, nat.DIM)).astype(np.int32)
    sg = rng.choice(np.float32([-1, 1]), size=(reps, nat.DIM)).astype(np.float32)
    c = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    if final == 0:
        h.check(nat.lib.b200ms_fde_configure(h.ptr, reps, ksim, proj, ctypes.c_float(1.0), c(sh), c(ai), c(sg)),
                "b200ms_fde_configure")
    else:
        inner = reps * (1 << ksim) * proj
        fi = rng.integers(0, final, size=inner).astype(np.int32)
        fs = rng.choice(np.float32([-1, 1]), size=inner).astype(np.float32)
        h.check(nat.lib.b200ms_fde_configure_ex(h.ptr, reps, ksim, proj, ctypes.c_float(1.0), c(sh), c(ai), c(sg), 0, final,
                                                c(fi), c(fs)), "b200ms_fde_configure_ex")
    return int(nat.lib.b200ms_fde_dim(h.ptr))


class Ctx:
    """One corpus kind: the index under test, A's and B's inputs, and what the cases attach or configure in mid-flight."""

    def __init__(self, kind):
        dtype, _, tier = soc.KINDS[kind]
        self.kind, self.dtype, self.tier = kind, dtype, tier
        self.n_pages = HOST_PAGES if tier == "host" else N_PAGES
        g = torch.Generator(device=DEV)
        g.manual_seed(2025)
        self.rows = unit_rows(g, self.n_pages * PAGE_ROWS, torch.bfloat16)  # the corpus as bf16 values (oracle input)
        self.idx = make_index(kind, self.rows, self.n_pages, PAGE_ROWS)
        self.q = {w: unit_rows(g, sum(LENS[w]), torch.float32) for w in LENS}
        self.q_list = {w: list(self.q[w].split(LENS[w])) for w in LENS}
        self.q_host = {w: [x.cpu().numpy() for x in self.q_list[w]] for w in LENS}
        self.q_pin = {w: self.q[w].cpu().pin_memory() for w in LENS}
        rng = np.random.default_rng(7)
        self.cand = {}
        for w, n_q in (("a", len(LENS["a"])), ("b", len(LENS["b"]))):
            c = rng.integers(0, self.n_pages if w == "a" else B_IDS, size=(n_q, N_CAND[w]))
            c[:, 5::9] = -1  # unused slots
            c[:, 3] = c[:, 1]  # a page in two slots
            self.cand[w] = torch.from_numpy(c).to(DEV)
        self.page_doc = (torch.arange(self.n_pages, device=DEV, dtype=torch.int32) // 4).contiguous()
        self.n_docs = self.n_pages // 4
        words = [self.idx.mask_from_pages(rng.random(self.n_pages) < f) for f in (0.5, 0.1)]
        self.masks = torch.from_numpy(np.stack(words).view(np.int32)).to(DEV)
        self.mask_index = {w: torch.tensor([i % 3 - 1 for i in range(len(LENS[w]))], dtype=torch.int32, device=DEV) for w in LENS}
        self.host_masks = {w: [None if i % 3 == 0 else words[i % 3 - 1] for i in range(len(LENS[w]))] for w in LENS}
        self.hq = rng.integers(0, 256, size=16).astype(np.uint8)  # a packed query row for hamming_batch
        self.merge_in = {}
        self.xchg = {}
        for w in LENS:
            n_q = len(LENS[w])
            sc = torch.from_numpy(rng.standard_normal((n_q, 2 * K)).astype(np.float32)).to(DEV)
            ids = torch.from_numpy(rng.permutation(10 * n_q * K)[: n_q * 2 * K].reshape(n_q, 2 * K)).to(DEV)
            self.merge_in[w] = (sc, ids)
            xb = torch.zeros(int(nat.lib.b200ms_xchg_bytes(n_q, K)), dtype=torch.uint8, device=DEV)
            xb[: n_q * K * 8].copy_(ids[:, :K].reshape(-1).view(torch.uint8))
            xb[n_q * K * 8: n_q * K * 12].copy_(sc[:, :K].reshape(-1).contiguous().view(torch.uint8))
            self.xchg[w] = xb
        self.idx.comm_init(bytes(128), 0, 1)  # world 1: bcast and allgather_topk without NCCL
        self._other = self._twin = self._fde = None
        torch.cuda.synchronize()

    def other(self):
        """A different, smaller corpus of the same kind (its own index keeps its rows alive)."""
        if self._other is None:
            g = torch.Generator(device=DEV)
            g.manual_seed(99)
            self._other = make_index(self.kind, unit_rows(g, OTHER_PAGES * OTHER_ROWS, torch.bfloat16), OTHER_PAGES, OTHER_ROWS)
        return self._other

    def twin(self):
        """The same packed rows behind a second handle."""
        if self._twin is None:
            t = MaxSimIndex(dtype=self.dtype)
            t.adopt_packed(self.idx.packed_rows(), [PAGE_ROWS] * self.n_pages)
            t._attach()
            self._twin = copy.copy(self)
            self._twin.idx = t
        return self._twin

    def fde(self):
        """FDE configuration "main" on the handle, and the finalized FDE matrix of the whole corpus."""
        if self._fde is None:
            dim = fde_configure(self.idx.h, "main")
            out = torch.empty((self.n_pages, dim), dtype=torch.float32, device=DEV)
            rows = torch.empty((self.n_pages, dim), dtype=torch.bfloat16, device=DEV)
            inv = torch.empty((self.n_pages,), dtype=torch.float32, device=DEV)
            h = self.idx.h
            h.check(nat.lib.b200ms_fde_encode_corpus(h.ptr, 0, self.n_pages, vp(out), cstream()), "fde_encode_corpus")
            h.check(nat.lib.b200ms_fde_finalize(h.ptr, vp(out), self.n_pages, vp(rows), vp(inv), cstream()), "fde_finalize")
            torch.cuda.synchronize()
            self._fde = (dim, rows, inv)
        return self._fde

    def reset(self):
        """Back to the state every run starts from: the corpus attached, FDE configuration "main"."""
        torch.cuda.synchronize()
        self.idx._attached = False
        self.idx._attach()
        if self._fde is not None:
            fde_configure(self.idx.h, "main")
        torch.cuda.synchronize()


@functools.lru_cache(maxsize=None)
def context(kind):
    return Ctx(kind)


# ---- the calls: each returns (outputs, after); `after` (or None) runs once the other call of the pair has been issued
def three(names, t):
    return dict(zip(names, t))


TOPK = ("scores", "ids", "counts")
DOCS = ("page_scores", "page_ids", "page_counts", "doc_counts")


def c_search_device(x, w):
    return three(TOPK, x.idx.search_device(x.q[w], LENS[w], K)), None


def c_search_device_masked(x, w):
    return three(TOPK, x.idx.search_device(x.q[w], LENS[w], K, allow_mask_dev=x.masks, mask_index_dev=x.mask_index[w])), None


def c_search_host(x, w):
    return three(TOPK, x.idx.search_host(x.q_host[w], K)), None


def c_search_host_masked(x, w):
    return three(TOPK, x.idx.search_host_masked(x.q_host[w], K, x.host_masks[w])), None


def c_rerank_device(x, w):
    return three(TOPK, x.idx.rerank(x.q[w], LENS[w], x.cand[w][0].contiguous(), K)), None


def c_rerank_batch_device(x, w):
    return three(TOPK, x.idx.rerank_batch(x.q[w], LENS[w], x.cand[w], K)), None


def c_explain_device(x, w):
    return three(("token_scores", "best_rows", "sim_map"), x.idx.explain(x.q_list[w], x.cand[w], map_rows=MAP_ROWS)), None


def c_search_docs_device(x, w):
    return three(DOCS, x.idx.search_docs_device(x.q[w], LENS[w], K, PER_DOC, x.page_doc, x.n_docs, allow_mask_dev=x.masks,
                                                mask_index_dev=x.mask_index[w])), None


def c_rerank_docs_batch_device(x, w):
    return three(DOCS, x.idx.rerank_docs_batch(x.q[w], LENS[w], x.cand[w], K, PER_DOC, x.page_doc, x.n_docs)), None


def c_score_topk(x, w):
    idx, h, n_q = x.idx, x.idx.h, len(LENS[w])
    scores, goff, n_pages, _ = idx.score_groups(x.q_list[w])
    goff_c = nat.i32_array(goff.tolist())
    sdt = nat.F32 if idx.float_scores else nat.I32
    ld = scores.shape[1]
    out = {"group_scores": scores,
           "scores": torch.empty((n_q, K), dtype=torch.float32, device=DEV),
           "ids": torch.empty((n_q, K), dtype=torch.int64, device=DEV),
           "counts": torch.empty((n_q,), dtype=torch.int32, device=DEV),
           "page_scores": torch.empty((n_q, K, PER_DOC), dtype=torch.float32, device=DEV),
           "page_ids": torch.empty((n_q, K, PER_DOC), dtype=torch.int64, device=DEV),
           "page_counts": torch.empty((n_q, K), dtype=torch.int32, device=DEV),
           "doc_counts": torch.empty((n_q,), dtype=torch.int32, device=DEV)}
    scale = ctypes.c_float(idx.score_scale)
    h.check(nat.lib.b200ms_topk(h.ptr, vp(scores), sdt, n_pages, ld, goff_c, n_q, None, K, scale, 0, vp(out["scores"]),
                                vp(out["ids"]), vp(out["counts"]), cstream()), "b200ms_topk")
    h.check(nat.lib.b200ms_topk_docs(h.ptr, vp(scores), sdt, n_pages, ld, goff_c, n_q, None, vp(x.page_doc), x.n_docs, K,
                                     PER_DOC, scale, 0, vp(out["page_scores"]), vp(out["page_ids"]), vp(out["page_counts"]),
                                     vp(out["doc_counts"]), cstream()), "b200ms_topk_docs")
    return out, None


def c_utilities(x, w):
    idx, h, n_q = x.idx, x.idx.h, len(LENS[w])
    out = {"bits": idx.sign_pack(x.q[w])}
    out["hamming"] = idx.hamming_distance_batch(x.hq, out["bits"])
    lens_c = nat.i32_array(LENS[w])
    packed = _aligned_bytes(int(nat.lib.b200ms_padded_rows(lens_c, n_q)) * nat.ROW_BYTES[nat.I8], DEV)
    h.check(nat.lib.b200ms_pack_pages(h.ptr, vp(x.q[w]), nat.F32, lens_c, n_q, vp(packed), nat.I8, ctypes.c_float(127.0),
                                      cstream()), "b200ms_pack_pages")
    out["packed"] = packed
    out.update(zip(("merge_scores", "merge_ids", "merge_counts"), idx.merge_topk(*x.merge_in[w], K)))
    idx.bcast(out["packed"])
    out.update(zip(("gather_scores", "gather_ids", "gather_counts"), idx.allgather_topk(x.xchg[w], n_q, K)))
    return out, None


def c_sharded_search(x, w):
    n_q = len(LENS[w])
    out = (torch.empty((n_q, K), dtype=torch.float32, device=DEV), torch.empty((n_q, K), dtype=torch.int64, device=DEV),
           torch.empty((n_q,), dtype=torch.int32, device=DEV))
    ticket = x.idx.sharded_search_begin(x.q[w], LENS[w], K, 0, out)
    return three(TOPK, out), lambda: x.idx.sharded_search_end(ticket)


def c_sharded_search_host(x, w):
    n_q = len(LENS[w])
    out = (torch.empty((n_q, K), dtype=torch.float32), torch.empty((n_q, K), dtype=torch.int64),
           torch.empty((n_q,), dtype=torch.int32))
    ticket = x.idx.sharded_search_host_begin(x.q_pin[w], LENS[w], K, 0)
    return three(TOPK, out), lambda: x.idx.sharded_search_host_end(ticket, *out)


def encode_queries(x, w, dim):
    h, n_q = x.idx.h, len(LENS[w])
    q_fde = torch.empty((n_q, dim), dtype=torch.float32, device=DEV)
    h.check(nat.lib.b200ms_fde_encode(h.ptr, vp(x.q[w]), nat.F32, nat.i32_array(LENS[w]), n_q, 0, vp(q_fde), cstream()),
            "b200ms_fde_encode")
    return q_fde


def c_fde_encode_scan(x, w):
    dim, rows, inv = x.fde()
    h, n_q = x.idx.h, len(LENS[w])
    q_fde = encode_queries(x, w, dim)
    scores = torch.empty((n_q, x.n_pages), dtype=torch.float32, device=DEV)
    h.check(nat.lib.b200ms_fde_scan(h.ptr, vp(rows), vp(inv), x.n_pages, vp(q_fde), n_q, vp(scores), x.n_pages, cstream()),
            "b200ms_fde_scan")
    return {"q_fde": q_fde, "fde_scores": scores}, None


def c_fde_encode_corpus(x, w):
    dim, _, _ = x.fde()
    h = x.idx.h
    first, n = (0, x.n_pages) if w == "a" else (1000, 2000)
    out = torch.empty((n, dim), dtype=torch.float32, device=DEV)
    rows = torch.empty((n, dim), dtype=torch.bfloat16, device=DEV)
    inv = torch.empty((n,), dtype=torch.float32, device=DEV)
    h.check(nat.lib.b200ms_fde_encode_corpus(h.ptr, first, n, vp(out), cstream()), "b200ms_fde_encode_corpus")
    h.check(nat.lib.b200ms_fde_finalize(h.ptr, vp(out), n, vp(rows), vp(inv), cstream()), "b200ms_fde_finalize")
    return {"fde": out, "fde_rows": rows, "inv_norm": inv}, None


def c_fde_configure(x, w, name="plain"):
    x.fde()
    return {"q_fde": encode_queries(x, w, fde_configure(x.idx.h, name))}, None


def c_fde_configure_ex(x, w):
    return c_fde_configure(x, w, "ex")


def c_set_corpus_search(x, w):
    o = x.other()
    x.idx.h.check(nat.lib.b200ms_set_corpus(x.idx.h.ptr, vp(o._buf), o.dtype, nat.i32_array(o._page_lens), o.n_pages),
                  "b200ms_set_corpus")
    return three(TOPK, x.idx.search_device(x.q[w], LENS[w], K)), None


def c_set_corpus_host_rerank(x, w):
    o = x.other()
    x.idx.h.check(nat.lib.b200ms_set_corpus_host(x.idx.h.ptr, vp(o._buf), o.dtype, nat.i32_array(o._page_lens), o.n_pages),
                  "b200ms_set_corpus_host")
    return three(TOPK, x.idx.rerank_batch(x.q[w], LENS[w], x.cand[w], K)), None


CALL_FNS = {name: globals()["c_" + name] for name in soc.CALLS}


def issue(x, call, w, stream):
    with torch.cuda.stream(stream):
        return CALL_FNS[call](x, w)


def finish(after, stream):
    if after is not None:
        with torch.cuda.stream(stream):
            after()


def to_host(out):
    res = {}
    for name, t in out.items():
        if t is None or isinstance(t, np.ndarray):  # no map requested / the host entry points' results
            res[name] = None if t is None else t.copy()
            continue
        t = t.detach()
        if t.dtype == torch.bfloat16:
            t = t.view(torch.int16)
        res[name] = t.cpu().numpy().copy()
    return res


def alone(x, call, w, stream):
    x.reset()
    out, after = issue(x, call, w, stream)
    finish(after, stream)
    torch.cuda.synchronize()
    return to_host(out)


def assert_same(got, want, what):
    assert got.keys() == want.keys(), what
    for name, w in want.items():
        g = got[name]
        if w is None:
            assert g is None, (what, name)
            continue
        assert g.shape == w.shape and g.dtype == w.dtype, (what, name, g.shape, w.shape)
        same = (g.view(np.uint8) == w.view(np.uint8)).reshape(g.shape + (-1,)).all(axis=-1) if g.size else np.ones(0, bool)
        if not same.all():
            first = tuple(int(i) for i in np.argwhere(~same)[0])
            raise AssertionError(f"{what}: output {name!r} differs from the call run alone in {int((~same).sum())} of "
                                 f"{same.size} entries, first at {first}: got {g[first]!r}, alone {w[first]!r}")


def check_against_oracle(x, res, n_check=6, n_sample=64):
    """The alone run of a full-scan search against oracle.scoring: each checked query's reported scores are the oracle's scores
    of the reported pages, and no sampled unreported page beats its k-th score beyond the dtype's tolerance."""
    rng = np.random.default_rng(3)
    queries = [q.cpu().numpy() for q in x.q_list["a"][:n_check]]
    for qi, q in enumerate(queries):
        n = int(res["counts"][qi])
        assert n == K, (qi, n)
        ids = res["ids"][qi, :n]
        others = np.setdiff1d(rng.choice(x.n_pages, size=n_sample, replace=False), ids)
        pages = [x.rows[p * PAGE_ROWS:(p + 1) * PAGE_ROWS].float().cpu().numpy() for p in np.concatenate([ids, others])]
        want = oracle_scores(x.dtype, [q], pages)[0]
        assert_scores(x.dtype, res["scores"][qi, :n], want[:n], f"query {qi}")
        kth = float(res["scores"][qi, n - 1])
        assert want[n:].max() <= kth + TOL[x.dtype] * max(abs(kth), 1e-3), (qi, want[n:].max(), kth)


PAIRS, IDS = soc.parametrize()


@pytest.mark.parametrize("case,kind", PAIRS, ids=IDS)
def test_calls_in_flight_together_return_their_alone_results(case, kind):
    x = context(kind)
    xb = x.twin() if case.handles == 2 else x
    s1 = torch.cuda.Stream(DEV)
    s2 = s1 if case.b_stream == "same" else torch.cuda.Stream(DEV)
    want_a = alone(x, case.a, "a", s1)
    want_b = alone(xb, case.b, "b", s2)
    if case.oracle:
        check_against_oracle(x, want_a)
    x.reset()
    xb.reset()
    out_a, after_a = issue(x, case.a, "a", s1)
    out_b, after_b = issue(xb, case.b, "b", s2)  # no synchronisation in between
    finish(after_a, s1)
    finish(after_b, s2)
    torch.cuda.synchronize()
    got_a, got_b = to_host(out_a), to_host(out_b)
    x.reset()
    assert_same(got_a, want_a, f"A = {case.a} on S1")
    assert_same(got_b, want_b, f"B = {case.b} issued while A ran")
