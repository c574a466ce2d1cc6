"""The FDE candidate stage (encoder, scan, candidate top-k) across the configurations the C-ABI accepts, not only the
reference's one (20 repetitions x 2^5 partitions x 16 dims = 10240).

(a) the encoder against the C oracle bit for bit: ksim 1..8, proj 1..64, proj << ksim below and at 512, 1..40
    repetitions, fill_empty_partitions, final projections; items of 0..4097 rows (the 2048-row segment boundary); f32 and
    bf16 sources; and b200ms_fde_encode_corpus (rebuild from packed rows) against add_pages;
(b) the scan against float64 on every path (wgmma, SIMT by option, by shape, by a base that is not 128-byte aligned) for
    every query-count class and dimension, including dimensions whose queries do not fit shared memory;
(c) the candidate top-k at the README's scale (131072 pages x 10240 dims): the float sliced top-k with exact ties across
    slices, negative scores and an allow mask;
(d) two-stage search end to end on three non-default configurations;
(e) a refused b200ms_fde_configure_ex leaves the handle's configuration as it was."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200 import fde  # noqa: E402
from morphik_core_b200.catalog import PageCatalog  # noqa: E402
from morphik_core_b200.index import MaxSimIndex, _vp  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import oracle_scores  # noqa: E402

# (ksim, proj, reps, fill_empty_partitions, final_projection_dimension) -- the same table as tests/test_fde_oracle_cpu.py
CONFIGS = [
    (1, 8, 1, False, 0),      # 2 partitions, 16 of 512 threads busy
    (3, 64, 7, True, 0),      # proj 64: proj << ksim = 512
    (8, 2, 1, True, 1000),    # 256 partitions: proj << ksim = 512; final projection wider than the encoding
    (5, 16, 40, False, 0),    # the reference's partitions and projection, 40 repetitions (20480 dims)
    (8, 1, 3, False, 0),      # proj 1
    (3, 3, 7, True, 16008),   # proj 3; final projection a multiple of 8 but not of 64
    (5, 16, 20, True, 16008),
    (4, 1, 40, True, 0),
]
CONFIG_IDS = [f"k{c[0]}-p{c[1]}-r{c[2]}-f{int(c[3])}-d{c[4]}" for c in CONFIGS]
ITEM_ROWS = (1, 0, 2, 2047, 2048, 2049, 4097)  # kFdeMaxSeg = 2048 rows are partitioned per segment
U = 2.0 ** -24  # fp32 unit roundoff


def cfg_of(ksim=5, proj=16, reps=20, fill=False, final=0, seed=1):
    return fde.FixedDimensionalEncodingConfig(num_repetitions=reps, num_simhash_projections=ksim, projection_dimension=proj,
                                              fill_empty_partitions=fill, final_projection_dimension=final, seed=seed)


def unit_rows(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-30)


def oracle_fde(x, cfg, m, is_doc):
    return orc.fde_encode_c_ex(x, m.simhash, m.ams_index, m.ams_sign, cfg.scale, is_doc, cfg.projection_dimension,
                               cfg.fill_empty_partitions, m.final_index, m.final_sign, cfg.final_projection_dimension)


def vp(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(ctypes.c_void_p)


def configure_raw(idx, reps, ksim, proj, sh, ai, sg, final_dim=0, fi=None, fs=None, fill=0):
    return nat.lib.b200ms_fde_configure_ex(idx.h.ptr, reps, ksim, proj, ctypes.c_float(1.0 / np.sqrt(max(proj, 1))), vp(sh),
                                           vp(ai), vp(sg), fill, final_dim, vp(fi), vp(fs))


# ------------------------------------------------------------------------------------------------ (a) encoder
@pytest.mark.parametrize("conf", CONFIGS, ids=CONFIG_IDS)
def test_encoder_configuration_sweep_bit_exact(conf):
    cfg = cfg_of(*conf)
    m = fde.fde_matrices_full(cfg)
    idx = MaxSimIndex(dtype="bf16")
    fde.configure_handle(idx, cfg, m)
    assert nat.lib.b200ms_fde_dim(idx.h.ptr) == cfg.fde_dimension
    rng = np.random.default_rng(sum(conf[:3]) + conf[4])
    items = [unit_rows(rng, n) for n in ITEM_ROWS]
    for src in ("f32", "bf16"):
        if src == "f32":
            dev_items, host_items = items, items
        else:
            dev_items = [torch.from_numpy(x).bfloat16().cuda() for x in items]
            host_items = [orc.bf16_round_np(x) for x in items]
        for is_doc in (False, True):
            got = fde.encode_items(idx, dev_items, is_doc, cfg.fde_dimension).cpu().numpy()
            assert got.shape == (len(items), cfg.fde_dimension)
            for i, x in enumerate(host_items):
                want = oracle_fde(x, cfg, m, is_doc)
                assert np.array_equal(got[i], want), (conf, src, is_doc, ITEM_ROWS[i], np.abs(got[i] - want).max())
            assert not got[1].any()  # the empty item

    # b200ms_fde_encode_corpus (first_page > 0, several batches) reproduces add_pages' rows from the packed bf16 rows
    lens = [3, 0, 2049, 1, 40, 2, 77, 2048, 5, 33]
    pages = [orc.bf16_round_np(unit_rows(rng, n)) for n in lens]
    two = fde.TwoStageIndex(dtype="bf16", config=cfg, matrices=m)
    two.add_pages(pages[:6])
    two.add_pages(pages[6:])
    F0, inv0 = [t.clone() for t in two.fde_rows()]
    two.rebuild_from_index(batch_pages=4)
    F1, inv1 = two.fde_rows()
    assert torch.equal(F0.view(torch.int16), F1.view(torch.int16)) and torch.equal(inv0, inv1), conf
    want = np.stack([orc.bf16_round_np(oracle_fde(p, cfg, m, True)) for p in pages])
    assert np.array_equal(F1.float().cpu().numpy(), want)


# ------------------------------------------------------------------------------------------------ (b) scan
SCAN_DIMS = (8, 64, 1280, 10240, 16008, 20480, 40960, 65544)  # 65544 floats: not even one query fits 227 KB of smem
SCAN_PAGES = (1, 127, 128, 129, 128 * 9 + 37)
SCAN_QS = (1, 2, 3, 4, 5, 31, 32, 33, 64, 65, 128, 129, 257)
# path -> (fde_gemm, base offset in bytes); "simt_shape" uses fde_gemm=1 on shapes the wgmma scan does not take
SCAN_PATHS = {"wgmma": (1, 0), "simt_option": (0, 0), "simt_shape": (1, 0), "simt_offset": (1, 16)}


def _wgmma_shape(fd, n_pages):
    return fd % 64 == 0 and n_pages >= 128


def _scan_cases():
    cases = []
    for path in SCAN_PATHS:
        shapes = [(fd, n) for fd in SCAN_DIMS for n in SCAN_PAGES
                  if (_wgmma_shape(fd, n) if path == "wgmma" else not _wgmma_shape(fd, n) if path == "simt_shape" else True)]
        dims = sorted({fd for fd, _ in shapes})
        for i in range(max(len(SCAN_QS), len(dims))):
            fd = dims[i % len(dims)]
            pages = [n for f, n in shapes if f == fd]
            cases.append((path, fd, pages[(i // len(dims) + i) % len(pages)], SCAN_QS[i % len(SCAN_QS)]))
    return cases


SCAN_CASES = _scan_cases()
_scan_handles = {}


def _scan_handle(fd):
    """A handle whose fde_dim is fd (the scan reads nothing else of the configuration)."""
    if fd not in _scan_handles:
        idx = MaxSimIndex(dtype="bf16")
        fde.configure_handle(idx, cfg_of(ksim=1, proj=8, reps=1, final=fd))
        _scan_handles[fd] = idx
    return _scan_handles[fd]


def _run_scan(idx, F_flat, off_elems, inv, q, n_pages, ld, sentinel):
    n_q, fd = q.shape
    scores = torch.full((n_q + 1, ld), sentinel, dtype=torch.float32, device="cuda")
    before = idx.launch_count()
    with torch.cuda.device(0):
        idx.h.check(nat.lib.b200ms_fde_scan(idx.h.ptr, _vp(F_flat[off_elems:]), _vp(inv), n_pages, _vp(q), n_q, _vp(scores), ld,
                                            idx._stream()), "b200ms_fde_scan")
    torch.cuda.synchronize()
    return scores, idx.launch_count() - before


def test_scan_cases_cover_every_path_query_class_and_dimension():
    for path in SCAN_PATHS:
        mine = [c for c in SCAN_CASES if c[0] == path]
        assert {c[3] for c in mine} == set(SCAN_QS), path
        want_dims = {fd for fd in SCAN_DIMS if path != "wgmma" or fd % 64 == 0}
        assert {c[1] for c in mine} == want_dims, path
    assert {c[2] for c in SCAN_CASES} == set(SCAN_PAGES)


@pytest.mark.parametrize("path,fd,n_pages,n_q", SCAN_CASES, ids=[f"{p}-d{f}-n{n}-q{q}" for p, f, n, q in SCAN_CASES])
def test_scan_matrix_against_float64(path, fd, n_pages, n_q):
    gemm, off_bytes = SCAN_PATHS[path]
    idx = _scan_handle(fd)
    idx.set_option("fde_gemm", gemm)
    gen = torch.Generator(device="cuda").manual_seed(fd * 1000 + n_pages * 7 + n_q)
    ld = n_pages + 3  # ld > n_pages: the columns past the corpus must keep the sentinel
    sentinel = -12345.5
    off = off_bytes // 2
    F_flat = torch.zeros(n_pages * fd + off, dtype=torch.bfloat16, device="cuda")
    F = F_flat[off:].view(n_pages, fd)
    zero_rows = torch.tensor([p for p in (n_pages - 2, 5) if 0 <= p < n_pages], dtype=torch.int64, device="cuda")

    # 1) Gaussian FDEs and fp32 queries: error within the path's model, relative to sum_i |q_i F_pi| * inv_p
    F.copy_(torch.randn((n_pages, fd), generator=gen, device="cuda").to(torch.bfloat16))
    F[zero_rows] = 0
    inv = 1.0 / torch.clamp(F.float().norm(dim=1), min=1e-30)
    inv[zero_rows] = 0
    q = torch.randn((n_q, fd), generator=gen, device="cuda")
    scores, launches = _run_scan(idx, F_flat, off, inv, q, n_pages, ld, sentinel)
    Fd, qd, invd = F.double(), q.double(), inv.double()
    want = (qd @ Fd.T) * invd
    mag = (qd.abs() @ Fd.abs().T) * invd
    if path == "wgmma":
        # hi + lo bf16 split of the query (~2^-17 relative per term) and fp32 tensor-core accumulation over K terms
        assert launches == 2 * ((n_q + 127) // 128)
        bound = (2.0 ** -17 + fd * 2 * U) * mag + U * want.abs()
    else:
        # fp32 fma chains: at most K roundings per score (plus the product with inv)
        props = torch.cuda.get_device_properties(0)
        optin = getattr(props, "shared_memory_per_block_optin", 232448)
        res = min(4, n_q, optin // (4 * fd))
        assert launches == -(-n_q // (res if res > 0 else 4))
        bound = fd * U * mag + U * want.abs()
    got = scores[:n_q, :n_pages].double()
    err = (got - want).abs()
    assert bool((err <= bound).all()), (path, fd, n_pages, n_q, float((err / bound.clamp(min=1e-300)).max()))
    assert bool((scores[:n_q, zero_rows] == 0).all())
    assert bool((scores[:n_q, n_pages:] == sentinel).all()) and bool((scores[n_q] == sentinel).all())

    # 2) small integers: every partial sum is exact in fp32 (|sum| <= 9 * K < 2^24) and the query's lo half is 0, so each
    # score is exactly fp32(dot) * inv -- a dropped, repeated or misplaced term changes it
    F.copy_(torch.randint(-3, 4, (n_pages, fd), generator=gen, device="cuda").to(torch.bfloat16))
    F[zero_rows] = 0
    inv = (1.0 / torch.clamp(F.float().norm(dim=1), min=1.0)).float()
    inv[zero_rows] = 0
    q = torch.randint(-3, 4, (n_q, fd), generator=gen, device="cuda").float()
    scores, _ = _run_scan(idx, F_flat, off, inv, q, n_pages, ld, sentinel)
    dots = (q.double() @ F.double().T)  # exact: integers below 2^53
    want = dots.float() * inv  # one fp32 rounding of an exact fp32 value, as in the kernel's epilogue
    assert torch.equal(scores[:n_q, :n_pages], want), (path, fd, n_pages, n_q)
    assert bool((scores[:n_q, n_pages:] == sentinel).all()) and bool((scores[n_q] == sentinel).all())


# ------------------------------------------------------------------------------------------------ (c) candidate top-k
def test_candidate_topk_at_readme_scale(monkeypatch):
    n, fd = 131072, 10240
    two = fde.TwoStageIndex(dtype="bf16")
    two._grow(n)
    F, inv = two._F[:n], two._inv[:n]
    gen = torch.Generator(device="cuda").manual_seed(3)
    for c in range(0, n, 16384):  # rows in a positive cone: every pairwise cosine is positive
        F[c:c + 16384] = (torch.randn((16384, fd), generator=gen, device="cuda") + 3.0).to(torch.bfloat16)
        inv[c:c + 16384] = torch.rsqrt(F[c:c + 16384].float().square().sum(dim=1))
    src = torch.tensor([(i * 613) % 65536 for i in range(100)], dtype=torch.int64, device="cuda")
    dst = src + 65536  # same tile row, the other half of the corpus: a different top-k slice for every slice count
    F[dst] = F[src]
    inv[dst] = inv[src]
    two._n = n
    queries = [F[src[0]].float(),                                 # ties at the top: src[0] and dst[0] score the same
               -F[src[1]].float(),                                # every cosine negative
               torch.randn(fd, generator=gen, device="cuda"),     # mixed signs
               F[src].float().sum(dim=0),                         # the duplicated rows near the top
               -torch.randn(fd, generator=gen, device="cuda").abs()]
    qf = torch.stack(queries).contiguous()
    # candidates() encodes its queries; here they are FDE vectors already, so the selection is tested on its own
    monkeypatch.setattr(fde, "encode_items", lambda index, items, is_doc, dim: torch.stack(list(items)).contiguous())
    s = two.fde_scores(qf)[:, :n]
    torch.cuda.synchronize()
    s_np = s.cpu().numpy()
    assert (s_np[1] < 0).all() and (s_np[4] < 0).all() and (s_np[2] > 0).any() and (s_np[2] < 0).any()
    assert s_np[0, int(src[0])] == s_np[0, int(dst[0])]
    # the scan's own scores against float64 (the wgmma bound of test_scan_matrix_against_float64)
    for c in range(0, n, 16384):
        Fd = F[c:c + 16384].double()
        want = (qf.double() @ Fd.T) * inv[c:c + 16384].double()
        mag = (qf.double().abs() @ Fd.abs().T) * inv[c:c + 16384].double()
        assert bool(((s[:, c:c + 16384].double() - want).abs() <= (2.0 ** -17 + fd * 2 * U) * mag + U * want.abs()).all())

    rng = np.random.default_rng(4)
    allow = rng.random(n) < 0.5
    allow[src.cpu().numpy()[:50]] = True
    allow[dst.cpu().numpy()[:50]] = True
    mask_dev = torch.from_numpy(PageCatalog.mask_words(allow).view(np.int32)).cuda()  # bit p & 31 of word p >> 5
    ids_all = np.arange(n, dtype=np.int64)
    for k in (10, 1000, 4096):
        for use_mask in (False, True):
            ti, ts, tc = two.candidates(queries, k, allow_mask_dev=mask_dev if use_mask else None)
            torch.cuda.synchronize()
            ti, ts, tc = ti.cpu().numpy(), ts.cpu().numpy(), tc.cpu().numpy()
            ids = ids_all[allow] if use_mask else ids_all
            for qi in range(len(queries)):
                order = np.lexsort((ids, -s_np[qi, ids].astype(np.float64)))[:k]
                want_ids = ids[order]
                assert int(tc[qi]) == k, (k, use_mask, qi)
                assert np.array_equal(ti[qi], want_ids), (k, use_mask, qi, np.flatnonzero(ti[qi] != want_ids)[:5])
                assert np.array_equal(ts[qi], s_np[qi, want_ids]), (k, use_mask, qi)
            # the exact tie at the top crosses slices and resolves to the lower id
            assert ti[0][:2].tolist() == [int(src[0]), int(dst[0])] and ts[0][0] == ts[0][1]


# ------------------------------------------------------------------------------------------------ (d) two-stage end to end
TWO_STAGE = [
    ("final16008", cfg_of(final=16008), 300),       # fde_dim % 64 != 0: always the SIMT scan, 64 KB per query
    ("ksim8-proj2", cfg_of(ksim=8, proj=2), 300),   # 256 partitions x 2 dims
    ("reps40-small", cfg_of(reps=40), 120),         # 20480 dims on a corpus under 128 pages: SIMT, 80 KB per query
]


@pytest.mark.parametrize("name,cfg,n_pages", TWO_STAGE, ids=[t[0] for t in TWO_STAGE])
def test_two_stage_search_on_non_default_configurations(name, cfg, n_pages):
    rng = np.random.default_rng(77)
    lens = [int(x) for x in rng.integers(20, 200, size=n_pages)]
    pages = [unit_rows(rng, n) for n in lens]
    queries = [unit_rows(rng, t) for t in (32, 20, 32, 40, 7)]
    planted = {}
    for qi, q in enumerate(queries):  # 6 relevant pages per query, none shared
        planted[qi] = {3 + qi + 20 * j for j in range(6)}
        for j, p in enumerate(sorted(planted[qi])):
            n = min(len(q), lens[p])
            pages[p][:n] = q[:n] + (0.02 * (j + 1)) * rng.standard_normal((n, 128)).astype(np.float32)
            pages[p] /= np.linalg.norm(pages[p], axis=1, keepdims=True)
    pages = [orc.bf16_round_np(p) for p in pages]  # bf16-valued, so that the FDEs rebuilt from packed rows are identical
    m = fde.fde_matrices_full(cfg)
    two = fde.TwoStageIndex(dtype="bf16", config=cfg, matrices=m)
    two.add_pages(pages[: n_pages // 2])
    two.add_pages(pages[n_pages // 2:])
    k, n_cand = 5, 40
    cand, cand_scores, cand_counts = two.candidates(queries, n_cand)
    torch.cuda.synchronize()
    cand, cand_scores = cand.cpu().numpy(), cand_scores.cpu().numpy()
    assert (cand_counts.cpu().numpy() == n_cand).all()
    # first stage against float64: the scores of the chosen pages, and no page left out that beats a chosen one by more
    # than the error bound
    F = np.stack([orc.bf16_round_np(oracle_fde(p, cfg, m, True)) for p in pages]).astype(np.float64)
    inv = np.float32(1.0) / np.sqrt((F * F).sum(axis=1)).astype(np.float32)
    fd = cfg.fde_dimension
    for qi, q in enumerate(queries):
        qf = oracle_fde(q, cfg, m, False).astype(np.float64)
        s = (F @ qf) * inv
        # (b)'s wgmma bound, covering the SIMT one, + 4 ulp for the device's rsqrtf of the row norm
        bound = (2.0 ** -17 + fd * 2 * U) * ((np.abs(F) @ np.abs(qf)) * inv) + 4 * U * np.abs(s)
        assert np.all(np.abs(cand_scores[qi] - s[cand[qi]]) <= bound[cand[qi]]), (name, qi)
        assert len(set(cand[qi].tolist())) == n_cand
        left_out = np.setdiff1d(np.arange(n_pages), cand[qi])
        assert s[left_out].max() <= s[cand[qi]].min() + 2 * bound.max(), (name, qi)
    # rerank == MaxSim oracle restricted to the candidates (ties -> earlier candidate slot)
    got_s, got_i, _ = two.search(queries, k, n_candidates=n_cand)
    for qi, q in enumerate(queries):
        full = oracle_scores("bf16", [q], pages)[0]
        cs = full[cand[qi]]
        order = np.lexsort((np.arange(n_cand), -cs))[:k]
        assert got_i[qi].tolist() == cand[qi][order].tolist(), (name, qi)
        np.testing.assert_allclose(got_s[qi], cs[order], rtol=3e-5)
        assert len(planted[qi] & set(got_i[qi].tolist())) >= 4, (name, qi)
    F0, inv0 = [t.clone() for t in two.fde_rows()]
    two.rebuild_from_index(batch_pages=n_pages // 3)
    F1, inv1 = two.fde_rows()
    assert torch.equal(F0.view(torch.int16), F1.view(torch.int16)) and torch.equal(inv0, inv1)


# ------------------------------------------------------------------------------------------------ (e) refused configuration
def test_refused_configuration_leaves_the_handle_as_it_was():
    cfg_a = cfg_of(reps=3)
    a = fde.fde_matrices_full(cfg_a)
    idx = MaxSimIndex(dtype="bf16")
    fde.configure_handle(idx, cfg_a, a)
    rng = np.random.default_rng(8)
    items = [unit_rows(rng, n) for n in (1, 9, 300, 2049)]

    def encode():
        return np.concatenate([fde.encode_items(idx, items, d, cfg_a.fde_dimension).cpu().numpy() for d in (False, True)])

    first = encode()
    assert np.array_equal(first[0], oracle_fde(items[0], cfg_a, a, False))
    assert np.array_equal(first[len(items)], oracle_fde(items[0], cfg_a, a, True))

    def refused(*args, **kw):
        rc = configure_raw(idx, *args, **kw)
        assert rc == -1, (args, rc)  # B200MS_EINVAL
        msg = nat.lib.b200ms_last_error(idx.h.ptr)
        assert msg and b"fde_configure" in msg, msg
        assert nat.lib.b200ms_fde_dim(idx.h.ptr) == cfg_a.fde_dimension
        assert np.array_equal(encode(), first), args[:3]

    # B: A's shape (so that nothing is read out of range) and other matrices, with one final_index entry past final_dim
    b = fde.fde_matrices_full(cfg_of(reps=3, final=1000, seed=99))
    bad_fi = b.final_index.copy()
    bad_fi[len(bad_fi) // 2] = 1000
    refused(3, 5, 16, b.simhash, b.ams_index, b.ams_sign, 1000, bad_fi, b.final_sign)
    bad_fi[len(bad_fi) // 2] = -1
    refused(3, 5, 16, b.simhash, b.ams_index, b.ams_sign, 1000, bad_fi, b.final_sign)

    def mats(reps, ksim, proj):
        return (np.ones((reps, 128, ksim), np.float32), np.zeros((reps, 128), np.int32), np.ones((reps, 128), np.float32))

    refused(1, 9, 1, *mats(1, 9, 1))          # ksim 9
    refused(1, 1, 65, *mats(1, 1, 65))        # proj 65
    refused(1, 6, 16, *mats(1, 6, 16))        # proj << ksim = 1024
    refused(1, 1, 3, *mats(1, 1, 3))          # proj << ksim = 6, not a multiple of 8
    refused(0, 5, 16, *mats(1, 5, 16))        # no repetitions
    refused(65536, 1, 8, *mats(65536, 1, 8))  # more repetitions than the encoder's grid.y holds
    sh, ai, sg = (x.copy() for x in (b.simhash, b.ams_index, b.ams_sign))
    ai[2, 127] = 16                            # ams_index out of range, in the last repetition
    refused(3, 5, 16, sh, ai, sg)
    ai[2, 127] = -1
    refused(3, 5, 16, sh, ai, sg)
    refused(3, 5, 16, b.simhash, b.ams_index, b.ams_sign, 12, b.final_index, b.final_sign)  # final_dim % 8 != 0
    refused(3, 5, 16, b.simhash, b.ams_index, b.ams_sign, 1000, None, b.final_sign)
    refused(3, 5, 16, None, b.ams_index, b.ams_sign)

    # the boundary configurations of the encoder sweep are accepted, and A can be restored afterwards
    for conf in CONFIGS:
        cfg = cfg_of(*conf)
        fde.configure_handle(idx, cfg)
        assert nat.lib.b200ms_fde_dim(idx.h.ptr) == cfg.fde_dimension
    fde.configure_handle(idx, cfg_a, a)
    assert np.array_equal(encode(), first)
