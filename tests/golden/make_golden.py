"""Generate the golden fixtures under tests/golden/ by EXECUTING reference code in the build container.

Run from the repo root:  MORPHIK_REFERENCE=<a morphik-core checkout> python tests/golden/make_golden.py
Needs that checkout and transformers, which is why the outputs (small .npz files) are committed next to this script.

What is executed:
  * core/utils/fast_ops.py of the checkout (loaded by file path; HAS_RUST is False here so the authoritative
    pure-Python fallbacks run): binary_quantize, binary_quantize_packed, hamming_distance(_batch).
  * transformers.models.colpali.processing_colpali.ColPaliProcessor.score_retrieval -- the port of
    colpali_engine v0.3.13 ``score_multi_vector`` that the reference calls at
    core/vector_store/fast_multivector_store.py:553-555 (colpali_engine itself is not installed; SURVEY F6).
The SQL ``max_sim`` (multi_vector_store.py:287-311) cannot be executed (no Postgres): its fixture holds only the
known answers implied by core/tests/unit/test_multivector.py and is marked ``derived``.
"""
import importlib.util
import os

import numpy as np
import torch

REF = os.environ.get("MORPHIK_REFERENCE", "")
OUT = os.path.dirname(os.path.abspath(__file__))


def load_fast_ops():
    spec = importlib.util.spec_from_file_location("ref_fast_ops", os.path.join(REF, "core/utils/fast_ops.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.HAS_RUST is False
    return mod


def gen_sign_pack(fo):
    rng = np.random.default_rng(20260922)
    x = rng.standard_normal((96, 128)).astype(np.float32)
    # edge values the Rust tests name (binary_ops.rs:299-306): 0.0 -> 0, plus -0.0, NaN, inf, denormals
    x[0, :8] = [1.0, -0.5, 0.1, -2.0, 0.0, 3.0, -1.0, 0.5]
    x[1, :8] = [1.0, -1.0, 1.0, -1.0, -1.0, 1.0, -1.0, 1.0]  # binary_ops.rs:309-319 -> 0b10100101
    x[2, :6] = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45]
    x[3] = 0.0
    packed = np.frombuffer(b"".join(fo.binary_quantize_packed(x)), dtype=np.uint8).reshape(96, 16)
    bools = np.array(fo.binary_quantize(x), dtype=bool)
    # float64 / odd dims go through the same entry point (multi_vector_store.py:334-345)
    x3 = np.array([[0.1, -0.2, 0.3], [-0.1, 0.2, -0.3]])  # test_multivector.py:94-109 -> "101", "010"
    bools3 = np.array(fo.binary_quantize(x3), dtype=bool)
    packed3 = np.frombuffer(b"".join(fo.binary_quantize_packed(x3)), dtype=np.uint8).reshape(2, 1)
    a = rng.integers(0, 256, size=(64, 16), dtype=np.uint8)
    b = rng.integers(0, 256, size=(64, 16), dtype=np.uint8)
    ham = np.array([fo.hamming_distance(bytes(a[i]), bytes(b[i])) for i in range(64)], dtype=np.int64)
    ham_batch = np.array(fo.hamming_distance_batch(bytes(a[0]), [bytes(r) for r in b]), dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "sign_pack.npz"), x=x, packed=packed, bools=bools, x3=x3, bools3=bools3,
                        packed3=packed3, ham_a=a, ham_b=b, ham=ham, ham_batch=ham_batch)


def unit_rows(rng, n, d=128):
    x = rng.standard_normal((n, d)).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def gen_float_maxsim():
    from transformers.models.colpali.processing_colpali import ColPaliProcessor

    rng = np.random.default_rng(4321)
    out = {}
    # case A: equal-length pages (the shape family of every BASELINE config), two queries of different length
    qa = [unit_rows(rng, 32), unit_rows(rng, 20)]
    pa = [unit_rows(rng, 64) for _ in range(12)]
    sa = ColPaliProcessor.score_retrieval(None, [torch.from_numpy(q) for q in qa], [torch.from_numpy(p) for p in pa],
                                          batch_size=128, output_dtype=torch.float32)
    out.update(a_q0=qa[0], a_q1=qa[1], a_pages=np.stack(pa), a_scores=sa.numpy())
    # case B: ragged pages inside one 128-batch -> zero-padding quirk (max includes the zero rows)
    lens_b = [5, 64, 1, 33, 64, 17, 40, 2]
    pb = [unit_rows(rng, n) for n in lens_b]
    qb = [-np.abs(unit_rows(rng, 8)), unit_rows(rng, 32)]  # first query is all-negative: makes the quirk visible
    pb[0] = np.abs(pb[0])
    pb[2] = np.abs(pb[2])
    sb = ColPaliProcessor.score_retrieval(None, [torch.from_numpy(q) for q in qb], [torch.from_numpy(p) for p in pb],
                                          batch_size=128, output_dtype=torch.float32)
    out.update(b_q0=qb[0], b_q1=qb[1], b_rows=np.concatenate(pb), b_lens=np.array(lens_b), b_scores=sb.numpy())
    # case C: batch_size smaller than the page count -> padding is per batch, not global
    sc = ColPaliProcessor.score_retrieval(None, [torch.from_numpy(q) for q in qb], [torch.from_numpy(p) for p in pb],
                                          batch_size=3, output_dtype=torch.float32)
    out.update(c_scores=sc.numpy(), c_batch=np.array(3))
    # case D: bf16-valued inputs (what the embedding model really emits: colpali_embedding_model.py:262)
    qd = torch.from_numpy(unit_rows(rng, 32)).bfloat16().float()
    pd = [torch.from_numpy(unit_rows(rng, 96)).bfloat16().float() for _ in range(16)]
    sd = ColPaliProcessor.score_retrieval(None, [qd], pd, batch_size=128, output_dtype=torch.float32)
    out.update(d_q=qd.numpy(), d_pages=torch.stack(pd).numpy(), d_scores=sd.numpy())
    # case E: the rerank call of FastMultiVectorStore.query_similar (fast_multivector_store.py:553-555): ONE query against the
    # candidate pages in FIRST-STAGE ORDER, one 128-batch (<= 75 candidates) -> the padding quirk follows the candidate list
    lens_e = [int(x) for x in rng.integers(3, 90, size=40)]
    pe = [torch.from_numpy(np.abs(unit_rows(rng, n))).bfloat16().float() for n in lens_e]  # bf16-valued, all-positive
    cand_e = rng.permutation(40)[:25]
    qe = [torch.from_numpy(-np.abs(unit_rows(rng, 20))).bfloat16().float(), torch.from_numpy(unit_rows(rng, 32)).bfloat16().float()]
    se = torch.stack([ColPaliProcessor.score_retrieval(None, [q], [pe[int(c)] for c in cand_e], batch_size=128,
                                                       output_dtype=torch.float32)[0] for q in qe])
    out.update(e_rows=torch.cat(pe).numpy(), e_lens=np.array(lens_e), e_cand=cand_e.astype(np.int64), e_q0=qe[0].numpy(),
               e_q1=qe[1].numpy(), e_scores=se.numpy())
    # split by case so that no fixture file exceeds 1 MB
    for name, cases in (("float_maxsim.npz", "abc"), ("float_maxsim_d.npz", "d"), ("float_maxsim_e.npz", "e")):
        np.savez_compressed(os.path.join(OUT, name), **{k: v for k, v in out.items() if k[0] in cases})


def gen_binary_known_answers():
    """Derived (not executed) known answers for SQL max_sim -- see module docstring."""
    # test_multivector.py:222-256: page1 = 3x[+1]*64,[-1]*64 ; page2 = complement ; query = one row like page1
    e1 = np.ones((3, 128), dtype=np.float32)
    e1[:, 64:] = -1
    e2 = -e1
    q = e1[:1].copy()
    np.savez_compressed(os.path.join(OUT, "binary_known.npz"), pattern_rows=np.concatenate([e1, e2]),
                        pattern_lens=np.array([3, 3]), pattern_query=q, pattern_scores=np.array([1.0, 0.0]),
                        derived=np.array(True))


if __name__ == "__main__":
    fo = load_fast_ops()
    gen_sign_pack(fo)
    gen_float_maxsim()
    gen_binary_known_answers()
    for f in sorted(os.listdir(OUT)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
