"""CPU check that the stream-order cases cover the C-ABI: every exported function of include/b200ms.h that takes a
`void* stream`, or that enqueues on the handle's own stream, must be run by some case of tests/stream_order_cases.py
(as call A or call B), so that a new entry point cannot skip tests/test_gpu_stream_order.py."""
import glob
import os
import re

import stream_order_cases as soc
from test_cabi_symbols import header_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_declarations():
    """name -> parameter list of every function the header declares."""
    text = open(os.path.join(ROOT, "include", "b200ms.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {m.group(1): " ".join(m.group(2).split()) for m in re.finditer(r"\b(b200ms_[a-z0-9_]+)\s*\(([^)]*)\)", text)}


def stream_takers():
    return {n for n, params in header_declarations().items() if re.search(r"\bvoid\s*\*\s*stream\b", params)}


def function_bodies():
    """name -> body of every top-level function definition in csrc/*.cu (a definition starts at column 0 and its body
    ends at the next closing brace at column 0)."""
    bodies = {}
    for path in sorted(glob.glob(os.path.join(ROOT, "morphik-core_b200", "csrc", "*.cu"))):
        src = open(path).read()
        for m in re.finditer(r"^[A-Za-z][^\n;{}]*?\b([A-Za-z_]\w*)\([^;{}]*?\)\s*(?:const\s*)?\{", src, flags=re.M):
            end = src.find("\n}\n", m.end())
            bodies[m.group(1)] = src[m.end():end if end >= 0 else len(src)]
    return bodies


def handle_stream_users():
    """Exported functions that enqueue on h->stream, directly (`s = h->stream`) or through a helper that does."""
    bodies = function_bodies()
    users = {n for n, b in bodies.items() if re.search(r"=\s*h->stream\b", b)}
    while True:
        more = {n for n, b in bodies.items() if n not in users and any(re.search(rf"\b{u}\(", b) for u in users)}
        if not more:
            break
        users |= more
    return {n for n in users if n.startswith("b200ms_")}


def test_parsers_see_the_known_entry_points():
    takers = stream_takers()
    assert {"b200ms_search_device", "b200ms_score", "b200ms_topk", "b200ms_fde_scan", "b200ms_explain_device",
            "b200ms_sharded_search_begin", "b200ms_send_device"} <= takers
    assert "b200ms_search_host" not in takers and "b200ms_set_corpus" not in takers
    users = handle_stream_users()
    assert {"b200ms_search_host", "b200ms_search_host_masked", "b200ms_set_corpus", "b200ms_set_corpus_host",
            "b200ms_fde_configure", "b200ms_fde_configure_ex", "b200ms_sharded_search_host_begin"} <= users, users


def test_every_enqueuing_export_has_a_case():
    needed = (stream_takers() | handle_stream_users()) - set(soc.MULTI_RANK_ONLY)
    missing = sorted(needed - soc.covered_exports())
    assert not missing, f"exported functions without a stream-order case in tests/stream_order_cases.py: {missing}"


def test_cases_name_real_exports_and_kinds():
    exports = set(header_symbols())
    named = {fn for fns in soc.CALLS.values() for fn in fns} | set(soc.MULTI_RANK_ONLY)
    assert named <= exports, sorted(named - exports)
    assert set(soc.MULTI_RANK_ONLY) <= stream_takers()
    for c in soc.CASES:
        assert c.a in soc.CALLS and c.b in soc.CALLS, c
        assert c.kinds and set(c.kinds) <= set(soc.KINDS), c
        assert c.b_stream in ("other", "same") and c.handles in (1, 2), c
    _, ids = soc.parametrize()
    assert len(ids) == len(set(ids))


def test_cases_cover_the_required_pairs():
    pairs = {(c.a, c.b, k) for c in soc.CASES for k in c.kinds if c.b_stream == "other" and c.handles == 1}
    for kind in ("bf16", "int8", "fp8", "b1_popc", "b1_wgmma"):
        assert ("search_device", "search_host", kind) in pairs, kind
    for kind in ("fp8", "b1_popc"):
        assert ("score_topk", "score_topk", kind) in pairs, kind
    assert any(a == "rerank_batch_device" and soc.KINDS[k][2] == "host" for a, _, k in pairs)
    assert any(a == "search_device" and b == "set_corpus_search" for a, b, _ in pairs)
    controls = [c for c in soc.CASES if c.b_stream == "same" or c.handles == 2]
    assert {c.b_stream for c in controls} == {"same", "other"} and {c.handles for c in controls} == {1, 2}
    # one oracle anchor per corpus dtype
    anchored = {soc.KINDS[k][0] for c in soc.CASES if c.oracle for k in c.kinds}
    assert anchored == {"bf16", "int8", "fp8", "binary"}
