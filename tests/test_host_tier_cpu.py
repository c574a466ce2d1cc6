"""CPU checks of the host-resident corpus tier: argument validation that happens before any GPU work, and the C-ABI surface
(exported, bound, documented)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["b200ms_set_corpus_host", "b200ms_host_alloc", "b200ms_host_free", "b200ms_last_gather_stats"]


def test_store_host_tier_needs_candidates_before_touching_the_gpu():
    from morphik_core_b200.store import B200MultiVectorStore

    with pytest.raises(ValueError, match="fde_candidates"):
        B200MultiVectorStore(corpus_tier="host")
    with pytest.raises(ValueError, match="fde_candidates"):
        B200MultiVectorStore(corpus_tier="host", fde_candidates=0)
    with pytest.raises(ValueError, match="corpus_tier"):
        B200MultiVectorStore(corpus_tier="disk", fde_candidates=10)


def test_index_rejects_unknown_tier():
    from morphik_core_b200.index import MaxSimIndex

    with pytest.raises(ValueError, match="tier"):
        MaxSimIndex(dtype="bf16", tier="nvme")


def test_host_tier_symbols_exported_bound_and_declared():
    from morphik_core_b200 import _native as nat

    header = open(os.path.join(ROOT, "include", "b200ms.h")).read()
    for s in NEW_SYMBOLS:
        assert re.search(rf"\b{s}\s*\(", header), s
        assert s in nat.EXPORTED
        assert getattr(nat.lib, s).argtypes is not None
    # no handle: EINVAL, never a crash
    assert nat.lib.b200ms_set_corpus_host(None, None, nat.BF16, None, 0) == -1
    assert nat.lib.b200ms_last_gather_stats(None, None, None, None, None) == -1
    assert nat.lib.b200ms_host_free(None, None) == 0


def test_host_stage_bytes_option_documented():
    header = open(os.path.join(ROOT, "include", "b200ms.h")).read()
    api = open(os.path.join(ROOT, "morphik-core_b200", "csrc", "api.cu")).read()
    assert '"host_stage_bytes"' in header and 'n == "host_stage_bytes"' in api
