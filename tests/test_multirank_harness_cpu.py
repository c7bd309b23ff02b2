"""The in-process rank harness of tests/multirank.py over the oracle-backed FakeEngine: the slicing and ordering of the
emulated all-to-all-v (source-rank major = map-id order, partition r on rank r % W) against the single-process oracle.
The GPU file tests/test_gpu_multirank_paths.py runs the same driver over the library."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.fake_engine import FakeEngine
from tests.multirank import group_dict, maps_by_rank, owned_parts, run_ranks
from tests.util import oracle_group, rand_pairs

AGG = {"group": 0, "sum": 1, "min": 2, "max": 3, "count": 4}


@pytest.mark.parametrize("op", list(AGG))
@pytest.mark.parametrize("W", [1, 2, 3, 8])
def test_harness_matches_single_process_oracle(W, op):
    rng = np.random.default_rng([W, AGG[op]])
    n, M, R = 6000, 2 * W + 1, 11
    keys, vals = rand_pairs(rng, n, 700, values="full")
    maps = maps_by_rank(n, M, W, lambda m, lo, hi: (keys[lo:hi], None if op == "count" else vals[lo:hi]))
    eng = FakeEngine()
    shs, _ = run_ranks(eng, W, AGG[op], maps, R, 0, 0, n_map=M)
    parts = owned_parts(eng, shs, R)
    if op == "group":
        assert [group_dict(*p) for p in parts] == oracle_group(keys, vals, M, R)
    else:
        want = O.shuffle(op, keys, None if op == "count" else vals, M, R)
        for p, w in zip(parts, want):
            assert dict(zip(p[0].tolist(), p[1].tolist())) == dict(zip(w["keys"].tolist(), w["combined"].tolist()))
