"""The cut agreement of sort_by_key over String keys across ranks, without a GPU: the restatement of
tests/str_sort_dist_ref.py gives every rank the cuts that make its partitions those of the one-process reference
(tests/str_sort_ref.py) over the same rows, for 1 to 8 ranks and 1 to 70 partitions, and stays within its round bound."""
import numpy as np
import pytest

from tests import str_sort_dist_ref as DR
from tests import str_sort_ref as SR


def _split(rows, W, rng, empty_ranks=()):
    """rows in map-id order, cut into W ascending blocks (as dist.map_block gives the ranks their map tasks)"""
    live = [r for r in range(W) if r not in empty_ranks]
    cuts = sorted(rng.integers(0, len(rows) + 1, len(live) - 1).tolist()) if live else []
    bounds = [0] + cuts + [len(rows)]
    blocks, j = [[] for _ in range(W)], 0
    for r in live:
        blocks[r] = rows[bounds[j]:bounds[j + 1]]
        j += 1
    return blocks


def _check(blocks, R):
    ranks = [DR.Rank(b) for b in blocks]
    kcut, trace = DR.agree_cuts(ranks, R)
    rows = [k for b in blocks for k in b]
    want = SR.partitions(rows, None, R)
    got = DR.rank_partitions(ranks, kcut, R)
    for p in range(R):
        # every rank's slice of partition p is exactly its keys in the reference partition
        wp = set(want[p][0])
        for r, rk in enumerate(ranks):
            assert got[r][p] == [k for k in rk.keys if k in wp], (p, r)
        n_rows = sum(ranks[r].row_off[kcut[r][p + 1]] - ranks[r].row_off[kcut[r][p]] for r in range(len(ranks)))
        assert n_rows == len(want[p][0]), (p, n_rows, len(want[p][0]))
    return trace


def _keysets(rng):
    prefix = "p" * 700
    return {
        "edges": [b"", b"k", b"k\x00", b"\x00", b"\x00\x00", b"\xff", b"\xff\x00", b"\xff" * 9, b"a", b"ab", b"abcdefg",
                  b"abcdefgh", b"abcdefg\x00", b"abcdefg\xff"],
        "chain": ["a" * i for i in range(1, 40)],
        "prefix700": [prefix + chr(97 + int(x)) * int(y) for x, y in zip(rng.integers(0, 26, 50), rng.integers(0, 4, 50))],
        "random": [bytes(rng.integers(0, 256, int(rng.integers(0, 20))).astype(np.uint8)) for _ in range(80)],
    }


@pytest.mark.parametrize("W", range(1, 9))
def test_cuts_equal_the_one_process_cuts(W):
    rng = np.random.default_rng(W)
    sets = _keysets(rng)
    for name, pool in sets.items():
        for R in sorted({1, 2, 3, 7, W, W + 1, 16, 31, 70}):
            n = int(rng.integers(1, 400))
            rows = [pool[i] for i in rng.integers(0, len(pool), n)]
            _check(_split(rows, W, rng), R)


@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_skewed_and_empty_inputs(W):
    rng = np.random.default_rng(100 + W)
    for R in (1, 2, 5, 13, 70):
        # one key holding most rows, and all rows one key
        rows = ["hot"] * 300 + [f"k{i}" for i in rng.integers(0, 50, 60)]
        rows = [rows[i] for i in rng.permutation(len(rows))]
        _check(_split(rows, W, rng), R)
        _check(_split(["only"] * 120, W, rng), R)
        # ranks with no rows, and N = 0
        _check(_split([f"x{i}" for i in rng.integers(0, 30, 90)], W, rng, empty_ranks=set(range(0, W, 2))), R)
        _check([[] for _ in range(W)], R)


def test_every_R_from_1_to_70():
    rng = np.random.default_rng(7)
    pool = _keysets(rng)["edges"] + [b"a" * i for i in range(1, 20)]
    rows = [pool[i] for i in rng.integers(0, len(pool), 500)]
    for W in (2, 3, 8):
        blocks = _split(rows, W, rng)
        for R in range(1, 71):
            _check(blocks, R)


def test_a_shared_word_costs_one_round():
    rng = np.random.default_rng(11)
    prefix = "q" * 700                                            # 100 words every key shares
    rows = [prefix + "%03d" % i for i in rng.integers(0, 1000, 600)]
    for W in (2, 4):
        trace = _check(_split(rows, W, rng), 9)
        for cut in trace["words"]:
            assert [w for w, _ in cut[:100]] == list(range(100))
            assert all(b == 0 for _, b in cut[:100])              # shared: one round, no bisection
            assert all(b <= 64 for _, b in cut)
        # bound: one round per shared word, plus the bisection of the words where the keys differ
        assert trace["rounds"] <= max(len(c) + sum(b for _, b in c) for c in trace["words"])
        assert trace["rounds"] <= 100 + 2 * (1 + 64)


def test_distinct_keys_stop_at_their_first_differing_word():
    rng = np.random.default_rng(12)
    rows = ["x" * 300 + "%06d" % i + "tail" * 50 for i in rng.permutation(5000)]   # unique past byte 306
    trace = _check(_split(rows, 3, rng), 8)
    for cut in trace["words"]:
        # 43 shared words, then the word where the keys differ; the rest of the key costs nothing once one is left
        assert len(cut) <= 43 + 2
