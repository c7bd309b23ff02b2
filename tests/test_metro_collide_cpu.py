"""tests/metro_collide_ref.py on the CPU: the block solver, every family's shared hash under the C oracle and both
numpy restatements, the wrap family's home at every index size, and the encode model's verdict on the parent's growth
rule and on this build's."""
import os
import re
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests import bytes_keys_ref as B
from tests import metro_collide_ref as MC
from tests import str_group_ref as S

STRKEYS = os.path.join(os.path.dirname(MC.__file__), os.pardir, "vega_b200", "csrc", "strkeys.cuh")
ENGINE = os.path.join(os.path.dirname(MC.__file__), os.pardir, "vega_b200", "csrc", "engine.cu")
KINDS = (MC.STR, MC.BYTES)


def oracle_hash(kind, k):
    """The C oracle's MetroHash64_1 of the stream the kind's Hash writes."""
    return O.metrohash64_1(k + b"\xff" if kind == MC.STR else struct.pack("<Q", len(k)) + k, 0)


def assert_one_hash(kind, keys, h=None):
    """Every key hashes to one value under the oracle and the kind's numpy restatement; returns it."""
    o, d = B.encode(list(keys))
    np_h = set((S.metro64_1_str if kind == MC.STR else B.metro64_1_bytes)(o, d).tolist())
    c_h = {oracle_hash(kind, k) for k in keys}
    assert np_h == c_h and len(c_h) == 1, (kind, len(np_h), len(c_h))
    if h is not None:
        assert c_h == {h}
    return c_h.pop()


def test_constants_match_the_engine():
    src = open(STRKEYS).read()
    assert re.search(r"STR_MAX_PROBE = (\d+);", src).group(1) == str(MC.STR_MAX_PROBE)
    assert re.search(r"str_bucket\(u64 h, u32 log_cap\) \{ return log_cap > 2 \? \(h >> \(66 - log_cap\)\)", src)
    assert re.search(r"STR_MAX_LOG_CAP = (\d+);", open(ENGINE).read()).group(1) == str(MC.STR_MAX_LOG_CAP)


def test_block_solver_reaches_any_state():
    rng = np.random.default_rng(0)
    a = tuple(rng.integers(0, 1 << 64, 1000, dtype=np.uint64) for _ in range(4))
    T = tuple(rng.integers(0, 1 << 64, 1000, dtype=np.uint64) for _ in range(4))
    w = MC.solve(a, T)
    assert all(np.array_equal(x, t) for x, t in zip(MC.block(a, w), T))
    # the block step against Python integers (one round of metro64_1_key's loop)
    rot = lambda v, k: ((v >> k) | (v << (64 - k))) & MC.MASK
    v = [int(x[0]) for x in a]
    ww = [int(x[0]) for x in w]
    v[0] = (rot((v[0] + ww[0] * MC.K[0]) & MC.MASK, 29) + v[2]) & MC.MASK
    v[1] = (rot((v[1] + ww[1] * MC.K[1]) & MC.MASK, 29) + v[3]) & MC.MASK
    v[2] = (rot((v[2] + ww[2] * MC.K[2]) & MC.MASK, 29) + v[0]) & MC.MASK
    v[3] = (rot((v[3] + ww[3] * MC.K[3]) & MC.MASK, 29) + v[1]) & MC.MASK
    assert v == [int(t[0]) for t in T]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [2, 3, 257, 3000])
def test_same_hash_keys_are_distinct_and_share_one_hash(kind, n):
    f = MC.same_hash(kind, n, seed=n)
    assert len(set(f.keys)) == n and {len(k) for k in f.keys} == {MC.DEFAULT_LEN[kind]}
    assert assert_one_hash(kind, f.keys) == f.hash
    # both blocks differ: no two keys share the free prefix, nor the solved block
    free, tail = MC.layout(kind, f.L)
    assert len({k[:free] for k in f.keys}) == n and len({k[free:free + 32] for k in f.keys}) == n
    if kind == MC.STR:
        assert all(k.endswith(MC.STR_TAIL) for k in f.keys)
    assert MC.same_hash(kind, n, seed=n).keys == f.keys                  # deterministic from the seed


@pytest.mark.parametrize("kind", KINDS)
def test_absent_keys_share_the_hash_and_are_not_in_the_family(kind):
    f = MC.same_hash(kind, 500, seed=11)
    ab = MC.absent(f, 300)
    assert len(set(ab)) == 300 and not set(ab) & set(f.keys)
    assert_one_hash(kind, ab, f.hash)


def test_bytes_keys_of_two_lengths_share_one_hash():
    f = MC.same_hash_lengths(200, seed=5)
    assert len(set(f.keys)) == 400 and sorted({len(k) for k in f.keys}) == [64, 96]
    assert_one_hash(MC.BYTES, f.keys)
    # the String pair would need a correction whose top byte keeps the 0xFF terminator: none of the short pairs has one
    assert MC.str_length_pair() is None
    for L1, L2 in MC.LENGTH_PAIRS:
        assert (MC.tail_shift(L1 + 1, L2 + 1) >> 56) not in (0x00, 0xFF)


@pytest.mark.parametrize("kind", KINDS)
def test_pairs_hold_one_hash_per_pair(kind):
    p = MC.pairs(kind, 400, seed=3)
    assert len(set(p)) == 800
    h = [oracle_hash(kind, k) for k in p]
    assert len(set(h)) == 400 and all(h[2 * i] == h[2 * i + 1] for i in range(400))
    o, d = B.encode(p)
    assert (S.metro64_1_str if kind == MC.STR else B.metro64_1_bytes)(o, d).tolist() == h


@pytest.mark.parametrize("kind", KINDS)
def test_wrap_is_homed_at_the_last_bucket_of_every_index_to_2_26_slots(kind):
    f = MC.wrap(kind, 300, seed=2)
    h = assert_one_hash(kind, f.keys)
    assert h >> (64 - MC.WRAP_BITS) == (1 << MC.WRAP_BITS) - 1
    for lc in range(4, 27):
        assert MC.home(h, lc) == (1 << (lc - 2)) - 1, lc
    assert MC.home(h, 40) != (1 << 38) - 1 or h == MC.MASK


def test_wrap_search_finds_states_with_the_top_bits_set():
    for kind in KINDS:
        T = MC.search_wrap(kind, 10, seed=5, chunk=1 << 12)
        f = MC.same_hash(kind, 4, T, seed=0)
        assert f.hash >> 54 == (1 << 10) - 1


# ---- the encode model ------------------------------------------------------------------------------------------------
def ordinary(n, seed=0):
    return np.random.default_rng(seed).integers(0, 1 << 64, n, dtype=np.uint64).tolist()


def mixed(n_family, n_plain=2000, seed=0):
    """Hashes of n_plain random keys with a same-hash family of n_family keys spread among them."""
    hs = ordinary(n_plain, seed) + [MC.same_hash(MC.BYTES, 2, seed=seed).hash] * n_family
    return [hs[i] for i in np.random.default_rng(seed + 1).permutation(len(hs))]


def test_model_parent_grows_until_the_index_cannot_be_allocated():
    hs = mixed(257)
    # default hint: 200k rows size the index at 2^19, and every size aborts on the 65-bucket chain
    _, out = MC.encode_model(hs, 200_000, fixed=False)
    assert out["ladder"] == [19, 21, 23, 25, 27, 29, 31] and out["error"] == "VB_ERR_OOM"
    # hint 1: the load ladder, then the chain, up to 2^32 slots (48 GiB), and no index past 2^33
    _, out = MC.encode_model(hs, 200_000, hint=1, fixed=False)
    assert out["ladder"][:5] == [4, 6, 8, 10, 12] and out["ladder"][-1] == 32 and out["error"] == "VB_ERR_TOO_LARGE"
    # alone, 256 keys fill exactly 64 buckets: the parent copes (with ordinary keys in the window, fewer fail)
    ix, out = MC.encode_model(mixed(256, n_plain=0), 200_000, fixed=False)
    assert out["error"] is None and out["ladder"] == [19]
    _, out = MC.encode_model(mixed(257, n_plain=0), 200_000, fixed=False)
    assert out["error"] == "VB_ERR_OOM"


@pytest.mark.parametrize("n_family", [257, 1024, 3000])
@pytest.mark.parametrize("hint", [0, 1])
def test_model_fix_bounds_the_index(n_family, hint):
    hs = mixed(n_family)
    ctrl, cout = MC.encode_model(ordinary(len(hs), seed=9), 200_000, hint=hint)
    ix, out = MC.encode_model(hs, 200_000, hint=hint)
    assert out["error"] is None and cout["error"] is None
    assert len(ix.entries) == len(hs)
    assert (1 << ix.log_cap) <= 4 * (1 << ctrl.log_cap), (out, cout)
    assert out["restarts"] <= cout["restarts"] + 1
    if hint == 0:                       # 2^19 slots already hold twice the call's rows: lifted from the start
        assert out["ladder"] == [19] and out["restarts"] == 0 and out["lifted"]
    # every key's chain ends at its own bucket: a lifted probe walks at most the family's chain
    fam = [i for i, h in enumerate(hs) if hs.count(h) > 1][:1]
    assert fam and ix.at[fam[0]] is not None


def test_model_random_keys_grow_as_the_parent_grows():
    for hint in (0, 1, 5000):
        for n in (100, 20_000):
            hs = ordinary(n, seed=n)
            a, oa = MC.encode_model(hs, 5 * n, hint=hint)
            b, ob = MC.encode_model(hs, 5 * n, hint=hint, fixed=False)
            assert oa["ladder"] == ob["ladder"] and a.log_cap == b.log_cap


def test_model_second_call_keeps_the_dictionary():
    hs = mixed(600)
    ix, _ = MC.encode_model(hs[:1000], 50_000, hint=1)
    ix2, out = MC.encode_model(hs, 50_000, ix=ix)       # the first 1000 keys again, then new ones
    assert out["error"] is None and len(ix2.entries) == len(hs)
