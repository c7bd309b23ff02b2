"""tests/slot_hash_ref.py on the CPU: the inverse of the slot hash, the home bucket of every key family at every table
size, and the insert model's verdict on chains at the HA_MAX_PROBE limit."""
import numpy as np
import pytest

from tests import slot_hash_ref as S

LOG_CAPS = range(4, 32)
PBITS = [(23, 2), (24, 3), (29, 8), (31, 8)]      # (log_cap, regions' top bits): min(8, log_cap - 21) in engine.cu


def test_slot_hash_matches_python_integers_and_inverts():
    rng = np.random.default_rng(0)
    keys = np.concatenate([rng.integers(0, 1 << 64, 20_000, dtype=np.uint64),
                           np.array([0, 1, S.MASK, 1 << 63, (1 << 32) - 1, 1 << 32], dtype=np.uint64)])

    def ref(x):                                   # common.cuh:slot_hash with Python integers
        x ^= x >> 32
        x = (x * S.M1) & S.MASK
        x ^= x >> 32
        return (x * S.M2) & S.MASK

    h = S.slot_hash(keys)
    assert h.tolist() == [ref(int(k)) for k in keys.tolist()]
    assert np.array_equal(S.slot_hash_inv(h), keys)
    assert np.array_equal(S.slot_hash(S.slot_hash_inv(keys)), keys)
    assert S.slot_hash(np.array([0], np.uint64))[0] == 0          # key 0: home bucket 0 at every size


def test_families_have_their_home_at_every_size():
    rng = np.random.default_rng(1)
    top = 0x1_5555_5555
    fam = S.same_home(rng, 3000, top)
    wr = S.wrap(rng, 500)
    absent = S.same_home(rng, 400, top, exclude=fam)
    for f in (fam, wr, absent):
        assert len(np.unique(f)) == len(f) and not np.isin(f, [0, S.MASK]).any()
    assert not np.isin(absent, fam).any()
    for lc in LOG_CAPS:
        nb = 1 << (lc - 2)
        assert (S.home_bucket(fam, lc) == top >> (S.TOP - (lc - 2))).all()
        assert (S.home_bucket(absent, lc) == top >> (S.TOP - (lc - 2))).all()
        assert (S.home_bucket(wr, lc) == nb - 1).all()
        assert S.home_bucket(np.array([0], np.uint64), lc)[0] == 0
    low = 0xABCDE
    cc = S.cache_clash(rng, 64, low)
    h = S.slot_hash(cc)
    assert (h & np.uint64((1 << 20) - 1) == low).all()
    for slots in (1024, 512):                     # HC_SLOTS and MA_HC_SLOTS: both choices collide
        assert len(np.unique(h & np.uint64(slots - 1))) == 1
        assert len(np.unique((h >> np.uint64(10)) & np.uint64(slots - 1))) == 1
    assert len(np.unique(S.home_bucket(cc, 20))) > 32          # spread over the table


@pytest.mark.parametrize("log_cap,pbits", PBITS)
def test_region_edge_keys_sit_on_the_last_bucket_of_each_region(log_cap, pbits):
    assert S.region_bits(log_cap) == pbits
    rng = np.random.default_rng(log_cap)
    keys = S.region_edge(rng, 3, log_cap)
    assert len(keys) == 3 << pbits
    per = 1 << (log_cap - 2 - pbits)
    homes = S.home_bucket(keys, log_cap)
    assert ((homes + np.uint64(1)) % np.uint64(per) == 0).all()
    assert sorted(set((homes // np.uint64(per)).tolist())) == list(range(1 << pbits))
    # the region of a row is its slot hash's top pbits: the edge key's chain continues in the next region
    assert np.array_equal(S.slot_hash(keys) >> np.uint64(64 - pbits), homes // np.uint64(per))


def test_i32_keys_share_a_home_bucket():
    keys = S.i32_same_home(np.random.default_rng(2), 900, 12, candidates=1 << 22)
    assert keys.dtype == np.int32 and len(np.unique(keys)) == 900 and not (keys == -1).any()
    assert len(np.unique(S.home_bucket(keys.astype(np.int64).view(np.uint64), 12))) == 1


@pytest.mark.parametrize("log_cap", [12, 13, 14, 20, 31])
def test_model_1024_same_home_keys_fit_and_1025_abort(log_cap):
    rng = np.random.default_rng(log_cap)
    fam = S.same_home(rng, 1025, 0x0_2468_ACE1)
    extra = np.array([0, S.MASK], dtype=np.uint64)               # bucket 0 and the special slot: not on the chain
    assert S.chain_model(np.concatenate([fam[:1024], extra]), log_cap) == (False, 256)
    assert S.chain_model(np.concatenate([fam, extra]), log_cap)[0]
    assert S.chain_model(fam[::-1], log_cap)[0]                  # in any order
    # a table that cannot grow lets the chain run on: the 1025th key loads a 257th bucket
    assert S.chain_model(fam, log_cap, limit=1 << (log_cap - 2)) == (False, 257)


def test_model_wrapped_chain_reaches_bucket_zero():
    rng = np.random.default_rng(3)
    wr = S.wrap(rng, 40)                                          # 10 buckets: the last one, then 0..8
    aborts, longest = S.chain_model(np.concatenate([np.array([0], np.uint64), wr]), 10)
    assert not aborts and longest == 11                           # key 0 holds a slot of bucket 0: one more bucket
    assert S.chain_model(wr, 10, limit=9)[0]
