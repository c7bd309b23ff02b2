"""tests/str_group_ref.py against what the suite already trusts: the C oracle's MetroHash64_1, oracle/pyref.py's
group_by_key, cogroup and HashPartitioner over str keys, and the "x" / "y" data of the reference's test_pair_rdd.rs."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import pyref as P
from tests import group_ref as G
from tests import str_group_ref as S


def _keys(ranks, lens=S.LENS):
    o, d = S.encode(ranks, lens)
    raw = d.tobytes()
    return [raw[int(o[i]):int(o[i + 1])] for i in range(len(ranks))]


def test_hash_matches_oracle_every_length():
    rng = np.random.default_rng(1)
    keys = [b""] + [bytes(rng.integers(0, 256, L, dtype=np.uint8)) for L in range(1, 301)]
    keys += [b"\xff" * L for L in range(0, 70)] + [b"\x00" * L for L in range(0, 70)]
    keys += [bytes(rng.integers(0, 256, int(rng.integers(0, 2000)), dtype=np.uint8)) for _ in range(300)]
    offs = np.r_[0, np.cumsum([len(k) for k in keys])].astype(np.uint64)
    data = np.frombuffer(b"".join(keys), dtype=np.uint8)
    want = [O.metrohash64_1(k + b"\xff") for k in keys]
    assert S.metro64_1_str(offs, data).tolist() == want
    # one length class read as one matrix (the fast path of decode and metro64_1_str)
    same = keys[120:121] * 5
    o = np.arange(6, dtype=np.uint64) * len(same[0])
    assert S.metro64_1_str(o, np.frombuffer(b"".join(same), dtype=np.uint8)).tolist() == want[120:121] * 5


def test_keys_cover_the_hash_steps_and_edge_bytes():
    ranks = S.distinct_ranks(70_000)
    ks = _keys(ranks)
    lens = {len(k) for k in ks}
    assert {0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 65, 100} <= lens
    assert ks[0] == b"" and ks[S.ALL_FF] == b"\xff" and ks[0xFFFF] == b"\xff\xff"
    assert any(b"\x00" in k for k in ks) and any(b"\xff" in k[8:] for k in ks)
    assert ks[1] == b"\x01" and ks[257] == b"\x01\x01" and ks[2] == b"\x02\x00"    # shared prefixes, NULs
    assert sum(1 for k in ks[256:] if 0 < len(k) < 8 and k[:1] in ks[1:256]) > 1000
    assert len(set(ks)) == len(ks)
    assert S.distinct_ranks(200).tolist()[:2] == [0, 1] and S.ALL_FF in S.distinct_ranks(200).tolist()


@pytest.mark.parametrize("lens", [S.LENS, (1100,)])
def test_encode_decode_round_trip_and_torch_bytes(lens):
    rng = np.random.default_rng(len(lens))
    ranks = np.r_[np.arange(3000), rng.integers(0, 1 << 62, 3000), [S.ALL_FF, 0xFFFFFF, (1 << 63) - 1]].astype(np.uint64)
    ranks = rng.permutation(ranks)
    o, d = S.encode(ranks, lens)
    assert np.array_equal(S.decode(o, d, lens), ranks)
    to, td = S.encode_torch(torch.from_numpy(ranks.view(np.int64)), lens)
    assert np.array_equal(to.numpy().view(np.uint64), o) and np.array_equal(td.numpy(), d)
    u = np.unique(ranks)
    assert len(set(_keys(u, lens))) == len(u)


def test_decode_catches_a_wrong_byte():
    ranks = S.distinct_ranks(5000)
    o, d = S.encode(ranks)
    for at in (int(o[300]), int(o[4000]) + 9, int(o[-1]) - 1):      # a rank byte, a pad byte, the last byte
        bad = d.copy()
        bad[at] ^= 0x40
        with pytest.raises(AssertionError):
            assert np.array_equal(S.decode(o, bad), ranks)
    short = o.copy()
    short[4000] += np.uint64(1)                                     # one key a byte longer, the next a byte shorter
    with pytest.raises(AssertionError):
        S.decode(short, d)


def _utf8_ranks(n):
    """Ranks whose keys are valid UTF-8 (pyref hashes str keys): NULs included, 0xFF never."""
    ranks = S.distinct_ranks(n)
    return ranks[[_valid(k) for k in _keys(ranks)]]


def _valid(k):
    try:
        k.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def _pyref_parts(keys, vals, M, R):
    """pyref.group_by_key per partition as (key offsets, key bytes, value offsets, values)."""
    by_part = [[] for _ in range(R)]
    for k, vs in P.group_by_key(list(zip(keys, vals)), M, R):
        by_part[P.get_partition(k, R)].append((k.encode(), vs))
    out = []
    for items in by_part:
        kb = [k for k, _ in items]
        out.append((np.r_[0, np.cumsum([len(k) for k in kb])].astype(np.uint64), np.frombuffer(b"".join(kb), np.uint8),
                    np.r_[0, np.cumsum([len(v) for _, v in items])].astype(np.uint64),
                    np.array([v for _, vs in items for v in vs], dtype=np.uint64)))
    return out


@pytest.mark.parametrize("R", [1, 7, 300])
def test_group_matches_pyref(R):
    rng = np.random.default_rng(R)
    pool = _utf8_ranks(3000)
    assert len(pool) > 300 and 0 in pool.tolist()
    ranks = pool[rng.integers(0, 400, 4000)]
    vals = rng.integers(0, 1 << 64, len(ranks), dtype=np.uint64)
    keys = [k.decode() for k in _keys(ranks)]
    parts = _pyref_parts(keys, vals.tolist(), 3, R)
    S.assert_str_group_equal(parts, ranks, vals, R)
    want = [P.get_partition(k, R) for k in keys[:500]]
    assert S.partition_of(ranks[:500], R).tolist() == want
    # a swapped pair of values and a key in the wrong partition fail
    ko, kb, vo, v = parts[0]
    big = int(np.argmax(np.diff(vo.astype(np.int64))))
    sw = v.copy()
    a, b = int(vo[big]), int(vo[big]) + 1
    sw[[a, b]] = sw[[b, a]]
    if sw[a] != sw[b]:
        with pytest.raises(AssertionError):
            S.assert_str_group_equal([(ko, kb, vo, sw)] + parts[1:], ranks, vals, R)
    if R > 1:
        with pytest.raises(AssertionError, match="another partition"):
            S.assert_str_group_equal([parts[1], parts[0]] + parts[2:], ranks, vals, R)


def test_reference_x_y_data():
    """tests/test_pair_rdd.rs:8-37: ("x", 1..7) and ("y", 1..8) grouped over 4 map tasks into 4 partitions."""
    keys = ["x"] * 7 + ["y"] * 8
    vals = list(range(1, 8)) + list(range(1, 9))
    parts = _pyref_parts(keys, vals, 4, 4)
    lens = (1,)                                   # ranks 0x78 / 0x79 are the one-byte keys "x" / "y"
    ranks = np.array([ord(k) for k in keys], np.uint64)
    assert _keys(ranks[[0, 7]], lens) == [b"x", b"y"]
    S.assert_str_group_equal(parts, ranks, np.array(vals, np.uint64), 4, lens=lens)


def test_cogroup_and_join_match_pyref():
    rng = np.random.default_rng(3)
    pool = _utf8_ranks(3000)
    R = 7
    ra, rb = pool[rng.integers(0, 300, 900)], pool[rng.integers(150, 500, 700)]
    va, vb = rng.integers(0, 1 << 64, len(ra), dtype=np.uint64), rng.integers(0, 1 << 64, len(rb), dtype=np.uint64)
    ka, kb = [k.decode() for k in _keys(ra)], [k.decode() for k in _keys(rb)]
    res = P.cogroup(list(zip(ka, va.tolist())), 3, list(zip(kb, vb.tolist())), 2, R)
    by_part = [[] for _ in range(R)]
    for k, (vs, ws) in res:
        by_part[P.get_partition(k, R)].append((k.encode(), vs, ws))
    parts, jparts = [], []
    for items in by_part:
        kbs = [k for k, _, _ in items]
        ko = np.r_[0, np.cumsum([len(k) for k in kbs])].astype(np.uint64)
        kd = np.frombuffer(b"".join(kbs), np.uint8)
        side = lambda i: (np.r_[0, np.cumsum([len(x[i]) for x in items])].astype(np.uint64),
                          np.array([v for x in items for v in x[i]], dtype=np.uint64))
        parts.append((ko, kd, [side(1), side(2)]))
        # the full outer join of the same lists: for v in vs { for w in ws }, a missing side as (0, valid 0)
        rows = [[(v, w, 1, 1) for v in vs for w in ws] or [(v, 0, 1, 0) for v in vs] or [(0, w, 0, 1) for w in ws]
                for _, vs, ws in items]
        flat = [x for r in rows for x in r]
        jparts.append((ko, kd, np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.uint64),
                       (np.array([x[0] for x in flat], np.uint64), np.array([x[1] for x in flat], np.uint64)),
                       (np.array([x[2] for x in flat], np.uint8), np.array([x[3] for x in flat], np.uint8))))
    placed = S.assert_str_cogroup_equal(parts, [(ra, va), (rb, vb)], R)
    G.assert_rows_equal(S.str_join_rows(jparts, R), G.join_rows("full", ra, va, rb, vb), G.JOIN_COLS)
    G.assert_rows_equal(S.str_join_rows(jparts, R, placed=placed), G.join_rows("full", ra, va, rb, vb), G.JOIN_COLS)
    with pytest.raises(AssertionError, match="partition of the checked key"):
        S.str_join_rows([jparts[1], jparts[0]] + jparts[2:], R, placed=placed)
    inner = [x for x in res if x[1][0] and x[1][1]]
    assert len(inner) > 50 and len(res) > len(inner) + 50


def test_byte_string_values_compare_by_their_bytes():
    rng = np.random.default_rng(4)
    ranks = S.rank_rows(rng, 3000, 500)
    vr = rng.integers(0, 1 << 40, len(ranks), dtype=np.uint64)
    R = 5
    part = S.partition_of(ranks, R)
    parts = []
    for r in range(R):
        order = np.argsort(ranks[part == r], kind="stable")
        kr, v = ranks[part == r][order], vr[part == r][order]
        uk, starts, cnt = G.runs(kr)
        ko, kd = S.encode(uk)
        vo, vd = S.encode(v)
        parts.append((ko, kd, np.r_[starts, len(kr)].astype(np.uint64), (vo, vd)))
    S.assert_str_group_equal(parts, ranks, vr, R)
    ko, kd, o, (vo, vd) = parts[0]
    bad = vd.copy()
    bad[int(vo[3]) + 1] ^= 1
    with pytest.raises(AssertionError):
        S.assert_str_group_equal([(ko, kd, o, (vo, bad))] + parts[1:], ranks, vr, R)
