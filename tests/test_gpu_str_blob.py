"""Bincode blobs of String-key reduce ops: vb_shuffle_reduce_blob encodes a sealed partition as the Vec<(String, C)>
vega stores in SHUFFLE_CACHE, vb_shuffle_map_blob takes such a map-side-combined bucket as a map task.  The encoder is
checked byte for byte against tests/str_blob_ref.py over the rows vb_shuffle_reduce_str returns; decoded buckets
against the pyref reduce over all rows (integer ops and f64 MIN / MAX bit for bit, f64 SUM within a bound)."""
import ctypes
import math
import struct

import numpy as np
import pytest
import torch

import vega_b200 as vb
from vega_b200 import _lib as L
from tests import str_blob_ref as B
from tests.test_gpu_str_keys import _fold, check_parts, key_pool, ref_parts, rows_from_pool
from tests.test_gpu_str_multirank import AGG, VCODE, columns, run_ranks
from tests.test_str_blob_cpu import corrupt_blobs

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
BIG = "m" * (1 << 20)
CASES = [("sum", "u64"), ("sum", "i64"), ("sum", "f64"), ("min", "i64"), ("max", "i64"), ("min", "f64"), ("max", "f64"),
         ("count", "u64")]


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def pool(rng):
    return sorted(set(key_pool(rng) + ["k" * n for n in range(1, 18)] + ["é" * 9, "日本語のキー", "🙂"]))


def rows(rng, n, vdt, finite=False, big=False):
    """n keys (with big, the 1 MiB key twice, at both ends) and values at full range; f64 with NaN, +-0 and infinities
    unless finite."""
    keys = rows_from_pool(rng, pool(rng), n)
    if big:
        keys[0] = keys[-1] = BIG
    if vdt == "u64":
        return keys, rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    if vdt == "i64":
        v = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64, endpoint=True)
        v[1:5] = [-2 ** 63, 2 ** 63 - 1, -1, 0]
        return keys, v
    v = rng.normal(0, 1e6, n)
    if not finite:
        at = rng.integers(0, n, 60)
        v[at] = np.array([math.nan, -0.0, 0.0, math.inf, -math.inf, 1e308] * 10)
    return keys, v


def build(sc, keys, vals, op, vdt, M, R, where="host"):
    kc, vc = columns(keys, None if op == "count" else vals, where)
    starts = vb.slice_starts(len(keys), M)
    sh = vb.StrShuffle(sc, M, R, VCODE[vdt], AGG[op])
    for m in range(M):
        sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    return sh


def str_pairs(sh, r):
    """Partition r as vb_shuffle_reduce_str returns it: [(key bytes, u64 bits)] in its key order."""
    ko, kb, comb = sh.reduce_raw(r)
    bits = comb.view(np.uint64).tolist()
    return [(kb[int(ko[i]):int(ko[i + 1])].tobytes(), bits[i]) for i in range(len(bits))]


def _bits(v, vdt):
    if vdt == "f64":
        return struct.unpack("<Q", struct.pack("<d", v))[0]
    return int(v) & M64


def combined_blob(keys, vals, op, vdt):
    """One map task's map-side-combined bucket, restated in Python (a key's partial in the op's combiner form)."""
    f = _fold("sum" if op == "count" else op, "u64" if op == "count" else vdt)
    acc = {}
    for k, v in zip(keys, [1] * len(keys) if op == "count" else vals.tolist()):
        acc[k] = f(acc[k], v) if k in acc else v
    return B.encode_str_pairs([(k, _bits(v, "u64" if op == "count" else vdt)) for k, v in acc.items()])


def parts_of(sh):
    return [{k: v for k, v in zip(p[0].tolist(), p[1].tolist())} for p in (sh.reduce(r) for r in range(sh.n_reduce))]


def check_against_ref(got, keys, vals, op, vdt, M, R):
    want = ref_parts(keys, vals, op, vdt, M, R)
    if op == "sum" and vdt == "f64":
        per_key = {}
        for k, v in zip(keys, vals.tolist()):
            per_key.setdefault(k, []).append(v)
        for g, w in zip(got, want):
            assert g.keys() == w.keys()
            for k, x in g.items():
                s_ = math.fsum(per_key[k])
                assert abs(x - s_) <= 1e-12 * sum(abs(v) for v in per_key[k]) + math.ulp(s_), (k, x, s_)
    else:
        check_parts(got, want, op, vdt)


# ---- encode ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 3, 257])
@pytest.mark.parametrize("op,vdt", CASES)
def test_encode_matches_reduce_str(sc, op, vdt, R):
    rng = np.random.default_rng(R * 31 + CASES.index((op, vdt)))
    keys, vals = rows(rng, 6000, vdt, big=True)
    sh = build(sc, keys, vals, op, vdt, 3, R)
    lib = sc._lib
    empty = 0
    for r in range(R):
        blob = sh.reduce_blob(r)
        pairs = str_pairs(sh, r)
        assert blob == B.encode_str_pairs(pairs), r
        assert sh.reduce_blob_size(r) == len(blob)
        if not pairs:
            assert blob == b"\x00" * 8
            empty += 1
        buf = torch.full((len(blob) + 32,), 0xAB, dtype=torch.uint8, device="cuda")     # storage: 256-byte aligned
        sh.reduce_blob_device(r, buf[16:16 + len(blob)])
        torch.cuda.synchronize()
        assert buf[16:16 + len(blob)].cpu().numpy().tobytes() == blob, r
        assert (buf[:16] == 0xAB).all() and (buf[16 + len(blob):] == 0xAB).all(), "wrote outside the blob"
        assert lib.vb_shuffle_reduce_blob(sh._h, r, ctypes.c_void_p(buf.data_ptr() + 8), L.VB_DEVICE) == L.VB_ERR_INVALID
    assert R < 257 or empty > 0
    got = {k: v for r in range(R) for k, v in B.decode_str_pairs(sh.reduce_blob(r))}
    assert BIG.encode() in got and all(("k" * n).encode() in got for n in range(1, 18)) and b"" in got
    sh.free()


# ---- decode ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op,vdt", CASES)
def test_decode_combined_buckets(sc, op, vdt):
    rng = np.random.default_rng(100 + CASES.index((op, vdt)))
    keys, vals = rows(rng, 8000, vdt, finite=(op == "sum"))
    M, R = 4, 3
    starts = vb.slice_starts(len(keys), M)
    sh = vb.StrShuffle(sc, M, R, VCODE[vdt], AGG[op])
    for m in range(M):
        lo, hi = int(starts[m]), int(starts[m + 1])
        sh.map_blob(m, combined_blob(keys[lo:hi], vals[lo:hi], op, vdt))
    sh.seal()
    check_against_ref(parts_of(sh), keys, vals, op, vdt, M, R)
    sh.free()


@pytest.mark.parametrize("op,vdt", [("sum", "u64"), ("min", "f64"), ("count", "u64")])
def test_mixed_rows_and_blobs(sc, op, vdt):
    """Map ids 0, 2, 4 as rows (host, device, borrowed), 1, 3, 5 as blobs, map 3 from device memory."""
    rng = np.random.default_rng(7)
    keys, vals = rows(rng, 9000, vdt)
    M, R = 6, 5
    starts = vb.slice_starts(len(keys), M)
    sh = vb.StrShuffle(sc, M, R, VCODE[vdt], AGG[op])
    lib = sc._lib
    for m in range(M):
        lo, hi = int(starts[m]), int(starts[m + 1])
        if m % 2 == 0:
            kc, vc = columns(keys, None if op == "count" else vals, ("host", "device", "borrowed")[m // 2])
            sh.map(m, kc, vc, lo, hi)
        elif m == 3:
            raw = np.frombuffer(combined_blob(keys[lo:hi], vals[lo:hi], op, vdt), dtype=np.uint8)
            blob = torch.zeros(len(raw) + 1, dtype=torch.uint8, device="cuda")
            blob[1:] = torch.from_numpy(raw.copy()).cuda()          # an odd address: the decoder's loads are aligned
            torch.cuda.synchronize()
            L.check(lib.vb_shuffle_map_blob(sh._h, m, ctypes.c_void_p(blob.data_ptr() + 1), len(raw), L.VB_DEVICE))
        else:
            sh.map_blob(m, combined_blob(keys[lo:hi], vals[lo:hi], op, vdt))
    sh.seal()
    check_against_ref(parts_of(sh), keys, vals, op, vdt, M, R)
    sh.free()


def test_resubmission_last_wins(sc):
    """rows -> blob on map 0, blob -> rows on map 1: the stale submission's keys and values are gone."""
    rng = np.random.default_rng(8)
    keys, vals = rows(rng, 4000, "u64")
    stale_keys = ["stale-%d" % i for i in range(50)]
    stale_vals = np.arange(50, dtype=np.uint64)
    M, R = 2, 3
    starts = vb.slice_starts(len(keys), M)
    sh = vb.StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM)
    kc, vc = columns(stale_keys, stale_vals, "host")
    sh.map(0, kc, vc, 0, 50)
    sh.map_blob(0, combined_blob(keys[:starts[1]], vals[:starts[1]], "sum", "u64"))
    sh.map_blob(1, combined_blob(stale_keys, stale_vals, "sum", "u64"))
    kc, vc = columns(keys, vals, "host")
    sh.map(1, kc, vc, int(starts[1]), int(starts[2]))
    sh.seal()
    check_against_ref(parts_of(sh), keys, vals, "sum", "u64", M, R)
    sh.free()


# ---- round trip -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op,vdt", [("sum", "i64"), ("max", "f64"), ("count", "u64")])
def test_round_trip_between_shuffles(sc, op, vdt):
    """Shuffle A's reduce blobs, every partition, fed to shuffle B as map tasks: B's partitions equal A's."""
    rng = np.random.default_rng(9)
    keys, vals = rows(rng, 7000, vdt)
    a = build(sc, keys, vals, op, vdt, 3, 4)
    b = vb.StrShuffle(sc, 4, 4, VCODE[vdt], AGG[op])
    for r in range(4):
        b.map_blob(r, a.reduce_blob(r))
    b.seal()
    ga, gb = parts_of(a), parts_of(b)
    for r in range(4):
        assert ga[r].keys() == gb[r].keys()
        for k in ga[r]:
            assert _bits(ga[r][k], vdt if op != "count" else "u64") == _bits(gb[r][k], vdt if op != "count" else "u64"), (r, k)
    a.free()
    b.free()


# ---- rejection ------------------------------------------------------------------------------------------------------
def test_corrupt_blobs_rejected_then_valid_blob_accepted(sc):
    sh = vb.StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM)
    for shape, blob in corrupt_blobs().items():
        with pytest.raises(vb.VegaB200Error) as e:
            sh.map_blob(0, blob)
        assert e.value.code == L.VB_ERR_INVALID, shape
    lib = sc._lib
    ok = B.encode_str_pairs([("ab", 3), ("", 4)])
    assert lib.vb_shuffle_map_blob(sh._h, 1, ok, len(ok), L.VB_HOST) == L.VB_ERR_INVALID      # map id
    sh.map_blob(0, ok)
    sh.seal()
    got = {}
    for p in parts_of(sh):
        got.update(p)
    assert got == {"ab": 3, "": 4}
    sh.free()


# ---- across ranks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 3])
def test_blobs_across_ranks(sc, W):
    rng = np.random.default_rng(10 + W)
    keys, vals = rows(rng, 6000, "i64")
    M, R = 5, 7
    one = build(sc, keys, vals, "max", "i64", M, R)
    shs = run_ranks(sc, W, "max", "i64", keys, vals, M, R)
    for d, sh in enumerate(shs):
        for r in range(R):
            blob = sh.reduce_blob(r)
            assert sh.reduce_blob_size(r) == len(blob)
            if r % W == d:
                assert dict(B.decode_str_pairs(blob)) == dict(str_pairs(one, r)), (d, r)
            else:
                assert blob == b"\x00" * 8, (d, r)
    x = vb.StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM, rank=0, world=2)
    ok = B.encode_str_pairs([("ab", 3)])
    assert sc._lib.vb_shuffle_map_blob(x._h, 0, ok, len(ok), L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    for sh in shs + [one, x]:
        sh.free()
