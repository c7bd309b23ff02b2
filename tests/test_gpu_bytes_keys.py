"""Byte-slice keys on the device (vb_shuffle_set_str_key(VB_STRKEY_BYTES), Python vb.BytesKeys): every op of the
String-key shuffle over keys placed as Rust hashes a `Vec<u8>`.  Every check is per partition: each output key must sit
in partition vb_get_partition_bytes(key) (tests/test_bytes_keys_cpu.py pins it to tests/bytes_keys_ref.py), not merely
appear in the collected multiset, so a kind that were silently ignored would fail here.  Values are checked against
plain Python folds."""
import ctypes
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from tests import multirank as MR
from tests import str_blob_ref as SB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
BYTES, STR = L.VB_STRKEY_BYTES, L.VB_STRKEY_STR
AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "group": L.VB_AGG_GROUP}
VCODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def key_pool(seed=0, n_rand=3000):
    """Distinct keys: every length 0..72 (random, all NUL, all 0xFF), non-UTF-8 bytes, short random keys."""
    rng = np.random.default_rng(seed)
    ks = [b""]
    for n in range(1, 73):
        ks += [bytes(rng.integers(0, 256, n, dtype=np.uint8)), b"\x00" * n, b"\xff" * n]
    ks += [b"\x80\xfe not utf-8", b"a\x00b", "é".encode(), b"\xc3"]
    ks += [bytes(rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8)) for _ in range(n_rand)]
    return list(dict.fromkeys(ks))


BIG = bytes(np.random.default_rng(99).integers(0, 256, 1 << 20, dtype=np.uint8))   # a 1 MiB key


def rows(n, seed=1, big=True):
    rng = np.random.default_rng(seed)
    pool = key_pool(seed)
    keys = [pool[i] for i in rng.integers(0, len(pool), n)] + pool[:80]
    if big:
        keys += [BIG, BIG]
    return [keys[i] for i in rng.permutation(len(keys))]


def values(n, vdt, seed=2):
    rng = np.random.default_rng(seed)
    if vdt == "u64":
        return rng.integers(0, 1 << 64, n, dtype=np.uint64)
    if vdt == "i64":
        return rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)
    return rng.integers(-1000, 1000, n).astype(np.float64)       # exact sums in any order


def bytes_col(keys, where):
    k = vb.BytesKeys.from_bytes(keys)
    if where == "host":
        return k
    return vb.BytesKeys(torch.from_numpy(k.offsets.view(np.int64)).cuda(), torch.from_numpy(k.data.copy()).cuda())


def val_col(v, where):
    return v if where == "host" else torch.from_numpy(v).cuda()


def part_of(k, R):
    return vb.lib().vb_get_partition_bytes(ctypes.c_char_p(k), len(k), R)


def check_placed(keys, r, R):
    """keys (from partition r) are bytes, distinct, and every one is placed by the Vec<u8> hash."""
    ks = list(keys)
    assert all(type(k) is bytes for k in ks)
    assert len(set(ks)) == len(ks), f"a key twice in partition {r}"
    bad = [k[:16] for k in ks if part_of(k, R) != r]
    assert not bad, f"partition {r} of {R}: {len(bad)} keys placed elsewhere, first {bad[0]!r}"


def fold(op, vdt, keys, vals):
    out = {}
    for k, v in zip(keys, vals.tolist() if vals is not None else [1] * len(keys)):
        if op == "count":
            out[k] = out.get(k, 0) + 1
        elif k not in out:
            out[k] = v
        elif op == "sum":
            out[k] = out[k] + v
        elif op == "min":
            out[k] = min(out[k], v)
        else:
            out[k] = max(out[k], v)
    if op == "sum" and vdt in ("u64", "i64"):
        out = {k: x & M64 for k, x in out.items()}
    return out


def norm(x, op, vdt):
    x = x.item() if hasattr(x, "item") else x
    return int(x) & M64 if op == "count" or vdt in ("u64", "i64") else x


def collect_reduce(sh, R, op, vdt):
    got = {}
    for r in range(R):
        ks, comb = sh.reduce(r)[:2]
        check_placed(ks, r, R)
        got.update({k: norm(c, op, vdt) for k, c in zip(ks.tolist(), comb.tolist())})
    return got


# ---- one process ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 3, 257])
@pytest.mark.parametrize("where", ["host", "device"])
def test_reduce_ops_and_counts(sc, where, R):
    keys = rows(6000, seed=R)
    M = 4
    for vdt in ("u64", "i64", "f64"):
        if where == "device" and vdt == "u64" and not hasattr(torch, "uint64"):
            continue
        v = values(len(keys), vdt, seed=R + 5)
        rdd = sc.parallelize(bytes_col(keys, where), M, values=val_col(v, where))
        for op in ("sum", "min", "max"):
            want = {k: norm(x, op, vdt) for k, x in fold(op, vdt, keys, v).items()}
            assert collect_reduce(rdd.reduce_by_key(op, R)._run(), R, op, vdt) == want, (vdt, op)
        assert collect_reduce(rdd.count_by_key(R)._run(), R, "count", vdt) == fold("count", vdt, keys, None)
    r = sc.parallelize(bytes_col(keys, where), M)
    cbv = r.count_by_value()
    assert collect_reduce(cbv._run(), cbv.num_slices, "count", "u64") == fold("count", "u64", keys, None)
    d = r.distinct(R)
    dsh = d.sh._run()
    got = []
    for p in range(R):
        ks = dsh.reduce(p)[0]
        check_placed(ks, p, R)
        got += ks.tolist()
    assert sorted(got) == sorted(set(keys))


def group_want(keys, vals):
    out = {}
    for k, v in zip(keys, vals.tolist()):
        out.setdefault(k, []).append(v)
    return out


@pytest.mark.parametrize("R", [1, 3, 257])
def test_group_by_key_and_partition_by_key(sc, R):
    keys = rows(5000, seed=10 + R)
    v = values(len(keys), "u64", seed=3)
    rdd = sc.parallelize(vb.BytesKeys.from_bytes(keys), 3, values=v)
    sh = rdd.group_by_key(R)._run()
    got = {}
    for r in range(R):
        ks, offs, vals = sh.reduce(r)
        check_placed(ks, r, R)
        o = offs.astype(np.int64)
        got.update({k: vals[o[i]:o[i + 1]].tolist() for i, k in enumerate(ks.tolist())})
    assert got == group_want(keys, v)                # values in input order
    parts = rdd.partition_by_key(R).glom()
    assert sorted(np.concatenate(parts).tolist()) == sorted(v.tolist())


def test_combine_by_key_mean(sc):
    keys = rows(8000, seed=21)
    u = values(len(keys), "u64", seed=4)
    f = values(len(keys), "f64", seed=5)
    R = 5
    c = sc.parallelize(vb.BytesKeys.from_bytes(keys), 4, values=(u, f)).combine_by_key(
        {"n": ("count", None), "s": ("sum", 0), "avg": ("mean", 1)}, R)
    cnt, s, fs = {}, {}, {}
    for k, a, b in zip(keys, u.tolist(), f.tolist()):
        cnt[k] = cnt.get(k, 0) + 1
        s[k] = (s.get(k, 0) + a) & M64
        fs[k] = fs.get(k, 0.0) + b
    for r in range(R):
        ks, outs = c.compute(r)
        check_placed(ks, r, R)
        for i, k in enumerate(ks.tolist()):
            assert int(outs["n"][i]) == cnt[k] and int(outs["s"][i]) == s[k]
            assert outs["avg"][i] == fs[k] / cnt[k]


def _side(sc, keys, seed, M=3):
    return sc.parallelize(vb.BytesKeys.from_bytes(keys), M, values=values(len(keys), "u64", seed=seed))


def test_cogroup_and_joins(sc):
    R = 7
    ka, kb, kc = rows(3000, seed=31), rows(2000, seed=32, big=False), rows(1500, seed=33, big=False)
    a, b, c = _side(sc, ka, 1), _side(sc, kb, 2), _side(sc, kc, 3)
    va, vb_, vc = (group_want(k, values(len(k), "u64", seed=s)) for k, s in ((ka, 1), (kb, 2), (kc, 3)))
    cg = vb.StrCoGroupedRdd([a, b, c], R)
    seen = set()
    for r in range(R):
        ks, lists = cg.compute(r)
        check_placed(ks, r, R)
        for i, k in enumerate(ks.tolist()):
            seen.add(k)
            for (o, v), want in zip(lists, (va, vb_, vc)):
                assert v[int(o[i]):int(o[i + 1])].tolist() == want.get(k, [])
    assert seen == set(va) | set(vb_) | set(vc)
    inner = {k for k in va if k in vb_ and k in vc}
    for r in range(R):
        k, (x, y, z) = cg.join_compute(r)
        check_placed(set(k.tolist()), r, R)
        assert set(k.tolist()) <= inner
        assert len(k) == sum(len(va[q]) * len(vb_[q]) * len(vc[q]) for q in inner if part_of(q, R) == r)
        k, cols = cg.outer_join_compute(r, 1)                  # left outer: every key of parent 0
        assert set(k.tolist()) == {q for q in va if part_of(q, R) == r}
    # narrow joins: a reduce result and a combine aggregate joined where they are, beside a GROUP side
    red = a.reduce_by_key("sum", R)
    comb = sc.parallelize(vb.BytesKeys.from_bytes(kb), 3, values=(values(len(kb), "u64", seed=2),)).combine_by_key(
        {"n": ("count", None)}, R)
    sums = {q: sum(x) & M64 for q, x in va.items()}
    nj = vb.StrCoGroupedRdd([red, comb.aggregate("n"), b], R)
    for r in range(R):
        k, (x, y, z) = nj.join_compute(r)
        check_placed(set(k.tolist()), r, R)
        for q, s_, n_ in zip(k.tolist(), x.tolist(), y.tolist()):
            assert s_ == sums[q] and n_ == len(vb_[q])


def test_sort_by_key_equals_the_string_kind(sc):
    keys = rows(4000, seed=41)
    v = values(len(keys), "u64", seed=6)
    k = vb.BytesKeys.from_bytes(keys)
    as_bytes = vb.StrSortedRdd(sc.parallelize(k, 3, values=v), 5)
    as_str = vb.StrSortedRdd(sc.parallelize(vb.StrKeys(k.offsets, k.data), 3, values=v), 5)
    for r in range(5):
        gb, gs = as_bytes.compute_raw(r), as_str.compute_raw(r)
        assert all(np.array_equal(x, y) for x, y in zip(gb, gs)), r
    ks, vs = as_bytes.collect()
    assert ks.tolist() == sorted(keys) and all(type(q) is bytes for q in ks.tolist())


def test_byte_string_values(sc):
    keys = rows(3000, seed=51, big=False)
    rng = np.random.default_rng(7)
    vals = [bytes(rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8)) for _ in keys]
    R = 4
    sh = sc.parallelize(vb.BytesKeys.from_bytes(keys), 3, values=vals).group_by_key(R)._run()
    want = {}
    for q, x in zip(keys, vals):
        want.setdefault(q, []).append(x)
    got = {}
    for r in range(R):
        ks, offs, vs = sh.reduce(r)
        check_placed(ks, r, R)
        o = offs.astype(np.int64)
        got.update({q: list(vs[o[i]:o[i + 1]]) for i, q in enumerate(ks.tolist())})
    assert got == want


def test_reduce_blobs(sc):
    keys = rows(5000, seed=61)
    v = values(len(keys), "u64", seed=8)
    R, M = 6, 4
    sh = sc.parallelize(vb.BytesKeys.from_bytes(keys), M, values=v).reduce_by_key("sum", R)._run()
    want = fold("sum", "u64", keys, v)
    blobs = []
    for r in range(R):
        ks, comb = sh.reduce(r)
        check_placed(ks, r, R)
        blob = sh.reduce_blob(r)
        assert blob == SB.encode_str_pairs(list(zip(ks.tolist(), comb.tolist())))     # byte for byte, Vec<(Vec<u8>, u64)>
        blobs.append(blob)
    # decode: every blob a map task of a new bytes-kind shuffle, and rows beside them as one more task
    extra = rows(500, seed=62, big=False)
    ev = values(len(extra), "u64", seed=9)
    out = vb.StrShuffle(sc, R + 1, 3, L.VB_U64, L.VB_AGG_SUM, key_kind=BYTES)
    for m, blob in enumerate(blobs):
        out.map_blob(m, blob)
    out.map(R, vb.rdd._StrCol(vb.BytesKeys.from_bytes(extra)), vb.rdd._Col(ev, role="value"), 0, len(extra))
    out.seal()
    both = dict(want)
    for q, x in fold("sum", "u64", extra, ev).items():
        both[q] = (both.get(q, 0) + x) & M64
    assert collect_reduce(out, 3, "sum", "u64") == both


def _collision_child():
    """Group and join under 4-bit index fingerprints: equal fingerprints of distinct keys resolve by their bytes."""
    with vb.Context(0) as sc:
        keys = rows(3000, seed=71, big=False)
        v = values(len(keys), "u64", seed=1)
        a = sc.parallelize(vb.BytesKeys.from_bytes(keys), 3, values=v)
        R = 3
        sh = a.group_by_key(R)._run()
        want = group_want(keys, v)
        for r in range(R):
            ks, offs, vals = sh.reduce(r)
            check_placed(ks, r, R)
            o = offs.astype(np.int64)
            for i, q in enumerate(ks.tolist()):
                assert vals[o[i]:o[i + 1]].tolist() == want[q]
        kb = keys[::3]
        b = sc.parallelize(vb.BytesKeys.from_bytes(kb), 2, values=values(len(kb), "u64", seed=2))
        wb = group_want(kb, values(len(kb), "u64", seed=2))
        n = sum(len(vb.StrCoGroupedRdd([a, b], R).join_compute(r)[0]) for r in range(R))
        assert n == sum(len(want[q]) * len(wb[q]) for q in wb)


def test_index_collisions_resolve_by_bytes():
    env = dict(os.environ, VEGA_B200_STR_FP_BITS="4")
    p = subprocess.run([sys.executable, "-c", "from tests.test_gpu_bytes_keys import _collision_child as f; f()"], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]


def test_refusals(sc):
    lib = vb.lib()
    ints = vb.Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)
    assert lib.vb_shuffle_set_str_key(ints._h, BYTES) == L.VB_ERR_INVALID
    s = vb.StrShuffle(sc, 1, 3, L.VB_U64, L.VB_AGG_GROUP)
    assert lib.vb_shuffle_set_str_key(s._h, 2) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_set_str_key(s._h, BYTES) == L.VB_OK
    assert lib.vb_shuffle_set_str_key(s._h, STR) == L.VB_OK                   # may change its mind before a map call
    keys = [b"x", b"y", b"x", b"\x00"]
    v = np.arange(4, dtype=np.uint64)
    s.map(0, vb.rdd._StrCol(vb.BytesKeys.from_bytes(keys)), vb.rdd._Col(v, role="value"), 0, 4)
    assert lib.vb_shuffle_set_str_key(s._h, BYTES) == L.VB_ERR_STATE
    s.seal()
    assert lib.vb_shuffle_set_str_key(s._h, BYTES) == L.VB_ERR_STATE
    t = vb.StrShuffle(sc, 1, 3, L.VB_U64, L.VB_AGG_GROUP, key_kind=BYTES)
    t.map(0, vb.rdd._StrCol(vb.BytesKeys.from_bytes(keys)), vb.rdd._Col(v, role="value"), 0, 4)
    t.seal()
    sides = (ctypes.c_void_p * 2)(s._h.value, t._h.value)
    n = ctypes.c_uint64()
    assert lib.vb_cogroup_n_str_size(sides, 2, 0, ctypes.byref(n), None, None) == L.VB_ERR_INVALID
    assert lib.vb_join_n_str_size(sides, 2, 0, 3, ctypes.byref(n), None, None) == L.VB_ERR_INVALID
    assert lib.vb_cogroup_n_str(sides, 2, 0, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_join_n_str(sides, 2, 0, 3, None, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    for sh, kind in ((s, STR), (t, BYTES)):                                  # both stay usable
        one = (ctypes.c_void_p * 1)(sh._h.value)
        tot = 0
        for r in range(3):
            nk = ctypes.c_uint64()
            assert lib.vb_cogroup_n_str_size(one, 1, r, ctypes.byref(nk), None, None) == L.VB_OK
            tot += nk.value
            ks = sh.reduce(r)[0]
            if kind == BYTES:
                check_placed([q for q in ks.tolist()], r, 3)
        assert tot == 3


# ---- across ranks: W ranks in one process through export / import --------------------------------------------------
def _swap(exports):
    recv = MR.swap_columns([(cols, (nk, nb, nk, nv)) for (nk, nb, nv), cols in exports])
    return [(tuple(cols), (n[0], n[1], n[3])) for cols, n in recv]


def run_ranks(sc, W, op, keys, vals, M, R):
    k = vb.rdd._StrCol(vb.BytesKeys.from_bytes(keys))
    vc = vb.rdd._Col(vals, role="value") if op != "count" else None
    starts = vb.slice_starts(len(keys), M)
    shs = [vb.StrShuffle(sc, M, R, L.VB_U64, AGG[op], rank=r, world=W, key_kind=BYTES) for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            sh.map(m, k, vc, int(starts[m]), int(starts[m + 1]))
    for sh, (cols, counts) in zip(shs, _swap([sh.export() for sh in shs])):
        sh.import_(*cols, *counts)
    for sh in shs:
        sh.seal()
    return shs


@pytest.mark.parametrize("W", [2, 3, 8])
def test_multirank_export_import(sc, W):
    keys = rows(6000, seed=80 + W)
    v = values(len(keys), "u64", seed=W)
    M, R = 9, 11
    for op in ("sum", "group"):
        shs = run_ranks(sc, W, op, keys, v, M, R)
        got = {}
        for d, sh in enumerate(shs):
            for r in range(R):
                p = sh.reduce(r)
                if r % W != d:
                    assert len(p[0]) == 0
                    continue
                check_placed(p[0], r, R)
                if op == "group":
                    o = p[1].astype(np.int64)
                    got.update({q: p[2][o[i]:o[i + 1]].tolist() for i, q in enumerate(p[0].tolist())})
                else:
                    got.update(zip(p[0].tolist(), p[1].tolist()))
        if op == "group":
            assert got == group_want(keys, v)
        else:
            assert got == fold("sum", "u64", keys, v)
        for sh in shs:
            sh.free()
    # combine_by_key: the accumulator columns cross ranks beside the keys
    kcol = vb.rdd._StrCol(vb.BytesKeys.from_bytes(keys))
    vcols = (vb.rdd._Col(v, role="value"),)
    multi = ([L.VB_U64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0)])
    shs = [vb.StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, rank=r, world=W, multi=multi, key_kind=BYTES) for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        starts = vb.slice_starts(len(keys), M)
        for m in range(lo, hi):
            sh.map_cols(m, kcol, vcols, int(starts[m]), int(starts[m + 1]))
    exports = [sh.export_cols() for sh in shs]
    recv = MR.swap_columns([([lens, data, accs.t()], [nk, nb, nk]) for (nk, nb), (lens, data, accs) in exports])
    for sh, (rc, rs) in zip(shs, recv):
        sh.import_cols(rc[0], rc[1], rc[2].t().contiguous(), rs[0], rs[1])
    cnt, s = fold("count", "u64", keys, None), fold("sum", "u64", keys, v)
    n_keys = 0
    for d, sh in enumerate(shs):
        sh.seal()
        for r in range(R):
            ko, kb, (c0, c1) = sh.reduce_cols(r, [np.uint64, np.uint64])
            ks = vb.rdd._decode_keys(ko, kb, BYTES)
            if r % W != d:
                assert len(ks) == 0
                continue
            check_placed(ks, r, R)
            n_keys += len(ks)
            assert all(int(a) == cnt[q] and int(b) == s[q] for q, a, b in zip(ks.tolist(), c0, c1))
        sh.free()
    assert n_keys == len(cnt)


# ---- across ranks: the library's NCCL exchange, two ranks on one GPU -----------------------------------------------
N_X, M_X, R_X = 20_000, 5, 7


def _x_run(sc, rank, world, kind=BYTES, combine=False):
    keys = rows(N_X, seed=90, big=False)
    v = values(len(keys), "u64", seed=11)
    starts = vb.slice_starts(len(keys), M_X)
    lo, hi = vdist.map_block(rank, world, M_X)
    bk = vb.BytesKeys.from_bytes(keys)
    maps = [(m, vb.BytesKeys(bk.offsets[starts[m]:starts[m + 1] + 1], bk.data), v[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    out = {}
    if combine:
        eng = vdist.StrCombineCudaEngine(sc, key_kind=kind)
        multi = ([L.VB_U64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0)])
        sh = vdist.run_str_combine_shuffle(eng, [(m, k, (x,)) for m, k, x in maps], M_X, R_X, multi, rank, world)
        for r in range(R_X):
            ko, kb, cols = eng.reduce(sh, r, [np.uint64, np.uint64])
            out[r] = dict(zip(vb.rdd._decode_keys(ko, kb, kind).tolist(), zip(*[c.tolist() for c in cols])))
    else:
        eng = vdist.StrCudaEngine(sc, key_kind=kind)
        sh = vdist.run_str_shuffle(eng, maps, M_X, R_X, L.VB_U64, L.VB_AGG_SUM, rank, world)
        for r in range(R_X):
            ks, comb = eng.reduce(sh, r)
            out[r] = dict(zip(ks.tolist(), comb.tolist()))
    sh.free()
    return out


def _x_child(rank, outdir):
    sys.path.insert(0, ROOT)
    sc = vb.Context(0)
    idf = os.path.join(outdir, "uid")
    try:
        if rank == 0:
            with open(idf + ".tmp", "wb") as f:
                f.write(sc.comm_unique_id())
            os.replace(idf + ".tmp", idf)
        else:
            deadline = time.monotonic() + 60
            while not os.path.exists(idf) and time.monotonic() < deadline:
                time.sleep(0.05)
        with open(idf, "rb") as f:
            sc.comm_init(rank, 2, f.read())
    except (vb.VegaB200Error, OSError) as e:
        with open(os.path.join(outdir, f"init_failed{rank}"), "w") as f:
            f.write(str(e))
        sys.exit(3)
    res = [_x_run(sc, rank, 2), _x_run(sc, rank, 2, combine=True)]
    codes = []
    for combine in (False, True):                     # rank 0 String, rank 1 bytes: both refuse before any send
        try:
            _x_run(sc, rank, 2, kind=(STR, BYTES)[rank], combine=combine)
            codes.append(None)
        except vb.VegaB200Error as e:
            codes.append(e.code)
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, codes), f)
    sc.close()


def test_nccl_exchange_two_ranks_on_one_gpu(tmp_path):
    d = str(tmp_path)
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1")
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    code = "import sys; from tests.test_gpu_bytes_keys import _x_child; _x_child(int(sys.argv[1]), sys.argv[2])"
    procs = [subprocess.Popen([sys.executable, "-c", code, str(r), d], cwd=ROOT, stdout=logs[r], stderr=subprocess.STDOUT,
                              env=dict(env, NCCL_HOSTID=f"vega-b200-bytes-rank{r}")) for r in range(2)]
    deadline = time.monotonic() + 300
    try:
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            if any(p.poll() not in (None, 0) for p in procs):
                deadline = min(deadline, time.monotonic() + 10)
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
    out = []
    for lg in logs:
        lg.seek(0)
        out.append(lg.read()[-3000:])
        lg.close()
    refused = [os.path.join(d, f"init_failed{r}") for r in range(2) if os.path.exists(os.path.join(d, f"init_failed{r}"))]
    if refused:
        pytest.skip("NCCL did not initialise two ranks: " + open(refused[0]).read())
    assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
    ranks = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(2)]
    with vb.Context(0) as sc:
        want = [_x_run(sc, 0, 1), _x_run(sc, 0, 1, combine=True)]
    for j in range(2):
        for r in range(R_X):
            got = ranks[r % 2][0][j][r]
            assert got == want[j][r], (j, r)
            assert len(ranks[(r + 1) % 2][0][j][r]) == 0
            check_placed(got.keys(), r, R_X)
    assert [ranks[q][1] for q in range(2)] == [[L.VB_ERR_INVALID] * 2] * 2


def test_example_group_by_bytes():
    """examples/group_by_bytes.cpp: examples/group_by.rs's data with b"x" / b"y" keys; exit 0 only on the expected result."""
    path = os.path.join(ROOT, "examples", "_build", "group_by_bytes")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    p = subprocess.run([path], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
