"""Sorted value lists on the device (vb_shuffle_set_value_order, sort_values=True).  Every case runs the same input in
input order and sorted: each partition must hold the same keys with the same list lengths, and each sorted list must
equal the input-order list sorted by tests/sorted_groups_ref.py, bit for bit.

The device sort (segsort.cuh) picks its path by list length: 1 (untouched), 2 to SS_T = 8192 values in shared memory
(one size class per power of two), longer lists through the radix passes.  LENS covers both sides of every edge."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":                  # a rank of the two-rank exchange below, started as a script
    sys.path.insert(0, ROOT)

import vega_b200 as vb  # noqa: E402
from tests import multirank as MR  # noqa: E402
from tests import sorted_groups_ref as S  # noqa: E402
from tests.test_gpu_reduce_paths import _col, _dev  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200 import dist as vdist  # noqa: E402
from vega_b200.rdd import JoinedRdd, Shuffle, StrShuffle, _Col  # noqa: E402

pytestmark = pytest.mark.gpu
T = 8192
LENS = [1, 2, 3, 31, 32, 33, T - 1, T, T + 1, 100_000]
CODE = {np.uint64: L.VB_U64, np.int64: L.VB_I64, np.float64: L.VB_F64}
PHI = np.uint64(0x9E3779B97F4A7C15)
ASC, INP = L.VB_VALORDER_ASC, L.VB_VALORDER_INPUT


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def keyed(rng, lens, n_small=3000, small_max=40):
    """Keys with the given list lengths plus n_small keys of 1..small_max values, rows shuffled."""
    lens = list(lens) + rng.integers(1, small_max + 1, n_small).tolist()
    labels = (np.arange(len(lens), dtype=np.uint64) + np.uint64(1)) * PHI
    keys = np.repeat(labels, lens)
    return keys[rng.permutation(len(keys))]


def run(sc, maps, R, vcode, order, agg=L.VB_AGG_GROUP):
    """One shuffle; maps[m] = (key column or rows, value column or None, start, stop) or None (map task skipped).
    Returns every partition as (keys, offsets, values)."""
    sh = Shuffle(sc, len(maps), R, L.VB_U64, vcode, agg, value_order=order)
    try:
        for m, mp in enumerate(maps):
            if mp is not None:
                sh.map(m, *mp)
        sh.seal()
        return [sh.reduce(r) for r in range(R)]
    finally:
        sh.free()


def check_sorted(plain, srt):
    """srt (sorted) against plain (input order), partition by partition."""
    assert len(plain) == len(srt)
    for (pk, po, pv), (sk, so, sv) in zip(plain, srt):
        assert len(pk) == len(sk) and len(pv) == len(sv)
        want = S.triples(pk, po, S.sort_lists(po, pv))
        got = S.triples(sk, so, sv)
        for w, g in zip(want, got):
            assert np.array_equal(w, g)


def sliced(kc, vc, n, M):
    s = vb.slice_starts(n, M)
    return [(kc, vc, int(s[m]), int(s[m + 1])) for m in range(len(s) - 1)]


def both(sc, maps, R, vcode, agg=L.VB_AGG_GROUP):
    plain, srt = run(sc, maps, R, vcode, INP, agg), run(sc, maps, R, vcode, ASC, agg)
    check_sorted(plain, srt)
    return plain, srt


@pytest.mark.parametrize("R", [1, 8, 300])
@pytest.mark.parametrize("dtype", [np.uint64, np.int64, np.float64], ids=["u64", "i64", "f64"])
def test_every_length_class(sc, dtype, R):
    rng = np.random.default_rng(R)
    keys = keyed(rng, LENS)
    vals = S.full_range(rng, len(keys), dtype)
    plain, _ = both(sc, sliced(_Col(keys), _Col(vals, role="value"), len(keys), 4), R, CODE[dtype])
    lens = np.concatenate([np.diff(o.astype(np.int64)) for _, o, _ in plain])
    assert set(LENS) <= set(lens.tolist())


@pytest.mark.parametrize("R", [1, 8, 300])
def test_one_key_of_2_24_values(sc, R):
    rng = np.random.default_rng(5)
    keys = keyed(rng, [(1 << 24) + 5, 3 * T], n_small=20_000)
    vals = S.full_range(rng, len(keys), np.float64)
    kd, vd = _dev(keys), _dev(vals)
    both(sc, sliced(_col(kd, L.VB_U64), _col(vd, L.VB_F64), len(keys), 3), R, L.VB_F64)


def test_many_tiny_lists(sc):
    rng = np.random.default_rng(9)
    keys = rng.integers(0, 1_500_000, 3_000_000).astype(np.uint64) * PHI
    vals = S.full_range(rng, len(keys), np.int64)
    both(sc, sliced(_col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_I64), len(keys), 2), 16, L.VB_I64)


@pytest.mark.parametrize("where", ["host_soa", "device_copy", "borrowed", "host_aos", "device_aos"])
def test_map_inputs(sc, where):
    rng = np.random.default_rng(3)
    keys = keyed(rng, [T + 100, 500, 2], n_small=5000)
    vals = S.full_range(rng, len(keys), np.uint64)
    n = len(keys)
    if where in ("host_aos", "device_aos"):
        rows = np.stack([keys, vals], axis=1)
        kc = _Col(rows, allow_rows=True) if where == "host_aos" else _col(_dev(rows), L.VB_U64, rows=True)
        maps = sliced(kc, None, n, 3)
    else:
        kc, vc = (_Col(keys), _Col(vals, role="value")) if where == "host_soa" else \
                 (_col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_U64))
        if where == "device_copy":
            kc.loc = vc.loc = L.VB_DEVICE
        maps = sliced(kc, vc, n, 3)
    both(sc, maps, 7, L.VB_U64)


def test_resubmitted_map_and_empty_shuffle(sc):
    rng = np.random.default_rng(4)
    keys = keyed(rng, [T + 1, 40], n_small=2000)
    vals = S.full_range(rng, len(keys), np.int64)
    stale = S.full_range(rng, len(keys), np.int64)
    for order in (INP, ASC):
        sh = Shuffle(sc, 2, 5, L.VB_U64, L.VB_I64, L.VB_AGG_GROUP, value_order=order)
        h = len(keys) // 2
        sh.map(0, _Col(keys), _Col(stale, role="value"), 0, h)
        sh.map(0, _Col(keys), _Col(vals, role="value"), 0, h)       # the stage is resubmitted: the second one counts
        sh.map(1, _Col(keys), _Col(vals, role="value"), h, len(keys))
        sh.seal()
        parts = [sh.reduce(r) for r in range(5)]
        sh.free()
        if order == INP:
            plain = parts
    check_sorted(plain, parts)
    empty = np.zeros(0, dtype=np.uint64)
    for order in (INP, ASC):
        parts = run(sc, [(_Col(empty), _Col(empty, role="value"), 0, 0)], 3, L.VB_U64, order)
        assert all(len(k) == 0 and len(v) == 0 for k, _, v in parts)


# ---- cogroup and the joins -------------------------------------------------------------------------------------------
def side(sc, keys, vals, R, order):
    sh = Shuffle(sc, 2, R, L.VB_U64, L.VB_I64, L.VB_AGG_COGROUP, value_order=order)
    for m, mp in enumerate(sliced(_Col(keys), _Col(vals, role="value"), len(keys), 2)):
        sh.map(m, *mp)
    sh.seal()
    return sh


def lists(keys, vals, order):
    """{key: its list} in input order, or sorted."""
    o = np.argsort(keys, kind="stable")
    k, v = keys[o], vals[o]
    cut = np.flatnonzero(np.diff(k)) + 1
    out = {}
    for kk, vv in zip(np.split(k, cut), np.split(v, cut)):
        if len(kk):
            out[int(kk[0])] = S.sort_lists([0, len(vv)], vv) if order == ASC else vv
    return out


def side_data(rng, n_keys, shift, n=40_000):
    keys = (rng.integers(0, n_keys, n).astype(np.uint64) + np.uint64(shift)) * PHI
    keys[:T + 10] = np.array([shift + 1], dtype=np.uint64) * PHI    # one list on the radix path on each side
    keys = keys[rng.permutation(len(keys))]
    return keys, S.full_range(rng, len(keys), np.int64)


def nested(lists_by_side, kinds):
    """{key: [row tuple]} of the N-way join (None for an optional side that lacks the key)."""
    out = {}
    for k in set().union(*[set(d) for d in lists_by_side]):
        cols = [d.get(k) for d in lists_by_side]
        if any(c is None and req for c, req in zip(cols, kinds)):
            continue
        rows = [()]
        for c in cols:
            rows = [r + (x,) for r in rows for x in (c.view(np.uint64).tolist() if c is not None else [None])]
        out[k] = rows
    return out


def by_key(k, cols):
    out = {}
    vals = [(c.data.view(np.uint64).tolist(), np.ma.getmaskarray(c).tolist()) if isinstance(c, np.ma.MaskedArray)
            else (np.asarray(c).view(np.uint64).tolist(), [False] * len(c)) for c in cols]
    for i, kk in enumerate(np.asarray(k).view(np.uint64).tolist()):
        out.setdefault(kk, []).append(tuple(None if m[i] else v[i] for v, m in vals))
    return out


@pytest.mark.parametrize("orders", [(ASC, ASC), (ASC, INP), (INP, ASC)], ids=["both", "left", "right"])
def test_cogroup_and_joins_follow_each_side(sc, orders):
    rng = np.random.default_rng(12)
    R = 6
    data = [side_data(rng, 3000, 0), side_data(rng, 3000, 1500)]
    shs = [side(sc, k, v, R, o) for (k, v), o in zip(data, orders)]
    want = [lists(k, v, o) for (k, v), o in zip(data, orders)]
    try:
        for kind, req in ((None, (True, True)), ("left", (True, False)), ("right", (False, True)), ("full", (False, False))):
            j = JoinedRdd.__new__(JoinedRdd)
            j.sc, j.num_slices, j.kind, j._shs = sc, R, kind, tuple(shs)
            k, v, w = j.collect()
            assert by_key(k, [v, w]) == nested(want, req), kind
        j = JoinedRdd.__new__(JoinedRdd)
        j.sc, j.num_slices, j.kind, j._shs = sc, R, None, tuple(shs)
        for k, (vs, ws) in j.cogroup_collect():
            for got, d in ((vs, want[0]), (ws, want[1])):
                exp = d.get(int(np.uint64(k)), np.zeros(0, dtype=np.int64))
                assert np.array_equal(np.asarray(got).view(np.uint64), exp.view(np.uint64))
    finally:
        for s in shs:
            s.free()


def test_filtered_inner_join_inherits_the_order(sc):
    """Both sides still lazy: the inner join groups only the keys on both sides, in internal shuffles cut from the
    user's (filtered_pair); those must sort as the user's shuffles do."""
    rng = np.random.default_rng(13)
    data = [side_data(rng, 4000, 0), side_data(rng, 4000, 3000)]
    for orders in ((ASC, ASC), (ASC, INP)):
        shs = [side(sc, k, v, 5, o) for (k, v), o in zip(data, orders)]
        want = [lists(k, v, o) for (k, v), o in zip(data, orders)]
        j = JoinedRdd.__new__(JoinedRdd)
        j.sc, j.num_slices, j.kind, j._shs = sc, 5, None, tuple(shs)
        k, v, w = j.collect()
        assert by_key(k, [v, w]) == nested(want, (True, True))
        for s in shs:
            s.free()


def test_n_way_with_mixed_sides(sc):
    rng = np.random.default_rng(14)
    R = 4
    orders = (ASC, INP, ASC)
    data = [side_data(rng, 2000, 700 * j, n=16_000) for j in range(3)]
    shs = [side(sc, k, v, R, o) for (k, v), o in zip(data, orders)]
    want = [lists(k, v, o) for (k, v), o in zip(data, orders)]
    cg = vb.CoGroupedRdd.__new__(vb.CoGroupedRdd)
    cg.rdds, cg.num_slices, cg.sc, cg._shs = [None] * 3, R, sc, shs
    try:
        for k, ls in cg.collect():
            for got, d in zip(ls, want):
                exp = d.get(int(np.uint64(k)), np.zeros(0, dtype=np.int64))
                assert np.array_equal(np.asarray(got).view(np.uint64), exp.view(np.uint64))
        k, cols = cg.join_collect()
        assert by_key(k, cols) == nested(want, (True, True, True))
        for mask in (0b101, 0):
            k, cols = cg.outer_join_collect(mask)
            assert by_key(k, cols) == nested(want, tuple(bool(mask >> j & 1) for j in range(3)))
    finally:
        for s in shs:
            s.free()


def test_pair_rdd_api(sc):
    rng = np.random.default_rng(15)
    (k1, v1), (k2, v2) = side_data(rng, 1000, 0), side_data(rng, 1000, 500)
    a, b = sc.parallelize(k1, 3, values=v1), sc.parallelize(k2, 2, values=v2)
    g0, g1 = a.group_by_key(5).collect(), a.group_by_key(5, sort_values=True).collect()
    check_sorted([(g0.keys, g0.offsets, g0.vals)], [(g1.keys, g1.offsets, g1.vals)])
    want = [lists(k1, v1, ASC), lists(k2, v2, ASC)]
    k, v, w = a.join(b, 4, sort_values=True).collect()
    assert by_key(k, [v, w]) == nested(want, (True, True))
    k, v, w = a.full_outer_join(b, 4, sort_values=True).collect()
    assert by_key(k, [v, w]) == nested(want, (False, False))
    k, cols = vb.CoGroupedRdd([a, b], 3, sort_values=True).join_collect()
    assert by_key(k, cols) == nested(want, (True, True))


# ---- String keys ----------------------------------------------------------------------------------------------------
def str_keys(rng, n):
    words = ["", "k\x00", "é-ключ"] + ["w%05d" % i for i in range(3000)]
    idx = rng.integers(0, len(words), n)
    idx[:T + 50] = 7                                               # one list on the radix path
    return [words[i] for i in idx[rng.permutation(n)]]


@pytest.mark.parametrize("kind", [L.VB_STRKEY_STR, L.VB_STRKEY_BYTES], ids=["str", "bytes"])
@pytest.mark.parametrize("dtype", [np.uint64, np.float64], ids=["u64", "f64"])
def test_string_group(sc, kind, dtype):
    rng = np.random.default_rng(21)
    n = 60_000
    keys = str_keys(rng, n)
    if kind == L.VB_STRKEY_BYTES:
        keys = [k.encode() for k in keys]
        keys = vb.BytesKeys.from_bytes(keys)
    vals = S.full_range(rng, n, dtype)
    res = []
    for order in (INP, ASC):
        sh = StrShuffle(sc, 3, 6, CODE[dtype], L.VB_AGG_GROUP, key_kind=kind, value_order=order)
        s = vb.slice_starts(n, 3)
        kc = vb.rdd._StrCol(keys)
        for m in range(3):
            sh.map(m, kc, _Col(vals, role="value"), int(s[m]), int(s[m + 1]))
        sh.seal()
        res.append([sh.reduce(r) for r in range(6)])
        sh.free()
    check_sorted(*[[(np.array([repr(x) for x in k]), o, v) for k, o, v in parts] for parts in res])


def test_str_cogrouped_joins(sc):
    rng = np.random.default_rng(22)
    k1, k2 = str_keys(rng, 30_000), str_keys(rng, 20_000)
    v1, v2 = S.full_range(rng, 30_000, np.int64), S.full_range(rng, 20_000, np.int64)
    a, b = sc.parallelize(k1, 3, values=v1), sc.parallelize(k2, 2, values=v2)
    cg = vb.StrCoGroupedRdd([a, b], 4, sort_values=True)
    ref = []
    for ks, vs in ((k1, v1), (k2, v2)):
        d = {}
        for kk, vv in zip(ks, vs.view(np.uint64).tolist()):
            d.setdefault(kk, []).append(vv)
        ref.append({kk: S.sort_lists([0, len(x)], np.array(x, dtype=np.uint64).view(np.int64)) for kk, x in d.items()})
    for k, ls in cg.collect():
        for got, d in zip(ls, ref):
            assert np.array_equal(np.asarray(got).view(np.uint64), d.get(k, np.zeros(0, dtype=np.int64)).view(np.uint64))
    k, cols = cg.outer_join_collect(0b01)
    got = {}
    vals = [(c.data.view(np.uint64).tolist(), np.ma.getmaskarray(c).tolist()) if isinstance(c, np.ma.MaskedArray)
            else (np.asarray(c).view(np.uint64).tolist(), [False] * len(c)) for c in cols]
    for i, kk in enumerate(k.tolist()):
        got.setdefault(kk, []).append(tuple(None if m[i] else v[i] for v, m in vals))
    want = {}
    for kk, vs in ref[0].items():
        ws = ref[1].get(kk)
        want[kk] = [(v, w) for v in vs.view(np.uint64).tolist() for w in (ws.view(np.uint64).tolist() if ws is not None else [None])]
    assert got == want


# ---- across ranks -------------------------------------------------------------------------------------------------
class SortedEngine(vdist.CudaEngine):
    def __init__(self, sc, order):
        super().__init__(sc)
        self.order = order

    def create(self, *a, **k):
        sh = super().create(*a, **k)
        vdist._set_value_order(sh, self.order)
        return sh


@pytest.mark.parametrize("W", [2, 3, 8])
def test_multirank_integer(sc, W):
    rng = np.random.default_rng(W)
    keys = keyed(rng, [T + 3, 600, 2], n_small=4000)
    vals = S.full_range(rng, len(keys), np.float64)
    M, R = 2 * W + 1, 2 * W + 3
    maps = MR.maps_by_rank(len(keys), M, W, lambda m, lo, hi: (keys[lo:hi], vals[lo:hi]))
    out = []
    for order in (INP, ASC):
        eng = SortedEngine(sc, order)
        shs, _ = MR.run_ranks(eng, W, L.VB_AGG_GROUP, maps, R, L.VB_U64, L.VB_F64, n_map=M)
        out.append(MR.owned_parts(eng, shs, R))
        for s in shs:
            s.free()
    check_sorted(*out)


@pytest.mark.parametrize("W", [2, 3, 8])
def test_multirank_string(sc, W):
    rng = np.random.default_rng(30 + W)
    n = 30_000
    keys = str_keys(rng, n)
    vals = S.full_range(rng, n, np.int64)
    M, R = W + 2, 2 * W + 1
    starts = vb.slice_starts(n, M)
    out = []
    for order in (INP, ASC):
        eng = vdist.StrCudaEngine(sc)
        shs = [StrShuffle(sc, M, R, L.VB_I64, L.VB_AGG_GROUP, rank=r, world=W, value_order=order) for r in range(W)]
        for r in range(W):
            lo, hi = vdist.map_block(r, W, M)
            for m in range(lo, hi):
                eng.map(shs[r], m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]])
        exports = [vdist._str_export(eng, sh, W) for sh in shs]
        for sh, (cols, splits) in zip(shs, MR.swap_columns(exports)):
            vdist._str_import(eng, sh, cols, splits)
        for sh in shs:
            sh.seal()
        parts = [None] * R
        for d, sh in enumerate(shs):
            for r in range(R):
                if r % W == d:
                    k, o, v = sh.reduce(r)
                    parts[r] = (np.array([repr(x) for x in k]), o, v)
        out.append(parts)
        for sh in shs:
            sh.free()
    check_sorted(*out)


# ---- the library's NCCL exchange, two ranks on one GPU ----------------------------------------------------------------
NX, MX, RX = 50_000, 5, 7


def _xdata():
    rng = np.random.default_rng(41)
    keys = keyed(rng, [T + 7, 300], n_small=5000)[:NX]
    vals = S.full_range(rng, len(keys), np.float64)
    words = ["w%04d" % i for i in range(1500)] + ["é-ключ"]
    strs = [words[i] for i in rng.integers(0, len(words), len(keys))]
    return keys, vals, strs


def _xcase(sc, case, order, rank, world):
    keys, vals, strs = _xdata()
    n = len(keys)
    starts = vb.slice_starts(n, MX)
    lo, hi = vdist.map_block(rank, world, MX)
    out = {}
    if case == "str":
        maps = [(m, strs[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        sh = vdist.run_str_shuffle(vdist.StrCudaEngine(sc), maps, MX, RX, L.VB_F64, L.VB_AGG_GROUP, rank, world,
                                   value_order=order)
        for r in range(RX):
            k, o, v = sh.reduce(r)
            out[r] = ([repr(x) for x in k], np.asarray(o).tolist(), np.asarray(v).view(np.uint64).tolist())
    else:
        maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        sh = vdist.run_shuffle(vdist.CudaEngine(sc), maps, MX, RX, L.VB_U64, L.VB_F64, L.VB_AGG_GROUP, rank, world,
                               p2p=case == "p2p", value_order=order)
        for r in range(RX):
            k, o, v = sh.reduce(r)
            out[r] = (np.asarray(k).view(np.uint64).tolist(), np.asarray(o).tolist(), np.asarray(v).view(np.uint64).tolist())
    sh.free()
    return out


XCASES = [("int", ASC), ("p2p", ASC), ("str", ASC)]


def _child(rank, outdir):
    c = vb.Context(0)
    idf = os.path.join(outdir, "uid")
    try:
        if rank == 0:
            with open(idf + ".tmp", "wb") as f:
                f.write(c.comm_unique_id())
            os.replace(idf + ".tmp", idf)
        else:
            deadline = time.monotonic() + 60
            while not os.path.exists(idf) and time.monotonic() < deadline:
                time.sleep(0.05)
        with open(idf, "rb") as f:
            c.comm_init(rank, 2, f.read())
    except (vb.VegaB200Error, OSError) as e:
        with open(os.path.join(outdir, f"init_failed{rank}"), "w") as f:
            f.write(str(e))
        sys.exit(3)
    res = {case: _xcase(c, case, order, rank, 2) for case, order in XCASES}
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    c.close()


@pytest.fixture(scope="module")
def xranks(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sorted_exchange"))
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1",
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), d], cwd=ROOT, stdout=logs[r],
                              stderr=subprocess.STDOUT, env=dict(env, NCCL_HOSTID=f"vega-b200-sorted{r}")) for r in range(2)]
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
        pytest.skip("NCCL did not initialise two ranks on one GPU: " + open(refused[0]).read())
    assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
    return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(2)]


@pytest.mark.parametrize("case", [c for c, _ in XCASES])
def test_nccl_exchange_two_ranks_on_one_gpu(xranks, sc, case):
    plain = _xcase(sc, case, INP, 0, 1)
    for r in range(RX):
        k, o, v = xranks[r % 2][case][r]
        pk, po, pv = plain[r]
        kd = None if case == "str" else np.uint64
        check_sorted([(np.array(pk, dtype=kd), np.array(po), np.array(pv, dtype=np.uint64).view(np.float64))],
                     [(np.array(k, dtype=kd), np.array(o), np.array(v, dtype=np.uint64).view(np.float64))])
        assert len(xranks[(r + 1) % 2][case][r][0]) == 0, f"partition {r} on the rank that does not own it"


# ---- errors ---------------------------------------------------------------------------------------------------------
def code(fn):
    with pytest.raises(vb.VegaB200Error) as e:
        fn()
    return e.value.code


def test_error_codes(sc):
    lib = sc._lib
    set_ = lambda sh, o: L.check(lib.vb_shuffle_set_value_order(sh._h, o))
    g = Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP)
    assert code(lambda: set_(g, 2)) == L.VB_ERR_INVALID
    assert code(lambda: set_(g, -1)) == L.VB_ERR_INVALID
    set_(g, ASC)
    set_(g, INP)
    set_(g, ASC)
    k = np.arange(10, dtype=np.uint64)
    g.map(0, _Col(k), _Col(k, role="value"), 0, 10)
    assert code(lambda: set_(g, ASC)) == L.VB_ERR_STATE
    g.seal()
    assert code(lambda: set_(g, INP)) == L.VB_ERR_STATE
    for agg in (L.VB_AGG_SUM, L.VB_AGG_MIN, L.VB_AGG_MAX, L.VB_AGG_COUNT, L.VB_AGG_SORT):
        s = Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, agg)
        assert code(lambda: set_(s, ASC)) == L.VB_ERR_INVALID
        if agg == L.VB_AGG_SUM:
            s.map(0, _Col(k), _Col(k, role="value"), 0, 10)
            s.seal()
            v = Shuffle.narrow(s, 0, L.VB_U64)
            assert code(lambda: set_(v, ASC)) == L.VB_ERR_INVALID      # the kind before the (sealed) state
            v.free()
        s.free()
    m = Shuffle(sc, 1, 2, L.VB_U64, None, None, multi=([L.VB_U64], [(L.VB_AGG_SUM, 0)]))
    assert code(lambda: set_(m, ASC)) == L.VB_ERR_INVALID
    for agg in (L.VB_AGG_GROUP, L.VB_AGG_COGROUP):
        b = Shuffle(sc, 1, 2, L.VB_U64, L.VB_BYTES, agg)
        assert code(lambda: set_(b, ASC)) == L.VB_ERR_UNSUPPORTED
        b.free()
    rp = vb.rdd.RepShuffle(sc, 1, 2, [L.VB_U64], False)
    assert code(lambda: set_(rp, ASC)) == L.VB_ERR_INVALID
    assert code(lambda: StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM, value_order=ASC)) == L.VB_ERR_INVALID
    assert code(lambda: StrShuffle(sc, 1, 2, L.VB_U64, None, sort=True, value_order=ASC)) == L.VB_ERR_INVALID
    bd = StrShuffle.bytes_dist(sc, 1, 2, 0, 2)
    assert code(lambda: set_(bd, ASC)) == L.VB_ERR_UNSUPPORTED
    bd.free()
    s = StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_GROUP)
    s.map(0, vb.rdd._StrCol(["a", "b"]), _Col(k[:2], role="value"), 0, 2)
    assert code(lambda: set_(s, ASC)) == L.VB_ERR_STATE
    s.free()
    with pytest.raises(TypeError):
        sc.parallelize(k, 1, values=["x"] * 10).group_by_key(2, sort_values=True)
    with pytest.raises(TypeError):
        sc.parallelize(k, 1, values=k).group_by_key(2, sort_values=1)


def test_cpp_example_runs():
    """examples/sorted_groups.cpp splits each user's sorted event times into sessions and joins with sorted_values; it
    exits 0 only on the expected sessions and on (v, w)-ordered join rows."""
    path = os.path.join(ROOT, "examples", "_build", "sorted_groups")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "user 7: sessions [[3, 5, 20], [90, 95]]" in out.stdout, out.stdout


if __name__ == "__main__":
    _child(int(sys.argv[1]), sys.argv[2])
