"""String keys across ranks, W ranks in one process and one context (vb_shuffle_create_str_dist, the string export /
import calls): the four exported columns of every rank are swapped with torch.cat, source-rank major, as the
all-to-all-v of vega_b200/dist.py would deliver them.  Every case asserts that partition r has keys only on rank
r % W, and that the owners' partitions equal both the one-process string shuffle over the same map tasks and
oracle/pyref.py: integer ops, COUNT and f64 MIN / MAX bit for bit, f64 SUM within the bound of any summation order,
GROUP lists in map-id order."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from tests import multirank as MR
from tests.test_gpu_str_keys import check_parts, key_pool, ref_parts, rows_from_pool
from tests.test_gpu_str_join import cogroup_part, join_part
from tests.util import rand_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "group": L.VB_AGG_GROUP}
VCODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


# ---- the W-rank harness ---------------------------------------------------------------------------------------------
def swap(exports):
    """exports[src] = ((n_keys, n_key_bytes, n_vals) per destination, (key_lens, key_bytes, val_counts, vals)) ->
    per destination (columns, counts per source), the sources concatenated in ascending order."""
    recv = MR.swap_columns([(cols, (nk, nb, nk, nv)) for (nk, nb, nv), cols in exports])
    return [(tuple(cols), (n[0], n[1], n[3])) for cols, n in recv]


def columns(keys, vals, where):
    """(_StrCol, _Col or None) of the whole input in `where`: host, device (copied in the call) or borrowed."""
    h = vb.StrKeys.from_strs(keys)
    if where == "host":
        kc = vb.rdd._StrCol(h)
        vc = vb.rdd._Col(vals, role="value") if vals is not None else None
        return kc, vc
    kc = vb.rdd._StrCol(vb.StrKeys(torch.from_numpy(h.offsets.view(np.int64)).cuda(), torch.from_numpy(h.data.copy()).cuda()))
    vc = vb.rdd._Col(torch.from_numpy(vals).cuda(), role="value") if vals is not None else None
    if where == "device":
        kc.loc = L.VB_DEVICE
        if vc is not None:
            vc.loc = L.VB_DEVICE
    return kc, vc


def run_ranks(sc, W, op, vdt, keys, vals, M, R, where="host", resubmit=None):
    """One shuffle on W ranks: rank r maps its map_block tasks (slices of one column), all export, swap, import,
    seal.  resubmit(sh, map_id) may map a task again before the export.  Returns the sealed shuffles by rank."""
    kc, vc = columns(keys, None if op == "count" else vals, where)
    starts = vb.slice_starts(len(keys), M) if keys else np.zeros(M + 1, dtype=np.int64)
    shs = [vb.StrShuffle(sc, M, R, VCODE[vdt], AGG[op], rank=r, world=W) for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            if resubmit:
                resubmit(sh, m)
            sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
    if W == 1:
        shs[0].seal()
        return shs
    exports = [sh.export() for sh in shs]
    for sh, (cols, counts) in zip(shs, swap(exports)):
        sh.import_(*cols, *counts)
    for sh in shs:
        sh.seal()
    return shs


def part_dict(p, op):
    keys = p[0].tolist()
    assert len(set(keys)) == len(keys), "a key twice in one partition"
    if op == "group":
        o, v = p[1].astype(np.int64), p[2]
        assert o[0] == 0 and o[-1] == len(v)
        return {k: v[o[i]:o[i + 1]].tolist() for i, k in enumerate(keys)}
    return dict(zip(keys, p[1].tolist()))


def owned(shs, op, R):
    """The owners' partitions, asserting that every other rank's copy of a partition is empty."""
    W = len(shs)
    out = [None] * R
    for d, sh in enumerate(shs):
        for r in range(R):
            p = sh.reduce(r)
            if r % W == d:
                out[r] = part_dict(p, op)
            else:
                assert len(p[0]) == 0, f"rank {d} holds keys of partition {r}, owned by rank {r % W}"
    return out


def bits_equal(got, want, op, vdt):
    """Bit for bit, NaN payloads included."""
    def b(x):
        if vdt == "f64" and op != "count":
            return np.float64(x).view(np.uint64).item()
        return int(x)
    for r, (g, w) in enumerate(zip(got, want)):
        assert g.keys() == w.keys(), r
        for k in w:
            if op == "group":
                assert [b(x) for x in g[k]] == [b(x) for x in w[k]], (r, k)
            else:
                assert b(g[k]) == b(w[k]), (r, k, g[k], w[k])


def f64_sum_within_bound(got, keys, vals):
    per_key = {}
    for k, v in zip(keys, vals.tolist()):
        per_key.setdefault(k, []).append(v)
    for g in got:
        for k, x in g.items():
            xs = per_key[k]
            if any(math.isnan(v) for v in xs) or (math.inf in xs and -math.inf in xs):
                assert math.isnan(x), k
            elif math.inf in xs or -math.inf in xs:
                assert x == (math.inf if math.inf in xs else -math.inf), k
            else:
                m, u = len(xs), 2.0 ** -53
                bound = (m - 1) * u / (1 - (m - 1) * u) * sum(abs(v) for v in xs) * (1 + 2 * m * u)
                s_ = math.fsum(xs)
                assert abs(x - s_) <= bound + math.ulp(s_), (k, x, s_)


def check_case(sc, W, op, vdt, keys, vals, M, R, where="host"):
    got = owned(run_ranks(sc, W, op, vdt, keys, vals, M, R, where), op, R)
    single = owned(run_ranks(sc, 1, op, vdt, keys, vals, M, R), op, R)
    assert sum(len(g) for g in got) == sum(len(s) for s in single)
    if op == "sum" and vdt == "f64":
        f64_sum_within_bound(got, keys, vals)
        f64_sum_within_bound(single, keys, vals)
        assert [g.keys() for g in got] == [s.keys() for s in single]
    else:
        bits_equal(got, single, op, vdt)
        check_parts(got, ref_parts(keys, vals, op, vdt, M, R), op, vdt)
    return got


def data(seed, n, op, vdt, mode, hot=0.2):
    """Word-like keys from the string pool (the empty key, NULs, non-ASCII, keys of 10 kB), one hot key carrying
    `hot` of the rows, and values over the full range of the dtype (or f64 specials)."""
    rng = np.random.default_rng(seed)
    keys = rows_from_pool(rng, key_pool(rng), n)
    for i in np.flatnonzero(rng.random(n) < hot):
        keys[i] = "the"
    _, vals = rand_pairs(rng, n, 100, vdtype=vdt, values=mode)
    return keys, vals


# ---- ops x dtypes x world -------------------------------------------------------------------------------------------
OPS = [("sum", "u64", "full"), ("sum", "i64", "full"), ("sum", "f64", "default"), ("sum", "f64", "cancel"),
       ("min", "u64", "full"), ("min", "i64", "full"), ("min", "f64", "special"),
       ("max", "u64", "full"), ("max", "i64", "full"), ("max", "f64", "special"),
       ("count", "u64", "default"), ("group", "u64", "full"), ("group", "f64", "special")]


@pytest.mark.parametrize("op,vdt,mode", OPS)
@pytest.mark.parametrize("W", [2, 3, 8])
def test_ops_match_single_process_and_reference(sc, op, vdt, mode, W):
    """W = 8 > M = 5: three ranks have no map task and only receive."""
    keys, vals = data(hash((op, vdt, mode, W)) & 0xFFFF, 6000, op, vdt, mode)
    check_case(sc, W, op, vdt, keys, vals, 5, 7)


@pytest.mark.parametrize("op,vdt,mode", [("sum", "i64", "full"), ("min", "f64", "special"), ("count", "u64", "default"),
                                         ("group", "u64", "full")])
def test_256_ranks(sc, op, vdt, mode):
    """world at its cap, far more ranks than map tasks and partitions than keys on most ranks."""
    keys, vals = data(11, 3000, op, vdt, mode)
    check_case(sc, 256, op, vdt, keys, vals, 6, 300)


@pytest.mark.parametrize("where", ["host", "device", "borrowed"])
@pytest.mark.parametrize("op", ["sum", "max", "count", "group"])
def test_input_locations(sc, where, op):
    keys, vals = data(7, 5000, op, "i64", "full")
    check_case(sc, 3, op, "i64", keys, vals, 4, 11, where)


def test_world_one_is_the_one_process_shuffle(sc):
    keys, vals = data(8, 3000, "group", "u64", "full")
    got = owned(run_ranks(sc, 1, "group", "u64", keys, vals, 3, 5), "group", 5)
    sh = vb.StrShuffle(sc, 3, 5, L.VB_U64, L.VB_AGG_GROUP, rank=0, world=1)
    kc, vc = columns(keys, vals, "host")
    starts = vb.slice_starts(len(keys), 3)
    for m in range(3):
        sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    assert owned([sh], "group", 5) == got
    check_parts(got, ref_parts(keys, vals, "group", "u64", 3, 5), "group", "u64")


def test_long_keys_and_one_hot_key(sc):
    """Keys above 1 KiB on every rank, and one key with half the rows: its GROUP list crosses every rank boundary."""
    rng = np.random.default_rng(9)
    pool = ["w%d" % i for i in range(300)] + ["L" * 1500 + str(i) for i in range(20)] + ["", "\x00", "a\x00b"]
    keys = rows_from_pool(rng, pool, 8000)
    for i in np.flatnonzero(rng.random(8000) < 0.5):
        keys[i] = "hot"
    vals = rng.integers(0, 1 << 64, 8000, dtype=np.uint64)
    for op in ("group", "sum", "count"):
        check_case(sc, 3, op, "u64", keys, vals, 7, 5)


# ---- resubmission, empty inputs --------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ["sum", "group", "count"])
def test_resubmitted_map_drops_its_stale_keys(sc, op):
    keys, vals = data(12, 2000, op, "u64", "full", hot=0.0)

    def stale(sh, m):
        kc, vc = columns([f"stale-{m}", "the", f"stale-{m}"], np.array([1, 2, 3], dtype=np.uint64), "host")
        sh.map(m, kc, None if op == "count" else vc, 0, 3)
    W, M, R = 3, 4, 5
    got = owned(run_ranks(sc, W, op, "u64", keys, vals, M, R, resubmit=stale), op, R)
    assert not any(k.startswith("stale-") for g in got for k in g)
    single = owned(run_ranks(sc, 1, op, "u64", keys, vals, M, R, resubmit=stale), op, R)
    bits_equal(got, single, op, "u64")
    check_parts(got, ref_parts(keys, vals, op, "u64", M, R), op, "u64")


@pytest.mark.parametrize("op", ["sum", "group", "count"])
@pytest.mark.parametrize("W", [2, 8])
def test_zero_rows(sc, op, W):
    shs = run_ranks(sc, W, op, "u64", [], np.zeros(0, dtype=np.uint64), 3, 4)
    assert all(len(p) == 0 for p in owned(shs, op, 4))
    for sh in shs:
        assert sh.reduce_size(0) == (0, 0, 0)


def test_export_columns_follow_the_wire_format(sc):
    """Destination-major columns: rank d's keys are exactly those of the partitions it owns, with u32 lengths, the
    bytes concatenated, u32 value counts and each key's values in map order."""
    keys = ["a", "bb", "a", "", "ccc", "bb", "a"]
    vals = np.arange(1, 8, dtype=np.uint64)
    W, R = 2, 5
    sh = vb.StrShuffle(sc, 2, R, L.VB_U64, L.VB_AGG_GROUP, rank=0, world=W)
    kc, vc = columns(keys, vals, "host")
    sh.map(0, kc, vc, 0, 4)
    sh.map(1, kc, vc, 4, 7)
    (nk, nb, nv), (lens, kbytes, cnts, vv) = sh.export()
    lens, kbytes, cnts, vv = (t.cpu().numpy() for t in (lens, kbytes, cnts, vv))
    assert sum(nk) == 4 and sum(nb) == 6 and sum(nv) == 7
    at_k = at_b = at_v = 0
    seen = {}
    for d in range(W):
        for _ in range(nk[d]):
            ln, c = int(lens[at_k]), int(cnts[at_k])
            raw = kbytes[at_b:at_b + ln].tobytes()
            assert sc._lib.vb_get_partition_str(ctypes.create_string_buffer(raw, max(ln, 1)), ln, R) % W == d
            k = raw.decode()
            seen[k] = vv[at_v:at_v + c].tolist()
            at_k, at_b, at_v = at_k + 1, at_b + ln, at_v + c
    assert seen == {"a": [1, 3, 7], "bb": [2, 6], "": [4], "ccc": [5]}
    sh.free()


# ---- forced fingerprint collisions at import ------------------------------------------------------------------------
def _fp_cases(sc):
    for op, vdt, mode in [("group", "u64", "full"), ("sum", "i64", "full"), ("min", "f64", "special"), ("count", "u64", "default")]:
        keys, vals = data(21, 4000, op, vdt, mode)
        check_case(sc, 3, op, vdt, keys, vals, 5, 6)


def test_forced_fingerprint_collisions():
    """VEGA_B200_STR_FP_BITS=4 keeps 4 bits of the hash in the index fingerprints, so the import's dictionary sees
    equal fingerprints of distinct keys all the time.  The switch is read once per process: a subprocess."""
    code = r'''
import vega_b200 as vb
from tests.test_gpu_str_multirank import _fp_cases
with vb.Context(0) as sc:
    _fp_cases(sc)
print("fp ok")
'''
    env = dict(os.environ, VEGA_B200_STR_FP_BITS="4")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and "fp ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


# ---- cogroup and join of multi-rank GROUP sides ---------------------------------------------------------------------
@pytest.mark.parametrize("n_sides", [2, 3])
def test_cogroup_and_join_of_multi_rank_sides(sc, n_sides):
    W, M, R = 3, 4, 7
    multi, single = [], []
    for j in range(n_sides):
        keys, vals = data(30 + j, 1500, "group", "u64", "full", hot=0.0)
        multi.append(run_ranks(sc, W, "group", "u64", keys, vals, M, R))
        single.append(run_ranks(sc, 1, "group", "u64", keys, vals, M, R)[0])
    full = (1 << n_sides) - 1
    for d in range(W):
        sides = [m[d] for m in multi]
        for r in range(R):
            if r % W != d:
                continue
            gk, gl, _ = cogroup_part(sc, sides, r)
            wk, wl, _ = cogroup_part(sc, single, r)
            got = {k: [v[o[i]:o[i + 1]].tolist() for o, v in gl] for i, k in enumerate(gk)}
            want = {k: [v[o[i]:o[i + 1]].tolist() for o, v in wl] for i, k in enumerate(wk)}
            assert got == want, r
            for mask in (full, 1):
                g = join_part(sc, sides, r, mask)
                w = join_part(sc, single, r, mask)
                gd = {k: [v[g[1][i]:g[1][i + 1]].tolist() for v in g[2]] + [v[g[1][i]:g[1][i + 1]].tolist() for v in g[3]]
                      for i, k in enumerate(g[0])}
                wd = {k: [v[w[1][i]:w[1][i + 1]].tolist() for v in w[2]] + [v[w[1][i]:w[1][i + 1]].tolist() for v in w[3]]
                      for i, k in enumerate(w[0])}
                assert gd == wd and g[5] == w[5], (r, mask)


# ---- the library's exchange and error codes -------------------------------------------------------------------------
def test_error_codes(sc):
    lib = sc._lib
    inv, st, uns, big = L.VB_ERR_INVALID, L.VB_ERR_STATE, L.VB_ERR_UNSUPPORTED, L.VB_ERR_TOO_LARGE
    h = ctypes.c_void_p()
    for rank, world in [(0, 0), (2, 2), (0, 257)]:
        assert lib.vb_shuffle_create_str_dist(sc._h, 1, 2, 3, L.VB_U64, L.VB_AGG_SUM, rank, world, ctypes.byref(h)) == inv
    assert lib.vb_shuffle_create_str_dist(None, 1, 2, 3, L.VB_U64, L.VB_AGG_SUM, 0, 2, ctypes.byref(h)) == inv
    assert lib.vb_shuffle_create_str_dist(sc._h, 1, 2, 3, L.VB_U64, L.VB_AGG_SORT, 0, 2, ctypes.byref(h)) == uns
    W = 2
    u = (ctypes.c_uint64 * W)()
    z = (ctypes.c_uint64 * W)()
    one = (ctypes.c_uint64 * W)(1, 0)
    p = ctypes.c_void_p()
    # world 1: the string export / import calls are in the wrong state; integer shuffles are not string shuffles
    s1 = vb.StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM, rank=0, world=1)
    assert lib.vb_shuffle_export_str_prepare(s1._h, u, u, u) == st
    assert lib.vb_shuffle_export_str_buffers(s1._h, None, None, None, None) == st
    assert lib.vb_shuffle_import_str(s1._h, None, None, None, None, z, z, z) == st
    assert lib.vb_shuffle_exchange(s1._h, L.VB_XCHG_NCCL) == uns
    ish = vb.Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, rank=0, world=2)
    assert lib.vb_shuffle_export_str_prepare(ish._h, u, u, u) == inv
    assert lib.vb_shuffle_import_str(ish._h, None, None, None, None, z, z, z) == inv
    for agg in (L.VB_AGG_SUM, L.VB_AGG_GROUP):
        sh = vb.StrShuffle(sc, 2, 3, L.VB_U64, agg, rank=0, world=W)
        hh = sh._h
        # the integer export / import / P2P calls and set_dist keep refusing string shuffles
        assert lib.vb_shuffle_export_prepare(hh, u) == uns
        assert lib.vb_shuffle_export_counts(hh, u) == uns
        assert lib.vb_shuffle_export_buffers(hh, ctypes.byref(p), ctypes.byref(p)) == uns
        assert lib.vb_shuffle_import(hh, None, None, z) == uns
        assert lib.vb_shuffle_import_arena(hh, z) == uns
        assert lib.vb_shuffle_export_direct(hh, z, z) == uns
        assert lib.vb_shuffle_set_dist(hh, 0, 2) == uns
        assert lib.vb_shuffle_set_dist(hh, 0, 1) == uns
        assert lib.vb_shuffle_exchange(hh, L.VB_XCHG_P2P) == uns
        assert lib.vb_shuffle_exchange(hh, L.VB_XCHG_NCCL) == st         # no communicator on this context
        # import before export, NULL arguments
        assert lib.vb_shuffle_import_str(hh, None, None, None, None, z, z, z) == st
        assert lib.vb_shuffle_export_str_buffers(hh, ctypes.byref(p), None, None, None) == st
        assert lib.vb_shuffle_export_str_prepare(hh, None, u, u) == inv
        assert lib.vb_shuffle_export_str_prepare(None, u, u, u) == inv
        assert lib.vb_shuffle_seal(hh) == st
        sh2 = vb.StrShuffle(sc, 2, 3, L.VB_U64, agg, rank=0, world=W)      # the failed seal leaves sh unusable
        hh = sh2._h
        kc, vc = columns(["x", "y"], np.array([1, 2], dtype=np.uint64), "host")
        sh2.map(0, kc, vc, 0, 2)
        L.check(lib.vb_shuffle_export_str_prepare(hh, u, u, u))
        assert lib.vb_shuffle_export_str_prepare(hh, u, u, u) == st       # twice
        kcm = vb.rdd._StrCol(vb.StrKeys.from_strs(["z"]))
        assert lib.vb_shuffle_map_str(hh, 1, ctypes.c_void_p(kcm.offs_ptr), ctypes.c_void_p(kcm.data_ptr), 1,
                                      vc.at(0), 1, L.VB_HOST) == st        # map after export
        # NULL columns with non-zero counts; reduce ops with n_vals != n_keys
        buf = torch.zeros(16, dtype=torch.int64, device="cuda")
        q = ctypes.c_void_p(buf.data_ptr())
        assert lib.vb_shuffle_import_str(hh, None, q, q, q, one, one, one) == inv
        assert lib.vb_shuffle_import_str(hh, q, None, q, q, one, one, one) == inv
        assert lib.vb_shuffle_import_str(hh, q, q, q, None, one, one, one) == inv
        if agg == L.VB_AGG_GROUP:
            assert lib.vb_shuffle_import_str(hh, q, q, None, q, one, one, one) == inv
        else:
            assert lib.vb_shuffle_import_str(hh, q, q, None, q, one, one, (ctypes.c_uint64 * W)(2, 0)) == inv
        # too large, decided from the counts alone (the pointers are never read)
        if agg == L.VB_AGG_GROUP:
            assert lib.vb_shuffle_import_str(hh, q, q, q, q, one, z, (ctypes.c_uint64 * W)(0xFFFFFFFE, 0)) == big
            assert lib.vb_shuffle_import_str(hh, q, q, q, q, one, z, (ctypes.c_uint64 * W)(0xFFFFFFFD, 0)) != big
            sh2.free()
            sh2 = vb.StrShuffle(sc, 2, 3, L.VB_U64, agg, rank=0, world=W)
            hh = sh2._h
            L.check(lib.vb_shuffle_export_str_prepare(hh, u, u, u))
        else:
            n = (ctypes.c_uint64 * W)(1 << 31, 0)
            assert lib.vb_shuffle_import_str(hh, q, q, None, q, n, z, n) == big
        assert lib.vb_shuffle_import_str(hh, q, q, q, q, (ctypes.c_uint64 * W)(1 << 31, 0), z,
                                         (ctypes.c_uint64 * W)(1 << 31, 0)) == big
        # a real import; then a second import, and an import after seal, are in the wrong state
        L.check(lib.vb_shuffle_import_str(hh, None, None, None, None, z, z, z))
        assert lib.vb_shuffle_import_str(hh, None, None, None, None, z, z, z) == st
        sh2.seal()
        assert lib.vb_shuffle_import_str(hh, None, None, None, None, z, z, z) == st
        assert lib.vb_shuffle_export_str_buffers(hh, ctypes.byref(p), None, None, None) == st
        assert lib.vb_shuffle_exchange(hh, L.VB_XCHG_P2P) == uns
        sh.free()
        sh2.free()
    ish.free()
    s1.free()


def test_imported_totals_must_add_up(sc):
    """Lengths or counts that disagree with the announced totals fail the seal with VB_ERR_INVALID."""
    lib = sc._lib
    W = 2
    for agg in (L.VB_AGG_SUM, L.VB_AGG_GROUP):
        sh = vb.StrShuffle(sc, 1, 3, L.VB_U64, agg, rank=1, world=W)
        u = (ctypes.c_uint64 * W)()
        L.check(lib.vb_shuffle_export_str_prepare(sh._h, u, u, u))
        lens = torch.tensor([3, 2], dtype=torch.int32, device="cuda")
        kb = torch.zeros(4, dtype=torch.uint8, device="cuda")
        cnt = torch.tensor([1, 1], dtype=torch.int32, device="cuda")
        vals = torch.zeros(2, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ptr = lambda t: ctypes.c_void_p(t.data_ptr())
        k2 = (ctypes.c_uint64 * W)(2, 0)
        L.check(lib.vb_shuffle_import_str(sh._h, ptr(lens), ptr(kb), ptr(cnt), ptr(vals), k2, (ctypes.c_uint64 * W)(4, 0), k2))
        assert lib.vb_shuffle_seal(sh._h) == L.VB_ERR_INVALID
        sh.free()
