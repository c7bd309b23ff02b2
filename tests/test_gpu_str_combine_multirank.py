"""combine_by_key over String keys across ranks, W ranks in one process and one context (vb_shuffle_create_str_multi_dist,
the _str_cols export / import calls): the exported key lengths, key bytes and [n_acc][keys] partials of every rank are
swapped with torch.cat, source-rank major, as the all-to-all-v of vega_b200/dist.py would deliver them.  Every case
asserts that partition r has keys only on rank r % W and that the owners' partitions equal the W = 1 shuffle over the
same map tasks (f64 SUM and MEAN within the bound of any summation order); the exported columns decode, in the
documented wire format, to each rank's own partials; and each rank's refused calls return their codes."""
import ctypes
import math

import numpy as np
import pytest
import torch

import vega_b200 as vb
from tests import multirank as MR
from tests.test_gpu_combine import SPECS
from tests.test_gpu_str_combine import bits, make_rows, mean_bound_ok, multi_of, out_dtypes, sum_bound_ok
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import StrShuffle, _Col, _StrCol

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def run_world(sc, W, multi, keys, cols, M, R, where="host", hint=0):
    """One String combine on W ranks -> (the shuffles by rank, every rank's export)."""
    n = len(keys)
    if where == "host":
        kcol, vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
    else:
        h = vb.StrKeys.from_strs(keys)
        kcol = _StrCol(vb.StrKeys(torch.from_numpy(h.offsets.view(np.int64)).cuda(), torch.from_numpy(h.data.copy()).cuda()))
        vcols = tuple(_Col(torch.from_numpy(c.copy()).cuda(), role="value") for c in cols)
    maps = MR.maps_by_rank(n, M, W, lambda m, lo, hi: (lo, hi))
    shs = [StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, hint=hint, rank=r, world=W, multi=multi) for r in range(W)]
    for r in range(W):
        for m, lo, hi in maps[r]:
            shs[r].map_cols(m, kcol, vcols, lo, hi)
    if W == 1:
        shs[0].seal()
        return shs, None
    exports = [sh.export_cols() for sh in shs]
    recv = MR.swap_columns([([lens, data, accs.t()], [nk, nb, nk]) for (nk, nb), (lens, data, accs) in exports])
    for sh, (rc, rs) in zip(shs, recv):
        sh.import_cols(rc[0], rc[1], rc[2].t().contiguous(), rs[0], rs[1])
    for sh in shs:
        sh.seal()
    return shs, exports


def owned(shs, R, dts):
    W = len(shs)
    out = [None] * R
    for d, sh in enumerate(shs):
        for r in range(R):
            ko, kb, outs = sh.reduce_cols(r, dts)
            keys = vb.rdd._decode_keys(ko, kb).tolist()
            if r % W == d:
                assert len(set(keys)) == len(keys)
                out[r] = dict(zip(keys, zip(*[o.tolist() for o in outs]))) if keys else {}
            else:
                assert not keys, f"rank {d} holds keys of partition {r}, owned by rank {r % W}"
    return out


def assert_same(got, want, spec, keys, cols):
    dts, aggs = SPECS[spec]
    per_key = {}
    for c, (d, _) in enumerate(dts):
        if d == "f64":
            for k, v in zip(keys, cols[c].tolist()):
                per_key.setdefault((c, k), []).append(v)
    for r, (g, w) in enumerate(zip(got, want)):
        assert g.keys() == w.keys(), r
        for a, (op, c) in enumerate(aggs):
            if dts[c][0] == "f64" and op == "sum":
                bad = [k for k in g if not sum_bound_ok(g[k][a], per_key[(c, k)])]
            elif dts[c][0] == "f64" and op == "mean":
                bad = [k for k in g if not mean_bound_ok(g[k][a], per_key[(c, k)])]
            else:
                bad = [k for k in g if bits(g[k][a]) != bits(w[k][a])]
            assert not bad, f"partition {r}, aggregate {a} ({op} of column {c}): {bad[:3]}"


@pytest.mark.parametrize("W", [1, 2, 3, 8, 256])
@pytest.mark.parametrize("spec", sorted(SPECS))
def test_owners_equal_one_process(sc, W, spec):
    n, M, R = 30_000, 12, 17 if W < 256 else 300
    keys, cols = make_rows(W * 7 + len(spec), spec, n)
    multi = multi_of(spec)
    want_shs, _ = run_world(sc, 1, multi, keys, cols, M, R)
    want = owned(want_shs, R, out_dtypes(spec))
    for sh in want_shs:
        sh.free()
    shs, _ = run_world(sc, W, multi, keys, cols, M, R, where="device" if W in (3, 8) else "host")
    got = owned(shs, R, out_dtypes(spec))
    for sh in shs:
        sh.free()
    assert_same(got, want, spec, keys, cols)


# every accumulator exact: u64 SUM, i64 MIN, f64 MAX (NaN rules), i64 MEAN (its sum and the internal COUNT)
WIRE = ([L.VB_U64, L.VB_I64, L.VB_F64],
        [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 2), (L.VB_AGG_MEAN, 1)])


def test_exported_columns_are_the_documented_wire_format(sc):
    from tests.util import rand_pairs
    rng = np.random.default_rng(4)
    W, M, R = 3, 6, 7
    keys, _ = make_rows(9, "mixed", 9000)
    cols = [rand_pairs(rng, len(keys), 50, "u64", values="full")[1], rand_pairs(rng, len(keys), 50, "i64", values="full")[1],
            rand_pairs(rng, len(keys), 50, "f64", values="special")[1]]
    starts = vb.slice_starts(len(keys), M)
    shs = [StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, rank=r, world=W, multi=WIRE) for r in range(W)]
    locals_ = []
    for r in range(W):
        lo, hi = vdist.map_block(r, W, M)
        # the rank's own rows through a one-process shuffle with one partition: its partials
        mine = StrShuffle(sc, 1, 1, L.VB_U64, L.VB_AGG_SUM,
                          multi=(WIRE[0], WIRE[1][:3] + [(L.VB_AGG_SUM, 1), (L.VB_AGG_COUNT, 0)]))
        a, b = int(starts[lo]), int(starts[hi])
        sel = keys[a:b]
        mine.map_cols(0, _StrCol(sel), tuple(_Col(c[a:b], role="value") for c in cols), 0, len(sel))
        mine.seal()
        ko, kb, outs = mine.reduce_cols(0, [np.uint64, np.int64, np.float64, np.int64, np.uint64])
        locals_.append(dict(zip(vb.rdd._decode_keys(ko, kb).tolist(), zip(*[o.view(np.uint64).tolist() for o in outs]))))
        mine.free()
        kcol, vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
        for m in range(lo, hi):
            shs[r].map_cols(m, kcol, vcols, int(starts[m]), int(starts[m + 1]))
    for r, sh in enumerate(shs):
        (nk, nb), (lens, data, accs) = sh.export_cols()
        assert len(nk) == len(nb) == W and accs.shape == (5, sum(nk)) and lens.numel() == sum(nk) and data.numel() == sum(nb)
        lens, raw, accs = lens.cpu().numpy().astype(np.int64), bytes(data.cpu().numpy()), accs.cpu().numpy().view(np.uint64)
        pos, i, got = 0, 0, {}
        for d in range(W):
            seg = lens[i:i + nk[d]]
            assert int(seg.sum()) == nb[d]
            for ln in seg.tolist():
                k = raw[pos:pos + ln].decode("utf-8", "surrogateescape")
                b = k.encode("utf-8", "surrogateescape")
                assert L.lib().vb_get_partition_str(ctypes.c_char_p(b), len(b), R) % W == d, "a key packed for another rank"
                got[k] = tuple(accs[:, i].tolist())
                pos, i = pos + ln, i + 1
        assert got.keys() == locals_[r].keys()
        for k, v in got.items():
            w = locals_[r][k]
            f64_nan = lambda x: "nan" if math.isnan(np.uint64(x).view(np.float64)) else x
            assert (v[0], v[1], f64_nan(v[2]), v[3], v[4]) == (w[0], w[1], f64_nan(w[2]), w[3], w[4]), k
    for sh in shs:
        sh.free()


def test_each_ranks_errors(sc):
    lib = L.lib()
    W, R = 2, 4
    multi = ([L.VB_U64], [(L.VB_AGG_SUM, 0), (L.VB_AGG_MEAN, 0)])

    def fresh():
        shs = [StrShuffle(sc, 2, R, L.VB_U64, L.VB_AGG_SUM, rank=r, world=W, multi=multi) for r in range(W)]
        for r, sh in enumerate(shs):
            ks = ["a", "bb", "a", "ccc", "d", "é", "", "ff", "g", "h"]
            sh.map_cols(r, _StrCol(ks), (_Col(np.arange(len(ks), dtype=np.uint64), role="value"),), 0, len(ks))
        return shs
    u64s = lambda *x: (ctypes.c_uint64 * len(x))(*x)
    shs = fresh()
    for sh in shs:
        # import before export, seal without import
        assert lib.vb_shuffle_import_str_cols(sh._h, None, None, None, 3, u64s(0, 0), u64s(0, 0)) == L.VB_ERR_STATE
        assert lib.vb_shuffle_seal(sh._h) == L.VB_ERR_STATE
    shs = fresh()
    exports = [sh.export_cols() for sh in shs]
    for sh in shs:
        assert lib.vb_shuffle_map_str_cols(sh._h, 0, None, None, 0, None, 0, L.VB_HOST) == L.VB_ERR_STATE      # map after export
        assert lib.vb_shuffle_export_str_cols_prepare(sh._h, u64s(0, 0), u64s(0, 0)) == L.VB_ERR_STATE      # second export
    recv = MR.swap_columns([([lens, data, accs.t()], [nk, nb, nk]) for (nk, nb), (lens, data, accs) in exports])
    d0 = next(d for d in range(W) if sum(recv[d][1][0]))               # a rank that receives keys
    (rc, rs) = recv[d0]
    lens, data, accs = rc[0], rc[1], rc[2].t().contiguous()
    s0 = shs[d0]._h
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    # a spec whose accumulator count differs
    assert lib.vb_shuffle_import_str_cols(s0, p(lens), p(data), p(accs), 2, u64s(*rs[0]), u64s(*rs[1])) == L.VB_ERR_INVALID
    # a NULL column with a non-zero count
    assert lib.vb_shuffle_import_str_cols(s0, None, p(data), p(accs), 3, u64s(*rs[0]), u64s(*rs[1])) == L.VB_ERR_INVALID
    # too large, decided from the counts
    assert lib.vb_shuffle_import_str_cols(s0, p(lens), p(data), p(accs), 3, u64s(1 << 31, 0), u64s(0, 0)) == L.VB_ERR_TOO_LARGE
    # key lengths that do not add up to the announced bytes: VB_ERR_INVALID at seal
    bad_bytes = u64s(rs[1][0] + 1, rs[1][1])
    tb = torch.cat([data, torch.zeros(1, dtype=torch.uint8, device=data.device)])
    assert lib.vb_shuffle_import_str_cols(s0, p(lens), p(tb), p(accs), 3, u64s(*rs[0]), bad_bytes) == L.VB_OK
    assert lib.vb_shuffle_import_str_cols(s0, p(lens), p(tb), p(accs), 3, u64s(*rs[0]), bad_bytes) == L.VB_ERR_STATE   # twice
    assert lib.vb_shuffle_seal(s0) == L.VB_ERR_INVALID
    # the other rank imports correctly and seals; then import after seal
    (rc1, rs1) = recv[1 - d0]
    shs[1 - d0].import_cols(rc1[0], rc1[1], rc1[2].t().contiguous(), rs1[0], rs1[1])
    shs[1 - d0].seal()
    assert lib.vb_shuffle_import_str_cols(shs[1 - d0]._h, None, None, None, 3, u64s(0, 0), u64s(0, 0)) == L.VB_ERR_STATE
    for sh in shs:
        sh.free()
