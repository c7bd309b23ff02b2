"""String-key group_by_key, cogroup and joins through each path of the String GROUP seal (seal_str_runs), against the
exact references of tests/str_group_ref.py: every key's bytes, its partition, and its value list element for element.

The seal turns dictionary entry ids into partition-major dense ids of the live entries (str_mark_live_kernel,
str_part_count_kernel, str_dense_kernel: an entry only a replaced submission referenced gets none), lays the key bytes
out in dense order with u64 offsets (str_gather_bytes_kernel), copies the runs into one (u32 entry id, u64 value)
buffer and sorts it with sort_id_pairs: the entry -> dense id translation first, then ceil(ceil_log2(max(D, 2)) / 8)
8-bit LSD passes.  The keys are placed by str_part_count_kernel, not by a multisplit, and no String map or seal step
launches any other kernel of the rp_scatter class, so:
  * rp_scatter launches of a one-process String GROUP = id-sort passes of the live D;
  * every pass is the gather sweep (rp_gsweep_kernel) on n >= 4 sweep tiles (45 056 rows), the last one recording the
    CSR itself (rp_gsweep_kernel<CSR>, offs[D] = n written from the host); below that rp_scatter_kernel runs every
    pass and csr_bounds_kernel computes the CSR.  The sort always reads the library's freshly allocated buffers, so
    the alignment of the caller's columns never selects the path;
  * the dictionary index grows 4x or more when it fills and the map call reruns (table_restarts).
Imported rows (across ranks) are encoded again and expanded to one entry id per value (str_expand_ids_kernel) before
the same seal.  Values are full-range i64, compared bit for bit, or byte strings compared by their bytes; every case
with D >= 3 has the empty key and the key b"\\xff".  String GROUP beyond 2^31 rows (the rp_scatter_kernel fallback past
SW_ROW_LIMIT) needs tens of GB and is not run here; nor is the two-process NCCL exchange (tests/test_gpu_str_dist.py)."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import vega_b200 as vb
from tests import group_ref as G
from tests import str_group_ref as S
from tests.test_gpu_str_multirank import swap
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import StrKeys, StrShuffle, _BytesCol, _Col, _StrCol

pytestmark = pytest.mark.gpu

GS_TILE_SOA = 1024 * 11                # gather-sweep tile of the (u32 id, u64 value) passes, GsPlan<u32, true, LD_KEY32_VAL_SOA>
SWEEP_MIN = 4 * GS_TILE_SOA            # 45 056 rows
BIG = (1 << 24) + (1 << 21)            # rows of the 2^24-key cases
LONG = (1100,)                         # key lengths of the > 4 GiB case


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    _, high = c.mem_info()
    print(f"\nString GROUP path matrix: context pool high-water mark {high / 2 ** 30:.2f} GiB")
    c.close()


def passes(D):
    bits = (max(D, 2) - 1).bit_length()
    return max(1, (bits + 7) // 8)


def full_i64(rng, n):
    return rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)


def key_col(ranks, where, lens=S.LENS):
    """The keys of ranks as the library receives them: host arrays, or device tensors borrowed by the map call."""
    if where == "host":
        return _StrCol(StrKeys(*S.encode(ranks, lens)))
    offs, data = S.encode_torch(torch.from_numpy(np.ascontiguousarray(ranks).view(np.int64)).cuda(), lens)
    return _StrCol(StrKeys(offs, data))


def val_col(vals, where):
    return _Col(vals, role="value") if where == "host" else _Col(torch.from_numpy(vals).cuda(), role="value")


def bytes_col(vranks, where):
    offs, data = S.encode(vranks)
    if where == "host":
        return _BytesCol(StrKeys(offs, data))
    return _BytesCol(StrKeys(torch.from_numpy(offs.view(np.int64)).cuda(), torch.from_numpy(data).cuda()))


def new_shuffle(sc, M, R, agg=L.VB_AGG_GROUP, vcode=L.VB_I64, hint=0, rank=0, world=1):
    return StrShuffle(sc, M, R, vcode, agg, hint=hint, rank=rank, world=world)


def map_slices(sh, kc, vc, n, M):
    s = vb.slice_starts(n, M)
    for m in range(len(s) - 1):
        sh.map(m, kc, vc, int(s[m]), int(s[m + 1]))


def gather_bytes(sh, refs):
    """Byte-string values of a shuffle's output references: (offsets, bytes)."""
    refs = np.ascontiguousarray(refs, dtype=np.uint64)
    n, nb = len(refs), ctypes.c_uint64()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    L.check(sh._lib.vb_shuffle_gather_bytes_size(sh._h, p(refs), n, L.VB_HOST, ctypes.byref(nb)))
    offs, data = np.empty(n + 1, np.uint64), np.empty(nb.value, np.uint8)
    L.check(sh._lib.vb_shuffle_gather_bytes(sh._h, p(refs), n, L.VB_HOST, p(offs), p(data), L.VB_HOST))
    return offs, data


def group_parts(sh, R, parts=None):
    """Every partition on the host: (key offsets, key bytes, value offsets, values or (value offsets, value bytes))."""
    out = []
    for r in range(R) if parts is None else parts:
        ko, kb, o, v = sh.reduce_raw(r) if sh.vcode != L.VB_BYTES else _refs_raw(sh, r)
        out.append((ko, kb, o, gather_bytes(sh, v) if sh.vcode == L.VB_BYTES else v))
    return out


def _refs_raw(sh, r):
    nk, nb, nv = sh.reduce_size(r)
    ko, kb, o, v = np.empty(nk + 1, np.uint64), np.empty(nb, np.uint8), np.empty(nk + 1, np.uint64), np.empty(nv, np.uint64)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    L.check(sh._lib.vb_shuffle_reduce_str(sh._h, r, p(ko), p(kb), None, p(o), p(v), L.VB_HOST))
    return ko, kb, o, v


def run_group(sc, kc, vc, n, M, R, hint=0, vcode=L.VB_I64):
    sh = new_shuffle(sc, M, R, vcode=vcode, hint=hint)
    try:
        map_slices(sh, kc, vc, n, M)
        sh.seal()
        return group_parts(sh, R), sh.stats()
    finally:
        sh.free()


def n_keys(parts):
    return sum(len(p[0]) - 1 for p in parts)


# ---- reduce side: SUM and COUNT over the same inputs -----------------------------------------------------------------
def assert_sum_count(sc, kc, vals, ranks, M, R, lens=S.LENS, device_keys=False):
    """String SUM (wrapping i64) and COUNT over the rows against exact numpy sums per key."""
    order = np.argsort(ranks, kind="stable")
    uk, starts, cnt = G.runs(ranks[order])
    want_sum = np.add.reduceat(vals.view(np.uint64)[order], starts) if len(starts) else np.zeros(0, np.uint64)
    vc = val_col(vals, "host" if kc.loc == L.VB_HOST else "dev")
    for agg, want in ((L.VB_AGG_SUM, want_sum), (L.VB_AGG_COUNT, cnt.astype(np.uint64))):
        sh = new_shuffle(sc, M, R, agg=agg)
        try:
            map_slices(sh, kc, vc if agg == L.VB_AGG_SUM else None, len(ranks), M)
            sh.seal()
            if device_keys:
                got_k, got_c = device_uniform_read(sh, 0, lens[0], agg)
            else:
                parts = [sh.reduce_raw(r) for r in range(R)]
                got_k, _ = S.str_keys_of(parts, R, lens)
                got_c = np.concatenate([G.u64(p[2]) for p in parts])
        finally:
            sh.free()
        o = np.argsort(got_k)
        assert np.array_equal(got_k[o], uk), f"agg {agg}: {len(got_k)} keys, want {len(uk)}"
        G.assert_rows_equal((got_k[o], got_c[o]), (uk, want), ("key", "value"))


def device_uniform_read(sh, r, u, agg):
    """Partition r through device outputs, keys all u bytes long: (ranks of the keys, combined values or (offsets,
    values)), checking every key byte on the device."""
    nk, nb, nv = sh.reduce_size(r)
    dev = "cuda"
    ko = torch.empty(nk + 1, dtype=torch.int64, device=dev)
    kb = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
    if agg == L.VB_AGG_GROUP:
        o = torch.empty(nk + 1, dtype=torch.int64, device=dev)
        v = torch.empty(max(nv, 1), dtype=torch.int64, device=dev)
        sh.reduce_device(r, out_key_offsets=ko, out_key_bytes=kb, out_offs=o, out_vals=v)
    else:
        comb = torch.empty(max(nk, 1), dtype=torch.int64, device=dev)
        sh.reduce_device(r, out_key_offsets=ko, out_key_bytes=kb, out_comb=comb)
    torch.cuda.synchronize()
    assert nb == nk * u and torch.equal(ko, torch.arange(nk + 1, device=dev) * u), "key offsets of fixed-length keys"
    m = kb[:nb].view(nk, u)
    pad = torch.from_numpy(S.pad(u)[8:]).to(dev)
    step = 1 << 18
    for a in range(0, nk, step):
        assert bool((m[a:a + step, 8:] == pad).all()), f"a pad byte of keys {a} .. {a + step} differs"
    ranks = m[:, :8].contiguous().view(torch.int64).flatten().cpu().numpy().view(np.uint64)
    assert np.array_equal(S.key_lens(ranks, (u,)), np.full(nk, u)), "a key that is not the encoding of its rank"
    if agg == L.VB_AGG_GROUP:
        return ranks, (o.cpu().numpy().view(np.uint64), v[:nv].cpu().numpy())
    return ranks, comb[:nk].cpu().numpy().view(np.uint64)


# ---- group_by_key: the path matrix -----------------------------------------------------------------------------------
# name: (D, rows, keys on the host or borrowed from the device, map tasks, R, hot-key share)
GROUP_CASES = {
    "one_key": (1, 3_000_000, "dev", 4, 7, 0.0),               # 1-pass sweep, one value run across every part and tile
    "d256_sweep": (256, 2_000_000, "dev", 3, 7, 0.0),          # 1 pass: rp_gsweep_kernel<CSR>
    "d256_small": (256, 40_000, "dev", 2, 7, 0.0),             # 1 pass: rp_scatter_kernel + csr_bounds_kernel
    "d257": (257, 2_000_000, "host", 3, 257, 0.0),             # first 2-pass D
    "d300_small": (300, 30_000, "host", 2, 7, 0.0),            # 2 passes on the scatter route
    "d65536": (1 << 16, 3_000_000, "dev", 2, 7, 0.0),          # last 2-pass D
    "d65537": ((1 << 16) + 1, 3_000_000, "dev", 2, 7, 0.0),    # first 3-pass D
    "d2^24": (1 << 24, BIG, "dev", 4, 7, 0.0),                 # last 3-pass D
    "d2^24+1": ((1 << 24) + 1, BIG, "dev", 4, 65536, 0.0),     # 4 passes, the largest R
    "hot": (100_000, 8_000_000, "dev", 2, 7, 0.6),             # one run across many tiles
}


@pytest.mark.parametrize("case", list(GROUP_CASES))
def test_group_path_matches_exact_reference(sc, case):
    D, n, where, M, R, hot = GROUP_CASES[case]
    rng = np.random.default_rng([list(GROUP_CASES).index(case), 11])
    ranks, vals = S.rank_rows(rng, n, D, hot=hot), full_i64(rng, n)
    if case.endswith("_small"):
        assert n < SWEEP_MIN                    # rp_scatter_kernel on every pass, csr_bounds_kernel
    else:
        assert n >= SWEEP_MIN                   # rp_gsweep_kernel on every pass, the last one rp_gsweep_kernel<CSR>
    kc = key_col(ranks, where)
    parts, st = run_group(sc, kc, val_col(vals, where), n, M, R)
    assert st["kernels"]["rp_scatter"]["launches"] == passes(D)
    assert n_keys(parts) == D > 0
    if hot:
        assert max(int(np.diff(p[2].astype(np.int64)).max(initial=0)) for p in parts) > 0.55 * n
    S.assert_str_group_equal(parts, ranks, vals, R)
    if case == "d2^24+1":                       # the fold over 2^24 + 1 dense ids on the reduce side
        assert_sum_count(sc, kc, vals, ranks, M, R)


def test_index_regrowth_in_first_and_later_calls(sc):
    """hint = 1: the index starts at 16 slots.  Map m brings the ranks [m D / 4, (m + 1) D / 4) for the first time,
    so the index grows in the first call and again in a later one, each time rerunning the call over every row."""
    rng = np.random.default_rng(40)
    D, n, M, R = 1 << 17, 2_000_000, 4, 7
    pool = S.distinct_ranks(D)
    q = D // M
    ranks = np.concatenate([rng.permutation(np.concatenate([pool[m * q:(m + 1) * q], pool[rng.integers(0, (m + 1) * q, n // M - q)]]))
                            for m in range(M)])
    vals = full_i64(rng, n)
    kc, vc = key_col(ranks, "host"), val_col(vals, "host")
    sh = new_shuffle(sc, M, R, hint=1)
    try:
        restarts = []
        for m in range(M):
            sh.map(m, kc, vc, m * (n // M), (m + 1) * (n // M))
            restarts.append(sh.stats()["table_restarts"])
        sh.seal()
        parts, st = group_parts(sh, R), sh.stats()
    finally:
        sh.free()
    assert restarts[0] >= 1 and restarts[-1] > restarts[0], restarts
    assert st["kernels"]["rp_scatter"]["launches"] == passes(D)
    assert n_keys(parts) == D
    S.assert_str_group_equal(parts, ranks, vals, R)


def test_resubmission_after_regrowth_leaves_dead_entries(sc):
    """Map 0 brings 75 000 keys (the index regrows), then is resubmitted with 60 000 rows over 200 other keys: the
    dictionary keeps 75 200 entries, of which 200 are live.  The dense ids, and the passes, follow the live D: one
    pass (3 if they followed the entries)."""
    rng = np.random.default_rng(41)
    R = 7
    stale = S.distinct_ranks(75_000, first=100_000)
    live = S.distinct_ranks(200)
    ranks = S.rows_over(rng, live, 60_000)
    vals = full_i64(rng, len(ranks))
    sh = new_shuffle(sc, 1, R, hint=1)
    try:
        sh.map(0, key_col(stale, "dev"), val_col(full_i64(rng, len(stale)), "dev"), 0, len(stale))
        assert sh.stats()["table_restarts"] >= 1
        sh.map(0, key_col(ranks, "dev"), val_col(vals, "dev"), 0, len(ranks))
        sh.seal()
        parts, st = group_parts(sh, R), sh.stats()
    finally:
        sh.free()
    assert len(ranks) >= SWEEP_MIN and passes(len(stale) + len(live)) == 3
    assert st["kernels"]["rp_scatter"]["launches"] == passes(len(live)) == 1
    assert n_keys(parts) == len(live)
    S.assert_str_group_equal(parts, ranks, vals, R)


def test_eight_threads_regrow_the_index(sc):
    """8 threads map 250 000 rows each over 2^17 keys into one shuffle with hint = 1."""
    rng = np.random.default_rng(42)
    D, M, per, R = 1 << 17, 8, 250_000, 17
    ranks, vals = S.rank_rows(rng, M * per, D), full_i64(rng, M * per)
    cols = [(key_col(ranks[m * per:(m + 1) * per], "dev"), val_col(vals[m * per:(m + 1) * per], "dev")) for m in range(M)]
    sh = new_shuffle(sc, M, R, hint=1)
    try:
        errs = []

        def work(m):
            try:
                sh.map(m, cols[m][0], cols[m][1], 0, per)
            except Exception as e:          # pragma: no cover - reported below
                errs.append(e)
        ts = [threading.Thread(target=work, args=(m,)) for m in range(M)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert not errs, errs
        sh.seal()
        parts, st = group_parts(sh, R), sh.stats()
    finally:
        sh.free()
    assert st["table_restarts"] >= 2
    assert st["kernels"]["rp_scatter"]["launches"] == passes(D)
    assert n_keys(parts) == D
    S.assert_str_group_equal(parts, ranks, vals, R)


def test_key_bytes_beyond_4_gib(sc):
    """4 * 10^6 keys of 1100 bytes (4.4 * 10^9 key bytes in one partition) over 4.5 * 10^6 rows: every key byte offset
    of the seal (arena, dense layout, gather destination, output copy) passes 2^32.  Read back through host and device
    outputs; SUM and COUNT over the same rows."""
    rng = np.random.default_rng(43)
    D, n, R = 4_000_000, 4_500_000, 1
    ranks = S.rows_over(rng, np.arange(D, dtype=np.uint64) * np.uint64(1_000_003) + np.uint64(7), n)
    vals = full_i64(rng, n)
    kc, vc = key_col(ranks, "dev", LONG), val_col(vals, "dev")
    sh = new_shuffle(sc, 1, R)
    try:
        map_slices(sh, kc, vc, n, 1)
        sh.seal()
        nk, nb, nv = sh.reduce_size(0)
        assert nk == D and nb == D * LONG[0] > (1 << 32) and nv == n
        assert sh.stats()["kernels"]["rp_scatter"]["launches"] == passes(D)
        parts = group_parts(sh, R)
        keys = S.str_keys_of(parts, R, LONG)
        G.assert_rows_equal(S.str_csr_triples(parts, R, LONG, keys=keys), G.group_triples(ranks, vals), G.GROUP_COLS)
        dk, (do, dv) = device_uniform_read(sh, 0, LONG[0], L.VB_AGG_GROUP)
        assert np.array_equal(dk, keys[0]) and np.array_equal(do, parts[0][2]) and np.array_equal(dv, parts[0][3])
    finally:
        sh.free()
    del parts
    assert_sum_count(sc, kc, vals, ranks, 1, R, lens=LONG, device_keys=True)


@pytest.mark.parametrize("D", [256, (1 << 16) + 1])
def test_byte_string_values(sc, D):
    """vb_shuffle_map_str_bytes: the values' bytes in list order (values of 0 to 100 bytes, NULs and 0xFF)."""
    rng = np.random.default_rng([44, D])
    n, M, R = 2_000_000, 3, 7
    ranks = S.rank_rows(rng, n, D)
    vr = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    where = "dev" if D == 256 else "host"
    parts, st = run_group(sc, key_col(ranks, where), bytes_col(vr, where), n, M, R, vcode=L.VB_BYTES)
    assert st["kernels"]["rp_scatter"]["launches"] == passes(D)
    assert n_keys(parts) == D
    S.assert_str_group_equal(parts, ranks, vr, R)


# ---- across ranks, in one process ------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,n", [(256, 1_000_000), ((1 << 16) + 1, 1_500_000)])
def test_multi_rank_import(sc, D, n):
    """W = 3 ranks, each key on every rank; the exported columns swapped with torch.cat.  Each rank's import is sealed
    over about n / 3 rows (>= 4 sweep tiles): its keys encoded again, each received value given its key's entry id
    by str_expand_ids_kernel, then the seal above.  Owned partitions equal the one-process shuffle and the
    reference; the others are empty."""
    rng = np.random.default_rng([45, D])
    W, M, R = 3, 6, 7
    ranks, vals = S.rank_rows(rng, n, D), full_i64(rng, n)
    assert n // W >= SWEEP_MIN
    kc, vc = key_col(ranks, "dev"), val_col(vals, "dev")
    starts = vb.slice_starts(n, M)
    shs = [new_shuffle(sc, M, R, rank=r, world=W) for r in range(W)]
    one = new_shuffle(sc, M, R)
    try:
        for r, sh in enumerate(shs):
            lo, hi = vdist.map_block(r, W, M)
            for m in range(lo, hi):
                sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
        exports = [sh.export() for sh in shs]
        for sh, (cols, counts) in zip(shs, swap(exports)):
            sh.import_(*cols, *counts)
        for sh in shs:
            sh.seal()
        map_slices(one, kc, vc, n, M)
        one.seal()
        owned = []
        for r in range(R):
            for d, sh in enumerate(shs):
                if d != r % W:
                    assert sh.reduce_size(r) == (0, 0, 0), f"rank {d} holds keys of partition {r}"
            owned += group_parts(shs[r % W], R, [r])
        single = group_parts(one, R)
    finally:
        for sh in shs + [one]:
            sh.free()
    assert n_keys(owned) == D
    G.assert_rows_equal(S.str_csr_triples(owned, R), S.str_csr_triples(single, R), G.GROUP_COLS)
    S.assert_str_group_equal(owned, ranks, vals, R)


# ---- cogroup and joins of two 4-pass sides ---------------------------------------------------------------------------
def _arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value for s in shs])


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def cogroup_raw(sc, shs, r):
    n, lib = len(shs), sc._lib
    nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * n)()
    L.check(lib.vb_cogroup_n_str_size(_arr(shs), n, r, ctypes.byref(nk), ctypes.byref(nb), nv))
    ko, kb = np.empty(nk.value + 1, np.uint64), np.empty(nb.value, np.uint8)
    sides = [(np.empty(nk.value + 1, np.uint64), np.empty(nv[j], np.uint64)) for j in range(n)]
    L.check(lib.vb_cogroup_n_str(_arr(shs), n, r, _p(ko), _p(kb), (ctypes.c_void_p * n)(*[_p(o) for o, _ in sides]),
                                 (ctypes.c_void_p * n)(*[_p(v) for _, v in sides]), L.VB_HOST))
    return ko, kb, sides


def join_raw(sc, shs, r, required):
    n, lib = len(shs), sc._lib
    nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    L.check(lib.vb_join_n_str_size(_arr(shs), n, r, required, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
    ko, kb, ro = np.empty(nk.value + 1, np.uint64), np.empty(nb.value, np.uint8), np.empty(nk.value + 1, np.uint64)
    vs = [np.empty(nr.value, np.uint64) for _ in shs]
    ok = [np.empty(nr.value, np.uint8) for _ in shs]
    L.check(lib.vb_join_n_str(_arr(shs), n, r, required, _p(ko), _p(kb), _p(ro), (ctypes.c_void_p * n)(*[_p(v) for v in vs]),
                              (ctypes.c_void_p * n)(*[_p(o) for o in ok]), L.VB_HOST))
    return ko, kb, ro, vs, ok


def test_cogroup_and_joins_four_passes_per_side(sc):
    """Two sides of 2^24 + 1 keys each, 2 % of the keys on both: each side is grouped whole at its seal in 4 passes.
    vb_cogroup_n_str, and vb_join_n_str with required = 0b11 (inner) and 0b00 (full outer)."""
    rng = np.random.default_rng(46)
    D, R = (1 << 24) + 1, 7
    pa = S.distinct_ranks(D)
    shared = rng.choice(pa, D // 50, replace=False)
    pb = np.concatenate([shared, np.arange(D, 2 * D - len(shared), dtype=np.uint64)])
    ra, rb = S.rows_over(rng, pa, D + (1 << 20)), S.rows_over(rng, pb, D + (1 << 19))
    va, vb_ = full_i64(rng, len(ra)), full_i64(rng, len(rb))
    shs = []
    try:
        for r_, v_, M in ((ra, va, 3), (rb, vb_, 2)):
            sh = new_shuffle(sc, M, R)
            shs.append(sh)
            map_slices(sh, key_col(r_, "dev"), val_col(v_, "dev"), len(r_), M)
            sh.seal()
            assert sh.stats()["kernels"]["rp_scatter"]["launches"] == passes(D) == 4
        placed = S.assert_str_cogroup_equal([cogroup_raw(sc, shs, r) for r in range(R)], [(ra, va), (rb, vb_)], R)
        for required, kind in ((0b11, "inner"), (0b00, "full")):
            parts = [join_raw(sc, shs, r, required) for r in range(R)]
            want = G.join_rows(kind, ra, va, rb, vb_)
            assert len(want[0]) >= (len(shared) if kind == "inner" else len(ra) + len(rb) - len(shared))
            G.assert_rows_equal(S.str_join_rows(parts, R, placed=placed), want, G.JOIN_COLS)   # keys hashed by the cogroup check
            del parts, want
    finally:
        for sh in shs:
            sh.free()
