"""sort_by_key through each path of seal_sort, against the exact checks of tests/sort_ref.py.

seal_sort runs one stable 8-bit LSD pass per key byte that varies (key_bits_kernel ORs and ANDs the order-transformed
keys; bytes on which every key agrees are skipped, and a sort with no varying byte still runs one pass, which copies
the rows out), then cuts the sorted keys into R partitions (sort_cuts_kernel).  The first pass reads the rows where
gather_maps leaves them: AoS rows adjacent in memory (one device (n, 2) tensor sliced into map tasks, or one host
map task copied to the device) in place, a single SoA map task in place, anything else copied to SoA (one
aos_to_soa_kernel per AoS map task, a device copy per SoA one).  Each pass runs the gather sweep
(rp_gsweep_kernel) when n >= 4 sweep tiles and both inputs are 16-byte aligned (and n < 2^31), otherwise
rp_scatter_kernel.  Each case places its input so that one path has to run and asserts the evidence:
  * rp_scatter launches (both scatter kernels count there) = key bytes that vary, or 1 when none does;
  * misc launches = key_bits_kernel + sort_cuts_kernel + one aos_to_soa_kernel per AoS map task copied to SoA;
  * no statistic separates the gather sweep from rp_scatter_kernel: the case asserts the property that selects it
    (n against 4 tiles, alignment) and names the kernel in a comment.
Values are row indices in map-id order, so every comparison also checks stability."""
import threading

import numpy as np
import pytest

import vega_b200 as vb
from tests import sort_ref as S
from tests.test_gpu_reduce_paths import _col, _dev
from vega_b200 import _lib as L
from vega_b200.rdd import Shuffle, _Col

pytestmark = pytest.mark.gpu

# gather-sweep tiles, GsPlan<u64, HAS_VAL, LDM>::T in gsweep.cuh (threads x rows per thread)
GS_T_KEY = 512 * 11             # u64 key only, SoA
GS_T_SOA = 1024 * 7             # (u64, u64) SoA: two key buffers
GS_T_AOS = 1024 * 11            # (u64, u64) AoS rows: one 16-byte row buffer
KCODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}
MID = 3_000_017                 # full tiles plus a partial one in each part; host AoS slices of 1,000,005 rows
BIG = 20_000_000                # AoS: each part holds 15 full tiles, the mbarrier phase wraps several times


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def _big_gpu():
    import torch
    return torch.cuda.get_device_properties(0).total_memory >= 60 * 2 ** 30


def passes(key_bits, kdtype):
    """Radix passes of seal_sort: key bytes that vary over the order-transformed keys, at least 1 (0 for no row)."""
    if len(key_bits) == 0:
        return 0
    ok = S.order_key(np.asarray(key_bits, np.int64), kdtype).view(np.uint64)
    varying = int(np.bitwise_or.reduce(ok)) ^ int(np.bitwise_and.reduce(ok))
    return max(1, sum(1 for b in range(8) if (varying >> (8 * b)) & 0xFF))


def sliced(kc, vc, n, M):
    s = vb.slice_starts(n, M) if n else np.array([0, 0])
    return [(m, kc, vc, int(s[m]), int(s[m + 1])) for m in range(len(s) - 1)]


def run_sort(sc, maps, M, R, kdtype, has_val, reverse=False):
    """One sort shuffle; maps = [(map id, key column or rows, value column, start, stop)].  Returns the host read of
    every partition and the statistics."""
    sh = Shuffle(sc, M, R, KCODE[kdtype], L.VB_U64, L.VB_AGG_SORT)
    sh.has_payload = has_val
    try:
        for m, kc, vc, a, b in (maps[::-1] if reverse else maps):
            sh.map(m, kc, vc, a, b)
        sh.seal()
        parts = [sh.reduce(r) for r in range(R)]
        st = sh.stats()
    finally:
        sh.free()
    return parts, st


# ---- 1. layout x key dtype x size ------------------------------------------------------------------------------------
# layout: (map tasks, has values, rows of one sweep tile of the first pass, AoS map tasks copied to SoA per map task)
LAYOUTS = {
    "host_soa": (4, True, GS_T_SOA, 0),          # copied into one owned SoA input
    "host_soa_keys": (3, False, GS_T_KEY, 0),
    "host_aos_1": (1, True, GS_T_AOS, 0),        # one owned AoS copy, read in place (LD_AOS64)
    "host_aos_3": (3, True, GS_T_SOA, 1),        # three owned AoS copies, not adjacent: aos_to_soa_kernel each
    "dev_soa": (1, True, GS_T_SOA, 0),           # one borrowed map task, read in place
    "dev_soa_misaligned": (1, True, GS_T_SOA, 0),
    "dev_soa_keys": (1, False, GS_T_KEY, 0),
    "dev_aos": (4, True, GS_T_AOS, 0),           # one (n, 2) tensor in 4 borrowed map tasks: adjacent, read in place
}


def place(layout, keys, vals):
    """(key column or rows, value column or None) of the layout; keys / vals are int64 patterns."""
    M, has_val, _, _ = LAYOUTS[layout]
    rows = np.stack([keys, vals], axis=1)
    if layout in ("host_soa", "host_soa_keys"):
        return _Col(keys), (_Col(vals, role="value") if has_val else None)
    if layout.startswith("host_aos"):
        return _Col(rows, allow_rows=True), None
    if layout == "dev_aos":
        kc = _col(_dev(rows), L.VB_U64, rows=True)
        assert kc.ptr % 16 == 0
        return kc, None
    mis = layout.endswith("misaligned")
    kc = _col(_dev(keys, misalign=mis), L.VB_U64)
    vc = _col(_dev(vals, misalign=mis), L.VB_U64) if has_val else None
    assert kc.ptr % 16 == (8 if mis else 0) and (vc is None or vc.ptr % 16 == kc.ptr % 16)
    return kc, vc


def _sizes(layout):
    T = LAYOUTS[layout][2]
    out = {"4T-1": 4 * T - 1, "4T": 4 * T, "3M": MID}
    if layout in ("host_aos_1", "dev_aos"):
        out["20M"] = BIG
    return out


MATRIX = [(lay, kd, sz) for lay in LAYOUTS for kd in ("u64", "i64", "f64") for sz in _sizes(lay)]


@pytest.mark.parametrize("layout, kdtype, size", MATRIX, ids=[f"{a}-{b}-{c}" for a, b, c in MATRIX])
def test_sort_layout_matches_oracle(sc, layout, kdtype, size):
    M, has_val, T, copies = LAYOUTS[layout]
    n = _sizes(layout)[size]
    rng = np.random.default_rng([MATRIX.index((layout, kdtype, size)), 11])
    keys = S.run_keys(rng, n, kdtype, max(len(S.EDGE[kdtype]), n // 64))
    vals = np.arange(n, dtype=np.int64)
    kc, vc = place(layout, keys, vals)
    maps = sliced(kc, vc, n, M)
    if copies:
        # the owned copies are 256-byte aligned allocations: a slice of 16 * rows bytes, not a multiple of 256, cannot
        # end where the next one starts, so gather_maps sees no adjacent run
        assert all((b - a) * 16 % 256 for _, _, _, a, b in maps[:-1])
    aligned = kc.ptr % 16 == 0
    if size == "4T-1":
        assert n < 4 * T                # every pass: rp_scatter_kernel (the first one with LD_AOS64 on AoS rows)
    elif not aligned:
        assert n >= 4 * GS_T_SOA        # pass 1 reads the caller's misaligned columns: rp_scatter_kernel; later
                                        # passes read the library's aligned buffers: rp_gsweep_kernel<u64, true, LD_SOA64>
    else:
        assert n >= 4 * T               # every pass: rp_gsweep_kernel (the first with LD_AOS64 on AoS rows, 4T: each
                                        # part is one partial tile)
    parts, st = run_sort(sc, maps, M, 8, kdtype, has_val)
    assert st["kernels"]["rp_scatter"]["launches"] == passes(keys, kdtype)
    assert st["kernels"]["misc"]["launches"] == 2 + copies * M
    S.assert_sort_equal(parts, keys, vals if has_val else None, 8, kdtype)


def test_misaligned_device_aos_rows_are_refused(sc):
    """Every AoS loader reads a row with one 16-byte load: device rows 8 bytes past a 16-byte boundary are refused
    before any kernel reads them, and the map task can then be submitted aligned."""
    import torch
    n = 50_000
    rng = np.random.default_rng(3)
    keys, vals = S.run_keys(rng, n, "u64", 500), np.arange(n, dtype=np.int64)
    rows = np.stack([keys, vals], axis=1)
    flat = torch.empty(2 * n + 1, dtype=torch.int64, device="cuda")
    flat[1:].copy_(torch.from_numpy(rows.reshape(-1)))
    bad = _col(flat[1:].view(n, 2), L.VB_U64, rows=True)
    assert bad.ptr % 16 == 8
    good = _col(_dev(rows), L.VB_U64, rows=True)
    sh = Shuffle(sc, 2, 4, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    try:
        for m, a, b in ((0, 0, n // 2), (1, n // 2, n)):
            with pytest.raises(vb.VegaB200Error) as e:
                sh.map(m, bad, None, a, b)
            assert e.value.code == L.VB_ERR_INVALID
            sh.map(m, good, None, a, b)
        sh.seal()
        parts = [sh.reduce(r) for r in range(4)]
    finally:
        sh.free()
    S.assert_sort_equal(parts, keys, vals, 4, "u64")


# ---- 2. skipped key bytes through AoS rows ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind, want_passes", [("high_byte", 1), ("below_1000", 2), ("all_equal", 1)])
def test_skipped_bytes_through_aos_rows(sc, kind, want_passes):
    """key_bits_kernel reads the keys of AoS rows (stride 2): the values (row indices) vary in bytes the keys do not.
    all_equal: the single pass reads the AoS rows and writes them out (rp_gsweep_kernel<u64, true, LD_AOS64>)."""
    n = 200_000
    rng = np.random.default_rng(len(kind))
    if kind == "high_byte":
        keys = (rng.integers(0, 256, n).astype(np.uint64) << np.uint64(56)).view(np.int64)
    elif kind == "below_1000":
        keys = rng.integers(0, 1000, n).astype(np.int64)
    else:
        keys = np.full(n, S.signed(0xFEDCBA9876543210), dtype=np.int64)
    vals = np.arange(n, dtype=np.int64)
    kc = _col(_dev(np.stack([keys, vals], axis=1)), L.VB_U64, rows=True)
    assert kc.ptr % 16 == 0 and n >= 4 * GS_T_AOS
    parts, st = run_sort(sc, sliced(kc, None, n, 4), 4, 8, "u64", True)
    assert passes(keys, "u64") == want_passes
    assert st["kernels"]["rp_scatter"]["launches"] == want_passes
    assert st["kernels"]["misc"]["launches"] == 2
    S.assert_sort_equal(parts, keys, vals, 8, "u64")


# ---- 3. the sortkv shape of tools/bench_ops.py -----------------------------------------------------------------------
def _sortkv_rows(sc, N):
    import torch
    rows = torch.empty((N, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=N, mode="uniform", n_distinct=max(1, N // 20))
    rows[:, 1] = torch.arange(N, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return rows


def _read_device(sh, R, n, has_val):
    """Every partition through reduce_device, into one key tensor and one value tensor; and the partition sizes."""
    import torch
    out_k = torch.empty(n, dtype=torch.int64, device="cuda")
    out_v = torch.empty(n, dtype=torch.int64, device="cuda") if has_val else None
    sizes, off = [], 0
    for r in range(R):
        nk, _ = sh.reduce_size(r)
        sh.reduce_device(r, out_keys=out_k[off:off + nk], out_comb=out_v[off:off + nk] if has_val else None)
        sizes.append(nk)
        off += nk
    assert off == n
    return out_k, out_v, sizes


def test_sortkv_shape_matches_oracle(sc):
    """int64 (N, 2) device rows in 8 borrowed map tasks, U64 keys, R = 8, at 2e7 rows: the host read against the
    oracle, and the device read equal to the host read."""
    N, M, R = 20_000_000, 8, 8
    rows = _sortkv_rows(sc, N)
    src = _Col(rows, allow_rows=True)
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    try:
        for m, kc, vc, a, b in sliced(src, None, N, M):
            sh.map(m, kc, vc, a, b)
        sh.seal()
        host = [sh.reduce(r) for r in range(R)]
        out_k, out_v, sizes = _read_device(sh, R, N, True)
        st = sh.stats()
    finally:
        sh.free()
    keys = rows[:, 0].cpu().numpy()
    vals = rows[:, 1].cpu().numpy()
    assert st["kernels"]["rp_scatter"]["launches"] == passes(keys, "u64")
    assert st["kernels"]["misc"]["launches"] == 2
    S.assert_sort_equal(host, keys, vals, R, "u64")
    assert sizes == [len(p[0]) for p in host]
    assert np.array_equal(out_k.cpu().numpy(), S.bits(np.concatenate([p[0] for p in host])))
    assert np.array_equal(out_v.cpu().numpy(), S.bits(np.concatenate([p[1] for p in host])))


def test_sortkv_shape_full_size_exact(sc):
    """The same at 5e8 rows (an 80 GB GPU), checked exactly on the device by check_sorted_exact."""
    import torch
    if not _big_gpu():
        pytest.skip("needs an 80 GB GPU")
    N, M, R = 500_000_000, 8, 8
    rows = _sortkv_rows(sc, N)
    src = _Col(rows, allow_rows=True)
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    try:
        for m, kc, vc, a, b in sliced(src, None, N, M):
            sh.map(m, kc, vc, a, b)
        sh.seal()
        out_k, out_v, sizes = _read_device(sh, R, N, True)
    finally:
        sh.free()
    S.check_sorted_exact(rows[:, 0], out_k, out_v, sizes, "u64")
    del rows, src, out_k, out_v
    torch.cuda.empty_cache()


# ---- 4. a key-only sort of more than 2^31 rows -----------------------------------------------------------------------
def test_keys_only_sort_above_2_31_rows(sc):
    """2^31 + 12,345 keys ((i mod D) * PHI + c) mod 2^64 in one borrowed map task (an 80 GB GPU): n >= 2^31, so every
    pass is rp_scatter_kernel<u64, false, LD_SOA64, DG_BITS> with u32 histogram offsets.  Checked exactly: keys never
    decrease, every key maps back to a rank below D, each rank has its exact row count, and the partition sizes
    follow the cut rule."""
    import torch
    if not _big_gpu():
        pytest.skip("needs an 80 GB GPU")
    n, D, c, R, chunk = (1 << 31) + 12_345, (1 << 20) + 7, 0x5DEECE66D, 8, 1 << 27
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        keys[a:b] = S.ranked_keys(torch.arange(a, b, dtype=torch.int64, device="cuda"), D, c)
    torch.cuda.synchronize()
    kc = _col(keys, L.VB_U64)
    sh = Shuffle(sc, 1, R, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    sh.has_payload = False
    try:
        sh.map(0, kc, None, 0, n)
        sh.seal()
        st = sh.stats()
        high_water = sc.mem_info()[1]
        del kc, keys                                       # the library holds its own sorted copy
        torch.cuda.empty_cache()
        sc.trim(0)
        out = torch.empty(n, dtype=torch.int64, device="cuda")
        sizes, off = [], 0
        for r in range(R):
            nk, _ = sh.reduce_size(r)
            sh.reduce_device(r, out_keys=out[off:off + nk])
            sizes.append(nk)
            off += nk
    finally:
        sh.free()
    print(f"\nkeys-only sort of {n} rows: library pool high-water {high_water / 2 ** 30:.1f} GiB")
    pool_keys = S.ranked_keys(np.arange(D, dtype=np.int64), D, c)
    assert st["kernels"]["rp_scatter"]["launches"] == passes(pool_keys, "u64")
    assert st["kernels"]["misc"]["launches"] == 2
    assert off == n
    counts = torch.zeros(D, dtype=torch.int64, device="cuda")
    for a in range(0, n, chunk):
        lo, b = max(a - 1, 0), min(n, a + chunk)
        ok = S.order_key(out[lo:b], "u64")
        assert bool((ok[1:] >= ok[:-1]).all()), f"keys decrease in rows [{lo}, {b})"
        rank = S.rank_of(out[a:b], c)
        assert bool(((rank >= 0) & (rank < D)).all()), f"a key in rows [{a}, {b}) is not one of the input's"
        counts += torch.bincount(rank, minlength=D)
        del ok, rank
    assert np.array_equal(counts.cpu().numpy(), S.rank_counts(n, D)), "rows per key differ from the input's"
    want = S.cuts_from_run_ends(S.ranked_run_ends(n, D, c), n, R)
    assert sizes == np.diff(want).tolist()
    del out
    torch.cuda.empty_cache()


# ---- 5. cut edges ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", ["1", "n-1", "n", "n+1", "65536"])
def test_cut_edges(sc, R):
    n = 300
    R = {"1": 1, "n-1": n - 1, "n": n, "n+1": n + 1, "65536": 65536}[R]
    rng = np.random.default_rng(R)
    keys, vals = S.run_keys(rng, n, "i64", 40, hot=0.3), np.arange(n, dtype=np.int64)
    kc, vc = place("dev_soa", keys, vals)
    parts, st = run_sort(sc, sliced(kc, vc, n, 1), 1, R, "i64", True)
    assert st["kernels"]["misc"]["launches"] == 2
    S.assert_sort_equal(parts, keys, vals, R, "i64")


def test_cut_positions_inside_one_long_run(sc):
    """90 % of the rows on one key, R = 16: several cut positions fall inside its run, so those partitions are empty."""
    n, R = 100_003, 16
    rng = np.random.default_rng(90)
    keys = S.run_keys(rng, n, "u64", 500, hot=0.9)
    vals = np.arange(n, dtype=np.int64)
    kc, vc = place("dev_soa", keys, vals)
    parts, _ = run_sort(sc, sliced(kc, vc, n, 1), 1, R, "u64", True)
    assert sum(len(p[0]) == 0 for p in parts) >= 10
    S.assert_sort_equal(parts, keys, vals, R, "u64")


# ---- 6. map order ------------------------------------------------------------------------------------------------------
def _order_case(seed, n=120_000):
    rng = np.random.default_rng(seed)
    return S.run_keys(rng, n, "u64", 2000, hot=0.2), np.arange(n, dtype=np.int64)


def test_map_tasks_submitted_in_reverse(sc):
    keys, vals = _order_case(61)
    kc, vc = place("host_soa", keys, vals)
    parts, _ = run_sort(sc, sliced(kc, vc, len(keys), 5), 5, 6, "u64", True, reverse=True)
    S.assert_sort_equal(parts, keys, vals, 6, "u64")


@pytest.mark.parametrize("layout", ["host_soa", "dev_aos"])
def test_map_tasks_from_eight_threads(sc, layout):
    keys, vals = _order_case(62)
    kc, vc = place(layout, keys, vals)
    maps = sliced(kc, vc, len(keys), 8)
    sh = Shuffle(sc, 8, 7, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    errors = []
    go = threading.Barrier(8)

    def submit(m, k, v, a, b):
        try:
            go.wait()
            sh.map(m, k, v, a, b)
        except Exception as e:          # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=submit, args=t) for t in maps]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        sh.seal()
        parts = [sh.reduce(r) for r in range(7)]
    finally:
        sh.free()
    S.assert_sort_equal(parts, keys, vals, 7, "u64")


def test_resubmitted_map_task_last_wins(sc):
    keys, vals = _order_case(63)
    other, _ = _order_case(64, n=50_000)
    n = len(keys)
    s = vb.slice_starts(n, 3)
    sh = Shuffle(sc, 3, 5, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    try:
        sh.map(1, _Col(other), _Col(np.arange(len(other), dtype=np.int64), role="value"), 0, len(other))
        for m in range(3):
            sh.map(m, _Col(keys), _Col(vals, role="value"), int(s[m]), int(s[m + 1]))
        sh.map(1, _Col(other), _Col(vals, role="value"), 0, 1000)        # replaced once more ...
        sh.map(1, _Col(keys), _Col(vals, role="value"), int(s[1]), int(s[2]))   # ... and the original rows win
        sh.seal()
        parts = [sh.reduce(r) for r in range(5)]
        assert sh.stats()["rows_in"] == n
    finally:
        sh.free()
    S.assert_sort_equal(parts, keys, vals, 5, "u64")


def test_mostly_empty_map_tasks(sc):
    """5 rows over 8 map tasks: five of them empty."""
    keys = np.array([S.INT64_MIN, -1, 7, S.INT64_MIN, 0], dtype=np.int64)
    vals = np.arange(5, dtype=np.int64)
    spans = [(0, 0), (0, 2), (2, 2), (2, 3), (3, 3), (3, 3), (3, 3), (3, 5)]
    maps = [(m, _Col(keys), _Col(vals, role="value"), a, b) for m, (a, b) in enumerate(spans)]
    for kdtype in ("u64", "i64"):
        parts, st = run_sort(sc, maps, 8, 3, kdtype, True)
        assert st["kernels"]["rp_scatter"]["launches"] == passes(keys, kdtype)
        S.assert_sort_equal(parts, keys, vals, 3, kdtype)


def test_aos_and_soa_map_tasks_in_one_shuffle(sc):
    """Device AoS, host SoA, host AoS and device SoA map tasks of one shuffle through vb_shuffle_map_aos / _soa: both
    AoS map tasks are copied to SoA by aos_to_soa_kernel."""
    keys, vals = _order_case(65, n=90_000)
    n = len(keys)
    rows = np.stack([keys, vals], axis=1)
    q = [0, 20_000, 45_000, 70_001, n]
    dev_rows = _col(_dev(rows), L.VB_U64, rows=True)
    dev_k, dev_v = _col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_U64)
    maps = [(0, dev_rows, None, q[0], q[1]), (1, _Col(keys), _Col(vals, role="value"), q[1], q[2]),
            (2, _Col(rows, allow_rows=True), None, q[2], q[3]), (3, dev_k, dev_v, q[3], q[4])]
    parts, st = run_sort(sc, maps, 4, 6, "u64", True)
    assert n >= 4 * GS_T_SOA            # every pass: rp_gsweep_kernel<u64, true, LD_SOA64> over the gathered columns
    assert st["kernels"]["misc"]["launches"] == 2 + 2
    assert st["kernels"]["rp_scatter"]["launches"] == passes(keys, "u64")
    S.assert_sort_equal(parts, keys, vals, 6, "u64")


# ---- 7. small inputs, outputs and errors -------------------------------------------------------------------------------
@pytest.mark.parametrize("has_val", [True, False], ids=["pairs", "keys"])
@pytest.mark.parametrize("n", [0, 1])
def test_empty_and_one_row(sc, n, has_val):
    keys = np.array([-5], dtype=np.int64)[:n]
    vals = np.arange(n, dtype=np.int64)
    for layout in ("host_soa", "dev_soa"):
        kc, vc = place(layout, keys, vals) if n else (_Col(keys), _Col(vals, role="value"))
        parts, st = run_sort(sc, [(0, kc, vc if has_val else None, 0, n)], 1, 3, "i64", has_val)
        assert st["kernels"]["rp_scatter"]["launches"] == n
        assert st["kernels"]["misc"]["launches"] == 2 * n
        S.assert_sort_equal(parts, keys, vals if has_val else None, 3, "i64")


@pytest.mark.parametrize("has_val", [True, False], ids=["pairs", "keys"])
def test_device_read_equals_host_read(sc, has_val):
    import torch
    n, R = 70_001, 5
    rng = np.random.default_rng(71)
    keys, vals = S.run_keys(rng, n, "f64", 900), np.arange(n, dtype=np.int64)
    kc, vc = place("dev_soa", keys, vals)
    sh = Shuffle(sc, 1, R, L.VB_F64, L.VB_U64, L.VB_AGG_SORT)
    sh.has_payload = has_val
    try:
        sh.map(0, kc, vc if has_val else None, 0, n)
        sh.seal()
        host = [sh.reduce(r) for r in range(R)]
        out_k, out_v, sizes = _read_device(sh, R, n, has_val)
    finally:
        sh.free()
    S.assert_sort_equal(host, keys, vals if has_val else None, R, "f64")
    assert sizes == [len(p[0]) for p in host]
    assert np.array_equal(out_k.cpu().numpy(), S.bits(np.concatenate([p[0] for p in host])))
    if has_val:
        S.check_sorted_exact(torch.from_numpy(keys).cuda(), out_k, out_v, sizes, "f64")
        assert np.array_equal(out_v.cpu().numpy(), S.bits(np.concatenate([p[1] for p in host])))


def test_values_of_a_key_only_sort_are_invalid(sc):
    import torch
    keys = np.arange(1000, dtype=np.int64)[::-1].copy()
    sh = Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SORT)
    try:
        sh.map(0, _Col(keys), None, 0, len(keys))
        sh.seal()
        with pytest.raises(vb.VegaB200Error) as e:
            sh.reduce(0)                                   # has_payload: asks for the values
        assert e.value.code == L.VB_ERR_INVALID
        k = torch.empty(sh.reduce_size(1)[0], dtype=torch.int64, device="cuda")
        with pytest.raises(vb.VegaB200Error) as e:
            sh.reduce_device(1, out_keys=k, out_comb=torch.empty_like(k))
        assert e.value.code == L.VB_ERR_INVALID
        sh.has_payload = False
        assert np.array_equal(np.concatenate([sh.reduce(r)[0] for r in range(2)]), np.arange(1000, dtype=np.uint64))
    finally:
        sh.free()


@pytest.mark.parametrize("kind", ["i32", "u32"])
def test_four_byte_keys_sort_in_their_own_order(sc, kind):
    """np.int32 keys sort signed (widened with sign extension), np.uint32 keys unsigned (zero extension)."""
    n, R = 60_000, 6
    rng = np.random.default_rng(len(kind) + 80)
    if kind == "i32":
        keys = rng.integers(-3000, 3000, n).astype(np.int32)
        edge = np.array([-1, -(1 << 31), (1 << 31) - 1, 0], dtype=np.int32)
    else:
        keys = (rng.integers(0, 3000, n) + (1 << 31) - 1500).astype(np.uint32)
        edge = np.array([(1 << 32) - 1, 1 << 31, (1 << 31) - 1, 0], dtype=np.uint32)
    keys[rng.choice(n, 400, replace=False)] = np.resize(edge, 400)
    vals = np.arange(n, dtype=np.int64)
    kdtype = "i64" if kind == "i32" else "u64"
    rdd = sc.parallelize((keys, vals), 3).sort_by_key(R)
    parts = [rdd.compute(r) for r in range(R)]
    assert rdd.stats()["kernels"]["rp_scatter"]["launches"] == passes(S.bits(keys), kdtype)
    S.assert_sort_equal(parts, S.bits(keys), vals, R, kdtype)
