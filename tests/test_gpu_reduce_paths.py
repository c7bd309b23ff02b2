"""reduce_by_key through every hash-aggregate path, over the full value range of every dtype, against exact references.

Each path asserts the statistic that proves it ran, so a change in kernel selection fails here instead of silently
testing another path.  Integer ops, COUNT and f64 MIN/MAX are compared bit for bit with the CPU oracle (NaN results
as one bit pattern); f64 SUM is checked per key by tests/util.py:assert_f64_sums against the exact reference of
tests/f64_sum_ref.py, bit-exact on values whose partial sums are all representable and within the order-independent
error bound otherwise."""
import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests.util import (assert_f64_sums, assert_parts_equal, bits_dict, f64_total_key, gpu_group_parts, oracle_group,
                        oracle_reduce_bits, rand_pairs)
from vega_b200 import _lib as L
from vega_b200.rdd import PairRdd, Rdd, Shuffle, _Col

pytestmark = pytest.mark.gpu

AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT}
CODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64, None: L.VB_U64}
# (op, value dtype, rand_pairs value mode); COUNT runs on keys alone (AoS rows carry values anyway)
OPS = [("sum", "u64", "full"), ("sum", "i64", "full"), ("sum", "f64", "exact"), ("sum", "f64", "subnormal"),
       ("sum", "f64", "cancel"), ("min", "u64", "full"), ("max", "u64", "full"), ("min", "i64", "full"),
       ("max", "i64", "full"), ("min", "f64", "special"), ("max", "f64", "special"), ("count", None, "full")]
OP_IDS = [f"{op}-{vdt or 'keys'}-{mode}" for op, vdt, mode in OPS]


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def _dev(a, misalign=False):
    """A torch CUDA tensor with the bits of a (1-D, or (n, 2) rows); misalign=True: its data starts 8 bytes past a
    16-byte boundary."""
    import torch
    h = torch.from_numpy(np.ascontiguousarray(a).view(np.int64))
    if not misalign:
        return h.cuda()
    t = torch.empty(h.numel() + 1, dtype=torch.int64, device="cuda")
    t[1:].copy_(h)
    return t[1:]


def _col(x, code, rows=False):
    c = _Col(x, allow_rows=rows, role="key")
    c.code = code                     # a torch int64 column carrying u64 or f64 bits
    return c


def run_reduce(sc, op, vdt, kcol, vcol, n, M, R, key_width=8, hint=0):
    """One shuffle: M map tasks over rows [0, n) as ParallelCollection slices them, seal, every reduce partition."""
    starts = vb.slice_starts(n, M)
    sh = Shuffle(sc, len(starts) - 1, R, L.VB_U64, CODE[vdt], AGG[op], key_width=key_width, hint=hint)
    try:
        for m in range(len(starts) - 1):
            sh.map(m, kcol, vcol, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        parts = [sh.reduce(r) for r in range(R)]
        st = sh.stats()
    finally:
        sh.free()
    return parts, st


def check_reduce(parts, op, vdt, mode, keys, vals, R, key_width=8):
    """Every key of every partition against the exact reference of the op."""
    if op == "sum" and vdt == "f64":
        got = [dict(zip(k.view(np.uint64).tolist(), c.tolist())) for k, c in parts]
        assert_f64_sums(got, keys, vals, R, key_width=key_width, exact=mode in ("exact", "subnormal"))
        return
    got = [bits_dict(k, c) for k, c in parts]
    want = oracle_reduce_bits(op, keys, None if op == "count" else vals, 4, R, vdt or "u64", key_width, threads=4)
    assert_parts_equal(got, want)


# ---- the path matrix -----------------------------------------------------------------------------------------------
# name: (rows, keys, hot-key share, R); _run_path places the input and asserts the statistic that proves the path ran
PATHS = {
    "register_small": (150_000, 20_000, 0.0, 7),          # host input, 3 map tasks of 50k rows: below the bulk kernel's 65,536
    "register_large": (2_000_001, 100_000, 0.0, 7),       # one device column sliced t[1:]: 8-byte misaligned
    "bulk_soa_tail": (1_000_003, 50_000, 0.0, 7),         # device columns, 1 map task, n % 1024 = 579 tail rows
    "bulk_aos": (1_000_003, 50_000, 0.0, 5),              # device (n, 2) rows, 2 map tasks
    "hot_key_cache": (8_000_000, 200_000, 0.12, 7),       # one map task, top key 12 % of rows: ~30 tiles per CTA
    "register_hot": (8_000_000, 200_000, 0.12, 7),        # the hot_key_cache rows as misaligned device columns: the
                                                          # register-staged kernel keeps its cache past the learning tiles
    "per_map_merge": (400_000, 100_000, 0.0, 7),          # host input, 4 map tasks: per-map tables merged at seal
    "shared_borrowed": (400_000, 100_000, 0.0, 7),        # device input, 4 map tasks at even starts: one shared table
    "restart_per_map": (300_000, 120_000, 0.0, 7),        # host input, hint=100: per-map tables overflow
    "restart_shared": (300_000, 120_000, 0.0, 7),         # device input, hint=100: the shared table overflows
    "partition_first": ((1 << 22) + 5, 300_000, 0.0, 7),  # device input, 1 map task, hint=3e6: 2^23-slot table
}


def _run_path(sc, path, op, vdt, keys, vals, n, R):
    """Place the input as the path needs it, run it, and assert the path's statistic."""
    has_v = op != "count"
    vcode = CODE[vdt]
    if path == "register_small":
        kc, vc = _Col(keys), (_Col(vals, role="value") if has_v else None)
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 3, R)
        assert st["hot_kernel_variant"] == 0
    elif path in ("register_large", "register_hot"):
        kc = _col(_dev(keys, misalign=True), L.VB_U64)
        vc = _col(_dev(vals, misalign=True), vcode) if has_v else None
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 1, R)
        assert st["hot_kernel_variant"] == 0
    elif path in ("bulk_soa_tail", "hot_key_cache"):
        kc = _col(_dev(keys), L.VB_U64)
        vc = _col(_dev(vals), vcode) if has_v else None
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 1, R)
        assert st["hot_kernel_variant"] == 1
    elif path == "bulk_aos":
        rows = _col(_dev(np.stack([keys, np.ascontiguousarray(vals).view(np.uint64)], axis=1)), vcode, rows=True)
        parts, st = run_reduce(sc, op, vdt, rows, None, n, 2, R)
        assert st["hot_kernel_variant"] == 1
    elif path == "per_map_merge":
        kc, vc = _Col(keys), (_Col(vals, role="value") if has_v else None)
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 4, R)
        assert st["kernels"]["merge"]["launches"] >= 1
    elif path == "shared_borrowed":
        kc = _col(_dev(keys), L.VB_U64)
        vc = _col(_dev(vals), vcode) if has_v else None
        assert all(s % 2 == 0 for s in vb.slice_starts(n, 4))
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 4, R)
        assert st["hot_kernel_variant"] == 1 and st["kernels"]["merge"]["launches"] == 0
    elif path == "restart_per_map":
        kc, vc = _Col(keys), (_Col(vals, role="value") if has_v else None)
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 2, R, hint=100)
        assert st["table_restarts"] >= 1
    elif path == "restart_shared":
        kc = _col(_dev(keys), L.VB_U64)
        vc = _col(_dev(vals), vcode) if has_v else None
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 4, R, hint=100)
        assert st["table_restarts"] >= 1
    elif path == "partition_first":
        kc = _col(_dev(keys), L.VB_U64)
        vc = _col(_dev(vals), vcode) if has_v else None
        parts, st = run_reduce(sc, op, vdt, kc, vc, n, 1, R, hint=3_000_000)
        assert st["table_slots"] >= 1 << 23
    else:
        raise ValueError(path)
    return parts, st


def _path_data(path, i_op):
    data = "hot_key_cache" if path == "register_hot" else path     # register_hot: the same rows, placed differently
    n, nkeys, hot, R = PATHS[data]
    op, vdt, mode = OPS[i_op]
    rng = np.random.default_rng([sorted(set(PATHS) - {"register_hot"}).index(data), i_op, 1])
    keys, vals = rand_pairs(rng, n, nkeys, vdt or "u64", values=mode, hot=hot)
    return n, R, keys, vals


@pytest.mark.parametrize("i_op", range(len(OPS)), ids=OP_IDS)
@pytest.mark.parametrize("path", list(PATHS))
def test_reduce_path_matches_exact_reference(sc, path, i_op):
    op, vdt, mode = OPS[i_op]
    n, R, keys, vals = _path_data(path, i_op)
    if path in ("hot_key_cache", "register_hot"):
        top = np.unique(keys, return_counts=True)[1].max()
        assert top > 0.05 * n
    parts, _ = _run_path(sc, path, op, vdt, keys, vals, n, R)
    check_reduce(parts, op, vdt, mode, keys, vals, R)


# ---- partition counts: both seal paths (unordered table split for R <= 256, ordered two-pass multisplit above) -----
@pytest.mark.parametrize("R", [1, 255, 256, 257, 1000, 65536])
def test_reduce_partition_counts(sc, R):
    rng = np.random.default_rng(R)
    for op, vdt in (("sum", "u64"), ("max", "i64")):
        keys, vals = rand_pairs(rng, 200_000, 60_000, vdt, values="full")
        parts, _ = run_reduce(sc, op, vdt, _Col(keys), _Col(vals, role="value"), len(keys), 3, R)
        check_reduce(parts, op, vdt, "full", keys, vals, R)


@pytest.mark.parametrize("R", [256, 257, 65536])
def test_group_by_key_partition_counts(sc, R):
    rng = np.random.default_rng(R + 1)
    keys, vals = rand_pairs(rng, 100_000, 30_000)
    assert gpu_group_parts(sc.parallelize((keys, vals), 3).group_by_key(R)) == oracle_group(keys, vals, 3, R)


def test_more_than_65536_partitions_is_unsupported(sc):
    with pytest.raises(vb.VegaB200Error) as e:
        Shuffle(sc, 1, 65537, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)
    assert e.value.code == -5
    keys = np.arange(10, dtype=np.uint64)
    with pytest.raises(vb.VegaB200Error) as e:
        sc.parallelize((keys, keys), 2).reduce_by_key("sum", 65537).collect()
    assert e.value.code == -5


# ---- 4-byte keys: widened to 64 bits (i32 -1 becomes the table's empty marker), hashed as 4 bytes ---------------------
@pytest.mark.parametrize("R", [7, 300])
@pytest.mark.parametrize("kind", ["i32", "u32"])
def test_four_byte_keys(sc, kind, R):
    rng = np.random.default_rng([R, len(kind)])
    n = 120_000
    if kind == "i32":
        keys = rng.integers(-3000, 3000, n).astype(np.int32)
        edge = np.array([-1, -(1 << 31), (1 << 31) - 1, 0], dtype=np.int32)
    else:
        keys = (rng.integers(0, 3000, n) + (1 << 31) - 1500).astype(np.uint32)     # straddles 2^31
        edge = np.array([(1 << 32) - 1, 1 << 31, (1 << 31) - 1, 0], dtype=np.uint32)
    keys[rng.choice(n, 400, replace=False)] = np.resize(edge, 400)
    wide = keys.astype(np.int64 if kind == "i32" else np.uint64).view(np.uint64)
    for op in ("sum", "min", "max"):
        _, vals = rand_pairs(rng, n, 1, "i64", values="full")
        kc = _Col(keys)
        assert kc.key_width == 4
        parts, _ = run_reduce(sc, op, "i64", kc, _Col(vals, role="value"), n, 3, R, key_width=4)
        check_reduce(parts, op, "i64", "full", wide, vals, R, key_width=4)


# ---- f64 sort keys: f64::total_cmp order, stable, cuts between bit-unequal keys --------------------------------------
@pytest.mark.parametrize("payload", [True, False])
@pytest.mark.parametrize("aligned", [True, False], ids=["gather_sweep", "radix_pass_misaligned"])
def test_f64_sort_keys_follow_total_order(sc, aligned, payload):
    rng = np.random.default_rng([int(aligned), int(payload)])
    n, R = 300_001, 8
    _, keys = rand_pairs(rng, n, 5000, "f64", values="special")
    keys[::7] = keys[3]                                       # a long run of one key
    vals = np.arange(n, dtype=np.uint64)
    M = 3 if aligned else 1                                   # slices of a misaligned column stay misaligned only at start 0
    kc = _col(_dev(keys, misalign=not aligned), L.VB_F64)
    if payload:
        rdd = PairRdd(sc, kc, _col(_dev(vals, misalign=not aligned), L.VB_U64), M).sort_by_key(R)
    else:
        rdd = Rdd(sc, kc, M).sort(R)
    gk, gv = rdd.collect()
    order = np.argsort(f64_total_key(keys), kind="stable")
    ok, ov, ps = O.sort_by_key(keys, vals if payload else None, R, "f64")
    assert np.array_equal(ok.view(np.uint64), keys.view(np.uint64)[order])          # the oracle is the total order
    assert np.array_equal(gk.view(np.uint64), ok.view(np.uint64))
    if payload:
        assert np.array_equal(gv.view(np.uint64), ov)
    sizes = [len(rdd.compute(r)[0]) for r in range(R)]
    assert sizes == np.diff(ps.astype(np.int64)).tolist()
