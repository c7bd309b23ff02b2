"""CPU-side checks of the semi and anti join: the restatement in tests/semi_join_ref.py against brute force on small
random cases, its array forms against the restatement, the Python mirror's argument errors (raised before any device
work), and the declarations of the four calls in the header, the Python binding and the Rust shim."""
import os
import random
import re

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import cogroup_n_ref as CN
from tests import semi_join_ref as SJ
from tests.test_join_n_outer_cpu import _NoDevice

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("vb_semi_join_n_size", "vb_semi_join_n", "vb_semi_join_n_str_size", "vb_semi_join_n_str")


def brute(parents, required, excluded):
    """{k: [side-0 values in input order]} of the kept keys, straight from the rows"""
    keysets = [{k for k, _ in rows} for rows, _ in parents]
    out = {}
    for k, v in parents[0][0]:
        if all(k in keysets[j] for j in range(len(parents)) if required >> j & 1) and \
                not any(k in keysets[j] for j in range(len(parents)) if excluded >> j & 1):
            out.setdefault(k, []).append(v)
    return out


def masks(n):
    for req in range(0, 1 << n, 2):
        for exc in range(0, 1 << n, 2):
            if not req & exc:
                yield req, exc


@pytest.mark.parametrize("n,seed", [(1, 0), (2, 1), (3, 2), (4, 3)])
def test_restatement_is_brute_force(n, seed):
    rng = random.Random(seed)
    keys = [0, 2 ** 64 - 1] + [rng.randrange(1 << 64) for _ in range(30)]
    parents = [([(rng.choice(keys), rng.randrange(1 << 64)) for _ in range(rng.randrange(0, 120))], rng.randrange(1, 5))
               for _ in range(n)]
    R = 3
    for req, exc in masks(n):
        got = {}
        for k, v in SJ.semi_join_n(parents, R, req, exc):
            got.setdefault(k, []).append(v)
        assert got == brute(parents, req, exc), (req, exc)


def test_special_cases():
    rng = random.Random(7)
    a = [(rng.randrange(20), rng.randrange(100)) for _ in range(200)]
    b = [(rng.randrange(10, 30), rng.randrange(100)) for _ in range(50)]
    sub = SJ.semi_join_n([(a, 3), (b, 2)], 4, 0, 0b10)
    semi = SJ.semi_join_n([(a, 3), (b, 2)], 4, 0b10, 0)
    assert sorted(sub) == sorted((k, v) for k, v in a if k not in {x for x, _ in b})
    assert sorted(semi) == sorted((k, v) for k, v in a if k in {x for x, _ in b})
    # both masks 0: side 0's rows as its group_by_key gives them
    want = [(k, v) for k, vs in P.group_by_key(a, 3, 4) for v in vs]
    assert SJ.semi_join_n([(a, 3), (b, 2)], 4, 0, 0) == want == SJ.semi_join_n([(a, 3)], 4, 0, 0)


@pytest.mark.parametrize("key_width", [8, 4])
def test_array_reference_matches_the_restatement(key_width):
    rng = np.random.default_rng(key_width)
    if key_width == 8:
        ks = [rng.integers(lo, lo + 40, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) for lo, n in ((0, 120), (20, 90), (30, 60))]
        ks[0][:2] = [0, 2 ** 64 - 1]
        to_py = int
    else:
        ks = [rng.integers(lo, lo + 40, n).astype(np.int32) for lo, n in ((-20, 120), (0, 90), (10, 60))]
        to_py = lambda k: int(k) & 0xFFFFFFFF
    vs = [rng.integers(1, 1 << 62, len(k)).astype(np.uint64) for k in ks]
    Ms, R = (3, 2, 4), 5
    parts = CN.ref_parts_n(list(zip(ks, vs, Ms)), R, key_width)
    parents = [([(to_py(x), int(y)) for x, y in zip(k, v)], M) for k, v, M in zip(ks, vs, Ms)]
    u64_of = {to_py(x): int(np.int64(x).view(np.uint64)) if key_width == 4 else int(x) for k in ks for x in k}
    for req, exc in masks(3):
        want = {}
        for k, v in SJ.semi_join_n(parents, R, req, exc, key_width):
            want.setdefault(u64_of[k], []).append(v)
        got = SJ.semi_of_parts(parts, req, exc)
        assert {k: l for d in got for k, l in d.items()} == want, (req, exc)
        for r, d in enumerate(got):
            assert all(P.get_partition(k if key_width == 8 else k & 0xFFFFFFFF, R, key_width) == r for k in d)
        lists = [{u64_of[to_py(x)]: [] for x in k} for k in ks]
        for j, (k, v) in enumerate(zip(ks, vs)):
            for x, y in zip(k, v):
                lists[j][u64_of[to_py(x)]].append(int(y))
        where = {k: r for r, d in enumerate(parts) for k in d}
        part = lambda k, R: where[k]
        if (req, exc) in ((0, 0b10), (0b10, 0b100)):    # the dict form agrees with the partition form
            assert SJ.semi_of_lists(lists, R, req, exc, part) == got


def test_python_mirror_argument_errors_before_device_work():
    k64 = np.arange(5, dtype=np.uint64)
    ctx = _NoDevice()
    a = vb.Context.parallelize(ctx, (k64, k64), 2)
    b = vb.Context.parallelize(ctx, (k64, np.arange(5, dtype=np.float64)), 3)
    cg = vb.CoGroupedRdd([a, b, a], 3)
    assert cg._semi_masks(0b10, 0b100) == (2, 4) and cg._semi_masks([1], [2]) == (2, 4) and cg._semi_masks(0, 0) == (0, 0)
    for req, exc in ((1, 0), (0, 1), (0b10, 0b10), (0b110, 0b100), (8, 0), (0, 1 << 16), ([0], []), ([], [3]), (-1, 0)):
        with pytest.raises(ValueError):
            cg.semi_join_compute(0, req, exc)
        with pytest.raises(ValueError):
            cg.semi_join_collect(req, exc)
    for req, exc in ((None, 0), (0, 1.0), ("1", 0), ([True], 0)):
        with pytest.raises(TypeError):
            cg.semi_join_compute(0, req, exc)
    # the RDD methods check their parents when called, before any device work
    sj = a.subtract_by_key(b, 3)
    assert isinstance(sj, vb.SemiJoinedRdd) and (sj.required, sj.excluded) == (0, 0b10)
    sj = a.semi_join(b, 3, sort_values=True)
    assert (sj.required, sj.excluded) == (0b10, 0)
    with pytest.raises(ValueError):
        a.subtract_by_key(b, 0)
    with pytest.raises(TypeError):
        a.semi_join(b, 3, sort_values=1)
    k32 = vb.Context.parallelize(ctx, (np.arange(5, dtype=np.int32), k64), 2)
    with pytest.raises(TypeError):
        a.subtract_by_key(k32, 3)                     # different key types
    s = vb.Context.parallelize(ctx, vb.StrKeys.from_strs(["a", "b"]), 2, values=np.arange(2, dtype=np.uint64))
    assert isinstance(s, vb.StrPairRdd)
    with pytest.raises(TypeError):
        a.subtract_by_key(s, 3)                       # an integer-key call on a String parent
    with pytest.raises(TypeError):
        s.subtract_by_key(a, 3)                       # and the reverse: StrPairRdd overrides the integer methods
    sj = s.semi_join(s, 2)
    assert isinstance(sj.cogrouped, vb.StrCoGroupedRdd) and (sj.required, sj.excluded) == (0b10, 0)
    with pytest.raises(ValueError):
        sj.cogrouped.semi_join_compute(0, 0b1, 0)


def test_declarations():
    h = open(os.path.join(ROOT, "include", "vega_b200.h")).read()
    rs = open(os.path.join(ROOT, "rust_shim", "vega_b200_sys.rs")).read()
    for name in CALLS:
        assert re.search(r"VB_API int32_t %s\(" % name, h), name
        assert re.search(r"pub fn %s\(" % name, rs), name
        assert name in vb.SYMBOLS
    sig = lambda name: re.search(r"VB_API int32_t %s\((.*?)\);" % name, h, re.S).group(1)
    assert "uint32_t required" in sig("vb_semi_join_n") and "uint32_t excluded" in sig("vb_semi_join_n_str_size")
    assert len(vb.SYMBOLS["vb_semi_join_n"][1]) == 8 and len(vb.SYMBOLS["vb_semi_join_n_str"][1]) == 10
    assert len(vb.SYMBOLS["vb_semi_join_n_size"][1]) == 6 and len(vb.SYMBOLS["vb_semi_join_n_str_size"][1]) == 8
