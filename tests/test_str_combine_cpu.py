"""combine_by_key over String keys without a GPU: the Python mirror's argument errors come before any device work, the
tuple-of-columns parallelize gives a StrPairRdd with value columns, and a world_size-2 gloo run of
dist.run_str_combine_shuffle's host logic (the swap of key and byte counts, the key lengths, key bytes and the
[keys][n_acc] partials split by destination, source-rank major receive order, ownership r % world).  The per-rank compute
is a pyref-backed stand-in for dist.StrCombineCudaEngine speaking the same wire columns; on the GPU the same
run_str_combine_shuffle drives the library (tests/test_gpu_str_combine_exchange.py)."""
import os
import pickle
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import vega_b200 as vb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
I64_MAX = (1 << 63) - 1


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_combine_by_key_needs_value_columns_as_a_tuple():
    """combine_by_key runs on a StrPairRdd of value columns given as a tuple; one plain value array keeps the
    single-column ops only, and its combine_by_key raises TypeError before any device work, as it always has."""
    sc = _NoDevice()
    keys = ["x", "y", "x"]
    vals = np.array([1, 2, 3], dtype=np.uint64)
    for a in (vb.Context.parallelize(sc, keys, 2, values=vals), vb.Context.parallelize(sc, (keys, vals), 2)):
        with pytest.raises(TypeError, match="value columns given as a tuple"):
            a.combine_by_key({"n": ("count", None)}, 2)
        assert a.reduce_by_key("sum", 3).num_slices == 3
    t = vb.Context.parallelize(sc, keys, 2, values=(vals,))
    assert isinstance(t, vb.StrPairRdd) and len(t.cols) == 1
    assert isinstance(t.combine_by_key({"n": ("count", None)}, 2), vb.StrCombinedRdd)
    assert t.reduce_by_key("sum", 3).num_slices == 3                  # one column: the single-column ops stay


def _cols(n=3):
    return (np.arange(n, dtype=np.uint64), np.arange(n, dtype=np.int64) - 1, np.linspace(0, 1, n))


def test_parallelize_tuple_of_value_columns():
    sc = _NoDevice()
    keys = ["a", "", "é"]
    for k in range(1, 5):
        p = vb.Context.parallelize(sc, keys, 2, values=(_cols() * 2)[:k])
        assert isinstance(p, vb.StrPairRdd) and len(p.cols) == k and p.n == 3
        assert [c.code for c in p.cols] == [vb._lib.VB_U64, vb._lib.VB_I64, vb._lib.VB_F64, vb._lib.VB_U64][:k]
        assert (p.vals is not None) == (k == 1)
    p = vb.Context.parallelize(sc, vb.StrKeys.from_strs(keys), 2, values=_cols())
    assert isinstance(p, vb.StrPairRdd) and len(p.cols) == 3
    with pytest.raises(ValueError):
        vb.Context.parallelize(sc, keys, 2, values=_cols() + _cols())          # five columns or more
    with pytest.raises(ValueError):
        vb.Context.parallelize(sc, keys, 2, values=(np.arange(3, dtype=np.uint64), np.arange(2, dtype=np.uint64)))
    with pytest.raises(ValueError):
        vb.Context.parallelize(sc, keys, 2, values=(np.zeros((3, 2), dtype=np.uint64),))
    with pytest.raises(TypeError):
        vb.Context.parallelize(sc, keys, 2, values=(np.arange(3, dtype=np.float32),))
    # a tuple of scalars stays one value column, as before
    p = vb.Context.parallelize(sc, keys, 2, values=(1, 2, 3))
    assert len(p.cols) == 1 and p.vals.n == 3


def test_combine_by_key_errors_before_device_work():
    sc = _NoDevice()
    p = vb.Context.parallelize(sc, ["a", "b", "a"], 2, values=_cols())
    ok = {"s": ("sum", 0), "lo": ("min", 1), "hi": ("max", 2), "avg": ("mean", 2), "n": ("count", None)}
    c = p.combine_by_key(ok, 5, hint=7)
    assert isinstance(c, vb.StrCombinedRdd) and c.names == list(ok) and c.num_slices == 5 and c.hint == 7
    assert c.spec == [(vb._lib.VB_AGG_SUM, 0), (vb._lib.VB_AGG_MIN, 1), (vb._lib.VB_AGG_MAX, 2), (vb._lib.VB_AGG_MEAN, 2),
                      (vb._lib.VB_AGG_COUNT, 0)]
    assert c.out_dtypes == [np.uint64, np.int64, np.float64, np.float64, np.uint64]
    bad = [({}, 2), ([("s", ("sum", 0))], 2), ({"s": ("sum",)}, 2), ({"s": ("avg", 0)}, 2), ({"s": ("sum", 3)}, 2),
           ({"s": ("sum", -1)}, 2), ({"s": ("sum", True)}, 2), ({"s": ("sum", "0")}, 2), ({"s": ("sum", 0)}, 0),
           ({f"m{i}": ("mean", 0) for i in range(8)}, 2), ({f"s{i}": ("sum", 0) for i in range(9)}, 2)]
    for aggs, n in bad:
        with pytest.raises(ValueError):
            p.combine_by_key(aggs, n)
    # the same errors as the integer combine, from the one shared parser
    q = vb.Context.parallelize(sc, np.arange(3, dtype=np.uint64), 2, values=_cols())
    for aggs, n in bad:
        with pytest.raises(ValueError) as e_int:
            q.combine_by_key(aggs, n)
        with pytest.raises(ValueError) as e_str:
            p.combine_by_key(aggs, n)
        assert str(e_int.value) == str(e_str.value)
    # several value columns: the single-column ops raise as an integer PairRdd with several columns does
    for rdd in (p, q):
        for method, args in [("reduce_by_key", ("sum", 2)), ("count_by_key", ()), ("group_by_key", (2,)), ("partition_by_key", (2,))]:
            with pytest.raises(TypeError, match="several value columns supports combine_by_key only"):
                getattr(rdd, method)(*args)
    one = vb.Context.parallelize(sc, ["a"], 1, values=(np.arange(1, dtype=np.int64),))
    assert one.combine_by_key({"n": ("count", None), "s": ("sum", 0)}, 1).out_dtypes == [np.uint64, np.int64]
    assert one.reduce_by_key("sum", 1).num_slices == 1                        # one column: the single-column ops stay
    assert not hasattr(vb.Context.parallelize(sc, ["a"], 1), "combine_by_key")        # keys only: no values to combine


def test_str_combine_is_not_a_join_parent():
    sc = _NoDevice()
    p = vb.Context.parallelize(sc, ["a", "b"], 1, values=_cols(2))
    c = p.combine_by_key({"s": ("sum", 0)}, 2)
    with pytest.raises(TypeError):
        vb.StrCoGroupedRdd([c, vb.Context.parallelize(sc, ["a"], 1, values=np.zeros(1, np.uint64))], 2)


# ---- the exchange's host logic over gloo -------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _signed(x):
    return x - (1 << 64) if x >= 1 << 63 else x


class FakeStrCombineEngine:
    """dist.StrCombineCudaEngine's calls on the CPU for the spec sum(v0) (wrapping u64), min(v1) (i64), count: three
    accumulators, placed by pyref.get_partition, wire columns as include/vega_b200.h documents them."""

    def create(self, n_map, n_reduce, multi, rank, world, hint=0):
        return {"R": n_reduce, "maps": {}, "recv": None}

    def map(self, sh, map_id, keys, cols):
        sh["maps"][map_id] = (list(keys), cols[0].tolist(), cols[1].tolist())

    def export(self, sh, world):
        from oracle import pyref
        comb = {}                                            # the rank's partial per key: [sum, min, count]
        for m in sorted(sh["maps"]):
            for k, a, b in zip(*sh["maps"][m]):
                s, lo, c = comb.get(k, (0, I64_MAX, 0))
                comb[k] = ((s + a) & M64, min(lo, b), c + 1)
        by_dst = [[k for k in comb if pyref.get_partition(k, sh["R"]) % world == d] for d in range(world)]
        order = [k for ks in by_dst for k in ks]
        enc = [k.encode("utf-8") for k in order]
        data = b"".join(enc)
        as_i64 = lambda xs: torch.tensor(np.array(xs, dtype=np.uint64).view(np.int64), dtype=torch.int64)
        accs = torch.stack([as_i64([comb[k][0] for k in order]), torch.tensor([comb[k][1] for k in order], dtype=torch.int64),
                            as_i64([comb[k][2] for k in order])]) if order else torch.empty((3, 0), dtype=torch.int64)
        cols = (torch.tensor([len(b) for b in enc], dtype=torch.int32),
                torch.frombuffer(bytearray(data), dtype=torch.uint8) if data else torch.empty(0, dtype=torch.uint8), accs)
        counts = ([len(ks) for ks in by_dst], [sum(len(k.encode()) for k in ks) for ks in by_dst])
        return counts, cols

    def import_(self, sh, cols, counts):
        lens, data, accs = cols
        assert accs.shape == (3, len(lens)) and sum(counts[0]) == len(lens) and sum(counts[1]) == len(data)
        sh["recv"] = cols

    def seal(self, sh):
        from oracle import pyref
        res = [dict() for _ in range(sh["R"])]
        if sh["recv"] is not None:
            lens, data, accs = sh["recv"]
            raw = bytes(data.numpy())
            sums, mins, cnts = accs[0].numpy().view(np.uint64).tolist(), accs[1].tolist(), accs[2].numpy().view(np.uint64).tolist()
            pos = 0
            for i, ln in enumerate(lens.tolist()):
                k = raw[pos:pos + ln].decode("utf-8")
                pos += ln
                part = res[pyref.get_partition(k, sh["R"])]
                s, lo, c = part.get(k, (0, I64_MAX, 0))
                part[k] = ((s + sums[i]) & M64, min(lo, mins[i]), c + cnts[i])
        sh["parts"] = res

    def reduce(self, sh, r, out_dtypes=None):
        return sh["parts"][r]


def _dataset():
    rng = np.random.default_rng(5)
    words = ["", "a", "é", "\x00x", "日本語", "the", "of"] + ["w%d" % i for i in range(150)] + ["long" * 200, "long" * 200 + "!"]
    n = 3000
    keys = [words[i] for i in rng.integers(0, len(words), n)]
    return keys, rng.integers(0, 1 << 64, n, dtype=np.uint64), rng.integers(-(1 << 63), I64_MAX, n, dtype=np.int64)


def _worker(rank, world, port, M, R, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from vega_b200 import dist as vdist
    from vega_b200.rdd import slice_starts
    keys, a, b = _dataset()
    starts = slice_starts(len(keys), M)
    lo, hi = vdist.map_block(rank, world, M)
    maps = [(m, keys[starts[m]:starts[m + 1]], (a[starts[m]:starts[m + 1]], b[starts[m]:starts[m + 1]])) for m in range(lo, hi)]
    stats = {}
    eng = FakeStrCombineEngine()
    sh = vdist.run_str_combine_shuffle(eng, maps, M, R, None, rank, world, stats=stats)
    res = {}
    for r in range(R):
        out = eng.reduce(sh, r)
        if r % world != rank:
            assert len(out) == 0, "a rank holds keys of a partition it does not own"
        res[r] = out
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats), f)
    dist.destroy_process_group()


@pytest.mark.parametrize("M,R", [(4, 5), (5, 1), (1, 3)])
def test_two_rank_str_combine_matches_pyref(M, R):
    """M = 1: rank 0 has no map task and only receives; R = 1: rank 1 owns nothing."""
    from oracle import pyref
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), M, R, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, a, b = _dataset()
    want = [dict() for _ in range(R)]
    for k, x, y in zip(keys, a.tolist(), b.tolist()):
        part = want[pyref.get_partition(k, R)]
        s, lo, c = part.get(k, (0, I64_MAX, 0))
        part[k] = ((s + x) & M64, min(lo, y), c + 1)
    for r in range(R):
        assert per_rank[r % world][0][r] == want[r], r
    sent = sum(s["sent_rows"] for _, s in per_rank)
    assert sent == sum(s["recv_rows"] for _, s in per_rank) and sent > 0


def test_all_to_all_v_on_one_rank():
    """The column layout of the String combine exchange without a peer: keys keep their order and bytes, the
    accumulators come back as [n_acc][keys]."""
    from vega_b200 import dist as vdist

    class Echo:
        def export(self, sh, world):
            return ([3], [5]), (torch.tensor([2, 0, 3], dtype=torch.int32), torch.arange(5, dtype=torch.uint8),
                                torch.arange(12, dtype=torch.int64).view(4, 3))

        def import_(self, sh, cols, counts):
            sh["got"] = (cols, counts)

    port = _free_port()
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        e, sh = Echo(), {}
        cols, splits = vdist._str_combine_export(e, sh, 1)
        rcols, rsplits = vdist.all_to_all_v(cols, splits)
        vdist._str_combine_import(e, sh, rcols, rsplits)
        (lens, data, accs), counts = sh["got"]
        want = e.export(sh, 1)[1]
        assert counts == ([3], [5]) and torch.equal(lens, want[0]) and torch.equal(data, want[1]) and torch.equal(accs, want[2])
    finally:
        dist.destroy_process_group()


class _NoDeviceEngine(FakeStrCombineEngine):
    def create(self, *a, **kw):
        raise AssertionError("argument errors must be raised before any shuffle is created")


@pytest.mark.parametrize("rank,world,ids", [(2, 2, []), (0, 0, []), (0, 257, []), (1, 2, [0]), (0, 2, [1, 0]), (0, 2, [0, 0])])
def test_argument_errors_before_device_work(rank, world, ids):
    """A rank outside the world, a world outside 1..256, map ids outside the rank's block or not ascending."""
    from vega_b200 import dist as vdist
    maps = [(m, ["k"], (np.zeros(1, np.uint64), np.zeros(1, np.int64))) for m in ids]
    with pytest.raises(ValueError):
        vdist.run_str_combine_shuffle(_NoDeviceEngine(), maps, 4, 3, None, rank, world)
