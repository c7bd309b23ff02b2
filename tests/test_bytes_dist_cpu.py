"""Byte-string values across ranks, the host logic (vega_b200/dist.py): the bytes engines' refusals before any device
work, and a world_size-2 gloo run of run_shuffle / run_str_shuffle through all_to_all_v with host-side stand-ins for
dist.BytesCudaEngine and dist.StrBytesCudaEngine that speak the same wire columns (keys or key lengths, key bytes and
value counts, then u32 value lengths and the values' bytes).  It checks the column and split bookkeeping of
_bytes_export / _bytes_import and the String pair: three and five columns, each split by its own count vector, received
source-rank major (= map-id order), partition r owned by rank r % world."""
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

from vega_b200 import _lib as L
from vega_b200 import dist as vdist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# ---- refusals -----------------------------------------------------------------------------------------------------------
class _NoContext:
    sc = None


def test_engines_take_byte_string_values_only():
    maps = [(0, np.arange(3, dtype=np.uint64), ["a", "b", "c"])]
    with pytest.raises(TypeError):
        vdist.run_shuffle(vdist.BytesCudaEngine(None), maps, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP, 0, 1)
    with pytest.raises(TypeError):
        vdist.run_str_shuffle(vdist.StrBytesCudaEngine(None), [(0, ["x"], ["a"])], 1, 2, L.VB_U64, L.VB_AGG_GROUP, 0, 1)
    with pytest.raises(TypeError):       # the bytes engines of the other key type
        vdist.run_shuffle(vdist.StrBytesCudaEngine(None), maps, 1, 2, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1)
    with pytest.raises(TypeError):
        vdist.run_str_shuffle(vdist.BytesCudaEngine(None), [(0, ["x"], ["a"])], 1, 2, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1)


@pytest.mark.parametrize("agg", [L.VB_AGG_SUM, L.VB_AGG_MIN, L.VB_AGG_MAX, L.VB_AGG_COUNT])
def test_ops_that_compute_on_values_are_refused(agg):
    with pytest.raises(TypeError):
        vdist.run_shuffle(vdist.BytesCudaEngine(None), [], 1, 2, L.VB_U64, L.VB_BYTES, agg, 0, 2)
    with pytest.raises(TypeError):
        vdist.run_str_shuffle(vdist.StrBytesCudaEngine(None), [], 1, 2, L.VB_BYTES, agg, 0, 2)
    with pytest.raises(TypeError):       # String keys: no COGROUP shuffle kind either
        vdist.run_str_shuffle(vdist.StrBytesCudaEngine(None), [], 1, 2, L.VB_BYTES, L.VB_AGG_COGROUP, 0, 2)


def test_rank_map_block_and_sort_refusals():
    eng, seng = vdist.BytesCudaEngine(_NoContext()), vdist.StrBytesCudaEngine(_NoContext())
    k, v = np.arange(2, dtype=np.uint64), [b"x", b"y"]
    for rank, world in ((2, 2), (0, 0), (0, 257)):
        with pytest.raises(ValueError):
            vdist.run_shuffle(eng, [], 4, 2, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, rank, world)
    with pytest.raises(ValueError):      # map 3 is rank 1's of 2 over 4 map tasks
        vdist.run_shuffle(eng, [(3, k, v)], 4, 2, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, 2)
    with pytest.raises(ValueError):      # not ascending
        vdist.run_str_shuffle(seng, [(1, ["a"], v[:1]), (0, ["b"], v[:1])], 4, 2, L.VB_BYTES, L.VB_AGG_GROUP, 0, 2)
    with pytest.raises(ValueError):      # sorts cross ranks inside the library only
        vdist.run_shuffle(eng, [], 4, 2, L.VB_U64, L.VB_BYTES, L.VB_AGG_SORT, 0, 2)
    with pytest.raises(ValueError):
        vdist.run_str_shuffle(seng, [], 4, 2, L.VB_BYTES, L.VB_AGG_SORT, 0, 2)


class _Sh:
    def map(self, *a):
        raise AssertionError("the library is not reached")


def test_map_refuses_mismatched_and_non_byte_string_columns():
    for eng, keys in ((vdist.BytesCudaEngine(None), np.arange(3, dtype=np.uint64)), (vdist.StrBytesCudaEngine(None), ["a", "b", "c"])):
        with pytest.raises(ValueError):
            eng.map(_Sh(), 0, keys, ["x", "y"])
        with pytest.raises(TypeError):
            eng.map(_Sh(), 0, keys, np.arange(3, dtype=np.uint64))
        with pytest.raises(TypeError):
            eng.map(_Sh(), 0, keys, ["x", b"y", "z"])
    with pytest.raises(TypeError):
        vdist.StrBytesCudaEngine(None).map(_Sh(), 0, [b"a", b"b"], ["x", "y"])


# ---- two ranks over gloo ------------------------------------------------------------------------------------------------
def _place(key, R):
    """The stand-in's partitioner for integer keys (any fixed function works: both ranks use it)."""
    return int(key) % R


def _wire_values(vals):
    lens = [len(v) for v in vals]
    return torch.tensor(lens, dtype=torch.int32), torch.frombuffer(bytearray(b"".join(vals)), dtype=torch.uint8) if sum(lens) \
        else torch.empty(0, dtype=torch.uint8)


def _read_values(lens, data):
    raw, out, pos = bytes(data.numpy()), [], 0
    for ln in lens.tolist():
        out.append(raw[pos:pos + ln])
        pos += ln
    return out


class FakeBytesEngine(vdist.BytesCudaEngine):
    """dist.BytesCudaEngine's calls on the CPU: GROUP of integer keys, rows packed destination-major in map order."""

    def __init__(self):
        super().__init__(None)

    def create(self, n_map, n_reduce, kcode, vcode, agg, rank, world, key_width=8, hint=0):
        return {"R": n_reduce, "maps": {}, "parts": None}

    def map(self, sh, map_id, keys, vals):
        sh["maps"][map_id] = list(zip(np.asarray(keys).tolist(), vals))

    def export(self, sh, world):
        rows = [row for m in sorted(sh["maps"]) for row in sh["maps"][m]]
        by_dst = [[(k, v) for k, v in rows if _place(k, sh["R"]) % world == d] for d in range(world)]
        keys = torch.tensor([k for rs in by_dst for k, _ in rs], dtype=torch.int64)
        lens, data = _wire_values([v for rs in by_dst for _, v in rs])
        return ([len(rs) for rs in by_dst], [sum(len(v) for _, v in rs) for rs in by_dst]), (keys, lens, data)

    def import_(self, sh, cols, counts):
        keys, lens, data = cols
        rows, nvb = counts
        assert sum(rows) == len(keys) == len(lens) and sum(nvb) == len(data) == int(lens.sum())
        sh["recv"] = list(zip(keys.tolist(), _read_values(lens, data)))

    def seal(self, sh):
        parts = [dict() for _ in range(sh["R"])]
        for k, v in sh.get("recv", [row for m in sorted(sh["maps"]) for row in sh["maps"][m]]):
            parts[_place(k, sh["R"])].setdefault(k, []).append(v)
        sh["parts"] = parts

    def reduce(self, sh, r):
        return sh["parts"][r]


class FakeStrBytesEngine(vdist.StrBytesCudaEngine):
    """dist.StrBytesCudaEngine's calls on the CPU: GROUP of String keys; each key once per destination with its values."""

    def __init__(self):
        super().__init__(None)

    def create(self, n_map, n_reduce, vcode, agg, rank, world, hint=0):
        return {"R": n_reduce, "maps": {}, "parts": None}

    def map(self, sh, map_id, keys, vals):
        sh["maps"][map_id] = list(zip(keys, vals))

    def _grouped(self, sh):
        g = {}
        for m in sorted(sh["maps"]):
            for k, v in sh["maps"][m]:
                g.setdefault(k, []).append(v)
        return g

    def export(self, sh, world):
        from oracle import pyref
        g = self._grouped(sh)
        by_dst = [[k for k in g if pyref.get_partition(k, sh["R"]) % world == d] for d in range(world)]
        ks = [k for d in by_dst for k in d]
        enc = [k.encode("utf-8") for k in ks]
        vals = [v for k in ks for v in g[k]]
        key_lens = torch.tensor([len(e) for e in enc], dtype=torch.int32)
        key_bytes = torch.frombuffer(bytearray(b"".join(enc)), dtype=torch.uint8) if any(enc) else torch.empty(0, dtype=torch.uint8)
        cnts = torch.tensor([len(g[k]) for k in ks], dtype=torch.int32)
        lens, data = _wire_values(vals)
        counts = ([len(d) for d in by_dst], [sum(len(k.encode()) for k in d) for d in by_dst],
                  [sum(len(g[k]) for k in d) for d in by_dst], [sum(len(v) for k in d for v in g[k]) for d in by_dst])
        return counts, (key_lens, key_bytes, cnts, lens, data)

    def import_(self, sh, cols, counts):
        key_lens, key_bytes, cnts, lens, data = cols
        nk, nkb, nv, nvb = counts
        assert sum(nk) == len(key_lens) == len(cnts) and sum(nkb) == len(key_bytes) and sum(nv) == len(lens) == int(cnts.sum())
        assert sum(nvb) == len(data) == int(lens.sum())
        keys = _read_values(key_lens, key_bytes)
        vals = _read_values(lens, data)
        rows, pos = [], 0
        for k, c in zip(keys, cnts.tolist()):
            rows += [(k.decode("utf-8"), v) for v in vals[pos:pos + c]]
            pos += c
        sh["recv"] = rows

    def seal(self, sh):
        from oracle import pyref
        parts = [dict() for _ in range(sh["R"])]
        rows = sh.get("recv", [row for m in sorted(sh["maps"]) for row in sh["maps"][m]])
        for k, v in rows:
            parts[pyref.get_partition(k, sh["R"])].setdefault(k, []).append(v)
        sh["parts"] = parts

    def reduce(self, sh, r):
        return sh["parts"][r]


def _dataset(s):
    rng = np.random.default_rng(9)
    n = 2000
    lens = rng.integers(0, 40, n)
    lens[::97] = 0
    raw = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
    o = np.concatenate([[0], np.cumsum(lens)])
    vals = [raw[o[i]:o[i + 1]] for i in range(n)]
    if s:
        words = ["", "a", "é", "\x00x"] + ["w%d" % i for i in range(150)]
        return [words[i] for i in rng.integers(0, len(words), n)], vals
    return rng.integers(0, 400, n).astype(np.uint64), vals


def _worker(rank, world, port, s, M, R, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from vega_b200 import dist as vd
    from vega_b200.rdd import slice_starts
    keys, vals = _dataset(s)
    starts = slice_starts(len(vals), M)
    lo, hi = vd.map_block(rank, world, M)
    maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    stats = {}
    if s:
        eng = FakeStrBytesEngine()
        sh = vd.run_str_shuffle(eng, maps, M, R, L.VB_BYTES, L.VB_AGG_GROUP, rank, world, stats=stats)
    else:
        eng = FakeBytesEngine()
        sh = vd.run_shuffle(eng, maps, M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, rank, world, stats=stats)
    res = {r: eng.reduce(sh, r) for r in range(R)}
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats), f)
    dist.destroy_process_group()


@pytest.mark.parametrize("s", [False, True], ids=["int", "str"])
@pytest.mark.parametrize("M,R", [(4, 5), (1, 3), (3, 1)])
def test_two_rank_bytes_shuffle_over_gloo(s, M, R):
    """M = 1: rank 0 maps nothing; R = 1: rank 1 receives nothing."""
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), s, M, R, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset(s)
    eng = FakeStrBytesEngine() if s else FakeBytesEngine()
    one = eng.create(M, R, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1) if s else eng.create(M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1)
    eng.map(one, 0, keys, vals)
    eng.seal(one)
    for r in range(R):
        assert per_rank[r % world][0][r] == eng.reduce(one, r), r
        assert not per_rank[(r + 1) % world][0][r]
    st = [x[1] for x in per_rank]
    assert st[0]["sent_rows"] == st[1]["recv_rows"] and st[1]["sent_rows"] == st[0]["recv_rows"]
    assert st[0]["sent_rows"] + st[1]["sent_rows"] > 0
