"""world_size-2 gloo test of the String exchange's host logic (vega_b200/dist.py: run_str_shuffle, all_to_all_v):
the swap of three counts per destination, the four columns split by keys, key bytes, keys and values, source-rank
major receive order (= map-id order), and partition ownership r % world.  The per-rank compute is a small pyref-backed
stand-in for dist.StrCudaEngine that speaks the same wire columns (u32 key lengths, key bytes, u32 value counts, u64
values); on the GPU the same run_str_shuffle drives the library (tests/test_gpu_str_dist.py)."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
SUM, COUNT, GROUP = 1, 4, 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class FakeStrEngine:
    """dist.StrCudaEngine's calls on the CPU: SUM (wrapping u64), COUNT and GROUP, placed by pyref.get_partition."""

    def create(self, n_map, n_reduce, vcode, agg, rank, world, hint=0):
        return {"R": n_reduce, "agg": agg, "world": world, "maps": {}, "recv": None}

    def map(self, sh, map_id, keys, vals):
        sh["maps"][map_id] = (list(keys), [1] * len(keys) if vals is None else [int(v) & M64 for v in vals])

    def export(self, sh, world):
        from oracle import pyref
        comb = {}                                       # map-side combine, in map-id order
        for m in sorted(sh["maps"]):
            for k, v in zip(*sh["maps"][m]):
                if sh["agg"] == GROUP:
                    comb.setdefault(k, []).append(v)
                else:
                    comb[k] = (comb.get(k, 0) + v) & M64
        by_dst = [[k for k in comb if pyref.get_partition(k, sh["R"]) % world == d] for d in range(world)]
        enc = {k: k.encode("utf-8") for k in comb}
        lens, data, cnts, vals = [], b"", [], []
        counts = ([], [], [])
        for ks in by_dst:
            vs = [x for k in ks for x in (comb[k] if sh["agg"] == GROUP else [comb[k]])]
            counts[0].append(len(ks))
            counts[1].append(sum(len(enc[k]) for k in ks))
            counts[2].append(len(vs))
            lens += [len(enc[k]) for k in ks]
            data += b"".join(enc[k] for k in ks)
            cnts += [len(comb[k]) for k in ks] if sh["agg"] == GROUP else []
            vals += vs
        i64 = lambda xs: torch.tensor(np.array(xs, dtype=np.uint64).view(np.int64))
        cols = (torch.tensor(lens, dtype=torch.int32), torch.frombuffer(bytearray(data), dtype=torch.uint8) if data else
                torch.empty(0, dtype=torch.uint8), torch.tensor(cnts, dtype=torch.int32) if sh["agg"] == GROUP else None, i64(vals))
        return counts, cols

    def import_(self, sh, cols, counts):
        assert sum(counts[0]) == len(cols[0]) and sum(counts[1]) == len(cols[1]) and sum(counts[2]) == len(cols[3])
        sh["recv"] = (cols, counts)

    def seal(self, sh):
        from oracle import pyref
        res = [dict() for _ in range(sh["R"])]
        if sh["recv"] is not None:
            (lens, data, cnts, vals), _ = sh["recv"]
            raw, vals = bytes(data.numpy()), vals.numpy().view(np.uint64).tolist()
            pos = vpos = 0
            for i, ln in enumerate(lens.tolist()):
                k = raw[pos:pos + ln].decode("utf-8")
                pos += ln
                part = res[pyref.get_partition(k, sh["R"])]
                if sh["agg"] == GROUP:
                    c = int(cnts[i])
                    part.setdefault(k, []).extend(vals[vpos:vpos + c])
                    vpos += c
                else:
                    part[k] = (part.get(k, 0) + vals[i]) & M64
        sh["parts"] = res

    def reduce(self, sh, r):
        return sh["parts"][r]


def _dataset():
    rng = np.random.default_rng(7)
    words = ["", "a", "é", "\x00x", "the", "of", "and"] + ["w%d" % i for i in range(200)] + ["long" * 300]
    n = 3000
    keys = [words[i] for i in rng.integers(0, len(words), n)]
    vals = rng.integers(0, 1 << 62, n).astype(np.uint64)
    return keys, vals


def _worker(rank, world, port, agg, M, R, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from vega_b200 import dist as vdist
    from vega_b200.rdd import slice_starts
    keys, vals = _dataset()
    starts = slice_starts(len(keys), M)
    lo, hi = vdist.map_block(rank, world, M)
    maps = [(m, keys[starts[m]:starts[m + 1]], None if agg == COUNT else vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    stats = {}
    eng = FakeStrEngine()
    sh = vdist.run_str_shuffle(eng, maps, M, R, 0, agg, rank, world, stats=stats)
    res = {}
    for r in range(R):
        out = eng.reduce(sh, r)
        if r % world != rank:
            assert len(out) == 0, "a rank holds keys of a partition it does not own"
        res[r] = out
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats), f)
    dist.destroy_process_group()


@pytest.mark.parametrize("agg,M,R", [(SUM, 4, 4), (COUNT, 5, 3), (GROUP, 4, 6), (GROUP, 3, 1), (SUM, 1, 5)])
def test_two_rank_string_shuffle_matches_pyref(agg, M, R):
    """M = 1: rank 0 has no map task and only receives."""
    from oracle import pyref
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), agg, M, R, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset()
    rows = list(zip(keys, [1] * len(keys) if agg == COUNT else [int(v) for v in vals]))
    res = pyref.group_by_key(rows, M, R) if agg == GROUP else pyref.reduce_by_key(rows, lambda a, b: (a + b) & M64, M, R)
    want = [dict() for _ in range(R)]
    for k, v in res:
        want[pyref.get_partition(k, R)][k] = list(v) if agg == GROUP else v
    for r in range(R):
        assert per_rank[r % world][0][r] == want[r], r
    sent = sum(s["sent_rows"] for _, s in per_rank)
    assert sent == sum(s["recv_rows"] for _, s in per_rank) and sent > 0
