"""world_size-2 gloo test of the combine_by_key exchange's host logic (vega_b200/dist.py: run_combine_shuffle,
all_to_all_v): the count swap, one row per distinct key carrying the key and every accumulator partial, source-rank
major receive order, and partition ownership r % world.  The per-rank compute is a numpy stand-in for
dist.CombineCudaEngine that speaks the same wire columns (u64 keys, u64 accumulators [n_acc][rows]); on the GPU the same
run_combine_shuffle drives the library (tests/test_gpu_combine_dist.py)."""
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
I64_MAX = (1 << 63) - 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _signed(x):
    return x - (1 << 64) if x >= 1 << 63 else x


class FakeCombineEngine:
    """dist.CombineCudaEngine's calls on the CPU for the spec sum(v0) (wrapping u64), min(v1) (i64), count: three
    accumulators, placed by oracle.get_partition."""

    def create(self, n_map, n_reduce, kcode, multi, rank, world, key_width=8, hint=0):
        return {"R": n_reduce, "maps": {}, "recv": None}

    def map(self, sh, map_id, keys, cols):
        sh["maps"][map_id] = (keys.tolist(), cols[0].tolist(), cols[1].tolist())

    def export(self, sh, world):
        from oracle import oracle as O
        comb = {}                                            # the rank's partial per key: [sum, min, count]
        for m in sorted(sh["maps"]):
            for k, a, b in zip(*sh["maps"][m]):
                s, lo, c = comb.get(k, (0, I64_MAX, 0))
                comb[k] = ((s + a) & M64, min(lo, b), c + 1)
        by_dst = [[k for k in comb if O.get_partition(k, sh["R"]) % world == d] for d in range(world)]
        order = [k for ks in by_dst for k in ks]
        as_i64 = lambda xs: torch.tensor(np.array(xs, dtype=np.uint64).view(np.int64), dtype=torch.int64)
        keys = as_i64(order)
        accs = torch.stack([as_i64([comb[k][0] for k in order]), torch.tensor([comb[k][1] for k in order], dtype=torch.int64),
                            as_i64([comb[k][2] for k in order])]) if order else torch.empty((3, 0), dtype=torch.int64)
        return [len(ks) for ks in by_dst], keys, accs

    def import_(self, sh, keys, accs, counts):
        assert accs.shape == (3, len(keys)) and sum(counts) == len(keys)
        sh["recv"] = (keys.numpy().view(np.uint64).tolist(), accs.numpy())

    def seal(self, sh):
        from oracle import oracle as O
        res = [dict() for _ in range(sh["R"])]
        if sh["recv"] is not None:
            keys, accs = sh["recv"]
            sums, mins, cnts = accs[0].view(np.uint64).tolist(), accs[1].tolist(), accs[2].view(np.uint64).tolist()
            for i, k in enumerate(keys):
                part = res[O.get_partition(k, sh["R"])]
                s, lo, c = part.get(k, (0, I64_MAX, 0))
                part[k] = ((s + sums[i]) & M64, min(lo, mins[i]), c + cnts[i])
        sh["parts"] = res

    def reduce(self, sh, r, out_dtypes=None):
        return sh["parts"][r]


def _dataset():
    rng = np.random.default_rng(11)
    n = 4000
    keys = rng.integers(0, 300, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    keys[::97] = np.uint64(M64)
    keys[1::89] = np.uint64(0)
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
    eng = FakeCombineEngine()
    sh = vdist.run_combine_shuffle(eng, maps, M, R, 0, None, rank, world, stats=stats)
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
def test_two_rank_combine_matches_numpy(M, R):
    """M = 1: rank 0 has no map task and only receives; R = 1: rank 1 owns nothing."""
    from oracle import oracle as O
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), M, R, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, a, b = _dataset()
    want = [dict() for _ in range(R)]
    for k, x, y in zip(keys.tolist(), a.tolist(), b.tolist()):
        part = want[O.get_partition(k, R)]
        s, lo, c = part.get(k, (0, I64_MAX, 0))
        part[k] = ((s + x) & M64, min(lo, y), c + 1)
    for r in range(R):
        assert per_rank[r % world][0][r] == want[r], r
    sent = sum(s["sent_rows"] for _, s in per_rank)
    assert sent == sum(s["recv_rows"] for _, s in per_rank) and sent > 0


def test_all_to_all_v_on_one_rank():
    """The column layout of the combine exchange step without a peer: rows keep their order, accumulators stay
    [n_acc][rows]."""
    from vega_b200 import dist as vdist
    port = _free_port()
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        k = torch.arange(5, dtype=torch.int64)
        a = torch.arange(15, dtype=torch.int64).view(3, 5)
        rk, ra, rc = vdist._combine_unpack(*vdist.all_to_all_v(*vdist._combine_pack([5], k, a)))
        assert rc == [5] and torch.equal(rk, k) and torch.equal(ra, a)
    finally:
        dist.destroy_process_group()


class _NoDeviceEngine(FakeCombineEngine):
    def create(self, *a, **kw):
        raise AssertionError("argument errors must be raised before any shuffle is created")


@pytest.mark.parametrize("rank,world,ids", [(2, 2, []), (0, 0, []), (0, 257, []), (1, 2, [0]), (0, 2, [1, 0]), (0, 2, [0, 0])])
def test_argument_errors_before_device_work(rank, world, ids):
    """A rank outside the world, a world outside 1..256, map ids outside the rank's block or not ascending."""
    from vega_b200 import dist as vdist
    maps = [(m, np.zeros(1, np.uint64), (np.zeros(1, np.uint64), np.zeros(1, np.int64))) for m in ids]
    with pytest.raises(ValueError):
        vdist.run_combine_shuffle(_NoDeviceEngine(), maps, 4, 3, 0, None, rank, world)
