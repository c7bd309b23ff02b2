"""String keys on two ranks with the real StrCudaEngine (export by destination rank, import, seal), checked against
oracle/pyref.py.  With >= 2 GPUs each rank has its own GPU and the exchange is the library's (vb_ctx_comm_init +
vb_shuffle_exchange: one grouped NCCL send/recv of the four columns); on a one-GPU box both ranks share GPU 0 and the
columns are staged through gloo on the host (run_str_shuffle's all_to_all_v)."""
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

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_ROWS = 60_000


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dataset():
    rng = np.random.default_rng(31)
    words = ["", "the", "\x00", "é-ключ"] + ["w%05d" % i for i in range(3000)] + ["L" * 1200 + str(i) for i in range(10)]
    keys = [words[i] for i in rng.integers(0, len(words), N_ROWS)]
    vals = rng.integers(0, 1 << 64, N_ROWS, dtype=np.uint64)
    return keys, vals


def _worker(rank, world, port, op, M, R, nccl, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if nccl else 0
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{dev}"))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    keys, vals = _dataset()
    starts = vb.slice_starts(N_ROWS, M)
    lo, hi = vdist.map_block(rank, world, M)
    sc = vb.Context(dev)
    if nccl:
        sc.comm_init(rank, world)
    eng = vdist.StrCudaEngine(sc)
    agg = {"sum": L.VB_AGG_SUM, "count": L.VB_AGG_COUNT, "group": L.VB_AGG_GROUP}[op]
    maps = [(m, keys[starts[m]:starts[m + 1]], None if op == "count" else vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    stats = {}
    sh = vdist.run_str_shuffle(eng, maps, M, R, L.VB_U64, agg, rank, world, stats=stats,
                               exchange_device=None if nccl else "cpu")
    res = {}
    for r in range(R):
        out = sh.reduce(r)
        if r % world != rank:
            assert len(out[0]) == 0
        res[r] = [np.asarray(x) for x in out]
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats), f)
    sh.free()
    sc.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("op,M,R", [("count", 4, 4), ("sum", 5, 7), ("group", 4, 6), ("group", 1, 3)])
def test_two_rank_string_shuffle_matches_pyref(op, M, R):
    """M = 1: rank 0 has no map task and only receives."""
    from tests.test_gpu_str_keys import check_parts, ref_parts
    world = 2
    nccl = torch.cuda.device_count() >= 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), op, M, R, nccl, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset()
    got = []
    for r in range(R):
        out = per_rank[r % world][0][r]
        ks = out[0].tolist()
        if op == "group":
            o = out[1].astype(np.int64)
            got.append({k: out[2][o[i]:o[i + 1]].tolist() for i, k in enumerate(ks)})
        else:
            got.append(dict(zip(ks, out[1].tolist())))
    check_parts(got, ref_parts(keys, vals, op, "u64", M, R), op, "u64")
    sent = sum(s["sent_rows"] for _, s in per_rank)
    assert sent == sum(s["recv_rows"] for _, s in per_rank) and sent > 0
