"""combine_by_key on two ranks with the real CombineCudaEngine (export by destination rank, import, seal), checked
against the CPU oracle's single-column references (tests/test_gpu_combine.py:check_combine).  With >= 2 GPUs each rank
has its own GPU and the exchange is the library's (vb_ctx_comm_init + vb_shuffle_exchange: one grouped NCCL send/recv
of the key and accumulator columns); on a one-GPU box both ranks share GPU 0 and the columns are staged through gloo on
the host (run_combine_shuffle's all_to_all_v)."""
import os
import pickle
import socket
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_ROWS = 120_000


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _multi(spec):
    """A spec of tests/test_gpu_combine.py; "reversed": "four"'s aggregates in reverse order (same columns, same n_acc)."""
    from tests.test_gpu_combine import AGG, CODE, SPECS
    dts, aggs = SPECS["four" if spec == "reversed" else spec]
    if spec == "reversed":
        aggs = aggs[::-1]
    return [CODE[d] for d, _ in dts], [(AGG[o], c) for o, c in aggs]


def _worker(rank, world, port, spec, M, R, nccl, outdir, spec_of_rank1=None):
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
    from tests.test_gpu_combine import SPECS, make_data, out_dtype
    keys, cols = make_data(41, spec, N_ROWS, 20_000)
    starts = vb.slice_starts(N_ROWS, M)
    lo, hi = vdist.map_block(rank, world, M)
    sc = vb.Context(dev)
    if nccl:
        sc.comm_init(rank, world)
    eng = vdist.CombineCudaEngine(sc)
    my_spec = spec_of_rank1 if (rank == 1 and spec_of_rank1) else spec
    maps = [(m, keys[starts[m]:starts[m + 1]], tuple(c[starts[m]:starts[m + 1]] for c in cols)) for m in range(lo, hi)]
    stats, res, code = {}, {}, L.VB_OK
    try:
        sh = vdist.run_combine_shuffle(eng, maps, M, R, L.VB_U64, _multi(my_spec), rank, world, stats=stats,
                                       exchange_device=None if nccl else "cpu")
    except vb.VegaB200Error as e:
        code = e.code
    else:
        outs = [out_dtype(spec, a) for a in range(len(SPECS[spec][1]))]
        for r in range(R):
            k, o = eng.reduce(sh, r, outs)
            if r % world != rank:
                assert len(k) == 0
            res[r] = (k, o)
        sh.free()
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats, code), f)
    sc.close()
    dist.destroy_process_group()


def _run(spec, M, R, nccl, spec_of_rank1=None):
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), spec, M, R, nccl, d, spec_of_rank1), nprocs=world, join=True)
        return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]


@pytest.mark.parametrize("spec,M,R", [("four", 4, 5), ("mixed", 5, 7), ("one", 1, 3)])
def test_two_rank_combine_matches_oracle(spec, M, R):
    """M = 1: rank 0 has no map task and only receives."""
    from tests.test_gpu_combine import check_combine, make_data
    per_rank = _run(spec, M, R, torch.cuda.device_count() >= 2)
    assert all(code == 0 for _, _, code in per_rank)
    keys, cols = make_data(41, spec, N_ROWS, 20_000)
    check_combine([per_rank[r % 2][0][r] for r in range(R)], spec, keys, cols, R)
    sent = sum(s["sent_rows"] for _, s, _ in per_rank)
    assert sent == sum(s["recv_rows"] for _, s, _ in per_rank) and sent > 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the library's NCCL exchange needs two GPUs")
def test_mismatched_specs_fail_on_every_rank():
    """Rank 1 aggregates the same columns with another spec: both ranks return VB_ERR_INVALID from the exchange, and
    neither waits in the send/recv group."""
    from vega_b200 import _lib as L
    per_rank = _run("four", 4, 5, True, spec_of_rank1="reversed")
    assert [code for _, _, code in per_rank] == [L.VB_ERR_INVALID, L.VB_ERR_INVALID]
