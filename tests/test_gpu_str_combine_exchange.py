"""The library's exchange (vb_ctx_comm_init + vb_shuffle_exchange) of a String-key combine_by_key with two ranks: two
child processes on ONE GPU (each with its own NCCL_HOSTID, talking over NCCL's loopback socket transport, as
tests/test_gpu_exchange_one_gpu.py does), and on two GPUs when the machine has them.  The owners' partitions must equal
the one-process shuffle over the same map tasks, the exchange stats must count the keys that crossed, and ranks whose
specs differ must both return VB_ERR_INVALID, as must ranks whose single-column String reduce ops differ (they share
the combine's exchange).  If NCCL refuses to initialise two ranks on one GPU, that case skips with NCCL's message."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
M, R, N = 5, 7, 60_000
TIMEOUT_S = 300


def _multi(rank_spec=0):
    from vega_b200 import _lib as L
    aggs = [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_MEAN, 1)]
    if rank_spec:
        aggs[2] = (L.VB_AGG_MAX, 1)                    # a different op on one rank
    return [L.VB_U64, L.VB_I64], aggs


def _data():
    rng = np.random.default_rng(13)
    vals = rng.integers(0, 1 << 64, N, dtype=np.uint64)
    i64 = rng.integers(-(1 << 62), 1 << 62, N).astype(np.int64)
    words = ["", "k\x00", "é-ключ"] + ["w%04d" % i for i in range(2000)] + ["L" * 700 + str(i) for i in range(5)]
    strs = [words[i] for i in rng.integers(0, len(words), N)]
    return strs, vals, i64


def _run(sc, rank, world, stats, rank_spec=0):
    """The String combine over the map tasks of `rank` (all of them for world 1) -> {partition: {key: outputs}}."""
    import vega_b200 as vb
    from vega_b200 import dist as vdist
    strs, vals, i64 = _data()
    starts = vb.slice_starts(N, M)
    lo, hi = vdist.map_block(rank, world, M)
    maps = [(m, strs[starts[m]:starts[m + 1]], (vals[starts[m]:starts[m + 1]], i64[starts[m]:starts[m + 1]])) for m in range(lo, hi)]
    eng = vdist.StrCombineCudaEngine(sc)
    sh = vdist.run_str_combine_shuffle(eng, maps, M, R, _multi(rank_spec), rank, world, stats=stats)
    out = {}
    for r in range(R):
        ko, kb, cols = eng.reduce(sh, r, [np.uint64, np.uint64, np.int64, np.int64, np.float64])
        keys = vb.rdd._decode_keys(ko, kb).tolist()
        out[r] = dict(zip(keys, zip(*[c.view(np.uint64).tolist() for c in cols])))
    sh.free()
    return out


def _child(rank, outdir, device):
    sys.path.insert(0, ROOT)
    import vega_b200 as vb
    sc = vb.Context(device)
    idf = os.path.join(outdir, "uid")
    try:
        if rank == 0:
            with open(idf + ".tmp", "wb") as f:
                f.write(sc.comm_unique_id())
            os.replace(idf + ".tmp", idf)
        else:
            deadline = time.monotonic() + 60
            while not os.path.exists(idf) and time.monotonic() < deadline:
                time.sleep(0.05)
        with open(idf, "rb") as f:
            sc.comm_init(rank, 2, f.read())
    except (vb.VegaB200Error, OSError) as e:
        with open(os.path.join(outdir, f"init_failed{rank}"), "w") as f:
            f.write(str(e))
        sys.exit(3)
    stats = {}
    res = _run(sc, rank, 2, stats)
    try:                                               # the specs differ: every rank refuses before any send
        _run(sc, rank, 2, {}, rank_spec=rank)
        mismatch = None
    except vb.VegaB200Error as e:
        mismatch = e.code
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    strs, vals, _ = _data()
    starts = vb.slice_starts(N, M)
    lo, hi = vdist.map_block(rank, 2, M)
    maps = [(m, strs[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    try:                                               # a single-column reduce_by_key, SUM on rank 0 and MAX on rank 1
        vdist.run_str_shuffle(vdist.StrCudaEngine(sc), maps, M, R, L.VB_U64, (L.VB_AGG_SUM, L.VB_AGG_MAX)[rank], rank, 2).free()
        op_mismatch = None
    except vb.VegaB200Error as e:
        op_mismatch = e.code
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats, mismatch, op_mismatch), f)
    sc.close()


def _launch(d, devices, hostids):
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1")
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), d, str(devices[r])], cwd=ROOT, stdout=logs[r],
                              stderr=subprocess.STDOUT, env=dict(env, **({"NCCL_HOSTID": hostids[r]} if hostids else {})))
             for r in range(2)]
    deadline = time.monotonic() + TIMEOUT_S
    try:
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            if any(p.poll() not in (None, 0) for p in procs):
                deadline = min(deadline, time.monotonic() + 10)
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
    out = []
    for lg in logs:
        lg.seek(0)
        out.append(lg.read()[-3000:])
        lg.close()
    refused = [os.path.join(d, f"init_failed{r}") for r in range(2) if os.path.exists(os.path.join(d, f"init_failed{r}"))]
    if refused:
        pytest.skip("NCCL did not initialise two ranks: " + open(refused[0]).read())
    assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
    return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(2)]


def _check(ranks):
    import vega_b200 as vb
    from vega_b200 import _lib as L
    with vb.Context(0) as sc:
        want = _run(sc, 0, 1, {})
    for r in range(R):
        assert ranks[r % 2][0][r] == want[r], f"partition {r}"     # integer columns and the i64 MEAN: bit for bit
        assert len(ranks[(r + 1) % 2][0][r]) == 0, f"partition {r} on rank {(r + 1) % 2}"
    st = [ranks[q][1] for q in range(2)]
    assert st[0]["sent_rows"] == st[1]["recv_rows"] and st[1]["sent_rows"] == st[0]["recv_rows"] > 0
    # the keys that crossed: rank q's exported keys owned by the other rank
    assert all(s["exchanges"] == 1 and s["exchange_kind"] == "nccl" for s in st)
    assert [ranks[q][2] for q in range(2)] == [L.VB_ERR_INVALID, L.VB_ERR_INVALID]
    assert [ranks[q][3] for q in range(2)] == [L.VB_ERR_INVALID, L.VB_ERR_INVALID]     # reduce ops that differ


def test_two_ranks_on_one_gpu(tmp_path):
    _check(_launch(str(tmp_path), (0, 0), ("vega-b200-rank0", "vega-b200-rank1")))


def test_two_gpus(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("fewer than two GPUs")
    _check(_launch(str(tmp_path), (0, 1), None))


if __name__ == "__main__":
    _child(int(sys.argv[1]), sys.argv[2], int(sys.argv[3]))
