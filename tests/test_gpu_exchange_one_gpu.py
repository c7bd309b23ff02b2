"""The library's own exchange (vb_ctx_comm_init + vb_shuffle_exchange) with two ranks on ONE GPU: two child processes
share device 0 and talk over NCCL's loopback socket transport.  NCCL refuses two ranks on one device within one host
id, so each child gets its own NCCL_HOSTID.  Every case (integer SUM, GROUP through NCCL and through the fused P2P
scatter, sort_by_key, a String-key SUM and a combine_by_key) compares the owners' partitions with the one-process
shuffle over the same map tasks, and the exchange stats with the rows that crossed.  If NCCL still refuses to
initialise, the test skips with NCCL's message."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
CASES = ("sum", "group_nccl", "group_p2p", "sort", "str_sum", "combine")
M, R, N = 5, 7, 60_000
TIMEOUT_S = 300


def _data():
    rng = np.random.default_rng(11)
    keys = rng.integers(0, 4000, N).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(5)
    vals = rng.integers(0, 1 << 64, N, dtype=np.uint64)
    i64 = rng.integers(-(1 << 62), 1 << 62, N).astype(np.int64)
    words = ["", "k\x00", "é-ключ"] + ["w%04d" % i for i in range(2000)] + ["L" * 700 + str(i) for i in range(5)]
    strs = [words[i] for i in rng.integers(0, len(words), N)]
    return keys, vals, i64, strs


def _run_case(sc, case, rank, world, stats):
    """One shuffle of `case` over the map tasks of `rank` (all of them for world 1) -> {partition: comparable value}."""
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    keys, vals, i64, strs = _data()
    starts = vb.slice_starts(N, M)
    lo, hi = vdist.map_block(rank, world, M)
    tasks = range(lo, hi)
    if case == "str_sum":
        maps = [(m, strs[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in tasks]
        sh = vdist.run_str_shuffle(vdist.StrCudaEngine(sc), maps, M, R, L.VB_U64, L.VB_AGG_SUM, rank, world, stats=stats)
        out = {r: dict(zip(*(lambda k, c: (list(k), c.tolist()))(*sh.reduce(r)[:2]))) for r in range(R)}
    elif case == "combine":
        multi = ([L.VB_U64, L.VB_I64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1)])
        maps = [(m, keys[starts[m]:starts[m + 1]], (vals[starts[m]:starts[m + 1]], i64[starts[m]:starts[m + 1]])) for m in tasks]
        eng = vdist.CombineCudaEngine(sc)
        sh = vdist.run_combine_shuffle(eng, maps, M, R, L.VB_U64, multi, rank, world, stats=stats)
        outs = [np.uint64, np.uint64, np.int64, np.int64]
        out = {}
        for r in range(R):
            k, cols = eng.reduce(sh, r, outs)
            out[r] = dict(zip(k.view(np.uint64).tolist(), zip(*[c.view(np.uint64).tolist() for c in cols])))
    else:
        agg = {"sum": L.VB_AGG_SUM, "group_nccl": L.VB_AGG_GROUP, "group_p2p": L.VB_AGG_GROUP, "sort": L.VB_AGG_SORT}[case]
        maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in tasks]
        sh = vdist.run_shuffle(vdist.CudaEngine(sc), maps, M, R, L.VB_U64, L.VB_U64, agg, rank, world, stats=stats,
                               p2p=case == "group_p2p")
        out = {}
        for r in range(R):
            p = [np.asarray(x) for x in sh.reduce(r)]
            if case == "sum":
                out[r] = dict(zip(p[0].view(np.uint64).tolist(), p[1].view(np.uint64).tolist()))
            elif case == "sort":
                out[r] = (p[0].view(np.uint64).tolist(), p[1].view(np.uint64).tolist())
            else:
                o = p[1].astype(np.int64)
                v = p[2].view(np.uint64).tolist()
                out[r] = {k: v[o[i]:o[i + 1]] for i, k in enumerate(p[0].view(np.uint64).tolist())}
    sh.free()
    return out


def _child(rank, outdir):
    """One rank: the NCCL unique id goes from rank 0 to rank 1 through a file in outdir."""
    sys.path.insert(0, ROOT)
    import vega_b200 as vb
    sc = vb.Context(0)
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
    res = {}
    for case in CASES:
        stats = {}
        res[case] = (_run_case(sc, case, rank, 2, stats), stats)
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sc.close()


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    """Both ranks' results, or a skip with NCCL's message.  A hard timeout kills both children."""
    d = str(tmp_path_factory.mktemp("exchange"))
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1", CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), d], cwd=ROOT, stdout=logs[r],
                              stderr=subprocess.STDOUT, env=dict(env, NCCL_HOSTID=f"vega-b200-rank{r}")) for r in range(2)]
    deadline = time.monotonic() + TIMEOUT_S
    try:
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            if any(p.poll() not in (None, 0) for p in procs):       # one rank failed: the other gets 10 s to finish
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
        pytest.skip("NCCL did not initialise two ranks on one GPU: " + open(refused[0]).read())
    assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
    return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(2)]


@pytest.fixture(scope="module")
def sc():
    import vega_b200 as vb
    with vb.Context(0) as c:
        yield c


@pytest.mark.parametrize("case", CASES)
def test_two_ranks_on_one_gpu_match_one_process(ranks, sc, case):
    want = _run_case(sc, case, 0, 1, {})
    for r in range(R):
        assert ranks[r % 2][case][0][r] == want[r], f"partition {r}"
        other = ranks[(r + 1) % 2][case][0][r]
        assert len(other if case != "sort" else other[0]) == 0, f"partition {r} on rank {(r + 1) % 2}"
    st = [ranks[q][case][1] for q in range(2)]
    print(f"\n{case} exchange stats: " + " | ".join(
        f"rank {q}: sent_rows={s['sent_rows']} recv_rows={s['recv_rows']} exchanges={s['exchanges']} kind={s['exchange_kind']}"
        for q, s in enumerate(st)))
    assert st[0]["sent_rows"] == st[1]["recv_rows"] and st[1]["sent_rows"] == st[0]["recv_rows"] > 0
    assert all(s["exchanges"] == 1 and s["exchange_kind"] == ("p2p" if case == "group_p2p" else "nccl") for s in st)


if __name__ == "__main__":
    _child(int(sys.argv[1]), sys.argv[2])
