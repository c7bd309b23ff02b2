"""The library's own exchange (vb_ctx_comm_init + vb_shuffle_exchange) of byte-string values with two ranks on ONE GPU:
two child processes share device 0 and talk over NCCL's loopback socket transport, each with its own NCCL_HOSTID (NCCL
refuses two ranks on one device within one host id).  Every case (integer GROUP, String GROUP, integer sort_by_key and
String sort_by_key with a byte-string payload) compares the owners' partitions, values gathered through the owning
rank's shuffle, with the one-process shuffle over the same map tasks, and checks that VB_XCHG_AUTO ran NCCL with the
rows that crossed.  If NCCL refuses to initialise, the test skips with NCCL's message."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
CASES = ("group", "str_group", "sort", "str_sort")
M, R, N = 5, 7, 30_000
TIMEOUT_S = 300


def _data():
    rng = np.random.default_rng(12)
    keys = rng.integers(0, 3000, N).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(5)
    words = ["", "k\x00", "é-ключ"] + ["w%04d" % i for i in range(1500)] + ["L" * 500 + str(i) for i in range(5)]
    strs = [words[i] for i in rng.integers(0, len(words), N)]
    lens = rng.integers(0, 65, N)
    lens[rng.random(N) < 0.01] = 4096
    lens[::101] = 0
    raw = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
    o = np.concatenate([[0], np.cumsum(lens)])
    return keys, strs, [raw[o[i]:o[i + 1]] for i in range(N)]


def _run_case(sc, case, rank, world, stats):
    """One shuffle of `case` over the map tasks of `rank` (all of them for world 1) -> {partition: comparable value}."""
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    keys, strs, vals = _data()
    starts = vb.slice_starts(N, M)
    lo, hi = vdist.map_block(rank, world, M)
    agg = L.VB_AGG_SORT if case.endswith("sort") else L.VB_AGG_GROUP
    out = {}
    if case.startswith("str"):
        maps = [(m, strs[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        eng = vdist.StrBytesCudaEngine(sc)
        sh = vdist.run_str_shuffle(eng, maps, M, R, L.VB_BYTES, agg, rank, world, stats=stats)
        sh.as_str = False
        for r in range(R):
            p = eng.reduce(sh, r)
            ko, kb = p[0].astype(np.int64), bytes(p[1])
            ks = [kb[ko[i]:ko[i + 1]] for i in range(len(ko) - 1)]
            if agg == L.VB_AGG_SORT:
                out[r] = list(zip(ks, p[2]))
            else:
                o = p[2].astype(np.int64)
                out[r] = {k: list(p[3][o[i]:o[i + 1]]) for i, k in enumerate(ks)}
    else:
        maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        eng = vdist.BytesCudaEngine(sc)
        sh = vdist.run_shuffle(eng, maps, M, R, L.VB_U64, L.VB_BYTES, agg, rank, world, stats=stats)
        sh.as_str = False
        for r in range(R):
            p = eng.reduce(sh, r)
            k = np.asarray(p[0]).view(np.uint64).tolist()
            if agg == L.VB_AGG_SORT:
                out[r] = list(zip(k, p[1]))
            else:
                o = np.asarray(p[1]).astype(np.int64)
                out[r] = {kk: list(p[2][o[i]:o[i + 1]]) for i, kk in enumerate(k)}
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
    d = str(tmp_path_factory.mktemp("bytes_exchange"))
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1", CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), d], cwd=ROOT, stdout=logs[r],
                              stderr=subprocess.STDOUT, env=dict(env, NCCL_HOSTID=f"vega-b200-bytes-rank{r}")) for r in range(2)]
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
        assert len(ranks[(r + 1) % 2][case][0][r]) == 0, f"partition {r} on rank {(r + 1) % 2}"
    st = [ranks[q][case][1] for q in range(2)]
    print(f"\n{case} exchange stats: " + " | ".join(
        f"rank {q}: sent_rows={s['sent_rows']} recv_rows={s['recv_rows']} exchanges={s['exchanges']} kind={s['exchange_kind']}"
        for q, s in enumerate(st)))
    assert st[0]["sent_rows"] == st[1]["recv_rows"] and st[1]["sent_rows"] == st[0]["recv_rows"] > 0
    assert all(s["exchanges"] == 1 and s["exchange_kind"] == "nccl" for s in st)


if __name__ == "__main__":
    _child(int(sys.argv[1]), sys.argv[2])
