"""repartition across ranks through the library's own NCCL exchange (vb_ctx_comm_init + vb_shuffle_exchange): two
child processes, one per rank, either both on GPU 0 (each with its own NCCL_HOSTID, over NCCL's loopback socket
transport) or on GPUs 0 and 1 (skipped below two GPUs).  Each rank maps its contiguous block of map ids; every partition
it owns must equal the one-process result exactly, in order, and every partition it does not own must be empty.  Ranks
that disagree on n_cols or has_bytes both get VB_ERR_INVALID before any send, and both shuffles can be freed.  If NCCL
refuses to initialise, the test skips with NCCL's message."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
M, N = 7, 20_000
CASES = [("u2", 5), ("u2", 300), ("b", 5), ("b", 300), ("u1b", 5), ("u1b", 300)]
SHAPES = {"u2": (2, False), "b": (0, True), "u1b": (1, True)}
TIMEOUT_S = 300


def _data():
    rng = np.random.default_rng(21)
    a = rng.integers(0, 1 << 62, N).astype(np.uint64)
    b = rng.integers(0, 1 << 62, N).astype(np.uint64)
    lens = rng.integers(0, 21, N)
    lens[::97] = 0
    raw = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
    o = np.concatenate([[0], np.cumsum(lens)])
    items = [raw[o[i]:o[i + 1]] for i in range(N)]
    starts = [int(x) for x in rng.integers(0, 1 << 63, M)]
    starts[2] = (1 << 64) - 3
    return a, b, items, starts


def _run_case(sc, shape, R, rank, world):
    """One repartition of `shape` over the map tasks of `rank` (all of them for world 1) -> per partition (cols, items)."""
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200.rdd import RepShuffle, StrKeys, _BytesCol, _Col
    a, b, items, starts = _data()
    n_cols, has_bytes = SHAPES[shape]
    bounds = [int(x) for x in vb.slice_starts(N, M)]
    cols = [_Col(a, role="value"), _Col(b, role="value")][:n_cols]
    bcol = None
    if has_bytes:
        offs = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.uint64)
        bcol = _BytesCol(StrKeys(offs, np.frombuffer(b"".join(items), dtype=np.uint8)))
        bcol.as_str = False
    sh = RepShuffle(sc, M, R, [L.VB_U64] * n_cols, has_bytes, as_str=False, rank=rank, world=world)
    for m in range((rank * M) // world, ((rank + 1) * M) // world):
        sh.map_items(m, starts[m], cols, bcol, bounds[m], bounds[m + 1])
    if world > 1:
        sh.exchange(L.VB_XCHG_AUTO)
    sh.seal()
    out = {}
    for r in range(R):
        c, it = sh.reduce(r)
        out[r] = ([x.tolist() for x in c], list(it) if it is not None else None)
    st = sh.exchange_stats() if world > 1 else None
    sh.free()
    return out, st


def _rdd_case(sc):
    a, _, _, starts = _data()
    return [p.tolist() for p in sc.parallelize(a, M).repartition(11, starts=starts).glom()]


def _child(rank, outdir, two_gpus):
    sys.path.insert(0, ROOT)
    import ctypes

    import vega_b200 as vb
    from vega_b200 import _lib as L
    sc = vb.Context(rank if two_gpus else 0)
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
    res = {case: _run_case(sc, case[0], case[1], rank, 2) for case in CASES}
    res["rdd"] = _rdd_case(sc)
    # disagreement: rank 0 has one column, rank 1 two (and bytes): every rank refuses before any send
    lib, codes = L.lib(), []
    for pair in (((1, 0), (2, 0)), ((1, 0), (1, 1))):
        n_cols, hb = pair[rank]
        h = ctypes.c_void_p()
        L.check(lib.vb_shuffle_create_repartition_dist(sc._h, 99, 2, 4, n_cols, hb, rank, 2, ctypes.byref(h)))
        x = np.arange(10, dtype=np.uint64)
        ptrs = (ctypes.c_void_p * 2)(x.ctypes.data, x.ctypes.data)
        offs = np.arange(11, dtype=np.uint64)
        L.check(lib.vb_shuffle_map_repartition(h, rank, 5, ptrs, offs.ctypes.data, x.ctypes.data, 10, 10, L.VB_HOST))
        codes.append(lib.vb_shuffle_exchange(h, L.VB_XCHG_NCCL))
        codes.append(lib.vb_shuffle_free(h))
    res["disagree"] = codes
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sc.close()


def _spawn(tmp_path_factory, two_gpus):
    d = str(tmp_path_factory.mktemp("rep_dist2" if two_gpus else "rep_dist1"))
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1")
    if not two_gpus:
        env["CUDA_VISIBLE_DEVICES"] = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
    logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(2)]
    procs = []
    for r in range(2):
        e = dict(env, NCCL_HOSTID=f"vega-b200-rep-rank{r}") if not two_gpus else env
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), d, "1" if two_gpus else "0"], cwd=ROOT,
                                      stdout=logs[r], stderr=subprocess.STDOUT, env=e))
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
        pytest.skip("NCCL did not initialise two ranks: " + open(refused[0]).read())
    assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
    return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(2)]


@pytest.fixture(scope="module")
def one_gpu(tmp_path_factory):
    return _spawn(tmp_path_factory, False)


@pytest.fixture(scope="module")
def two_gpus(tmp_path_factory):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    return _spawn(tmp_path_factory, True)


@pytest.fixture(scope="module")
def sc():
    import vega_b200 as vb
    with vb.Context(0) as c:
        yield c


def _check(ranks, sc):
    from vega_b200 import _lib as L
    for case in CASES:
        want, _ = _run_case(sc, case[0], case[1], 0, 1)
        R = case[1]
        for r in range(R):
            assert ranks[r % 2][case][0][r] == want[r], f"{case} partition {r}"
            assert len(ranks[(r + 1) % 2][case][0][r][0][0] if SHAPES[case[0]][0] else ranks[(r + 1) % 2][case][0][r][1]) == 0
        st = [ranks[q][case][1] for q in range(2)]
        assert st[0]["sent_rows"] == st[1]["recv_rows"] > 0 and st[1]["sent_rows"] == st[0]["recv_rows"] > 0
        assert all(s["exchanges"] == 1 and s["exchange_kind"] == "nccl" for s in st)
    want = [p.tolist() for p in sc.parallelize(_data()[0], M).repartition(11, starts=_data()[3]).glom()]
    for r in range(11):
        assert ranks[r % 2]["rdd"][r] == want[r] and ranks[(r + 1) % 2]["rdd"][r] == []
    for q in range(2):
        assert ranks[q]["disagree"] == [L.VB_ERR_INVALID, L.VB_OK, L.VB_ERR_INVALID, L.VB_OK]


def test_two_ranks_on_one_gpu(one_gpu, sc):
    _check(one_gpu, sc)


def test_two_gpus(two_gpus, sc):
    _check(two_gpus, sc)


if __name__ == "__main__":
    _child(int(sys.argv[1]), sys.argv[2], sys.argv[3] == "1")
