"""sort_by_key over String keys across ranks (vb_shuffle_create_str_sort_dist + vb_shuffle_exchange).  Two and three
ranks run as child processes on ONE GPU over NCCL's loopback socket transport, each with its own NCCL_HOSTID (NCCL
refuses two ranks on one device within one host id); the NCCL id goes through a file.  Every owned partition must be
the one-process sort's (vb_shuffle_create_str_sort over the same map tasks) and tests/str_sort_ref.py's, key bytes and
payload bits row for row; the other ranks hold it empty.  Ranks that disagree, too many partitions and the P2P mode are
refused with the same code on every rank.  If NCCL refuses to initialise, the tests skip with NCCL's message.  One case
runs with one rank per GPU through mp.spawn and skips below two GPUs."""
import ctypes
import os
import pickle
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import str_sort_ref as SR  # noqa: E402

pytestmark = pytest.mark.gpu
TIMEOUT_S = 600
U64, I64, F64 = 0, 1, 2


def _cases():
    """name -> (keys as bytes in map-id order, payload array or None, vcode, M, R)"""
    rng = np.random.default_rng(21)
    words = [b"", b"k\x00", b"k", "é-ключ".encode(), b"\xff", b"\x00"] + [b"w%04d" % i for i in range(2000)] + \
        [b"L" * 700 + b"%d" % i for i in range(5)] + [b"L" * 700]
    n = 60_000
    mixed = [words[i] for i in rng.integers(0, len(words), n)]
    pos = np.arange(n, dtype=np.uint64)                               # payload = input position: checks stability
    f = rng.standard_normal(20_000)
    bits = f.view(np.uint64)
    bits[::7] = np.uint64(0x7FF8000000000000)
    bits[1::11] = np.uint64(0xFFF8000000000001)
    bits[2::13] = np.uint64(0x7FF0000000000123)
    f[3::17] = -0.0
    hot = [b"hot-key" if i < 8000 else words[int(j)] for i, j in zip(rng.permutation(20_000), rng.integers(0, 2000, 20_000))]
    nd = 200_000
    lens = rng.integers(2, 18, nd)
    raw = rng.integers(0, 256, int(lens.sum())).astype(np.uint8).tobytes()
    ends = np.cumsum(lens)
    distinct = list({raw[e - l:e]: None for e, l in zip(ends.tolist(), lens.tolist())})
    distinct = [distinct[i] for i in rng.permutation(len(distinct))]
    # 95 % of the rows share a 700-byte prefix: the cuts fall inside it and walk its 100 shared words on the device
    tails = [b"", b"\x00", b"\xff", b"\xff" * 9] + [b"%d" % i for i in range(300)]
    long_prefix = [b"P" * 700 + tails[int(i)] if r < 0.95 else words[int(i) % len(words)]
                   for i, r in zip(rng.integers(0, len(tails), 20_000), rng.random(20_000))]
    return {
        "mixed": (mixed, pos, U64, 5, 7),
        "prefix700": (long_prefix, pos[:20_000], U64, 4, 9),
        "f64": ([words[i] for i in rng.integers(0, len(words), 20_000)], f, F64, 4, 5),
        "key_only": (mixed[:30_000], None, None, 4, 6),
        "hot": (hot, np.arange(20_000, dtype=np.int64) - 7, I64, 6, 16),
        "single": ([b"same"] * 5000, np.arange(5000, dtype=np.uint64), U64, 3, 5),
        "distinct": (distinct, np.arange(len(distinct), dtype=np.uint64), U64, 6, 13),
        "r1": (mixed[:5000], pos[:5000], U64, 4, 1),
        "r_gt_n": (mixed[:20], pos[:20], U64, 4, 50),
        "m_lt_w": (mixed[:3000], pos[:3000], U64, 1, 4),
        "empty": ([], np.zeros(0, dtype=np.uint64), U64, 3, 4),
    }


def _col(keys):
    import vega_b200 as vb
    offs = np.zeros(len(keys) + 1, dtype=np.uint64)
    np.cumsum(np.fromiter((len(k) for k in keys), dtype=np.uint64, count=len(keys)), out=offs[1:])
    return vb.StrKeys(offs, np.frombuffer(b"".join(keys), dtype=np.uint8) if keys else np.zeros(0, dtype=np.uint8))


def _run(sc, name, case, rank, world, stats):
    """The shuffle of `case` over the map tasks of `rank` (all of them for world 1) -> [partition (keys, payload bits)]"""
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    keys, vals, vcode, M, R = case
    starts = [len(keys) * m // M for m in range(M + 1)]
    lo, hi = vdist.map_block(rank, world, M)
    maps = [(m, _col(keys[starts[m]:starts[m + 1]]), None if vals is None else vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    eng = vdist.StrCudaEngine(sc)
    sh = vdist.run_str_shuffle(eng, maps, M, R, vcode, L.VB_AGG_SORT, rank, world, stats=stats)
    out = []
    for r in range(R):
        ko, kb, v = eng.reduce(sh, r)
        ks = [kb[int(ko[i]):int(ko[i + 1])].tobytes() for i in range(len(ko) - 1)]
        out.append((ks, None if v is None else v.view(np.uint64).tolist()))
    sh.free()
    return out


def _errors(sc, rank, world):
    """Each refused exchange's return code on this rank."""
    from vega_b200 import _lib as L
    lib = sc._lib
    got = {}

    def attempt(name, vdt, R, mode=L.VB_XCHG_NCCL):
        h = ctypes.c_void_p()
        L.check(lib.vb_shuffle_create_str_sort_dist(sc._h, 900 + len(got), 2 * world, R, vdt, rank, world, ctypes.byref(h)))
        offs, data = np.array([0, 1, 3], dtype=np.uint64), np.frombuffer(b"abc", dtype=np.uint8)
        v = np.array([1, 2], dtype=np.uint64)
        for m in (2 * rank, 2 * rank + 1):
            L.check(lib.vb_shuffle_map_str(h, m, ctypes.c_void_p(offs.ctypes.data), ctypes.c_void_p(data.ctypes.data), 3,
                                           ctypes.c_void_p(v.ctypes.data) if vdt >= 0 else None, 2, L.VB_HOST))
        got[name] = lib.vb_shuffle_exchange(h, mode)
        lib.vb_shuffle_free(h)

    attempt("val_dtype", U64 if rank == 0 else I64, 4)
    attempt("key_only_vs_payload", U64 if rank == 0 else -1, 4)
    attempt("n_reduce", U64, 4 if rank == 0 else 5)
    attempt("n_reduce_4097", U64, 4097)
    attempt("p2p", U64, 4, L.VB_XCHG_P2P)
    return got


def _child(rank, world, outdir):
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
            sc.comm_init(rank, world, f.read())
    except (vb.VegaB200Error, OSError) as e:
        with open(os.path.join(outdir, f"init_failed{rank}"), "w") as f:
            f.write(str(e))
        sys.exit(3)
    res = {}
    for name, case in _cases().items():
        stats = {}
        res[name] = (_run(sc, name, case, rank, world, stats), stats)
    res["errors"] = _errors(sc, rank, world)
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sc.close()


def _launch(world):
    """Every rank's results, or a skip with NCCL's message.  A hard timeout kills every child."""
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1",
                   CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
        logs = [open(os.path.join(d, f"log{r}"), "w+") for r in range(world)]
        procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), str(world), d], cwd=ROOT, stdout=logs[r],
                                  stderr=subprocess.STDOUT, env=dict(env, NCCL_HOSTID=f"vega-b200-rank{r}")) for r in range(world)]
        deadline = time.monotonic() + TIMEOUT_S
        try:
            while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
                if any(p.poll() not in (None, 0) for p in procs):       # one rank failed: the others get 10 s to finish
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
        refused = [os.path.join(d, f"init_failed{r}") for r in range(world) if os.path.exists(os.path.join(d, f"init_failed{r}"))]
        if refused:
            pytest.skip("NCCL did not initialise the ranks on one GPU: " + open(refused[0]).read())
        assert all(p.returncode == 0 for p in procs), f"exit codes {[p.returncode for p in procs]}\n" + "\n----\n".join(out)
        return [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]


_RESULTS = {}


def _ranks(world):
    if world not in _RESULTS:
        _RESULTS[world] = _launch(world)
    return _RESULTS[world]


@pytest.fixture(scope="module")
def sc():
    import vega_b200 as vb
    with vb.Context(0) as c:
        yield c


@pytest.fixture(scope="module")
def cases():
    return _cases()


def _reference(case):
    keys, vals, vcode, M, R = case
    want = SR.partitions(keys, vals, R)
    return [(k, None if v is None else np.asarray(v).view(np.uint64).tolist()) for k, v in want]


@pytest.mark.parametrize("name", ["mixed", "prefix700", "f64", "key_only", "hot", "single", "distinct", "r1", "r_gt_n", "m_lt_w", "empty"])
@pytest.mark.parametrize("world", [2, 3])
def test_ranks_on_one_gpu_match_one_process(sc, cases, world, name):
    from vega_b200 import dist as vdist
    ranks = _ranks(world)
    case = cases[name]
    R = case[4]
    one = _run(sc, name, case, 0, 1, {})
    ref = _reference(case)
    for r in range(R):
        assert one[r] == ref[r], f"one-process partition {r}"
        assert ranks[r % world][name][0][r] == one[r], f"partition {r}"
        for q in range(world):
            if q != r % world:
                assert ranks[q][name][0][r] == ([], None if case[1] is None else []), f"partition {r} on rank {q}"
    st = [ranks[q][name][1] for q in range(world)]
    assert all(s["exchanges"] == 1 and s["exchange_kind"] == "nccl" for s in st)
    assert sum(s["sent_rows"] for s in st) == sum(s["recv_rows"] for s in st)
    if name == "prefix700":
        # the restatement over the same local keys: the agreement walks the shared prefix word by word
        from tests import str_sort_dist_ref as DR
        keys, M = case[0], case[3]
        starts = [len(keys) * m // M for m in range(M + 1)]
        blocks = [keys[starts[vdist.map_block(q, world, M)[0]]:starts[vdist.map_block(q, world, M)[1]]] for q in range(world)]
        trace = DR.agree_cuts([DR.Rank(b) for b in blocks], R)[1]
        assert max(len(cut) for cut in trace["words"]) > 100
        assert sum(1 for cut in trace["words"] if len(cut) > 100) >= R // 2
    if name in ("mixed", "distinct"):
        assert all(s["recv_rows"] > 0 for s in st)
        print(f"\n{name} W={world}: " + " | ".join(f"rank {q}: prepare {s['prepare_wall_ms']:.1f} ms, counts {s['counts_wall_ms']:.1f} ms, "
                                                   f"post {s['post_wall_ms']:.1f} ms" for q, s in enumerate(st)))


@pytest.mark.parametrize("world", [2, 3])
def test_refusals_are_the_same_on_every_rank(world):
    from vega_b200 import _lib as L
    ranks = _ranks(world)
    want = {"val_dtype": L.VB_ERR_INVALID, "key_only_vs_payload": L.VB_ERR_INVALID, "n_reduce": L.VB_ERR_INVALID,
            "n_reduce_4097": L.VB_ERR_UNSUPPORTED, "p2p": L.VB_ERR_UNSUPPORTED}
    for q in range(world):
        assert ranks[q]["errors"] == want, f"rank {q}"


def test_calls_refused_without_a_communicator(sc):
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    lib = sc._lib
    inv, uns, state = L.VB_ERR_INVALID, L.VB_ERR_UNSUPPORTED, L.VB_ERR_STATE
    h = ctypes.c_void_p()
    assert lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 2, 3, U64, 2, 2, ctypes.byref(h)) == inv          # rank >= world
    assert lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 2, 3, U64, 0, 257, ctypes.byref(h)) == inv        # world > 256
    assert lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 2, 3, 7, 0, 2, ctypes.byref(h)) == inv            # val_dtype
    assert lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 2, 0, U64, 0, 2, ctypes.byref(h)) == inv          # n_reduce 0
    L.check(lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 2, 3, U64, 0, 2, ctypes.byref(h)))
    offs, data = np.array([0, 1, 2], dtype=np.uint64), np.frombuffer(b"ba", dtype=np.uint8)
    v = np.array([1, 2], dtype=np.uint64)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)
    L.check(lib.vb_shuffle_map_str(h, 0, p(offs), p(data), 2, p(v), 2, L.VB_HOST))
    u = ctypes.c_uint64()
    n3 = (ctypes.c_uint64 * 2)()
    assert lib.vb_shuffle_export_str_prepare(h, ctypes.byref(u), ctypes.byref(u), ctypes.byref(u)) == uns
    assert lib.vb_shuffle_export_str_buffers(h, None, None, None, None) == uns
    assert lib.vb_shuffle_import_str(h, None, None, None, None, n3, n3, n3) == uns
    assert lib.vb_shuffle_export_str_cols_prepare(h, ctypes.byref(u), ctypes.byref(u)) == uns
    assert lib.vb_shuffle_export_str_cols_buffers(h, None, None, None, None) == uns
    assert lib.vb_shuffle_import_str_cols(h, None, None, None, 1, n3, n3) == uns
    assert lib.vb_shuffle_set_dist(h, 0, 2) == uns
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_P2P) == uns
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_NCCL) == state                                            # no communicator
    assert lib.vb_shuffle_seal(h) == state                                                                # no exchange
    lib.vb_shuffle_free(h)
    # world 1 is the one-process shuffle
    L.check(lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 1, 2, -1, 0, 1, ctypes.byref(h)))
    L.check(lib.vb_shuffle_map_str(h, 0, p(offs), p(data), 2, None, 2, L.VB_HOST))
    L.check(lib.vb_shuffle_seal(h))
    assert lib.vb_shuffle_reduce_str_size(h, 0, ctypes.byref(u), None, None) == 0 and u.value == 1
    lib.vb_shuffle_free(h)
    # the Python path without the library's communicator says what it needs
    with pytest.raises(ValueError, match="vb_ctx_comm_init"):
        vdist.run_str_shuffle(vdist.StrCudaEngine(sc), [(0, ["a"], None)], 2, 2, None, L.VB_AGG_SORT, 0, 2)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _spawn_worker(rank, world, port, outdir):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    import vega_b200 as vb
    sc = vb.Context(rank)
    sc.comm_init(rank, world)
    res = {n: _run(sc, n, c, rank, world, {}) for n, c in _cases().items() if n in ("mixed", "key_only", "hot")}
    with open(os.path.join(outdir, f"s{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sc.close()
    dist.destroy_process_group()


def test_two_gpus_one_rank_each(cases):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("one rank per GPU needs >= 2 GPUs")
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_spawn_worker, args=(world, _free_port(), d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"s{r}.pkl"), "rb")) for r in range(world)]
    for name in ("mixed", "key_only", "hot"):
        ref = _reference(cases[name])
        for r in range(cases[name][4]):
            assert per_rank[r % world][name][r] == ref[r], f"{name} partition {r}"


if __name__ == "__main__":
    _child(int(sys.argv[1]), int(sys.argv[2]), sys.argv[3])
