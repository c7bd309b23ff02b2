"""sort_by_key over String keys across ranks (DESIGN.md §5.8): two ranks as two processes on ONE GPU.

The exchange runs over NCCL's loopback socket transport (each process has its own NCCL_HOSTID), so the post time says
nothing about NVLink; the cut agreement's rounds are host round trips of the same kind.  `rows` rows (default 5e7)
with i64 payloads, 8 map slices -> 8 partitions, rank r maps slices map_block(r, 2, 8).  Key sets as in §5.7
(tools/bench_str_sort.py): uniform 1e4 / uniform 1e6 word-like keys, all distinct, and URL keys with a 32-byte shared
prefix.  Per key set and rank, one JSON line:
  prepare_ms / counts_ms / post_ms   vb_shuffle_exchange_stats: the local sort, the all-gathers with the cut
                                      agreement, the grouped send/recv (median of 3 after a warm-up);
  seal_ms                             the owner's seal: re-encode and re-sort of the received rows;
  total_ms                            first map call to the end of the seal;
  rounds                              the agreement's all-gathers from tests/str_sort_dist_ref.py over the same local
                                      keys (all distinct: over the first `ROUND_ROWS` rows only, see `rounds_rows`);
  one_process_ms                      the one-process String sort of all rows on this GPU;
  int_rank_sort_w2_ms                 the W = 2 integer sort of the keys' ranks through the same communicator;
  identical                           the owned partitions equal the one-process result (keys and payload bits).
The card name and power limit are read in the same process; nothing is written outside a temporary directory.
    python tools/bench_str_sort_dist.py [rows=5e7]
"""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
W, M, R = 2, 8, 8
ROUND_ROWS = 2_000_000
KEY_SETS = [("uniform 1e4", "uniform", 10_000), ("uniform 1e6", "uniform", 1_000_000), ("all distinct", "unique", 0),
            ("url, 32-byte shared prefix", "uniform", 1_000_000)]


def _keys(sc, name, mode, D, n):
    import torch
    from bench_str_sort import url_keys            # the §5.7 URL keys, so both key sets stay the same
    from tests.test_gpu_str_keys import _device_words
    ranks = torch.empty(n, dtype=torch.int64, device="cuda")
    vals = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, out_vals=vals, n=n, mode=mode, n_distinct=max(D, 1), seed_k=5)
    ranks &= (1 << 63) - 1 if mode == "unique" else (1 << 28) - 1
    return ranks, vals, (url_keys(ranks) if name.startswith("url") else _device_words(ranks))


def _rounds(keys_of, ranks, rank_rows):
    """The agreement's rounds from the restatement, every rank's distinct local keys taken from its rows."""
    import torch
    from tests import str_sort_dist_ref as DR
    rk = []
    for lo, hi in rank_rows:
        u, cnt = torch.unique(ranks[lo:hi], return_counts=True)
        ks = keys_of(u)
        offs, data = ks.offsets.cpu().numpy(), ks.data.cpu().numpy().tobytes()
        pairs = sorted(zip((data[offs[i]:offs[i + 1]] for i in range(len(u))), cnt.cpu().tolist()))
        r = DR.Rank([])
        r.keys = [k for k, _ in pairs]
        r.row_off = [0]
        for _, c in pairs:
            r.row_off.append(r.row_off[-1] + c)
        rk.append(r)
    return DR.agree_cuts(rk, R)[1]["rounds"]


def _child(rank, outdir, n):
    import torch
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    from vega_b200.rdd import Shuffle, StrShuffle, _Col, _StrCol
    from bench_str_sort import url_keys
    from tests.test_gpu_str_keys import _device_words
    sc = vb.Context(0)
    idf = os.path.join(outdir, "uid")
    if rank == 0:
        with open(idf + ".tmp", "wb") as f:
            f.write(sc.comm_unique_id())
        os.replace(idf + ".tmp", idf)
    else:
        while not os.path.exists(idf):
            time.sleep(0.05)
    with open(idf, "rb") as f:
        sc.comm_init(rank, W, f.read())
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    starts = vb.slice_starts(n, M)
    lo, hi = vdist.map_block(rank, W, M)

    def timed(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, r

    def dist_sort(K, V):
        sh = StrShuffle(sc, M, R, L.VB_I64, L.VB_AGG_SORT, rank=rank, world=W, sort=True)
        for m in range(lo, hi):
            sh.map(m, K, V, int(starts[m]), int(starts[m + 1]))
        sh.exchange(L.VB_XCHG_NCCL)
        t_seal = timed(sh.seal)[0]
        return sh, t_seal

    def one_sort(K, V):
        sh = StrShuffle(sc, M, R, L.VB_I64, L.VB_AGG_SORT, sort=True)
        for m in range(M):
            sh.map(m, K, V, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        return sh

    def int_sort(ranks, V):
        k = _Col(ranks)
        k.code = L.VB_U64
        sh = Shuffle(sc, M, R, L.VB_U64, L.VB_I64, L.VB_AGG_SORT, rank=rank, world=W)
        for m in range(lo, hi):
            sh.map(m, k, V, int(starts[m]), int(starts[m + 1]))
        sh.exchange(L.VB_XCHG_NCCL)
        sh.seal()
        sh.free()

    def device_part(sh, r):
        nk, nb, _ = sh.reduce_size(r)
        ko = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        kb = torch.empty(nb, dtype=torch.uint8, device="cuda")
        v = torch.empty(nk, dtype=torch.int64, device="cuda")
        sh.reduce_device(r, out_key_offsets=ko, out_key_bytes=kb, out_comb=v)
        torch.cuda.synchronize()
        return ko, kb, v

    for ki, (name, mode, D) in enumerate(KEY_SETS):
        # the ranks build their keys in turn: the builder's temporaries of two processes at once do not fit one GPU
        turn = lambda q: os.path.join(outdir, f"built{ki}_{q}")
        while rank and not os.path.exists(turn(rank - 1)):
            time.sleep(0.05)
        ranks, vals, keys = _keys(sc, name, mode, D, n)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        open(turn(rank), "w").close()
        K, V = _StrCol(keys), _Col(vals, role="value")
        runs = []
        for i in range(4):
            t, (sh, t_seal) = timed(lambda: dist_sort(K, V))
            st = sh.exchange_stats()
            if i == 3:
                one = one_sort(K, V)
                same = True
                for r in range(rank, R, W):
                    a, b = device_part(sh, r), device_part(one, r)
                    same &= all(torch.equal(x, y) for x, y in zip(a, b))
                one.free()
            sh.free()
            if i:
                runs.append((t, t_seal, st))
        med = lambda f: round(statistics.median(f(x) for x in runs), 2)
        case = {"keys": name, "rank": rank, "world": W, "rows": n, "rows_this_rank": int(starts[hi] - starts[lo]),
                "gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "transport": "NCCL sockets over loopback, one GPU",
                "prepare_ms": med(lambda x: x[2]["prepare_wall_ms"]), "counts_ms": med(lambda x: x[2]["counts_wall_ms"]),
                "post_ms": med(lambda x: x[2]["post_wall_ms"]), "seal_ms": med(lambda x: x[1]), "total_ms": med(lambda x: x[0]),
                "sent_rows": runs[-1][2]["sent_rows"], "recv_rows": runs[-1][2]["recv_rows"], "identical": bool(same)}
        timed(lambda: one_sort(K, V).free())
        case["one_process_ms"] = round(statistics.median(timed(lambda: one_sort(K, V).free())[0] for _ in range(3)), 2)
        timed(lambda: int_sort(ranks, V))
        case["int_rank_sort_w2_ms"] = round(statistics.median(timed(lambda: int_sort(ranks, V))[0] for _ in range(3)), 2)
        if rank == 0:
            keys_of = url_keys if name.startswith("url") else _device_words
            rn = n if mode != "unique" else min(n, ROUND_ROWS)
            rs = vb.slice_starts(rn, M)
            bounds = [(int(rs[vdist.map_block(q, W, M)[0]]), int(rs[vdist.map_block(q, W, M)[1]])) for q in range(W)]
            case["rounds"] = _rounds(keys_of, ranks[:rn], bounds)
            case["rounds_rows"] = rn
        print(json.dumps(case), flush=True)
        del ranks, vals, keys, K, V
        torch.cuda.empty_cache()
    sc.close()


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", NCCL_IB_DISABLE="1", PYTHONPATH=ROOT,
                   CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
        procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "--child", str(r), d, str(n)], cwd=ROOT,
                                  env=dict(env, NCCL_HOSTID=f"vega-b200-bench{r}")) for r in range(W)]
        try:
            deadline = time.monotonic() + 1800
            while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
                if any(p.poll() not in (None, 0) for p in procs):
                    deadline = min(deadline, time.monotonic() + 10)
                time.sleep(0.5)
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
            for p in procs:
                p.wait()
    sys.exit(max(abs(p.returncode) for p in procs))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        _child(int(sys.argv[2]), sys.argv[3], int(sys.argv[4]))
    else:
        main()
