"""Bincode blobs of a String-key count_by_key (DESIGN.md §5.12): the encode of every reduce partition to a device buffer
against a device-to-device cudaMemcpy of the same bytes, and the decode of CPU-encoded blobs from pinned host memory.

Workload: a word count, 5e7 rows over about 1e6 distinct words of 1 to 20 bytes (a bijective base-26 stem, which
makes every word distinct, padded with digits to a length drawn per word), uniform, 8 map tasks and 8 partitions.  The
blobs hold the ~1e6 combined (word, count) records.  Encode: vb_shuffle_reduce_blob of all 8 partitions (each call ends
in a synchronise), host clock over the loop, and the device time of the encode kernel from the shuffle's K_MISC
counter.  Copy: the same 8 byte counts copied device to device, each copy followed by a synchronise, host clock.  Decode:
vb_shuffle_map_blob of the 8 blobs (encoded by tests/str_blob_ref.py on the host) from pinned host memory into a fresh
shuffle, host clock, seal excluded.  Medians of 5 runs after a warm-up.  The card's name and power limit are read in the
same process.  Prints one JSON line; writes nothing.
    python tools/bench_str_blob.py [rows=5e7] [distinct=1e6]
"""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from tests import str_blob_ref as B  # noqa: E402

REPS = 5


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def dictionary(D, rng):
    """D distinct words of 1 to 20 bytes: bijective base-26 stem of i (letters) + digits up to a drawn length."""
    words = []
    want = rng.integers(1, 21, D)
    for i in range(D):
        x, s = i + 1, []
        while x:
            x -= 1
            s.append(97 + x % 26)
            x //= 26
        stem = bytes(s)
        words.append(stem + b"0123456789" * 2)
        words[-1] = words[-1][:max(len(stem), int(want[i]))]
    lens = np.array([len(w) for w in words], dtype=np.int64)
    offs = np.zeros(D + 1, dtype=np.int64)
    offs[1:] = np.cumsum(lens)
    return torch.from_numpy(offs).cuda(), torch.from_numpy(np.frombuffer(b"".join(words), dtype=np.uint8).copy()).cuda()


def rows(n, D, seed):
    """n keys drawn uniformly from the dictionary, built on the device."""
    doffs, dbytes = dictionary(D, np.random.default_rng(seed))
    g = torch.Generator(device="cuda").manual_seed(seed)
    ranks = torch.randint(0, D, (n,), generator=g, device="cuda")
    lens = doffs[1:][ranks] - doffs[:-1][ranks]
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    row = torch.repeat_interleave(torch.arange(n, device="cuda"), lens, output_size=total)
    j = torch.arange(total, device="cuda") - offs[:-1][row]
    data = dbytes[doffs[:-1][ranks][row] + j]
    del row, j, ranks, lens
    return vb.StrKeys(offs, data)


def misc_ms(sh):
    return sh.stats()["kernels"]["misc"]["ms"]


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
    D = int(float(sys.argv[2])) if len(sys.argv) > 2 else 1_000_000
    name, limit = card()
    keys = rows(n, D, 11)
    torch.cuda.empty_cache()
    ones = torch.ones(n, dtype=torch.int64, device="cuda")
    R = M = 8
    with vb.Context(0, profile=True) as sc:
        lib = sc._lib
        sh = sc.parallelize(keys, M, values=ones).count_by_key(R)._run()
        sizes = [sh.reduce_blob_size(r) for r in range(R)]
        total = sum(sizes)
        out = [torch.empty(s, dtype=torch.uint8, device="cuda") for s in sizes]
        src = [torch.empty(s, dtype=torch.uint8, device="cuda") for s in sizes]
        dst = [torch.empty(s, dtype=torch.uint8, device="cuda") for s in sizes]

        def encode():
            for r in range(R):
                sh.reduce_blob_device(r, out[r])

        def copy():
            for r in range(R):
                dst[r].copy_(src[r])
                torch.cuda.synchronize()

        def timed(f):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        encode(); copy()
        t_enc, t_copy, t_kern = [], [], []
        for _ in range(REPS):           # alternated, so both see the same machine state
            k0 = misc_ms(sh)
            t_enc.append(timed(encode))
            t_kern.append((misc_ms(sh) - k0) / 1e3)
            t_copy.append(timed(copy))
        blobs = [sh.reduce_blob(r) for r in range(R)]
        assert all(bytes(o.cpu().numpy()) == b for o, b in zip(out, blobs)), "device and host blobs differ"
        # CPU-encoded buckets: the same records encoded by the host codec, in pinned host memory
        cpu = []
        for r in range(R):
            ko, kb, comb = sh.reduce_raw(r)
            pairs = [(kb[int(ko[i]):int(ko[i + 1])].tobytes(), int(c)) for i, c in enumerate(comb.tolist())]
            b = B.encode_str_pairs(pairs)
            assert b == blobs[r]
            t = torch.empty(len(b), dtype=torch.uint8, pin_memory=True)
            t.numpy()[:] = np.frombuffer(b, dtype=np.uint8)
            cpu.append(t)

        def decode_once():
            d = vb.StrShuffle(sc, R, R, L.VB_U64, L.VB_AGG_COUNT)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for m in range(R):
                L.check(lib.vb_shuffle_map_blob(d._h, m, ctypes.c_void_p(cpu[m].data_ptr()), cpu[m].numel(), L.VB_HOST))
            t = time.perf_counter() - t0
            return d, t

        d, _ = decode_once()
        d.seal()
        assert [d.reduce_size(r) for r in range(R)] == [sh.reduce_size(r) for r in range(R)], "decoded shuffle differs"
        d.free()
        t_dec = []
        for _ in range(REPS):
            d, t = decode_once()
            t_dec.append(t)
            d.free()
        distinct = sum(sh.reduce_size(r)[0] for r in range(R))
        sh.free()
    med = statistics.median
    gbps = lambda t: round(total / t / 1e9, 2)
    res = {"gpu": name, "power_limit": limit, "rows": n, "distinct_words": distinct, "key_bytes_in": int(keys.data.numel()),
           "maps": M, "partitions": R, "blob_bytes": total,
           "encode_ms": round(med(t_enc) * 1e3, 3), "encode_GBps": gbps(med(t_enc)),
           "encode_kernel_ms": round(med(t_kern) * 1e3, 3), "encode_kernel_GBps": gbps(med(t_kern)),
           "copy_d2d_ms": round(med(t_copy) * 1e3, 3), "copy_d2d_GBps": gbps(med(t_copy)),
           "encode_over_copy": round(med(t_copy) / med(t_enc), 3),
           "decode_ms": round(med(t_dec) * 1e3, 3), "decode_GBps": gbps(med(t_dec)),
           "decode_over_copy": round(med(t_copy) / med(t_dec), 3)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
