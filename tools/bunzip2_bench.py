#!/usr/bin/env python3
"""bzip2 input on a GPU box: bench-like FASTQ (cfb_synth_reads through bench.py's helpers, 100 bp, CFB_BZ2_BENCH_READS
reads, default 4 M) compressed two ways, as one level-9 stream and as one stream per 900 KB piece (as pbzip2 writes), then
  - the device decompressor's rate on each (decompressed GB/s, best of 3 after a warm-up, host clock around whole-file
    runs into host memory, each ending in a device synchronise),
  - one host core running libbz2 (Python's bz2) on the same bytes,
  - `centrifuge-class` file-to-file reads/s on the .fq, .fq.gz and .fq.bz2 (files in /dev/shm), and whether the TSVs match,
  - blocks and rejected block starts, the card's name and power limit.
One JSON line on stdout.  --profile instead prints the device time per k_bz_* kernel of one whole-file run
(torch.profiler).  Env: CFB_BZ2_BENCH_READS, CFB_CLI_GBP (index size, default 1 Gbp), CFB_BZ2_PASS_KB."""
import bz2
import ctypes as C
import gzip
import json
import os
import re
import subprocess
import sys
import time
import zlib
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")


def decompress_device(comp, out):
    """whole-file run through the ABI into the reused host buffer `out`: (seconds, bytes out, stats)"""
    g = capi.Bunzip2(0, 0)
    L = capi.lib()
    src = np.frombuffer(comp, dtype=np.uint8)
    pos, total = 0, 0
    n_out, n_in = C.c_uint64(), C.c_uint64()
    t0 = time.perf_counter()
    while True:
        rc = L.cfb_bunzip2_run(g.h, C.c_void_p(src.ctypes.data + pos), C.c_uint64(len(comp) - pos), C.c_int(1),
                               out.ctypes.data_as(C.c_void_p), C.c_uint64(out.size), C.byref(n_out), C.byref(n_in))
        if rc:
            raise capi.CfbError(L.cfb_last_error().decode())
        pos += n_in.value
        total += n_out.value
        if not n_out.value and not n_in.value:
            break
    dt = time.perf_counter() - t0              # cfb_bunzip2_run synchronises its stream before it returns
    st = g.stats()
    g.close()
    return dt, total, st


def _bz9(piece):
    return bz2.compress(piece, 9)


def main():
    n = int(os.environ.get("CFB_BZ2_BENCH_READS", 4000000))
    profile = "--profile" in sys.argv
    sys.argv = ["bench.py", "--index-gbp", os.environ.get("CFB_CLI_GBP", "1"), "--rdlen", "100"]
    a = bench.parse_args()
    base, d = bench.get_index(a)
    work = "/dev/shm" if os.path.isdir("/dev/shm") else d
    fq, fqz, fqb = (os.path.join(work, "bz_bench.fq" + x) for x in ("", ".gz", ".bz2"))
    t0 = time.time()
    with open(fq, "wb") as f:
        for s in range(0, n, 2000000):
            f.write(bench.make_reads(a, min(2000000, n - s), 1000 + s).fastq(0, start=s).tobytes())
    with open(fq, "rb") as f:
        plain = f.read()
    with Pool(min(16, os.cpu_count() or 1)) as pool:
        pieces = [plain[i:i + 900000] for i in range(0, len(plain), 900000)]
        multi = b"".join(pool.map(_bz9, pieces))
        one = pool.apply_async(_bz9, (plain,))
        gz = pool.apply_async(gzip.compress, (plain, 6))
        one, gz = one.get(), gz.get()
    with open(fqb, "wb") as f:
        f.write(one)
    with open(fqz, "wb") as f:
        f.write(gz)
    print("[bunzip2_bench] %d reads: %.2f GB FASTQ, %.3f GB bzip2 (one level-9 stream), %.3f GB as %d streams, %.0f s to write"
          % (n, len(plain) / 1e9, len(one) / 1e9, len(multi) / 1e9, len(pieces), time.time() - t0), file=sys.stderr, flush=True)
    out = np.empty(1 << 28, dtype=np.uint8)
    if profile:
        import torch
        decompress_device(one, out)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            dt, _, st = decompress_device(one, out)
        per = {}
        for e in prof.key_averages():
            if e.key.startswith("k_bz_") or "k_bz_" in e.key:
                name = re.search(r"k_bz_\w+", e.key).group(0)
                per[name] = per.get(name, 0) + e.device_time_total / 1e3
        print(json.dumps({"reads": n, "fastq_bytes": len(plain), "wall_s": round(dt, 3), "kernel_ms": {k: round(v, 2) for k, v in sorted(per.items(), key=lambda x: -x[1])},
                          "blocks": st["blocks"], "rejected": st["rejected"]}))
        for p in (fq, fqz, fqb):
            os.remove(p)
        return
    res = {}
    for tag, comp in (("one_stream", one), ("pbzip2", multi)):
        decompress_device(comp, out)                            # warm-up: module load, buffer growth
        runs = [decompress_device(comp, out) for _ in range(3)]
        assert all(r[1] == len(plain) for r in runs)
        res[tag] = dict(bytes=len(comp), device_gb_per_s=round(len(plain) / min(r[0] for r in runs) / 1e9, 3),
                        device_s=[round(r[0], 3) for r in runs], blocks=runs[0][2]["blocks"], rejected=runs[0][2]["rejected"])
    t0 = time.perf_counter()
    host = bz2.decompress(one)
    host_s = time.perf_counter() - t0
    assert host == plain
    del host

    def cli(path):
        o, r = os.path.join(work, "bz_bench.tsv"), os.path.join(work, "bz_bench.rep")
        t0 = time.time()
        p = subprocess.run([EXE, "-q", "-x", base, "-U", path, "-S", o, "--report-file", r], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                           env=dict(os.environ, CFB_TEXT_STATS="1"))
        dt = time.time() - t0
        if p.returncode:
            raise RuntimeError(p.stderr.decode()[-2000:])
        with open(o, "rb") as f:
            digest = zlib.crc32(f.read())
        return dt, digest, p.stderr.decode()
    cli(fq)                                                   # warm-up: index into the page cache
    t_plain, d_plain, _ = cli(fq)
    t_gz, d_gz, _ = cli(fqz)
    t_bz, d_bz, err = cli(fqb)
    m = re.search(r"bunzip2: .*", err)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    print(json.dumps({
        "reads": n, "fastq_bytes": len(plain), **res,
        "host_libbz2_one_core_gb_per_s": round(len(plain) / host_s / 1e9, 3),
        "cli_reads_per_s_fq": round(n / t_plain), "cli_reads_per_s_fq_gz": round(n / t_gz), "cli_reads_per_s_fq_bz2": round(n / t_bz),
        "cli_same_tsv": d_plain == d_gz == d_bz, "cli_bunzip2_line": m.group(0) if m else None, "gpu": gpu[0] if gpu else None,
    }))
    for p in (fq, fqz, fqb, os.path.join(work, "bz_bench.tsv"), os.path.join(work, "bz_bench.rep")):
        if os.path.exists(p):
            os.remove(p)


if __name__ == "__main__":
    main()
