#!/usr/bin/env python3
"""Gzip input on a GPU box: bench-like FASTQ (cfb_synth_reads through bench.py's helpers, 100 bp, CFB_GZ_BENCH_READS reads,
default 10 M) compressed as one member at level 6, then
  - the device inflater's rate (decompressed GB/s, host clock around whole-file inflates that end in a device synchronise,
    after one warm-up inflate; the output is copied to host memory, as centrifuge-class does),
  - one host core running zlib on the same bytes,
  - `centrifuge-class` file-to-file reads/s on the .fq and on the .fq.gz (files in /dev/shm),
  - chunks and re-decoded chunks, the card's name and power limit.
One JSON line on stdout.  Env: CFB_GZ_BENCH_READS, CFB_CLI_GBP (index size, default 1 Gbp), CFB_GZ_CHUNK_KB."""
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")


def inflate_device(gz, out):
    """whole-file inflate through the ABI into the reused buffer `out`: (seconds, bytes out, stats)"""
    g = capi.Gunzip(0, 0)
    L = capi.lib()
    src = np.frombuffer(gz, dtype=np.uint8)
    pos, total = 0, 0
    n_out, n_in = C.c_uint64(), C.c_uint64()
    t0 = time.perf_counter()
    while True:
        rc = L.cfb_gunzip_run(g.h, C.c_void_p(src.ctypes.data + pos), C.c_uint64(len(gz) - pos), C.c_int(1),
                              out.ctypes.data_as(C.c_void_p), C.c_uint64(out.size), C.byref(n_out), C.byref(n_in))
        if rc:
            raise capi.CfbError(L.cfb_last_error().decode())
        pos += n_in.value
        total += n_out.value
        if not n_out.value and not n_in.value:
            break
    dt = time.perf_counter() - t0
    st = g.stats()
    g.close()
    return dt, total, st


def main():
    n = int(os.environ.get("CFB_GZ_BENCH_READS", 10000000))
    sys.argv = ["bench.py", "--index-gbp", os.environ.get("CFB_CLI_GBP", "1"), "--rdlen", "100"]
    a = bench.parse_args()
    base, d = bench.get_index(a)
    work = "/dev/shm" if os.path.isdir("/dev/shm") else d
    fq, fqz = os.path.join(work, "gz_bench.fq"), os.path.join(work, "gz_bench.fq.gz")
    comp = zlib.compressobj(6, zlib.DEFLATED, 31)
    t0 = time.time()
    with open(fq, "wb") as f, open(fqz, "wb") as z:
        for s in range(0, n, 2000000):
            m = bench.make_reads(a, min(2000000, n - s), 1000 + s).fastq(0, start=s).tobytes()
            f.write(m)
            z.write(comp.compress(m))
        z.write(comp.flush())
    plain_bytes, gz_bytes = os.path.getsize(fq), os.path.getsize(fqz)
    print("[gunzip_bench] %d reads: %.2f GB FASTQ, %.2f GB gzip (level 6, one member), %.0f s to write" % (n, plain_bytes / 1e9, gz_bytes / 1e9, time.time() - t0), file=sys.stderr, flush=True)
    with open(fqz, "rb") as f:
        gz = f.read()
    out = np.empty(1 << 28, dtype=np.uint8)
    inflate_device(gz, out)                                   # warm-up: module load, buffer growth
    runs = [inflate_device(gz, out) for _ in range(3)]
    dev_s = min(r[0] for r in runs)
    assert all(r[1] == plain_bytes for r in runs)
    t0 = time.perf_counter()
    host_out = zlib.decompress(gz, 31)
    host_s = time.perf_counter() - t0
    assert len(host_out) == plain_bytes
    del host_out

    def cli(path):
        o, r = os.path.join(work, "gz_bench.tsv"), os.path.join(work, "gz_bench.rep")
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
    t_gz, d_gz, err = cli(fqz)
    m = re.search(r"gunzip: .*", err)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    print(json.dumps({
        "reads": n, "fastq_bytes": plain_bytes, "gzip_bytes": gz_bytes,
        "device_inflate_gb_per_s": round(plain_bytes / dev_s / 1e9, 3), "device_inflate_s": [round(r[0], 3) for r in runs],
        "host_zlib_one_core_gb_per_s": round(plain_bytes / host_s / 1e9, 3),
        "chunks": runs[0][2]["chunks"], "redecoded_chunks": runs[0][2]["redone"],
        "cli_reads_per_s_fq": round(n / t_plain), "cli_reads_per_s_fq_gz": round(n / t_gz), "cli_same_tsv": d_plain == d_gz,
        "cli_gunzip_line": m.group(0) if m else None, "gpu": gpu[0] if gpu else None,
    }))
    for p in (fq, fqz, os.path.join(work, "gz_bench.tsv"), os.path.join(work, "gz_bench.rep")):
        if os.path.exists(p):
            os.remove(p)


if __name__ == "__main__":
    main()
