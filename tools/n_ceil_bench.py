#!/usr/bin/env python3
"""File-to-file time of `centrifuge-class` on an N-dense FASTQ under `--n-ceil L,0,1` against the default ceiling, on a GPU
box.  Every read of the file is a 100 bp read of bench.py's synthetic index with an N at every third base (33 Ns), so
the default ceiling (15 Ns) filters all of them and L,0,1 passes all of them, with hit lists of up to one null hit per N.
Both runs go through the device text operator; the [cfb] lines give its spans, fallbacks and long units.
Env: CFB_NCEIL_READS (default 10M), CFB_NCEIL_GBP (default 1 -> 1 Gbp index), CFB_NCEIL_DIR (work directory)."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")


def run(args):
    t0 = time.time()
    p = subprocess.run([EXE] + args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
    dt = time.time() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr.decode()[-2000:])
    return dt, " | ".join(l for l in p.stderr.decode().splitlines() if l.startswith("[cfb]"))


def main():
    n = int(os.environ.get("CFB_NCEIL_READS", 10000000))
    sys.argv = ["bench.py", "--index-gbp", os.environ.get("CFB_NCEIL_GBP", "1"), "--rdlen", "100"]
    a = bench.parse_args()
    base, d = bench.get_index(a)
    work = os.environ.get("CFB_NCEIL_DIR", "/dev/shm" if os.path.isdir("/dev/shm") else d)
    fq = os.path.join(work, "n_ceil_bench.fq")
    t0 = time.time()
    with open(fq, "wb") as f:
        for s in range(0, n, 2000000):
            r = bench.make_reads(a, min(2000000, n - s), 2000 + s)
            r.codes[0][:, ::3] = 4
            f.write(r.fastq(0, start=s).tobytes())
    print("[n_ceil_bench] %d N-dense reads, %.2f GB FASTQ written in %.1f s" % (n, os.path.getsize(fq) / 1e9, time.time() - t0), flush=True)
    out, rep = os.path.join(work, "n_ceil_out.tsv"), os.path.join(work, "n_ceil_out.rep")
    try:
        for tag, extra in (("default ceiling", []), ("--n-ceil L,0,1", ["--n-ceil", "L,0,1"]),
                           ("default ceiling (2nd run)", []), ("--n-ceil L,0,1 (2nd run)", ["--n-ceil", "L,0,1"])):
            dt, st = run(["-q", "-x", base, "-U", fq, "-S", out, "--report-file", rep] + extra)
            with open(out, "rb") as f:
                rows = sum(1 for _ in f) - 1
            print("[n_ceil_bench] %s: wall %.2f s, %.1f M reads/s, %d rows; %s" % (tag, dt, n / dt / 1e6, rows, st), flush=True)
    finally:
        for p in (fq, out, rep):
            if os.path.exists(p):
                os.remove(p)


if __name__ == "__main__":
    main()
