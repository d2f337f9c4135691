#!/usr/bin/env python3
"""FASTQ -> TSV throughput of `centrifuge-class` with the default columns against the column list the `centrifuge`
wrapper asks for when it writes reads back out (--un / --al / --un-conc / --al-conc: the default list plus
readSeq,readQual, with --passthrough), alternating the two in one run on the same files.  Prints reads/s and the
CFB_TEXT_STATS time breakdown (reader busy / device wait / writer busy) of every run.
Env: CFB_CLI_GBP (default 1 -> 1 Gbp index), CFB_COLS_READS (10M single reads), CFB_COLS_PAIRS (5M 2 x 150 pairs),
CFB_COLS_REPS (2 runs per list and input)."""
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")
DEFAULT = []
WRAPPER = ["--tab-fmt-cols", "readID,seqID,taxID,score,2ndBestScore,hitLength,queryLength,numMatches,readSeq,readQual", "--passthrough"]


def write_fastq(a, n, paths):
    for s in range(0, n, 2000000):
        k = min(2000000, n - s)
        m = bench.make_reads(a, k, 1000 + s)
        for mate, p in enumerate(paths):
            with open(p, "ab" if s else "wb") as f:
                f.write(m.fastq(mate, start=s, suffix=(b"/%d" % (mate + 1)) if len(paths) == 2 else b"").tobytes())


def main():
    gbp = os.environ.get("CFB_CLI_GBP", "1")
    reps = int(os.environ.get("CFB_COLS_REPS", 2))
    cases = [("SE 100 bp", int(os.environ.get("CFB_COLS_READS", 10000000)), ["--rdlen", "100"]),
             ("PE 2 x 150 bp", int(os.environ.get("CFB_COLS_PAIRS", 5000000)), ["--rdlen", "150", "--paired"])]
    for tag, n, extra in cases:
        if n <= 0:
            continue
        sys.argv = ["bench.py", "--index-gbp", gbp] + extra
        a = bench.parse_args()
        base, d = bench.get_index(a)
        work = os.environ.get("CFB_CLI_DIR", "/dev/shm" if os.path.isdir("/dev/shm") else d)
        paths = [os.path.join(work, "cols_bench_%d.fq" % m) for m in range(2 if a.paired else 1)]
        t0 = time.time()
        write_fastq(a, n, paths)
        print("[cols_bench] %s: %d units, %.2f GB FASTQ written in %.1f s" % (tag, n, sum(os.path.getsize(p) for p in paths) / 1e9, time.time() - t0), flush=True)
        inp = ["-1", paths[0], "-2", paths[1]] if a.paired else ["-U", paths[0]]
        out, rep = os.path.join(work, "cols_out.tsv"), os.path.join(work, "cols_out.rep")
        for r in range(reps):
            for name, cols in (("default columns", DEFAULT), ("wrapper columns", WRAPPER)):
                t0 = time.time()
                p = subprocess.run([EXE, "-q", "-x", base] + inp + cols + ["-S", out, "--report-file", rep], stdout=subprocess.DEVNULL,
                                   stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
                dt = time.time() - t0
                if p.returncode != 0:
                    raise RuntimeError(p.stderr.decode()[-2000:])
                err = p.stderr.decode()
                m = re.search(r"reads ([0-9.e+-]+) s", err)
                t_reads = float(m.group(1)) if m else dt
                print("[cols_bench] %s, %s, run %d: %.2f M units/s (reads phase %.2f s, wall %.2f s, TSV %.2f GB); %s" % (
                    tag, name, r + 1, n / t_reads / 1e6, t_reads, dt, os.path.getsize(out) / 1e9,
                    " | ".join(l for l in err.splitlines() if l.startswith("[cfb] text"))), flush=True)
        for f in paths + [out, rep]:
            if os.path.exists(f):
                os.remove(f)


if __name__ == "__main__":
    main()
