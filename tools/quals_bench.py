#!/usr/bin/env python3
"""File-to-file time of `centrifuge-class` on the same reads written with four quality encodings, on a GPU box: phred33
(no option), phred64 (--phred64), Solexa (--solexa-quals) and integer (--int-quals, two-digit tokens).  The reads are
10 M 100 bp reads of bench.py's synthetic index; each encoding runs with the default columns and with readQual, through
the device text operator and with --host-parse.  The [cfb] lines give the operator's spans and fallbacks.  The card's
name and power limit are printed with the numbers.
Env: CFB_QUALS_READS (default 10M), CFB_QUALS_GBP (default 1 -> 1 Gbp index), CFB_QUALS_DIR (work directory),
CFB_QUALS_HOST=0 skips the --host-parse runs, CFB_QUALS_ONLY=<names> runs only the listed encodings (comma-separated)."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")
ENCODINGS = (("phred33", []), ("phred64", ["--phred64"]), ("solexa", ["--solexa-quals"]), ("integer", ["--int-quals"]))
# phred33 byte -> the encoding's bytes: +31 for phred64 and Solexa (any byte is a Solexa value), "NN " for integers
_SHIFT = np.arange(256, dtype=np.uint8) + np.uint8(31)
_TOKENS = np.array([[ord("0") + max(b - 33, 0) // 10 % 10, ord("0") + max(b - 33, 0) % 10, ord(" ")] for b in range(256)], dtype=np.uint8)


def run(args):
    t0 = time.time()
    p = subprocess.run([EXE] + args, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
    dt = time.time() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr.decode()[-2000:])
    return dt, " | ".join(l for l in p.stderr.decode().splitlines() if l.startswith("[cfb]"))


def recode(fq, enc):
    """the records of a phred33 FASTQ chunk with their quality lines written in `enc`"""
    if enc == "phred33":
        return fq
    lines = fq.split(b"\n")
    quals = lines[3::4]
    if enc in ("phred64", "solexa"):
        lines[3::4] = [_SHIFT[np.frombuffer(q, dtype=np.uint8)].tobytes() for q in quals]
    else:
        lines[3::4] = [_TOKENS[np.frombuffer(q, dtype=np.uint8)].tobytes()[:-1] for q in quals]
    return b"\n".join(lines)


def card():
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, check=True)
        return p.stdout.decode().strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown card (%s)" % e


def main():
    n = int(os.environ.get("CFB_QUALS_READS", 10000000))
    host = os.environ.get("CFB_QUALS_HOST", "1") != "0"
    sys.argv = ["bench.py", "--index-gbp", os.environ.get("CFB_QUALS_GBP", "1"), "--rdlen", "100"]
    a = bench.parse_args()
    base, d = bench.get_index(a)
    work = os.environ.get("CFB_QUALS_DIR", "/dev/shm" if os.path.isdir("/dev/shm") else d)
    print("[quals_bench] %s" % card(), flush=True)
    only = os.environ.get("CFB_QUALS_ONLY")
    encodings = [(e, o) for e, o in ENCODINGS if not only or e in only.split(",")]
    files = {e: os.path.join(work, "quals_bench.%s.fq" % e) for e, _ in encodings}
    out, rep = os.path.join(work, "quals_out.tsv"), os.path.join(work, "quals_out.rep")
    try:
        t0 = time.time()
        fo = {e: open(p, "wb") for e, p in files.items()}
        for s in range(0, n, 2000000):
            fq = bench.make_reads(a, min(2000000, n - s), 2000 + s).fastq(0, start=s).tobytes()
            for e, f in fo.items():
                f.write(recode(fq, e))
        for f in fo.values():
            f.close()
        print("[quals_bench] %d reads written in %d encodings in %.1f s (%s)" %
              (n, len(files), time.time() - t0, ", ".join("%s %.2f GB" % (e, os.path.getsize(p) / 1e9) for e, p in files.items())), flush=True)
        for e, opts in encodings:
            for cols in ([], ["--tab-fmt-cols", "readID,taxID,readQual"]):
                for hp in ([False, True] if host else [False]):
                    args = ["-q", "-x", base, "-U", files[e], "-S", out, "--report-file", rep] + opts + cols + (["--host-parse"] if hp else [])
                    dt, st = run(args)
                    print("[quals_bench] %-8s %-13s %-11s wall %.2f s, %.2f M reads/s; %s" %
                          (e, "readQual" if cols else "default cols", "--host-parse" if hp else "device", dt, n / dt / 1e6, st), flush=True)
    finally:
        for p in list(files.values()) + [out, rep]:
            if os.path.exists(p):
                os.remove(p)


if __name__ == "__main__":
    main()
