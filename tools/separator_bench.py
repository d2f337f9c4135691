#!/usr/bin/env python3
"""What `centrifuge-class --separator` saves when many samples are classified against one index: 16 FASTQ inputs of
1 M bench reads on the 9 Gbp bench index, classified three ways on one GPU -- one --separator run (one index load,
one report per input), 16 separate runs (16 index loads), and one run over the concatenated inputs without --separator.
Prints one JSON line: the card and its power limit, the three wall times, the index-load time the runs print
(CFB_TEXT_STATS=1), and the per-input overhead of --separator, (separator - concatenated) / inputs."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

EXE = os.path.join(ROOT, "centrifuge_b200", "centrifuge-class")


def run(args, cwd):
    t0 = time.perf_counter()
    p = subprocess.run([EXE] + args, cwd=cwd, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
    dt = time.perf_counter() - t0
    err = p.stderr.decode()
    if p.returncode != 0:
        raise RuntimeError(err[-2000:])
    load = float(re.search(r"\[cfb\] index load ([0-9.]+) s", err).group(1))
    fb = int(re.search(r"(\d+) fallbacks\)", err).group(1))
    return dt, load, fb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", type=int, default=16)
    ap.add_argument("--reads", type=int, default=1000000, help="reads per input")
    ap.add_argument("--index-gbp", default="9")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    sys.argv = ["bench.py", "--index-gbp", args.index_gbp]
    a = bench.parse_args()
    base, _ = bench.get_index(a)
    work = tempfile.mkdtemp(prefix="separator_bench_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    try:
        files = []
        cat = os.path.join(work, "all.fq")
        with open(cat, "wb") as g:
            for i in range(args.inputs):
                data = bench.make_reads(a, args.reads, 5000 + i).fastq(0).tobytes()
                files.append(os.path.join(work, "in%02d.fq" % i))
                with open(files[-1], "wb") as f:
                    f.write(data)
                g.write(data)
        common = ["-q", "-x", base]
        res = {"gpu": gpu, "index_gbp": float(args.index_gbp), "inputs": args.inputs, "reads_per_input": args.reads}
        run(common + ["-U", files[0], "-S", os.path.join(work, "warm.tsv"), "--report-file", os.path.join(work, "warm.rep")], work)   # page cache
        dt, load, fb = run(common + ["--separator", "-U", ",".join(files), "-S", os.path.join(work, "sep.tsv")], work)
        res.update(separator_s=dt, separator_index_load_s=load, separator_fallbacks=fb)
        tot, loads = 0.0, []
        for i, f in enumerate(files):
            dt, load, _ = run(common + ["-U", f, "-S", os.path.join(work, "one.tsv"), "--report-file", os.path.join(work, "one.rep")], work)
            tot += dt; loads.append(load)
        res.update(separate_runs_s=tot, separate_index_load_s_median=sorted(loads)[len(loads) // 2])
        dt, load, _ = run(common + ["-U", cat, "-S", os.path.join(work, "cat.tsv"), "--report-file", os.path.join(work, "cat.rep")], work)
        res.update(concatenated_s=dt, concatenated_index_load_s=load)
        res["per_input_overhead_s"] = (res["separator_s"] - res["concatenated_s"]) / args.inputs
        res["saved_s"] = res["separate_runs_s"] - res["separator_s"]
        print(json.dumps(res), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
