#!/usr/bin/env python3
"""Regenerates tests/golden/* from the seeded generators and the UNMODIFIED reference binaries in
oracle/_ref (built from the reference sources by `make -C oracle ref`).  Run with CFB_REFERENCE_TREE=<reference sources>; the
outputs are committed so that the oracle stays pinned where the reference is not available.

  adv.{1,2,3,4}.cf.xz   index of tools/synth.py:write_adversarial (seed 33) built by centrifuge-build-bin
  adv_t<T>o<O>.{1,2,3,4}.cf.xz   the same genomes built with -t/--ftabchars T and -o/--offrate O (GEOMETRIES below)
  adv.reads.fa.xz       its reads
  adv.<case>.tsv.xz / adv.<case>.report.tsv   centrifuge-class output per option set (CASES below)
  example.*             output of the reference's own example fixture (MANUAL.markdown:1586-1603)
"""
import lzma
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import synth  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
CASES = {
    "default": [],
    "k1": ["-k", "1"],
    "k50": ["-k", "50"],
    "minhit15": ["--min-hitlen", "15"],
    "host": ["--host-taxids", "100,1005", "-k", "2"],
    "excl": ["--exclude-taxids", "10"],
    "family": ["--classification-rank", "family"],
    "notraverse": ["--no-traverse"],
}
# (ftabChars, offRate) of the other committed builds of the adv genomes: every sampled row (-o 0), the smallest ftab (-t 1)
# and long resolve walks (-o 7).  -t 12 is not committed (its ftab alone is 134 MB): tests build it and check its digest.
GEOMETRIES = {"adv_t6o0": (6, 0), "adv_t1o2": (1, 2), "adv_t8o7": (8, 7)}


def xz(src, dst):
    with open(src, "rb") as f, lzma.open(dst, "wb", preset=9) as g:
        g.write(f.read())


def main():
    tmp = tempfile.mkdtemp()
    synth.write_adversarial(tmp, seed=33, n_reads=3000)
    base = os.path.join(tmp, "adv")
    subprocess.check_call([os.path.join(REF, "centrifuge-build-bin"), "-p", "4", "--conversion-table", os.path.join(tmp, "conv.tsv"),
                           "--taxonomy-tree", os.path.join(tmp, "nodes.dmp"), "--name-table", os.path.join(tmp, "names.dmp"),
                           os.path.join(tmp, "genomes.fa"), base], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    for k in "1234":
        xz("%s.%s.cf" % (base, k), os.path.join(HERE, "adv.%s.cf.xz" % k))
    for name, (t, o) in GEOMETRIES.items():
        gbase = os.path.join(tmp, name)
        subprocess.check_call([os.path.join(REF, "centrifuge-build-bin"), "-p", "4", "-t", str(t), "-o", str(o),
                               "--conversion-table", os.path.join(tmp, "conv.tsv"), "--taxonomy-tree", os.path.join(tmp, "nodes.dmp"),
                               "--name-table", os.path.join(tmp, "names.dmp"), os.path.join(tmp, "genomes.fa"), gbase],
                              stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        for k in "1234":
            xz("%s.%s.cf" % (gbase, k), os.path.join(HERE, "%s.%s.cf.xz" % (name, k)))
    xz(os.path.join(tmp, "reads.fa"), os.path.join(HERE, "adv.reads.fa.xz"))
    for name, opts in CASES.items():
        out, rep = os.path.join(tmp, name + ".tsv"), os.path.join(tmp, name + ".rep")
        subprocess.check_call([os.path.join(REF, "centrifuge-class"), "-f", "-x", base, "-U", os.path.join(tmp, "reads.fa"),
                               "-S", out, "--report-file", rep] + opts, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        xz(out, os.path.join(HERE, "adv.%s.tsv.xz" % name))
        shutil.copy(rep, os.path.join(HERE, "adv.%s.report.tsv" % name))
    ex = os.path.join(os.environ["CFB_REFERENCE_TREE"], "example")
    if os.path.exists(ex):
        out, rep = os.path.join(tmp, "ex.tsv"), os.path.join(tmp, "ex.rep")
        subprocess.check_call([os.path.join(REF, "centrifuge-class"), "-f", "-x", ex + "/index/test", "-U", ex + "/reads/input.fa",
                               "-S", out, "--report-file", rep], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        shutil.copy(out, os.path.join(HERE, "example.tsv"))
        shutil.copy(rep, os.path.join(HERE, "example.report.tsv"))
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
