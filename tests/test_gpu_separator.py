"""`centrifuge-class --separator` on the GPU: one TSV with a separator line after every input's rows, and one report per
input, byte for byte what the unmodified reference writes (recorded digests, tests/golden/separator_digests.json).
Checked through the text operator (plain, gzip and bzip2 inputs, with a record-level fallback on a CR-LF file in the
middle of the run), through the record-level reader, to a file and to stdout, on one and on two GPUs, and under the
`centrifuge` wrapper's FIFO protocol."""
import errno
import os
import queue
import re
import select
import subprocess
import threading
import time

import pytest

import util
import util_separator as us

pytestmark = pytest.mark.gpu

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
STATS = re.compile(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units")
# -k 50 and -s/-u run on the record-level reader
CASES = {"default": [], "k1": ["-k", "1"], "k50": ["-k", "50"], "no_abundance": ["--no-abundance"], "skip_upto": ["-s", "20", "-u", "100"]}
TEXT_CASES = {"default", "k1", "no_abundance"}


def n_devices():
    from centrifuge_b200 import capi
    return int(capi.lib().cfb_device_count())


@pytest.fixture(scope="module")
def inputs(adv_reads, tmp_path_factory):
    d = tmp_path_factory.mktemp("separator")
    reads = us.adv_regular_reads(adv_reads)
    return {ext: us.write_inputs(d, reads, ext)[1] for ext in ("", ".gz", ".bz2")}


def run(args, cwd, out="out.tsv"):
    """(outputs, --report-file written, fallbacks of the text operator)"""
    got, written, err = us.run(EXE, args, cwd, out, env=dict(os.environ, CFB_TEXT_STATS="1"))
    return got, written, int(STATS.search(err).group(3))


@pytest.mark.parametrize("case", sorted(CASES))
def test_separator_matches_reference(case, adv_base, inputs, tmp_path):
    args = ["-q", "-x", adv_base] + inputs[""] + CASES[case]
    want, want_written = us.reference_outputs(case, args, tmp_path)
    got, written, fb = run(args, tmp_path / "plain")
    util.assert_matches(got, want, case)
    util.assert_matches(written, want_written, case)
    assert got[0].count(us.SEP) == 5 and len(got[1]) == 5
    assert fb == (1 if case in TEXT_CASES else 0)                  # only the CR-LF input leaves the text operator
    for ext in (".gz", ".bz2"):
        got_c, written_c, fb_c = run(["-q", "-x", adv_base] + inputs[ext] + CASES[case], tmp_path / ext[1:])
        assert (got_c, written_c) == (got, written), ext
        assert fb_c == fb, ext
    got_h, _, fb_h = run(args + ["--host-parse"], tmp_path / "host")
    assert got_h == got and fb_h == 0
    got_s, _, _ = run(args, tmp_path / "stdout", out="-")
    assert got_s == got


@pytest.mark.skipif(n_devices() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("case", ["default", "k1"])
def test_two_gpu_separator_is_byte_identical(case, adv_base, inputs, tmp_path):
    args = ["-q", "-x", adv_base] + inputs[""] + CASES[case]
    want, _ = us.reference_outputs(case, args, tmp_path)
    got, _, fb = run(args + ["--devices", "0-1"], tmp_path / "two")
    util.assert_matches(got, want, case)
    assert fb == 1


# ------------------------------------------------------------------------------ the wrapper's FIFO protocol
TIMEOUT = 300


def open_fifo_writer(path, proc, deadline):
    """O_NONBLOCK open for writing: ENXIO until the process opens the FIFO for reading.  Never blocks past the deadline."""
    while True:
        try:
            return os.open(path, os.O_WRONLY | os.O_NONBLOCK)
        except OSError as e:
            if e.errno != errno.ENXIO:
                raise
        if proc.poll() is not None or time.monotonic() > deadline:
            raise AssertionError("centrifuge-class did not open %s for reading" % path)
        time.sleep(0.01)


def write_all(fd, data, proc, deadline):
    view = memoryview(data)
    while view:
        try:
            view = view[os.write(fd, view[:1 << 16]):]
        except BlockingIOError:
            if proc.poll() is not None or time.monotonic() > deadline:
                raise AssertionError("centrifuge-class stopped reading its input")
            select.select([], [fd], [], 0.1)


def test_wrapper_fifo_protocol(adv_base, adv_reads, tmp_path):
    """As `centrifuge --sample-sheet` drives it: every input is a FIFO, and input i+1 is written only after input i's
    separator line has come out of stdout, at which point input i's report must be complete."""
    reads = us.adv_regular_reads(adv_reads)
    datas = [us.fastq(reads[0:300]), b"", us.fastq(reads[300:700]), us.fastq(reads[700:1500])]
    plain = []
    for i, data in enumerate(datas):
        plain.append(str(tmp_path / ("plain%d.fq" % i)))
        with open(plain[-1], "wb") as f:
            f.write(data)
    want, _ = us.reference_outputs("fifo", ["-q", "-x", adv_base, "-U", ",".join(plain)], tmp_path)
    fifos = [str(tmp_path / ("fifo%d" % i)) for i in range(len(datas))]
    for p in fifos:
        os.mkfifo(p)
    cwd = tmp_path / "run"
    cwd.mkdir()
    proc = subprocess.Popen([EXE, "--separator", "-q", "-x", adv_base, "-U", ",".join(fifos), "-S", "-", "--report-file", "rep.tsv"],
                            cwd=str(cwd), stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    out, err, seps = [], [], queue.Queue()

    def pump_out():
        for line in iter(proc.stdout.readline, b""):
            out.append(line)
            if line == us.SEP:
                seps.put(len(out))

    pumps = [threading.Thread(target=pump_out, daemon=True), threading.Thread(target=lambda: err.append(proc.stderr.read()), daemon=True)]
    for t in pumps:
        t.start()
    deadline = time.monotonic() + TIMEOUT
    snapshots = []
    try:
        for i, data in enumerate(datas):
            fd = open_fifo_writer(fifos[i], proc, deadline)
            try:
                write_all(fd, data, proc, deadline)
            finally:
                os.close(fd)
            try:
                seps.get(timeout=max(0.1, deadline - time.monotonic()))
            except queue.Empty:
                raise AssertionError("no separator line for input %d within %d s" % (i, TIMEOUT))
            seen = us.reports(cwd)                                  # as they are when input i's separator line arrives
            assert [n for n, _ in seen] == ["centrifuge_report_%d.tsv" % k for k in range(i + 1)]
            snapshots.append(seen[i])
        assert proc.wait(timeout=max(1, deadline - time.monotonic())) == 0
    finally:
        if proc.poll() is None:
            proc.kill()
        proc.wait()
        for t in pumps:
            t.join(timeout=10)
    # the reports as read at their separator lines are the reference's complete reports
    util.assert_matches((b"".join(out), snapshots, us.stderr_lines(b"".join(err))), want)
    assert us.reports(cwd) == snapshots and not (cwd / "rep.tsv").exists()
