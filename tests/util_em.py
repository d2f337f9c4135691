"""Plain-Python restatement of SpeciesMetrics::calculateAbundance's iteration (aln_sink.h:196-495) on a flattened
tie-set table, an order-exact numpy form of the same loops, the reference's table construction from a classification
TSV (addSpeciesCounts and the prologue of calculateAbundance), and a seeded generator of such tables.  Test
infrastructure: Python floats are IEEE doubles and the loops add in the reference's order, so results are comparable
bit for bit."""
import math
import os

import numpy as np

SIZE_MAX = 2 ** 64 - 1                                   # numeric_limits<size_t>::max(): "no genome size known"
X86_NAN = 0xFFF8000000000000                             # what x86 SSE arithmetic makes of 0/0 and inf/inf


def em_python(count, key_off, target, length, p):
    """SpeciesMetrics::calculateAbundance iteration (aln_sink.h:410-480) on the flattened table."""
    n, K = len(p), len(count)

    def step(p):
        pn = [0.0] * n
        for k in range(K):
            tg = target[key_off[k]:key_off[k + 1]]
            psum = 0.0
            for j in tg:
                psum += p[j]
            if psum == 0.0:
                continue
            for j in tg:
                pn[j] += count[k] * (p[j] / psum)
        s = 0.0
        for i in range(n):
            s += pn[i] / length[i]
        return [pn[i] / length[i] / s for i in range(n)]

    it = 0
    while True:
        pn = step(p)
        pn2 = step(pn)
        ssr = ssv = 0.0
        pr = [0.0] * n; pv = [0.0] * n
        for i in range(n):
            pr[i] = pn[i] - p[i]; ssr += pr[i] * pr[i]
            pv[i] = pn2[i] - pn[i] - pr[i]; ssv += pv[i] * pv[i]
        if ssv > 0.0:
            g = -math.sqrt(ssr / ssv)
            pn2 = [max(0.0, p[i] - 2 * g * pr[i] + g * g * pv[i]) for i in range(n)]
            pn = step(pn2)
        diff = 0.0
        for i in range(n):
            diff += (p[i] - pn[i]) if p[i] > pn[i] else (pn[i] - p[i])
        if diff < 0.0000000001:
            break
        it += 1
        if it >= 10000:
            break
        p = pn
    return p, it, diff


def _seq_sum(x):
    """Sum in ascending index order from 0.0, one addition at a time (np.sum would add pairwise)."""
    return float(np.add.accumulate(np.concatenate([[0.0], x]))[-1])


def em_numpy(count, key_off, target, length, p0, species_sum=_seq_sum):
    """em_python's operations in em_python's order, vectorised: np.bincount adds its weights in index order, so the
    per-key sums (contributions in key order) and the per-species sums (contributions in (key, position) order) are
    the sequential loops' doubles; sums over species add one at a time.  Division by zero and NaN follow IEEE (x86's
    default NaN) instead of raising.  species_sum replaces the sums over species (np.sum: a reordered variant)."""
    count = np.asarray(count, dtype=np.uint64).astype(np.float64)       # (double)uint64: rounds to nearest
    key_off = np.asarray(key_off, dtype=np.int64)
    target = np.asarray(target, dtype=np.int64)
    length = np.asarray(length, dtype=np.uint64).astype(np.float64)
    p = np.array(p0, dtype=np.float64)
    n, K = len(p), len(count)
    key_of = np.repeat(np.arange(K), np.diff(key_off))

    def step(p):
        psum = np.bincount(key_of, weights=p[target], minlength=K)
        live = psum[key_of] != 0.0                                      # keys whose psum is 0 add nothing
        k, j = key_of[live], target[live]
        pn = np.bincount(j, weights=count[k] * (p[j] / psum[k]), minlength=n)
        s = species_sum(pn / length)
        return pn / length / s

    it = 0
    with np.errstate(all="ignore"):
        while True:
            pn = step(p)
            pn2 = step(pn)
            pr = pn - p
            pv = pn2 - pn - pr
            ssr, ssv = species_sum(pr * pr), species_sum(pv * pv)
            if ssv > 0.0:
                g = -math.sqrt(ssr / ssv)
                x = p - 2 * g * pr + g * g * pv
                pn2 = np.where(0.0 < x, x, 0.0)                         # std::max(0.0, x): NaN -> 0.0
                pn = step(pn2)
            diff = species_sum(np.where(p > pn, p - pn, pn - p))
            if diff < 0.0000000001:
                break
            it += 1
            if it >= 10000:
                break
            p = pn
    return p, it, diff


def _ptr(a, t):
    import ctypes as C
    return a.ctypes.data_as(C.POINTER(t))


def _em_args(count, key_off, target, length, p0):
    import ctypes as C
    a = [np.array(count, dtype=np.uint64), np.array(key_off, dtype=np.uint64), np.array(target, dtype=np.uint32),
         np.array(length, dtype=np.uint64), np.array(p0, dtype=np.float64)]
    iters, diff = C.c_uint64(), C.c_double()
    args = [C.c_uint64(len(a[4])), C.c_uint64(len(a[0])), _ptr(a[0], C.c_uint64), _ptr(a[1], C.c_uint64), _ptr(a[2], C.c_uint32),
            _ptr(a[3], C.c_uint64), _ptr(a[4], C.c_double), C.byref(iters), C.byref(diff)]
    return a, args, iters, diff


def host_em(count, key_off, target, length, p0):
    """cfb_em_abundance_host, the product's host loop: (p, iterations, last difference)."""
    import ctypes as C
    import util
    a, args, iters, diff = _em_args(count, key_off, target, length, p0)
    assert C.CDLL(util.PRODUCT_LIB).cfb_em_abundance_host(*args) == 0
    return a[4], iters.value, diff.value


def device_em(count, key_off, target, length, p0, device=0):
    """cfb_em_abundance on `device`: (p, iterations, last difference)."""
    import ctypes as C
    import util
    a, args, iters, diff = _em_args(count, key_off, target, length, p0)
    assert C.CDLL(util.PRODUCT_LIB).cfb_em_abundance(C.c_int(device), *args) == 0
    return a[4], iters.value, diff.value


def bits(x):
    """IEEE bit patterns of doubles (NaN payloads and signs included), for exact comparison."""
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def fmt_double(x):
    """operator<<(ostream&, double) with the default precision (%g), as glibc prints NaN: with its sign."""
    if math.isnan(x):
        return "-nan" if math.copysign(1.0, x) < 0 else "nan"
    return "%g" % x


def em_stderr_lines(iters, diff):
    """The two lines centrifuge-class writes to stderr after the EM (aln_sink.h:471-472)."""
    return ["Number of iterations in EM algorithm: %d" % iters,
            "Probability diff. (P - P_prev) in the last iteration: %s" % fmt_double(diff)]


def em_lines_of(stderr):
    return [ln for ln in stderr.decode().splitlines() if "EM algorithm" in ln or "Probability diff" in ln]


def run_class(exe, args, tmp, env=None):
    """centrifuge-class `args` -S/--report-file into tmp: (report bytes, EM stderr lines, whole stderr)."""
    import subprocess
    rep = os.path.join(str(tmp), "em.rep")
    p = subprocess.run([exe] + list(args) + ["-S", os.path.join(str(tmp), "em.tsv"), "--report-file", rep],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=env)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    with open(rep, "rb") as f:
        return f.read(), em_lines_of(p.stderr), p.stderr.decode()


# the option sets of the committed adv goldens (tests/golden/make_golden.py)
ADV_CASES = {
    "default": [], "k1": ["-k", "1"], "k50": ["-k", "50"], "minhit15": ["--min-hitlen", "15"],
    "host": ["--host-taxids", "100,1005", "-k", "2"], "excl": ["--exclude-taxids", "10"],
    "family": ["--classification-rank", "family"], "notraverse": ["--no-traverse"],
}


def adv_reference_em_lines(case, adv_base, adv_reads, tmp):
    """Recorded digest of the reference binary's two EM lines on the adv reads with ADV_CASES[case] (util.reference)."""
    import util
    return util.reference("em/adv/" + case, lambda: run_class(util.REF_CLASS, ["-f", "-x", adv_base, "-U", adv_reads] + ADV_CASES[case], tmp)[1])


# ----------------------------------------------------------------------------- the table, from classification output
def observed_from_tsv(rows):
    """SpeciesMetrics::addSpeciesCounts (aln_sink.h:142-172) over single-end classification TSV rows (default columns,
    header excluded): {sorted taxIDs: reads}.  A classified read's maximum score is (queryLength-15)^2, an unclassified
    read's 0 (classifier.h:530-535); the rows of one read are consecutive."""
    observed, cur = {}, []
    for row in rows:
        f = row.split("\t")
        taxid, score, qlen, nresult = int(f[2]), int(f[3]), int(f[6]), int(f[7])
        max_score = 0 if f[1] == "unclassified" else ((qlen - 15) ** 2 if qlen > 15 else 0)
        if score >= max_score:
            cur.append(taxid)
            if len(cur) == nresult:
                key = tuple(sorted(cur))
                observed[key] = observed.get(key, 0) + 1
                cur = []
    return observed


def _ids_order(ids):
    return (len(ids), ids)                               # SpeciesMetrics::IDs::operator< (aln_sink.h:63-71)


def flatten(observed, tree, sizes):
    """The prologue of calculateAbundance (aln_sink.h:274-417) on `observed`: tree = {taxid: (parent, is_leaf)},
    sizes = {taxid: genome size}.  Returns (count, key_off, target, length, p0, taxids): the flattened table, the start
    vector, and the taxid of every species slot."""
    keys = sorted(observed, key=_ids_order)
    leaves = sorted({t for ids in keys for t in ids if t in tree and tree[t][1]})
    leaf_set = set(leaves)
    anc = {}
    for ids in keys:
        for tid in ids:
            if tid in leaf_set or tid in anc:
                continue
            ch = []
            for leaf in leaves:
                t = leaf
                while t in tree:
                    par = tree[t][0]
                    if tid == par:
                        ch.append(leaf)
                    if t == par:
                        break
                    t = par
            anc[tid] = sorted(ch)
    t2n, p, length = {}, [], []
    for ids in keys:
        for tid in ids:
            if tid not in leaf_set:
                continue
            if tid not in t2n:
                t2n[tid] = len(p)
                p.append(1.0 / len(ids) * observed[ids])
                length.append(sizes.get(tid, SIZE_MAX))
            else:
                p[t2n[tid]] += 1.0 / len(ids) * observed[ids]
    with np.errstate(all="ignore"):
        pa, la = np.array(p, dtype=np.float64), np.array(length, dtype=np.uint64).astype(np.float64)
        p0 = pa / la / _seq_sum(pa / la)
    count, key_off, target = [], [0], []
    for ids in keys:
        for tid in ids:
            if tid in t2n:
                target.append(t2n[tid])
            elif tid in anc:
                target += [t2n[c] for c in anc[tid] if c in t2n]
        count.append(observed[ids])
        key_off.append(len(target))
    taxids = [0] * len(t2n)
    for tid, j in t2n.items():
        taxids[j] = tid
    return count, key_off, target, length, p0, taxids


def index_tree(base):
    """{taxid: (parent, is_leaf)} of an index's taxonomy, read through the host-only index loader."""
    from centrifuge_b200 import capi
    ix = capi.Index(base, -1)
    try:
        tree = {}
        for t in ix.node_taxids():
            par, _, leaf = ix.tax_node(int(t))
            tree[int(t)] = (par, bool(leaf))
        return tree
    finally:
        ix.close()


def report_abundance(report):
    """{taxid: (genomeSize, abundance text)} of a report file's rows."""
    out = {}
    for ln in report.decode().splitlines()[1:]:
        f = ln.split("\t")
        out[int(f[1])] = (int(f[3]), f[6])
    return out


# ----------------------------------------------------------------------------- generated tables
KINDS = ("random", "empty", "zero", "dups", "wide", "skew", "counts", "lengths", "singletons", "slow", "underflow", "nan")


def random_problem(seed, n, K, kind="random"):
    """A seeded flattened table of n species and K keys.  kind selects a shape the EM must get right:
      random      1-4 targets per key, duplicates allowed
      empty       a fifth of the keys have no targets (ids that are neither a leaf nor an ancestor of one)
      zero        some keys reach only species whose start value is 0, so their psum is 0
      dups        keys that name one species several times
      wide        keys of 500 and more targets (an ancestor expanded to its leaves)
      skew        species 0 in 40 % of the keys (its incidence list is long)
      counts      counts of 1, 2^53 + 1 and 2^64 - 1 (not exact as doubles)
      lengths     genome sizes of 1 and SIZE_MAX ("no size")
      singletons  one target per key: a fixed point after the first step, so ssv == 0 at iteration 1
      slow        every key three neighbours on a chain of species: slow to converge (seed 2, n=300, K=500: 323 iterations)
      underflow   species 0 in every key, all others start near 1e-200: their changes square to 0, so ssv == 0 and the
                  third step is guarded off although p still moves
      nan         one genome size of 0: every value turns NaN and the loop runs to the 10 000-iteration cap"""
    rng = np.random.default_rng(seed)
    count, key_off, target = [], [0], []
    for k in range(K):
        if kind == "singletons":
            sz = 1
        elif kind == "empty":
            sz = 0 if k % 5 == 2 else int(rng.integers(1, 5))
        elif kind == "wide" and k % 7 == 0:
            sz = int(rng.integers(500, 700))
        elif kind == "dups":
            sz = int(rng.integers(2, 7))
        else:
            sz = int(rng.integers(1, 5))
        if kind == "wide" and sz >= 500:
            lo = int(rng.integers(0, max(1, n - sz)))
            ids = np.arange(lo, lo + sz) % n                   # sorted leaf list of an ancestor
        elif kind == "dups":
            ids = rng.integers(0, min(n, 3), size=sz)
        elif kind == "slow":                               # windows of 3 neighbours along a chain of species
            a = int(rng.integers(0, max(1, n - 2)))
            ids = np.arange(a, a + 3) % n
        else:
            ids = rng.integers(0, n, size=sz)              # duplicates allowed: an ancestor and its own leaf in one key
        if kind == "skew" and rng.random() < 0.4:
            ids = np.concatenate([ids, [0]])
        target += [int(x) for x in ids]
        count.append(int(rng.integers(1, 5000)))
        key_off.append(len(target))
    length = [int(x) for x in rng.integers(1000, 5_000_000, size=n)]
    if n > 6:
        length[3] = SIZE_MAX                             # "no size known" (numeric_limits<size_t>::max())
    p0 = rng.random(n); p0[rng.random(n) < 0.15] = 0.0   # species nobody hit
    if kind == "zero":
        dead = rng.random(n) < 0.4
        p0[dead] = 0.0
        for k in range(0, K, 3):                         # every third key reaches dead species only
            d = np.flatnonzero(dead)
            if len(d):
                target[key_off[k]:key_off[k + 1]] = [int(x) for x in rng.choice(d, size=key_off[k + 1] - key_off[k])]
    if kind == "counts":
        count = [[1, 2 ** 53 + 1, 2 ** 64 - 1][k % 3] if k % 2 == 0 else c for k, c in enumerate(count)]
    if kind == "lengths":
        length = [[1, SIZE_MAX][j % 2] if j % 3 != 2 else L for j, L in enumerate(length)]
    if kind == "underflow":                              # species 0 in every key; the others' values square to 0
        for k in range(K):
            target.insert(key_off[k] + k, 0)
        key_off = [o + k for k, o in enumerate(key_off)]
        p0 = np.concatenate([[1.0], 1e-200 * rng.random(n - 1)])
    if kind == "nan":
        length[min(1, n - 1)] = 0
        p0[min(1, n - 1)] = 0.5
    if p0.sum() == 0:
        p0[0] = 1.0
    p0 = [float(x) for x in p0 / p0.sum()]
    return count, key_off, target, length, p0


# (seed, n, K, kind) of the generated tables both EM forms are checked on: every n and K at the edges of the 8-wide
# serial sums and of the 256-thread blocks, then one table per shape
MATRIX = ([(10 + i, n, K, "random") for i, (n, K) in enumerate((n, K) for n in (1, 2, 7, 8, 9, 255, 256, 257) for K in (1, 255, 256, 257))]
          + [(1, 60, 400, "empty"), (1, 60, 400, "zero"), (1, 60, 400, "dups"), (1, 1000, 300, "wide"), (1, 300, 20000, "skew"),
             (1, 60, 400, "counts"), (1, 60, 400, "lengths"), (1, 60, 400, "singletons"), (2, 300, 500, "slow"), (1, 50, 300, "underflow"), (1, 20, 200, "nan")])


LARGE = (7, 4000, 87400, "bench")       # em_bench's generator at 262 660 contributions, just above the device threshold
BENCH = (7, 20000, 400000, "bench")     # tools/em_bench.py's own table: 1 200 732 contributions


def problem(seed, n, K, kind):
    """MATRIX entry -> table; kind "bench" is bench_problem(n, K)."""
    return bench_problem(n, K, seed) if kind == "bench" else random_problem(seed, n, K, kind)


def bench_problem(n=20000, K=400000, seed=7):
    """tools/em_bench.py's table: reads tie within "genera" of 10 neighbouring species (1-5 targets per key)."""
    rng = np.random.default_rng(seed)
    sz = rng.integers(1, 6, size=K)
    key_off = np.concatenate([[0], np.cumsum(sz)]).astype(np.uint64)
    g = rng.integers(0, n // 10, size=K)
    target = (np.repeat(g, sz) * 10 + rng.integers(0, 10, size=int(sz.sum()))).astype(np.uint32)
    count = rng.integers(1, 2000, size=K).astype(np.uint64)
    length = rng.integers(500000, 8000000, size=n).astype(np.uint64)
    p0 = rng.random(n); p0 /= p0.sum()
    return count, key_off, target, length, p0
