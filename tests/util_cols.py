"""Recorded reference outputs of the --tab-fmt-cols tests: the same scheme as util.reference (SHA-256 digests of what the
unmodified reference produced, re-recorded with CFB_RECORD_REFERENCE=1), kept in a file of their own,
tests/golden/tab_cols_digests.json."""
import atexit
import json
import os

import util

DIGESTS = os.path.join(util.GOLDEN, "tab_cols_digests.json")
_digests = None
_recorded = {}


def reference(key, run):
    """Digest of what the reference produced for the case named `key`; run() produces that output with the reference
    and is called only when recording."""
    global _digests
    if util.RECORD:
        if not util.have_ref():
            raise RuntimeError("CFB_RECORD_REFERENCE=1 needs the reference binaries under oracle/_ref (make -C oracle ref)")
        d = util.digest(run())
        if not _recorded:
            atexit.register(_save)
        _recorded[key] = d
        return d
    if _digests is None:
        with open(DIGESTS) as f:
            _digests = json.load(f)
    if key not in _digests:
        raise KeyError("no recorded reference output for %r (re-record, see tests/util.py)" % key)
    return _digests[key]


def _save():
    old = {}
    if os.path.exists(DIGESTS):
        with open(DIGESTS) as f:
            old = json.load(f)
    old.update(_recorded)
    with open(DIGESTS, "w") as f:
        json.dump(old, f, indent=0, sort_keys=True)
        f.write("\n")
