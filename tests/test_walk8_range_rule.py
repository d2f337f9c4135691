"""walk8's range rule (DESIGN.md 3), checked on the host against one LF step at a time.

When both end rows of a range [top, bot) follow the read's next eight bases, the range after them is exactly
[W8(top), W8(bot - 1) + 1), whatever the rows in between do.  tests/native/walk8_rule.cpp restates k_build_walk8's entry on
the host twin of a committed index, takes random ranges (single rows to a few hundred rows, some with an end row within eight
steps of '$') and 16-base extensions, and compares every jump the rule accepts with the range the base-by-base walk reaches.
It also checks walk8_retry: every jump tried before it after a failed one fails too."""
import ctypes as C
import os
import subprocess

import pytest

import util


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("walk8_rule") / "walk8_rule.so")
    csrc = os.path.join(util.ROOT, "centrifuge_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(util.ROOT, "tests", "native", "walk8_rule.cpp"), os.path.join(csrc, "cf_index.cpp")])
    lib = C.CDLL(so)
    lib.w8_check.restype = C.c_longlong
    return lib


@pytest.mark.parametrize("name", ["adv", "example"])
def test_end_rows_decide_a_range_jump(checker, name):
    base = util.golden_index(name)
    st = (C.c_ulonglong * 9)()
    err = C.create_string_buffer(256)
    r = checker.w8_check(base.encode(), C.c_uint64(7), C.c_uint32(200000), st, err, C.c_size_t(256))
    assert r >= 0, err.value.decode()
    trials, ok, ok_range, ok_wide, narrowed, rejected, near_end, retries, bad = list(st)
    assert bad == 0 and r == 0, list(st)
    assert trials == 200000 and ok > 0 and rejected > 0 and retries > 0
    assert ok_range > 0 and ok_wide > 0           # ranges of width >= 5 jump
    assert narrowed > 0                           # ... including ranges whose interior rows drop out on the way
    assert near_end > 0                           # end rows that meet '$' within the eight steps
