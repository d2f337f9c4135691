"""Every device allocation, pinned buffer, stream and event of the library is owned by the types of cf_buf.cuh (DBuf, HBuf,
Stream, Event), which free what they hold when they go.  No other source under centrifuge_b200/csrc allocates or frees one
itself, except cfb_host_alloc / cfb_host_free, which hand raw pinned memory to the caller."""
import os
import re

import util

CSRC = os.path.join(util.ROOT, "centrifuge_b200", "csrc")
RAW = re.compile(r"\b(cudaMalloc\w*|cudaHostAlloc|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
CODE = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
CALLER_OWNED = ("cfb_host_alloc", "cfb_host_free")


def code_only(text):
    """comments and string literals blanked to spaces, so line numbers stay"""
    return CODE.sub(lambda m: re.sub(r"[^\n]", " ", m.group(0)), text)


def without_bodies(text, names):
    """the bodies of the named function definitions blanked"""
    for name in names:
        for m in re.finditer(r"\b%s\s*\([^;{]*\)\s*\{" % name, text):
            depth, i = 0, m.end() - 1
            while True:
                depth += {"{": 1, "}": -1}.get(text[i], 0)
                if depth == 0:
                    break
                i += 1
            text = text[:m.end()] + re.sub(r"[^\n]", " ", text[m.end():i]) + text[i:]
    return text


def raw_calls(path):
    with open(path) as f:
        text = without_bodies(code_only(f.read()), CALLER_OWNED)
    return ["%s:%d: %s" % (os.path.basename(path), text.count("\n", 0, m.start()) + 1, m.group(1)) for m in RAW.finditer(text)]


def test_code_only_strips_comments_and_strings():
    text = 'a(); // cudaFree(x)\nb("cudaMalloc(") /* cudaEventDestroy(e)\n */ cudaFree(p);'
    got = code_only(text)
    assert got.count("\n") == text.count("\n")
    assert [m.group(1) for m in RAW.finditer(got)] == ["cudaFree"]
    assert [m.group(1) for m in RAW.finditer(without_bodies("void* cfb_host_alloc(size_t n) { if(1) { cudaHostAlloc(&p, n, 0); } }", CALLER_OWNED))] == []


def test_only_cf_buf_allocates_or_frees():
    found = []
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h", ".cpp")) and name != "cf_buf.cuh":
            found += raw_calls(os.path.join(CSRC, name))
    assert not found, "raw CUDA allocation, stream or event calls outside cf_buf.cuh:\n" + "\n".join(found)
    assert raw_calls(os.path.join(CSRC, "cf_buf.cuh"))      # the owners themselves are what the pattern finds
