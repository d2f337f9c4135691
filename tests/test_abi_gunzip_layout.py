"""cfb_gunzip_state, the resume state of the gzip inflater, against its ctypes mirror (capi.GunzipState): a C probe
compiled against include/cfb200.h prints the size and every field offset."""
import ctypes as C
import os
import subprocess

import util

FIELDS = ("in_offset", "out_offset", "bit", "hdr_bit", "member_bytes", "crc", "win_len", "phase", "members", "window")


def test_gunzip_state_matches_the_c_header(tmp_path):
    from centrifuge_b200 import capi
    src = tmp_path / "probe.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"cfb200.h\"\nint main(void) {\n"
                   + '  printf("size %zu\\n", sizeof(cfb_gunzip_state));\n'
                   + "".join('  printf("%s %%zu\\n", offsetof(cfb_gunzip_state, %s));\n' % (f, f) for f in FIELDS)
                   + "  return 0;\n}\n")
    exe = str(tmp_path / "probe")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(util.ROOT, "include"), "-o", exe, str(src)])
    got = dict((k, int(v)) for k, v in (l.split() for l in subprocess.check_output([exe]).decode().splitlines()))
    assert got.pop("size") == C.sizeof(capi.GunzipState)
    assert got == {f: getattr(capi.GunzipState, f).offset for f in FIELDS}
