"""CPU test of the ctypes mirrors in ``diff_gaussian_rasterization/_C.py`` against ``include/gsrast.h``: every struct the
header defines has a ``Structure`` of the same name with the same members in the same order, and the host C compiler
gives the same ``sizeof`` and the same ``offsetof`` for every member.  A mirror that is out of step with the header would
hand every pointer after the first wrong field to the wrong slot without any error."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "gsrast.h")


def header_structs():
    """{name: [member, ...]} for every ``typedef struct Name { ... } Name;`` in the header, members in order."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    for name, body, alias in re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*(\w+)\s*;", src, flags=re.S):
        assert name == alias, (name, alias)
        members = []
        for decl in body.split(";"):
            if decl.strip():
                members += [re.search(r"(\w+)\s*(\[[^\]]*\])?\s*$", part).group(1) for part in decl.split(",")]
        out[name] = members
    return out


def host_cc():
    for cc in (os.environ.get("CC"), "cc", "gcc", "clang"):
        if cc and shutil.which(cc):
            return cc
    return None


def test_ctypes_mirrors_match_the_header(tmp_path):
    cc = host_cc()
    if cc is None:
        pytest.skip("no host C compiler")
    from diff_gaussian_rasterization import _C
    structs = header_structs()
    assert "GsrForwardArgs" in structs and "GsrBackwardArgs" in structs
    for name, members in structs.items():
        assert hasattr(_C, name), f"{name} is defined in gsrast.h but has no ctypes mirror in _C.py"
        assert [f[0] for f in getattr(_C, name)._fields_] == members, name

    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "gsrast.h"', "int main(void) {"]
    for name, members in structs.items():
        lines.append(f'    printf("{name} sizeof %zu\\n", sizeof({name}));')
        lines += [f'    printf("{name} {m} %zu\\n", offsetof({name}, {m}));' for m in members]
    lines += ["    return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c11", "-I", os.path.dirname(HEADER), str(tmp_path / "layout.c"), "-o", str(exe)],
                   check=True, capture_output=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")

    want = []
    for name, members in structs.items():
        cls = getattr(_C, name)
        want.append(f"{name} sizeof {ctypes.sizeof(cls)}")
        want += [f"{name} {m} {getattr(cls, m).offset}" for m in members]
    assert got[:-1] == want
