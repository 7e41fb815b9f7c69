"""
The ctypes mirrors of the C ABI's argument structs (``lkpy_b200/_lib.py``) have the layout the header
declares: a C program compiled against ``include/lkpy_b200.h`` prints every field offset and struct size,
and each must equal what ``ctypes`` computes.  A field added, removed, reordered or retyped on one side
only would otherwise pass garbage to the kernels without any error.  CPU only.
"""

import ctypes as C
import shutil
import subprocess
from pathlib import Path

from lkpy_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
STRUCTS = {
    "lk_als_args": _lib.LkAlsArgs,
    "lk_knn_geom": _lib.LkKnnGeom,
    "lk_knn_build_args": _lib.LkKnnBuildArgs,
    "lk_knn_score_args": _lib.LkKnnScoreArgs,
}


def test_ctypes_structs_match_header(tmp_path):
    expected, lines = [], []
    for cname, cls in STRUCTS.items():
        for field in cls._fields_:
            name = field[0]
            expected.append((f"{cname}.{name}", getattr(cls, name).offset))
            lines.append(f'    printf("{cname}.{name} %zu\\n", offsetof({cname}, {name}));')
        expected.append((f"sizeof {cname}", C.sizeof(cls)))
        lines.append(f'    printf("sizeof {cname} %zu\\n", sizeof({cname}));')
    src = tmp_path / "layout.c"
    src.write_text(
        "#include <stddef.h>\n#include <stdio.h>\n#include \"lkpy_b200.h\"\n\nint main(void)\n{\n"
        + "\n".join(lines)
        + "\n    return 0;\n}\n"
    )
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to read the header's layout"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    got = [(line.rsplit(" ", 1)[0], int(line.rsplit(" ", 1)[1])) for line in out]
    assert got == expected
