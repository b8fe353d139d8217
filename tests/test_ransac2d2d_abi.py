"""CPU checks of okb_ransac_2d2d_batch's boundary: abi.Ransac2dJob / Ransac2dCam / Ransac2dResult and
ransac2d_outlier_dtype against the header's structs (size and every offset, as a C compiler lays them out), and the
capi wrapper's export."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from okvis_b200 import abi, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = [("okb_ransac2d_job", abi.Ransac2dJob), ("okb_ransac2d_cam", abi.Ransac2dCam),
           ("okb_ransac2d_result", abi.Ransac2dResult)]


def _layout(name, fields):
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"okvis_b200.h\"\nint main(void) {\n"
    src += '  printf("%%zu", sizeof(%s));\n' % name
    src += "".join('  printf(" %%zu", offsetof(%s, %s));\n' % (name, f) for f in fields)
    src += "  return 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "layout.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "layout"), os.path.join(d, "layout.c")])
        return [int(v) for v in subprocess.check_output([os.path.join(d, "layout")], text=True).split()]


def test_struct_layouts_match_header():
    for name, cls in STRUCTS:
        fields = [f for f, _ in cls._fields_]
        got = _layout(name, fields)
        assert got[0] == C.sizeof(cls), name
        assert got[1:] == [getattr(cls, f).offset for f in fields], name
    fields = list(abi.ransac2d_outlier_dtype.names)
    got = _layout("okb_ransac2d_outlier", fields)
    assert got[0] == abi.ransac2d_outlier_dtype.itemsize
    assert got[1:] == [abi.ransac2d_outlier_dtype.fields[f][1] for f in fields]


def test_capi_export():
    assert callable(capi.Context.ransac_2d2d_batch)
    assert hasattr(capi.lib(), "okb_ransac_2d2d_batch")
    assert np.dtype(abi.ransac2d_outlier_dtype).itemsize == 16
