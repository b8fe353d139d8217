"""CPU checks of okb_detect_describe_store_batch's boundary: abi.DetectStoreJob against the header's struct (size and
every offset, as a C compiler lays it out), and the capi wrapper's exports."""
import ctypes as C
import os
import subprocess
import tempfile

from okvis_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("win", "feat_slot", "n_cams", "_pad", "images", "out_kp", "out_desc", "n_out")


def test_detect_store_job_layout_matches_header():
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"okvis_b200.h\"\nint main(void) {\n"
    src += '  printf("%zu", sizeof(okb_detect_store_job));\n'
    src += "".join('  printf(" %%zu", offsetof(okb_detect_store_job, %s));\n' % f for f in FIELDS)
    src += "  return 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "layout.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "layout"), os.path.join(d, "layout.c")])
        got = [int(v) for v in subprocess.check_output([os.path.join(d, "layout")], text=True).split()]
    assert got[0] == C.sizeof(abi.DetectStoreJob) == 48
    assert got[1:] == [getattr(abi.DetectStoreJob, f).offset for f in FIELDS]
