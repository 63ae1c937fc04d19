"""tools/pipe_census.py: the pipe classes it sorts SASS into, and that it finds the record and mark passes of the built
warp kernel (static, no GPU)."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pipe_census  # noqa: E402

LIB = os.path.join(ROOT, "peritext_b200", "libperitext_b200.so")


@pytest.mark.parametrize("text,cls", [
    ("ISETP.NE.AND P0, PT, R1, RZ, PT", "INT"),
    ("@!P0 LOP3.LUT R2, R2, 0x2, RZ, 0xfc, !PT", "INT"),
    ("VIADDMNMX.U32 R21, R31, 0x20, R14, PT", "INT"),
    ("IMAD.WIDE.U32 R20, R21, 0x4, R26", "IMAD"),
    ("@P1 IMAD.MOV.U32 R6, RZ, RZ, 0xffff", "IMAD"),
    ("ATOMS.OR RZ, [R6], R21", "mem"),
    ("LDG.E.64.CONSTANT R26, desc[UR8][R26.64]", "mem"),
    ("@!P0 BRA `(.L_x_1)", "ctrl"),
    ("VOTE.ANY R24, PT, P2", "shfl/vote"),
    ("UMOV UR4, 0xffffffff", "other"),
])
def test_pipe_class(text, cls):
    assert pipe_census.pipe_class(text) == cls


@pytest.mark.skipif(not (os.path.exists(LIB) and shutil.which("cuobjdump") and shutil.which("nvdisasm")),
                    reason="needs the built library and the CUDA binary tools")
def test_census_finds_both_passes():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pipe_census.py"), LIB], capture_output=True, text=True,
                         check=True).stdout
    assert "\nA+B: " in out and "\nG: " in out
