"""The row kernels built into the library are exactly the layouts the row dispatch can select (tests/row_paths.py
mirrors it): no reachable layout is missing, and no unreachable one is compiled.  Reads the kernel names of the built
library with cuobjdump, which works without a GPU."""
import os
import re
import shutil
import sys

import pytest

from tests import row_paths as rp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNEL = re.compile(r"(vtrace_rows_fwd|upgo_rows_fwd|ppo_rows_fwd|softmax_grad_rows)(?:_(staged|loop))?(?:_kernel)?"
                    r"(?:<(\d+), (\d+), (true|false)>)?$")
FAMILY = {"vtrace_rows_fwd": "vtrace", "upgo_rows_fwd": "upgo", "ppo_rows_fwd": "ppo", "softmax_grad_rows": "grad"}


def built_layouts():
    from di_hpc_b200 import build
    from tools import sass_opcodes
    names = list(sass_opcodes.listing(build.build()))
    out = []
    for name in sass_opcodes.demangle(names):
        m = KERNEL.match(name)
        if not m:
            continue
        family, path, kmax, width, g1 = m.groups()
        if path:
            out.append((FAMILY[family], path))
        else:
            out.append((FAMILY[family], int(width), g1 == "true", int(kmax)))
    return out


def test_built_row_kernels_are_the_selectable_layouts():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not on PATH")
    built = built_layouts()
    assert len(built) == len(set(built))
    want = rp.row_layouts()
    assert set(built) == want, (sorted(set(built) - want, key=str), sorted(want - set(built), key=str))
    # per family: 34 register layouts, the staged and the looping kernel
    assert len(want) == 4 * 36
