"""The hardware claims of DESIGN.md, checked on the built library itself (cuobjdump works without a GPU): sm_90a only,
TMA tensor loads AND stores in the headline GAE kernels, bulk copies where the docs say so -- and no floating-point
atomic anywhere (every reduction has a fixed order)."""
import os
import re
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from di_hpc_b200 import build
    from tools import sass_opcodes
    lib = build.build()
    kernels, atomics, arch = sass_opcodes.parse(lib)
    assert len(kernels) > 100
    return kernels, atomics, arch


def pick(kernels, fragment):
    hit = {k: c for k, c in kernels.items() if fragment in k}
    assert hit, "no kernel matching %r in the library" % fragment
    return hit


def test_only_sm_90a_cubins(sass):
    _, _, arch = sass
    assert arch == {"sm_90a"}, arch


def test_headline_gae_kernels_use_tma_loads_and_tma_stores(sass):
    kernels, _, _ = sass
    for frag in ("gae_fwd_tma_st", "gae_bwd_tma_st"):
        for name, c in pick(kernels, frag).items():
            assert c["UTMALDG"] > 0 and c["UTMASTG"] > 0 and c["SYNCS"] > 0, (name, c["UTMALDG"], c["UTMASTG"])


def test_scan_kernels_of_the_other_ops_use_tma_loads(sass):
    kernels, _, _ = sass
    for frag in ("td_lambda_fwd_tma", "vtrace_scan_tma", "upgo_scan_tma"):
        for name, c in pick(kernels, frag).items():
            assert c["UTMALDG"] > 0, name


def test_c51_lane_kernel_gathers_with_tma_and_stores_in_bulk(sass):
    kernels, _, _ = sass
    for name, c in pick(kernels, "dist_nstep_fwd_lane_kernel").items():
        assert c["UTMALDG"] > 0 and c["UBLKCP"] > 0, (name, dict(c))


def test_backward_scatter_writes_with_bulk_copies(sass):
    kernels, _, _ = sass
    for name, c in pick(kernels, "scatter_rows_bulk_kernel").items():
        assert c["UBLKCP"] > 0 and c["STG"] <= 8, (name, c["UBLKCP"], c["STG"])  # (STG: the tail rows only)


def test_no_floating_point_atomics(sass):
    _, atomics, _ = sass
    for name, ops in atomics.items():
        for op in ops:
            assert ".F32" not in op and ".F64" not in op and ".F16" not in op, (name, op)
        # the only kernels with atomics at all are the ticket / done counters of the look-back scans
        assert "lookback" in name, (name, sorted(ops))


def test_against_compares_instruction_lines_with_anonymous_namespace_masked(sass, capsys):
    from di_hpc_b200 import build
    from tools import sass_opcodes
    kernels, _, _ = sass
    lib = build.build()
    listing = sass_opcodes.listing(lib)
    assert len(listing) == len(kernels)
    assert sum(map(len, listing.values())) == sum(c["_total"] for c in kernels.values())
    assert not [k for k in listing if re.search(r"_GLOBAL__N__[0-9a-f]{8}_", k)]
    assert sass_opcodes.against(lib, lib) == 0
    assert "instruction text differs: 0" in capsys.readouterr().out
