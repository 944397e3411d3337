"""What the compiler made of the CTU search's transform-unit path (no GPU needed): the functions that evaluate a
transform unit work on shared memory only (the team's arena slot, the shared tables, the context models), so their
SASS must reach it with LDS / STS, not with generic LD / ST, and must not touch the thread's stack (LDL / STL:
by-reference arguments, run-time-indexed local arrays, spills), which at three CTAs per SM has next to no L1 behind it.
Reads the SASS of the built library with cuobjdump / nvdisasm (tools/sass_census.py prints the whole census)."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kvazaar_b200", "libkvzcuda.so")
sys.path.insert(0, os.path.join(ROOT, "tools"))

# device functions by the name tools/ncu_ctu_summary.py gives them, a prefix standing for every template instance
SHARED_ONLY = ("rdoq_team", "rdoq_sign_hiding", "fwd_pass", "inv_pass", "dequant_block")
# The 4x4 instances have one caller each, tu_core_t<2>, and ptxas compiles them into its frame: they reload a few of its
# spilled values (LDL of the caller's slots, no STL of their own).  Those reloads may not grow.
LDL_ALLOWED = {"rdoq_teamILi2": 1, "dequant_blockILi2": 3}


@pytest.fixture(scope="module")
def census():
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not on PATH")
    if not os.path.exists(LIB):
        pytest.skip("kvazaar_b200/libkvzcuda.so not built")
    from sass_census import census as take
    return take(LIB)


def test_both_instantiations_present(census):
    assert sorted(census) == ["h", "t"], "ctu_frame_kernel<uint8_t> and <uint16_t> expected in the library"
    for kern, fns in census.items():
        for name in SHARED_ONLY:
            assert any(f.startswith(name) for f in fns), f"{name} is no function of its own in ctu_frame_kernel<{kern}>"


@pytest.mark.parametrize("name", SHARED_ONLY)
def test_transform_unit_path_addresses_shared_memory_as_shared(census, name):
    bad = []
    for kern, fns in sorted(census.items()):
        for f, c in sorted(fns.items()):
            if f.startswith(name) and (c["LD"] or c["ST"] or c["LDL"] > LDL_ALLOWED.get(f, 0) or c["STL"]):
                bad.append(f"ctu_frame_kernel<{kern}> {f}: LD {c['LD']} ST {c['ST']} LDL {c['LDL']} STL {c['STL']}")
    assert not bad, "generic or local memory instructions:\n" + "\n".join(bad)
