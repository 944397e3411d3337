"""What the compiler made of the CTU search above the transform-unit jobs (no GPU needed): the search spine, the rough
search and the leader's cost walks take the CTA's shared state block (CtuST) instead of a context on the caller's
stack, and reach it through sm(), so the leader's serial sections load and store with LDS / STS.  Reads the SASS of the
built library with cuobjdump / nvdisasm (tools/sass_census.py prints the whole census)."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kvazaar_b200", "libkvzcuda.so")
sys.path.insert(0, os.path.join(ROOT, "tools"))

INST = ("h", "t")       # ctu_frame_kernel<uint8_t>, <uint16_t>: the suffix tools/ncu_ctu_summary.py gives the functions

# leader functions that only touch shared state: no generic and no local memory instructions.  mock_encode_coding_unit
# and cu_rd_cost_luma_leaf keep a few reloads of their caller's spill slots (LDL, no STL of their own): they may not grow.
LEADER_SHARED_ONLY = ("cost_accurate_node", "cost_tr_split_accurate", "cu_rd_cost_luma_leaf", "cu_rd_cost_chroma_leaf",
                      "cu_rd_cost_chroma_leaf_of_level", "mock_encode_coding_unit", "rough_search_replay", "rough_mode_costs")
LDL_ALLOWED = {"mock_encode_coding_unit": 6, "cu_rd_cost_luma_leaf": 3}

# rough_costs_all_modes: its only generic loads are those of the source block (global memory)
ROUGH_LD_MAX = 160

# the search spine: its stack traffic (by-reference arguments, spills) may not grow past {instantiation: (LDL, STL)}
SPINE_LOCAL_MAX = {
    "search_ctu": {"h": (120, 25), "t": (120, 25)},
    "search_cu_intra": {"h": (138, 64), "t": (138, 64)},
    "intra_recon_leaf": {"h": (132, 88), "t": (135, 92)},
    "search_cu_intra_chroma": {"h": (34, 6), "t": (47, 7)},
    "intra_recon_cu": {"h": (13, 33), "t": (13, 33)},
}


@pytest.fixture(scope="module")
def census():
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not on PATH")
    if not os.path.exists(LIB):
        pytest.skip("kvazaar_b200/libkvzcuda.so not built")
    from sass_census import census as take
    return take(LIB)


def fn(census, name, kern):
    """The census row of function `name` in ctu_frame_kernel<kern>; it must be a function of its own."""
    f = census[kern].get(name + ("Ih" if kern == "h" else "It"))
    assert f is not None, f"{name} is no function of its own in ctu_frame_kernel<{kern}>"
    return f


@pytest.mark.parametrize("name", LEADER_SHARED_ONLY)
def test_leader_cost_walks_address_shared_memory_as_shared(census, name):
    bad = []
    for kern in INST:
        c = fn(census, name, kern)
        if c["LD"] or c["ST"] or c["LDL"] > LDL_ALLOWED.get(name, 0) or c["STL"]:
            bad.append(f"ctu_frame_kernel<{kern}> {name}: LD {c['LD']} ST {c['ST']} LDL {c['LDL']} STL {c['STL']}")
    assert not bad, "generic or local memory instructions:\n" + "\n".join(bad)


def test_rough_search_reads_only_its_source_generically(census):
    for kern in INST:
        c = fn(census, "rough_costs_all_modes", kern)
        assert not (c["ST"] or c["LDL"] or c["STL"]), f"ctu_frame_kernel<{kern}> rough_costs_all_modes: {c}"
        assert c["LD"] <= ROUGH_LD_MAX, f"ctu_frame_kernel<{kern}> rough_costs_all_modes: {c['LD']} generic loads"


@pytest.mark.parametrize("name", sorted(SPINE_LOCAL_MAX))
def test_search_spine_stack_traffic_does_not_grow(census, name):
    for kern in INST:
        c = fn(census, name, kern)
        ldl, stl = SPINE_LOCAL_MAX[name][kern]
        assert c["LDL"] <= ldl and c["STL"] <= stl, \
            f"ctu_frame_kernel<{kern}> {name}: LDL {c['LDL']} STL {c['STL']}, at most {ldl} / {stl}"
