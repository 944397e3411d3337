"""Fractional motion search (include/kvz_cuda.h: kvz_cuda_me_frac_search_batch; search_frac, src/search_inter.c:974-1168).

Checker: the UNMODIFIED reference's own search_frac (oracle/ref_me.c includes src/search_inter.c where it lies; its filter
stages, kvz_get_extended_block and SATD functions are the compiled reference's selected strategies) and its committed
outputs (tests/golden/me_search.npz, `frac/...`).  CPU: the host build of the device code (TEST INFRASTRUCTURE); GPU: the
product through the C ABI.  Bar: best MV, bits and cost identical for every PU -- incl. the AMP heights (16x12, 16x4)
where the reference's four-candidate SATD counts rows 0-7 twice, and the truncation of the MV cost into its unsigned
cost accumulator.  (The file sorts last on purpose: this kernel was written after the round's GPU budget was spent, its
`-m gpu` tests run for the first time at the round-end check.)
"""
import ctypes as C
import os

import numpy as np
import pytest

from _me_cases import (MC_CASES, make_mc_case, mc_refs_struct, run_mc_host_api, run_mc_reference, BIPRED_CASES, BIPRED_RESULT, CASES, FRAC_CASES, GPU_FIRST_RUN_DONE, MERGE_CASES, MERGE_COST, RESULT, make_bipred_case, make_merge_case,
                       merge_refs_struct, run_bipred_host_api, run_bipred_reference, run_merge_host_api, run_merge_reference)
from _me_cases import grid_case, make_frac_case, run_frac_host_api, run_frac_reference, run_host_api, run_reference, same
from test_me_search import _explain, _hostsim, check_cuda_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", "me_search.npz"))
    out = np.zeros(len(g["frac/" + name + "/bits"]), RESULT)
    out["mv"], out["bits"], out["cost"] = g["frac/" + name + "/mv"], g["frac/" + name + "/bits"], g["frac/" + name + "/cost"]
    return out


@pytest.mark.parametrize("name", sorted(FRAC_CASES))
def test_reference_matches_golden(name, ref, ref10):
    p, level, cur, rf, pus = make_frac_case(name)
    want = run_frac_reference(ref if p.bitdepth == 8 else ref10, p, level, cur, rf, pus)
    assert same(want, _golden(name)), _explain(want, _golden(name), pus)


@pytest.mark.parametrize("name", sorted(FRAC_CASES))
def test_hostbuild_matches_golden(name):
    p, level, cur, rf, pus = make_frac_case(name)
    got = run_frac_host_api(_hostsim(), p, level, cur, rf, pus)
    assert same(got, _golden(name)), _explain(got, _golden(name), pus)
    assert ((got["mv"] % 4) != 0).any(1).mean() > 0.25          # fractional positions do win


def test_hostbuild_integer_then_fractional_matches_reference(ref):
    """the chain of search_pu_inter: integer search, then search_frac from its result (--preset slow: hexbs, subme 4)"""
    p, cur, rf, pus = grid_case(208, 136, 8, 8)
    lib = _hostsim()
    integer = run_host_api(lib, p, cur, rf, pus)
    assert same(integer, run_reference(ref, p, cur, rf, pus))
    pus2 = pus.copy()
    pus2["start_mv"] = integer["mv"]
    got, want = run_frac_host_api(lib, p, 4, cur, rf, pus2), run_frac_reference(ref, p, 4, cur, rf, pus2)
    assert same(got, want), _explain(got, want, pus2)


# ---- merge analysis (kvz_cuda_me_merge_cost_batch; search_pu_inter's merge loop, src/search_inter.c:1667-1730)
def _golden_merge(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", "me_search.npz"))
    return g["merge/" + name].view(MERGE_COST), tuple(g["merge/" + name + "/bits"])


def _explain_merge(got, want, pus):
    bad = [i for i in range(len(pus)) if got[i].tobytes() != want[i].tobytes()]
    i = bad[0]
    return f"{len(bad)} of {len(pus)} PUs differ; first: PU {i} {pus[i]}\n got  {got[i]}\n want {want[i]}"


@pytest.mark.parametrize("name", sorted(MERGE_CASES))
def test_merge_reference_matches_golden(name, ref, ref10):
    p, c, cur, planes, pus, cu = make_merge_case(name)
    want, bits = run_merge_reference(ref if p.bitdepth == 8 else ref10, p, c, cur, planes, pus, cu)
    gold, gbits = _golden_merge(name)
    assert bits == gbits and want.tobytes() == gold.tobytes(), _explain_merge(want, gold, pus)


@pytest.mark.parametrize("name", sorted(MERGE_CASES))
def test_merge_hostbuild_matches_golden(name):
    p, c, cur, planes, pus, _ = make_merge_case(name)
    gold, bits = _golden_merge(name)
    got = run_merge_host_api(_hostsim(), p, c, cur, planes, pus, bits)
    assert got.tobytes() == gold.tobytes(), _explain_merge(got, gold, pus)
    assert got["size"].max() >= 3 and got["size"].min() <= 1           # several accepted candidates; PUs where (almost) none may be used


# ---- bi-prediction from the two best uni-predictions (kvz_cuda_me_bipred_batch; src/search_inter.c:1937-2031)
def _golden_bipred(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", "me_search.npz"))
    return g["bipred/" + name].view(BIPRED_RESULT)


@pytest.mark.parametrize("name", sorted(BIPRED_CASES))
def test_bipred_reference_and_hostbuild_match_golden(name, ref, ref10):
    p, c, cur, planes, pus = make_bipred_case(name)
    want = run_bipred_reference(ref if p.bitdepth == 8 else ref10, p, c, cur, planes, pus)
    assert want.tobytes() == _golden_bipred(name).tobytes()
    got = run_bipred_host_api(_hostsim(), p, c, cur, planes, pus)
    bad = [i for i in range(len(pus)) if got[i].tobytes() != want[i].tobytes()]
    assert not bad, (len(bad), pus[bad[0]], got[bad[0]], want[bad[0]])
    assert bool(want["valid"].any()) == bool(c["bipred"])


# ---- motion compensation (kvz_cuda_me_predict_batch; kvz_inter_pred_pu luma + chroma, src/inter.c:604-668)
def _mc_digest(planes3):
    import hashlib
    return np.frombuffer(b"".join(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest() for a in planes3), np.uint8)


def _golden_mc(name):
    return np.load(os.path.join(ROOT, "tests", "golden", "me_search.npz"))["mc/" + name]


@pytest.mark.parametrize("name", sorted(MC_CASES))
def test_mc_reference_and_hostbuild_match_golden(name, ref, ref10):
    p, c, planes, us, vs, pus, cu = make_mc_case(name)
    want = run_mc_reference(ref if p.bitdepth == 8 else ref10, p, c, planes, us, vs, pus, cu)
    assert np.array_equal(_mc_digest(want), _golden_mc(name))
    got = run_mc_host_api(_hostsim(), p, c, planes, us, vs, pus)
    for g, w_, what in zip(got, want, "YUV"):
        assert np.array_equal(g, w_), (what, int((g != w_).sum()))
    assert (want[0] != 0).mean() > 0.99                       # the PUs tile the whole picture


# ------------------------------------------------------------------------------------------------ GPU (the product)
LATER = sorted(set(CASES) - set(GPU_FIRST_RUN_DONE))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in LATER if "satd_final" not in n])
def test_cuda_integer_search_cases_added_later(cuda_lib, name, ref, ref10):
    """tz and full search cases of tools/me_cases.py (added after the first search cases; same check_mv primitive)"""
    check_cuda_case(cuda_lib, name, ref, ref10)


def _dev(kb, p, level, cur, rf, pus):
    import torch
    out = kb.me_frac_search_batch(p, level, kb.to_dev(cur), kb.to_dev(rf), kb.to_dev(pus))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(RESULT).copy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FRAC_CASES))
def test_cuda_matches_golden_and_reference(cuda_lib, name, ref, ref10):
    kb = cuda_lib
    p, level, cur, rf, pus = make_frac_case(name)
    got = _dev(kb, p, level, cur, rf, pus)
    assert same(got, _golden(name)), _explain(got, _golden(name), pus)
    want = run_frac_reference(ref if p.bitdepth == 8 else ref10, p, level, cur, rf, pus)
    assert same(got, want), _explain(got, want, pus)
    got_host = run_frac_host_api(C.CDLL(kb.LIB_PATH), p, level, cur, rf, pus)           # host-buffer entry
    assert same(got_host, want)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,bd,size", [(1920, 1080, 8, 16), (832, 480, 10, 32), (1920, 1080, 8, 64)])
def test_cuda_integer_then_fractional_full_picture(cuda_lib, ref, ref10, w, h, bd, size):
    """every PU of a picture: integer search on the device, fractional search from its result, both against the reference"""
    import torch
    kb = cuda_lib
    shim = ref if bd == 8 else ref10
    p, cur, rf, pus = grid_case(w, h, bd, size)
    d_cur, d_ref = kb.to_dev(cur), kb.to_dev(rf)
    integer = kb.me_search_batch(p, d_cur, d_ref, kb.to_dev(pus)).cpu().numpy().view(RESULT).copy()
    assert same(integer, run_reference(shim, p, cur, rf, pus))
    pus2 = pus.copy()
    pus2["start_mv"] = integer["mv"]
    got = kb.me_frac_search_batch(p, 4, d_cur, d_ref, kb.to_dev(pus2))
    torch.cuda.synchronize()
    got = got.cpu().numpy().view(RESULT).copy()
    want = run_frac_reference(shim, p, 4, cur, rf, pus2)
    assert same(got, want), _explain(got, want, pus2)



@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in LATER if "satd_final" in n])
def test_cuda_integer_search_with_final_hadamard_cost(cuda_lib, name, ref, ref10):
    """cfg.fme_level == 0: the integer kernel's second instantiation (winner's cost recomputed with the Hadamard cost)"""
    check_cuda_case(cuda_lib, name, ref, ref10)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MERGE_CASES))
def test_cuda_merge_analysis_matches_golden_and_reference(cuda_lib, name, ref, ref10):
    import torch
    kb = cuda_lib
    p, c, cur, planes, pus, cu = make_merge_case(name)
    want, bits = run_merge_reference(ref if p.bitdepth == 8 else ref10, p, c, cur, planes, pus, cu)
    d_planes = [kb.to_dev(pl) for pl in planes]
    rf = merge_refs_struct(c, [t.data_ptr() for t in d_planes], p.width, bits)
    out = kb.me_merge_cost_batch(p, rf, kb.to_dev(cur), kb.to_dev(pus))
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(MERGE_COST).copy()
    assert got.tobytes() == want.tobytes(), _explain_merge(got, want, pus)
    assert got.tobytes() == _golden_merge(name)[0].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BIPRED_CASES))
def test_cuda_bipred_matches_golden_and_reference(cuda_lib, name, ref, ref10):
    import torch
    kb = cuda_lib
    p, c, cur, planes, pus = make_bipred_case(name)
    want = run_bipred_reference(ref if p.bitdepth == 8 else ref10, p, c, cur, planes, pus)
    d_planes = [kb.to_dev(pl) for pl in planes]
    rf = merge_refs_struct(c, [t.data_ptr() for t in d_planes], p.width, (0.0, 0.0, 0.0))
    out = kb.me_bipred_batch(p, rf, kb.to_dev(cur), kb.to_dev(pus))
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(BIPRED_RESULT).copy()
    assert got.tobytes() == want.tobytes() and got.tobytes() == _golden_bipred(name).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MC_CASES))
def test_cuda_motion_compensation_matches_golden_and_reference(cuda_lib, name, ref, ref10):
    import torch
    kb = cuda_lib
    p, c, planes, us, vs, pus, cu = make_mc_case(name)
    want = run_mc_reference(ref if p.bitdepth == 8 else ref10, p, c, planes, us, vs, pus, cu)
    dy, du, dv = [kb.to_dev(a) for a in planes], [kb.to_dev(a) for a in us], [kb.to_dev(a) for a in vs]
    rf = mc_refs_struct(c, [t.data_ptr() for t in dy], [t.data_ptr() for t in du], [t.data_ptr() for t in dv])
    oy, ou, ov = [torch.zeros_like(t) for t in (dy[0], du[0], dv[0])]
    kb.me_predict_batch(p, rf, kb.to_dev(pus), oy, ou, ov)
    torch.cuda.synchronize()
    got = [t.cpu().numpy().view(planes[0].dtype) for t in (oy, ou, ov)]
    for g, w_, what in zip(got, want, "YUV"):
        assert np.array_equal(g, w_), (what, int((g != w_).sum()))
    assert np.array_equal(_mc_digest(got), _golden_mc(name))


# ------------------------------------------------------------------------------------------------ CTU driver, chroma mode search
@pytest.mark.gpu
def test_cuda_ctu_driver_chroma_mode_search(cuda_lib, tmp_path):
    """the --intra-chroma-search fix of the CTU driver (scan order of the candidates; CPU: tests/test_ctu_driver.py) on the device"""
    import test_ctu_driver as T
    T._identity(tmp_path, cuda_lib.LIB_PATH, 264, 136, 1, "veryslow", 15, True, extra=("--intra-chroma-search",))


# ------------------------------------------------------------------------------------------------ 10-bit drop-in encode
# (kept in this last file for the same reason: first hardware run at the round-end check)
def _tenbit_encode(tmp_path, cuda):
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from synth_yuv import synth_frame
    enc = os.path.join(ROOT, "oracle", "_ref", "kvz_cuda_encode_10b")
    if not os.path.exists(enc):
        pytest.skip("oracle/_ref/kvz_cuda_encode_10b missing (make -C integration needs /root/reference)")
    w, h = 128, 64
    clip = str(tmp_path / "in.yuv")
    with open(clip, "wb") as f:
        for i in range(3):
            f.write(synth_frame(w, h, 1234, i).tobytes())
    out = str(tmp_path / ("cuda.hevc" if cuda else "host.hevc"))
    cmd = [enc] + (["--cuda"] if cuda else []) + [clip, f"{w}x{h}", out, "preset=fast", "qp=30", "period=16", "gop=0", "threads=2", "owf=1"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1500:]
    return open(out, "rb").read(), r.stderr, clip, (w, h)


def test_tenbit_host_program_matches_reference_cli(tmp_path):
    """the 10-bit build of the drop-in host (8-bit input scaled to 10 bits) writes what the 10-bit reference CLI writes"""
    import subprocess
    cli = os.path.join(ROOT, "oracle", "_ref", "kvazaar_10b")
    if not os.path.exists(cli):
        pytest.skip("oracle/_ref/kvazaar_10b missing")
    a, _, clip, (w, h) = _tenbit_encode(tmp_path, cuda=False)
    out = str(tmp_path / "cli.hevc")
    r = subprocess.run([cli, "-i", clip, "--input-res", f"{w}x{h}", "-o", out, "--preset", "fast", "-q", "30", "-p", "16", "--gop", "0", "--threads", "2",
                        "--owf", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1500:]
    assert len(a) > 100 and a == open(out, "rb").read()


@pytest.mark.gpu
def test_tenbit_bitstream_identical_with_cuda_strategies(cuda_lib, tmp_path):
    """VERDICT r1 item 3: the 10-bit reference encoder (inter, FME, bipred) with every strategy pointer bound to CUDA"""
    import re
    a, _, _, _ = _tenbit_encode(tmp_path, cuda=False)
    b, log, _, _ = _tenbit_encode(tmp_path, cuda=True)
    m = re.search(r"(\d+) strategy pointers bound", log)
    assert m and int(m.group(1)) >= 60, log[-1500:]
    assert len(a) > 100 and a == b, f"10-bit bitstreams differ ({len(a)} vs {len(b)} bytes)"
