"""CTU search driver (include/kvz_cuda_ctu.h): bitstream identity with the unmodified reference encoder.

The reference CLI is linked twice from the same unmodified sources (oracle/Makefile): `kvazaar` (all reference) and
`kvazaar_ctu` (the four CTU-job functions redirected to a provider of the kvz_cuda_ctu_* ABI by
integration/kvz_ctu_hooks.c).  The provider is
  * CPU tests: tests/hostsim/libkvzctu_hostsim.so -- the driver's single-source algorithm (csrc/ctu/*.h) compiled for
    the host with a one-thread "CTA" (TEST INFRASTRUCTURE: checks the control flow without a GPU);
  * GPU tests: kvazaar_b200/libkvzcuda.so -- the product.
Gate: `cmp` of the .hevc files (BASELINE.md 3, steps 4-5), and `verify` mode (the reference searches as well and
every CU field / coefficient / SAO parameter / context model is compared per CTU).
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
HOSTSIM = os.path.join(ROOT, "tests", "hostsim", "libkvzctu_hostsim.so")
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _need(*names):
    paths = [os.path.join(REF_DIR, n) for n in names]
    for p in paths:
        if not os.path.exists(p):
            pytest.skip(f"{p} missing (make -C oracle ref ctu needs /root/reference)")
    return paths


def _hostsim():
    if not os.path.exists(HOSTSIM):
        src = os.path.join(ROOT, "tests", "hostsim", "ctu_hostsim.cpp")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unused-function", "-Wno-unknown-pragmas",
                               "-o", HOSTSIM, src])
    return HOSTSIM


def _clip(tmp_path, w, h, frames, noisy=False):
    from synth_yuv import synth_frame, noisy_frame
    p = str(tmp_path / f"clip_{w}x{h}_{frames}{'n' if noisy else ''}.yuv")
    f = noisy_frame if noisy else synth_frame
    seed = 5 if noisy else 1234
    with open(p, "wb") as fh:
        for i in range(frames):
            fh.write(f(w, h, seed, i).tobytes())
    return p


def _encode(binary, clip, w, h, out, preset, qp, env=None, extra=()):
    e = dict(os.environ)
    e.pop("KVZ_CTU_PROVIDER", None)
    e.pop("KVZ_CTU_MODE", None)
    e.update(env or {})
    r = subprocess.run([binary, "-i", clip, "--input-res", f"{w}x{h}", "-o", out, "--preset", preset, "-q", str(qp), "-p", "1", *extra],
                       env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1500)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stderr


def _identity(tmp_path, provider, w, h, frames, preset, qp, noisy=False, extra=(), verify=True, clip=None):
    ref_bin, ctu_bin = _need("kvazaar", "kvazaar_ctu")
    clip = clip or _clip(tmp_path, w, h, frames, noisy)
    a, b = str(tmp_path / "ref.hevc"), str(tmp_path / "ctu.hevc")
    _encode(ref_bin, clip, w, h, a, preset, qp, extra=extra)
    log = _encode(ctu_bin, clip, w, h, b, preset, qp, env={"KVZ_CTU_PROVIDER": provider}, extra=extra)
    assert "CTU search driver active" in log, log[-1500:]
    ra, rb = open(a, "rb").read(), open(b, "rb").read()
    assert len(ra) > 100
    assert ra == rb, f"bitstreams differ ({len(ra)} vs {len(rb)} bytes)"
    if verify:
        log = _encode(ctu_bin, clip, w, h, str(tmp_path / "ver.hevc"), preset, qp,
                      env={"KVZ_CTU_PROVIDER": provider, "KVZ_CTU_MODE": "verify", "KVZ_CUDA_CTU_DEBUG": "1"}, extra=extra)
        m = re.search(r"verify finished, (\d+) mismatches", log)
        assert m and int(m.group(1)) == 0, log[-3000:]
    return len(ra)


# ------------------------------------------------------------------------------------------------ CPU (host build)
def test_abi_header_matches_both_providers():
    """every function include/kvz_cuda_ctu.h declares is exported by libkvzcuda.so and by the host test build"""
    txt = open(os.path.join(ROOT, "include", "kvz_cuda_ctu.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    names = sorted(set(re.findall(r"\b(kvz_cuda_ctu_[a-z0-9_]+)\s*\(", txt)))
    assert len(names) >= 7
    import kvazaar_b200 as kb
    for path in (kb.LIB_PATH, _hostsim()):
        lib = C.CDLL(path)
        missing = [n for n in names if not hasattr(lib, n)]
        assert not missing, (path, missing)


@pytest.mark.parametrize("w,h,frames,preset,qp,noisy", [
    (64, 64, 3, "ultrafast", 32, False),        # BASELINE config 1
    (264, 200, 2, "medium", 27, False),         # partial CTUs on both edges; rd=0, RDOQ, SAO
    (264, 200, 1, "veryslow", 22, False),       # rd=3: RDO of candidates, chroma search, sign hiding, transform skip
    (136, 72, 1, "veryslow", 22, True),         # high levels, band SAO, transform skip picked
    (200, 136, 1, "medium", 27, True),
    (128, 128, 1, "slow", 37, False),           # rd=1; coarse QP: zero CBFs, early termination
    (128, 64, 2, "faster", 22, False),
])
def test_hostbuild_bitstream_identical(tmp_path, w, h, frames, preset, qp, noisy):
    _identity(tmp_path, _hostsim(), w, h, frames, preset, qp, noisy)


@pytest.mark.parametrize("w,h,preset,qp,noisy", [(136, 72, "veryslow", 15, True), (264, 136, "slower", 29, True), (192, 64, "veryslow", 15, False)])
def test_hostbuild_chroma_mode_search(tmp_path, w, h, preset, qp, noisy):
    """--intra-chroma-search (no preset sets it): the candidates are predicted with their own mode but quantised and costed
    in the scan order of the mode the CU record still holds (the luma mode) -- found by tools/sweep_ctu_hostsim.py"""
    _identity(tmp_path, _hostsim(), w, h, 1, preset, qp, noisy, extra=("--intra-chroma-search",))


def test_hostbuild_out_of_scope_falls_through(tmp_path):
    """a configuration outside the driver's scope (inter pictures) must run the reference path untouched"""
    ref_bin, ctu_bin = _need("kvazaar", "kvazaar_ctu")
    clip = _clip(tmp_path, 128, 64, 3)
    a, b = str(tmp_path / "a.hevc"), str(tmp_path / "b.hevc")
    args = dict(w=128, h=64, preset="ultrafast", qp=30)
    for binary, out, env in ((ref_bin, a, None), (ctu_bin, b, {"KVZ_CTU_PROVIDER": _hostsim()})):
        e = dict(os.environ)
        e.update(env or {})
        r = subprocess.run([binary, "-i", clip, "--input-res", "128x64", "-o", out, "--preset", "ultrafast", "-q", "30", "-p", "8"],
                           env=e, stderr=subprocess.PIPE, text=True, timeout=300)
        assert r.returncode == 0
        assert "CTU search driver active" not in r.stderr
    assert open(a, "rb").read() == open(b, "rb").read()
    del args


# ------------------------------------------------------------------------------------------------ GPU (the product)
def _cuda_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import kvazaar_b200 as kb
    return kb.LIB_PATH


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,frames,preset,qp,noisy", [
    (64, 64, 3, "ultrafast", 32, False),        # BASELINE config 1 at its named size
    (264, 200, 2, "medium", 27, False),
    (264, 200, 2, "veryslow", 22, False),
    (264, 200, 2, "veryslow", 22, True),
    (264, 200, 2, "medium", 27, True),
    (832, 480, 3, "slow", 32, False),
    (416, 240, 2, "veryslow", 37, True),
])
def test_cuda_bitstream_identical_small(tmp_path, w, h, frames, preset, qp, noisy):
    _identity(tmp_path, _cuda_lib(), w, h, frames, preset, qp, noisy)


@pytest.mark.gpu
def test_cuda_bitstream_identical_config2_1080p_medium(tmp_path):
    """BASELINE config 2 at its named size: 1920x1080 --preset medium -q 27 -p 1, 16 frames"""
    _identity(tmp_path, _cuda_lib(), 1920, 1080, 16, "medium", 27, verify=False)


@pytest.mark.gpu
def test_cuda_bitstream_identical_config3_2160p_veryslow(tmp_path):
    """BASELINE config 3 (the headline) at its named size: 3840x2160 --preset veryslow -q 22 -p 1, 8 frames"""
    _identity(tmp_path, _cuda_lib(), 3840, 2160, 8, "veryslow", 22, verify=False)


# ------------------------------------------------------------------------------------------------ golden bitstreams
# tests/golden/ctu_bitstreams.json: sha256 of what the unmodified reference writes (tools/make_golden_bitstreams.py, run in
# the container that has /root/reference); these tests need neither /root/reference nor the plain reference binary.
def _golden():
    import json
    return json.load(open(os.path.join(ROOT, "tests", "golden", "ctu_bitstreams.json")))


def _golden_check(tmp_path, provider, name):
    import hashlib
    g = _golden()[name]
    (ctu_bin,) = _need("kvazaar_ctu")
    clip = _clip(tmp_path, g["w"], g["h"], g["frames"], g["noisy"])
    out = str(tmp_path / "g.hevc")
    log = _encode(ctu_bin, clip, g["w"], g["h"], out, g["preset"], g["qp"], env={"KVZ_CTU_PROVIDER": provider})
    assert "CTU search driver active" in log
    data = open(out, "rb").read()
    assert len(data) == g["bytes"] and hashlib.sha256(data).hexdigest() == g["sha256"], name


@pytest.mark.parametrize("name", sorted(_golden()))
def test_hostbuild_golden_bitstreams(tmp_path, name):
    _golden_check(tmp_path, _hostsim(), name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_golden()))
def test_cuda_golden_bitstreams(tmp_path, name):
    _golden_check(tmp_path, _cuda_lib(), name)
