"""CTU search driver at 10 bits (Main 10, kvz_cuda_ctu_config.bitdepth = 10): bitstream identity with the unmodified
10-bit reference encoder.

Same gate as tests/test_ctu_driver.py, on the KVZ_BIT_DEPTH=10 builds of the reference: `kvazaar_10b` (all reference) and
`kvazaar_ctu_10b` (the CTU job redirected to a provider by integration/kvz_ctu_hooks.c).  Input is either genuine
10-bit samples (tools/synth_yuv.py, --input-bitdepth 10) or 8-bit samples that the reference shifts up.
"""
import ctypes as C
import hashlib
import json
import os
import re

import pytest

from test_ctu_driver import ROOT, _cuda_lib, _encode, _need

GOLDEN_10B = os.path.join(ROOT, "tests", "golden", "ctu_bitstreams_10b.json")
HOSTSIM_10B = os.path.join(ROOT, "tests", "hostsim", "libkvzctu_hostsim_10b.so")


def _hostsim():
    """the host build with both instantiations of the algorithm (tests/hostsim/ctu_hostsim_10b.cpp)"""
    if not os.path.exists(HOSTSIM_10B):
        import subprocess
        src = os.path.join(ROOT, "tests", "hostsim", "ctu_hostsim_10b.cpp")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unused-function", "-Wno-unknown-pragmas",
                               "-o", HOSTSIM_10B, src])
    return HOSTSIM_10B


def _clip(tmp_path, w, h, frames, noisy, input_bitdepth):
    from synth_yuv import frame_fn
    f = frame_fn(noisy, input_bitdepth)
    p = str(tmp_path / f"clip_{w}x{h}_{frames}{'n' if noisy else ''}_{input_bitdepth}.yuv")
    with open(p, "wb") as fh:
        for i in range(frames):
            a = f(w, h, 5 if noisy else 1234, i)
            fh.write(a.astype("<u2").tobytes() if input_bitdepth == 10 else a.tobytes())
    return p


def _identity10(tmp_path, provider, w, h, frames, preset, qp, noisy=False, input_bitdepth=10, extra=(), verify=True):
    ref_bin, ctu_bin = _need("kvazaar_10b", "kvazaar_ctu_10b")
    clip = _clip(tmp_path, w, h, frames, noisy, input_bitdepth)
    extra = ("--input-bitdepth", str(input_bitdepth), *extra)
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


# (w, h, frames, preset, qp, noisy, extra, input bit depths)
CASES = [
    (64, 64, 3, "ultrafast", 32, False, (), (10, 8)),
    (264, 200, 2, "medium", 27, False, (), (10, 8)),        # partial CTUs on both edges
    (264, 200, 1, "veryslow", 22, False, (), (10,)),
    (136, 72, 1, "veryslow", 22, True, (), (10, 8)),        # band SAO and transform skip get picked
    (200, 136, 1, "medium", 27, True, (), (10,)),
    (128, 128, 1, "slow", 37, False, (), (10,)),
    (192, 64, 1, "veryslow", 15, True, (), (10,)),          # large levels, SAO offsets above 7
    (136, 72, 1, "veryslow", 15, True, ("--intra-chroma-search",), (10,)),
]
PARAMS = [pytest.param(w, h, fr, pr, qp, nz, ex, ib, id=f"{w}x{h}-{pr}-q{qp}{'-noisy' if nz else ''}{'-chroma' if ex else ''}-in{ib}")
          for (w, h, fr, pr, qp, nz, ex, ibs) in CASES for ib in ibs]


# ------------------------------------------------------------------------------------------------ CPU (host build)
def _config(bitdepth):
    import numpy as np
    c = np.zeros(1, dtype=np.dtype([("v", "<i4", (21,)), ("lambda", "<f8"), ("lambda_sqrt", "<f8")], align=True))
    # width, height, qp, rdo, pu_depth_intra_min, pu_depth_intra_max, ..., wpp, bitdepth (kvz_cuda_ctu_config)
    c["v"][0][:6] = (64, 64, 32, 2, 1, 4)
    c["v"][0][19] = 1
    c["v"][0][20] = bitdepth
    return c


def test_abi_bitdepth_accepted_and_rejected():
    """bitdepth 0 and 8 mean 8-bit, 10 means 10-bit; every other value is refused by both providers"""
    import kvazaar_b200 as kb
    assert _config(0).itemsize == 104
    for path in (kb.LIB_PATH, _hostsim()):
        lib = C.CDLL(path)
        lib.kvz_cuda_ctu_config_supported.argtypes = [C.c_void_p]
        for bd, want in ((0, 0), (8, 0), (10, 0), (9, -1), (12, -1), (16, -1)):
            c = _config(bd)
            assert lib.kvz_cuda_ctu_config_supported(c.ctypes.data) == want, (path, bd)


def test_abi_struct_sizes_unchanged():
    """the config and result structs keep their layout: bitdepth took the place of the config's padding word and the
    sample pointers became `const void *`"""
    import subprocess
    import tempfile
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "kvz_cuda_ctu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(kvz_cuda_ctu_config), sizeof(kvz_cuda_ctu_result), sizeof(kvz_cuda_ctu_device_result),
         offsetof(kvz_cuda_ctu_config, bitdepth), offsetof(kvz_cuda_ctu_config, lambda));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        open(c, "w").write(prog)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", exe, c])
        assert subprocess.check_output([exe], text=True).split() == ["104", "96", "48", "80", "88"]


@pytest.mark.parametrize("w,h,frames,preset,qp,noisy,extra,input_bitdepth", PARAMS)
def test_hostbuild_10bit_bitstream_identical(tmp_path, w, h, frames, preset, qp, noisy, extra, input_bitdepth):
    _identity10(tmp_path, _hostsim(), w, h, frames, preset, qp, noisy, input_bitdepth, extra)


def _golden():
    return json.load(open(GOLDEN_10B))


def _golden_check(tmp_path, provider, name):
    g = _golden()[name]
    (ctu_bin,) = _need("kvazaar_ctu_10b")
    clip = _clip(tmp_path, g["w"], g["h"], g["frames"], g["noisy"], 10)
    out = str(tmp_path / "g.hevc")
    log = _encode(ctu_bin, clip, g["w"], g["h"], out, g["preset"], g["qp"], env={"KVZ_CTU_PROVIDER": provider},
                  extra=("--input-bitdepth", "10"))
    assert "CTU search driver active" in log
    data = open(out, "rb").read()
    assert len(data) == g["bytes"] and hashlib.sha256(data).hexdigest() == g["sha256"], name


@pytest.mark.parametrize("name", sorted(_golden()))
def test_hostbuild_10bit_golden_bitstreams(tmp_path, name):
    _golden_check(tmp_path, _hostsim(), name)


def test_hostbuild_10bit_out_of_scope_falls_through(tmp_path):
    """a 10-bit configuration outside the driver's scope (inter pictures, -p 8) runs the reference path untouched"""
    ref_bin, ctu_bin = _need("kvazaar_10b", "kvazaar_ctu_10b")
    clip = _clip(tmp_path, 128, 64, 3, False, 10)
    a, b = str(tmp_path / "a.hevc"), str(tmp_path / "b.hevc")
    import subprocess
    for binary, out, env in ((ref_bin, a, None), (ctu_bin, b, {"KVZ_CTU_PROVIDER": _hostsim()})):
        e = dict(os.environ)
        e.pop("KVZ_CTU_PROVIDER", None)
        e.update(env or {})
        r = subprocess.run([binary, "-i", clip, "--input-res", "128x64", "--input-bitdepth", "10", "-o", out, "--preset", "ultrafast",
                            "-q", "30", "-p", "8"], env=e, stderr=subprocess.PIPE, text=True, timeout=300)
        assert r.returncode == 0
        assert "CTU search driver active" not in r.stderr
    assert open(a, "rb").read() == open(b, "rb").read()


# ------------------------------------------------------------------------------------------------ GPU (the product)
@pytest.mark.gpu
@pytest.mark.parametrize("w,h,frames,preset,qp,noisy,extra,input_bitdepth", PARAMS)
def test_cuda_10bit_bitstream_identical(tmp_path, w, h, frames, preset, qp, noisy, extra, input_bitdepth):
    _identity10(tmp_path, _cuda_lib(), w, h, frames, preset, qp, noisy, input_bitdepth, extra)


@pytest.mark.gpu
def test_cuda_10bit_bitstream_identical_832x480_slow(tmp_path):
    _identity10(tmp_path, _cuda_lib(), 832, 480, 3, "slow", 32)


@pytest.mark.gpu
def test_cuda_10bit_bitstream_identical_1080p_medium(tmp_path):
    _identity10(tmp_path, _cuda_lib(), 1920, 1080, 4, "medium", 27, verify=False)


@pytest.mark.gpu
def test_cuda_10bit_bitstream_identical_2160p_veryslow(tmp_path):
    _identity10(tmp_path, _cuda_lib(), 3840, 2160, 2, "veryslow", 22, verify=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_golden()))
def test_cuda_10bit_golden_bitstreams(tmp_path, name):
    _golden_check(tmp_path, _cuda_lib(), name)
