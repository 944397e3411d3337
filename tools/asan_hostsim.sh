#!/bin/bash
# TEST INFRASTRUCTURE: the single-source device algorithms (CTU search driver, motion search) compiled for the host with
# AddressSanitizer + UndefinedBehaviorSanitizer and run on the parity cases -- an out-of-bounds read or signed overflow in
# that source is one on the device too.  CPU only; needs oracle/_ref (the reference encoder with the CTU hooks).
#   bash tools/asan_hostsim.sh        -> prints one line per run, "issues 0" everywhere when clean
set -e
cd "$(dirname "$0")/.."
FLAGS="-O1 -g -std=c++17 -fPIC -shared -ffp-contract=off -fsanitize=address,undefined -Wall -Wno-unused-function -Wno-unknown-pragmas"
g++ $FLAGS -o /tmp/libkvzme_hostsim_asan.so tests/hostsim/me_hostsim.cpp
g++ $FLAGS -o /tmp/libkvzctu_hostsim_asan.so tests/hostsim/ctu_hostsim.cpp
g++ $FLAGS -o /tmp/libkvzctu_hostsim_10b_asan.so tests/hostsim/ctu_hostsim_10b.cpp
ASAN=$(g++ -print-file-name=libasan.so)
LD_PRELOAD=$ASAN ASAN_OPTIONS=detect_leaks=0 python - <<'PY'
import ctypes as C, os, pathlib, subprocess, sys, tempfile
ROOT = os.getcwd()
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
from _me_cases import *
host = C.CDLL("/tmp/libkvzme_hostsim_asan.so")
gold = np.load(os.path.join(ROOT, "tests", "golden", "me_search.npz"))
def tight(a):
    b = np.empty(a.shape, a.dtype); b[...] = a; return b          # exactly-sized heap buffers: ASan sees any overrun
for name in CASES:
    p, cur, ref, pus = make_case(name)
    assert np.array_equal(run_host_api(host, p, tight(cur), tight(ref), tight(pus))["cost"], gold[name + "/cost"]), name
for name in FRAC_CASES:
    p, level, cur, ref, pus = make_frac_case(name)
    assert np.array_equal(run_frac_host_api(host, p, level, tight(cur), tight(ref), tight(pus))["cost"], gold["frac/" + name + "/cost"]), name
for name in CAND_CASES:
    f, crp, clx, cus, col, pus = make_cand_case(name)
    assert run_cand_host_api(host, f, tight(cus), tight(col), tight(pus)).tobytes() == gold["cand/" + name].tobytes(), name
for name in MERGE_CASES:
    p, c, cur, planes, pus, cu = make_merge_case(name)
    bits = tuple(gold["merge/" + name + "/bits"])
    got = run_merge_host_api(host, p, c, tight(cur), [tight(pl) for pl in planes], tight(pus), bits)
    assert got.tobytes() == gold["merge/" + name].tobytes(), name
for name in BIPRED_CASES:
    p, c, cur, planes, pus = make_bipred_case(name)
    got = run_bipred_host_api(host, p, c, tight(cur), [tight(pl) for pl in planes], tight(pus))
    assert got.tobytes() == gold["bipred/" + name].tobytes(), name
import hashlib
for name in MC_CASES:
    p, c, planes, us, vs, pus, cu = make_mc_case(name)
    got = run_mc_host_api(host, p, c, [tight(a) for a in planes], [tight(a) for a in us], [tight(a) for a in vs], tight(pus))
    assert np.array_equal(np.frombuffer(b"".join(hashlib.sha256(a.tobytes()).digest() for a in got), np.uint8), gold["mc/" + name]), name
print("motion search host build: issues 0, results equal to the golden outputs")
PY
python - <<'PY'
import os, pathlib, subprocess, sys, tempfile
ROOT = os.getcwd()
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import test_ctu_driver as T
tmp = pathlib.Path(tempfile.mkdtemp(prefix="kvza_", dir="/tmp"))
ctu_bin = os.path.join(T.REF_DIR, "kvazaar_ctu")
asan = subprocess.check_output(["g++", "-print-file-name=libasan.so"], text=True).strip()
for (w, h, preset, qp, noisy) in [(264, 200, "veryslow", 22, False), (200, 136, "medium", 27, True), (136, 72, "veryslow", 22, True),
                                  (128, 128, "slow", 37, False), (72, 72, "placebo", 30, True)]:
    clip = T._clip(tmp, w, h, 1, noisy)
    e = dict(os.environ)
    e.update({"KVZ_CTU_PROVIDER": "/tmp/libkvzctu_hostsim_asan.so", "LD_PRELOAD": asan, "ASAN_OPTIONS": "detect_leaks=0:halt_on_error=0"})
    r = subprocess.run([ctu_bin, "-i", clip, "--input-res", f"{w}x{h}", "-o", str(tmp / "o.hevc"), "--preset", preset, "-q", str(qp), "-p", "1",
                        "--threads", "2"], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    issues = [ln for ln in r.stderr.splitlines() if "ERROR" in ln or "runtime error" in ln]
    print(f"CTU driver host build {w}x{h} {preset} q{qp}: rc {r.returncode}, active {'CTU search driver active' in r.stderr}, issues {len(issues)}")
# the same at 10 bits (kvazaar_ctu_10b, genuine 10-bit content, the host build with both instantiations): the wider accumulators
import test_ctu_driver_10bit as T10
ctu10 = os.path.join(T.REF_DIR, "kvazaar_ctu_10b")
for (w, h, preset, qp, noisy) in [(264, 200, "veryslow", 22, False), (200, 136, "medium", 27, True), (136, 72, "veryslow", 15, True),
                                  (192, 64, "veryslow", 15, True), (72, 72, "placebo", 30, True)]:
    clip = T10._clip(tmp, w, h, 1, noisy, 10)
    e = dict(os.environ)
    e.update({"KVZ_CTU_PROVIDER": "/tmp/libkvzctu_hostsim_10b_asan.so", "LD_PRELOAD": asan, "ASAN_OPTIONS": "detect_leaks=0:halt_on_error=0"})
    r = subprocess.run([ctu10, "-i", clip, "--input-res", f"{w}x{h}", "--input-bitdepth", "10", "-o", str(tmp / "o.hevc"), "--preset", preset,
                        "-q", str(qp), "-p", "1", "--threads", "2"], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    issues = [ln for ln in r.stderr.splitlines() if "ERROR" in ln or "runtime error" in ln]
    print(f"CTU driver host build 10-bit {w}x{h} {preset} q{qp}: rc {r.returncode}, active {'CTU search driver active' in r.stderr}, issues {len(issues)}")
PY
