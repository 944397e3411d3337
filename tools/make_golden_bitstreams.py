#!/usr/bin/env python
"""Regenerates tests/golden/ctu_bitstreams.json: sha256 of the bitstreams the UNMODIFIED reference (oracle/_ref/kvazaar,
compiled from /root/reference by oracle/Makefile) writes for small synthetic clips (tools/synth_yuv.py).  The CTU search
driver must reproduce them byte for byte (tests/test_ctu_driver.py::test_*_golden_bitstreams).

    python tools/make_golden_bitstreams.py                 # 8-bit:  tests/golden/ctu_bitstreams.json
    python tools/make_golden_bitstreams.py --bitdepth 10   # 10-bit: tests/golden/ctu_bitstreams_10b.json from
                                                           #         oracle/_ref/kvazaar_10b, genuine 10-bit clips
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from synth_yuv import synth_frame, noisy_frame, frame_fn  # noqa: E402

CASES = [  # name, w, h, frames, preset, qp, noisy
    ("config1_64x64_ultrafast_q32", 64, 64, 3, "ultrafast", 32, False),
    ("192x128_medium_q27", 192, 128, 2, "medium", 27, False),
    ("136x72_veryslow_q22_noisy", 136, 72, 1, "veryslow", 22, True),
    ("128x128_slow_q37", 128, 128, 1, "slow", 37, False),
    ("200x136_veryslow_q27", 200, 136, 1, "veryslow", 27, False),
]


def make_clip(path, w, h, frames, noisy):
    with open(path, "wb") as f:
        for i in range(frames):
            f.write((noisy_frame(w, h, 5, i) if noisy else synth_frame(w, h, 1234, i)).tobytes())


def make_clip_10b(path, w, h, frames, noisy):
    f10 = frame_fn(noisy, 10)
    with open(path, "wb") as f:
        for i in range(frames):
            f.write(f10(w, h, 5 if noisy else 1234, i).astype("<u2").tobytes())


def main():
    ten = "--bitdepth" in sys.argv and sys.argv[sys.argv.index("--bitdepth") + 1] == "10"
    ref = os.path.join(ROOT, "oracle", "_ref", "kvazaar_10b" if ten else "kvazaar")
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, w, h, frames, preset, qp, noisy in CASES:
            clip, hevc = os.path.join(d, "c.yuv"), os.path.join(d, "o.hevc")
            (make_clip_10b if ten else make_clip)(clip, w, h, frames, noisy)
            extra = ["--input-bitdepth", "10"] if ten else []
            subprocess.check_call([ref, "-i", clip, "--input-res", f"{w}x{h}", "-o", hevc, "--preset", preset, "-q", str(qp), "-p", "1", *extra],
                                  stderr=subprocess.DEVNULL)
            data = open(hevc, "rb").read()
            out[name] = {"w": w, "h": h, "frames": frames, "preset": preset, "qp": qp, "noisy": noisy, "bytes": len(data),
                         "sha256": hashlib.sha256(data).hexdigest()}
    os.makedirs(os.path.join(ROOT, "tests", "golden"), exist_ok=True)
    with open(os.path.join(ROOT, "tests", "golden", "ctu_bitstreams_10b.json" if ten else "ctu_bitstreams.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
