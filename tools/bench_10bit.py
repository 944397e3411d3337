#!/usr/bin/env python
"""Main 10 throughput of the CTU search driver: one JSON line for 3840x2160 --preset veryslow -q 22 -p 1 at 10 bits.

    python tools/bench_10bit.py [--frames 8] [--steps 2] [--warmup 1]

  e2e_fps            frames/s through the reference encoder with the CTU job on the device (kvz_stream_bench_ctu_10b)
  device_fps         pictures/s of the driver alone (tools/ctu_devbench.py --bitdepth 10)
  reference_fps      frames/s of the unmodified 10-bit reference on this host's cores (kvz_stream_bench_ref_10b)
  bitstream_identical  the two encoders wrote the same bytes
plus the card's name and power limit and the host's core count.  Needs a GPU and oracle/_ref/ as build() leaves it;
scratch files go to a temporary directory.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
REF = os.path.join(ROOT, "oracle", "_ref")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="3840x2160")
    ap.add_argument("--frames", type=int, default=4, help="pictures per timed step")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--device-frames", type=int, default=8)
    a = ap.parse_args()
    w, h = map(int, a.res.split("x"))
    import kvazaar_b200 as kb
    from synth_yuv import synth_frame_10b
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    out = {"workload": f"{w}x{h} veryslow q22 -p 1, 10-bit", "gpu": gpu, "host_cores": os.cpu_count()}
    with tempfile.TemporaryDirectory() as d:
        clip = os.path.join(d, "clip.yuv")
        with open(clip, "wb") as f:
            for i in range(4):
                f.write(synth_frame_10b(w, h, 1234, i).astype("<u2").tobytes())
        args = [str(a.frames), str(a.steps), str(a.warmup), "0", "preset=veryslow", "qp=22", "period=1", "input-bitdepth=10"]
        res = {}
        for arm, binary, env in (("ctu", "kvz_stream_bench_ctu_10b", {"KVZ_CTU_PROVIDER": kb.LIB_PATH}), ("ref", "kvz_stream_bench_ref_10b", {})):
            e = dict(os.environ)
            e.pop("KVZ_CTU_PROVIDER", None)
            e.update(env)
            hevc = os.path.join(d, arm + ".hevc")
            r = subprocess.run([os.path.join(REF, binary), clip, a.res, hevc, *args], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
            assert r.returncode == 0, r.stderr[-2000:]
            if env:
                assert "CTU search driver active" in r.stderr, r.stderr[-2000:]
            res[arm] = (json.loads(r.stdout.strip().splitlines()[-1]), open(hevc, "rb").read())
        out["e2e_fps"] = round(res["ctu"][0]["fps"], 3)
        out["reference_fps"] = round(res["ref"][0]["fps"], 3)
        out["bitstream_identical"] = res["ctu"][1] == res["ref"][1]
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ctu_devbench.py"), "--res", a.res, "--preset", "veryslow", "--frames",
                            str(a.device_frames), "--bitdepth", "10"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        m = re.search(r"([0-9.]+) pictures/s", r.stdout)
        out["device_fps"] = float(m.group(1))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
