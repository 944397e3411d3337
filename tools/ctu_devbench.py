#!/usr/bin/env python
"""Throughput of the CTU search driver alone (no encoder around it): pictures/s through kvz_cuda_ctu_submit/wait with
`slots` pictures in flight.  With a `make PROF=1` build kvz_cuda_ctu_close prints the phase profile.

    python tools/ctu_devbench.py --res 1920x1080 --preset medium --frames 32 --slots 16
    python tools/ctu_devbench.py --res 3840x2160 --preset veryslow --frames 8 --bitdepth 10    # Main 10 (uint16 samples)
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "width", "height", "qp", "rdo", "pu_depth_intra_min", "pu_depth_intra_max", "rdoq_enable", "rdoq_skip", "signhide_enable",
        "trskip_enable", "sao_type", "deblock_enable", "deblock_beta", "deblock_tc", "cu_split_termination", "intra_rdo_et",
        "combine_intra_cus", "intra_chroma_search", "full_intra_search", "wpp", "bitdepth")] + [("lambda_", C.c_double), ("lambda_sqrt", C.c_double)]


class Result(C.Structure):
    _fields_ = [("cu", C.c_void_p), ("cu_stride", C.c_int32), ("width_in_lcu", C.c_int32), ("height_in_lcu", C.c_int32), ("pad", C.c_int32),
                ("coeff", C.c_void_p), ("sao", C.c_void_p), ("rec_y", C.c_void_p), ("rec_u", C.c_void_p), ("rec_v", C.c_void_p),
                ("dbg_ctx", C.c_void_p), ("dbg_y", C.c_void_p), ("dbg_u", C.c_void_p), ("dbg_v", C.c_void_p)]


# the fields the reference's presets set (src/cfg.c:486-736) that the intra CTU search reads
PRESETS = {
    "ultrafast": dict(rdo=0, pu=(2, 3), rdoq=0, signhide=0, trskip=0, sao=0),
    "medium": dict(rdo=0, pu=(1, 4), rdoq=1, signhide=0, trskip=0, sao=3),
    "slow": dict(rdo=1, pu=(1, 4), rdoq=1, signhide=0, trskip=0, sao=3),
    "veryslow": dict(rdo=3, pu=(1, 4), rdoq=1, signhide=1, trskip=1, sao=3),
}


def make_config(w, h, preset, qp, bitdepth=8):
    p = PRESETS[preset]
    c = Config()
    c.bitdepth = bitdepth
    c.width, c.height, c.qp, c.rdo = w, h, qp, p["rdo"]
    c.pu_depth_intra_min, c.pu_depth_intra_max = p["pu"]
    c.rdoq_enable, c.rdoq_skip, c.signhide_enable, c.trskip_enable = p["rdoq"], 0, p["signhide"], p["trskip"]
    c.sao_type, c.deblock_enable, c.deblock_beta, c.deblock_tc = p["sao"], 1, 0, 0
    c.cu_split_termination, c.intra_rdo_et, c.combine_intra_cus, c.intra_chroma_search, c.full_intra_search, c.wpp = 0, 0, 1, 0, 0, 1
    c.lambda_ = 0.57 * 2.0 ** ((qp - 12) / 3.0)          # fixed-QP lambda (rate_control.c:678-691)
    c.lambda_sqrt = float(np.sqrt(c.lambda_))
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--preset", default="medium")
    ap.add_argument("--qp", type=int, default=None)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--distinct", type=int, default=4, help="distinct synthetic pictures (cycled)")
    ap.add_argument("--bitdepth", type=int, default=8, choices=[8, 10])
    a = ap.parse_args()
    w, h = map(int, a.res.split("x"))
    qp = a.qp if a.qp is not None else {"ultrafast": 32, "medium": 27, "slow": 27, "veryslow": 22}[a.preset]
    import kvazaar_b200 as kb
    from synth_yuv import frame_fn
    lib = C.CDLL(kb.LIB_PATH)
    lib.kvz_cuda_ctu_open.restype = C.c_void_p
    lib.kvz_cuda_ctu_open.argtypes = [C.POINTER(Config), C.c_int]
    lib.kvz_cuda_ctu_submit.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_int]
    lib.kvz_cuda_ctu_wait.argtypes = [C.c_void_p, C.c_int, C.POINTER(Result)]
    lib.kvz_cuda_ctu_release.argtypes = [C.c_void_p, C.c_int]
    lib.kvz_cuda_ctu_close.argtypes = [C.c_void_p]
    lib.kvz_cuda_ctu_launches.restype = C.c_uint64
    lib.kvz_cuda_ctu_launches.argtypes = [C.c_void_p]
    lib.kvz_cuda_last_error.restype = C.c_char_p
    cfg = make_config(w, h, a.preset, qp, a.bitdepth)
    enc = lib.kvz_cuda_ctu_open(C.byref(cfg), a.slots)
    assert enc, lib.kvz_cuda_last_error()
    ctx = np.zeros(192, np.uint8)
    assert lib.kvz_cuda_cabac_ctx_init(qp, 2, ctx.ctypes.data_as(C.c_void_p)) == 0       # KVZ_SLICE_I = 2
    frames = [frame_fn(False, a.bitdepth)(w, h, 1234, i) for i in range(a.distinct)]

    def submit(i):
        f = frames[i % len(frames)]
        y, u, v = f[:w * h], f[w * h:w * h * 5 // 4], f[w * h * 5 // 4:]
        s = lib.kvz_cuda_ctu_submit(enc, y.ctypes.data, u.ctypes.data, v.ctypes.data, w, w // 2, ctx.ctypes.data, cfg.lambda_, cfg.lambda_sqrt, qp)
        assert s >= 0, lib.kvz_cuda_last_error()
        return s

    res = Result()
    # warm-up: one picture
    s = submit(0)
    assert lib.kvz_cuda_ctu_wait(enc, s, C.byref(res)) == 0, lib.kvz_cuda_last_error()
    lib.kvz_cuda_ctu_release(enc, s)
    t0 = time.perf_counter()
    pending, nxt, done, first_latency = [], 0, 0, None
    while done < a.frames:
        while nxt < a.frames and len(pending) < a.slots:
            pending.append(submit(nxt))
            nxt += 1
        s = pending.pop(0)
        assert lib.kvz_cuda_ctu_wait(enc, s, C.byref(res)) == 0, lib.kvz_cuda_last_error()
        if first_latency is None:
            first_latency = time.perf_counter() - t0
        lib.kvz_cuda_ctu_release(enc, s)
        done += 1
    dt = time.perf_counter() - t0
    nctu = ((w + 63) // 64) * ((h + 63) // 64)
    print(f"ctu_devbench {a.res} {a.preset} q{qp} {a.bitdepth}-bit: {a.frames} pictures, {a.slots} in flight: {a.frames / dt:.2f} pictures/s, "
          f"{a.frames * nctu / dt:.0f} CTU/s, first picture after {first_latency * 1e3:.0f} ms, launches {lib.kvz_cuda_ctu_launches(enc)}", flush=True)
    lib.kvz_cuda_ctu_close(enc)


if __name__ == "__main__":
    main()
