#!/usr/bin/env python
"""Deterministic synthetic I420 clips.
   tools/synth_yuv.py W H FRAMES out.yuv [seed] [--noisy] [--bitdepth 10]
default: the clip of SURVEY.md 8(d) (ramp + drifting sinusoid + small noise);
--noisy: strong noise, flat patches and sharp edges (exercises high coefficient levels, band SAO, transform skip);
--bitdepth 10: the same scenes with genuine 10-bit samples (uint16 little-endian, 0..1023): the smooth parts are
evaluated at 10-bit precision and the noise has its own low-order bits, so the samples are not multiples of 4."""
import sys
import numpy as np


def synth_frame(width, height, seed=1234, frame_idx=0):
    r = np.random.default_rng(seed + frame_idx)
    y, x = np.mgrid[0:height, 0:width]
    luma = (x + y) * 0.11 + 60 * np.sin((x + 3 * frame_idx) / 37.0) * np.cos(y / 29.0) + 128 + r.integers(-4, 5, (height, width))
    cy, cx = np.mgrid[0:height // 2, 0:width // 2]
    u = 128 + 40 * np.sin(cx / 23.0 + frame_idx * 0.1) + r.integers(-2, 3, cx.shape)
    v = 128 + 40 * np.cos(cy / 19.0) + r.integers(-2, 3, cx.shape)
    return np.concatenate([np.clip(p, 0, 255).astype(np.uint8).ravel() for p in (luma, u, v)])


def noisy_frame(width, height, seed=5, frame_idx=0):
    r = np.random.default_rng(seed * 1000 + frame_idx)
    y, x = np.mgrid[0:height, 0:width]
    base = 128 + 70 * np.sin(x / 9.0 + frame_idx) * np.cos(y / 7.0) + r.integers(-40, 41, (height, width))
    base[(x // 16 + y // 16) % 3 == 0] = r.integers(0, 256)
    base[((x // 4) % 2 == 0) & ((y // 32) % 2 == 1)] += 60
    cy, cx = np.mgrid[0:height // 2, 0:width // 2]
    u = 128 + 50 * np.sin(cx / 5.0) + r.integers(-20, 21, cx.shape)
    v = 128 + 50 * np.cos(cy / 3.0) + r.integers(-30, 31, cx.shape)
    return np.concatenate([np.clip(p, 0, 255).astype(np.uint8).ravel() for p in (base, u, v)])


def synth_frame_10b(width, height, seed=1234, frame_idx=0):
    """synth_frame at 10 bits"""
    r = np.random.default_rng(seed + frame_idx)
    y, x = np.mgrid[0:height, 0:width]
    luma = 4 * ((x + y) * 0.11 + 60 * np.sin((x + 3 * frame_idx) / 37.0) * np.cos(y / 29.0) + 128) + r.integers(-16, 17, (height, width))
    cy, cx = np.mgrid[0:height // 2, 0:width // 2]
    u = 4 * (128 + 40 * np.sin(cx / 23.0 + frame_idx * 0.1)) + r.integers(-8, 9, cx.shape)
    v = 4 * (128 + 40 * np.cos(cy / 19.0)) + r.integers(-8, 9, cx.shape)
    return np.concatenate([np.clip(np.rint(p), 0, 1023).astype(np.uint16).ravel() for p in (luma, u, v)])


def noisy_frame_10b(width, height, seed=5, frame_idx=0):
    """noisy_frame at 10 bits"""
    r = np.random.default_rng(seed * 1000 + frame_idx)
    y, x = np.mgrid[0:height, 0:width]
    base = 4 * (128 + 70 * np.sin(x / 9.0 + frame_idx) * np.cos(y / 7.0)) + r.integers(-160, 161, (height, width))
    base[(x // 16 + y // 16) % 3 == 0] = r.integers(0, 1024)
    base[((x // 4) % 2 == 0) & ((y // 32) % 2 == 1)] += 240
    cy, cx = np.mgrid[0:height // 2, 0:width // 2]
    u = 4 * (128 + 50 * np.sin(cx / 5.0)) + r.integers(-80, 81, cx.shape)
    v = 4 * (128 + 50 * np.cos(cy / 3.0)) + r.integers(-120, 121, cx.shape)
    return np.concatenate([np.clip(np.rint(p), 0, 1023).astype(np.uint16).ravel() for p in (base, u, v)])


def frame_fn(noisy=False, bitdepth=8):
    if bitdepth == 10:
        return noisy_frame_10b if noisy else synth_frame_10b
    return noisy_frame if noisy else synth_frame


if __name__ == "__main__":
    argv = sys.argv[1:]
    bitdepth = 8
    if "--bitdepth" in argv:
        i = argv.index("--bitdepth")
        bitdepth = int(argv[i + 1])
        del argv[i:i + 2]
    args = [a for a in argv if not a.startswith("--")]
    noisy = "--noisy" in argv
    w, h, n, out = int(args[0]), int(args[1]), int(args[2]), args[3]
    seed = int(args[4]) if len(args) > 4 else (5 if noisy else 1234)
    f = frame_fn(noisy, bitdepth)
    with open(out, "wb") as fh:
        for i in range(n):
            fh.write(f(w, h, seed, i).astype("<u2" if bitdepth == 10 else np.uint8).tobytes())
