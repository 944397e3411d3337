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


def extreme_pictures(w, h, bitdepth=8, seed=3):
    """One 4:2:0 picture of each kind of extreme content -> {name: bytes} (16-bit little-endian samples above 8 bits):
    flat, black, white, 1-pixel checkerboard, stripes, full-range noise, edges, ramps, blocks.  They drive clipping,
    all-zero residuals, transform skip and saturated SAO."""
    m = (1 << bitdepth) - 1
    k = (m + 1) >> 8
    r = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    cy, cx = yy[:h // 2, :w // 2], xx[:h // 2, :w // 2]

    def planes(y, u=None, v=None):
        mid = np.full((h // 2, w // 2), 128 * k)
        out = [np.clip(p, 0, m) for p in (y, mid if u is None else u, mid if v is None else v)]
        return b"".join((p.astype(np.uint8) if bitdepth == 8 else p.astype("<u2")).tobytes() for p in out)
    return {
        "flat128": planes(np.full((h, w), 128 * k)),
        "black": planes(np.zeros((h, w)), np.zeros((h // 2, w // 2)), np.zeros((h // 2, w // 2))),
        "white": planes(np.full((h, w), m), np.full((h // 2, w // 2), m), np.full((h // 2, w // 2), m)),
        "checker1": planes(((xx + yy) % 2) * m, ((cx + cy) % 2) * m, m - ((cx + cy) % 2) * m),
        "vstripes": planes((xx % 4 < 2) * m),
        "hstripes8": planes((yy % 16 < 8) * 200 * k + 20 * k),
        "fullnoise": planes(r.integers(0, m + 1, (h, w)), r.integers(0, m + 1, (h // 2, w // 2)), r.integers(0, m + 1, (h // 2, w // 2))),
        "diag_edge": planes((xx > yy * 2) * 180 * k + 40 * k, (cx > cy) * 100 * k + 60 * k),
        "ramp": planes(xx * m // w, cy * m // (h // 2), cx * m // (w // 2)),
        "blocks": planes(((xx // 8 + yy // 8) % 2) * 120 * k + 60 * k + r.integers(-2 * k, 2 * k + 1, (h, w))),
    }


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
