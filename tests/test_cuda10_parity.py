"""10-bit (kvz_pixel = uint16_t) parity of the batched strategy entry points at the edges of the 10-bit range.

The checker is the reference compiled with KVZ_BIT_DEPTH=10 (`ref10`): its generic entry is the bit-exactness gate, and
every other implementation that build registers for the same type must agree with it on the same case.  The oracle's
10-bit build (`orc10`) is used only for the plane form of bi-prediction, which the reference has no entry for; a CPU test
pins it against the reference's `bipred_average`.

The seeded cases are module-level functions.  The GPU tests run them through the CUDA kernels (tolerance zero); the CPU
"reach" tests run the same cases through the reference and show that they reach the edge they exist for (clipped
outputs, saturated levels, the packed Hadamard lane bound of satd.cuh), so that a change to a generator cannot quietly
drop it.
"""
import numpy as np
import pytest

import _cases as cs

U16 = np.uint16
PMAX = 1023


def rp(r, n, kind="uniform"):
    return cs.rand_pix(r, n, U16, kind)


def dev16(kb, a):
    return kb.to_dev(np.ascontiguousarray(a))          # uint16 travels as int16


def host(t):
    return t.cpu().numpy()


def host16(t):
    return t.cpu().numpy().view(U16)


def costs(t):
    """Cost outputs are uint32_t in the C ABI (carried in an int32 tensor): a 64x64 10-bit SSD goes past 2^31."""
    return t.cpu().numpy().view(np.uint32)


_REGISTRY = {}


def impls(ref10, type_):
    """The implementations the 10-bit reference registers for `type_`, generic first."""
    if not _REGISTRY:
        for t, name, _ in ref10.entries():
            _REGISTRY.setdefault(t, []).append(name)
    names = _REGISTRY[type_]
    assert "generic" in names, type_
    return ["generic"] + sorted(set(names) - {"generic"})


def others(ref10, type_):
    return impls(ref10, type_)[1:]


# ============================================================================================ Walsh-Hadamard worst cases
def walsh(n):
    """n x n Sylvester Hadamard matrix of +-1."""
    h = np.ones((1, 1), np.int64)
    while h.shape[0] < n:
        h = np.block([[h, h], [h, -h]])
    return h


def walsh_pattern(n, k):
    """The k-th of the n*n two-dimensional Walsh-Hadamard basis patterns (+-1)."""
    w = walsh(n)
    return np.outer(w[k // n], w[k % n])


def hadamard_sum(d):
    """Sum of |H d H^T| in exact integers (H = the Sylvester matrix of d's size)."""
    w = walsh(d.shape[0])
    return int(np.abs(w @ d.astype(np.int64) @ w.T).sum())


def satd_block(d):
    """The reference's rounding of one Hadamard block: 4x4 (s + 1) >> 1, 8x8 (s + 2) >> 2."""
    s = hadamard_sum(d)
    return (s + 1) >> 1 if d.shape[0] == 4 else (s + 2) >> 2


SATD8_WALSH = (PMAX * 64 + 2) >> 2                     # one 8x8 block with all its energy in one coefficient
SATD4_WALSH = (PMAX * 16 + 1) >> 1                     # the same for 4x4


def packed_lane_peak(d):
    """Largest |value| after the five butterfly stages satd.cuh materialises for an 8x8 block (horizontal distances
    1 and 4, vertical 1, 2, 4; the distance-2 horizontal stage is folded into the absolute sum).  satd.cuh carries two
    such values per 32-bit register, so this must stay below 2^15."""
    x = d.astype(np.int64).copy()

    def bfly(a, axis, dist):
        a = np.moveaxis(a, axis, 0).copy()
        for i in range(a.shape[0]):
            if i & dist == 0:
                p, q = a[i].copy(), a[i + dist].copy()
                a[i], a[i + dist] = p + q, p - q
        return np.moveaxis(a, 0, axis)

    for dist in (1, 4):
        x = bfly(x, 1, dist)
    for dist in (1, 2, 4):
        x = bfly(x, 0, dist)
    return int(np.abs(x).max())


def walsh_pair(sign):
    """(a, b) with a = 1023 where `sign` is +1 and 0 elsewhere, b = 1023 - a: a - b = 1023 * sign."""
    a = np.where(sign > 0, PMAX, 0).astype(U16)
    return a, (PMAX - a).astype(U16)


def walsh_square_cases(n):
    """Sign blocks of n x n: every 4x4 / 8x8 basis pattern (and its negation); for n >= 16 the 8x8 patterns tiled,
    one pattern over the whole block and mixed patterns per 8x8 tile."""
    out = []
    if n <= 8:
        for k in range(n * n):
            out += [walsh_pattern(n, k), -walsh_pattern(n, k)]
        return out
    t = n // 8
    for k in range(0, 64, 3):
        out.append(np.tile(walsh_pattern(8, k), (t, t)))
    for m in range(8):
        blk = np.zeros((n, n), np.int64)
        for ty in range(t):
            for tx in range(t):
                blk[ty * 8:ty * 8 + 8, tx * 8:tx * 8 + 8] = walsh_pattern(8, (m * 11 + ty * 7 + tx * 13) % 64) * (1 if (ty + tx + m) % 2 else -1)
        out.append(blk)
    return out


def satd_nxn_closed(n):
    return SATD4_WALSH if n == 4 else ((n // 8) ** 2 * SATD8_WALSH) >> 2


def any_size_tiles(w, h):
    """(y, x, size) of the sub-blocks satd_any_size visits (strategies-picture.h SATD_ANY_SIZE): a first column of 4x4
    blocks when w % 8, a first row of 4x4 blocks when h % 8, 8x8 blocks for the rest."""
    tiles, x0, y0 = [], 0, 0
    if w % 8:
        tiles += [(y, 0, 4) for y in range(0, h, 4)]
        x0 = 4
    if h % 8:
        tiles += [(0, x, 4) for x in range(x0, w, 4)]
        y0 = 4
    tiles += [(y, x, 8) for y in range(y0, h, 8) for x in range(x0, w, 8)]
    return tiles


def quad_tiles(w, h):
    """The sub-blocks satd_any_size_quad visits (picture-generic.c SATD_ANY_SIZE_MULTI_GENERIC), including its quirk:
    the first row of 4x4 blocks starts at column 0 again, and the 8x8 rows start at row 0 when h % 8 == 4."""
    tiles = []
    wm8 = w % 8
    if wm8:
        tiles += [(y, 0, 4) for y in range(0, h, 4)]
        w -= 4
    if h % 8:
        tiles += [(0, x, 4) for x in range(0, w, 4)]
        h -= 4
    tiles += [(y, x, 8) for y in range(h % 8, h, 8) for x in range(wm8, w, 8)]
    return tiles


def satd_tiles(diff, tiles):
    """Plain model of satd_any_size / satd_any_size_quad at 10 bits: per-tile Hadamard, sum >> (10 - 8)."""
    return sum(satd_block(diff[y:y + s, x:x + s]) for y, x, s in tiles) >> 2


def walsh_fill(w, h, tiles, seed):
    """A w x h sign block in which every tile of `tiles` is a Walsh-Hadamard basis pattern of the tile's size."""
    sign = np.ones((h, w), np.int64)
    for i, (y, x, s) in enumerate(tiles):
        sign[y:y + s, x:x + s] = walsh_pattern(s, (seed * 5 + i * 7) % (s * s)) * (1 if (seed + i) % 3 else -1)
    return sign


ANY_DIMS = (4, 8, 12, 16, 24, 32, 48, 64)
ANY_SHAPES = [(w, h) for w in ANY_DIMS for h in ANY_DIMS]
QUAD_SHAPES = [(w, h) for w in (8, 12, 16, 24, 32, 48, 64) for h in ANY_DIMS] + [(4, 8), (4, 16)]
SA, SB, SLOT = 80, 76, 64                              # strides of the two planes, rows per case


def any_size_case():
    """Planes a (stride SA) and b (stride SB), one 64-row slot per (shape, variant): in slot i the w x h block at
    descs[i] is a Walsh fill of the satd_any_size tiling.  Returns (a, b, [(w, h, off_a, off_b, sign)])."""
    cases = [(w, h, v) for (w, h) in ANY_SHAPES for v in range(2)]
    a = np.zeros(SA * SLOT * len(cases), U16)
    b = np.zeros(SB * SLOT * len(cases), U16)
    out = []
    for i, (w, h, v) in enumerate(cases):
        sign = walsh_fill(w, h, any_size_tiles(w, h), i + v)
        pa, pb = walsh_pair(sign)
        xa, xb = (i * 3) % (SA - w + 1), (i * 5) % (SB - w + 1)
        oa, ob = i * SLOT * SA + xa, i * SLOT * SB + xb
        for y in range(h):
            a[oa + y * SA: oa + y * SA + w] = pa[y]
            b[ob + y * SB: ob + y * SB + w] = pb[y]
        out.append((w, h, oa, ob, sign))
    return cs.al(a), cs.al(b), out


QS, QROWS = 64, 64


def quad_case():
    """Four prediction planes and an original (all stride QS), one QROWS-row slot per shape: the original is 1023 on a
    Walsh fill.  8x8 tiles are laid from the block's origin
    (shifted by 4 when w % 8 == 4), so every tile the quad visits is a basis pattern whenever w % 8 == 0 or h % 8 == 0.
    Predictions 0 and 2 are 1023 - original (the Walsh maximum), 1 and 3 equal the original (cost 0)."""
    n = len(QUAD_SHAPES)
    orig = np.zeros(QS * QROWS * n + 64, U16)
    preds = [np.zeros(QS * QROWS * n + 64, U16) for _ in range(4)]
    out = []
    for i, (w, h) in enumerate(QUAD_SHAPES):
        grid = [(y, x, 8) for y in range(0, h - 7, 8) for x in range(w % 8, w - 7, 8)]
        if w % 8:
            grid += [(y, 0, 4) for y in range(0, h, 4)]
        if h % 8:
            grid += [(h - 4, x, 4) for x in range(0, w, 4)]
        o = i * QS * QROWS
        so = walsh_fill(w, h, grid, i)
        oa, _ = walsh_pair(so)
        for y in range(h):
            orig[o + y * QS: o + y * QS + w] = oa[y]
        for k in range(4):
            pk = oa if k % 2 else (PMAX - oa).astype(U16)
            for y in range(h):
                preds[k][o + y * QS: o + y * QS + w] = pk[y]
        out.append((w, h, o))
    return [cs.al(p) for p in preds], cs.al(orig), out


def quad_model(preds, orig, w, h, o):
    d = [orig[o:o + QS * QROWS].reshape(QROWS, QS).astype(np.int64) - p[o:o + QS * QROWS].reshape(QROWS, QS) for p in preds]
    return [satd_tiles(dk, quad_tiles(w, h)) for dk in d]


def dual_case(n):
    """cost_nxn_multi_batch / satd_NxN_dual layout: per block two modes 1024 samples apart.  Mode 0 is the Walsh case's
    b (all the energy in one coefficient), mode 1 the same for even blocks and equal to the original (cost 0) for odd
    ones, so that a swap of modes shows.  (At 64x64 the two modes overlap, as in the reference's pred_buffer: both b.)"""
    sq = walsh_square_cases(n)
    count = len(sq)
    pitch = (1024 + n * n + 15) // 16 * 16
    preds = np.zeros(count * pitch, U16)
    origs = np.zeros(count * n * n, U16)
    for i in range(count):
        a, b = walsh_pair(sq[i])
        origs[i * n * n:(i + 1) * n * n] = a.ravel()
        preds[i * pitch: i * pitch + n * n] = b.ravel()
        preds[i * pitch + 1024: i * pitch + 1024 + n * n] = (a if i % 2 and n < 64 else b).ravel()
    return cs.al(preds), cs.al(origs), pitch, count


def dual_closed(n, i):
    return [satd_nxn_closed(n), 0 if i % 2 and n < 64 else satd_nxn_closed(n)]


def rough_walsh_case(log2w, inverted):
    """A 10-bit picture for the fused rough search: the source is Walsh patterns (0/1023) over a reconstruction of
    zeros, so the references -- and with them DC, planar and every angular mode -- predict 0 except in the first block
    (no neighbours: 512).  `inverted` mirrors both (source 1023 - pattern over a reconstruction of 1023s)."""
    pic_w, pic_h = 96, 64
    w = 1 << log2w
    src = np.zeros((pic_h, pic_w), U16)
    for j in range(pic_h // w):
        for i in range(pic_w // w):
            k = j * (pic_w // w) + i
            if w == 4:
                sign = walsh_pattern(4, k % 16)
            else:
                sign = np.tile(walsh_pattern(8, (k * 5) % 64), (w // 8, w // 8))
            src[j * w:(j + 1) * w, i * w:(i + 1) * w] = np.where(sign > 0, PMAX, 0)
    rec = np.zeros_like(src)
    if inverted:
        src, rec = (PMAX - src).astype(U16), np.full_like(rec, PMAX)
    return cs.al(src.ravel()), cs.al(rec.ravel()), pic_w, pic_h


def rough_reference(ref10, log2w, src, rec, pic_w, pic_h):
    """build_reference + intra_predict (filter_boundary 1) + satd_NxN of the 10-bit reference: [block, mode] costs."""
    w = 1 << log2w
    bx, by = pic_w // w, pic_h // w
    out = np.zeros((bx * by, 35), np.int64)
    for j in range(by):
        for i in range(bx):
            top, left = ref10.intra_build_reference(log2w, 0, i * w, j * w, pic_w, pic_h, rec, pic_w)
            blk = cs.al(np.ascontiguousarray(src.reshape(pic_h, pic_w)[j * w:(j + 1) * w, i * w:(i + 1) * w]).ravel())
            for mode in range(35):
                pred = cs.al(ref10.intra_predict(log2w, mode, 0, top, left, 1))
                out[j * bx + i, mode] = ref10.nxn("satd", w, pred, blk)
    return out


# ============================================================================================ transforms
def transform_cases(n):
    """(name, block, in_range): residuals in +-1023, saturated +-1023 residuals in Walsh patterns, coefficients over
    the whole int16 range (in_range False: compared with the generic entry only, AVX2 saturates)."""
    r = cs.rng(200 + n)
    w = walsh(n)
    out = [("residual", r.integers(-PMAX, PMAX + 1, n * n).astype(np.int16), True),
           ("residual_extreme", ((r.integers(0, 2, n * n) * 2 - 1) * PMAX).astype(np.int16), True)]
    for k in (0, 1, n - 1, n * n // 2 + 1, n * n - 1):
        out.append((f"walsh{k}", (np.outer(w[k // n], w[k % n]) * PMAX).astype(np.int16).ravel(), True))
    for kind in ("full", "sparse", "small"):
        out.append((kind, cs.rand_coeffs(r, n * n, kind).astype(np.int16), False))
    out.append(("int16_max", np.full(n * n, 32767, np.int16), False))
    out.append(("int16_min", np.full(n * n, -32768, np.int16), False))
    return out


TR_SIZES = (4, 8, 16, 32)


# ============================================================================================ quant / dequant
QUANT_QPS = (0, 1, 22, 37, 50, 51)


def quant_blocks(ref10, n, qp):
    """Coefficient blocks for quant: forward DCTs (10-bit) of +-1023 and Walsh residuals, and raw int16 blocks."""
    r = cs.rng(300 + n * 64 + qp)
    blocks = []
    for k in range(4):
        res = r.integers(-PMAX, PMAX + 1, n * n).astype(np.int16) if k % 2 else \
            (walsh_pattern(n, (k * 5 + qp) % (n * n)) * PMAX).astype(np.int16).ravel()
        blocks.append(ref10.transform(f"dct_{n}x{n}", 10, res, n))
    for kind in ("full", "sparse", "small"):
        blocks.append(cs.rand_coeffs(r, n * n, kind))
    blocks.append(cs.al((r.integers(-3, 4, n * n) * (r.random(n * n) < 0.3)).astype(np.int16)))  # odd-parity groups
    return [cs.al(b, np.int16) for b in blocks]


def quant_types(n):
    return (0, 2) if n < 32 else (0,)


def dequant_levels(n):
    """Levels for dequant incl. +-32767 so that the int16 clip is reached at high qp_scaled."""
    r = cs.rng(400 + n)
    full = cs.rand_coeffs(r, n * n, "full")
    ext = np.where(r.integers(0, 2, n * n) > 0, 32767, -32767).astype(np.int16)
    mid = r.integers(-300, 301, n * n).astype(np.int16)
    small = r.integers(-4, 5, n * n).astype(np.int16)
    return [cs.al(x, np.int16) for x in (full, ext, mid, small)]


DEQUANT_QPS = (0, 22, 37, 51)


# ============================================================================================ quantize_residual
QR_STRIDE = 256                                          # 8 slots of 32 columns
QR_CONTENTS = ("noise", "sat_src", "sat_pred", "equal", "walsh")


def qres_case(seed):
    """Source / prediction planes and TU records: every TU in its own 32x32 slot (so reconstruction footprints are
    disjoint); widths 4-32, colours 0/1/2 (chroma up to 16), scans 0-2, 4x4 luma transform skip, intra and inter CUs,
    and the contents noise, saturated (1023 over 0 and 0 over 1023), prediction == source and Walsh +-1023."""
    import kvazaar_b200.api as api
    r = cs.rng(seed)
    recs = []
    for n in (4, 8, 16, 32):
        for ci, content in enumerate(QR_CONTENTS):
            for k in range(6):
                color = k % 3 if n < 32 else 0
                trskip = 1 if (n == 4 and color == 0 and (k + ci) % 2 == 0) else 0
                recs.append((n, content, color, (k + ci) % 3, trskip, (k // 3 + ci) % 2))
    rows = 32 * ((len(recs) + 7) // 8)
    src = np.zeros((rows, QR_STRIDE), U16)
    pred = np.zeros((rows, QR_STRIDE), U16)
    tus = np.zeros(len(recs), api.TU)
    n_coeff = 0
    for i, (n, content, color, scan, trskip, intra) in enumerate(recs):
        y, x = (i // 8) * 32, (i % 8) * 32
        if content == "noise":
            s = r.integers(0, PMAX + 1, (n, n))
            p = np.clip(s + r.integers(-200, 201, (n, n)), 0, PMAX)
        elif content == "sat_src":
            s, p = np.full((n, n), PMAX), np.zeros((n, n))
        elif content == "sat_pred":
            s, p = np.zeros((n, n)), np.full((n, n), PMAX)
        elif content == "equal":
            s = r.integers(0, PMAX + 1, (n, n))
            p = s
        else:
            s, p = walsh_pair(walsh_pattern(n, (i * 7) % (n * n)))
        src[y:y + n, x:x + n] = s
        pred[y:y + n, x:x + n] = p
        off = y * QR_STRIDE + x
        tus[i] = (off, off, off, n_coeff, n, color, scan, trskip, intra, 0, 0, 0)
        n_coeff += n * n
    return cs.al(src.ravel()), cs.al(pred.ravel()), tus, n_coeff, recs


QR_QPS = (0, 30, 51)


def tile(plane, off, w, h, stride):
    return np.stack([plane[off + y * stride: off + y * stride + w] for y in range(h)])


def qres_reference(ref10, qp, signhide, src, pred, t, impl="generic"):
    n = int(t["width"])
    o = int(t["off_ref"])
    s = cs.al(tile(src, o, n, n, QR_STRIDE))
    p = cs.al(tile(pred, o, n, n, QR_STRIDE))
    has, rec, coeff = ref10.quantize_residual(qp, n, int(t["color"]), int(t["scan_idx"]), int(t["use_trskip"]),
                                              int(t["cu_is_intra"]), n, s, p, 1, signhide, 0, impl)
    return has, rec[:n * n].reshape(n, n), coeff


# ============================================================================================ intra
def intra_refs(log2w):
    """Reference rows (top, left; 2w + 1 samples, corner shared) with 0/1023 steps, so the DC, vertical and horizontal
    edge filters over- and undershoot, plus random extreme and uniform rows."""
    r = cs.rng(500 + log2w)
    n = 2 * (1 << log2w) + 1
    out = []
    for corner, tv, lv in ((0, PMAX, PMAX), (PMAX, 0, 0), (0, 0, PMAX), (PMAX, PMAX, 0)):
        top = np.full(n, tv, U16)
        left = np.full(n, lv, U16)
        top[0] = left[0] = corner
        out.append((top, left))
    steps = np.where((np.arange(n) // 2) % 2, PMAX, 0).astype(U16)
    out.append((steps.copy(), (PMAX - steps).astype(U16)))
    for kind in ("extreme", "uniform"):
        t, l = cs.rand_refs(r, log2w, U16, kind)
        out.append((t, l))
    return [(cs.al(t), cs.al(l)) for t, l in out]


def edge_filter_unclipped(log2w, mode, top, left):
    """The unclipped values of the vertical (26) / horizontal (10) boundary filters of a luma block smaller than 32:
    first column top[1] + ((left[y] - left[0]) >> 1), first row left[1] + ((top[x] - top[0]) >> 1)."""
    w = 1 << log2w
    t, l = top.astype(np.int64), left.astype(np.int64)
    if mode == 26:
        return t[1] + ((l[1:w + 1] - l[0]) >> 1)
    return l[1] + ((t[1:w + 1] - t[0]) >> 1)


PIC_W, PIC_H = 200, 136


def intra_plane_case():
    """Luma with a band of 0/1023 rows on top; uniform below and in chroma (so substituted runs stand out)."""
    r = cs.rng(600)
    luma = rp(r, PIC_W * PIC_H)
    luma[: PIC_W * 24] = rp(r, PIC_W * 24, "extreme")
    return {0: luma, 1: rp(r, PIC_W * PIC_H // 4)}


def block_positions(log2w, color):
    step = (1 << log2w) << (1 if color else 0)
    return [(lx, ly) for ly in range(0, PIC_H - step + 1, step) for lx in range(0, PIC_W - step + 1, step)]


# ============================================================================================ interpolation
SAMPLE_SHAPES = [(4, 4), (8, 4), (4, 8), (16, 4), (4, 16), (16, 12), (24, 32), (32, 32), (48, 64), (64, 64)]
SAMPLE_KINDS = ("luma", "luma_hi", "chroma", "chroma_hi")
S_STRIDE, S_ROWS = 160, 96


def sample_case():
    """Extreme 0/1023 content (the filters over- and undershoot, so the pixel outputs clip) with a uniform lower part,
    and for every kind the shapes x every fraction: descriptors (off_src, w, h, fx, fy)."""
    r = cs.rng(700)
    src = rp(r, S_STRIDE * S_ROWS, "extreme")
    src[S_STRIDE * 80:] = rp(r, S_STRIDE * (S_ROWS - 80))
    descs = {}
    for kind in SAMPLE_KINDS:
        chroma = kind.startswith("chroma")
        frac = 8 if chroma else 4
        d = []
        for (w, h) in SAMPLE_SHAPES:
            if chroma and (w > 32 or h > 32):
                continue
            for fy in range(frac):
                for fx in range(frac):
                    y, x = int(r.integers(4, S_ROWS - 4 - h)), int(r.integers(4, S_STRIDE - 4 - w))
                    d.append((y * S_STRIDE + x, w, h, fx, fy))
        descs[kind] = d
    return src, descs


FME_SHAPES = [(8, 8), (16, 16), (16, 8), (32, 32), (64, 64), (8, 16), (24, 32)]
FME_OFFS = [(ox, oy) for ox in (-1, 0, 1) for oy in (-1, 0, 1)]
F_STRIDE, F_ROWS = 128, 100


def fme_case():
    r = cs.rng(800)
    src = rp(r, F_STRIDE * F_ROWS)
    src[: F_STRIDE * 50] = rp(r, F_STRIDE * 50, "extreme")
    offs = {}
    for (w, h) in FME_SHAPES:
        offs[(w, h)] = [int(r.integers(8, F_ROWS - 8 - h - 1)) * F_STRIDE + int(r.integers(8, F_STRIDE - 8 - w - 1))
                        for _ in FME_OFFS]
    return src, offs


EXT_W, EXT_H, EXT_S = 80, 48, 88
EXT_PLACES = [(-6, 4), (70, 10), (20, -5), (20, 44), (-10, -10), (76, 46), (-40, 8), (100, 60)]
EXT_SIZES = [(8, 8), (16, 4), (32, 16)]
EXT_PADS = [(3, 4, 3, 4, 0), (3, 4, 3, 4, 1), (1, 2, 1, 2, 3)]


# ============================================================================================ picture group
B_SA, B_SB, B_ROWS = 208, 176, 160


def block_cost_case():
    """Extreme planes on the 8-bit test's shape grid, with one side's lower half the complement of the other's."""
    r = cs.rng(900)
    a = rp(r, B_SA * B_ROWS, "extreme")
    b = rp(r, B_SB * B_ROWS)
    b[: B_SB * 80] = rp(r, B_SB * 80, "extreme")
    b[B_SB * 80:] = PMAX - a[: B_SA * (B_ROWS - 80)].reshape(-1, B_SA)[:, :B_SB].ravel()   # a 64x64 SSD above 2^31
    descs = []
    for i in range(len(ANY_SHAPES) * 2):
        w, h = ANY_SHAPES[i % len(ANY_SHAPES)]
        ya, xa = int(r.integers(0, B_ROWS - 64)), int(r.integers(0, B_SA - 64))
        yb, xb = int(r.integers(0, B_ROWS - 64)), int(r.integers(0, B_SB - 64))
        side = int(r.integers(1, w)) if w > 1 else 0
        descs.append((ya * B_SA + xa, yb * B_SB + xb, w, h, side if i % 2 else 0, 0 if i % 2 else side))
    return a, b, descs


def pixel_var_bufs():
    r = cs.rng(950)
    return [rp(r, 4096, "extreme"), rp(r, 4096, "smooth"), cs.al(np.full(4096, PMAX, U16)), rp(r, 4096),
            cs.al(np.zeros(4096, U16))]


BIPRED_SHAPES = [(8, 8), (16, 8), (64, 64), (8, 32), (4, 4)]


def bipred_case():
    """Per shape: two pixel blocks (extreme 0/1023) and two 14-bit intermediates with values near both ends of
    int16, so that the averages clip at 0 and 1023."""
    r = cs.rng(960)
    out = []
    for (w, h) in BIPRED_SHAPES:
        px = [rp(r, w * h, "extreme"), rp(r, w * h)]
        im = []
        for _ in range(2):
            x = np.where(r.integers(0, 2, w * h) > 0, r.integers(24000, 32768, w * h), r.integers(-32768, -24000, w * h))
            x[::5] = r.integers(-2000, 18000, x[::5].size)
            im.append(cs.al(x.astype(np.int16)))
        out.append((w, h, px, im))
    return out


# ============================================================================================ SAO
SAO_SHAPES = [(64, 64), (32, 32), (56, 64), (64, 24), (8, 8), (16, 40)]


def sao_block_case():
    """Original / reconstruction blocks (uniform, extreme, smooth; reconstruction off by up to 40), edge classes,
    edge offsets over +-31 and band positions 0 and 28-31."""
    r = cs.rng(1000)
    shapes = SAO_SHAPES * 3
    origs, recs = [], []
    for i, (bw, bh) in enumerate(shapes):
        o = rp(r, bw * bh, cs.KINDS[i % 3])
        origs.append(o)
        recs.append(cs.al(np.clip(o.astype(int) + r.integers(-40, 41, bw * bh), 0, PMAX).astype(U16)))
    eo = (np.arange(len(shapes)) % 4).astype(np.int8)
    offsets = r.integers(-31, 32, (len(shapes), 5)).astype(np.int32)
    offsets[::4] = [0, 31, 31, -31, -31]
    band_pos = np.array([[0, 28, 29, 30, 31][i % 5] for i in range(len(shapes))], np.int32)
    bands = r.integers(-31, 32, (len(shapes), 4)).astype(np.int32)
    bands[::3] = [31, -31, 31, -31]
    return shapes, origs, recs, eo, offsets, band_pos, bands


SR_STRIDE, SR_NEW_STRIDE, SR_ROWS = 200, 136, 140
SR_SHAPES = [(64, 64), (32, 20), (10, 54), (54, 10), (1, 1), (3, 64)]


def sao_rec_case():
    """Reconstruction near 0 (rows 0-69) and near 1023 (rows 70-139), and descriptors over types 0/1/2, all edge
    classes, colours 0/1/2, offsets +-31 and band positions at both ends; every block keeps a one-sample halo."""
    r = cs.rng(1100)
    half = SR_STRIDE * SR_ROWS // 2
    rec = cs.al(np.concatenate([r.integers(0, 24, half), r.integers(PMAX - 24, PMAX + 1, half)]).astype(U16))
    descs = []
    for i in range(72):
        bw, bh = SR_SHAPES[i % 6]
        y = 1 + (i % 3) + (0 if (i // 3) % 2 == 0 else SR_ROWS // 2)
        x = 1 + int(r.integers(0, SR_STRIDE - bw - 2))
        type_ = [2, 1, 2, 0, 1, 2][(i // 6) % 6]
        offs = r.integers(-31, 32, 10).astype(np.int32)
        if i % 2:
            offs[:] = [0, 31, 31, -31, -31, 0, -31, -31, 31, 31] if type_ == 2 else [31, 31, -31, -31, 0, -31, -31, 31, 31, 0]
        bp = [[0, 31], [28, 0], [31, 29], [30, 28]][i % 4]
        descs.append((y * SR_STRIDE + x, bw, bh, type_, (i // 2) % 4, i % 3, bp, offs))
    return rec, descs


# ============================================================================================ checksum
CHECKSUM_CASES = [(3, 5, 3), (1920, 8, 2000), (3840, 2160, 3840)]


def checksum_data(w, h, stride):
    r = cs.rng(1200 + w)
    return rp(r, stride * h)


# ############################################################################################ GPU tests: CUDA vs ref10
@pytest.mark.gpu
@pytest.mark.parametrize("n", (4, 8, 16, 32, 64))
def test_walsh_satd_nxn(cuda_lib, ref10, n):
    kb = cuda_lib
    sq = walsh_square_cases(n)
    pairs = [walsh_pair(s) for s in sq]
    a = cs.al(np.concatenate([p[0].ravel() for p in pairs]))
    b = cs.al(np.concatenate([p[1].ravel() for p in pairs]))
    got = host(kb.satd_nxn_batch(n, dev16(kb, a), dev16(kb, b), len(pairs)))
    for i in range(len(pairs)):
        ai, bi = cs.al(a[i * n * n:(i + 1) * n * n]), cs.al(b[i * n * n:(i + 1) * n * n])
        want = ref10.nxn("satd", n, ai, bi)
        assert want == satd_nxn_closed(n), (n, i)
        assert got[i] == want, (n, i, int(got[i]), want)
    # the plain batch and the multi-mode entry with one mode are the same computation
    plain = host(kb.cost_nxn_multi_batch(1, n, dev16(kb, a), n * n, 0, 1, dev16(kb, b), len(pairs))).ravel()
    assert np.array_equal(plain, got)


@pytest.mark.gpu
@pytest.mark.parametrize("n", (4, 8, 16, 32, 64))
def test_walsh_cost_nxn_multi_dual(cuda_lib, ref10, n):
    kb = cuda_lib
    preds, origs, pitch, count = dual_case(n)
    for use_satd, kind in ((1, "satd"), (0, "sad")):
        got = host(kb.cost_nxn_multi_batch(use_satd, n, dev16(kb, preds), pitch, 1024, 2, dev16(kb, origs), count))
        for i in range(count):
            p = cs.al(preds[i * pitch: i * pitch + 1024 + n * n])
            o = cs.al(origs[i * n * n:(i + 1) * n * n])
            want = ref10.nxn_dual(kind, n, p, o)
            for impl in others(ref10, f"{kind}_{n}x{n}_dual"):
                assert np.array_equal(ref10.nxn_dual(kind, n, p, o, impl), want), (kind, n, impl)
            if use_satd:
                assert list(want) == dual_closed(n, i), (n, i)
            assert list(got[i]) == list(want), (kind, n, i)


@pytest.mark.gpu
def test_walsh_block_cost_satd_any(cuda_lib, ref10):
    kb = cuda_lib
    a, b, cases = any_size_case()
    descs = np.zeros(len(cases), kb.BLK)
    for i, (w, h, oa, ob, _) in enumerate(cases):
        descs[i] = (oa, ob, w, h, 0, 0)
    got = host(kb.block_cost_batch(kb.OP_SATD_ANY, dev16(kb, a), SA, dev16(kb, b), SB, descs))
    for i, (w, h, oa, ob, sign) in enumerate(cases):
        want = ref10.satd_any_size(w, h, a[oa:], SA, b[ob:], SB)
        assert want == satd_tiles(1023 * sign, any_size_tiles(w, h)), (w, h)
        assert got[i] == want, (w, h, int(got[i]), want)


@pytest.mark.gpu
def test_walsh_satd_any_size_quad(cuda_lib, ref10):
    kb = cuda_lib
    preds, orig, cases = quad_case()
    base = cs.al(np.concatenate(preds))
    plen = preds[0].size
    descs = np.zeros(len(cases), kb.QUAD)
    for i, (w, h, o) in enumerate(cases):
        descs[i]["off_pred"] = [k * plen + o for k in range(4)]
        descs[i]["off_orig"] = o
        descs[i]["w"], descs[i]["h"] = w, h
    got = host(kb.satd_any_size_quad_batch(dev16(kb, base), QS, dev16(kb, orig), QS, descs))
    for i, (w, h, o) in enumerate(cases):
        want = ref10.satd_any_size_quad(w, h, [p[o:] for p in preds], QS, orig[o:], QS)
        assert list(want) == quad_model(preds, orig, w, h, o), (w, h)
        assert list(got[i]) == list(want), (w, h, list(got[i]), list(want))


@pytest.mark.gpu
@pytest.mark.parametrize("log2w", (2, 3, 4, 5))
def test_walsh_intra_rough_search(cuda_lib, ref10, log2w):
    kb = cuda_lib
    for inverted in (0, 1):
        src, rec, pic_w, pic_h = rough_walsh_case(log2w, inverted)
        got = host(kb.intra_rough_search_frame(log2w, dev16(kb, src), dev16(kb, rec), pic_w, pic_w, pic_h))
        want = rough_reference(ref10, log2w, src, rec, pic_w, pic_h)
        assert np.array_equal(got, want), (log2w, inverted, np.argwhere(got != want)[:4])


@pytest.mark.gpu
@pytest.mark.parametrize("n", TR_SIZES)
def test_transform_batch_10bit(cuda_lib, ref10, n):
    kb = cuda_lib
    cases = transform_cases(n)
    x = cs.al(np.concatenate([c[1] for c in cases]), np.int16)
    kinds = [(kb.TR_DCT, f"dct_{n}x{n}"), (kb.TR_IDCT, f"idct_{n}x{n}")]
    if n == 4:
        kinds += [(kb.TR_DST, "fast_forward_dst_4x4"), (kb.TR_IDST, "fast_inverse_dst_4x4")]
    fwd_out = {}
    for kind, name in kinds:
        got = host(kb.transform_batch(kind, n, 10, dev16(kb, x), len(cases)))
        for i, (label, blk, in_range) in enumerate(cases):
            want = ref10.transform(name, 10, blk, n)
            if in_range:
                for impl in others(ref10, name):
                    assert np.array_equal(ref10.transform(name, 10, blk, n, impl), want), (name, label, impl)
            assert np.array_equal(got[i * n * n:(i + 1) * n * n], want), (name, label)
        fwd_out[name] = got
    # inverse of the forward outputs of in-range residuals: what an encoder's reconstruction sees
    pairs = [(f"dct_{n}x{n}", f"idct_{n}x{n}", kb.TR_IDCT)]
    if n == 4:
        pairs.append(("fast_forward_dst_4x4", "fast_inverse_dst_4x4", kb.TR_IDST))
    for fwd, inv, kinv in pairs:
        coef = fwd_out[fwd]
        got = host(kb.transform_batch(kinv, n, 10, dev16(kb, coef), len(cases)))
        for i, (label, _, in_range) in enumerate(cases):
            c = cs.al(coef[i * n * n:(i + 1) * n * n], np.int16)
            want = ref10.transform(inv, 10, c, n)
            if in_range:
                for impl in others(ref10, inv):
                    assert np.array_equal(ref10.transform(inv, 10, c, n, impl), want), (inv, label, impl)
            assert np.array_equal(got[i * n * n:(i + 1) * n * n], want), (inv, label)


@pytest.mark.gpu
@pytest.mark.parametrize("qp", QUANT_QPS)
def test_quant_batch_10bit(cuda_lib, ref10, qp):
    kb = cuda_lib
    for n in TR_SIZES:
        blocks = quant_blocks(ref10, n, qp)
        reps = [(b, s) for s in range(3) for b in range(len(blocks))]
        x = dev16(kb, np.concatenate([blocks[b] for b, _ in reps]))
        scans = dev16(kb, np.array([s for _, s in reps], np.int8))
        for intra in (0, 1):
            for signhide in (0, 1):
                for type_ in quant_types(n):
                    q = host(kb.quant_batch(kb.quant_params(qp, 10, intra, signhide), x, n, type_, scans, len(reps)))
                    for i, (b, s) in enumerate(reps):
                        want = ref10.quant(qp, blocks[b], n, n, type_, s, 1, intra, signhide)
                        for impl in others(ref10, "quant"):
                            assert np.array_equal(ref10.quant(qp, blocks[b], n, n, type_, s, 1, intra, signhide, impl), want), \
                                (qp, n, b, s, intra, signhide, type_, impl)
                        assert np.array_equal(q[i * n * n:(i + 1) * n * n], want), (qp, n, b, s, intra, signhide, type_)


@pytest.mark.gpu
@pytest.mark.parametrize("qp", DEQUANT_QPS)
def test_dequant_batch_10bit(cuda_lib, ref10, qp):
    kb = cuda_lib
    for n in TR_SIZES:
        levels = dequant_levels(n)
        x = dev16(kb, np.concatenate(levels))
        for type_ in ((0, 2, 3) if n < 32 else (0,)):
            got = host(kb.dequant_batch(kb.quant_params(qp, 10), x, n, type_, len(levels)))
            for i, lv in enumerate(levels):
                want = ref10.dequant(qp, lv, n, n, type_, 1)
                assert np.array_equal(got[i * n * n:(i + 1) * n * n], want), (qp, n, type_, i)


@pytest.mark.gpu
@pytest.mark.parametrize("qp", QR_QPS)
def test_quantize_residual_batch_10bit(cuda_lib, ref10, qp):
    import torch
    kb = cuda_lib
    src, pred, tus, n_coeff, recs = qres_case(4100 + qp)
    for signhide in (0, 1):
        rec = torch.zeros(src.size, dtype=torch.int16, device="cuda")
        coeff = torch.zeros(n_coeff, dtype=torch.int16, device="cuda")
        has = host(kb.quantize_residual_batch(kb.quant_params(qp, 10, 1, signhide), dev16(kb, src), dev16(kb, pred),
                                              QR_STRIDE, rec, QR_STRIDE, coeff, tus))
        rec_h, coeff_h = host16(rec), host(coeff)
        for i, t in enumerate(tus):
            n = int(t["width"])
            want_has, want_rec, want_coeff = qres_reference(ref10, qp, signhide, src, pred, t)
            o = int(t["off_rec"])
            got_rec = tile(rec_h, o, n, n, QR_STRIDE)
            label = (qp, signhide, i, recs[i])
            assert has[i] == want_has, label
            assert np.array_equal(coeff_h[t["off_coeff"]: t["off_coeff"] + n * n], want_coeff), label
            assert np.array_equal(got_rec, want_rec), label


@pytest.mark.gpu
@pytest.mark.parametrize("log2w", (2, 3, 4, 5))
def test_intra_predict_batch_10bit(cuda_lib, ref10, log2w):
    kb = cuda_lib
    refs = intra_refs(log2w)
    ww = 1 << (2 * log2w)
    count = len(refs) * 35
    top = np.concatenate([refs[i // 35][0] for i in range(count)])
    left = np.concatenate([refs[i // 35][1] for i in range(count)])
    modes = (np.arange(count) % 35).astype(np.int8)
    dt, dl, dm = dev16(kb, top), dev16(kb, left), dev16(kb, modes)
    raw = host16(kb.intra_predict_batch(0, log2w, 0, 0, dt, dl, dm, count))
    for i in range(count):
        t, l, m = refs[i // 35][0], refs[i // 35][1], int(modes[i])
        name = "intra_pred_planar" if m == 0 else ("intra_pred_filtered_dc" if m == 1 else "angular_pred")
        want = ref10.planar(log2w, t, l) if m == 0 else (ref10.filtered_dc(log2w, t, l) if m == 1 else ref10.angular(log2w, m, t, l))
        for impl in others(ref10, name):
            w2 = ref10.planar(log2w, t, l, impl) if m == 0 else (ref10.filtered_dc(log2w, t, l, impl) if m == 1 else ref10.angular(log2w, m, t, l, impl))
            assert np.array_equal(w2, want), (log2w, m, impl)
        assert np.array_equal(raw[i * ww:(i + 1) * ww], want), (log2w, m, i // 35)
    for color in (0, 1):
        for fb in (0, 1):
            full = host16(kb.intra_predict_batch(1, log2w, color, fb, dt, dl, dm, count))
            for i in range(count):
                t, l, m = refs[i // 35][0], refs[i // 35][1], int(modes[i])
                want = ref10.intra_predict(log2w, m, color, t, l, fb)
                assert np.array_equal(full[i * ww:(i + 1) * ww], want), (log2w, m, color, fb, i // 35)


@pytest.mark.gpu
def test_intra_build_reference_batch_10bit(cuda_lib, ref10):
    kb = cuda_lib
    planes = intra_plane_case()
    for log2w in (2, 3, 4, 5):
        for color in (0, 1):
            stride = PIC_W >> (1 if color else 0)
            xy = block_positions(log2w, color)
            top, left = kb.intra_build_reference_batch(log2w, color, dev16(kb, planes[color]), stride, PIC_W, PIC_H, xy)
            top, left = host16(top), host16(left)
            for i, (lx, ly) in enumerate(xy):
                o = ref10.intra_build_reference(log2w, color, lx, ly, PIC_W, PIC_H, planes[color], stride)
                assert np.array_equal(top[i], o[0]) and np.array_equal(left[i], o[1]), (log2w, color, lx, ly)


@pytest.mark.gpu
def test_sample_batch_10bit(cuda_lib, ref10):
    import torch
    kb = cuda_lib
    src, descs = sample_case()
    dsrc = dev16(kb, src)
    kinds = {"luma": kb.IPOL_LUMA, "luma_hi": kb.IPOL_LUMA_HI, "chroma": kb.IPOL_CHROMA, "chroma_hi": kb.IPOL_CHROMA_HI}
    type_names = {"luma": "sample_quarterpel_luma", "luma_hi": "sample_quarterpel_luma_hi",
                  "chroma": "sample_octpel_chroma", "chroma_hi": "sample_octpel_chroma_hi"}
    for name, kind in kinds.items():
        d = np.zeros(len(descs[name]), kb.IPOL)
        off = 0
        for i, (o, w, h, fx, fy) in enumerate(descs[name]):
            d[i] = (o, off, w, h, fx, fy)
            off += w * h + (-(w * h)) % 8
        dst = torch.zeros(off, dtype=torch.int16, device="cuda")
        for w in sorted(set(int(x) for x in d["w"])):     # each block is written with dst_stride = its own width
            kb.sample_batch(kind, dsrc, S_STRIDE, dst, w, d[d["w"] == w])
        out = host(dst)
        for t in d:
            w, h = int(t["w"]), int(t["h"])
            want = ref10.sample(name, src, int(t["off_src"]), S_STRIDE, w, h, int(t["mvx"]), int(t["mvy"]))
            for impl in others(ref10, type_names[name]):
                assert np.array_equal(ref10.sample(name, src, int(t["off_src"]), S_STRIDE, w, h, int(t["mvx"]), int(t["mvy"]), impl=impl), want)
            got = out[t["off_dst"]: t["off_dst"] + w * h]
            assert np.array_equal(got if name.endswith("_hi") else got.view(U16), want), (name, w, h, int(t["mvx"]), int(t["mvy"]))


@pytest.mark.gpu
@pytest.mark.parametrize("fme_level", (1, 2, 3, 4))
def test_filter_fme_batch_10bit(cuda_lib, ref10, fme_level):
    import torch
    kb = cuda_lib
    src, src_offs = fme_case()
    dsrc = dev16(kb, src)
    for (w, h) in FME_SHAPES:
        count = len(FME_OFFS)
        offs = src_offs[(w, h)]
        filt = torch.zeros(count * 4 * 4096, dtype=torch.int16, device="cuda")
        im = torch.zeros(count * 5 * kb.IPOL_IM_SIZE, dtype=torch.int16, device="cuda")
        cols = torch.zeros(count * 5 * kb.IPOL_FIRST_COLS, dtype=torch.int16, device="cuda")
        states = [ref10.fme_state() for _ in range(count)]
        for stage in range(4):
            kb.filter_fme_batch(stage, dsrc, F_STRIDE, offs, w, h, filt, im, fme_level, cols, np.array(FME_OFFS, np.int8))
            f = host16(filt).reshape(count, 4, 64, 64)
            imh = host(im).reshape(count, 5, kb.IPOL_IM_SIZE)
            ch = host(cols).reshape(count, 5, kb.IPOL_FIRST_COLS)
            for b in range(count):
                ref10.filter_fme(stage, src, offs[b], F_STRIDE, w, h, states[b], fme_level, FME_OFFS[b][0], FME_OFFS[b][1])
                want = states[b][0].reshape(4, 64, 64)
                label = (w, h, fme_level, stage, FME_OFFS[b])
                assert np.array_equal(f[b][:, :h, :w], want[:, :h, :w]), label
                wim = states[b][1].reshape(5, -1)
                for k in ((0, 1) if stage < 2 else (0, 1, 3, 4)):
                    assert np.array_equal(imh[b, k, : (h + 8) * 64].reshape(-1, 64)[:, :w],
                                          wim[k, : (h + 8) * 64].reshape(-1, 64)[:, :w]), label + (k,)
                wc = states[b][2].reshape(5, -1)
                for k in ((0, 2) if stage < 2 else (0, 1, 2, 3)):
                    assert np.array_equal(ch[b, k, : h + 8], wc[k, : h + 8]), label + (k,)


@pytest.mark.gpu
def test_extend_block_10bit(cuda_lib, ref10):
    kb = cuda_lib
    src = rp(cs.rng(850), EXT_S * EXT_H, "extreme")
    n_copied = 0
    for (bx, by) in EXT_PLACES:
        for (bw, bh) in EXT_SIZES:
            for pads in EXT_PADS:
                o = ref10.get_extended_block(src, EXT_W, EXT_H, EXT_S, bx, by, bw, bh, *pads)
                if not o[0]:
                    continue          # block + padding inside the frame: the reference returns a pointer, no copy
                got = host16(kb.extend_block(dev16(kb, src), EXT_W, EXT_H, EXT_S, bx, by, bw, bh, *pads))
                assert np.array_equal(got, o[1][: got.size]), (bx, by, bw, bh, pads)
                n_copied += 1
    assert n_copied > 0


@pytest.mark.gpu
def test_block_costs_10bit(cuda_lib, ref10):
    kb = cuda_lib
    a, b, dl = block_cost_case()
    descs = np.array([(oa, ob, w, h, 0, 0) for (oa, ob, w, h, _, _) in dl], kb.BLK)
    hd = np.array(dl, kb.BLK)
    da, db = dev16(kb, a), dev16(kb, b)
    sad = costs(kb.block_cost_batch(kb.OP_REG_SAD, da, B_SA, db, B_SB, descs))
    ver = costs(kb.block_cost_batch(kb.OP_VER_SAD, da, B_SA, db, B_SB, descs))
    hor = costs(kb.block_cost_batch(kb.OP_HOR_SAD, da, B_SA, db, B_SB, hd))
    satd = costs(kb.block_cost_batch(kb.OP_SATD_ANY, da, B_SA, db, B_SB, descs))
    for i, d in enumerate(hd):
        w, h, oa, ob = int(d["w"]), int(d["h"]), int(d["off_a"]), int(d["off_b"])
        assert sad[i] == ref10.reg_sad(a[oa:], b[ob:], w, h, B_SA, B_SB), (i, w, h)
        assert ver[i] == ref10.ver_sad(a[oa:], b[ob:], w, h, B_SA), (i, w, h)
        assert hor[i] == ref10.hor_sad(a[oa:], b[ob:], w, h, B_SA, B_SB, int(d["left"]), int(d["right"])), (i, w, h)
        assert satd[i] == ref10.satd_any_size(w, h, a[oa:], B_SA, b[ob:], B_SB), (i, w, h)
    ssd_d = descs[[i for i, d in enumerate(descs) if d["w"] == d["h"] and d["w"] in (4, 8, 16, 32, 64)]]
    ssd = costs(kb.block_cost_batch(kb.OP_SSD, da, B_SA, db, B_SB, ssd_d))
    for i, d in enumerate(ssd_d):
        assert ssd[i] == ref10.pixels_calc_ssd(a[d["off_a"]:], b[d["off_b"]:], B_SA, B_SB, int(d["w"])), i


@pytest.mark.gpu
def test_pixel_var_batch_10bit(cuda_lib, ref10):
    kb = cuda_lib
    bufs = pixel_var_bufs()
    got = host(kb.pixel_var_batch(dev16(kb, np.concatenate(bufs)), 4096, len(bufs)))
    for i, buf in enumerate(bufs):
        assert got[i] == ref10.pixel_var(buf), i                    # equal doubles: same summation order


@pytest.mark.gpu
def test_bipred_average_plane_10bit(cuda_lib, orc10):
    import torch
    kb = cuda_lib
    for (w, h, px, im) in bipred_case():
        for f0 in (0, 1):
            for f1 in (0, 1):
                l0, l1 = im[0] if f0 else px[0], im[1] if f1 else px[1]
                dst = torch.zeros(64 * 64, dtype=torch.int16, device="cuda")
                kb.bipred_average_plane(dst, 64, dev16(kb, l0), dev16(kb, l1), f0, f1, w, h, 10)
                want = orc10.bipred_average_plane(l0, l1, f0, f1, w, h, 64)
                got = host16(dst)
                assert np.array_equal(got[: h * 64].reshape(h, 64)[:, :w], want[: h * 64].reshape(h, 64)[:, :w]), (w, h, f0, f1)


@pytest.mark.gpu
def test_sao_stats_and_distortions_10bit(cuda_lib, ref10):
    kb = cuda_lib
    shapes, origs, recs, eo, offsets, band_pos, bands = sao_block_case()
    blks = np.zeros(len(shapes), kb.SAO_BLK)
    off = 0
    for i, (bw, bh) in enumerate(shapes):
        blks[i] = (off, off, bw, bh, 0, 0)
        off += bw * bh
    do, dr = dev16(kb, np.concatenate(origs)), dev16(kb, np.concatenate(recs))
    stats = host(kb.sao_edge_stats_batch(10, do, dr, blks))
    dd = host(kb.sao_edge_ddistortion_batch(10, do, dr, blks, eo, offsets))
    bd = host(kb.sao_band_ddistortion_batch(10, do, dr, blks, band_pos, bands))
    for i, (bw, bh) in enumerate(shapes):
        o, rc = origs[i], recs[i]
        for e in range(4):
            assert np.array_equal(stats[i, e].ravel(), ref10.calc_sao_edge_dir(o, rc, e, bw, bh)), (i, e)
        assert dd[i] == ref10.sao_edge_ddistortion(o, rc, bw, bh, int(eo[i]), offsets[i]), i
        assert bd[i] == ref10.sao_band_ddistortion(o, rc, bw, bh, int(band_pos[i]), bands[i]), i


@pytest.mark.gpu
def test_sao_reconstruct_batch_10bit(cuda_lib, ref10):
    import torch
    kb = cuda_lib
    rec, dl = sao_rec_case()
    descs = np.zeros(len(dl), kb.SAO_REC)
    for i, (off_rec, bw, bh, type_, eo, color, bp, offs) in enumerate(dl):
        descs[i]["off_rec"], descs[i]["off_new"] = off_rec, i * 64 * SR_NEW_STRIDE
        descs[i]["bw"], descs[i]["bh"] = bw, bh
        descs[i]["type"], descs[i]["eo_class"], descs[i]["color"] = type_, eo, color
        descs[i]["band_position"], descs[i]["offsets"] = bp, offs
    new = torch.zeros(len(dl) * 64 * SR_NEW_STRIDE, dtype=torch.int16, device="cuda")
    kb.sao_reconstruct_batch(10, dev16(kb, rec), SR_STRIDE, new, SR_NEW_STRIDE, descs)
    out = host16(new)
    for i, (off_rec, bw, bh, type_, eo, color, bp, offs) in enumerate(dl):
        got = out[i * 64 * SR_NEW_STRIDE:][: bh * SR_NEW_STRIDE].reshape(bh, SR_NEW_STRIDE)[:, :bw]
        assert np.array_equal(got, sao_rec_reference(ref10, rec, dl[i])), (i, bw, bh, type_, eo, color)


def sao_rec_reference(ref10, rec, d, impl="generic"):
    off_rec, bw, bh, type_, eo, color, bp, offs = d
    if type_ == 0:
        return np.stack([rec[off_rec + y * SR_STRIDE: off_rec + y * SR_STRIDE + bw] for y in range(bh)])
    return ref10.sao_reconstruct_color(rec, off_rec, type_, eo, bp, offs, SR_STRIDE, SR_NEW_STRIDE, bw, bh, color,
                                       impl).reshape(bh, SR_NEW_STRIDE)[:, :bw]


@pytest.mark.gpu
def test_array_checksum_10bit(cuda_lib, ref10):
    kb = cuda_lib
    for (w, h, stride) in CHECKSUM_CASES:
        data = checksum_data(w, h, stride)
        want = ref10.array_checksum(data, h, w, stride)
        for impl in others(ref10, "array_checksum"):
            assert np.array_equal(ref10.array_checksum(data, h, w, stride, impl), want), (w, h, impl)
        assert np.array_equal(host(kb.array_checksum(dev16(kb, data), h, w, stride)), want), (w, h)


# ############################################################################################ CPU: pins and reach
def test_orc10_bipred_plane_vs_ref10(orc10, ref10):
    """The plane form of bi-prediction in the oracle's 10-bit build == the reference's 10-bit bipred_average (luma and
    both chroma planes, every flag combination), on the cases the GPU test uses."""
    r = cs.rng(970)
    for (w, h, px, im) in bipred_case():
        if w < 8 or h < 8:
            continue
        cpx = [dict(y=p, u=rp(r, w * h // 4, "extreme"), v=rp(r, w * h // 4)) for p in px]
        cim = [dict(y=m, u=cs.al(m[: w * h // 4]), v=cs.al(m[w * h // 4: w * h // 2])) for m in im]
        for f0 in range(4):
            for f1 in range(4):
                for impl in impls(ref10, "bipred_average"):
                    ry, ru, rv = ref10.bipred_average(cpx[0], cpx[1], cim[0], cim[1], 0, 0, w, h, f0, f1, impl)
                    oy = orc10.bipred_average_plane(cim[0]["y"] if f0 & 1 else cpx[0]["y"], cim[1]["y"] if f1 & 1 else cpx[1]["y"],
                                                    f0 & 1, f1 & 1, w, h, 64)
                    assert np.array_equal(oy[: h * 64].reshape(h, 64)[:, :w], ry.reshape(64, 64)[:h, :w]), (w, h, f0, f1)
                    for pl, rr in (("u", ru), ("v", rv)):
                        o = orc10.bipred_average_plane(cim[0][pl] if f0 & 2 else cpx[0][pl], cim[1][pl] if f1 & 2 else cpx[1][pl],
                                                       (f0 >> 1) & 1, (f1 >> 1) & 1, w // 2, h // 2, 32)
                        assert np.array_equal(o[: h // 2 * 32].reshape(h // 2, 32)[:, : w // 2],
                                              rr.reshape(32, 32)[: h // 2, : w // 2]), (w, h, f0, f1, pl)


def test_reach_walsh_closed_form_and_lane_peak(ref10):
    """Every Walsh case's reference SATD equals the closed form, and the 8x8 cases bring a packed Hadamard lane of
    satd.cuh to 1023 * 32 = 32736, 32 short of 2^15."""
    for n in (4, 8, 16, 32, 64):
        for s in walsh_square_cases(n):
            a, b = walsh_pair(s)
            assert ref10.nxn("satd", n, cs.al(a.ravel()), cs.al(b.ravel())) == satd_nxn_closed(n), n
            if n == 8:
                assert packed_lane_peak(a.astype(np.int64) - b) == PMAX * 32
        preds, origs, pitch, count = dual_case(n)
        for i in range(count):
            got = ref10.nxn_dual("satd", n, cs.al(preds[i * pitch: i * pitch + 1024 + n * n]), cs.al(origs[i * n * n:(i + 1) * n * n]))
            assert list(got) == dual_closed(n, i), (n, i)
    a, b, cases = any_size_case()
    for (w, h, oa, ob, sign) in cases:
        n8 = sum(1 for t in any_size_tiles(w, h) if t[2] == 8)
        n4 = len(any_size_tiles(w, h)) - n8
        closed = (n8 * SATD8_WALSH + n4 * SATD4_WALSH) >> 2
        assert sum(ww * ww for _, _, ww in any_size_tiles(w, h)) == w * h        # the tiling covers the block
        assert satd_tiles(PMAX * sign, any_size_tiles(w, h)) == closed
        assert ref10.satd_any_size(w, h, a[oa:], SA, b[ob:], SB) == closed, (w, h)
    preds, orig, qcases = quad_case()
    for (w, h, o) in qcases:
        want = ref10.satd_any_size_quad(w, h, [p[o:] for p in preds], QS, orig[o:], QS)
        assert list(want) == quad_model(preds, orig, w, h, o), (w, h)
        if w % 8 == 0 or h % 8 == 0:
            tiles = quad_tiles(w, h)
            n8 = sum(1 for t in tiles if t[2] == 8)
            closed = (n8 * SATD8_WALSH + (len(tiles) - n8) * SATD4_WALSH) >> 2
            assert list(want) == [closed, 0, closed, 0], (w, h)


@pytest.mark.parametrize("log2w", (2, 3, 4, 5))
def test_reach_walsh_rough_search(ref10, log2w):
    """Away from the first block the references are flat, every mode predicts the flat value, and each block's cost is
    the closed form of its Walsh pattern."""
    w = 1 << log2w
    for inverted in (0, 1):
        src, rec, pic_w, pic_h = rough_walsh_case(log2w, inverted)
        costs = rough_reference(ref10, log2w, src, rec, pic_w, pic_h)
        assert (costs[1:] == satd_nxn_closed(w)).all(), (log2w, inverted)
        assert (costs[0] != satd_nxn_closed(w)).any()


def test_reach_transform_inputs(ref10):
    for n in TR_SIZES:
        cases = transform_cases(n)
        x = np.concatenate([c[1] for c in cases]).astype(np.int64)
        assert x.min() == -32768 and x.max() == 32767
        walsh_blocks = [c[1] for c in cases if c[0].startswith("walsh")]
        assert all(np.abs(b).min() == PMAX for b in walsh_blocks)
        # the DC Walsh case puts the whole block into one coefficient
        dc = ref10.transform(f"dct_{n}x{n}", 10, walsh_blocks[0], n)
        assert np.count_nonzero(dc) == 1 and abs(int(dc[0])) > 0


def test_reach_quant_levels_and_sign_hiding(ref10):
    """QP 51 chroma and QP 0 quantise to non-zero levels, and sign hiding changes at least one block."""
    for n in TR_SIZES:
        for qp, type_ in ((51, quant_types(n)[-1]), (0, 0), (0, quant_types(n)[-1])):
            blocks = quant_blocks(ref10, n, qp)
            assert any(np.count_nonzero(ref10.quant(qp, b, n, n, type_, 0, 1, 1, 0)) for b in blocks), (n, qp, type_)
        changed = 0
        for qp in QUANT_QPS:
            for b in quant_blocks(ref10, n, qp):
                for scan in range(3):
                    changed += not np.array_equal(ref10.quant(qp, b, n, n, 0, scan, 1, 1, 0), ref10.quant(qp, b, n, n, 0, scan, 1, 1, 1))
        assert changed > 0, n


def test_reach_dequant_clip(ref10):
    """Dequantised outputs hit -32768 and 32767 (the int16 clip) at QP 51."""
    for n in TR_SIZES:
        out = np.concatenate([ref10.dequant(51, lv, n, n, 0, 1) for lv in dequant_levels(n)])
        assert out.min() == -32768 and out.max() == 32767, n


def test_reach_quantize_residual(ref10):
    """The seeded TUs give blocks with and without coefficients, reconstructions at 0 and 1023, transform skip in use,
    and every colour / scan / intra-inter combination."""
    for qp in QR_QPS:
        src, pred, tus, _, recs = qres_case(4100 + qp)
        has_set, lo, hi = set(), False, False
        for t in tus:
            h, rec, _ = qres_reference(ref10, qp, 1, src, pred, t)
            has_set.add(bool(h))
            lo |= bool((rec == 0).any())
            hi |= bool((rec == PMAX).any())
        assert has_set == {True, False} and lo and hi, qp
        assert {(c, s, i) for (_, _, c, s, _, i) in recs} == {(c, s, i) for c in range(3) for s in range(3) for i in range(2)}
        assert any(tr for (_, _, _, _, tr, _) in recs)


@pytest.mark.parametrize("log2w", (2, 3, 4))
def test_reach_intra_edge_filter_clips(ref10, log2w):
    """The vertical / horizontal edge filters of luma blocks under 32 go outside 0..1023 unclipped on the seeded
    references -- at both ends -- and the reference clips them."""
    below = above = False
    for top, left in intra_refs(log2w):
        for mode in (10, 26):
            u = edge_filter_unclipped(log2w, mode, top, left)
            out = ref10.intra_predict(log2w, mode, 0, top, left, 1).reshape(1 << log2w, 1 << log2w)
            edge = out[:, 0] if mode == 26 else out[0, :]
            assert np.array_equal(edge, np.clip(u, 0, PMAX)), (log2w, mode)
            below |= bool((u < 0).any())
            above |= bool((u > PMAX).any())
    assert below and above


def test_reach_intra_build_reference(ref10):
    """The 200x136 picture gives exactly one block with no neighbours (all 512) and blocks whose below-left or
    above-right half is unavailable (filled by repeating the last available sample)."""
    planes = intra_plane_case()
    for log2w in (2, 3, 4, 5):
        n = 1 << log2w
        for color in (0, 1):
            stride = PIC_W >> (1 if color else 0)
            all512 = partial = 0
            for (lx, ly) in block_positions(log2w, color):
                top, left = ref10.intra_build_reference(log2w, color, lx, ly, PIC_W, PIC_H, planes[color], stride)
                if (top == 512).all() and (left == 512).all():
                    all512 += 1
                elif (left[n + 1:] == left[n]).all() or (top[n + 1:] == top[n]).all():
                    partial += 1
            assert all512 == 1 and partial > 0, (log2w, color)


def test_reach_sample_clips(ref10):
    """Luma and chroma pixel outputs clip: their 14-bit forms lie outside the 10-bit range by more than rounding."""
    src, descs = sample_case()
    for hi_name in ("luma_hi", "chroma_hi"):
        low = high = False
        for (o, w, h, fx, fy) in descs[hi_name]:
            if fx == 0 and fy == 0:
                continue
            v = ref10.sample(hi_name, src, o, S_STRIDE, w, h, fx, fy).astype(np.int64)
            low |= bool((v < -32).any())
            high |= bool((v > (PMAX + 2) * 16).any())
        assert low and high, hi_name
    for name in ("luma", "chroma"):
        outs = np.concatenate([ref10.sample(name, src, o, S_STRIDE, w, h, fx, fy) for (o, w, h, fx, fy) in descs[name][:64]])
        assert outs.min() == 0 and outs.max() == PMAX


def test_reach_block_cost_ssd_above_int32(ref10):
    a, b, dl = block_cost_case()
    big = [ref10.pixels_calc_ssd(a[oa:], b[ob:], B_SA, B_SB, w) for (oa, ob, w, h, _, _) in dl if w == h == 64]
    assert max(big) >= 2 ** 31


def test_reach_bipred_clips(orc10):
    low = high = False
    for (w, h, _, im) in bipred_case():
        u = (im[0].astype(np.int64) + im[1] + 16) >> 5
        low |= bool((u < 0).any())
        high |= bool((u > PMAX).any())
        out = orc10.bipred_average_plane(im[0], im[1], 1, 1, w, h, w)
        assert out.min() == 0 and out.max() == PMAX
    assert low and high


def test_reach_sao(ref10):
    """Offsets reach +-31, band positions 0 and 28-31 occur, and reconstructions clip at 0 and at 1023."""
    _, _, _, _, offsets, band_pos, bands = sao_block_case()
    assert offsets.min() == -31 and offsets.max() == 31 and bands.min() == -31 and bands.max() == 31
    assert set(band_pos.tolist()) == {0, 28, 29, 30, 31}
    rec, dl = sao_rec_case()
    assert {d[3] for d in dl} == {0, 1, 2} and {d[4] for d in dl} == {0, 1, 2, 3} and {d[5] for d in dl} == {0, 1, 2}
    assert {(d[1], d[2]) for d in dl} == set(SR_SHAPES)
    clip0 = clip1023 = False
    for d in dl:
        off_rec, bw, bh = d[0], d[1], d[2]
        if d[3] == 0:
            continue
        got = sao_rec_reference(ref10, rec, d).astype(np.int64)
        src = np.stack([rec[off_rec + y * SR_STRIDE: off_rec + y * SR_STRIDE + bw] for y in range(bh)]).astype(np.int64)
        clip0 |= bool(((got == 0) & (src > 0)).any())
        clip1023 |= bool(((got == PMAX) & (src < PMAX)).any())
    assert clip0 and clip1023
