"""CTU search driver: the back half of every CTU's job -- ctu_store, ctu_deblock, ctu_sao_search, ctu_track_models and
ctu_sao_apply of kvazaar_b200/csrc/ctu/ctu_frame.h -- against the reference's own CTU job, CTU by CTU, on INJECTED CTU
decisions (CU records, pre-deblock reconstruction, coefficients, source), never on a search.

  * tests/cuda/ctu_frame_probe.cu runs the driver's code with search_ctu replaced by injection: the host build
    (tests/hostsim/libkvzctu_frame_probe_host.so, one-thread CTA) and the device build (tests/cuda/libkvzctu_frame_probe.so,
    one 128-thread CTA per CTU, one launch per wavefront anti-diagonal);
  * oracle/ref_frame.c (oracle/_ref/libkvzref_frame{,_10b}.so) encodes one picture with the reference, its
    kvz_search_lcu replaced at link time by the same injection, and captures what the reference's CTU job made of it.

Compared exactly: the deblocked and the final picture, the 184 model bytes at every CTU's start and after its syntax,
and both SAO records of every CTU.  The generator makes decisions the reference's search could have made and content
chosen for the operation under test: DC steps across transform units for every deblocking decision, saturated
pictures, reconstruction = source + bias so that SAO offsets clip, samples gathered in the first and last bands, flat
areas where SAO costs tie.
"""
import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np
import pytest

from test_ctu_driver import ROOT
from test_rdoq import lambda_for

PROBE_SRC = os.path.join(ROOT, "tests", "cuda", "ctu_frame_probe.cu")
PROBE_HOST = os.path.join(ROOT, "tests", "hostsim", "libkvzctu_frame_probe_host.so")
PROBE_CUDA = os.path.join(ROOT, "tests", "cuda", "libkvzctu_frame_probe.so")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
CFG = np.dtype([("v", "<i4", (21,)), ("lambda", "<f8"), ("lambda_sqrt", "<f8")], align=True)    # CtuConfig
CUREC = np.dtype([("type", "u1"), ("depth", "u1"), ("part_size", "u1"), ("tr_depth", "u1"), ("tr_skip", "u1"), ("qp", "u1"),
                  ("mode", "i1"), ("mode_chroma", "i1"), ("cbf", "<u2"), ("pad", "<u2")])                  # CuRec / cu_info_t
SAO = np.dtype([("type", "<i4"), ("eo_class", "<i4"), ("ddistortion", "<i4"), ("merge_left_flag", "<i4"), ("merge_up_flag", "<i4"),
                ("band_position", "<i4", (2,)), ("offsets", "<i4", (10,))])                                 # SaoRec / sao_info_t
assert CUREC.itemsize == 12 and SAO.itemsize == 68
CTX = 184
FILLS = (0x00, 0xA5)
SIZES = ((64, 64), (72, 72), (136, 200), (200, 136), (264, 136))
WIDE = (1000, 520)          # 16 x 9 CTUs: eight CTUs on the widest anti-diagonals; 40- and 8-pixel partial CTUs
QPS = (0, 1, 15, 30, 37, 45, 51)
DEBLOCK = (None, (0, 0), (-6, -6), (6, 6), (-3, 3))     # None: off; else (beta, tc) offsets
SAO_TYPES = (0, 1, 2, 3)                                 # off, edge, band, both
THEMES = ("steps", "bias", "bands0", "flat", "bands28", "sat0", "satmax", "noise")


def _probe_host():
    if not os.path.exists(PROBE_HOST):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unused-function", "-Wno-unknown-pragmas",
                               "-x", "c++", "-o", PROBE_HOST, PROBE_SRC])
    return PROBE_HOST


def _ref_frame_lib(bitdepth):
    so = os.path.join(REF_DIR, "libkvzref_frame.so" if bitdepth == 8 else "libkvzref_frame_10b.so")
    return so if os.path.exists(so) else None


# ------------------------------------------------------------------------------------------------ decisions
def zorder(width, x, y):
    """xy_to_zorder: offset of the 4-aligned position (x, y) inside an lcu_coeff_t plane of `width`"""
    r = 0
    if width == 64:
        r += (x >> 5) * 1024 + (y >> 5) * 2048
        x &= 31
        y &= 31
    if width >= 32:
        r += (x >> 4) * 256 + (y >> 4) * 512
        x &= 15
        y &= 15
    if width >= 16:
        r += (x >> 3) * 64 + (y >> 3) * 128
        x &= 7
        y &= 7
    if width >= 8:
        r += (x >> 2) * 16 + (y >> 2) * 32
    return r


def cbf_bit(depth, plane):
    return (0x10 >> depth) << (5 * plane)


@dataclass
class Case:
    bd: int
    w: int
    h: int
    qp: int
    sao: int
    dbk: object
    trskip: int
    theme: str
    lam: float
    cu: np.ndarray = None           # [h / 4][w / 4] CUREC
    coeff: np.ndarray = None        # [nctu][6144] int16, lcu_coeff_t layout
    src: np.ndarray = None          # Y, U, V planes back to back
    rec: np.ndarray = None          # pre-deblock reconstruction, same layout
    stats: dict = field(default_factory=dict)

    @property
    def wl(self):
        return (self.w + 63) // 64

    @property
    def hl(self):
        return (self.h + 63) // 64

    @property
    def nctu(self):
        return self.wl * self.hl

    @property
    def max(self):
        return (1 << self.bd) - 1

    @property
    def pix(self):
        return np.uint8 if self.bd == 8 else np.uint16

    @property
    def cmax(self):
        return (1 << (min(self.bd, 10) - 5)) - 1

    def name(self):
        d = "off" if self.dbk is None else f"{self.dbk[0]}:{self.dbk[1]}"
        return f"{self.bd}b {self.w}x{self.h} qp {self.qp} sao {self.sao} deblock {d} ts {self.trskip} {self.theme} lambda {self.lam:.4f}"

    def planes(self, a):
        ny, nc = self.w * self.h, self.w * self.h // 4
        return a[:ny].reshape(self.h, self.w), a[ny:ny + nc].reshape(self.h // 2, self.w // 2), a[ny + nc:].reshape(self.h // 2, self.w // 2)


class Gen:
    """Seeded legal decisions and targeted content for one case."""

    def __init__(self, case, rng):
        self.c, self.r = case, rng
        c = case
        self.cu = np.zeros((c.h // 4, c.w // 4), CUREC)
        self.coeff = np.zeros((c.nctu, 6144), np.int16)
        self.tus = []               # (plane, x, y, n) in picture samples of the plane: the transform units, for content
        self.n = dict(border_split=0, nxn=0, cu64=0, tr_skip=0)
        # how deep the quadtree goes: the mix changes with the case so that every size meets every other
        self.p_split = (rng.uniform(0.3, 1.0), rng.uniform(0.2, 0.9), rng.uniform(0.2, 0.9))
        self.p_nxn = rng.uniform(0.2, 0.8)
        self.p_zero = rng.uniform(0.1, 0.6)

    def levels(self, n):
        r = self.r
        q = np.zeros(n * n, np.int16)
        if r.random() < self.p_zero:
            return q
        k = int(r.integers(1, max(2, n * n // 4)))
        pos = r.choice(n * n, k, replace=False)
        mag = r.integers(1, 4, k)
        big = r.random(k) < 0.15
        mag[big] = r.integers(4, 3000, int(big.sum()))          # Golomb-Rice escapes
        q[pos] = mag * r.choice([-1, 1], k)
        return q

    def put(self, ctu, plane, xl, yl, n, q):
        """levels of the unit at CTU-local (xl, yl) of its plane (chroma: chroma samples)"""
        off = (0, 4096, 5120)[plane] + zorder(64 if plane == 0 else 32, xl, yl)
        self.coeff[ctu, off:off + n * n] = q

    def fill(self, x, y, size, **kv):
        blk = self.cu[y >> 2:(y + size) >> 2, x >> 2:(x + size) >> 2]
        for k, v in kv.items():
            blk[k] = v

    def ctu(self, cx, cy):
        self.tree(cx, cy, cx * 64, cy * 64, 0)

    def tree(self, cx, cy, x, y, d):
        c, r = self.c, self.r
        size = 64 >> d
        if x >= c.w or y >= c.h:
            return
        if x + size > c.w or y + size > c.h:
            self.n["border_split"] += 1
            split = True
        else:
            split = d < 3 and r.random() < self.p_split[d]
        if split:
            h = size // 2
            for (ox, oy) in ((0, 0), (h, 0), (0, h), (h, h)):
                self.tree(cx, cy, x + ox, y + oy, d + 1)
            return
        self.leaf(cx, cy, x, y, d)

    def chroma_mode(self, luma):
        cands = [34 if m == luma else m for m in (0, 26, 10, 1)] + [luma]
        return cands[int(self.r.integers(0, 5))]

    def leaf(self, cx, cy, x, y, d):
        c, r = self.c, self.r
        ctu = cy * c.wl + cx
        xl, yl = x & 63, y & 63
        nxn = d == 3 and r.random() < self.p_nxn
        size = 64 >> d
        if nxn:
            modes = [int(m) for m in r.integers(0, 35, 4)]
            self.fill(x, y, 8, type=1, depth=3, part_size=3, tr_depth=4, qp=c.qp, mode_chroma=self.chroma_mode(modes[0]), cbf=0, tr_skip=0)
            for j in range(4):
                px, py = x + 4 * (j & 1), y + 4 * (j >> 1)
                q = self.levels(4)
                rec = self.cu[py >> 2, px >> 2]
                rec["mode"] = modes[j]
                if q.any():
                    rec["cbf"] |= cbf_bit(4, 0)
                    if c.trskip and r.random() < 0.5:
                        rec["tr_skip"] = 1
                        self.n["tr_skip"] += 1
                self.put(ctu, 0, px & 63, py & 63, 4, q)
                self.tus.append((0, px, py, 4))
            tl = self.cu[y >> 2, x >> 2]
            for p in (1, 2):            # the 8x8 CU's one 4x4 chroma unit: bits at depth 4 on its top-left record
                q = self.levels(4)
                if q.any():
                    tl["cbf"] |= cbf_bit(4, p)
                self.put(ctu, p, xl // 2, yl // 2, 4, q)
            self.tus.append((1, x // 2, y // 2, 4))
            self.n["nxn"] += 1
            return
        mode = int(r.integers(0, 35))
        trd = 1 if d == 0 else d
        self.fill(x, y, size, type=1, depth=d, part_size=0, tr_depth=trd, qp=c.qp, mode=mode, mode_chroma=self.chroma_mode(mode), cbf=0, tr_skip=0)
        tsz = 64 >> trd
        offs = ((0, 0), (32, 0), (0, 32), (32, 32)) if d == 0 else ((0, 0),)
        for (ox, oy) in offs:            # each unit's bits on its top-left record (kvz_intra_recon_cu)
            rec = self.cu[(y + oy) >> 2, (x + ox) >> 2]
            for p in (0, 1, 2):
                n = tsz if p == 0 else tsz // 2
                q = self.levels(n)
                if q.any():
                    rec["cbf"] |= cbf_bit(trd, p)
                self.put(ctu, p, (xl + ox) if p == 0 else (xl + ox) // 2, (yl + oy) if p == 0 else (yl + oy) // 2, n, q)
            self.tus.append((0, x + ox, y + oy, tsz))
            self.tus.append((1, (x + ox) // 2, (y + oy) // 2, tsz // 2))
        if d == 0:
            # the 64x64 CU's parent bits: set when one of the units 1..3 has them (cbf_set_conditionally)
            tl = self.cu[y >> 2, x >> 2]
            kids = [int(self.cu[(y + oy) >> 2, (x + ox) >> 2]["cbf"]) for (ox, oy) in offs[1:]]
            for p in (0, 1, 2):
                if any(k & cbf_bit(1, p) for k in kids):
                    tl["cbf"] |= cbf_bit(0, p)
            self.n["cu64"] += 1

    # ---- content
    def content(self):
        c, r, mx = self.c, self.r, self.c.max
        s = 1 << (c.bd - 8)
        theme = c.theme
        ny, nc = c.w * c.h, c.w * c.h // 4
        rec = np.zeros(ny + 2 * nc, np.int64)
        src = np.zeros_like(rec)
        ry, ru, rv = c.planes(rec)
        sy, su, sv = c.planes(src)
        for (py, ps) in ((ry, sy), (ru, su), (rv, sv)):
            hh, ww = py.shape
            if theme in ("steps", "noise", "bias"):
                # one DC per transform unit, steps of every size between them, textures of every strength inside
                base = int(r.integers(mx // 4, 3 * mx // 4))
                py[:] = base
            elif theme in ("bands0", "bands28"):
                # samples in four bands at one end, the other bands empty
                bands = [0, 1, 2, 3] if theme == "bands0" else [28, 29, 30, 31]
                py[:] = r.choice(bands, (hh, ww)) * (mx + 1) // 32 + r.integers(0, (mx + 1) // 32, (hh, ww))
            elif theme == "flat":
                py[:] = int(r.integers(0, mx + 1))
            elif theme == "dips":
                py[:] = (mx + 1) // 2
                py[2::4, 2::4] -= 2 << (c.bd - 8)       # a band of their own; local minima in every direction
            elif theme == "sat0":
                py[:] = np.minimum(r.integers(0, 3 * s, (hh, ww)), mx)
            elif theme == "satmax":
                py[:] = np.maximum(mx - r.integers(0, 3 * s, (hh, ww)), 0)
        if theme in ("steps", "noise", "bias"):
            for (plane, x, y, n) in self.tus:
                for t in ((ry,) if plane == 0 else (ru, rv)):
                    hh, ww = t.shape
                    if x >= ww or y >= hh:
                        continue
                    step = int(r.choice([0, 1, 2, 3, 5, 8, 12, 20, 40, 90])) * s * int(r.choice([-1, 1]))
                    tex = int(r.choice([0, 0, 1, 2, 3, 6])) * s
                    blk = t[y:y + n, x:x + n]
                    blk += step
                    if tex:
                        blk += r.integers(-tex, tex + 1, blk.shape)
            if theme == "noise":
                rec[:] = r.integers(0, mx + 1, rec.size)
            np.clip(rec, 0, mx, out=rec)
        # the source: the reconstruction plus a bias field (large, so that offsets clip), or nearly the reconstruction
        if theme == "bias":
            # edge statistics keep 8-bit precision: at 10 bits the bias must reach 4 * 31 for the offsets to clip
            bias = int(r.choice([-1, 1])) * (int(r.integers(c.cmax + 1, 2 * c.cmax + 2)) << (c.bd - 8))
            src[:] = rec + bias + r.integers(-1, 2, rec.size)
        elif theme in ("bands0", "bands28"):
            src[:] = rec + (9 if theme == "bands0" else -9) * s + r.integers(-2 * s, 2 * s + 1, rec.size)
        elif theme == "flat":
            src[:] = rec
        elif theme == "dips":
            src[:] = rec + (rec < (mx + 1) // 2)
        elif theme in ("sat0", "satmax"):
            src[:] = rec + (1 if theme == "sat0" else -1) * r.integers(0, 12 * s, rec.size)
        else:
            amp = int(r.choice([1, 3, 10])) * s
            src[:] = rec + r.integers(-amp, amp + 1, rec.size)
        np.clip(src, 0, mx, out=src)
        return src.astype(c.pix), rec.astype(c.pix)


def make_case(bd, w, h, qp, sao, dbk, trskip, theme, seed, lam=None):
    rng = np.random.default_rng(seed)
    c = Case(bd, w, h, qp, sao, dbk, trskip, theme, lam if lam is not None else lambda_for(qp) * float(rng.uniform(0.5, 2.0)))
    g = Gen(c, rng)
    for cy in range(c.hl):
        for cx in range(c.wl):
            g.ctu(cx, cy)
    c.cu, c.coeff = g.cu, g.coeff
    c.src, c.rec = g.content()
    c.stats = dict(g.n)
    return c


def make_cases(bd):
    """Every size, QP, deblocking switch, SAO type, transform-skip switch and theme, each with the others cycling."""
    out = []
    for i in range(35):
        w, h = SIZES[i % len(SIZES)]
        out.append(make_case(bd, w, h, QPS[i % len(QPS)], SAO_TYPES[(i // 5) % 4], DEBLOCK[i % len(DEBLOCK)], (i // 7) % 2,
                             THEMES[(i + i // 7) % len(THEMES)], 1000 * bd + i))
    # QP 51 with the tc offsets that reach the clip of the tc index at 53
    for j, dbk in enumerate(((0, 0), (6, 6), (-3, 3))):
        out.append(make_case(bd, 136, 72, 51, 3, dbk, j & 1, "steps", 3000 + 10 * bd + j))
    # exact ties: isolated one-sample dips, one too dark, in flat pictures at a lambda that makes every SAO rate cost 0;
    # at 8 bits edge and band offsets then lower the distortion by the same amount, so `edge <= band` and the merge
    # choices' `<=` / `<` decide (at 10 bits the edge statistics' rounding breaks the tie)
    for j, sao in enumerate((3, 3, 2, 1)):
        out.append(make_case(bd, (64, 136, 200, 136)[j], (64, 72, 136, 200)[j], (0, 1, 15, 30)[j], sao, None, 0, "dips", 5000 + 10 * bd + j, lam=0.01))
    # the wide picture: eight CTUs per anti-diagonal
    out.append(make_case(bd, *WIDE, 30, 3, (0, 0), 1, "steps", 4000 + bd))
    out.append(make_case(bd, *WIDE, 37, 3, (-3, 3), 0, "bias", 4100 + bd))
    return out


# ------------------------------------------------------------------------------------------------ running
def _cfg(c):
    cfg = np.zeros(1, CFG)
    v = cfg[0]["v"]
    v[0:6] = (c.w, c.h, c.qp, 3, 1, 4)
    v[9] = c.trskip
    v[10] = c.sao
    v[11:14] = (0, 0, 0) if c.dbk is None else (1, c.dbk[0], c.dbk[1])
    v[19] = 1                   # wpp
    v[20] = c.bd
    cfg[0]["lambda"] = c.lam
    cfg[0]["lambda_sqrt"] = np.sqrt(c.lam)
    return cfg


def _leaders(c, rot):
    return np.array([32 * ((i + rot) % 4) for i in range(c.nctu)], np.int32)


def _P(a):
    return C.c_void_p(a.ctypes.data)


def run_probe(lib_path, c, ctx_init, fill=0, rot=0, raster=0):
    lib = C.CDLL(lib_path)
    n = c.src.size
    cfg = _cfg(c)
    cu = np.ascontiguousarray(c.cu)
    dbk, out = np.zeros(n, c.pix), np.zeros(n, c.pix)
    sao = np.zeros((c.nctu, 2), SAO)
    cs, ce = np.zeros((c.nctu, CTX), np.uint8), np.zeros((c.nctu, CTX), np.uint8)
    info = np.zeros(4, np.int32)
    ctx = np.ascontiguousarray(ctx_init, np.uint8)
    lead = _leaders(c, rot)
    rc = lib.kvz_ctu_frame_probe_run(c.bd, _P(cfg), _P(ctx), _P(c.src), _P(cu), _P(c.rec), _P(c.coeff), _P(lead), fill, raster,
                                     _P(dbk), _P(out), _P(sao), _P(cs), _P(ce), _P(info))
    assert rc == 0, f"kvz_ctu_frame_probe_run failed: {c.name()}"
    return dict(dbk=dbk, out=out, sao=sao, ctx_start=cs, ctx_end=ce, widest=int(info[0]))


def run_reference(c):
    so = _ref_frame_lib(c.bd)
    assert so, f"oracle/_ref/libkvzref_frame for {c.bd} bits missing: make -C oracle ref builds it"
    lib = C.CDLL(so)
    n = c.src.size
    cu = np.ascontiguousarray(c.cu)
    dbk, out = np.zeros(n, c.pix), np.zeros(n, c.pix)
    sao = np.zeros((c.nctu, 2), SAO)
    cs, ce = np.zeros((c.nctu, CTX), np.uint8), np.zeros((c.nctu, CTX), np.uint8)
    lam = np.zeros((c.nctu, 2), np.float64)
    qp = np.zeros(c.nctu, np.int32)
    visits = np.zeros((c.nctu, 2), np.int32)
    beta, tc = (0, 0) if c.dbk is None else c.dbk
    lib.kvzref_frame_run.argtypes = [C.c_int] * 8 + [C.c_double] + [C.c_void_p] * 12
    rc = lib.kvzref_frame_run(c.w, c.h, c.qp, c.sao, int(c.dbk is not None), beta, tc, c.trskip, c.lam, _P(c.src), _P(c.rec), _P(cu),
                              _P(c.coeff), _P(dbk), _P(out), _P(sao), _P(cs), _P(ce), _P(lam), _P(qp), _P(visits))
    assert rc == 0, f"kvzref_frame_run failed: {c.name()}"
    assert (visits == 1).all(), f"{c.name()}: every CTU searched and coded once: {visits.tolist()}"
    assert (qp == c.qp).all() and (lam[:, 0] == c.lam).all(), f"{c.name()}: the reference ran at QP {set(qp.tolist())}, lambda {set(lam[:, 0].tolist())}"
    return dict(dbk=dbk, out=out, sao=sao, ctx_start=cs, ctx_end=ce)


# ------------------------------------------------------------------------------------------------ comparing
# Fields of sao_info_t the reference leaves unwritten, so they hold whatever its stack held (sao.c sao_search_best_mode and
# the edge / band searches it calls):
#   * luma, every type: offsets[6..9] (a luma record has one set of offsets, [0..4]; edge writes [5] as 0, band keeps its 0);
#   * band, luma: offsets[0] and band_position[1]; band, chroma: offsets[0] and offsets[5] (copied from an unset entry of
#     the band search's temporary offsets; the band position of the unused second buffer is never written);
#   * type none: the record is the losing edge or band record with its type cleared, so only what both write is compared.
# Every other field -- type, eo_class, ddistortion, both merge flags, the band positions in use, the offsets in use -- is
# compared exactly.
def sao_fields(rec, chroma):
    t = int(rec["type"])
    o = rec["offsets"]
    f = dict(type=t, eo_class=int(rec["eo_class"]), ddistortion=int(rec["ddistortion"]), merge_left=int(rec["merge_left_flag"]),
             merge_up=int(rec["merge_up_flag"]), band_position0=int(rec["band_position"][0]))
    used = [1, 2, 3, 4] + ([6, 7, 8, 9] if chroma else [5])
    if t == 2:
        used += [0, 5]
    if chroma or t == 2:
        f["band_position1"] = int(rec["band_position"][1])
    for i in sorted(set(used)):
        f[f"offsets[{i}]"] = int(o[i])
    return f


# cu_qp_delta_abs[2..3] (model bytes 26 and 27): kvz_init_contexts initialises two of the four, so the other two hold what
# the reference's encoder state held; no syntax of this scope codes them.  Every other model byte is compared.
MODELS_UNSET = (26, 27)


def compare(c, got, want, with_sao=True, models_unset=()):
    """-> list of mismatch descriptions: the first differing sample of each picture, every differing CTU's models and SAO
    records"""
    bad = []
    keep = np.setdiff1d(np.arange(CTX), models_unset)
    for key in ("dbk", "out"):
        if not np.array_equal(got[key], want[key]):
            for pi, (g, w) in enumerate(zip(c.planes(got[key]), c.planes(want[key]))):
                diff = np.argwhere(g != w)
                if diff.size:
                    y, x = diff[0]
                    sh = 0 if pi == 0 else 1
                    bad.append(f"{'deblocked' if key == 'dbk' else 'final'} picture, plane {'YUV'[pi]}: CTU ({(x << sh) // 64},{(y << sh) // 64}) "
                               f"sample ({x},{y}): want {int(w[y, x])}, got {int(g[y, x])} ({len(diff)} samples differ)")
                    break
    for key, what in (("ctx_start", "models at the CTU's start"), ("ctx_end", "models after the CTU's syntax")):
        g, w = got[key][:, keep], want[key][:, keep]
        for i in np.flatnonzero((g != w).any(axis=1))[:4]:
            j = int(keep[np.flatnonzero(g[i] != w[i])[0]])
            bad.append(f"{what}, CTU ({i % c.wl},{i // c.wl}): model {j}: want {want[key][i, j]}, got {got[key][i, j]}")
    if with_sao and c.sao:
        for i in range(c.nctu):
            for k in (0, 1):
                fw, fg = sao_fields(want["sao"][i, k], k), sao_fields(got["sao"][i, k], k)
                if fw != fg:
                    d = {n: (fw.get(n), fg.get(n)) for n in sorted(set(fw) | set(fg)) if fw.get(n) != fg.get(n)}
                    bad.append(f"SAO {'chroma' if k else 'luma'} record, CTU ({i % c.wl},{i // c.wl}): (want, got) {d}")
    return bad


def _assert_same(c, got, want, against, models_unset=()):
    bad = compare(c, got, want, models_unset=models_unset)
    assert not bad, f"{c.name()}: differs from {against}:\n" + "\n".join(bad[:12])


# ------------------------------------------------------------------------------------------------ coverage
def _dbk_params(c):
    beta_off, tc_off = c.dbk
    s = 1 << (c.bd - 8)
    bi = min(max(c.qp + 2 * beta_off, 0), 51)
    beta = (0 if bi < 16 else (bi - 10 if bi < 29 else 2 * bi - 38)) * s
    tct = [0] * 18 + [1] * 9 + [2] * 4 + [3] * 4 + [4] * 3 + [5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24]
    tc = tct[min(max(c.qp + 2 + 2 * tc_off, 0), 53)] * s
    return beta, tc


def luma_decisions(c):
    """The decisions of the vertical luma edges, read off the pre-deblock picture (the first pass reads nothing the pass
    itself has changed) -> set of 'strong', 'weak', 'weak-no-side' (neither p1 nor q1 filtered), 'none'"""
    if c.dbk is None:
        return set()
    beta, tc = _dbk_params(c)
    y_pl = c.planes(c.rec)[0].astype(np.int64)
    out = set()
    side = (beta + (beta >> 1)) >> 3
    for x in range(8, c.w, 8):
        for y in range(0, c.h, 4):
            r = c.cu[y >> 2, x >> 2]
            if x % (64 >> int(r["tr_depth"])) and x % (64 >> int(r["depth"])):
                continue
            b = y_pl[y:y + 4, x - 4:x + 4]
            d2 = lambda l, a: abs(int(b[l, a]) - 2 * int(b[l, a + 1]) + int(b[l, a + 2]))
            dp0, dq0, dp3, dq3 = d2(0, 1), d2(0, 4), d2(3, 1), d2(3, 4)
            dp, dq = dp0 + dp3, dq0 + dq3
            if dp + dq >= beta:
                out.add("none")
                continue
            strong = all(2 * (dpl + dql) < (beta >> 2) and abs(int(b[l, 3]) - int(b[l, 4])) < ((5 * tc + 1) >> 1) and
                         abs(int(b[l, 0]) - int(b[l, 3])) + abs(int(b[l, 4]) - int(b[l, 7])) < (beta >> 3)
                         for l, dpl, dql in ((0, dp0, dq0), (3, dp3, dq3)))
            if strong:
                out.add("strong")
                continue
            deltas = [abs((9 * (int(b[l, 4]) - int(b[l, 3])) - 3 * (int(b[l, 5]) - int(b[l, 2])) + 8) >> 4) for l in range(4)]
            if any(dl < 10 * tc for dl in deltas) and tc > 0:
                out.add("weak" if (dp < side or dq < side) else "weak-no-side")
            else:
                out.add("none")
    return out


def coverage(cases, wants):
    cov = dict(sao_type=set(), eo_class=set(), merge=set(), cmax=0, band_last=0, band0=0, dbk=set(), chroma_edge=0,
               border_split=0, nxn=0, cu64=0, tr_skip=0, qps=set(), dbk_switch=set(), sao_switch=set(), sizes=set(), widest=0)
    for c, w in zip(cases, wants):
        cov["qps"].add(c.qp)
        cov["dbk_switch"].add(c.dbk)
        cov["sao_switch"].add(c.sao)
        cov["sizes"].add((c.w, c.h))
        for k in ("border_split", "nxn", "cu64", "tr_skip"):
            cov[k] += c.stats[k]
        if c.sao:
            for i in range(c.nctu):
                sl = w["sao"][i, 0]
                if sl["merge_left_flag"]:
                    cov["merge"].add("left")
                    continue
                if sl["merge_up_flag"]:
                    cov["merge"].add("up")
                    continue
                for k in (0, 1):
                    s = w["sao"][i, k]
                    t = int(s["type"])
                    cov["sao_type"].add(t)
                    if t == 2:
                        cov["eo_class"].add(int(s["eo_class"]))
                    if t == 1:
                        bp = [int(s["band_position"][j]) for j in range(1 + k)]
                        cov["band_last"] += 27 in bp and bool((c.planes(w["dbk"])[k] >> (c.bd - 5) == 31).any())
                        cov["band0"] += 0 in bp
                    if t:
                        offs = s["offsets"][[1, 2, 3, 4] + ([6, 7, 8, 9] if k else [])]
                        cov["cmax"] += int((np.abs(offs) == c.cmax).any())
        cov["dbk"] |= luma_decisions(c)
        if c.dbk is not None:
            pre, post = c.planes(c.rec), c.planes(w["dbk"])
            cov["chroma_edge"] += int(not np.array_equal(pre[1], post[1]) or not np.array_equal(pre[2], post[2]))
    return cov


def _check_coverage(cases, wants):
    cov = coverage(cases, wants)
    assert cov["qps"] == set(QPS) and cov["dbk_switch"] == set(DEBLOCK) and cov["sao_switch"] == set(SAO_TYPES), cov
    assert set(SIZES) | {WIDE} <= cov["sizes"], cov
    assert cov["sao_type"] == {0, 1, 2} and cov["eo_class"] == {0, 1, 2, 3} and cov["merge"] == {"left", "up"}, cov
    # the band search tries the starts 0..27 (sao.c calc_sao_band_offsets: band < 28), so the last start is 27, here
    # chosen on content whose samples reach band 31: a start of 28 would cover them
    assert cov["cmax"] and cov["band_last"] and cov["band0"], cov
    assert {"strong", "weak", "weak-no-side", "none"} <= cov["dbk"] and cov["chroma_edge"], cov
    assert cov["border_split"] and cov["nxn"] and cov["cu64"] and cov["tr_skip"], cov
    return cov


# ------------------------------------------------------------------------------------------------ CPU (host build)
_CASES = {}


def _cases(bd):
    if bd not in _CASES:
        _CASES[bd] = make_cases(bd)
    return _CASES[bd]


@pytest.mark.parametrize("bitdepth", [8, 10])
def test_hostprobe_frame_stage_matches_reference(ref, ref10, bitdepth):
    """Host build == the reference's CTU job, CTU by CTU; and unchanged by the fill byte, the leader warps and raster
    instead of wavefront order."""
    r = ref if bitdepth == 8 else ref10
    host = _probe_host()
    cases = _cases(bitdepth)
    wants = []
    for c in cases:
        ctx = r.init_contexts(c.qp, 2)
        want = run_reference(c)
        wants.append(want)
        got = run_probe(host, c, ctx, FILLS[0], 0)
        _assert_same(c, got, want, "the reference", MODELS_UNSET)
        for fill, rot, raster in ((FILLS[1], 1, 0), (FILLS[1], 2, 1)):
            _assert_same(c, run_probe(host, c, ctx, fill, rot, raster), want, f"the reference (fill {fill:#x}, leaders +{rot}, "
                                                                             f"{'raster' if raster else 'diagonal'} order)", MODELS_UNSET)
        assert got["widest"] == max(sum(1 for y in range(c.hl) if 0 <= d - 2 * y < c.wl) for d in range(c.wl + 2 * c.hl))
    _check_coverage(cases, wants)


def test_frame_probe_rejects_bad_arguments():
    c = make_case(8, 72, 72, 30, 3, (0, 0), 0, "steps", 7)
    lib = C.CDLL(_probe_host())
    ctx = np.zeros(CTX, np.uint8)
    n = c.src.size
    bufs = [np.zeros(n, c.pix), np.zeros(n, c.pix), np.zeros((c.nctu, 2), SAO), np.zeros((c.nctu, CTX), np.uint8), np.zeros((c.nctu, CTX), np.uint8),
            np.zeros(4, np.int32)]
    cu = np.ascontiguousarray(c.cu)

    def call(cfg, bd=8, lead=None):
        lead = _leaders(c, 0) if lead is None else lead
        return lib.kvz_ctu_frame_probe_run(bd, _P(cfg), _P(ctx), _P(c.src), _P(cu), _P(c.rec), _P(c.coeff), _P(lead), 0, 0, *[_P(b) for b in bufs])

    assert call(_cfg(c)) == 0
    for idx, val in ((19, 0), (0, 68), (1, 70), (2, 52), (10, 4), (12, 7), (13, -7), (20, 10)):
        cfg = _cfg(c)
        cfg[0]["v"][idx] = val
        assert call(cfg) == -1, (idx, val)
    assert call(_cfg(c), bd=9) == -1
    assert call(_cfg(c), lead=np.full(c.nctu, 16, np.int32)) == -1


# ------------------------------------------------------------------------------------------------ GPU (the product's code)
@pytest.mark.gpu
@pytest.mark.parametrize("bitdepth", [8, 10])
def test_cuda_frame_stage_matches_host_and_reference(ref, ref10, bitdepth):
    """The device (128-thread CTAs, block-scope atomics into the arena, two item-strided deblocking passes, neighbours'
    records and samples through L2, rotating leader warps) against the one-thread host build on the same seeded cases,
    and against the reference's CTU job where its library is present."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(PROBE_CUDA), f"{PROBE_CUDA} missing: build() runs `make probe`"
    r = ref if bitdepth == 8 else ref10
    host = _probe_host()
    have_ref = _ref_frame_lib(bitdepth) is not None
    widest = 0
    wants = []
    for c in _cases(bitdepth):
        ctx = r.init_contexts(c.qp, 2)
        want = run_probe(host, c, ctx, FILLS[0], 0)
        if have_ref:
            _assert_same(c, want, run_reference(c), "the reference (host build)", MODELS_UNSET)
        wants.append(want)
        for fill, rot in ((FILLS[0], 0), (FILLS[1], 1)):
            got = run_probe(PROBE_CUDA, c, ctx, fill, rot)
            _assert_same(c, got, want, f"the host build (device, fill {fill:#x}, leaders +{rot})")
            widest = max(widest, got["widest"])
    assert widest >= 8, f"the widest diagonal launch had {widest} CTAs"
