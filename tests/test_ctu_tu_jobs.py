"""CTU search driver: the transform-unit jobs (ctu_leaf.h tu_eval / tu_core and coeff_cost_serial, dealt to teams by
ctu_search.h for_tu_tasks) against the compiled reference, unit by unit.

tests/cuda/ctu_tu_probe.cu runs batches of jobs through the driver's own code, the way search_cu_intra and
intra_recon_leaf issue them, and returns every job's prediction, levels, reconstruction, cbf, SSD, transform-skip choice,
coefficient-group mask and coefficient bits.  Two providers run the same seeded batches through the same test body:
  * CPU: tests/hostsim/libkvzctu_probe_host.so, the one-thread CTA of the host build, compared exactly with what the
    reference returns for the same unit (oracle/ref_tu.c kvzref_intra_tu: kvz_intra_predict,
    kvz_quantize_residual(_trskip), kvz_pixels_calc_ssd, kvz_get_coeff_cost);
  * GPU: tests/cuda/libkvzctu_probe.so (make probe), one 128-thread CTA per batch, so the jobs run on the CTA, warp and
    half-warp teams -- the code the host build never executes -- compared exactly with the host build on those batches,
    and so with the reference.
The second half of the module encodes small pictures with configurations that force each team path and the QP extremes
through the driver (bitstream identity and verify mode), on the host build and on the device.
"""
import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np
import pytest

from test_ctu_driver import ROOT, _cuda_lib, _hostsim, _identity
from test_ctu_driver_10bit import _hostsim as _hostsim10, _identity10
from test_rdoq import lambda_for

PROBE_SRC = os.path.join(ROOT, "tests", "cuda", "ctu_tu_probe.cu")
PROBE_HOST = os.path.join(ROOT, "tests", "hostsim", "libkvzctu_probe_host.so")
PROBE_CUDA = os.path.join(ROOT, "tests", "cuda", "libkvzctu_probe.so")
CFG = np.dtype([("v", "<i4", (21,)), ("lambda", "<f8"), ("lambda_sqrt", "<f8")], align=True)    # CtuConfig
CTX = 184
MAXN = 1024
REFLEN = 68
QPS = (0, 1, 4, 12, 22, 30, 37, 45, 51)
FILLS = (0x00, 0xA5)


def _probe_host():
    if not os.path.exists(PROBE_HOST):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unused-function", "-Wno-unknown-pragmas",
                               "-x", "c++", "-o", PROBE_HOST, PROBE_SRC])
    return PROBE_HOST


def _probe_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(PROBE_CUDA), f"{PROBE_CUDA} missing: build() runs `make probe`"
    return PROBE_CUDA


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Task:
    color: int
    log2n: int
    mode: int
    scan: int
    depth: int          # the CU record of the reference: depth, tr_depth, NxN
    tr_depth: int
    nxn: int
    alt: int            # -1: tu_eval; 0 / 1: the transform / transform-skip alternative of a 4x4 luma unit
    src: np.ndarray
    cls: str = ""


@dataclass
class Batch:
    kind: str
    qp: int
    lam: float
    rdoq: int
    rdoq_skip: int
    signhide: int
    trskip: int
    cabac0: np.ndarray
    sc: np.ndarray
    refs: dict                      # colour -> (top, left), unfiltered, 2n + 1 samples
    tasks: list = field(default_factory=list)
    leader_tid: int = 0


def _scan(rng, log2n):
    return int(rng.integers(0, 3)) if log2n <= 3 else 0


class Gen:
    """Seeded batches at one bit depth, shaped like the batches the driver issues."""

    def __init__(self, ref, bitdepth, seed):
        self.ref, self.bd, self.rng = ref, bitdepth, np.random.default_rng(seed)
        self.max = (1 << bitdepth) - 1
        self.pix = np.uint8 if bitdepth == 8 else np.uint16
        self.nb = 0
        self.modes = {}             # (colour, log2n) -> units so far: the modes of a unit size cycle through all 35

    def refs_of(self, log2n, theme):
        n2 = 2 * (1 << log2n) + 1
        r = self.rng
        if theme == "sat_hi":
            return np.zeros(n2, self.pix), np.zeros(n2, self.pix)
        if theme == "sat_lo":
            return np.full(n2, self.max, self.pix), np.full(n2, self.max, self.pix)
        if r.random() < 0.3:
            return r.integers(0, self.max + 1, n2).astype(self.pix), r.integers(0, self.max + 1, n2).astype(self.pix)
        base = int(r.integers(0, self.max + 1))
        walk = lambda: np.clip(base + np.cumsum(r.integers(-(self.max >> 4), (self.max >> 4) + 1, n2)), 0, self.max).astype(self.pix)
        return walk(), walk()

    def source(self, b, color, log2n, mode, theme):
        n, r, mx = 1 << log2n, self.rng, self.max
        if theme == "sat_hi":
            return "max", np.full(n * n, mx, self.pix)
        if theme == "sat_lo":
            return "zero", np.zeros(n * n, self.pix)
        cls = "noisy" if theme == "noisy" else ["smooth", "noisy", "checker", "pred", "pm1", "hstripe"][int(r.integers(0, 6))]
        yy, xx = np.mgrid[0:n, 0:n]
        if cls == "smooth":
            a = int(r.integers(0, mx + 1)) + (xx * int(r.integers(-3, 4)) + yy * int(r.integers(-3, 4))) * (mx >> 7) + r.integers(-2, 3, (n, n))
        elif cls == "noisy":
            a = r.integers(0, mx + 1, (n, n))
        elif cls == "checker":
            a = ((xx + yy) % 2) * mx
        elif cls == "hstripe":        # highest vertical frequency: levels in the coefficient groups of the lower rows
            a = (yy % 2) * mx // 2 + mx // 4 + r.integers(-1, 2, (n, n))
        else:
            top, left = b.refs[color]
            p = self.ref.intra_predict(log2n, mode, color, top, left, int(color == 0)).astype(np.int64).reshape(n, n)
            a = p if cls == "pred" else p + r.choice([-1, 1], (n, n))
        return cls, np.clip(a, 0, mx).astype(self.pix).ravel()

    def batch(self, kind, units, theme=None):
        """units: [(color, log2n, depth, tr_depth, nxn, alt, mode or None)]; one unit size per colour, as in the driver."""
        r = self.rng
        k = self.nb
        self.nb += 1
        qp = QPS[k % len(QPS)]
        sw = k % 16                 # with QPS[k % 9]: every (QP, switches) pair once in 144 batches
        if theme is None:
            theme = ("sat_hi", "sat_lo")[k % 2] if k % 7 == 3 else "mixed"
        if r.random() < 0.5:
            cabac0 = self.ref.init_contexts(qp, 2)
            sc = cabac0.copy()
            idx = r.choice(CTX, 40, replace=False)           # the search models have moved on from the coder's
            sc[idx] = r.integers(0, 126, 40)
        else:
            cabac0, sc = r.integers(0, 126, CTX).astype(np.uint8), r.integers(0, 126, CTX).astype(np.uint8)
        b = Batch(kind, qp, lambda_for(qp) * float(r.uniform(0.5, 2.0)), sw & 1, (sw >> 1) & 1, (sw >> 2) & 1, (sw >> 3) & 1,
                  cabac0, sc, {}, leader_tid=32 * (k % 4))
        for (color, log2n, *_rest) in units:
            if color not in b.refs:
                b.refs[color] = self.refs_of(log2n, theme)
        for (color, log2n, depth, tr_depth, nxn, alt, mode) in units:
            i = self.modes.get((color, log2n), 0)
            self.modes[(color, log2n)] = i + 1
            mode = (i * 13 + 7 * (color + log2n)) % 35 if mode is None else mode
            cls, src = self.source(b, color, log2n, mode, theme)
            b.tasks.append(Task(color, log2n, mode, _scan(r, log2n), depth, tr_depth, nxn, alt, src, cls))
        return b


def _rdo_units(depth, k, trskip, chroma=True, alts=True):
    """search_cu_intra's RDO batch: the luma units of k candidates (both transform-skip alternatives at depth 4), then
    (U, V) of each candidate.  The temporary CU has depth = tr_depth = depth, NxN at depth 4."""
    l2y = 6 - depth
    l2c = 5 - depth if depth < 4 else 2
    nxn = int(depth == 4)
    split = depth == 4 and trskip and alts
    u = []
    for _ in range(k):
        u += [(0, l2y, depth, depth, nxn, 0, None), (0, l2y, depth, depth, nxn, 1, None)] if split else [(0, l2y, depth, depth, nxn, -1, None)]
    if chroma:
        for _ in range(k):
            u += [(1, l2c, depth, depth, nxn, -1, None), (2, l2c, depth, depth, nxn, -1, None)]
    return u


def _leaf_units(depth, chroma=True):
    """intra_recon_leaf's [Y, U, V]: the CU record of the search (depth 4: an NxN CU of depth 3, tr_depth 4)."""
    cu_depth, nxn = (3, 1) if depth == 4 else (depth, 0)
    l2c = 5 - depth if depth < 4 else 2
    u = [(0, 6 - depth, cu_depth, depth, nxn, -1, None)]
    if chroma:
        u += [(1, l2c, cu_depth, depth, nxn, -1, None), (2, l2c, cu_depth, depth, nxn, -1, None)]
    return u


def make_batches(ref, bitdepth, seed=11, rounds=3):
    g = Gen(ref, bitdepth, seed)
    out = []
    # 1. every class on its own
    for _ in range(rounds * 2):
        for color, log2n in ((0, 2), (0, 3), (0, 4), (0, 5), (1, 2), (2, 3), (1, 4)):
            depth = 6 - log2n if color == 0 else (5 - log2n if log2n > 2 else 4)
            alts = (-1, 0, 1) if (color, log2n) == (0, 2) else (-1,)
            for alt in alts:
                out.append(g.batch("single", [(color, log2n, depth, depth, int(depth == 4), alt, None)]))
    for _ in range(rounds):
        for depth in (1, 2, 3, 4):
            for k in (1, 2, 3, 5):
                for ts in (0, 1):
                    b = g.batch(f"rdo{depth}", _rdo_units(depth, k, ts))
                    b.trskip = ts if depth == 4 else b.trskip
                    out.append(b)
            # the CU's chroma is not reconstructed at odd 4x4 / 8x8 positions: luma candidates only
            out.append(g.batch(f"rdo{depth}-luma", _rdo_units(depth, 3, 0, chroma=False)))
        # 6. depth 4, an odd number of luma units: the last one alone on a lower half-warp
        for k in (1, 3, 5):
            b = g.batch("rdo4-odd", _rdo_units(4, k, 0, chroma=False) + _rdo_units(4, 1, 0)[1:])
            b.trskip = 0
            out.append(b)
        # 7. 32 tasks: 4x4 only (half-warps), and 8x8 luma with 4x4 chroma (whole warps)
        b = g.batch("max32-4", _rdo_units(4, 8, 1))
        b.trskip = 1
        out.append(b)
        out.append(g.batch("max32-8", [(0, 3, 3, 3, 0, -1, None)] * 16 + [(1 + (i & 1), 2, 3, 3, 0, -1, None) for i in range(16)]))
        # 8. intra_recon_leaf
        for depth in (1, 2, 3, 4):
            out.append(g.batch(f"leaf{depth}", _leaf_units(depth)))
            out.append(g.batch(f"leaf{depth}-luma", _leaf_units(depth, chroma=False)))
    # intra_recon_leaf at depth 4 with transform skip: tu_eval's own decision between the two alternatives
    for i in range(2 * len(QPS)):
        b = g.batch("leaf4-ts", _leaf_units(4, chroma=i % 2 == 0))
        b.trskip = 1
        out.append(b)
    # RDOQ's sign hiding with a lambda that makes its rate-distortion factor (inv_quant^2 * 2^(2 (qp / 6)) / lambda / 16,
    # at every bit depth) a number of tens with a fraction above one half: its rounding then decides which level changes
    for i in range(48):
        depth = 1 + i % 3
        b = g.batch("rdoq-sh", _rdo_units(depth, 2, 0), theme="noisy")
        b.qp = QPS[i % len(QPS)]
        inv = (40, 45, 51, 57, 64, 72)[b.qp % 6]
        b.lam = inv * inv * 4.0 ** (b.qp // 6) / 16 / (20 + 4 * i + float(g.rng.uniform(0.55, 0.95)))
        b.rdoq, b.signhide = 1, 1
        out.append(b)
    # 32x32 units with levels in the groups of the second mask word (raster group 32 and above)
    for qp in (0, 1, 4):
        b = g.batch("cg-hi", [(0, 5, 1, 1, 0, -1, None)] * 2 + [(1, 4, 1, 1, 0, -1, None), (2, 4, 1, 1, 0, -1, None)], theme="mixed")
        b.qp, b.lam = qp, lambda_for(qp)
        for t in b.tasks:
            n = 1 << t.log2n
            yy = np.arange(n * n) // n
            t.src = np.clip((yy % 2) * g.max // 2 + g.max // 4, 0, g.max).astype(g.pix)
            t.cls = "hstripe"
        out.append(b)
    return out


# ------------------------------------------------------------------------------------------------ running
def run_probe(lib_path, bitdepth, batches, fill):
    lib = C.CDLL(lib_path)
    pix = np.uint8 if bitdepth == 8 else np.uint16
    nb = len(batches)
    tasks = [t for b in batches for t in b.tasks]
    nt = len(tasks)
    cfg = np.zeros(nb, CFG)
    bt = np.zeros((nb, 4), np.int32)
    cab = np.zeros((nb, 2, CTX), np.uint8)
    refs = np.zeros((nb, 3, 2, REFLEN), pix)
    td = np.zeros((nt, 8), np.int32)
    src = np.zeros((nt, MAXN), pix)
    first = 0
    for i, b in enumerate(batches):
        v = cfg[i]["v"]
        v[:6] = (64, 64, b.qp, 3, 1, 4)
        v[6:10] = (b.rdoq, b.rdoq_skip, b.signhide, b.trskip)
        v[20] = bitdepth
        cfg[i]["lambda"] = b.lam
        cfg[i]["lambda_sqrt"] = np.sqrt(b.lam)
        bt[i] = (first, len(b.tasks), b.leader_tid, 0)
        cab[i, 0], cab[i, 1] = b.cabac0, b.sc
        for col, (top, left) in b.refs.items():
            refs[i, col, 0, :top.size], refs[i, col, 1, :left.size] = top, left
        for j, t in enumerate(b.tasks):
            td[first + j, :6] = (t.color, t.log2n, t.mode, t.scan, t.tr_depth - t.depth + t.nxn, t.alt)
            src[first + j, :t.src.size] = t.src
        first += len(b.tasks)
    pred, rec = np.zeros((nt, MAXN), pix), np.zeros((nt, MAXN), pix)
    q = np.zeros((nt, MAXN), np.int16)
    oi = np.zeros((nt, 8), np.int32)
    mask = np.zeros(nt, np.uint64)
    bits = np.zeros(nt, np.float64)
    p = lambda a: C.c_void_p(a.ctypes.data)
    rc = lib.kvz_ctu_probe_run(bitdepth, nb, p(cfg), p(bt), p(cab), p(refs), nt, p(td), p(src), fill, p(pred), p(rec), p(q), p(oi), p(mask), p(bits))
    assert rc == 0, "kvz_ctu_probe_run failed"
    out = []
    for k, t in enumerate(tasks):
        nn = 1 << (2 * t.log2n)
        out.append(dict(pred=pred[k, :nn].copy(), rec=rec[k, :nn].copy(), coeff=q[k, :nn].copy(), has=int(oi[k, 0]), ssd=int(oi[k, 1]),
                        tr_skip=int(oi[k, 2]), team=int(oi[k, 3]), first=int(oi[k, 4]), cg_mask=int(mask[k]), bits=float(bits[k])))
    return out


def reference(ref, batches):
    out = []
    for b in batches:
        for t in b.tasks:
            top, left = b.refs[t.color]
            out.append(ref.intra_tu(b.qp, b.lam, b.rdoq, b.rdoq_skip, b.signhide, b.trskip, b.cabac0, b.sc, t.color, t.log2n, t.depth,
                                    t.tr_depth, t.nxn, t.mode, t.scan, t.alt, top, left, t.src))
    return out


def cg_mask_of(coeff, log2n):
    n = 1 << log2n
    nz = (coeff.reshape(n // 4, 4, n // 4, 4) != 0).any(axis=(1, 3)).ravel()
    return sum(1 << int(g) for g in np.flatnonzero(nz))


FIELDS = ("pred", "coeff", "rec", "has", "ssd", "tr_skip", "bits")


def compare(batches, got, want):
    """-> list of mismatch descriptions naming the batch, the task, its team and the field"""
    bad = []
    k = 0
    for bi, b in enumerate(batches):
        for ti, t in enumerate(b.tasks):
            g, w = got[k], want[k]
            k += 1
            fields = [f for f in FIELDS if not (np.array_equal(g[f], w[f]) if isinstance(w[f], np.ndarray) else g[f] == w[f])]
            if g["cg_mask"] != cg_mask_of(g["coeff"], t.log2n):
                fields.append("cg_mask")
            if fields:
                bad.append(f"batch {bi} ({b.kind}, qp {b.qp}, rdoq {b.rdoq}/{b.rdoq_skip} sh {b.signhide} ts {b.trskip}) task {ti} "
                           f"(colour {t.color} {1 << t.log2n}x{1 << t.log2n} mode {t.mode} scan {t.scan} alt {t.alt} {t.cls}) on team "
                           f"{g['team']}@{g['first']}: {', '.join(fields)}")
    return bad


def check_jobs(lib_path, bitdepth, batches, want, against):
    """Runs the batches with two fill bytes and every batch's tasks alone; all must equal `want`.  -> outputs"""
    runs = [run_probe(lib_path, bitdepth, batches, f) for f in FILLS]
    for f, got in zip(FILLS, runs):
        bad = compare(batches, got, want)
        assert not bad, f"{len(bad)} of {len(want)} units differ from {against} (fill {f:#x}):\n" + "\n".join(bad[:12])
    # every task alone in a batch of its own, with its batch's configuration and models
    alone = []
    for b in batches:
        if len(b.tasks) > 1:
            for t in b.tasks:
                alone.append(Batch(b.kind + "-alone", b.qp, b.lam, b.rdoq, b.rdoq_skip, b.signhide, b.trskip, b.cabac0, b.sc,
                                   {t.color: b.refs[t.color]}, [t], b.leader_tid))
    got = run_probe(lib_path, bitdepth, alone, FILLS[1])
    bad = compare(alone, got, [w for b, ws in _split(batches, want) if len(b.tasks) > 1 for w in ws])
    assert not bad, f"{len(bad)} units differ when run alone:\n" + "\n".join(bad[:12])
    return runs[0]


def _split(batches, flat):
    k = 0
    for b in batches:
        yield b, flat[k:k + len(b.tasks)]
        k += len(b.tasks)


def coverage(batches, want):
    """what the cases reached, from the reference's outputs"""
    tasks = [t for b in batches for t in b.tasks]
    return dict(
        tasks=len(tasks),
        modes={(t.color, t.log2n): set() for t in tasks},
        has0=sum(w["has"] == 0 for w in want),
        ts1=sum(w["tr_skip"] == 1 for w in want),
        cg_hi=sum((cg_mask_of(w["coeff"], t.log2n) >> 32) != 0 for t, w in zip(tasks, want)),
        qps={b.qp for b in batches},
        switches={(b.rdoq, b.rdoq_skip, b.signhide, b.trskip) for b in batches},
        scans={(t.log2n, t.scan) for t in tasks if t.log2n <= 3},
    )


def _check_coverage(batches, want):
    c = coverage(batches, want)
    assert c["has0"] > 0 and c["ts1"] > 0 and c["cg_hi"] > 0, c
    assert c["qps"] == set(QPS) and len(c["switches"]) == 16, c
    assert {(l, s) for l in (2, 3) for s in range(3)} <= c["scans"], c
    for t in (t for b in batches for t in b.tasks):
        c["modes"][(t.color, t.log2n)].add(t.mode)
    thin = {k: len(v) for k, v in c["modes"].items() if len(v) < 35}
    assert not thin, f"not every mode was used: {thin}"
    return c["tasks"]


# ------------------------------------------------------------------------------------------------ CPU (host build)
@pytest.mark.parametrize("bitdepth", [8, 10])
def test_hostprobe_tu_jobs_match_reference(ref, ref10, bitdepth):
    r = ref if bitdepth == 8 else ref10
    batches = make_batches(r, bitdepth)
    want = reference(r, batches)
    got = check_jobs(_probe_host(), bitdepth, batches, want, "the reference")
    _check_coverage(batches, want)
    assert {g["team"] for g in got} == {1}


# ------------------------------------------------------------------------------------------------ GPU (the product's code)
@pytest.mark.gpu
@pytest.mark.parametrize("bitdepth", [8, 10])
def test_cuda_tu_jobs_match_reference(ref, ref10, bitdepth):
    """The device's teams against the one-thread host build of the same jobs, on the same seeded batches: the host build
    equals the reference unit by unit on exactly these batches (test_hostprobe_tu_jobs_match_reference), so the device
    is held to the reference without needing the reference's transform-unit entry point where the device runs."""
    r = ref if bitdepth == 8 else ref10
    cuda = _probe_cuda()
    batches = make_batches(r, bitdepth)
    want = run_probe(_probe_host(), bitdepth, batches, FILLS[0])
    got = check_jobs(cuda, bitdepth, batches, want, "the host build")
    _check_coverage(batches, want)
    # the team shapes the jobs ran on: the whole CTA, whole warps, half-warps, and the upper half of a warp
    teams = {(b.kind, g["team"]) for b, gs in _split(batches, got) for g in gs}
    shapes = {s for _, s in teams}
    assert {128, 32, 16} <= shapes, f"team shapes reached: {sorted(shapes)}"
    assert any(g["team"] == 16 and g["first"] % 32 == 16 for g in got), "no unit ran on the upper half of a warp"
    kinds = {k: {s for kk, s in teams if kk == k} for k, _ in teams}
    # 16x16 units run on warps when four of their slots fit the arena: at 8 bits, not at 10
    assert kinds["rdo4"] == {16} and kinds["rdo3"] == {32}, kinds
    assert kinds["rdo2"] == ({32} if bitdepth == 8 else {128}) and kinds["rdo1"] == ({128, 32} if bitdepth == 8 else {128}), kinds


# ------------------------------------------------------------------------------------------------ whole pictures
# Configurations that force each team path and the QP extremes through the driver.  None of them uses ultrafast, superfast
# or veryfast: their --fast-residual-cost 28 sends every picture below QP 28 to the reference instead of the driver.
# (bit depth, w, h, preset, qp, extra switches, content: None = synthetic, "noisy", or an extreme picture of synth_yuv)
GRID = [
    (8, 136, 72, "veryslow", 22, "--pu-depth-intra 4-4 --rd 3 --transform-skip", "noisy"),    # half-warp pairs, both alternatives
    (8, 136, 72, "medium", 27, "--pu-depth-intra 4-4 --rd 2 --no-transform-skip", None),      # unpaired halves
    (8, 136, 72, "medium", 30, "--pu-depth-intra 4-4 --rdoq-skip --signhide", "noisy"),       # quant_block's sign hiding on halves
    (8, 264, 200, "veryslow", 22, "--pu-depth-intra 3-3 --rd 3", None),                       # 8x8 luma + 4x4 chroma on warps
    (8, 136, 72, "medium", 22, "--pu-depth-intra 2-2 --no-rdoq --signhide", "noisy"),         # 16x16 on warps
    (8, 264, 200, "veryslow", 27, "--pu-depth-intra 1-1 --rd 3", None),                       # 32x32 on the CTA, 16x16 on warps
    (8, 136, 72, "medium", 22, "--pu-depth-intra 1-4 --rd 0", "noisy"),
    (8, 136, 72, "medium", 27, "--pu-depth-intra 1-4 --rd 1", "noisy"),
    (8, 136, 72, "veryslow", 0, "", "noisy"),
    (8, 136, 72, "medium", 1, "", None),
    (8, 264, 200, "veryslow", 51, "", None),
    (8, 136, 72, "veryslow", 4, "", "black"),
    (8, 136, 72, "veryslow", 12, "", "white"),
    (8, 136, 72, "veryslow", 22, "", "checker1"),
    (8, 136, 72, "medium", 1, "", "fullnoise"),
    (10, 264, 200, "veryslow", 27, "--pu-depth-intra 1-1 --rd 3", None),     # 16x16 units fall back to the CTA at 10 bits
    (10, 136, 72, "veryslow", 22, "--pu-depth-intra 2-2", "noisy"),
    (10, 136, 72, "veryslow", 22, "--pu-depth-intra 4-4 --rd 3 --transform-skip", "noisy"),
    (10, 136, 72, "veryslow", 0, "", "noisy"),
    (10, 136, 72, "medium", 51, "", None),
    (10, 136, 72, "veryslow", 4, "", "black"),
    (10, 136, 72, "veryslow", 12, "", "white"),
    (10, 136, 72, "veryslow", 22, "", "checker1"),
    (10, 136, 72, "medium", 1, "", "fullnoise"),
]
GRID_PARAMS = [pytest.param(*c, id=f"{c[0]}b-{c[1]}x{c[2]}-{c[3]}-q{c[4]}{c[5].replace(' ', '')}-{c[6] or 'synth'}") for c in GRID]


def _grid_case(tmp_path, provider, bitdepth, w, h, preset, qp, extra, content):
    """bitstream identity and verify mode; both helpers assert "CTU search driver active" """
    clip = None
    if content not in (None, "noisy"):
        from synth_yuv import extreme_pictures
        clip = str(tmp_path / f"{content}.yuv")
        with open(clip, "wb") as f:
            f.write(extreme_pictures(w, h, bitdepth)[content])
    if bitdepth == 8:
        _identity(tmp_path, provider, w, h, 1, preset, qp, content == "noisy", tuple(extra.split()), clip=clip)
    else:
        _identity10(tmp_path, provider, w, h, 1, preset, qp, content == "noisy", 10, tuple(extra.split()), clip=clip)


@pytest.mark.parametrize("bitdepth,w,h,preset,qp,extra,content", GRID_PARAMS)
def test_hostbuild_team_paths_bitstream_identical(tmp_path, bitdepth, w, h, preset, qp, extra, content):
    _grid_case(tmp_path, _hostsim() if bitdepth == 8 else _hostsim10(), bitdepth, w, h, preset, qp, extra, content)


@pytest.mark.gpu
@pytest.mark.parametrize("bitdepth,w,h,preset,qp,extra,content", GRID_PARAMS)
def test_cuda_team_paths_bitstream_identical(tmp_path, bitdepth, w, h, preset, qp, extra, content):
    _grid_case(tmp_path, _cuda_lib(), bitdepth, w, h, preset, qp, extra, content)
