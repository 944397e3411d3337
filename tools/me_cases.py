"""Inputs of the integer-motion-search parity tests (tests/test_me_search.py, tools/make_golden_me.py): record layouts of
include/kvz_cuda.h (kvz_cuda_me_*), deterministic pictures / PU lists, and the ctypes plumbing shared by the three
implementations (reference shim, host build of the device code, the CUDA library)."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from kvazaar_b200.api import ME_MERGE as MERGE, ME_PU as PU, ME_RESULT as RESULT, MeParams as Params

assert MERGE.itemsize == 12 and PU.itemsize == 84 and RESULT.itemsize == 24 and C.sizeof(Params) == 56      # include/kvz_cuda.h

# PU shapes the reference searches: 2Nx2N / 2NxN / Nx2N of CUs 8..64 and the asymmetric (AMP) splits
SHAPES = [(8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 16), (32, 16), (16, 32), (64, 32), (32, 64), (8, 4), (4, 8),
          (16, 4), (16, 12), (4, 16), (12, 16), (32, 8), (32, 24), (8, 32), (24, 32), (64, 16), (64, 48), (16, 64), (48, 64)]

# name -> (width, height, bitdepth, params, seed, pus)
CASES = {
    "hexbs_et_sensitive":   dict(w=208, h=136, bd=8, algo=0, steps=-1, et=2, mvc=0, wpp=0, delay=0, qp=27, seed=1, n=400),
    "hexbs_et_on_wpp_sao":  dict(w=208, h=136, bd=8, algo=0, steps=-1, et=1, mvc=0, wpp=1, delay=10, qp=32, seed=2, n=400),
    "hexbs_et_off_margin":  dict(w=136, h=72, bd=8, algo=0, steps=-1, et=0, mvc=4, wpp=1, delay=8, qp=22, seed=3, n=400),
    "hexbs_steps2_frame":   dict(w=320, h=192, bd=8, algo=0, steps=2, et=0, mvc=1, wpp=0, delay=0, qp=37, seed=4, n=400),
    "hexbs_steps0":         dict(w=128, h=128, bd=8, algo=0, steps=0, et=2, mvc=0, wpp=1, delay=0, qp=27, seed=5, n=300),
    "dia_et_sensitive":     dict(w=208, h=136, bd=8, algo=7, steps=-1, et=2, mvc=0, wpp=0, delay=0, qp=27, seed=6, n=400),
    "dia_et_off_steps3":    dict(w=136, h=72, bd=8, algo=7, steps=3, et=0, mvc=4, wpp=1, delay=10, qp=30, seed=7, n=400),
    "hexbs_noisy":          dict(w=208, h=136, bd=8, algo=0, steps=-1, et=0, mvc=0, wpp=0, delay=0, qp=17, seed=8, n=400, noisy=True),
    "hexbs_10bit":          dict(w=208, h=136, bd=10, algo=0, steps=-1, et=1, mvc=0, wpp=1, delay=10, qp=27, seed=9, n=400),
    "dia_10bit_margin":     dict(w=136, h=72, bd=10, algo=7, steps=-1, et=2, mvc=4, wpp=0, delay=0, qp=32, seed=10, n=300),
    "tz_et_off":            dict(w=208, h=136, bd=8, algo=1, steps=-1, et=0, mvc=0, wpp=0, delay=0, qp=27, seed=11, n=300),
    "tz_wpp_sao_10bit":     dict(w=208, h=136, bd=10, algo=1, steps=-1, et=1, mvc=0, wpp=1, delay=10, qp=22, seed=12, n=300),
    "tz_noisy_margin":      dict(w=136, h=72, bd=8, algo=1, steps=-1, et=0, mvc=4, wpp=0, delay=0, qp=37, seed=13, n=200, noisy=True),
    "full8_et_off":         dict(w=136, h=72, bd=8, algo=3, steps=-1, et=0, mvc=0, wpp=1, delay=8, qp=27, seed=14, n=120),
    "full8_frame":          dict(w=128, h=128, bd=8, algo=3, steps=-1, et=2, mvc=1, wpp=0, delay=0, qp=32, seed=15, n=120),
    "full16_small":         dict(w=136, h=72, bd=8, algo=4, steps=-1, et=0, mvc=0, wpp=0, delay=0, qp=27, seed=16, n=40),
}


def lambda_sqrt(qp):
    return float(np.sqrt(0.57 * 2.0 ** ((qp - 12) / 3.0)))


def pictures(w, h, bd, seed, noisy=False):
    """current and reference luma planes: smooth structure + texture, the current picture = the reference moved by a
    spatially varying amount (so the searches travel several steps) + noise"""
    r = np.random.default_rng(1000 + seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 110 + 60 * np.sin(xx / 9.0 + seed) * np.cos(yy / 7.0) + 35 * np.sin((xx + 2 * yy) / 3.3)
    tex = r.integers(-25, 26, (h, w))
    ref = np.clip(base + tex, 0, 255)
    sx = (3 + 4 * np.sin(yy / 40.0)).astype(int)
    sy = (-2 + 3 * np.cos(xx / 50.0)).astype(int)
    cx = np.clip(xx + sx, 0, w - 1)
    cy = np.clip(yy + sy, 0, h - 1)
    amp = 40 if noisy else 4
    cur = np.clip(ref[cy, cx] + r.integers(-amp, amp + 1, (h, w)), 0, 255)
    if bd == 10:
        ref = ref * 4 + r.integers(0, 4, (h, w))
        cur = cur * 4 + r.integers(0, 4, (h, w))
        return np.ascontiguousarray(cur.astype(np.uint16)), np.ascontiguousarray(ref.astype(np.uint16))
    return np.ascontiguousarray(cur.astype(np.uint8)), np.ascontiguousarray(ref.astype(np.uint8))


def pu_list(w, h, seed, n):
    r = np.random.default_rng(2000 + seed)
    pus = np.zeros(n, PU)
    for i in range(n):
        pw, ph = SHAPES[int(r.integers(0, len(SHAPES)))]
        while pw > w or ph > h:
            pw, ph = SHAPES[int(r.integers(0, len(SHAPES)))]
        # positions on the 4-sample grid; a good share touching the picture borders
        edge = r.integers(0, 6)
        x = int(r.integers(0, (w - pw) // 4 + 1)) * 4
        y = int(r.integers(0, (h - ph) // 4 + 1)) * 4
        if edge == 0:
            x = 0
        elif edge == 1:
            x = (w - pw) // 4 * 4
        elif edge == 2:
            y = 0
        elif edge == 3:
            y = (h - ph) // 4 * 4
        pus[i]["x"], pus[i]["y"], pus[i]["w"], pus[i]["h"] = x, y, pw, ph
        pus[i]["mv_cand"] = r.integers(-40, 41, (2, 2))
        if r.integers(0, 4) == 0:
            pus[i]["mv_cand"][1] = pus[i]["mv_cand"][0]
        kind = r.integers(0, 5)
        if kind == 0:
            pus[i]["start_mv"] = 0
        elif kind == 1:
            pus[i]["start_mv"] = r.integers(-600, 601, 2)          # far away, often outside the picture / not allowed
        else:
            pus[i]["start_mv"] = r.integers(-48, 49, 2)
        nm = int(r.integers(0, 6))
        pus[i]["num_merge"] = nm
        for m in range(nm):
            pus[i]["merge"][m]["dir"] = int(r.integers(1, 4))
            pus[i]["merge"][m]["mv"] = r.integers(-64, 65, (2, 2))
            if r.integers(0, 5) == 0:
                pus[i]["merge"][m]["mv"] = 0
            if r.integers(0, 6) == 0 and kind != 0:
                pus[i]["merge"][m]["mv"][:] = pus[i]["start_mv"]       # the start MV is one of the merge candidates
    return pus


def make_case(name):
    c = CASES[name]
    p = Params()
    p.width, p.height, p.bitdepth = c["w"], c["h"], c["bd"]
    p.ime_algorithm, p.me_max_steps, p.me_early_termination = c["algo"], c["steps"], c["et"]
    p.mv_constraint, p.wpp_owf, p.delay_px = c["mvc"], c["wpp"], c["delay"]
    p.max_ref_lcu_right, p.max_ref_lcu_down = 1, 1                  # encoder.c:193-194
    p.lambda_sqrt = lambda_sqrt(c["qp"])
    p.satd_final = c.get("satd_final", 0)
    cur, ref = pictures(c["w"], c["h"], c["bd"], c["seed"], c.get("noisy", False))
    return p, cur, ref, pu_list(c["w"], c["h"], c["seed"], c["n"])


def grid_case(w, h, bd, size=16, seed=77, qp=27):
    """every size x size PU of a picture (the shape of a frame-level call)"""
    p = Params()
    p.width, p.height, p.bitdepth = w, h, bd
    p.ime_algorithm, p.me_max_steps, p.me_early_termination = 0, -1, 1       # --preset slow: hexbs, early termination on
    p.mv_constraint, p.wpp_owf, p.delay_px = 0, 1, 10
    p.max_ref_lcu_right, p.max_ref_lcu_down = 1, 1
    p.lambda_sqrt = lambda_sqrt(qp)
    cur, ref = pictures(w, h, bd, seed)
    nx, ny = w // size, h // size
    pus = np.zeros(nx * ny, PU)
    r = np.random.default_rng(seed)
    for j in range(ny):
        for i in range(nx):
            u = pus[j * nx + i]
            u["x"], u["y"], u["w"], u["h"] = i * size, j * size, size, size
            u["mv_cand"] = r.integers(-24, 25, (2, 2))
            u["start_mv"] = r.integers(-32, 33, 2)
            u["num_merge"] = 2
            u["merge"][0]["dir"], u["merge"][1]["dir"] = 1, 2
            u["merge"][0]["mv"] = r.integers(-32, 33, (2, 2))
            u["merge"][1]["mv"] = r.integers(-32, 33, (2, 2))
    return p, cur, ref, pus


def run_host_api(lib, p, cur, ref, pus):
    """kvz_cuda_call_me_search of `lib` (host buffers): the CUDA library or the host build of the device code"""
    out = np.zeros(len(pus), RESULT)
    lib.kvz_cuda_call_me_search.argtypes = [C.POINTER(Params), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = lib.kvz_cuda_call_me_search(C.byref(p), cur.ctypes.data, cur.shape[1], ref.ctypes.data, ref.shape[1], pus.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out


def run_reference(ref_shim, p, cur, ref, pus):
    """the unmodified reference's own functions (oracle/ref_me.c)"""
    out = np.zeros(len(pus), RESULT)
    ctx = ref_shim.ctx(27, 0, 0, p.width, p.height)
    f = ref_shim.lib.kvzref_me_search
    f.argtypes = [C.c_void_p, C.POINTER(Params), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = f(ctx, C.byref(p), cur.ctypes.data, cur.shape[1], ref.ctypes.data, ref.shape[1], pus.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out


def same(a, b):
    """decisions and costs identical (the diagnostic point count is not part of the reference's result)"""
    return np.array_equal(a["mv"], b["mv"]) and np.array_equal(a["bits"], b["bits"]) and np.array_equal(a["cost"], b["cost"])


# ------------------------------------------------------------------------------------------------ AMVP / merge candidates
from kvazaar_b200.api import ME_CU as CU, ME_CAND_PU as CAND_PU, ME_CAND_OUT as CAND_OUT, MeFrame as Frame  # noqa: E402

assert CU.itemsize == 12 and CAND_PU.itemsize == 12 and CAND_OUT.itemsize == 80 and C.sizeof(Frame) == 260

CAND_CASES = {
    # name -> picture size, reference structure
    "p_one_ref":        dict(w=208, h=136, poc=5, slice_b=0, tmvp=1, max_merge=5, pocs=[4], l0=[0], l1=[], seed=1, n=500),
    "p_four_refs":      dict(w=264, h=200, poc=9, slice_b=0, tmvp=1, max_merge=5, pocs=[8, 7, 5, 1], l0=[0, 1, 2, 3], l1=[], seed=2, n=500),
    "b_gop":            dict(w=264, h=200, poc=4, slice_b=1, tmvp=1, max_merge=5, pocs=[0, 8, 2, 6], l0=[0, 2], l1=[1, 3], seed=3, n=500),
    "b_lowdelay":       dict(w=208, h=136, poc=7, slice_b=1, tmvp=1, max_merge=4, pocs=[6, 5, 3], l0=[0, 1, 2], l1=[0, 1, 2], seed=4, n=500),
    "p_no_tmvp_merge2": dict(w=136, h=72, poc=3, slice_b=0, tmvp=0, max_merge=2, pocs=[2, 1], l0=[0, 1], l1=[], seed=5, n=400),
    "b_poc1_future":    dict(w=136, h=136, poc=1, slice_b=1, tmvp=1, max_merge=5, pocs=[0, 2], l0=[0], l1=[1], seed=6, n=400),
    "b_far_pocs":       dict(w=320, h=192, poc=300, slice_b=1, tmvp=1, max_merge=5, pocs=[100, 299, 600, 301], l0=[1, 0], l1=[3, 2], seed=7, n=500),
}


def cu_image(w, h, r, list_sizes, inter_share=0.7):
    """CU records of a picture: tiled with blocks of 8..64 samples; each block not set / intra / inter with random motion"""
    wl, hl = (w + 63) // 64 * 64, (h + 63) // 64 * 64
    im = np.zeros((hl // 4, wl // 4), CU)

    def fill(x, y, size):
        if size > 8 and (size == 64 or r.integers(0, 3) != 0) and r.integers(0, 4) != 0:
            for k in range(4):
                fill(x + (k % 2) * size // 2, y + (k // 2) * size // 2, size // 2)
            return
        parts = [(x, y, size, size)]
        if r.integers(0, 4) == 0:            # two PUs side by side / on top of each other
            parts = [(x, y, size // 2, size), (x + size // 2, y, size // 2, size)] if r.integers(0, 2) else \
                    [(x, y, size, size // 2), (x, y + size // 2, size, size // 2)]
        for (px, py, pw, ph) in parts:
            rec = np.zeros((), CU)
            t = r.random()
            if t < inter_share:
                rec["type"] = 2
                dirs = [1] if list_sizes[1] == 0 else [1, 2, 3]
                d = int(dirs[int(r.integers(0, len(dirs)))])
                rec["mv_dir"] = d
                for l in range(2):
                    if d & (1 << l):
                        rec["mv"][l] = r.integers(-80, 81, 2) if r.integers(0, 5) else 0
                        rec["mv_ref"][l] = int(r.integers(0, list_sizes[l]))
                    else:                   # what the unused list holds must not matter: put junk there
                        rec["mv"][l] = r.integers(-9, 10, 2)
                        rec["mv_ref"][l] = int(r.integers(0, 4))
            elif t < inter_share + 0.2:
                rec["type"] = 1
            im[py // 4:(py + ph) // 4, px // 4:(px + pw) // 4] = rec

    for y in range(0, hl, 64):
        for x in range(0, wl, 64):
            fill(x, y, 64)
    # some repeated motion so that duplicate pruning happens
    return im


def make_cand_case(name):
    c = CAND_CASES[name]
    r = np.random.default_rng(3000 + c["seed"])
    f = Frame()
    f.width, f.height, f.poc, f.slice_b, f.tmvp_enable, f.max_merge = c["w"], c["h"], c["poc"], c["slice_b"], c["tmvp"], c["max_merge"]
    f.used_size = len(c["pocs"])
    for i, p in enumerate(c["pocs"]):
        f.pocs[i] = p
    sizes = [len(c["l0"]), len(c["l1"])]
    f.ref_LX_size[0], f.ref_LX_size[1] = sizes
    for l, lst in enumerate((c["l0"], c["l1"])):
        for i, v in enumerate(lst):
            f.ref_LX[l][i] = v
    # the colocated picture (ref_LX[0][0]): the POCs it referred to, and its own reference lists
    col_poc = c["pocs"][c["l0"][0]]
    col_pic_ref_pocs = np.array([col_poc - 1 - int(r.integers(0, 6)) if i % 3 else col_poc + 1 + int(r.integers(0, 4)) for i in range(16)], np.int32)
    col_ref_LXs = r.integers(0, 16, (2, 16)).astype(np.uint8)
    for l in range(2):
        for i in range(16):
            f.col_ref_pocs[l][i] = int(col_pic_ref_pocs[col_ref_LXs[l][i]])
    cus = cu_image(c["w"], c["h"], r, [sizes[0], sizes[1]])
    col = cu_image(c["w"], c["h"], r, [4, 4], inter_share=0.8)
    # a few neighbours with identical motion (duplicate pruning in the merge list)
    flat = cus.reshape(-1)
    inter = np.nonzero(flat["type"] == 2)[0]
    for _ in range(len(inter) // 6):
        a, b = r.choice(inter, 2)
        flat[b] = flat[a]
    n = c["n"]
    pus = np.zeros(n, CAND_PU)
    # PUs as the encoder forms them: a CU of 8..64 samples on its own grid, one of the part modes the inter search tries
    # (2Nx2N, 2NxN, Nx2N, the four asymmetric splits for CUs >= 16), either PU of it
    for i in range(n):
        while True:
            size = int((8, 16, 32, 64)[int(r.integers(0, 4))])
            if size <= c["w"] and size <= c["h"]:
                break
        cx = int(r.integers(0, c["w"] // size)) * size
        cy = int(r.integers(0, c["h"] // size)) * size
        mode = int(r.integers(0, 7 if size >= 16 else 3))
        q = size // 4
        split = {0: None, 1: ("h", size // 2), 2: ("v", size // 2), 3: ("h", q), 4: ("h", size - q), 5: ("v", q), 6: ("v", size - q)}[mode]
        ipu = int(r.integers(0, 2)) if split else 0
        x, y, pw, ph = cx, cy, size, size
        if split:
            kind, at = split
            if kind == "h":
                y, ph = (cy, at) if ipu == 0 else (cy + at, size - at)
            else:
                x, pw = (cx, at) if ipu == 0 else (cx + at, size - at)
        pus[i]["x"], pus[i]["y"], pus[i]["w"], pus[i]["h"] = x, y, pw, ph
        pus[i]["mv_ref"] = [int(r.integers(0, max(1, sizes[0]))), int(r.integers(0, max(1, sizes[1])))]
        pus[i]["use_a1"], pus[i]["use_b1"] = int(ipu == 0 or pw >= ph), int(ipu == 0 or pw <= ph)       # search_inter.c:1628-1633
        if r.integers(0, 8) == 0:
            pus[i]["use_a1"], pus[i]["use_b1"] = int(r.integers(0, 2)), int(r.integers(0, 2))
    return f, col_pic_ref_pocs, col_ref_LXs, cus, col, pus


def run_cand_host_api(lib, f, cus, col, pus):
    out = np.zeros(len(pus), CAND_OUT)
    lib.kvz_cuda_call_me_candidates.argtypes = [C.POINTER(Frame), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = lib.kvz_cuda_call_me_candidates(C.byref(f), cus.ctypes.data, cus.shape[1], col.ctypes.data, col.shape[1], cus.shape[0], pus.ctypes.data,
                                         len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out


def run_cand_reference(ref_shim, f, col_pic_ref_pocs, col_ref_LXs, cus, col, pus):
    out = np.zeros(len(pus), CAND_OUT)
    ctx = ref_shim.ctx(27, 0, 0, f.width, f.height)
    fn = ref_shim.lib.kvzref_me_candidates
    fn.argtypes = [C.c_void_p, C.POINTER(Frame), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = fn(ctx, C.byref(f), col_pic_ref_pocs.ctypes.data, col_ref_LXs.ctypes.data, cus.ctypes.data, cus.shape[1], col.ctypes.data, col.shape[1],
            cus.shape[0], pus.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out


# ------------------------------------------------------------------------------------------------ fractional search
FRAC_CASES = {
    # name -> base search case (pictures, PUs, limits) + cfg.fme_level
    "frac4_hexbs":        dict(base="hexbs_et_sensitive", level=4),
    "frac4_wpp_sao":      dict(base="hexbs_et_on_wpp_sao", level=4),
    "frac4_margin":       dict(base="hexbs_et_off_margin", level=4),
    "frac2_frame":        dict(base="hexbs_steps2_frame", level=2),
    "frac1":              dict(base="dia_et_sensitive", level=1),
    "frac3_noisy":        dict(base="hexbs_noisy", level=3),
    "frac4_10bit":        dict(base="hexbs_10bit", level=4),
    "frac2_10bit_margin": dict(base="dia_10bit_margin", level=2),
}


def make_frac_case(name, int_results=None):
    """the PUs of the base case; the fractional search starts from a full-pel MV (what the integer search returns): here
    a deterministic one near the content's motion, clipped so that the PU stays within reach of the picture"""
    c = FRAC_CASES[name]
    p, cur, rf, pus = make_case(c["base"])
    r = np.random.default_rng(4000 + CASES[c["base"]]["seed"])
    pus = pus.copy()
    start = r.integers(-12, 13, (len(pus), 2)) * 4
    far = r.integers(0, 8, len(pus)) == 0
    start[far] = r.integers(-80, 81, (int(far.sum()), 2)) * 4            # some far outside the picture
    pus["start_mv"] = start
    return p, c["level"], cur, rf, pus


def run_frac_host_api(lib, p, level, cur, ref, pus):
    out = np.zeros(len(pus), RESULT)
    lib.kvz_cuda_call_me_frac_search.argtypes = [C.POINTER(Params), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = lib.kvz_cuda_call_me_frac_search(C.byref(p), level, cur.ctypes.data, cur.shape[1], ref.ctypes.data, ref.shape[1], pus.ctypes.data, len(pus),
                                          out.ctypes.data)
    assert rc == 0, rc
    return out


def run_frac_reference(ref_shim, p, level, cur, ref, pus):
    out = np.zeros(len(pus), RESULT)
    ctx = ref_shim.ctx(27, 0, 0, p.width, p.height)
    f = ref_shim.lib.kvzref_me_frac_search
    f.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = f(ctx, C.byref(p), level, cur.ctypes.data, cur.shape[1], ref.ctypes.data, ref.shape[1], pus.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out

# cfg.fme_level == 0 (--preset ultrafast): the integer winner's cost is recomputed as Hadamard cost (search_inter.c:1385-1397)
CASES["hexbs_satd_final"] = dict(w=208, h=136, bd=8, algo=0, steps=-1, et=2, mvc=0, wpp=1, delay=8, qp=32, seed=17, n=300, satd_final=1)
CASES["dia_satd_final_10bit"] = dict(w=136, h=72, bd=10, algo=7, steps=-1, et=1, mvc=0, wpp=0, delay=0, qp=27, seed=18, n=200, satd_final=1)

# the search cases of tests/test_me_search.py's -m gpu tests; the GPU tests of the cases added later live in
# tests/test_zz_me_frac.py, which sorts last
GPU_FIRST_RUN_DONE = ["dia_10bit_margin", "dia_et_off_steps3", "dia_et_sensitive", "hexbs_10bit", "hexbs_et_off_margin", "hexbs_et_on_wpp_sao",
                      "hexbs_et_sensitive", "hexbs_noisy", "hexbs_steps0", "hexbs_steps2_frame"]


class RefShim:
    """oracle/_ref/libkvzref_shim[_10b].so without the test suite's loader (tests/_oracle.py:Ref offers the same two members):
    the compiled, unmodified reference plus oracle/ref_me.c.  TEST / BASELINE INFRASTRUCTURE."""

    def __init__(self, bitdepth=8):
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        so = os.path.join(root, "oracle", "_ref", "libkvzref_shim.so" if bitdepth == 8 else "libkvzref_shim_10b.so")
        self.lib = C.CDLL(so)
        self.lib.kvzref_ctx_open.restype = C.c_void_p
        assert self.lib.kvzref_init() == 1
        self._ctx = {}

    def ctx(self, qp=22, signhide=0, rdoq=0, w=64, h=64):
        key = (qp, signhide, rdoq, w, h)
        if key not in self._ctx:
            c = self.lib.kvzref_ctx_open(w, h, qp, signhide, rdoq)
            assert c
            self._ctx[key] = C.c_void_p(c)
        return self._ctx[key]


# ------------------------------------------------------------------------------------------------ merge analysis
from kvazaar_b200.api import ME_MERGE_COST as MERGE_COST, MeRefs as Refs  # noqa: E402

assert MERGE_COST.itemsize == 96 and C.sizeof(Refs) == 256

MERGE_CASES = {
    "merge_p_one_ref":    dict(w=208, h=136, bd=8, pics=1, l0=[0], l1=[], bipred=0, mvc=0, wpp=0, delay=0, qp=27, ctx=(30, 11), seed=1, n=300),
    "merge_b_two_refs":   dict(w=208, h=136, bd=8, pics=2, l0=[0, 1], l1=[1, 0], bipred=1, mvc=0, wpp=1, delay=10, qp=32, ctx=(5, 70), seed=2, n=300),
    "merge_b_four_refs":  dict(w=264, h=200, bd=8, pics=4, l0=[0, 2, 1], l1=[3, 1], bipred=1, mvc=4, wpp=0, delay=0, qp=22, ctx=(62, 62), seed=3, n=300),
    "merge_b_nobipred":   dict(w=136, h=72, bd=8, pics=2, l0=[0], l1=[1], bipred=0, mvc=1, wpp=1, delay=8, qp=37, ctx=(100, 3), seed=4, n=250),
    "merge_b_10bit":      dict(w=208, h=136, bd=10, pics=3, l0=[0, 1], l1=[2, 0], bipred=1, mvc=0, wpp=1, delay=10, qp=27, ctx=(17, 40), seed=5, n=250),
}
PART_MODES = [0, 1, 2, 4, 5, 6, 7]          # part_mode_t of the generator's split kinds: 2Nx2N 2NxN Nx2N 2NxnU 2NxnD nLx2N nRx2N


def make_merge_case(name):
    c = MERGE_CASES[name]
    r = np.random.default_rng(6000 + c["seed"])
    w, h, bd = c["w"], c["h"], c["bd"]
    p = Params()
    p.width, p.height, p.bitdepth = w, h, bd
    p.mv_constraint, p.wpp_owf, p.delay_px = c["mvc"], c["wpp"], c["delay"]
    p.max_ref_lcu_right, p.max_ref_lcu_down = 1, 1
    p.lambda_sqrt = lambda_sqrt(c["qp"])
    cur, ref0 = pictures(w, h, bd, 50 + c["seed"])
    planes = [ref0] + [pictures(w, h, bd, 60 + 7 * k + c["seed"], noisy=(k == 2))[1] for k in range(1, c["pics"])]
    sizes = [len(c["l0"]), len(c["l1"])]
    n = c["n"]
    pus = np.zeros(n, PU)
    cu = np.zeros((n, 5), np.int32)
    for i in range(n):
        while True:
            size = int((8, 16, 32, 64)[int(r.integers(0, 4))])
            if size <= w and size <= h:
                break
        cx, cy = int(r.integers(0, w // size)) * size, int(r.integers(0, h // size)) * size
        mode = int(r.integers(0, 7 if size >= 16 else 3))
        q = size // 4
        split = {0: None, 1: ("h", size // 2), 2: ("v", size // 2), 3: ("h", q), 4: ("h", size - q), 5: ("v", q), 6: ("v", size - q)}[mode]
        ipu = int(r.integers(0, 2)) if split else 0
        x, y, pw, ph = cx, cy, size, size
        if split:
            kind, at = split
            if kind == "h":
                y, ph = (cy, at) if ipu == 0 else (cy + at, size - at)
            else:
                x, pw = (cx, at) if ipu == 0 else (cx + at, size - at)
        pus[i]["x"], pus[i]["y"], pus[i]["w"], pus[i]["h"] = x, y, pw, ph
        cu[i] = (cx, cy, size, PART_MODES[mode], ipu)
        nm = int(r.integers(1, 6))
        pus[i]["num_merge"] = nm
        for m in range(nm):
            dirs = [1] if sizes[1] == 0 else [1, 2, 3, 3]
            d = int(dirs[int(r.integers(0, len(dirs)))])
            mc = pus[i]["merge"][m]
            mc["dir"] = d
            for l in range(2):
                used = d & (1 << l)
                if used or r.integers(0, 3) == 0:          # the list a candidate does not use sometimes holds leftovers
                    rng = 600 if r.integers(0, 12) == 0 else 40
                    mc["mv"][l] = r.integers(-rng, rng + 1, 2)
                    if r.integers(0, 3) == 0:
                        mc["mv"][l] = (mc["mv"][l] >> 2) << 2  # integer MVs: the copy path
                    mc["ref"][l] = int(r.integers(0, max(1, sizes[l])))
            if m > 0 and r.integers(0, 5) == 0:
                pus[i]["merge"][m] = pus[i]["merge"][int(r.integers(0, m))]       # duplicates
    return p, c, cur, planes, pus, cu


def merge_refs_struct(c, plane_ptrs, width, bits):
    rf = Refs()
    for i in range(16):
        rf.plane[i] = plane_ptrs[i if i < len(plane_ptrs) else 0]
        rf.stride[i] = width
    for l, lst in enumerate((c["l0"], c["l1"])):
        for i, v in enumerate(lst):
            rf.ref_LX[l][i] = v
    rf.bipred = c["bipred"]
    rf.merge_flag_bits, rf.merge_idx_bits[0], rf.merge_idx_bits[1] = bits
    return rf


def run_merge_reference(ref_shim, p, c, cur, planes, pus, cu):
    out = np.zeros(len(pus), MERGE_COST)
    bits = (C.c_double * 3)()
    ctx = ref_shim.ctx(27, 0, 0, p.width, p.height)
    ptrs = (C.c_void_p * 16)(*[planes[i if i < len(planes) else 0].ctypes.data for i in range(16)])
    lx = np.zeros((2, 16), np.uint8)
    lx[0, :len(c["l0"])] = c["l0"]
    lx[1, :len(c["l1"])] = c["l1"]
    sizes = (C.c_int32 * 2)(len(c["l0"]), len(c["l1"]))
    f = ref_shim.lib.kvzref_me_merge_cost
    f.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    cu = np.ascontiguousarray(cu, np.int32)
    rc = f(ctx, C.byref(p), len(planes), ptrs, lx.ctypes.data, sizes, c["bipred"], c["ctx"][0], c["ctx"][1], bits, cur.ctypes.data, cur.shape[1],
           pus.ctypes.data, cu.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out, (bits[0], bits[1], bits[2])


def run_merge_host_api(lib, p, c, cur, planes, pus, bits):
    out = np.zeros(len(pus), MERGE_COST)
    rf = merge_refs_struct(c, [pl.ctypes.data for pl in planes], p.width, bits)
    lib.kvz_cuda_me_merge_cost_batch.argtypes = [C.POINTER(Params), C.POINTER(Refs), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    rc = lib.kvz_cuda_me_merge_cost_batch(C.byref(p), C.byref(rf), cur.ctypes.data, cur.shape[1], pus.ctypes.data, len(pus), out.ctypes.data, None)
    assert rc == 0, rc
    return out


# ------------------------------------------------------------------------------------------------ bi-prediction from two uni-predictions
from kvazaar_b200.api import ME_BIPRED_PU as BIPRED_PU, ME_BIPRED_RESULT as BIPRED_RESULT  # noqa: E402

assert BIPRED_PU.itemsize == 28 and BIPRED_RESULT.itemsize == 16


def make_bipred_case(name):
    """the pictures, reference lists and PU geometry of a B merge case; MVs / reference indices / AMVP candidates at random"""
    p, c, cur, planes, mpus, _ = make_merge_case(name)
    r = np.random.default_rng(7000 + c["seed"])
    n = len(mpus)
    pus = np.zeros(n, BIPRED_PU)
    for k in ("x", "y", "w", "h"):
        pus[k] = mpus[k]
    pus["mv"] = r.integers(-48, 49, (n, 2, 2))
    ints = r.integers(0, 3, (n, 2)) == 0
    pus["mv"][ints] = (pus["mv"][ints] >> 2) << 2                 # integer MVs: the copy path of one or both lists
    far = r.integers(0, 15, n) == 0
    pus["mv"][far] = r.integers(-500, 501, (int(far.sum()), 2, 2))
    pus["mv_ref"][:, 0] = r.integers(0, len(c["l0"]), n)
    pus["mv_ref"][:, 1] = r.integers(0, max(1, len(c["l1"])), n)
    pus["mv_cand"] = r.integers(-40, 41, (n, 2, 2))
    same = r.integers(0, 4, n) == 0
    pus["mv_cand"][same, 1] = pus["mv_cand"][same, 0]
    return p, c, cur, planes, pus


def run_bipred_reference(ref_shim, p, c, cur, planes, pus):
    out = np.zeros(len(pus), BIPRED_RESULT)
    ctx = ref_shim.ctx(27, 0, 0, p.width, p.height)
    ptrs = (C.c_void_p * 16)(*[planes[i if i < len(planes) else 0].ctypes.data for i in range(16)])
    lx = np.zeros((2, 16), np.uint8)
    lx[0, :len(c["l0"])] = c["l0"]
    lx[1, :len(c["l1"])] = c["l1"]
    f = ref_shim.lib.kvzref_me_bipred
    f.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    rc = f(ctx, C.byref(p), len(planes), ptrs, lx.ctypes.data, c["bipred"], cur.ctypes.data, cur.shape[1], pus.ctypes.data, len(pus), out.ctypes.data)
    assert rc == 0, rc
    return out


def run_bipred_host_api(lib, p, c, cur, planes, pus):
    out = np.zeros(len(pus), BIPRED_RESULT)
    rf = merge_refs_struct(c, [pl.ctypes.data for pl in planes], p.width, (0.0, 0.0, 0.0))
    lib.kvz_cuda_me_bipred_batch.argtypes = [C.POINTER(Params), C.POINTER(Refs), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    rc = lib.kvz_cuda_me_bipred_batch(C.byref(p), C.byref(rf), cur.ctypes.data, cur.shape[1], pus.ctypes.data, len(pus), out.ctypes.data, None)
    assert rc == 0, rc
    return out


BIPRED_CASES = ["merge_b_two_refs", "merge_b_four_refs", "merge_b_nobipred", "merge_b_10bit"]


# ------------------------------------------------------------------------------------------------ motion compensation
from kvazaar_b200.api import ME_MC_PU as MC_PU, MeMcRefs as McRefs  # noqa: E402

assert MC_PU.itemsize == 20 and C.sizeof(McRefs) == 416
MC_CASES = ["merge_p_one_ref", "merge_b_two_refs", "merge_b_four_refs", "merge_b_10bit"]


def chroma_planes(w, h, bd, seed):
    r = np.random.default_rng(8000 + seed)
    yy, xx = np.mgrid[0:h // 2, 0:w // 2]
    u = np.clip(128 + 50 * np.sin(xx / 5.0 + seed) + r.integers(-20, 21, (h // 2, w // 2)), 0, 255)
    v = np.clip(128 + 50 * np.cos(yy / 4.0 - seed) + r.integers(-20, 21, (h // 2, w // 2)), 0, 255)
    if bd == 10:
        return (u * 4 + r.integers(0, 4, u.shape)).astype(np.uint16), (v * 4 + r.integers(0, 4, v.shape)).astype(np.uint16)
    return u.astype(np.uint8), v.astype(np.uint8)


def make_mc_case(name):
    """the pictures / reference lists of a merge case (plus chroma planes); the picture tiled with CUs of 8..64 in random part modes,
    every PU with random motion (fractional, integer, far outside the picture) from one or two lists"""
    p, c, _, planes, _, _ = make_merge_case(name)
    r = np.random.default_rng(9000 + c["seed"])
    w, h, bd = p.width, p.height, p.bitdepth
    us, vs = zip(*[chroma_planes(w, h, bd, 10 * c["seed"] + k) for k in range(len(planes))])
    sizes = [len(c["l0"]), len(c["l1"])]
    pus, cu = [], []

    def add(cx, cy, size):
        if size > 8 and (cx + size > w or cy + size > h or r.integers(0, 3) != 0):
            for k in range(4):
                if cx + (k % 2) * size // 2 < w and cy + (k // 2) * size // 2 < h:
                    add(cx + (k % 2) * size // 2, cy + (k // 2) * size // 2, size // 2)
            return
        if cx + size > w or cy + size > h:
            return
        mode = int(r.integers(0, 7 if size >= 16 else 3))
        q = size // 4
        split = {0: None, 1: ("h", size // 2), 2: ("v", size // 2), 3: ("h", q), 4: ("h", size - q), 5: ("v", q), 6: ("v", size - q)}[mode]
        for ipu in range(2 if split else 1):
            x, y, pw, ph = cx, cy, size, size
            if split:
                kind, at = split
                if kind == "h":
                    y, ph = (cy, at) if ipu == 0 else (cy + at, size - at)
                else:
                    x, pw = (cx, at) if ipu == 0 else (cx + at, size - at)
            rec = np.zeros((), MC_PU)
            rec["x"], rec["y"], rec["w"], rec["h"] = x, y, pw, ph
            dirs = [1] if sizes[1] == 0 else [1, 2, 3, 3]
            d = int(dirs[int(r.integers(0, len(dirs)))])
            if d == 3 and pw + ph <= 12:
                d = 1                                                  # 8x4 / 4x8 PUs are never bi-predicted
            rec["dir"] = d
            for l in range(2):
                rng = 700 if r.integers(0, 15) == 0 else 48
                rec["mv"][l] = r.integers(-rng, rng + 1, 2)
                k = r.integers(0, 4)
                if k == 0:
                    rec["mv"][l] = (rec["mv"][l] >> 2) << 2            # integer luma MV (chroma may still be fractional)
                elif k == 1:
                    rec["mv"][l] = (rec["mv"][l] >> 3) << 3            # integer for chroma too: the copy path
                rec["mv_ref"][l] = int(r.integers(0, max(1, sizes[l])))
            pus.append(rec)
            cu.append((cx, cy, size, PART_MODES[mode], ipu))

    for cy in range(0, h, 64):
        for cx in range(0, w, 64):
            add(cx, cy, 64)
    return p, c, planes, list(us), list(vs), np.array(pus, MC_PU), np.array(cu, np.int32)


def mc_refs_struct(c, ys, us, vs):
    rf = McRefs()
    for i in range(len(ys)):
        rf.y[i], rf.u[i], rf.v[i] = ys[i], us[i], vs[i]
    for l, lst in enumerate((c["l0"], c["l1"])):
        for i, v in enumerate(lst):
            rf.ref_LX[l][i] = v
    return rf


def run_mc_reference(ref_shim, p, c, planes, us, vs, pus, cu):
    dt = planes[0].dtype
    oy, ou, ov = np.zeros((p.height, p.width), dt), np.zeros((p.height // 2, p.width // 2), dt), np.zeros((p.height // 2, p.width // 2), dt)
    ctx = ref_shim.ctx(27, 0, 0, p.width, p.height)

    def arr(lst):
        return (C.c_void_p * 16)(*[np.ascontiguousarray(lst[i if i < len(lst) else 0]).ctypes.data for i in range(16)])
    lx = np.zeros((2, 16), np.uint8)
    lx[0, :len(c["l0"])] = c["l0"]
    lx[1, :len(c["l1"])] = c["l1"]
    f = ref_shim.lib.kvzref_me_predict
    f.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                  C.c_void_p, C.c_void_p]
    cu = np.ascontiguousarray(cu, np.int32)
    rc = f(ctx, C.byref(p), len(planes), arr(planes), arr(us), arr(vs), lx.ctypes.data, pus.ctypes.data, cu.ctypes.data, len(pus), oy.ctypes.data,
           ou.ctypes.data, ov.ctypes.data)
    assert rc == 0, rc
    return oy, ou, ov


def run_mc_host_api(lib, p, c, planes, us, vs, pus):
    dt = planes[0].dtype
    oy, ou, ov = np.zeros((p.height, p.width), dt), np.zeros((p.height // 2, p.width // 2), dt), np.zeros((p.height // 2, p.width // 2), dt)
    keep = [np.ascontiguousarray(a) for a in list(planes) + list(us) + list(vs)]
    n = len(planes)
    rf = mc_refs_struct(c, [a.ctypes.data for a in keep[:n]], [a.ctypes.data for a in keep[n:2 * n]], [a.ctypes.data for a in keep[2 * n:]])
    lib.kvz_cuda_me_predict_batch.argtypes = [C.POINTER(Params), C.POINTER(McRefs), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = lib.kvz_cuda_me_predict_batch(C.byref(p), C.byref(rf), pus.ctypes.data, len(pus), oy.ctypes.data, ou.ctypes.data, ov.ctypes.data, None)
    assert rc == 0, rc
    return oy, ou, ov
