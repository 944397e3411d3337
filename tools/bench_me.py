#!/usr/bin/env python
"""Device timing of the motion-search kernels (SURVEY 8f rank 4) next to the reference's own functions on one host thread.

    python tools/bench_me.py [--res 1920x1080] [--pu 16] [--algo hexbs|dia|tz|full8] [--bitdepth 8] [--iters 20] [--fme-level 4]

Every pu x pu block of a synthetic picture pair goes through (the settings of --preset slow: early termination on, WPP + SAO
limits): the integer search (kvz_cuda_me_search_batch), then the fractional search from its results
(kvz_cuda_me_frac_search_batch), the AMVP / merge candidate derivation of as many PUs from a random CU image
(kvz_cuda_me_candidates_batch), and the merge analysis of those candidates (kvz_cuda_me_merge_cost_batch).  CUDA events on the launching stream around `iters` launches after 3 warm-up launches.
The reference arm is oracle/ref_me.c (the reference's search_inter.c compiled in place, its selected AVX2 strategies) on ONE
host thread: a per-core baseline, not the target.  One JSON line.  bench.py runs this in a subprocess after its own
measurement and attaches the line as "me_search".
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def timed(fn, iters):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(res="1920x1080", pu=16, algo="hexbs", bitdepth=8, iters=20, fme_level=4, with_reference=True):
    import kvazaar_b200 as kb
    from me_cases import (CAND_OUT, CAND_PU, RESULT, CAND_CASES, RefShim, cu_image, grid_case, make_cand_case, run_cand_reference,
                          run_frac_reference, run_reference, same)
    w, h = map(int, res.split("x"))
    kb.init(0)
    p, cur, rf, pus = grid_case(w, h, bitdepth, pu)
    p.ime_algorithm = {"hexbs": 0, "tz": 1, "full8": 3, "full16": 4, "dia": 7}[algo]
    d_cur, d_ref, d_pus = kb.to_dev(cur), kb.to_dev(rf), kb.to_dev(pus)
    px = 1 if bitdepth == 8 else 2
    peak = 3350.0     # H100 SXM data sheet (HBM3) unless measured
    mp = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(mp):
        peak = float(json.load(open(mp))["hbm_gbs"])
    alg = 2 * w * h * px                       # both luma planes read once (the PU records and results are ~1 % of that)
    line = {"workload": f"{res} {bitdepth}-bit luma, every {pu}x{pu} PU, --preset slow settings ({algo}, early termination on, WPP + SAO limits)",
            "pus": int(len(pus)), "iters": iters, "algorithmic_bytes_per_launch": alg, "hbm_peak_GBps": peak}

    # ---- integer search
    out = kb.me_search_batch(p, d_cur, d_ref, d_pus)
    ms = timed(lambda: kb.me_search_batch(p, d_cur, d_ref, d_pus, out), iters)
    integer = out.cpu().numpy().view(RESULT).copy()
    line["integer"] = {"kernel": "me_search_kernel", "ms_per_launch": ms, "pus_per_s": len(pus) / ms * 1e3, "points_per_pu": float(integer["points"].mean()),
                       "sad_pixels_per_s": float(integer["points"].sum()) * pu * pu / ms * 1e3, "GBps": alg / ms / 1e6, "frac_of_hbm_peak": alg / ms / 1e6 / peak}
    # ---- fractional search from the integer results
    pus2 = pus.copy()
    pus2["start_mv"] = integer["mv"]
    d_pus2 = kb.to_dev(pus2)
    out2 = kb.me_frac_search_batch(p, fme_level, d_cur, d_ref, d_pus2)
    ms2 = timed(lambda: kb.me_frac_search_batch(p, fme_level, d_cur, d_ref, d_pus2, out2), iters)
    frac = out2.cpu().numpy().view(RESULT).copy()
    line["fractional"] = {"kernel": "me_frac_kernel", "fme_level": fme_level, "ms_per_launch": ms2, "pus_per_s": len(pus) / ms2 * 1e3,
                          "positions_per_pu": float(frac["points"].mean()), "GBps": alg / ms2 / 1e6, "frac_of_hbm_peak": alg / ms2 / 1e6 / peak}
    # ---- candidates: as many PUs, CU records of a picture of this size
    f, crp, clx, _, _, _ = make_cand_case("p_four_refs")
    f.width, f.height = w, h
    r = np.random.default_rng(5)
    cus, col = cu_image(w, h, r, [4, 0]), cu_image(w, h, r, [4, 4], inter_share=0.8)
    cpus = np.zeros(len(pus), CAND_PU)
    for k in ("x", "y", "w", "h"):
        cpus[k] = pus[k]
    cpus["use_a1"], cpus["use_b1"] = 1, 1
    d_cus, d_col = kb.to_dev(cus.view(np.uint8).reshape(cus.shape[0], -1)), kb.to_dev(col.view(np.uint8).reshape(col.shape[0], -1))
    d_cpus = kb.to_dev(cpus)
    out3 = kb.me_candidates_batch(f, d_cus, d_col, d_cpus)
    ms3 = timed(lambda: kb.me_candidates_batch(f, d_cus, d_col, d_cpus, out3), iters)
    cand = out3.cpu().numpy().view(CAND_OUT).copy()
    line["candidates"] = {"kernel": "me_cand_kernel", "ms_per_launch": ms3, "pus_per_s": len(cpus) / ms3 * 1e3}

    # ---- merge analysis of the same PUs with the derived merge candidates (P slice, four reference pictures)
    from me_cases import MERGE_COST, PU, merge_refs_struct, pictures, run_merge_reference
    planes = [rf] + [pictures(w, h, bitdepth, 90 + k)[1] for k in range(1, 4)]
    mcase = {"l0": [0, 1, 2, 3], "l1": [], "bipred": 0, "ctx": (30, 11)}
    mpus = np.zeros(len(pus), PU)
    for k in ("x", "y", "w", "h"):
        mpus[k] = pus[k]
    mpus["num_merge"] = cand["num_merge"]
    mpus["merge"] = cand["merge"]
    d_planes = [kb.to_dev(pl) for pl in planes]
    mbits = (2.128, 1.376, 0.702)
    mcu = np.stack([pus["x"], pus["y"], pus["w"], np.zeros(len(pus)), np.zeros(len(pus))], 1).astype(np.int32)
    shim_m = None
    if with_reference:
        shim_m = RefShim(bitdepth)
        t = time.perf_counter(); want4, mbits = run_merge_reference(shim_m, p, mcase, cur, planes, mpus, mcu); t_m = time.perf_counter() - t
    refs_struct = merge_refs_struct(mcase, [t_.data_ptr() for t_ in d_planes], w, mbits)
    d_mpus = kb.to_dev(mpus)
    out4 = kb.me_merge_cost_batch(p, refs_struct, d_cur, d_mpus)
    ms4 = timed(lambda: kb.me_merge_cost_batch(p, refs_struct, d_cur, d_mpus, out4), iters)
    mres = out4.cpu().numpy().view(MERGE_COST).copy()
    line["merge_analysis"] = {"kernel": "me_merge_kernel", "ms_per_launch": ms4, "pus_per_s": len(pus) / ms4 * 1e3,
                              "candidates_costed_per_pu": float(mres["size"].mean())}
    if with_reference:
        line["merge_analysis"].update({"reference_one_thread_ms": t_m * 1e3, "identical": bool(mres.tobytes() == want4.tobytes())})

    if with_reference:
        shim = RefShim(bitdepth)
        t = time.perf_counter(); want = run_reference(shim, p, cur, rf, pus); t_int = time.perf_counter() - t
        t = time.perf_counter(); want2 = run_frac_reference(shim, p, fme_level, cur, rf, pus2); t_frac = time.perf_counter() - t
        line["integer"].update({"reference_one_thread_ms": t_int * 1e3, "identical": bool(same(integer, want))})
        line["fractional"].update({"reference_one_thread_ms": t_frac * 1e3, "identical": bool(same(frac, want2))})
        if bitdepth == 8:
            t = time.perf_counter(); want3 = run_cand_reference(shim, f, crp, clx, cus, col, cpus); t_c = time.perf_counter() - t
            line["candidates"].update({"reference_one_thread_ms": t_c * 1e3, "identical": bool(cand.tobytes() == want3.tobytes())})
        line["cpu_baseline"] = {"kind": "reference", "cores": 1, "sample": "the same PUs through oracle/ref_me.c (the reference's own functions), one host thread"}
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--pu", type=int, default=16)
    ap.add_argument("--algo", default="hexbs", choices=["hexbs", "tz", "full8", "full16", "dia"])
    ap.add_argument("--bitdepth", type=int, default=8, choices=[8, 10])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--fme-level", type=int, default=4)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    print(json.dumps(measure(a.res, a.pu, a.algo, a.bitdepth, a.iters, a.fme_level, not a.no_reference)))


if __name__ == "__main__":
    main()
