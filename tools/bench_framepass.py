#!/usr/bin/env python
"""bench.py -- frames/s of the per-CTU strategy-kernel hot path (the frame-level pass of framepass.cu).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA path
    python bench.py --impl reference --steps K --warmup W    # the reference's own CPU (AVX2) strategy functions

Workload (BASELINE.json configs[1]): 1920x1080 8-bit synthetic I420, all-intra, QP 27 ("medium": SAO on, no
sign hiding).  One STEP = `frames_per_step` frames through the frame-level pass: for every quadtree depth
(32/16/8/4) rough search of all 35 intra modes + SATD, mode selection, prediction + transform + quantisation +
reconstruction + SSD for luma and chroma, then SAO statistics/decision/reconstruction and the picture checksum.
`value` is frames/s with the frames already resident in HBM; `e2e` goes through the host-buffer C-ABI entry point
(kvz_cuda_fp_run_host: pinned host frame in, 28 MB result blob out, copies inside the timed region).
This is the hot PATH's throughput, not whole-encoder fps: mode decision / RDOQ / CABAC stay on the host and are
outside this round's scope (DESIGN.md).  Multi-GPU: frames are sharded one set per rank, no collective (all-intra
frames are independent), scaling = weak.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

W, H, QP, SIGNHIDE, RDOQ, TRSKIP, BITDEPTH = 1920, 1080, 27, 0, 0, 0, 8
WORKLOAD = "1920x1080 8-bit synthetic I420, all-intra, QP27 (preset medium: SAO on, signhide off), frame-level hot-path pass"


def set_workload(name, rdoq):
    """configs[1] (default, the one the metric is quoted on) or the configs[2] shape (2160p, QP22, sign hiding)."""
    global W, H, QP, SIGNHIDE, RDOQ, TRSKIP, BITDEPTH, WORKLOAD
    RDOQ = int(rdoq)
    q = "RDOQ on" if RDOQ else "RDOQ off (kvz_quant)"
    WORKLOAD = f"1920x1080 8-bit synthetic I420, all-intra, QP27 (preset medium: deblock + SAO on, signhide off, {q}), frame-level hot-path pass"
    if name == "2160p":
        W, H, QP, SIGNHIDE, TRSKIP = 3840, 2160, 22, 1, 1
        WORKLOAD = f"3840x2160 8-bit synthetic I420, all-intra, QP22 (preset veryslow shape: deblock + SAO on, signhide on, transform skip on, {q}), frame-level hot-path pass"


def set_workload_4320p10(rdoq):
    """configs[4] shape: 7680x4320 10-bit (the intra hot path of it; tiles / inter exchange are dist.py's business)."""
    global W, H, QP, SIGNHIDE, RDOQ, TRSKIP, BITDEPTH, WORKLOAD
    W, H, QP, SIGNHIDE, TRSKIP, BITDEPTH, RDOQ = 7680, 4320, 22, 0, 0, 10, int(rdoq)
    q = "RDOQ on" if RDOQ else "RDOQ off (kvz_quant)"
    WORKLOAD = f"7680x4320 10-bit synthetic I420, all-intra, QP22 (preset slow shape: deblock + SAO on, signhide off, {q}), frame-level hot-path pass"


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet, HBM3)"


def synth_frames(n):
    from test_framepass import synth_frame
    if BITDEPTH == 8:
        return [synth_frame(W, H, frame_idx=i) for i in range(n)]
    out = []
    for i in range(n):                       # 10-bit: the 8-bit pattern scaled by 4 plus two fresh low bits
        f8 = synth_frame(W, H, frame_idx=i).astype(np.uint16)
        out.append((f8 * 4 + np.random.default_rng(i).integers(0, 4, f8.size).astype(np.uint16)).astype(np.uint16))
    return out


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region (one streaming nvidia-smi process, 100 ms period)."""
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.proc, self.rows = index, None, []

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            time.sleep(0.35)          # first sample is out before the timed region starts
        except Exception:
            self.proc = None
        return self

    def __exit__(self, *a):
        if self.proc:
            time.sleep(0.15)
            self.proc.terminate()
            try:
                out, _ = self.proc.communicate(timeout=5)
            except Exception:
                self.proc.kill()
                out = ""
            for ln in out.splitlines():
                c = [x.strip() for x in ln.split(",")]
                if len(c) >= 7:
                    self.rows.append(c)

    def summary(self):
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        sm = sorted(float(r[0]) for r in self.rows)
        reasons = []
        for i, name in enumerate(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap")):
            if any(r[3 + i] == "Active" for r in self.rows):
                reasons.append(name)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": float(self.rows[0][1]), "reasons": reasons,
                "power_w_max": max(float(r[2]) for r in self.rows), "samples": len(self.rows)}


def run_reference(args):
    """The reference's own CPU implementation of the path: its strategy function pointers (AVX2 where selected),
    driven by oracle/ref_framepass.c with all host threads.  One step = `ref_frames` frames (bounded sample)."""
    from _oracle import Ref, ref_frame_pass
    import kvazaar_b200 as kb
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    ref = Ref(BITDEPTH)
    cores = os.cpu_count() or 1
    lay = kb.fp_layout_for(W, H, QP, SIGNHIDE, BITDEPTH)
    from _oracle import aligned, al
    frames = [al(f) for f in synth_frames(4)]
    blob = aligned(int(lay.host_bytes), np.uint8)
    nper = args.ref_frames
    for _ in range(max(1, args.warmup)):
        ref_frame_pass(ref, frames[0], W, H, QP, lay, nthreads=cores, signhide=SIGNHIDE, blob=blob, src_is_aligned=True, rdoq=RDOQ, trskip=TRSKIP)
    t0 = time.perf_counter()
    for s in range(args.steps):
        for f in range(nper):
            ref_frame_pass(ref, frames[(s * nper + f) % len(frames)], W, H, QP, lay, nthreads=cores, signhide=SIGNHIDE, blob=blob, src_is_aligned=True, rdoq=RDOQ, trskip=TRSKIP)
    dt = time.perf_counter() - t0
    fps = args.steps * nper / dt
    sample = f"{args.steps * nper} frames {W}x{H} through the reference's selected strategy functions ({ref.selected_name('satd_8x8')})"
    line = {"impl": "reference", "metric": "hot-path frames/sec at fixed QP (per-CTU strategy kernels, all depths)", "value": fps,
            "unit": "frames/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000 * dt / args.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8" if BITDEPTH == 8 else "u16", "data": "synthetic",
            "config": {"workload": WORKLOAD, "frames_per_step": nper},
            "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": cores, "kind": "reference", "sample": sample},
            "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def cpu_baseline(budget_s=15.0):
    """Bounded sample of the same workload on the host cores, through oracle/_ref when present (kind=reference)."""
    from _oracle import Ref, ref_frame_pass
    import kvazaar_b200 as kb
    try:
        ref = Ref(BITDEPTH)
    except Exception as e:  # pragma: no cover
        return {"value": None, "unit": "frames/s", "cores": 0, "kind": "reference", "sample": f"unavailable: {e}"}
    cores = os.cpu_count() or 1
    lay = kb.fp_layout_for(W, H, QP, SIGNHIDE, BITDEPTH)
    from _oracle import aligned, al
    frames = [al(f) for f in synth_frames(2)]
    blob = aligned(int(lay.host_bytes), np.uint8)
    ref_frame_pass(ref, frames[0], W, H, QP, lay, nthreads=cores, signhide=SIGNHIDE, blob=blob, src_is_aligned=True, rdoq=RDOQ, trskip=TRSKIP)
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < budget_s and n < 2000:
        ref_frame_pass(ref, frames[n % 2], W, H, QP, lay, nthreads=cores, signhide=SIGNHIDE, blob=blob, src_is_aligned=True, rdoq=RDOQ, trskip=TRSKIP)
        n += 1
    dt = time.perf_counter() - t0
    out = {"value": n / dt, "unit": "frames/s", "cores": cores, "kind": "reference",
           "sample": f"{n} frames {W}x{H} in {dt:.1f}s through oracle/_ref strategy pointers ({ref.selected_name('satd_8x8')}), {cores} threads"}
    # context: the unmodified reference ENCODER (whole pipeline incl. mode decision, RDOQ, CABAC) on the same input
    cli = os.path.join(ROOT, "oracle", "_ref", "kvazaar" if BITDEPTH == 8 else "kvazaar_10b")
    if os.path.exists(cli) and BITDEPTH == 8:       # (the 4320p 10-bit whole-encoder run would take minutes: skipped)
        try:
            yuv = f"/tmp/kvz_bench_{H}p.yuv"
            np.concatenate(synth_frames(4)).tofile(yuv)
            r = subprocess.run([cli, "-i", yuv, "--input-res", f"{W}x{H}", "-o", "/tmp/kvz_bench.hevc", "--preset", "veryslow" if W > 1920 else "medium", "-q", str(QP),
                                "-p", "1"], capture_output=True, text=True, timeout=120)
            for ln in (r.stderr + r.stdout).splitlines():
                if ln.strip().startswith("FPS:"):
                    out["reference_encoder_fps"] = float(ln.split(":")[1])
        except Exception:
            pass
    return out


def run_cuda(args):
    import torch
    import torch.distributed as dist
    import kvazaar_b200 as kb

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    kb.init(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    L = kb.lib()
    fps_step = args.frames_per_step
    inflight = args.inflight
    streams = [torch.cuda.Stream() for _ in range(inflight)]
    passes = [kb.FramePass(W, H, QP, SIGNHIDE, RDOQ, 0.0, TRSKIP, BITDEPTH) for _ in range(inflight)]
    frames_np = synth_frames(fps_step)
    # every rank gets its own frames (sharding = frame i of the job -> rank i mod world)
    frames_np = [np.roll(f, rank * 977) for f in frames_np]
    frames_dev = [kb.to_dev(f) for f in frames_np]
    frames_pin = [torch.from_numpy(f.copy()).pin_memory() for f in frames_np]
    results_pin = [torch.empty(passes[0].host_bytes, dtype=torch.uint8).pin_memory() for _ in range(inflight)]

    def step_dev():
        for i in range(fps_step):
            with torch.cuda.stream(streams[i % inflight]):
                passes[i % inflight].run_dev(frames_dev[i])

    def step_host():
        for i in range(fps_step):
            with torch.cuda.stream(streams[i % inflight]):
                passes[i % inflight].run_host(frames_pin[i], results_pin[i % inflight])

    # compact result: head of the blob + bitmap + non-zero coefficient chunks (lossless, kvz_cuda_fp_run_host_compact);
    # the chunk budget is 1/8 of the region and checked after the run
    lay0 = passes[0].layout
    budget = int(lay0.n_chunks) // 8
    small_pin = [torch.empty(int(lay0.coeff_begin), dtype=torch.uint8).pin_memory() for _ in range(inflight)]
    compact_pin = [torch.empty(int(lay0.compact_header_bytes) + 32 * budget, dtype=torch.uint8).pin_memory() for _ in range(inflight)]

    def step_host_compact():
        for i in range(fps_step):
            with torch.cuda.stream(streams[i % inflight]):
                passes[i % inflight].run_host_compact(frames_pin[i], small_pin[i % inflight], compact_pin[i % inflight], budget)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        main = torch.cuda.current_stream()
        e0.record(main)
        for s in streams:
            s.wait_stream(main)
        for _ in range(steps):
            fn()
        for s in streams:
            main.wait_stream(s)
        e1.record(main)
        barrier()
        ms = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t[0])
        return ms

    for _ in range(max(3, args.warmup)):
        step_dev()
    barrier()
    launches0 = kb.launch_count()
    with ClockSampler(local) as clk:
        ms = timed(step_dev, args.steps)
    launches = kb.launch_count() - launches0
    value = world * fps_step * args.steps / (ms / 1000.0)

    # ---- e2e: host buffers through the C-ABI, copies inside the timed region.  Headline e2e = the compact result
    # (what a host that feeds CABAC needs); e2e_full_blob = every coefficient of every depth as dense int16.
    for _ in range(3):
        step_host()
    ms_e2e_full = timed(step_host, args.steps)
    e2e_full = world * fps_step * args.steps / (ms_e2e_full / 1000.0)
    for _ in range(3):
        step_host_compact()
    ms_e2e = timed(step_host_compact, args.steps)
    e2e = world * fps_step * args.steps / (ms_e2e / 1000.0)
    nonzero_chunks = max(int(c.numpy()[:4].view(np.uint32)[0]) for c in compact_pin)
    d2h_compact = int(lay0.coeff_begin) + int(lay0.compact_header_bytes) + 32 * budget
    compact_ok = nonzero_chunks <= budget
    if not compact_ok:            # denser content than the budget: the dense blob is the end-to-end result then
        e2e, ms_e2e, d2h_compact = e2e_full, ms_e2e_full, passes[0].host_bytes

    # ---- live per-stage timing (CUDA events on the launching stream) -> roofline of the dominant kernel
    peak, peak_src = peaks()
    fp = passes[0]
    L.kvz_cuda_fp_set_timing(fp.h, 1)
    with torch.cuda.stream(streams[0]):
        for i in range(max(8, fps_step)):
            fp.run_dev(frames_dev[i % fps_step])
    torch.cuda.synchronize()
    NST = 40
    ms_stage = (C.c_double * NST)()
    runs = C.c_int()
    L.kvz_cuda_fp_get_timing(fp.h, ms_stage, C.byref(runs))
    L.kvz_cuda_fp_set_timing(fp.h, 0)
    stage_ms = [ms_stage[i] / max(1, runs.value) for i in range(NST)]
    names = [f"{k}_w{32 >> d}" for d in range(4) for k in ("rough_search", "recon_luma", "rdoq_luma", "recon_luma_inv", "bits_luma",
                                                           "recon_chroma", "rdoq_chroma", "recon_chroma_inv", "bits_chroma")] + \
            ["deblock", "sao_stats_decide", "sao_reconstruct", "checksum"]
    stages = {names[i]: round(stage_ms[i], 4) for i in range(NST) if stage_ms[i] > 0.0005}
    # per-LAUNCH time of each kernel (chroma stages hold two launches: U and V; deblocking two passes)
    per_launch = [stage_ms[i] / (2 if names[i].startswith("recon_chroma") or names[i] == "deblock" else 1) for i in range(NST)]
    dom = int(np.argmax(per_launch))

    def alg_bytes(name):
        """Bytes one launch must move through HBM (DESIGN.md section 4)."""
        kind, wtxt = name.rsplit("_w", 1) if "_w" in name else (name, "0")
        w = int(wtxt)
        if kind == "rough_search":       # source block + 4w+1 reference samples in, 35 costs out
            return (W // w) * (H // w) * (w * w + 4 * w + 1 + 35 * 4)
        if kind in ("recon_luma", "recon_luma_inv"):   # source + refs in; reconstruction + int16 coefficients + has + ssd out
            return (W // w) * (H // w) * (w * w + 4 * w + 1 + w * w + 2 * w * w + 5)
        if kind in ("recon_chroma", "recon_chroma_inv"):   # one of the two chroma planes, blocks of w/2
            wc = w // 2
            return (W // w) * (H // w) * (wc * wc + 4 * wc + 1 + wc * wc + 2 * wc * wc + 5)
        if kind == "bits_luma":          # int16 levels in, one double per block out
            return W * H * 2 + (W // w) * (H // w) * 8
        if kind == "bits_chroma":        # U and V in one launch
            return 2 * ((W // 2) * (H // 2) * 2 + (W // w) * (H // w) * 8)
        if kind == "rdoq_luma":          # int16 coefficients in, int16 levels out
            return W * H * 4
        if kind == "rdoq_chroma":        # U and V in one launch
            return 2 * (W // 2) * (H // 2) * 4
        if kind == "deblock":            # per pass (launch): the three reconstruction planes in and out + 20-byte CU records in
            return 2 * W * H * 3 // 2 + (W // 4) * (H // 4) * 20
        if kind == "sao_stats_decide":   # source + reconstruction of all three planes in, 40+4+1 ints per CTU-plane out
            return 2 * W * H * 3 // 2 + 3 * ((W + 63) // 64) * ((H + 63) // 64) * 46 * 4
        return None

    roof = None
    alg = alg_bytes(names[dom])
    if alg:
        ach = alg / (per_launch[dom] / 1000.0) / 1e9
        kname = {"rough_search": "rough_search_u8_kernel", "recon_luma": "intra_recon_kernel", "recon_chroma": "intra_recon_kernel",
                 "recon_luma_inv": "intra_recon_kernel", "recon_chroma_inv": "intra_recon_kernel", "rdoq_luma": "rdoq_grid_kernel",
                 "rdoq_chroma": "rdoq_grid_kernel", "bits_luma": "coeff_cost_grid_kernel", "bits_chroma": "coeff_cost_grid_kernel",
                 "sao_stats_decide": "sao_ctu_kernel", "deblock": "deblock_pass_kernel"}.get(names[dom].rsplit("_w", 1)[0], names[dom])
        roof = {"kernel": f"{kname} [{names[dom]}]", "bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                "traffic": None, "ms_per_launch": per_launch[dom],
                "algorithmic_bytes_per_launch": alg, "peak_source": peak_src,
                "note": ("RDOQ is HM's serial per-TU chain (one lane of a warp walks the scan in double precision): latency bound; "
                         if names[dom].startswith("rdoq") else
                         "fused per-block kernels keep predictions / transforms on chip: they are instruction-issue bound, not HBM bound; ")
                        + "roofline_satd_batch is the HBM-streaming kernel of the north star"}

    # ---- the batched SATD kernel of the north_star (block pairs streamed from HBM), inputs > L2
    n_pairs = 4 * 1024 * 1024            # 4M 8x8 pairs = 512 MiB of pixels > 50 MB L2
    g = torch.Generator(device="cuda").manual_seed(7)
    a = torch.randint(0, 256, (n_pairs * 64,), dtype=torch.uint8, device="cuda", generator=g)
    b = torch.randint(0, 256, (n_pairs * 64,), dtype=torch.uint8, device="cuda", generator=g)
    out = torch.empty(n_pairs, dtype=torch.int32, device="cuda")       # no allocation inside the timed launches
    for _ in range(3):
        kb.satd_nxn_batch(8, a, b, n_pairs, out)
    torch.cuda.synchronize()
    reps = 20
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i in range(reps):                        # one event pair per launch: host-side gaps between launches are not kernel time
        evs[i][0].record()
        kb.satd_nxn_batch(8, a, b, n_pairs, out)
        evs[i][1].record()
    torch.cuda.synchronize()
    per = [e0.elapsed_time(e1) for e0, e1 in evs]
    ms_satd = float(np.mean(per))                # the reported figure is the MEAN launch duration
    alg_satd = n_pairs * (2 * 64 + 4)        # SURVEY.md 8(d): 2*N*N*s + 4 bytes per block pair
    ach_satd = alg_satd / (ms_satd / 1000.0) / 1e9
    roof_satd = {"kernel": "satd_nxn_kernel<u8,8> (kvz_cuda_satd_nxn_batch)", "bound": "hbm", "achieved": ach_satd, "peak": peak,
                 "unit": "GB/s", "frac": ach_satd / peak, "traffic": None, "ms_per_launch": ms_satd, "pairs_per_launch": n_pairs,
                 "algorithmic_bytes_per_launch": alg_satd, "peak_source": peak_src, "checksum": int(out.to(torch.int64).sum()),
                 "ms_per_launch_min_median_max": [round(float(np.min(per)), 5), round(float(np.median(per)), 5), round(float(np.max(per)), 5)]}
    del a, b

    if rank == 0:
        line = {"metric": "hot-path frames/sec at fixed QP (per-CTU strategy kernels, all depths)", "value": value, "unit": "frames/s",
                "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms / args.steps,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8" if BITDEPTH == 8 else "u16", "data": "synthetic",
                "config": {"workload": WORKLOAD, "frames_per_step": fps_step, "frames_in_flight": inflight, "parallelism": f"frames/{world}",
                           "l2": f"working set per step ({fps_step} distinct {passes[0].frame_bytes / 1e6:.1f} MB frames + {inflight} result/scratch blobs of "
                                 f"{passes[0].host_bytes / 1e6:.0f}+ MB each) exceeds the 50 MB L2"},
                "e2e": {"value": e2e, "unit": "frames/s", "h2d_bytes_per_step": fps_step * passes[0].frame_bytes,
                        "d2h_bytes_per_step": fps_step * d2h_compact, "ms_per_step": ms_e2e / args.steps,
                        "result": "compact: blob head + bitmap + non-zero 32-byte coefficient chunks (lossless)" if compact_ok
                                  else "dense blob (the compact chunk budget was exceeded)",
                        "nonzero_chunks_per_frame": nonzero_chunks, "chunk_budget": budget},
                "e2e_full_blob": {"value": e2e_full, "unit": "frames/s", "d2h_bytes_per_step": fps_step * passes[0].host_bytes,
                                  "ms_per_step": ms_e2e_full / args.steps},
                "gpu_launches": int(launches), "clocks": clk.summary(), "roofline": roof, "roofline_satd_batch": roof_satd,
                "stage_ms_per_frame": stages}
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline()
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="cuda", choices=["cuda", "reference"])
    ap.add_argument("--frames-per-step", type=int, default=8)
    ap.add_argument("--inflight", type=int, default=4, help="frames in flight (one stream + one result blob each)")
    ap.add_argument("--ref-frames", type=int, default=8, help="frames per step of the reference arm (bounded sample)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--workload", default="1080p", choices=["1080p", "2160p", "4320p10"], help="1080p = BASELINE configs[1] (default)")
    ap.add_argument("--rdoq", type=int, default=1, choices=[0, 1], help="1 (default): quantise with kvz_rdoq as the medium / veryslow presets do; 0: kvz_quant")
    args = ap.parse_args()
    if args.workload == "4320p10":
        set_workload_4320p10(args.rdoq)
    else:
        set_workload(args.workload, args.rdoq)
    if args.impl == "reference":
        run_reference(args)
    else:
        run_cuda(args)


if __name__ == "__main__":
    main()
