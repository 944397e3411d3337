"""Times kvz_cuda_satd_nxn_batch(8) -- the HBM-streaming kernel of the north star -- on 4 Mi block pairs (512 MiB of input,
more than L2) with CUDA events.  `--json`: one JSON object (bench.py attaches it to its line as "roofline_satd_batch")."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import kvazaar_b200 as kb  # noqa: E402
kb.init(0)
n = 4 * 1024 * 1024
g = torch.Generator(device="cuda").manual_seed(7)
a = torch.randint(0, 256, (n * 64,), dtype=torch.uint8, device="cuda", generator=g)
b = torch.randint(0, 256, (n * 64,), dtype=torch.uint8, device="cuda", generator=g)
for _ in range(3):
    kb.satd_nxn_batch(8, a, b, n)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20):
    o = kb.satd_nxn_batch(8, a, b, n)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 20
peak, src = 3350.0, "fallback (H100 SXM data sheet, HBM3)"
mp = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
if os.path.exists(mp):
    peak, src = float(json.load(open(mp))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
alg = n * 132                      # SURVEY 8(d): 2 * 64 bytes in + 4 bytes out per 8x8 pair
if "--json" in sys.argv:
    print(json.dumps({"kernel": "satd_nxn_kernel<u8,8> (kvz_cuda_satd_nxn_batch)",
                      "bound": "hbm", "achieved": alg / ms / 1e6, "peak": peak, "unit": "GB/s", "frac": alg / ms / 1e6 / peak, "traffic": None,
                      "ms_per_launch": ms, "pairs_per_launch": n, "algorithmic_bytes_per_launch": alg, "peak_source": src,
                      "checksum": int(o.to(torch.int64).sum()), "timing": "CUDA events over 20 launches after 3 warm-up launches; inputs (512 MiB) exceed L2"}))
else:
    print(f"{ms:.4f} ms  {alg / ms / 1e6:.0f} GB/s  frac {alg / ms / 1e6 / peak:.3f}  sum {int(o.to(torch.int64).sum())}")
