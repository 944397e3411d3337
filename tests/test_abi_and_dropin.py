"""C-ABI surface (CPU) and drop-in tests (GPU): the reference's own greatest suites over the "cuda" entries and
bitstream identity of the unmodified reference encoder with the cuda strategies bound in."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def _header_functions():
    txt = open(os.path.join(ROOT, "include", "kvz_cuda.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    names = set(re.findall(r"\b(kvz_(?:cuda|strategy)_[a-z0-9_]+)\s*\(", txt))
    names -= {"kvz_cuda_register_fn"}
    return sorted(names)


def test_library_exports_every_declared_symbol():
    """include/kvz_cuda.h <-> libkvzcuda.so: every declared entry point is exported (no compute call is made)."""
    import kvazaar_b200 as kb
    lib = C.CDLL(kb.LIB_PATH)
    names = _header_functions()
    assert len(names) > 60
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_no_device_degrades_to_not_registering():
    """Without a GPU the registrars must report success and register nothing (SURVEY.md 8b 'Errors')."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    import kvazaar_b200 as kb
    lib = kb.lib()
    calls = []
    CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_void_p)
    cb = CB(lambda o, t, n, p, f: calls.append(t) or 1)
    lib.kvz_cuda_set_register_fn(cb)
    assert lib.kvz_strategy_register_picture_cuda(None, 8) == 1
    lib.kvz_cuda_set_register_fn(None)
    assert calls == []
    assert lib.kvz_cuda_strategy_fptr(b"satd_8x8", 8)           # the table itself is there
    with pytest.raises(kb.KvzCudaError):
        kb.satd_nxn_batch(8, None, None, 0)                     # compute entry points refuse loudly


def _yuv(path, w, h, frames, seed=3):
    from test_framepass import synth_frame
    np.concatenate([synth_frame(w, h, seed=seed, frame_idx=i) for i in range(frames)]).tofile(path)


def _need(*names):
    paths = [os.path.join(REF_DIR, n) for n in names]
    for p in paths:
        if not os.path.exists(p):
            pytest.skip(f"{p} not built (needs /root/reference at build time)")
    return paths


def test_host_program_matches_reference_cli(tmp_path):
    """integration/kvz_cuda_encode.c without --cuda is just the reference library: same bytes as the CLI."""
    enc, cli = _need("kvz_cuda_encode", "kvazaar")
    yuv = str(tmp_path / "a.yuv")
    _yuv(yuv, 64, 64, 2)
    a, b = str(tmp_path / "a.hevc"), str(tmp_path / "b.hevc")
    subprocess.check_call([enc, yuv, "64x64", a, "preset=ultrafast", "qp=32", "period=1", "threads=0", "owf=0"],
                          stderr=subprocess.DEVNULL)
    subprocess.check_call([cli, "-i", yuv, "--input-res", "64x64", "-o", b, "--preset", "ultrafast", "-q", "32", "-p", "1",
                           "--threads", "0", "--owf", "0"], stderr=subprocess.DEVNULL, stdout=subprocess.DEVNULL)
    assert open(a, "rb").read() == open(b, "rb").read()


@pytest.mark.gpu
def test_reference_greatest_suites_over_cuda_entries():
    """tests/{sad,intra_sad,satd,dct,coeff_sum}_tests.c of the reference, unmodified, iterating a strategy list that
    contains the cuda entries (integration/test_strategies_cuda.c)."""
    (exe,) = _need("kvazaar_tests_cuda")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    m = re.search(r"(\d+) cuda entries appended", out)
    assert m and int(m.group(1)) >= 40, out[-2000:]
    assert r.returncode == 0, out[-3000:]
    assert re.search(r"Pass: \d+, fail: 0", out) or "fail: 0" in out, out[-2000:]


DROPIN_CASES = [
    # BASELINE.json configs[0]: 64x64 ultrafast -q 32 -p 1
    ("cfg0_ultrafast_intra", 64, 64, 2, ["preset=ultrafast", "qp=32", "period=1"]),
    # medium (RDOQ on the device between our forward and inverse halves, SAO full)
    ("medium_intra_rdoq_sao", 64, 64, 1, ["preset=medium", "qp=27", "period=1"]),
    # inter: hexbs ME, fractional ME (FME filters), bipred, merge -> ipol + sad + satd_any_size(+quad)
    ("fast_inter", 128, 64, 3, ["preset=fast", "qp=30", "period=16", "gop=0"]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h,frames,opts", DROPIN_CASES)
def test_bitstream_identical_with_cuda_strategies(tmp_path, name, w, h, frames, opts):
    """The unmodified reference encoder produces the same .hevc with every strategy pointer bound to CUDA."""
    (enc,) = _need("kvz_cuda_encode")
    yuv = str(tmp_path / "in.yuv")
    _yuv(yuv, w, h, frames)
    ref_out, cuda_out = str(tmp_path / "ref.hevc"), str(tmp_path / "cuda.hevc")
    common = [yuv, f"{w}x{h}"]
    extra = opts + ["threads=2", "owf=1"]
    subprocess.check_call([enc] + common + [ref_out] + extra, stderr=subprocess.DEVNULL, timeout=600)
    r = subprocess.run([enc, "--cuda"] + common + [cuda_out] + extra, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"(\d+) strategy pointers bound", r.stderr)
    assert m and int(m.group(1)) >= 60, r.stderr
    a, b = open(ref_out, "rb").read(), open(cuda_out, "rb").read()
    assert len(a) > 100
    assert a == b, f"{name}: bitstreams differ ({len(a)} vs {len(b)} bytes)"


def _sel_encode(tmp_path, env=None):
    sel, ref = _need("kvazaar_sel", "kvazaar")
    clip = str(tmp_path / "sel64.yuv")
    _yuv(clip, 64, 64, 2)
    outs, logs = [], []
    for binary, e2 in ((ref, {}), (sel, env or {})):
        e = dict(os.environ)
        for k in list(e):
            if k.startswith("KVAZAAR_OVERRIDE_"):
                del e[k]
        e.update(e2)
        out = str(tmp_path / f"o{len(outs)}.hevc")
        r = subprocess.run([binary, "-i", clip, "--input-res", "64x64", "-o", out, "--preset", "ultrafast", "-q", "32", "-p", "1"],
                           env=e, stderr=subprocess.PIPE, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-1500:]
        outs.append(open(out, "rb").read())
        logs.append(r.stderr)
    return outs, logs[1]


def _chosen(log, strategy_type):
    """the line DEBUG_STRATEGYSELECTOR marks with '>' in the block of `strategy_type` (strategyselector.c:309-320)"""
    block = log.split(f"Choosing strategy for {strategy_type}:\n", 1)[1].split("Choosing strategy for", 1)[0]
    return [ln for ln in block.splitlines() if ln.startswith(">")][0]


def test_selection_library_without_device_keeps_host_strategies(tmp_path):
    """CPU: the selector-wrapped reference registers nothing without a device and encodes like the plain reference"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    outs, log = _sel_encode(tmp_path)
    assert outs[0] == outs[1] and len(outs[0]) > 100
    assert "cuda" not in _chosen(log, "satd_8x8")


@pytest.mark.gpu
def test_selection_through_the_reference_selector(tmp_path):
    """The cuda entries registered inside kvz_strategyselector_init through kvz_strategyselector_register
    (strategyselector.c:233-273): priority 50 wins the choice (:296), KVAZAAR_OVERRIDE_<type>=cuda|generic both work
    (:286-306), and the bitstream of BASELINE config 1 stays identical in every case."""
    outs, log = _sel_encode(tmp_path)
    assert outs[0] == outs[1] and len(outs[0]) > 100
    for t in ("satd_8x8", "dct_8x8", "angular_pred", "sao_edge_ddistortion", "quant", "array_checksum", "filter_hpel_blocks_hor_ver_luma"):
        assert "> cuda (50" in _chosen(log, t), (t, _chosen(log, t))
    outs, log = _sel_encode(tmp_path, {"KVAZAAR_OVERRIDE_satd_8x8": "generic", "KVAZAAR_OVERRIDE_dct_8x8": "cuda"})
    assert outs[0] == outs[1]
    assert "choosing satd_8x8:generic" in log and "choosing dct_8x8:cuda" in log
