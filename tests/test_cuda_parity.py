"""GPU parity tests: every batched entry point of libkvzcuda.so (called through the C ABI via ctypes) must be
bit-exact against the oracle (oracle/kvz_oracle.c) on seeded inputs, against the reference's own golden
constants, and -- at full frame sizes -- satisfy size-independent properties.  Integer work: tolerance is zero.
"""
import numpy as np
import pytest

import _cases as cs

pytestmark = pytest.mark.gpu


def dev(kb, a):
    return kb.to_dev(a)


def host(t):
    return t.cpu().numpy()


# --------------------------------------------------------------------------- picture group
@pytest.mark.parametrize("n", (4, 8, 16, 32, 64))
def test_sad_satd_nxn_batch(cuda_lib, orc, n):
    kb = cuda_lib
    r = cs.rng(1000 + n)
    count = 257
    a = np.concatenate([cs.rand_pix(r, n * n, kind=cs.KINDS[i % 3]) for i in range(count)])
    b = np.concatenate([cs.rand_pix(r, n * n, kind=cs.KINDS[(i // 3) % 3]) for i in range(count)])
    sad = host(kb.sad_nxn_batch(n, dev(kb, a), dev(kb, b), count))
    satd = host(kb.satd_nxn_batch(n, dev(kb, a), dev(kb, b), count))
    for i in range(count):
        ai, bi = a[i * n * n:(i + 1) * n * n], b[i * n * n:(i + 1) * n * n]
        assert sad[i] == orc.sad_nxn(n, ai, bi), (n, i)
        assert satd[i] == orc.satd_nxn(n, ai, bi), (n, i)


def test_satd8_large_batch(cuda_lib, orc):
    """A batch of more than 4096 pairs; the odd count exercises a partial last CTA."""
    kb = cuda_lib
    r = cs.rng(1050)
    count = 3 * 4096 + 77
    a = r.integers(0, 256, count * 64).astype(np.uint8)
    b = r.integers(0, 256, count * 64).astype(np.uint8)
    a[: 64 * 300] = cs.rand_pix(r, 64 * 300, kind="extreme")
    got = host(kb.satd_nxn_batch(8, dev(kb, a), dev(kb, b), count))
    for i in list(range(0, 600)) + list(range(count - 300, count)) + list(range(4000, 4200)):
        assert got[i] == orc.satd_nxn(8, cs.al(a[i * 64:(i + 1) * 64]), cs.al(b[i * 64:(i + 1) * 64])), i
    # and the whole batch against the multi-mode entry point with one mode
    plain = host(kb.cost_nxn_multi_batch(1, 8, dev(kb, a), 64, 0, 1, dev(kb, b), count)).ravel()
    assert np.array_equal(got, plain)


@pytest.mark.parametrize("test", (0, 1, 2))
def test_satd_reference_goldens(cuda_lib, test):
    """The known answers of the reference's satd_tests (tests/satd_tests.c:122,140,159)."""
    kb = cuda_lib
    for log_w in range(2, 7):
        n = 1 << log_w
        a, b = cs.satd_test_bufs(test, log_w)
        got = host(kb.satd_nxn_batch(n, dev(kb, np.concatenate([a, b])), dev(kb, np.concatenate([b, a])), 2))
        assert list(got) == [cs.SATD_GOLDEN[test][log_w - 2]] * 2


def test_intra_sad_reference_goldens(cuda_lib):
    kb = cuda_lib
    for log_w in range(2, 7):
        n = 1 << log_w
        a, b = cs.intra_sad_bufs(0, log_w)
        assert int(kb.sad_nxn_batch(n, dev(kb, a), dev(kb, b), 1)[0]) == 255 * n * n
        a, b = cs.intra_sad_bufs(1, log_w)
        assert int(kb.sad_nxn_batch(n, dev(kb, a), dev(kb, b), 1)[0]) == int(np.abs(a.astype(int) - b.astype(int)).sum())


@pytest.mark.parametrize("n", (4, 8, 16, 32, 64))
def test_dual_costs(cuda_lib, orc, n):
    """satd_NxN_dual / sad_NxN_dual: pred_buffer layout, two modes 32*32 pixels apart."""
    kb = cuda_lib
    r = cs.rng(1100 + n)
    count = 33
    pitch = 2 * 1024 + (n * n if n == 64 else 0) + 1024      # per-block pitch, multiple of 16
    pitch = (pitch + 15) // 16 * 16
    preds = np.zeros(count * pitch, np.uint8)
    orig = np.concatenate([cs.rand_pix(r, n * n) for _ in range(count)])
    for i in range(count):
        preds[i * pitch: i * pitch + 1024 + n * n] = cs.rand_pix(r, 1024 + n * n, kind=cs.KINDS[i % 3])
    for use_satd in (0, 1):
        got = host(kb.cost_nxn_multi_batch(use_satd, n, dev(kb, preds), pitch, 1024, 2, dev(kb, orig), count))
        for i in range(count):
            p = cs.al(preds[i * pitch: i * pitch + 1024 + n * n])
            o = orig[i * n * n:(i + 1) * n * n]
            want = orc.satd_nxn_dual(n, p, o) if use_satd else orc.sad_nxn_dual(n, p, o)
            assert list(got[i]) == list(want), (n, use_satd, i)


def test_strided_block_costs(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(1200)
    sa, sb, rows = 208, 176, 160
    a = cs.rand_pix(r, sa * rows)
    b = cs.rand_pix(r, sb * rows, kind="smooth")
    shapes = [(w, h) for w in (4, 8, 12, 16, 24, 32, 48, 64) for h in (4, 8, 12, 16, 24, 32, 48, 64)]
    descs = np.zeros(len(shapes) * 3, kb.BLK)
    for i in range(len(descs)):
        w, h = shapes[i % len(shapes)]
        ya, xa = int(r.integers(0, rows - 64)), int(r.integers(0, sa - 64))
        yb, xb = int(r.integers(0, rows - 64)), int(r.integers(0, sb - 64))
        descs[i] = (ya * sa + xa, yb * sb + xb, w, h, 0, 0)
    da, db = dev(kb, a), dev(kb, b)
    sad = host(kb.block_cost_batch(kb.OP_REG_SAD, da, sa, db, sb, descs))
    satd = host(kb.block_cost_batch(kb.OP_SATD_ANY, da, sa, db, sb, descs))
    ver = host(kb.block_cost_batch(kb.OP_VER_SAD, da, sa, db, sb, descs))
    for i, d in enumerate(descs):
        w, h = int(d["w"]), int(d["h"])
        pa, pb = a[d["off_a"]:], b[d["off_b"]:]
        assert sad[i] == orc.reg_sad(pa, pb, w, h, sa, sb), (i, w, h)
        assert satd[i] == orc.satd_any_size(w, h, pa, sa, pb, sb), (i, w, h)
        assert ver[i] == orc.ver_sad(pa, pb, w, h, sa), (i, w, h)
    # SSD uses width only
    ssd_d = descs[[i for i, d in enumerate(descs) if d["w"] == d["h"] and d["w"] in (4, 8, 16, 32, 64)]]
    ssd = host(kb.block_cost_batch(kb.OP_SSD, da, sa, db, sb, ssd_d))
    for i, d in enumerate(ssd_d):
        assert ssd[i] == orc.pixels_calc_ssd(a[d["off_a"]:], b[d["off_b"]:], sa, sb, int(d["w"]))
    # hor_sad: exactly one of left/right non-zero (src/image.c:326-387)
    hd = descs.copy()
    for i in range(len(hd)):
        w = int(hd[i]["w"])
        side = int(r.integers(1, w))
        if i % 2:
            hd[i]["left"] = side
        else:
            hd[i]["right"] = side
    hs = host(kb.block_cost_batch(kb.OP_HOR_SAD, da, sa, db, sb, hd))
    for i, d in enumerate(hd):
        assert hs[i] == orc.hor_sad(a[d["off_a"]:], b[d["off_b"]:], int(d["w"]), int(d["h"]), sa, sb, int(d["left"]),
                                    int(d["right"])), i


def test_satd_any_size_quad_with_reference_quirk(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(1300)
    ps, os_, rows = 64, 96, 64
    pred = cs.rand_pix(r, 4 * ps * rows + 64)
    orig = cs.rand_pix(r, os_ * rows + 64)
    shapes = [(w, h) for w in (8, 12, 16, 24, 32, 48, 64) for h in (4, 8, 12, 16, 24, 32, 48, 64)] + [(4, 8), (4, 16)]
    descs = np.zeros(len(shapes), kb.QUAD)
    for i, (w, h) in enumerate(shapes):
        descs[i]["off_pred"] = [k * ps * rows for k in range(4)]
        descs[i]["off_orig"] = 0
        descs[i]["w"], descs[i]["h"] = w, h
    got = host(kb.satd_any_size_quad_batch(dev(kb, pred), ps, dev(kb, orig), os_, descs))
    for i, (w, h) in enumerate(shapes):
        preds4 = [pred[k * ps * rows:] for k in range(4)]
        assert list(got[i]) == list(orc.satd_any_size_quad(w, h, preds4, ps, orig, os_)), (w, h)


def test_bipred_and_pixel_var(cuda_lib, orc):
    import torch
    kb = cuda_lib
    r = cs.rng(1400)
    for (w, h) in [(8, 8), (16, 8), (64, 64), (8, 32)]:
        px = [cs.rand_pix(r, w * h) for _ in range(2)]
        im = [r.integers(-2000, 18000, w * h).astype(np.int16) for _ in range(2)]
        for f0 in (0, 1):
            for f1 in (0, 1):
                dst = torch.zeros(64 * 64, dtype=torch.uint8, device="cuda")
                kb.bipred_average_plane(dst, 64, dev(kb, im[0] if f0 else px[0]), dev(kb, im[1] if f1 else px[1]), f0, f1, w, h)
                want = orc.bipred_average_plane(im[0] if f0 else px[0], im[1] if f1 else px[1], f0, f1, w, h, 64)
                assert np.array_equal(host(dst)[: h * 64].reshape(h, 64)[:, :w], want[: h * 64].reshape(h, 64)[:, :w])
    bufs = np.concatenate([cs.rand_pix(r, 4096, kind=k) for k in cs.KINDS])
    got = host(kb.pixel_var_batch(dev(kb, bufs), 4096, 3))
    for i in range(3):
        assert got[i] == orc.pixel_var(cs.al(bufs[i * 4096:(i + 1) * 4096]))      # exact: same summation order


# --------------------------------------------------------------------------- dct group
@pytest.mark.parametrize("n", (4, 8, 16, 32))
def test_transform_batch(cuda_lib, orc, n):
    kb = cuda_lib
    r = cs.rng(2000 + n)
    kinds = ["residual", "full", "sparse", "small"]
    count = 41
    blocks = [cs.dct_test_buf()[: n * n]] + [cs.rand_coeffs(r, n * n, kinds[i % 4]) for i in range(count - 1)]
    x = np.concatenate(blocks)
    for kind, fn in ((kb.TR_DCT, orc.dct), (kb.TR_IDCT, orc.idct)):
        got = host(kb.transform_batch(kind, n, 8, dev(kb, x), count))
        for i in range(count):
            assert np.array_equal(got[i * n * n:(i + 1) * n * n], fn(n, 8, blocks[i])), (n, kind, i)
    if n == 4:
        for kind, fn in ((kb.TR_DST, orc.dst4), (kb.TR_IDST, orc.idst4)):
            got = host(kb.transform_batch(kind, 4, 8, dev(kb, x), count))
            for i in range(count):
                assert np.array_equal(got[i * 16:(i + 1) * 16], fn(8, blocks[i])), (kind, i)


# --------------------------------------------------------------------------- quant group
@pytest.mark.parametrize("signhide", (0, 1))
@pytest.mark.parametrize("qp", (17, 22, 27, 32, 51))
def test_quant_dequant_batch(cuda_lib, orc, qp, signhide):
    kb = cuda_lib
    r = cs.rng(3000 + qp)
    for n in (4, 8, 16, 32):
        kinds = ["residual", "full", "sparse", "small"]
        count = 24
        blocks = []
        for i in range(count):
            c = cs.rand_coeffs(r, n * n, kinds[i % 4])
            blocks.append(orc.dct(n, 8, c) if kinds[i % 4] == "residual" else c)
        x = dev(kb, np.concatenate(blocks))
        scans = (np.arange(count) % 3).astype(np.int8)
        for intra in (0, 1):
            for type_ in ((0, 2) if n < 32 else (0,)):
                prm = kb.quant_params(qp, 8, intra, signhide)
                q = host(kb.quant_batch(prm, x, n, type_, dev(kb, scans), count))
                for i in range(count):
                    want = orc.quant(qp, blocks[i], n, n, type_, int(scans[i]), 1, intra, signhide)
                    assert np.array_equal(q[i * n * n:(i + 1) * n * n], want), (n, i, intra, type_)
        for dq_type in ((0, 2, 3) if n < 32 else (0,)):
            dq = host(kb.dequant_batch(kb.quant_params(qp), dev(kb, q), n, dq_type, count))
            for i in range(count):
                assert np.array_equal(dq[i * n * n:(i + 1) * n * n], orc.dequant(qp, q[i * n * n:(i + 1) * n * n], n, n, dq_type, 1))


@pytest.mark.parametrize("qp", (22, 27, 37))
def test_quantize_residual_batch(cuda_lib, orc, qp):
    import torch
    kb = cuda_lib
    r = cs.rng(4000 + qp)
    stride, rows = 256, 64
    for signhide in (0, 1):
        src = cs.rand_pix(r, stride * rows, kind="uniform")
        pred = np.clip(src.astype(int) + r.integers(-20, 21, src.size), 0, 255).astype(np.uint8)
        pred[: stride * 8] = cs.rand_pix(r, stride * 8, kind="extreme")
        tus, n_coeff = [], 0
        for n in (4, 8, 16, 32):
            for k in range(12):
                y, x = int(r.integers(0, rows - n + 1)), int(r.integers(0, (stride - n) // 32)) * 32 + (k % 2) * 0
                color = k % 3 if n < 32 else 0
                tus.append((y * stride + x, y * stride + x, (len(tus) % 2) * 0 + y * stride + x, n_coeff, n, color,
                            k % 3, 1 if (n == 4 and k % 4 == 3) else 0, (k // 2) % 2, 0, 0, 0))
                n_coeff += n * n
        # make TU footprints in rec disjoint: give every TU its own 32-wide column band / row band
        tus_arr = np.zeros(len(tus), kb.TU)
        for i, t in enumerate(tus):
            tus_arr[i] = t
            tus_arr[i]["off_rec"] = (i // 8) * 32 * 512 + (i % 8) * 32
        rec = torch.zeros(512 * 32 * (len(tus) // 8 + 1), dtype=torch.uint8, device="cuda")
        coeff = torch.zeros(n_coeff, dtype=torch.int16, device="cuda")
        prm = kb.quant_params(qp, 8, 1, signhide)
        has = host(kb.quantize_residual_batch(prm, dev(kb, src), dev(kb, pred), stride, rec, 512, coeff, tus_arr))
        rec_h, coeff_h = host(rec), host(coeff)
        for i, t in enumerate(tus_arr):
            n = int(t["width"])
            o = orc.quantize_residual(qp, n, int(t["color"]), int(t["scan_idx"]), int(t["use_trskip"]), int(t["cu_is_intra"]),
                                      stride, src[t["off_ref"]:], pred[t["off_pred"]:], 1, signhide)
            assert has[i] == o[0], i
            assert np.array_equal(coeff_h[t["off_coeff"]: t["off_coeff"] + n * n], o[2]), (i, n)
            got_rec = rec_h[t["off_rec"]:][: n * 512].reshape(n, 512)[:, :n] if n * 512 <= rec_h.size - t["off_rec"] else None
            want_rec = o[1].reshape(n, stride)[:, :n]
            rr = np.stack([rec_h[t["off_rec"] + y * 512: t["off_rec"] + y * 512 + n] for y in range(n)])
            assert np.array_equal(rr, want_rec), (i, n)


def test_coeff_helpers_batch(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(5000)
    data, expected = cs.coeff_sum_case()
    assert int(kb.coeff_abs_sum_batch(dev(kb, data), 4096, 1)[0]) == expected     # tests/coeff_sum_tests.c:51-54
    for n in (4, 8, 16, 32):
        blocks = [cs.rand_coeffs(r, n * n, k) for k in ("full", "sparse", "small")]
        x = dev(kb, np.concatenate(blocks))
        w = int(r.integers(0, 2 ** 63))
        s = host(kb.coeff_abs_sum_batch(x, n * n, 3))
        c = host(kb.fast_coeff_cost_batch(x, n, w, 3))
        for i in range(3):
            assert s[i] == orc.coeff_abs_sum(blocks[i])
            assert c[i] / 256.0 == orc.fast_coeff_cost(blocks[i], n, w)


# --------------------------------------------------------------------------- intra group
@pytest.mark.parametrize("log2w", (2, 3, 4, 5))
def test_intra_predict_batch(cuda_lib, orc, log2w):
    kb = cuda_lib
    r = cs.rng(6000 + log2w)
    n = 2 * (1 << log2w) + 1
    ww = 1 << (2 * log2w)
    refs = [cs.rand_refs(r, log2w, kind=cs.KINDS[i % 3]) for i in range(6)]
    count = 6 * 35
    top = np.concatenate([refs[i // 35][0] for i in range(count)])
    left = np.concatenate([refs[i // 35][1] for i in range(count)])
    modes = (np.arange(count) % 35).astype(np.int8)
    dt, dl, dm = dev(kb, top), dev(kb, left), dev(kb, modes)
    raw = host(kb.intra_predict_batch(0, log2w, 0, 0, dt, dl, dm, count))
    for i in range(count):
        t, l, m = refs[i // 35][0], refs[i // 35][1], int(modes[i])
        want = orc.planar(log2w, t, l) if m == 0 else (orc.filtered_dc(log2w, t, l) if m == 1 else orc.angular(log2w, m, t, l))
        assert np.array_equal(raw[i * ww:(i + 1) * ww], want), (log2w, m)
    for color in (0, 1):
        for fb in (0, 1):
            full = host(kb.intra_predict_batch(1, log2w, color, fb, dt, dl, dm, count))
            for i in range(count):
                t, l, m = refs[i // 35][0], refs[i // 35][1], int(modes[i])
                assert np.array_equal(full[i * ww:(i + 1) * ww], orc.intra_predict(log2w, m, color, t, l, fb)), (log2w, m, color, fb)
    assert n  # silence


def test_intra_build_reference_batch(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(7000)
    pic_w, pic_h = 200, 136
    planes = {0: cs.rand_pix(r, pic_w * pic_h), 1: cs.rand_pix(r, pic_w * pic_h // 4)}
    for log2w in (2, 3, 4, 5):
        w = 1 << log2w
        for color in (0, 1):
            step = w << (1 if color else 0)
            stride = pic_w >> (1 if color else 0)
            xy = [(lx, ly) for ly in range(0, pic_h - step + 1, step) for lx in range(0, pic_w - step + 1, step)]
            top, left = kb.intra_build_reference_batch(log2w, color, dev(kb, planes[color]), stride, pic_w, pic_h, xy)
            top, left = host(top), host(left)
            for i, (lx, ly) in enumerate(xy):
                o = orc.intra_build_reference(log2w, color, lx, ly, pic_w, pic_h, planes[color], stride)
                assert np.array_equal(top[i], o[0]) and np.array_equal(left[i], o[1]), (log2w, color, lx, ly)


@pytest.mark.parametrize("log2w", (2, 3, 4, 5))
def test_intra_rough_search_frame(cuda_lib, orc, log2w):
    """Fused refs -> 35 predictions -> SATD; equals build_reference + intra_predict + satd_NxN of the oracle."""
    kb = cuda_lib
    r = cs.rng(8000 + log2w)
    pic_w, pic_h = 136, 72
    src = cs.rand_pix(r, pic_w * pic_h, kind="smooth")
    rec = np.clip(src.astype(int) + r.integers(-6, 7, src.size), 0, 255).astype(np.uint8)
    costs = host(kb.intra_rough_search_frame(log2w, dev(kb, src), dev(kb, rec), pic_w, pic_w, pic_h))
    w = 1 << log2w
    bx, by = pic_w // w, pic_h // w
    assert costs.shape == (bx * by, 35)
    for j in range(by):
        for i in range(bx):
            x0, y0 = i * w, j * w
            top, left = orc.intra_build_reference(log2w, 0, x0, y0, pic_w, pic_h, rec, pic_w)
            blk = cs.al(np.ascontiguousarray(src.reshape(pic_h, pic_w)[y0:y0 + w, x0:x0 + w]).ravel())
            for mode in range(35):
                pred = cs.al(orc.intra_predict(log2w, mode, 0, top, left, 1))
                assert costs[j * bx + i, mode] == orc.satd_nxn(w, pred, blk), (log2w, i, j, mode)


# --------------------------------------------------------------------------- ipol group
def test_sample_batch(cuda_lib, orc):
    import torch
    kb = cuda_lib
    r = cs.rng(9000)
    stride, rows = 160, 120
    src = cs.rand_pix(r, stride * rows)
    src[: stride * 40] = cs.rand_pix(r, stride * 40, kind="extreme")
    shapes = [(4, 4), (8, 4), (8, 8), (16, 12), (24, 32), (32, 32), (64, 64), (48, 64), (16, 64)]
    for kind, name in ((kb.IPOL_LUMA, "luma"), (kb.IPOL_LUMA_HI, "luma_hi"), (kb.IPOL_CHROMA, "chroma"), (kb.IPOL_CHROMA_HI, "chroma_hi")):
        chroma = kind >= kb.IPOL_CHROMA
        descs, off = [], 0
        for (w, h) in shapes:
            if chroma and (w > 32 or h > 32):
                continue
            for _ in range(4):
                y, x = int(r.integers(8, rows - 8 - h)), int(r.integers(8, stride - 8 - w))
                descs.append((y * stride + x, off, w, h, int(r.integers(0, 8)), int(r.integers(0, 8))))
                off += w * h + (-(w * h)) % 8
        d = np.array(descs, kb.IPOL)
        hi = kind & 1
        dst = torch.zeros(off, dtype=torch.int16 if hi else torch.uint8, device="cuda")
        # each block is written with dst_stride = its own width: launch per distinct width
        for w in sorted(set(int(x) for x in d["w"])):
            kb.sample_batch(kind, dev(kb, src), stride, dst, w, d[d["w"] == w])
        out = host(dst)
        for t in d:
            w, h = int(t["w"]), int(t["h"])
            want = orc.sample(name, src, int(t["off_src"]), stride, w, h, int(t["mvx"]), int(t["mvy"]))
            assert np.array_equal(out[t["off_dst"]: t["off_dst"] + w * h], want), (name, w, h, int(t["mvx"]), int(t["mvy"]))


def test_filter_fme_batch(cuda_lib, orc):
    import torch
    kb = cuda_lib
    r = cs.rng(9100)
    stride, rows = 128, 100
    src = cs.rand_pix(r, stride * rows)
    src[: stride * 50] = cs.rand_pix(r, stride * 50, kind="extreme")
    for (w, h) in [(8, 8), (16, 16), (16, 8), (32, 32), (64, 64), (8, 16), (24, 32)]:
        offs = [(ox, oy) for ox in (-1, 0, 1) for oy in (-1, 0, 1)]
        count = len(offs)
        src_off = [int(r.integers(8, rows - 8 - h - 1)) * stride + int(r.integers(8, stride - 8 - w - 1)) for _ in range(count)]
        filt = torch.zeros(count * 4 * 4096, dtype=torch.uint8, device="cuda")
        im = torch.zeros(count * 5 * kb.IPOL_IM_SIZE, dtype=torch.int16, device="cuda")
        cols = torch.zeros(count * 5 * kb.IPOL_FIRST_COLS, dtype=torch.int16, device="cuda")
        states = [orc.fme_state() for _ in range(count)]
        dsrc = dev(kb, src)
        for stage in range(4):
            kb.filter_fme_batch(stage, dsrc, stride, src_off, w, h, filt, im, 2, cols, np.array(offs, np.int8))
            f = host(filt).reshape(count, 4, 64, 64)
            imh = host(im).reshape(count, 5, kb.IPOL_IM_SIZE)
            ch = host(cols).reshape(count, 5, kb.IPOL_FIRST_COLS)
            for b in range(count):
                orc.filter_fme(stage, src, src_off[b], stride, w, h, states[b], 2, offs[b][0], offs[b][1])
                want = states[b][0].reshape(4, 64, 64)
                assert np.array_equal(f[b][:, :h, :w], want[:, :h, :w]), (w, h, stage, offs[b])
                wim = states[b][1].reshape(5, -1)
                for k in ((0, 1) if stage < 2 else (0, 1, 3, 4)):
                    assert np.array_equal(imh[b, k, : (h + 8) * 64].reshape(-1, 64)[:, :w], wim[k, : (h + 8) * 64].reshape(-1, 64)[:, :w])
                wc = states[b][2].reshape(5, -1)
                for k in ((0, 2) if stage < 2 else (0, 1, 2, 3)):
                    assert np.array_equal(ch[b, k, : h + 8], wc[k, : h + 8]), (w, h, stage, k)


def test_extend_block(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(9200)
    sw, sh, ss = 80, 48, 88
    src = cs.rand_pix(r, ss * sh)
    for (bx, by) in [(-6, 4), (70, 10), (20, -5), (20, 44), (-10, -10), (76, 46), (-40, 8), (100, 60)]:
        for (bw, bh) in [(8, 8), (16, 4), (32, 16)]:
            for pads in [(3, 4, 3, 4, 0), (3, 4, 3, 4, 1), (1, 2, 1, 2, 3)]:
                o = orc.get_extended_block(src, sw, sh, ss, bx, by, bw, bh, *pads)
                if not o[0]:
                    continue      # block + padding inside the frame: the reference returns a pointer, no copy
                got = host(kb.extend_block(dev(kb, src), sw, sh, ss, bx, by, bw, bh, *pads))
                assert np.array_equal(got, o[1][: got.size]), (bx, by, bw, bh, pads)


# --------------------------------------------------------------------------- sao group
def test_sao_batches(cuda_lib, orc):
    import torch
    kb = cuda_lib
    r = cs.rng(10000)
    shapes = [(64, 64), (32, 32), (56, 64), (64, 24), (8, 8), (16, 40)] * 3
    blks = np.zeros(len(shapes), kb.SAO_BLK)
    origs, recs, off = [], [], 0
    for i, (bw, bh) in enumerate(shapes):
        o = cs.rand_pix(r, bw * bh, kind=cs.KINDS[i % 3])
        rc = np.clip(o.astype(int) + r.integers(-3, 4, bw * bh), 0, 255).astype(np.uint8)
        origs.append(o); recs.append(rc)
        blks[i] = (off, off, bw, bh, 0, 0)
        off += bw * bh
    do, dr = dev(kb, np.concatenate(origs)), dev(kb, np.concatenate(recs))
    stats = host(kb.sao_edge_stats_batch(8, do, dr, blks))
    for i, (bw, bh) in enumerate(shapes):
        for eo in range(4):
            assert np.array_equal(stats[i, eo].ravel(), orc.calc_sao_edge_dir(8, origs[i], recs[i], eo, bw, bh)), (i, eo)
    eo_cls = (np.arange(len(shapes)) % 4).astype(np.int8)
    offsets = r.integers(-7, 8, (len(shapes), 5)).astype(np.int32)
    offsets[::3, 0] = 0
    dd = host(kb.sao_edge_ddistortion_batch(8, do, dr, blks, eo_cls, offsets))
    band_pos = r.integers(0, 32, len(shapes)).astype(np.int32)
    bands = r.integers(-7, 8, (len(shapes), 4)).astype(np.int32)
    bd = host(kb.sao_band_ddistortion_batch(8, do, dr, blks, band_pos, bands))
    for i, (bw, bh) in enumerate(shapes):
        assert dd[i] == orc.sao_edge_ddistortion(8, origs[i], recs[i], bw, bh, int(eo_cls[i]), offsets[i]), i
        assert bd[i] == orc.sao_band_ddistortion(8, origs[i], recs[i], bw, bh, int(band_pos[i]), bands[i]), i
    # reconstruct
    stride, new_stride, rows = 200, 136, 70
    rec = cs.rand_pix(r, stride * rows)
    descs = np.zeros(30, kb.SAO_REC)
    placed = []
    for i in range(len(descs)):
        bw, bh = [(64, 64), (32, 20), (10, 54), (54, 10), (1, 1), (3, 64)][i % 6]
        y, x = 1 + (i % 3), 1 + int(r.integers(0, stride - bw - 2))
        descs[i]["off_rec"] = y * stride + x
        descs[i]["off_new"] = (i * 70) * new_stride
        descs[i]["bw"], descs[i]["bh"] = bw, bh
        descs[i]["type"] = [2, 1, 2, 0, 1][i % 5]
        descs[i]["eo_class"] = i % 4
        descs[i]["color"] = i % 3
        descs[i]["band_position"] = [int(r.integers(0, 32)), int(r.integers(0, 32))]
        descs[i]["offsets"] = r.integers(-7, 8, 10)
        placed.append((bw, bh))
    new = torch.zeros(30 * 70 * new_stride, dtype=torch.uint8, device="cuda")
    kb.sao_reconstruct_batch(8, dev(kb, rec), stride, new, new_stride, descs)
    out = host(new)
    for i, d in enumerate(descs):
        bw, bh = placed[i]
        got = out[d["off_new"]:][: bh * new_stride].reshape(bh, new_stride)[:, :bw]
        if d["type"] == 0:
            want = np.stack([rec[d["off_rec"] + y * stride: d["off_rec"] + y * stride + bw] for y in range(bh)])
        else:
            want = orc.sao_reconstruct_color(8, rec, int(d["off_rec"]), int(d["type"]), int(d["eo_class"]), d["band_position"],
                                             d["offsets"], stride, new_stride, bw, bh, int(d["color"])).reshape(bh, new_stride)[:, :bw]
        assert np.array_equal(got, want), (i, bw, bh, int(d["type"]))


# --------------------------------------------------------------------------- nal group
def test_array_checksum(cuda_lib, orc):
    kb = cuda_lib
    r = cs.rng(11000)
    for (w, h, stride) in [(64, 64, 64), (1920, 8, 1920), (3, 5, 3), (520, 300, 520), (960, 540, 1024), (3840, 2160, 3840)]:
        data = cs.rand_pix(r, stride * h)
        got = host(kb.array_checksum(dev(kb, data), h, w, stride))
        assert np.array_equal(got, orc.array_checksum(data, h, w, stride)), (w, h)


# --------------------------------------------------------------------------- size-independent properties at full size
def test_full_frame_properties_2160p(cuda_lib):
    """At BASELINE sizes the oracle is too slow; check properties instead: SATD/SAD of identical planes is 0,
    SAD is symmetric, the checksum is linear in a per-pixel byte toggle, DCT->IDCT of small residuals round-trips."""
    import torch
    kb = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(5)
    w, h = 3840, 2160
    a = torch.randint(0, 256, (h * w,), dtype=torch.uint8, device="cuda", generator=g)
    b = torch.randint(0, 256, (h * w,), dtype=torch.uint8, device="cuda", generator=g)
    count = h * w // 64
    assert int(kb.satd_nxn_batch(8, a, a, count).abs().sum()) == 0
    s1, s2 = kb.sad_nxn_batch(8, a, b, count), kb.sad_nxn_batch(8, b, a, count)
    assert torch.equal(s1, s2)
    total = int(s1.to(torch.int64).sum())
    assert total == int((a.to(torch.int16) - b.to(torch.int16)).abs().to(torch.int64).sum())
    # SATD >= |DC difference| / ... : weaker but size independent: satd(a,b) == satd(b,a)
    assert torch.equal(kb.satd_nxn_batch(8, a, b, count), kb.satd_nxn_batch(8, b, a, count))
    c0 = kb.array_checksum(a, h, w, w).cpu().numpy()
    a2 = a.clone()
    a2[123456] ^= 0xFF
    c1 = kb.array_checksum(a2, h, w, w).cpu().numpy()
    v0, v1 = int.from_bytes(bytes(c0), "big"), int.from_bytes(bytes(c1), "big")
    x, y = 123456 % w, 123456 // w
    mask = ((x & 0xff) ^ (y & 0xff) ^ (x >> 8) ^ (y >> 8)) & 0xff
    old = int(a[123456]) ^ mask
    new = (int(a[123456]) ^ 0xFF) ^ mask
    assert (v1 - v0) % (1 << 32) == (new - old) % (1 << 32)
    res = torch.randint(-255, 256, (count * 64,), dtype=torch.int16, device="cuda", generator=g)
    coef = kb.transform_batch(kb.TR_DCT, 8, 8, res, count)
    back = kb.transform_batch(kb.TR_IDCT, 8, 8, coef, count)
    assert int((back.to(torch.int32) - res.to(torch.int32)).abs().max()) <= 2
