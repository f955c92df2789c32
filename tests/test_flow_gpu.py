"""GPU: RAFT band HBM-bound stages through the C ABI vs the reference fixture and the oracle:
K11 pre-process, K13+K14 correlation pyramid, K15 lookup, K20 HSV encode."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import raft as oraft
from prisma_b200.synthetic import synthetic_frame
from prisma_b200._lib import check, fptr, lib, u8ptr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,W", [(240, 320), (482, 854), (270, 481), (720, 1280), (1080, 1920)])
@pytest.mark.parametrize("kind", ["synthetic", "noise"])
def test_raft_preprocess(H, W, kind):
    """K11 against cv2 itself (flow_raft.py:100: cv2.resize(frame, None, fx=0.75, fy=0.75, INTER_CUBIC)), including sizes
    where src*fx is not an integer (the sampling step stays 1/fx; 482x854 differs on 70 % of the bytes if the step is
    re-derived from the rounded output size).  The 8-bit cubic of this OpenCV build is IPP's float pipeline, round half to
    even; the kernel is byte-equal to it except at exact .5 ties of the real-valued result, where IPP's closed, CPU-
    dispatched operation order decides: every differing byte must be such a tie (|exact - (n + .5)| < 1e-4, the float32
    rounding noise of a 16-tap sum of values up to 255), by 1 LSB.  Flat regions make exact ties common on the
    smooth synthetic frames; bound 1e-3 of the bytes.  Padding / normalisation are exact."""
    img = synthetic_frame(H, W, 2) if kind == "synthetic" else np.random.default_rng(H).integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref_rs = oraft.raft_preprocess(img)  # 3 x hs x ws float (0..255), via cv2
    hs, ws = ref_rs.shape[-2:]
    pad = oraft.input_pad(hs, ws)
    hp, wp = hs + pad[2] + pad[3], ws + pad[0] + pad[1]
    rs = np.empty((hs, ws, 3), np.uint8)
    chw = np.empty((3, hp, wp), np.float32)
    check(lib().prisma_flow_preprocess(0, u8ptr(img), H, W, 0.75, u8ptr(rs), fptr(chw)))
    ref_u8 = ref_rs.permute(1, 2, 0).numpy().astype(np.uint8)
    diff = rs != ref_u8
    if diff.any():
        exact = oraft.cubic_resize_f64(img, 0.75)
        tie = np.abs(exact - np.floor(exact) - 0.5)[diff]
        lsb = np.abs(rs.astype(int) - ref_u8.astype(int))[diff]
        assert tie.max() < 1e-4 and lsb.max() == 1, (tie.max(), lsb.max())
    assert diff.mean() <= 1e-3, diff.mean()
    # pad + normalise exactly as the reference does, applied to OUR resized image
    t = torch.from_numpy(rs).permute(2, 0, 1).float()[None]
    exp = 2 * (torch.nn.functional.pad(t, pad, mode="replicate") / 255.0) - 1.0
    assert np.array_equal(chw, exp[0].numpy())


def test_flow_encode_matches_reference(golden_dir):
    """K20 on the reference's own flow: u8 frame within 1 LSB (arctan2 ulp), max displacement bit-exact."""
    g = np.load(os.path.join(golden_dir, "raft_240x320.npz"))
    flow = np.ascontiguousarray(g["flow_fwd"])
    h, w = flow.shape[:2]
    rgb = np.empty((h, w, 3), np.uint8)
    mx = C.c_float()
    check(lib().prisma_flow_encode(0, fptr(flow), h, w, u8ptr(rgb), C.byref(mx)))
    assert np.float32(mx.value) == g["flow_max"]
    d = np.abs(rgb.astype(int) - g["flow_rgb"].astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-3, (d.max(), (d > 0).mean())
    # full 1080p*0.75 size against the oracle, and the zero-flow last frame (reference: NaN -> 0)
    rng = np.random.default_rng(1)
    flow = (rng.standard_normal((810, 1440, 2), dtype=np.float32) * 5).astype(np.float32)
    rgb = np.empty((810, 1440, 3), np.uint8)
    check(lib().prisma_flow_encode(0, fptr(flow), 810, 1440, u8ptr(rgb), C.byref(mx)))
    ref, rmax = oraft.process_flow(flow)
    assert np.float32(mx.value) == np.float32(rmax)
    d = np.abs(rgb.astype(int) - ref.astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-3
    z = np.zeros((8, 8, 2), np.float32)
    rgbz = np.full((8, 8, 3), 7, np.uint8)
    check(lib().prisma_flow_encode(0, fptr(z), 8, 8, u8ptr(rgbz), C.byref(mx)))
    assert mx.value == 0.0 and not rgbz.any()


def _corr(batch, h8, w8):
    h = C.c_void_p()
    check(lib().prisma_flowcorr_create(0, batch, h8, w8, C.byref(h)))
    return h


def test_corr_pyramid_and_lookup_match_reference(golden_dir):
    """K13-K15 vs the reference CorrBlock outputs in the fixture (fp16 features, fp32 accumulation)."""
    g = np.load(os.path.join(golden_dir, "raft_240x320.npz"))
    fm1 = np.ascontiguousarray(g["fmap1"].astype(np.float32))
    fm2 = np.ascontiguousarray(g["fmap2"].astype(np.float32))
    B, Cc, h8, w8 = fm1.shape
    P = h8 * w8
    h = _corr(B, h8, w8)
    l = lib()
    check(l.prisma_flowcorr_set_fmaps(h, fptr(fm1), fptr(fm2)))
    ms = C.c_float()
    check(l.prisma_flowcorr_build(h, 1, C.byref(ms)))
    scale = np.abs(g["corr_l0_rows"]).max()
    l0 = np.empty((64, P), np.float32)
    check(l.prisma_flowcorr_read_level(h, 0, 0, 0, 64, fptr(l0)))
    assert np.abs(l0 - g["corr_l0_rows"].reshape(64, -1)).max() <= 1e-3 * scale
    n3 = (h8 >> 3) * (w8 >> 3)
    l3 = np.empty((64, n3), np.float32)
    check(l.prisma_flowcorr_read_level(h, 3, 0, 0, 64, fptr(l3)))
    assert np.abs(l3 - g["corr_l3_rows"].reshape(64, -1)).max() <= 1e-3 * scale
    # the full pyramid against the oracle (all levels, both images)
    pyr = oraft.corr_pyramid(torch.from_numpy(fm1), torch.from_numpy(fm2))
    for lvl in range(4):
        n = (h8 >> lvl) * (w8 >> lvl)
        for b in range(B):
            got = np.empty((P, n), np.float32)
            check(l.prisma_flowcorr_read_level(h, lvl, b, 0, P, fptr(got)))
            ref = pyr[lvl][b * P:(b + 1) * P, 0].reshape(P, n).numpy()
            assert np.abs(got - ref).max() <= 1e-3 * scale, (lvl, b)
    # lookup at the fixture's coordinates (random offsets up to ~6 px, some outside the volume)
    coords = np.ascontiguousarray(g["coords"])
    out = np.empty((B, 324, h8, w8), np.float32)
    check(l.prisma_flowcorr_lookup(h, fptr(coords), fptr(out), 1, C.byref(ms)))
    ref = g["lookup"].astype(np.float32)
    # both the engine's lookup output (the fp16 A operand of convc1) and the fixture are fp16: 2 x 2^-11 relative
    assert np.abs(out - ref).max() <= 1.5e-3 * np.abs(ref).max()
    # far outside the volume everything is zero (zeros padding)
    far = coords + 1000.0
    check(l.prisma_flowcorr_lookup(h, fptr(np.ascontiguousarray(far)), fptr(out), 1, C.byref(ms)))
    assert not out.any()
    l.prisma_engine_destroy(h)


def test_corr_full_size_properties():
    """BASELINE config-3 size (1080p*0.75 -> 102x180, P = 18360, fwd+bwd): size-independent properties.
    (a) L0 of the backward pair is the transpose of L0 of the forward pair; (b) level l+1 == 2x2 mean of level l;
    (c) a row sum equals <f1[i], sum_j f2[j]> / 16 (checksum against a CPU dot product)."""
    h8, w8, Cc = 102, 180, 256
    P = h8 * w8
    rng = np.random.default_rng(0)
    fa = rng.standard_normal((Cc, h8, w8), dtype=np.float32).astype(np.float16).astype(np.float32)
    fb = rng.standard_normal((Cc, h8, w8), dtype=np.float32).astype(np.float16).astype(np.float32)
    fm1 = np.ascontiguousarray(np.stack([fa, fb]))
    fm2 = np.ascontiguousarray(np.stack([fb, fa]))
    h = _corr(2, h8, w8)
    l = lib()
    check(l.prisma_flowcorr_set_fmaps(h, fptr(fm1), fptr(fm2)))
    ms = C.c_float()
    check(l.prisma_flowcorr_build(h, 3, C.byref(ms)))
    work = (C.c_double * 2)()
    check(l.prisma_flowcorr_work(h, work))
    print("corr build %.3f ms  %.1f GB/s algorithmic  %.1f TFLOP/s" % (ms.value, work[1] / ms.value / 1e6, work[0] / ms.value / 1e9))
    rows = 96
    a = np.empty((rows, P), np.float32)
    check(l.prisma_flowcorr_read_level(h, 0, 0, 0, rows, fptr(a)))
    # (a) transpose symmetry: bwd[j, i] == fwd[i, j] for i < rows -> read all bwd rows, first `rows` columns
    bwd = np.empty((P, P), np.float32)
    check(l.prisma_flowcorr_read_level(h, 0, 1, 0, P, fptr(bwd)))
    assert np.abs(bwd[:, :rows].T - a).max() <= 1e-4 * np.abs(a).max()
    # (b) pyramid linearity
    prev = a.reshape(rows, h8, w8)
    for lvl in range(1, 4):
        hh, ww = h8 >> lvl, w8 >> lvl
        got = np.empty((rows, hh * ww), np.float32)
        check(l.prisma_flowcorr_read_level(h, lvl, 0, 0, rows, fptr(got)))
        pooled = prev[:, :hh * 2, :ww * 2].reshape(rows, hh, 2, ww, 2).mean(axis=(2, 4))
        assert np.abs(got.reshape(rows, hh, ww) - pooled).max() <= 2e-3 * np.abs(a).max(), lvl
        prev = got.reshape(rows, hh, ww)
    # (c) checksum of checksums
    s2 = fb.reshape(Cc, P).astype(np.float64).sum(axis=1)
    ref = (fa.reshape(Cc, P)[:, :rows].astype(np.float64).T @ s2) / 16.0
    assert np.abs(a.astype(np.float64).sum(axis=1) - ref).max() <= 1e-3 * np.abs(ref).max() + 1e-2
    del bwd
    l.prisma_engine_destroy(h)


def test_consistency_masks_and_u16_encode(golden_dir):
    """compute_fwdbwd_mask + encode_flow vs the reference outputs in the fixture (random-weight flows: all-false masks)
    and vs the oracle (cv2.remap) on a synthetic, mostly consistent flow pair where the mask is non-trivial."""
    import ctypes as C
    l = lib()

    def run(fwd, bwd):
        h, w = fwd.shape[:2]
        fm = np.empty((h, w), np.uint8); bm = np.empty((h, w), np.uint8)
        fu = np.empty((h, w, 3), np.uint16); bu = np.empty((h, w, 3), np.uint16)
        check(l.prisma_flow_masks(0, fptr(fwd), fptr(bwd), h, w, u8ptr(fm), u8ptr(bm),
                                  fu.ctypes.data_as(C.POINTER(C.c_uint16)), bu.ctypes.data_as(C.POINTER(C.c_uint16))))
        return fm.astype(bool), bm.astype(bool), fu, bu

    g = np.load(os.path.join(golden_dir, "raft_240x320.npz"))
    fm, bm, fu, bu = run(np.ascontiguousarray(g["flow_fwd"]), np.ascontiguousarray(g["flow_bwd"]))
    assert np.array_equal(fm, g["fwd_mask"]) and np.array_equal(bm, g["bwd_mask"])
    assert np.array_equal(fu, g["flow_u16"])
    # synthetic pair: smooth forward flow, backward = -forward sampled at the target + a disturbance in one corner
    H, W = 540, 960
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    fwd = np.stack([6 * np.sin(yy / 70) + 2.5, 4 * np.cos(xx / 90) - 1.25], -1).astype(np.float32)
    bwd = (-fwd + 0.3 * np.sin(xx / 13)[..., None]).astype(np.float32)
    bwd[:120, :200] += 7.0
    fm, bm, fu, bu = run(fwd, bwd)
    rfm, rbm = oraft.compute_fwdbwd_mask(fwd, bwd)
    assert 0.05 < rfm.mean() < 0.999
    assert (fm != rfm).mean() < 1e-4 and (bm != rbm).mean() < 1e-4   # remap rounding ties only
    assert np.array_equal(fu[..., :2], oraft.encode_flow(fwd.copy(), fm)[..., :2])
    assert np.array_equal(fu, oraft.encode_flow(fwd.copy(), fm))
