"""GPU: the whole Depth-Anything band path (prisma_depth_infer through the C ABI) vs the reference fixtures and the
CPU oracle.  Tolerance (north_star): depth floats within 1e-3 relative -- asserted as max|d| <= 1e-3 * max|ref| and
relative L2 <= 1e-3; the u8 frame may differ by the propagated float error only."""
import os

import numpy as np
import pytest
import torch

from oracle import da as oda
from prisma_b200.synthetic import synthetic_frame
from prisma_b200.seeded_weights import make_da_weights

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max()), float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def vits_engine():
    from prisma_b200.depth import DepthAnythingEngine
    eng = DepthAnythingEngine("vits", make_da_weights("vits", 0))
    yield eng
    eng.close()


@pytest.mark.parametrize("tag", ["vits_160x208", "vits_480x640"])
def test_depth_band_matches_reference_fixture(golden_dir, vits_engine, tag):
    g = np.load(os.path.join(golden_dir, f"da_{tag}.npz"))
    H, W = [int(v) for v in g["frame_hw"]]
    img = synthetic_frame(H, W, int(g["frame_index"]))
    rgb, dmin, dmax, pred = vits_engine.infer_encoded(img, want_depth=True)
    wn, hn = oda.da_get_size(W, H)
    T, D = 1 + (hn // 14) * (wn // 14), 384
    report = {}
    net = vits_engine.read_tap("net_input", (3, hn, wn))
    report["net_input"] = float(np.abs(net[:, ::4, ::4] - g["net_input_s4"]).max())
    feat3 = vits_engine.read_tap("feat3", (T - 1, D))  # patch tokens (cls dropped)
    report["feat3"] = _rel(feat3[::7], g["feat3_s7"])
    depth = vits_engine.read_tap("net_depth", (hn, wn))
    report["net_depth"] = _rel(depth[::2, ::2], g["depth_s2"])
    report["prediction"] = _rel(pred, g["prediction"])
    report["minmax"] = (abs(dmin - float(g["dmin"])) / float(g["dmax"]), abs(dmax - float(g["dmax"])) / float(g["dmax"]))
    report["rgb_max_lsb"] = int(np.abs(rgb.astype(int) - g["rgb"].astype(int)).max())
    report["rgb_mean_lsb"] = float(np.abs(rgb.astype(int) - g["rgb"].astype(int)).mean())
    print(tag, report)
    assert report["net_input"] <= 5e-7 * 3
    assert report["feat3"][0] <= 5e-3 and report["feat3"][1] <= 2e-3   # intermediate tokens (fp16 operands)
    assert report["net_depth"][0] <= TOL and report["net_depth"][1] <= TOL
    assert report["prediction"][0] <= TOL and report["prediction"][1] <= TOL
    assert max(report["minmax"]) <= TOL
    # the u8 heat frame (what the band writes into <band>.mp4) against the REFERENCE's frame.  heat_to_rgb has slope
    # 6 * 0.65 per unit of normalised depth (encode.py:13-33), so an error e of the normalised depth moves a channel by at
    # most 255 * 3.9 * e before the truncating cast: the frame may differ by the propagated float error only (the seeded weights span
    # only 0.236..0.280 of depth, so a 1e-3 normalised-depth error is a few LSB at most).
    span = float(g["dmax"]) - float(g["dmin"])
    e_norm = (float(np.abs(pred - g["prediction"]).max()) + 2 * max(report["minmax"]) * float(g["dmax"])) / span
    lsb_bound = int(np.ceil(255 * 3.9 * e_norm)) + 1
    assert report["rgb_max_lsb"] <= min(lsb_bound, 3), (report["rgb_max_lsb"], lsb_bound)
    assert report["rgb_mean_lsb"] <= 0.15, report["rgb_mean_lsb"]


def test_depth_band_matches_oracle_720p(vits_engine):
    """BASELINE config-2 frame size (720p) with the ViT-S weights: CUDA vs the CPU oracle on the same frame."""
    img = synthetic_frame(720, 1280, 5)
    pred = vits_engine.infer(img)
    sd = make_da_weights("vits", 0)
    ref = oda.da_infer(sd, img, "vits")
    m, l2 = _rel(pred, ref)
    print("720p vits: max-rel %.3e  rel-L2 %.3e" % (m, l2))
    assert m <= TOL and l2 <= TOL
    # determinism / idempotence: the same frame twice gives identical bits
    assert np.array_equal(pred, vits_engine.infer(img))


def test_batch_equals_single_frames(vits_engine):
    """prisma_depth_infer_batch(n frames) == n x prisma_depth_infer: frame sharding / batching invariance."""
    frames = [synthetic_frame(240, 320, t) for t in range(3)]
    rgb_b, mins_b, maxs_b, pred_b = vits_engine.infer_batch(frames, want_depth=True)
    for i, f in enumerate(frames):
        rgb, dmin, dmax, pred = vits_engine.infer_encoded(f, want_depth=True)
        assert np.array_equal(pred, pred_b[i]) and np.array_equal(rgb, rgb_b[i])
        assert np.float32(dmin) == mins_b[i] and np.float32(dmax) == maxs_b[i]


def test_streamed_clip_equals_single_frames(vits_engine):
    """prisma_depth_infer_stream (overlapped copies, ragged last pass, pinned and pageable buffers) == per-frame calls."""
    from prisma_b200.depth import pinned_empty
    frames = np.stack([synthetic_frame(240, 320, t) for t in range(7)])
    single = [vits_engine.infer_encoded(f, want_depth=True) for f in frames]
    pin_in = pinned_empty(frames.shape, np.uint8)
    pin_in[...] = frames
    pin_rgb = pinned_empty(frames.shape, np.uint8)
    for src, out_rgb, pf in ((frames, None, 2), (pin_in, pin_rgb, 3), (pin_in, None, 4)):
        rgb, mins, maxs, pred = vits_engine.infer_clip(src, pass_frames=pf, want_depth=True, out_rgb=out_rgb)
        for i, (r1, mn, mx, p1) in enumerate(single):
            assert np.array_equal(rgb[i], r1) and np.array_equal(pred[i], p1), (pf, i)
            assert np.float32(mn) == mins[i] and np.float32(mx) == maxs[i]


def test_still_image_path_matches_video_path_and_png_oracle(vits_engine):
    """process_image (bands/depth_anything.py:146-174): prisma_depth_infer_image = the same prediction as the video path,
    encoded with write_depth's PNG variant (bit-exact against the pinned oracle on the engine's own prediction)."""
    img = synthetic_frame(240, 320, 3)
    png, dmin, dmax, pred = vits_engine.infer_image(img, want_depth=True)
    assert np.array_equal(pred, vits_engine.infer(img))
    ref_png, rmin, rmax = oda.da_write_depth_rgb(pred, True)
    assert np.array_equal(png, ref_png)
    assert np.float32(dmin) == np.float32(pred.min()) and np.float32(dmax) == np.float32(pred.max())


def test_depth_vitl_720p_matches_oracle():
    """The bench configuration itself (BASELINE configs[1]): ViT-L on a 720p frame, CUDA vs the pinned oracle."""
    from prisma_b200.depth import DepthAnythingEngine
    sd = make_da_weights("vitl", 0)
    eng = DepthAnythingEngine("vitl", sd)
    img = synthetic_frame(720, 1280, 5)
    pred = eng.infer(img)
    eng.close()
    ref = oda.da_infer(sd, img, "vitl")
    err = float(np.abs(pred - ref).max() / np.abs(ref).max())
    l2 = float(np.linalg.norm(pred - ref) / np.linalg.norm(ref))
    assert err < 1e-3 and l2 < 1e-3, (err, l2)


def test_depth_vitl_1080p_matches_oracle():
    """BASELINE metric frame size (1080p, the bench headline): ViT-L end to end, CUDA vs the pinned oracle, floats and
    the encoded u8 frame (same propagated-error bound as the fixture test)."""
    from prisma_b200.depth import DepthAnythingEngine
    sd = make_da_weights("vitl", 0)
    eng = DepthAnythingEngine("vitl", sd)
    img = synthetic_frame(1080, 1920, 7)
    rgb, dmin, dmax, pred = eng.infer_encoded(img, want_depth=True)
    eng.close()
    ref = oda.da_infer(sd, img, "vitl")
    err = float(np.abs(pred - ref).max() / np.abs(ref).max())
    l2 = float(np.linalg.norm(pred - ref) / np.linalg.norm(ref))
    ref_rgb, rmin, rmax = oda.da_encode(ref)
    lsb = np.abs(rgb.astype(int) - ref_rgb.astype(int))
    e_norm = (float(np.abs(pred - ref).max()) + abs(dmin - rmin) + abs(dmax - rmax)) / (rmax - rmin)
    print("1080p vitl: max-rel %.3e rel-L2 %.3e; u8 frame max %d LSB mean %.3f LSB (bound %d)" %
          (err, l2, lsb.max(), lsb.mean(), int(np.ceil(255 * 3.9 * e_norm)) + 1))
    assert err < 1e-3 and l2 < 1e-3, (err, l2)
    assert abs(dmin - rmin) <= 1e-3 * abs(rmax) and abs(dmax - rmax) <= 1e-3 * abs(rmax)
    assert lsb.max() <= int(np.ceil(255 * 3.9 * e_norm)) + 1 and lsb.mean() <= 0.25, (lsb.max(), lsb.mean())
