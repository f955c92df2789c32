"""depth_midas --model midas3-small: the DPT_Large network behind the hub's small_transform (fit inside 256 x 256), against
oracle/midas_small.py (oracle/midas.py's network behind the 256-pixel transform).  Same taps and tolerances as
tests/test_midas_gpu.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import midas as om
from oracle import midas_small as oms
from prisma_b200.synthetic import synthetic_frame
from prisma_b200.seeded_weights import make_midas_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_midas_small_size_arithmetic():
    # small_transform: Resize(256, 256, keep AR, x32, "upper_bound"); np.round(4.5) == 4 for the 1080p height
    assert om.midas_get_size(640, 480, target=256) == (256, 192)
    assert om.midas_get_size(1920, 1080, target=256) == (256, 128) and om.midas_get_size(1280, 720, target=256) == (256, 128)
    assert om.midas_get_size(480, 640, target=256) == (192, 256) and om.midas_get_size(320, 240, target=256) == (256, 192)
    assert om.midas_get_size(200, 360, target=256) == (128, 256)
    img = synthetic_frame(48, 64, 0)
    assert oms.midas_small_preprocess(img).shape == (3, 192, 256)
    assert np.array_equal(om.midas_preprocess(img), oms.midas_small_preprocess(img, target=384))


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max()), float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def tiny():
    from prisma_b200.depth import MidasEngine
    sd = make_midas_weights("dpt_tiny", 0)
    eng = MidasEngine(sd, variant="dpt_tiny", net_side=256)
    yield eng, sd
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(240, 320), (360, 200)])
def test_midas_small_matches_oracle(tiny, hw):
    eng, sd = tiny
    img = synthetic_frame(hw[0], hw[1], 1)
    pred = eng.infer(img)
    wn, hn = om.midas_get_size(hw[1], hw[0], target=256)
    taps = {}
    x = torch.from_numpy(oms.midas_small_preprocess(img)).unsqueeze(0)
    assert x.shape[-2:] == (hn, wn) and max(hn, wn) == 256
    net_in = eng.read_tap("net_input", (3, hn, wn))
    assert np.array_equal(net_in, x[0].numpy())
    with torch.no_grad():
        ref_net = om.midas_model(sd, x, "dpt_tiny", taps=taps)[0].numpy()
    tok = eng.read_tap("tokens", tuple(taps["tokens"].shape[1:]))
    m, l2 = rel(tok, taps["tokens"][0].numpy())
    assert m < 1e-3 and l2 < 1e-3, ("tokens", m, l2)      # the 24 x 24 position table resized bilinearly to this grid
    net = eng.read_tap("net_depth", (hn, wn))
    m, l2 = rel(net, ref_net)
    assert m < 1e-3 and l2 < 1e-3, ("net_depth", m, l2)
    ref = oms.midas_small_infer(sd, img, "dpt_tiny")
    m, l2 = rel(pred, ref)
    assert m < 1e-3 and l2 < 1e-3, ("prediction", m, l2)


@pytest.mark.gpu
def test_net_side_is_checked():
    from prisma_b200._lib import PrismaError
    from prisma_b200.depth import DepthAnythingEngine, MidasEngine
    with pytest.raises(PrismaError):
        MidasEngine(None, variant="dpt_tiny", net_side=320)
    from prisma_b200._lib import lib
    da = DepthAnythingEngine("vits")
    assert lib().prisma_depth_set_net_side(da._h, 256) < 0          # a Depth-Anything engine has no MiDaS transform
    da.close()
    eng = MidasEngine(make_midas_weights("dpt_tiny", 0), variant="dpt_tiny", net_side=256)
    eng.infer(synthetic_frame(64, 96, 0))
    assert lib().prisma_depth_set_net_side(eng._h, 384) < 0         # only before the first frame
    eng.close()


@pytest.mark.gpu
def test_midas_small_dpt_large_640x480_matches_oracle():
    """One 640x480 frame through the full-size DPT_Large graph behind small_transform (256x192 input, 193 tokens)."""
    from prisma_b200.depth import MidasEngine
    sd = make_midas_weights("dpt_large", 0)
    eng = MidasEngine(sd, net_side=256)
    img = synthetic_frame(480, 640, 0)
    pred = eng.infer(img)
    eng.close()
    ref = oms.midas_small_infer(sd, img, "dpt_large")
    m, l2 = rel(pred, ref)
    assert m < 1e-3 and l2 < 1e-3, (m, l2)


@pytest.mark.gpu
def test_midas_small_band_writes_video_csv_and_metadata(tmp_path):
    import cv2
    folder = tmp_path / "clip"
    folder.mkdir()
    w = cv2.VideoWriter(str(folder / "rgba.mp4"), cv2.VideoWriter_fourcc(*"mp4v"), 24.0, (320, 240))
    for t in range(3):
        w.write(synthetic_frame(240, 320, t)[..., ::-1].copy())
    w.release()
    json.dump({"bands": {"rgba": {"url": "rgba.mp4"}}, "width": 320, "height": 240, "frames": 3, "fps": 24.0},
              open(folder / "metadata.json", "w"))
    rc = subprocess.call([sys.executable, os.path.join(ROOT, "bands", "depth_midas.py"), "-i", str(folder), "-n", "-d",
                          "frames", "--model", "midas3-small", "--seeded-weights"])
    assert rc == 0
    meta = json.load(open(folder / "metadata.json"))
    band = meta["bands"]["depth_midas"]
    assert band["url"] == "depth_midas.mp4" and os.path.getsize(folder / "depth_midas.mp4") > 0
    assert band["values"] == {"min": {"type": "float", "url": "depth_midas_min.csv"},
                              "max": {"type": "float", "url": "depth_midas_max.csv"}}
    mins = [float(l) for l in open(folder / "depth_midas_min.csv")]
    maxs = [float(l) for l in open(folder / "depth_midas_max.csv")]
    assert len(mins) == 3 and all(b > a for a, b in zip(mins, maxs))
    pred = np.load(folder / "frames" / "00000.npy")
    assert pred.shape == (240, 320) and pred.dtype == np.float32 and np.float32(pred.min()) == np.float32(mins[0])
