"""--ply of the depth bands: prisma_depth_point_cloud (flip, 5x5 median, unprojection, 15-byte records) against the
reference's own write_pcl output (tests/golden/pcl_37x53.npz) and the oracle restatement (oracle/pcl.py), bit for bit;
the PLY file layout; the bands' still-image runs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pcl as opcl
from prisma_b200.depth import PLY_VERTEX_DTYPE
from prisma_b200.synthetic import synthetic_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = (b"ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
          b"property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")


def _synthetic_depth(h, w, t):
    """An f32 depth with many ties (u8-derived) and a wide range."""
    f = synthetic_frame(h, w, t)
    return (f[..., 0].astype(np.float32) * np.float32(0.5) + f[..., 2].astype(np.float32) // 16 + np.float32(0.125)).astype(np.float32)


def _records(d, rgb, flip):
    """np.rec.fromarrays(...).astype(dtype).tobytes() of the oracle's x, y, z and the frame's colours."""
    v = opcl.point_cloud(d, rgb, flip)
    c = rgb.reshape(-1, 3)
    return np.rec.fromarrays([v["x"], v["y"], v["z"], c[:, 0], c[:, 1], c[:, 2]],
                             names="x,y,z,red,green,blue").astype(PLY_VERTEX_DTYPE).tobytes()


def test_write_ply_is_header_then_records(tmp_path):
    from bands.common.ply import write_ply
    v = np.zeros(3, PLY_VERTEX_DTYPE)
    v["x"] = [1.5, -2.0, 0.25]
    v["blue"] = [1, 2, 255]
    path = str(tmp_path / "a.ply")
    write_ply(path, v)
    data = open(path, "rb").read()
    assert data == HEADER % 3 + v.tobytes() and len(data) == len(HEADER % 3) + 45
    with pytest.raises(ValueError):
        write_ply(path, np.zeros((3, 4), np.float32))


@pytest.fixture(scope="module")
def eng():
    from prisma_b200.depth import DepthAnythingEngine
    e = DepthAnythingEngine("vits")  # the point cloud needs no weights
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [0, 1])
def test_point_cloud_matches_reference_fixture(eng, golden_dir, flip):
    g = np.load(os.path.join(golden_dir, "pcl_37x53.npz"))
    got = eng.point_cloud(g["depth"], g["rgb"], flip)
    ref = g[f"vertices_flip{flip}"]
    assert got.dtype == PLY_VERTEX_DTYPE and got.tobytes() == ref.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(240, 320), (1080, 1920), (37, 53), (33, 65), (5, 3), (1, 1)])
@pytest.mark.parametrize("flip", [0, 1])
def test_point_cloud_matches_oracle(eng, hw, flip):
    h, w = hw
    d = _synthetic_depth(h, w, 0)
    if h * w == 1:
        d[:] = 2.5
        flip = 0  # one pixel: max == min, and the reference's flip divides by zero
    rgb = synthetic_frame(h, w, 1)
    got = eng.point_cloud(d, rgb, flip)
    assert got.shape == (h * w,) and got.tobytes() == _records(d, rgb, flip)


@pytest.mark.gpu
def test_point_cloud_rejects_mismatched_frame(eng):
    from prisma_b200._lib import PrismaError
    with pytest.raises(PrismaError):
        eng.point_cloud(np.zeros((4, 5), np.float32), np.zeros((4, 6, 3), np.uint8), 1)


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    n = int(data[:end].split(b"element vertex ")[1].split(b"\n")[0])
    assert data[:end] == HEADER % n
    return n, np.frombuffer(data[end:], PLY_VERTEX_DTYPE)


@pytest.mark.gpu
@pytest.mark.parametrize("band,extra,flip", [
    ("depth_anything", ["--encoder", "vits"], 1),
    ("depth_anything", ["--encoder", "vits", "--metric", "indoor"], 0),
    ("depth_midas", [], 1),
])
def test_band_writes_ply_for_a_still_image(tmp_path, band, extra, flip):
    import cv2
    h, w = 96, 128
    img = synthetic_frame(h, w, 0)
    src = str(tmp_path / "frame.png")
    cv2.imwrite(src, img[..., ::-1].copy())
    rc = subprocess.call([sys.executable, os.path.join(ROOT, "bands", band + ".py"), "-i", src, "--seeded-weights", "-p", "-n"]
                         + extra)
    assert rc == 0
    n, v = _read_ply(str(tmp_path / (band + ".ply")))
    assert n == h * w and v.size == h * w
    pred = np.load(str(tmp_path / (band + ".npy")))
    assert pred.shape == (h, w)
    assert v.tobytes() == _records(pred, img, flip)  # the band's own prediction through write_pcl(..., flip)
