"""--ply point cloud: the oracle restatement (oracle/pcl.py) against the reference's own write_pcl output (CPU)."""
import os

import numpy as np

from oracle import pcl as opcl
from prisma_b200.depth import PLY_VERTEX_DTYPE


def _fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "pcl_37x53.npz"))


def test_fixture_covers_ties_and_border_extremes(golden_dir):
    g = _fixture(golden_dir)
    d = g["depth"]
    assert d.dtype == np.float32 and d.shape == (37, 53)
    assert np.unique(d).size < d.size // 4                        # many ties inside every 5x5 window
    assert d[0, 0] == d.max() and d[-1, -2] == d.min() == 0.0      # extremes on the borders, where the window is replicated


def test_oracle_matches_reference_write_pcl(golden_dir):
    g = _fixture(golden_dir)
    for flip in (0, 1):
        ref = g[f"vertices_flip{flip}"]
        got = opcl.point_cloud(g["depth"], g["rgb"], flip)
        assert ref.dtype == PLY_VERTEX_DTYPE and PLY_VERTEX_DTYPE.itemsize == 15
        assert np.array_equal(got, ref) and got.tobytes() == ref.tobytes(), flip


def test_oracle_steps_match_reference_fields(golden_dir):
    """Each step on its own: z = -median(flip(depth)), x and y are that depth times the fixed ray."""
    g = _fixture(golden_dir)
    H, W = g["depth"].shape
    for flip in (0, 1):
        ref = g[f"vertices_flip{flip}"].reshape(H, W)
        d = opcl.pcl_flip(g["depth"]) if flip else g["depth"]
        med = opcl.median5(d)
        assert np.array_equal(-med, ref["z"])
        xyz = opcl.unproject(med)
        assert np.array_equal(xyz[..., 0], ref["x"]) and np.array_equal(xyz[..., 1], ref["y"])
        assert np.array_equal(np.stack([ref["red"], ref["green"], ref["blue"]], -1), g["rgb"])
    # the flip is not the identity on this depth, and it maps the extremes onto each other
    f = opcl.pcl_flip(g["depth"])
    assert not np.array_equal(f, g["depth"]) and f[0, 0] == g["depth"].min() and f[-1, -2] == g["depth"].max()


def test_median_matches_opencv():
    """Independent cross-check of the median restatement on random f32 data with ties (OpenCV is installed here)."""
    import cv2
    rng = np.random.default_rng(0)
    for h, w in ((5, 5), (7, 13), (64, 33)):
        d = (rng.integers(0, 9, (h, w)) * 0.37).astype(np.float32)
        assert np.array_equal(opcl.median5(d), cv2.medianBlur(d, 5))
