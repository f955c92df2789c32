"""CPU oracle: the depth bands' --ply point cloud (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

Restates write_pcl (bands/common/io.py:201-211) -> create_point_cloud (common/geom.py:5-24) -> save_point_cloud's records
(geom.py:27-47) in numpy, without OpenCV or plyfile.  Pinned bit for bit against the reference's own functions by
tests/golden/pcl_37x53.npz (written by oracle/tools/make_pcl_golden.py, tests/test_oracle_pcl_golden.py).
"""
import numpy as np

from prisma_b200.depth import PLY_VERTEX_DTYPE


def pcl_flip(depth):
    """io.py:203-208, float32 throughout: numpy keeps the f32 min / max and the Python 1.0 in f32."""
    d = np.asarray(depth, np.float32)
    mn, mx = d.min(), d.max()
    t = (d - mn) / (mx - mn)
    t = np.float32(1.0) - t
    return mn + t * (mx - mn)


def median5(depth):
    """cv2.medianBlur(depth, 5) on f32: the 13th smallest of each 5x5 window, borders replicated."""
    d = np.asarray(depth, np.float32)
    H, W = d.shape
    p = np.pad(d, 2, mode="edge")
    win = np.stack([p[dy:dy + H, dx:dx + W] for dy in range(5) for dx in range(5)])
    return np.partition(win, 12, axis=0)[12]


def unproject(blurred):
    """create_point_cloud after the blur (geom.py:8-24) with u0 = W/2, v0 = H/2, fx = fy = 1000: f32 (H, W, 3)."""
    H, W = blurred.shape
    u = np.arange(W, dtype=np.float32) - np.float32(W / 2)
    v = np.arange(H, dtype=np.float32) - np.float32(H / 2)
    x = np.broadcast_to(u / np.float32(1000.0), (H, W))
    y = np.broadcast_to((v / np.float32(1000.0))[:, None], (H, W))
    pcl = np.stack([x, -y, -np.ones((H, W), np.float32)], axis=2)
    return blurred[:, :, None] * pcl


def point_cloud(depth, rgb, flip):
    """write_pcl(depth, rgb, flip): the H*W vertex records save_point_cloud writes, as a structured array."""
    d = pcl_flip(depth) if flip else np.asarray(depth, np.float32)
    xyz = unproject(median5(d)).reshape(-1, 3)
    c = np.asarray(rgb, np.uint8).reshape(-1, 3)
    return np.rec.fromarrays([xyz[:, 0], xyz[:, 1], xyz[:, 2], c[:, 0], c[:, 1], c[:, 2]],
                             dtype=PLY_VERTEX_DTYPE).view(np.ndarray).astype(PLY_VERTEX_DTYPE)
