"""Pin oracle/pcl.py against the reference's own --ply code and write tests/golden/pcl_37x53.npz (TEST INFRASTRUCTURE).

Runs ONLY where a checkout of the reference is available at REF, like oracle/tools/make_golden.py.  It calls the reference's
write_pcl (bands/common/io.py:201-211 -> common/geom.py) with and without the flip, on an f32 depth with ties (u8-derived
values) and extreme values on the borders.  plyfile is not installed: a stand-in captures the vertex array save_point_cloud
hands to PlyElement.describe, which is exactly what plyfile writes after its header.

    python oracle/tools/make_pcl_golden.py        # from the repository root
"""
import os
import sys
import types

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference"
sys.dont_write_bytecode = True
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REF, "bands"))

import numpy as np  # noqa: E402

from oracle import pcl as opcl  # noqa: E402
from prisma_b200.synthetic import synthetic_frame  # noqa: E402

GOLD = os.path.join(REPO, "tests", "golden")


def _reference_write_pcl():
    """common.io.write_pcl with plyfile replaced by a stand-in that records the vertex array it is given."""
    captured = []
    ply = types.ModuleType("plyfile")
    ply.PlyElement = types.SimpleNamespace(describe=lambda arr, name: (name, arr))

    class PlyData:
        def __init__(self, elements, text=False):
            assert len(elements) == 1 and elements[0][0] == "vertex" and text is False
            self.arr = elements[0][1]

        def write(self, filename):
            captured.append(self.arr)

    ply.PlyData = PlyData
    sys.modules["plyfile"] = ply
    for m in ("av", "decord"):  # container deps of common.io that are not installed
        sys.modules.setdefault(m, types.ModuleType(m))
    import common.io as rio

    def write_pcl(depth, rgb, flip):
        captured.clear()
        rio.write_pcl(os.devnull, depth.copy(), rgb.copy(), flip=bool(flip))
        return captured[0]
    return write_pcl


def golden_pcl(H=37, W=53):
    write_pcl = _reference_write_pcl()
    frame = synthetic_frame(H, W, 0)
    depth = (frame[..., 0].astype(np.float32) * np.float32(0.25) + frame[..., 1].astype(np.float32) // 64 + np.float32(2.0))
    depth[0, :7] = 1.0e4                    # far outliers along the top border and in a corner
    depth[-1, -9:] = 0.0                    # zeros along the bottom border
    depth[5:12, 0] = 3.0e-6                 # tiny values down the left border
    depth[:, -1] = depth[:, -1].max()       # a constant right border: ties across the replicated edge
    depth = depth.astype(np.float32)
    rgb = synthetic_frame(H, W, 1)
    out = {}
    for flip in (0, 1):
        ref = write_pcl(depth, rgb, flip)
        mine = opcl.point_cloud(depth, rgb, flip)
        assert ref.dtype == mine.dtype and ref.tobytes() == mine.tobytes(), flip
        out[f"vertices_flip{flip}"] = ref
    np.savez_compressed(os.path.join(GOLD, f"pcl_{H}x{W}.npz"), depth=depth, rgb=rgb, **out)
    print(f"[pcl] oracle == reference write_pcl (flip 0 and 1, {H}x{W}); wrote fixture")


if __name__ == "__main__":
    golden_pcl()
