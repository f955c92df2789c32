"""Binary PLY writer for the depth bands' --ply output (the reference's save_point_cloud, bands/common/geom.py:27-47).

The reference writes through `plyfile` (PlyData([PlyElement.describe(vertices, 'vertex')], text=False)), which is not a
dependency here.  The header below is restated from plyfile's format rules for one 'vertex' element of the dtype
(f4 -> "float", u1 -> "uchar", "\\n" line ends, binary_little_endian 1.0, no comments); it is not pinned against plyfile
output.  The body is the records as they are: 15 packed little-endian bytes per vertex.
"""
import numpy as np

from prisma_b200.depth import PLY_VERTEX_DTYPE


def ply_header(n):
    return ("ply\n"
            "format binary_little_endian 1.0\n"
            f"element vertex {n}\n"
            "property float x\n"
            "property float y\n"
            "property float z\n"
            "property uchar red\n"
            "property uchar green\n"
            "property uchar blue\n"
            "end_header\n").encode("ascii")


def write_ply(path, vertices):
    """Write a structured array of PLY_VERTEX_DTYPE (DepthAnythingEngine.point_cloud) as a binary PLY file."""
    v = np.ascontiguousarray(vertices)
    if v.dtype != PLY_VERTEX_DTYPE or v.ndim != 1:
        raise ValueError(f"expected a 1-D array of {PLY_VERTEX_DTYPE}, got {v.dtype} {v.shape}")
    with open(path, "wb") as f:
        f.write(ply_header(len(v)))
        f.write(v.tobytes())
