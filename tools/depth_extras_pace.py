"""Pace of the depth bands' extras: the --ply point cloud at 1080p and depth_midas --model midas3-small at 720p.

    python tools/depth_extras_pace.py [--reps 20] [--out FILE.json]

point cloud : prisma_depth_point_cloud on a 1080p prediction with the flip (the bands' relative-depth case).  Kernel times
              come from torch.profiler (CUDA activities), the mean over --reps calls after one warm-up call: the min / max
              pass of the flip, the 5x5 median (reads 4 B, writes 4 B per pixel) and the unproject-and-pack (reads 4 + 3 B,
              writes 15 B per pixel), with the bytes per pixel over kernel time as achieved bandwidth.  `call_ms` is the whole
              call on the host clock, host-to-device and device-to-host copies included.
midas3-small: frames/s of the DPT_Large engine behind the 256-pixel transform at 1280x720 with the frames resident on the
              device (prisma_depth_infer_resident, CUDA events), next to the 384-pixel midas3 for scale; seeded weights.
Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.autograd import DeviceType

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from prisma_b200.depth import DepthAnythingEngine, MidasEngine  # noqa: E402
from prisma_b200.seeded_weights import make_midas_weights  # noqa: E402
from prisma_b200.synthetic import synthetic_frame  # noqa: E402

KERNELS = {"k_minmax_plain": None, "k_pcl_median5": (4, 4), "k_pcl_unproject_pack": (7, 15)}  # bytes read, written per pixel


def point_cloud_pace(reps, h=1080, w=1920):
    f = synthetic_frame(h, w, 0)
    pred = (f[..., 0].astype(np.float32) * 0.01 + f[..., 1].astype(np.float32) * 0.001 + 1.0).astype(np.float32)
    eng = DepthAnythingEngine("vits")
    eng.point_cloud(pred, f, True)
    t0 = time.perf_counter()
    for _ in range(reps):
        eng.point_cloud(pred, f, True)
    call_ms = (time.perf_counter() - t0) * 1e3 / reps
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.point_cloud(pred, f, True)
    eng.close()
    out = dict(frame=[h, w], call_ms=call_ms, kernels={})
    for name, bpp in KERNELS.items():
        ks = [e for e in prof.events() if name in e.name and e.device_type == DeviceType.CUDA]
        assert len(ks) == reps, (name, len(ks))
        us = sum(e.time_range.elapsed_us() for e in ks) / reps
        k = dict(us=us)
        if bpp:
            k["bytes_per_pixel"] = sum(bpp)
            k["GB_per_s"] = h * w * sum(bpp) / us / 1e3
        out["kernels"][name] = k
    out["median_and_pack_us"] = out["kernels"]["k_pcl_median5"]["us"] + out["kernels"]["k_pcl_unproject_pack"]["us"]
    return out


def midas_pace(reps, batch, h=720, w=1280):
    sd = make_midas_weights("dpt_large", 0)
    out = {}
    for model, side in (("midas3-small", 256), ("midas3", 384)):
        eng = MidasEngine(sd, net_side=side)
        eng.time_resident(h, w, 2, batch)
        ms = eng.time_resident(h, w, reps, batch)
        eng.close()
        out[model] = dict(net_side=side, frame=[h, w], batch=batch, ms_per_pass=ms, frames_per_s=batch * 1e3 / ms)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi, point_cloud=point_cloud_pace(a.reps),
               midas=midas_pace(a.reps, a.batch))
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
