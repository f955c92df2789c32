#!/usr/bin/env python3
"""PRISMA orchestrator -- the reference's process.py surface (flags :76-99, defaults :18-56, band order :163-290) on top
of the H100 bands.

    python process.py -i clip.mp4 [-d depth_anything|depth_midas|...|all] [-f flow_raft|flow_gmflow|all] [-e N] [-b] [-m] ...

Same contract as the reference: creates the PRISMA folder next to the input (or --output), writes metadata.json, stores
the input as the `rgba` band (bands/rgba.py), fills width / height / fps / frames / duration and the camera guesses
(:188-203), then launches ONE SUBPROCESS PER BAND (`python3 bands/<band>.py -i <folder> [extra] [--subpath sub]`, :60-73)
with the reference's default extra arguments (`mask_mmdet --sdf`, `depth_anything --metric outdoor`, :46-56), the mask band
unconditionally (:207), the depth band(s), and for videos the flow band(s); finally the default-band aliases
`depth`, `flow`, `flow_bwd`, `flow_mask`, `flow_mask_bwd` (:246-287).

What differs, and is printed when it happens: bands outside SURVEY.md section 8 (depth_marigold, depth_zoedepth,
depth_patchfusion, flow_gmflow, camera_colmap) are not built here.  Where the reference's DEFAULT would pick one of them
(`depth_patchfusion` for images, `flow_gmflow` for videos) the accelerated band of the same kind runs instead
(depth_anything / flow_raft); an explicit request for one of them is reported and skipped.  Extra flags of this
implementation: --seeded-weights (no checkpoints offline), --encoder, --gpus N (frame sharding inside every band).
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bands.common.meta import add_band, create_metadata, is_video, load_metadata, set_default_band, write_metadata  # noqa: E402
from bands.common.media import VideoReader, open_rgb  # noqa: E402

# defaults of the reference (process.py:18-56)
DEPTH_VIDEO_DEFAULT = "depth_anything"
DEPTH_IMAGE_DEFAULT = "depth_patchfusion"
DEPTH_BANDS = ["depth_midas", "depth_marigold", "depth_zoedepth", "depth_patchfusion", "depth_anything"]
DEPTH_OPTIONS = DEPTH_BANDS + ["all"]
FLOW_DEFAULT = "flow_gmflow"
FLOW_BANDS = ["flow_gmflow", "flow_raft"]
FLOW_OPTIONS = FLOW_BANDS + ["all"]
SUBFOLDERS = {"rgba": "images", "mask_mmdet": "mask", "flow_raft": "flow_raft", "flow_gmflow": "flow_gmflow",
              "depth_zoedepth": "depth_zoedepth", "depth_midas": "depth_midas", "depth_marigold": "depth_marigold",
              "depth_patchfusion": "depth_patchfusion", "depth_anything": "depth_anything", "camera_colmap": "sparse"}
EXTRA_ARGS = {"rgba": "", "mask_mmdet": "--sdf ", "depth_midas": " ", "depth_marigold": "", "depth_zoedepth": "",
              "depth_patchfusion": "", "depth_anything": "--metric outdoor ", "flow_raft": "", "flow_gmflow": ""}

ACCELERATED = {"rgba", "depth_anything", "depth_midas", "flow_raft", "mask_mmdet"}
SHARDED = {"depth_anything", "depth_midas", "flow_raft", "mask_mmdet"}   # bands with --gpus N
OWN_ARGS = ""   # --seeded-weights etc., appended to every inference band (set in main)


def run(band, input_folder, output_file="", subpath=False, extra_args=""):
    """reference process.py:60-73, with subprocess instead of os.system so a failing band is reported."""
    print("\n# ", band.upper())
    if band not in ACCELERATED:
        print(f"[process] band '{band}' is outside the H100 hot path (SURVEY.md section 8): skipped")
        return 1
    cmd = [sys.executable, os.path.join(ROOT, "bands", band + ".py"), "-i", input_folder]
    if output_file != "":
        cmd += ["--output", output_file]
    cmd += extra_args.split()
    if band != "rgba":
        cmd += OWN_ARGS.split()
    if subpath:
        cmd += ["--subpath", SUBFOLDERS[band]]
    print(" ".join(cmd), "\n")
    return subprocess.call(cmd)


def main(argv=None):
    global OWN_ARGS
    parser = argparse.ArgumentParser()
    parser.add_argument('--input', '-i', help="input file", type=str, required=True)
    parser.add_argument('--output', help="folder name", type=str, default='')
    parser.add_argument('--record3d', help="Record3D video", action='store_true')
    # global video properties
    parser.add_argument('--fps', '-r', help='fix framerate', type=float, default=24)
    parser.add_argument('--extra', '-e', help='Save extra data [>0 frames|PLYs; >1 FLOs; >2 NPY]', type=int, default=0)
    # Depth
    parser.add_argument('--rgbd', help='Where the depth is', type=str, default=None)
    parser.add_argument('--depth', '-d', help='Depth bands', type=str, default=None, choices=DEPTH_OPTIONS)
    parser.add_argument('--ply', '-p', help='Save ply for images', action='store_true')
    parser.add_argument('--npy', '-n', help='Save npy version of files', action='store_true')
    # Flow
    parser.add_argument('--flow', '-f', help='Flow bands', type=str, default=None, choices=FLOW_OPTIONS)
    parser.add_argument('--flo', help='Save flo files for raft', action='store_true')
    parser.add_argument('--flow_backwards', '-b', help="Save backwards video", action='store_true')
    parser.add_argument('--flow_mask', '-m', help="Save mask of videos", action='store_true')
    # this implementation
    parser.add_argument('--seeded-weights', action='store_true', help="seeded random weights in every band (offline testing)")
    parser.add_argument('--encoder', type=str, default="vitl", choices=["vits", "vitb", "vitl"], help="depth_anything encoder")
    parser.add_argument('--gpus', type=int, default=1, help="shard the frames of every band over this many GPUs")
    args = parser.parse_args(argv)

    # 1. input parameters (:103-108)
    input_path = args.input
    input_folder = os.path.dirname(input_path)
    input_basename = os.path.basename(input_path).rsplit(".", 1)[0]
    # 2. folder + metadata (:110-115)
    folder_name = args.output if args.output else os.path.join(input_folder, input_basename)
    data = create_metadata(folder_name)
    video = is_video(input_path)
    extension = "mp4" if video else "png"
    name_rgba = "rgba." + extension
    path_rgba = os.path.join(folder_name, name_rgba)
    extra_rgba_args = EXTRA_ARGS["rgba"]
    if args.record3d:  # :125-160: camera intrinsics + depth range from the container's Record3D track
        try:
            from pymediainfo import MediaInfo  # noqa: F401
        except ImportError:
            print("[process] --record3d needs pymediainfo (reference common/meta.py:148-156), which is not installed")
            return 2
        import json
        info = json.loads(MediaInfo.parse(input_path).to_json())
        rec = json.loads(info["tracks"][0]["movie_more"])
        args.rgbd = "right"
        height = VideoReader(input_path).height if video else open_rgb(input_path).shape[0]
        cam = rec["intrinsicMatrix"]
        data["focal_length"] = max(cam[0], cam[4])
        data["principal_point"] = [cam[6], cam[7]]
        data["field_of_view"] = 2 * np.arctan(0.5 * height / data["focal_length"]) * 180 / np.pi
        extra_rgba_args += "--encoding_depth hue "
        add_band(data, "depth", url="depth." + extension)
        rng = rec["rangeOfEncodedDepth"]
        data["bands"]["depth"]["values"] = {"min": {"type": "float", "value": rng[0]}, "max": {"type": "float", "value": rng[1]}}
    # 3. rgba band (:163-174)
    add_band(data, "rgba", url=name_rgba)
    if args.rgbd:
        extra_rgba_args += "--rgbd " + args.rgbd
    if video:
        extra_rgba_args += " --fps " + str(args.fps)
    write_metadata(folder_name, data)
    run("rgba", input_path, path_rgba, subpath=True, extra_args=extra_rgba_args)
    data = load_metadata(folder_name)
    # 4. metadata (:176-203)
    if video:
        r = VideoReader(path_rgba)
        data["width"], data["height"], data["fps"], data["frames"] = r.width, r.height, r.get_avg_fps(), len(r)
        data["duration"] = float(data["frames"]) / float(data["fps"])
    else:
        img = open_rgb(path_rgba)
        data["width"], data["height"] = img.shape[1], img.shape[0]
    if "principal_point" not in data:
        data["principal_point"] = [float(data["width"] / 2), float(data["height"] / 2)]
    if "focal_length" not in data:
        data["focal_length"] = float(data["height"] * data["width"]) ** 0.5
    if "field_of_view" not in data:
        data["field_of_view"] = 2 * np.arctan(0.5 * data["height"] / data["focal_length"]) * 180 / np.pi
    write_metadata(folder_name, data)

    # 5. bands (:205-290)
    if args.extra > 0:
        args.ply = True
    if args.extra > 1:
        args.flo = True
    if args.extra > 2:
        args.npy = True
    OWN_ARGS = ("--seeded-weights " if args.seeded_weights else "")
    shard = f"--gpus {args.gpus} " if (args.gpus > 1 and video) else ""

    # 5.a mask (always)
    run("mask_mmdet", folder_name, subpath=True, extra_args=EXTRA_ARGS["mask_mmdet"] + shard)

    # 5.b depth
    depth_args = ("--ply " if args.ply else "") + ("--npy " if args.npy else "")
    if args.depth is None:
        args.depth = DEPTH_VIDEO_DEFAULT if video else DEPTH_IMAGE_DEFAULT
        if args.depth not in ACCELERATED:
            print(f"[process] the reference's default depth band for this input ({args.depth}) is outside the H100 hot "
                  f"path; running depth_anything instead")
            args.depth = "depth_anything"
    ran_depth = []
    for band in (DEPTH_BANDS if args.depth == "all" else [args.depth]):
        extra = depth_args + EXTRA_ARGS.get(band, "")
        if band == "depth_anything":
            extra += f"--encoder {args.encoder} "
        if band in SHARDED:
            extra += shard
        if band == "depth_patchfusion" and video:
            extra += "--mode=p49 "
        if run(band, folder_name, subpath=args.extra, extra_args=extra) == 0:
            ran_depth.append(band)
    if args.rgbd is None:  # default depth band (:246-254)
        if args.depth == "all":
            default = DEPTH_VIDEO_DEFAULT if video else DEPTH_IMAGE_DEFAULT
            if default not in ran_depth and ran_depth:
                default = "depth_anything" if "depth_anything" in ran_depth else ran_depth[0]
            set_default_band(folder_name, "depth", default)
        else:
            set_default_band(folder_name, "depth", args.depth)

    if video:
        # 5.c flow
        if args.flow is None:
            args.flow = FLOW_DEFAULT
            if args.flow not in ACCELERATED:
                print(f"[process] the reference's default flow band ({args.flow}) is outside the H100 hot path; running "
                      f"flow_raft instead")
                args.flow = "flow_raft"
        flow_args = ("--backwards " if args.flow_backwards else "") + ("--mask " if args.flow_mask else "")
        for band in (FLOW_BANDS if args.flow == "all" else [args.flow]):
            extra = flow_args + EXTRA_ARGS.get(band, "") + (shard if band in SHARDED else "")
            run(band, folder_name, subpath=args.flo, extra_args=extra)
        flow_default = args.flow
        if args.flow == "all":
            flow_default = FLOW_DEFAULT if FLOW_DEFAULT in ACCELERATED else "flow_raft"
        set_default_band(folder_name, "flow", flow_default)
        set_default_band(folder_name, "flow_bwd", flow_default + "_bwd")
        set_default_band(folder_name, "flow_mask", flow_default + "_mask")
        set_default_band(folder_name, "flow_mask_bwd", flow_default + "_mask_bwd")
        # 5.d camera
        run("camera_colmap", folder_name, subpath=True)
    return 0


if __name__ == '__main__':
    sys.exit(main())
