#!/usr/bin/env python3
"""rgba band -- drop-in for the reference's bands/rgba.py (SURVEY.md section 8f row 4): stores the input as the PRISMA
folder's `rgba` band (video: re-muxed without audio at --fps, optionally every frame as <subpath>/%06d.png; image:
rgba.png) and, for side-by-side RGB-D recordings (--rgbd left|right|top|bottom), splits the colour half from the depth
half (depth optionally re-encoded from hue to the heat map, --encoding_depth hue).

Same CLI as reference rgba.py:149-163, same outputs and metadata keys (:166-199).  This band does no inference: it is
container / pixel-copy work, and the only arithmetic on the path (hue -> heat re-encode of Record3D depth, :62-64) is
per-pixel numpy as in the reference.  Frames are decoded / encoded with OpenCV (bands/common/media.py): decord, PyAV and
ffmpeg, which the reference uses (:77,85; common/io.py:246-305), are not in this image, and the engine has no hardware video codec path, so
"encode on the GPU" is not an option on this part at all (NVDEC exists; see DESIGN.md section 7).
"""
import argparse
import os
import shutil
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bands.common.media import VideoReader, VideoWriter, create_folder, open_rgb, write_rgb  # noqa: E402
from bands.common.meta import get_target, get_url, is_video, load_metadata, write_metadata  # noqa: E402

BAND = "rgba"
data = None


def hue_to_rgb(hue):
    """common/encode.py:13-23 (hue in [0,1] -> fully saturated RGB in [0,1])."""
    hue = np.asarray(hue, np.float64)
    rgb = np.zeros(hue.shape + (3,))
    for i, off in enumerate((0.0, 4.0, 2.0)):
        rgb[..., i] = np.clip(np.abs(np.fmod(hue * 6.0 + off, 6.0) - 3.0) - 1.0, 0.0, 1.0)
    return rgb


def heat_to_rgb(heat):
    """common/encode.py:31-33."""
    return hue_to_rgb((1.0 - heat) * 0.65)


def rgb_to_hue360(rgb_u8):
    """Hue channel of common/encode.py:36-70 rgb_to_hsv (degrees), for --encoding_depth hue."""
    rgb = rgb_u8.astype(np.float64) / 255.0
    mx, mn = rgb.max(-1), rgb.min(-1)
    d = mx - mn
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    h = np.zeros_like(mx)
    m = d > 0
    rm, gm, bm = m & (mx == r), m & (mx == g) & (mx != r), m & (mx == b) & (mx != r) & (mx != g)
    h[rm] = (60.0 * ((g - b)[rm] / d[rm]) + 360.0) % 360.0
    h[gm] = 60.0 * ((b - r)[gm] / d[gm]) + 120.0
    h[bm] = 60.0 * ((r - g)[bm] / d[bm]) + 240.0
    return h


def crops(width, height, where):
    """rgba.py:29-40: (rgb_crop, depth_crop) as [x, y, w, h]."""
    if where == "left":
        return [width // 2, 0, width // 2, height], [0, 0, width // 2, height]
    if where == "right":
        return [0, 0, width // 2, height], [width // 2, 0, width // 2, height]
    if where == "top":
        return [0, height // 2, width, height // 2], [0, 0, width, height // 2]
    return [0, 0, width, height // 2], [0, height // 2, width, height // 2]


def cut(frame, c):
    return frame[c[1]:c[1] + c[3], c[0]:c[0] + c[2], :]


def subfolder(output_file, sub):
    if not sub:
        return None
    p = os.path.join(os.path.dirname(output_file), sub)
    create_folder(p)
    return p


def process_video(args):
    reader = VideoReader(args.tmp if os.path.exists(args.tmp) else args.input)
    fps = args.fps
    if args.rgbd == "none":  # prune (:74-96): pass-through without audio
        sub = subfolder(args.output, args.subpath)
        out = VideoWriter(reader.width, reader.height, fps, args.output)
        for i, frame in enumerate(reader):
            if sub:
                write_rgb(os.path.join(sub, str(i).zfill(6) + ".png"), frame)
            out.write(frame)
        out.close()
        return
    rgb_c, dep_c = crops(reader.width, reader.height, args.rgbd)
    sub_rgb, sub_dep = subfolder(args.output, args.subpath), subfolder(args.output_depth, args.subpath_depth)
    rgb_v = VideoWriter(rgb_c[2], rgb_c[3], fps, args.output)
    dep_v = VideoWriter(dep_c[2], dep_c[3], fps, args.output_depth)
    for i, frame in enumerate(reader):
        rgb, dep = cut(frame, rgb_c), cut(frame, dep_c)
        if args.encoding_depth == "hue":  # Record3D encodes depth as hue; PRISMA's depth bands are heat maps (:62-64)
            dep = (heat_to_rgb(np.clip(rgb_to_hue360(dep) / 360.0, 0.0, 1.0)) * 255.0).astype(np.uint8)
        if sub_rgb:
            write_rgb(os.path.join(sub_rgb, str(i).zfill(6) + ".png"), rgb)
        if sub_dep:
            write_rgb(os.path.join(sub_dep, str(i).zfill(6) + ".png"), dep)
        rgb_v.write(np.ascontiguousarray(rgb))
        dep_v.write(np.ascontiguousarray(dep))
    rgb_v.close()
    dep_v.close()


def process_image(args):
    write_rgb(args.output, open_rgb(args.tmp if os.path.exists(args.tmp) else args.input))


def main(argv=None):
    global data
    parser = argparse.ArgumentParser()
    parser.add_argument('--input', '-i', help="input", type=str, required=True)
    parser.add_argument('--tmp', '-t', help="tmp", type=str, default="tmp")
    parser.add_argument('--fps', '-r', help='fix framerate of videos', type=float, default=24)
    parser.add_argument('--output', '-o', help="output", type=str, default="")
    parser.add_argument('--subpath', help="subpath to frames", type=str, default=None)
    parser.add_argument('--rgbd', help='Where the depth is', choices=["none", "left", "right", "top", "bottom"], default='none')
    parser.add_argument('--encoding_depth', help="encoding for depth", choices=["none", "hue"], default="none")
    parser.add_argument('--output_depth', help="output file for depth", type=str, default="depth")
    parser.add_argument('--subpath_depth', help="subpath to frames for depth", type=str, default=None)
    args = parser.parse_args(argv)

    data = load_metadata(args.input)
    meta_path = args.input
    if data:  # a PRISMA folder: metadata defaults (:166-173)
        args.tmp = get_url(args.input, data, "rgba")
        args.input = args.tmp
        args.output = get_target(args.tmp, data, band=BAND, target=args.output, force_extension='png')
        if args.rgbd != "none":
            args.output_depth = get_target(args.tmp, data, band='depth', target="")
    else:
        folder = os.path.dirname(args.input)
        ext = args.input.rsplit(".", 1)[1]
        if args.tmp == "tmp":
            args.tmp = os.path.join(folder, "tmp." + ext)
        if ext != "mp4":
            ext = "png"
        if args.output == "":
            args.output = os.path.join(folder, BAND + "." + ext)
        elif os.path.isdir(args.output):
            args.output = os.path.join(args.output, BAND + "." + ext)
        args.output_depth = os.path.join(os.path.dirname(args.output), args.output_depth + "." + ext)
        if os.path.abspath(args.tmp) != os.path.abspath(args.input):
            shutil.copyfile(args.input, args.tmp)  # the reference works on a copy (:108,121)

    if os.path.abspath(args.output) == os.path.abspath(args.input):
        # in-place request (the folder's rgba band is the input): nothing to transcode
        return 0
    if is_video(args.input):
        process_video(args)
    else:
        process_image(args)
    if not data and os.path.exists(args.tmp) and os.path.abspath(args.tmp) != os.path.abspath(args.input):
        os.remove(args.tmp)
    write_metadata(meta_path, data)
    return 0


if __name__ == '__main__':
    sys.exit(main())
