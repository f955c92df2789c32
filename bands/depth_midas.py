#!/usr/bin/env python3
"""depth_midas band on the H100 engine -- drop-in for the reference's bands/depth_midas.py.

Same plugin surface: BAND / MODELS_VERSIONS, init_model(model_version), infer(img, model_version, normalize),
process_image(args), process_video(args), the CLI flags of bands/depth_midas.py:182-192, the outputs (depth_midas.mp4|png,
depth_midas_min.csv, depth_midas_max.csv, optional <sub>/%05d.npy|png) and the metadata.json keys (:87-99,163-174).
The hub transform, the DPT_Large forward, the bicubic(align_corners=True) resize and the heat encode run in
libprisma_b200.so; there is no CPU path.

Built: --model midas3 (the default: DPT_Large + default_transform, fit inside 384 x 384) and midas3-small (the same network
and checkpoint behind the hub's small_transform, fit inside 256 x 256).  midas2 / midas2-small (the ResNeXt-101 MiDaS v2.1
network) raise instead of falling back.  --ply writes depth_midas.ply next to a still image's output (reference :102-103);
video runs ignore it, as the reference does.
Additions: --weights (the upstream dpt_large_384.pt state_dict or .npz), --seeded-weights, --device.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bands.common.depth_loop import process_depth_video  # noqa: E402
from bands.common.sharded import ENV_RANK, ShardContext, launch  # noqa: E402
from bands.common.media import open_rgb, write_rgb  # noqa: E402
from bands.common.ply import write_ply  # noqa: E402
from bands.common.meta import get_target, get_url, is_video, load_metadata, write_metadata  # noqa: E402

BAND = "depth_midas"
DEVICE = 0
MODELS_VERSIONS = ["midas2-small", "midas2", "midas3-small", "midas3"]
WEIGHTS = "models/dpt_large_384.pt"

model = None
data = None
args = None


def _load_state_dict(a):
    if a.seeded_weights:
        from prisma_b200.seeded_weights import make_midas_weights
        return make_midas_weights("dpt_large", 0)
    path = a.weights or WEIGHTS
    if path.endswith(".npz"):
        return dict(np.load(path))
    import torch
    sd = torch.load(path, map_location="cpu")
    return sd.get("state_dict", sd)


NET_SIDES = {"midas3": 384, "midas3-small": 256}  # hub default_transform / small_transform


def init_model(model_version="midas3"):
    """reference :29-46."""
    global model
    if model_version not in NET_SIDES:
        raise NotImplementedError("only --model midas3 / midas3-small (DPT_Large) are built; %s is not" % model_version)
    from prisma_b200.depth import MidasEngine
    model = MidasEngine(_load_state_dict(args), device=args.device if args else DEVICE, net_side=NET_SIDES[model_version])
    return model


def infer(img, model_version="midas3", normalize=False):
    """HxWx3 u8 RGB -> HxW f32 (reference :49-75)."""
    if model is None:
        init_model(model_version)
    return model.infer(np.asarray(img), normalize=normalize)


def process_image(a):
    img = open_rgb(a.input)
    rgb, dmin, dmax, pred = model.infer_image(img, want_depth=True)  # write_depth's PNG encoding (io.py:138-166)
    if a.npy:
        np.save(os.path.join(os.path.dirname(a.output), BAND + ".npy"), pred)
    if a.ply:  # reference :102-103: write_pcl(..., flip=True)
        write_ply(os.path.join(os.path.dirname(a.output), BAND + ".ply"), model.point_cloud(pred, img, flip=True))
    write_rgb(a.output, rgb)
    if data:
        data["bands"][BAND]["values"] = {"min": {"value": dmin, "type": "float"}, "max": {"value": dmax, "type": "float"}}


def process_video(a, ctx=None):
    process_depth_video(model, a, data, BAND, ctx)


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--input", "-i", help="Input image/video", type=str, required=True)
    p.add_argument("--output", "-o", help="Output image/video", type=str, default="")
    p.add_argument("--npy", "-n", help="Save numpy data", action="store_true")
    p.add_argument("--ply", "-p", help="Create point cloud PLY", action="store_true")
    p.add_argument("--subpath", "-d", help="subpath to frames", type=str, default="")
    p.add_argument("--model", type=str, choices=MODELS_VERSIONS, default="midas3")
    p.add_argument("--weights", type=str, default="", help="DPTDepthModel state_dict (.pt/.npz)")
    p.add_argument("--seeded-weights", action="store_true", help="seeded random weights (offline testing)")
    p.add_argument("--device", type=int, default=DEVICE)
    p.add_argument("--gpus", type=int, default=1, help="shard the frames of a video over this many GPUs (one worker each)")
    p.add_argument("--device-list", type=str, default="", help="GPU ordinals of the workers (default 0..gpus-1)")
    return p


def main(argv=None):
    global args, data
    args = build_parser().parse_args(argv)
    data = load_metadata(args.input)
    if data:
        args.input = get_url(args.input, data, "rgba")
        args.output = get_target(args.input, data, band=BAND, target=args.output, force_extension="png")
    elif args.output == "":
        args.output = os.path.join(os.path.dirname(args.input), BAND + os.path.splitext(args.input)[1])
    if args.gpus > 1 and ENV_RANK not in os.environ and is_video(args.output):
        devices = [int(d) for d in args.device_list.split(",")] if args.device_list else None
        launch(os.path.abspath(__file__), argv if argv is not None else sys.argv[1:], args.gpus, devices)
        return  # rank 0 of the workers wrote the video, the csv pair and the metadata
    ctx = ShardContext.from_env(args.device)
    init_model(args.model)
    if is_video(args.output):
        process_video(args, ctx)
    else:
        process_image(args)
    if ctx.is_writer():
        write_metadata(args.input, data)
    ctx.close()


if __name__ == "__main__":
    main()
