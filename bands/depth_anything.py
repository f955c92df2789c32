#!/usr/bin/env python3
"""depth_anything band on the H100 engine -- drop-in for the reference's bands/depth_anything.py.

Same plugin surface (SURVEY.md section 8b): module constants/globals, init_model(), infer(img, normalize),
process_image(args), process_video(args), the CLI flags of bands/depth_anything.py:255-265, the outputs
(<band>.mp4|png, <band>_min.csv, <band>_max.csv, optional <sub>/%05d.npy) and the metadata.json keys
(:155-166,241-251).  The model call and the numpy encode are replaced by libprisma_b200.so; there is no CPU path.

`--metric indoor|outdoor` runs the ZoeDepth metric head (no flip in the encode, reference :188).
Additions: --weights (state_dict: torch .pth/.pt or .npz), --seeded-weights (offline test weights), --device.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bands.common.meta import get_target, get_url, is_video, load_metadata, write_metadata  # noqa: E402
from bands.common.depth_loop import process_depth_video  # noqa: E402
from bands.common.sharded import ENV_RANK, ShardContext, launch  # noqa: E402
from bands.common.media import open_rgb, write_rgb  # noqa: E402

BAND = "depth_anything"
DEVICE = 0
WEIGHTS = "models/depth_anything_{}14.pth"
METRIC_WEIGHTS = {"indoor": "models/depth_anything_metric_depth_indoor.pt",     # reference :38-39
                  "outdoor": "models/depth_anything_metric_depth_outdoor.pt"}

model = None
data = None
args = None


def _load_state_dict(a):
    if a.seeded_weights:
        # seeded random weights (no checkpoint is reachable offline)
        from prisma_b200.seeded_weights import make_da_weights, make_zoe_weights
        return make_zoe_weights(a.encoder, 0) if a.metric != "none" else make_da_weights(a.encoder, 0)
    path = a.weights or (METRIC_WEIGHTS[a.metric] if a.metric != "none" else WEIGHTS.format(a.encoder))
    if path.endswith(".npz"):
        return dict(np.load(path))
    import torch
    sd = torch.load(path, map_location="cpu")
    return sd.get("state_dict", sd)


def init_model():
    """reference :48-76: relative model, or (--metric indoor|outdoor, :52-57) the ZoeDepth metric model."""
    global model
    from prisma_b200.depth import DepthAnythingEngine, ZoeDepthEngine
    if args.metric != "none":
        model = ZoeDepthEngine(_load_state_dict(args), device=args.device, encoder=args.encoder)
    else:
        model = DepthAnythingEngine(args.encoder, _load_state_dict(args), device=args.device)
    return model


def infer(img, normalize=False):
    """HxWx3 u8 RGB -> HxW f32 (reference :100-143)."""
    if model is None:
        init_model()
    return model.infer(img, normalize=normalize)


def process_image(a):
    img = open_rgb(a.input)
    rgb, dmin, dmax, pred = model.infer_image(img, want_depth=True)  # write_depth's PNG encoding (io.py:138-166)
    if a.npy:
        np.save(os.path.splitext(a.output)[0] + ".npy", pred)
    write_rgb(a.output, rgb)
    if data:
        data["bands"][BAND]["values"] = {"min": {"type": "float", "value": dmin}, "max": {"type": "float", "value": dmax}}


def process_video(a, ctx=None):
    process_depth_video(model, a, data, BAND, ctx, flip=(a.metric == "none"))  # reference :188


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--input", "-i", help="Input image/video", type=str, required=True)
    p.add_argument("--output", "-o", help="Output image/video", type=str, default="")
    p.add_argument("--npy", "-n", help="Save numpy data", action="store_true")
    p.add_argument("--ply", "-p", help="Create point cloud PLY", action="store_true")
    p.add_argument("--subpath", "-d", help="subpath to frames", type=str, default="")
    p.add_argument("--encoder", type=str, default="vitl", choices=["vits", "vitb", "vitl"])
    p.add_argument("--metric", help="Use a metric model", type=str, default="none", choices=["none", "indoor", "outdoor"])
    p.add_argument("--weights", type=str, default="", help="DPT_DINOv2 state_dict (.pth/.npz)")
    p.add_argument("--seeded-weights", action="store_true", help="seeded random weights (offline testing)")
    p.add_argument("--device", type=int, default=DEVICE)
    p.add_argument("--gpus", type=int, default=1, help="shard the frames of a video over this many GPUs (one worker each)")
    p.add_argument("--device-list", type=str, default="", help="GPU ordinals of the workers (default 0..gpus-1)")
    return p


def main(argv=None):
    global args, data
    args = build_parser().parse_args(argv)
    if args.metric != "none" and args.encoder != "vitl" and not args.seeded_weights:
        raise ValueError("the metric checkpoints are ViT-L models (base_models/depth_anything.py:339)")
    if args.ply:
        print("--ply is outside the engine's scope (optional export, SURVEY.md section 2); ignored")
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
    init_model()
    if is_video(args.output):
        process_video(args, ctx)
    else:
        process_image(args)
    if ctx.is_writer():
        write_metadata(args.input, data)
    ctx.close()


if __name__ == "__main__":
    main()
