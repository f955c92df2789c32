#!/usr/bin/env python3
"""mask band (mask_mmdet) on the H100 engine -- drop-in for the reference's bands/mask_mmdet.py.

Same plugin surface: BAND / CLASSES / CONFIDENCE_THRESHOLD constants, init_model(), process_image(args),
process_video(args), the CLI flags of bands/mask_mmdet.py:165-174 (-i -o -c --sdf --subpath), the outputs (mask.png|mp4,
optional <subpath>/%05d.png with the inverted mask for COLMAP) and the metadata.json keys (bands.mask.{url,ids,folder},
:159-161).  SOLOv2 (inference_detector) and the union of the instance masks run in libprisma_b200.so; there is no CPU path.

--sdf: the clamped signed distance field of the union (snowy.generate_sdf in the reference) is an exact Euclidean
distance transform on the GPU (prisma_mask_sdf).
Additions: --weights (the mmdet checkpoint .pth or .npz), --seeded-weights, --device, --gpus / --device-list (frame sharding),
--lanes (engines per GPU working on consecutive frames at once, prisma_b200/mask.py:SoloV2Lanes).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bands.common.media import VideoReader, VideoWriter, create_folder, open_rgb, write_rgb  # noqa: E402
from bands.common.meta import get_target, get_url, is_video, load_metadata, write_metadata  # noqa: E402

BAND = "mask"
DEVICE = 0
CONFIG = "models/solov2_r101_fpn_3x_coco.py"
MODEL = "models/solov2_r101_fpn_3x_coco_20220511_095119-c559a076.pth"
CLASSES = ['person', 'bird', 'cat', 'dog', 'horse', 'sheep', 'cow', 'elephant', 'bear', 'zebra', 'giraffe']
CONFIDENCE_THRESHOLD = 0.5

model = None
data = None
args = None


def _load_state_dict(a):
    if a.seeded_weights:
        from prisma_b200.seeded_weights import make_solo_weights
        return make_solo_weights("r101", 0)
    path = a.weights or MODEL
    if path.endswith(".npz"):
        return dict(np.load(path))
    import torch
    sd = torch.load(path, map_location="cpu")
    return sd.get("state_dict", sd)  # mmcv checkpoints: {state_dict, meta{CLASSES}} (apis/inference.py:46-48)


def init_model():
    """reference :38-41."""
    global model
    from prisma_b200.mask import SoloV2Lanes
    lanes = getattr(args, "lanes", 4) if is_video(getattr(args, "output", "") or "") else 1   # a still image needs one engine
    # precision: "exact" (default) = the whole network in fp32-class arithmetic (3xTF32, fp32 accumulation): the reference's
    # instance list itself (north_star: mask ids bit-exact); "mixed" = fp16 backbone + fp32-class head and decode (half the GPU
    # time, instances at the 0.05 score filter may differ); "fast" = fp16 everywhere
    variant = "r101" + {"fast": "-fast", "exact": "-exact"}.get(getattr(args, "precision", "exact"), "")
    model = SoloV2Lanes(_load_state_dict(args), device=args.device, lanes=lanes, variant=variant)
    return model


def frame_masks(rgb, confidence):
    """The loop body of process_image / process_video (:113-146): HxWx3 u8 mask frame (the union on every channel)."""
    u = model.infer(rgb, confidence=confidence)["union"]
    return np.repeat(u[..., None], 3, axis=-1)


def encode_sdf(masks):
    """--sdf (:116-118,150-152): a clamped signed distance field of the union in the GREEN channel."""
    from prisma_b200.mask import sdf_green
    masks = masks.copy()
    masks[..., 1] = sdf_green(masks[..., 0], device=args.device)
    return masks


def process_image(a):
    masks = frame_masks(open_rgb(a.input), a.confidence)
    if a.sdf:
        masks = encode_sdf(masks)
    write_rgb(a.output, masks)
    if data is not None:
        data["bands"][BAND] = {"url": os.path.basename(a.output), "ids": CLASSES}


def process_video(a, ctx=None):
    """reference :131-161 over this rank's frames (independent frames: no halo); ordered frames go to the writer rank."""
    from bands.common.sharded import OrderedStreams, ShardContext
    ctx = ctx or ShardContext()
    reader = VideoReader(a.input)
    streams = OrderedStreams(ctx, {"mask": lambda: VideoWriter(reader.width, reader.height, reader.get_avg_fps(), a.output)})
    folder = os.path.dirname(a.output)
    sub = ""
    if a.subpath != "":
        sub = os.path.join(folder, a.subpath)
        create_folder(sub)
    start, stop, _ = ctx.frames(len(reader))
    if start > 0:
        reader.seek(start)
    if stop > start:
        def frames():  # this rank's frames, read lazily (the lanes keep a few of them in flight)
            for k, frame in enumerate(reader):
                yield frame
                if start + k + 1 >= stop:
                    return
        for k, res in enumerate(model.map(frames(), confidence=a.confidence)):
            f = start + k
            masks = np.repeat(res["union"][..., None], 3, axis=-1)
            if sub:  # COLMAP wants black-on-white masks (:148-149)
                write_rgb(os.path.join(sub, "{:05d}.png".format(f)), 255 - masks)
            if a.sdf:
                masks = encode_sdf(masks)
            streams.write("mask", masks)
    streams.finish()
    if ctx.is_writer() and data is not None:
        data["bands"][BAND] = {"url": os.path.basename(a.output), "ids": CLASSES}
        if a.subpath != "":
            data["bands"][BAND]["folder"] = a.subpath


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--input", "-i", help="input", type=str, required=True)
    p.add_argument("--output", "-o", help="output", type=str, default="")
    p.add_argument("--confidence", "-c", help="confidence threshold", type=float, default=CONFIDENCE_THRESHOLD)
    p.add_argument("--sdf", "-s", help="Encode SDF on GREEN channel", action="store_true")
    p.add_argument("--subpath", help="Mask Subpath to frames", type=str, default="")
    p.add_argument("--weights", type=str, default="", help="mmdet SOLOv2 checkpoint (.pth/.npz)")
    p.add_argument("--seeded-weights", action="store_true", help="seeded random weights (offline testing)")
    p.add_argument("--device", type=int, default=DEVICE)
    p.add_argument("--precision", choices=("fast", "mixed", "exact"), default="exact",
                   help="exact: fp32-class everywhere (the reference's instances); mixed: fp16 backbone, fp32-class head + decode; fast: fp16")
    p.add_argument("--lanes", type=int, default=4, help="engines per GPU that take consecutive frames concurrently (video)")
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
    from bands.common.sharded import ENV_RANK, ShardContext, launch
    if args.gpus > 1 and ENV_RANK not in os.environ and is_video(args.output):
        devices = [int(d) for d in args.device_list.split(",")] if args.device_list else None
        launch(os.path.abspath(__file__), argv if argv is not None else sys.argv[1:], args.gpus, devices)
        return  # rank 0 of the workers wrote the video and the metadata
    ctx = ShardContext.from_env(args.device)
    init_model()
    if is_video(args.output):
        process_video(args, ctx)
    else:
        process_image(args)
    if data and ctx.is_writer():
        write_metadata(args.input, data)
    ctx.close()


if __name__ == "__main__":
    main()
