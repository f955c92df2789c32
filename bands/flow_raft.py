#!/usr/bin/env python3
"""flow_raft band on the H100 engine -- drop-in for the reference's bands/flow_raft.py.

Same plugin surface: BAND / ITERATIONS / MODEL constants, init_model(args), infer(args, prev, curr),
process_video(args), the CLI flags of bands/flow_raft.py:170-189, the outputs (flow_raft.mp4, flow_raft.csv with the
per-frame max displacement, optional flow_raft_bwd.mp4, flow_raft_mask[_bwd].mp4, <subpath>_fwd|_bwd/%04d.flo,
<subpath_mask>_fwd|_bwd/%04d.png) and the metadata.json keys (:143-166).
The model (RAFT, 12-20 GRU iterations), the x`scale` cubic resize, the HSV encode, the forward/backward consistency
masks and the 16-bit flow PNG payload are computed in libprisma_b200.so.  --small raises (commented out in the
reference too); --alternate_corr /
--mixed_precision are accepted for CLI compatibility: the engine has one (fp16-operand, fp32-accumulate) path and
always builds the correlation pyramid on the GPU.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bands.common.meta import get_target, get_url, load_metadata, write_metadata  # noqa: E402
from bands.common.media import VideoReader, VideoWriter  # noqa: E402

BAND = "flow_raft"
ITERATIONS = 20
MODEL = "models/raft-sintel.pth"

model = None
data = None


def _load_state_dict(a):
    if a.seeded_weights:
        from prisma_b200.seeded_weights import make_raft_weights
        return make_raft_weights(0)
    import torch
    return torch.load(a.model, map_location="cpu")  # keys carry the DataParallel "module." prefix (:42-44)


def init_model(args):
    global model
    from prisma_b200.flow import RaftFlowEngine
    model = RaftFlowEngine(_load_state_dict(args), device=args.device, iterations=args.iterations, scale=args.scale)
    return model


def infer(args, prev_frame, curr_frame, want_rgb=False, reuse_prev=False):
    """(fwd_flow, bwd_flow, fwd_mask, bwd_mask) like the reference's infer (:51-66), plus the engine's result dict;
    frames are HxWx3 u8 RGB at the source resolution (the x scale resize of :100 happens inside the engine)."""
    from prisma_b200.flow import consistency_masks
    r = model.infer_pair(prev_frame, curr_frame, want_rgb=want_rgb, reuse_prev=reuse_prev)
    fwd_mask = bwd_mask = None
    if args.output_mask != "" or args.subpath_mask != "":
        fwd_mask, bwd_mask, r["fwd_u16"], r["bwd_u16"] = consistency_masks(r["fwd"], r["bwd"], want_u16=True,
                                                                           device=args.device)
    return r["fwd"], r["bwd"], fwd_mask, bwd_mask, r


def write_flow(args, r, streams, idx, fwd_mask=None, bwd_mask=None):
    """One frame's outputs (reference common/flow.py:64-98): ordered video frames + the max displacement go to `streams`
    (bands/common/sharded.OrderedStreams), per-frame files are written here.  The reference's .flo branch (:90-93) calls
    this very function with (path, flow) and cannot run; the Middlebury writer it means (common/io.py:175-198) is used."""
    from prisma_b200.flow import write_flo
    streams.write("fwd", r["fwd_rgb"])  # the VideoWriter rescales to the source size, as the reference's does
    streams.scalars(r["max_fwd"])
    if fwd_mask is not None and args.output_mask != "":
        streams.write("fwd_mask", np.repeat((fwd_mask.astype(np.uint8) * 255)[..., None], 3, axis=-1))
    if bwd_mask is not None and args.output_mask != "" and args.backwards:
        streams.write("bwd_mask", np.repeat((bwd_mask.astype(np.uint8) * 255)[..., None], 3, axis=-1))
    if args.backwards:
        streams.write("bwd", r["bwd_rgb"])
    if args.subpath != "":
        write_flo(os.path.join(args.subpath + "_fwd", "%04d.flo" % idx), r["fwd"])
        if args.backwards:
            write_flo(os.path.join(args.subpath + "_bwd", "%04d.flo" % idx), r["bwd"])
    if args.subpath_mask != "":
        import cv2
        cv2.imwrite(os.path.join(args.subpath_mask + "_fwd", "%04d.png" % idx), r["fwd_u16"])
        if args.backwards:
            cv2.imwrite(os.path.join(args.subpath_mask + "_bwd", "%04d.png" % idx), r["bwd_u16"])


def process_video(args, ctx=None, chunk=16):
    """The reference's loop (:97-141) over this rank's frames.  Output index j = the flow from frame j to frame j + 1
    (j < T - 1) and the all-zero last frame (j = T - 1).  A rank that owns the `curr` frames [start, stop) reads from
    start - 1 (one halo frame) and produces the outputs [start - 1, stop - 1); the rank that owns the last frame appends
    the zero frame.  Frames go through the engine in chunks (prisma_flow_infer_stream: uploads / downloads overlapped, each
    frame encoded once)."""
    from bands.common.sharded import OrderedStreams, ShardContext
    from prisma_b200.flow import consistency_masks
    ctx = ctx or ShardContext()
    reader = VideoReader(args.input)
    T = len(reader)
    base = args.output.rsplit(".", 1)[0]
    fps = reader.get_avg_fps()
    new_writer = lambda name: (lambda: VideoWriter(reader.width, reader.height, fps, name))
    mask_base = args.output_mask.rsplit(".", 1)[0] if args.output_mask != "" else ""
    streams = OrderedStreams(ctx, {"fwd": new_writer(args.output), "bwd": new_writer(base + "_bwd.mp4"),
                                   "fwd_mask": new_writer(args.output_mask), "bwd_mask": new_writer(mask_base + "_bwd.mp4")})
    want_masks = args.output_mask != "" or args.subpath_mask != ""
    want_flow = want_masks or args.subpath != ""
    start, stop, first = ctx.frames(T, halo=1)
    if first > 0:
        reader.seek(first)
    state = dict(cont=False, idx=first)

    def flush(frs):
        r = model.infer_clip(np.ascontiguousarray(np.stack(frs)), continue_clip=state["cont"], want_flow=want_flow, want_rgb=True)
        state["cont"] = True
        for j in range(r["pairs"]):
            rec = dict(fwd_rgb=r["fwd_rgb"][j], bwd_rgb=r["bwd_rgb"][j], max_fwd=float(r["max_fwd"][j]))
            fm = bm = None
            if want_flow:
                rec["fwd"], rec["bwd"] = r["fwd"][j], r["bwd"][j]
            if want_masks:
                fm, bm, rec["fwd_u16"], rec["bwd_u16"] = consistency_masks(rec["fwd"], rec["bwd"], want_u16=True, device=args.device)
            write_flow(args, rec, streams, state["idx"], fm, bm)
            state["idx"] += 1

    pending, n_read = [], 0
    if stop > first:
        for frame in reader:
            pending.append(frame)
            n_read += 1
            if len(pending) == chunk:
                flush(pending)
                pending = []
            if first + n_read >= stop:
                break
        if pending:
            flush(pending)
    if stop == T and T > 0 and start < stop:
        # last frame (:116-126): zero flow (the reference's 0/0 -> NaN -> u8 cast gives a black frame) and all-false masks.
        # Emitted at the engine's output size; the reference allocates them at the source size, and the writer rescales
        # either to the same black frame.
        hs, ws = model.out_size(reader.height, reader.width)
        zero = np.zeros((hs, ws, 2), np.float32)
        black = np.zeros((hs, ws, 3), np.uint8)
        u16 = np.zeros((hs, ws, 3), np.uint16)
        u16[..., :2] = 32768
        rec = dict(fwd=zero, bwd=zero, fwd_rgb=black, bwd_rgb=black, max_fwd=0.0, fwd_u16=u16, bwd_u16=u16)
        mask = np.zeros((hs, ws), bool) if want_masks else None
        write_flow(args, rec, streams, T - 1, mask, mask)
    table = streams.finish()
    if not ctx.is_writer():
        return
    with open(base + ".csv", "w") as f:
        f.writelines("{}\n".format(row[0]) for row in table)
    if data:
        data["bands"][BAND] = {"url": BAND + ".mp4", "values": {"dist": {"type": "float", "url": BAND + ".csv"}}}
        if args.subpath != "":
            data["bands"][BAND]["folder"] = args.subpath
        if args.backwards:
            data["bands"][BAND + "_bwd"] = {"url": BAND + "_bwd.mp4"}
            if args.subpath != "":
                data["bands"][BAND + "_bwd"]["folder"] = args.subpath + "_bwd"
        if args.output_mask != "":
            data["bands"][BAND + "_mask"] = {"url": BAND + "_mask.mp4"}
            if args.backwards:
                data["bands"][BAND + "_mask_bwd"] = {"url": BAND + "_mask_bwd.mp4"}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--input", "-i", help="input", type=str, required=True)
    p.add_argument("--output", "-o", help="output", type=str, default="")
    p.add_argument("--subpath", help="path to flo files", type=str, default="")
    p.add_argument("--backwards", "-b", help="Backward video", action="store_true")
    p.add_argument("--mask", action="store_true", help="Compute mask as well")
    p.add_argument("--output_mask", help="output dense", type=str, default="")
    p.add_argument("--subpath_mask", help="path to flo files", type=str, default="")
    p.add_argument("--iterations", help="number of iterations", type=int, default=ITERATIONS)
    p.add_argument("--model", "-m", help="model path", type=str, default=MODEL)
    p.add_argument("--scale", type=float, default=0.75)
    p.add_argument("--raft_model", default="models/raft-things.pth", help="[RAFT] restore checkpoint")
    p.add_argument("--small", action="store_true", help="[RAFT] use small model")
    p.add_argument("--mixed_precision", action="store_true", help="[RAFT] use mixed precision")
    p.add_argument("--alternate_corr", action="store_true", help="[RAFT] use efficent correlation implementation")
    p.add_argument("--seeded-weights", action="store_true", help="seeded random weights (offline testing)")
    p.add_argument("--device", type=int, default=0)
    p.add_argument("--gpus", type=int, default=1, help="shard the frames over this many GPUs (one worker each, 1-frame halo)")
    p.add_argument("--device-list", type=str, default="", help="GPU ordinals of the workers (default 0..gpus-1)")
    return p


def main(argv=None):
    global data
    args = build_parser().parse_args(argv)
    if args.small:
        raise NotImplementedError("the small RAFT variant is commented out in the reference (raft.py:28-33) and not built")
    data = load_metadata(args.input)
    if data:
        args.input = get_url(args.input, data, "rgba")
        args.output = get_target(args.input, data, band=BAND, target=args.output)
        if args.mask:
            args.output_mask = get_target(args.input, data, band=BAND + "_mask")
    elif args.output == "":
        args.output = os.path.join(os.path.dirname(args.input), BAND + ".mp4")
    input_folder = os.path.dirname(args.input)
    for attr in ("subpath", "subpath_mask"):  # reference :208-218
        if getattr(args, attr) != "":
            setattr(args, attr, os.path.join(input_folder, getattr(args, attr)))
            os.makedirs(getattr(args, attr) + "_fwd", exist_ok=True)
            if args.backwards:
                os.makedirs(getattr(args, attr) + "_bwd", exist_ok=True)
    from bands.common.sharded import ENV_RANK, ShardContext, launch
    if args.gpus > 1 and ENV_RANK not in os.environ:
        devices = [int(d) for d in args.device_list.split(",")] if args.device_list else None
        launch(os.path.abspath(__file__), argv if argv is not None else sys.argv[1:], args.gpus, devices)
        return  # rank 0 of the workers wrote the videos, the csv and the metadata
    ctx = ShardContext.from_env(args.device)
    init_model(args)
    process_video(args, ctx)
    if ctx.is_writer():
        write_metadata(args.input, data)
    ctx.close()


if __name__ == "__main__":
    main()
