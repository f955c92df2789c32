"""How much of each RAFT update-block GEMM is its epilogue: every update-block launch of the bench geometry (1080p x 0.75,
4 pairs per pass, forward and backward: 8 images of 102 x 180 at 1/8 scale in shared-border pad-2 maps, M = 151 552 rows)
runs through prisma_debug_gemm_ep twice -- with its real epilogue, and with its destinations (and the ConvGRU gate inputs)
removed, so that it still reads the accumulators and applies bias and activation but loads and stores nothing.  The
difference of the two kernel times is the epilogue time the MMAs do not hide.

    python tools/gemm_epilogue_pace.py [--bn 0 128 256] [--reps 10] [--out FILE.json]

Kernel times come from torch.profiler (CUDA activities), the mean over --reps launches after one warm-up launch.  The library
is the one prisma_b200._lib loads (PRISMA_B200_LIB selects another build, e.g. to compare two trees).  Needs an H100.
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch
from torch.autograd import DeviceType

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from prisma_b200._lib import DebugEpilogue, lib  # noqa: E402

ROW_PADDED, ROW_TOK2PAD = 1, 2
B, H8, W8, PAD = 8, 102, 180, 2
HP, WP = H8 + PAD, W8 + PAD              # shared border: pad zero rows / columns after every image / row
IMG_ROWS = (HP * WP + 31) // 32 * 32     # image row counts are multiples of 32
M = B * IMG_ROWS                         # 151 552
GEOM = dict(row_map=ROW_PADDED, img_rows=IMG_ROWS, in_w=WP, in_h=HP, pad=PAD, lead=0, out_lead=0)

# name, input channels, (kh, kw), taps per position (hi / lo weight slabs), N, epilogue kind
LAUNCHES = [
    ("convc1", 384, (1, 1), 1, 256, "relu_f16"),
    ("convc2", 256, (3, 3), 1, 192, "relu_f16"),
    ("convf1", 256, None, 1, 128, "tok2pad"),
    ("convf2", 128, (3, 3), 1, 64, "relu_f16"),
    ("motion_conv", 256, (3, 3), 1, 128, "relu_copy"),
    ("gru_zr", 384, (1, 5), 1, 256, "gru1"),
    ("gru_q", 384, (5, 1), 1, 128, "gru2"),
    ("flow_head1", 128, (3, 3), 1, 256, "relu_f16"),
    ("flow_head2", 256, (1, 1), 2, 20, "f32"),
]


def _offsets(khw, split):
    if khw is None:
        return [0]
    kh, kw = khw
    return [(ky - kh // 2) * WP + (kx - kw // 2) for ky in range(kh) for kx in range(kw) for _ in range(split)]


def _epilogue(kind, N, real, bufs):
    """DebugEpilogue of one launch; real=False keeps bias, activation and row mapping but no destination or gate input."""
    f = dict(bias=bufs["bias"].data_ptr(), act=2)
    if kind == "tok2pad":
        f.update(row_map=ROW_TOK2PAD, in_w=W8, in_h=H8, out_wp=WP, out_img_rows=IMG_ROWS, out_pad=PAD, out_lead=0)
    else:
        f.update(GEOM)
    if kind == "gru1":
        f["act"] = 3
    elif kind == "gru2":
        f["act"] = 4
    elif kind == "f32":
        f["act"] = 0
    if not real:
        return DebugEpilogue(**f)
    if kind in ("relu_f16", "tok2pad"):
        f.update(out_f16=bufs["f16"].data_ptr(), out_f16_ld=256 if kind == "relu_f16" else 128)
    elif kind == "relu_copy":
        f.update(out_f16=bufs["f16_384"].data_ptr(), out_f16_ld=384, out_f16_relu=bufs["f16_384b"].data_ptr(), out_f16_relu_ld=384)
    elif kind == "gru1":
        f.update(out_f32=bufs["f32_256"].data_ptr(), out_f32_ld=256, gru=1, gru_h=bufs["h"].data_ptr(),
                 gru_rh=bufs["f16_384b"].data_ptr(), gru_rh_ld=384)
    elif kind == "gru2":
        f.update(out_f32=bufs["h"].data_ptr(), out_f32_ld=128, out_f16=bufs["f16_384"].data_ptr(), out_f16_ld=384, gru=2,
                 gru_h=bufs["h"].data_ptr(), gru_z=bufs["f32_256"].data_ptr())
    elif kind == "f32":
        f.update(out_f32=bufs["f32_256"].data_ptr(), out_f32_ld=32)
    return DebugEpilogue(**f)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--bn", type=int, nargs="+", default=[0, 128, 256], help="tile widths to force (0 = the library's choice)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_epilogue_pace needs an H100"
    L = lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    A = (torch.rand((M, 384), generator=g, device="cuda") - 0.5).half()
    W = ((torch.rand((256, 5 * 384 * 2), generator=g, device="cuda") - 0.5) / 16).half()
    bufs = dict(bias=torch.rand(256, device="cuda") - 0.5,
                f16=torch.zeros((M, 256), dtype=torch.float16, device="cuda"),
                f16_384=torch.zeros((M, 384), dtype=torch.float16, device="cuda"),
                f16_384b=torch.zeros((M, 384), dtype=torch.float16, device="cuda"),
                f32_256=torch.rand((M, 256), generator=g, device="cuda"),
                h=torch.rand((M, 128), generator=g, device="cuda") - 0.5)
    results = []
    print(f"{'launch':12s} {'bn':>4s} {'real us':>9s} {'no-dst us':>9s} {'exposed us':>10s} {'TFLOP/s':>8s}")
    for name, cin, khw, split, N, kind in LAUNCHES:
        offs = _offsets(khw, split)
        a_rows, m = (B * H8 * W8, B * H8 * W8) if kind == "tok2pad" else (M, M)
        K = len(offs) * cin
        wk = W[:, :K].contiguous()
        offs_c = (C.c_int * len(offs))(*offs)
        for bn in a.bn:
            if bn == 256 and N <= 128:
                continue
            times = {}
            for real in (True, False):
                ep = _epilogue(kind, N, real, bufs)

                def launch():
                    rc = L.prisma_debug_gemm_ep(0, A.data_ptr(), a_rows, cin, 384, wk.data_ptr(), 256, m, N, len(offs), offs_c,
                                                bn, 0, 0, C.byref(ep))
                    assert rc == 0, L.prisma_last_error().decode()
                launch()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.reps):
                        launch()
                ks = [e for e in prof.events() if "gemm_tc_kernel" in e.name and e.device_type == DeviceType.CUDA]
                assert len(ks) == a.reps, [e.name for e in prof.events()][:8]
                times[real] = sum(e.time_range.elapsed_us() for e in ks) / len(ks)
            flop = 2.0 * B * H8 * W8 * K * N
            r = dict(launch=name, bn=bn, N=N, K=K, real_us=times[True], no_dst_us=times[False],
                     exposed_us=times[True] - times[False], tflops=flop / times[True] / 1e6)
            results.append(r)
            print(f"{name:12s} {bn:4d} {r['real_us']:9.1f} {r['no_dst_us']:9.1f} {r['exposed_us']:10.1f} {r['tflops']:8.1f}")
    for bn in a.bn:
        rs = [r for r in results if r["bn"] == bn]
        print(f"bn {bn}: sum real {sum(r['real_us'] for r in rs):.1f} us, exposed {sum(r['exposed_us'] for r in rs):.1f} us "
              f"over {len(rs)} launches")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(0), results=results), f, indent=1)


if __name__ == "__main__":
    main()
