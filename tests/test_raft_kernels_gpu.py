"""GPU: the RAFT band's pointwise and gather kernels (raft_kernels.cu), each through its kernel-level C entry, against a
float64 reference computed from the kernel's own (fp32 or fp16-rounded) inputs.

Every bound is per element and derived from the kernel's arithmetic; u = 2^-24 is the fp32 unit roundoff and 2^-11 the fp16
one.  The entries fill their destinations with all-ones bytes (NaN) before the launch and return all of it, maps included in
the engine's shared-border layout (pixel (y, x) of image b at row b * img_rows + y (W + pad) + x), so each test also checks
that exactly the intended cells were written.  The reference helpers (`_*_ref`) are plain numpy / torch and run without a GPU.

Geometries are those the engine reaches: 1080p x 0.75 (stem 408 x 720, coarse 102 x 180), 720p x 0.75 (stem 272 x 480,
coarse 68 x 120) and a 270 x 481 frame (202 x 361 after scaling, padded [3, 4, 3, 3] to 208 x 368: coarse 26 x 46), plus
tiny ones; B up to 8 directions, the limit of DirFrames.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from prisma_b200._lib import check, fptr, lib

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24  # fp32 unit roundoff
U16 = 2.0 ** -11  # fp16 unit roundoff
SUB16 = 2.0 ** -25  # half the spacing of fp16 subnormals: the absolute rounding error below 2^-14
EPS = float(np.float32(1e-5))  # InstanceNorm2d eps, as the kernels take it: the fp32 1e-5f, widened to double

# (stem H, stem W) = the padded frame halved; coarse = stem / 4
STEM_1080P, STEM_720P, STEM_270X481 = (408, 720), (272, 480), (104, 184)
COARSE_1080P, COARSE_720P, COARSE_270X481 = (102, 180), (68, 120), (26, 46)


def _f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check_bound(out, ref, bound, what):
    err = np.abs(out.astype(np.float64) - ref)
    worst = float((err / bound).max())
    print(f"{what}: max|err| {err.max():.3e}, max err/bound {worst:.3f}")
    assert np.all(err <= bound), f"{what}: {int((err > bound).sum())} elements over the bound (worst ratio {worst:.2f})"
    return worst


def _check_written(out, mask, what):
    """mask = cells the kernel must write: no NaN (poison) left there, and poison untouched everywhere else."""
    assert not np.isnan(out[mask]).any(), f"{what}: {int(np.isnan(out[mask]).sum())} intended cells not written"
    assert np.isnan(out[~mask]).all(), f"{what}: {int((~np.isnan(out[~mask])).sum())} cells written outside the destination"


def _img_rows(H, W, pad):
    return -(-(H + pad) * (W + pad) // 32) * 32


def _pixel_rows(B, H, W, pad):
    """[B][H][W] map row of every interior pixel in the shared-border layout."""
    b, y, x = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), indexing="ij")
    return b * _img_rows(H, W, pad) + y * (W + pad) + x


def _interior(B, H, W, pad, C, cols=None):
    """Boolean [B * img_rows][C] mask of the interior pixels' cells (all columns, or `cols`)."""
    m = np.zeros((B * _img_rows(H, W, pad), C), bool)
    rows = _pixel_rows(B, H, W, pad).ravel()
    if cols is None:
        m[rows] = True
    else:
        m[np.ix_(rows, np.asarray(cols))] = True
    return m


def _coords(rng, B, H, W, max_flow):
    """coords0 = the pixel grid, coords1 = coords0 + a flow whose magnitudes spread log-uniformly over [1e-6, max_flow] with
    random signs; both [B][2][H][W] fp32."""
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    c0 = np.ascontiguousarray(np.broadcast_to(np.stack([xs, ys])[None], (B, 2, H, W)), np.float32)
    mag = np.exp(rng.uniform(np.log(1e-6), np.log(max_flow), (B, 2, H, W)))
    flow = mag * rng.choice([-1.0, 1.0], (B, 2, H, W))
    return c0, (c0 + flow).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------ stem im2col
def _stem_im2col_ref(x):
    """conv1 (7x7, stride 2, padding 3) im2col in the documented K order k = (c*7 + ky)*8 + kx: row b*Ho*Wo + oy*Wo + ox holds
    fp16(x[b, c, 2 oy - 3 + ky, 2 ox - 3 + kx]) (+0 outside the image); columns kx = 7 and k >= 168 are +0."""
    B, _, H, W = x.shape
    Ho, Wo = H // 2, W // 2
    xp = np.zeros((B, 3, H + 7, W + 7), np.float16)
    xp[:, :, 3:H + 3, 3:W + 3] = x.astype(np.float16)
    ref = np.zeros((B, Ho, Wo, 3, 7, 8), np.float16)
    for ky in range(7):
        for kx in range(7):
            ref[..., ky, kx] = xp[:, :, ky:ky + 2 * Ho:2, kx:kx + 2 * Wo:2].transpose(0, 2, 3, 1)
    out = np.zeros((B * Ho * Wo, 192), np.float16)
    out[:, :168] = ref.reshape(B * Ho * Wo, 168)
    return out.astype(np.float32)


@pytest.mark.parametrize("B,H,W", [
    (1, 2 * STEM_1080P[0], 2 * STEM_1080P[1]), (2, 2 * STEM_720P[0], 2 * STEM_720P[1]),
    (8, 2 * STEM_270X481[0], 2 * STEM_270X481[1]), (2, 16, 24), (8, 8, 8), (1, 2, 14)])
def test_stem_im2col_bit_exact(B, H, W):
    """Bit-exact against the numpy im2col, every border pixel included (the kernel's fast path needs the seven taps inside
    the row; the first and last output columns take the border path)."""
    rng = np.random.default_rng(B * H + W)
    x = (rng.standard_normal((B, 3, H, W), dtype=np.float32) * 1.5).astype(np.float32)
    x[:, :, ::5, ::3] = rng.uniform(-1e-6, 1e-6, x[:, :, ::5, ::3].shape)  # fp16 subnormals: round-to-nearest below 2^-14
    ref = _stem_im2col_ref(x)
    out = np.empty(ref.shape, np.float32)
    check(lib().prisma_debug_raft_stem_im2col(0, fptr(x), B, H, W, fptr(out)))
    _check_written(out, np.ones(out.shape, bool), "stem im2col")
    assert np.array_equal(_bits(out), _bits(ref)), f"stem im2col: {int((_bits(out) != _bits(ref)).sum())} cells differ"
    zero_cols = np.r_[np.arange(7, 168, 8), np.arange(168, 192)]
    assert np.all(_bits(out[:, zero_cols]) == 0)  # +0.0


# ------------------------------------------------------------------------------------------------------------------ statistics
def _stats_ref(S, Q, HW, eS, eQ):
    """float64 (mean, rstd) from sums S and sums of squares Q over HW pixels, and the bounds of a kernel whose S and Q are
    off by at most eS and eQ, which then forms var = Q/HW - mean^2 (clamped at 0) and 1/sqrt(var + eps) and rounds both
    to fp32: mean within eS/HW + u|mean|; rstd within the interval 1/sqrt(var +- dvar + eps), dvar = eQ/HW + (2|mean| +
    eS/HW) eS/HW, plus u rstd.  dvar grows as mean^2 (the one-pass E[x^2] - mean^2)."""
    mean = S / HW
    var = np.maximum(Q / HW - mean * mean, 0.0)
    rstd = 1.0 / np.sqrt(var + EPS)
    em = eS / HW
    dvar = eQ / HW + (2 * np.abs(mean) + em) * em + 8 * 2.0 ** -53 * (Q / HW + mean * mean)  # last: the double steps
    lo, hi = 1.0 / np.sqrt(var + dvar + EPS), 1.0 / np.sqrt(np.maximum(var - dvar, 0.0) + EPS)
    b_mean = em * (1 + U32) + U32 * np.abs(mean) + 1e-300
    b_rstd = np.maximum(hi - rstd, rstd - lo) * (1 + U32) + U32 * rstd
    return mean, rstd, b_mean, b_rstd


def _check_stats(stats, mean, rstd, b_mean, b_rstd, what):
    r1 = _check_bound(stats[..., 0], mean, b_mean, f"{what} mean")
    r2 = _check_bound(stats[..., 1], rstd, b_rstd, f"{what} rstd")
    return r1, r2


def _channels_with_ratios(rng, B, HW, C):
    """x [B][HW][C]: channel c has |mean|/std = RATIOS[c % 7] (0 ... 300), an all-zero channel (c % 7 == 5) or a constant
    channel (c % 7 == 6), with std spread over 1e-2 .. 1e2 across the channels."""
    ratios = np.array([0.0, 3.0, 30.0, 100.0, 300.0, 0.0, 0.0])
    kind = np.arange(C) % 7
    std = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), C))
    mean = ratios[kind] * std * rng.choice([-1.0, 1.0], C)
    x = mean + std * rng.standard_normal((B, HW, C))
    x[:, :, kind == 5] = 0.0
    x[:, :, kind == 6] = 1.3 * std[kind == 6]
    return x.astype(np.float32), kind, ratios


@pytest.mark.parametrize("B,HW,C", [
    (2, 300, 64), (1, 512, 64), (8, 513, 64), (1, STEM_1080P[0] * STEM_1080P[1], 64),
    (2, 300, 96), (2, 513, 96), (1, 512, 128), (2, 5000, 128)])
def test_instnorm_stats_dense(B, HW, C):
    """The stem's dense path: k_in_partial sums 512-row blocks in fp32 (each of blockDim / C thread groups runs a
    sequential sum over its rows, s += v and q = fmaf(v, v, q), then the groups are added: at most ceil(512 / groups) +
    groups roundings per partial), k_in_final adds the partials and forms the statistics in double.  So eS <= d u sum|x|
    and eQ <= d u sum x^2, d = ceil(512 / groups) + groups; the statistics bound follows (_stats_ref)."""
    rng = np.random.default_rng(B * HW + C)
    x, kind, ratios = _channels_with_ratios(rng, B, HW, C)
    stats = np.empty((B, C, 2), np.float32)
    check(lib().prisma_debug_instnorm_stats(0, fptr(x), B, HW, C, fptr(stats)))
    _check_written(stats, np.ones(stats.shape, bool), "instnorm stats")
    groups = (4 * C if C <= 64 else 2 * C) // C
    d = -(-512 // groups) + groups
    xd = x.astype(np.float64)
    S, Q = xd.sum(1), (xd * xd).sum(1)
    mean, rstd, b_mean, b_rstd = _stats_ref(S, Q, HW, d * U32 * np.abs(xd).sum(1), d * U32 * Q)
    _check_stats(stats, mean, rstd, b_mean, b_rstd, f"instnorm stats B{B} HW{HW} C{C}")
    rel = np.abs(stats[..., 1] - rstd) / rstd
    real = np.abs(mean) / np.sqrt(np.maximum(Q / HW - mean * mean, 1e-300))
    for k in (3, 4):
        sel = kind == k
        print(f"  |mean|/std {ratios[k]:.0f} (measured {real[:, sel].min():.0f}..{real[:, sel].max():.0f}): rstd relative "
              f"error vs float64 {rel[:, sel].max():.2e} (bound {(b_rstd / rstd)[:, sel].max():.2e})")
    # the all-zero channels: mean +0 exactly, rstd = fp32(1 / sqrt(eps)) computed in double
    assert np.all(_bits(stats[:, kind == 5, 0]) == 0)
    assert np.all(stats[:, kind == 5, 1] == np.float32(1.0 / np.sqrt(EPS)))


def _slab_partials(rng, B, spi, C):
    """fp32 per-slab (sum, sum of squares) of 32 pixel values each, [B*spi][2][C], with a per-image, per-channel mean
    of up to 30 standard deviations; some slabs empty (all zero), as the pad slabs of the conv epilogue are."""
    mean = rng.uniform(-30, 30, (B, 1, 1, C)) * rng.uniform(0.01, 2, (1, 1, 1, C))
    v = mean + rng.uniform(0.01, 2, (1, 1, 1, C)) * rng.standard_normal((B, spi, 32, C))
    v[:, ::7] = 0.0
    part = np.stack([v.sum(2), (v * v).sum(2)], axis=2)  # [B][spi][2][C]
    return part.reshape(B * spi, 2, C).astype(np.float32)


@pytest.mark.parametrize("B,spi,C", [
    (2, 40, 64),     # spi < 72: stage 1 leaves some of its 72 stripes empty
    (1, 72, 96),     # one slab per stripe
    (2, 1000, 128),  # 13 or 14 slabs per stripe: the stripes differ in length
    (2, 9216, 64),   # the stem-resolution map at 1080p: (409 * 721) rows in 9216 slabs of 32
    (8, 73, 96),     # one stripe of two slabs
    (1, 1, 128)])
def test_instnorm_slab_stats(B, spi, C):
    """Stage 1 adds stripes of slabs in double over 72 blocks per image, stage 2 adds the 72 partials in double and forms the
    statistics.  The reference is the float64 sum of the same fp32 partials, so the bound is the final fp32 rounding of mean
    and rstd plus the double additions."""
    rng = np.random.default_rng(B * spi + C)
    part = _slab_partials(rng, B, spi, C)
    HW = spi * 32 - 5
    stats = np.empty((B, C, 2), np.float32)
    check(lib().prisma_debug_instnorm_slab_stats(0, fptr(part), B, spi, C, HW, fptr(stats)))
    _check_written(stats, np.ones(stats.shape, bool), "slab stats")
    p = part.astype(np.float64).reshape(B, spi, 2, C)
    S, Q = p[:, :, 0].sum(1), p[:, :, 1].sum(1)
    dd = (spi + 80) * 2.0 ** -53
    mean, rstd, b_mean, b_rstd = _stats_ref(S, Q, HW, dd * np.abs(p[:, :, 0]).sum(1), dd * Q)
    _check_stats(stats, mean, rstd, b_mean, b_rstd, f"slab stats B{B} spi{spi} C{C}")


@pytest.mark.parametrize("sub,N", [(1, 64), (2, 128), (1, 96)])
def test_instnorm_slab_stats_of_a_conv(sub, N):
    """A real conv with the stat_part epilogue (ROW_PAD2TOK over a pad-1 shared-border map, as RaftEngine::add_conv_in runs
    it) chained into the slab statistics, against the float64 statistics of the conv's own fp32 output.  Each slab sum
    takes at most 34 fp32 roundings (test_gemm_epilogue_gpu.py), then the double stages."""
    from test_gemm_epilogue_gpu import (ROW_PAD2TOK, Geometry, conv_offsets, dev, fp16_values, make_ep, nan32, run_ok,
                                        upload_a16, upload_w16)
    rng = np.random.default_rng(90 + sub + N)
    src = Geometry(2, 2 * 23, 2 * 37, 1, shared=True, align32=True)
    Cin = 64
    A = src.embed(fp16_values(rng.standard_normal((src.B, src.H, src.W, Cin)) + 0.5))
    w = fp16_values(rng.standard_normal((N, 9, Cin)) / 24.0)
    bias = rng.uniform(-3, 3, N).astype(np.float32).astype(np.float64)
    Ho, Wo = src.H // sub, src.W // sub
    M = src.rows
    nslab = -(-M // 256) * 8  # the slabs of every tile, CTA-pair tiles included
    dense = nan32(src.B * Ho * Wo, N)
    part = torch.zeros((nslab + 8, 2 * N), dtype=torch.float32, device="cuda")
    ep = make_ep(bias=dev(bias), out_f32=dense, out_f32_ld=N, stat_part=part, row_map=ROW_PAD2TOK, **src.src_geom(sub))
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, M, N, conv_offsets(3, 3, src.Wp), ep)
    spi = src.img_rows // 32
    slab = np.ascontiguousarray(part.cpu().numpy()[:src.B * spi])
    y = dense.double().cpu().numpy().reshape(src.B, Ho * Wo, N)
    assert not np.isnan(y).any()
    stats = np.empty((src.B, N, 2), np.float32)
    check(lib().prisma_debug_instnorm_slab_stats(0, fptr(slab), src.B, spi, N, Ho * Wo, fptr(stats)))
    S, Q = y.sum(1), (y * y).sum(1)
    mean, rstd, b_mean, b_rstd = _stats_ref(S, Q, Ho * Wo, 34 * U32 * np.abs(y).sum(1), 34 * U32 * Q)
    _check_stats(stats, mean, rstd, b_mean, b_rstd, f"conv -> slab stats sub{sub} N{N}")


# ------------------------------------------------------------------------------------------------------------------ apply
def _apply_ref(x, stats, skip_kind, skip, skip_stats):
    """float64 relu(skip + relu((x - mean) rstd)) from the kernel's fp32 x and statistics (skip: fp16-rounded map, or raw
    fp32 normalised with its own statistics), and the bound: (x - m) and the product r: 2 fp32 roundings; the skip add 1
    (fp16 map) or the skip's own 2 plus the add (raw); then the fp16 output (2^-11 |y| or 2^-25 below 2^-14)."""
    m, r = stats[..., 0].astype(np.float64)[:, None, None], stats[..., 1].astype(np.float64)[:, None, None]
    t = (x.astype(np.float64) - m) * r
    y = np.maximum(t, 0.0)
    e = 2.01 * U32 * np.abs(t)
    if skip_kind == 1:
        s = y + skip.astype(np.float64)
        y, e = np.maximum(s, 0.0), e + 1.01 * U32 * np.abs(s)
    elif skip_kind == 2:
        sm, sr = skip_stats[..., 0].astype(np.float64)[:, None, None], skip_stats[..., 1].astype(np.float64)[:, None, None]
        t2 = (skip.astype(np.float64) - sm) * sr
        s = y + t2
        y, e = np.maximum(s, 0.0), e + 2.01 * U32 * np.abs(t2) + 1.01 * U32 * np.abs(s)
    return y, e + U16 * (y + e) + SUB16


@pytest.mark.parametrize("B,H,W,C,skip_kind", [
    (1, *STEM_1080P, 64, 0), (2, *STEM_720P, 64, 1), (2, 68, 120, 64, 2),
    (2, 136, 240, 96, 0), (8, 52, 92, 96, 1), (2, 136, 240, 96, 2),
    (2, *COARSE_720P, 128, 0), (2, *COARSE_270X481, 128, 1), (8, 2, 3, 128, 2), (3, 1, 1, 64, 1)])
def test_instnorm_apply(B, H, W, C, skip_kind):
    """Normalise + ReLU (+ skip, + ReLU) into a pad-1 fp16 map: only the interior is written; pad columns, pad rows and
    tail rows keep their fill."""
    rng = np.random.default_rng(B * H * W + C + skip_kind)
    mu = rng.uniform(-5, 5, (B, C))
    sd = rng.uniform(0.05, 4, (B, C))
    x = (mu[:, None, None] + sd[:, None, None] * rng.standard_normal((B, H, W, C))).astype(np.float32)
    stats = np.stack([mu, 1.0 / sd], -1).astype(np.float32)
    skip = skip_stats = None
    if skip_kind == 1:
        skip = _f16(np.maximum(rng.standard_normal((B, H, W, C)), 0) * 2)
    elif skip_kind == 2:
        smu, ssd = rng.uniform(-2, 2, (B, C)), rng.uniform(0.1, 3, (B, C))
        skip = (smu[:, None, None] + ssd[:, None, None] * rng.standard_normal((B, H, W, C))).astype(np.float32)
        skip_stats = np.stack([smu, 1.0 / ssd], -1).astype(np.float32)
    out = np.empty((B * _img_rows(H, W, 1), C), np.float32)
    check(lib().prisma_debug_instnorm_apply(0, fptr(x), fptr(stats), B, H, W, C, skip_kind, fptr(skip), fptr(skip_stats),
                                            fptr(out)))
    _check_written(out, _interior(B, H, W, 1, C), "instnorm apply")
    ref, bound = _apply_ref(x, stats, skip_kind, skip, skip_stats)
    got = out[_pixel_rows(B, H, W, 1)]
    _check_bound(got, ref, bound, f"instnorm apply B{B} {H}x{W} C{C} skip{skip_kind}")


# ------------------------------------------------------------------------------------------------------------------ GRU operands
@pytest.mark.parametrize("B,H,W,frames", [
    (2, *COARSE_1080P, [0, 1]), (8, *COARSE_720P, [0, 1, 1, 2, 2, 3, 3, 4]), (8, *COARSE_270X481, list(range(8))),
    (4, 2, 3, [0, 1, 1, 2]), (8, 1, 1, [0, 1, 1, 2, 2, 3, 3, 4])])
def test_gru_operands(B, H, W, frames):
    """cnet split then flow columns on the NaN-filled pad-2 GRU operand maps.  Direction b reads the context features of
    frame frames[b] (the clip layout [0, 1, 1, 2, ...] is not the identity).  h_master = tanhf(net) within tanhf's 2 ulp
    of float64 tanh; hx[:, :128] = fp16(h_master) bit for bit, so within one fp16 ulp of fp16(tanh); the ReLU half
    (hx and rhx channels 128..255) and the flow columns 382..383 (fp16 of the fp32 c1 - c0) bit-exact.  Exactly hx channels
    0..255 and 382..383, rhx channels 128..255 and 382..383 and h_master's interior are written."""
    rng = np.random.default_rng(B * H * W + sum(frames))
    F = max(frames) + 1
    P = H * W
    cn = (rng.standard_normal((F, P, 256)) * 3).astype(np.float32)
    cn[:, ::5, ::3] = 0.0
    cn[:, 1::7, :128] *= 10  # tanh saturation
    c0, c1 = _coords(rng, B, H, W, 300.0)
    ir = _img_rows(H, W, 2)
    hm = np.empty((B * ir, 128), np.float32)
    hx = np.empty((B * ir, 384), np.float32)
    rhx = np.empty((B * ir, 384), np.float32)
    df = (C.c_int * B)(*frames)
    check(lib().prisma_debug_raft_gru_operands(0, fptr(cn), F, B, H, W, df, fptr(c0), fptr(c1), fptr(hm), fptr(hx), fptr(rhx)))
    _check_written(hm, _interior(B, H, W, 2, 128), "h_master")
    _check_written(hx, _interior(B, H, W, 2, 384, np.r_[0:256, 382, 383]), "hx")
    _check_written(rhx, _interior(B, H, W, 2, 384, np.r_[128:256, 382, 383]), "rhx")
    rows = _pixel_rows(B, H, W, 2).reshape(B, P)
    src = cn[np.asarray(frames)]  # [B][P][256]
    t = np.tanh(src[..., :128].astype(np.float64))
    h = hm[rows]
    _check_bound(h, t, 2 * np.spacing(np.abs(t).astype(np.float32)).astype(np.float64), f"h_master B{B} {H}x{W}")
    hxi, rhxi = hx[rows], rhx[rows]
    assert np.array_equal(_bits(hxi[..., :128]), _bits(_f16(h)))
    ft = _f16(t)
    assert np.all(np.abs(hxi[..., :128] - ft) <= np.spacing(np.abs(ft).astype(np.float16)).astype(np.float32))
    relu = _f16(np.maximum(src[..., 128:], 0))
    assert np.array_equal(_bits(hxi[..., 128:256]), _bits(relu))
    assert np.array_equal(_bits(rhxi[..., 128:256]), _bits(relu))
    flow = _f16((c1 - c0).reshape(B, 2, P).transpose(0, 2, 1))
    assert np.array_equal(_bits(hxi[..., 382:]), _bits(flow))
    assert np.array_equal(_bits(rhxi[..., 382:]), _bits(flow))


# ------------------------------------------------------------------------------------------------------------------ flow im2col
def _flow_im2col_ref(c0, c1):
    """convf1's im2col: row b*H*W + y*W + x, k = ch*49 + ky*7 + kx < 98 holds v = fp32(c1 - c0) at (y + ky - 3, x + kx - 3)
    (0 outside), split hi = fp16(v) in columns [0, 98) and lo = fp16(v - hi) (fp32 difference) in [128, 226); the rest +0.
    Returns (out, v)."""
    B, _, H, W = c0.shape
    v = (c1 - c0).astype(np.float32)
    vp = np.zeros((B, 2, H + 6, W + 6), np.float32)
    vp[:, :, 3:H + 3, 3:W + 3] = v
    taps = np.zeros((B, H, W, 2, 7, 7), np.float32)
    for ky in range(7):
        for kx in range(7):
            taps[..., ky, kx] = vp[:, :, ky:ky + H, kx:kx + W].transpose(0, 2, 3, 1)
    taps = taps.reshape(B * H * W, 98)
    hi = _f16(taps)
    lo = _f16(taps - hi)
    out = np.zeros((B * H * W, 256), np.float32)
    out[:, :98], out[:, 128:226] = hi, lo
    return out, taps


@pytest.mark.parametrize("B,H,W", [
    (2, *COARSE_1080P), (8, *COARSE_720P), (4, *COARSE_270X481), (8, 2, 3), (3, 1, 1), (2, 5, 9)])
def test_flow_im2col_hi_lo(B, H, W):
    """hi == fp16(v) and lo == fp16(v - hi) bit for bit for flows from 1e-6 to 300 px of either sign, every border, the zero
    columns 98..127 and 226..255 (+0); and hi + lo within 2^-22 |v| + 2^-25 of v (lo's own rounding: relative 2^-11 of a
    remainder below 2^-11 |v|, or the fp16 subnormal spacing)."""
    rng = np.random.default_rng(B * H + W)
    c0, c1 = _coords(rng, B, H, W, 300.0)
    ref, v = _flow_im2col_ref(c0, c1)
    out = np.empty(ref.shape, np.float32)
    check(lib().prisma_debug_raft_flow_im2col(0, fptr(c0), fptr(c1), B, H, W, fptr(out)))
    _check_written(out, np.ones(out.shape, bool), "flow im2col")
    assert np.array_equal(_bits(out), _bits(ref)), f"flow im2col: {int((_bits(out) != _bits(ref)).sum())} cells differ"
    assert np.all(_bits(out[:, np.r_[98:128, 226:256]]) == 0)
    s = out[:, :98].astype(np.float64) + out[:, 128:226]
    bound = 2.0 ** -22 * np.abs(v) + SUB16
    _check_bound(s, v.astype(np.float64), bound, f"flow im2col hi + lo B{B} {H}x{W}")
    miss = np.abs(out[:, :98] - v.astype(np.float64)) > bound
    assert miss[v != 0].mean() > 0.3  # hi alone misses the bound for most taps: the lo half is needed


# ------------------------------------------------------------------------------------------------------------------ FlowHead gather
def _flow_head2_ref(u, b0, b1, coords1):
    """coords1 + (b0, b1) + sum over the 3x3 taps t of u[p + t][2t + o] (zero outside the image), float64; bound: the kernel's
    9 tap additions and the final one, 10 fp32 roundings of partial sums at most |b| + sum|u| + |coords1|."""
    B, H, W, _ = u.shape
    ud = np.zeros((B, H + 2, W + 2, 18))
    ud[:, 1:H + 1, 1:W + 1] = u[..., :18]
    acc = np.zeros((B, H, W, 2))
    mag = np.zeros((B, H, W, 2))
    for t in range(9):
        dy, dx = t // 3, t % 3
        tap = ud[:, dy:dy + H, dx:dx + W, 2 * t:2 * t + 2]
        acc += tap
        mag += np.abs(tap)
    bias = np.array([b0, b1], np.float64)
    c = coords1.astype(np.float64).transpose(0, 2, 3, 1)
    ref = c + bias + acc
    bound = 10 * U32 * (np.abs(bias) + mag + np.abs(c)) + 1e-38
    return ref.transpose(0, 3, 1, 2), bound.transpose(0, 3, 1, 2)


@pytest.mark.parametrize("B,H,W", [(3, *COARSE_1080P), (3, *COARSE_270X481), (3, 1, 1), (3, 2, 3), (8, 4, 5)])
def test_flow_head2_gather(B, H, W):
    """B >= 3, so the top taps of images 1 and 2 read the previous image's pad and tail rows (zero in the map, as the 1x1
    GEMM leaves them) and image 0's skip the rows before the map.  Columns 18..31 of u are NaN: never read."""
    rng = np.random.default_rng(B * H * W + 7)
    u = (rng.standard_normal((B, H, W, 32)) * rng.uniform(0.1, 3, (B, H, W, 1))).astype(np.float32)
    u[..., 18:] = np.nan
    b0, b1 = np.float32(0.3125), np.float32(-1.7)
    c0, c1 = _coords(rng, B, H, W, 50.0)
    out = np.empty_like(c1)
    check(lib().prisma_debug_raft_flow_head2(0, fptr(u), B, H, W, float(b0), float(b1), fptr(c1), fptr(out)))
    _check_written(out, np.ones(out.shape, bool), "flow head2")
    ref, bound = _flow_head2_ref(u, float(b0), float(b1), c1)
    _check_bound(out, ref, bound, f"flow head2 B{B} {H}x{W}")


# ------------------------------------------------------------------------------------------------------------------ convex up-sampling
def _convex_upsample_ref(mask, c0, c1, Hs, Ws, pad_top, pad_left):
    """oracle.raft.upsample_flow in float64 on the kernel's fp32 flow c1 - c0, cropped to rows pad_top .. pad_top + Hs and
    columns pad_left .. pad_left + Ws, [B][Hs][Ws][2]; bound: the softmax weights p_k = exp(w_k - max) / sum are off by a
    relative 2E + 9u (E = u max_k |w_k - max| for the fp32 argument plus expf's 2 ulp; the 9-term sum and the division), and
    the 9-tap sum of p_k 8 flow_k takes at most 11 more roundings: (2E + 20u) sum_k p_k 8 |flow_k|."""
    from oracle import raft as oraft
    B, H, W, _ = mask.shape
    flow = torch.from_numpy((c1 - c0).astype(np.float32).astype(np.float64))
    m = torch.from_numpy(mask.astype(np.float64)).permute(0, 3, 1, 2)
    with torch.no_grad():
        up = oraft.upsample_flow(flow, m)
        mag = oraft.upsample_flow(flow.abs(), m)  # sum_k p_k 8 |flow_k|
    w = mask.astype(np.float64).reshape(B, H, W, 9, 64)
    E = U32 * (w.max(3) - w.min(3)) + 4 * U32  # [B][H][W][64], sub-pixel a*8 + b
    E = torch.from_numpy(E).permute(0, 3, 1, 2).reshape(B, 1, 8, 8, H, W).permute(0, 1, 4, 2, 5, 3).reshape(B, 1, 8 * H, 8 * W)
    bound = (2 * E + 20 * U32) * mag + 1e-36
    crop = lambda t: t[:, :, pad_top:pad_top + Hs, pad_left:pad_left + Ws].permute(0, 2, 3, 1).numpy()
    return crop(up), crop(bound.expand(-1, 2, -1, -1))


def _upsample_mask(rng, B, H, W):
    """Logits [B][H][W][576] (channel k*64 + a*8 + b): random with spreads up to ~120 across the nine k (exp underflows
    fp32 for the smallest), and every fifth pixel with nine equal logits (uniform weights)."""
    spread = rng.choice([0.5, 5.0, 40.0, 120.0], (B, H, W, 1, 64))
    m = rng.uniform(-0.5, 0.5, (B, H, W, 9, 64)) * spread
    flat = m.reshape(B, H * W, 9, 64)
    flat[:, ::5] = rng.uniform(-3, 3, (B, flat[:, ::5].shape[1], 1, 64))
    return np.ascontiguousarray(flat.reshape(B, H, W, 576), np.float32)


def _run_convex(B, H, W, Hs, Ws, pad_top, pad_left, seed, max_flow=30.0):
    rng = np.random.default_rng(seed)
    mask = _upsample_mask(rng, B, H, W)
    c0, c1 = _coords(rng, B, H, W, max_flow)
    out = np.empty((B, Hs, Ws, 2), np.float32)
    check(lib().prisma_debug_raft_convex_upsample(0, fptr(mask), fptr(c0), fptr(c1), B, H, W, Hs, Ws, pad_top, pad_left,
                                                  fptr(out)))
    # each output cell comes from one (coarse pixel, sub-pixel) (the crop is a shift), so every cell written and equal to the
    # reference value of that one source is every cell written exactly once
    _check_written(out, np.ones(out.shape, bool), "convex upsample")
    ref, bound = _convex_upsample_ref(mask, c0, c1, Hs, Ws, pad_top, pad_left)
    return _check_bound(out, ref, bound, f"convex upsample B{B} {H}x{W} -> {Hs}x{Ws} pad ({pad_top}, {pad_left})")


@pytest.mark.parametrize("pad_top", [0, 1, 2, 3])
@pytest.mark.parametrize("pad_left", [0, 1, 2, 3])
def test_convex_upsample_crop(pad_top, pad_left):
    """Every (pad_top, pad_left) InputPadder can give, with bottom / right pads from 0 to 4."""
    H, W = 5, 7
    pad_bottom, pad_right = (pad_top + 2 * pad_left) % 5, (3 * pad_top + pad_left + 1) % 5
    _run_convex(2, H, W, 8 * H - pad_top - pad_bottom, 8 * W - pad_left - pad_right, pad_top, pad_left, 10 * pad_top + pad_left)


@pytest.mark.parametrize("B,H,W,Hs,Ws,pad_top,pad_left", [
    (2, *COARSE_270X481, 202, 361, 3, 3),   # 270 x 481 x 0.75: pads [left 3, right 4, top 3, bottom 3]
    (2, *COARSE_1080P, 810, 1440, 3, 0),   # 1080p x 0.75: pads [0, 0, 3, 3]
    (8, *COARSE_720P, 540, 960, 2, 0),     # 720p x 0.75: pads [0, 0, 2, 2]
    (8, 1, 1, 5, 4, 1, 2)])
def test_convex_upsample_engine_geometries(B, H, W, Hs, Ws, pad_top, pad_left):
    _run_convex(B, H, W, Hs, Ws, pad_top, pad_left, B * H * W, max_flow=300.0)


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_raft_pair_with_left_pad_matches_oracle():
    """A 270 x 481 frame pair scales to 202 x 361, which InputPadder pads on all four sides ([3, 4, 3, 3]): the convex
    up-sampler's row and column crops both run.  Forward and backward flow against the oracle at the band's 1e-3 of the
    largest displacement."""
    from oracle import raft as oraft
    from prisma_b200.flow import RaftFlowEngine
    from prisma_b200.seeded_weights import make_raft_weights
    from prisma_b200.synthetic import synthetic_frame
    from test_raft_gpu import _oracle, _rel
    H, W = 270, 481
    eng = RaftFlowEngine(make_raft_weights(0), iterations=12, scale=0.75)
    f0, f1 = synthetic_frame(H, W, 0), synthetic_frame(H, W, 1)
    out = eng.infer_pair(f0, f1)
    hs, ws = eng.out_size(H, W)
    rs = eng.read_tap("resized", (2, hs, ws, 3)).astype(np.uint8)
    eng.close()
    pad = oraft.input_pad(hs, ws)
    assert (hs, ws) == (202, 361) and all(p > 0 for p in pad), pad
    _, _, up = _oracle(f0, f1, rs[0], rs[1], 12)
    fwd_ref = up[0].permute(1, 2, 0).numpy()
    bwd_ref = up[1].permute(1, 2, 0).numpy()
    assert out["fwd"].shape == fwd_ref.shape == (202, 361, 2)
    r = (_rel(out["fwd"], fwd_ref), _rel(out["bwd"], bwd_ref))
    print("270x481 raft: fwd", r[0], "bwd", r[1], "max|flow|", float(np.abs(fwd_ref).max()))
    assert r[0][0] <= 1e-3 and r[1][0] <= 1e-3, r
