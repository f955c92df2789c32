"""GPU: the ViT-encoder and DPT-resampling kernels of the depth bands, each through its kernel-level C entry, against a
float64 reference computed from the kernel's own (fp16-rounded) inputs.

Every bound is per element and derived from the kernel's arithmetic; u = 2^-24 is the fp32 unit roundoff and 2^-11 the fp16
one.  The entries fill their destinations with all-ones bytes (NaN) before the launch and return all of it, so each test
also checks that exactly the intended cells were written.  The reference helpers (`_*_ref`) are plain numpy / torch and run
without a GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from prisma_b200._lib import check, fptr, lib

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24  # fp32 unit roundoff
U16 = 2.0 ** -11  # fp16 unit roundoff
SUB16 = 2.0 ** -25  # half the spacing of fp16 subnormals: the absolute rounding error below 2^-14


def _f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


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


# ------------------------------------------------------------------------------------------------------------------ attention
def _attention_ref(qkv16, batch, T, heads):
    """float64 softmax(q k^T) v per image and head from the kernel's fp16 operands (q = fp16(q * 1/8), as the entry scales it),
    with the per-element bound of the kernel's arithmetic:
      * P is rounded to fp16 for the PV product (relative 2^-11 on each p; absolute 2^-25 below 2^-14) while the row sum
        l = sum p stays fp32:  (2^-11 sum p|v| + 2^-25 sum_{p < 2^-13} |v|) / sum p;
      * the scores come from a 64-term fp32 MMA sum (error ds <= 16 u sum|q||k|) and feed ex2.approx through
        s * log2e - m * log2e in fp32 (de <= 8 u max|s|): p moves by a relative 2 (ds + de);
      * l sums n keys in fp32 (n u); O accumulates 9 fp32 steps per KV tile plus the rescales ((9 tiles + 8) 2^-23);
      * the output is rounded to fp16 (2^-11 |o|, or 2^-25 below 2^-14).
    Returns ref [batch*T][D], bound [batch*T][D]."""
    D = heads * 64
    x = qkv16.reshape(batch, T, 3, heads, 64).astype(np.float64)
    q = _f16(qkv16.reshape(batch, T, 3, heads, 64)[:, :, 0] * np.float32(0.125)).astype(np.float64)
    k, v = x[:, :, 1], x[:, :, 2]
    ref = np.empty((batch, T, heads, 64))
    bound = np.empty((batch, T, heads, 64))
    n_tiles = -(-T // 128)
    c_acc = T * U32 + (9 * n_tiles + 8) * 2 * U32 + 2 * U32
    for b in range(batch):
        for h in range(heads):
            qq, kk, vv = q[b, :, h], k[b, :, h], v[b, :, h]
            s = qq @ kk.T
            m = s.max(axis=1, keepdims=True)
            p = np.exp(s - m)
            l = p.sum(axis=1, keepdims=True)
            av = np.abs(vv)
            pv = p @ av
            ds = 16 * U32 * (np.abs(qq) @ np.abs(kk).T).max(axis=1, keepdims=True)
            de = 8 * U32 * np.abs(s).max(axis=1, keepdims=True)
            o = (p @ vv) / l
            ref[b, :, h] = o
            bound[b, :, h] = ((U16 + 2 * (ds + de) + c_acc) * pv + SUB16 * ((p < 2.0 ** -13) @ av)) / l \
                + U16 * np.abs(o) + SUB16
    return ref.reshape(batch * T, D), bound.reshape(batch * T, D)


def _run_attention(qkv, batch, T, heads):
    out = np.empty((batch * T, heads * 64), np.float32)
    ms = C.c_float()
    check(lib().prisma_debug_attention_batch(0, fptr(qkv), fptr(out), batch, T, heads, 1, C.byref(ms)))
    return out


def _random_qkv(rng, batch, T, heads, scale=1.0):
    return _f16(rng.standard_normal((batch * T, 3 * heads * 64), dtype=np.float32) * scale)


@pytest.mark.parametrize("batch,T,heads", [
    (1, 5, 6), (2, 5, 16), (3, 127, 12), (2, 128, 6), (3, 129, 16), (1, 129, 12),
    (2, 1370, 6), (3, 1370, 12), (1, 1370, 16), (2, 2443, 16), (3, 2443, 6), (1, 127, 6)])
def test_attention_random(batch, T, heads):
    rng = np.random.default_rng(1000 * batch + T + heads)
    qkv = _random_qkv(rng, batch, T, heads, 1.5)
    out = _run_attention(qkv, batch, T, heads)
    _check_written(out, np.ones(out.shape, bool), "attention")
    ref, bound = _attention_ref(qkv, batch, T, heads)
    _check_bound(out, ref, bound, f"attention b{batch} T{T} h{heads}")


@pytest.mark.parametrize("batch,T,heads", [(2, 129, 6), (3, 1370, 12), (2, 5, 16), (3, 2443, 6)])
def test_attention_no_leak_across_images(batch, T, heads):
    """In image b+1, the first keys score far above everything image b's queries see (s ~ +12 vs |s| < 1) and carry
    v = 60.  Keys of image b+1 sit in image b's last ragged KV tile and queries of image b+1 in its trailing query tile:
    any attention across the boundary moves image b's output by tens."""
    rng = np.random.default_rng(T + heads)
    D = heads * 64
    qkv = (rng.standard_normal((batch, T, 3, heads, 64), dtype=np.float32) * 0.3)
    u = np.zeros(64, np.float32); u[7] = 1.0
    qkv[:, :, 0] += 4.0 * u          # every query points along u (score 0.125 * 4 * 24 = 12 with a planted key)
    n_leak = min(4, T)
    for b in range(1, batch):
        qkv[b, :n_leak, 1] = 24.0 * u  # planted keys: first rows of image b+1
        qkv[b, :n_leak, 2] = 60.0
    qkv = _f16(qkv.reshape(batch * T, 3 * D))
    out = _run_attention(qkv, batch, T, heads)
    _check_written(out, np.ones(out.shape, bool), "attention leak")
    ref, bound = _attention_ref(qkv, batch, T, heads)
    _check_bound(out, ref, bound, f"attention leak b{batch} T{T}")
    assert np.abs(out[:T]).max() < 5.0  # image 0 never sees a planted key


@pytest.mark.parametrize("batch,T,heads", [(2, 1370, 6), (3, 129, 12), (1, 2443, 16)])
def test_attention_online_softmax_rescaling(batch, T, heads):
    """Per row the largest score sits either in the first KV tile (key 0) or in the last, ragged one (key T-1), so both the
    alpha = 1 and the alpha << 1 paths of the online softmax run; the spread of the scaled scores reaches ~90, so
    exp underflows fp16 (and fp32) for most keys of those rows."""
    rng = np.random.default_rng(7 * T + heads)
    D = heads * 64
    qkv = rng.standard_normal((batch, T, 3, heads, 64), dtype=np.float32) * 0.5
    u1 = np.zeros(64, np.float32); u1[3] = 1.0
    u2 = np.zeros(64, np.float32); u2[40] = 1.0
    qkv[:, 0, 1] = 24.0 * u1
    qkv[:, T - 1, 1] = 24.0 * u2
    amp = np.linspace(0.0, 30.0, T, dtype=np.float32)          # 0.125 * 30 * 24 = 90
    row_dir = np.where((np.arange(T) % 2 == 0)[:, None], u1, u2)  # even rows: max in tile 0; odd rows: in the last tile
    qkv[:, :, 0] += (amp[:, None] * row_dir)[None, :, None, :]
    qkv = _f16(qkv.reshape(batch * T, 3 * D))
    out = _run_attention(qkv, batch, T, heads)
    _check_written(out, np.ones(out.shape, bool), "attention rescale")
    ref, bound = _attention_ref(qkv, batch, T, heads)
    _check_bound(out, ref, bound, f"attention rescale b{batch} T{T}")


# ------------------------------------------------------------------------------------------------------------------ LayerNorm
def _layernorm_ref(x_rows, g, b):
    """float64 LayerNorm (eps 1e-6) of fp32 rows, and the bound of the kernel's fp32 statistics + fp16 output:
      mean: 32 sequential + 5 butterfly fp32 adds and the 1/D product: dm <= 40 u mean|x|;
      rstd: squares summed the same way, rsqrtf (2 ulp), /D: relative dr <= 48 u;
      y = (x - m) rstd g + b: 4 fp32 roundings, then fp16 (2^-11 |y|, or 2^-25 below 2^-14)."""
    x = torch.from_numpy(x_rows.astype(np.float64))
    D = x.shape[1]
    ref = torch.layer_norm(x, (D,), torch.from_numpy(g.astype(np.float64)), torch.from_numpy(b.astype(np.float64)), 1e-6).numpy()
    xd = x.numpy()
    mean = xd.mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(xd.var(axis=1, keepdims=True) + 1e-6)
    dm = 40 * U32 * np.abs(xd).mean(axis=1, keepdims=True)
    gd, bd = np.abs(g.astype(np.float64)), np.abs(b.astype(np.float64))
    core = np.abs(xd - mean) * rstd * gd
    bound = gd * rstd * (dm + U32 * np.abs(xd - mean)) + core * 48 * U32 + 4 * U32 * (core + bd) + U16 * np.abs(ref) + SUB16
    return ref, bound


@pytest.mark.parametrize("rows,D,skip_per,B", [
    (1001, 384, 0, 1), (13, 768, 0, 1), (7, 1024, 0, 1),
    (2 * 1369, 384, 1369, 2), (3 * 1369, 1024, 1369, 3), (2 * 2442, 768, 2442, 2), (3 * 2442, 1024, 2442, 3)])
def test_layernorm(rows, D, skip_per, B):
    rng = np.random.default_rng(rows + D)
    in_rows = rows // skip_per * (skip_per + 1) if skip_per else rows
    x = rng.standard_normal((in_rows, D), dtype=np.float32) * 2 + 0.3
    # rows whose mean is many times their standard deviation (mean 1000, std 0.5; mean -300, std 0.01)
    x[5::17] = 1000.0 + 0.5 * rng.standard_normal((len(x[5::17]), D), dtype=np.float32)
    x[11::23] = -300.0 + 0.01 * rng.standard_normal((len(x[11::23]), D), dtype=np.float32)
    if skip_per:  # cls rows: distinctive values, so a cls row normalised in place of a patch row fails grossly
        cls_rows = np.arange(B) * (skip_per + 1)
        x[cls_rows] = 5e3 * np.sin(np.arange(D, dtype=np.float32))[None] + 7e3
    g = (1 + 0.2 * rng.standard_normal(D)).astype(np.float32)
    b = (0.1 * rng.standard_normal(D)).astype(np.float32)
    y = np.empty((rows, D), np.float32)
    check(lib().prisma_debug_layernorm_skip(0, fptr(x), fptr(g), fptr(b), fptr(y), rows, D, skip_per))
    _check_written(y, np.ones(y.shape, bool), "layernorm")
    src = x.reshape(B, skip_per + 1, D)[:, 1:].reshape(rows, D) if skip_per else x
    ref, bound = _layernorm_ref(src, g, b)
    _check_bound(y, ref, bound, f"layernorm rows{rows} D{D} skip{skip_per}")


# ------------------------------------------------------------------------------------------------------------------ pos-embed
def _cubic_weights(t):
    """torch's upsample_bicubic2d tap weights (A = -0.75) at fractional offsets t, float64: [..., 4]."""
    A = -0.75
    c1 = lambda x: ((A + 2) * x - (A + 3)) * x * x + 1
    c2 = lambda x: ((A * x - 5 * A) * x + 8 * A) * x - 4 * A
    return np.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], axis=-1)


def _pos_taps(n_out, S):
    """Source taps of interpolate_pos_encoding along one axis: torch's float32 coordinate (float)(1/scale_factor) with
    scale_factor = (n + 0.1)/S, src = scale (dst + 0.5) - 0.5 in float32; clamped taps.  Also the spacing of src (one
    float32 ulp: the coordinate a fused multiply-add would produce instead)."""
    scale = np.float32(1.0 / ((n_out + 0.1) / S))
    src = scale * (np.arange(n_out, dtype=np.float32) + np.float32(0.5)) - np.float32(0.5)
    i0 = np.floor(src).astype(np.int64)
    t = (src - i0.astype(np.float32)).astype(np.float64)
    idx = np.clip(i0[:, None] - 1 + np.arange(4)[None], 0, S - 1)
    return idx, _cubic_weights(t), np.spacing(np.abs(src)).astype(np.float64)


def _pos_embed_ref(pos, cls, S, ph, pw):
    """float64 F.interpolate(bicubic, scale_factor=((ph+.1)/S, (pw+.1)/S)) of the S x S grid with float32 coordinates,
    row 0 = pos[0] + cls; bound per element:
      tap weights evaluated in fp32 (absolute <= 32 u each) and a 16-term fp32 sum (24 u sum |w_y w_x pos|);
      one float32 ulp of the source coordinate (fused or not) moves a weight by <= 1.5 ulp (|dw/dt| <= 1.35)."""
    D = pos.shape[1]
    grid = pos[1:].astype(np.float64).reshape(S, S, D)
    iy, wy, sy = _pos_taps(ph, S)
    ix, wx, sx = _pos_taps(pw, S)
    g_abs = np.abs(grid)
    tmp = np.einsum("xi,yxid->yxd", wx, grid[:, ix])               # [S][pw][D]
    ref = np.einsum("yj,yjxd->yxd", wy, tmp[iy])                  # [ph][pw][D]
    awx, awy = np.abs(wx), np.abs(wy)
    t_abs = np.einsum("xi,yxid->yxd", awx, g_abs[:, ix])
    s_w = np.einsum("yj,yjxd->yxd", awy, t_abs[iy])               # sum |w_y w_x pos|
    t_sum = g_abs[:, ix].sum(axis=2)                              # [S][pw][D]: sum_i |pos|
    s_all = t_sum[iy].sum(axis=1)                                 # sum over the 16 taps of |pos|
    s_wy = np.einsum("yj,yjxd->yxd", awy, t_sum[iy])              # sum |w_y| |pos|
    s_wx = t_abs[iy].sum(axis=1)                                  # sum |w_x| |pos|
    bound = 24 * U32 * s_w + 32 * U32 * (s_wy + s_wx) + 2 * U32 * s_all \
        + 1.5 * (sy[:, None, None] * s_wx + sx[None, :, None] * s_wy)
    row0 = pos[0].astype(np.float64) + cls.astype(np.float64)
    ref = np.concatenate([row0[None], ref.reshape(ph * pw, D)])
    bound = np.concatenate([U32 * np.abs(row0)[None], bound.reshape(ph * pw, D)])
    return ref, bound


def _pos_table(S=37, D=384, seed=0):
    rng = np.random.default_rng(seed)
    pos = (0.03 * rng.standard_normal((1 + S * S, D))).astype(np.float32)
    pos[1:] += (0.05 * np.sin(np.arange(S * S)[:, None] * 0.37 + np.arange(D)[None] * 0.11)).astype(np.float32)
    cls = (0.05 * rng.standard_normal(D)).astype(np.float32)
    return pos, cls


def _run_pos_embed(pos, cls, S, D, ph, pw):
    out = np.empty((1 + ph * pw, D), np.float32)
    check(lib().prisma_debug_pos_embed(0, fptr(pos), fptr(cls), S, D, ph, pw, fptr(out)))
    return out


def test_pos_embed_square_grid_is_the_table():
    """A 37 x 37 grid (every square or near-square depth_anything frame: 518 x 518 input) takes the table unchanged, as
    interpolate_pos_encoding does (vision_transformer.py:183-184): bit for bit, and row 0 = pos[0] + cls in fp32."""
    from oracle import da as oda
    S, D = 37, 384
    pos, cls = _pos_table(S, D)
    out = _run_pos_embed(pos, cls, S, D, S, S)
    _check_written(out, np.ones(out.shape, bool), "pos_embed 37x37")
    assert np.array_equal(out[1:].view(np.uint32), pos[1:].view(np.uint32))
    assert np.array_equal(out[0].view(np.uint32), (pos[0] + cls).view(np.uint32))
    ora = oda.interpolate_pos_encoding(torch.from_numpy(pos)[None], S, S)[0].numpy()
    assert np.array_equal(out[1:].view(np.uint32), ora[1:].view(np.uint32))


@pytest.mark.parametrize("ph,pw", [(37, 66), (37, 49), (28, 37), (66, 37), (2, 2), (74, 74)])
def test_pos_embed_resampled(ph, pw):
    from oracle import da as oda
    S, D = 37, 384
    pos, cls = _pos_table(S, D, seed=ph * 100 + pw)
    out = _run_pos_embed(pos, cls, S, D, ph, pw)
    _check_written(out, np.ones(out.shape, bool), f"pos_embed {ph}x{pw}")
    ref, bound = _pos_embed_ref(pos, cls, S, ph, pw)
    _check_bound(out, ref, bound, f"pos_embed {ph}x{pw}")
    assert np.array_equal(out[0].view(np.uint32), (pos[0] + cls).view(np.uint32))
    # the oracle's own fp32 interpolation (torch CPU; its row 0 is pos[0] alone), whose rounding obeys the same bound:
    # within twice of it
    ora = oda.interpolate_pos_encoding(torch.from_numpy(pos)[None], ph, pw)[0].numpy()
    _check_bound(out[1:], ora[1:].astype(np.float64), 2 * bound[1:], f"pos_embed {ph}x{pw} vs oracle fp32")


# ------------------------------------------------------------------------------------------------------------------ patchify
def _patchify_ref(x, patch):
    """im2col of the patch-embed conv: row b*P + py*pw + px, column c*p*p + ky*p + kx, fp16-rounded, zero padded."""
    B, _, h, w = x.shape
    ph, pw = h // patch, w // patch
    kpad = -(-3 * patch * patch // 64) * 64
    t = x[:, :, :ph * patch, :pw * patch].reshape(B, 3, ph, patch, pw, patch).transpose(0, 2, 4, 1, 3, 5)
    ref = np.zeros((B * ph * pw, kpad), np.float32)
    ref[:, :3 * patch * patch] = _f16(t.reshape(B * ph * pw, 3 * patch * patch))
    return ref


@pytest.mark.parametrize("patch,h,w", [(14, 14 * 5 + 9, 14 * 7 + 3), (16, 16 * 6, 16 * 4 + 15)])
def test_patchify_bit_exact(patch, h, w):
    rng = np.random.default_rng(patch)
    B = 2
    x = (rng.standard_normal((B, 3, h, w), dtype=np.float32) * 2).astype(np.float32)
    ref = _patchify_ref(x, patch)
    out = np.empty(ref.shape, np.float32)
    check(lib().prisma_debug_patchify(0, fptr(x), B, h, w, patch, fptr(out)))
    _check_written(out, np.ones(out.shape, bool), "patchify")
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    assert np.all(out[:, 3 * patch * patch:].view(np.uint32) == 0)  # the pad columns are +0.0


# ------------------------------------------------------------------------------------------------------------------ readout
@pytest.mark.parametrize("B,T,D", [(1, 577, 768), (3, 577, 1024), (3, 5, 768), (1, 2, 1024)])
def test_readout_concat_bit_exact(B, T, D):
    rng = np.random.default_rng(B * T + D)
    x = (rng.standard_normal((B * T, D), dtype=np.float32) * 3).astype(np.float32)
    xb = x.reshape(B, T, D)
    ref = np.concatenate([xb[:, 1:], np.broadcast_to(xb[:, :1], (B, T - 1, D))], axis=2).reshape(B * (T - 1), 2 * D)
    ref = _f16(ref)
    out = np.empty(ref.shape, np.float32)
    check(lib().prisma_debug_readout_concat(0, fptr(x), B, T, D, fptr(out)))
    _check_written(out, np.ones(out.shape, bool), "readout_concat")
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------ upsample_ac
def _ac_linear_taps(n_in, n_out):
    """torch's align_corners=True bilinear source taps in float32: scale = (in-1)/(out-1), src = scale * dst,
    i0 = (int)src, i1 = i0 + (i0 < in-1), l1 = src - i0, l0 = 1 - l1."""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    src = np.float32(scale) * np.arange(n_out, dtype=np.float32)
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    return i0, i1, l0.astype(np.float64), l1.astype(np.float64)


def _upsample_ac_ref(x16, oh, ow):
    """float64 bilinear (align_corners=True) of fp16 NHWC maps with float32 coordinates; bound: fp16 rounding of the output
    (2^-11 |ref| + 2^-25) plus the kernel's 6 fp32 roundings of the 4-tap sum (6 u sum w |x|)."""
    B, ih, iw, Cc = x16.shape
    y0, y1, ly0, ly1 = _ac_linear_taps(ih, oh)
    x0, x1, lx0, lx1 = _ac_linear_taps(iw, ow)
    fy0, fy1 = ly0[:, None, None], ly1[:, None, None]
    fx0, fx1 = lx0[None, :, None], lx1[None, :, None]
    ref = np.empty((B, oh, ow, Cc))
    bound = np.empty((B, oh, ow, Cc))
    for b in range(B):  # one image at a time keeps the float64 temporaries small
        x = x16[b].astype(np.float64)
        r0, r1 = x[y0], x[y1]
        ref[b] = fy0 * (fx0 * r0[:, x0] + fx1 * r0[:, x1]) + fy1 * (fx0 * r1[:, x0] + fx1 * r1[:, x1])
        a0, a1 = np.abs(r0), np.abs(r1)
        mag = fy0 * (fx0 * a0[:, x0] + fx1 * a0[:, x1]) + fy1 * (fx0 * a1[:, x0] + fx1 * a1[:, x1])
        bound[b] = U16 * np.abs(ref[b]) + SUB16 + 6 * U32 * mag
    return ref, bound


@pytest.mark.parametrize("ih,iw,C,oh,ow,relu_copy", [
    (19, 33, 256, 37, 66, 1),      # refinenet4 -> level 3 of a 720p ViT-L frame
    (37, 66, 128, 74, 132, 0),     # x2 fusion step
    (74, 132, 64, 148, 264, 1),    # x2 fusion step
    (148, 264, 64, 296, 528, 1),   # refinenet1 x2
    (296, 528, 64, 518, 924, 1),   # final resize to the 518 x 924 network input (720p)
    (1, 7, 64, 5, 13, 1),          # a single input row
])
def test_upsample_ac(ih, iw, C, oh, ow, relu_copy):
    rng = np.random.default_rng(ih * iw + C)
    B = 2
    x = _f16(rng.standard_normal((B, ih, iw, C), dtype=np.float32) * 2)
    out = np.empty((B, oh + 2, ow + 2, C), np.float32)
    out_relu = np.empty_like(out)
    check(lib().prisma_debug_upsample_ac(0, fptr(x), B, ih, iw, C, oh, ow, relu_copy, fptr(out), fptr(out_relu)))
    interior = np.zeros(out.shape, bool)
    interior[:, 1:-1, 1:-1] = True
    _check_written(out, interior, "upsample_ac")  # the one-pixel border still holds the fill
    ref, bound = _upsample_ac_ref(x, oh, ow)
    _check_bound(out[:, 1:-1, 1:-1], ref, bound, f"upsample_ac {ih}x{iw}->{oh}x{ow} C{C}")
    if relu_copy:
        _check_written(out_relu, interior, "upsample_ac relu")
        inner = out[:, 1:-1, 1:-1]
        expect = np.where(inner > 0, inner, np.float32(0))
        assert np.array_equal(out_relu[:, 1:-1, 1:-1].view(np.uint32), expect.view(np.uint32))
    else:
        assert np.isnan(out_relu).all()


# ------------------------------------------------------------------------------------------------------------------ bicubic
def _ac_cubic_taps(n_in, n_out):
    """align_corners=True bicubic source taps in float32: scale = (in-1)/(out-1), src = scale * dst, clamped taps."""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    src = np.float32(scale) * np.arange(n_out, dtype=np.float32)
    i0 = np.floor(src).astype(np.int64)
    t = (src - i0.astype(np.float32)).astype(np.float64)
    return np.clip(i0[:, None] - 1 + np.arange(4)[None], 0, n_in - 1), _cubic_weights(t)


def _upsample_bicubic_ref(x, oh, ow):
    """float64 bicubic (align_corners=True, A = -0.75) with float32 coordinates; bound: tap weights evaluated in fp32
    (absolute <= 32 u each) and two 4-tap fp32 sums, rows then columns (16 u sum |w_y w_x x|)."""
    iy, wy = _ac_cubic_taps(x.shape[0], oh)
    ix, wx = _ac_cubic_taps(x.shape[1], ow)
    xd = x.astype(np.float64)
    tmp = np.einsum("xi,yxi->yx", wx, xd[:, ix])        # [ih][ow]
    ref = np.einsum("yj,yjx->yx", wy, tmp[iy])           # [oh][ow]
    ax = np.abs(xd)
    t_w = np.einsum("xi,yxi->yx", np.abs(wx), ax[:, ix])
    t_1 = ax[:, ix].sum(axis=2)
    s_w = np.einsum("yj,yjx->yx", np.abs(wy), t_w[iy])
    s_wy = np.einsum("yj,yjx->yx", np.abs(wy), t_1[iy])
    s_wx = t_w[iy].sum(axis=1)
    return ref, 16 * U32 * s_w + 32 * U32 * (s_wy + s_wx)


@pytest.mark.parametrize("ih,iw,oh,ow", [(224, 384, 720, 1280), (224, 384, 1080, 1920), (384, 384, 480, 480),
                                         (288, 384, 240, 320)])
def test_upsample_bicubic(ih, iw, oh, ow):
    rng = np.random.default_rng(ih + iw + oh)
    yy, xx = np.mgrid[0:ih, 0:iw]
    x = (3 + np.sin(yy * 0.05) * np.cos(xx * 0.031) + 0.3 * rng.standard_normal((ih, iw))).astype(np.float32)
    out = np.empty((oh, ow), np.float32)
    check(lib().prisma_debug_upsample_bicubic(0, fptr(x), ih, iw, fptr(out), oh, ow))
    _check_written(out, np.ones(out.shape, bool), "upsample_bicubic")
    ref, bound = _upsample_bicubic_ref(x, oh, ow)
    _check_bound(out, ref, bound, f"bicubic {ih}x{iw}->{oh}x{ow}")
    tv = F.interpolate(torch.from_numpy(x)[None, None], (oh, ow), mode="bicubic", align_corners=True)[0, 0].numpy()
    _check_bound(out, tv.astype(np.float64), 2 * bound, f"bicubic {ih}x{iw}->{oh}x{ow} vs torch fp32")


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_square_frame_tokens_and_depth():
    """ViT-S on a 540 x 540 frame (518 x 518 input, the 37 x 37 grid): the patch-embed tokens against the oracle's
    vit_tokens in float64 from the engine's own net input with fp16 operands, and the prediction against the oracle at the
    band's 1e-3 tolerance.  Token bound: the fp16 x fp16 products are exact; the fp32 MMA sum runs 10 k-blocks of 64
    (depth <= 48 additions, each within 2^-23 of its result): 48 * 2^-23 * sum |x||w|, plus the bias and pos-embed adds
    (2^-23 |t|).  A resampled position table (5e-3 of the tokens' range) exceeds it many times over."""
    from oracle import da as oda
    from prisma_b200.depth import DepthAnythingEngine
    from prisma_b200.seeded_weights import make_da_weights
    from prisma_b200.synthetic import synthetic_frame
    sd = make_da_weights("vits", 0)
    img = synthetic_frame(540, 540, 2)
    eng = DepthAnythingEngine("vits", sd)
    pred = eng.infer(img)
    wn, hn = oda.da_get_size(540, 540)
    assert (wn, hn) == (518, 518)
    T, D = 1 + 37 * 37, 384
    net = eng.read_tap("net_input", (3, hn, wn))
    tok = eng.read_tap("tokens", (T, D))
    eng.close()
    sd64 = {k: v.double() for k, v in sd.items()}
    x = torch.from_numpy(net.astype(np.float64))[None]
    with torch.no_grad():
        ref = oda.vit_tokens(sd64, x, q=lambda t: t.half().double())[0].numpy()
        q = lambda t: t.half().double()
        mag = F.conv2d(q(x).abs(), q(sd64["pretrained.patch_embed.proj.weight"]).abs(), stride=14)
        mag = mag.flatten(2).transpose(1, 2)[0].numpy()
    bound = np.empty((T, D))
    bound[0] = U32 * np.abs(ref[0])
    bound[1:] = 48 * 2 * U32 * mag + 2 * 2 * U32 * np.abs(ref[1:])
    _check_bound(tok, ref, bound, "square-frame tokens")
    ref_pred = oda.da_infer(sd, img, "vits")
    m = float(np.abs(pred - ref_pred).max() / np.abs(ref_pred).max())
    l2 = float(np.linalg.norm(pred - ref_pred) / np.linalg.norm(ref_pred))
    print(f"square-frame depth: max-rel {m:.3e}, rel-L2 {l2:.3e}")
    assert m <= 1e-3 and l2 <= 1e-3
