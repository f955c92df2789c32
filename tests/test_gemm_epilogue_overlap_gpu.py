"""The fused epilogue of the shifted-row GEMM across many tiles per CTA.

The fp16 register-epilogue kernels (BN 32 / 64 / 128) hand every tile's accumulators to an epilogue warpgroup through one
shared-memory buffer guarded by two mbarriers, while the consumers run the next tile's MMAs; BN 256 keeps the consumer-run
epilogue.  test_gemm_epilogue_gpu.py covers each feature at M <= 2000, where a CTA sees at most one tile.  Here every case has
enough rows that each of the 132 CTAs runs at least 3 tiles, plus a ragged last tile, so the hand-off is reused with both
barrier parities; a K = 64 ConvGRU case makes the consumers finish a tile's MMAs long before the epilogue has read the
previous one.  The float64 epilogue model, the NaN-poisoned destinations and the row mapper are those of
test_gemm_epilogue_gpu.py.
"""
import numpy as np
import pytest
import torch

from test_gemm_epilogue_gpu import (ROW_LINEAR, ROW_PADDED, ROW_PAD2TOK, U, Geometry, _ru, assert_cells, check_f16,
                                    conv_offsets, dev, epilogue_ref, exact_rows, exact_w, expected_buffer, fp16_values,
                                    make_ep, map_cells, nan16, nan32, ref_acc, run_ok, upload_a16, upload_w16)

SMS = 132  # H100 SXM


def _tiles_per_cta(M, N, bn):
    return (-(-M // 128) * -(-N // bn)) / SMS


@pytest.mark.gpu
@pytest.mark.parametrize("act,M,N,K,bn", [
    (0, 51_203, 100, 64, 32),     # the accumulator itself, bit-exact
    (1, 26_011, 136, 128, 64),    # exact-erf GELU
    (2, 50_777, 120, 64, 128),
    (3, 50_801, 96, 64, 32),      # fast sigmoid
    (4, 25_777, 128, 72, 64),     # fast tanh
    (5, 51_001, 64, 100, 128),    # softplus
    (6, 40_403, 264, 64, 256),    # sigmoid with expf + IEEE division; 256-wide tiles (consumer-run epilogue)
])
def test_activations_many_tiles(act, M, N, K, bn):
    """alpha acc + bias -> activation -> fp32 and fp16 destinations of a pitch wider than N, past the last row NaN."""
    assert _tiles_per_cta(M, N, bn) >= 3 and M % 128 != 0
    rng = np.random.default_rng(1000 + act)
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = None if act == 0 else rng.uniform(-8, 8, N).astype(np.float32).astype(np.float64)
    alpha = 1.0 if act == 0 else 0.75
    out32, out16 = nan32(M + 40, N + 12), nan16(M + 40, N + 20)
    ep = make_ep(alpha=alpha, act=act, bias=None if bias is None else dev(bias), out_f32=out32, out_f32_ld=N + 12,
                 out_f16=out16, out_f16_ld=N + 20)
    run_ok(upload_a16(A, _ru(K, 8) + 8), upload_w16(w), K, M, N, [0], ep, bn=bn)
    rows, cols = map_cells(M, N, {})
    r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(alpha=alpha, bias=bias, act=act))
    exp, tol = expected_buffer(out32.shape, rows, cols, r["v"], r["e"])
    if act == 0:
        assert np.all(tol[~np.isnan(tol)] == 0)
    assert_cells(out32, exp, tol, "out_f32")
    check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "out_f16")


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_residuals_relu_copy_shared_border_conv(bn):
    """3x3 ROW_PADDED conv over a shared-border map (random operands) + bias + res_a + res_b, stored as fp16 x and relu(x)
    copies of the same geometry; the borders, the alignment rows and the extra image stay NaN."""
    rng = np.random.default_rng(2000 + bn)
    g = Geometry(5, 60, 201, 1, shared=True, align32=True)
    Cin, N = 64, 64 if bn <= 64 else 136
    assert _tiles_per_cta(g.rows, N, bn) >= 3 and g.rows % 128 != 0
    A = g.embed(fp16_values(rng.standard_normal((g.B, g.H, g.W, Cin))))
    w = fp16_values(rng.standard_normal((N, 9, Cin)) / 24.0)
    offs = conv_offsets(3, 3, g.Wp)
    acc, mag = ref_acc(A, w, offs, g.rows)
    eacc = U * 9 * Cin * mag
    bias = rng.standard_normal(N).astype(np.float32).astype(np.float64)
    res_a = fp16_values(rng.standard_normal((g.rows, N)))
    res_b = fp16_values(rng.standard_normal((g.rows, N)))
    rows_total = g.rows + g.img_rows
    o16, o16r = nan16(rows_total, N + 8), nan16(rows_total, N + 8)
    ep = make_ep(bias=dev(bias), res_a=dev(res_a, torch.float16), res_a_ld=N, res_b=dev(res_b, torch.float16), res_b_ld=N,
                 out_f16=o16, out_f16_ld=N + 8, out_f16_relu=o16r, out_f16_relu_ld=N + 8, row_map=ROW_PADDED, **g.src_geom())
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, g.rows, N, offs, ep, bn=bn)
    rows, cols = map_cells(g.rows, N, dict(row_map=ROW_PADDED, **g.src_geom()))
    r = epilogue_ref(acc, eacc, rows, cols, dict(bias=bias, res_a=res_a, res_b=res_b))
    check_f16(o16, o16.shape, rows, cols, r["v"], r["e"], "out_f16")
    check_f16(o16r, o16r.shape, rows, cols, np.maximum(r["v"], 0), r["e"], "out_f16_relu")


@pytest.mark.gpu
@pytest.mark.parametrize("gru,bn,Cin,kh,kw", [
    (1, 128, 96, 1, 5),
    (1, 256, 96, 1, 5),
    (2, 64, 96, 5, 1),
    (2, 128, 96, 5, 1),
    (1, 128, 64, 1, 1),   # K = 64: one K block per tile, the consumers wait on the hand-off
    (2, 128, 64, 1, 1),
])
def test_convgru_many_tiles(gru, bn, Cin, kh, kw):
    """The ConvGRU gate epilogues in the RaftEngine::add_conv layout (shared border 2): gru 1 writes z (columns < 128) and
    r * h; gru 2 writes h' = (1 - z) h + z q in place of h and its fp16 operand copy."""
    rng = np.random.default_rng(3000 + gru * 100 + bn + Cin + kh)
    src = Geometry(3, 100, 189, 2, shared=True, align32=True)
    N = 256 if gru == 1 else 128
    M = src.rows
    assert _tiles_per_cta(M, N, bn) >= 3 and M % 128 != 0
    A = src.embed(exact_rows(rng, src.B * src.H * src.W, Cin).reshape(src.B, src.H, src.W, Cin))
    w = exact_w(rng, N, kh * kw, Cin, wmax=8)
    offs = conv_offsets(kh, kw, src.Wp)
    acc, _ = ref_acc(A, w, offs, M)
    bias = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    geom = dict(row_map=ROW_PADDED, **src.src_geom())
    rows, cols = map_cells(M, N, geom)
    h0 = rng.uniform(-1, 1, (M, 128)).astype(np.float32).astype(np.float64)
    A_dev, W_dev = upload_a16(A, _ru(Cin, 8) + 8), upload_w16(w)
    if gru == 1:
        out, rh = nan32(M + 64, 264), nan16(M + 64, 136)
        ep = make_ep(bias=dev(bias), act=3, out_f32=out, out_f32_ld=264, gru=1, gru_h=dev(h0), gru_rh=rh, gru_rh_ld=136, **geom)
        run_ok(A_dev, W_dev, Cin, M, N, offs, ep, bn=bn)
        r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=3, gru=1, gru_h=h0))
        zc = r["z_cols"]
        exp, tol = expected_buffer(out.shape, rows[:, zc], cols[:, zc], r["v"][:, zc], r["e"][:, zc])
        assert_cells(out, exp, tol, "z (out_f32)")
        check_f16(rh, rh.shape, rows[:, ~zc], cols[:, ~zc] - 128, r["rh"][:, ~zc], r["erh"][:, ~zc], "r * h (gru_rh)")
    else:
        z = np.full((M, 256), np.nan)
        z[:, :128] = rng.uniform(0, 1, (M, 128)).astype(np.float32)
        h = dev(h0)
        out16 = nan16(M + 64, 136)
        ep = make_ep(bias=dev(bias), act=4, out_f32=h, out_f32_ld=128, out_f16=out16, out_f16_ld=136, gru=2, gru_h=h,
                     gru_z=dev(z), **geom)
        run_ok(A_dev, W_dev, Cin, M, N, offs, ep, bn=bn)
        r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=4, gru=2, gru_h=h0, gru_z=z))
        stored = rows >= 0
        assert_cells(h, np.where(stored, r["v"], h0), np.where(stored, r["e"], 0.0), "h' (out_f32, in place)")
        check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "h' (out_f16)")


@pytest.mark.gpu
@pytest.mark.parametrize("N,bn", [(64, 32), (96, 128), (128, 256)])
def test_instnorm_statistics_many_tiles(N, bn):
    """stat_part of a stride-1 ROW_PAD2TOK conv over a shared-border map: every 32-row slab of every tile writes the sum and
    sum of squares of its valid stored values; slabs without a valid row hold exact zeros."""
    rng = np.random.default_rng(4000 + N + bn)
    src = Geometry(3, 90, 191, 1, shared=True, align32=True)
    Cin = 64
    M = src.rows
    assert _tiles_per_cta(M, N, bn) >= 3 and M % 128 != 0
    A = src.embed(fp16_values(rng.standard_normal((src.B, src.H, src.W, Cin))))
    w = fp16_values(rng.standard_normal((N, 1, Cin)) / 8.0)
    acc, mag = ref_acc(A, w, [0], M)
    eacc = U * Cin * mag
    bias = rng.standard_normal(N).astype(np.float32).astype(np.float64)
    nslab = _ru(M, 128) // 32
    dense = nan32(src.B * src.H * src.W + 20, N)
    stats = nan32((nslab + 6) * 2, N)
    geom = dict(row_map=ROW_PAD2TOK, **src.src_geom(1))
    ep = make_ep(bias=dev(bias), out_f32=dense, out_f32_ld=N, stat_part=stats, **geom)
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, M, N, [0], ep, bn=bn)
    rows, cols = map_cells(M, N, geom)
    r = epilogue_ref(acc, eacc, rows, cols, dict(bias=bias))
    exp, tol = expected_buffer(dense.shape, rows, cols, r["v"], r["e"])
    assert_cells(dense, exp, tol, "dense out_f32")
    ok = np.zeros((nslab * 32, N), bool)
    ok[:M] = rows >= 0
    v, e = np.zeros((nslab * 32, N)), np.zeros((nslab * 32, N))
    v[:M], e[:M] = np.where(rows >= 0, r["v"], 0), np.where(rows >= 0, r["e"], 0)
    v, e = v.reshape(nslab, 32, N), e.reshape(nslab, 32, N)
    exp = np.full((nslab + 6, 2, N), np.nan)
    tol = np.full((nslab + 6, 2, N), np.nan)
    exp[:nslab, 0], exp[:nslab, 1] = v.sum(1), (v * v).sum(1)
    tol[:nslab, 0] = e.sum(1) + 32 * U * np.abs(v).sum(1)
    tol[:nslab, 1] = (2 * np.abs(v) * e + e * e).sum(1) + 34 * U * (v * v).sum(1)
    empty = ~ok.reshape(nslab, 32, N).any(1)
    assert empty.any() and (~empty).any()
    tol[:nslab][np.repeat(empty[:, None, :], 2, 1)] = 0.0
    assert_cells(stats, exp.reshape(-1, N), tol.reshape(-1, N), "stat_part")


@pytest.mark.gpu
@pytest.mark.parametrize("bn,copy", [(32, True), (64, False)])
def test_dpt_head_many_tiles(bn, copy):
    """The fused DPT output head (N == 32) over a symmetric-border map of many tiles: depth written dense, optionally with the
    32 ReLU'd activations."""
    rng = np.random.default_rng(5000 + bn)
    g = Geometry(2, 150, 191, 1)
    Cin, N = 64, 32
    assert _tiles_per_cta(g.rows, N, bn) >= 3 and g.rows % 128 != 0
    A = g.embed(exact_rows(rng, g.B * g.H * g.W, Cin).reshape(g.B, g.H, g.W, Cin))
    w = exact_w(rng, N, 9, Cin, wmax=8)
    offs = conv_offsets(3, 3, g.Wp)
    acc, _ = ref_acc(A, w, offs, g.rows)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    hw = rng.uniform(-1, 1, N).astype(np.float32).astype(np.float64)
    hb = float(np.float32(0.375))
    npix = g.B * g.H * g.W
    head = nan32(npix + 50, 1)
    act32 = nan16(npix + 50, 40) if copy else None
    ep = make_ep(bias=dev(bias), act=2, head_w=dev(hw), head_b=hb, head_out=head, out_f16=act32, out_f16_ld=40 if copy else 0,
                 row_map=ROW_PADDED, **g.src_geom())
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, g.rows, N, offs, ep, bn=bn)
    pix_rows = g.pixel_rows().ravel()
    hv = np.maximum(acc[pix_rows] + bias, 0.0)
    ehv = U * np.abs(acc[pix_rows] + bias)
    depth = hb + hv @ hw
    edepth = ehv @ np.abs(hw) + 34 * U * (abs(hb) + np.abs(hv) @ np.abs(hw))
    pix = np.arange(npix)
    exp, tol = expected_buffer(head.shape, pix, np.zeros_like(pix), np.maximum(depth, 0), edepth)
    assert_cells(head, exp, tol, "head_out")
    if copy:
        prow, pcol = np.repeat(pix[:, None], N, 1), np.broadcast_to(np.arange(N), (npix, N))
        check_f16(act32, act32.shape, prow, pcol, hv, ehv, "head out_f16")


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [64, 128])
def test_device_row_count_many_tiles(bn):
    """m_dev: only the first round_up(*m_dev, 128) rows are computed and stored, whether that leaves several tiles per CTA,
    fewer tiles than CTAs, or none."""
    rng = np.random.default_rng(6000 + bn)
    M, N, K = 60_000, 128, 64
    assert _tiles_per_cta(M, N, bn) >= 3
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    A_dev, W_dev = upload_a16(A, K), upload_w16(w)
    rows_all, cols = map_cells(M, N, {})
    r = epilogue_ref(acc, np.zeros_like(acc), rows_all, cols, dict(bias=bias, act=3))
    for m in (0, 5_000, 51_111, M):
        m_dev = torch.tensor([m], dtype=torch.int32, device="cuda")
        shape = (M + 20, N + 12)
        out = nan16(*shape)
        ep = make_ep(bias=dev(bias), act=3, m_dev=m_dev, out_f16=out, out_f16_ld=N + 12, row_map=ROW_LINEAR)
        run_ok(A_dev, W_dev, K, M, N, [0], ep, bn=bn)
        rows = np.where(rows_all < min(M, _ru(m, 128)), rows_all, -1)
        check_f16(out, shape, rows, cols, r["v"], r["e"], f"m_dev={m}")
